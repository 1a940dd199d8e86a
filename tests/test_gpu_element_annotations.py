"""Element sets that keep annotations on the GPU (m3tsz_element_set_*_annotated, DESIGN.md §4.12), in both int_optimized
modes, Gauge and Counter, with and without transformations (Reset included): the reference's annotation goldens
through the device calls; random sequences over several add calls with consumes between them, equal to the CPU model
(tests/element_set_ann_model.py) in bytes, results, statuses, records and watermarks; byte identity with
aggregate_tiles_types(annotations=True) where the two rules agree; the capacity stops with grow and resend; the
argument checks; 100 k elements sampled against the model; and sets whose datapoints carry no annotation writing the
plain calls' bytes."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

import agg_oracle_lib as A
from element_set_ann_model import AnnotatedElementModel, annotated_points, sparse_annotations
from m3_b200 import capi
from test_element_set_model import _bits, random_series

pytestmark = pytest.mark.gpu

SEC = 1_000_000_000
RES = 60 * SEC
START = 1_600_000_020 * SEC  # a whole minute
DEV = "cuda"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "m3tsz_tile_annotation_goldens.json")
# annotation.Payload{OpenMetricsFamilyType: COUNTER, OpenMetricsHandleValueResets: true}, and a few others
PAYLOADS = [bytes([0x08, 0x01, 0x10, 0x01]), b"gauge", bytes(range(1, 40)), b"x" * 120]


@pytest.fixture(scope="module")
def codecs():
    from m3_b200.codec import BatchCodec
    return {True: BatchCodec(0, int_optimized=True), False: BatchCodec(0, int_optimized=False)}


def _point_major(cols, P=None):
    """per-element lists [(t, value bits, annotation)] -> (ts [P, N], values [P, N], n_points [N], annotations) on the
    device"""
    N = len(cols)
    P = max([len(c) for c in cols] + [1]) if P is None else P
    ts = np.zeros((P, N), dtype=np.int64)
    vb = np.zeros((P, N), dtype=np.uint64)
    for s, c in enumerate(cols):
        for i, (t, v, _) in enumerate(c):
            ts[i, s], vb[i, s] = t, v
    n = np.array([len(c) for c in cols], dtype=np.int32)
    ann = tuple(torch.from_numpy(a).to(DEV) for a in sparse_annotations(cols))
    return (torch.from_numpy(ts).to(DEV), torch.from_numpy(vb.view(np.float64)).to(DEV), torch.from_numpy(n).to(DEV),
            ann)


def _add(es, cols):
    ts, vals, n, ann = _point_major(cols)
    res, st = es.add(ts, vals, n, annotations=ann)
    res = res.cpu().numpy()
    return [res[: len(c), s].tolist() for s, c in enumerate(cols)], st.cpu().numpy().tolist()


def _rows(es):
    snap = es.stream()
    out, ln = snap.out.cpu().numpy(), snap.out_len.cpu().numpy()
    return [out[r, : ln[r]].tobytes() for r in range(len(ln))]


def _new(codec, N, metric, types, ops=(), discard=False, R=4, capacity=128, stride=None):
    return codec.element_set(torch.full((N,), START, dtype=torch.int64, device=DEV), metric, types, RES,
                             transforms=ops, discard_nan=discard, open_windows=R, stride=stride,
                             annotation_capacity=capacity)


def _models(N, metric, types, ops=(), discard=False, R=4, capacity=128, int_opt=True):
    return [AnnotatedElementModel(metric, types, RES, ops, discard, open_windows=R, capacity=capacity, start_ns=START,
                                  int_optimized=int_opt) for _ in range(N)]


def _check_against(es, models):
    rows = _rows(es)
    N, k = es.n_elements, len(es.agg_types)
    for s, m in enumerate(models):
        want = m.streams()
        for j in range(k):
            assert rows[j * N + s] == want[j], (s, j)
    elem, wm = es.elem.cpu().numpy(), es.watermark.cpu().numpy()
    for s, m in enumerate(models):
        assert elem[s].tobytes() == m.state.tobytes(), s
        assert int(wm[s]) == m.watermark, s


def _golden_types(metric):
    return [A.AGG_LAST, A.AGG_SUM] if metric == A.METRIC_GAUGE else [A.AGG_SUM]


@pytest.mark.parametrize("int_opt", [True, False])
def test_goldens_through_the_device_calls(codecs, int_opt):
    """each golden datapoint as its own add call; the open window's slot holds the golden's annotation, and the
    flushed rows equal the model's (every datapoint of the window written with it)"""
    with open(GOLDEN) as f:
        cases = json.load(f)["cases"]
    codec = codecs[int_opt]
    for case in cases:
        assert case["step_ns"] == 10 * SEC
        metric, types = case["metric_type"], _golden_types(case["metric_type"])
        es = codec.element_set(torch.full((1,), case["start_ns"], dtype=torch.int64, device=DEV), metric, types,
                               case["step_ns"], open_windows=case["n_windows"], annotation_capacity=64)
        m = AnnotatedElementModel(metric, types, case["step_ns"], open_windows=case["n_windows"], capacity=64,
                                  start_ns=case["start_ns"], int_optimized=int_opt)
        for t, v, a in case["datapoints"]:
            dp = [[(int(t), _bits(v), bytes.fromhex(a))]]
            assert _add(es, dp) == ([[0]], [0])
            assert m.add(dp[0]) == ([0], 0)
        ln, by = es.ann_len.cpu().numpy(), es.ann_bytes.cpu().numpy()
        start, cnt = es.win["start"].cpu().numpy(), es.win["count"].cpu().numpy()
        for w, want in enumerate(case["want_windows"]):
            ws = case["start_ns"] + w * case["step_ns"]
            r = [r for r in range(es.open_windows) if cnt[r, 0] and start[r, 0] == ws]
            assert len(r) == 1, (case["name"], w)
            assert by[r[0], 0, : ln[r[0], 0]].tobytes() == bytes.fromhex(want), (case["name"], w)
        end = case["start_ns"] + case["n_windows"] * case["step_ns"]
        assert es.consume(end).tolist() == [0]
        m.consume(end)
        _check_against(es, [m])


CASES = [
    (A.METRIC_GAUGE, [1, 2, 3], []),
    (A.METRIC_GAUGE, [1, 4, 9], [4, 3, 5]),
    (A.METRIC_GAUGE, [4, 7], [5]),
    (A.METRIC_COUNTER, [7], []),
    (A.METRIC_COUNTER, [2, 7, 8], [3]),
    (A.METRIC_COUNTER, [7, 9], [4, 5]),
]


def _random_cols(rng, N, metric, clock):
    """up to five datapoints per element around the clock: late ones to older (open or closed) windows, NaN values,
    about half with an annotation"""
    cols = []
    for _ in range(N):
        pts = []
        for _ in range(int(rng.integers(0, 6))):
            t = clock + int(rng.integers(-3 * RES, RES)) // SEC * SEC
            if metric == A.METRIC_COUNTER:
                v = float(rng.choice([rng.integers(-1000, 1000), np.nan]))
            else:
                v = float(rng.choice([rng.normal() * 100, np.nan, np.inf]))
            pts.append((max(t, START), _bits(v)))
        cols.append(annotated_points(pts, rng, PAYLOADS))
    return cols


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("n_calls", [1, 2, 5, 17])
def test_random_sequences_equal_the_model(codecs, int_opt, case, n_calls):
    metric, types, ops = CASES[case]
    codec = codecs[int_opt]
    rng = np.random.default_rng(1000 * case + 10 * n_calls + int_opt)
    N, R, discard = 64, 3, bool(case % 2)
    es = _new(codec, N, metric, types, ops, discard, R=R, capacity=128, stride=16384)
    models = _models(N, metric, types, ops, discard, R=R, capacity=128, int_opt=int_opt)
    clock = START + 2 * RES
    for call in range(n_calls):
        cols = _random_cols(rng, N, metric, clock)
        got_r, got_s = _add(es, cols)
        for s, m in enumerate(models):
            assert (got_r[s], got_s[s]) == m.add(cols[s]), (call, s)
        clock += int(rng.integers(0, 3)) * RES // 2
        if call + 1 < n_calls and rng.random() < 0.6:
            target = clock - int(rng.integers(0, 2)) * RES
            assert es.consume(target).tolist() == [0] * N
            for m in models:
                m.consume(target)
    assert es.consume(clock + 4 * RES).tolist() == [0] * N
    for m in models:
        m.consume(clock + 4 * RES)
    _check_against(es, models)


def _tiles_annotated(codec, cols, metric, types, ops, n_windows):
    """aggregate_tiles_types(annotations=True) over annotated streams of the same datapoints -> bytes per row"""
    N = len(cols)
    P = max([len(c) for c in cols] + [1])
    ts = np.zeros((N, P), dtype=np.int64)
    vb = np.zeros((N, P), dtype=np.uint64)
    for s, c in enumerate(cols):
        for i, (t, v, _) in enumerate(c):
            ts[s, i], vb[s, i] = t, v
    n = torch.tensor([len(c) for c in cols], dtype=torch.int32, device=DEV)
    start = torch.full((N,), START, dtype=torch.int64, device=DEV)
    ann = tuple(torch.from_numpy(a).to(DEV) for a in sparse_annotations(cols))
    enc = codec.encode(torch.from_numpy(ts).to(DEV), torch.from_numpy(vb.view(np.float64)).to(DEV), start,
                       n_points=n, annotations=ann)
    assert int(enc.status.abs().sum()) == 0
    offs = torch.arange(N, dtype=torch.int64, device=DEV) * enc.out.shape[1]
    out, _ = codec.aggregate_tiles_types(enc.out.view(-1), offs, START, RES, n_windows, types, metric_type=metric,
                                         lengths=enc.out_len, transforms=ops, discard_nan=False,
                                         state=codec.element_state(N), annotations=True)
    assert int(out.status.abs().sum()) == 0
    packed = out.packed.cpu().numpy()
    o, ln = out.offsets.reshape(-1).cpu().numpy(), out.out_len.reshape(-1).cpu().numpy()
    return [packed[o[r]: o[r] + ln[r]].tobytes() for r in range(len(ln))]


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("n_calls", [1, 2, 5, 17])
def test_equals_aggregate_tiles_annotated_in_order(codecs, int_opt, case, n_calls):
    """Where the two rules agree, the bytes do.  The tile path takes a window's annotation from the source stream,
    which writes an annotation only where it differs from the last one written: its window keeps the last one WRITTEN
    there.  The element keeps the last non-empty one it was given.  With the datapoints in window order, let L(w) be
    the last non-empty annotation given up to window w.  Both outputs have written L(w) last after window w (an
    element window's non-empty annotation is L(w); a tile window has one only when the source wrote in it, and then
    it is L(w); without one L(w) = L(w - 1)), and both write at w exactly when L(w) != L(w - 1), which needs an
    annotation in w that differs from L(w - 1).  That holds only while every window writes its datapoints: a window
    that the NaN discard drops writes nothing, so no discard here."""
    metric, types, ops = CASES[case]
    codec = codecs[int_opt]
    rng = np.random.default_rng(500 + 10 * case + n_calls + int_opt)
    N, W = 70, 8
    cols = [annotated_points(random_series(rng, START, RES, W, metric), rng, PAYLOADS[:2], 0.4) for _ in range(N)]
    es = _new(codec, N, metric, types, ops, False, R=W, capacity=64)
    cuts = [np.sort(rng.integers(0, len(c) + 1, n_calls - 1)).tolist() for c in cols]
    for call in range(n_calls):
        parts = [c[([0] + cuts[s] + [len(c)])[call]: ([0] + cuts[s] + [len(c)])[call + 1]] for s, c in enumerate(cols)]
        res, st = _add(es, parts)
        assert all(r == [0] * len(p) for r, p in zip(res, parts)) and st == [0] * N
        pending = [c[([0] + cuts[s] + [len(c)])[call + 1]:] for s, c in enumerate(cols)]
        firsts = [p[0][0] - (p[0][0] - START) % RES for p in pending if p]
        if call + 1 < n_calls and firsts:
            assert es.consume(min(firsts)).tolist() == [0] * N
    assert es.consume(START + W * RES).tolist() == [0] * N
    assert _rows(es) == _tiles_annotated(codec, cols, metric, types, ops, W)


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("metric", [A.METRIC_GAUGE, A.METRIC_COUNTER])
def test_annotation_capacity_stop_grow_and_resend(codecs, int_opt, metric):
    codec = codecs[int_opt]
    rng = np.random.default_rng(77 + int_opt + metric)
    N, W = 96, 6
    types, ops = ([1, 8] if metric == A.METRIC_GAUGE else [7, 8]), [4, 5]
    cols = [annotated_points(random_series(rng, START, RES, W, metric), rng, [b"ab", b"y" * 30, b"z" * 100], 0.3)
            for _ in range(N)]
    full = _new(codec, N, metric, types, ops, R=W, capacity=128)
    _add(full, cols)
    es = _new(codec, N, metric, types, ops, R=W, capacity=32)
    res, st = _add(es, cols)
    assert capi.ERR_CAPACITY in st
    for s, c in enumerate(cols):
        stop = next((i for i, (_, _, a) in enumerate(c) if len(a) > 32), None)
        assert res[s] == [0] * len(c) if stop is None else res[s] == [0] * stop + [capi.ERR_CAPACITY] * (len(c) - stop)
    again = [[p for i, p in enumerate(c) if res[s][i] == capi.ERR_CAPACITY] for s, c in enumerate(cols)]
    es.grow(annotation_capacity=128)
    res2, st2 = _add(es, again)
    assert st2 == [0] * N and all(r == [0] * len(a) for r, a in zip(res2, again))
    assert es.consume(START + W * RES).tolist() == [0] * N
    assert full.consume(START + W * RES).tolist() == [0] * N
    assert _rows(es) == _rows(full)
    assert torch.equal(es.elem, full.elem) and torch.equal(es.watermark, full.watermark)


@pytest.mark.parametrize("int_opt", [True, False])
def test_consume_capacity_from_annotation_room_alone(codecs, int_opt):
    codec = codecs[int_opt]
    cols = [[(START + 5 * SEC, _bits(1.0), b"q" * 200)], []]
    plain = codec.element_set(torch.full((2,), START, dtype=torch.int64, device=DEV), A.METRIC_GAUGE, [1], RES,
                              stride=64)
    ts, vals, n, _ = _point_major(cols)
    plain.add(ts, vals, n)
    assert plain.consume(START + RES).tolist() == [0, 0]  # 64 bytes take the datapoint without its annotation
    es = _new(codec, 2, A.METRIC_GAUGE, [1], capacity=256, stride=64)
    assert _add(es, cols) == ([[0], []], [0, 0])
    before = es.state()
    assert es.consume(START + RES).tolist() == [capi.ERR_CAPACITY, 0]
    after = es.state()
    assert torch.equal(before["ann_len"], after["ann_len"]) and torch.equal(before["ann_bytes"], after["ann_bytes"])
    assert all(torch.equal(before["win"][f], after["win"][f]) for f in before["win"])
    assert int(es.watermark[0]) == -(1 << 63) and int(es.out.num_encoded[0]) == 0
    es.grow(stride=320)
    assert es.consume(START + RES).tolist() == [0, 0]
    m = _models(1, A.METRIC_GAUGE, [1], capacity=256, int_opt=int_opt)[0]
    m.add(cols[0])
    m.consume(START + RES)
    assert _rows(es)[0] == m.streams()[0]


def test_argument_checks(codecs):
    codec = codecs[True]
    es = _new(codec, 4, A.METRIC_GAUGE, [1], capacity=64)
    L = capi.lib()
    d = es._desc()
    ts, vals, n, ann = _point_major([[(START, _bits(1.0), b"a")]] * 4)
    res = torch.zeros(ts.shape, dtype=torch.int8, device=DEV)
    st = torch.zeros(4, dtype=torch.int32, device=DEV)
    status = torch.zeros(4, dtype=torch.int32, device=DEV)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def p(t):
        if t is None or isinstance(t, C.c_void_p):
            return t if t is not None else C.c_void_p(0)
        return C.c_void_p(t.data_ptr())

    def add(a, a_off=ann[0], a_ent=ann[1], a_bytes=ann[2]):
        return L.m3tsz_element_set_add_annotated(codec.ctx.handle, C.byref(codec.opts), C.byref(d),
                                                 C.byref(a) if a is not None else None, p(ts), p(vals), ts.shape[0],
                                                 p(n), p(a_off), p(a_ent), p(a_bytes), p(res), p(st), stream)

    def consume(a):
        return L.m3tsz_element_set_consume_annotated(codec.ctx.handle, C.byref(codec.opts), C.byref(d),
                                                     C.byref(a) if a is not None else None, START + RES,
                                                     capi.UNIT_S, p(status), stream)

    def desc(**kw):
        a = es._ann()
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    bad = [None, desc(reserved=1), desc(capacity=0), desc(capacity=12), desc(capacity=capi.MAX_ELEMENT_ANNOTATION + 8),
           desc(d_len=None), desc(d_bytes=None), desc(d_len=es.ann_len.data_ptr() + 2),
           desc(d_bytes=es.ann_bytes.data_ptr() + 4)]
    for a in bad:
        assert add(a) == capi.ERR_INVALID_ARG
        assert consume(a) == capi.ERR_INVALID_ARG
    good = desc()
    assert add(good, a_ent=None) == capi.ERR_INVALID_ARG
    assert add(good, a_bytes=None) == capi.ERR_INVALID_ARG
    assert add(good, a_off=C.c_void_p(ann[0].data_ptr() + 4)) == capi.ERR_INVALID_ARG  # misaligned offsets
    assert add(good, a_ent=C.c_void_p(ann[1].data_ptr() + 4)) == capi.ERR_INVALID_ARG  # misaligned entries
    torch.cuda.synchronize()
    assert int(es.win["count"].sum()) == 0  # nothing launched
    assert add(good, a_off=None, a_ent=None, a_bytes=None) == capi.OK  # no annotations in this call
    assert add(good) == capi.OK
    assert consume(good) == capi.OK
    torch.cuda.synchronize()
    assert status.tolist() == [0] * 4


@pytest.mark.parametrize("int_opt", [True, False])
def test_100k_elements_sampled_against_the_model(codecs, int_opt):
    codec = codecs[int_opt]
    rng = np.random.default_rng(21 + int_opt)
    N, metric, types, ops = 100_000, A.METRIC_COUNTER, [7, 9], [5]
    es = _new(codec, N, metric, types, ops, R=3, capacity=64, stride=codec.encode_bound(64) + 4096)
    sample = rng.choice(N, 300, replace=False)
    models = {int(s): _models(1, metric, types, ops, R=3, capacity=64, int_opt=int_opt)[0] for s in sample}
    pay = np.frombuffer(b"".join(PAYLOADS[:3]), dtype=np.uint8)
    lens = [len(x) for x in PAYLOADS[:3]]
    starts = np.cumsum([0] + lens[:-1])
    for step in range(12):
        n = rng.integers(0, 4, N).astype(np.int32)
        t = START + step * 20 * SEC + rng.integers(-90, 30, (3, N)) * SEC
        t = np.maximum(t, START)
        v = rng.integers(-1000, 1000, (3, N)).astype(np.float64)
        v[rng.random((3, N)) < 0.02] = np.nan
        which = rng.integers(-1, 3, (3, N))  # -1: no annotation
        # the sparse list: element-major, rows in order
        has = (which >= 0) & (np.arange(3)[:, None] < n[None, :])
        cnt = has.sum(0)
        off = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
        ss, ii = np.nonzero(has.T)
        ent = np.zeros(max(1, len(ss)), dtype=[("dp_index", "<u4"), ("length", "<u4"), ("byte_offset", "<u8")])
        w = which[ii, ss]
        ent["dp_index"][: len(ss)] = ii
        ent["length"][: len(ss)] = np.array(lens)[w]
        ent["byte_offset"][: len(ss)] = starts[w]
        a = (torch.from_numpy(off).to(DEV), torch.from_numpy(ent.view(np.uint8).reshape(-1, 16)).to(DEV),
             torch.from_numpy(pay.copy()).to(DEV))
        res, _ = es.add(torch.from_numpy(t).to(DEV).contiguous(), torch.from_numpy(v).to(DEV).contiguous(),
                        torch.from_numpy(n).to(DEV), annotations=a)
        res = res.cpu().numpy()
        for s, m in models.items():
            pts = [(int(t[i, s]), _bits(v[i, s]), PAYLOADS[which[i, s]] if which[i, s] >= 0 else b"")
                   for i in range(n[s])]
            r, _ = m.add(pts)
            assert res[: n[s], s].tolist() == r, (step, s)
        if step % 3 == 2:
            target = START + (step // 3) * RES
            assert int(es.consume(target).abs().sum()) == 0
            for m in models.values():
                m.consume(target)
    rows = _rows(es)
    elem, wm = es.elem.cpu().numpy(), es.watermark.cpu().numpy()
    for s, m in models.items():
        want = m.streams()
        for j in range(len(types)):
            assert rows[j * N + s] == want[j], (s, j)
        assert elem[s].tobytes() == m.state.tobytes() and int(wm[s]) == m.watermark


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_without_annotations_the_plain_bytes(codecs, int_opt, case):
    metric, types, ops = CASES[case]
    codec = codecs[int_opt]
    rng = np.random.default_rng(900 + case + int_opt)
    N, W = 50, 6
    cols = [random_series(rng, START, RES, W, metric) for _ in range(N)]
    start = torch.full((N,), START, dtype=torch.int64, device=DEV)
    plain = codec.element_set(start, metric, types, RES, transforms=ops, discard_nan=bool(case % 2), open_windows=W)
    es = _new(codec, N, metric, types, ops, bool(case % 2), R=W, capacity=8)
    ts, vals, n, _ = _point_major([[(t, v, b"") for t, v in c] for c in cols])
    r1, s1 = plain.add(ts, vals, n)
    r2, s2 = es.add(ts, vals, n)
    assert torch.equal(r1, r2) and torch.equal(s1, s2)
    for target in (START + 3 * RES, START + W * RES):
        assert torch.equal(plain.consume(target), es.consume(target))
    assert _rows(plain) == _rows(es)
    assert torch.equal(plain.elem, es.elem) and torch.equal(plain.watermark, es.watermark)
