"""Timer element sets on the GPU (m3tsz_element_set_*_timer, DESIGN.md §4.12), in both int_optimized modes: the
reference's Timer and CM stream expectations through the device calls; samples added over 1 / 2 / 5 / 17 calls (single
samples and BatchTimer batches) with consumes in between, equal to the CPU model (tests/element_timer_model.py) in
every written datapoint, value bits included, and in the element records, for the default 11-type element, a
quantile-only element with an unsorted quantile list and an element with transformations; grow-and-resend after
capacity stops on open windows and on sample_capacity; closed windows and invalid batch continuations; argument checks and the refusals of the other calls; 100 k elements sampled against the
model; a run on a caller's non-blocking stream behind a sleep."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

import timer_oracle_lib as T
from element_timer_model import TimerElementModel
from m3_b200 import capi
from test_gpu_elements import _decoded_rows

pytestmark = pytest.mark.gpu

SEC = 1_000_000_000
RES = 60 * SEC
START = 1_600_000_020 * SEC  # a whole minute
DEV = "cuda"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "m3tsz_timer_goldens.json")


@pytest.fixture(scope="module")
def codecs():
    from m3_b200.codec import BatchCodec
    return {True: BatchCodec(0, int_optimized=True), False: BatchCodec(0, int_optimized=False)}


def _timer_set(codec, N, types, ops=(), discard=False, R=4, cap=64, eps=1e-3, every=1024, stride=None):
    return codec.element_set(torch.full((N,), START, dtype=torch.int64, device=DEV), capi.METRIC_TIMER, types, RES,
                             transforms=ops, discard_nan=discard, open_windows=R, sample_capacity=cap, eps=eps,
                             insert_and_compress_every=every, stride=stride)


def _point_major(cols):
    """per-element rows [(t, value, continues)] -> ts, values, n_points, batch on the device"""
    N = len(cols)
    P = max([len(c) for c in cols] + [1])
    ts = np.zeros((P, N), dtype=np.int64)
    vs = np.zeros((P, N), dtype=np.float64)
    bt = np.zeros((P, N), dtype=np.int8)
    for s, c in enumerate(cols):
        for i, (t, v, b) in enumerate(c):
            ts[i, s], vs[i, s], bt[i, s] = t, v, b
    n = np.array([len(c) for c in cols], dtype=np.int32)
    return (torch.from_numpy(ts).to(DEV), torch.from_numpy(vs).to(DEV), torch.from_numpy(n).to(DEV),
            torch.from_numpy(bt).to(DEV))


def _add(es, models, cols):
    ts, vs, n, bt = _point_major(cols)
    res, st = es.add(ts, vs, n, batch=bt)
    res, st = res.cpu().numpy(), st.cpu().numpy().tolist()
    for s, m in enumerate(models):
        want_r, want_s = m.add([(t, v) for t, v, _ in cols[s]], [b for _, _, b in cols[s]])
        assert res[: len(cols[s]), s].tolist() == want_r and st[s] == want_s, s
    return st


def _encoded(codec, rows):
    """rows of datapoints [(t, value bits)] through the batch encoder (start START, seconds, as the element sets'
    output rows) and back: what the same datapoints read as after the codec's value encoding"""
    R = len(rows)
    P = max([len(r) for r in rows] + [1])
    ts = np.full((R, P), START, dtype=np.int64)
    vb = np.zeros((R, P), dtype=np.uint64)
    for i, r in enumerate(rows):
        for j, (t, v) in enumerate(r):
            ts[i, j], vb[i, j] = t, v
    n = torch.tensor([len(r) for r in rows], dtype=torch.int32, device=DEV)
    enc = codec.encode(torch.from_numpy(ts).to(DEV), torch.from_numpy(vb.view(np.float64)).to(DEV),
                       torch.full((R,), START, dtype=torch.int64, device=DEV), n_points=n)
    offs = torch.arange(R, dtype=torch.int64, device=DEV) * enc.out.shape[1]
    dec = codec.decode(enc.out.view(-1), offs, P, lengths=enc.out_len)
    dt, dv, dn = dec.ts.cpu().numpy(), dec.values.cpu().numpy().view(np.uint64), dec.n_points.cpu().numpy()
    return [list(zip(dt[i, : dn[i]].tolist(), dv[i, : dn[i]].tolist())) if rows[i] else [] for i in range(R)]


def _consume_and_check(codec, es, models, target, acc):
    st = es.consume(target).cpu().numpy().tolist()
    assert st == [0] * len(models)
    k = len(es.agg_types)
    for s, m in enumerate(models):
        for j, (t, v) in enumerate(m.consume(target)):
            acc[j * len(models) + s] += list(zip(t.tolist(), np.asarray(v).view(np.uint64).tolist()))
    rows = _decoded_rows(codec, es, cap=256)
    assert rows == _encoded(codec, acc)
    elem = es.elem.cpu().numpy()
    for s, m in enumerate(models):
        if k <= 8:
            assert elem[s].tobytes() == m.state.tobytes(), s
        assert int(es.watermark[s]) == m.watermark


def _random_rows(rng, W, batchy):
    """one element's rows over W windows: single samples, or batches of 1 .. 40 at one timestamp"""
    rows = []
    for w in range(W):
        for _ in range(int(rng.integers(0, 4))):
            t = START + w * RES + int(rng.integers(0, 60)) * SEC
            n = int(rng.integers(1, 41)) if batchy else 1
            for i in range(n):
                r = rng.random()
                v = float("nan") if r < 0.03 else -0.0 if r < 0.08 else 0.0 if r < 0.13 else \
                    float(np.round(rng.exponential(50), int(rng.integers(0, 3))))
                rows.append((t, v, 1 if i else 0))
    return rows


CASES = [
    (list(capi.DEFAULT_TIMER_TYPES), []),
    ([capi.AGG_MEDIAN, capi.AGG_P10, capi.AGG_P90, capi.AGG_P99, capi.AGG_P25, capi.AGG_P75], []),
    ([capi.AGG_MAX, capi.AGG_COUNT, capi.AGG_P50, capi.AGG_P99], [capi.TRANSFORM_INCREASE, capi.TRANSFORM_RESET]),
]


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("n_calls", [1, 2, 5, 17])
def test_adds_over_calls_equal_the_model(codecs, int_opt, case, n_calls):
    types, ops = CASES[case]
    codec = codecs[int_opt]
    rng = np.random.default_rng(1000 * case + 10 * n_calls + int_opt)
    N, W = 48, 6
    every = [2, 7, 1024][case]
    cap = 512
    es = _timer_set(codec, N, types, ops, discard=True, R=W + 1, cap=cap, every=every,
                    stride=int(capi.lib().m3tsz_encode_bound_units(64, 1)))
    models = [TimerElementModel(types, RES, ops, True, W + 1, cap, 1e-3, every) for _ in range(N)]
    cols = [_random_rows(rng, W, batchy=bool(s % 2)) for s in range(N)]
    acc = [[] for _ in range(len(types) * N)]
    # cut each element's rows into n_calls parts at batch boundaries; consume the windows ended before each part
    for call in range(n_calls):
        parts = []
        for c in cols:
            starts = [i for i, (_, _, b) in enumerate(c) if not b] + [len(c)]
            lo = starts[len(starts) * call // n_calls] if call else 0
            hi = starts[len(starts) * (call + 1) // n_calls] if call + 1 < n_calls else len(c)
            parts.append(c[lo:hi])
        assert _add(es, models, parts) == [0] * N
        if call + 1 < n_calls:
            _consume_and_check(codec, es, models, START + (W * (call + 1) // n_calls) * RES, acc)
    _consume_and_check(codec, es, models, START + (W + 1) * RES, acc)


@pytest.mark.parametrize("case", json.load(open(GOLDEN))["cases"], ids=lambda c: c["name"])
def test_goldens_through_the_device(codecs, case):
    codec = codecs[True]
    batches = [list(b) for b, times in case["batches"] for _ in range(times)]
    rows = [(START + SEC, v, 1 if i else 0) for b in batches for i, v in enumerate(b)]
    n = len(rows)
    es = _timer_set(codec, 1, case["types"], R=1, cap=n, eps=case["eps"], every=case["every"])
    ts, vs, npts, bt = _point_major([rows])
    res, st = es.add(ts, vs, npts, batch=bt)
    assert int(st[0]) == 0 and int(res.abs().sum()) == 0
    assert int(es.consume(START + RES)[0]) == 0
    got = _decoded_rows(codec, es)
    want, _ = T.timer_window(batches, case["types"], case["eps"], case["every"])
    assert got == _encoded(codec, [[(START + RES, int(np.array([w]).view(np.uint64)[0]))] for w in want])
    for j, ty in enumerate(case["types"]):
        assert len(got[j]) == 1
        if str(ty) in case["want"]:
            assert np.array([got[j][0][1]], dtype=np.uint64).view(np.float64)[0] == case["want"][str(ty)], ty


def test_grow_and_resend_gives_the_unstopped_result(codecs):
    codec = codecs[False]
    types = list(capi.DEFAULT_TIMER_TYPES)
    rng = np.random.default_rng(11)
    N = 16
    cols = [_random_rows(rng, 3, batchy=True) for _ in range(N)]
    big = _timer_set(codec, N, types, R=4, cap=4096, every=5)
    ts, vs, n, bt = _point_major(cols)
    assert int(big.add(ts, vs, n, batch=bt)[1].abs().sum()) == 0
    assert int(big.consume(START + 4 * RES).abs().sum()) == 0
    small = _timer_set(codec, N, types, R=1, cap=8, every=5)
    pending = cols
    for _ in range(64):
        ts, vs, n, bt = _point_major(pending)
        res, st = small.add(ts, vs, n, batch=bt)
        res = res.cpu().numpy()
        refused = [[r for i, r in enumerate(c) if res[i, s] == capi.ERR_CAPACITY] for s, c in enumerate(pending)]
        if not any(refused):
            break
        small.grow(open_windows=min(4, small.open_windows + 1), sample_capacity=small.sample_capacity * 2)
        pending = refused
    assert not any(refused)
    assert int(small.consume(START + 4 * RES).abs().sum()) == 0
    assert _decoded_rows(codec, small) == _decoded_rows(codec, big)
    assert torch.equal(small.elem, big.elem) and torch.equal(small.watermark, big.watermark)


def test_closed_windows_and_invalid_batches(codecs):
    codec = codecs[True]
    types = [capi.AGG_COUNT, capi.AGG_P50]
    es = _timer_set(codec, 3, types, R=2, cap=16)
    models = [TimerElementModel(types, RES, (), False, 2, 16) for _ in range(3)]
    _add(es, models, [[(START + SEC, 1.0, 0)], [(START + SEC, 2.0, 0)], [(START + SEC, 3.0, 0)]])
    _consume_and_check(codec, es, models, START + RES, [[] for _ in range(6)])
    st = _add(es, models, [[(START + 2 * SEC, 4.0, 0), (START + 2 * SEC, 5.0, 1)],  # closed window
                           [(START + RES, 6.0, 1)],  # a continuation in row 0
                           [(START + RES, 7.0, 0), (START + RES + SEC, 8.0, 1)]])  # another timestamp
    assert st == [0, capi.ERR_INVALID_ARG, capi.ERR_INVALID_ARG]


def test_argument_checks_and_refusals(codecs):
    codec = codecs[True]
    lib = capi.lib()
    es = _timer_set(codec, 4, [capi.AGG_MIN, capi.AGG_P99], cap=8)
    d, sd = es._desc(), es._streams()
    ctx, opts = codec.ctx.handle, C.byref(codec.opts)
    ts = torch.zeros((1, 4), dtype=torch.int64, device=DEV)
    vs = torch.zeros((1, 4), dtype=torch.float64, device=DEV)
    res = torch.zeros((1, 4), dtype=torch.int8, device=DEV)
    st = torch.zeros(4, dtype=torch.int32, device=DEV)
    P = lambda t: C.c_void_p(t.data_ptr())

    def add(d_=None, sd_=None):
        return lib.m3tsz_element_set_add_timer(ctx, opts, C.byref(d_ or d), None if sd_ is False else C.byref(sd_ or sd),
                                               P(ts), P(vs), 1, None, None, P(res), P(st), None)

    assert add() == capi.OK
    assert add(sd_=False) == capi.ERR_INVALID_ARG
    for field, bad in (("sample_capacity", 0), ("eps", 0.0), ("eps", float("inf")), ("eps", float("nan")),
                       ("insert_and_compress_every", 0), ("reserved", 1), ("d_value", sd.d_value + 4),
                       ("d_header", None)):
        x = capi.ElementTimerStreams.from_buffer_copy(sd)
        setattr(x, field, bad)
        assert add(sd_=x) == capi.ERR_INVALID_ARG, field
    for types, ops in (([capi.AGG_LAST], []), ([capi.AGG_MAX, capi.AGG_MIN], []), ([0], []),
                       (list(range(2, 11)), [capi.TRANSFORM_ABSOLUTE]), ([25], [])):
        x = capi.ElementSet.from_buffer_copy(d)
        arr, oa = (C.c_int32 * len(types))(*types), (C.c_int32 * max(1, len(ops)))(*ops)
        x.agg_types, x.n_types = C.cast(arr, C.POINTER(C.c_int32)), len(types)
        x.ops, x.n_ops = C.cast(oa, C.POINTER(C.c_int32)), len(ops)
        assert add(d_=x) == capi.ERR_INVALID_ARG, types
    all23 = [t for t in range(2, 25)]
    es23 = _timer_set(codec, 4, all23, cap=8)
    assert int(es23.add(ts, vs)[1].abs().sum()) == 0
    # the other element-set calls refuse a Timer set; the Timer calls refuse the others
    assert lib.m3tsz_element_set_add(ctx, opts, C.byref(d), P(ts), P(vs), 1, None, P(res), P(st), None) == \
        capi.ERR_INVALID_ARG
    assert lib.m3tsz_element_set_consume(ctx, opts, C.byref(d), START, 1, P(st), None) == capi.ERR_INVALID_ARG
    with pytest.raises(ValueError):
        es.forward(START, torch.zeros(1, dtype=torch.int64, device=DEV), torch.zeros(0, dtype=torch.int32, device=DEV),
                   es)
    g = codec.element_set(torch.full((4,), START, dtype=torch.int64, device=DEV), capi.METRIC_GAUGE, [capi.AGG_MAX],
                          RES)
    assert lib.m3tsz_element_set_add_timer(ctx, opts, C.byref(g._desc()), C.byref(sd), P(ts), P(vs), 1, None, None,
                                           P(res), P(st), None) == capi.ERR_INVALID_ARG
    assert lib.m3tsz_element_set_consume_timer(ctx, opts, C.byref(g._desc()), C.byref(sd), START, 1, P(st), None) == \
        capi.ERR_INVALID_ARG
    # the tile calls keep refusing metric type 2
    state = torch.zeros(1, dtype=torch.int64, device=DEV)
    assert lib.m3tsz_aggregate_tiles_ex(ctx, opts, P(state), 8, P(state), None, 1, START, RES, 1, capi.METRIC_TIMER,
                                        capi.AGG_MAX, 1, 16, P(state), 8, P(state), P(state), P(st), None, None,
                                        None) == capi.ERR_INVALID_ARG
    es.reset(torch.full((4,), START, dtype=torch.int64, device=DEV))
    assert int(es.win["count"].abs().sum()) == 0 and int(es.watermark[0]) == -(1 << 63)


def test_large_set_sampled(codecs):
    codec = codecs[True]
    types = list(capi.DEFAULT_TIMER_TYPES)
    N, W, P = 100_000, 2, 12
    g = torch.Generator(device="cpu").manual_seed(3)
    ts = (START + (torch.arange(P) // 6 * RES + (torch.arange(P) % 6) * 10 * SEC)).view(P, 1).expand(P, N).contiguous()
    vs = torch.round(torch.rand((P, N), generator=g, dtype=torch.float64) * 1000) / 10
    es = _timer_set(codec, N, types, R=W + 1, cap=16)
    res, st = es.add(ts.to(DEV), vs.to(DEV))
    assert int(st.abs().sum()) == 0
    assert int(es.consume(START + 2 * RES).abs().sum()) == 0
    snap = es.stream()
    sample = np.random.default_rng(1).choice(N, 200, replace=False)
    dec = codec.decode(snap.out.view(-1), es.out.offsets(), 4, lengths=snap.out_len)
    dt, dv = dec.ts.cpu().numpy(), dec.values.cpu().numpy().view(np.uint64)
    got, want = [], []
    for s in sample.tolist():
        m = TimerElementModel(types, RES, (), False, W + 1, 16)
        m.add([(int(ts[i, s]), float(vs[i, s])) for i in range(P)])
        for j, (t, v) in enumerate(m.consume(START + 2 * RES)):
            want.append(list(zip(t.tolist(), np.asarray(v).view(np.uint64).tolist())))
            got.append(list(zip(dt[j * N + s, :2].tolist(), dv[j * N + s, :2].tolist())))
    assert got == _encoded(codec, want)


def test_on_a_non_blocking_stream_behind_a_sleep(codecs):
    codec = codecs[True]
    types = [capi.AGG_MAX, capi.AGG_P50, capi.AGG_P99]
    N = 64
    rng = np.random.default_rng(9)
    cols = [_random_rows(rng, 2, batchy=True) for _ in range(N)]
    ref = _timer_set(codec, N, types, R=3, cap=256)
    ts, vs, n, bt = _point_major(cols)
    ref.add(ts, vs, n, batch=bt)
    ref.consume(START + 2 * RES)
    want = _decoded_rows(codec, ref)
    es = _timer_set(codec, N, types, R=3, cap=256)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(20_000_000)
        es.add(ts, vs, n, batch=bt)
        es.consume(START + 2 * RES)
    s.synchronize()
    torch.cuda.synchronize()
    assert _decoded_rows(codec, es) == want
