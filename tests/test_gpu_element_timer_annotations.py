"""Timer element sets that keep annotations on the GPU (m3tsz_element_set_add_timer_annotated /
_consume_timer_annotated, DESIGN.md §4.12), in both int_optimized modes: single samples and BatchTimer batches with an
annotation on a random subset of batches, added over 1 / 2 / 5 / 17 calls with consumes in between, equal byte for byte
in every output row to the CPU model (tests/element_timer_ann_model.py) and its reference encoder; the reference's
Timer annotation golden through the device; without any annotation, the plain Timer calls' bytes, slots and streams;
the annotation-capacity and sample-room stops with grow and resend, and a consume stopped by annotation room; the
broken-batch refusal; the argument checks and cross-refusals; 100 k elements sampled; a run on a caller's non-blocking
stream."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from element_set_ann_model import sparse_annotations
from element_timer_ann_model import AnnotatedTimerModel
from m3_b200 import capi

pytestmark = pytest.mark.gpu

SEC = 1_000_000_000
RES = 60 * SEC
START = 1_600_000_020 * SEC
DEV = "cuda"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "m3tsz_timer_annotation_goldens.json")
PAYLOADS = [b"a", b"prom", b"0123456789abcdef", b"p" * 40]
TYPES = [capi.AGG_MAX, capi.AGG_COUNT, capi.AGG_P50, capi.AGG_P99]


@pytest.fixture(scope="module")
def codecs():
    from m3_b200.codec import BatchCodec
    return {True: BatchCodec(0, int_optimized=True), False: BatchCodec(0, int_optimized=False)}


def _new(codec, N, types=TYPES, ops=(), R=4, cap=64, capacity=64, stride=None):
    return codec.element_set(torch.full((N,), START, dtype=torch.int64, device=DEV), capi.METRIC_TIMER, types, RES,
                             transforms=ops, open_windows=R, sample_capacity=cap, annotation_capacity=capacity,
                             stride=stride)


def _models(N, int_opt, types=TYPES, ops=(), R=4, cap=64, capacity=64):
    return [AnnotatedTimerModel(types, RES, ops, False, R, cap, capacity=capacity, start_ns=START,
                                int_optimized=int_opt) for _ in range(N)]


def _inputs(cols):
    """per-element rows [(t, value, continues, annotation)] -> device ts, values, n_points, batch, annotations"""
    N = len(cols)
    P = max([len(c) for c in cols] + [1])
    ts = np.zeros((P, N), dtype=np.int64)
    vs = np.zeros((P, N), dtype=np.float64)
    bt = np.zeros((P, N), dtype=np.int8)
    for s, c in enumerate(cols):
        for i, (t, v, b, _) in enumerate(c):
            ts[i, s], vs[i, s], bt[i, s] = t, v, b
    n = np.array([len(c) for c in cols], dtype=np.int32)
    ann = tuple(torch.from_numpy(a).to(DEV) for a in sparse_annotations([[(0, 0, a) for *_, a in c] for c in cols]))
    d = lambda a: torch.from_numpy(a).to(DEV)
    return d(ts), d(vs), d(n), d(bt), ann


def _add(es, models, cols):
    ts, vs, n, bt, ann = _inputs(cols)
    res, st = es.add(ts, vs, n, annotations=ann, batch=bt)
    res, st = res.cpu().numpy(), st.cpu().numpy().tolist()
    for s, m in enumerate(models):
        c = cols[s]
        want = m.add([(t, v) for t, v, _, _ in c], [b for _, _, b, _ in c], [a for *_, a in c])
        assert (res[: len(c), s].tolist(), st[s]) == want, s
    return res, st


def _rows(es):
    snap = es.stream()
    out, ln = snap.out.cpu().numpy(), snap.out_len.cpu().numpy()
    return [out[r, : ln[r]].tobytes() for r in range(len(ln))]


def _consume_and_check(es, models, target):
    assert es.consume(target).cpu().numpy().tolist() == [0] * len(models)
    for m in models:
        m.consume(target)
    rows, N = _rows(es), es.n_elements
    for s, m in enumerate(models):
        for j, want in enumerate(m.streams()):
            assert rows[j * N + s] == want, (s, j)
        assert es.elem[s].cpu().numpy().tobytes() == m.state.tobytes() and int(es.watermark[s]) == m.watermark


def _random_cols(rng, N, W, p_ann=0.4, batchy=True):
    cols = []
    for _ in range(N):
        rows = []
        for w in range(W):
            for _ in range(int(rng.integers(0, 3))):
                t = START + w * RES + int(rng.integers(0, 60)) * SEC
                a = PAYLOADS[int(rng.integers(0, len(PAYLOADS)))] if rng.random() < p_ann else b""
                for i in range(int(rng.integers(1, 6)) if batchy else 1):
                    v = float("nan") if rng.random() < 0.03 else float(np.round(rng.exponential(50), 1))
                    rows.append((t, v, 1 if i else 0, b"" if i else a))
        cols.append(rows)
    return cols


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("calls", [1, 2, 5, 17])
def test_adds_over_calls_equal_the_model(codecs, int_opt, calls):
    rng = np.random.default_rng(calls * 2 + int_opt)
    N, W = 64, 6
    es, models = _new(codecs[int_opt], N), _models(N, int_opt)
    cols = _random_cols(rng, N, W, batchy=calls % 2 == 1)
    for c in range(calls):  # each call takes the rows of some windows (a batch shares one timestamp), consumed after
        lo, hi = c * W // calls, (c + 1) * W // calls
        _add(es, models, [[r for r in col if lo <= (r[0] - START) // RES < hi] for col in cols])
        _consume_and_check(es, models, START + hi * RES)
    _consume_and_check(es, models, START + (W + 1) * RES)


def test_golden_through_the_device(codecs):
    for case in json.load(open(GOLDEN))["cases"]:
        es, models = _new(codecs[True], 1), _models(1, True)
        cols = [[(START + SEC, v, 0, (a or "").encode()) for v, a in case["adds"]]]
        _add(es, models, cols)
        assert int(es.ann_len[0, 0]) == len(case["want"])
        assert es.ann_bytes[0, 0, : len(case["want"])].cpu().numpy().tobytes() == case["want"].encode()
        _consume_and_check(es, models, START + RES)


@pytest.mark.parametrize("int_opt", [True, False])
def test_without_annotations_equals_the_plain_calls(codecs, int_opt):
    rng = np.random.default_rng(9)
    N = 128
    a = _new(codecs[int_opt], N)
    p = codecs[int_opt].element_set(torch.full((N,), START, dtype=torch.int64, device=DEV), capi.METRIC_TIMER, TYPES,
                                    RES, open_windows=4, sample_capacity=64)
    for step in range(3):
        cols = _random_cols(rng, N, 2, p_ann=0.0)
        ts, vs, n, bt, ann = _inputs(cols)
        ra, sa = a.add(ts, vs, n, annotations=ann, batch=bt)
        rp, sp = p.add(ts, vs, n, batch=bt)
        assert torch.equal(ra, rp) and torch.equal(sa, sp)
        target = START + (step + 1) * RES
        assert torch.equal(a.consume(target), p.consume(target))
        assert _rows(a) == _rows(p)
        sa_, sp_ = a.state(), p.state()
        bits = lambda x: x.view(torch.uint8)  # (NaN sums and samples compare by their bits)
        for f in sp_["win"]:
            assert torch.equal(bits(sa_["win"][f]), bits(sp_["win"][f]))
        for f in sp_["streams"]:
            assert torch.equal(bits(sa_["streams"][f]), bits(sp_["streams"][f]))


def test_capacity_stops_then_grow_and_resend(codecs):
    es, models = _new(codecs[True], 3, R=1, cap=4, capacity=8), _models(3, True, R=1, cap=4, capacity=8)
    cols = [[(START + SEC, 1.0, 0, b"x" * 16), (START + 2 * SEC, 2.0, 0, b"")],  # annotation too long
            [(START + SEC, 1.0, 0, b"ok"), (START + RES, 2.0, 0, b"")],  # second window: no slot
            [(START + SEC, float(i), 1 if i else 0, b"") for i in range(6)]]  # batch past the sample room
    res, st = _add(es, models, cols)
    assert st == [capi.ERR_CAPACITY] * 3
    es.grow(open_windows=2, sample_capacity=8, annotation_capacity=16)
    for m in models:
        m.m.R, m.m.cap, m.capacity = 2, 8, 16
    again = [[r for i, r in enumerate(c) if res[i, s] == capi.ERR_CAPACITY] for s, c in enumerate(cols)]
    assert _add(es, models, again)[1] == [0, 0, 0]
    _consume_and_check(es, models, START + 2 * RES)


def test_consume_stopped_by_annotation_room(codecs):
    # one datapoint: 2 words + 10 + 4 without its annotation, (64 + 3) / 4 + 4 = 20 with it
    stride = 4 * (2 + 10 + 4 + 20 - 1) // 16 * 16
    es = _new(codecs[True], 2, types=[capi.AGG_MAX], stride=stride)
    ts, vs, n, bt, ann = _inputs([[(START + SEC, 1.0, 0, b"z" * 64)], [(START + SEC, 1.0, 0, b"")]])
    es.add(ts, vs, n, annotations=ann, batch=bt)
    assert es.consume(START + RES).cpu().tolist() == [capi.ERR_CAPACITY, 0]
    es.grow(stride=stride + 64)
    assert es.consume(START + RES).cpu().tolist() == [0, 0]


def test_broken_batch_and_closed_windows(codecs):
    es, models = _new(codecs[True], 3, capacity=8), _models(3, True, capacity=8)
    cols = [[(START + SEC, 1.0, 0, b""), (START + SEC, 2.0, 1, b"late")],  # annotation on a continuation
            [(START + SEC, 1.0, 0, b"a")], [(START + SEC, 1.0, 0, b"b")]]
    assert _add(es, models, cols)[1] == [capi.ERR_INVALID_ARG, 0, 0]
    assert int(es.win["count"].sum()) == 2
    _consume_and_check(es, models, START + RES)
    # a closed batch with a too-long annotation is closed, and the element goes on
    cols = [[], [(START + SEC, 1.0, 0, b"y" * 16), (START + RES + SEC, 1.0, 0, b"c")], []]
    res, st = _add(es, models, cols)
    assert res[:2, 1].tolist() == [capi.ERR_AGGREGATION_CLOSED, 0] and st[1] == 0


def test_argument_checks_and_cross_refusals(codecs):
    codec = codecs[True]
    L = capi.lib()
    es, plain = _new(codec, 4), codec.element_set(torch.full((4,), START, dtype=torch.int64, device=DEV),
                                                   capi.METRIC_TIMER, TYPES, RES, sample_capacity=8)
    gauge = codec.element_set(torch.full((4,), START, dtype=torch.int64, device=DEV), capi.METRIC_GAUGE, [1], RES,
                              annotation_capacity=8)
    ts = torch.zeros((1, 4), dtype=torch.int64, device=DEV)
    vs = torch.zeros((1, 4), dtype=torch.float64, device=DEV)
    out8 = torch.zeros((1, 4), dtype=torch.int8, device=DEV)
    st = torch.zeros(4, dtype=torch.int32, device=DEV)
    h, o = codec.ctx.handle, C.byref(codec.opts)
    p = lambda t: C.c_void_p(t.data_ptr())
    cs = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def add(d, streams, ann):
        return L.m3tsz_element_set_add_timer_annotated(h, o, C.byref(d), streams, ann, p(ts), p(vs), 1, None, None,
                                                       None, None, None, p(out8), p(st), cs)

    def consume(d, streams, ann):
        return L.m3tsz_element_set_consume_timer_annotated(h, o, C.byref(d), streams, ann, START, 1, p(st), cs)

    good = es._ann()
    for call in (add, consume):
        assert call(es._desc(), C.byref(es._streams()), C.byref(good)) == 0
        assert call(es._desc(), C.byref(es._streams()), None) == capi.ERR_INVALID_ARG
        assert call(gauge._desc(), C.byref(es._streams()), C.byref(gauge._ann())) == capi.ERR_INVALID_ARG
        for field, bad in (("capacity", 12), ("capacity", 0), ("reserved", 1)):
            a = es._ann()
            setattr(a, field, bad)
            assert call(es._desc(), C.byref(es._streams()), C.byref(a)) == capi.ERR_INVALID_ARG
    # the Gauge / Counter annotated calls keep refusing Timer sets
    assert L.m3tsz_element_set_add_annotated(h, o, C.byref(es._desc()), C.byref(good), p(ts), p(vs), 1, None, None,
                                             None, None, p(out8), p(st), cs) == capi.ERR_INVALID_ARG
    assert L.m3tsz_element_set_consume_annotated(h, o, C.byref(es._desc()), C.byref(good), START, 1, p(st),
                                                 cs) == capi.ERR_INVALID_ARG
    torch.cuda.synchronize()
    with pytest.raises(ValueError):
        es.forward(START, torch.zeros(1, dtype=torch.int64, device=DEV), torch.zeros(0, dtype=torch.int32, device=DEV),
                   plain)


def test_100k_elements_sampled(codecs):
    rng = np.random.default_rng(11)
    N = 100_000
    es = _new(codecs[True], N, capacity=16)
    cols = _random_cols(rng, N, 2, p_ann=0.5, batchy=False)
    cols = [[r[:3] + (r[3][:16],) for r in c] for c in cols]
    ts, vs, n, bt, ann = _inputs(cols)
    _, st = es.add(ts, vs, n, annotations=ann, batch=bt)
    assert int((st != 0).sum()) == 0
    assert int((es.consume(START + 2 * RES) != 0).sum()) == 0
    rows = _rows(es)
    for s in rng.choice(N, 64, replace=False).tolist():
        m = AnnotatedTimerModel(TYPES, RES, capacity=16, start_ns=START)
        c = cols[s]
        m.add([(t, v) for t, v, _, _ in c], [b for _, _, b, _ in c], [a for *_, a in c])
        m.consume(START + 2 * RES)
        for j, want in enumerate(m.streams()):
            assert rows[j * N + s] == want, (s, j)


def test_on_a_non_blocking_stream(codecs):
    rng = np.random.default_rng(12)
    N = 256
    es, models = _new(codecs[False], N), _models(N, False)
    cols = _random_cols(rng, N, 2)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()  # (created non-blocking by torch)
    with torch.cuda.stream(s):
        torch.cuda._sleep(1_000_000)
        _add(es, models, cols)
        _consume_and_check(es, models, START + 2 * RES)
