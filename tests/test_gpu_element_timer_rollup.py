"""Timer element sets through a rollup on the GPU (m3tsz_element_set_forward_timer, DESIGN.md §4.12), in both
int_optimized modes and with contiguous and random membership: samples added over 1 / 2 / 5 / 17 calls with forwards
and group consumes in between, equal to the CPU model (tests/element_timer_rollup_model.py) in every written datapoint,
value bits included, and in the statuses, records and watermarks; the group set's state (slots, stream headers and
arenas) and bytes equal to a twin group set fed by add_timer with the forwarded values in listed order, one row per
value; the reference's Timer rollup goldens through the device; grow-and-retry after both capacity stops; the host
checks and the refusals of the other forward calls; 100 k sources sampled against the model; a run on a caller's
non-blocking stream behind a sleep."""
import ctypes as C
import json
import math
import os

import numpy as np
import pytest
import torch

from element_set_model import window_start
from element_timer_rollup_model import TimerGroupModel, TimerSourceModel, forward
from m3_b200 import capi
from test_gpu_element_timers import _encoded, _point_major, _random_rows, _timer_set
from test_gpu_elements import _decoded_rows

pytestmark = pytest.mark.gpu

SEC = 1_000_000_000
RES = 60 * SEC
START = 1_600_000_020 * SEC  # a whole minute
DEV = "cuda"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "m3tsz_timer_rollup_goldens.json")


@pytest.fixture(scope="module")
def codecs():
    from m3_b200.codec import BatchCodec
    return {True: BatchCodec(0, int_optimized=True), False: BatchCodec(0, int_optimized=False)}


def _source_set(codec, N, src_type, ops=(), discard=False, R=4, cap=64, every=1024, eps=1e-3):
    return _timer_set(codec, N, [src_type], ops, discard, R=R, cap=cap, eps=eps, every=every, stride=0)


def _groups(kind, S, G, rng):
    """contiguous: group g is sources g * S / G .. ; random: 1 .. 7 random sources each, some listed twice"""
    if kind == "contiguous":
        off = np.arange(G + 1, dtype=np.int64) * (S // G)
        mem = np.arange(off[-1], dtype=np.int32)
    else:
        lens = rng.integers(1, 8, G)
        off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        mem = rng.integers(0, S, int(off[-1])).astype(np.int32)
    return off, mem


def _dev(off, mem):
    return torch.from_numpy(np.asarray(off, dtype=np.int64)).to(DEV), \
        torch.from_numpy(np.asarray(mem, dtype=np.int32)).to(DEV)


def _add_sources(es, models, cols):
    ts, vs, n, bt = _point_major(cols)
    res, st = es.add(ts, vs, n, batch=bt)
    res, st = res.cpu().numpy(), st.cpu().numpy().tolist()
    for s, m in enumerate(models):
        want = m.add([(t, v) for t, v, _ in cols[s]], [b for _, _, b in cols[s]])
        assert (res[: len(cols[s]), s].tolist(), st[s]) == want, s


def _forwarded_by_group(sms, target, off, mem):
    """the values each group takes, in listed order: [(window start, value)] per group, from the model"""
    pend = [s.pending(target)[0] for s in sms]
    return [[(ws, v) for i in range(int(off[g]), int(off[g + 1])) for ws, v, ok in pend[int(mem[i])] if ok]
            for g in range(len(off) - 1)]


def _check_group_rows(codec, es, gms, target, acc):
    st = es.consume(target).cpu().numpy().tolist()
    assert st == [0] * len(gms)
    for g, m in enumerate(gms):
        for j, (t, v) in enumerate(m.consume(target)):
            acc[j * len(gms) + g] += list(zip(t.tolist(), np.asarray(v).view(np.uint64).tolist()))
    assert _decoded_rows(codec, es, cap=256) == _encoded(codec, acc)
    elem = es.elem.cpu().numpy()
    for g, m in enumerate(gms):
        assert elem[g].tobytes() == m.state.tobytes(), g
        assert int(es.watermark[g]) == m.watermark


def _bits(t):
    return t.view(torch.int64) if t.dtype == torch.float64 else t


def _same_state(a, b):
    """slots, stream headers and arenas, records and watermarks, bit for bit (NaN sums and samples included)"""
    sa, sb = a.state(), b.state()
    for f in sa["win"]:
        assert torch.equal(_bits(sa["win"][f]), _bits(sb["win"][f])), f
    for f in sa["streams"]:
        assert torch.equal(_bits(sa["streams"][f]), _bits(sb["streams"][f])), f
    assert torch.equal(sa["watermark"], sb["watermark"]) and torch.equal(sa["elem"], sb["elem"])


PIPES = [(capi.AGG_P99, [], [capi.AGG_MAX, capi.AGG_P50, capi.AGG_P99], [], False),
         (capi.AGG_MAX, [capi.TRANSFORM_ABSOLUTE], list(capi.DEFAULT_TIMER_TYPES), [], True)]


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("kind", ["contiguous", "random"])
@pytest.mark.parametrize("n_calls", [1, 2, 5, 17])
def test_adds_over_calls_equal_the_model(codecs, int_opt, kind, n_calls):
    codec = codecs[int_opt]
    rng = np.random.default_rng(100 * n_calls + 10 * int_opt + (kind == "random"))
    src_type, pre, types, post, discard = PIPES[(n_calls + int_opt) % 2]
    S, G, W = 48, 8, 6
    every = [2, 7, 1024][n_calls % 3]
    off, mem = _groups(kind, S, G, rng)
    doff, dmem = _dev(off, mem)
    src = _source_set(codec, S, src_type, pre, discard, R=W + 1, cap=512, every=every)
    grp = _timer_set(codec, G, types, post, discard, R=W + 1, cap=512, every=every,
                     stride=int(capi.lib().m3tsz_encode_bound_units(64, 1)))
    twin = _timer_set(codec, G, types, post, discard, R=W + 1, cap=512, every=every,
                      stride=int(capi.lib().m3tsz_encode_bound_units(64, 1)))
    sms = [TimerSourceModel(src_type, RES, pre, discard, W + 1, 512, 1e-3, every) for _ in range(S)]
    gms = [TimerGroupModel(types, RES, post, discard, W + 1, 512, 1e-3, every) for _ in range(G)]
    cols = [_random_rows(rng, W, batchy=bool(s % 2)) for s in range(S)]
    acc = [[] for _ in range(len(types) * G)]
    for call in range(n_calls):
        parts = []
        for c in cols:
            starts = [i for i, (_, _, b) in enumerate(c) if not b] + [len(c)]
            lo = starts[len(starts) * call // n_calls] if call else 0
            hi = starts[len(starts) * (call + 1) // n_calls] if call + 1 < n_calls else len(c)
            parts.append(c[lo:hi])
        _add_sources(src, sms, parts)
        target = START + (W * (call + 1) // n_calls) * RES if call + 1 < n_calls else START + (W + 1) * RES
        vals = _forwarded_by_group(sms, target, off, mem)
        sst, gst = src.forward_timer(target, doff, dmem, grp)
        assert (sst.cpu().numpy().tolist(), gst.cpu().numpy().tolist()) == forward(sms, gms, target, off, mem)
        # the twin takes the same values through add_timer, one row (one Timer.Add) per value
        ts, vs, n, _ = _point_major([[(ws, v, 0) for ws, v in vals[g]] for g in range(G)])
        twin.add(ts, vs, n)
        _same_state(grp, twin)
        es = src.elem.cpu().numpy()
        for s, m in enumerate(sms):
            assert es[s].tobytes() == m.state.tobytes() and int(src.watermark[s]) == m.watermark, s
        _check_group_rows(codec, grp, gms, target, acc)
        assert int(twin.consume(target).abs().sum()) == 0
        assert _decoded_rows(codec, twin, cap=256) == _decoded_rows(codec, grp, cap=256)


def _set_at(codec, N, types, res, ops=(), discard=False, R=4, cap=64, eps=1e-3, every=1024, stride=None):
    """a Timer set of resolution `res`"""
    return codec.element_set(torch.full((N,), START, dtype=torch.int64, device=DEV), capi.METRIC_TIMER, types, res,
                             transforms=ops, discard_nan=discard, open_windows=R, sample_capacity=cap, eps=eps,
                             insert_and_compress_every=every, stride=stride)


def test_goldens_through_the_device(codecs):
    g = json.load(open(GOLDEN))
    codec = codecs[False]  # (float mode: the decoded values are the written ones)
    for case in g["add_unique"]:
        res = case["resolution_s"] * SEC
        steps = case["steps"]
        base = 1_600_000_000 * SEC  # (a whole 10 s: the goldens' times are seconds after it)
        for upto in range(1, len(steps) + 1):
            src = _set_at(codec, len(steps), [capi.AGG_MAX], res, R=2, cap=4, stride=0, eps=case["eps"],
                          every=case["every"])
            grp = _set_at(codec, 1, case["types"], res, R=4, cap=16, eps=case["eps"], every=case["every"])
            for i, st in enumerate(steps[:upto]):
                at, v = st["add"]
                t = base + at * SEC
                ts, vs, n, _ = _point_major([[(t, v, 0)] if j == i else [] for j in range(len(steps))])
                assert int(src.add(ts, vs, n)[1].abs().sum()) == 0
                doff, dmem = _dev([0, 1], [i])
                sst, gst = src.forward_timer(window_start(t, res) + res, doff, dmem, grp)
                assert int(sst[i]) == 0 and int(gst[0]) == 0
            st = steps[upto - 1]
            if "want" not in st:
                continue
            ws = base + st["window_s"] * SEC
            slot = int((grp.win["start"][:, 0] == ws).nonzero()[0, 0])
            assert int(grp.win["count"][slot, 0]) == st["want"]["count"]
            assert math.isclose(float(grp.win["sum"][slot, 0]), st["want"]["sum"], rel_tol=1e-10)
            if "sum_sq" in st["want"]:
                assert math.isclose(float(grp.win["sum_sq"][slot, 0]), st["want"]["sum_sq"], rel_tol=1e-10)
            if "q0.5" in st["want"]:
                assert int(grp.consume(ws + res)[0]) == 0
                rows = _decoded_rows(codec, grp)
                p50 = rows[case["types"].index(capi.AGG_P50)]
                assert np.array([p50[-1][1]], dtype=np.uint64).view(np.float64)[0] == st["want"]["q0.5"]
    for case in g["pipeline"]:
        res = case["resolution_s"] * SEC
        base = 1_600_000_000 * SEC
        src = _set_at(codec, 1, [case["src_type"]], res, case["pre_ops"], case["discard_nan"], R=4, cap=8, stride=0)
        grp = _set_at(codec, 1, case["rollup_types"], res, R=4, cap=8)
        rows = [(base + ws * SEC, x, 0) for ws, xs in case["windows"] for x in xs]
        ts, vs, n, _ = _point_major([rows])
        assert int(src.add(ts, vs, n)[1].abs().sum()) == 0
        doff, dmem = _dev([0, 1], [0])
        want = []
        for c in case["consumes"]:
            sst, gst = src.forward_timer(base + c["target_s"] * SEC, doff, dmem, grp)
            assert int(sst[0]) == 0 and int(gst[0]) == 0
            want += c["want"]
        assert int(grp.consume(base + 10_000 * SEC)[0]) == 0
        got = _decoded_rows(codec, grp)[0]
        assert [t for t, _ in got] == [base + t * SEC for t, _ in want]
        for (_, gv), (_, wv) in zip(got, want):
            x = np.array([gv], dtype=np.uint64).view(np.float64)[0]
            assert math.isnan(x) if wv == "NaN" else x == wv


def _stop_case(codec, R, cap):
    """4 sources, each a sample in two windows, into one group of R open windows and `cap` samples"""
    types = [capi.AGG_MAX, capi.AGG_P50, capi.AGG_P99]
    src = _source_set(codec, 4, capi.AGG_P99, R=4, cap=16)
    grp = _timer_set(codec, 1, types, R=R, cap=cap)
    cols = [[(START + SEC * (s + 1), float(s), 0), (START + RES + SEC, float(-s), 0)] for s in range(4)]
    ts, vs, n, _ = _point_major(cols)
    assert int(src.add(ts, vs, n)[1].abs().sum()) == 0
    return src, grp


@pytest.mark.parametrize("stop", ["open_windows", "sample_capacity"])
def test_capacity_stop_then_grow_and_retry(codecs, stop):
    codec = codecs[True]
    doff, dmem = _dev([0, 4], [0, 1, 2, 3])
    big_src, big = _stop_case(codec, 4, 64)
    sst, gst = big_src.forward_timer(START + 2 * RES, doff, dmem, big)
    assert int(sst.abs().sum()) == 0 and int(gst[0]) == 0
    src, grp = _stop_case(codec, 1, 64) if stop == "open_windows" else _stop_case(codec, 4, 3)
    before = src.state()
    sst, gst = src.forward_timer(START + 2 * RES, doff, dmem, grp)
    assert sst.cpu().tolist() == [capi.ERR_CAPACITY] * 4 and gst.cpu().tolist() == [capi.ERR_CAPACITY]
    assert int(grp.win["count"].abs().sum()) == 0
    after = src.state()
    for f in ("start", "count", "sum", "sum_sq"):
        assert torch.equal(before["win"][f], after["win"][f])
    assert torch.equal(before["watermark"], after["watermark"]) and torch.equal(before["elem"], after["elem"])
    grp.grow(open_windows=4, sample_capacity=64)
    sst, gst = src.forward_timer(START + 2 * RES, doff, dmem, grp)
    assert int(sst.abs().sum()) == 0 and int(gst[0]) == 0
    assert int(big.consume(START + 2 * RES)[0]) == 0 and int(grp.consume(START + 2 * RES)[0]) == 0
    assert _decoded_rows(codec, grp) == _decoded_rows(codec, big)
    assert torch.equal(src.watermark, big_src.watermark)


def test_host_checks_and_refusals(codecs):
    codec = codecs[True]
    lib = capi.lib()
    ctx, opts = codec.ctx.handle, C.byref(codec.opts)
    src = _source_set(codec, 4, capi.AGG_P99, cap=8)
    grp = _timer_set(codec, 2, [capi.AGG_MAX, capi.AGG_P50], cap=8)
    doff, dmem = _dev([0, 2, 4], [0, 1, 2, 3])
    sst = torch.zeros(4, dtype=torch.int32, device=DEV)
    gst = torch.zeros(2, dtype=torch.int32, device=DEV)
    P = lambda t: C.c_void_p(t.data_ptr())

    def call(d=None, sd=None, gd=None, gsd=None, off=None, mem=None, n_members=4, n_groups=2, s_st=None, g_st=None):
        sd = src._streams() if sd is None else sd
        gsd = grp._streams() if gsd is None else gsd
        return lib.m3tsz_element_set_forward_timer(
            ctx, opts, C.byref(d or src._desc()), None if sd is False else C.byref(sd), START,
            off if off is not None else P(doff), mem if mem is not None else P(dmem), n_members, n_groups,
            C.byref(gd or grp._desc()), None if gsd is False else C.byref(gsd), s_st if s_st is not None else P(sst),
            g_st if g_st is not None else P(gst), None)

    assert call() == capi.OK
    torch.cuda.synchronize()
    bad = capi.ERR_INVALID_ARG
    assert call(sd=False) == bad and call(gsd=False) == bad
    for es in (src, grp):
        streams = es._streams()
        for field, value in (("sample_capacity", 0), ("eps", 0.0), ("eps", float("nan")),
                             ("insert_and_compress_every", 0), ("reserved", 1), ("d_value", streams.d_value + 4),
                             ("d_header", None)):
            x = capi.ElementTimerStreams.from_buffer_copy(streams)
            setattr(x, field, value)
            assert (call(sd=x) if es is src else call(gsd=x)) == bad, field
    # not Timer sets, a source of two types, a resolution or group-count mismatch
    gauge = codec.element_set(torch.full((4,), START, dtype=torch.int64, device=DEV), capi.METRIC_GAUGE,
                              [capi.AGG_MAX], RES, stride=0)
    assert call(d=gauge._desc()) == bad and call(gd=gauge._desc()) == bad
    two = _timer_set(codec, 4, [capi.AGG_MAX, capi.AGG_P99], cap=8, stride=0)
    assert call(d=two._desc(), sd=two._streams()) == bad
    x = capi.ElementSet.from_buffer_copy(grp._desc())
    x.resolution_ns = 2 * RES
    assert call(gd=x) == bad
    assert call(n_groups=3) == bad
    # shared slots or streams
    assert call(gd=src._desc(), gsd=src._streams(), n_groups=4) == bad
    assert call(gsd=src._streams()) == bad
    # group arrays and statuses
    assert call(off=C.c_void_p(doff.data_ptr() + 4)) == bad and call(mem=C.c_void_p(0)) == bad
    assert call(s_st=C.c_void_p(0)) == bad and call(g_st=C.c_void_p(gst.data_ptr() + 2)) == bad
    assert call(n_members=(1 << 40) + 1) == bad
    # the other forward calls keep refusing Timer sets, and forward_timer the other sets
    assert lib.m3tsz_element_set_forward(ctx, opts, C.byref(src._desc()), START, P(doff), P(dmem), 4, 2,
                                         C.byref(grp._desc()), P(sst), P(gst), None) == bad
    with pytest.raises(ValueError):
        src.forward(START, doff, dmem, grp)
    with pytest.raises(ValueError):
        gauge.forward_timer(START, doff, dmem, grp)


def test_large_set_sampled(codecs):
    codec = codecs[True]
    types = [capi.AGG_MAX, capi.AGG_P50, capi.AGG_P99]
    S, G, P = 100_000, 1_000, 6
    gen = torch.Generator(device="cpu").manual_seed(5)
    ts = (START + torch.arange(P) * 10 * SEC).view(P, 1).expand(P, S).contiguous()
    vs = torch.round(torch.rand((P, S), generator=gen, dtype=torch.float64) * 10000) / 10
    rng = np.random.default_rng(2)
    off = np.arange(G + 1, dtype=np.int64) * (S // G)
    mem = rng.permutation(S).astype(np.int32)
    src = _source_set(codec, S, capi.AGG_P99, R=2, cap=8)
    grp = _timer_set(codec, G, types, R=2, cap=128)
    assert int(src.add(ts.to(DEV), vs.to(DEV))[1].abs().sum()) == 0
    doff, dmem = _dev(off, mem)
    sst, gst = src.forward_timer(START + RES, doff, dmem, grp)
    assert int(sst.abs().sum()) == 0 and int(gst.abs().sum()) == 0
    assert int(grp.consume(START + RES).abs().sum()) == 0
    rows = _decoded_rows(codec, grp)
    got, want = [], []
    for g in np.random.default_rng(3).choice(G, 40, replace=False).tolist():
        gm = TimerGroupModel(types, RES, open_windows=2, sample_capacity=128)
        sms = []
        for s in mem[off[g]: off[g + 1]].tolist():
            m = TimerSourceModel(capi.AGG_P99, RES, open_windows=2, sample_capacity=8)
            m.add([(int(ts[i, s]), float(vs[i, s])) for i in range(P)])
            sms.append(m)
        forward(sms, [gm], START + RES, [0, len(sms)], list(range(len(sms))))
        for j, (t, v) in enumerate(gm.consume(START + RES)):
            want.append(list(zip(t.tolist(), np.asarray(v).view(np.uint64).tolist())))
            got.append(rows[j * G + g])
    assert got == _encoded(codec, want)


def test_on_a_non_blocking_stream_behind_a_sleep(codecs):
    codec = codecs[True]
    types = [capi.AGG_MAX, capi.AGG_P50, capi.AGG_P99]
    S, G = 64, 8
    rng = np.random.default_rng(9)
    off, mem = _groups("random", S, G, rng)
    doff, dmem = _dev(off, mem)
    cols = [_random_rows(rng, 2, batchy=True) for _ in range(S)]
    ts, vs, n, bt = _point_major(cols)

    def run():
        src = _source_set(codec, S, capi.AGG_P99, R=3, cap=256)
        grp = _timer_set(codec, G, types, R=3, cap=1024)
        src.add(ts, vs, n, batch=bt)
        src.forward_timer(START + 2 * RES, doff, dmem, grp)
        grp.consume(START + 2 * RES)
        return grp

    want = _decoded_rows(codec, run())
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(20_000_000)
        grp = run()
    s.synchronize()
    torch.cuda.synchronize()
    assert _decoded_rows(codec, grp) == want
