"""Element sets through a rollup on the GPU (m3tsz_element_set_forward, DESIGN.md §4.12), in both int_optimized modes:
datapoints added to a source set over several calls, forwarded into a group set and consumed at flush ticks give
byte for byte the rows, and the records, of m3tsz_aggregate_tiles_rollup over streams of the same datapoints; a
CAPACITY stop and a retry of the failed groups; closed group windows; NaN cases and the group side's discard rule
against the CPU model (tests/element_rollup_model.py); argument checks; and 100 k sources sampled against the model."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import agg_oracle_lib as A
import oracle_lib as O
from element_rollup_model import ERR_CAPACITY, ERR_CLOSED, ERR_INVALID_ARG, OK, GroupModel, SourceModel, forward
from m3_b200 import capi
from test_element_set_model import _bits
from test_gpu_elements import _decoded_rows, _point_major, _rows

pytestmark = pytest.mark.gpu

SEC = 1_000_000_000
RES = 60 * SEC
START = 1_600_000_020 * SEC  # a whole minute
DEV = "cuda"
GAUGE, COUNTER = A.METRIC_GAUGE, A.METRIC_COUNTER
LAST, MIN, MAX, SUM = 1, 2, 3, 7
# (metric, source type, pre-ops, rollup types, post-ops): Counter Sum + [Increase] -> Rollup [Sum] -> [Add], and
# Gauge Last -> Rollup [Min, Max, Sum]
PIPES = [(COUNTER, SUM, [3], [SUM], [4]), (GAUGE, LAST, [], [MIN, MAX, SUM], [])]


@pytest.fixture(scope="module")
def codecs():
    from m3_b200.codec import BatchCodec
    return {True: BatchCodec(0, int_optimized=True), False: BatchCodec(0, int_optimized=False)}


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def finite_series(rng, n_windows, metric):
    """[(t, value bits)]: windows in order, datapoints out of order inside each, finite values"""
    pts = []
    for w in range(n_windows):
        if rng.random() < 0.25:
            continue
        for o in rng.integers(0, RES // SEC, int(rng.integers(1, 5))):
            v = float(rng.integers(0, 1000)) if metric == COUNTER else float(rng.normal() * 100)
            pts.append((START + w * RES + int(o) * SEC, _bits(v)))
    return pts


def memberships(rng, S, G, kind):
    if kind == "contiguous":
        off = np.linspace(0, S, G + 1).astype(np.int64)
        return off, np.arange(S, dtype=np.int32)
    n = G * 4
    return np.arange(0, n + 1, 4, dtype=np.int64), rng.integers(0, S, n).astype(np.int32)


def sets(codec, S, G, pipe, discard, R=8, src_R=8):
    metric, src_type, pre, types, post = pipe
    zeros = lambda n: torch.full((n,), START, dtype=torch.int64, device=DEV)
    src = codec.element_set(zeros(S), metric, [src_type], RES, transforms=pre, discard_nan=discard,
                            open_windows=src_R, stride=0)
    grp = codec.element_set(zeros(G), metric, types, RES, transforms=post, discard_nan=discard, open_windows=R)
    return src, grp


def tile_rollup(codec, cols, pipe, discard, off, mem, n_windows):
    """aggregate_tiles_rollup over streams of the same datapoints -> (bytes per row, source records, group records)"""
    metric, src_type, pre, types, post = pipe
    S, G = len(cols), len(off) - 1
    P = max([len(c) for c in cols] + [1])
    ts = np.zeros((S, P), dtype=np.int64)
    vb = np.zeros((S, P), dtype=np.uint64)
    for s, c in enumerate(cols):
        for i, (t, v) in enumerate(c):
            ts[s, i], vb[s, i] = t, v
    n = torch.tensor([len(c) for c in cols], dtype=torch.int32, device=DEV)
    enc = codec.encode(_dev(ts), _dev(vb.view(np.float64)), torch.full((S,), START, dtype=torch.int64, device=DEV),
                       n_points=n)
    assert int(enc.status.abs().sum()) == 0
    offs = torch.arange(S, dtype=torch.int64, device=DEV) * enc.out.shape[1]
    xs, gs = codec.transform_state(S), codec.element_state(G)
    out, _, sst = codec.aggregate_tiles_rollup(enc.out.view(-1), offs, START, RES, n_windows, src_type, _dev(off),
                                               _dev(mem), types, metric_type=metric, pre_transforms=pre,
                                               post_transforms=post, discard_nan=discard, src_state=xs,
                                               group_state=gs, lengths=enc.out_len)
    assert int(out.status.abs().sum()) == 0 and int(sst.abs().sum()) == 0
    packed = out.packed.cpu().numpy()
    o, ln = out.offsets.reshape(-1).cpu().numpy(), out.out_len.reshape(-1).cpu().numpy()
    return [packed[o[r]: o[r] + ln[r]].tobytes() for r in range(len(ln))], xs, gs


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("pipe", range(len(PIPES)))
@pytest.mark.parametrize("kind", ["contiguous", "random"])
@pytest.mark.parametrize("n_calls", [1, 2, 5, 17])
def test_equals_aggregate_tiles_rollup(codecs, int_opt, pipe, kind, n_calls):
    codec = codecs[int_opt]
    rng = np.random.default_rng(1000 * pipe + 10 * n_calls + int_opt + (kind == "random") * 7)
    S, G, W = 60, 9, 8
    metric = PIPES[pipe][0]
    cols = [finite_series(rng, W, metric) for _ in range(S)]
    off, mem = memberships(rng, S, G, kind)
    discard = bool(n_calls % 2)
    src, grp = sets(codec, S, G, PIPES[pipe], discard)
    cuts = [np.sort(rng.integers(0, len(c) + 1, n_calls - 1)).tolist() for c in cols]
    d_off, d_mem = _dev(off), _dev(mem)
    for call in range(n_calls):
        parts = [c[([0] + cuts[s] + [len(c)])[call]: ([0] + cuts[s] + [len(c)])[call + 1]] for s, c in enumerate(cols)]
        res, st = src.add(*_point_major(parts))
        assert int(st.abs().sum()) == 0 and int(res.abs().sum()) == 0
        # a flush tick that closes no window a later datapoint falls in
        pending = [c[([0] + cuts[s] + [len(c)])[call + 1]:] for s, c in enumerate(cols)]
        firsts = [p[0][0] - (p[0][0] - START) % RES for p in pending if p]
        if call + 1 < n_calls and firsts:
            sst, gst = src.forward(min(firsts), d_off, d_mem, grp)
            assert int(sst.abs().sum()) == 0 and int(gst.abs().sum()) == 0
            assert int(grp.consume(min(firsts)).abs().sum()) == 0
    sst, gst = src.forward(START + W * RES, d_off, d_mem, grp)
    assert int(sst.abs().sum()) == 0 and int(gst.abs().sum()) == 0
    assert int(grp.consume(START + W * RES).abs().sum()) == 0
    want, xs, gs = tile_rollup(codec, cols, PIPES[pipe], discard, off, mem, W)
    assert _rows(grp) == want
    assert torch.equal(grp.elem, gs)
    assert torch.equal(src.elem[:, :96], xs)


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("pipe", range(len(PIPES)))
def test_capacity_stop_and_retry_of_the_failed_groups(codecs, int_opt, pipe):
    """groups with too few open windows fold nothing and hold their members back; growing and forwarding again with
    only the failed groups listed (the others' ranges empty) gives the unstopped bytes and records"""
    codec = codecs[int_opt]
    rng = np.random.default_rng(77 + pipe + int_opt)
    S, G, W = 48, 8, 5
    metric = PIPES[pipe][0]
    cols = [finite_series(rng, W, metric) for _ in range(S)]
    off, mem = memberships(rng, S, G, "random")
    src, grp = sets(codec, S, G, PIPES[pipe], False, R=2)
    res, st = src.add(*_point_major(cols))
    assert int(st.abs().sum()) == 0
    sst, gst = src.forward(START + W * RES, _dev(off), _dev(mem), grp)
    gst, sst = gst.cpu().numpy(), sst.cpu().numpy()
    failed = [g for g in range(G) if gst[g] != OK]
    assert failed and set(gst.tolist()) <= {OK, ERR_CAPACITY}
    held = {int(m) for g in failed for m in mem[off[g]: off[g + 1]]}
    assert {s for s in range(S) if sst[s] != OK} == held and set(sst[list(held)].tolist()) == {ERR_CAPACITY}
    grp.grow(open_windows=W)
    lens = np.array([off[g + 1] - off[g] if g in failed else 0 for g in range(G)])
    off2 = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    mem2 = np.concatenate([mem[off[g]: off[g + 1]] for g in failed]).astype(np.int32)
    sst, gst = src.forward(START + W * RES, _dev(off2), _dev(mem2), grp)
    assert int(sst.abs().sum()) == 0 and int(gst.abs().sum()) == 0
    assert int(grp.consume(START + W * RES).abs().sum()) == 0
    want, xs, gs = tile_rollup(codec, cols, PIPES[pipe], False, off, mem, W)
    assert _rows(grp) == want
    assert torch.equal(grp.elem, gs) and torch.equal(src.elem[:, :96], xs)


def _models(pipe, S, G, discard, R=8):
    metric, src_type, pre, types, post = pipe
    return ([SourceModel(metric, src_type, RES, pre, discard, open_windows=R) for _ in range(S)],
            [GroupModel(metric, types, RES, post, discard, open_windows=R) for _ in range(G)])


def _noisy_series(rng, n_windows, metric):
    pts = []
    for w in range(n_windows):
        for o in rng.integers(0, RES // SEC, int(rng.integers(0, 4))):
            if metric == COUNTER:
                v = float(rng.choice([rng.integers(-1000, 1000), np.nan, 9.1e18]))
            else:
                v = float(rng.choice([rng.normal() * 100, np.nan, np.inf, -np.inf, 0.0, -0.0]))
            pts.append((START + w * RES + int(o) * SEC, _bits(v)))
    return pts


@pytest.mark.parametrize("pipe", [PIPES[0], PIPES[1], (GAUGE, LAST, [1, 2], [LAST, SUM], [5])])
@pytest.mark.parametrize("discard", [False, True])
def test_nan_cases_and_closed_windows_against_the_model(codecs, pipe, discard):
    """NaN / +-Inf values, a lagging source whose late window reaches a consumed group window (AGGREGATION_CLOSED),
    sources in several groups or in none, every group's rows, source records and statuses against the model"""
    codec = codecs[True]
    rng = np.random.default_rng(5 + discard)
    S, G, W = 40, 7, 6
    metric = pipe[0]
    src, grp = sets(codec, S, G, pipe, discard)
    sms, gms = _models(pipe, S, G, discard)
    off = np.array([0, 3, 3, 9, 12, 20, 22, 30], dtype=np.int64)
    mem = rng.integers(0, S - 4, 30).astype(np.int32)  # the last four sources are in no group
    want_rows = [[[] for _ in pipe[3]] for _ in range(G)]
    for tick in range(W):
        cols = [[p for p in _noisy_series(rng, W, metric) if p[0] < START + (tick + 1) * RES
                 and (s % 5 != 0 or p[0] >= START + (tick - 1) * RES)] if rng.random() < 0.7 else []
                for s in range(S)]
        res, st = src.add(*_point_major(cols))
        for s, m in enumerate(sms):
            wr, ws_ = m.add(cols[s])
            assert res[: len(cols[s]), s].cpu().tolist() == wr and int(st[s]) == ws_
        target = START + tick * RES
        sst, gst = src.forward(target, _dev(off), _dev(mem), grp)
        wst, wgst = forward(sms, gms, target, off, mem)
        assert sst.cpu().tolist() == wst and gst.cpu().tolist() == wgst
        assert int(grp.consume(target).abs().sum()) == 0
        for g, m in enumerate(gms):
            for j, (t, v) in enumerate(m.consume(target)):
                want_rows[g][j] += list(zip(t.tolist(), v.view(np.uint64).tolist()))
    rows = _rows(grp)  # (bytes: the int-optimised encoding writes -0.0 as 0)
    for g in range(G):
        for j in range(len(pipe[3])):
            t = np.array([x for x, _ in want_rows[g][j]], dtype=np.int64)
            v = np.array([x for _, x in want_rows[g][j]], dtype=np.uint64).view(np.float64)
            assert rows[j * G + g] == (O.encode_series(t, v, START, O.UNIT_S, True) if len(t) else b""), (g, j)
    for s, m in enumerate(sms):
        assert src.elem[s].cpu().numpy().tobytes() == m.state.tobytes()
        assert int(src.watermark[s]) == m.watermark


def test_group_side_discard_writes_a_nan_rollup_value(codecs):
    """discard_nan, no post-ops, +Inf + -Inf in a Sum: the group set writes the NaN (the element set's rule: discard
    only with ops), where aggregate_tiles_rollup drops it"""
    codec = codecs[True]
    pipe = (GAUGE, LAST, [], [SUM], [])
    src, grp = sets(codec, 2, 1, pipe, True)
    src.add(*_point_major([[(START, _bits(math.inf))], [(START, _bits(-math.inf))]]))
    sst, gst = src.forward(START + RES, _dev(np.array([0, 2])), _dev(np.array([0, 1], dtype=np.int32)), grp)
    assert int(sst.abs().sum()) == 0 and int(gst.abs().sum()) == 0
    assert int(grp.consume(START + RES).abs().sum()) == 0
    (row,) = _decoded_rows(codec, grp)
    assert len(row) == 1 and row[0][0] == START + RES and math.isnan(np.array([row[0][1]]).view(np.float64)[0])
    cols = [[(START, _bits(math.inf))], [(START, _bits(-math.inf))]]
    want, _, _ = tile_rollup(codec, cols, pipe, True, np.array([0, 2]), np.array([0, 1], dtype=np.int32), 1)
    assert want == [b""]


def test_argument_checks(codecs):
    codec = codecs[True]
    zeros = lambda n: torch.full((n,), START, dtype=torch.int64, device=DEV)
    src = codec.element_set(zeros(4), COUNTER, [SUM], RES, stride=0)
    off, mem = _dev(np.array([0, 2, 4])), _dev(np.array([0, 1, 2, 3], dtype=np.int32))
    ok = codec.element_set(zeros(2), COUNTER, [SUM], RES)
    assert int(src.forward(START, off, mem, ok)[0].abs().sum()) == 0
    bad = [codec.element_set(zeros(2), GAUGE, [SUM], RES),             # metric type
           codec.element_set(zeros(2), COUNTER, [SUM], 2 * RES),       # resolution
           codec.element_set(zeros(3), COUNTER, [SUM], RES)]           # n_groups
    for g in bad:
        with pytest.raises(capi.M3tszError):
            src.forward(START, off, mem, g)
    two = codec.element_set(zeros(4), COUNTER, [MIN, SUM], RES, stride=0)  # two source types
    with pytest.raises(capi.M3tszError):
        two.forward(START, off, mem, ok)
    with pytest.raises(capi.M3tszError):  # a set forwarding into itself
        src.forward(START, _dev(np.array([0, 0, 0, 0, 0])), mem, src)
    # the output-less set: consume and stream refuse it, and so does the C call
    with pytest.raises(ValueError):
        src.consume(START)
    with pytest.raises(ValueError):
        src.stream()
    d = src._desc()
    st = torch.zeros(4, dtype=torch.int32, device=DEV)
    rc = capi.lib().m3tsz_element_set_consume(codec.ctx.handle, C.byref(codec.opts), C.byref(d), START, capi.UNIT_S,
                                              st.data_ptr(), None)
    assert rc == capi.ERR_INVALID_ARG
    # NULL members with members counted
    gd = ok._desc()
    rc = capi.lib().m3tsz_element_set_forward(codec.ctx.handle, C.byref(codec.opts), C.byref(d), START, off.data_ptr(),
                                              None, 4, 2, C.byref(gd), st.data_ptr(), st.data_ptr(), None)
    assert rc == capi.ERR_INVALID_ARG


def test_invalid_groups_on_the_device(codecs):
    codec = codecs[True]
    pipe = PIPES[1]
    S, G = 3, 3
    src, grp = sets(codec, S, G, pipe, False)
    sms, gms = _models(pipe, S, G, False)
    cols = [[(START, _bits(1.0))]] * S
    src.add(*_point_major(cols))
    for s, m in enumerate(sms):
        m.add(cols[s])
    off, mem = np.array([0, 2, 1, 4], dtype=np.int64), np.array([7, 0, 1, 1], dtype=np.int32)
    sst, gst = src.forward(START + RES, _dev(off), _dev(mem), grp)
    wst, wgst = forward(sms, gms, START + RES, off, mem)
    assert gst.cpu().tolist() == wgst == [ERR_INVALID_ARG, ERR_INVALID_ARG, OK]
    assert sst.cpu().tolist() == wst


def test_large_set_sampled(codecs):
    """100 k sources, 10 k groups of 10 random members; sampled groups' rows and their members' records against the
    model"""
    codec = codecs[True]
    pipe = PIPES[0]
    rng = np.random.default_rng(21)
    S, G, W = 100_000, 10_000, 3
    off = np.arange(0, G * 10 + 1, 10, dtype=np.int64)
    mem = rng.integers(0, S, G * 10).astype(np.int32)
    src, grp = sets(codec, S, G, pipe, True, R=4, src_R=4)
    n = rng.integers(0, 4, (W, S))
    ts = np.zeros((int(n.sum(0).max()), S), dtype=np.int64)
    vals = np.zeros(ts.shape, dtype=np.float64)
    counts = np.zeros(S, dtype=np.int32)
    cols = [[] for _ in range(S)]
    sample = sorted(rng.choice(G, 40, replace=False).tolist())
    srcs = sorted({int(m) for g in sample for m in mem[off[g]: off[g + 1]]})
    in_sample = set(srcs)
    for w in range(W):
        for s in range(S):
            for _ in range(n[w, s]):
                t = START + w * RES + int(rng.integers(0, 60)) * SEC
                v = float(rng.integers(0, 1000))
                ts[counts[s], s], vals[counts[s], s] = t, v
                counts[s] += 1
                if s in in_sample:
                    cols[s].append((t, _bits(v)))
    res, st = src.add(_dev(ts), _dev(vals), _dev(counts))
    assert int(st.abs().sum()) == 0
    sst, gst = src.forward(START + W * RES, _dev(off), _dev(mem), grp)
    assert int(sst.abs().sum()) == 0 and int(gst.abs().sum()) == 0
    assert int(grp.consume(START + W * RES).abs().sum()) == 0
    rows = _decoded_rows(codec, grp, cap=16)
    sms = {s: SourceModel(COUNTER, SUM, RES, pipe[2], True, open_windows=4) for s in srcs}
    for s in srcs:
        sms[s].add(cols[s])
    for g in sample:
        gm = GroupModel(COUNTER, pipe[3], RES, pipe[4], True, open_windows=4)
        members = [int(m) for m in mem[off[g]: off[g + 1]]]
        # the group's fold over its members' pending windows (the sources commit after every group folded)
        pend = {m: sms[m].pending(START + W * RES)[0] for m in set(members)}
        for m in members:
            for ws, v, fwd in pend[m]:
                if fwd:
                    gm.add_unique(ws, v)
        (t, v), = gm.consume(START + W * RES)
        assert rows[g] == list(zip(t.tolist(), v.view(np.uint64).tolist())), g
    for s in srcs:
        _, rec = sms[s].pending(START + W * RES)
        assert src.elem[s].cpu().numpy().tobytes() == rec.tobytes()
