"""Tile aggregation through a rollup on the GPU (m3tsz_aggregate_tiles_rollup: the fused decode, the forward stage, the
fold and the multi-type element stage over the groups): bytes, out_len, n_tiles, row and source statuses and both
kinds of record against the composed oracle (rollup_oracle_lib), in both int_optimized modes and both stream
addressings; source blocks; listed order; bad groups; re-runs, CAPACITY and split calls; argument checks; and the
equivalence with aggregate_tiles_types for one-member groups."""
import math

import numpy as np
import pytest
import torch

import agg_oracle_lib as A
import elem_oracle_lib as E
import oracle_lib as O
import rollup_oracle_lib as R
import xf_oracle_lib as X
from m3_b200 import capi
from test_gpu_transforms import N_WIN, R0, START, WIN, _batch, _csr, _padded, codecs  # noqa: F401
from test_tile_blocks_oracle import random_series

pytestmark = pytest.mark.gpu

AB, PS, INC, ADD, RST = 1, 2, 3, 4, 5
LAST, MIN, MAX, MEAN, COUNT, SUM, SUMSQ, STDEV = 1, 2, 3, 4, 6, 7, 8, 9
GAUGE, COUNTER = A.METRIC_GAUGE, A.METRIC_COUNTER
GAUGE_ALL = [1, 2, 3, 4, 6, 7, 8, 9]
COUNTER_ALL = [2, 3, 4, 6, 7, 8, 9]
ERR_INVALID_ARG, ERR_CAPACITY = capi.ERR_INVALID_ARG, capi.ERR_CAPACITY

# (metric, source type, pre-ops, rollup types, post-ops)
PIPELINES = [
    (COUNTER, SUM, [INC], [SUM], [ADD]),  # the documented Prometheus counter rollup
    (GAUGE, LAST, [], [MIN, MAX, SUM], []),
    (GAUGE, LAST, [AB, PS], GAUGE_ALL, [ADD]),
    (COUNTER, SUM, [PS], COUNTER_ALL, [ADD, RST]),
    (GAUGE, MAX, [RST], [LAST, MEAN, COUNT], [INC]),
    (COUNTER, MAX, [], [MIN, MAX, SUMSQ, STDEV], [RST]),
    (GAUGE, STDEV, [ADD], [LAST, SUMSQ], [AB, ADD]),
]


def membership(rng, S, G, max_len=7, spare=8):
    """random groups over sources 0 .. S - spare - 1 (the last `spare` sources are in no group): empty groups,
    duplicates, sources in several groups"""
    lists = [list(rng.integers(0, S - spare, int(rng.integers(0, max_len + 1)))) for _ in range(G)]
    lists[0] = []
    lists[1] = [3, 3, 5]
    off = np.zeros(G + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(x) for x in lists])
    return off, np.array([m for x in lists for m in x], dtype=np.int32)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


class Expect:
    def __init__(self, decoded, int_opt, G):
        self.decoded, self.int_opt = decoded, int_opt
        self.src_state = np.zeros(len(decoded), dtype=X.XF_STATE_DTYPE)
        self.group_state = np.zeros(G, dtype=E.ELEM_STATE_DTYPE)

    def call(self, r0, n_win, pipe, off, mem, discard, saved_rows=None):
        metric, src, pre, types, post = pipe
        return R.aggregate_tiles_rollup(self.decoded, self.int_opt, r0, WIN, n_win, metric, src, pre, off, mem, types,
                                        post, discard, self.src_state, self.group_state, saved_rows)


def run(codec, inputs, r0, n_win, pipe, off, mem, discard, src_state, group_state, capacity=None):
    blob, o, lengths, blocks = inputs
    metric, src, pre, types, post = pipe
    return codec.aggregate_tiles_rollup(blob, o, r0, WIN, n_win, src, dev(off), dev(mem), types, metric_type=metric,
                                        pre_transforms=pre, post_transforms=post, discard_nan=discard,
                                        src_state=src_state, group_state=group_state, lengths=lengths, blocks=blocks,
                                        capacity=capacity)


def layout(streams, addressing):
    blob, o, lengths = _csr(streams) if addressing == "csr" else _padded(streams)
    return blob, o, lengths, None


def block_layout(series):
    segs = [b for blocks in series for b in blocks]
    blob, o, lengths = _padded(segs)
    bo = np.zeros(len(series) + 1, dtype=np.int64)
    bo[1:] = np.cumsum([len(b) for b in series])
    return blob, o, lengths, dev(bo)


def check(res, exp_rows, exp_src, only=None):
    r, nt, sst = res
    st, ln, of = r.status.cpu().numpy(), r.out_len.cpu().numpy(), r.offsets.cpu().numpy()
    packed, nt = r.packed.cpu().numpy(), nt.cpu().numpy()
    for j, row in enumerate(exp_rows):
        for g, (e_st, e_bytes, e_n) in enumerate(row):
            if only is not None and g not in only:
                continue
            assert st[j, g] == e_st, (j, g, st[j, g], e_st)
            if e_st:
                assert ln[j, g] == 0 and nt[j, g] == 0, (j, g)
                continue
            assert nt[j, g] == e_n, (j, g, nt[j, g], e_n)
            assert ln[j, g] == len(e_bytes) and packed[of[j, g]: of[j, g] + ln[j, g]].tobytes() == e_bytes, (j, g)
    if exp_src is not None:
        assert sst.cpu().numpy().tolist() == list(exp_src)


def check_states(exp, src_state, group_state):
    s = src_state.cpu().numpy().copy().view(X.XF_STATE_DTYPE).reshape(-1)
    g = group_state.cpu().numpy().copy().view(E.ELEM_STATE_DTYPE).reshape(-1)
    assert s.tobytes() == exp.src_state.tobytes()
    assert g.tobytes() == exp.group_state.tobytes()


@pytest.mark.parametrize("discard", [True, False])
@pytest.mark.parametrize("addressing", ["csr", "lengths"])
@pytest.mark.parametrize("int_opt", [True, False])
def test_rollup_against_oracle(codecs, int_opt, addressing, discard):
    codec = codecs[int_opt]
    streams = _batch(int_opt, S=70, both_inf=not discard)
    S, G = len(streams), 41
    decoded = R.decode_sources(streams, int_opt, blocks=False)
    inputs = layout(streams, addressing)
    rng = np.random.default_rng(3)
    for pipe in PIPELINES:
        off, mem = membership(rng, S, G)
        exp = Expect(decoded, int_opt, G)
        xs, gs = codec.transform_state(S), codec.element_state(G)
        for r0, n_win in ((R0, 5), (R0 + 5 * WIN, N_WIN - 5)):  # two calls: the records carry over
            res = run(codec, inputs, r0, n_win, pipe, off, mem, discard, xs, gs)
            rows, src = exp.call(r0, n_win, pipe, off, mem, discard)
            torch.cuda.synchronize()
            check(res, rows, src)
            check_states(exp, xs, gs)


@pytest.mark.parametrize("int_opt", [True, False])
def test_blocks(codecs, int_opt):
    codec = codecs[int_opt]
    # NULL blocks against one block per series: the same outputs
    streams = _batch(int_opt, S=40, damage=False)
    off, mem = membership(np.random.default_rng(8), 40, 23)
    pipe = PIPELINES[2]
    a = run(codec, layout(streams, "lengths"), R0, N_WIN, pipe, off, mem, True, None, None)
    b = run(codec, block_layout([[s] for s in streams]), R0, N_WIN, pipe, off, mem, True, None, None)
    torch.cuda.synchronize()
    for x, y in zip((a[0].status, a[0].out_len, a[1], a[2]), (b[0].status, b[0].out_len, b[1], b[2])):
        assert torch.equal(x, y)
    for j in range(len(pipe[3])):
        for g in range(23):
            ra = a[0].packed[int(a[0].offsets[j, g]): int(a[0].offsets[j, g]) + int(a[0].out_len[j, g])]
            rb = b[0].packed[int(b[0].offsets[j, g]): int(b[0].offsets[j, g]) + int(b[0].out_len[j, g])]
            assert torch.equal(ra, rb), (j, g)
    # 0-12 blocks per series against the composition
    from test_tile_blocks_oracle import N_WIN as BN, R0 as BR0, STEP
    assert STEP == WIN
    rng = np.random.default_rng(21)
    series = [random_series(rng, (0, 1, 2, 5, 12)[i % 5], int_opt, False) for i in range(37)]
    decoded = R.decode_sources(series, int_opt, blocks=True)
    off, mem = membership(rng, 37, 19)
    for pipe in (PIPELINES[0], PIPELINES[4]):
        exp = Expect(decoded, int_opt, 19)
        xs, gs = codec.transform_state(37), codec.element_state(19)
        res = run(codec, block_layout(series), BR0, BN, pipe, off, mem, True, xs, gs)
        rows, src = exp.call(BR0, BN, pipe, off, mem, True)
        torch.cuda.synchronize()
        check(res, rows, src)
        check_states(exp, xs, gs)


def test_listed_order_wins(codecs):
    """three members whose Gauge sum depends on the order: 1e16 + 1 + 1 != 1 + 1 + 1e16"""
    codec = codecs[True]
    vals = [1e16, 1.0, 1.0]
    streams = [O.encode_series(np.array([R0 + 10 * 10 ** 9], dtype=np.int64), np.array([v]), START, O.UNIT_S, True)
               for v in vals]
    off = np.array([0, 3, 6], dtype=np.int64)
    mem = np.array([0, 1, 2, 1, 2, 0], dtype=np.int32)
    pipe = (GAUGE, LAST, [], [SUM], [])
    res = run(codec, layout(streams, "csr"), R0, 2, pipe, off, mem, True, None, None)
    rows, _ = R.aggregate_tiles_rollup(R.decode_sources(streams, True, False), True, R0, WIN, 2, GAUGE, LAST, [], off,
                                       mem, [SUM], [], True, np.zeros(3, X.XF_STATE_DTYPE),
                                       np.zeros(2, E.ELEM_STATE_DTYPE))
    torch.cuda.synchronize()
    check(res, rows, [0, 0, 0])
    assert rows[0][0][1] != rows[0][1][1]  # the two orders write different bits
    assert (1e16 + 1.0) + 1.0 != (1.0 + 1.0) + 1e16


def test_bad_groups_fail_alone(codecs):
    codec = codecs[True]
    streams = _batch(True, S=20, damage=False)
    decoded = R.decode_sources(streams, True, False)
    # g0 ok, g1 decreasing range, g2 index >= S, g3 ok, g4 past n_members
    off = np.array([0, 3, 2, 5, 7, 12], dtype=np.int64)
    mem = np.array([0, 1, 2, 4, 99, 6, 7, 8, 9, 10], dtype=np.int32)
    pipe = PIPELINES[1]
    exp = Expect(decoded, True, 5)
    xs, gs = codec.transform_state(20), codec.element_state(5)
    res = run(codec, layout(streams, "csr"), R0, N_WIN, pipe, off, mem, True, xs, gs)
    rows, src = exp.call(R0, N_WIN, pipe, off, mem, True)
    torch.cuda.synchronize()
    st = res[0].status.cpu().numpy()
    assert (st[:, [1, 2, 4]] == ERR_INVALID_ARG).all() and (st[:, [0, 3]] == 0).all()
    check(res, rows, src)
    check_states(exp, xs, gs)


@pytest.mark.parametrize("int_opt", [True, False])
def test_rerun_of_failed_groups(codecs, int_opt):
    """a truncated member fails every group that lists it; re-running those groups with their members (the stream
    repaired) gives the records and rows of one unstopped call"""
    codec = codecs[int_opt]
    good = _batch(int_opt, S=50, damage=False)
    bad = list(good)
    bad[7] = bad[7][: max(1, len(bad[7]) // 2)]
    off, mem = membership(np.random.default_rng(4), 50, 30)
    mem[2] = 7  # at least one group lists source 7
    pipe = PIPELINES[0]
    unstopped = Expect(R.decode_sources(good, int_opt, False), int_opt, 30)
    want_rows, _ = unstopped.call(R0, N_WIN, pipe, off, mem, True)
    xs, gs = codec.transform_state(50), codec.element_state(30)
    res = run(codec, layout(bad, "csr"), R0, N_WIN, pipe, off, mem, True, xs, gs)
    torch.cuda.synchronize()
    failed = [g for g in range(30) if res[0].status[0, g].item() != 0]
    assert failed and all(7 in mem[off[g]: off[g + 1]].tolist() for g in failed)
    check(res, want_rows, None, only=[g for g in range(30) if g not in failed])
    # the re-run: the failed groups, their members, their records
    srcs = sorted({int(m) for g in failed for m in mem[off[g]: off[g + 1]]})
    idx = {s: i for i, s in enumerate(srcs)}
    sub_mem = np.array([idx[int(m)] for g in failed for m in mem[off[g]: off[g + 1]]], dtype=np.int32)
    sub_off = np.zeros(len(failed) + 1, dtype=np.int64)
    sub_off[1:] = np.cumsum([off[g + 1] - off[g] for g in failed])
    si, gi = torch.tensor(srcs, device="cuda"), torch.tensor(failed, device="cuda")
    sx, sg = xs[si].contiguous(), gs[gi].contiguous()
    res2 = run(codec, layout([good[s] for s in srcs], "csr"), R0, N_WIN, pipe, sub_off, sub_mem, True, sx, sg)
    xs[si], gs[gi] = sx, sg
    torch.cuda.synchronize()
    check(res2, [[row[g] for g in failed] for row in want_rows], None)
    check_states(unstopped, xs, gs)


def test_capacity_then_retry(codecs):
    codec = codecs[True]
    streams = _batch(True, S=60, damage=False)
    decoded = R.decode_sources(streams, True, False)
    off, mem = membership(np.random.default_rng(6), 60, 33)
    pipe = PIPELINES[3]
    exp = Expect(decoded, True, 33)
    xs, gs = codec.transform_state(60), codec.element_state(33)
    res = run(codec, layout(streams, "csr"), R0, N_WIN, pipe, off, mem, True, xs, gs, capacity=3000)
    torch.cuda.synchronize()
    st = res[0].status.cpu().numpy()
    assert (st == ERR_CAPACITY).any() and (st == 0).any()
    saved = lambda g: bool((st[:, g] == 0).all())
    rows, _ = exp.call(R0, N_WIN, pipe, off, mem, True, saved_rows=saved)
    check(res, [[row[g] if saved(g) else (ERR_CAPACITY, b"", 0) for g in range(33)] for row in rows], None,
          only=[g for g in range(33) if saved(g)])
    check_states(exp, xs, gs)
    # the retry of the failed groups with their members, with room, gives the unstopped result
    full = Expect(decoded, True, 33)
    want, _ = full.call(R0, N_WIN, pipe, off, mem, True)
    failed = [g for g in range(33) if not saved(g)]
    srcs = sorted({int(m) for g in failed for m in mem[off[g]: off[g + 1]]})
    idx = {s: i for i, s in enumerate(srcs)}
    sub_mem = np.array([idx[int(m)] for g in failed for m in mem[off[g]: off[g + 1]]], dtype=np.int32)
    sub_off = np.zeros(len(failed) + 1, dtype=np.int64)
    sub_off[1:] = np.cumsum([off[g + 1] - off[g] for g in failed])
    si, gi = torch.tensor(srcs, device="cuda"), torch.tensor(failed, device="cuda")
    sx, sg = xs[si].contiguous(), gs[gi].contiguous()
    res2 = run(codec, layout([streams[s] for s in srcs], "csr"), R0, N_WIN, pipe, sub_off, sub_mem, True, sx, sg)
    xs[si], gs[gi] = sx, sg
    torch.cuda.synchronize()
    check(res2, [[row[g] for g in failed] for row in want], None)
    check_states(full, xs, gs)


@pytest.mark.parametrize("records", [True, False])
@pytest.mark.parametrize("n_calls", [1, 2, 5])
def test_split_calls(codecs, n_calls, records):
    """consecutive calls over a split window range write the datapoints of one call; without records every call
    starts new elements, as the oracle with fresh records does"""
    codec = codecs[True]
    streams = _batch(True, S=45, damage=True)
    decoded = R.decode_sources(streams, True, False)
    off, mem = membership(np.random.default_rng(9), 45, 20)
    pipe = PIPELINES[3]
    edges = np.linspace(0, N_WIN, n_calls + 1).astype(int)
    exp = Expect(decoded, True, 20)
    xs, gs = (codec.transform_state(45), codec.element_state(20)) if records else (None, None)
    for a, b in zip(edges[:-1], edges[1:]):
        if not records:
            exp = Expect(decoded, True, 20)
        res = run(codec, layout(streams, "csr"), R0 + int(a) * WIN, int(b - a), pipe, off, mem, True, xs, gs)
        rows, src = exp.call(R0 + int(a) * WIN, int(b - a), pipe, off, mem, True)
        torch.cuda.synchronize()
        check(res, rows, src)
        if records:
            check_states(exp, xs, gs)


def test_invalid_arguments(codecs):
    codec = codecs[True]
    streams = _batch(True, S=8, damage=False)
    off, mem = np.array([0, 2], dtype=np.int64), np.array([0, 1], dtype=np.int32)
    inputs = layout(streams, "csr")
    bad = [
        (GAUGE, LAST, [], [MAX, MIN], []),              # type order
        (GAUGE, LAST, [], [], []),                      # no types
        (GAUGE, LAST, [], [1, 2, 3, 4, 6, 7, 8, 9, 9], []),  # nine types
        (COUNTER, LAST, [], [SUM], []),                 # a source type invalid for the metric
        (GAUGE, LAST, [PS, INC], [SUM], []),            # two derivatives in one list
        (GAUGE, LAST, [], [SUM], [INC, PS]),
        (COUNTER, SUM, [], [LAST], []),                 # Last for a Counter
        (GAUGE, LAST, [6], [SUM], []),                  # unknown op
    ]
    for pipe in bad:
        with pytest.raises(capi.M3tszError) as e:
            run(codec, inputs, R0, N_WIN, pipe, off, mem, True, None, None)
        assert e.value.status == ERR_INVALID_ARG, pipe


@pytest.mark.parametrize("int_opt", [True, False])
def test_one_member_groups_equal_tiles_types(codecs, int_opt):
    """Last -> Rollup [Last] with one member per group and no pre-ops is the local element of Last.  Without
    discard_nan: with it, the source drops a NaN window that the local element would still run through its ops"""
    codec = codecs[int_opt]
    streams = _batch(int_opt, S=64)
    S = len(streams)
    inputs = layout(streams, "csr")
    off = np.arange(S + 1, dtype=np.int64)
    mem = np.arange(S, dtype=np.int32)[::-1].copy()
    for post in ([], [ADD], [INC, RST]):
        a, na, sa = run(codec, inputs, R0, N_WIN, (GAUGE, LAST, [], [LAST], post), off, mem, False, None, None)
        b, nb = codec.aggregate_tiles_types(inputs[0], inputs[1], R0, WIN, N_WIN, [LAST], transforms=post,
                                            discard_nan=False)
        torch.cuda.synchronize()
        order = torch.from_numpy(mem.astype(np.int64)).cuda()
        assert torch.equal(a.status[0], b.status[0][order]) and torch.equal(na[0], nb[0][order])
        for g in range(S):
            s = int(mem[g])
            ra = a.packed[int(a.offsets[0, g]): int(a.offsets[0, g]) + int(a.out_len[0, g])]
            rb = b.packed[int(b.offsets[0, s]): int(b.offsets[0, s]) + int(b.out_len[0, s])]
            assert torch.equal(ra, rb), (post, g)


@pytest.mark.parametrize("discard", [True, False])
def test_nan_sources_without_pre_ops(codecs, discard):
    """Gauge Last -> Rollup [Count, Min, Sum] with no pre-ops: with discard_nan a NaN window value is not forwarded
    (generic_elem.go:892-894), so it adds nothing to Count, and a window whose members are all NaN writes nothing"""
    codec = codecs[True]
    sec = 10 ** 9
    pts = [([R0 + 5 * sec, R0 + WIN + 5 * sec, R0 + 2 * WIN + 5 * sec], [1.5, math.nan, math.nan]),
           ([R0 + 7 * sec, R0 + WIN + 7 * sec, R0 + 2 * WIN + 7 * sec], [math.nan, 2.5, math.nan])]
    streams = [O.encode_series(np.array(t, dtype=np.int64), np.array(v), START, O.UNIT_S, True) for t, v in pts]
    off, mem = np.array([0, 2], dtype=np.int64), np.array([0, 1], dtype=np.int32)
    pipe = (GAUGE, LAST, [], [MIN, COUNT, SUM], [])
    exp = Expect(R.decode_sources(streams, True, False), True, 1)
    xs, gs = codec.transform_state(2), codec.element_state(1)
    res = run(codec, layout(streams, "csr"), R0, 3, pipe, off, mem, discard, xs, gs)
    rows, src = exp.call(R0, 3, pipe, off, mem, discard)
    torch.cuda.synchronize()
    check(res, rows, src)
    check_states(exp, xs, gs)
    n = res[1].cpu().numpy()[:, 0].tolist()
    assert n == ([2, 2, 2] if discard else [3, 3, 3])  # window 2 (all NaN) writes nothing with discard_nan
    t, v, cnt, err = O.decode_series(res[0].packed[int(res[0].offsets[1, 0]): int(res[0].offsets[1, 0]) +
                                                   int(res[0].out_len[1, 0])].cpu().numpy().tobytes(), True)
    assert err == 0 and v[:cnt].tolist() == ([1.0, 1.0] if discard else [2.0, 2.0, 2.0])


@pytest.mark.parametrize("metric,src,types", [(COUNTER, SUM, [SUM]), (GAUGE, LAST, [LAST])])
def test_golden_forward_through_the_call(codecs, metric, src, types):
    """testPipeline's source element (Absolute, PerSecond, DiscardNaNAggregatedValues off) through a one-member
    rollup: the rows are the forwarded values of the reference test (the Counter's through int64())"""
    import json
    import os
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "m3tsz_rollup_goldens.json")) as f:
        case = [c for c in json.load(f)["forward"] if c["metric_type"] == metric][0]
    codec = codecs[True]
    step = case["step_ns"]
    ends = [t for t, _ in case["windows"]]
    r0 = ends[0] - step
    stream = O.encode_series(np.array([t - step for t in ends], dtype=np.int64),
                             np.array([v for _, v in case["windows"]]), r0 - step, O.UNIT_S, True)
    blob, o, lengths = _csr([stream])
    res = codec.aggregate_tiles_rollup(blob, o, r0, step, len(ends), src, dev(np.array([0, 1], dtype=np.int64)),
                                       dev(np.array([0], dtype=np.int32)), types, metric_type=metric,
                                       pre_transforms=case["ops"], discard_nan=case["discard_nan"])
    torch.cuda.synchronize()
    r = res[0]
    row = r.packed[int(r.offsets[0, 0]): int(r.offsets[0, 0]) + int(r.out_len[0, 0])].cpu().numpy().tobytes()
    t, v, n, err = O.decode_series(row, True)
    assert err == 0 and t[:n].tolist() == [tt for tt, _ in case["want"]]
    for got, (_, w) in zip(v[:n].tolist(), case["want"]):
        if metric == COUNTER:  # Counter.Update(int64(value)): NaN is MinInt64
            assert got == (-(2.0 ** 63) if w == "NaN" else float(int(w)))
        else:
            assert (w == "NaN" and math.isnan(got)) or got == w


def test_large_batch_sampled(codecs):
    """100 k sources, 10 k groups of 10 random members (each source in one group on average), sampled against the
    oracle"""
    codec = codecs[True]
    rng = np.random.default_rng(12)
    base = _batch(True, S=256, damage=True, n_max=120)
    pick = rng.integers(0, len(base), 100_000)
    streams = [base[i] for i in pick]
    S, G = len(streams), 10_000
    mem = rng.integers(0, S, G * 10).astype(np.int32)
    off = np.arange(0, G * 10 + 1, 10, dtype=np.int64)
    pipe = PIPELINES[0]
    xs, gs = codec.transform_state(S), codec.element_state(G)
    res = run(codec, layout(streams, "csr"), R0, N_WIN, pipe, off, mem, True, xs, gs)
    torch.cuda.synchronize()
    sample = sorted(rng.choice(G, 60, replace=False).tolist())
    srcs = sorted({int(m) for g in sample for m in mem[off[g]: off[g + 1]]})
    idx = {s: i for i, s in enumerate(srcs)}
    sub_mem = np.array([idx[int(m)] for g in sample for m in mem[off[g]: off[g + 1]]], dtype=np.int32)
    sub_off = np.arange(0, len(sample) * 10 + 1, 10, dtype=np.int64)
    exp = Expect(R.decode_sources([streams[s] for s in srcs], True, False), True, len(sample))
    rows, src = exp.call(R0, N_WIN, pipe, sub_off, sub_mem, True)
    r, nt, sst = res
    st, ln, of = r.status.cpu().numpy(), r.out_len.cpu().numpy(), r.offsets.cpu().numpy()
    packed = r.packed.cpu().numpy()
    assert sst.cpu().numpy()[srcs].tolist() == src
    gsh = gs.cpu().numpy().copy().view(E.ELEM_STATE_DTYPE).reshape(-1)
    for i, g in enumerate(sample):
        e_st, e_bytes, e_n = rows[0][i]
        assert st[0, g] == e_st and (e_st or packed[of[0, g]: of[0, g] + ln[0, g]].tobytes() == e_bytes), g
        assert nt[0, g].item() == e_n or e_st, g
        assert gsh[g].tobytes() == exp.group_state[i].tobytes(), g
