"""Tile aggregation through a rollup that keeps annotations on the GPU (m3tsz_aggregate_tiles_rollup_annotated: the
annotated fused decode, the annotated forward and fold variants and the multi-type element stage's IN = 7): bytes,
out_len, n_tiles, row and source statuses and both kinds of record against the composed oracle
(rollup_ann_oracle_lib), in both int_optimized modes, one stream per source and source blocks; discard_nan on and
off with annotated NaN windows; the last listed member winning; every valid rollup type, Reset before and after the
rollup; bad groups and a failed source; CAPACITY and the retry of the failed groups; split calls; argument checks;
byte equality with m3tsz_aggregate_tiles_rollup on sources without annotations; one-member groups against
m3tsz_aggregate_tiles_annotated; a 100 k source batch; and the Prometheus payload read back from the rolled-up rows."""
import numpy as np
import pytest
import torch

import ann_oracle_lib as N
import oracle_lib as O
import rollup_ann_oracle_lib as RA
import rollup_oracle_lib as R
from m3_b200 import capi
from test_gpu_tile_annotations import PROM_COUNTER_PAYLOAD, _first_annotation, annotated_batch
from test_gpu_tile_rollup import (ADD, COUNTER, ERR_CAPACITY, ERR_INVALID_ARG, GAUGE, INC, LAST, MAX, MIN,
                                  PIPELINES, RST, SUM, Expect, block_layout, check, check_states, dev, layout,
                                  membership)
from test_gpu_transforms import N_WIN, R0, START, WIN, _batch, codecs  # noqa: F401
from test_tile_blocks_oracle import random_series

pytestmark = pytest.mark.gpu

SEC = 10 ** 9


class ExpectAnn(Expect):
    """the composed oracle with the records of the plain rollup's Expect; `decoded` from RA.decode_sources"""

    def call(self, r0, n_win, pipe, off, mem, discard, saved_rows=None):
        metric, src, pre, types, post = pipe
        return RA.aggregate_tiles_rollup_annotated(self.decoded, self.int_opt, r0, WIN, n_win, metric, src, pre, off,
                                                   mem, types, post, discard, self.src_state, self.group_state,
                                                   saved_rows)


def run(codec, inputs, r0, n_win, pipe, off, mem, discard, src_state, group_state, capacity=None, annotations=True):
    blob, o, lengths, blocks = inputs
    metric, src, pre, types, post = pipe
    return codec.aggregate_tiles_rollup(blob, o, r0, WIN, n_win, src, dev(off), dev(mem), types, metric_type=metric,
                                        pre_transforms=pre, post_transforms=post, discard_nan=discard,
                                        src_state=src_state, group_state=group_state, lengths=lengths, blocks=blocks,
                                        capacity=capacity, annotations=annotations)


def groups_with(off, mem, extra):
    """the groups (off, mem) plus one group per list in `extra`"""
    lists = [mem[off[g]: off[g + 1]].tolist() for g in range(len(off) - 1)] + extra
    o = np.zeros(len(lists) + 1, dtype=np.int64)
    o[1:] = np.cumsum([len(x) for x in lists])
    return o, np.array([m for x in lists for m in x], dtype=np.int32)


@pytest.mark.parametrize("discard", [True, False])
@pytest.mark.parametrize("addressing", ["csr", "lengths"])
@pytest.mark.parametrize("int_opt", [True, False])
def test_against_oracle(codecs, int_opt, addressing, discard):
    """every pipeline (every valid rollup type, Reset in the pre- and post-ops); the last source is truncated inside
    an annotation, and a group that lists it fails; bad groups (a member index >= S, a decreasing range, a range
    past n_members) fail alone; the records carry over two calls"""
    codec = codecs[int_opt]
    streams = annotated_batch(int_opt)
    S = len(streams)
    decoded = RA.decode_sources(streams, int_opt, blocks=False)
    assert decoded[S - 1][3] != 0
    inputs = layout(streams, addressing)
    rng = np.random.default_rng(31)
    for pipe in PIPELINES:
        off, mem = membership(rng, S, 37)
        off, mem = groups_with(off, mem, [[S - 1, 0], [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10], [4, 1, 4], [2, S + 5]])
        failed_src, bad_index = len(off) - 5, len(off) - 2
        # then a decreasing range, a valid one over [4, 1, 4] again, and one past n_members
        off = np.concatenate([off, [off[-1] - 5, off[-1] - 2, off[-1] + 5]]).astype(np.int64)
        G = len(off) - 1
        bad = [failed_src, bad_index, G - 3, G - 1]
        exp = ExpectAnn(decoded, int_opt, G)
        xs, gs = codec.transform_state(S), codec.element_state(G)
        for r0, n_win in ((R0, 5), (R0 + 5 * WIN, N_WIN - 5)):
            res = run(codec, inputs, r0, n_win, pipe, off, mem, discard, xs, gs)
            rows, src = exp.call(r0, n_win, pipe, off, mem, discard)
            torch.cuda.synchronize()
            assert all(rows[j][g][0] != 0 for j in range(len(pipe[3])) for g in bad)
            assert all(rows[j][G - 2][0] == 0 for j in range(len(pipe[3])))
            check(res, rows, src)
            check_states(exp, xs, gs)


@pytest.mark.parametrize("int_opt", [True, False])
def test_blocks(codecs, int_opt):
    """0-12 annotated source blocks per series (the block decode's batch-addressed references)"""
    from test_tile_blocks_oracle import N_WIN as BN, R0 as BR0, STEP
    assert STEP == WIN
    codec = codecs[int_opt]
    rng = np.random.default_rng(22)
    series = [random_series(rng, (0, 1, 2, 5, 12)[i % 5], int_opt, True) for i in range(37)]
    decoded = RA.decode_sources(series, int_opt, blocks=True)
    off, mem = membership(rng, 37, 19)
    for pipe in (PIPELINES[0], PIPELINES[1], PIPELINES[3]):
        for discard in (True, False):
            exp = ExpectAnn(decoded, int_opt, 19)
            xs, gs = codec.transform_state(37), codec.element_state(19)
            res = run(codec, block_layout(series), BR0, BN, pipe, off, mem, discard, xs, gs)
            rows, src = exp.call(BR0, BN, pipe, off, mem, discard)
            torch.cuda.synchronize()
            check(res, rows, src)
            check_states(exp, xs, gs)


def _one_point(t, v, a):
    enc = O.Encoder(START, True)
    assert enc.encode(int(t), float(v), O.UNIT_S, a) == 0
    return enc.stream()


@pytest.mark.parametrize("discard", [True, False])
def test_listed_order_and_nan(codecs, discard):
    """window 0: sources a / b / none / NaN carrying "n".  The last listed member with an annotation wins; a NaN that
    discard_nan drops does not count, one forwarded without it does; a member in two groups gives both"""
    codec = codecs[True]
    t = R0 + 10 * SEC
    streams = [_one_point(t, 1.0, b"a"), _one_point(t, 2.0, b"bb"), _one_point(t, 3.0, b""),
               _one_point(t, float("nan"), b"n")]
    off = np.array([0, 3, 5, 6, 8, 9], dtype=np.int64)
    mem = np.array([0, 1, 2, 1, 0, 2, 0, 3, 3], dtype=np.int32)
    pipe = (GAUGE, LAST, [], [MIN, SUM], [])
    res = run(codec, layout(streams, "csr"), R0, 2, pipe, off, mem, discard, None, None)
    exp = ExpectAnn(RA.decode_sources(streams, True, False), True, 5)
    rows, src = exp.call(R0, 2, pipe, off, mem, discard)
    torch.cuda.synchronize()
    check(res, rows, src)
    want = [b"bb", b"a", None, b"a" if discard else b"n", None if discard else b"n"]
    for g, a in enumerate(want):
        if res[0].out_len[0, g] == 0:
            assert g == 4 and discard  # (its only member's NaN was dropped)
        else:
            assert _first_annotation(codec, res[0], g) == ((a, 1) if a else (b"", 0)), g


@pytest.mark.parametrize("int_opt", [True, False])
def test_unannotated_sources_equal_rollup(codecs, int_opt):
    """no source annotated: the bytes, statuses, counts and records of m3tsz_aggregate_tiles_rollup"""
    codec = codecs[int_opt]
    streams = _batch(int_opt, S=70)
    inputs = layout(streams, "lengths")
    rng = np.random.default_rng(5)
    for pipe in PIPELINES:
        off, mem = membership(rng, 70, 41)
        outs = []
        for ann in (False, True):
            xs, gs = codec.transform_state(70), codec.element_state(41)
            r, nt, sst = run(codec, inputs, R0, N_WIN, pipe, off, mem, True, xs, gs, annotations=ann)
            rows = [[r.packed[int(r.offsets[j, g]): int(r.offsets[j, g]) + int(r.out_len[j, g])].cpu().numpy()
                     .tobytes() for g in range(41)] for j in range(len(pipe[3]))]
            outs.append((rows, r.status.cpu(), r.out_len.cpu(), nt.cpu(), sst.cpu(), xs.cpu(), gs.cpu()))
        a, b = outs
        assert a[0] == b[0]
        for x, y in zip(a[1:], b[1:]):
            assert torch.equal(x, y)


@pytest.mark.parametrize("int_opt", [True, False])
def test_one_member_groups_equal_tiles_annotated(codecs, int_opt):
    """Last -> Rollup [Last] with one member per group, no pre-ops and no discard is the local element with
    annotations"""
    codec = codecs[int_opt]
    streams = annotated_batch(int_opt)
    S = len(streams)
    inputs = layout(streams, "csr")
    off = np.arange(S + 1, dtype=np.int64)
    mem = np.arange(S, dtype=np.int32)[::-1].copy()
    for post in ([], [ADD], [INC, RST]):
        a, na, _ = run(codec, inputs, R0, N_WIN, (GAUGE, LAST, [], [LAST], post), off, mem, False, None, None)
        b, nb = codec.aggregate_tiles_types(inputs[0], inputs[1], R0, WIN, N_WIN, [LAST], transforms=post,
                                            discard_nan=False, annotations=True)
        torch.cuda.synchronize()
        order = torch.from_numpy(mem.astype(np.int64)).cuda()
        assert torch.equal(a.status[0], b.status[0][order]) and torch.equal(na[0], nb[0][order])
        for g in range(S):
            s = int(mem[g])
            ra = a.packed[int(a.offsets[0, g]): int(a.offsets[0, g]) + int(a.out_len[0, g])]
            rb = b.packed[int(b.offsets[0, s]): int(b.offsets[0, s]) + int(b.out_len[0, s])]
            assert torch.equal(ra, rb), (post, g)


def _subset(off, mem, groups):
    srcs = sorted({int(m) for g in groups for m in mem[off[g]: off[g + 1]]})
    idx = {s: i for i, s in enumerate(srcs)}
    sub_mem = np.array([idx[int(m)] for g in groups for m in mem[off[g]: off[g + 1]]], dtype=np.int32)
    sub_off = np.zeros(len(groups) + 1, dtype=np.int64)
    sub_off[1:] = np.cumsum([off[g + 1] - off[g] for g in groups])
    return srcs, sub_off, sub_mem


def test_capacity_then_retry(codecs):
    """a packed buffer too small: CAPACITY on some group rows, never a shorter stream; re-running exactly the failed
    groups with their members gives the result of one unstopped call"""
    codec = codecs[True]
    streams = annotated_batch(True)[:-1]
    S = len(streams)
    decoded = RA.decode_sources(streams, True, False)
    off, mem = membership(np.random.default_rng(6), S, 33)
    pipe = PIPELINES[3]
    exp = ExpectAnn(decoded, True, 33)
    # half the bytes the rows take with room (each row's slot adds its group's member bytes, so the capacity has to be
    # a share of the real total to leave some rows written)
    total = int(run(codec, layout(streams, "csr"), R0, N_WIN, pipe, off, mem, True, None, None)[0].total.item())
    xs, gs = codec.transform_state(S), codec.element_state(33)
    res = run(codec, layout(streams, "csr"), R0, N_WIN, pipe, off, mem, True, xs, gs, capacity=total // 2)
    torch.cuda.synchronize()
    st = res[0].status.cpu().numpy()
    assert (st == ERR_CAPACITY).any() and (st == 0).any()
    saved = lambda g: bool((st[:, g] == 0).all())
    rows, _ = exp.call(R0, N_WIN, pipe, off, mem, True, saved_rows=saved)
    check(res, rows, None, only=[g for g in range(33) if saved(g)])
    assert (res[0].out_len.cpu().numpy()[st != 0] == 0).all()
    check_states(exp, xs, gs)
    full = ExpectAnn(decoded, True, 33)
    want, _ = full.call(R0, N_WIN, pipe, off, mem, True)
    failed = [g for g in range(33) if not saved(g)]
    srcs, sub_off, sub_mem = _subset(off, mem, failed)
    si, gi = torch.tensor(srcs, device="cuda"), torch.tensor(failed, device="cuda")
    sx, sg = xs[si].contiguous(), gs[gi].contiguous()
    res2 = run(codec, layout([streams[s] for s in srcs], "csr"), R0, N_WIN, pipe, sub_off, sub_mem, True, sx, sg)
    xs[si], gs[gi] = sx, sg
    torch.cuda.synchronize()
    check(res2, [[row[g] for g in failed] for row in want], None)
    check_states(full, xs, gs)


@pytest.mark.parametrize("n_calls", [1, 2, 5])
def test_split_calls(codecs, n_calls):
    """consecutive calls over a split window range: each call's rows are the oracle's with the carried records"""
    codec = codecs[True]
    streams = annotated_batch(True, seed=9)
    S = len(streams)
    decoded = RA.decode_sources(streams, True, False)
    off, mem = membership(np.random.default_rng(9), S, 20)
    pipe = PIPELINES[0]
    edges = np.linspace(0, N_WIN, n_calls + 1).astype(int)
    exp = ExpectAnn(decoded, True, 20)
    xs, gs = codec.transform_state(S), codec.element_state(20)
    for a, b in zip(edges[:-1], edges[1:]):
        res = run(codec, layout(streams, "csr"), R0 + int(a) * WIN, int(b - a), pipe, off, mem, True, xs, gs)
        rows, src = exp.call(R0 + int(a) * WIN, int(b - a), pipe, off, mem, True)
        torch.cuda.synchronize()
        check(res, rows, src)
        check_states(exp, xs, gs)


def test_invalid_arguments(codecs):
    codec = codecs[True]
    streams = annotated_batch(True)[:8]
    off, mem = np.array([0, 2], dtype=np.int64), np.array([0, 1], dtype=np.int32)
    inputs = layout(streams, "csr")
    bad = [
        (GAUGE, LAST, [], [MAX, MIN], []),
        (GAUGE, LAST, [], [], []),
        (COUNTER, LAST, [], [SUM], []),
        (GAUGE, LAST, [2, 3], [SUM], []),
        (COUNTER, SUM, [], [LAST], []),
        (GAUGE, LAST, [6], [SUM], []),
    ]
    for pipe in bad:
        with pytest.raises(capi.M3tszError) as e:
            run(codec, inputs, R0, N_WIN, pipe, off, mem, True, None, None)
        assert e.value.status == ERR_INVALID_ARG, pipe


def test_large_batch_sampled(codecs):
    """100 k sources, 10 k groups of 10 random members, sampled against the oracle"""
    codec = codecs[True]
    rng = np.random.default_rng(12)
    base = annotated_batch(True, seed=12)
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
    srcs, sub_off, sub_mem = _subset(off, mem, sample)
    exp = ExpectAnn(RA.decode_sources([streams[s] for s in srcs], True, False), True, len(sample))
    rows, src = exp.call(R0, N_WIN, pipe, sub_off, sub_mem, True)
    r, nt, sst = res
    st, ln, of = r.status.cpu().numpy(), r.out_len.cpu().numpy(), r.offsets.cpu().numpy()
    packed = r.packed.cpu().numpy()
    assert sst.cpu().numpy()[srcs].tolist() == src
    for i, g in enumerate(sample):
        e_st, e_bytes, e_n = rows[0][i]
        assert st[0, g] == e_st and (e_st or packed[of[0, g]: of[0, g] + ln[0, g]].tobytes() == e_bytes), g
        assert nt[0, g].item() == e_n or e_st, g


def test_prometheus_counter_payload_round_trip(codecs):
    """Increase -> Rollup [Sum] -> Add over counters whose every source block carries the OpenMetrics counter payload
    on its first datapoint: the first annotation of every rolled-up row, as the Prometheus conversion reads it, is
    that payload"""
    from test_tile_blocks_oracle import B0, BS, N_WIN as BN, R0 as BR0, encode
    codec = codecs[True]
    rng = np.random.default_rng(40)
    series = []
    for s in range(64):
        blocks, v = [], float(rng.integers(0, 100))
        for b in range(4):
            t, dps = B0 + b * BS + int(rng.integers(1, 20)) * SEC, []
            while t < B0 + (b + 1) * BS:
                v += float(rng.integers(0, 10))
                dps.append([t, v, O.UNIT_S, PROM_COUNTER_PAYLOAD if not dps else b""])
                t += int(rng.integers(10, 50)) * SEC
            blocks.append(encode(dps, True, B0 + b * BS))
        series.append(blocks)
    off = np.arange(0, 65, 8, dtype=np.int64)
    mem = rng.permutation(64).astype(np.int32)
    pipe = PIPELINES[0]
    res = run(codec, block_layout(series), BR0, BN, pipe, off, mem, True, None, None)
    exp = ExpectAnn(RA.decode_sources(series, True, blocks=True), True, 8)
    rows, src = exp.call(BR0, BN, pipe, off, mem, True)
    torch.cuda.synchronize()
    check(res, rows, src)
    for g in range(8):
        assert int(res[0].out_len[0, g]) > 0
        got, cnt = _first_annotation(codec, res[0], g)
        assert got == PROM_COUNTER_PAYLOAD and cnt >= 1, g
    # the plain rollup writes none
    plain = run(codec, block_layout(series), BR0, BN, pipe, off, mem, True, None, None, annotations=False)
    torch.cuda.synchronize()
    assert _first_annotation(codec, plain[0], 0)[1] == 0


def test_goldens_through_the_call(codecs):
    """the reference's AddUnique annotation steps (tests/golden/m3tsz_rollup_annotation_goldens.json), each
    forwarded value one source, all steps' sources one group rolled up with [Count, Sum]: the device's rows are the
    composed oracle's, which tests/test_rollup_annotation_goldens.py checks against the goldens"""
    from test_rollup_annotation_goldens import COUNT, COUNTER as G_COUNTER, LAST as G_LAST, SUM as G_SUM, _ann, \
        _cases, _stream
    codec = codecs[True]
    for case in _cases():
        step, starts = case["resolution_ns"], case["window_starts_ns"]
        streams = [_stream(st["at_ns"], v, _ann(st["annotation"])) for st in case["steps"] for v in st["values"]]
        n = len(streams)
        off, mem = np.array([0, n], dtype=np.int64), np.arange(n, dtype=np.int32)
        pipe = (case["metric_type"], G_SUM if case["metric_type"] == G_COUNTER else G_LAST, [], [COUNT, G_SUM], [])
        r = codec.aggregate_tiles_rollup(*layout(streams, "csr")[:2], starts[0], step, len(starts), pipe[1],
                                         dev(off), dev(mem), pipe[3], metric_type=pipe[0], discard_nan=False,
                                         annotations=True)
        exp = ExpectAnn(RA.decode_sources(streams, True, False), True, 1)
        metric, src, pre, types, post = pipe
        rows, srcs = RA.aggregate_tiles_rollup_annotated(exp.decoded, True, starts[0], step, len(starts), metric, src,
                                                         pre, off, mem, types, post, False, exp.src_state,
                                                         exp.group_state)
        torch.cuda.synchronize()
        check(r, rows, srcs)
        assert b"testAnnotation" in N.decode_annotated(rows[1][0][1], True)[2]
