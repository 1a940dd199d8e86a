"""Element-set rollups across shards on the GPU (m3tsz_element_set_forward_write / _add_forwarded, DESIGN.md §4.12), in
both int_optimized modes: sources split over K source sets written as forwarded batches and added to a group set give
byte for byte the rows, records, watermarks and open windows of one m3tsz_element_set_forward over a single set that
holds every source (each group's members listed shard by shard), and the same source-set state; shuffled arrival
against the CPU model (tests/element_forwarded_model.py); redelivery; every capacity stop with grow and retry; closed
and invalid records; the host checks; 100 k groups; and a run on a caller's non-blocking stream."""
import ctypes as C

import numpy as np
import pytest
import torch

import agg_oracle_lib as A
from element_forwarded_model import ForwardedGroupModel, SourceModel, add_forwarded, forward_write
from m3_b200 import capi
from m3_b200.codec import ForwardedBatch
from test_gpu_elements import _point_major, _rows

pytestmark = pytest.mark.gpu

SEC = 1_000_000_000
RES = 60 * SEC
START = 1_600_000_020 * SEC
DEV = "cuda"
GAUGE, COUNTER = A.METRIC_GAUGE, A.METRIC_COUNTER
LAST, MIN, MAX, SUM = 1, 2, 3, 7
OK, CAP, INV, CLOSED, DUP = 0, capi.ERR_CAPACITY, capi.ERR_INVALID_ARG, capi.ERR_AGGREGATION_CLOSED, \
    capi.ERR_DUPLICATE_SOURCE
# (metric, source type, pre-ops, rollup types, post-ops)
PIPES = [(COUNTER, SUM, [3], [SUM], [4]), (GAUGE, LAST, [2], [MIN, MAX, SUM], [5]), (GAUGE, LAST, [], [LAST, SUM], [])]


@pytest.fixture(scope="module")
def codecs():
    from m3_b200.codec import BatchCodec
    return {True: BatchCodec(0, int_optimized=True), False: BatchCodec(0, int_optimized=False)}


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _bits(v):
    return int(np.array([v], dtype=np.float64).view(np.uint64)[0])


def _cols(rng, S, W, metric, nan=0.0):
    cols = []
    for _ in range(S):
        pts = []
        for w in range(W):
            if rng.random() < 0.25:
                continue
            for o in np.sort(rng.integers(0, 60, int(rng.integers(1, 4)))):
                v = float(rng.integers(0, 1000)) if metric == COUNTER else float(rng.normal() * 100)
                if rng.random() < nan:
                    v = float("nan")
                pts.append((START + w * RES + int(o) * SEC, _bits(v)))
        cols.append(pts)
    return cols


def _membership(rng, S, G, per=5):
    off = np.arange(0, G * per + 1, per, dtype=np.int64)
    return off, rng.integers(0, S, G * per).astype(np.int32)


def _split(off, mem, K):
    """each group's members by shard (source s on shard s % K, local index s // K), keeping their order: per shard
    (group_off, members), and the single set's members listed shard by shard"""
    G = len(off) - 1
    parts, whole = [], [[] for _ in range(G)]
    for k in range(K):
        o, m = [0], []
        for g in range(G):
            mine = [int(x) for x in mem[off[g]:off[g + 1]] if x % K == k]
            m += [x // K for x in mine]
            whole[g] += mine
            o.append(len(m))
        parts.append((np.array(o, dtype=np.int64), np.array(m, dtype=np.int32)))
    o = np.cumsum([0] + [len(w) for w in whole]).astype(np.int64)
    return parts, o, np.array([x for w in whole for x in w], dtype=np.int32)


def _open_windows(es):
    """each element's open slots as sorted (start, field values...) tuples: slot placement aside, the windows"""
    w = {f: a.cpu().numpy() for f, a in es.win.items()}
    fields = sorted(w)
    out = []
    for s in range(es.n_elements):
        rows = [tuple(w[f][r, s].tobytes() for f in fields) for r in range(es.open_windows) if w["count"][r, s]]
        out.append(sorted(rows, key=lambda t: np.frombuffer(t[fields.index("start")], dtype=np.int64)[0]))
    return out


def _world(codec, pipe, S, G, K, discard, R=8, cap=64):
    metric, src_type, pre, types, post = pipe
    at = lambda n: torch.full((n,), START, dtype=torch.int64, device=DEV)
    one = codec.element_set(at(S), metric, [src_type], RES, transforms=pre, discard_nan=discard, open_windows=8,
                            stride=0)
    shards = [codec.element_set(at(len(range(k, S, K))), metric, [src_type], RES, transforms=pre,
                                discard_nan=discard, open_windows=8, stride=0) for k in range(K)]
    ref = codec.element_set(at(G), metric, types, RES, transforms=post, discard_nan=discard, open_windows=R)
    grp = codec.element_set(at(G), metric, types, RES, transforms=post, discard_nan=discard, open_windows=R,
                            source_capacity=cap)
    return one, shards, ref, grp


def _add(one, shards, cols, K):
    r, st = one.add(*_point_major(cols))
    assert int(st.abs().sum()) == 0 and int(r.abs().sum()) == 0
    for k, sh in enumerate(shards):
        r, st = sh.add(*_point_major(cols[k::K]))
        assert int(st.abs().sum()) == 0 and int(r.abs().sum()) == 0


def _write_all(shards, target, parts, order=None):
    batches = []
    for k, (o, m) in enumerate(parts):
        b, st, gst = shards[k].forward_write(target, _dev(o), _dev(m), k)
        assert int(st.abs().sum()) == 0 and int(gst.abs().sum()) == 0
        assert b.counts[0] == b.counts[2] and b.counts[1] == b.counts[3]
        batches.append(b)
    return batches


def _same_sources(one, shards, K):
    for k, sh in enumerate(shards):
        idx = torch.arange(k, one.n_elements, K, device=DEV)
        assert torch.equal(sh.elem, one.elem[idx]) and torch.equal(sh.watermark, one.watermark[idx])
        assert torch.equal(sh.win["count"], one.win["count"][:, idx])


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("pipe", range(len(PIPES)))
@pytest.mark.parametrize("K", [1, 2, 5])
def test_shards_compose_to_one_forward(codecs, int_opt, pipe, K):
    codec = codecs[int_opt]
    rng = np.random.default_rng(100 * pipe + 10 * K + int_opt)
    S, G, W = 60, 11, 6
    discard = bool(K % 2)
    cols = _cols(rng, S, W, PIPES[pipe][0], nan=0.1)
    off, mem = _membership(rng, S, G)
    mem[1] = mem[0]  # a member listed twice
    parts, o1, m1 = _split(off, mem, K)
    one, shards, ref, grp = _world(codec, PIPES[pipe], S, G, K, discard)
    _add(one, shards, cols, K)
    for target in (START + 3 * RES, START + W * RES):
        sst, gst = one.forward(target, _dev(o1), _dev(m1), ref)
        assert int(sst.abs().sum()) == 0 and int(gst.abs().sum()) == 0
        res, st = grp.add_forwarded(_write_all(shards, target, parts))
        assert int(st.abs().sum()) == 0 and int(res.abs().sum()) == 0
        assert _open_windows(grp) == _open_windows(ref)
        assert int(ref.consume(target).abs().sum()) == 0 and int(grp.consume(target).abs().sum()) == 0
        assert torch.equal(grp.watermark, ref.watermark) and torch.equal(grp.elem, ref.elem)
    assert _rows(grp) == _rows(ref)
    _same_sources(one, shards, K)


@pytest.mark.parametrize("metric", [GAUGE, COUNTER])
def test_shuffled_arrival_against_the_model(codecs, metric):
    codec = codecs[True]
    rng = np.random.default_rng(7 + metric)
    S, G, W, K = 50, 9, 4, 3
    pipe = PIPES[0] if metric == COUNTER else PIPES[2]
    cols = _cols(rng, S, W, metric)
    off, mem = _membership(rng, S, G)
    parts, _, _ = _split(off, mem, K)
    one, shards, _, grp = _world(codec, pipe, S, G, K, False)
    _add(one, shards, cols, K)
    b = ForwardedBatch.concat(_write_all(shards, START + W * RES, parts))
    perm = rng.permutation(b.metrics.shape[0])
    shuffled = ForwardedBatch(b.metrics[_dev(perm)], b.values, b.counts)
    res, st = grp.add_forwarded(shuffled)
    f = shuffled.fields()
    vals = b.values.cpu().numpy()
    recs = [(int(f["key"][i]), int(f["time_ns"][i]), vals[f["value_off"][i]: f["value_off"][i] + f["n_values"][i]]
             .tolist(), int(f["source_id"][i]), 0, 0) for i in range(len(perm))]
    model = [ForwardedGroupModel(metric, pipe[3], RES, open_windows=8, source_capacity=64) for _ in range(G)]
    mres, mst = add_forwarded(model, recs)
    assert res.cpu().tolist() == mres and st.cpu().tolist() == mst
    w = {f: a.cpu().numpy() for f, a in grp.win.items()}
    for g in range(G):
        for r in range(grp.open_windows):
            if not w["count"][r, g]:
                continue
            a = model[g].aggregates(int(w["start"][r, g]))
            for fld, v in a.items():
                got = w[fld][r, g]
                assert got.tobytes() == np.array([v], dtype=got.dtype).tobytes(), (g, fld)


@pytest.mark.parametrize("metric", [GAUGE, COUNTER])
def test_keys_and_invalid_groups_against_the_model(codecs, metric):
    """the writer's keys (a permutation: group g's records go to element keys[g]) and its invalid groups (a decreasing
    range, a range past n_members, a member past the sources), which write nothing and hold their members back, against
    the CPU model; the records then added give the model's results and group windows"""
    codec = codecs[False]
    rng = np.random.default_rng(31 + metric)
    S, G, W = 24, 8, 4
    pipe = PIPES[0] if metric == COUNTER else PIPES[2]
    src_type, pre = pipe[1], pipe[2]
    cols = _cols(rng, S, W, metric)
    at = lambda n: torch.full((n,), START, dtype=torch.int64, device=DEV)
    src = codec.element_set(at(S), metric, [src_type], RES, transforms=pre, open_windows=8, stride=0)
    grp = codec.element_set(at(G), metric, pipe[3], RES, transforms=pipe[4], open_windows=8, source_capacity=32)
    models = [SourceModel(metric, src_type, RES, pre, open_windows=8) for _ in range(S)]
    r, st = src.add(*_point_major(cols))
    assert int(st.abs().sum()) == 0
    for s, m in enumerate(models):
        m.add(cols[s])
    off, mem = _membership(rng, S, G, per=4)
    mem[3 * 4 + 1] = S + 5  # group 3 lists a source past the sources
    off[6] = off[7] + 1  # group 6's range decreases
    off[G] = len(mem) + 2  # group 7's runs past n_members
    keys = rng.permutation(G).astype(np.int64)
    gms = [ForwardedGroupModel(metric, pipe[3], RES, open_windows=8, source_capacity=32) for _ in range(G)]
    for target in (START + 2 * RES, START + W * RES):
        b, sst, gst = src.forward_write(target, _dev(off), _dev(mem), 3, keys=_dev(keys))
        want, wst, wgst, wcounts = forward_write(models, target, off, mem, 3, keys)
        assert gst.cpu().tolist() == wgst and sst.cpu().tolist() == wst and b.counts == wcounts
        assert {g for g in range(G) if wgst[g] == INV} == {3, 6, 7}
        f = b.fields()
        vals = b.values.cpu().numpy()
        got = [(int(f["key"][i]), int(f["time_ns"][i]),
                vals[f["value_off"][i]: f["value_off"][i] + f["n_values"][i]].tolist(), int(f["source_id"][i]),
                int(f["version"][i]), int(f["reserved"][i])) for i in range(b.counts[0])]
        assert [r[:2] + r[3:] for r in got] == [r[:2] + r[3:] for r in want]
        assert all(np.array(a[2]).tobytes() == np.array(w[2]).tobytes() for a, w in zip(got, want))
        assert torch.equal(src.watermark.cpu(), torch.tensor([m.watermark for m in models]))
        # the members of the invalid groups were held back and forward their windows again in the second call: the
        # valid groups that list them get those records twice from the same source, which refuses them
        res, st = grp.add_forwarded(b)
        wres, wst = add_forwarded(gms, want)
        assert res.cpu().tolist() == wres and st.cpu().tolist() == wst
    w = {k: a.cpu().numpy() for k, a in grp.win.items()}
    for g in range(G):
        for r in range(grp.open_windows):
            if w["count"][r, g] and int(w["start"][r, g]) in gms[g].windows:
                for fld, v in gms[g].aggregates(int(w["start"][r, g])).items():
                    assert w[fld][r, g].tobytes() == np.array([v], dtype=w[fld].dtype).tobytes(), (g, fld)


def test_redelivery(codecs):
    codec = codecs[False]
    rng = np.random.default_rng(11)
    S, G, W, K = 40, 8, 4, 2
    cols = _cols(rng, S, W, COUNTER)
    off, mem = _membership(rng, S, G)
    parts, _, _ = _split(off, mem, K)
    one, shards, _, grp = _world(codec, PIPES[0], S, G, K, False)
    _add(one, shards, cols, K)
    batches = _write_all(shards, START + W * RES, parts)
    res, _ = grp.add_forwarded(batches)
    assert int(res.abs().sum()) == 0
    before = grp.state()
    res, st = grp.add_forwarded(batches)
    assert set(res.cpu().tolist()) == {DUP} and int(st.abs().sum()) == 0
    b = ForwardedBatch.concat(batches)
    idx = _dev(rng.integers(0, b.metrics.shape[0], 25))
    res, _ = grp.add_forwarded(ForwardedBatch(b.metrics[idx], b.values, b.counts))
    assert set(res.cpu().tolist()) == {DUP}
    after = grp.state()
    for f in before["win"]:
        assert torch.equal(before["win"][f], after["win"][f])
    assert torch.equal(before["source_bits"], after["source_bits"])


@pytest.mark.parametrize("limit,resend", [("windows", "refused"), ("windows", "whole"), ("sources", "refused"),
                                          ("sources", "whole"), ("metrics", None), ("values", None)])
def test_capacity_grow_and_retry(codecs, limit, resend):
    """an add stopped by open windows or source ids resends the refused records, or the whole batch, after a grow; a
    writer stopped by its record or value buffer writes again exactly the failed groups"""
    codec = codecs[True]
    rng = np.random.default_rng(13)
    S, G, W, K = 40, 10, 5, 2
    cols = _cols(rng, S, W, GAUGE)
    off, mem = _membership(rng, S, G)
    parts, o1, m1 = _split(off, mem, K)
    one, shards, ref, grp = _world(codec, PIPES[2], S, G, K, False, R=2 if limit == "windows" else 8,
                                   cap=32 if limit == "sources" else 64)
    ref.grow(open_windows=8)
    _add(one, shards, cols, K)
    target = START + W * RES
    one.forward(target, _dev(o1), _dev(m1), ref)
    if limit in ("metrics", "values"):
        batches = []
        for k, (o, m) in enumerate(parts):
            b, st, gst = shards[k].forward_write(target, _dev(o), _dev(m), k + 32,
                                                 metric_capacity=8 if limit == "metrics" else None,
                                                 value_capacity=40 if limit == "values" else None)
            g = gst.cpu().tolist()
            assert CAP in g and g.index(CAP) > 0 and set(g[g.index(CAP):]) == {CAP} and b.counts[0] < b.counts[2]
            batches.append(b)
            failed = [i for i in range(G) if g[i] == CAP]
            o2 = np.zeros(G + 1, dtype=np.int64)
            mm = []
            for i in range(G):
                if i in failed:
                    mm += m[o[i]:o[i + 1]].tolist()
                o2[i + 1] = len(mm)
            b2, st2, gst2 = shards[k].forward_write(target, _dev(o2), _dev(np.array(mm, dtype=np.int32)), k + 32)
            assert int(gst2.abs().sum()) == 0
            batches.append(b2)
        res, st = grp.add_forwarded(batches)
        assert int(res.abs().sum()) == 0
    else:
        batches = _write_all(shards, target, parts)
        if limit == "sources":  # source ids 32, 33 do not fit a capacity of 32
            for b in batches:
                b.metrics[:, 28:32] = torch.tensor([32 + b.metrics[0, 28].item(), 0, 0, 0], dtype=torch.uint8,
                                                   device=DEV)
        res, st = grp.add_forwarded(batches)
        r = res.cpu().numpy()
        assert (r == CAP).any() and (st.cpu().numpy() == CAP).any()
        grp.grow(open_windows=8, source_capacity=64)
        b = ForwardedBatch.concat(batches)
        if resend == "refused":
            b = ForwardedBatch(b.metrics[_dev(np.nonzero(r == CAP)[0])], b.values, b.counts)
        res2, st2 = grp.add_forwarded(b)
        assert int(st2.abs().sum()) == 0
        assert set(res2.cpu().tolist()) <= ({OK} if resend == "refused" else {OK, DUP})
    assert _open_windows(grp) == _open_windows(ref)
    assert int(ref.consume(target).abs().sum()) == 0 and int(grp.consume(target).abs().sum()) == 0
    assert _rows(grp) == _rows(ref)


def test_closed_and_invalid_records(codecs):
    codec = codecs[True]
    at = lambda n: torch.full((n,), START, dtype=torch.int64, device=DEV)
    grp = codec.element_set(at(2), COUNTER, [SUM], RES, open_windows=4, source_capacity=32)
    t = START + RES
    recs = [(0, t, 0, 1, 0, 0, 0), (7, t, 0, 1, 0, 0, 0), (0, t, 0, 0, 1, 0, 0), (0, t, 0, 1, 1, 1, 0),
            (0, t, 0, 1, 1, 0, 3), (0, t, 1, 5, 1, 0, 0), (1, t + 17 * SEC, 1, 1, 0, 0, 0), (0, t, 1, 1, 0, 0, 0)]
    m = np.zeros((len(recs), 40), dtype=np.uint8)
    for i, (k, tt, vo, nv, sid, ver, rsv) in enumerate(recs):
        m[i] = np.frombuffer(np.array([(k, tt, vo, nv, sid, ver, rsv)], dtype=[
            ("k", "<u8"), ("t", "<i8"), ("vo", "<u8"), ("nv", "<u4"), ("sid", "<u4"), ("v", "<u4"),
            ("r", "<u4")]).tobytes(), dtype=np.uint8)
    b = ForwardedBatch(_dev(m), _dev(np.array([3.0, 4.0])), (len(recs), 2, len(recs), 2))
    res, st = grp.add_forwarded(b)
    assert res.cpu().tolist() == [OK, INV, INV, INV, INV, INV, OK, DUP] and int(st.abs().sum()) == 0
    assert grp.win["sum"][:, 0].sum().item() == 3 and grp.win["sum"][:, 1].sum().item() == 4
    assert int(grp.consume(START + 2 * RES).abs().sum()) == 0
    res, _ = grp.add_forwarded(ForwardedBatch(_dev(m[:1]), _dev(np.array([3.0])), (1, 1, 1, 1)))
    assert res.cpu().tolist() == [CLOSED]


def test_host_checks_and_refusals(codecs):
    codec = codecs[True]
    at = lambda n: torch.full((n,), START, dtype=torch.int64, device=DEV)
    tm = codec.element_set(at(2), capi.METRIC_TIMER, [MAX], RES, sample_capacity=8, stride=0)
    off, mem = _dev(np.array([0, 1], dtype=np.int64)), _dev(np.array([0], dtype=np.int32))
    with pytest.raises(ValueError):
        tm.forward_write(START, off, mem, 0)
    with pytest.raises(ValueError):
        tm.add_forwarded([])
    plain = codec.element_set(at(2), COUNTER, [SUM], RES)
    with pytest.raises(ValueError):
        plain.add_forwarded([])
    grp = codec.element_set(at(2), COUNTER, [SUM], RES, source_capacity=32)
    L, ctx, opts = capi.lib(), codec.ctx.handle, C.byref(codec.opts)
    res = torch.zeros(1, dtype=torch.int8, device=DEV)
    st = torch.zeros(2, dtype=torch.int32, device=DEV)
    m = torch.zeros((1, 40), dtype=torch.uint8, device=DEV)
    v = torch.zeros(1, dtype=torch.float64, device=DEV)
    for cap, rsv in ((0, 0), (48, 0), (65536 + 32, 0), (32, 1)):
        s = capi.ElementSources()
        s.d_bits, s.capacity, s.reserved = grp.source_bits.data_ptr(), cap, rsv
        assert L.m3tsz_element_set_add_forwarded(ctx, opts, C.byref(grp._desc()), C.byref(s), m.data_ptr(), 1,
                                                 v.data_ptr(), 1, res.data_ptr(), st.data_ptr(), None) == INV
    s = capi.ElementSources()
    s.d_bits, s.capacity = grp.source_bits.data_ptr(), 32
    assert L.m3tsz_element_set_add_forwarded(ctx, opts, C.byref(tm._desc()), C.byref(s), m.data_ptr(), 1,
                                             v.data_ptr(), 1, res.data_ptr(), st.data_ptr(), None) == INV
    assert L.m3tsz_element_set_add_forwarded(ctx, opts, C.byref(grp._desc()), C.byref(s), m.data_ptr() + 4, 1,
                                             v.data_ptr(), 1, res.data_ptr(), st.data_ptr(), None) == INV
    assert L.m3tsz_element_set_add_forwarded(ctx, opts, C.byref(grp._desc()), None, m.data_ptr(), 1,
                                             v.data_ptr(), 1, res.data_ptr(), st.data_ptr(), None) == INV
    src = codec.element_set(at(2), COUNTER, [SUM], RES, stride=0)
    cnt = torch.zeros(4, dtype=torch.int64, device=DEV)
    gs = torch.zeros(1, dtype=torch.int32, device=DEV)
    call = lambda d, nm, counts: L.m3tsz_element_set_forward_write(
        ctx, opts, C.byref(d), START, off.data_ptr(), mem.data_ptr(), nm, 1, None, 0, m.data_ptr(), 1, v.data_ptr(),
        1, counts, st.data_ptr(), gs.data_ptr(), None)
    assert call(src._desc(), 1, cnt.data_ptr()) == OK
    assert call(src._desc(), (1 << 40) + 1, cnt.data_ptr()) == INV
    assert call(src._desc(), 1, None) == INV
    assert call(tm._desc(), 1, cnt.data_ptr()) == INV
    assert call(plain._desc(), 1, cnt.data_ptr()) == OK  # (a set with output rows forwards too)
    two = codec.element_set(at(2), GAUGE, [MIN, MAX], RES, stride=0)
    assert call(two._desc(), 1, cnt.data_ptr()) == INV
    assert capi.status_string(DUP) == "duplicate forwarding source"


def test_100k_groups(codecs):
    codec = codecs[True]
    rng = np.random.default_rng(21)
    S, G, K, W = 200_000, 100_000, 4, 2
    metric, src_type, pre, types, post = PIPES[0]
    ts = np.zeros((2 * W, S), dtype=np.int64)
    vb = rng.integers(0, 1000, (2 * W, S)).astype(np.float64)
    for w in range(W):
        ts[2 * w] = START + w * RES + rng.integers(0, 30, S) * SEC
        ts[2 * w + 1] = ts[2 * w] + 10 * SEC
    off, mem = _membership(rng, S, G, per=10)
    parts, o1, m1 = _split(off, mem, K)
    one, shards, ref, grp = _world(codec, PIPES[0], S, G, K, False)
    r, st = one.add(_dev(ts), _dev(vb))
    assert int(st.abs().sum()) == 0
    for k, sh in enumerate(shards):
        r, st = sh.add(_dev(ts[:, k::K]), _dev(vb[:, k::K]))
        assert int(st.abs().sum()) == 0
    target = START + W * RES
    one.forward(target, _dev(o1), _dev(m1), ref)
    res, st = grp.add_forwarded(_write_all(shards, target, parts))
    assert int(res.abs().sum()) == 0 and int(st.abs().sum()) == 0
    for f in ref.win:
        a, b = ref.win[f], grp.win[f]
        order_a = torch.argsort(ref.win["start"] + (ref.win["count"] == 0) * (1 << 62), dim=0)
        order_b = torch.argsort(grp.win["start"] + (grp.win["count"] == 0) * (1 << 62), dim=0)
        live = torch.gather(ref.win["count"], 0, order_a) != 0
        assert torch.equal(torch.gather(a, 0, order_a)[live], torch.gather(b, 0, order_b)[live]), f
    assert int(ref.consume(target).abs().sum()) == 0 and int(grp.consume(target).abs().sum()) == 0
    sa, sb = ref.stream(), grp.stream()
    idx = _dev(rng.integers(0, G, 2000))
    assert torch.equal(sa.out_len[idx], sb.out_len[idx]) and torch.equal(sa.out[idx], sb.out[idx])
    assert torch.equal(sa.out_len, sb.out_len)


def test_non_blocking_stream(codecs):
    codec = codecs[True]
    rng = np.random.default_rng(5)
    S, G, W, K = 30, 6, 3, 2
    cols = _cols(rng, S, W, COUNTER)
    off, mem = _membership(rng, S, G)
    parts, o1, m1 = _split(off, mem, K)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        one, shards, ref, grp = _world(codec, PIPES[0], S, G, K, False)
        _add(one, shards, cols, K)
        one.forward(START + W * RES, _dev(o1), _dev(m1), ref)
        res, st = grp.add_forwarded(_write_all(shards, START + W * RES, parts))
        ref.consume(START + W * RES)
        grp.consume(START + W * RES)
    s.synchronize()
    assert int(res.abs().sum()) == 0 and _rows(grp) == _rows(ref)
