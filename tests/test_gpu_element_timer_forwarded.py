"""Timer element-set rollups across shards on the GPU (m3tsz_element_set_forward_write_timer / _add_forwarded_timer,
DESIGN.md §4.12), in both int_optimized modes: sources split over K = 1, 2 and 5 Timer source sets written as
forwarded batches and added to a Timer group set give one m3tsz_element_set_forward_timer over a single set that holds
every source (each group's members listed shard by shard): the group windows matched by start (count, sum, sum_sq and
the CM stream's header and samples), the consumed rows' bytes, the watermarks and the source state.  Against the CPU
model (tests/element_timer_forwarded_model.py): shuffled arrival, keys and invalid groups, redelivery, closed and
invalid records, and both capacity stops with grow and resend.  Also the host checks, 100 k groups, and a run on a
caller's non-blocking stream."""
import ctypes as C

import numpy as np
import pytest
import torch

from element_timer_forwarded_model import (TimerForwardedGroupModel, TimerSourceModel, add_forwarded_timer,
                                           forward_write)
from m3_b200 import capi
from m3_b200.codec import ForwardedBatch
from test_gpu_element_timer_rollup import _bits, _check_group_rows
from test_gpu_element_timers import _point_major, _random_rows, _timer_set
from test_gpu_elements import _rows

pytestmark = pytest.mark.gpu

SEC = 1_000_000_000
RES = 60 * SEC
START = 1_600_000_020 * SEC  # a whole minute
DEV = "cuda"
OK, CAP, INV, CLOSED, DUP = 0, capi.ERR_CAPACITY, capi.ERR_INVALID_ARG, capi.ERR_AGGREGATION_CLOSED, \
    capi.ERR_DUPLICATE_SOURCE
TYPES = [capi.AGG_MAX, capi.AGG_P50, capi.AGG_P99]
STRIDE = 1 << 12
REC_DTYPE = np.dtype([("key", "<u8"), ("time_ns", "<i8"), ("value_off", "<u8"), ("n_values", "<u4"),
                      ("source_id", "<u4"), ("version", "<u4"), ("reserved", "<u4")])


@pytest.fixture(scope="module")
def codecs():
    from m3_b200.codec import BatchCodec
    return {True: BatchCodec(0, int_optimized=True), False: BatchCodec(0, int_optimized=False)}


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _membership(rng, S, G, per=5):
    off = np.arange(0, G * per + 1, per, dtype=np.int64)
    mem = rng.integers(0, S, G * per).astype(np.int32)
    mem[1] = mem[0]  # a member listed twice
    return off, mem


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


def _windows(es):
    """per element {window start: (count, sum, sum_sq, stream header, the stream's used sample entries and pending
    heap entries) as bytes}: the windows, slot placement aside.  (A slot's entries past those are left from the
    windows it held before.)"""
    w = {f: a.cpu().numpy() for f, a in es.win.items()}
    st = {f: a.cpu().numpy() for f, a in es.streams.items()}
    out = []
    for s in range(es.n_elements):
        d = {}
        for r in range(es.open_windows):
            if w["count"][r, s]:
                h = st["header"][r, s]
                n_used, n_a, n_b = (int(h[o: o + 4].view(np.int32)[0]) for o in (36, 48, 52))
                used = {"heap_a": n_a, "heap_b": n_b}
                d[int(w["start"][r, s])] = (tuple(w[f][r, s].tobytes() for f in ("count", "sum", "sum_sq")) +
                                            (h.tobytes(),) + tuple(st[f][r, : used.get(f, n_used), s].tobytes()
                                                                   for f, _ in es._STREAM_ARRAYS))
        out.append(d)
    return out


def _write_all(shards, target, parts):
    batches = []
    for k, (o, m) in enumerate(parts):
        b, st, gst = shards[k].forward_write_timer(target, _dev(o), _dev(m), k)
        assert int(st.abs().sum()) == 0 and int(gst.abs().sum()) == 0
        assert b.counts[0] == b.counts[2] and b.counts[1] == b.counts[3]
        batches.append(b)
    return batches


def _records(b):
    """a ForwardedBatch as model records [(key, time_ns, [values], source_id, version, reserved)]"""
    f = b.fields()
    vals = b.values.cpu().numpy()
    return [(int(f["key"][i]), int(f["time_ns"][i]), vals[f["value_off"][i]: f["value_off"][i] + f["n_values"][i]]
             .tolist(), int(f["source_id"][i]), int(f["version"][i]), int(f["reserved"][i]))
            for i in range(b.metrics.shape[0])]


def _batch(records):
    """model records -> a ForwardedBatch on the device"""
    rec = np.zeros(len(records), dtype=REC_DTYPE)
    vals = []
    for i, (key, t, vs, sid, ver, rsv) in enumerate(records):
        rec[i] = (key, t, len(vals), len(vs), sid, ver, rsv)
        vals += vs
    m = _dev(rec.view(np.uint8).reshape(-1, 40)) if len(records) else \
        torch.zeros((0, 40), dtype=torch.uint8, device=DEV)
    v = _dev(np.array(vals, dtype=np.float64))
    return ForwardedBatch(m, v, (len(records), len(vals), len(records), len(vals)))


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("K", [1, 2, 5])
def test_shards_compose_to_one_forward(codecs, int_opt, K):
    codec = codecs[int_opt]
    rng = np.random.default_rng(10 * K + int_opt)
    S, G, W = 40, 9, 5
    every = [3, 1024][int_opt]
    pre = [capi.TRANSFORM_PERSECOND]
    off, mem = _membership(rng, S, G)
    parts, o1, m1 = _split(off, mem, K)
    cols = [_random_rows(rng, W, batchy=bool(s % 2)) for s in range(S)]
    one = _timer_set(codec, S, [capi.AGG_P99], pre, R=W + 1, cap=512, every=every, stride=0)
    shards = [_timer_set(codec, len(range(k, S, K)), [capi.AGG_P99], pre, R=W + 1, cap=512, every=every, stride=0)
              for k in range(K)]
    ref = _timer_set(codec, G, TYPES, R=W + 1, cap=512, every=every, stride=STRIDE)
    grp = codec.element_set(torch.full((G,), START, dtype=torch.int64, device=DEV), capi.METRIC_TIMER, TYPES, RES,
                            open_windows=W + 1, sample_capacity=512, insert_and_compress_every=every, stride=STRIDE,
                            source_capacity=32)
    ts, vs, n, bt = _point_major(cols)
    r, st = one.add(ts, vs, n, batch=bt)
    assert int(st.abs().sum()) == 0
    for k, sh in enumerate(shards):
        ts, vs, n, bt = _point_major(cols[k::K])
        r, st = sh.add(ts, vs, n, batch=bt)
        assert int(st.abs().sum()) == 0
    for target in (START + 3 * RES, START + (W + 1) * RES):
        sst, gst = one.forward_timer(target, _dev(o1), _dev(m1), ref)
        assert int(sst.abs().sum()) == 0 and int(gst.abs().sum()) == 0
        res, st = grp.add_forwarded_timer(_write_all(shards, target, parts))
        assert int(st.abs().sum()) == 0 and int(res.abs().sum()) == 0
        assert _windows(grp) == _windows(ref)
        assert int(ref.consume(target).abs().sum()) == 0 and int(grp.consume(target).abs().sum()) == 0
        assert torch.equal(grp.watermark, ref.watermark) and torch.equal(grp.elem, ref.elem)
    assert _rows(grp) == _rows(ref)
    for k, sh in enumerate(shards):
        idx = torch.arange(k, S, K, device=DEV)
        assert torch.equal(sh.elem, one.elem[idx]) and torch.equal(sh.watermark, one.watermark[idx])
        for f in sh.win:
            assert torch.equal(_bits(sh.win[f]), _bits(one.win[f][:, idx])), f
        for f in sh.streams:
            a, b = sh.streams[f], one.streams[f]
            assert torch.equal(_bits(a), _bits(b[:, idx] if f == "header" else b[:, :, idx])), f


def _noise(rng, recs, G, clock):
    """redeliveries, invalid records (a key past the elements, a version, no values), late records and a source id
    past the capacity, mixed into a batch"""
    out = list(recs)
    for _ in range(int(rng.integers(3, 9))):
        kind = int(rng.integers(0, 5))
        if kind == 0 and recs:
            out.insert(int(rng.integers(0, len(out) + 1)), recs[int(rng.integers(0, len(recs)))])
        elif kind == 1:
            out.append((int(rng.integers(0, G + 2)), clock, [1.0], 1, int(rng.integers(0, 2)), 0))
        elif kind == 2:
            out.append((int(rng.integers(0, G)), clock, [], 1, 0, 0))
        elif kind == 3:
            out.append((int(rng.integers(0, G)), clock - 6 * RES, [2.0], 3, 0, 0))
        else:
            out.append((int(rng.integers(0, G)), clock, [3.0, float("nan")], 40, 0, 0))
    return out


@pytest.mark.parametrize("int_opt", [True, False])
def test_against_the_model(codecs, int_opt):
    """keys and invalid groups on the writer; shuffled arrival, redelivery, closed and invalid records on the add;
    both capacity stops (open windows and samples) grown and resent; the group rows consumed, against the model"""
    codec = codecs[int_opt]
    rng = np.random.default_rng(3 + int_opt)
    S, G, W, K = 24, 8, 6, 2
    src_type, pre = capi.AGG_MAX, [capi.TRANSFORM_ABSOLUTE]
    srcs = [_timer_set(codec, S, [src_type], pre, R=W + 1, cap=256, every=7, stride=0) for _ in range(K)]
    sms = [[TimerSourceModel(src_type, RES, pre, False, W + 1, 256, 1e-3, 7) for _ in range(S)] for _ in range(K)]
    grp = codec.element_set(torch.full((G,), START, dtype=torch.int64, device=DEV), capi.METRIC_TIMER, TYPES, RES,
                            open_windows=1, sample_capacity=2, insert_and_compress_every=7, stride=STRIDE,
                            source_capacity=32)
    gms = [TimerForwardedGroupModel(TYPES, RES, (), False, 1, 2, 1e-3, 7, source_capacity=32) for _ in range(G)]
    for k in range(K):
        cols = [_random_rows(rng, W, batchy=bool(s % 3 == 0)) for s in range(S)]
        ts, vs, n, bt = _point_major(cols)
        r, st = srcs[k].add(ts, vs, n, batch=bt)
        assert int(st.abs().sum()) == 0
        for s, m in enumerate(sms[k]):
            m.add([(t, v) for t, v, _ in cols[s]], [b for _, _, b in cols[s]])
    memb = []
    for k in range(K):
        off, mem = _membership(rng, S, G, per=3)
        if k == 1:
            mem[2 * 3 + 1] = S + 5  # group 2 lists a source past the sources
            off[5] = off[6] + 1  # group 5's range decreases
        memb.append((off, mem))
    keys = rng.permutation(G).astype(np.int64)
    acc = [[] for _ in range(len(TYPES) * G)]
    stops, seen = set(), set()
    for target in (START + 2 * RES, START + 4 * RES, START + (W + 1) * RES):
        recs = []
        for k in range(K):
            off, mem = memb[k]
            b, sst, gst = srcs[k].forward_write_timer(target, _dev(off), _dev(mem), k, keys=_dev(keys))
            want, wst, wgst, wcounts = forward_write(sms[k], target, off, mem, k, keys)
            assert gst.cpu().tolist() == wgst and sst.cpu().tolist() == wst and b.counts == wcounts
            got = _records(b)
            assert [r[:2] + r[3:] for r in got] == [r[:2] + r[3:] for r in want]
            assert all(np.array(a[2]).tobytes() == np.array(w[2]).tobytes() for a, w in zip(got, want))
            recs += got
        batch = _noise(rng, recs, G, target)
        batch = [batch[i] for i in rng.permutation(len(batch))]
        res, st = grp.add_forwarded_timer(_batch(batch))
        wres, wst = add_forwarded_timer(gms, batch)
        assert res.cpu().tolist() == wres and st.cpu().tolist() == wst
        seen.update(wres)
        for g in range(G):  # which limit stopped each stopped element
            if wst[g] == CAP:
                i = next(i for i, b in enumerate(batch) if b[0] == g and wres[i] == CAP)
                ws, m = batch[i][1] // RES * RES - RES, gms[g]
                stops.add("source id" if batch[i][3] >= 32 else
                          "samples" if ws in m.windows or len(m.windows) < m.R else "windows")
        while CAP in wst:  # grow and resend the refused records, or the whole batch
            grp.grow(open_windows=grp.open_windows + 3, sample_capacity=grp.sample_capacity * 4)
            for m in gms:
                m.R, m.cap = grp.open_windows, grp.sample_capacity
            again = [b for b, x in zip(batch, wres) if x == CAP] if rng.random() < 0.5 else batch
            again = [b for b in again if b[3] < 32]
            res, st = grp.add_forwarded_timer(_batch(again))
            wres, wst = add_forwarded_timer(gms, again)
            assert res.cpu().tolist() == wres and st.cpu().tolist() == wst
            batch = again
        redo = grp.add_forwarded_timer(_batch(recs))[0].cpu().tolist()
        assert redo == add_forwarded_timer(gms, recs)[0] and set(redo) <= {DUP, CLOSED}
        _check_group_rows(codec, grp, gms, target, acc)
    assert seen >= {OK, CAP, INV, CLOSED, DUP}
    assert stops >= {"samples", "windows"}, stops


def test_host_checks_and_refusals(codecs):
    codec = codecs[True]
    at = lambda n: torch.full((n,), START, dtype=torch.int64, device=DEV)
    tm = _timer_set(codec, 2, [capi.AGG_MAX], stride=0)
    tg = codec.element_set(at(2), capi.METRIC_TIMER, TYPES, RES, sample_capacity=8, source_capacity=32)
    plain_tm = _timer_set(codec, 2, TYPES)
    ctr = codec.element_set(at(2), capi.METRIC_COUNTER, [capi.AGG_SUM], RES, stride=0)
    cg = codec.element_set(at(2), capi.METRIC_COUNTER, [capi.AGG_SUM], RES, source_capacity=32)
    off, mem = _dev(np.array([0, 1], dtype=np.int64)), _dev(np.array([0], dtype=np.int32))
    with pytest.raises(ValueError):
        ctr.forward_write_timer(START, off, mem, 0)
    with pytest.raises(ValueError):
        cg.add_forwarded_timer([])
    with pytest.raises(ValueError):
        plain_tm.add_forwarded_timer([])  # (no source_capacity)
    with pytest.raises(ValueError):
        tm.forward_write(START, off, mem, 0)
    with pytest.raises(ValueError):
        tg.add_forwarded([])
    b, sst, gst = tm.forward_write_timer(START, off, mem, 0)
    assert b.counts == (0, 0, 0, 0) and int(gst.abs().sum()) == 0
    res, st = tg.add_forwarded_timer(b)
    assert res.numel() == 0 and int(st.abs().sum()) == 0

    L, ctx, opts = capi.lib(), codec.ctx.handle, C.byref(codec.opts)
    res = torch.zeros(1, dtype=torch.int8, device=DEV)
    st = torch.zeros(2, dtype=torch.int32, device=DEV)
    m = torch.zeros((1, 40), dtype=torch.uint8, device=DEV)
    v = torch.zeros(1, dtype=torch.float64, device=DEV)
    cnt = torch.zeros(4, dtype=torch.int64, device=DEV)
    gs = torch.zeros(1, dtype=torch.int32, device=DEV)
    src = capi.ElementSources()
    src.d_bits, src.capacity = tg.source_bits.data_ptr(), 32

    def write(es, streams, nm=1, counts=cnt.data_ptr()):
        return L.m3tsz_element_set_forward_write_timer(
            ctx, opts, C.byref(es._desc()), streams, START, off.data_ptr(), mem.data_ptr(), nm, 1, None, 0,
            m.data_ptr(), 1, v.data_ptr(), 1, counts, st.data_ptr(), gs.data_ptr(), None)

    def add(es, streams, sources=C.byref(src), metrics=m.data_ptr()):
        return L.m3tsz_element_set_add_forwarded_timer(ctx, opts, C.byref(es._desc()), streams, sources, metrics, 1,
                                                       v.data_ptr(), 1, res.data_ptr(), st.data_ptr(), None)

    assert write(tm, C.byref(tm._streams())) == OK
    assert write(tm, None) == INV
    assert write(tm, C.byref(tm._streams()), nm=(1 << 40) + 1) == INV
    assert write(tm, C.byref(tm._streams()), counts=None) == INV
    assert write(plain_tm, C.byref(plain_tm._streams())) == INV  # three types
    assert write(ctr, C.byref(tm._streams())) == INV  # a Counter set
    bad = tm._streams()
    bad.sample_capacity = 0
    assert write(tm, C.byref(bad)) == INV
    assert add(tg, C.byref(tg._streams())) == OK
    assert add(tg, None) == INV
    assert add(tg, C.byref(tg._streams()), sources=None) == INV
    assert add(tg, C.byref(tg._streams()), metrics=m.data_ptr() + 4) == INV
    assert add(cg, C.byref(tg._streams())) == INV  # a Counter set
    # the Gauge / Counter pair keeps refusing Timer sets
    assert L.m3tsz_element_set_forward_write(
        ctx, opts, C.byref(tm._desc()), START, off.data_ptr(), mem.data_ptr(), 1, 1, None, 0, m.data_ptr(), 1,
        v.data_ptr(), 1, cnt.data_ptr(), st.data_ptr(), gs.data_ptr(), None) == INV
    assert L.m3tsz_element_set_add_forwarded(ctx, opts, C.byref(tg._desc()), C.byref(src), m.data_ptr(), 1,
                                             v.data_ptr(), 1, res.data_ptr(), st.data_ptr(), None) == INV


def test_100k_groups(codecs):
    codec = codecs[True]
    rng = np.random.default_rng(21)
    S, G, K, W = 200_000, 100_000, 4, 2
    ts = np.zeros((2 * W, S), dtype=np.int64)
    vs = np.round(rng.exponential(50, (2 * W, S)), 1)
    for w in range(W):
        ts[2 * w] = START + w * RES + rng.integers(0, 30, S) * SEC
        ts[2 * w + 1] = ts[2 * w] + 10 * SEC
    off, mem = _membership(rng, S, G, per=10)
    parts, o1, m1 = _split(off, mem, K)
    one = _timer_set(codec, S, [capi.AGG_P99], R=W + 1, cap=8, stride=0)
    shards = [_timer_set(codec, len(range(k, S, K)), [capi.AGG_P99], R=W + 1, cap=8, stride=0) for k in range(K)]
    ref = _timer_set(codec, G, TYPES, R=W + 1, cap=32, stride=STRIDE)
    grp = codec.element_set(torch.full((G,), START, dtype=torch.int64, device=DEV), capi.METRIC_TIMER, TYPES, RES,
                            open_windows=W + 1, sample_capacity=32, stride=STRIDE, source_capacity=32)
    r, st = one.add(_dev(ts), _dev(vs))
    assert int(st.abs().sum()) == 0
    for k, sh in enumerate(shards):
        r, st = sh.add(_dev(ts[:, k::K]), _dev(vs[:, k::K]))
        assert int(st.abs().sum()) == 0
    target = START + W * RES
    sst, gst = one.forward_timer(target, _dev(o1), _dev(m1), ref)
    assert int(gst.abs().sum()) == 0
    res, st = grp.add_forwarded_timer(_write_all(shards, target, parts))
    assert int(res.abs().sum()) == 0 and int(st.abs().sum()) == 0
    order = lambda es: torch.argsort(es.win["start"] + (es.win["count"] == 0) * (1 << 62), dim=0)
    oa, ob = order(ref), order(grp)
    live = torch.gather(ref.win["count"], 0, oa) != 0
    for f in ref.win:
        a, b = _bits(ref.win[f]), _bits(grp.win[f])
        assert torch.equal(torch.gather(a, 0, oa)[live], torch.gather(b, 0, ob)[live]), f
    assert int(ref.consume(target).abs().sum()) == 0 and int(grp.consume(target).abs().sum()) == 0
    sa, sb = ref.stream(), grp.stream()
    assert torch.equal(sa.out_len, sb.out_len)
    idx = _dev(rng.integers(0, sa.out.shape[0], 2000))
    assert torch.equal(sa.out[idx], sb.out[idx])


def test_non_blocking_stream(codecs):
    codec = codecs[True]
    rng = np.random.default_rng(5)
    S, G, W, K = 30, 6, 3, 2
    off, mem = _membership(rng, S, G)
    parts, o1, m1 = _split(off, mem, K)
    cols = [_random_rows(rng, W, batchy=True) for s in range(S)]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        one = _timer_set(codec, S, [capi.AGG_P50], R=W + 1, cap=256, stride=0)
        shards = [_timer_set(codec, len(range(k, S, K)), [capi.AGG_P50], R=W + 1, cap=256, stride=0)
                  for k in range(K)]
        ref = _timer_set(codec, G, TYPES, R=W + 1, cap=64, stride=STRIDE)
        grp = codec.element_set(torch.full((G,), START, dtype=torch.int64, device=DEV), capi.METRIC_TIMER, TYPES,
                                RES, open_windows=W + 1, sample_capacity=64, stride=STRIDE, source_capacity=32)
        ts, vs, n, bt = _point_major(cols)
        one.add(ts, vs, n, batch=bt)
        for k, sh in enumerate(shards):
            ts, vs, n, bt = _point_major(cols[k::K])
            sh.add(ts, vs, n, batch=bt)
        torch.cuda._sleep(50_000_000)
        one.forward_timer(START + W * RES, _dev(o1), _dev(m1), ref)
        res, st = grp.add_forwarded_timer(_write_all(shards, START + W * RES, parts))
        ref.consume(START + W * RES)
        grp.consume(START + W * RES)
    s.synchronize()
    assert int(res.abs().sum()) == 0 and int(st.abs().sum()) == 0 and _rows(grp) == _rows(ref)
