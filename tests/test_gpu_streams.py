"""The device entry points on a caller's non-blocking stream, and one context shared by calls on several streams.

Every call here runs behind torch.cuda._sleep on a torch pool stream (non-blocking, so work left on the legacy stream
is not ordered against it):

(a) a call whose inputs are copied over valid decoys after the sleep, on the same stream, gives byte for byte what it
    gives on the default stream: a call that ran any of its work on another stream would read a decoy;
(b) the whole sweep completes on its stream while a sleep still holds the legacy default stream;
(c) a call returns before its stream has run it, except for the device entry points the header lists as blocking;
(d) calls that use the context's scratch are ordered in the order they are issued, whatever their streams: a device
    call on one stream and a later one on another, or a later *_host call, never run before the earlier call.

Decoys and real inputs share every shape: streams sit in fixed-stride slots, so a misordered read sees the decoy's
streams, never an address outside the buffers."""
import ctypes as C
import os
import re
import time

import numpy as np
import pytest
import torch

from m3_b200 import capi
from m3_b200.codec import DecodeResult, DownsampleResult, EncodeResult, PackedResult

pytestmark = pytest.mark.gpu

SEC = 1_000_000_000
START = 1_599_955_200 * SEC  # day-aligned
S, P = 96, 48  # S even (point-major encode: the TMA input stage); S - 1 odd (the cp.async stage)
WIN = 300 * SEC
NW = 12
TARGET = START + 6 * WIN
SENT = 0xA5  # every output byte a call does not write keeps it
LAST, MIN, MAX, SUM = capi.AGG_LAST, capi.AGG_MIN, capi.AGG_MAX, capi.AGG_SUM
ADD = capi.TRANSFORM_ADD
HEADER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "include", "m3tsz_b200.h")

# the device entry points include/m3tsz_b200.h lists as blocking the host
BLOCKING = {"m3tsz_compact_streams", "m3tsz_aggregate_tiles_annotated", "m3tsz_aggregate_tiles_blocks",
            "m3tsz_aggregate_tiles_rollup_annotated"}


@pytest.fixture(scope="module")
def codec():
    from m3_b200.codec import BatchCodec
    return BatchCodec(0, int_optimized=True)


# ---------------------------------------------------------------------------------------------------- inputs
def _inputs(codec, seed):
    """One valid batch: S series of P datapoints (irregular timestamps, values of two decimals), their encoded
    streams in slots of one stride, and every index the calls below take.  Same shapes for every seed."""
    rng = np.random.default_rng(seed)
    dt = rng.integers(20, 100, size=(S, P)) * SEC
    ts = START + np.cumsum(dt, axis=1) - dt[:, :1]
    vals = np.round(100 + np.cumsum(rng.normal(0, 1, size=(S, P)), axis=1), 2)
    n = rng.integers(P // 2, P + 1, size=S).astype(np.int32)
    d = {"ts": torch.from_numpy(ts).cuda(), "vals": torch.from_numpy(vals).cuda(),
         "start": torch.full((S,), START, dtype=torch.int64, device="cuda"),
         "n": torch.from_numpy(n).cuda()}
    d["tsT"], d["valsT"] = d["ts"].t().contiguous(), d["vals"].t().contiguous()
    enc = codec.encode(d["ts"], d["vals"], d["start"], unit=capi.UNIT_S, n_points=d["n"])
    torch.cuda.synchronize()
    assert int(enc.status.abs().sum()) == 0
    stride = enc.out.shape[1]
    keep = torch.arange(stride, device="cuda")[None, :] < enc.out_len[:, None]
    d["blob"] = (enc.out * keep).reshape(-1).contiguous()  # zero past each stream's end
    d["len"] = enc.out_len.clone()
    d["off_csr"] = torch.arange(S + 1, dtype=torch.int64, device="cuda") * stride
    d["off"] = d["off_csr"][:S].contiguous()
    # out-of-order halves for the buffer buckets: the second half of every series first
    h = P // 2
    d["ts_ooo"] = torch.cat([d["ts"][:, h:], d["ts"][:, :h]], 1).contiguous()
    d["vals_ooo"] = torch.cat([d["vals"][:, h:], d["vals"][:, :h]], 1).contiguous()
    return d


@pytest.fixture(scope="module")
def real(codec):
    return _inputs(codec, 1)


@pytest.fixture(scope="module")
def decoy(codec):
    return _inputs(codec, 2)


def _full(shape, dtype):
    t = torch.empty(shape, dtype=dtype, device="cuda")
    t.view(-1).view(torch.uint8).fill_(SENT)
    return t


def _stream_ptr():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _i32s(*xs):
    return (C.c_int32 * len(xs))(*xs)


# ---------------------------------------------------------------------------------------------------- the calls
# Each case makes its calls on the current stream from the input dict d and returns the tensors it produced or
# changed; `post` (optional) turns their host copies into what must match.

def _events_post(a):
    """the event table is filled in whatever order the series reach it: its rows sorted"""
    ev = a[6]
    return a[:6] + [ev[np.lexsort(ev.T[::-1])], a[7]]


def _decode(point_major=False, lengths=False, events=0):
    def fn(codec, d):
        shape = (P, S) if point_major else (S, P)
        out = DecodeResult(ts=_full(shape, torch.int64), values=_full(shape, torch.float64),
                           n_points=_full(S, torch.int32), status=_full(S, torch.int32), unit=_full(S, torch.uint8),
                           annotations=None)
        off = d["off"] if lengths else d["off_csr"]
        r = codec.decode(d["blob"], off, P, out=out, lengths=d["len"] if lengths else None, want_events=events,
                         point_major=point_major)
        return [r.ts, r.values, r.n_points, r.status, r.unit] + ([r.unit_first, r.events, r.event_count]
                                                                  if events else [])
    return fn


def _downsample(kind):
    def fn(codec, d):
        counter = kind == "counter"
        agg = torch.int64 if counter else torch.float64
        mk = lambda dt: _full((NW, S), dt)
        out = DownsampleResult(sum=mk(agg), count=mk(torch.int64), min=mk(agg), max=mk(agg),
                               n_points=_full(S, torch.int32), status=_full(S, torch.int32),
                               last=mk(torch.float64) if kind == "last" else None,
                               last_at=mk(torch.int64) if kind == "last" else None,
                               # the Gauge's sumSq without last / lastAt, and the Counter without sumSq: the
                               # kernel keeps those in context scratch
                               sum_sq=mk(agg) if kind == "sumsq" else None,
                               metric=capi.METRIC_COUNTER if counter else capi.METRIC_GAUGE)
        if kind in ("plain", "last"):
            r = codec.decode_downsample(d["blob"], d["off_csr"], START, WIN, NW, out=out, want_last=kind == "last")
        else:
            r = codec._decode_downsample_ex(d["blob"], d["off_csr"], START, WIN, NW, out, False,
                                            out.metric, kind == "sumsq", None)
        return [t for t in (r.sum, r.count, r.min, r.max, r.n_points, r.status, r.last, r.last_at, r.sum_sq)
                if t is not None]
    return fn


def _encode(point_major=False, odd=False):
    def fn(codec, d):
        n = S - 1 if odd else S
        stride = codec.encode_bound(P)
        out = EncodeResult(out=_full((n, stride), torch.uint8), out_len=_full(n, torch.int64),
                           status=_full(n, torch.int32))
        if point_major:
            ts, vals = (d["tsT"][:, :n].contiguous(), d["valsT"][:, :n].contiguous()) if odd else (d["tsT"], d["valsT"])
        else:
            ts, vals = d["ts"], d["vals"]
        r = codec.encode(ts, vals, d["start"][:n], n_points=d["n"][:n], out=out, point_major=point_major)
        return [r.out, r.out_len, r.status]
    return fn


def _packed_canon(packed, offsets, out_len, total):
    """a packed buffer whose streams sit in completion order: the streams in row order, and the bytes past the end"""
    packed, offsets, out_len = packed.reshape(-1), offsets.reshape(-1), out_len.reshape(-1)
    end = int(total.reshape(-1)[0])
    rows = [packed[o: o + n].tobytes() if 0 <= o and o + n <= packed.size else b"?"
            for o, n in zip(offsets.tolist(), out_len.tolist())]
    return [np.frombuffer(b"|".join(rows), dtype=np.uint8), packed[end:]]


def _encode_packed(codec, d):
    cap = S * codec.encode_bound(P)
    out = PackedResult(packed=_full(cap, torch.uint8), offsets=_full(S, torch.int64), out_len=_full(S, torch.int64),
                       status=_full(S, torch.int32), total=_full(1, torch.int64))
    r = codec.encode_packed(d["ts"], d["vals"], d["start"], n_points=d["n"], align=64, out=out)
    return [r.packed, r.offsets, r.out_len, r.status, r.total]


def _encode_packed_post(a):
    return _packed_canon(a[0], a[1], a[2], a[4]) + a[2:]


def _compact(codec, d):
    stride = codec.encode_bound(P)
    enc = EncodeResult(out=_full((S, stride), torch.uint8), out_len=_full(S, torch.int64),
                       status=_full(S, torch.int32))
    codec.encode(d["ts"], d["vals"], d["start"], n_points=d["n"], out=enc)
    packed, offsets = codec.compact(enc, align=16, capacity=S * (stride + 16))
    return [packed, offsets, enc.out_len, enc.status]


def _compact_post(a):
    """the streams at their offsets (the alignment padding between them is not written)"""
    packed, offsets, out_len = a[:3]
    rows = [packed[o: o + n].tobytes() for o, n in zip(offsets[:-1].tolist(), out_len.tolist())]
    return [np.frombuffer(b"|".join(rows), dtype=np.uint8)] + a[1:]


def _encoder_set(codec, d):
    es = codec.encoder_set(d["start"], codec.encode_bound(P))
    h = P // 2
    n1, s1 = es.append(d["ts"][:, :h].contiguous(), d["vals"][:, :h].contiguous())
    n2, s2 = es.append(d["ts"][:, h:].contiguous(), d["vals"][:, h:].contiguous(), n_points=d["n"] - h)
    snap = es.stream()
    return [es.state, es.buf, snap.out_len, n1, s1, n2, s2]


def _bucket_write(codec, d):
    bs = codec.bucket_set(d["start"], codec.encode_bound(P), encoders=4, pool_records=2 * S)
    h = P // 2
    r1, s1 = bs.write(d["ts_ooo"][:, :h].contiguous(), d["vals_ooo"][:, :h].contiguous())
    r2, s2 = bs.write(d["ts_ooo"][:, h:].contiguous(), d["vals_ooo"][:, h:].contiguous())
    pr = bs.primary
    return [pr.state, pr.buf, bs.pool, bs.pool_buf, bs.pool_count, bs.table, r1, s1, r2, s2]


def _bucket_post(a):
    """overflow records are taken from the pool in whatever order the series get there: each series' encoders in
    encoder order, whichever records hold them"""
    state, buf, pool, pool_buf, count, table = a[:6]
    rec = np.where(table >= 0, table, 0)
    opened = (table >= 0)[:, :, None]
    return [state, buf, np.where(opened, pool[rec], 0), np.where(opened, pool_buf[rec], 0), count,
            table >= 0] + a[6:]


class _TileOut:
    """sentinel-filled packed outputs for up to two rows per series, and the records a tile call may carry"""

    def __init__(self, codec, n_src):
        n = 2 * n_src
        self.cap = n * (codec.encode_bound(NW) + codec.encode_bound(P) + 64)
        self.packed = _full(self.cap, torch.uint8)
        self.offsets, self.out_len = _full(n, torch.int64), _full(n, torch.int64)
        self.status, self.n_tiles = _full(n, torch.int32), _full(n, torch.int32)
        self.total = _full(1, torch.int64)
        self.src_status = _full(n_src, torch.int32)

    def args(self):
        return (64, self.packed.data_ptr(), self.cap, self.offsets.data_ptr(), self.out_len.data_ptr(),
                self.status.data_ptr(), self.n_tiles.data_ptr(), self.total.data_ptr())

    def tensors(self):
        return [self.packed, self.offsets, self.out_len, self.status, self.n_tiles, self.total, self.src_status]


TILE_FN = {"batch": "m3tsz_aggregate_tiles_batch", "ex": "m3tsz_aggregate_tiles_ex",
           "transform": "m3tsz_aggregate_tiles_transform", "types": "m3tsz_aggregate_tiles_types",
           "annotated": "m3tsz_aggregate_tiles_annotated", "blocks": "m3tsz_aggregate_tiles_blocks",
           "blocks_annotated": "m3tsz_aggregate_tiles_blocks", "rollup": "m3tsz_aggregate_tiles_rollup",
           "rollup_annotated": "m3tsz_aggregate_tiles_rollup_annotated"}


def _tiles(name):
    def fn(codec, d):
        L, h, o = capi.lib(), codec.ctx.handle, C.byref(codec.opts)
        src = (d["blob"].data_ptr(), d["blob"].numel(), d["off_csr"].data_ptr(), None)
        out = _TileOut(codec, S)
        st = _stream_ptr()
        if name == "batch":
            rc = L.m3tsz_aggregate_tiles_batch(h, o, *src, S, START, WIN, NW, LAST, capi.UNIT_S, *out.args(), st)
            return [rc] + out.tensors()
        if name == "ex":
            rc = L.m3tsz_aggregate_tiles_ex(h, o, *src, S, START, WIN, NW, capi.METRIC_COUNTER, SUM, capi.UNIT_S,
                                            *out.args(), st)
            return [rc] + out.tensors()
        if name == "transform":
            state = codec.transform_state(S)
            rc = L.m3tsz_aggregate_tiles_transform(h, o, *src, S, START, WIN, NW, capi.METRIC_GAUGE, LAST,
                                                   capi.UNIT_S, *out.args(), _i32s(ADD), 1, 1, state.data_ptr(), st)
            return [rc, state] + out.tensors()
        state = codec.element_state(S)
        if name in ("types", "annotated"):
            f = L.m3tsz_aggregate_tiles_types if name == "types" else L.m3tsz_aggregate_tiles_annotated
            rc = f(h, o, *src, S, START, WIN, NW, capi.METRIC_GAUGE, _i32s(MIN, MAX), 2, capi.UNIT_S, *out.args(),
                   _i32s(ADD), 1, 1, state.data_ptr(), st)
            return [rc, state] + out.tensors()
        if name in ("blocks", "blocks_annotated"):
            blocks = torch.arange(S + 1, dtype=torch.int64, device="cuda")  # one source block per series
            rc = L.m3tsz_aggregate_tiles_blocks(h, o, *src, S, blocks.data_ptr(), S, START, WIN, NW,
                                                capi.METRIC_GAUGE, _i32s(MIN, MAX), 2, capi.UNIT_S, *out.args(),
                                                _i32s(ADD), 1, 1, state.data_ptr(),
                                                1 if name == "blocks_annotated" else 0, st)
            return [rc, state] + out.tensors()
        # group g: sources 3g .. 3g + 2
        G = S // 3
        group_off = torch.arange(0, S + 1, 3, dtype=torch.int64, device="cuda")
        members = torch.arange(S, dtype=torch.int32, device="cuda")
        src_state, group_state = codec.transform_state(S), codec.element_state(G)
        f = getattr(L, TILE_FN[name])
        rc = f(h, o, *src, S, None, S, START, WIN, NW, capi.METRIC_GAUGE, SUM, _i32s(ADD), 1, group_off.data_ptr(),
               members.data_ptr(), S, G, _i32s(MIN, MAX), 2, _i32s(ADD), 1, 1, src_state.data_ptr(),
               group_state.data_ptr(), capi.UNIT_S, *out.args(), out.src_status.data_ptr(), st)
        return [rc, src_state, group_state] + out.tensors()
    return fn


def _tiles_post(a):
    rc, rest = a[0], a[1:]
    packed, offsets, out_len, status, n_tiles, total, src_status = rest[-7:]
    assert int(rc[0]) == 0, int(rc[0])
    return rest[:-7] + _packed_canon(packed, offsets, out_len, total) + [out_len, status, n_tiles, total, src_status]


def _element_set(annotated):
    def fn(codec, d):
        es = codec.element_set(d["start"], capi.METRIC_GAUGE, [MIN, MAX], WIN, open_windows=NW + 2,
                               annotation_capacity=16 if annotated else 0)
        r, st = es.add(d["tsT"], d["valsT"], d["n"])
        cst = es.consume(TARGET)
        snap = es.stream()
        return list(es.win.values()) + [es.elem, es.watermark, es.out.state, es.out.buf, snap.out_len, r, st, cst] + (
            [es.ann_len, es.ann_bytes] if annotated else [])
    return fn


def _element_forward(codec, d):
    G = S // 3
    group_off = torch.arange(0, S + 1, 3, dtype=torch.int64, device="cuda")
    members = torch.arange(S, dtype=torch.int32, device="cuda")
    src = codec.element_set(d["start"], capi.METRIC_GAUGE, [SUM], WIN, open_windows=NW + 2, stride=0)
    groups = codec.element_set(d["start"][:G].contiguous(), capi.METRIC_GAUGE, [MIN, MAX], WIN,
                               open_windows=NW + 2)
    r, st = src.add(d["tsT"], d["valsT"], d["n"])
    sst, gst = src.forward(TARGET, group_off, members, groups)
    cst = groups.consume(TARGET)
    snap = groups.stream()
    return (list(src.win.values()) + [src.elem, src.watermark] + list(groups.win.values()) +
            [groups.elem, groups.watermark, groups.out.buf, groups.out.state, snap.out_len, r, st, sst, gst, cst])


def _merge(point_major):
    def fn(codec, d):
        ident = torch.arange(S + 1, dtype=torch.int64, device="cuda")
        series_off = torch.arange(0, S + 1, 3, dtype=torch.int64, device="cuda")  # three replicas per series
        seq_status = torch.zeros(S, dtype=torch.int32, device="cuda")
        ts, vals = (d["tsT"], d["valsT"]) if point_major else (d["ts"], d["vals"])
        t, v, n, st = codec.merge_series(ts, vals, d["n"], seq_status, ident, ident, series_off, 2 * P,
                                         point_major=point_major)
        return [t, v, n, st, torch.tensor([1 if point_major else 0])]
    return fn


def _rows_post(a):
    """(ts [R, cap] or [cap, R] when a[-1] says point-major, values, n [R], status): the rows' first n entries"""
    t, v, n, st = a[:4]
    pm = len(a) > 4 and int(a[4][0]) == 1
    if pm:
        t, v = t.T, v.T
    keep = np.arange(t.shape[1])[None, :] < n[:, None]
    return [np.where(keep, t, 0), np.where(keep, v.view(np.int64), 0), n, st]


def _prom(codec, d):
    t, v, n, st = codec.prom_convert(d["ts"], d["vals"], d["n"])
    return [t, v, n, st]


def _checksum(codec, d):
    c, st = codec.segment_checksums(d["blob"], d["off"], lengths=d["len"])
    return [c, st]


# name -> (the calls, post, the C entry points it makes)
CASES = {
    "decode": (_decode(), None, {"m3tsz_decode_batch_ex"}),
    "decode_point_major": (_decode(point_major=True), None, {"m3tsz_decode_batch_ex"}),
    "decode_lengths": (_decode(lengths=True), None, {"m3tsz_decode_batch_ex"}),
    "decode_events": (_decode(events=64), _events_post, {"m3tsz_decode_batch_ex"}),
    "downsample": (_downsample("plain"), None, {"m3tsz_decode_downsample_batch"}),
    "downsample_last": (_downsample("last"), None, {"m3tsz_decode_downsample_last_batch"}),
    "downsample_ex_sumsq": (_downsample("sumsq"), None, {"m3tsz_decode_downsample_ex"}),
    "downsample_ex_counter": (_downsample("counter"), None, {"m3tsz_decode_downsample_ex"}),
    "encode": (_encode(), None, {"m3tsz_encode_batch_ex"}),
    "encode_point_major_even": (_encode(point_major=True), None, {"m3tsz_encode_batch_ex"}),
    "encode_point_major_odd": (_encode(point_major=True, odd=True), None, {"m3tsz_encode_batch_ex"}),
    "encode_packed": (_encode_packed, _encode_packed_post, {"m3tsz_encode_batch_packed_ex"}),
    "compact": (_compact, _compact_post, {"m3tsz_encode_batch_ex", "m3tsz_compact_streams"}),
    "encoder_set": (_encoder_set, None, {"m3tsz_encoder_set_reset", "m3tsz_encoder_set_append",
                                         "m3tsz_encoder_set_stream"}),
    "bucket_write": (_bucket_write, _bucket_post, {"m3tsz_encoder_set_reset", "m3tsz_encoder_set_write"}),
    "element_set": (_element_set(False), None, {"m3tsz_element_set_reset", "m3tsz_element_set_add",
                                                "m3tsz_element_set_consume", "m3tsz_encoder_set_stream"}),
    "element_set_annotated": (_element_set(True), None, {"m3tsz_element_set_reset",
                                                         "m3tsz_element_set_add_annotated",
                                                         "m3tsz_element_set_consume_annotated",
                                                         "m3tsz_encoder_set_stream"}),
    "element_forward": (_element_forward, None, {"m3tsz_element_set_reset", "m3tsz_element_set_add",
                                                 "m3tsz_element_set_forward", "m3tsz_element_set_consume",
                                                 "m3tsz_encoder_set_stream"}),
    "merge": (_merge(False), _rows_post, {"m3tsz_merge_series_batch_ex"}),
    "merge_point_major": (_merge(True), _rows_post, {"m3tsz_merge_series_batch_ex"}),
    "prom_convert": (_prom, _rows_post, {"m3tsz_prom_convert_batch"}),
    "checksum": (_checksum, None, {"m3tsz_checksum_batch"}),
}
for _t in TILE_FN:
    # (blocks without annotations makes the same C call as blocks_annotated, but does not block)
    CASES["tiles_" + _t] = (_tiles(_t), _tiles_post,
                            {"m3tsz_aggregate_tiles_blocks(plain)" if _t == "blocks" else TILE_FN[_t]})


def _blocks_host(name):
    return bool(CASES[name][2] & BLOCKING)


def _host(fn, post, tensors):
    torch.cuda.synchronize()
    a = [t.cpu().numpy() if isinstance(t, torch.Tensor) else np.array([t]) for t in tensors]
    return post(a) if post else a


def _same(got, want, what):
    assert len(got) == len(want), what
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape and g.dtype == w.dtype, (what, i, g.shape, w.shape)
        assert g.tobytes() == w.tobytes(), (what, i)


# ---------------------------------------------------------------------------------------------------- sleeps
@pytest.fixture(scope="module")
def cycles_per_s():
    """the spin kernel's clock rate, timed once with events"""
    torch.cuda._sleep(1000)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 50_000_000
    e0.record()
    torch.cuda._sleep(n)
    e1.record()
    e1.synchronize()
    return n / (e0.elapsed_time(e1) / 1e3)


def _sleep(cycles_per_s, seconds):
    assert seconds <= 1.0
    torch.cuda._sleep(int(cycles_per_s * seconds))


@pytest.fixture(scope="module")
def reference(codec, real):
    """every case on the default stream over the real inputs, run twice (the second run warms the first's scratch
    sizes and allocations); the two must agree"""
    ref = {}
    for name, (fn, post, _) in CASES.items():
        a = _host(fn, post, fn(codec, dict(real)))
        _same(_host(fn, post, fn(codec, dict(real))), a, name + " (repeat)")
        ref[name] = a
    return ref


def _warm(codec, real, stream):
    """the whole sweep on `stream`, twice: the allocator then holds blocks for every call's tensors there, and
    the context's scratch has the sizes of these shapes"""
    for _ in range(2):
        with torch.cuda.stream(stream):
            for fn, _, _ in CASES.values():
                fn(codec, dict(real))
        stream.synchronize()


@pytest.fixture(scope="module")
def side(codec, real, reference):
    st = torch.cuda.Stream()
    _warm(codec, real, st)
    return st


@pytest.fixture(scope="module")
def streams2(codec, real, reference):
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    _warm(codec, real, s1)
    _warm(codec, real, s2)
    return s1, s2


# ---------------------------------------------------------------------------------------------------- (a)
@pytest.mark.parametrize("name", list(CASES))
def test_side_stream_over_decoys(codec, real, decoy, reference, side, cycles_per_s, name):
    """inputs copied over decoys behind a sleep, on the call's stream: the call sees only the real inputs, and
    writes what it writes on the default stream"""
    fn, post, _ = CASES[name]
    bufs = {k: v.clone() for k, v in decoy.items()}
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        _sleep(cycles_per_s, 0.05)
        for k, v in bufs.items():
            v.copy_(real[k])
        res = fn(codec, bufs)
    side.synchronize()
    _same(_host(fn, post, res), reference[name], name)


def test_decoys_differ(codec, real, decoy, reference):
    """the decoys are a different batch: a call that read them would give other results"""
    for name, (fn, post, _) in CASES.items():
        got = _host(fn, post, fn(codec, dict(decoy)))
        assert any(g.tobytes() != w.tobytes() for g, w in zip(got, reference[name])), name


# ---------------------------------------------------------------------------------------------------- (b)
def test_no_dependence_on_legacy_stream(codec, real, reference, side, cycles_per_s):
    """with the legacy default stream held by a sleep, the whole sweep completes on a pool stream"""
    results = {}
    torch.cuda.synchronize()
    _sleep(cycles_per_s, 1.0)  # on the legacy default stream
    with torch.cuda.stream(side):
        for name, (fn, _, _) in CASES.items():
            results[name] = fn(codec, dict(real))
    side.synchronize()
    held = not torch.cuda.default_stream().query()
    torch.cuda.synchronize()
    assert held, "a call waited for the legacy default stream"
    for name, (fn, post, _) in CASES.items():
        _same(_host(fn, post, results[name]), reference[name], name)


# ---------------------------------------------------------------------------------------------------- (c)
def _header_blocking():
    text = open(HEADER).read()
    m = re.search(r"Device entry points that block the host(.*?)\n \*\n", text, re.S)
    assert m, "the header's list of blocking device entry points"
    return set(re.findall(r"m3tsz_\w+", m.group(1)))


def test_blocking_list_is_the_headers():
    assert _header_blocking() == BLOCKING


@pytest.mark.parametrize("name", list(CASES))
def test_which_calls_block(codec, real, reference, side, cycles_per_s, name):
    """a call behind a sleep returns before its stream runs it, unless the header lists it as blocking, in which
    case it waits for the sleep"""
    fn, post, _ = CASES[name]
    secs = 0.3
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        _sleep(cycles_per_s, secs)
        t0 = time.perf_counter()
        res = fn(codec, dict(real))
        took = time.perf_counter() - t0
        pending = not side.query()
    side.synchronize()
    _same(_host(fn, post, res), reference[name], name)
    if _blocks_host(name):
        assert took > secs / 2, "%s is listed as blocking but returned after %.3f s" % (name, took)
    else:
        assert pending, "%s blocked the host (%.3f s)" % (name, took)


# ---------------------------------------------------------------------------------------------------- (d)
def _host_inputs(real):
    return real["blob"].cpu(), real["off_csr"].cpu()


def _downsample_host(codec, real):
    hb, ho = _host_inputs(real)
    f = lambda dt: torch.full((NW, S), -7, dtype=dt)
    outs = [f(torch.float64), f(torch.int64), f(torch.float64), f(torch.float64),
            torch.full((S,), -7, dtype=torch.int32), torch.full((S,), -7, dtype=torch.int32)]
    codec.decode_downsample_host(hb, ho, START, WIN, NW, *outs)
    return [t.numpy() for t in outs]


def _decode_host(codec, real):
    hb, ho = _host_inputs(real)
    outs = [torch.full((S, P), -7, dtype=torch.int64), torch.full((S, P), -7, dtype=torch.float64),
            torch.full((S,), -7, dtype=torch.int32), torch.full((S,), -7, dtype=torch.int32)]
    codec.decode_host(hb, ho, P, *outs)
    return [t.numpy() for t in outs]


def _encode_host(codec, real):
    ts, vals, start = real["ts"].cpu(), real["vals"].cpu(), real["start"].cpu()
    cap = S * codec.encode_bound(P)
    packed = torch.full((cap,), SENT, dtype=torch.uint8)
    offsets = torch.full((S + 1,), -7, dtype=torch.int64)
    out_len = torch.full((S,), -7, dtype=torch.int64)
    status = torch.full((S,), -7, dtype=torch.int32)
    codec.encode_host(ts, vals, start, capi.UNIT_S, packed, offsets, out_len, status, align=16)
    return [packed.numpy()[: int(offsets[-1])], offsets.numpy(), out_len.numpy(), status.numpy()]


HOST_CALLS = {"downsample_host": _downsample_host, "decode_host": _decode_host, "encode_host": _encode_host}

# (device call A, host call B): B uses scratch slots A uses (the windows, n_points / status), or, for compaction
# and the host encode, the context's overflow flag
DEVICE_THEN_HOST = [("tiles_batch", "downsample_host"), ("tiles_types", "downsample_host"),
                    ("tiles_rollup", "downsample_host"), ("downsample_ex_sumsq", "downsample_host"),
                    ("tiles_ex", "decode_host"), ("element_set", "decode_host"), ("compact", "encode_host")]


@pytest.mark.parametrize("a,b", DEVICE_THEN_HOST)
def test_host_call_waits_for_device_call(codec, real, reference, streams2, cycles_per_s, a, b):
    """a device call A on one stream behind a sleep, then a *_host call B on the same context: B returns after A
    has run, and both give what they give alone"""
    fn, post, _ = CASES[a]
    alone_b = HOST_CALLS[b](codec, real)  # (also sizes B's scratch before A is queued)
    s1 = streams2[0]
    torch.cuda.synchronize()
    with torch.cuda.stream(s1):
        _sleep(cycles_per_s, 0.3)
        res = fn(codec, dict(real))
    got_b = HOST_CALLS[b](codec, real)
    a_ran = s1.query()
    s1.synchronize()
    assert a_ran, "%s returned before the earlier %s ran" % (b, a)
    _same(_host(fn, post, res), reference[a], a)
    _same(got_b, alone_b, b)


# (A on stream 1, B on stream 2), both using context scratch
TWO_STREAMS = [("tiles_types", "tiles_ex"), ("tiles_batch", "downsample_ex_sumsq"),
               ("tiles_ex", "downsample_ex_counter"), ("tiles_rollup", "tiles_annotated"),
               ("tiles_batch", "encode_packed"), ("encode_packed", "tiles_blocks"),
               ("bucket_write", "bucket_write"), ("element_set", "element_set_annotated"),
               ("element_forward", "element_set"), ("tiles_transform", "compact"),
               ("downsample_ex_counter", "tiles_rollup_annotated")]


@pytest.mark.parametrize("a,b", TWO_STREAMS)
def test_two_streams_one_context(codec, real, reference, streams2, cycles_per_s, a, b):
    """A on stream 1 behind a sleep, then B on stream 2 of the same context: B's stream does not complete before
    A has run, and both give what they give alone"""
    (fa, pa, _), (fb, pb, _) = CASES[a], CASES[b]
    s1, s2 = streams2
    torch.cuda.synchronize()
    with torch.cuda.stream(s1):
        _sleep(cycles_per_s, 0.3)
        ra = fa(codec, dict(real))
    with torch.cuda.stream(s2):
        rb = fb(codec, dict(real))
    b_waits = _blocks_host(b) or not s2.query()
    s2.synchronize()
    a_ran = s1.query()
    s1.synchronize()
    assert a_ran, "%s on its stream completed before the earlier %s ran" % (b, a)
    assert b_waits
    _same(_host(fa, pa, ra), reference[a], a)
    _same(_host(fb, pb, rb), reference[b], b)
