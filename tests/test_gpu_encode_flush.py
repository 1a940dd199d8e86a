"""GPU encode: what the output tile's flushes may and may not write.

Every flush of the encoder moves a warp's tile to 32 output streams at once.  These tests put lanes that flush
very different amounts into the same warp (int-like next to float series, constant next to random, ragged lengths,
lanes without a series, long annotations on a few lanes, series that run out of capacity) and check, for every
stream, the bytes up to `out_len`, the zero padding up to the next 16-byte boundary, and that nothing else in the
stream's slot or in its neighbours' slots was written."""
import numpy as np
import pytest

import oracle_lib as O

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
SEC = 1_000_000_000
START = 1599955200 * SEC
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def codecs():
    from m3_b200.codec import BatchCodec
    return {True: BatchCodec(0, True), False: BatchCodec(0, False)}


def _mixed(S, P, seed):
    """[S, P] inputs whose neighbouring series produce very different amounts of output: random-walk floats,
    int-like counters, constants, 2-digit decimals, full-width random doubles and repeats, by s % 6.  n_points
    is ragged: 0, 1, P and every length up to min(63, P) appear, so some series end right after a flush."""
    rng = np.random.default_rng(seed)
    ts = START + np.cumsum(rng.integers(1, 4, size=(S, P)), axis=1) * 10 * SEC
    fam = np.arange(S) % 6
    walk = np.cumsum(rng.normal(size=(S, P)), axis=1)
    vals = np.empty((S, P), dtype=np.float64)
    vals[fam == 0] = 100 + walk[fam == 0]
    vals[fam == 1] = np.cumsum(rng.integers(0, 50, size=(S, P)), axis=1)[fam == 1]
    vals[fam == 2] = 42.0
    vals[fam == 3] = np.round(walk[fam == 3], 2)
    vals[fam == 4] = rng.normal(size=(S, P))[fam == 4] * 1e9
    vals[fam == 5] = rng.integers(0, 3, size=(S, P))[fam == 5] * 0.5
    n_pts = rng.integers(0, P + 1, size=S).astype(np.int32)
    n_pts[:64] = np.minimum(np.arange(64), P)
    n_pts[64:72] = [0, 1, P, P, 0, 1, P, 2]
    return ts, vals, n_pts


def _oracle(ts, vals, n, int_opt):
    return O.encode_series(ts[:n], vals[:n], START, O.UNIT_S, int_opt) if n else b""


def _check_slots(buf, out_len, status, expected, stride):
    """buf: uint8 [rows, stride] with rows >= len(expected), filled with SENTINEL before the encode.  For every
    status-0 series: [0, out_len) == expected, [out_len, round16(out_len)) == 0, the rest of the slot untouched;
    rows past the series (slots of lanes without a series) are untouched."""
    S = len(expected)
    for s in range(S):
        if status[s] != 0:
            continue
        n = int(out_len[s])
        r16 = (n + 15) & ~15
        assert buf[s, :n].tobytes() == expected[s], s
        assert not buf[s, n:r16].any(), s
        assert (buf[s, r16:] == SENTINEL).all(), (s, n)
    assert (buf[S:] == SENTINEL).all()


def _encode_into_sentinel(codec, ts, vals, n_pts, stride, point_major, annotations=None):
    from m3_b200.codec import EncodeResult
    S, P = ts.shape
    rows = (S + 31) // 32 * 32 + 32  # the slots a lane past n_series would have, and one more warp's
    buf = torch.full((rows, stride), SENTINEL, dtype=torch.uint8, device="cuda")
    out = EncodeResult(out=buf[:S], out_len=torch.empty(S, dtype=torch.int64, device="cuda"),
                       status=torch.empty(S, dtype=torch.int32, device="cuda"))
    t, v = torch.from_numpy(ts).cuda(), torch.from_numpy(vals).cuda()
    if point_major:
        t, v = t.t().contiguous(), v.t().contiguous()
    codec.encode(t, v, torch.full((S,), START, dtype=torch.int64, device="cuda"), unit=O.UNIT_S,
                 n_points=torch.from_numpy(n_pts).cuda(), annotations=annotations, out=out,
                 point_major=point_major)
    torch.cuda.synchronize()
    return buf.cpu().numpy(), out.out_len.cpu().numpy(), out.status.cpu().numpy()


@pytest.mark.parametrize("stride_mod", [16, 32, 128])
@pytest.mark.parametrize("S", [333, 334])  # odd: lane-local input fills, even: tensor copies; neither fills a warp
@pytest.mark.parametrize("int_opt", [True, False])
def test_mixed_warps_and_stride_alignment(codecs, stride_mod, S, int_opt):
    P = 300
    codec = codecs[int_opt]
    ts, vals, n_pts = _mixed(S, P, seed=S + stride_mod)
    stride = (codec.encode_bound(P) + 127) // 128 * 128 + stride_mod % 128
    expected = [_oracle(ts[s], vals[s], int(n_pts[s]), int_opt) for s in range(S)]
    res = {}
    for pm in (False, True):
        buf, out_len, status = _encode_into_sentinel(codec, ts, vals, n_pts, stride, pm)
        assert (status == 0).all()
        _check_slots(buf, out_len, status, expected, stride)
        res[pm] = buf
    assert np.array_equal(res[False], res[True])


@pytest.mark.parametrize("point_major", [False, True])
def test_capacity_error_next_to_full_series(codecs, point_major):
    """A slot too small for the random-double series but ample for the constant ones: the failing series stop
    with a capacity error, and their neighbours' slots hold exactly their streams."""
    from m3_b200 import capi
    S, P = 160, 400
    codec = codecs[True]
    ts, vals, n_pts = _mixed(S, P, seed=7)
    n_pts[:] = P
    stride = 1024 + 16
    expected = [_oracle(ts[s], vals[s], P, True) for s in range(S)]
    buf, out_len, status = _encode_into_sentinel(codec, ts, vals, n_pts, stride, point_major)
    fam = np.arange(S) % 6
    assert (status[fam == 4] == capi.ERR_CAPACITY).all()
    assert (status[fam == 2] == 0).all()
    assert set(np.unique(status)) <= {0, capi.ERR_CAPACITY}
    _check_slots(buf, out_len, status, expected, stride)


@pytest.mark.parametrize("packed", [False, True])
def test_long_annotations_on_a_few_lanes(codecs, packed):
    """Annotations of hundreds of bytes on three lanes of a warp drive the annotation loop's repeated flushes
    while the other lanes have nothing to flush (series-major inputs: point-major ones take no annotations)."""
    S, P = 96, 200
    rng = np.random.default_rng(11)
    codec = codecs[True]
    ts, vals, n_pts = _mixed(S, P, seed=11)
    n_pts[:] = P
    entries, series_off, blob = [], [0], bytearray()
    expected = []
    for s in range(S):
        anns = {}
        if s % 32 in (3, 17, 30):
            for i in sorted(rng.choice(P, size=4, replace=False)):
                anns[int(i)] = bytes(rng.integers(0, 256, size=int(rng.integers(200, 700)), dtype=np.uint8))
        for i, a in anns.items():
            entries.append((i, len(a), len(blob)))
            blob += a
        series_off.append(len(entries))
        e = O.Encoder(0, True)
        e.reset(START)
        for i in range(P):
            assert e.encode(int(ts[s, i]), float(vals[s, i]), O.UNIT_S, anns.get(i, b"")) == 0
        expected.append(e.stream() or b"")
    ent = np.zeros(len(entries), dtype=[("dp", "<u4"), ("len", "<u4"), ("off", "<u8")])
    for k, e in enumerate(entries):
        ent[k] = e
    ann = (torch.tensor(series_off, dtype=torch.int64, device="cuda"),
           torch.from_numpy(ent.view(np.uint8).reshape(-1, 16).copy()).cuda(),
           torch.frombuffer(bytearray(bytes(blob) + b"\0"), dtype=torch.uint8).cuda())
    stride = codec.encode_bound(P) + (4 * 700 + 64 + 15) // 16 * 16 + 16
    if not packed:
        buf, out_len, status = _encode_into_sentinel(codec, ts, vals, n_pts, stride, False, annotations=ann)
        assert (status == 0).all()
        _check_slots(buf, out_len, status, expected, stride)
        return
    pk = codec.encode_packed(torch.from_numpy(ts).cuda(), torch.from_numpy(vals).cuda(),
                             torch.full((S,), START, dtype=torch.int64, device="cuda"), unit=O.UNIT_S,
                             annotations=ann, align=16, capacity=S * stride, slot_bytes=stride)
    torch.cuda.synchronize()
    assert int((pk.status != 0).sum()) == 0
    h_pk, h_off, h_len = pk.packed.cpu().numpy(), pk.offsets.cpu().numpy(), pk.out_len.cpu().numpy()
    for s in range(S):
        a = int(h_off[s])
        assert h_pk[a: a + int(h_len[s])].tobytes() == expected[s], s


def _stream_bytes(blob, off, lens):
    """The bytes of every stream, concatenated (device tensors): blob[off[s] : off[s] + lens[s]] for all s."""
    total = int(lens.sum())
    first = torch.cumsum(lens, 0) - lens
    rep = torch.repeat_interleave(torch.arange(lens.numel(), device="cuda"), lens)
    return blob[off[rep] + torch.arange(total, device="cuda") - first[rep]]


@pytest.mark.parametrize("align", [1, 16, 64])
@pytest.mark.parametrize("point_major", [False, True])
def test_packed_several_batches_per_warp(codecs, align, point_major):
    """Packed output: several times more series than the resident warps' scratch slots (an H100 holds at most
    132 SMs x 5 blocks x 128 of them), so every warp encodes several batches into the same slots; a slot size
    that is 16 bytes past a 32-byte multiple.  Every stream equals the segment encode of the same inputs, and a
    sample equals the oracle's."""
    S, P = 300_000, 24
    codec = codecs[True]
    ts, vals, n_pts = _mixed(S, P, seed=align)
    t, v = torch.from_numpy(ts).cuda(), torch.from_numpy(vals).cuda()
    start = torch.full((S,), START, dtype=torch.int64, device="cuda")
    n = torch.from_numpy(n_pts).cuda()
    seg = codec.encode(t, v, start, unit=O.UNIT_S, n_points=n)
    if point_major:
        t, v = t.t().contiguous(), v.t().contiguous()
    slot = codec.encode_bound(P) // 32 * 32 + 16
    pk =codec.encode_packed(t, v, start, unit=O.UNIT_S, n_points=n, align=align, slot_bytes=slot,
                             point_major=point_major)
    torch.cuda.synchronize()
    assert int((seg.status != 0).sum()) == 0 and int((pk.status != 0).sum()) == 0
    assert torch.equal(pk.out_len, seg.out_len)
    lens = pk.out_len
    alen = (lens + align - 1) // align * align
    assert int(pk.total[0]) == int(alen.sum())
    assert int((pk.offsets % align).sum()) == 0
    nz = alen > 0  # (an empty stream takes no space: its offset may equal the next stream's)
    order = torch.argsort(pk.offsets[nz])
    o_sorted, a_sorted = pk.offsets[nz][order], alen[nz][order]
    assert bool((o_sorted[1:] >= o_sorted[:-1] + a_sorted[:-1]).all())  # no two streams overlap
    seg_off = torch.arange(S, dtype=torch.int64, device="cuda") * seg.out.shape[1]
    assert torch.equal(_stream_bytes(pk.packed, pk.offsets, lens), _stream_bytes(seg.out.view(-1), seg_off, lens))
    if align >= 16:  # the copy moves whole 16-byte groups: the stream's zero padding comes along
        pad = (16 - lens % 16) % 16
        assert not bool(_stream_bytes(pk.packed, pk.offsets + lens, pad).any())
    h_pk, h_off, h_len = pk.packed.cpu().numpy(), pk.offsets.cpu().numpy(), lens.cpu().numpy()
    for s in list(range(0, 72)) + list(range(S - 40, S)) + list(range(1000, S, 9973)):
        a = int(h_off[s])
        assert h_pk[a: a + int(h_len[s])].tobytes() == _oracle(ts[s], vals[s], int(n_pts[s]), True), s


def test_tile_reencode_with_empty_windows(codecs):
    """The tile aggregation's re-encode (Gauge aggregates read directly, packed output) on series with gaps,
    so that some windows are empty and lanes of a warp emit different numbers of datapoints."""
    rng = np.random.default_rng(5)
    S, P, step, nw = 200, 360, 300 * SEC, 200
    codec = codecs[True]
    gaps = rng.integers(1, 60, size=(S, P))
    gaps[rng.random(size=(S, P)) < 0.02] = 3000  # ~ 10 empty windows after each jump
    ts = START + np.cumsum(gaps, axis=1) * 10 * SEC
    vals = np.round(100 + np.cumsum(rng.normal(size=(S, P)), axis=1), 1)
    vals[1::4] = rng.normal(size=(S, P))[1::4] * 1e6
    enc = codec.encode(torch.from_numpy(ts).cuda(), torch.from_numpy(vals).cuda(),
                       torch.full((S,), START, dtype=torch.int64, device="cuda"), unit=O.UNIT_S)
    packed, offsets = codec.compact(enc, align=16)
    tiles, n_tiles = codec.aggregate_tiles(packed, offsets, START, step, nw)
    torch.cuda.synchronize()
    assert int((tiles.status != 0).sum()) == 0
    h_pk, h_off, h_len = tiles.packed.cpu().numpy(), tiles.offsets.cpu().numpy(), tiles.out_len.cpu().numpy()
    h_n = n_tiles.cpu().numpy()
    assert (h_n < nw).any() and (h_n > 0).all()
    for s in range(S):
        t_ts, t_v = O.aggregate_tiles_series(ts[s], vals[s], START, step, nw, O.AGG_LAST)
        assert h_n[s] == len(t_ts), s
        exp = O.encode_series(t_ts, t_v, START, O.UNIT_S, True)
        a = int(h_off[s])
        assert h_pk[a: a + int(h_len[s])].tobytes() == exp, s
