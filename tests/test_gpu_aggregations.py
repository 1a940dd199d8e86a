"""The Gauge with expensive aggregations (sumSq) and the Counter on the GPU: the fused downsample modes behind
m3tsz_decode_downsample_ex and the tile aggregation of m3tsz_aggregate_tiles_ex, bit for bit against the CPU oracle
(tests/agg_oracle.c), in both int_optimized modes."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import agg_oracle_lib as A
import oracle_lib as O

pytestmark = pytest.mark.gpu

SEC = 1_000_000_000
WIN = 60 * SEC
N_WIN = 12
R0 = 1_700_000_040 * SEC  # range start (window-aligned)
START = R0 - 10 * WIN     # encoder start

SPECIALS = [math.nan, math.inf, -math.inf, -0.0, 0.0, 2.0 ** 63, -2.0 ** 63, 9.3e18, -9.3e18, -1.5, 1.5, -2.5,
            3.0e18, 4.0e9, -4.0e9, 1e-300, 123.456]


@pytest.fixture(scope="module")
def codecs():
    from m3_b200.codec import BatchCodec
    return {True: BatchCodec(0, int_optimized=True), False: BatchCodec(0, int_optimized=False)}


def _series(rng, n, specials=True):
    """n datapoints: seconds steps of 1..90 s with occasional steps back (out of order), starting before the range
    and running past its end; values mix the special ones, integers and fractions."""
    t = R0 - int(rng.integers(0, 4)) * WIN + int(rng.integers(0, 60)) * SEC
    ts, vals = [], []
    for _ in range(n):
        ts.append(t)
        r = rng.random()
        if specials and r < 0.3:
            vals.append(SPECIALS[int(rng.integers(0, len(SPECIALS)))])
        elif r < 0.65:
            vals.append(float(int(rng.integers(-1000, 100000))))
        else:
            vals.append(float(np.round(rng.normal(0, 1000), 3)))
        t += (int(rng.integers(1, 91)) if rng.random() > 0.12 else -int(rng.integers(1, 400))) * SEC
        if rng.random() < 0.03:
            t += 5 * WIN  # leave empty windows behind
    return np.array(ts, dtype=np.int64), np.array(vals, dtype=np.float64)


def _batch(int_opt, S=96, seed=7, specials=True, damage=True):
    """Ragged series (windows out of phase across lanes), some truncated or with flipped bytes.  Returns the host
    streams and the CSR blob + offsets on the device."""
    rng = np.random.default_rng(seed)
    streams = []
    for s in range(S):
        ts, vals = _series(rng, int(rng.integers(1, 200)), specials)
        b = O.encode_series(ts, vals, START, O.UNIT_S, int_opt)
        if damage and s % 11 == 3:
            b = b[: max(1, len(b) * 3 // 5)]  # truncated
        elif damage and s % 13 == 5 and len(b) > 24:
            a = bytearray(b)
            a[len(a) // 2] ^= 0xA5  # corrupt
            b = bytes(a)
        streams.append(b)
    off = np.zeros(S + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(b) for b in streams])
    blob = np.frombuffer(b"".join(streams) + b"\0" * 16, dtype=np.uint8).copy()
    return streams, torch.from_numpy(blob).cuda(), torch.from_numpy(off).cuda()


def _padded(streams):
    """The same streams at 64-byte aligned starts: (blob, starts, lengths) for offsets + lengths addressing."""
    starts, pos = [], 0
    for b in streams:
        starts.append(pos)
        pos += (len(b) + 63) // 64 * 64
    blob = np.zeros(pos + 16, dtype=np.uint8)
    for p, b in zip(starts, streams):
        blob[p: p + len(b)] = np.frombuffer(b, dtype=np.uint8)
    lens = [len(b) for b in streams]
    t = lambda a: torch.tensor(a, dtype=torch.int64, device="cuda")
    return torch.from_numpy(blob).cuda(), t(starts), t(lens)


def _bits(a):
    return a.cpu().numpy().view(np.uint64)


def _same_f64(got, exp):
    """Bit-equal, except that a NaN sum (+Inf and -Inf in one window) only has to be NaN on both sides: the
    NaN's payload is the hardware's, as in the existing Gauge modes."""
    g, e = got.view(np.uint64), exp.view(np.uint64)
    return bool(((g == e) | (np.isnan(got) & np.isnan(exp))).all())


def _decoded(codec, blob, off, S, lengths=None):
    d = codec.decode(blob, off, 16384, lengths=lengths)
    torch.cuda.synchronize()
    n = d.n_points.cpu().numpy()
    return d.ts.cpu().numpy(), d.values.cpu().numpy(), n


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("addressing", ["csr", "lengths"])
def test_gauge_sum_sq_and_counter_downsample(codecs, int_opt, addressing):
    from m3_b200 import capi
    codec = codecs[int_opt]
    streams, blob, off = _batch(int_opt)
    S = len(streams)
    lengths = None
    if addressing == "lengths":
        blob, off, lengths = _padded(streams)
    ref = codec.decode_downsample(blob, off, R0, WIN, N_WIN, want_last=True, lengths=lengths)
    g = codec.decode_downsample(blob, off, R0, WIN, N_WIN, want_sum_sq=True, lengths=lengths)
    c = codec.decode_downsample(blob, off, R0, WIN, N_WIN, metric=capi.METRIC_COUNTER, lengths=lengths)
    ts, vals, n = _decoded(codec, blob, off, S, lengths)
    torch.cuda.synchronize()
    assert g.sum_sq.dtype == torch.float64 and c.sum.dtype == torch.int64 and c.sum_sq.dtype == torch.int64
    # the Gauge's sumSq mode is mode 2 plus sumSq: every shared output is identical, n_points / status too
    for a, b in ((g.sum, ref.sum), (g.count, ref.count), (g.min, ref.min), (g.max, ref.max), (g.last, ref.last),
                 (g.last_at, ref.last_at), (g.n_points, ref.n_points), (g.status, ref.status),
                 (c.n_points, ref.n_points), (c.status, ref.status), (c.count, ref.count)):
        assert torch.equal(a.view(torch.int64) if a.dtype == torch.float64 else a,
                           b.view(torch.int64) if b.dtype == torch.float64 else b)
    st = ref.status.cpu().numpy()
    assert (st != 0).sum() >= 1  # damaged streams are in the batch
    assert (n == ref.n_points.cpu().numpy()).all()
    gh = [x.cpu().numpy() for x in (g.sum, g.count, g.min, g.max, g.last, g.last_at, g.sum_sq)]
    ch = [x.cpu().numpy() for x in (c.sum, c.count, c.min, c.max, c.sum_sq)]
    for s in range(S):
        k = int(n[s])
        exp = A.downsample_gauge_ex(ts[s, :k], vals[s, :k], R0, WIN, N_WIN)
        assert _same_f64(gh[0][:, s], exp[0]), s
        assert (gh[1][:, s] == exp[1]).all() and (gh[5][:, s] == exp[5]).all(), s
        for j in (2, 3, 4, 6):
            assert (gh[j][:, s].view(np.uint64) == exp[j].view(np.uint64)).all(), (s, j)
        if k:  # against the stream's own oracle decode where it is intact
            ots, ovals, on, oerr = O.decode_series(streams[s], int_opt, cap=256)
            if oerr == 0:
                assert on == k and (ots == ts[s, :k]).all()
        cexp = A.downsample_counter(ts[s, :k], vals[s, :k], R0, WIN, N_WIN)
        for j in range(5):
            assert (ch[j][:, s] == cexp[j]).all(), (s, j)


@pytest.mark.parametrize("int_opt", [True, False])
def test_downsample_ex_rejects_bad_outputs(codecs, int_opt):
    from m3_b200 import capi
    codec = codecs[int_opt]
    streams, blob, off = _batch(int_opt, S=8, damage=False)
    S = len(streams)
    mk = lambda dt: torch.empty((N_WIN, S), dtype=dt, device="cuda")
    f, i = mk(torch.float64), mk(torch.int64)
    L = capi.lib()
    cases = []
    o = capi.DownsampleOutputs(); o.metric_type = 2; o.d_count = i.data_ptr(); cases.append(o)  # unknown metric
    o = capi.DownsampleOutputs(); o.metric_type = capi.METRIC_COUNTER; o.d_count = i.data_ptr()
    o.d_counter_sum = o.d_counter_min = o.d_counter_max = i.data_ptr(); o.d_sum = f.data_ptr(); cases.append(o)
    o = capi.DownsampleOutputs(); o.metric_type = capi.METRIC_COUNTER; o.d_count = i.data_ptr()
    o.d_counter_sum = o.d_counter_min = i.data_ptr(); cases.append(o)  # no max
    o = capi.DownsampleOutputs(); o.metric_type = capi.METRIC_GAUGE; o.d_count = i.data_ptr()
    o.d_sum = o.d_min = o.d_max = o.d_sum_sq = f.data_ptr(); o.d_counter_sum_sq = i.data_ptr(); cases.append(o)
    o = capi.DownsampleOutputs(); o.metric_type = capi.METRIC_GAUGE; o.d_count = i.data_ptr()
    o.d_sum = o.d_min = o.d_sum_sq = f.data_ptr(); cases.append(o)  # no max
    n0 = codec.launch_count()
    for o in cases:
        rc = L.m3tsz_decode_downsample_ex(codec.ctx.handle, C.byref(codec.opts), blob.data_ptr(), blob.numel(),
                                          off.data_ptr(), None, S, R0, WIN, N_WIN, C.byref(o), None)
        assert rc == capi.ERR_INVALID_ARG
    assert codec.launch_count() == n0


GAUGE_TYPES = [1, 2, 3, 4, 6, 7, 8, 9]
COUNTER_TYPES = [2, 3, 4, 6, 7, 8, 9]


def _tile_check(codec, streams, blob, off, int_opt, metric, agg, lengths=None):
    S = len(streams)
    r, n_tiles = codec.aggregate_tiles(blob, off, R0, WIN, N_WIN, agg_type=agg, metric_type=metric, lengths=lengths)
    ts, vals, n = _decoded(codec, blob, off, S, lengths)
    torch.cuda.synchronize()
    st, g_len, g_off = r.status.cpu().numpy(), r.out_len.cpu().numpy(), r.offsets.cpu().numpy()
    packed, nt = r.packed.cpu().numpy(), n_tiles.cpu().numpy()
    for s in range(S):
        _, _, _, err = O.decode_series(streams[s], int_opt, cap=256)
        if err != 0:
            assert st[s] == err and g_len[s] == 0 and nt[s] == 0, s
            continue
        assert st[s] == 0, (s, st[s])
        k = int(n[s])
        tts, tvals = A.aggregate_tiles_series_ex(ts[s, :k], vals[s, :k], R0, WIN, N_WIN, metric, agg)
        assert nt[s] == len(tts), s
        exp = O.encode_series(tts, tvals, R0, O.UNIT_S, int_opt) if len(tts) else b""
        assert packed[g_off[s]: g_off[s] + g_len[s]].tobytes() == exp, (s, metric, agg)
    return r, n_tiles


@pytest.mark.parametrize("int_opt", [True, False])
def test_tiles_ex_every_valid_pair(codecs, int_opt):
    """No +Inf and -Inf in one window here (a NaN sum's payload is the hardware's; see _same_f64); +Inf alone still
    makes a NaN Stdev (Inf - Inf), whose bits are amd64's."""
    codec = codecs[int_opt]
    rng = np.random.default_rng(3)
    streams = []
    for s in range(64):
        ts, vals = _series(rng, int(rng.integers(1, 200)), specials=False)
        if s % 4 == 1:  # special values, one infinity sign per series
            pick = rng.choice([math.nan, math.inf if s % 8 == 1 else -math.inf, -0.0, 2.0 ** 63, -2.0 ** 63,
                               -1.5, 3.0e18, 4.0e9], size=len(vals))
            vals = np.where(rng.random(len(vals)) < 0.4, pick, vals)
        b = O.encode_series(ts, vals, START, O.UNIT_S, int_opt)
        streams.append(b[: len(b) // 2] if s == 9 else b)  # one truncated source stream
    off = np.zeros(len(streams) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(b) for b in streams])
    blob = torch.from_numpy(np.frombuffer(b"".join(streams) + b"\0" * 16, dtype=np.uint8).copy()).cuda()
    off = torch.from_numpy(off).cuda()
    for agg in GAUGE_TYPES:
        _tile_check(codec, streams, blob, off, int_opt, A.METRIC_GAUGE, agg)
    for agg in COUNTER_TYPES:
        _tile_check(codec, streams, blob, off, int_opt, A.METRIC_COUNTER, agg)
    pblob, pstarts, plens = _padded(streams)
    _tile_check(codec, streams, pblob, pstarts, int_opt, A.METRIC_COUNTER, 9, lengths=plens)
    _tile_check(codec, streams, pblob, pstarts, int_opt, A.METRIC_GAUGE, 9, lengths=plens)


@pytest.mark.parametrize("int_opt", [True, False])
def test_tiles_ex_gauge_old_types_match_batch(codecs, int_opt):
    from m3_b200 import capi
    codec = codecs[int_opt]
    streams, blob, off = _batch(int_opt, S=64, seed=11, specials=False)
    S = len(streams)
    for agg in (1, 2, 3, 4, 6, 7):
        a, na = codec.aggregate_tiles(blob, off, R0, WIN, N_WIN, agg_type=agg)
        b, nb = _tiles_ex_raw(codec, blob, off, S, capi.METRIC_GAUGE, agg)
        torch.cuda.synchronize()
        assert torch.equal(a.status, b.status) and torch.equal(na, nb) and torch.equal(a.out_len, b.out_len)
        pa, pb = a.packed.cpu().numpy(), b.packed.cpu().numpy()
        oa, ob, ln = a.offsets.cpu().numpy(), b.offsets.cpu().numpy(), a.out_len.cpu().numpy()
        for s in range(S):
            assert (pa[oa[s]: oa[s] + ln[s]] == pb[ob[s]: ob[s] + ln[s]]).all(), (s, agg)


def _tiles_ex_raw(codec, blob, off, S, metric, agg):
    from m3_b200 import capi
    from m3_b200.codec import PackedResult
    dev = codec.device
    cap = S * codec.encode_bound(N_WIN)
    out = PackedResult(packed=torch.empty(cap, dtype=torch.uint8, device=dev),
                       offsets=torch.empty(S, dtype=torch.int64, device=dev),
                       out_len=torch.empty(S, dtype=torch.int64, device=dev),
                       status=torch.empty(S, dtype=torch.int32, device=dev),
                       total=torch.zeros(1, dtype=torch.int64, device=dev))
    n_tiles = torch.empty(S, dtype=torch.int32, device=dev)
    rc = capi.lib().m3tsz_aggregate_tiles_ex(
        codec.ctx.handle, C.byref(codec.opts), blob.data_ptr(), blob.numel(), off.data_ptr(), None, S, R0, WIN,
        N_WIN, metric, agg, O.UNIT_S, 64, out.packed.data_ptr(), cap, out.offsets.data_ptr(),
        out.out_len.data_ptr(), out.status.data_ptr(), n_tiles.data_ptr(), out.total.data_ptr(), None)
    return (out, n_tiles) if rc == 0 else rc


@pytest.mark.parametrize("int_opt", [True, False])
def test_tiles_invalid_pairs_launch_nothing(codecs, int_opt):
    from m3_b200 import capi
    codec = codecs[int_opt]
    streams, blob, off = _batch(int_opt, S=8, damage=False)
    n0 = codec.launch_count()
    bad = [(capi.METRIC_COUNTER, 1), (capi.METRIC_GAUGE, 5), (capi.METRIC_COUNTER, 10), (capi.METRIC_GAUGE, 0),
           (2, 7), (0, 7), (4, 9), (capi.METRIC_GAUGE, 12)]
    for metric, agg in bad:
        assert _tiles_ex_raw(codec, blob, off, len(streams), metric, agg) == capi.ERR_INVALID_ARG, (metric, agg)
    assert codec.launch_count() == n0
    # the batch call keeps rejecting the expensive types
    for agg in (8, 9):
        with pytest.raises(capi.M3tszError):
            rc = capi.lib().m3tsz_aggregate_tiles_batch(
                codec.ctx.handle, C.byref(codec.opts), blob.data_ptr(), blob.numel(), off.data_ptr(), None,
                len(streams), R0, WIN, N_WIN, agg, O.UNIT_S, 64, None, 0, None, None, None, None, None, None)
            codec.ctx.check(rc, "m3tsz_aggregate_tiles_batch")
    assert codec.launch_count() == n0


@pytest.mark.parametrize("int_opt", [True, False])
def test_sum_sq_and_counter_16k_x_1440_every_window(codecs, int_opt):
    from m3_b200 import capi, synth
    S, P = 16_384, 1440
    codec = codecs[int_opt]
    ts, vals, start = synth.gaussian_walk(S, P, "cuda", seed=99)
    enc = codec.encode(ts, vals, start, unit=O.UNIT_S)
    packed, offsets = codec.compact(enc, align=64)
    s0 = int(start[0].item())
    n_win = 288
    ref = codec.decode_downsample(packed, offsets, s0, 300 * SEC, n_win, want_last=True)
    g = codec.decode_downsample(packed, offsets, s0, 300 * SEC, n_win, want_sum_sq=True)
    c = codec.decode_downsample(packed, offsets, s0, 300 * SEC, n_win, metric=capi.METRIC_COUNTER)
    torch.cuda.synchronize()
    assert int((g.status != 0).sum()) == 0 and int((c.status != 0).sum()) == 0
    for a, b in ((g.sum, ref.sum), (g.min, ref.min), (g.max, ref.max), (g.last, ref.last)):
        assert torch.equal(a.view(torch.int64), b.view(torch.int64))
    assert torch.equal(g.count, ref.count) and torch.equal(c.count, ref.count)
    total = int(offsets[-1].item())
    o_ts, o_vals, o_n, o_st = O.decode_batch(packed[:total].cpu().numpy(), offsets.cpu().numpy().astype(np.uint64),
                                             P, int_opt, n_threads=8)
    assert (o_st == 0).all() and (o_n == P).all()
    gsq = g.sum_sq.cpu().numpy().view(np.uint64)
    ch = [x.cpu().numpy() for x in (c.sum, c.min, c.max, c.sum_sq)]
    for s in range(S):
        exp = A.downsample_gauge_ex(o_ts[s], o_vals[s], s0, 300 * SEC, n_win)
        assert (gsq[:, s] == exp[6].view(np.uint64)).all(), s
        cs, cc, cmn, cmx, csq = A.downsample_counter(o_ts[s], o_vals[s], s0, 300 * SEC, n_win)
        for got, e in zip(ch, (cs, cmn, cmx, csq)):
            assert (got[:, s] == e).all(), s
