"""GPU decode: the ring fills, checked through every decode mode against the oracle.

A refill event is warp-wide: lanes that consume their streams at very different rates (constants next to full-width
random doubles) differ in whether they take a chunk at every event, and each fill asks L2 for the whole 128-byte line
around its request.  These tests put such lanes into ragged warps, start the streams at every byte offset mod 128
(CSR offsets and offsets + lengths), end the last stream at the buffer's last byte with a size that is not a multiple
of 16 (so the line around the last chunk runs past the buffer), and add empty streams, lanes rejected with
INVALID_ARG and lanes whose annotations run past the ring.  Series-major, point-major and the fused downsample (with and without `last`) are compared with the
oracle bit for bit, `n_points` and `status` included."""
import numpy as np
import pytest

import oracle_lib as O

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
SEC = 1_000_000_000
START = 1599955200 * SEC
S = 301  # 9 full warps + a ragged one of 13 lanes
P = 240


@pytest.fixture(scope="module")
def codecs():
    from m3_b200.codec import BatchCodec
    return {True: BatchCodec(0, True), False: BatchCodec(0, False)}


def _streams(int_opt, seed):
    """S oracle-encoded streams, by s % 6: constants, full-width random doubles (about 25 times the constants'
    bytes per datapoint), a random walk, int-like counters, 2-digit decimals, and repeats of a few values.  Lengths are ragged (empty streams included); lanes 7, 100 and 290
    carry annotations of 300-900 bytes, longer than the 256-byte ring."""
    rng = np.random.default_rng(seed)
    ts = START + np.cumsum(rng.integers(1, 4, size=(S, P)), axis=1) * 10 * SEC
    walk = np.cumsum(rng.normal(size=(S, P)), axis=1)
    fam = np.arange(S) % 6
    ts[fam == 0] = START + np.arange(1, P + 1) * 10 * SEC  # constants at a fixed step: 2-3 bits per datapoint
    # full-width doubles at irregular steps (32-bit delta-of-delta buckets)
    ts[fam == 1] = START + np.cumsum(rng.integers(1, 5000, size=(S, P)), axis=1)[fam == 1] * SEC
    vals = np.empty((S, P), dtype=np.float64)
    vals[fam == 0] = 42.0
    vals[fam == 1] = np.ldexp(rng.random(size=(S, P)) - 0.5, rng.integers(-900, 900, size=(S, P)))[fam == 1]
    vals[fam == 2] = (100 + walk)[fam == 2]
    vals[fam == 3] = np.cumsum(rng.integers(0, 50, size=(S, P)), axis=1)[fam == 3]
    vals[fam == 4] = np.round(walk, 2)[fam == 4]
    vals[fam == 5] = (rng.integers(0, 3, size=(S, P)) * 0.5)[fam == 5]
    n_pts = rng.integers(P // 2, P + 1, size=S)
    n_pts[[3, 40, 41, 77, 200, 299]] = 0
    n_pts[[5, 64, 150]] = 1
    out = []
    for s in range(S):
        n = int(n_pts[s])
        if s in (7, 100, 290):
            e = O.Encoder(START, int_opt)
            for i in range(n):
                ann = bytes(rng.integers(0, 256, size=300 + 300 * (i % 3), dtype=np.uint8)) if i in (2, 60, 61) else b""
                e.encode(int(ts[s, i]), float(vals[s, i]), O.UNIT_S, annotation=ann)
            out.append(e.stream())
        else:
            out.append(O.encode_series(ts[s, :n], vals[s, :n], START, O.UNIT_S, int_opt) if n else b"")
    return out


def _layout(streams, shift):
    """Byte starts in one buffer: the i-th non-empty stream starts at (shift + 37 i) mod 128 (every residue once per
    128 streams), the last one ends at the buffer's last byte with a size = 13 mod 128.  Returns (starts, total)."""
    live = [i for i, b in enumerate(streams) if b]
    starts = np.zeros(len(streams), dtype=np.int64)
    pos = 0
    for j, i in enumerate(live):
        n = len(streams[i])
        want = (13 - n) % 128 if i == live[-1] else (shift + 37 * j) % 128
        pos += (want - pos) % 128
        starts[i] = pos
        pos += n
    assert pos % 16 == 13
    return starts, pos


def _fill(streams, starts, total, seed):
    buf = np.random.default_rng(seed).integers(0, 256, size=total, dtype=np.uint8)
    for st, b in zip(starts, streams):
        buf[st:st + len(b)] = np.frombuffer(b, dtype=np.uint8)
    return buf


def _csr(streams, shift, seed):
    """CSR offsets over a buffer where a stream's range runs on to the next stream's start: the junk after a stream's
    end-of-stream marker is never decoded.  Empty streams stay empty."""
    starts, total = _layout(streams, shift)
    buf = _fill(streams, starts, total, seed)
    off = np.zeros(len(streams) + 1, dtype=np.int64)
    off[-1] = total
    nxt = total
    for i in range(len(streams) - 1, -1, -1):
        off[i] = starts[i] if streams[i] else nxt
        nxt = off[i]
    return buf, off


def _oracle(streams, int_opt):
    blob = b"".join(streams)
    off = np.zeros(len(streams) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(b) for b in streams])
    return O.decode_batch(np.frombuffer(blob, dtype=np.uint8), off, P + 8, int_opt)


def _dev(buf):
    # the exact buffer: the decoder must not read past streams_bytes
    return torch.from_numpy(np.ascontiguousarray(buf)).cuda()


def _check_decode(codec, d, off, lengths, expected, bad=()):
    e_ts, e_v, e_n, e_st = expected
    cap = P + 8
    lens = None if lengths is None else torch.from_numpy(lengths).cuda()
    o = torch.from_numpy(off).cuda()
    sm = codec.decode(d, o, cap, lengths=lens)
    pm = codec.decode(d, o, cap, lengths=lens, point_major=True)
    torch.cuda.synchronize()
    for r in (sm, pm):
        n, st = r.n_points.cpu().numpy(), r.status.cpu().numpy()
        for s in range(S):
            if s in bad:
                assert n[s] == 0 and st[s] == 101, s  # M3TSZ_ERR_INVALID_ARG
            else:
                assert n[s] == e_n[s] and st[s] == e_st[s], (s, n[s], e_n[s], st[s], e_st[s])
    n = sm.n_points.cpu().numpy()
    s_ts, s_v = sm.ts.cpu().numpy(), sm.values.cpu().numpy().view(np.uint64)
    p_ts, p_v = pm.ts.cpu().numpy().T, pm.values.cpu().numpy().view(np.uint64).T
    ev = e_v.view(np.uint64)
    for s in range(S):
        k = int(n[s])
        assert (s_ts[s, :k] == e_ts[s, :k]).all() and (s_v[s, :k] == ev[s, :k]).all(), s
        assert (p_ts[s, :k] == s_ts[s, :k]).all() and (p_v[s, :k] == s_v[s, :k]).all(), s


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("shift", [0, 1, 63])
def test_mixed_rates_csr(codecs, int_opt, shift):
    streams = _streams(int_opt, 5 + shift)
    buf, off = _csr(streams, shift, shift)
    _check_decode(codecs[int_opt], _dev(buf), off, None, _oracle(streams, int_opt))


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("shift", [0, 90])
def test_mixed_rates_offsets_and_lengths(codecs, int_opt, shift):
    """Streams placed anywhere among junk bytes, (start, length) per series; lanes 30, 31, 33 and 300 point past the
    end of the buffer and are rejected next to live lanes."""
    streams = _streams(int_opt, 17 + shift)
    starts, total = _layout(streams, shift)
    buf = _fill(streams, starts, total, 99)
    lengths = np.array([len(b) for b in streams], dtype=np.int64)
    bad = (30, 31, 33, 300)
    for s in bad:
        starts[s], lengths[s] = total - 3, 100
    _check_decode(codecs[int_opt], _dev(buf), starts, lengths, _oracle(streams, int_opt), bad)


@pytest.mark.parametrize("want_last", [False, True])
@pytest.mark.parametrize("int_opt", [True, False])
def test_fused_downsample(codecs, int_opt, want_last):
    streams = _streams(int_opt, 3)
    buf, off = _csr(streams, 11, 4)
    window, n_win = 300 * SEC, 32
    r = codecs[int_opt].decode_downsample(_dev(buf), torch.from_numpy(off).cuda(), START, window, n_win,
                                          want_last=want_last)
    torch.cuda.synchronize()
    e_ts, e_v, e_n, e_st = _oracle(streams, int_opt)
    n, st = r.n_points.cpu().numpy(), r.status.cpu().numpy()
    got = [x.cpu().numpy().view(np.uint64) for x in (r.sum, r.count, r.min, r.max)]
    last = r.last.cpu().numpy().view(np.uint64) if want_last else None
    for s in range(S):
        assert n[s] == e_n[s] and st[s] == e_st[s], (s, n[s], e_n[s], st[s], e_st[s])
        k = int(e_n[s])
        es, ec, emn, emx, el = O.downsample_series(e_ts[s, :k], e_v[s, :k], START, window, n_win)
        for g, e in zip(got, (es, ec, emn, emx)):
            assert (g[:, s] == np.ascontiguousarray(e).view(np.uint64)).all(), s
        if want_last:
            assert (last[:, s] == el.view(np.uint64)).all(), s
