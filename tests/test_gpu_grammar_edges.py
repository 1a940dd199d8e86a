"""The GPU codec at the edges of the M3TSZ grammar: the corpus of tests/grammar_edges.py through every encode tier
and decode path, against the oracle.

Which copy of the grammar runs is a warp vote, so the corpus runs in two layouts.  Uniform warps: the 32 lanes of a
warp take the same series template, each lane with its own values and start (`grammar_edges.corpus(lane)`), so
they reach each cell at the same datapoint and the voted tiers take it (the encoder's hot tier, second tier and
point-major tile stage; the decoder's hot candidate and general fast path).  Mixed warps: templates interleaved
lane by lane, so the general path and the complete grammar take the cells.  Both with an even and an odd number of
series (the encoder's tensor-copy and lane-local input fills).  Each (int_optimized, unit) group is one batch,
under a codec whose default unit is that unit.

- Encode (series-major, point-major, packed): bytes, out_len and status; a series that fails (a delta-of-delta
  past 32 bits) holds the datapoints before the failing one.
- The encoder set, one datapoint per append over the whole batch, so the state record is saved and loaded at
  every grammar state: every snapshot is the oracle's Stream() of the prefix.
- The widest codes in a slot whose capacity stop falls on every row of a tile.
- Decode of the oracle's streams (series- and point-major, CSR and offsets + lengths) and of the GPU's own streams.
- The fused downsample (plain, last, sumSq; Counter on the int-optimised groups), with warps on the hot path whose
  datapoints land exactly on a window end and 1 ns before one."""
import functools

import numpy as np
import pytest

import agg_oracle_lib as A
import grammar_edges as G
import oracle_lib as O
from test_gpu_encode_flush import _check_slots, _encode_into_sentinel
from test_gpu_encode_groups import _check, _encode, _expected

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
LANES = 32
GROUPS = [(m, u) for m in (False, True) for u in (1, 2, 3, 4)]


@functools.lru_cache(maxsize=None)
def _lanes():
    return [G.corpus(lane) for lane in range(LANES)]


@functools.lru_cache(maxsize=None)
def _codec(int_opt, unit):
    from m3_b200.codec import BatchCodec
    return BatchCodec(0, int_opt, default_unit=unit)


@functools.lru_cache(maxsize=None)
def _batch(int_opt, unit, layout, odd):
    """(ts [S, P], vals [S, P], start [S], series) of the group in the layout; S odd or even"""
    lanes = _lanes()
    idx = [i for i, s in enumerate(lanes[0]) if s.int_opt == int_opt and s.unit == unit]
    if layout == "uniform":
        series = [lanes[l][i] for i in idx for l in range(LANES)]
    else:  # the templates interleaved: neighbouring lanes are 37 templates apart (lane variants 0-1, then 2-3)
        k = 37 if len(idx) % 37 else 41
        order = [idx[(j * k) % len(idx)] for j in range(len(idx))]
        series = [lanes[j % 2][i] for j, i in enumerate(order)] + [lanes[2 + j % 2][i] for j, i in enumerate(order)]
    if (len(series) % 2 == 1) != odd:
        series = series + [lanes[5][idx[0]]]
    ts = np.stack([s.ts for s in series])
    vals = np.stack([s.vals for s in series])
    start = np.array([s.start for s in series], dtype=np.int64)
    return ts, vals, start, series


class Oracle:
    """the oracle's streams (bytes of the datapoints before a failing one), status and datapoints encoded"""

    def __init__(self, ts, vals, start, int_opt, unit):
        S, P = ts.shape
        self.out, ln, self.status = O.encode_batch(ts, vals, start, unit, int_opt, default_unit=unit, n_threads=16)
        self.len = ln.astype(np.int64)
        self.n_ok = np.full(S, P, dtype=np.int64)
        self.streams = [self.out[s, : self.len[s]].tobytes() for s in range(S)]
        for s in np.nonzero(self.status)[0]:
            e = O.Encoder(int(start[s]), int_opt, unit)
            for i in range(P):
                if e.encode(int(ts[s, i]), float(vals[s, i]), unit):
                    break
            self.n_ok[s] = i
            self.streams[s] = (e.stream() or b"") if i else b""
            self.len[s] = len(self.streams[s])
        self.stride = (max(self.len.max(), 1) + 15) // 16 * 16
        self.padded = self.out[:, : self.stride].copy()  # (zero past each stream)
        for s in np.nonzero(self.status)[0]:
            self.padded[s] = 0
            self.padded[s, : self.len[s]] = np.frombuffer(self.streams[s], dtype=np.uint8)


@functools.lru_cache(maxsize=None)
def _case(int_opt, unit, layout, odd):
    ts, vals, start, series = _batch(int_opt, unit, layout, odd)
    return ts, vals, start, Oracle(ts, vals, start, int_opt, unit)


def _same_streams(buf, out_len, e, rows=None):
    """buf [S, >= len] uint8: every stream's bytes and length as the oracle's"""
    rows = np.arange(len(e.len)) if rows is None else rows
    assert (out_len[rows] == e.len[rows]).all(), rows[out_len[rows] != e.len[rows]][:10]
    w = e.stride
    mask = np.arange(w)[None, :] < e.len[rows, None]
    got = buf[rows, :w] if buf.shape[1] >= w else np.pad(buf[rows], ((0, 0), (0, w - buf.shape[1])))
    bad = ((got != e.padded[rows]) & mask).any(axis=1)
    assert not bad.any(), rows[bad][:10]


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("odd", [False, True])
@pytest.mark.parametrize("layout", ["uniform", "mixed"])
@pytest.mark.parametrize("int_opt,unit", GROUPS)
def test_encode_against_oracle(int_opt, unit, layout, odd):
    codec = _codec(int_opt, unit)
    ts, vals, start, e = _case(int_opt, unit, layout, odd)
    S, P = ts.shape
    d_ts, d_v, d_st = _t(ts), _t(vals), _t(start)
    sm = codec.encode(d_ts, d_v, d_st, unit=unit)
    pm = codec.encode(d_ts.t().contiguous(), d_v.t().contiguous(), d_st, unit=unit, point_major=True)
    pk = codec.encode_packed(d_ts, d_v, d_st, unit=unit, align=16)
    torch.cuda.synchronize()
    ok = np.nonzero(e.status == 0)[0]
    for r in (sm, pm):
        st, ln, out = r.status.cpu().numpy(), r.out_len.cpu().numpy(), r.out.cpu().numpy()
        assert (st == e.status).all(), np.nonzero(st != e.status)[0][:10]
        _same_streams(out, ln, e, ok)
    p_out, p_off, p_len, p_st = (x.cpu().numpy() for x in (pk.packed, pk.offsets, pk.out_len, pk.status))
    assert (p_st == e.status).all()
    got = np.zeros((S, e.stride), dtype=np.uint8)
    for s in ok:
        got[s, : p_len[s]] = p_out[p_off[s]: p_off[s] + p_len[s]]
    _same_streams(got, p_len, e, ok)
    # the GPU's streams decode as the oracle's do (a failing series: the datapoints before the failing one)
    r = codec.decode(sm.out.view(-1), torch.arange(S, dtype=torch.int64, device="cuda") * sm.out.shape[1], P,
                     lengths=sm.out_len)
    torch.cuda.synchronize()
    rows, _, x_ts, x_v, mask = _oracle_decode(e, int_opt, unit, P)
    assert (r.status.cpu().numpy()[rows] == 0).all() and (r.n_points.cpu().numpy()[rows] == e.n_ok[rows]).all()
    assert ((r.ts.cpu().numpy()[rows] == x_ts) | ~mask).all()
    assert ((r.values.cpu().numpy().view(np.uint64)[rows] == x_v.view(np.uint64)) | ~mask).all()
    n_fail = int((e.status != 0).sum())
    print("encode int_opt=%s unit=%d %s S=%d: %d series fail (delta-of-delta overflow)" % (int_opt, unit, layout, S,
                                                                                          n_fail))


def _oracle_decode(e, int_opt, unit, cap):
    """the oracle's decode of the oracle's non-empty streams (a series whose first datapoint fails has none):
    (rows, their streams, ts [len(rows), cap], values [len(rows), cap], mask of the datapoints)"""
    rows = np.nonzero(e.n_ok > 0)[0]
    streams = [e.streams[s] for s in rows]
    off = np.zeros(len(rows) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(b) for b in streams])
    blob = np.frombuffer(b"".join(streams) + b"\0", dtype=np.uint8)
    ts, v, n, st = O.decode_batch(blob, off, cap, int_opt, unit, n_threads=16)
    assert (st == 0).all() and (n == e.n_ok[rows]).all()
    return rows, streams, ts, v, np.arange(cap)[None, :] < e.n_ok[rows, None]


def _csr(streams):
    off = np.zeros(len(streams) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(b) for b in streams])
    blob = np.frombuffer(b"".join(streams) + b"\0", dtype=np.uint8).copy()
    return _t(blob[: max(int(off[-1]), 1)]), _t(off), None


def _scattered(streams):
    """offsets + lengths: stream i at byte (37 i + 5) mod 128 of its own stretch, random bytes between"""
    rng = np.random.default_rng(len(streams))
    starts, pos = [], 0
    for i, b in enumerate(streams):
        pos += (37 * i + 5 - pos) % 128
        starts.append(pos)
        pos += len(b)
    buf = rng.integers(0, 256, size=pos + 1, dtype=np.uint8)
    for st, b in zip(starts, streams):
        buf[st: st + len(b)] = np.frombuffer(b, dtype=np.uint8)
    return _t(buf), _t(np.array(starts, dtype=np.int64)), _t(np.array([len(b) for b in streams], dtype=np.int64))


@pytest.mark.parametrize("odd", [False, True])
@pytest.mark.parametrize("layout", ["uniform", "mixed"])
@pytest.mark.parametrize("int_opt,unit", GROUPS)
def test_decode_oracle_streams(int_opt, unit, layout, odd):
    codec = _codec(int_opt, unit)
    ts, vals, start, e = _case(int_opt, unit, layout, odd)
    S, P = ts.shape
    rows, streams, x_ts, x_v, mask = _oracle_decode(e, int_opt, unit, P)
    for place in (_csr, _scattered):
        blob, off, lengths = place(streams)
        for pm in (False, True):
            r = codec.decode(blob, off, P, lengths=lengths, point_major=pm)
            torch.cuda.synchronize()
            assert (r.status.cpu().numpy() == 0).all() and (r.n_points.cpu().numpy() == e.n_ok[rows]).all()
            g_ts, g_v = r.ts.cpu().numpy(), r.values.cpu().numpy().view(np.uint64)
            if pm:
                g_ts, g_v = g_ts.T, g_v.T
            assert ((g_ts == x_ts) | ~mask).all(), (place.__name__, pm)
            assert ((g_v == x_v.view(np.uint64)) | ~mask).all(), (place.__name__, pm)


@pytest.mark.parametrize("layout", ["uniform", "mixed"])
@pytest.mark.parametrize("int_opt,unit", GROUPS)
def test_append_one_datapoint_per_call(int_opt, unit, layout):
    """every datapoint index is a call boundary: the state record is saved and loaded at every grammar state, and
    every snapshot is the oracle's Stream() of the prefix; a failing datapoint stops its series"""
    codec = _codec(int_opt, unit)
    odd = layout == "mixed"
    ts, vals, start, e = _case(int_opt, unit, layout, odd)
    S, P = ts.shape
    d_ts, d_v = _t(ts), _t(vals)
    es = codec.encoder_set(_t(start), codec.encode_bound(P))
    pm = layout == "uniform"  # the point-major input stage on the uniform warps, the series-major one on the others
    for i in range(P):
        take = (i < e.n_ok) | (i == e.n_ok)  # the failing datapoint is offered once
        n = _t(take.astype(np.int32))
        a, b = d_ts[:, i: i + 1], d_v[:, i: i + 1]
        if pm:
            a, b = a.t(), b.t()
        n_app, st = es.append(a.contiguous(), b.contiguous(), n_points=n, unit=unit, point_major=pm)
        snap = es.stream()
        torch.cuda.synchronize()
        n_app, st = n_app.cpu().numpy(), st.cpu().numpy()
        fails = i == e.n_ok
        assert (st[fails] == e.status[fails]).all() and (n_app[fails] == 0).all(), i
        assert (st[~fails] == 0).all() and (n_app[~fails] == take[~fails]).all(), i
        k = np.minimum(i + 1, e.n_ok)
        ex = _prefixes(int_opt, unit, layout, odd)[i]
        _same_streams(snap.out.cpu().numpy(), snap.out_len.cpu().numpy(), ex, np.nonzero(k == i + 1)[0])
        short = np.nonzero(k < i + 1)[0]  # after a failure: the stream of the datapoints before it
        _same_streams(snap.out.cpu().numpy(), snap.out_len.cpu().numpy(), e, short)


@functools.lru_cache(maxsize=None)
def _prefixes(int_opt, unit, layout, odd):
    ts, vals, start, _ = _case(int_opt, unit, layout, odd)
    return [Oracle(ts[:, : i + 1], vals[:, : i + 1], start, int_opt, unit) for i in range(ts.shape[1])]


@pytest.mark.parametrize("point_major", [False, True])
@pytest.mark.parametrize("int_opt", [False, True])
def test_widest_codes_capacity_stop_on_every_row(int_opt, point_major):
    """slots sized so that the capacity stop of the widest codes falls on every row of a 4-row input tile: the
    stop, out_len, status and bytes of the per-datapoint model, and nothing written past a finished stream"""
    from m3_b200 import capi
    from m3_b200.codec import BatchCodec
    codec = BatchCodec(0, int_opt)
    Pw = 64
    series = [s for lane in range(LANES) for s in G.widest(lane, Pw) if s.int_opt == int_opt]
    ts = np.stack([s.ts for s in series])
    vals = np.stack([s.vals for s in series])
    S = len(series)
    n_pts = np.full(S, Pw, dtype=np.int32)
    n_pts[::7] = Pw - 1 - np.arange(len(n_pts[::7])) % 5
    stops = set()
    for stride in range(96, 96 + 16 * 14, 16):
        expected = [_expected(ts[s], vals[s], int(n_pts[s]), int_opt, stride // 4) for s in range(S)]
        stops |= {k % 4 for _, st, k in expected if st == capi.ERR_CAPACITY}
        _check(_encode(codec, ts, vals, n_pts, stride, point_major), expected)
    assert stops == {0, 1, 2, 3}, stops
    stride = codec.encode_bound(Pw)
    buf, out_len, status = _encode_into_sentinel(codec, ts, vals, n_pts, stride, point_major)
    assert (status == 0).all()
    _check_slots(buf, out_len, status, [_expected(ts[s], vals[s], int(n_pts[s]), int_opt, stride // 4)[0]
                                        for s in range(S)], stride)


# ---------------------------------------------------------------------------------------------------------------
# fused downsample
# ---------------------------------------------------------------------------------------------------------------
N_WIN = 17


def _window_edge_series(int_opt, unit):
    """32-lane warps of a steady cadence equal to the window, every datapoint exactly on a window end, or 1 ns
    before one (from a start 1 ns before the unit's grid: the first datapoint changes the unit, and the timestamps
    decode exactly): the hot path's window advance at its edge.  (start, ts, values) per lane."""
    win = 20 * G.UNIT_NS[unit]
    out = []
    for back in (0, 1):
        for lane in range(LANES):
            ts = G.START0 - back + win * np.arange(1, G.P + 1, dtype=np.int64)
            out.append((G.START0 - back, ts, np.array(G._walk(lane, G.P, 11 + back))))
    return out


@pytest.mark.parametrize("layout", ["uniform", "mixed"])
@pytest.mark.parametrize("int_opt,unit", GROUPS)
def test_fused_downsample(int_opt, unit, layout):
    codec = _codec(int_opt, unit)
    ts, vals, start, e = _case(int_opt, unit, layout, layout == "mixed")
    S, P = ts.shape
    keep, streams, x_ts, x_v, _ = _oracle_decode(e, int_opt, unit, P)
    S = len(keep)
    rows = [(x_ts[j, : e.n_ok[s]], x_v[j, : e.n_ok[s]]) for j, s in enumerate(keep)]
    for w_start, w_ts, w_v in _window_edge_series(int_opt, unit):  # their own warps, after the corpus' last warp
        b = O.encode_series(w_ts, w_v, w_start, unit, int_opt, default_unit=unit)
        streams.append(b)
        d_ts, d_v, n, st = O.decode_series(b, int_opt, unit)
        assert st == 0 and n == G.P and (d_ts == w_ts).all()
        rows.append((d_ts, d_v))
    pad = (-S) % 32  # (the first stream again up to a whole warp)
    streams = streams[:S] + streams[:1] * pad + streams[S:]
    rows = rows[:S] + rows[:1] * pad + rows[S:]
    win = 20 * G.UNIT_NS[unit]
    blob, off, _ = _csr(streams)
    kinds = ["plain", "last", "sum_sq"] + (["counter"] if int_opt else [])
    for kind in kinds:
        kw = {"last": {"want_last": True}, "sum_sq": {"want_sum_sq": True}, "plain": {}}.get(kind, {})
        if kind == "counter":
            from m3_b200 import capi
            kw = {"metric": capi.METRIC_COUNTER}
        r = codec.decode_downsample(blob, off, G.START0, win, N_WIN, **kw)
        torch.cuda.synchronize()
        assert (r.status.cpu().numpy() == 0).all()
        assert (r.n_points.cpu().numpy() == [len(t) for t, _ in rows]).all()
        h = lambda t: t.cpu().numpy()
        if kind in ("plain", "last"):
            exp = [O.downsample_series(t, v, G.START0, win, N_WIN) for t, v in rows]
        elif kind == "sum_sq":
            exp = [A.downsample_gauge_ex(t, v, G.START0, win, N_WIN) for t, v in rows]
        else:
            exp = [A.downsample_counter(t, v, G.START0, win, N_WIN) for t, v in rows]
        exp = [np.stack([x[j] for x in exp], axis=1) for j in range(len(exp[0]))]
        if kind == "counter":
            for g, x in zip((r.sum, r.count, r.min, r.max, r.sum_sq), exp):
                assert (h(g) == x).all()
            continue
        g_sum, x_sum = h(r.sum), exp[0]
        assert ((g_sum.view(np.uint64) == x_sum.view(np.uint64)) | (np.isnan(g_sum) & np.isnan(x_sum))).all(), kind
        assert (h(r.count) == exp[1]).all(), kind
        for g, x in ((r.min, exp[2]), (r.max, exp[3])):
            assert (h(g).view(np.uint64) == x.view(np.uint64)).all(), kind
        if kind == "last":
            assert (h(r.last).view(np.uint64) == exp[4].view(np.uint64)).all()
        if kind == "sum_sq":
            assert (h(r.last).view(np.uint64) == exp[4].view(np.uint64)).all() and (h(r.last_at) == exp[5]).all()
            assert (h(r.sum_sq).view(np.uint64) == exp[6].view(np.uint64)).all()
