"""The two kernels that consume decoded rows on the fetch path, at their edges, on the device against the oracle:

* the series merge (m3tsz_merge.cu) with NaN payloads, +-Inf and +-0 at equal timestamps, where the equal-timestamp
  strategies sort with < / > (false on NaN) and count frequencies by == (0 for NaN, one key for +-0), on both sides
  of the fast kernel's replica limit, from arrays and from real streams decoded on the device;
* the Prometheus epilogue (m3tsz_query.cu) with ragged warps and blocks, every mode, empty / one / full rows, output
  capacity overflow, timestamps on resolution boundaries, at the tolerance limit and below zero, special values and
  counter resets to +-0;
* rows whose count exceeds their capacity (what decode and merge report when they hit it), which the epilogue
  refuses without reading them -- given directly, and produced by decode and by merge.

The merge only moves values, so every bit is compared.  The epilogue's cumulative sum is arithmetic: a NaN it makes
from non-NaN inputs (Inf - Inf) is the GPU's, and where two NaNs meet in it the H100 does not always keep the one
amd64 keeps (DESIGN.md section 6).  Any NaN is accepted there and in the sums that carry such a NaN; every other
output, a NaN carried from one input included, is compared bit for bit."""
import math

import numpy as np
import pytest

import oracle_lib as O
import test_independent_merge as M
from test_gpu_merge import assert_same, gpu_merge
from test_independent_query_rows import _go_div

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

SEC = 1_000_000_000
ERR_CAPACITY, ERR_INVALID_ARG = 100, 101


@pytest.fixture(scope="module")
def codec():
    from m3_b200.codec import BatchCodec
    return BatchCodec(0, True)


# ------------------------------------------------------------------ merge at special values
SHAPES = {  # (replicas, readers per slice)
    "fast_path": ((1, 4), (1, 1)),        # the fast kernel's shape (strategy 0)
    "several_readers": ((1, 4), (2, 4)),
    "many_replicas": ((5, 12), (1, 4)),   # beyond the fast kernel's 4 replicas
}


@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("strategy", [0, 1, 2, 3])
def test_merge_special_values(codec, strategy, shape):
    reps, rds = SHAPES[shape]
    rng = np.random.default_rng(2100 + strategy * 7 + sorted(SHAPES).index(shape))
    series = M.special_value_series(rng, 150, replicas=reps, readers=rds)
    for start, end in ((0, 0), M.SPECIAL_RANGE):
        got, exp = gpu_merge(codec, series, start=start, end=end, strategy=strategy)
        assert_same(got, exp)
        assert (exp[3] == 0).all() and int(exp[2].sum()) > 0


def _upload_streams(streams):
    blob = b"".join(streams)
    off = np.zeros(len(streams) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(x) for x in streams])
    buf = torch.zeros(len(blob) + 16, dtype=torch.uint8, device="cuda")
    buf[: len(blob)] = torch.frombuffer(bytearray(blob), dtype=torch.uint8).cuda()
    return buf[: len(blob)], off


def _rf3_streams(rng, S, P, start, values):
    """RF = 3, one block: each replica misses a few writes, and the replicas' values at a timestamp often differ"""
    streams = []
    for s in range(S):
        t = start + (np.arange(P) * 10 + rng.integers(0, 5, size=P)) * SEC
        base = values(rng, P)
        for r in range(3):
            keep = rng.random(P) < 0.9
            v = np.where(rng.random(P) < 0.5, values(rng, P), base)
            streams.append(O.encode_series(t[keep], v[keep], start, O.UNIT_S, True))
    return streams


def _special(rng, k):
    return np.array(M.SPECIAL_VALUES)[rng.integers(0, len(M.SPECIAL_VALUES), size=k)]


@pytest.mark.parametrize("strategy", [0, 1, 2, 3])
def test_decode_then_merge_special_values(codec, strategy):
    """real M3TSZ streams carrying the special values (the codec keeps NaN payloads), decoded and merged on the
    device == the oracle's decode and merge, every bit"""
    rng = np.random.default_rng(2200 + strategy)
    S, P = 64, 40
    start = 1599955200 * SEC
    streams = _rf3_streams(rng, S, P, start, _special)
    buf, off = _upload_streams(streams)
    dec = codec.decode(buf, torch.from_numpy(off).cuda(), P)
    n_seq = len(streams)
    ar = lambda stop, step: torch.arange(0, stop, step, dtype=torch.int64, device="cuda")
    got = codec.merge_series(dec.ts, dec.values, dec.n_points, dec.status, ar(n_seq + 1, 1), ar(n_seq + 1, 1),
                             ar(n_seq + 1, 3), P, 0, 0, strategy)
    torch.cuda.synchronize()
    got = [x.cpu().numpy() for x in got]
    got[2] = got[2].view(np.uint32)
    o_ts, o_val, o_n, o_st = O.decode_batch(np.frombuffer(b"".join(streams), dtype=np.uint8), off, P)
    assert (o_st == 0).all()
    assert (dec.n_points.cpu().numpy().view(np.uint32) == o_n).all()
    sq = np.arange(n_seq + 1, dtype=np.uint64)
    exp = O.series_merge_batch(o_ts, o_val, o_n, o_st, sq, sq, sq[::3], strategy=strategy, out_cap=P)
    assert_same(got, exp)
    assert np.isnan(exp[1]).any() and np.isinf(exp[1]).any()


# ------------------------------------------------------------------ Prometheus epilogue
T_FILL, V_FILL = -777, 0x7FF4DEADBEEF0001  # output prefill: an int and a NaN bit pattern nobody computes
Q = 15 * SEC                            # timestamps are whole quanta (plus a per-series offset)
RES = 60 * SEC                          # resolution: every fourth quantum is a window boundary
ORIGIN = 1599955200 * SEC               # a multiple of RES
UNTIL = ORIGIN + 37 * Q                 # a timestamp many series have exactly
TOL = 1e-3
MODES = {"plain": (False, False), "tolerance": (True, False), "resets": (False, True), "both": (True, True)}
EDGE_VALUES = M.SPECIAL_VALUES + [1e308, -1.0]


def _edge_rows(rng, rows, cap):
    """rows of `cap` datapoints: timestamps on the resolution boundaries and 1 ns / 1 ms - 1 ns beside them, from
    ORIGIN or from below zero across it; values of four families -- counters whose resets go to +0 or -0,
    dips around the tolerance (the exact limit included), special values, counters with special values"""
    ts = np.zeros((rows, cap), dtype=np.int64)
    vals = np.zeros((rows, cap), dtype=np.float64)
    for s in range(rows):
        origin = ORIGIN if s % 2 == 0 else -20 * Q
        offset = (0, 0, -1, 1, 999_999)[(s // 2) % 5]
        ts[s] = origin + offset + np.cumsum(rng.choice([1, 1, 2, 3], size=cap)) * Q
        fam = (s // 10) % 4
        cur = 0.0
        for i in range(cap):
            if fam == 0 or fam == 3:
                if rng.random() < 0.15:
                    cur = float(rng.choice([0.0, -0.0]))
                else:
                    cur = cur + float(rng.integers(0, 5))
                v = cur
                if fam == 3 and rng.random() < 0.1:
                    v = EDGE_VALUES[int(rng.integers(0, len(EDGE_VALUES)))]
            elif fam == 1:
                prev = vals[s, i - 1] if i else 1000.0
                v = prev * (1 - float(rng.choice([1e-5, 1e-4, TOL, 1e-2]))) if rng.random() < 0.3 else prev + 1.5
            else:
                v = EDGE_VALUES[int(rng.integers(0, len(EDGE_VALUES)))]
            vals[s, i] = v
    return ts, vals


def _counts(rng, S, cap):
    n = rng.integers(0, cap + 1, size=S).astype(np.uint32)
    n[: min(S, 3)] = [0, 1, cap][: min(S, 3)] if S > 1 else [cap]
    return n


def prom(codec, ts, vals, n, S, resolution, handle, tol, until, out_cap):
    """m3tsz_prom_convert_batch over the first S rows of ts / vals (host or device; they may have more rows) into
    outputs prefilled with T_FILL / V_FILL -> host arrays (ts_ms, value bits, n_out, status)"""
    from m3_b200 import capi
    from m3_b200.codec import _cuda_stream_ptr, _ptr
    d = lambda a: a if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a)).cuda()
    d_ts, d_v, d_n = d(ts), d(vals), d(n if torch.is_tensor(n) else n.astype(np.uint32).view(np.int32))
    d_h = None if handle is None else d(np.asarray(handle, dtype=np.uint8))
    t_out = torch.full((S, out_cap), T_FILL, dtype=torch.int64, device="cuda")
    v_out = torch.full((S, out_cap), V_FILL, dtype=torch.int64, device="cuda").view(torch.float64)
    n_out = torch.full((S,), 12345, dtype=torch.int32, device="cuda")
    st = torch.full((S,), -1, dtype=torch.int32, device="cuda")
    rc = capi.lib().m3tsz_prom_convert_batch(
        codec.ctx.handle, _ptr(d_ts), _ptr(d_v), d_ts.shape[1], _ptr(d_n), S, int(resolution), _ptr(d_h),
        float(tol), int(until), _ptr(t_out), _ptr(v_out), out_cap, _ptr(n_out), _ptr(st),
        _cuda_stream_ptr(codec.device))
    codec.ctx.check(rc, "m3tsz_prom_convert_batch")
    torch.cuda.synchronize()
    return (t_out.cpu().numpy(), v_out.cpu().numpy().view(np.uint64), n_out.cpu().numpy().view(np.uint32),
            st.cpu().numpy())


def _loose_nan(ts, vals, resolution, handle, tol, until):
    """per output sample of iteratorToPromResult: whether its value is a NaN whose bits are not the one input NaN
    it was carried from -- made by the cumulative sum from non-NaN inputs (Inf - Inf, Inf + -Inf), or where two
    NaNs met (a NaN sum plus a NaN difference, a NaN minus a NaN); a NaN sum stays what it is until then"""
    if not handle:
        return []
    out = []
    first, cum, loose = True, 0.0, False
    prev_t, prev_v = 0, 0.0
    for t, v in zip(ts.tolist(), vals.tolist()):
        if tol > 0 and t < until and not first and v < prev_v and v > prev_v * (1 - tol):
            v = prev_v
        if _go_div(t, resolution) != _go_div(prev_t, resolution) and not first:
            out.append(loose)
        if v < prev_v:
            d, d_loose = v, False
        else:
            d = v - prev_v
            d_loose = math.isnan(d) and math.isnan(v) == math.isnan(prev_v)
        if not math.isnan(cum + d):
            loose = False
        elif math.isnan(cum) != math.isnan(d):
            loose = loose if math.isnan(cum) else d_loose
        else:
            loose = True
        cum += d
        prev_t, prev_v, first = t, v, False
    if not first:
        out.append(loose)
    return out


def assert_series(s, ts, vals, k, resolution, handle, tol, until, out_cap, got):
    """series s == the oracle's conversion of its k datapoints, with the NaN rule of the module docstring"""
    t_out, v_out, n_out, st = got
    e_ts, e_v = O.prom_convert_series(ts[:k], vals[:k], resolution, handle, tol, until)
    assert int(n_out[s]) == len(e_ts), (s, int(n_out[s]), len(e_ts))
    assert int(st[s]) == (ERR_CAPACITY if len(e_ts) > out_cap else 0), (s, int(st[s]))
    m = min(len(e_ts), out_cap)
    assert (t_out[s, :m] == e_ts[:m]).all(), s
    g, e = v_out[s, :m], e_v[:m].view(np.uint64)
    loose = np.array(_loose_nan(ts[:k], vals[:k], resolution, handle, tol, until)[:m] or [False] * m, dtype=bool)
    assert len(loose) == m, s
    exact = ~loose
    assert (g[exact] == e[exact]).all(), (s, [hex(int(x)) for x in g[exact][g[exact] != e[exact]][:4]])
    assert np.isnan(g[loose].view(np.float64)).all() and np.isnan(e[loose].view(np.float64)).all(), s
    assert (t_out[s, m:] == T_FILL).all() and (v_out[s, m:] == V_FILL).all(), s  # nothing past the samples
    return loose.sum()


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("S", [1, 31, 33, 257, 4099])
def test_prom_edges(codec, S, mode):
    use_tol, use_resets = MODES[mode]
    rng = np.random.default_rng(2300 + S + sorted(MODES).index(mode))
    cap = 48
    ts, vals = _edge_rows(rng, S, cap)
    n = _counts(rng, S, cap)
    tol, until = (TOL, UNTIL) if use_tol else (0.0, 0)
    handle = (rng.random(S) < 0.75).astype(np.uint8) if use_resets else None
    hits_until = int((ts == UNTIL).any(axis=1).sum())
    for out_cap in (cap + 1, 7):  # room for every sample, and fewer than most series produce
        got = prom(codec, ts, vals, n, S, RES, handle, tol, until, out_cap)
        for s in range(S):
            h = bool(handle[s]) if handle is not None else False
            assert_series(s, ts[s], vals[s], int(n[s]), RES, h, tol, until, out_cap, got)
        if S > 1:
            assert (got[3] == ERR_CAPACITY).any() == (out_cap == 7)
    if S >= 257 and use_tol:
        assert hits_until > 10  # t == tolerance_until is in the batch


@pytest.mark.parametrize("mode", ["plain", "resets", "both"])
@pytest.mark.parametrize("S", [33, 257])
def test_prom_refuses_rows_shorter_than_their_count(codec, S, mode):
    """a middle series and the last one have n_points > cap: INVALID_ARG, n_out 0, output rows still holding
    their prefill.  The input is the first S rows of a larger tensor whose extra rows hold sentinels, which would
    be converted if the last series' row were read past its end."""
    use_tol, use_resets = MODES[mode]
    rng = np.random.default_rng(2400 + S + len(mode))
    cap, extra = 40, 2
    ts, vals = _edge_rows(rng, S + extra, cap)
    ts[S:], vals[S:] = ORIGIN, 4321.0
    n = _counts(rng, S, cap)
    mid, last = S // 2, S - 1
    n[mid - 1], n[mid], n[last] = cap, cap + 1, cap + cap // 2
    tol, until = (TOL, UNTIL) if use_tol else (0.0, 0)
    handle = np.ones(S, dtype=np.uint8) if use_resets else None
    big_ts, big_v = torch.from_numpy(ts).cuda(), torch.from_numpy(vals).cuda()
    for out_cap in (cap + 1, cap + cap):
        got = prom(codec, big_ts[:S], big_v[:S], n, S, RES, handle, tol, until, out_cap)
        t_out, v_out, n_out, st = got
        for s in range(S):
            if s in (mid, last):
                assert int(st[s]) == ERR_INVALID_ARG and int(n_out[s]) == 0, (s, int(st[s]), int(n_out[s]))
                assert (t_out[s] == T_FILL).all() and (v_out[s] == V_FILL).all(), s
            else:
                assert_series(s, ts[s], vals[s], int(n[s]), RES, use_resets, tol, until, out_cap, got)


def test_decode_capacity_then_prom(codec):
    """decode with max_points below some streams' lengths (status CAPACITY, n_points = the full count) ->
    the epilogue on the decoded arrays: those series are refused, the others equal the oracle's decode and
    conversion"""
    rng = np.random.default_rng(2500)
    S, P, cap = 96, 64, 40
    start = 1599955200 * SEC
    lens = rng.integers(1, P + 1, size=S)
    lens[-1] = cap - 3  # the last row is not over-long: its reads stay inside the allocation either way
    streams = []
    for s in range(S):
        t = start + np.cumsum(rng.integers(1, 90, size=lens[s])) * SEC
        v = np.cumsum(rng.integers(0, 7, size=lens[s])).astype(np.float64)
        v[rng.random(lens[s]) < 0.05] = 0.0
        streams.append(O.encode_series(t, v, start, O.UNIT_S, True))
    buf, off = _upload_streams(streams)
    dec = codec.decode(buf, torch.from_numpy(off).cuda(), cap)
    torch.cuda.synchronize()
    d_n, d_st = dec.n_points.cpu().numpy().view(np.uint32), dec.status.cpu().numpy()
    assert (d_n == lens).all() and ((d_st == ERR_CAPACITY) == (lens > cap)).all()
    assert 10 < int((lens > cap).sum()) < S - 10
    o_ts, o_val, o_n, o_st = O.decode_batch(np.frombuffer(b"".join(streams), dtype=np.uint8), off, P)
    for handle in (None, np.ones(S, dtype=np.uint8)):
        got = prom(codec, dec.ts, dec.values, dec.n_points, S, 300 * SEC, handle, 0.0, 0, cap + 1)
        for s in range(S):
            if lens[s] > cap:
                assert int(got[3][s]) == ERR_INVALID_ARG and int(got[2][s]) == 0, s
                assert (got[0][s] == T_FILL).all() and (got[1][s] == V_FILL).all(), s
            else:
                assert_series(s, o_ts[s], o_val[s], int(o_n[s]), 300 * SEC, handle is not None, 0.0, 0, cap + 1, got)


def test_merge_capacity_then_prom(codec):
    """RF = 3 decode -> merge with out_cap below some merged lengths (status CAPACITY, n_out = the full count) ->
    the epilogue on the merge output: those series are refused, the others equal the oracle's decode, merge and
    conversion"""
    rng = np.random.default_rng(2600)
    S, P, out_cap = 64, 60, 48
    start = 1599955200 * SEC
    counter = lambda rng, k: np.cumsum(rng.integers(0, 4, size=k)).astype(np.float64)
    streams = []
    for s in range(S):
        p = int(rng.integers(20, P + 1)) if s < S - 1 else 30  # the last series stays inside its row
        streams += _rf3_streams(rng, 1, p, start, counter)
    buf, off = _upload_streams(streams)
    dec = codec.decode(buf, torch.from_numpy(off).cuda(), P)
    n_seq = len(streams)
    ar = lambda stop, step: torch.arange(0, stop, step, dtype=torch.int64, device="cuda")
    m_ts, m_val, m_n, m_st = codec.merge_series(dec.ts, dec.values, dec.n_points, dec.status, ar(n_seq + 1, 1),
                                                ar(n_seq + 1, 1), ar(n_seq + 1, 3), out_cap)
    torch.cuda.synchronize()
    o_ts, o_val, o_n, o_st = O.decode_batch(np.frombuffer(b"".join(streams), dtype=np.uint8), off, P)
    sq = np.arange(n_seq + 1, dtype=np.uint64)
    e_ts, e_val, e_n, e_st = O.series_merge_batch(o_ts, o_val, o_n, o_st, sq, sq, sq[::3], out_cap=P)
    over = e_n > out_cap
    assert (m_n.cpu().numpy().view(np.uint32) == e_n).all()
    assert ((m_st.cpu().numpy() == ERR_CAPACITY) == over).all() and 5 < int(over.sum()) < S - 5
    for handle in (None, np.ones(S, dtype=np.uint8)):
        got = prom(codec, m_ts, m_val, m_n, S, 300 * SEC, handle, 0.0, 0, out_cap + 1)
        for s in range(S):
            if over[s]:
                assert int(got[3][s]) == ERR_INVALID_ARG and int(got[2][s]) == 0, s
                assert (got[0][s] == T_FILL).all() and (got[1][s] == V_FILL).all(), s
            else:
                assert_series(s, e_ts[s], e_val[s], int(e_n[s]), 300 * SEC, handle is not None, 0.0, 0,
                              out_cap + 1, got)
