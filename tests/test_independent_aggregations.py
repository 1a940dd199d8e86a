"""The Gauge's expensive aggregations (sumSq, Stdev) and the Counter, without a GPU: the CPU oracle against the
reference's test tables (tests/golden/m3tsz_agg_goldens.json), against a second, pure-Python
restatement of src/aggregator/aggregation/{gauge,counter,common}.go written from the reference (Python ints masked
to 64 bits, Go/amd64 int64(float64)), and, for every valid (metric, aggregation type) pair of the tile aggregation,
against the independent encoder of tests/indep_m3tsz.py.  Also compiles the two copies of the amd64 conversion and
the kernels' stdev (m3tsz_common.cuh, m3tsz_encode.cu) for the host and checks them against the oracle."""
import ctypes as C
import json
import math
import os
import struct

import numpy as np
import pytest

import agg_oracle_lib as A
import oracle_lib as O
from host_build import compile, cut, fn, source_text

SEC = 1_000_000_000
M64 = (1 << 64) - 1
HERE = os.path.dirname(os.path.abspath(__file__))
AMD64_NAN = 0xFFF8000000000000  # the invalid-operation NaN of SSE2 (Inf - Inf, sqrt(-x))


def bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def f64(b):
    return struct.unpack("<d", struct.pack("<Q", b & M64))[0]


def s64(u):
    u &= M64
    return u - (1 << 64) if u >> 63 else u


def go_int64(v):
    """int64(v) on amd64 (CVTTSD2SQ): truncation; NaN, +-Inf and |v| >= 2^63 (except -2^63) -> MinInt64."""
    if v != v or v >= 2.0 ** 63 or v < -(2.0 ** 63):
        return -(1 << 63)
    return int(v)  # Python int() truncates toward zero


def stdev(count, sum_sq, sum_):
    """common.go:29-37; every NaN is amd64's default NaN."""
    div = s64(count * (count - 1))
    if div == 0:
        return 0.0
    num = float(count) * sum_sq - sum_ * sum_
    q = num / float(div)
    if q != q or q < 0:
        return f64(AMD64_NAN)
    return math.sqrt(q)


def window_of(t, start, window):
    return (t - start) // window  # Python floor division = Truncate for the window start


def gauge_windows(ts, vals, start, window, n_windows):
    """Gauge with HasExpensiveAggregations per window: gauge.go:74-103."""
    go_nan = f64(0x7FF8000000000001)  # math.NaN()
    ws = [dict(sum=0.0, sum_sq=0.0, count=0, mn=go_nan, mx=go_nan, last=0.0, last_at=None)
          for _ in range(n_windows)]
    for t, v in zip(ts, vals):
        w = window_of(t, start, window)
        if not 0 <= w < n_windows:
            continue
        g = ws[w]
        if g["last_at"] is None or t > g["last_at"]:
            g["last_at"], g["last"] = t, v
        g["count"] += 1
        if v != v:
            continue
        g["sum"] += v
        if g["mx"] != g["mx"] or g["mx"] < v:
            g["mx"] = v
        if g["mn"] != g["mn"] or g["mn"] > v:
            g["mn"] = v
        g["sum_sq"] += v * v
    return ws


def counter_windows(ts, vals, start, window, n_windows):
    """Counter fed int64(value): counter.go:44-78, int64 arithmetic wrapping like Go."""
    ws = [dict(sum=0, sum_sq=0, count=0, mn=(1 << 63) - 1, mx=-(1 << 63)) for _ in range(n_windows)]
    for t, v in zip(ts, vals):
        w = window_of(t, start, window)
        if not 0 <= w < n_windows:
            continue
        c, x = ws[w], go_int64(v)
        c["sum"] = s64(c["sum"] + x)
        c["count"] += 1
        if c["mx"] < x:
            c["mx"] = x
        if c["mn"] > x:
            c["mn"] = x
        c["sum_sq"] = s64(c["sum_sq"] + x * x)
    return ws


def gauge_value_of(agg, g):
    return {1: g["last"], 2: g["mn"], 3: g["mx"], 4: (g["sum"] / float(g["count"])) if g["count"] else 0.0,
            6: float(g["count"]), 7: g["sum"], 8: g["sum_sq"], 9: stdev(g["count"], g["sum_sq"], g["sum"])}[agg]


def counter_value_of(agg, c):
    return {2: float(c["mn"]), 3: float(c["mx"]), 4: (float(c["sum"]) / float(c["count"])) if c["count"] else 0.0,
            6: float(c["count"]), 7: float(c["sum"]), 8: float(c["sum_sq"]),
            9: stdev(c["count"], float(c["sum_sq"]), float(c["sum"]))}[agg]


SPECIALS = [math.nan, math.inf, -math.inf, -0.0, 0.0, 2.0 ** 63, -(2.0 ** 63), 2.0 ** 63 - 1024, -1.5, 1.5, -2.5,
            0.9999, -0.9999, 3.0e18, 4.0e9, -4.0e9, 9.3e18, 1e-300]


def random_series(rng, n, start, window, n_windows):
    """Stream order with steps back (out of order), datapoints before and after the range, special values and values
    whose sums / squares wrap int64."""
    t = start - 2 * window + int(rng.integers(0, window // SEC)) * SEC
    ts, vals = [], []
    for _ in range(n):
        ts.append(t)
        r = rng.random()
        if r < 0.35:
            vals.append(SPECIALS[int(rng.integers(0, len(SPECIALS)))])
        elif r < 0.7:
            vals.append(float(int(rng.integers(-10 ** 6, 10 ** 6))))
        else:
            vals.append(float(np.round(rng.normal(0, 500), 2)))
        step = int(rng.integers(1, 2 * window // SEC)) * SEC
        t += step if rng.random() > 0.15 else -3 * step
    return np.array(ts, dtype=np.int64), np.array(vals, dtype=np.float64)


def _beq(a, b):
    return bits(float(a)) == bits(float(b))


def test_conversion_and_stdev_match_restatement():
    for v in SPECIALS + [-1.0, 1.0, -(2.0 ** 63) + 1024, 123456.789, -123456.789]:
        assert A.go_int64(v) == go_int64(v), v
    assert go_int64(-1.5) == -1 and go_int64(-0.0) == 0 and go_int64(-(2.0 ** 63)) == -(1 << 63)
    assert go_int64(2.0 ** 63) == -(1 << 63) and go_int64(math.nan) == -(1 << 63)
    rng = np.random.default_rng(5)
    for _ in range(2000):
        c = int(rng.integers(-3, 10 ** 6))
        sq = float(rng.choice([0.0, math.inf, float(rng.random() * 1e12)]))
        s = float(rng.choice([0.0, math.inf, -math.inf, float(rng.normal() * 1e6)]))
        assert _beq(A.stdev(c, sq, s), stdev(c, sq, s)), (c, sq, s)
    assert _beq(A.stdev(3, 0.0, 5.0), f64(AMD64_NAN))  # negative numerator: NaN, amd64's


@pytest.mark.parametrize("seed", range(6))
def test_gauge_and_counter_windows_match_oracle(seed):
    rng = np.random.default_rng(900 + seed)
    start, window, n_windows = 1599955200 * SEC, 60 * SEC, 10
    for _ in range(30):
        ts, vals = random_series(rng, int(rng.integers(0, 300)), start, window, n_windows)
        o = A.downsample_gauge_ex(ts, vals, start, window, n_windows)
        for w, g in enumerate(gauge_windows(ts.tolist(), vals.tolist(), start, window, n_windows)):
            assert o[1][w] == g["count"]
            assert o[5][w] == (g["last_at"] or 0)
            for j, k in ((0, "sum"), (2, "mn"), (3, "mx"), (4, "last"), (6, "sum_sq")):
                assert _beq(o[j][w], g[k]) or (math.isnan(o[j][w]) and math.isnan(g[k]) and k == "sum"), (w, k)
        oc = A.downsample_counter(ts, vals, start, window, n_windows)
        for w, c in enumerate(counter_windows(ts.tolist(), vals.tolist(), start, window, n_windows)):
            assert [int(oc[j][w]) for j in range(5)] == [c["sum"], c["count"], c["mn"], c["mx"], c["sum_sq"]], w


def test_counter_wraps():
    ts = np.arange(6, dtype=np.int64) * SEC
    vals = np.array([3.0e18, 3.0e18, 3.0e18, 4.0e9, -1.5, 2.0 ** 63])
    s, c, mn, mx, sq = A.downsample_counter(ts, vals, 0, 60 * SEC, 1)
    exp = counter_windows(ts.tolist(), vals.tolist(), 0, 60 * SEC, 1)[0]
    assert int(s[0]) == exp["sum"] and int(sq[0]) == exp["sum_sq"] and int(mn[0]) == -(1 << 63)
    assert int(mx[0]) == 3 * 10 ** 18 and s64(9 * 10 ** 18 + 4 * 10 ** 9 - 1 - (1 << 63)) == exp["sum"]


def test_goldens():
    g = json.load(open(os.path.join(HERE, "golden", "m3tsz_agg_goldens.json")))
    val = lambda x: math.nan if x == "NaN" else x
    for case in g["gauge"]:
        n = len(case["values"])
        ts = np.array(case["times"], dtype=np.int64) * SEC + 10 * SEC
        s, c, mn, mx, last, last_at, sq = A.downsample_gauge_ex(ts, np.array(case["values"], dtype=np.float64),
                                                                0, 3600 * SEC, 1)
        for t, want in case["value_of"].items():
            got = A.gauge_value_of_ex(int(t), s[0], c[0], mn[0], mx[0], last[0], sq[0])
            assert (math.isnan(got) and math.isnan(val(want))) or got == want, (case["name"], t)
        if "stdev" in case:
            want, delta = case["stdev"]
            assert abs(A.gauge_value_of_ex(9, s[0], c[0], mn[0], mx[0], last[0], sq[0]) - want) <= delta
        assert c[0] == n
    for case in g["counter"]:
        ts = np.arange(len(case["values"]), dtype=np.int64) * SEC
        s, c, mn, mx, sq = A.downsample_counter(ts, np.array(case["values"], dtype=np.float64), 0, 3600 * SEC, 1)
        assert int(s[0]) == case["sum"]
        for t, want in case["value_of"].items():
            assert A.counter_value_of(int(t), s[0], c[0], mn[0], mx[0], sq[0]) == want, (case["name"], t)
        if "stdev" in case:
            want, delta = case["stdev"]
            assert abs(A.counter_value_of(9, s[0], c[0], mn[0], mx[0], sq[0]) - want) <= delta
        for t, want in case.get("invalid_value_of", {}).items():
            assert A.counter_value_of(int(t), s[0], c[0], mn[0], mx[0], sq[0]) == want
    for case in g["stdev"]:
        assert abs(A.stdev(case["count"], case["sum_sq"], case["sum"]) - case["want"]) <= case["delta"]


PAIRS = [(A.METRIC_GAUGE, a) for a in (1, 2, 3, 4, 6, 7, 8, 9)] + [(A.METRIC_COUNTER, a) for a in (2, 3, 4, 6, 7, 8, 9)]


@pytest.mark.parametrize("metric,agg", PAIRS)
def test_tiles_every_valid_pair_match_restatement_and_independent_encoder(metric, agg):
    import indep_m3tsz as I
    rng = np.random.default_rng(7000 + 10 * metric + agg)
    start, step, n_windows = 1599955200 * SEC, 300 * SEC, 24
    for _ in range(12):
        n = int(rng.integers(0, 300))
        ts = np.sort(start + rng.integers(0, n_windows * step // SEC, size=n) * SEC)
        vals = np.round(rng.normal(size=n) * 50, int(rng.integers(0, 3)))
        if n:
            vals[rng.integers(0, n, size=max(1, n // 20))] = rng.choice([math.nan, 3.0e18, -1.5, math.inf])
        t_o, v_o = A.aggregate_tiles_series_ex(ts, vals, start, step, n_windows, metric, agg)
        ws = (counter_windows if metric == A.METRIC_COUNTER else gauge_windows)(ts.tolist(), vals.tolist(), start,
                                                                             step, n_windows)
        vo = counter_value_of if metric == A.METRIC_COUNTER else gauge_value_of
        exp = [(start + (i + 1) * step, vo(agg, w)) for i, w in enumerate(ws) if w["count"]]
        assert t_o.tolist() == [e[0] for e in exp]
        for a, (_, b) in zip(v_o.tolist(), exp):
            assert _beq(a, b) or (math.isnan(a) and math.isnan(b) and agg in (4, 7)), (a, b)
        if metric == A.METRIC_GAUGE and agg == 1:
            continue  # covered by test_independent_query_rows
        if exp:
            mine = I.encode(start, [(t, v, O.UNIT_S, b"") for t, v in zip(t_o.tolist(), v_o.tolist())], True)
            assert mine == O.encode_series(t_o, v_o, start, O.UNIT_S, True)


# ---- the device functions, compiled for the host ----
EXPORTS = r"""
extern "C" {
int64_t dev_i64(double v) { return go_f64_to_i64(v); }
uint64_t dev_u64(double v) { return go_f64_to_u64_via_i64(v); }
double dev_stdev(int64_t c, double sq, double s) { return agg_stdev(c, sq, s); }
}
"""


def test_device_conversion_and_stdev_on_host():
    com, enc = source_text("m3tsz_common.cuh"), source_text("m3tsz_encode.cu")
    body = "\n".join([cut(com, fn("go_f64_to_i64")), cut(enc, fn("go_f64_to_u64_via_i64")), cut(com, fn("agg_stdev"))])
    L = compile("agg_host", body, EXPORTS)
    L.dev_i64.restype, L.dev_i64.argtypes = C.c_int64, [C.c_double]
    L.dev_u64.restype, L.dev_u64.argtypes = C.c_uint64, [C.c_double]
    L.dev_stdev.restype, L.dev_stdev.argtypes = C.c_double, [C.c_int64, C.c_double, C.c_double]
    rng = np.random.default_rng(11)
    vals = SPECIALS + [f64(int(b)) for b in rng.integers(0, 1 << 63, size=2000, dtype=np.uint64)]
    vals += [float(x) for x in rng.normal(size=2000) * 1e19]
    for v in vals:
        assert L.dev_i64(v) == A.go_int64(v) and L.dev_u64(v) == (A.go_int64(v) & M64), v
    for _ in range(3000):
        c = int(rng.integers(-3, 10 ** 7))
        sq = float(rng.choice([0.0, math.inf, float(rng.random() * 1e15)]))
        s = float(rng.choice([0.0, math.inf, -math.inf, float(rng.normal() * 1e7)]))
        assert _beq(L.dev_stdev(c, sq, s), A.stdev(c, sq, s)), (c, sq, s)
