"""A pure-Python restatement of the rollup's fold and source forward, written from the Go source
(aggregation/gauge.go:74-101, aggregation/counter.go:52-78, GenericElem.AddUnique generic_elem.go:246-281 and
processValue's forward branch generic_elem.go:892-937), checked bit for bit against the composed oracle
(rollup_oracle_lib): fold values, forwarded values and records, on random values, memberships and call splits."""
import math
import struct

import numpy as np

import agg_oracle_lib as A
import elem_oracle_lib as E
import oracle_lib as O
import rollup_oracle_lib as R
import xf_oracle_lib as X

GO_NAN = struct.unpack("<d", struct.pack("<Q", 0x7FF8000000000001))[0]
SEC = 10 ** 9
STEP = 60 * SEC
R0 = 1_700_000_040 * SEC


def bits(x):
    return struct.unpack("<Q", struct.pack("<d", float(x)))[0]


def go_int64(v):
    if not (-9223372036854775808.0 <= v < 9223372036854775808.0):
        return -(1 << 63)
    return int(v)


def wrap(x):
    x &= (1 << 64) - 1
    return x - (1 << 64) if x >> 63 else x


def amd64_add(a, x):
    """ADDSD of a total and a non-NaN value: a NaN total keeps its payload, Inf + -Inf is the default NaN"""
    r = a + x
    if r == r:
        return r
    if a != a:
        return a
    return struct.unpack("<d", struct.pack("<Q", 0xFFF8000000000000))[0]


def fold_gauge(values):
    """NewGauge, then Gauge.Update of every value at one timestamp"""
    s, c, mn, mx, last, sq, last_at = 0.0, 0, GO_NAN, GO_NAN, 0.0, 0.0, None
    for x in values:
        if last_at is None:  # lastAt.IsZero(); an equal timestamp is never After it
            last_at, last = 1, x
        c += 1
        if math.isnan(x):
            continue
        s = amd64_add(s, x)
        if math.isnan(mx) or mx < x:
            mx = x
        if math.isnan(mn) or mn > x:
            mn = x
        sq = amd64_add(sq, x * x)
    return s, c, mn, mx, last, sq


def fold_counter(values):
    s, c, mn, mx, sq = 0, 0, (1 << 63) - 1, -(1 << 63), 0
    for x in values:
        v = go_int64(x)
        s = wrap(s + v)
        c += 1
        mx = max(mx, v)
        mn = min(mn, v)
        sq = wrap(sq + v * v)
    return s, c, mn, mx, sq


SPECIALS = [GO_NAN, struct.unpack("<d", struct.pack("<Q", 0x7FF8000000000abc))[0], math.inf, -math.inf, 0.0, -0.0,
            2.0 ** 63, -(2.0 ** 63), 2.0 ** 64, 4.0e9, 3.0e18, -1.5, 1e16, 1.0]


def random_values(rng, n):
    return [SPECIALS[int(rng.integers(0, len(SPECIALS)))] if rng.random() < 0.5 else float(rng.normal(0, 1e3))
            for _ in range(n)]


def test_fold_matches_the_oracle():
    rng = np.random.default_rng(1)
    for _ in range(3000):
        vs = random_values(rng, int(rng.integers(0, 9)))
        g, o = fold_gauge(vs), R.fold_gauge(vs)
        assert [bits(x) for x in (g[0], g[2], g[3], g[4], g[5])] == [bits(x) for x in (o[0], o[2], o[3], o[4], o[5])]
        assert g[1] == o[1]
        assert fold_counter(vs) == R.fold_counter(vs)


def test_fold_edges():
    # equal timestamps: Last is the first member's value, NaN payload included
    nan_b = struct.unpack("<d", struct.pack("<Q", 0x7FF8000000000abc))[0]
    assert bits(R.fold_gauge([nan_b, 1.0, 2.0])[4]) == 0x7FF8000000000abc
    assert R.fold_gauge([nan_b, 1.0])[1] == 2
    # +-0 in both orders: the first is kept by min and max
    assert bits(R.fold_gauge([-0.0, 0.0])[2]) == bits(-0.0) and bits(R.fold_gauge([0.0, -0.0])[3]) == bits(0.0)
    # int64(): NaN and values >= 2^63 are MinInt64; the sums wrap
    assert R.fold_counter([math.nan, 2.0 ** 63])[0] == 0 and R.fold_counter([math.nan])[2] == -(1 << 63)
    assert R.fold_counter([3.0e18] * 4)[0] == wrap(4 * 3000000000000000000)
    assert R.fold_counter([4.0e9, 4.0e9])[4] == wrap(2 * 4000000000 ** 2)
    # Inf + -Inf: the default NaN, kept by later adds
    assert bits(R.fold_gauge([math.inf, -math.inf, 1.0])[0]) == 0xFFF8000000000000


def forward(ts, vals, metric, src, ops, discard, st):
    """restated source element: ValueOf(src) of each non-empty window, the op chain (xf oracle's arithmetic), a
    discarded NaN dropped, the value alone forwarded"""
    wt, wv = A.aggregate_tiles_series_ex(ts, vals, R0, STEP, 12, metric, src)
    out = {}
    for t, v in zip(wt.tolist(), wv.tolist()):
        to, vo = X.transform_series(ops, False, STEP, st, [t], [v])
        x = float(vo[0])
        if discard and math.isnan(x):
            continue
        out[(t - R0) // STEP - 1] = x
    return out


def series(rng):
    n = int(rng.integers(1, 60))
    ts = R0 - STEP + np.cumsum(rng.integers(1, 40, n)) * SEC
    vals = np.array(random_values(rng, n))
    return ts.astype(np.int64), vals


def test_forward_matches_the_oracle():
    rng = np.random.default_rng(2)
    for metric, src, ops in ((A.METRIC_COUNTER, A.AGG_SUM, [3]), (A.METRIC_GAUGE, A.AGG_LAST, [1, 2]),
                             (A.METRIC_GAUGE, A.AGG_MAX, [5, 4]), (A.METRIC_COUNTER, A.AGG_MIN, [])):
        for discard in (True, False):
            for _ in range(20):
                ts, vals = series(rng)
                a, b = X.new_transform_state(), X.new_transform_state()
                got = forward(ts, vals, metric, src, ops, discard, a)
                want = R.forward_series(ts, vals, R0, STEP, 12, metric, src, ops, discard, b)
                assert {k: bits(v) for k, v in got.items()} == {k: bits(v) for k, v in want.items()}
                assert a.tobytes() == b.tobytes()


def restated_call(decoded, metric, src, pre, off, mem, types, post, discard, xs, gs, w0, n_win):
    """the whole call from the restated pieces and the element oracle; records updated in place"""
    fwd, ok = [], []
    new = []
    for s, (ts, vals, err) in enumerate(decoded):
        st = xs[s: s + 1].copy()
        wt, wv = A.aggregate_tiles_series_ex(ts, vals, R0 + w0 * STEP, STEP, n_win, metric, src)
        f = {}
        for t, v in zip(wt.tolist(), wv.tolist()):
            to, vo = X.transform_series(pre, False, STEP, st, [t], [v])
            if not (discard and math.isnan(float(vo[0]))):
                f[(t - R0) // STEP - 1 - w0] = float(vo[0])
        fwd.append(f)
        new.append(st[0])
        ok.append(err == 0)
    rows = []
    for g in range(len(off) - 1):
        ms = [int(m) for m in mem[off[g]: off[g + 1]]]
        wt, wv = [], []
        for w in range(n_win):
            vs = [fwd[m][w] for m in ms if w in fwd[m]]
            if vs:
                wt.append(R0 + (w0 + w + 1) * STEP)
                if metric == A.METRIC_COUNTER:
                    s_, c, mn, mx, sq = fold_counter(vs)
                    wv.append([A.counter_value_of(a, s_, c, mn, mx, sq) for a in types])
                else:
                    s_, c, mn, mx, last, sq = fold_gauge(vs)
                    wv.append([A.gauge_value_of_ex(a, s_, c, mn, mx, last, sq) for a in types])
        st = gs[g: g + 1].copy()
        res = E.element_series(post, discard, STEP, len(types), st, np.array(wt, dtype=np.int64),
                               np.array(wv, dtype=np.float64).reshape(len(wt), len(types)))
        gs[g] = st[0]
        rows.append([O.encode_series(t, v, R0 + w0 * STEP, O.UNIT_S, True) if len(t) else b"" for t, v in res])
    for s in range(len(decoded)):
        xs[s] = new[s]
    return rows


def test_calls_match_the_oracle_across_splits():
    rng = np.random.default_rng(3)
    pipes = [(A.METRIC_COUNTER, A.AGG_SUM, [3], [7], [4]), (A.METRIC_GAUGE, A.AGG_LAST, [], [2, 3, 7], []),
             (A.METRIC_GAUGE, A.AGG_MEAN, [1, 2], [1, 4, 6, 8, 9], [4, 5]),
             (A.METRIC_COUNTER, A.AGG_MAX, [5], [2, 3, 9], [3])]
    for metric, src, pre, types, post in pipes:
        decoded = [(ts, vals, 0) for ts, vals in (series(rng) for _ in range(12))]
        lists = [list(rng.integers(0, 12, int(rng.integers(0, 5)))) for _ in range(7)]
        off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
        mem = np.array([m for x in lists for m in x], dtype=np.int32)
        for discard in (True, False):
            for edges in ([0, 12], [0, 5, 12], [0, 2, 3, 7, 11, 12]):
                xs1, gs1 = np.zeros(12, X.XF_STATE_DTYPE), np.zeros(7, E.ELEM_STATE_DTYPE)
                xs2, gs2 = np.zeros(12, X.XF_STATE_DTYPE), np.zeros(7, E.ELEM_STATE_DTYPE)
                for a, b in zip(edges[:-1], edges[1:]):
                    want, src_st = R.aggregate_tiles_rollup(decoded, True, R0 + a * STEP, STEP, b - a, metric, src,
                                                            pre, off, mem, types, post, discard, xs1, gs1)
                    got = restated_call(decoded, metric, src, pre, off, mem, types, post, discard, xs2, gs2, a, b - a)
                    assert src_st == [0] * 12
                    assert all(r[0] == 0 for row in want for r in row)
                    assert [[want[j][g][1] for j in range(len(types))] for g in range(7)] == got
                    assert xs1.tobytes() == xs2.tobytes() and gs1.tobytes() == gs2.tobytes()


def test_one_member_group_is_the_element():
    """one member, no pre-ops, NaN-free values: the rollup element sees the source's own window values"""
    rng = np.random.default_rng(4)
    for metric, src, post in ((A.METRIC_GAUGE, A.AGG_LAST, [4]), (A.METRIC_COUNTER, A.AGG_SUM, [3, 5])):
        for _ in range(10):
            n = int(rng.integers(1, 60))
            ts = (R0 - STEP + np.cumsum(rng.integers(1, 40, n)) * SEC).astype(np.int64)
            vals = np.round(rng.normal(0, 1e3, n)).astype(np.float64)
            gs = np.zeros(1, E.ELEM_STATE_DTYPE)
            rows, _ = R.aggregate_tiles_rollup([(ts, vals, 0)], True, R0, STEP, 12, metric, src, [],
                                               np.array([0, 1]), np.array([0], dtype=np.int32), [src], post, True,
                                               np.zeros(1, X.XF_STATE_DTYPE), gs)
            st = E.new_element_state()
            t, v = E.aggregate_tiles_types_series(ts, vals, R0, STEP, 12, metric, [src], post, True, st)[0]
            assert rows[0][0][1] == (O.encode_series(t, v, R0, O.UNIT_S, True) if len(t) else b"")
            assert gs.tobytes() == st.tobytes()


def _goldens():
    import json
    import os
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "m3tsz_rollup_goldens.json")) as f:
        return json.load(f)


def _num(x):
    return math.nan if x == "NaN" else float(x)


def test_goldens_forward():
    """testPipeline's forwarded values: Absolute, PerSecond on each window's value, only the value forwarded"""
    for case in _goldens()["forward"]:
        step = case["step_ns"]
        ends = [t for t, _ in case["windows"]]
        r0 = ends[0] - step
        # one datapoint per window, at the window's start: its ValueOf(Sum / Last) is the datapoint's value
        ts = np.array([t - step for t in ends], dtype=np.int64)
        vals = np.array([v for _, v in case["windows"]], dtype=np.float64)
        st = X.new_transform_state()
        got = R.forward_series(ts, vals, r0, step, len(ends), case["metric_type"], case["src_type"], case["ops"],
                               case["discard_nan"], st)
        want = {(t - r0) // step - 1: _num(v) for t, v in case["want"]}
        assert sorted(got) == sorted(want), case["name"]
        for w, v in want.items():
            assert (math.isnan(v) and math.isnan(got[w])) or got[w] == v, (case["name"], w, got[w], v)
        assert float(st["prev_v"][0]) == case["consumed"]


def test_goldens_folds():
    """the rollup element's AddUnique: the restatement and the oracle reproduce what the reference tests assert"""
    for case in _goldens()["folds"]:
        for step in case["steps"]:
            vs, want = step["values"], step["want"]
            eps = want.get("eps", 0.0)
            if case["metric_type"] == A.METRIC_COUNTER:
                outs = [fold_counter(vs), R.fold_counter(vs)]
                got = [dict(sum=o[0], count=o[1], max=o[3], sum_sq=o[4]) for o in outs]
            else:
                outs = [fold_gauge(vs), R.fold_gauge(vs)]
                got = [dict(sum=o[0], count=o[1], max=o[3], sum_sq=o[5]) for o in outs]
            for g in got:
                for k, v in want.items():
                    if k == "eps":
                        continue
                    if eps and k == "sum":
                        assert abs(g[k] - v) <= eps * abs(v), (case["name"], k, g[k], v)
                    else:
                        assert g[k] == v, (case["name"], vs, k, g[k], v)


def test_goldens_flush_timestamps():
    """a rollup window receives its values at a timestamp aligned to its resolution (the source window's end here)
    and the forwarded list writes it at that window's start: the same timestamp, so the tile timestamps of the rollup
    rows are the source windows' ends"""
    case = _goldens()["flush"]
    res = case["resolution_ns"]
    for added, want in zip(case["added_at_ns"], case["want_flush_ns"]):
        assert added - added % res == want  # AddUnique's Truncate, then forwardedMetricTimestampNanos
    for el in case["elements"]:
        v = [el["value"]]
        if el["metric_type"] == A.METRIC_COUNTER:
            s_, c, mn, mx, sq = fold_counter(v)
            assert A.counter_value_of(case["agg_type"], s_, c, mn, mx, sq) == el["value"]
        else:
            s_, c, mn, mx, last, sq = fold_gauge(v)
            assert A.gauge_value_of_ex(case["agg_type"], s_, c, mn, mx, last, sq) == el["value"]
