"""The element-rollup model (tests/element_rollup_model.py) against the reference's rollup tables
(tests/golden/m3tsz_rollup_goldens.json) fed as adds, a forward and a group consume, against the tile rollup's
oracle (rollup_oracle_lib.aggregate_tiles_rollup) fed in one add, one forward and one consume, and its closed and
commit rules on their own."""
import json
import math
import os

import numpy as np

import agg_oracle_lib as A
import oracle_lib as O
import rollup_oracle_lib as R
import xf_oracle_lib as X
from element_rollup_model import (ERR_CAPACITY, ERR_CLOSED, ERR_INVALID_ARG, OK, GroupModel, SourceModel,
                                  forward)
from elem_oracle_lib import ELEM_STATE_DTYPE

SEC = 1_000_000_000
GAUGE, COUNTER = A.METRIC_GAUGE, A.METRIC_COUNTER
LAST, MIN, MAX, SUM = 1, 2, 3, 7


def _goldens():
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "m3tsz_rollup_goldens.json")) as f:
        return json.load(f)


def _bits(v):
    return int(np.array([v], dtype=np.float64).view(np.uint64)[0])


def _same(a, b):
    return (math.isnan(a) and math.isnan(b)) or a == b


def test_goldens_forward_through_a_group():
    """testPipeline: each window's value through Absolute, PerSecond is forwarded and written by a one-member group at
    the source window's end; the source's record keeps the last value consumed"""
    for case in _goldens()["forward"]:
        step, metric = case["step_ns"], case["metric_type"]
        src = SourceModel(metric, case["src_type"], step, case["ops"], case["discard_nan"], open_windows=8)
        rollup = SUM if metric == COUNTER else LAST
        grp = GroupModel(metric, [rollup], step, open_windows=8)
        src.add([(t - step, _bits(v)) for t, v in case["windows"]])
        st, gst = forward([src], [grp], case["windows"][-1][0], [0, 1], [0])
        assert st == [OK] and gst == [OK]
        (ts, vs), = grp.consume(case["windows"][-1][0])
        assert ts.tolist() == [t for t, _ in case["want"]], case["name"]
        for got, (_, w) in zip(vs.tolist(), case["want"]):
            if metric == COUNTER:  # the rollup element's Counter.Update(int64(value)): NaN is MinInt64
                assert got == (-(2.0 ** 63) if w == "NaN" else float(int(w))), case["name"]
            else:
                assert _same(got, math.nan if w == "NaN" else w), case["name"]
        assert float(np.frombuffer(src.state.tobytes()[:96], dtype=X.XF_STATE_DTYPE)["prev_v"][0]) == \
            case["consumed"]


def test_goldens_folds_as_forwards():
    """AddUnique's tables: each step's values come from that many one-window sources listed in order"""
    for case in _goldens()["folds"]:
        metric = case["metric_type"]
        for step in case["steps"]:
            vs, want = step["values"], step["want"]
            srcs = [SourceModel(metric, SUM if metric == COUNTER else LAST, 10 * SEC) for _ in vs]
            for s, v in zip(srcs, vs):
                s.add([(100 * SEC, _bits(v))])
            grp = GroupModel(metric, [SUM], 10 * SEC)
            st, gst = forward(srcs, [grp], 110 * SEC, [0, len(vs)], list(range(len(vs))))
            assert gst == [OK] and st == [OK] * len(vs)
            a = grp.aggregates(100 * SEC)
            for k, v in want.items():
                if k == "eps":
                    continue
                if "eps" in want and k == "sum":
                    assert abs(a[k] - v) <= want["eps"] * abs(v), (case["name"], k)
                else:
                    assert a[k] == v, (case["name"], vs, k, a[k], v)


def test_goldens_flush_timestamps():
    """a value added in the source window that ends at added_at is written by the group at added_at"""
    case = _goldens()["flush"]
    res = case["resolution_ns"]
    for el in case["elements"]:
        metric = el["metric_type"]
        for added, want in zip(case["added_at_ns"], case["want_flush_ns"]):
            src = SourceModel(metric, SUM if metric == COUNTER else LAST, res)
            src.add([(added - res, _bits(el["value"]))])
            grp = GroupModel(metric, [case["agg_type"]], res)
            forward([src], [grp], added, [0, 1], [0])
            (ts, vs), = grp.consume(added)
            assert ts.tolist() == [want] and vs.tolist() == [el["value"]]


PIPES = [  # (metric, src type, pre-ops, rollup types, post-ops)
    (COUNTER, SUM, [3], [SUM], [4]),
    (GAUGE, LAST, [], [MIN, MAX, SUM], []),
    (GAUGE, LAST, [1, 2], [LAST, SUM], [5]),
]


def test_one_call_equals_the_tile_rollup():
    """every datapoint in one add, one forward, one group consume: the tile rollup's rows, statuses and records (on
    finite values, where the two sides' discard rules agree)"""
    rng = np.random.default_rng(5)
    step, n_win = 10 * SEC, 6
    r0 = 1_700_000_000 * SEC // step * step
    for metric, src_type, pre, types, post in PIPES:
        for it in range(4):
            S, G = 12, 5
            cols = []
            for s in range(S):
                n = int(rng.integers(0, 12))
                ts = np.sort(rng.choice(n_win * 10, n, replace=False)) * (step // 10) + r0
                vs = (rng.integers(0, 1000, n) if metric == COUNTER else rng.normal(size=n) * 10).astype(np.float64)
                cols.append((ts.astype(np.int64), vs))
            members = rng.integers(0, S, int(rng.integers(G, 3 * G))).astype(np.int32)
            cut = np.sort(rng.integers(0, len(members) + 1, G - 1))
            group_off = np.concatenate([[0], cut, [len(members)]]).astype(np.int64)
            discard = bool(it % 2)
            srcs = [SourceModel(metric, src_type, step, pre, discard, open_windows=n_win) for _ in range(S)]
            grps = [GroupModel(metric, types, step, post, discard, open_windows=n_win) for _ in range(G)]
            for s, (ts, vs) in zip(srcs, cols):
                assert s.add([(int(t), _bits(v)) for t, v in zip(ts, vs)])[1] == OK
            end = r0 + n_win * step
            st, gst = forward(srcs, grps, end, group_off, members)
            assert st == [OK] * S and gst == [OK] * G
            xs = np.zeros(S, dtype=X.XF_STATE_DTYPE)
            gs = np.zeros(G, dtype=ELEM_STATE_DTYPE)
            rows, sst = R.aggregate_tiles_rollup([(ts, vs, 0) for ts, vs in cols], True, r0, step, n_win, metric,
                                                 src_type, pre, group_off, members, types, post, discard, xs, gs)
            for g in range(G):
                out = grps[g].consume(end)
                for j in range(len(types)):
                    b = O.encode_series(out[j][0], out[j][1], r0, O.UNIT_S, True) if len(out[j][0]) else b""
                    assert rows[j][g] == (0, b, len(out[j][0])), (metric, it, g, j)
                assert grps[g].state.tobytes() == gs[g].tobytes()
            for s in range(S):
                assert srcs[s].state.tobytes()[:96] == xs[s].tobytes()


def test_closed_group_window():
    """a group window that ended by the group's watermark drops its values; the group's other windows still fold and
    the sources commit"""
    res = 10 * SEC
    a, b = SourceModel(GAUGE, LAST, res), SourceModel(GAUGE, LAST, res)
    grp = GroupModel(GAUGE, [SUM], res)
    a.add([(0, _bits(1.0))])
    forward([a, b], [grp], res, [0, 2], [0, 1])
    assert grp.consume(res)[0][0].tolist() == [res]
    b.add([(0, _bits(2.0)), (res, _bits(3.0))])  # b's window [0, res) was never due: still open
    st, gst = forward([a, b], [grp], 2 * res, [0, 2], [0, 1])
    assert gst == [ERR_CLOSED] and st == [OK, OK]
    assert list(grp.windows) == [res] and grp.windows[res] == [3.0]
    assert b.windows == {} and b.watermark == 2 * res


def test_commit_rule_and_retry():
    """a CAPACITY group holds back its members (their windows, record and watermark), a source in another group that
    succeeded is held back too but that group keeps its fold; growing and re-running exactly the failed group gives
    the unstopped result"""
    res = 10 * SEC

    def setup(R_small):
        srcs = [SourceModel(COUNTER, SUM, res, [3]) for _ in range(3)]
        for i, s in enumerate(srcs):
            s.add([(w * res + i, _bits(float(10 * w + i))) for w in range(3)])
        grps = [GroupModel(COUNTER, [SUM], res, open_windows=R_small), GroupModel(COUNTER, [SUM], res)]
        return srcs, grps

    off, mem = [0, 2, 4], [0, 1, 1, 2]
    srcs, grps = setup(2)
    st, gst = forward(srcs, grps, 3 * res, off, mem)
    assert gst == [ERR_CAPACITY, OK] and st == [ERR_CAPACITY, ERR_CAPACITY, OK]
    assert grps[0].windows == {} and len(srcs[0].windows) == 3 and srcs[2].windows == {}
    grps[0].R = 4
    st, gst = forward(srcs, grps[:1], 3 * res, [0, 2], [0, 1])
    assert gst == [OK] and st == [OK, OK, OK]
    want_s, want_g = setup(4)
    forward(want_s, want_g, 3 * res, off, mem)
    for g, w in zip(grps, want_g):
        assert g.windows == w.windows
    for s, w in zip(srcs, want_s):
        assert s.state.tobytes() == w.state.tobytes() and s.watermark == w.watermark


def test_invalid_groups_hold_back_what_they_name():
    res = 10 * SEC
    srcs = [SourceModel(GAUGE, LAST, res) for _ in range(3)]
    for s in srcs:
        s.add([(0, _bits(1.0))])
    grps = [GroupModel(GAUGE, [SUM], res) for _ in range(3)]
    # group 0 names source 7; group 1's range decreases; group 2 lists sources 0, 1, 1: it folds source 0's value,
    # which group 0 holds back, and source 1's twice
    st, gst = forward(srcs, grps, res, [0, 2, 1, 4], [7, 0, 1, 1])
    assert gst == [ERR_INVALID_ARG, ERR_INVALID_ARG, OK]
    assert st == [ERR_INVALID_ARG, OK, OK] and grps[2].windows == {0: [1.0, 1.0, 1.0]}
    assert grps[0].windows == {} and srcs[0].windows and not srcs[1].windows and not srcs[2].windows


def test_group_side_discard_keeps_the_element_set_rule():
    """with discard_nan, no post-ops and a NaN rollup value (+Inf + -Inf in a Sum) the group set writes it, where the
    tile rollup drops it"""
    res = 10 * SEC
    srcs = [SourceModel(GAUGE, LAST, res, [], True) for _ in range(2)]
    srcs[0].add([(0, _bits(math.inf))])
    srcs[1].add([(0, _bits(-math.inf))])
    grp = GroupModel(GAUGE, [SUM], res, [], True)
    forward(srcs, [grp], res, [0, 2], [0, 1])
    (ts, vs), = grp.consume(res)
    assert ts.tolist() == [res] and math.isnan(vs[0])
    rows, _ = R.aggregate_tiles_rollup([(np.array([0], dtype=np.int64), np.array([v]), 0) for v in (math.inf, -math.inf)],
                                       True, 0, res, 1, GAUGE, LAST, [], [0, 2], [0, 1], [SUM], [], True,
                                       np.zeros(2, dtype=X.XF_STATE_DTYPE), np.zeros(1, dtype=ELEM_STATE_DTYPE))
    assert rows[0][0] == (0, b"", 0)
