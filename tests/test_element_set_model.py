"""The element sets' CPU model (tests/element_set_model.py) on the reference's element tables
(tests/golden/m3tsz_element_consume_goldens.json), against the tile element oracle, and with the reference's rule for
late writes pinned next to this library's."""
import json
import os

import numpy as np
import pytest

import agg_oracle_lib as A
import elem_oracle_lib as E
from element_set_model import ERR_CAPACITY, ERR_CLOSED, OK, ElementModel, window_start

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SEC = 1_000_000_000


def _load(name):
    with open(os.path.join(GOLDEN, name)) as f:
        return json.load(f)


def _bits(v):
    return int(np.array([v], dtype=np.float64).view(np.uint64)[0])


def add_case_datapoints(case):
    """an "adds" case's datapoints [(t, value)], read from the annotation goldens where it says so"""
    if "datapoints_from" not in case:
        return [(t, v) for t, v in case["datapoints"]]
    src = {c["name"]: c for c in _load(case["datapoints_from"])["cases"]}[case["name"]]
    return [(t, v) for t, v, _ in src["datapoints"]]


def window_fields(model, ws):
    """what the element tests assert on a window: its aggregates and Mean"""
    a = model.aggregates(ws)
    a["mean"] = model.value_of(ws, A.AGG_MEAN)
    return a


@pytest.mark.parametrize("case", _load("m3tsz_element_consume_goldens.json")["adds"], ids=lambda c: c["name"])
def test_goldens_add(case):
    m = ElementModel(case["metric_type"], case["agg_types"], case["resolution_ns"])
    dps = add_case_datapoints(case)
    assert len(dps) == len(case["want_windows"])
    for (t, v), want in zip(dps, case["want_windows"]):
        assert m.add([(t, _bits(v))]) == ([OK], OK)
        assert sorted(m.windows) == [w["start_ns"] for w in want]
        for w in want:
            got = window_fields(m, w["start_ns"])
            for f, x in w.items():
                if f != "start_ns":
                    assert got[f] == x, (case["name"], w["start_ns"], f)


@pytest.mark.parametrize("case", _load("m3tsz_element_consume_goldens.json")["consumes"], ids=lambda c: c["name"])
def test_goldens_consume(case):
    m = ElementModel(case["metric_type"], case["agg_types"], case["resolution_ns"])
    assert m.add([(t, _bits(v)) for t, v in case["windows"]]) == ([OK] * len(case["windows"]), OK)
    for step in case["steps"]:
        got = m.consume(step["target_ns"])
        assert [list(zip(t.tolist(), v.tolist())) for t, v in got] == [[tuple(x) for x in w] for w in step["want"]]


def test_window_start_is_go_truncation():
    # a resolution that divides a day: floor division; 7 s: counted from the zero time (62135596800 % 7 == 3)
    assert window_start(-1, 60 * SEC) == -60 * SEC
    assert window_start(59 * SEC, 60 * SEC) == 0
    assert window_start(0, 7 * SEC) == -4 * SEC
    assert window_start(3 * SEC, 7 * SEC) == 3 * SEC


def random_series(rng, start, res, n_windows, metric_type, whole_seconds=True):
    """datapoints [(t, value bits)] in arrival order: windows in order, datapoints out of order inside each"""
    pts = []
    for w in range(n_windows):
        if rng.random() < 0.25:
            continue
        n = int(rng.integers(1, 5))
        off = rng.integers(0, res // SEC, n) * SEC if whole_seconds else rng.integers(0, res, n)
        for o in off:
            if metric_type == A.METRIC_COUNTER:
                v = float(rng.integers(-1000, 1000))
            else:
                v = float(rng.choice([rng.normal() * 100, np.nan, np.inf, -np.inf, 0.0], p=[.85, .05, .04, .03, .03]))
            pts.append((start + w * res + int(o), _bits(v)))
    return pts


@pytest.mark.parametrize("metric_type", [A.METRIC_GAUGE, A.METRIC_COUNTER])
def test_model_equals_tile_element_oracle(metric_type):
    rng = np.random.default_rng(7 + metric_type)
    res, start = 60 * SEC, 1_600_000_020 * SEC
    for it in range(60):
        n_windows = int(rng.integers(1, 12))
        types = sorted(rng.choice([2, 3, 4, 6, 7, 8, 9] + ([1] if metric_type == A.METRIC_GAUGE else []),
                                  int(rng.integers(1, 4)), replace=False).tolist())
        ops = [[], [3], [1, 2], [4], [5], [4, 3, 5]][it % 6]
        pts = random_series(rng, start, res, n_windows, metric_type)
        m = ElementModel(metric_type, types, res, ops, True, open_windows=n_windows)
        assert m.add(pts)[1] == OK
        got = m.consume(start + n_windows * res)
        ts = np.array([t for t, _ in pts], dtype=np.int64)
        vs = np.array([v for _, v in pts], dtype=np.uint64).view(np.float64)
        st = E.new_element_state()
        # (the oracle discards NaN with any list; the tile calls and the element sets only with transformations)
        exp = E.aggregate_tiles_types_series(ts, vs, start, res, n_windows, metric_type, types, ops, len(ops) > 0, st)
        for j in range(len(types)):
            assert np.array_equal(got[j][0], exp[j][0])
            assert np.array_equal(got[j][1].view(np.uint64), exp[j][1].view(np.uint64)), (it, j)
        assert m.state.tobytes() == st.tobytes()


def test_late_writes_reference_rule_and_watermark_rule():
    """GenericElem keeps only the last consumed window closed: a write to an older one opens a fresh window, which
    the next Consume flushes after the later one it already flushed (Increase then sees its previous value go
    backwards).  Here every window up to the watermark is closed and each output stays in time order."""
    res = 10 * SEC
    runs = {}
    for rule in ("reference", "watermark"):
        m = ElementModel(A.METRIC_GAUGE, [A.AGG_LAST], res, ops=[3], rule=rule, open_windows=None)
        assert m.add([(211 * SEC, _bits(5.0)), (221 * SEC, _bits(7.0))]) == ([OK, OK], OK)
        first = m.consume(230 * SEC)
        late = m.add([(212 * SEC, _bits(9.0)), (222 * SEC, _bits(1.0))])[0]
        second = m.consume(240 * SEC)
        runs[rule] = (first, late, second)
    ref_first, ref_late, ref_second = runs["reference"]
    assert ref_late == [OK, ERR_CLOSED]  # 210 s was dropped from the element; 220 s is the one it keeps closed
    assert ref_second[0][0].tolist() == [220 * SEC]  # the 210 s window again, behind 230 s
    wm_first, wm_late, wm_second = runs["watermark"]
    assert wm_late == [ERR_CLOSED, ERR_CLOSED]
    assert len(wm_second[0][0]) == 0
    assert [x.tolist() for x in wm_first[0]] == [x.tolist() for x in ref_first[0]] == [[220 * SEC, 230 * SEC],
                                                                                        [5.0, 2.0]]


def test_capacity_stops_the_rest_of_the_element():
    m = ElementModel(A.METRIC_COUNTER, [A.AGG_SUM], 10 * SEC, open_windows=2)
    res, st = m.add([(1 * SEC, _bits(1.0)), (11 * SEC, _bits(2.0)), (21 * SEC, _bits(3.0)), (2 * SEC, _bits(4.0))])
    assert (res, st) == ([OK, OK, ERR_CAPACITY, ERR_CAPACITY], ERR_CAPACITY)
