"""The annotated element-set model (tests/element_set_ann_model.py) on the reference's annotation cases
(tests/golden/m3tsz_tile_annotation_goldens.json: TestGaugeReturnsLastNonEmptyAnnotation,
TestCounterReturnsLastNonEmptyAnnotation and the TestCounterElemAddUnion* annotation steps, which are the element's
own rule) fed as adds, against the window rule of the annotation oracle (ann_oracle_lib.window_annotations) on random
in-order sequences, and on the cases that rule cannot state: late datapoints, refused ones and the capacity stop."""
import json
import os

import numpy as np
import pytest

import agg_oracle_lib as A
import ann_oracle_lib as N
from element_set_ann_model import AnnotatedElementModel, annotated_points
from element_set_model import ERR_CAPACITY, ERR_CLOSED, OK
from test_element_set_model import _bits, random_series

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "m3tsz_tile_annotation_goldens.json")
SEC = 1_000_000_000
PAYLOADS = [bytes([0x08, 0x01, 0x10, 0x01]), b"gauge", b"longer payload"]


def _goldens():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


def _types(metric):
    return [A.AGG_LAST] if metric == A.METRIC_GAUGE else [A.AGG_SUM]


@pytest.mark.parametrize("case", _goldens(), ids=lambda c: c["name"])
@pytest.mark.parametrize("one_call", [True, False])
def test_goldens_as_adds(case, one_call):
    m = AnnotatedElementModel(case["metric_type"], _types(case["metric_type"]), case["step_ns"],
                              open_windows=case["n_windows"], start_ns=case["start_ns"])
    dps = [(int(t), _bits(v), bytes.fromhex(a)) for t, v, a in case["datapoints"]]
    if one_call:
        assert m.add(dps) == ([OK] * len(dps), OK)
    else:
        for dp in dps:
            assert m.add([dp]) == ([OK], OK)
    for w, want in enumerate(case["want_windows"]):
        ws = case["start_ns"] + w * case["step_ns"]
        assert m.window_annotation(ws) == bytes.fromhex(want), (case["name"], w)
    out = m.consume(case["start_ns"] + case["n_windows"] * case["step_ns"])
    want = [bytes.fromhex(a) for a in case["want_windows"]]
    assert out[0][2] == [want[w] for w in range(case["n_windows"])
                         if case["start_ns"] + (w + 1) * case["step_ns"] in out[0][0].tolist()]


@pytest.mark.parametrize("metric", [A.METRIC_GAUGE, A.METRIC_COUNTER])
def test_window_rule_equals_the_oracle(metric):
    rng = np.random.default_rng(40 + metric)
    res, start = 60 * SEC, 1_600_000_020 * SEC
    for it in range(60):
        n_windows = int(rng.integers(1, 10))
        pts = annotated_points(random_series(rng, start, res, n_windows, metric), rng, PAYLOADS, 0.5)
        m = AnnotatedElementModel(metric, _types(metric), res, open_windows=n_windows)
        assert m.add(pts)[1] == OK
        ts = np.array([t for t, _, _ in pts], dtype=np.int64)
        ids = np.array([i if a else -1 for i, (_, _, a) in enumerate(pts)], dtype=np.int64)
        win = N.window_annotations(ts, ids, start, res, n_windows)
        for w in range(n_windows):
            ws = start + w * res
            if ws in m.ann:
                assert m.window_annotation(ws) == (pts[win[w]][2] if win[w] >= 0 else b""), (it, w)
            else:
                assert win[w] == -1


def test_every_flushed_datapoint_carries_its_window_annotation():
    """the Reset datapoint included; no annotation crosses windows"""
    res = 10 * SEC
    m = AnnotatedElementModel(A.METRIC_COUNTER, [A.AGG_SUM], res, ops=[5], open_windows=4)
    assert m.add([(211 * SEC, _bits(5.0), b"a"), (215 * SEC, _bits(1.0), b""), (221 * SEC, _bits(7.0), b"")]) == \
        ([OK] * 3, OK)
    ts, _, anns = m.consume(240 * SEC)[0]
    assert ts.tolist() == [220 * SEC, 225 * SEC, 230 * SEC, 235 * SEC] and anns == [b"a", b"a", b"", b""]


def test_late_refused_and_nan_datapoints():
    res = 10 * SEC
    m = AnnotatedElementModel(A.METRIC_GAUGE, [A.AGG_LAST], res, open_windows=4)
    assert m.add([(211 * SEC, _bits(1.0), b"old"), (221 * SEC, _bits(2.0), b"new"),
                  (212 * SEC, _bits(float("nan")), b"late")]) == ([OK] * 3, OK)
    assert m.window_annotation(210 * SEC) == b"late" and m.window_annotation(220 * SEC) == b"new"
    m.consume(220 * SEC)
    assert m.add([(213 * SEC, _bits(3.0), b"closed")]) == ([ERR_CLOSED], OK)
    assert m.window_annotation(220 * SEC) == b"new" and 210 * SEC not in m.ann


def test_capacity_stops_the_element():
    res = 10 * SEC
    m = AnnotatedElementModel(A.METRIC_GAUGE, [A.AGG_LAST], res, open_windows=4, capacity=8)
    got = m.add([(211 * SEC, _bits(1.0), b"12345678"), (212 * SEC, _bits(1.0), b"123456789"),
                 (213 * SEC, _bits(1.0), b"")])
    assert got == ([OK, ERR_CAPACITY, ERR_CAPACITY], ERR_CAPACITY)
    assert m.window_annotation(210 * SEC) == b"12345678"
    # a closed window is refused before its annotation is looked at
    m.consume(220 * SEC)
    assert m.add([(215 * SEC, _bits(1.0), b"far too long")]) == ([ERR_CLOSED], OK)
