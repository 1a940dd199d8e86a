"""The annotated Timer element-set model (tests/element_timer_ann_model.py) against the reference's Timer annotation
golden, and against the models it composes: without annotations it is the Timer model, on single-row batches its
annotations are the annotated Gauge model's, and a one-member group through the annotated Timer rollup is the annotated
Timer model."""
import json
import os

import numpy as np

from element_set_ann_model import AnnotatedElementModel
from element_set_model import ERR_CAPACITY, ERR_INVALID_ARG, OK
from element_timer_ann_model import AnnotatedTimerGroup, AnnotatedTimerModel, AnnotatedTimerSource, forward
from element_timer_model import TimerElementModel

SEC = 1_000_000_000
RES = 10 * SEC
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "m3tsz_timer_annotation_goldens.json")
TYPES = [3, 14, 20]
PAYLOADS = [b"", b"", b"a", b"prom", b"0123456789abcdef"]


def _bits(v):
    return int(np.array([v], dtype=np.float64).view(np.uint64)[0])


def test_golden_last_non_empty_annotation():
    for case in json.load(open(GOLDEN))["cases"]:
        m = AnnotatedTimerModel(TYPES, RES, capacity=64)
        rows = [(RES + SEC, v) for v, _ in case["adds"]]
        anns = [(a or "").encode() for _, a in case["adds"]]
        assert m.add(rows, None, anns) == ([OK] * len(rows), OK)
        assert m.window_annotation(RES) == case["want"].encode()
        assert all(per == [case["want"].encode()] for _, _, per in m.consume(2 * RES))


def _random_rows(rng, clock):
    rows, marks, anns = [], [], []
    for _ in range(int(rng.integers(0, 4))):
        t = clock + int(rng.integers(-2 * RES, RES)) // SEC * SEC
        for i in range(int(rng.integers(1, 4))):
            rows.append((t, float(rng.choice([rng.normal(), np.nan, 1.0]))))
            marks.append(1 if i else 0)
            anns.append(b"" if i else PAYLOADS[int(rng.integers(0, len(PAYLOADS)))])
    return rows, marks, anns


def test_without_annotations_equals_the_timer_model():
    rng = np.random.default_rng(3)
    a, p = AnnotatedTimerModel(TYPES, RES, open_windows=2, sample_capacity=8), TimerElementModel(TYPES, RES, (), False,
                                                                                                 2, 8)
    clock = 10 * RES
    for _ in range(60):
        rows, marks, _ = _random_rows(rng, clock)
        assert a.add(rows, marks) == p.add(rows, marks)
        clock += int(rng.integers(0, 2)) * RES
        got, want = a.consume(clock), p.consume(clock)
        for (gt, gv, ga), (wt, wv) in zip(got, want):
            assert np.array_equal(gt, wt) and np.array_equal(gv.view(np.uint64), wv.view(np.uint64))
            assert all(x == b"" for x in ga)


def test_single_row_batches_take_the_gauge_rule():
    rng = np.random.default_rng(4)
    for _ in range(20):
        t_m = AnnotatedTimerModel(TYPES, RES, open_windows=3, capacity=8)
        g_m = AnnotatedElementModel(1, [1], RES, open_windows=3, capacity=8)
        clock = 10 * RES
        for _ in range(20):
            pts = [(clock + int(rng.integers(-2 * RES, RES)) // SEC * SEC, float(rng.normal()),
                    PAYLOADS[int(rng.integers(0, len(PAYLOADS)))]) for _ in range(int(rng.integers(0, 5)))]
            got = t_m.add([(t, v) for t, v, _ in pts], None, [a for _, _, a in pts])
            assert got == g_m.add([(t, _bits(v), a) for t, v, a in pts])
            assert t_m.ann == g_m.ann
            clock += int(rng.integers(0, 2)) * RES
            t_m.consume(clock)
            g_m.consume(clock)


def test_annotation_on_a_continuation_row_is_refused():
    m = AnnotatedTimerModel(TYPES, RES, capacity=8)
    rows = [(RES, 1.0), (RES, 2.0)]
    assert m.add(rows, [0, 1], [b"", b"x"]) == ([ERR_INVALID_ARG] * 2, ERR_INVALID_ARG)
    assert m.m.windows == {} and m.ann == {}
    assert m.add(rows, [0, 1], [b"x", b""]) == ([OK] * 2, OK) and m.ann == {RES: b"x"}
    assert m.add([(RES, 3.0)], None, [b"y" * 9]) == ([ERR_CAPACITY], ERR_CAPACITY) and m.ann == {RES: b"x"}


def test_one_member_group_equals_the_annotated_timer_model():
    rng = np.random.default_rng(5)
    src = AnnotatedTimerSource(20, RES, capacity=16)
    grp = AnnotatedTimerGroup(TYPES, RES, capacity=16)
    ref = AnnotatedTimerModel(TYPES, RES, capacity=16)
    clock = 10 * RES
    for _ in range(40):
        pts = [(clock + int(rng.integers(-RES, RES)) // SEC * SEC, float(rng.normal()),
                PAYLOADS[int(rng.integers(0, len(PAYLOADS)))]) for _ in range(int(rng.integers(0, 3)))]
        src.add([(t, v) for t, v, _ in pts], None, [a for _, _, a in pts])
        clock += int(rng.integers(0, 2)) * RES
        fw = src.forwarded(clock)
        assert forward([src], [grp], clock, [0, 1], [0]) == ([OK], [OK])
        for ws, v, a in fw:  # each forwarded value is one Timer.Add at the window's start
            ref.add([(ws, v)], None, [a])
        got, want = grp.consume(clock), ref.consume(clock)
        for (gt, gv, ga), (wt, wv, wa) in zip(got, want):
            assert np.array_equal(gt, wt) and np.array_equal(gv.view(np.uint64), wv.view(np.uint64)) and ga == wa
