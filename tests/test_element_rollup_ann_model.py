"""The annotated element-rollup model (tests/element_rollup_ann_model.py) against the reference's AddUnique tests of a
rollup element's annotation (tests/golden/m3tsz_rollup_annotation_goldens.json) fed as adds and forwards, against
the element-rollup model without annotations, and against the annotated element-set model for one-member groups."""
import json
import os

import numpy as np
import pytest

import agg_oracle_lib as A
from element_rollup_ann_model import (ERR_CAPACITY, ERR_CLOSED, OK, AnnotatedGroup, AnnotatedSource, forward)
from element_rollup_model import GroupModel, SourceModel
from element_rollup_model import forward as plain_forward
from element_set_ann_model import AnnotatedElementModel

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "m3tsz_rollup_annotation_goldens.json")
SEC = 1_000_000_000
GAUGE, COUNTER = A.METRIC_GAUGE, A.METRIC_COUNTER
LAST, MIN, MAX, COUNT, SUM = 1, 2, 3, 6, 7


def _bits(v):
    return int(np.array([v], dtype=np.float64).view(np.uint64)[0])


def _cases():
    return json.load(open(GOLDEN))["cases"]


def _ann(h):
    return b"" if h is None else bytes.fromhex(h)


@pytest.mark.parametrize("case", _cases(), ids=lambda c: c["name"])
def test_goldens_as_forwards(case):
    """each step's values are that many new sources, each with one datapoint at the step's time carrying the step's
    annotation; the step is one forward listing them in order into the one group, whose windows stay open across the
    steps.  What the reference asserts after each step must hold for the group's window."""
    step, starts = case["resolution_ns"], case["window_starts_ns"]
    metric = case["metric_type"]
    src_type = SUM if metric == COUNTER else LAST
    n = sum(len(st["values"]) for st in case["steps"])
    srcs = [AnnotatedSource(metric, src_type, step, capacity=64) for _ in range(n)]
    grp = AnnotatedGroup(metric, [COUNT, SUM], step, capacity=64)
    k = 0
    for st in case["steps"]:
        mem = list(range(k, k + len(st["values"])))
        for s, v in zip(mem, st["values"]):
            assert srcs[s].add([(st["at_ns"], _bits(v), _ann(st["annotation"]))]) == ([OK], OK)
        k += len(mem)
        target = starts[-1] + step
        sst, gst = forward(srcs, [grp], target, [0, len(mem)], mem)
        assert gst == [OK] and sst == [OK] * n
        for want in st["want"]:
            ws = starts[want["window"]]
            a = grp.m.aggregates(ws)
            for name in ("count", "sum"):
                if name in want:
                    assert a[name] == want[name], (case["name"], want, name)
            if "annotation" in want:
                assert grp.window_annotation(ws) == _ann(want["annotation"]), (case["name"], want)


PIPES = [  # (metric, src type, pre-ops, rollup types, post-ops)
    (COUNTER, SUM, [3], [SUM], [4]),
    (GAUGE, LAST, [], [MIN, MAX, SUM], []),
    (GAUGE, LAST, [1, 2], [LAST, SUM], [5]),
]


def _memberships(rng, S, G):
    lens = rng.integers(0, 5, G)
    mem = rng.integers(0, S + (1 if rng.random() < 0.2 else 0), int(lens.sum()))
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int64), mem.astype(np.int64)


@pytest.mark.parametrize("pipe", range(len(PIPES)))
def test_without_annotations_equals_the_element_rollup_model(pipe):
    metric, src_type, pre, types, post = PIPES[pipe]
    rng = np.random.default_rng(11 + pipe)
    res = 10 * SEC
    for it in range(6):
        S, G, R, RG = 10, 4, 3, int(rng.integers(1, 4))
        discard = bool(it % 2)
        a_src = [AnnotatedSource(metric, src_type, res, pre, discard, R, capacity=16) for _ in range(S)]
        a_grp = [AnnotatedGroup(metric, types, res, post, discard, RG, capacity=16) for _ in range(G)]
        p_src = [SourceModel(metric, src_type, res, pre, discard, R) for _ in range(S)]
        p_grp = [GroupModel(metric, types, res, post, discard, RG) for _ in range(G)]
        off, mem = _memberships(rng, S, G)
        clock = 0
        for step in range(8):
            for s in range(S):
                pts = [(clock + int(rng.integers(-2 * res, res)), _bits(float(rng.choice([1.0, 2.5, np.nan]))))
                       for _ in range(int(rng.integers(0, 3)))]
                assert a_src[s].add([(t, v, b"") for t, v in pts]) == p_src[s].add(pts)
            clock += res
            target = clock - int(rng.integers(0, 2)) * res
            assert forward(a_src, a_grp, target, off, mem) == plain_forward(p_src, p_grp, target, off, mem)
            for a, p in zip(a_src + a_grp, p_src + p_grp):
                assert repr(a.m.windows) == repr(p.windows) and a.state.tobytes() == p.state.tobytes()
                assert a.watermark == p.watermark
            if rng.random() < 0.5:
                for a, p in zip(a_grp, p_grp):
                    got, want = a.consume(target), p.consume(target)
                    for (ta, va, aa), (tp, vp) in zip(got, want):
                        assert np.array_equal(ta, tp) and np.array_equal(va.view(np.uint64), vp.view(np.uint64))
                        assert all(x == b"" for x in aa)


@pytest.mark.parametrize("metric", [GAUGE, COUNTER])
def test_one_member_groups_equal_the_annotated_element_set_model(metric):
    """a group of one source with the source's type (Gauge Last, Counter Sum) and no ops writes what an annotated
    element of that type fed the source's datapoints writes: the same values, each with its window's annotation"""
    rng = np.random.default_rng(3 + metric)
    res = 10 * SEC
    src_type = SUM if metric == COUNTER else LAST
    payloads = [b"", b"", b"a", b"prom", b"0123456789abcdef"]
    S = 6
    srcs = [AnnotatedSource(metric, src_type, res, open_windows=4, capacity=16) for _ in range(S)]
    grps = [AnnotatedGroup(metric, [src_type], res, open_windows=8, capacity=16) for _ in range(S)]
    elems = [AnnotatedElementModel(metric, [src_type], res, open_windows=4, capacity=16) for _ in range(S)]
    off, mem = np.arange(S + 1), np.arange(S)
    clock = 0
    for step in range(12):
        for s in range(S):
            pts = [(clock + int(rng.integers(-2 * res, res)), _bits(float(rng.integers(-50, 50))),
                    payloads[int(rng.integers(0, len(payloads)))]) for _ in range(int(rng.integers(0, 4)))]
            assert srcs[s].add(pts) == elems[s].add(pts)
        clock += res
        target = clock - int(rng.integers(0, 2)) * res
        sst, gst = forward(srcs, grps, target, off, mem)
        assert sst == [OK] * S and set(gst) <= {OK, ERR_CLOSED}
        for g, e in zip(grps, elems):
            got, want = g.consume(target), e.consume(target)
            for (tg, vg, ag), (te, ve, ae) in zip(got, want):
                assert np.array_equal(tg, te) and np.array_equal(vg, ve) and ag == ae


def test_rule_details():
    """listed order with a member listed twice, a NaN dropped by discard_nan, a NaN carried without it, a closed group
    window, an open group window keeping its annotation, and the annotation capacity stop with its retry"""
    res = 10 * SEC
    mk = lambda discard=False: AnnotatedSource(GAUGE, LAST, res, discard_nan=discard, capacity=32)
    a, b = mk(), mk()
    grp = AnnotatedGroup(GAUGE, [SUM], res, capacity=32)
    a.add([(0, _bits(1.0), b"a")])
    b.add([(0, _bits(2.0), b"b")])
    forward([a, b], [grp], res, [0, 3], [0, 1, 0])
    assert grp.window_annotation(0) == b"a" and grp.m.windows[0] == [1.0, 2.0, 1.0]
    # the group window stays open: a forward that brings no annotation keeps it, one that brings one replaces it
    for ann, want in ((b"", b"a"), (b"bb", b"bb")):
        c = mk()
        assert c.add([(1, _bits(3.0), ann)]) == ([OK], OK)
        assert forward([c], [grp], res, [0, 1], [0]) == ([OK], [OK])
        assert grp.window_annotation(0) == want
    # discard_nan drops a NaN and its annotation; without it the NaN carries its annotation
    for discard, want in ((True, b"bb"), (False, b"nan")):
        c = mk(discard)
        c.add([(3, _bits(float("nan")), b"nan")])
        forward([c], [grp], res, [0, 1], [0])
        assert grp.window_annotation(0) == want
    grp.consume(res)
    # a closed group window: the value and its annotation are dropped
    c = mk()
    c.add([(4, _bits(1.0), b"late")])
    sst, gst = forward([c], [grp], res, [0, 1], [0])
    assert gst == [ERR_CLOSED] and 0 not in grp.ann
    # an annotation longer than the group's capacity: CAPACITY, the member held back, then a retry after growing
    small = AnnotatedGroup(GAUGE, [SUM], res, capacity=8)
    d = mk()
    d.add([(res, _bits(1.0), b"x" * 20)])
    sst, gst = forward([d], [small], 2 * res, [0, 1], [0])
    assert gst == [ERR_CAPACITY] and sst == [ERR_CAPACITY] and small.m.windows == {} and d.m.windows
    small.capacity = 32
    sst, gst = forward([d], [small], 2 * res, [0, 1], [0])
    assert gst == [OK] and sst == [OK] and small.window_annotation(res) == b"x" * 20
