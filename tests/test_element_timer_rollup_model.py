"""The Timer element-rollup model (tests/element_timer_rollup_model.py) against the reference's Timer rollup goldens
(tests/golden/m3tsz_timer_rollup_goldens.json), against the Timer element-set model for one-member groups, and the
one-value-per-Timer.Add rule of its fold."""
import json
import math
import os

import numpy as np

from element_set_model import window_start
from element_timer_model import TimerElementModel
from element_timer_rollup_model import OK, TimerGroupModel, TimerSourceModel, forward
from indep_timer import Timer

SEC = 1_000_000_000
MAX = 3


def goldens():
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                           "m3tsz_timer_rollup_goldens.json")) as f:
        return json.load(f)


def check_add_unique_want(w, want):
    """a group window's Timer against a golden step's checks (sums InEpsilon 1e-10, the rest exact)"""
    if "count" in want:
        assert w.count == want["count"]
    if "sum" in want:
        assert math.isclose(w.sum, want["sum"], rel_tol=1e-10)
    if "sum_sq" in want:
        assert math.isclose(w.sum_sq, want["sum_sq"], rel_tol=1e-10)
    if "q0.5" in want:
        w.stream.flush()
        assert w.stream.quantile(0.5) == want["q0.5"]


def add_unique_as_forwards(case):
    """the golden's AddUnique steps as forwards: step i is source i (type Max, one sample: the value) forwarded alone
    into group 0 at a target after its window -> (sources, group, [(step, forward statuses)])"""
    res = case["resolution_s"] * SEC
    steps = case["steps"]
    srcs = [TimerSourceModel(MAX, res, eps=case["eps"], every=case["every"]) for _ in steps]
    grp = TimerGroupModel(case["types"], res, open_windows=4, eps=case["eps"], every=case["every"])
    out = []
    for i, st in enumerate(steps):
        at, v = st["add"]
        assert srcs[i].add([(at * SEC, v)]) == ([OK], OK)
        target = window_start(at * SEC, res) + res
        out.append((i, forward(srcs, [grp], target, [0, 1], [i])))
    return srcs, grp, out


def test_add_unique_goldens():
    for case in goldens()["add_unique"]:
        res = case["resolution_s"] * SEC
        direct = TimerGroupModel(case["types"], res, eps=case["eps"], every=case["every"])
        _, grp, out = add_unique_as_forwards(case)
        for (i, (sst, gst)), st in zip(out, case["steps"]):
            at, v = st["add"]
            assert direct.add_unique(window_start(at * SEC, res), v)
            assert (sst[i], gst) == (OK, [OK])
        for m in (direct, grp):  # (the checks at the end of each window's steps still hold: later steps go elsewhere)
            for st in case["steps"]:
                if "want" in st and st is [s for s in case["steps"] if s.get("window_s") == st["window_s"]][-1]:
                    check_add_unique_want(m.windows[st["window_s"] * SEC], st["want"])
        # and step by step on a fresh group
        g = TimerGroupModel(case["types"], res, eps=case["eps"], every=case["every"])
        for st in case["steps"]:
            at, v = st["add"]
            g.add_unique(window_start(at * SEC, res), v)
            if "want" in st:
                check_add_unique_want(g.windows[st["window_s"] * SEC], st["want"])


def test_pipeline_goldens():
    for case in goldens()["pipeline"]:
        res = case["resolution_s"] * SEC
        src = TimerSourceModel(case["src_type"], res, case["pre_ops"], case["discard_nan"])
        grp = TimerGroupModel(case["rollup_types"], res, open_windows=4)
        for ws, samples in case["windows"]:
            assert src.add([(ws * SEC, x) for x in samples])[1] == OK
        for c in case["consumes"]:
            fwd, _ = src.pending(c["target_s"] * SEC)
            got = [[(ws + res) // SEC, v] for ws, v, ok in fwd if ok]
            want = c["want"]
            assert len(got) == len(want)
            for (gt, gv), (wt, wv) in zip(got, want):
                assert gt == wt
                assert math.isnan(gv) if wv == "NaN" else gv == wv
            assert forward([src], [grp], c["target_s"] * SEC, [0, 1], [0]) == ([0], [OK])
            for (wt, wv) in want:  # a one-member group's Max is the forwarded value
                got_v = grp.windows[(wt * SEC) - res].values()[0]
                assert math.isnan(got_v) if wv == "NaN" else got_v == wv


def _random_source(rng, res, clock):
    return [(clock + int(rng.integers(-2 * res, res)) // SEC * SEC,
             float("nan") if rng.random() < 0.05 else float(np.round(rng.normal() * 50, 1)))
            for _ in range(int(rng.integers(0, 5)))]


def test_one_member_group_equals_the_timer_element_model():
    """a one-member group is a TimerElementModel fed the forwarded values as one-row batches"""
    rng = np.random.default_rng(3)
    res = 10 * SEC
    for it in range(40):
        types = [[2, 3, 14, 20], [4, 6, 7, 8, 9], [5, 10, 18, 23]][it % 3]
        ops, discard = [[], [1], [2]][it % 3], bool(it % 2)
        src = TimerSourceModel([20, 3, 4][it % 3], res, ops, discard, open_windows=3, sample_capacity=64)
        grp = TimerGroupModel(types, res, open_windows=4, sample_capacity=64, every=int(rng.choice([1, 2, 3, 1024])))
        twin = TimerElementModel(types, res, open_windows=4, sample_capacity=64, every=grp.every)
        clock = 10 * res
        for step in range(10):
            src.add(_random_source(rng, res, clock))
            clock += int(rng.integers(0, 2)) * res
            target = clock - int(rng.integers(0, 2)) * res
            fwd, _ = src.pending(target)
            sst, gst = forward([src], [grp], target, [0, 1], [0])
            if gst == [OK]:
                for ws, v, ok in fwd:
                    if ok:
                        assert twin.add([(ws, v)])[1] == OK
            if rng.random() < 0.5:
                a, b = grp.consume(target), twin.consume(target)
                for (ta, va), (tb, vb) in zip(a, b):
                    assert np.array_equal(ta, tb)
                    assert np.array_equal(np.asarray(va).view(np.uint64), np.asarray(vb).view(np.uint64))


def test_single_value_adds_differ_from_one_batch():
    """k values into one window are k one-value AddBatch calls, each reading the insertion point afresh; folding them
    as one batch of k gives other quantiles on some inputs"""
    rng = np.random.default_rng(11)
    types = [14, 18, 19, 20]
    differ = 0
    for _ in range(100):  # (a difference needs inserts inside the batch and compressions that merge samples)
        every, eps = int(rng.choice([1, 2, 3, 5, 16])), float(rng.choice([0.01, 0.05, 0.1]))
        vals = [float(x) for x in np.round(rng.normal(size=int(rng.integers(20, 300))) * 10, 1)]
        one, singles = Timer(types, eps, every), Timer(types, eps, every)
        one.add_batch(vals)
        for v in vals:
            singles.add_batch([v])
        a, b = one.values(), singles.values()
        assert one.count == singles.count and one.sum == singles.sum
        differ += a != b
    assert differ > 0
