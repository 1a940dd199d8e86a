"""A second statement of an element with several aggregation types, in pure Python, written from the Go source
(GenericElem.processValue's loop over e.aggTypes, src/aggregator/aggregator/generic_elem.go:830-889, and
src/metrics/transformation/{unary,binary,unary_multi}.go), not from the C oracle.  The bit-level NaN rules (amd64 SSE)
are those of test_independent_transforms.py.

Per window, for each type in order: the Add op at position i is one closure (one sum for every type); the binary op
reads (prevStartTime's timestamp, consumedValues[type]) and writes consumedValues[type]; discarding a NaN drops only
that type's datapoints.  It must reproduce tests/golden/m3tsz_element_types_goldens.json, agree with the oracle
(tests/elem_oracle.c) bit for bit, final state included, on random type sets, op lists and call splits, and give the
single-type oracle's results (tests/xf_oracle.c) for one type and, type by type, for any list without Add."""
import json
import os

import numpy as np
import pytest

import agg_oracle_lib as A
import elem_oracle_lib as E
import xf_oracle_lib as X
from test_independent_transforms import (ABSOLUTE, ADD, GO_NAN, INCREASE, PERSECOND, RESET, _splits, _val, b2f, f2b,
                                         i64, is_nan, random_pipeline, random_windows, sse)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "m3tsz_element_types_goldens.json")
GAUGE_TYPES = [1, 2, 3, 4, 6, 7, 8, 9]  # Last, Min, Max, Mean, Count, Sum, SumSq, Stdev
COUNTER_TYPES = [2, 3, 4, 6, 7, 8, 9]


class MultiElement:
    """one element: cState.prevStartTime (the previous flushed window, shared), fState.consumedValues (one per type)
    and the closure of every Add op (one per op, shared by the types)"""

    def __init__(self, n_ops, n_types):
        self.prev_t = None
        self.consumed = [GO_NAN] * n_types
        self.sums = [0] * n_ops  # bits of +0

    def flush(self, ops, step, discard_nan, t, values):
        """processValue for one non-empty window ending at t, values[j] the bits of type j's value: the datapoints
        each type writes"""
        out = []
        binary = False
        for j, v in enumerate(values):
            extra = None
            for k, op in enumerate(ops):
                if op == ABSOLUTE:
                    v &= 0x7FFFFFFFFFFFFFFF
                elif op == ADD:
                    if not is_nan(v):
                        self.sums[k] = sse("+", self.sums[k], v)
                    v = self.sums[k]
                elif op in (PERSECOND, INCREASE):
                    # prev := {Value: nan}; if cState.prevStartTime > 0 { prev = (prevTimestamp, consumedValues[j]) }
                    prev_t, prev_v = (self.prev_t, self.consumed[j]) if self.prev_t is not None else (0, GO_NAN)
                    curr = v
                    if op == PERSECOND:
                        if prev_t >= t or is_nan(prev_v) or is_nan(curr):
                            v = GO_NAN
                        else:
                            diff = sse("-", curr, prev_v)
                            if not is_nan(diff) and b2f(diff) < 0:
                                v = GO_NAN
                            else:
                                v = sse("/", sse("*", diff, f2b(1e9)), f2b(float(i64(t - prev_t))))
                    else:
                        if prev_t >= t or is_nan(curr):
                            v = GO_NAN
                        else:
                            diff = sse("-", curr, f2b(0.0) if is_nan(prev_v) else prev_v)
                            v = GO_NAN if (not is_nan(diff) and b2f(diff) < 0) else diff
                    self.consumed[j] = curr  # fState.consumedValues[aggTypeIdx] = curr.Value
                    binary = True
                elif op == RESET:
                    half = step // 2 if step >= 0 else -((-step) // 2)
                    extra = (i64(t + int(max(float(half), 1.0))), 0)
            if discard_nan and is_nan(v):
                out.append([])
                continue
            dps = [(t, v)]
            if extra is not None and extra[0] != 0:
                dps.append(extra)
            out.append(dps)
        if binary:
            self.prev_t = t
        return out

    def state_record(self):
        """the same state as an m3tsz_element_state record"""
        st = E.new_element_state()
        if self.prev_t is not None:
            st["has_prev"] = 1
            st["prev_t"] = self.prev_t
        cons = np.zeros(8, dtype=np.uint64)
        if self.prev_t is not None:
            cons[:len(self.consumed)] = self.consumed
        st["prev_v"] = cons[:1].view(np.float64)[0]
        st["prev_v_more"][0] = cons[1:].view(np.float64)
        sums = np.zeros(8, dtype=np.uint64)
        sums[:len(self.sums)] = self.sums
        st["sum"][0] = sums.view(np.float64)
        return st


def _goldens():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


@pytest.mark.parametrize("case", _goldens(), ids=lambda c: c["name"])
def test_goldens_independent(case):
    k = len(case["agg_types"])
    e = MultiElement(len(case["ops"]), k)
    for call in case["calls"]:
        got = [[] for _ in range(k)]
        for t, vs in call["windows"]:
            for j, dps in enumerate(e.flush(case["ops"], case["step_ns"], case["discard_nan"], t,
                                            [_val(v) for v in vs])):
                got[j] += dps
        assert got == [[(t, _val(v)) for t, v in w] for w in call["want"]], case["name"]


@pytest.mark.parametrize("case", _goldens(), ids=lambda c: c["name"])
def test_goldens_oracle(case):
    k = len(case["agg_types"])
    st = E.new_element_state()
    for call in case["calls"]:
        t = np.array([w[0] for w in call["windows"]], dtype=np.int64)
        v = np.array([[_val(x) for x in w[1]] for w in call["windows"]], dtype=np.uint64).reshape(len(t), k)
        res = E.element_series(case["ops"], case["discard_nan"], case["step_ns"], k, st, t, v.view(np.float64))
        for j in range(k):
            to, vo = res[j]
            assert list(zip(to.tolist(), vo.view(np.uint64).tolist())) == [(a, _val(b)) for a, b in call["want"][j]]


def random_types(rng, metric=None):
    pool = GAUGE_TYPES if (metric or A.METRIC_GAUGE) == A.METRIC_GAUGE else COUNTER_TYPES
    k = int(rng.integers(1, len(pool) + 1))
    return sorted(int(x) for x in rng.choice(pool, size=k, replace=False))


def random_element_pipeline(rng):
    """random_pipeline, with Add (at a random position) in most lists"""
    ops = random_pipeline(rng)
    if rng.random() < 0.6 and ADD not in ops:
        ops[int(rng.integers(0, len(ops)))] = ADD
    return ops


def _element_windows(rng, n, k):
    step, ts, v0 = random_windows(rng, n)
    cols = [v0] + [random_windows(rng, n)[2] for _ in range(k - 1)]
    return step, ts, [[cols[j][i] for j in range(k)] for i in range(n)]


def test_random_elements_match_oracle():
    rng = np.random.default_rng(20261017)
    for it in range(1500):
        k = int(rng.integers(1, 9))
        ops = random_element_pipeline(rng)
        discard = bool(rng.random() < 0.5)
        step, ts, vs = _element_windows(rng, int(rng.integers(0, 20)), k)
        e = MultiElement(len(ops), k)
        st = E.new_element_state()
        for a, b in _splits(rng, len(ts)):
            exp = [[] for _ in range(k)]
            for t, v in zip(ts[a:b], vs[a:b]):
                for j, dps in enumerate(e.flush(ops, step, discard, t, v)):
                    exp[j] += dps
            res = E.element_series(ops, discard, step, k, st, np.array(ts[a:b], dtype=np.int64),
                                   np.array(vs[a:b], dtype=np.uint64).reshape(b - a, k).view(np.float64))
            for j in range(k):
                got = list(zip(res[j][0].tolist(), res[j][1].view(np.uint64).tolist()))
                assert got == exp[j], (it, ops, discard, step, j)
        assert e.state_record().tobytes() == st.tobytes(), (it, ops, k)


def test_add_is_shared_across_types():
    """two types, [Add]: type 1's value adds onto type 0's in the same window (no sequence of single-type calls
    can write this)"""
    e = MultiElement(1, 2)
    out = e.flush([ADD], 10, True, 100, [f2b(1.0), f2b(10.0)])
    assert out == [[(100, f2b(1.0))], [(100, f2b(11.0))]]
    out = e.flush([ADD], 10, True, 110, [f2b(2.0), f2b(20.0)])
    assert out == [[(110, f2b(13.0))], [(110, f2b(33.0))]]
    st = E.new_element_state()
    res = E.element_series([ADD], True, 10, 2, st, np.array([100, 110], dtype=np.int64),
                           np.array([[1.0, 10.0], [2.0, 20.0]]))
    assert res[0][1].tolist() == [1.0, 13.0] and res[1][1].tolist() == [11.0, 33.0]


def _single_type_oracle(ops, discard, step, ts, col):
    st = X.new_transform_state()
    to, vo = X.transform_series(ops, discard, step, st, np.array(ts, dtype=np.int64),
                                np.array(col, dtype=np.uint64).view(np.float64))
    return list(zip(to.tolist(), vo.view(np.uint64).tolist())), st


def test_single_type_and_no_add_match_single_type_oracle():
    """k = 1: the transformation oracle's datapoints and state (the first 96 bytes); any k without Add: type by type"""
    rng = np.random.default_rng(99)
    for it in range(800):
        k = 1 if it % 2 == 0 else int(rng.integers(2, 9))
        ops = random_pipeline(rng)
        if k > 1:
            ops = [op if op != ADD else ABSOLUTE for op in ops]
        discard = bool(rng.random() < 0.5)
        step, ts, vs = _element_windows(rng, int(rng.integers(0, 20)), k)
        e = MultiElement(len(ops), k)
        got = [[] for _ in range(k)]
        for t, v in zip(ts, vs):
            for j, dps in enumerate(e.flush(ops, step, discard, t, v)):
                got[j] += dps
        for j in range(k):
            exp, st1 = _single_type_oracle(ops, discard, step, ts, [v[j] for v in vs])
            assert got[j] == exp, (it, ops, j)
            if k == 1:
                assert e.state_record().tobytes()[:96] == st1.tobytes(), (it, ops)
                assert e.state_record().tobytes()[96:] == bytes(64)


def test_random_tiles_match_oracle():
    """decode -> downsample -> ValueOf of every type -> the element: the oracle's tile path equals the independent
    element over the aggregation oracle's tiles"""
    rng = np.random.default_rng(11)
    for it in range(150):
        n = int(rng.integers(0, 120))
        step = 60 * 10 ** 9
        ts = np.sort(rng.integers(0, 20 * step, size=n)).astype(np.int64)
        vals = np.array([float(rng.integers(-50, 500)) for _ in range(n)], dtype=np.float64)
        metric = A.METRIC_GAUGE if rng.random() < 0.5 else A.METRIC_COUNTER
        types = random_types(rng, metric)
        ops = random_element_pipeline(rng)
        discard = bool(rng.random() < 0.5)
        wt, wv = E.element_windows(ts, vals, 0, step, 20, metric, types)
        e = MultiElement(len(ops), len(types))
        exp = [[] for _ in types]
        for i, t in enumerate(wt.tolist()):
            for j, dps in enumerate(e.flush(ops, step, discard, t, wv[i].view(np.uint64).tolist())):
                exp[j] += dps
        st = E.new_element_state()
        res = E.aggregate_tiles_types_series(ts, vals, 0, step, 20, metric, types, ops, discard, st)
        for j in range(len(types)):
            assert list(zip(res[j][0].tolist(), res[j][1].view(np.uint64).tolist())) == exp[j], (it, j)
        assert e.state_record().tobytes() == st.tobytes(), it
