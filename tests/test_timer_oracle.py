"""The Timer oracles (tests/timer_oracle.c and the independent pure-Python restatement tests/indep_timer.py) reproduce
the reference's Timer and CM stream expectations (tests/golden/m3tsz_timer_goldens.json) and agree with each other bit
for bit on random sequences: +-0 and NaN samples, duplicates, batches of 1 to 3000 values, several insert/compress
periods and eps values, unsorted quantile lists and elements without quantile types.  The element model
(tests/element_timer_model.py) states the batch and capacity rules."""
import json
import os

import numpy as np
import pytest

import timer_oracle_lib as T
from element_timer_model import TimerElementModel
from indep_timer import Timer, pooled_quantiles

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "m3tsz_timer_goldens.json")


def _load():
    with open(GOLDEN) as f:
        return json.load(f)


def _batches(case):
    return [list(b) for b, times in case["batches"] for _ in range(times)]


def _bits(a):
    return np.asarray(a, dtype=np.float64).view(np.uint64).tolist()


@pytest.mark.parametrize("case", _load()["cases"], ids=lambda c: c["name"])
def test_goldens(case):
    batches = _batches(case)
    got_c, _ = T.timer_window(batches, case["types"], case["eps"], case["every"])
    t = Timer(case["types"], case["eps"], case["every"])
    for b in batches:
        t.add_batch(b)
    got_py = t.values()
    assert _bits(got_c) == _bits(got_py)
    for j, ty in enumerate(case["types"]):
        if str(ty) in case["want"]:
            assert got_c[j] == case["want"][str(ty)], (ty, got_c[j])


@pytest.mark.parametrize("case", _load()["tolerance"], ids=lambda c: c["name"])
def test_tolerance_properties(case):
    n = case["n"]
    vals = np.arange(n, dtype=np.float64)
    if case["order"] == "decreasing":
        vals = vals[::-1]
    got, _ = T.timer_window([[float(v)] for v in vals], case["types"], case["eps"], case["every"])
    assert got[0] == 0.0 and got[1] == n - 1
    margin = n * case["eps"]
    for j, ty in enumerate(case["types"]):
        q = case["quantiles"].get(str(ty))
        if q is not None:
            assert n * q - margin <= got[j] <= n * q + margin, (ty, got[j])


def test_quantile_list_is_listed_order():
    assert pooled_quantiles([5, 10, 18]) == [0.5, 0.1, 0.9]
    assert pooled_quantiles([5, 14, 20, 23, 24]) == [0.5, 0.99, 0.25, 0.75]
    assert pooled_quantiles([2, 3, 4, 6, 7, 8, 9]) == []
    # Quantile(q) is the first listed quantile >= q: with [0.5, 0.1, 0.9], P10 reads the median's slot
    t = Timer([5, 10, 18])
    t.add_batch([float(i) for i in range(1, 201)])
    med, p10, p90 = t.values()
    assert p10 == med and p90 > med


TYPE_LISTS = [[2, 3, 4, 5, 6, 7, 8, 9, 14, 19, 20], [5, 10, 18], [14, 20, 23, 24], [2, 3, 6, 7], [20],
              [2, 3, 4, 5, 6, 7, 8, 9] + list(range(10, 25)), [3, 10, 11, 12, 13, 21, 22]]


def _random_value(rng, pool):
    r = rng.random()
    if r < 0.05:
        return float("nan")
    if r < 0.12:
        return 0.0
    if r < 0.19:
        return -0.0
    if r < 0.45 and pool:
        return pool[int(rng.integers(0, len(pool)))]  # a duplicate
    return float(np.round(rng.normal() * 100, int(rng.integers(0, 4))))


def random_batches(rng):
    batches, pool = [], []
    for _ in range(int(rng.integers(1, 7))):
        r = rng.random()
        n = int(rng.integers(1, 6)) if r < 0.7 else int(rng.integers(6, 60)) if r < 0.995 else \
            int(rng.integers(120, 3001))
        b = [_random_value(rng, pool) for _ in range(n)]
        pool += [v for v in b[:8] if v == v]
        batches.append(b)
    return batches


def test_oracles_agree_on_random_sequences():
    rng = np.random.default_rng(20261018)
    for it in range(10000):
        types = TYPE_LISTS[it % len(TYPE_LISTS)]
        every = [1, 2, 3, 7, 64, 1024][int(rng.integers(0, 6))]
        eps = [1e-3, 0.01, 0.05, 0.3][int(rng.integers(0, 4))]
        batches = random_batches(rng)
        got_c, peak = T.timer_window(batches, types, eps, every)
        t = Timer(types, eps, every)
        size = 0
        for b in batches:
            t.add_batch(b)
            size = max(size, t.stream.size())
        assert _bits(got_c) == _bits(t.values()), (it, types, every, eps)
        assert peak == size, it


def test_model_batch_and_capacity_rules():
    sec = 1_000_000_000
    m = TimerElementModel([2, 3, 20], 60 * sec, open_windows=2, sample_capacity=4)
    # a continuation in row 0, or with another timestamp, refuses the element
    assert m.add([(1 * sec, 1.0)], [1]) == ([101], 101)
    assert m.add([(1 * sec, 1.0), (2 * sec, 2.0)], [0, 1]) == ([101, 101], 101)
    assert m.windows == {}
    # a batch beyond the slot's capacity stops the element, later rows too
    res, st = m.add([(1 * sec, 1.0), (1 * sec, 2.0), (1 * sec, 3.0), (61 * sec, 4.0), (1 * sec, 5.0)], [0, 1, 1, 0, 0])
    assert (res, st) == ([0, 0, 0, 0, 0], 0)
    res, st = m.add([(2 * sec, 6.0), (2 * sec, 7.0), (62 * sec, 8.0)], [0, 1, 0])
    assert (res, st) == ([100, 100, 100], 100)
    # a third window with R = 2 open
    assert m.add([(125 * sec, 1.0)]) == ([100], 100)
    out = m.consume(120 * sec)
    assert [len(t) for t, _ in out] == [2, 2, 2]
    assert m.add([(1 * sec, 1.0)]) == ([17], 0)
