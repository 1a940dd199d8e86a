"""A second statement of the aggregator's transformations of a flushed window, in pure Python, written from the Go
source (src/metrics/transformation/{unary,binary,unary_multi}.go and GenericElem.processValue,
src/aggregator/aggregator/generic_elem.go:804-950), not from the C oracle.  NaN rules are spelled out on bit patterns
rather than left to the host's arithmetic: math.NaN() is 0x7FF8000000000001, an invalid operation on amd64 (Inf -
Inf) makes 0xFFF8000000000000, and an operation with one NaN operand returns that operand's NaN, quieted.

It must reproduce the reference's own test tables (tests/golden/m3tsz_transform_goldens.json) and agree with the
oracle (tests/xf_oracle.c) bit for bit, final state included, on random op lists over NaN payloads, +-Inf, +-0,
decreasing values, gaps between windows and call splits."""
import json
import math
import os
import struct

import numpy as np
import pytest

import agg_oracle_lib as A
import xf_oracle_lib as X

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "m3tsz_transform_goldens.json")

ABSOLUTE, PERSECOND, INCREASE, ADD, RESET = 1, 2, 3, 4, 5
GO_NAN = 0x7FF8000000000001   # math.NaN(), emptyDatapoint's value
AMD64_NAN = 0xFFF8000000000000  # the default NaN of an invalid operation
QUIET = 0x0008000000000000
MASK = (1 << 64) - 1


def f2b(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def b2f(b):
    return struct.unpack("<d", struct.pack("<Q", b & MASK))[0]


def is_nan(b):
    return (b & 0x7FF0000000000000) == 0x7FF0000000000000 and (b & 0x000FFFFFFFFFFFFF) != 0


def i64(x):
    x &= MASK
    return x - (1 << 64) if x >> 63 else x


def sse(op, a, b):
    """a op b on bit patterns the way an amd64 SSE instruction (dest a, source b) returns NaNs"""
    if is_nan(a):
        return a | QUIET
    if is_nan(b):
        return b | QUIET
    fa, fb = b2f(a), b2f(b)
    if op == "+":
        r = fa + fb
    elif op == "-":
        r = fa - fb
    elif op == "*":
        r = fa * fb
    else:
        r = fa / fb  # (the divisor here is t - prev_t > 0)
    return AMD64_NAN if math.isnan(r) else f2b(r)


class Element:
    """the state of one element for one aggregation type: the binary op's previous window (consumedValues at
    prevStartTime) and the closure of every Add op (transformAdd's `curr`)"""

    def __init__(self, n_ops):
        self.prev = None  # (t, value bits)
        self.sums = [0] * n_ops  # bits of +0

    def flush(self, ops, step, discard_nan, t, v):
        """processValue for one non-empty window ending at t with value bits v: the datapoints written"""
        extra = None
        for k, op in enumerate(ops):
            if op == ABSOLUTE:  # math.Abs: the sign bit
                v &= 0x7FFFFFFFFFFFFFFF
            elif op == ADD:  # if !math.IsNaN(dp.Value) { curr += dp.Value }; return curr
                if not is_nan(v):
                    self.sums[k] = sse("+", self.sums[k], v)
                v = self.sums[k]
            elif op in (PERSECOND, INCREASE):
                prev_t, prev_v = self.prev if self.prev is not None else (0, GO_NAN)
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
                        pv = f2b(0.0) if is_nan(prev_v) else prev_v
                        diff = sse("-", curr, pv)
                        v = GO_NAN if (not is_nan(diff) and b2f(diff) < 0) else diff
                self.prev = (t, curr)  # consumedValues keeps the op's input
            elif op == RESET:  # resetWindow := int64(math.Max(float64(resolution/2), 1))
                half = step // 2 if step >= 0 else -((-step) // 2)  # Go's / truncates toward zero
                rw = int(max(float(half), 1.0))
                extra = (i64(t + rw), 0)
            else:
                raise ValueError(op)
        if discard_nan and is_nan(v):
            return []
        out = [(t, v)]
        if extra is not None and extra[0] != 0:
            out.append(extra)
        return out

    def state_record(self):
        """the same state as a m3tsz_transform_state record"""
        st = X.new_transform_state()
        if self.prev is not None:
            st["has_prev"] = 1
            st["prev_t"] = self.prev[0]
            st["prev_v"] = b2f(self.prev[1])
        sums = np.zeros(8, dtype=np.uint64)
        sums[:len(self.sums)] = self.sums
        st["sum"][0] = sums.view(np.float64)
        return st


def _val(x):
    if isinstance(x, str):
        assert x.startswith("NaN:")
        return int(x[4:], 16)
    return f2b(float(x))


def _goldens():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


@pytest.mark.parametrize("case", _goldens(), ids=lambda c: c["name"])
def test_goldens_independent(case):
    e = Element(len(case["ops"]))
    if case["state"]:
        e.prev = (case["state"]["prev_t"], _val(case["state"]["prev_v"]))
    for call in case["calls"]:
        got = []
        for t, v in call["windows"]:
            got += e.flush(case["ops"], case["step_ns"], case["discard_nan"], t, _val(v))
        assert got == [(t, _val(v)) for t, v in call["want"]], case["name"]
    if "consumed" in case:
        assert e.prev[1] == f2b(case["consumed"][-1])


def _oracle_state(case):
    st = X.new_transform_state()
    if case["state"]:
        st["has_prev"] = case["state"]["has_prev"]
        st["prev_t"] = case["state"]["prev_t"]
        st["prev_v"] = b2f(_val(case["state"]["prev_v"]))
    return st


@pytest.mark.parametrize("case", _goldens(), ids=lambda c: c["name"])
def test_goldens_oracle(case):
    st = _oracle_state(case)
    for call in case["calls"]:
        t = np.array([w[0] for w in call["windows"]], dtype=np.int64)
        v = np.array([_val(w[1]) for w in call["windows"]], dtype=np.uint64).view(np.float64)
        to, vo = X.transform_series(case["ops"], case["discard_nan"], case["step_ns"], st, t, v)
        assert list(zip(to.tolist(), vo.view(np.uint64).tolist())) == [(t, _val(v)) for t, v in call["want"]]
    if "consumed" in case:
        assert float(st["prev_v"][0]) == case["consumed"][-1]


SPECIAL_BITS = [0x7FF8000000000001, 0xFFF8000000000000, 0x7FF8000000000000, 0x7FF8DEADBEEF0000, 0xFFF800000000ABCD,
                f2b(math.inf), f2b(-math.inf), f2b(0.0), f2b(-0.0), f2b(1e308), f2b(-1e308), f2b(5e-324)]


def random_pipeline(rng):
    """a valid op list: 1..8 ops, at most one PerSecond / Increase"""
    n = int(rng.integers(1, 9))
    ops, binary = [], False
    for _ in range(n):
        op = int(rng.integers(1, 6))
        if op in (PERSECOND, INCREASE):
            if binary:
                op = ADD
            binary = True
        ops.append(op)
    return ops


def random_windows(rng, n, t0=None):
    """n non-empty windows: increasing ends with gaps, values from specials, decreasing runs and ordinary ones"""
    step = int(rng.choice([1, 2, 3, 10 ** 9, 10 * 10 ** 9 + 1, 60 * 10 ** 9]))
    t = int(rng.integers(-5, 5)) * step if t0 is None else t0
    ts, vs = [], []
    x = float(rng.normal(0, 100))
    for _ in range(n):
        t += step * (1 if rng.random() < 0.7 else int(rng.integers(2, 6)))
        r = rng.random()
        if r < 0.25:
            b = SPECIAL_BITS[int(rng.integers(0, len(SPECIAL_BITS)))]
        else:
            x += float(rng.normal(5, 20)) if r < 0.8 else -float(rng.integers(0, 50))
            b = f2b(x)
        ts.append(t)
        vs.append(b)
    return step, ts, vs


def _splits(rng, n):
    cuts = sorted(set(int(c) for c in rng.integers(0, n + 1, size=int(rng.integers(0, 4)))))
    bounds = [0] + cuts + [n]
    return [(bounds[i], bounds[i + 1]) for i in range(len(bounds) - 1)]


def test_random_chains_match_oracle():
    rng = np.random.default_rng(20261016)
    for it in range(1500):
        ops = random_pipeline(rng)
        discard = bool(rng.random() < 0.5)
        step, ts, vs = random_windows(rng, int(rng.integers(0, 25)))
        e = Element(len(ops))
        st = X.new_transform_state()
        for a, b in _splits(rng, len(ts)):
            exp = []
            for t, v in zip(ts[a:b], vs[a:b]):
                exp += e.flush(ops, step, discard, t, v)
            to, vo = X.transform_series(ops, discard, step, st, np.array(ts[a:b], dtype=np.int64),
                                        np.array(vs[a:b], dtype=np.uint64).view(np.float64))
            got = list(zip(to.tolist(), vo.view(np.uint64).tolist()))
            assert got == exp, (it, ops, discard, step)
        assert e.state_record().tobytes() == st.tobytes(), (it, ops)


def test_random_tiles_match_oracle():
    """decode -> downsample -> ValueOf -> transformations: the oracle's tile path equals the independent chain over
    the oracle's own non-transformed tiles"""
    rng = np.random.default_rng(7)
    for it in range(200):
        n = int(rng.integers(0, 120))
        step = 60 * 10 ** 9
        ts = np.sort(rng.integers(0, 20 * step, size=n)).astype(np.int64)
        vals = np.array([b2f(SPECIAL_BITS[int(rng.integers(0, 8))]) if rng.random() < 0.2 else
                         float(rng.integers(-50, 500)) for _ in range(n)], dtype=np.float64)
        metric, agg = ((A.METRIC_GAUGE, int(rng.choice([1, 2, 3, 7]))) if rng.random() < 0.5 else
                       (A.METRIC_COUNTER, int(rng.choice([2, 3, 4, 6, 7]))))
        ops = random_pipeline(rng)
        discard = bool(rng.random() < 0.5)
        wt, wv = A.aggregate_tiles_series_ex(ts, vals, 0, step, 20, metric, agg)
        e = Element(len(ops))
        exp = []
        for t, v in zip(wt.tolist(), wv.view(np.uint64).tolist()):
            exp += e.flush(ops, step, discard, t, v)
        st = X.new_transform_state()
        to, vo = X.aggregate_tiles_transform_series(ts, vals, 0, step, 20, metric, agg, ops, discard, st)
        assert list(zip(to.tolist(), vo.view(np.uint64).tolist())) == exp, it
        assert e.state_record().tobytes() == st.tobytes(), it


def test_reset_datapoint_at_zero_is_not_written():
    e = Element(1)
    assert e.flush([RESET], 2, False, -1, f2b(3.0)) == [(-1, f2b(3.0))]
    st = X.new_transform_state()
    to, vo = X.transform_series([RESET], False, 2, st, np.array([-1, 1], dtype=np.int64), np.array([3.0, 4.0]))
    assert to.tolist() == [-1, 1, 2] and vo.tolist() == [3.0, 4.0, 0.0]
