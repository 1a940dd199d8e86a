"""The rollup fold's device code, compiled for the host from the .cu source text: `rollup_gauge_init`,
`rollup_gauge_add`, `rollup_counter_init`, `rollup_counter_add` and `rollup_add` with their accumulators
(m3tsz_encode.cu) and `go_f64_to_i64` (m3tsz_common.cuh).  A driver folds a window's values in listed order the way
the fold kernel's lane does, and must equal the oracle (tests/rollup_oracle.c) bit for bit on NaN payloads, +-Inf,
+-0 in both orders, values >= 2^63 or NaN through int64(), wrapping sums and the equal-timestamp Last.  A CPU
regression harness for the device source; nothing of it ships."""
import ctypes as C
import math
import struct

import numpy as np
import pytest

import rollup_oracle_lib as R
from host_build import compile, constants, cut, fn, source_text

DRIVER = r"""
extern "C" void dev_fold_gauge(const double *v, size_t n, double *out5, int64_t *count) {
  RollupGaugeAcc a;
  rollup_gauge_init(a);
  for (size_t i = 0; i < n; i++) rollup_gauge_add(a, v[i]);
  out5[0] = a.sum;
  out5[1] = a.mn;
  out5[2] = a.mx;
  out5[3] = a.last;
  out5[4] = a.sq;
  *count = a.cnt;
}
extern "C" void dev_fold_counter(const double *v, size_t n, int64_t *out5) {
  RollupCounterAcc a;
  rollup_counter_init(a);
  for (size_t i = 0; i < n; i++) rollup_counter_add(a, v[i]);
  out5[0] = a.sum;
  out5[1] = a.cnt;
  out5[2] = a.mn;
  out5[3] = a.mx;
  out5[4] = a.sq;
}
"""


@pytest.fixture(scope="module")
def dev():
    enc, com = source_text("m3tsz_encode.cu"), source_text("m3tsz_common.cuh")
    parts = [constants(enc, r"kXf\w*"), cut(com, fn("go_f64_to_i64"))]
    for name in ("xf_isnan", "xf_bits"):
        parts.append(cut(enc, fn(name)))
    parts += [cut(enc, r"struct RollupGaugeAcc\b"), cut(enc, r"struct RollupCounterAcc\b")]
    for name in ("rollup_gauge_init", "rollup_counter_init", "rollup_add", "rollup_gauge_add", "rollup_counter_add"):
        parts.append(cut(enc, fn(name)))
    lib = compile("dev_rollup_host", "\n".join(parts), DRIVER)
    vp = C.c_void_p
    lib.dev_fold_gauge.restype = None
    lib.dev_fold_gauge.argtypes = [vp, C.c_size_t, vp, vp]
    lib.dev_fold_counter.restype = None
    lib.dev_fold_counter.argtypes = [vp, C.c_size_t, vp]
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _f(b):
    return struct.unpack("<d", struct.pack("<Q", b))[0]


def _bits(x):
    return struct.unpack("<Q", struct.pack("<d", float(x)))[0]


def _gauge(lib, vs):
    v = np.ascontiguousarray(vs, dtype=np.float64)
    o = np.zeros(5, dtype=np.float64)
    c = np.zeros(1, dtype=np.int64)
    lib.dev_fold_gauge(_p(v), len(v), _p(o), _p(c))
    return [_bits(x) for x in o], int(c[0])


def _counter(lib, vs):
    v = np.ascontiguousarray(vs, dtype=np.float64)
    o = np.zeros(5, dtype=np.int64)
    lib.dev_fold_counter(_p(v), len(v), _p(o))
    return [int(x) for x in o]


SPECIALS = [_f(0x7FF8000000000001), _f(0x7FF8000000000abc), _f(0xFFF8000000000000), math.inf, -math.inf, 0.0, -0.0,
            2.0 ** 63, -(2.0 ** 63), 2.0 ** 64, 9.3e18, 4.0e9, 3.0e18, -1.5, 1e16, 1.0, 5e-324]


def _oracle_gauge(vs):
    s, c, mn, mx, last, sq = R.fold_gauge(vs)
    return [_bits(x) for x in (s, mn, mx, last, sq)], c


def test_fold_edges(dev):
    cases = [[], [_f(0x7FF8000000000abc), 1.0, 2.0], [-0.0, 0.0], [0.0, -0.0], [math.inf, -math.inf, 1.0],
             [math.nan, 2.0 ** 63, -(2.0 ** 63)], [3.0e18] * 5, [4.0e9] * 3, [1e16, 1.0, 1.0], [1.0, 1.0, 1e16],
             [-math.inf], [math.inf, math.inf], [math.nan] * 3]
    for vs in cases:
        assert _gauge(dev, vs) == _oracle_gauge(vs), vs
        assert _counter(dev, vs) == list(R.fold_counter(vs)), vs


def test_fold_random(dev):
    rng = np.random.default_rng(17)
    for _ in range(4000):
        n = int(rng.integers(0, 10))
        vs = [SPECIALS[int(rng.integers(0, len(SPECIALS)))] if rng.random() < 0.5 else float(rng.normal(0, 1e6))
              for _ in range(n)]
        assert _gauge(dev, vs) == _oracle_gauge(vs), vs
        assert _counter(dev, vs) == list(R.fold_counter(vs)), vs
