"""The value classifier the encode kernel runs -- `maybe_int`, `go_f64_to_u64_via_i64`, `convert_to_int_float`
(m3_b200/csrc/m3tsz_encode.cu) and `mult_pow10` (m3tsz_common.cuh) -- compiled FOR THE HOST from the device source
text itself (the function bodies are cut out of the .cu files at test time; CUDA's round-to-nearest intrinsics are
mapped onto the IEEE operations they are, the build contracts no FMA, like the kernels' -fmad=false) and
compared with the oracle's convertToIntFloat: same (value bits, multiplier, isFloat) for every current multiplier
on the reference's families, ulp neighbourhoods of decimals, random bit patterns and the special values.  This is a
CPU check of the DEVICE code's arithmetic, not a CPU path of the product: the shared object it builds lives in a
temporary directory and only this test loads it."""
import ctypes as C
import random

import numpy as np
import pytest

import oracle_lib as O
from host_build import compile, constants, cut, fn, source_text

EXPORTS = r"""
extern "C" {
int dev_maybe_int(double v) { return maybe_int(v) ? 1 : 0; }
uint64_t dev_f64_to_u64(double v) { return go_f64_to_u64_via_i64(v); }
void dev_convert(double v, int cur, double *val, int *mult, int *is_float) {
  bool f = false;
  convert_to_int_float(v, cur, *val, *mult, f);
  *is_float = f ? 1 : 0;
}
}
"""


@pytest.fixture(scope="module")
def dev():
    enc, com = source_text("m3tsz_encode.cu"), source_text("m3tsz_common.cuh")
    body = "\n".join([constants(com, "kMaxMult"), cut(com, fn("mult_pow10")), cut(enc, fn("maybe_int")),
                      cut(enc, fn("go_f64_to_u64_via_i64")), cut(enc, fn("convert_to_int_float"))])
    assert "__dmul_rn" in body and "trunc(" in body  # still the separately rounded form
    lib = compile("dev_host", body, EXPORTS)
    lib.dev_maybe_int.restype, lib.dev_maybe_int.argtypes = C.c_int, [C.c_double]
    lib.dev_f64_to_u64.restype, lib.dev_f64_to_u64.argtypes = C.c_uint64, [C.c_double]
    lib.dev_convert.restype = None
    lib.dev_convert.argtypes = [C.c_double, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    return lib


def _values():
    r = random.Random(41)
    vals = []
    for num_dig, num_dec in [(0, 0), (2, 0), (10, 0), (13, 0), (18, 0), (0, 6), (3, 6), (7, 6), (0, 1), (1, 3), (5, 3),
                             (2, 16), (9, 2), (11, 3), (12, 1), (6, 5), (8, 4)]:
        for _ in range(250):
            dig = r.getrandbits(62) % 10 ** num_dig
            v = float(dig) if num_dec == 0 else float("%d.%d" % (dig, r.getrandbits(62) % 10 ** num_dec))
            vals += [v, -v]
    base = np.array([(r.getrandbits(r.randrange(1, 50)) + 1) / 10.0 ** r.randrange(0, 7) for _ in range(2500)])
    bits = base.view(np.int64)
    for j in (-12, -8, -3, -2, -1, 0, 1, 2, 3, 8, 12, 100):
        vals += (bits + j).view(np.float64).tolist()
    vals += (-base).tolist()
    rb = np.random.default_rng(43).integers(0, 2 ** 63, size=3000, dtype=np.int64).view(np.float64)
    vals += rb.tolist() + (-rb).tolist()
    vals += [0.0, -0.0, float("inf"), float("-inf"), float("nan"), 2.0 ** 63, -2.0 ** 63, 2.0 ** 63 - 1024, 1e13,
             1e13 - 0.5, 9999999999999.9, 1e300, -1e300, 5e-324, 1e-7, 0.1, 0.9, 0.95, 0.05]
    return vals


def test_device_convert_to_int_float_equals_oracle(dev):
    val, mult, isf = C.c_double(), C.c_int(), C.c_int()
    n = n_int = 0
    for v in _values():
        for cur in range(7):
            ov, om, of, err = O.convert_to_int_float(v, cur)
            assert err == 0
            dev.dev_convert(v, cur, C.byref(val), C.byref(mult), C.byref(isf))
            assert (mult.value, bool(isf.value)) == (om, of), (v, cur)
            a, b = np.float64(val.value).view(np.uint64), np.float64(ov).view(np.uint64)
            assert a == b or (val.value != val.value and ov != ov), (v, cur, val.value, ov)
            if not of:  # whatever the classifier calls an int, the cheap filter must have let through
                assert dev.dev_maybe_int(v) == 1, (v, cur)
                n_int += 1
            n += 1
    assert n > 300000 and n_int > 40000


def test_device_maybe_int_equals_its_numpy_restatement(dev):
    from test_int_filter_property import maybe_int
    vals = np.array(_values(), dtype=np.float64)
    got = np.array([dev.dev_maybe_int(float(v)) for v in vals], dtype=bool)
    assert (got == maybe_int(vals)).all()
    assert 0.2 < got.mean() < 0.9  # both verdicts occur


def test_device_float_to_int_conversion_follows_amd64(dev):
    """int64(float64) as the reference's host executes it (CVTTSD2SQ): out of range and NaN give 0x8000000000000000
    (SURVEY Appendix B #3; reachable through a first value <= -2^63)."""
    for v, exp in [(0.0, 0), (1.9, 1), (-1.9, (1 << 64) - 1), (2.0 ** 62, 1 << 62), (2.0 ** 63, 1 << 63),
                   (-2.0 ** 63, 1 << 63), (1e300, 1 << 63), (-1e300, 1 << 63), (float("nan"), 1 << 63),
                   (float("inf"), 1 << 63), (9.2e18, 9200000000000000000)]:
        assert dev.dev_f64_to_u64(v) == exp, v
