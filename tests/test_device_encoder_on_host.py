"""The ENCODER's device functions, compiled for the host from the .cu source text and driven one series at a time
the way a lane of the kernel drives them: `EncLane`, `put32` / `put64`, the value classifier, `track_new_sig`,
`sig_mult_hdr`, `xor_code`, `encode_value<INT_OPT>`, `encode_time`, `tier2_candidate<INT_OPT>` /
`tier2_commit<INT_OPT>` are cut out of m3_b200/csrc/m3tsz_encode.cu (and the constants / unit helpers out of
m3tsz_common.cuh) at test time.  Only what is PTX is replaced by a plain C++ statement of the same contract: the
predicated-store merge `emit_code_p` (here: put32 + put64 of the same bits), `lz_tz` / `shl64_clamp`, the CUDA
intrinsics.  Two drivers -- every datapoint through the general path, and the second tier wherever
`tier2_candidate` says so (the kernel picks per warp vote, so any mix has to give the same bytes) -- must both
reproduce the ORACLE's bytes on the reference's families, unit changes, jittered timestamps, special values and
Gaussian walks, in both modes.  A CPU regression harness for the device source; nothing of it ships."""
import ctypes as C
import os
import random
import re
import subprocess
import tempfile

import numpy as np
import pytest

import oracle_lib as O

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
CSRC = os.path.join(ROOT, "m3_b200", "csrc")
SEC = 10 ** 9

SHIM = r"""
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
enum { M3TSZ_ERR_DOD_OVERFLOW = 4, M3TSZ_ERR_UNRECOGNIZED_UNIT = 6 };
static inline double __dmul_rn(double a, double b) { return a * b; }
static inline double __dsub_rn(double a, double b) { return a - b; }
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline long long __double2ll_rz(double a) { return (long long)a; }
static inline long long __double_as_longlong(double a) { long long r; memcpy(&r, &a, 8); return r; }
static inline double __longlong_as_double(long long a) { double r; memcpy(&r, &a, 8); return r; }
static inline int __clzll(long long v) { return v ? __builtin_clzll((unsigned long long)v) : 64; }
// funnel shift right, shift amount clamped to 32 (PTX shf.r.clamp)
static inline uint32_t __funnelshift_rc(uint32_t lo, uint32_t hi, uint32_t sh) {
  if (sh > 32) sh = 32;
  const uint64_t v = ((uint64_t)hi << 32) | lo;
  return (uint32_t)(v >> sh);
}
constexpr int ENC_STRIDE = 33;
// ---- PTX helpers of m3tsz_common.cuh restated (their contracts are in the comments there) ----
static inline uint64_t shl64(uint64_t x, int n) { return n >= 64 ? 0ull : x << n; }
static inline uint64_t shr64(uint64_t x, int n) { return n >= 64 ? 0ull : x >> n; }
static inline uint64_t shl64_clamp(uint64_t x, uint32_t n) { return n > 63 ? 0ull : x << n; }
static inline uint64_t shr64_clamp(uint64_t x, uint32_t n) { return n > 63 ? 0ull : x >> n; }
static inline void lz_tz(uint64_t v, int &lz, int &tz) {
  if (!v) { lz = 64; tz = 0; return; }
  lz = __builtin_clzll(v);
  tz = __builtin_ctzll(v);
}
"""

# emit_code_p: header (low hb bits of hdr) followed by the payload given LEFT-ALIGNED in P (top plen bits)
EMIT = r"""
inline void emit_code_p(EncLane &s, uint32_t *tile, int lane, uint32_t hdr, int hb, uint64_t P, int plen) {
  if (hb > 0) put32(s, tile, lane, hb >= 32 ? hdr : (hdr & ((1u << hb) - 1u)), hb);
  if (plen > 0) put64(s, tile, lane, P >> (64 - plen), plen);
}
"""

DRIVER = r"""
template <bool INT_OPT>
static long long drive(const int64_t *ts, const double *vals, const uint8_t *units, size_t n, int64_t start, int unit,
                       int default_unit, int use_tier2, uint8_t *out, size_t cap, int *n_tier2, uint8_t *tiers) {
  std::vector<uint32_t> tile((n * 6 + 64) * ENC_STRIDE, 0u);
  EncLane s;
  memset(&s, 0, sizeof(s));
  s.plz = 64;
  s.prev_time = start;
  s.unit = initial_time_unit(start, default_unit);
  if (n) put64(s, tile.data(), 0, (uint64_t)start, 64);
  bool steady = false;
  *n_tier2 = 0;
  for (size_t i = 0; i < n && s.err == 0; i++) {
    const int64_t t = ts[i];
    const double v = vals[i];
    const int u = units ? (int)units[i] : unit;
    uint64_t fb;
    memcpy(&fb, &v, 8);
    const int64_t delta = (int64_t)((uint64_t)t - (uint64_t)s.prev_time);
    Tier2 c2;
    if (use_tier2 && u == s.unit && tier2_candidate<INT_OPT>(s, steady, delta, fb, v, c2)) {
      s.prev_time = t;
      s.prev_delta = delta;
      tier2_commit<INT_OPT>(s, tile.data(), 0, fb, c2);
      s.n_enc++;
      (*n_tier2)++;
      if (tiers) tiers[i] = 2;
    } else {
      uint32_t hdr;
      int hb;
      encode_time(s, tile.data(), 0, t, u, hdr, hb);
      if (s.err == 0) {
        uint64_t payload;
        int plen;
        encode_value<INT_OPT>(s, v, hdr, hb, payload, plen);
        emit_code(s, tile.data(), 0, hdr, hb, payload, plen);
        s.n_enc++;
      }
      if (tiers) tiers[i] = 1;
    }
    steady = (u == s.unit) && (s.unit >= 1 && s.unit <= 4) && s.n_enc > 0;
  }
  if (s.err) return -(long long)s.err;
  if (s.n_enc == 0) return 0;
  put32(s, tile.data(), 0, (kMarkerOpcode << 2) | (uint32_t)kMarkerEOS, kMarkerBits);
  const uint64_t bits = (uint64_t)s.k * 32ull + s.sh;
  const size_t nbytes = (size_t)((bits + 7) / 8);
  if (nbytes > cap) return -1000;
  for (size_t b = 0; b < nbytes; b++) {
    const size_t w = b / 4;
    const uint32_t word = w < s.k ? tile[w * ENC_STRIDE] : s.carry;
    out[b] = (uint8_t)(word >> (24 - 8 * (b % 4)));
  }
  return (long long)nbytes;
}
extern "C" long long dev_encode_series(const int64_t *ts, const double *vals, const uint8_t *units, size_t n,
                                       int64_t start, int unit, int int_opt, int default_unit, int use_tier2,
                                       uint8_t *out, size_t cap, int *n_tier2, uint8_t *tiers) {
  return int_opt ? drive<true>(ts, vals, units, n, start, unit, default_unit, use_tier2, out, cap, n_tier2, tiers)
                 : drive<false>(ts, vals, units, n, start, unit, default_unit, use_tier2, out, cap, n_tier2, tiers);
}
"""


def _cut(src, pattern):
    """the definition that `pattern` starts (a function, struct or enum), braces matched; a preceding template<> line
    is kept"""
    m = re.search(pattern, src)
    assert m, pattern
    start = m.start()
    prev = src.rfind("\n", 0, start - 1)
    if src[prev + 1: start].strip().startswith("template"):
        start = prev + 1
    i = src.index("{", m.end())
    depth = 0
    for j in range(i, len(src)):
        if src[j] == "{":
            depth += 1
        elif src[j] == "}":
            depth -= 1
            if depth == 0:
                end = j + 1
                if src[end: end + 1] == ";":
                    end += 1
                return src[start:end]
    raise AssertionError(pattern)


def _fn(name):
    return r"__device__[^\n;{]*\b%s\s*\(" % re.escape(name)


def build_dev_encoder():
    """Compiles the encoder's general path and second tier for the host (g++ only) and returns the loaded library:
    `dev_encode_series(ts, vals, units, n, start, unit, int_opt, default_unit, use_tier2, out, cap, &n_tier2,
    tiers)` returns the stream's length, or minus the status; `tiers` (may be NULL) receives per datapoint 1 for
    the general path and 2 for the second tier."""
    enc = open(os.path.join(CSRC, "m3tsz_encode.cu")).read()
    com = open(os.path.join(CSRC, "m3tsz_common.cuh")).read()
    consts = "\n".join(re.findall(r"^constexpr [^\n]*\bk(?:Marker|MaxMult)[^\n]*$", com, flags=re.M))
    parts = [consts, _cut(com, r"enum SchemeKind"),
             _cut(com, r"__host__ __device__[^\n{;]*\bunit_is_valid\s*\("),
             _cut(com, r"__host__ __device__[^\n{;]*\bunit_nanos\s*\("),
             _cut(com, r"__host__ __device__[^\n{;]*\bscheme_kind_for_unit\s*\("),
             _cut(com, r"__host__ __device__[^\n{;]*\binitial_time_unit\s*\("),
             _cut(com, _fn("num_sig")), _cut(com, _fn("mult_pow10")),
             _cut(enc, r"struct EncLane"), _cut(enc, _fn("put32")), _cut(enc, _fn("put64")), EMIT,
             _cut(enc, _fn("emit_code"))]
    for name in ("maybe_int", "go_f64_to_u64_via_i64", "convert_to_int_float", "track_new_sig", "sig_mult_hdr",
                 "xor_code", "encode_value", "encode_time"):
        parts.append(_cut(enc, _fn(name)))
    parts += [_cut(enc, r"struct Tier2"), _cut(enc, _fn("div_unit")), _cut(enc, _fn("tier2_candidate")),
              _cut(enc, _fn("tier2_commit"))]
    body = "\n".join(parts)
    assert "asm" not in body, "a PTX block slipped into the host build"
    d = tempfile.mkdtemp(prefix="m3dev_enc_host_")
    path = os.path.join(d, "dev_enc_host.cpp")
    open(path, "w").write(SHIM + body + DRIVER)
    so = os.path.join(d, "dev_enc_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-w", path, "-o", so])
    lib = C.CDLL(so)
    lib.dev_encode_series.restype = C.c_longlong
    lib.dev_encode_series.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int64, C.c_int, C.c_int,
                                      C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_int), C.c_void_p]
    return lib


@pytest.fixture(scope="module")
def dev():
    return build_dev_encoder()


def _dev_encode(dev, ts, vals, start, unit, int_opt, use_tier2, units=None):
    ts = np.ascontiguousarray(ts, dtype=np.int64)
    vals = np.ascontiguousarray(vals, dtype=np.float64)
    un = None if units is None else np.ascontiguousarray(units, dtype=np.uint8)
    out = np.zeros(64 + 24 * len(ts), dtype=np.uint8)
    nt = C.c_int()
    n = dev.dev_encode_series(ts.ctypes.data, vals.ctypes.data, None if un is None else un.ctypes.data, len(ts),
                              int(start), int(unit), int(int_opt), 1, int(use_tier2), out.ctypes.data, len(out),
                              C.byref(nt), None)
    assert n >= 0, n
    return out[:n].tobytes(), nt.value


def _gen(r, num_dig, num_dec):
    dig = r.getrandbits(62) % 10 ** num_dig
    return float(dig) if num_dec == 0 else float("%d.%d" % (dig, r.getrandbits(62) % 10 ** num_dec))


def _series(int_opt):
    r = random.Random(71 + int(int_opt))
    rng = np.random.default_rng(73 + int(int_opt))
    start = 1599955200 * SEC
    fams = [(12, 0), (7, 6), (0, 1), (2, 16), (5, 3), (3, 0), (18, 0), (1, 2), (0, 6), (4, 4), (9, 2), (0, 0)]
    for num_dig, num_dec in fams:
        for rep in range(3):
            P = 250
            ts = start + np.cumsum(rng.choice([1, 10, 60, 60, 60, 300, 4000, 10 ** 6], size=P)).astype(np.int64) * SEC
            if rep == 0:
                ts = start + np.arange(1, P + 1, dtype=np.int64) * 60 * SEC
            vals = np.array([_gen(r, num_dig, num_dec) for _ in range(P)])
            if rep == 1:
                vals *= rng.choice([-1.0, 1.0], size=P)
            if rep == 2:
                idx = rng.integers(1, P, size=P // 4)
                vals[idx] = vals[idx - 1]
                oth = rng.integers(0, P, size=P // 8)
                vals[oth] = [_gen(r, *fams[r.randrange(len(fams))]) for _ in oth]
            yield ts, vals, start
    for k in range(12):
        P = 300
        ts = start + np.arange(1, P + 1, dtype=np.int64) * 60 * SEC
        if k % 3 == 0:
            vals = 100.0 + np.cumsum(rng.normal(size=P))
        elif k % 3 == 1:
            vals = np.round(np.cumsum(rng.normal(size=P) * 10.0 ** rng.integers(0, 12)))
        else:
            vals = np.round(rng.normal(size=P) * 5, int(rng.integers(0, 7)))
            sp = [np.nan, np.inf, -np.inf, -0.0, 2.0 ** 63, -2.0 ** 63, 1e300, -1e300, 5e-324, 0.0, 9.2e18, 1e13]
            vals[::23] = (sp * 2)[: len(vals[::23])]
        yield ts, vals, start


@pytest.mark.parametrize("int_opt", [True, False])
def test_device_encoder_functions_reproduce_oracle_bytes(dev, int_opt):
    n = n_t2 = n_dp = 0
    for ts, vals, start in _series(int_opt):
        exp = O.encode_series(ts, vals, start, O.UNIT_S, int_opt)
        general, zero = _dev_encode(dev, ts, vals, start, O.UNIT_S, int_opt, use_tier2=False)
        mixed, t2 = _dev_encode(dev, ts, vals, start, O.UNIT_S, int_opt, use_tier2=True)
        assert zero == 0
        assert general == exp, n
        assert mixed == exp, n
        n += 1
        n_t2 += t2
        n_dp += len(ts)
    assert n == 48 and n_t2 > 0.3 * n_dp  # the second tier really carried a large share of the datapoints


@pytest.mark.parametrize("int_opt", [True, False])
def test_device_encoder_time_units_and_unit_changes(dev, int_opt):
    """all four scheme units as the series' unit, and per-datapoint unit changes (marker + 64-bit delta-of-delta)"""
    rng = np.random.default_rng(91)
    start = 1599955200 * SEC
    for unit, step in ((O.UNIT_S, SEC), (O.UNIT_MS, 10 ** 6), (O.UNIT_US, 10 ** 3), (O.UNIT_NS, 1)):
        P = 200
        ts = start + np.cumsum(rng.integers(1, 5000, size=P)).astype(np.int64) * step
        vals = np.round(rng.normal(size=P) * 100, 2)
        e = O.Encoder(start, int_opt)
        for t, v in zip(ts.tolist(), vals.tolist()):
            assert e.encode(t, v, unit, b"") == 0
        for tier2 in (False, True):
            got, _ = _dev_encode(dev, ts, vals, start, unit, int_opt, tier2)
            assert got == e.stream(), (unit, tier2)
    P = 240
    ts = start + np.cumsum(rng.integers(1, 5000, size=P)).astype(np.int64) * 10 ** 6
    vals = np.round(rng.normal(size=P) * 100, 1)
    units = np.full(P, O.UNIT_S, dtype=np.uint8)
    units[40:80] = O.UNIT_MS
    units[80:120] = O.UNIT_US
    units[120:121] = O.UNIT_NS
    units[200:] = O.UNIT_MS
    e = O.Encoder(start, int_opt)
    for t, v, u in zip(ts.tolist(), vals.tolist(), units.tolist()):
        assert e.encode(t, v, u, b"") == 0
    for tier2 in (False, True):
        got, _ = _dev_encode(dev, ts, vals, start, O.UNIT_S, int_opt, tier2, units=units)
        assert got == e.stream(), tier2
