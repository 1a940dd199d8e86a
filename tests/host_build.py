"""Test support for the host harnesses (not a test module; nothing of it ships).

The `test_device_*_on_host.py` harnesses cut `__device__` functions, structs and constants out of the CUDA sources at
test time, compile them for the host with g++ and drive them against the oracle.  This module is the plumbing they
share: `cut` / `fn` / `constants` to take code out of the sources, one `PRELUDE` that stands in for what CUDA and PTX
provide, one `compile` (the kernels' arithmetic: no FMA contraction, as nvcc's -fmad=false), the builders that several
harnesses drive (the encoder's lane, its append path, the decoder's complete grammar), and `build_c_oracle` for the
tile-path C oracles tests/*_oracle.c."""
import atexit
import ctypes as C
import functools
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np

TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
CSRC = os.path.join(ROOT, "m3_b200", "csrc")


@functools.lru_cache(maxsize=None)
def source_text(name):
    """the text of m3_b200/csrc/<name>"""
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def cut(src, pattern):
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


def fn(name):
    """the pattern of a `__device__` function's definition, for `cut`"""
    return r"__device__[^\n;{]*\b%s\s*\(" % re.escape(name)


def constants(src, names):
    """the `constexpr` lines of `src` that define a name matching the regex `names`, as they are written there"""
    lines = re.findall(r"^constexpr [\w ]+?\b(?:%s) = [^\n]*$" % names, src, flags=re.M)
    assert lines, names
    return "\n".join(lines)


# What CUDA and PTX provide, for device code compiled by g++: the qualifiers, the thread indices (a driver sets
# them before it calls a kernel body), the intrinsics the cut code calls -- each the IEEE-rounded operation or the
# plain statement of its contract -- and the PTX helpers of m3tsz_common.cuh.  Status codes and record types come from
# the public header itself.
PRELUDE = r"""
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>
#include "%s"
#define __device__
#define __host__
#define __global__
#define __forceinline__ inline
#define __noinline__
#define __launch_bounds__(...)
struct Dim3 { unsigned x, y, z; };
static thread_local Dim3 threadIdx, blockIdx, blockDim;
struct uint4 { uint32_t x, y, z, w; };
static inline double __dmul_rn(double a, double b) { return a * b; }
static inline double __dsub_rn(double a, double b) { return a - b; }
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline double __ddiv_rn(double a, double b) { return a / b; }
static inline double __dsqrt_rn(double a) { return std::sqrt(a); }
static inline long long __double2ll_rz(double a) { return (long long)a; }
static inline double __ull2double_rn(unsigned long long a) { return (double)a; }
static inline double __ll2double_rn(long long a) { return (double)a; }
static inline long long __double_as_longlong(double a) { long long r; memcpy(&r, &a, 8); return r; }
static inline double __longlong_as_double(long long a) { double r; memcpy(&r, &a, 8); return r; }
static inline int __clzll(long long v) { return v ? __builtin_clzll((unsigned long long)v) : 64; }
// funnel shift right, shift amount clamped to 32 (PTX shf.r.clamp)
static inline uint32_t __funnelshift_rc(uint32_t lo, uint32_t hi, uint32_t sh) {
  if (sh > 32) sh = 32;
  const uint64_t v = ((uint64_t)hi << 32) | lo;
  return (uint32_t)(v >> sh);
}
// funnel shift left by (sh & 31): the high word of (hi:lo) << sh  (PTX shf.l.wrap)
static inline uint32_t __funnelshift_l(uint32_t lo, uint32_t hi, uint32_t sh) {
  sh &= 31;
  return sh ? ((hi << sh) | (lo >> (32 - sh))) : hi;
}
static inline uint32_t __byte_perm(uint32_t v, uint32_t, uint32_t sel) {  // only the byte swap is used
  if (sel != 0x0123) __builtin_trap();
  return __builtin_bswap32(v);
}
static inline uint32_t __ldg(const uint32_t *p) { return *p; }
static inline uint4 __ldg(const uint4 *p) { return *p; }
static inline uint32_t __dp4a(uint32_t a, uint32_t b, uint32_t c) {
  for (int i = 0; i < 4; i++) c += ((a >> (8 * i)) & 0xffu) * ((b >> (8 * i)) & 0xffu);
  return c;
}
// one thread at a time: the atomics are plain read-modify-writes
static inline unsigned long long atomicAdd(unsigned long long *p, unsigned long long v) {
  const unsigned long long o = *p;
  *p += v;
  return o;
}
static inline uint32_t atomicAdd(uint32_t *p, uint32_t v) { const uint32_t o = *p; *p += v; return o; }
static inline uint32_t atomicSub(uint32_t *p, uint32_t v) { const uint32_t o = *p; *p -= v; return o; }
// ---- PTX helpers of m3tsz_common.cuh restated ----
// Go shift semantics: x >> n == 0 and x << n == 0 for n >= 64.
static inline uint64_t shl64(uint64_t x, int n) { return n >= 64 ? 0ull : x << n; }
static inline uint64_t shr64(uint64_t x, int n) { return n >= 64 ? 0ull : x >> n; }
// PTX shifts: amounts above 63 (incl. "negative" ones read as unsigned) shift everything out
static inline uint64_t shl64_clamp(uint64_t x, uint32_t n) { return n > 63 ? 0ull : x << n; }
static inline uint64_t shr64_clamp(uint64_t x, uint32_t n) { return n > 63 ? 0ull : x >> n; }
// encoding.LeadingAndTrailingZeros (encoding.go:33-43): (64, 0) for v == 0
static inline void lz_tz(uint64_t v, int &lz, int &tz) {
  if (!v) { lz = 64; tz = 0; return; }
  lz = __builtin_clzll(v);
  tz = __builtin_ctzll(v);
}
""" % os.path.join(ROOT, "include", "m3tsz_b200.h")


@functools.lru_cache(maxsize=None)
def _dir():
    """one temporary directory per process, removed at exit"""
    d = tempfile.mkdtemp(prefix="m3_host_build_")
    atexit.register(shutil.rmtree, d, ignore_errors=True)
    return d


def compile(name, body, driver):
    """PRELUDE + body (the code cut from the sources, and a harness' own restatements) + driver (its extern "C"
    exports), compiled by g++ as the kernels are by nvcc -fmad=false, loaded"""
    assert "asm" not in body, "a PTX block slipped into the host build"
    path = os.path.join(_dir(), name + ".cpp")
    assert not os.path.exists(path), "%s built twice in one process" % name
    with open(path, "w") as f:
        f.write(PRELUDE + body + driver)
    so = os.path.join(_dir(), name + ".so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-w", path, "-o", so])
    return C.CDLL(so)


def build_c_oracle(name):
    """tests/<name>_oracle.c -> tests/libm3tsz_<name>_oracle.so, with oracle/Makefile's flags (and its CC override),
    rebuilt when the source is newer than the library; returns the library's path"""
    src = os.path.join(TESTS, name + "_oracle.c")
    lib = os.path.join(TESTS, "libm3tsz_%s_oracle.so" % name)
    if os.path.exists(lib) and os.path.getmtime(lib) >= os.path.getmtime(src):
        return lib
    with open(os.path.join(ROOT, "oracle", "Makefile")) as f:
        cflags = re.search(r"^CFLAGS \?= (.*)$", f.read(), flags=re.M).group(1).split()
    subprocess.check_call([os.environ.get("CC", "gcc")] + cflags + ["-shared", "-o", lib, src, "-lm"])
    return lib


# ---- the encoder's lane ----

# emit_code_p: header (low hb bits of hdr) followed by the payload given LEFT-ALIGNED in P (top plen bits)
EMIT = r"""
inline void emit_code_p(EncLane &s, uint32_t *tile, int lane, uint32_t hdr, int hb, uint64_t P, int plen) {
  if (hb > 0) put32(s, tile, lane, hb >= 32 ? hdr : (hdr & ((1u << hb) - 1u)), hb);
  if (plen > 0) put64(s, tile, lane, P >> (64 - plen), plen);
}
"""


def _units():
    """the marker constants, kMaxMult and the time-unit helpers of m3tsz_common.cuh"""
    com = source_text("m3tsz_common.cuh")
    return [constants(com, r"kMarker\w*|kMaxMult"), cut(com, r"enum SchemeKind")] + [
        cut(com, r"__host__ __device__[^\n{;]*\b%s\s*\(" % name)
        for name in ("unit_is_valid", "unit_nanos", "scheme_kind_for_unit", "initial_time_unit")]


def encoder_lane(state=False):
    """the encoder's general path and second tier (m3tsz_encode.cu), and with `state` the open-encoder state and its
    load / save / snapshot functions the append path adds"""
    enc, com = source_text("m3tsz_encode.cu"), source_text("m3tsz_common.cuh")
    parts = _units() + [constants(enc, "ENC_STRIDE"), cut(com, fn("num_sig")), cut(com, fn("mult_pow10")),
                        cut(enc, r"struct EncLane"), cut(enc, fn("put32")), cut(enc, fn("put64")), EMIT,
                        cut(enc, fn("emit_code"))]
    for name in ("maybe_int", "go_f64_to_u64_via_i64", "convert_to_int_float", "track_new_sig", "sig_mult_hdr",
                 "xor_code", "encode_value", "encode_time"):
        parts.append(cut(enc, fn(name)))
    parts += [cut(enc, r"struct Tier2"), cut(enc, fn("div_unit")), cut(enc, fn("tier2_candidate")),
              cut(enc, fn("tier2_commit"))]
    if state:
        parts += [cut(com, r"__host__ __device__[^\n{;]*\bxxh64\s*\("), cut(enc, r"struct EncStateInternal")]
        for name in ("enc_state_tag", "enc_state_reset", "enc_state_load", "enc_state_save", "enc_check_time",
                     "enc_snapshot_words"):
            parts.append(cut(enc, fn(name)))
    return "\n".join(parts)


ENCODE_DRIVER = r"""
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


@functools.lru_cache(maxsize=None)
def build_dev_encoder():
    """Compiles the encoder's general path and second tier for the host (g++ only) and returns the loaded library:
    `dev_encode_series(ts, vals, units, n, start, unit, int_opt, default_unit, use_tier2, out, cap, &n_tier2,
    tiers)` returns the stream's length, or minus the status; `tiers` (may be NULL) receives per datapoint 1 for
    the general path and 2 for the second tier."""
    lib = compile("dev_enc_host", encoder_lane(), ENCODE_DRIVER)
    lib.dev_encode_series.restype = C.c_longlong
    lib.dev_encode_series.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int64, C.c_int, C.c_int,
                                      C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_int), C.c_void_p]
    return lib


APPEND_DRIVER = r"""
// one append call on one encoder: what a lane of encode_kernel<., false, ., true> does with its series
template <bool INT_OPT>
static long long append_call(m3tsz_encoder_state *st, uint8_t *slot, const int64_t *ts, const double *vals,
                             const uint8_t *units, int unit, size_t n, const uint32_t *ann_off,
                             const uint32_t *ann_len, const uint8_t *ann_bytes, int use_tier2, int *err) {
  std::vector<uint32_t> tile((n * 40 + 64) * ENC_STRIDE, 0u);
  EncLane s;
  memset(&s, 0, sizeof(s));
  uint64_t ann_cs = 0;
  *err = enc_state_load<INT_OPT>(*st, s, tile.data(), 0, ann_cs);
  if (*err) return 0;
  const uint32_t n0 = s.n_enc;
  if (n && s.n_enc == 0) put64(s, tile.data(), 0, (uint64_t)s.prev_time, 64);
  for (size_t i = 0; i < n; i++) {
    const int64_t t = ts[i];
    const double v = vals[i];
    const int u = units ? (int)units[i] : unit;
    *err = enc_check_time(s, t, u);
    if (*err) break;
    if (ann_len[i]) {  // timestamp_encoder.go:166-195 with the checksum carried in the state
      const uint64_t h = xxh64(ann_bytes + ann_off[i], ann_len[i]);
      if (h != ann_cs) {
        put32(s, tile.data(), 0, (kMarkerOpcode << 2) | (uint32_t)kMarkerAnnotation, kMarkerBits);
        uint64_t ux = ((uint64_t)(ann_len[i] - 1)) << 1;
        while (ux >= 0x80) {
          put32(s, tile.data(), 0, (uint32_t)(ux & 0x7f) | 0x80u, 8);
          ux >>= 7;
        }
        put32(s, tile.data(), 0, (uint32_t)ux, 8);
        for (uint32_t b = 0; b < ann_len[i]; b++) put32(s, tile.data(), 0, ann_bytes[ann_off[i] + b], 8);
      }
      ann_cs = h;
    }
    const bool steady = (u == s.unit) && (s.unit >= 1 && s.unit <= 4) && s.n_enc > 0;
    uint64_t fb;
    memcpy(&fb, &v, 8);
    const int64_t delta = (int64_t)((uint64_t)t - (uint64_t)s.prev_time);
    Tier2 c2;
    if (use_tier2 && tier2_candidate<INT_OPT>(s, steady, delta, fb, v, c2)) {
      s.prev_time = t;
      s.prev_delta = delta;
      tier2_commit<INT_OPT>(s, tile.data(), 0, fb, c2);
    } else {
      uint32_t hdr;
      int hb;
      encode_time(s, tile.data(), 0, t, u, hdr, hb);
      if (s.err) {  // enc_check_time let through a datapoint encode_time refuses
        *err = -1;
        return -1;
      }
      uint64_t payload;
      int plen;
      encode_value<INT_OPT>(s, v, hdr, hb, payload, plen);
      emit_code(s, tile.data(), 0, hdr, hb, payload, plen);
    }
    s.n_enc++;
  }
  // the epilogue's flush: whole sectors to the slot, <= 7 words stay
  const uint32_t done = s.k & ~7u;
  for (uint32_t w = 0; w < done; w++)
    for (int b = 0; b < 4; b++) slot[(s.words_out + w) * 4ull + b] = (uint8_t)(tile[w * ENC_STRIDE] >> (24 - 8 * b));
  for (uint32_t w = done; w < s.k; w++) tile[(w - done) * ENC_STRIDE] = tile[w * ENC_STRIDE];
  s.words_out += done;
  s.k -= done;
  if (s.n_enc != n0) enc_state_save<INT_OPT>(*st, s, tile.data(), 0, ann_cs);
  return (long long)(s.n_enc - n0);
}
extern "C" long long dev_append(m3tsz_encoder_state *st, uint8_t *slot, const int64_t *ts, const double *vals,
                                const uint8_t *units, int unit, size_t n, const uint32_t *ann_off,
                                const uint32_t *ann_len, const uint8_t *ann_bytes, int int_opt, int use_tier2,
                                int *err) {
  return int_opt ? append_call<true>(st, slot, ts, vals, units, unit, n, ann_off, ann_len, ann_bytes, use_tier2, err)
                 : append_call<false>(st, slot, ts, vals, units, unit, n, ann_off, ann_len, ann_bytes, use_tier2, err);
}
extern "C" void dev_reset(m3tsz_encoder_state *st, int64_t start, int default_unit, int int_opt) {
  enc_state_reset(*st, start, default_unit, int_opt != 0);
}
// the snapshot kernel's work for one encoder; returns Len()
extern "C" uint64_t dev_snapshot(const m3tsz_encoder_state *st, uint8_t *slot) {
  uint32_t w[12];
  uint64_t at = 0;
  const uint32_t n = enc_snapshot_words(*st, w, at);
  for (uint32_t i = 0; i < n; i++)
    for (int b = 0; b < 4; b++) slot[(at + i) * 4 + b] = (uint8_t)(w[i] >> (24 - 8 * b));
  return st->num_encoded ? (st->bits + kMarkerBits + 7) / 8 : 0;
}
"""


def build_dev_append(name="dev_append_host", body="", driver=""):
    """Compiles the encoder's lane with its open-encoder state, plus `body` and `driver`, and returns the loaded
    library: `dev_reset(state, start, default_unit, int_opt)`, `dev_append(state, slot, ts, vals, units, unit, n,
    ann_off, ann_len, ann_bytes, int_opt, use_tier2, &err)` (one append call: the datapoints taken, `err` the status)
    and `dev_snapshot(state, slot)` (writes the stream's tail into the slot, returns Len())."""
    lib = compile(name, encoder_lane(state=True) + "\n" + body, APPEND_DRIVER + driver)
    vp = C.c_void_p
    lib.dev_append.restype = C.c_longlong
    lib.dev_append.argtypes = [vp, vp, vp, vp, vp, C.c_int, C.c_size_t, vp, vp, vp, C.c_int, C.c_int,
                               C.POINTER(C.c_int)]
    lib.dev_reset.restype = None
    lib.dev_reset.argtypes = [vp, C.c_int64, C.c_int, C.c_int]
    lib.dev_snapshot.restype = C.c_uint64
    lib.dev_snapshot.argtypes = [vp, vp]
    return lib


# ---- the decoder's complete grammar ----

DECODE_DRIVER = r"""
template <bool INT_OPT>
static int drive(const uint8_t *buf, uint64_t nbytes, uint64_t o0, uint64_t o1, int default_unit, int64_t *ts,
                 uint64_t *vals, uint32_t *bitpos, uint32_t cap, uint32_t *n_out, m3tsz_dp_event *events,
                 uint64_t ev_cap, unsigned long long *ev_count, int *units, uint32_t *ann) {
  DecState s;
  memset(&s, 0, sizeof(s));
  s.scheme = kSchemeNone;
  // the kernel's addressing: base = the stream's first word rounded down to a 16-word boundary
  const uint64_t w = o0 >> 2;
  s.wbase = w & ~(uint64_t)15;
  s.pos = (uint32_t)(w - s.wbase) * 32u + (uint32_t)(o0 & 3) * 8u;
  s.end = s.pos + (uint32_t)(o1 - o0) * 8u;
  const uint32_t pos0 = s.pos;
  SlowSrc src;
  src.base = buf;
  src.nbytes = nbytes;
  src.ring_lane = nullptr;
  src.ring_safe = 0;
  EventSink ev;
  ev.events = events;
  ev.capacity = ev_cap;
  ev.count = ev_count;
  ev.series = 0;
  ev.pos0 = pos0;
  while (!s.done && s.err == 0 && s.n < cap) {
    int64_t t = 0;
    uint64_t v = 0;
    if (decode_dp_slow<INT_OPT>(s, src, default_unit, t, v, &ev)) {
      ts[s.n] = t;
      vals[s.n] = v;
      bitpos[s.n] = s.pos - pos0;  // the stream bit after the datapoint
      s.n++;
    }
  }
  *n_out = s.n;
  units[0] = s.emit_unit;  // unit at the last datapoint produced
  units[1] = s.first_unit;  // ... at the first
  units[2] = s.unit;        // unit in force when the decode stopped
  // the first annotation, as the kernel's m3tsz_annotation_ref holds it
  ann[0] = s.ann_count ? s.ann_bit - pos0 : 0u;
  ann[1] = s.ann_len;
  ann[2] = s.ann_count;
  return s.err;
}
extern "C" int dev_decode(const uint8_t *buf, uint64_t nbytes, uint64_t o0, uint64_t o1, int int_opt, int default_unit,
                          int64_t *ts, uint64_t *vals, uint32_t *bitpos, uint32_t cap, uint32_t *n_out,
                          m3tsz_dp_event *events, uint64_t ev_cap, unsigned long long *ev_count, int *units,
                          uint32_t *ann) {
  return int_opt ? drive<true>(buf, nbytes, o0, o1, default_unit, ts, vals, bitpos, cap, n_out, events, ev_cap,
                               ev_count, units, ann)
                 : drive<false>(buf, nbytes, o0, o1, default_unit, ts, vals, bitpos, cap, n_out, events, ev_cap,
                                ev_count, units, ann);
}
"""


@functools.lru_cache(maxsize=None)
def build_dev_decoder():
    """Compiles the decoder's complete grammar for the host (g++ only) and returns the loaded library."""
    dec, com = source_text("m3tsz_decode.cu"), source_text("m3tsz_common.cuh")
    m = re.search(r"#define M3_RD\(nbits, var\).*?\n  \}\n", dec, flags=re.S)
    assert m
    parts = _units() + [constants(dec, "DEC_RING|DEC_QUADS"), cut(com, fn("sign_extend")),
                        cut(com, fn("mult_pow10")), cut(com, fn("load_be32")), cut(dec, r"struct DecState"),
                        cut(dec, r"struct SlowSrc"), cut(dec, r"struct EventSink"), cut(dec, fn("push_event")),
                        cut(dec, fn("gpeek64")), m.group(0), cut(dec, fn("decode_dp_slow"))]
    lib = compile("dev_dec_host", "\n".join(parts), DECODE_DRIVER)
    lib.dev_decode.restype = C.c_int
    return lib


class DevDecode:
    """One stream through the complete grammar: `status`, `dps` [(ts, value bits)], `bitpos` (the stream bit after
    each datapoint), `emit_unit` / `first_unit` / `unit` (at the last and first datapoint, and when the decode
    stopped), `ann` (the first annotation: bit offset from the stream's first bit, length, count) and `events`
    (uint8 [E, 32] rows of m3tsz_dp_event, series 0)."""

    def __init__(self, dev, stream, int_opt, lead=0, cap=4096, default_unit=1, ev_cap=256):
        buf = np.zeros(lead + len(stream) + 64, dtype=np.uint8)
        buf[lead: lead + len(stream)] = np.frombuffer(stream, dtype=np.uint8)
        ts = np.zeros(cap, dtype=np.int64)
        vals = np.zeros(cap, dtype=np.uint64)
        bitpos = np.zeros(cap, dtype=np.uint32)
        n = C.c_uint32()
        events = np.zeros((ev_cap, 32), dtype=np.uint8)
        evc = C.c_ulonglong(0)
        units = np.zeros(3, dtype=np.int32)
        ann = np.zeros(3, dtype=np.uint32)
        p = lambda a: C.c_void_p(a.ctypes.data)
        self.status = dev.dev_decode(p(buf), C.c_uint64(lead + len(stream)), C.c_uint64(lead),
                                     C.c_uint64(lead + len(stream)), int(int_opt), int(default_unit), p(ts), p(vals),
                                     p(bitpos), C.c_uint32(cap), C.byref(n), p(events), C.c_uint64(ev_cap),
                                     C.byref(evc), p(units), p(ann))
        k = n.value
        self.ts, self.vals, self.bitpos = ts[:k], vals[:k], bitpos[:k]
        self.dps = list(zip(self.ts.tolist(), self.vals.tolist()))
        self.emit_unit, self.first_unit, self.unit = (int(u) for u in units)
        self.ann = tuple(int(a) for a in ann)
        assert evc.value <= ev_cap
        self.events = events[: evc.value]
