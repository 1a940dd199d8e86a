// m3tsz_encode.cu -- batch M3TSZ encode for sm_90a (+ stream compaction).
//
// Mapping (DESIGN.md §4): one LANE per series, 32 series per warp.  The
// int-optimised value grammar is a sequential state machine per series
// (maxMult / isFloat / IntSigBitsTracker, m3tsz/encoder.go:148-250), so each
// lane runs its series' encoder while the WARP cooperates on memory:
// (ts, value) inputs are staged through a transposed shared-memory tile from
// coalesced 128-byte loads, each datapoint's code (<= 32-bit header + <= 64-bit
// payload) is merged into a per-lane bit accumulator with funnel shifts, full
// 32-bit words go to a transposed output tile, and pairs of lanes write their
// two series' words back in whole 32-byte sectors.
//
// Format: SURVEY.md Appendix A; reference encode path
//   m3tsz/encoder.go:90-250, m3tsz/timestamp_encoder.go:72-259,
//   m3tsz/float_encoder_iterator.go:69-103, m3tsz/int_sig_bits_tracker.go:35-91,
//   m3tsz/m3tsz.go:78-119, ostream.go:133-221, scheme.go:198-220.
#include <cstring>
#include <type_traits>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cuda.h>  // CUtensorMap (types only: the encoder is resolved through cudaGetDriverEntryPoint)

#include "m3tsz_common.cuh"
#include "m3tsz_kernels.h"

namespace m3tsz {

constexpr int ENC_WARPS = 4;
constexpr int ENC_STRIDE = 33;
constexpr int ENC_IN_T = 8;     // datapoints per input tile of the series-major stage (double buffered, cp.async)
// output tile words per lane (smaller tile = more L1): the 24 words that 16-byte flushes used, plus 4 for the
// larger leftover of whole-sector flushes, so a flush cycle still adds about as many words as before
constexpr int ENC_OUT_W = 28;
// Residency the launch bounds promise.  The series-major stage (IN = 0) uses ~48 KB of shared memory per block,
// so the 132 KB carveout below holds 2 of them; the point-major stage (IN = 1) uses ~31 KB and fits 4; the Gauge
// stage (IN = 2) has no input tiles and fits more.
constexpr int ENC_MIN_BLOCKS = 2;
constexpr int ENC_MIN_BLOCKS_PM = 4;
constexpr int ENC_MIN_BLOCKS_AGG = 4;
constexpr int ENC_GUARD = 10;   // words a single datapoint (no annotation) may add
constexpr int ENC_OUT_TILE_WORDS = ENC_OUT_W * ENC_STRIDE;
// A flush writes whole 32-byte sectors and leaves up to 7 words in the tile.  The tile is flushed once it holds
// more than ENC_OUT_W - ENC_GUARD words; that must be at least one sector, so every flush makes room.
static_assert(ENC_OUT_W - ENC_GUARD >= 8, "output tile too small for sector flushes");
// rows per input tile of the point-major input stage (IN = 1).  Tensor copies do not allocate L1 lines, so one
// copy per array costs the same whatever the box; the tile size sets the shared memory per warp and with it the
// residency.  Measured with ENC_NSTAGE_PM (ENC_CARVEOUT_KB has the numbers): 4 x 2 (4 blocks at 132 KB) was the
// fastest; 2 x 2 (5 blocks), 2 x 4 and 4 x 3 (3 blocks) were slower.
constexpr int ENC_IN_T_PM = 4;
// input tiles in flight per warp in the point-major stage (a ring of stages, one mbarrier each)
constexpr int ENC_NSTAGE_PM = 2;
// input stage IN: 0 series-major tiles (8 rows: one 64-byte segment per series and array), 1 point-major
// tiles, 2 Gauge aggregates read directly (no input tiles), 4 the same through the transformations
// IN = 3 (append mode only): a bucket write's share of one encoder (DESIGN.md §4.11).  Each lane reads its own
// series' datapoints directly (the lanes of the overflow pass belong to scattered series) and takes the ones the
// route kernel sent to its encoder.
template <int IN>
__host__ __device__ constexpr int enc_in_t() {
  return IN == 1 ? ENC_IN_T_PM : ENC_IN_T;
}
template <int IN>
__host__ __device__ constexpr int enc_nstage() {
  return IN == 1 ? ENC_NSTAGE_PM : 2;
}
// The point-major stage (IN = 1) fills its tiles by TMA tensor copies: the arrays are described as 2-D tensors
// [points][series] of 8-byte elements (cuTensorMapEncodeTiled, box = IN_T rows x 32 series), so one
// cp.async.bulk.tensor.2d per array moves a whole tile; rows past the end and series past n_series are
// zero-filled by the hardware, which makes ragged batches and the last partial tile the same code.  A tile row is
// then 32 datapoints exactly (no padding column: the copies' destinations must be 16-byte aligned, and the
// lane-local reads are conflict-free either way).  Needs 16-byte aligned arrays and an even n_series < 2^31, else
// the stage keeps the lane-local 8-byte cp.async fills.
template <int IN>
__host__ __device__ constexpr bool enc_bulk() {
  return IN == 1;
}
// the two tensor maps of the point-major input arrays, a __grid_constant__ kernel parameter
struct EncTensorMaps {
  alignas(64) CUtensorMap ts;
  alignas(64) CUtensorMap val;
  int ok;  // 0: not built (unaligned arrays, odd n_series, no driver entry point): cp.async fills
};
// datapoints (8-byte cells) per input tile row
template <int IN>
__host__ __device__ constexpr int enc_in_stride() {
  return enc_bulk<IN>() ? 32 : ENC_STRIDE;
}
// The tile stage with transformations (IN = 4) keeps every lane's m3tsz_transform_state in shared memory behind the
// output tile (in registers the sums pushed the int-optimised kernel past its 128 registers into spills).  A lane's
// record is padded to 104 bytes (26 words): the 16 lanes of a half-warp's 8-byte access then hit distinct bank pairs.
struct XfSlot {
  m3tsz_transform_state st;
  uint64_t pad;
};
static_assert(sizeof(XfSlot) == 104 && (ENC_OUT_TILE_WORDS * 4) % 8 == 0, "transformation state slots");
// The multi-type stage (IN = 5) keeps an element's record there instead, rearranged for the chain: `w` is the
// m3tsz_transform_state xf_window runs on (its prev_v is loaded with the type that runs), pv[j] is type j's
// binary-op input, and `reserved` the record's last word.  The lane's source series and type sit behind it, out of
// the registers (in them the int-optimised kernel spilled).  184 bytes (23 8-byte words, an odd number): the 16
// lanes of a half-warp's 8-byte access hit distinct bank pairs, as in XfSlot.
struct XfElem {
  m3tsz_transform_state w;
  double pv[M3TSZ_MAX_ELEMENT_TYPES];
};
struct XfElemSlot {
  XfElem e;
  uint64_t reserved;
  uint64_t src;  // the lane's source series (row % tile_n_src)
  uint32_t ty;   // its type (row / tile_n_src)
  uint32_t all;  // the list has an Add op: the lane runs every type
};
static_assert(sizeof(XfElemSlot) == 184, "element state slots");
template <int IN>
__host__ __device__ constexpr size_t enc_warp_smem() {
  const size_t raw =
      ((IN == 0 || IN == 1) ? 2 * (size_t)enc_nstage<IN>() * (enc_in_t<IN>() * enc_in_stride<IN>()) * 8 : 0) +
      (size_t)ENC_OUT_TILE_WORDS * 4 + (enc_bulk<IN>() ? 8 * enc_nstage<IN>() : 0) +  // (+ one mbarrier per stage)
      (IN == 4 ? 32 * sizeof(XfSlot) : 0) + ((IN == 5 || IN == 6 || IN == 7) ? 32 * sizeof(XfElemSlot) : 0);
  return enc_bulk<IN>() ? ((raw + 127) & ~(size_t)127) : raw;  // tensor copies land on 128-byte boundaries
}

struct EncLane {
  uint32_t carry, sh, k, words_out;
  int64_t prev_time, prev_delta;
  uint64_t prev_bits;
  int plz, ptz;  // leading / trailing zeros of the previous XOR ((64, 0) for a zero XOR)
  double int_val;
  int unit;
  int num_sig, hi_lower_sig, n_lower_sig, max_mult;
  int err;
  uint32_t n_enc;
  bool is_float;
};

// ---- bit output -----------------------------------------------------------
// appends the low n (1..32) bits of v
__device__ __forceinline__ void put32(EncLane &s, uint32_t *tile, int lane, uint32_t v, int n) {
  const uint32_t c0 = v << (32 - n);
  const uint32_t m0 = s.carry | __funnelshift_rc(c0, 0u, s.sh);
  const uint32_t m1 = __funnelshift_rc(0u, c0, s.sh);
  const uint32_t tot = s.sh + (uint32_t)n;
  if (tot >= 32) {
    tile[s.k * ENC_STRIDE + lane] = m0;
    s.k++;
    s.carry = m1;
    s.sh = tot - 32;
  } else {
    s.carry = m0;
    s.sh = tot;
  }
}
// appends the low n (0..64) bits of v
__device__ __forceinline__ void put64(EncLane &s, uint32_t *tile, int lane, uint64_t v, int n) {
  if (n > 32) {
    put32(s, tile, lane, (uint32_t)(v >> 32), n - 32);
    put32(s, tile, lane, (uint32_t)v, 32);
  } else if (n > 0) {
    put32(s, tile, lane, (uint32_t)v, n);
  }
}

// appends header (low hb bits of hdr, hb 0..32) followed by a payload given
// LEFT-ALIGNED in P (its top plen bits, plen 0..64; bits below must be zero): one
// merge of up to 96 bits into the accumulator.
__device__ __forceinline__ void emit_code_p(EncLane &s, uint32_t *tile, int lane, uint32_t hdr, int hb,
                                            uint64_t P, int plen) {
  const uint32_t H = hb ? (hdr << (32 - hb)) : 0u;
  const uint32_t Ph = (uint32_t)(P >> 32), Pl = (uint32_t)P;
  const uint32_t c0 = H | __funnelshift_rc(Ph, 0u, (uint32_t)hb);
  const uint32_t c1 = __funnelshift_rc(Pl, Ph, (uint32_t)hb);
  const uint32_t c2 = __funnelshift_rc(0u, Pl, (uint32_t)hb);
  const uint32_t m0 = s.carry | __funnelshift_rc(c0, 0u, s.sh);
  const uint32_t m1 = __funnelshift_rc(c1, c0, s.sh);
  const uint32_t m2 = __funnelshift_rc(c2, c1, s.sh);
  const uint32_t m3 = __funnelshift_rc(0u, c2, s.sh);
  const uint32_t tot = s.sh + (uint32_t)(hb + plen);
  const uint32_t full = tot >> 5;
  // predicated stores (kept out of the compiler's hands: it turns the chain into a
  // divergent branch region otherwise)
  const uint32_t ta = (uint32_t)__cvta_generic_to_shared(tile + s.k * ENC_STRIDE + lane);
  asm volatile(
      "{\n\t.reg .pred p0, p1, p2;\n\t"
      "setp.gt.u32 p0, %0, 0;\n\tsetp.gt.u32 p1, %0, 1;\n\tsetp.gt.u32 p2, %0, 2;\n\t"
      "@p0 st.shared.u32 [%1], %2;\n\t@p1 st.shared.u32 [%1+132], %3;\n\t@p2 st.shared.u32 [%1+264], %4;\n\t}"
      ::"r"(full), "r"(ta), "r"(m0), "r"(m1), "r"(m2)
      : "memory");
  static_assert(ENC_STRIDE * 4 == 132, "store offsets above");
  const uint32_t c01 = full == 0 ? m0 : m1, c23 = full == 2 ? m2 : m3;
  s.carry = full < 2 ? c01 : c23;
  s.k += full;
  s.sh = tot & 31u;
}
// same with the payload right-aligned (its low plen bits)
__device__ __forceinline__ void emit_code(EncLane &s, uint32_t *tile, int lane, uint32_t hdr, int hb,
                                          uint64_t payload, int plen) {
  emit_code_p(s, tile, lane, hdr, hb, plen ? (payload << (64 - plen)) : 0ull, plen);
}

// ---- convertToIntFloat (m3tsz.go:78-119) ----------------------------------
// Cheap NECESSARY condition for convertToIntFloat(v, cur) to return an int for
// any cur in [0,6]: if some v*10^m lies within one ulp of an integer, then
// fl(|v|*1e6) lies within 4 ulps of an integer (DESIGN.md §4.2 has the proof);
// tested with margin 8.  Returns true ("maybe int") for everything it cannot
// rule out, including NaN/Inf/huge/tiny values.
__device__ __forceinline__ bool maybe_int(double v) {
  const double a = fabs(v);
  const double p = __dmul_rn(a, 1000000.0);
  // on the (otherwise idle) FP64 pipe: p - rint(p) is exact, and p * 2^-49 lies in
  // [8, 16) ulps of p, so "far" implies more than 8 ulps from the nearest integer
  const double r = __dsub_rn(p, rint(p));
  const bool far = fabs(r) > __dmul_rn(p, 0x1p-49);
  const bool in_rng = (p >= 1.0) && (p < 0x1p48);   // NaN fails both: "maybe int"
  const bool tiny_v = (p < 0.5) && (a >= 1e-300);   // only N = 0 is near, i.e. v ~ 0
  return !((in_rng && far) || tiny_v);
}

// Go int64(float64) on amd64 (CVTTSD2SQ): out of range / NaN -> 0x8000000000000000
__device__ __forceinline__ uint64_t go_f64_to_u64_via_i64(double a) {
  if (!(a >= -9223372036854775808.0 && a < 9223372036854775808.0)) return 0x8000000000000000ull;
  return (uint64_t)__double2ll_rz(a);
}

__device__ __noinline__ void convert_to_int_float(double v, int cur, double &val, int &mult,
                                                  bool &is_float) {
  if (cur == 0 && v < 9223372036854775807.0) {
    const double i = trunc(v);
    if (__dsub_rn(v, i) == 0.0) {
      val = i;
      mult = 0;
      is_float = false;
      return;
    }
  }
  const double sign = (v < 0.0) ? -1.0 : 1.0;
  for (int m = cur; m <= kMaxMult; m++) {
    const double x = __dmul_rn(__dmul_rn(v, mult_pow10(m)), sign);
    if (x >= 1e13) break;
    const double i = trunc(x);
    const double r = __dsub_rn(x, i);
    if (r == 0.0) {
      val = __dmul_rn(sign, i);
      mult = m;
      is_float = false;
      return;
    } else if (r < 0.1) {
      const double below = __longlong_as_double(__double_as_longlong(x) - 1);  // Nextafter(x, 0)
      if (below <= i) {
        val = __dmul_rn(sign, i);
        mult = m;
        is_float = false;
        return;
      }
    } else if (r > 0.9) {
      const double next = __dadd_rn(i, 1.0);
      const double above = __longlong_as_double(__double_as_longlong(x) + 1);  // Nextafter(x, next)
      if (above >= next) {
        val = __dmul_rn(sign, next);
        mult = m;
        is_float = false;
        return;
      }
    }
  }
  val = v;
  mult = 0;
  is_float = true;
}

// IntSigBitsTracker.TrackNewSig, int_sig_bits_tracker.go:68-91
__device__ __forceinline__ int track_new_sig(EncLane &s, int ns) {
  int new_sig = s.num_sig;
  if (ns > s.num_sig) {
    new_sig = ns;
  } else if (s.num_sig - ns >= 3) {
    if (s.n_lower_sig == 0)
      s.hi_lower_sig = ns;
    else if (ns > s.hi_lower_sig)
      s.hi_lower_sig = ns;
    s.n_lower_sig++;
    if (s.n_lower_sig >= 5) {
      new_sig = s.hi_lower_sig;
      s.n_lower_sig = 0;
    }
  } else {
    s.n_lower_sig = 0;
  }
  return new_sig;
}

// writeIntSigMult (encoder.go:235-250) + WriteIntSig (int_sig_bits_tracker.go:48-62):
// appends to the header accumulator
__device__ __forceinline__ void sig_mult_hdr(EncLane &s, int sig, int mult, bool float_changed,
                                             uint32_t &hdr, int &hb) {
  if (s.num_sig != sig) {
    if (sig == 0) {
      hdr = (hdr << 2) | 2u;  // '1' '0'
      hb += 2;
    } else {
      hdr = (hdr << 8) | (3u << 6) | (uint32_t)(sig - 1);  // '1' '1' + 6 bits
      hb += 8;
    }
  } else {
    hdr <<= 1;  // '0'
    hb += 1;
  }
  s.num_sig = sig;
  if (mult > s.max_mult) {
    hdr = (hdr << 4) | 8u | (uint32_t)mult;
    hb += 4;
    s.max_mult = mult;
  } else if (s.max_mult == mult && float_changed) {
    hdr = (hdr << 4) | 8u | (uint32_t)s.max_mult;
    hb += 4;
  } else {
    hdr <<= 1;
    hb += 1;
  }
}

// XOR code (float_encoder_iterator.go:75-103) appended after `hb` prefix bits
__device__ __forceinline__ void xor_code(EncLane &s, uint64_t fb, uint32_t &hdr, int &hb,
                                         uint64_t &payload, int &plen) {
  const uint64_t x = s.prev_bits ^ fb;
  int cl, ct;
  lz_tz(x, cl, ct);  // (64, 0) for x == 0
  if (x == 0) {
    hdr <<= 1;
    hb += 1;
    plen = 0;
  } else if (cl >= s.plz && ct >= s.ptz) {
    hdr = (hdr << 2) | 2u;
    hb += 2;
    payload = x >> s.ptz;
    plen = 64 - s.plz - s.ptz;
  } else {
    const int nm = 64 - cl - ct;
    hdr = (hdr << 14) | (3u << 12) | ((uint32_t)cl << 6) | (uint32_t)(nm - 1);
    hb += 14;
    payload = x >> ct;
    plen = nm;
  }
  s.plz = cl;  // PrevXOR := x
  s.ptz = ct;
  s.prev_bits = fb;
}

// value grammar: encoder.go:112-231.  Produces header bits appended to
// (hdr, hb) and the payload.
template <bool INT_OPT>
__device__ __forceinline__ void encode_value(EncLane &s, double v, uint32_t &hdr, int &hb,
                                             uint64_t &payload, int &plen) {
  const bool first = (s.n_enc == 0);
  const uint64_t vbits = (uint64_t)__double_as_longlong(v);
  payload = 0;
  plen = 0;
  if (!INT_OPT) {
    if (first) {  // writeFullFloat
      s.prev_bits = vbits;
      lz_tz(vbits, s.plz, s.ptz);  // PrevXOR := bits
      payload = vbits;
      plen = 64;
    } else {
      xor_code(s, vbits, hdr, hb, payload, plen);
    }
    return;
  }
  double val = v;
  int mult = 0;
  bool isf = true;
  if (maybe_int(v)) {
    // out-parameters of the (noinline) exact classifier live on the stack: keep
    // them out of the common path
    double v2;
    int m2;
    bool f2;
    convert_to_int_float(v, first ? 0 : s.max_mult, v2, m2, f2);
    val = v2;
    mult = m2;
    isf = f2;
  }
  if (first) {  // writeFirstValue :112-146
    if (isf) {
      hdr = (hdr << 1) | 1u;
      hb += 1;
      s.prev_bits = vbits;
      lz_tz(vbits, s.plz, s.ptz);  // PrevXOR := bits
      payload = vbits;
      plen = 64;
      s.is_float = true;
      s.max_mult = mult;
    } else {
      hdr <<= 1;  // opcodeIntMode
      hb += 1;
      s.int_val = val;
      uint32_t neg_diff = 1;
      double a = val;
      if (val < 0.0) {
        neg_diff = 0;
        a = -val;
      }
      const uint64_t vb = go_f64_to_u64_via_i64(a);
      const int ns = num_sig(vb);
      sig_mult_hdr(s, ns, mult, false, hdr, hb);
      hdr = (hdr << 1) | neg_diff;
      hb += 1;
      payload = vb;
      plen = s.num_sig;
    }
    return;
  }
  // writeNextValue :148-172
  double diff = 0.0;
  if (!isf) diff = __dsub_rn(s.int_val, val);
  if (isf || diff >= 9223372036854775807.0 || diff <= -9223372036854775808.0) {
    const uint64_t fb = (uint64_t)__double_as_longlong(val);  // writeFloatVal :176-198
    if (!s.is_float) {
      hdr = (hdr << 3) | 1u;  // update, no-repeat, float-mode
      hb += 3;
      s.prev_bits = fb;
      lz_tz(fb, s.plz, s.ptz);  // PrevXOR := bits
      payload = fb;
      plen = 64;
      s.is_float = true;
      s.max_mult = mult;
    } else if (fb == s.prev_bits) {
      hdr = (hdr << 2) | 1u;  // update, repeat
      hb += 2;
    } else {
      hdr = (hdr << 1) | 1u;  // no-update
      hb += 1;
      xor_code(s, fb, hdr, hb, payload, plen);
    }
    return;
  }
  // writeIntVal :201-231
  if (diff == 0.0 && !s.is_float && mult == s.max_mult) {
    hdr = (hdr << 2) | 1u;
    hb += 2;
    return;
  }
  uint32_t neg = 0;
  if (diff < 0.0) {
    neg = 1;
    diff = -diff;
  }
  const uint64_t db = go_f64_to_u64_via_i64(diff);
  const int ns = num_sig(db);
  const int new_sig = track_new_sig(s, ns);
  const bool float_changed = s.is_float;
  if (mult > s.max_mult || s.num_sig != new_sig || float_changed) {
    hdr <<= 3;  // update, no-repeat, int-mode
    hb += 3;
    sig_mult_hdr(s, new_sig, mult, float_changed, hdr, hb);
    hdr = (hdr << 1) | neg;
    hb += 1;
    payload = db;
    plen = s.num_sig;
    s.is_float = false;
  } else {
    hdr = (hdr << 2) | 2u | neg;  // no-update + sign
    hb += 2;
    payload = db;
    plen = s.num_sig;
  }
  s.int_val = val;
}

// timestamp grammar: timestamp_encoder.go:104-246 (annotation handled by caller).
// Small codes are returned in (hdr, hb); 32/64-bit fields are written directly.
__device__ __forceinline__ void encode_time(EncLane &s, uint32_t *tile, int lane, int64_t t, int u,
                                            uint32_t &hdr, int &hb) {
  hdr = 0;
  hb = 0;
  const int64_t delta = (int64_t)((uint64_t)t - (uint64_t)s.prev_time);
  const int64_t dd = (int64_t)((uint64_t)delta - (uint64_t)s.prev_delta);
  s.prev_time = t;
  if (u != s.unit && unit_is_valid(u)) {  // maybeWriteTimeUnitChange :141-162
    put32(s, tile, lane, (kMarkerOpcode << 2) | (uint32_t)kMarkerTimeUnit, kMarkerBits);
    put32(s, tile, lane, (uint32_t)u, 8);
    s.unit = u;
    put64(s, tile, lane, (uint64_t)dd, 64);  // writeDeltaOfDeltaTimeUnitChanged :197-203
    s.prev_delta = 0;
    return;
  }
  if (!unit_is_valid(u)) {
    s.err = M3TSZ_ERR_UNRECOGNIZED_UNIT;
    s.prev_delta = delta;
    return;
  }
  s.prev_delta = delta;
  const int kind = scheme_kind_for_unit(u);
  if (dd == 0) {
    hb = (kind == kSchemeZero) ? 0 : 1;
    return;
  }
  const int64_t dod = dd / unit_nanos(u);  // ToNormalizedDuration, x/time/time.go:55-57
  if (u <= 2 && dod != (int64_t)(int32_t)dod) {
    s.err = M3TSZ_ERR_DOD_OVERFLOW;
    return;
  }
  if (kind == kSchemeZero) return;
  if (dod == 0) {
    hb = 1;
  } else if (dod >= -64 && dod <= 63) {
    hdr = (2u << 7) | ((uint32_t)dod & 0x7fu);
    hb = 9;
  } else if (dod >= -256 && dod <= 255) {
    hdr = (6u << 9) | ((uint32_t)dod & 0x1ffu);
    hb = 12;
  } else if (dod >= -2048 && dod <= 2047) {
    hdr = (14u << 12) | ((uint32_t)dod & 0xfffu);
    hb = 16;
  } else {
    put32(s, tile, lane, 0xfu, 4);
    put64(s, tile, lane, (uint64_t)dod, kind == kScheme32 ? 32 : 64);
  }
}

// ---- second-tier candidate (see the kernel's datapoint step) ---------------
struct Tier2 {
  uint32_t thdr;  // delta-of-delta code
  int thb;
  int kind;       // 0 float XOR, 1 float repeat, 2 int diff, 3 int repeat
  uint32_t neg;
  uint64_t db;    // |diff| as integer (kind 2)
  double val;     // converted value (kind 2)
  int n_lower, hi_lower;  // tracker state after this datapoint (kind 2)
  int new_sig;            // significant bits in force after this datapoint (kind 2)
};

// ToNormalizedDuration (x/time/time.go:55-57) with the unit's constant divisor
__device__ __forceinline__ int64_t div_unit(int64_t dd, int u) {
  switch (u) {
    case 1: return dd / 1000000000LL;
    case 2: return dd / 1000000LL;
    case 3: return dd / 1000LL;
    default: return dd;
  }
}

// True when this datapoint can be coded without touching the mode / header
// state: same s/ms/us/ns unit, not the first datapoint, delta-of-delta within the
// 12-bit bucket, and the value is (a) float mode, certainly not int-like, or
// (b) int mode, int-like at the current multiplier, diff in int64 range (a
// significant-bits update is fine, a multiplier or mode change is not).
// Nothing in `s` is modified.
template <bool INT_OPT>
__device__ __forceinline__ bool tier2_candidate(const EncLane &s, bool base, int64_t delta, uint64_t fb,
                                                double v, Tier2 &c) {
  bool ok = base && (s.unit >= 1 && s.unit <= 4) && s.n_enc > 0;
  const int64_t dd = (int64_t)((uint64_t)delta - (uint64_t)s.prev_delta);
  const int64_t dod = div_unit(dd, s.unit);
  ok = ok && (dod >= -2048 && dod <= 2047);
  const uint32_t ud = (uint32_t)dod;
  if (dod == 0) {
    c.thdr = 0;
    c.thb = 1;
  } else if (dod >= -64 && dod <= 63) {
    c.thdr = (2u << 7) | (ud & 0x7fu);
    c.thb = 9;
  } else if (dod >= -256 && dod <= 255) {
    c.thdr = (6u << 9) | (ud & 0x1ffu);
    c.thb = 12;
  } else {
    c.thdr = (14u << 12) | (ud & 0xfffu);
    c.thb = 16;
  }
  c.kind = 0;
  c.neg = 0;
  c.db = 0;
  c.val = 0.0;
  c.n_lower = s.n_lower_sig;
  c.hi_lower = s.hi_lower_sig;
  c.new_sig = s.num_sig;
  if (!INT_OPT) return ok;
  if (s.is_float) {
    c.kind = (fb == s.prev_bits) ? 1 : 0;
    return ok && !maybe_int(v);
  }
  // convertToIntFloat at m = max_mult only (m3tsz.go:78-119); anything that would
  // move on to a larger multiplier is left to the general path
  const double sign = (v < 0.0) ? -1.0 : 1.0;
  const double x = __dmul_rn(__dmul_rn(v, mult_pow10(s.max_mult)), sign);
  const double i = trunc(x);
  const double r = __dsub_rn(x, i);
  const bool exact = (r == 0.0);
  const bool lo = (r < 0.1) && (__longlong_as_double(__double_as_longlong(x) - 1) <= i);
  const double next = __dadd_rn(i, 1.0);
  const bool hi = (r > 0.9) && (__longlong_as_double(__double_as_longlong(x) + 1) >= next);
  ok = ok && (x < 1e13) && (exact || lo || hi);
  c.val = __dmul_rn(sign, (hi && !exact) ? next : i);
  double diff = __dsub_rn(s.int_val, c.val);
  ok = ok && (diff < 9223372036854775807.0) && (diff > -9223372036854775808.0);
  if (diff == 0.0) {
    c.kind = 3;
    return ok;
  }
  c.kind = 2;
  if (diff < 0.0) {
    c.neg = 1;
    diff = -diff;
  }
  c.db = ok ? (uint64_t)__double2ll_rz(diff) : 1ull;
  const int ns = num_sig(c.db);
  // IntSigBitsTracker.TrackNewSig without committing (int_sig_bits_tracker.go:68-91)
  c.new_sig = s.num_sig;
  if (ns > s.num_sig) {
    c.new_sig = ns;
  } else if (s.num_sig - ns >= 3) {
    c.hi_lower = (c.n_lower == 0 || ns > c.hi_lower) ? ns : c.hi_lower;
    c.n_lower++;
    if (c.n_lower >= 5) {
      c.new_sig = c.hi_lower;
      c.n_lower = 0;
    }
  } else {
    c.n_lower = 0;
  }
  return ok;
}

template <bool INT_OPT>
__device__ __forceinline__ void tier2_commit(EncLane &s, uint32_t *tile, int lane, uint64_t fb, const Tier2 &c) {
  if (!INT_OPT || c.kind == 0) {
    const uint32_t pre = INT_OPT ? ((c.thdr << 1) | 1u) : c.thdr;  // + '1' no-update
    const int pb = c.thb + (INT_OPT ? 1 : 0);
    const uint64_t x = s.prev_bits ^ fb;
    int cl, ct;
    lz_tz(x, cl, ct);
    const bool zero = (x == 0);
    const bool cont = !zero && cl >= s.plz && ct >= s.ptz;
    const int nm = 64 - cl - ct;
    const uint64_t P = shl64(x, cont ? s.plz : cl);
    const int plen = zero ? 0 : (cont ? 64 - s.plz - s.ptz : nm);
    const uint32_t hdr = zero ? (pre << 1)
                              : (cont ? ((pre << 2) | 2u)
                                      : ((pre << 14) | (3u << 12) | ((uint32_t)cl << 6) | (uint32_t)(nm - 1)));
    const int hb = pb + (zero ? 1 : (cont ? 2 : 14));
    s.plz = cl;
    s.ptz = ct;
    s.prev_bits = fb;
    emit_code_p(s, tile, lane, hdr, hb, P, plen);
  } else if (c.kind == 2) {  // '1' no-update + sign + num_sig bits (encoder.go:224-230)
    s.n_lower_sig = c.n_lower;
    s.hi_lower_sig = c.hi_lower;
    s.int_val = c.val;
    uint32_t hdr = (c.thdr << 1) | 1u;  // '1' no-update
    int hb = c.thb + 1;
    if (c.new_sig != s.num_sig) {
      // '0' update '0' no-repeat '0' int mode, new significant bits, '0' same multiplier
      // (writeIntSigMult, encoder.go:235-250)
      if (c.new_sig == 0) {
        hdr = (c.thdr << 6) | (2u << 1);
        hb = c.thb + 6;
      } else {
        hdr = (c.thdr << 12) | (3u << 7) | ((uint32_t)(c.new_sig - 1) << 1);
        hb = c.thb + 12;
      }
      s.num_sig = c.new_sig;
    }
    const uint64_t P = s.num_sig ? (c.db << (64 - s.num_sig)) : 0ull;
    emit_code_p(s, tile, lane, (hdr << 1) | c.neg, hb + 1, P, s.num_sig);
  } else {  // '0' update + '1' repeat (float: encoder.go:186-189, int: :202-206)
    emit_code_p(s, tile, lane, (c.thdr << 2) | 1u, c.thb + 2, 0ull, 0);
  }
}

// the append mode's own per-lane variables (encode_kernel)
struct EncAppendVars {
  uint32_t n_enc0 = 0;  // datapoints the encoder held before this call
  uint64_t ann_cs = 0;  // XXH64 of the last annotation written
};
struct EncNoVars {};

// ---- encoder sets: the state record between appends (DESIGN.md §4.6) ------------------------------------------
// m3tsz_encoder_state.internal: what EncLane holds besides the public prefix.  The output tile's leftover words
// (fewer than a sector) and the partial word wait here, so the slot only receives whole sectors and words_out
// stays a multiple of 8; words_out = bits / 32 - k.  prev_time is last_ts (start_ns before the first datapoint).
struct EncStateInternal {
  uint32_t left[7];  // leftover words, stream order
  uint32_t carry;    // partial word: its top `sh` bits
  int64_t prev_delta;
  uint64_t prev_bits;
  double int_val;
  uint64_t meta;  // sh:5 k:3 plz:7 ptz:7 unit:4 num_sig:7 hi_lower_sig:7 n_lower_sig:3 max_mult:3 is_float:1, tag:16
  uint64_t reserved[2];
};
static_assert(sizeof(EncStateInternal) == sizeof(((m3tsz_encoder_state *)0)->internal), "state layout");
static_assert(sizeof(m3tsz_encoder_state) == 128, "state layout");
// the tag records the mode the state was reset in (an append in the other mode is refused)
__host__ __device__ __forceinline__ uint64_t enc_state_tag(bool int_opt) { return int_opt ? 0xe3a1u : 0xe3a0u; }

// Reset(start), encoder.go:262-279 (+ NewTimestampEncoder's empty-annotation checksum, timestamp_encoder.go:56)
__host__ __device__ __forceinline__ void enc_state_reset(m3tsz_encoder_state &st, int64_t start, int default_unit,
                                                         bool int_opt) {
  memset(&st, 0, sizeof(st));
  st.start_ns = start;
  st.ann_checksum = xxh64(nullptr, 0);
  EncStateInternal &in = *reinterpret_cast<EncStateInternal *>(st.internal);
  in.meta = (64ull << 8) | ((uint64_t)initial_time_unit(start, default_unit) << 22) | (enc_state_tag(int_opt) << 48);
}

// state -> lane (+ leftover words into the lane's tile column).  M3TSZ_ERR_INVALID_ARG when the state was reset in
// the other mode (nothing is loaded then).
template <bool INT_OPT>
__device__ __forceinline__ int enc_state_load(const m3tsz_encoder_state &st, EncLane &s, uint32_t *tile, int lane,
                                              uint64_t &ann_cs) {
  const EncStateInternal &in = *reinterpret_cast<const EncStateInternal *>(st.internal);
  const uint64_t m = in.meta;
  if ((m >> 48) != enc_state_tag(INT_OPT)) return M3TSZ_ERR_INVALID_ARG;
  s.sh = (uint32_t)(m & 31u);
  s.k = (uint32_t)((m >> 5) & 7u);
  s.plz = (int)((m >> 8) & 127u);
  s.ptz = (int)((m >> 15) & 127u);
  s.unit = (int)((m >> 22) & 15u);
  s.num_sig = (int)((m >> 26) & 127u);
  s.hi_lower_sig = (int)((m >> 33) & 127u);
  s.n_lower_sig = (int)((m >> 40) & 7u);
  s.max_mult = (int)((m >> 43) & 7u);
  s.is_float = ((m >> 46) & 1u) != 0;
  for (uint32_t i = 0; i < s.k; i++) tile[i * ENC_STRIDE + lane] = in.left[i];
  s.carry = in.carry;
  s.words_out = (uint32_t)(st.bits >> 5) - s.k;
  s.n_enc = (uint32_t)st.num_encoded;
  s.prev_time = st.num_encoded ? st.last_ts : st.start_ns;
  s.prev_delta = in.prev_delta;
  s.prev_bits = in.prev_bits;
  s.int_val = in.int_val;
  s.err = 0;
  ann_cs = st.ann_checksum;
  return 0;
}

// lane -> state, after a flush that left s.k <= 7 words in the tile
template <bool INT_OPT>
__device__ __forceinline__ void enc_state_save(m3tsz_encoder_state &st, const EncLane &s, const uint32_t *tile,
                                               int lane, uint64_t ann_cs) {
  EncStateInternal &in = *reinterpret_cast<EncStateInternal *>(st.internal);
  for (uint32_t i = 0; i < 7; i++) in.left[i] = i < s.k ? tile[i * ENC_STRIDE + lane] : 0u;
  in.carry = s.carry;
  in.prev_delta = s.prev_delta;
  in.prev_bits = s.prev_bits;
  in.int_val = s.int_val;
  in.meta = (uint64_t)s.sh | ((uint64_t)s.k << 5) | ((uint64_t)s.plz << 8) | ((uint64_t)s.ptz << 15) |
            ((uint64_t)s.unit << 22) | ((uint64_t)s.num_sig << 26) | ((uint64_t)s.hi_lower_sig << 33) |
            ((uint64_t)s.n_lower_sig << 40) | ((uint64_t)s.max_mult << 43) | ((uint64_t)s.is_float << 46) |
            (enc_state_tag(INT_OPT) << 48);
  st.num_encoded = s.n_enc;
  st.last_ts = s.prev_time;
  // LastEncoded().Value (encoder.go:305-319), as the batch encoder's d_last_value
  st.last_value = (INT_OPT && s.is_float) ? __longlong_as_double((long long)s.prev_bits) : (INT_OPT ? s.int_val : 0.0);
  st.ann_checksum = ann_cs;
  st.bits = ((uint64_t)s.words_out + s.k) * 32ull + s.sh;
}

// The checks encode_time makes on a datapoint (timestamp_encoder.go:104-164), made before anything of it is
// written: append mode drops a failing datapoint as a whole, annotation included.
__device__ __forceinline__ int enc_check_time(const EncLane &s, int64_t t, int u) {
  if (!unit_is_valid(u)) return M3TSZ_ERR_UNRECOGNIZED_UNIT;
  if (u != s.unit || u > 2) return 0;  // a unit change writes a 64-bit delta-of-delta; us / ns have 64-bit buckets
  const int64_t delta = (int64_t)((uint64_t)t - (uint64_t)s.prev_time);
  const int64_t dod = div_unit((int64_t)((uint64_t)delta - (uint64_t)s.prev_delta), u);
  return dod != (int64_t)(int32_t)dod ? M3TSZ_ERR_DOD_OVERFLOW : 0;
}

// Stream()'s tail at the committed position (scheme.go:198-211): the leftover words, the partial word with the
// end-of-stream marker, zero words up to a whole 16-byte group.  Fills w (big-endian word values) and returns the
// number of words (0, 4, 8 or 12) that go to the slot from word `at` on (the committed words_out).
__host__ __device__ __forceinline__ uint32_t enc_snapshot_words(const m3tsz_encoder_state &st, uint32_t w[12],
                                                                uint64_t &at) {
  if (st.num_encoded == 0) return 0;
  const EncStateInternal &in = *reinterpret_cast<const EncStateInternal *>(st.internal);
  const uint32_t sh = (uint32_t)(in.meta & 31u), k = (uint32_t)((in.meta >> 5) & 7u);
  at = (st.bits >> 5) - k;
  uint32_t n = 0;
  for (; n < k; n++) w[n] = in.left[n];
  const uint64_t eos = (uint64_t)((kMarkerOpcode << 2) | (uint32_t)kMarkerEOS) << (64 - kMarkerBits);
  const uint64_t acc = ((uint64_t)in.carry << 32) | (eos >> sh);
  w[n++] = (uint32_t)(acc >> 32);
  if (sh + kMarkerBits > 32) w[n++] = (uint32_t)acc;
  while (n & 3u) w[n++] = 0u;
  return n;
}

// ---- bucket writes: routing (DESIGN.md §4.11) ------------------------------------------------------------------
// What the router keeps of one encoder of a bucket during a call: lastWriteAt, what enc_check_time reads, the
// LastEncoded value and annotation checksum as of the call's start, and an upper bound of the stream's bits.
struct RouteEnc {
  int64_t lw;  // lastWriteAt (buffer.go:1228-1231): 0 before the first write
  int64_t prev_time, prev_delta;
  double last_value;
  uint64_t ann_cs;
  uint64_t bits;  // >= the bits the append will have written, the first datapoint's 64-bit start included
  uint64_t n_enc;
  int unit;
  int32_t rec;      // pool record, -1 for encoder 0
  uint32_t n_call;  // datapoints of this call routed to it
};

__device__ __forceinline__ void route_enc_load(const m3tsz_encoder_state &st, RouteEnc &r, int32_t rec) {
  const EncStateInternal &in = *reinterpret_cast<const EncStateInternal *>(st.internal);
  r.n_enc = st.num_encoded;
  r.lw = r.n_enc ? st.last_ts : 0;
  r.prev_time = r.n_enc ? st.last_ts : st.start_ns;
  r.prev_delta = in.prev_delta;
  r.unit = (int)((in.meta >> 22) & 15u);
  r.last_value = st.last_value;
  r.ann_cs = st.ann_checksum;
  r.bits = st.bits + (r.n_enc ? 0u : 64u);
  r.rec = rec;
  r.n_call = 0;
}

// datapoint j of series s in the inputs' layout
__device__ __forceinline__ uint64_t route_at(const RouteParams &p, uint64_t s, uint32_t j) {
  return p.point_major ? (uint64_t)j * p.n_series + s : s * p.points_stride + j;
}

// LastEncoded().Value of encoder `enc` after the datapoints of this call routed to it before datapoint j_end: its
// state as of the call's start, then the encoder's own value step for each of them (the time step does not touch
// the value state).  Only int-optimised mode needs it: without, the value is always 0.
template <bool INT_OPT>
__device__ __noinline__ double route_last_value(const RouteParams &p, const m3tsz_encoder_state &st, uint64_t s,
                                                uint32_t j_end, int enc, uint32_t *tile, int lane) {
  EncLane e;
  uint64_t cs;
  enc_state_load<INT_OPT>(st, e, tile, lane, cs);
  for (uint32_t j = 0; j < j_end; j++) {
    const uint64_t at = route_at(p, s, j);
    if (p.target[at] != (uint8_t)enc) continue;
    uint32_t hdr = 0;
    int hb = 0, plen;
    uint64_t payload;
    encode_value<INT_OPT>(e, p.val[at], hdr, hb, payload, plen);
    e.n_enc++;
  }
  return e.is_float ? __longlong_as_double((long long)e.prev_bits) : e.int_val;
}

// BufferBucket.write for every datapoint of series s in call order (buffer.go:1261-1364): the target of each
// datapoint (p.target), its result (p.result) and the series' status; opens pool records and lists the ones that
// take datapoints in p.touched.  `tile` is a 7-row column of shared memory for enc_state_load's leftover words.
template <bool INT_OPT>
__device__ __forceinline__ void route_series(const RouteParams &p, uint64_t s, uint32_t *tile, int lane) {
  const uint32_t n = p.n_points ? p.n_points[s] : (uint32_t)p.points_stride;
  if (n == 0) {
    p.status[s] = M3TSZ_OK;
    return;
  }
  const m3tsz_encoder_state &st0 = p.state[s];
  if (n > p.points_stride ||
      (reinterpret_cast<const EncStateInternal *>(st0.internal)->meta >> 48) != enc_state_tag(INT_OPT)) {
    p.status[s] = M3TSZ_ERR_INVALID_ARG;
    return;
  }
  RouteEnc r0;
  route_enc_load(st0, r0, -1);
  const int64_t start = st0.start_ns;
  RouteEnc ro[M3TSZ_MAX_BUCKET_ENCODERS - 1];
  int n_open = 0;  // encoders open, 0 until the overflow encoders are loaded (in-order traffic never needs them)
  int32_t *row = p.table + s * (uint64_t)(p.n_encoders - 1);
  uint64_t ann_i = 0, ann_end = 0;
  if (p.ann_series_off) {
    ann_i = p.ann_series_off[s];
    ann_end = p.ann_series_off[s + 1];
  }
  int32_t status = M3TSZ_OK;
  for (uint32_t j = 0; j < n; j++) {
    const uint64_t at = route_at(p, s, j);
    const uint8_t *a_ptr = nullptr;
    uint32_t a_len = 0;
    if (ann_i < ann_end && p.ann_entries[ann_i].dp_index == j) {
      a_ptr = p.ann_bytes + p.ann_entries[ann_i].byte_offset;
      a_len = p.ann_entries[ann_i].length;
      ann_i++;
    }
    int res = M3TSZ_ERR_CAPACITY;
    int tgt = 0xff;
    if (status == M3TSZ_OK) {
      const int64_t t = p.ts[at];
      const double v = p.val[at];
      const int u = p.units ? (int)p.units[at] : p.unit;
      // the append's room check for this datapoint: its worst case, its annotation and a snapshot's tail
      const uint64_t ann_words = a_len ? (a_len + 3) / 4 + 4 : 0;
      bool have_cs = false;
      uint64_t cs = 0;
      auto ann_cs = [&]() {
        if (!have_cs) cs = xxh64(a_ptr, a_len);
        have_cs = true;
        return cs;
      };
      // 0: go on with the next encoder, 1: write here, 2: unchanged, 3: LastEncoded failed
      auto scan = [&](const RouteEnc &r, int i) {
        if (t == r.lw) {
          if (r.n_enc == 0) return 3;
          double lv = r.last_value;
          if (INT_OPT && r.n_call)
            lv = route_last_value<INT_OPT>(p, i ? p.pool_state[r.rec] : st0, s, j, i, tile, lane);
          return (lv == v && r.ann_cs == ann_cs()) ? 2 : 0;
        }
        return t > r.lw ? 1 : 0;
      };
      // the write's checks, made before it is committed: the encoder's time checks, then room in its slot
      auto check = [&](const RouteEnc &r, uint64_t slot_words) {
        EncLane e;
        e.unit = r.unit;
        e.prev_time = r.prev_time;
        e.prev_delta = r.prev_delta;
        const int err = enc_check_time(e, t, u);
        if (err) return err;
        return (r.bits >> 5) + ENC_GUARD + 4 + ann_words > slot_words ? (int)M3TSZ_ERR_CAPACITY : 0;
      };
      // encode_time's state update, and the datapoint's worst case: a unit change writes a marker and a 64-bit
      // delta-of-delta (83 bits), else at most '1111' + 64 bits; the value at most 80 bits
      auto commit = [&](RouteEnc &r) {
        const int64_t delta = (int64_t)((uint64_t)t - (uint64_t)r.prev_time);
        r.bits += (u != r.unit ? 83u : 68u) + 80u + 32u * ann_words;
        if (u != r.unit) {
          r.unit = u;
          r.prev_delta = 0;
        } else {
          r.prev_delta = delta;
        }
        r.prev_time = t;
        r.lw = t;
        r.n_enc++;
        r.n_call++;
        if (a_len) r.ann_cs = ann_cs();
      };
      int k = scan(r0, 0), hit = k == 1 ? 0 : -1;
      if (k == 0) {
        if (n_open == 0) {
          n_open = 1;
          for (; n_open < p.n_encoders && row[n_open - 1] >= 0; n_open++)
            route_enc_load(p.pool_state[row[n_open - 1]], ro[n_open - 1], row[n_open - 1]);
        }
        for (int i = 1; i < n_open && k == 0; i++) {
          k = scan(ro[i - 1], i);
          if (k == 1) hit = i;
        }
      }
      if (k == 2) {
        res = -1;
      } else if (k == 3) {
        res = M3TSZ_ERR_NO_DATAPOINTS;
      } else if (hit == 0) {
        res = check(r0, p.slot_words);
        if (res == 0) commit(r0);
      } else if (hit > 0) {
        res = check(ro[hit - 1], p.pool_slot_words);
        if (res == 0) commit(ro[hit - 1]);
      } else if (n_open >= p.n_encoders) {
        res = M3TSZ_ERR_TOO_MANY_ENCODERS;
      } else {
        // a new encoder: Reset(block start), opened only once its first write is known to succeed
        RouteEnc &r = ro[n_open - 1];
        m3tsz_encoder_state fresh;
        enc_state_reset(fresh, start, p.default_unit, INT_OPT);
        route_enc_load(fresh, r, -1);
        res = check(r, p.pool_slot_words);
        if (res == 0) {
          const uint32_t rec = atomicAdd(p.pool_count, 1u);
          if (rec >= p.pool_capacity) {
            atomicSub(p.pool_count, 1u);
            res = M3TSZ_ERR_CAPACITY;
          } else {
            p.pool_state[rec] = fresh;
            row[n_open - 1] = (int32_t)rec;
            r.rec = (int32_t)rec;
            commit(r);
            hit = n_open++;
          }
        }
      }
      if (res == 0) tgt = hit;
      if (res == M3TSZ_ERR_CAPACITY) status = M3TSZ_ERR_CAPACITY;
    }
    p.target[at] = (uint8_t)tgt;
    p.result[at] = (int8_t)res;
  }
  p.status[s] = status;
  uint32_t n_touched = 0;
  for (int i = 1; i < n_open; i++) n_touched += ro[i - 1].n_call ? 1u : 0u;
  if (n_touched) {
    uint32_t k = atomicAdd(p.n_touched, n_touched);
    for (int i = 1; i < n_open; i++)
      if (ro[i - 1].n_call) p.touched[k++] = RouteTouched{(uint32_t)ro[i - 1].rec, (uint32_t)s, (uint32_t)i, 0u};
  }
}

__device__ __forceinline__ uint32_t enc_smem_addr(const void *p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void enc_cp_async8(uint32_t dst, const void *src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(dst), "l"(src) : "memory");
}
// ---- TMA tensor copies + mbarrier (point-major input stage) ----
__device__ __forceinline__ void enc_mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void enc_mbar_init_fence() {
  // make the initialised barriers visible to the async proxy (the tensor copies' complete_tx)
  asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
}
__device__ __forceinline__ void enc_mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(bar), "r"(bytes) : "memory");
}
// one box of a 2-D tensor (tensor map in param space) -> shared memory; c0 = innermost coordinate
__device__ __forceinline__ void enc_tma_2d(uint32_t dst, const CUtensorMap *tm, int c0, int c1, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];\n" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void enc_mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n"
      "ENC_MBAR_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra ENC_MBAR_DONE;\n\t"
      "bra ENC_MBAR_WAIT;\n"
      "ENC_MBAR_DONE:\n\t}"
      ::"r"(bar), "r"(parity)
      : "memory");
}

// ---------------------------------------------------------------------------
// the aggregator's transformations on a window's value (DESIGN.md §4.8, GenericElem.processValue,
// src/aggregator/aggregator/generic_elem.go:830-889), run by the lane that owns the series
// ---------------------------------------------------------------------------
constexpr uint64_t kXfEmptyNaN = 0x7FF8000000000001ull;  // emptyDatapoint's value: Go's math.NaN()
constexpr uint64_t kXfOpNaN = 0xFFF8000000000000ull;     // amd64's default NaN of an invalid operation (Inf - Inf)

__device__ __forceinline__ bool xf_isnan(double x) { return x != x; }
__device__ __forceinline__ double xf_bits(uint64_t b) { return __longlong_as_double((long long)b); }

// perSecond, metrics/transformation/binary.go:49-60.  Neither input is NaN past the first test, so the only NaN the
// arithmetic makes is Inf - Inf; `diff < 0` is false for it and the rest carries it.
__device__ __forceinline__ double xf_per_second(int64_t pt, double pv, int64_t t, double v) {
  if (pt >= t || xf_isnan(pv) || xf_isnan(v)) return xf_bits(kXfEmptyNaN);
  const double diff = __dsub_rn(v, pv);
  if (xf_isnan(diff)) return xf_bits(kXfOpNaN);
  if (diff < 0) return xf_bits(kXfEmptyNaN);
  const int64_t dt = (int64_t)((uint64_t)t - (uint64_t)pt);
  return __ddiv_rn(__dmul_rn(diff, 1e9), __ll2double_rn(dt));
}

// increase, binary.go:66-88
__device__ __forceinline__ double xf_increase(int64_t pt, double pv, int64_t t, double v) {
  if (pt >= t || xf_isnan(v)) return xf_bits(kXfEmptyNaN);
  const double diff = __dsub_rn(v, xf_isnan(pv) ? 0.0 : pv);
  if (xf_isnan(diff)) return xf_bits(kXfOpNaN);
  return diff < 0 ? xf_bits(kXfEmptyNaN) : diff;
}

// One non-empty window (end t, value v) through the op list `ops` (op k in bits 4k .. 4k + 3, 0 ends the list).
// Updates st (the binary op's previous window, the Add sums) and v; extra_t = the Reset datapoint's timestamp, 0 for
// none (a Reset datapoint at 0 is not written either, generic_elem.go:920).  The loop is unrolled, so st.sum[k] has
// a fixed offset.
__device__ __forceinline__ void xf_window(uint32_t ops, int64_t step, m3tsz_transform_state &st, int64_t t,
                                          double &v, int64_t &extra_t) {
  extra_t = 0;
#pragma unroll
  for (int k = 0; k < M3TSZ_MAX_TRANSFORMS; k++) {
    const uint32_t op = (ops >> (4 * k)) & 0xfu;
    if (op == 0) break;
    if (op == M3TSZ_TRANSFORM_ABSOLUTE) {  // math.Abs, unary.go:35-40
      v = xf_bits((uint64_t)__double_as_longlong(v) & 0x7FFFFFFFFFFFFFFFull);
    } else if (op == M3TSZ_TRANSFORM_ADD) {  // unary.go:46-54: curr += v unless v is NaN
      if (!xf_isnan(v)) {
        const double a = st.sum[k];
        double r = __dadd_rn(a, v);
        // amd64 ADDSD keeps a NaN operand's payload (quieted); only `a` can be one here.  Inf + -Inf: default NaN
        if (xf_isnan(r))
          r = xf_isnan(a) ? xf_bits((uint64_t)__double_as_longlong(a) | 0x0008000000000000ull) : xf_bits(kXfOpNaN);
        st.sum[k] = r;
      }
      v = st.sum[k];
    } else if (op == M3TSZ_TRANSFORM_PERSECOND || op == M3TSZ_TRANSFORM_INCREASE) {
      // prev = the previous non-empty window's input to this op (consumedValues), (0, NaN) without one
      const int64_t pt = st.has_prev ? st.prev_t : 0;
      const double pv = st.has_prev ? st.prev_v : xf_bits(kXfEmptyNaN);
      const double in = v;
      v = op == M3TSZ_TRANSFORM_PERSECOND ? xf_per_second(pt, pv, t, in) : xf_increase(pt, pv, t, in);
      st.has_prev = 1;
      st.prev_t = t;
      st.prev_v = in;
    } else if (op == M3TSZ_TRANSFORM_RESET) {  // unary_multi.go:46-54: int64(math.Max(float64(step / 2), 1))
      const int64_t rw = (int64_t)__double2ll_rz(fmax(__ll2double_rn(step / 2), 1.0));
      extra_t = (int64_t)((uint64_t)t + (uint64_t)rw);
    }
  }
}

// One non-empty window (end t) of an element with several aggregation types (generic_elem.go:830-889, the loop over
// e.aggTypes): types i0 .. i1 - 1 in order each take their value value_of(i) through xf_window, with the element's
// Add sums (e.w.sum: a type adds after the types before it), the previous window as it was before this window (the
// element's has_prev / prev_t) and the type's own binary-op input e.pv[i] (consumedValues[i]), which the type then
// records.  take(i, v, extra_t) gets each type's result and Reset timestamp.  A lane whose list has an Add op runs
// every type (i0 = 0, i1 = n_types) to keep the sums; without one, a type depends on nothing of the others.
template <class ValueOf, class Take>
__device__ __forceinline__ void xf_element_window(uint32_t ops, int64_t step, XfElem &e, uint32_t i0, uint32_t i1,
                                                  int64_t t, ValueOf value_of, Take take) {
  const int32_t has_prev = e.w.has_prev;
  const int64_t prev_t = e.w.prev_t;
#pragma unroll 1
  for (uint32_t i = i0; i < i1; i++) {
    double v = value_of(i);
    int64_t extra_t = 0;
    e.w.has_prev = has_prev;
    e.w.prev_t = prev_t;
    e.w.prev_v = e.pv[i];
    xf_window(ops, step, e.w, t, v, extra_t);
    e.pv[i] = e.w.prev_v;
    take(i, v, extra_t);
  }
}

// The window value of the tile stages (IN = 2 / 4 / 5): ValueOf(agg) of window-major element o with count c.  The
// switches are uniform across a warp, except in an IN = 5 warp whose 32 rows straddle two types.
__device__ __forceinline__ double tile_value_of(const EncodeParams &p, bool counter, int agg, uint64_t o, int64_t c) {
  double v = 0.0;
  if (counter) {
    // Counter.ValueOf, counter.go:112-134: float64() of the int64 aggregates (uniform switch)
    switch (agg) {
      case M3TSZ_AGG_MIN: v = __ll2double_rn(__ldg(p.tile_imin + o)); break;
      case M3TSZ_AGG_MAX: v = __ll2double_rn(__ldg(p.tile_imax + o)); break;
      case M3TSZ_AGG_MEAN:
        v = c == 0 ? 0.0 : __ddiv_rn(__ll2double_rn(__ldg(p.tile_isum + o)), __ll2double_rn(c));
        break;
      case M3TSZ_AGG_COUNT: v = __ll2double_rn(c); break;
      case M3TSZ_AGG_SUM: v = __ll2double_rn(__ldg(p.tile_isum + o)); break;
      case M3TSZ_AGG_SUMSQ: v = __ll2double_rn(__ldg(static_cast<const int64_t *>(p.tile_sum_sq) + o)); break;
      case M3TSZ_AGG_STDEV:
        v = agg_stdev(c, __ll2double_rn(__ldg(static_cast<const int64_t *>(p.tile_sum_sq) + o)),
                      __ll2double_rn(__ldg(p.tile_isum + o)));
        break;
      default: break;
    }
  } else {
    switch (agg) {  // Gauge.ValueOf, gauge.go:144-165 (uniform switch)
      case M3TSZ_AGG_LAST: v = __ldg(p.tile_last + o); break;
      case M3TSZ_AGG_MIN: v = __ldg(p.tile_min + o); break;
      case M3TSZ_AGG_MAX: v = __ldg(p.tile_max + o); break;
      case M3TSZ_AGG_MEAN: v = c == 0 ? 0.0 : __ddiv_rn(__ldg(p.tile_sum + o), __ll2double_rn(c)); break;
      case M3TSZ_AGG_COUNT: v = __ll2double_rn(c); break;
      case M3TSZ_AGG_SUM: v = __ldg(p.tile_sum + o); break;
      case M3TSZ_AGG_SUMSQ: v = __ldg(static_cast<const double *>(p.tile_sum_sq) + o); break;
      case M3TSZ_AGG_STDEV:
        v = agg_stdev(c, __ldg(static_cast<const double *>(p.tile_sum_sq) + o), __ldg(p.tile_sum + o));
        break;
      default: break;
    }
  }
  return v;
}

// PACKED = false: one warp per 32-series batch, every series writes its own slot
//   p.out + s * p.out_stride (fixed stride).
// PACKED = true : persistent warps fetch batches from a counter, encode into a per-warp
//   scratch slot set (reused batch after batch), then allocate exact space in the packed
//   buffer with ONE atomicAdd per batch (sum of the 32 aligned lengths) and copy their
//   streams there with coalesced 16-byte loads/stores -- the separate compaction pass
//   (scan + gather over all bytes) and the [S][stride] slot buffer disappear; the copies
//   of finished warps overlap the bit packing of the others.  Streams land in completion
//   order: p.packed_off[s] / p.out_len[s] are the index entry (Offset, Size) of stream s
//   (persist/schema/types.go:70-78).
// IN = 0: series-major inputs ts/val[S][stride], staged through transposed shared-memory tiles;
// IN = 1: point-major inputs ts/val[stride][S]: the same tiles, filled lane-locally (a tile row is 32
//         consecutive elements of the array: coalesced sources, no shuffles).  Direct LDG.64 with two rows
//         in flight was slower: the loads' latency is exposed;
// IN = 2: the Gauge aggregates of the fused decode+downsample kernel (window-major): datapoint i of a
//         series = (tile_start + (i+1)*tile_step, Gauge.ValueOf(agg)) unless window i is empty
//         (count == 0: skipped) -- the tile aggregation's re-encode without a gather pass.
// IN = 4: IN = 2 with the aggregator's transformations (xf_window, p.xf_ops): the lane runs each non-empty window's
//         value through the op list as it loads the row, and skips a NaN result when p.xf_discard_nan is set.
//         With a Reset op a window takes two rows: 2i its datapoint, 2i + 1 the Reset datapoint (or skipped).  The
//         prologue loads the series' p.xf_state record (zeros without one), the epilogue saves it when the
//         series' status is OK.
// IN = 5: IN = 4 for an element's several aggregation types (xf_element_window): lane row r is source series
//         r % p.tile_n_src under type r / p.tile_n_src; with an Add op the lane runs every type of the window to
//         keep the shared sums and writes its own.  The prologue loads the series' p.xf_elem record, the epilogue
//         writes the lane's part of the new one to p.xf_elem_out (launch_tiles_types_status commits it).
// APPEND: encoder-set append (DESIGN.md §4.6).  Every lane continues the open encoder p.state[s] in slot p.out +
//   s * out_stride: the prologue loads the state (leftover words into the output tile), each datapoint is checked
//   before anything of it is written, and the epilogue flushes whole sectors and saves the state instead of
//   writing the tail.
template <bool INT_OPT, bool PACKED, int IN, bool APPEND = false>
__global__ void __launch_bounds__(ENC_WARPS * 32,
                                  IN >= 2 ? ENC_MIN_BLOCKS_AGG : (IN == 1 ? ENC_MIN_BLOCKS_PM : ENC_MIN_BLOCKS))
    encode_kernel(const EncodeParams p, const __grid_constant__ EncTensorMaps tmaps) {
  static_assert(!APPEND || (!PACKED && IN != 2 && IN != 4 && IN != 5 && IN != 6 && IN != 7),
                "append mode writes its own slots from staged inputs");
  // the tile aggregation's re-encode (IN = 4: with transformations, IN = 5: an element's several types)
  constexpr bool TILES = IN == 2 || IN == 4 || IN == 5 || IN == 6 || IN == 7;
  // IN = 6: IN = 5 that writes each window's annotation (p.tile_ann), read from the source streams; IN = 7: the same
  // over several source blocks per series, whose references hold the payload's bit offset in the whole batch
  constexpr bool ELEM = IN == 5 || IN == 6 || IN == 7, TANN = IN == 6 || IN == 7, TBLK = IN == 7;
  static_assert(IN != 3 || APPEND, "the routed input stage continues open encoders");
  extern __shared__ __align__(128) uint32_t smem[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  // the direct input stages (IN != 0) need no input tiles: only the output tile lives in shared memory
  constexpr bool STAGED = (IN == 0 || IN == 1);  // inputs go through the shared-memory tiles
  constexpr int IN_T = enc_in_t<IN>();  // datapoints per input tile
  static_assert((IN_T & (IN_T - 1)) == 0, "tile rows must be a power of two");
  constexpr uint32_t NSTAGE = (uint32_t)enc_nstage<IN>();  // input tiles in flight (ring of buffers)
  constexpr int IN_STRIDE = enc_in_stride<IN>();  // cells per tile row
  constexpr int IN_TILE_DW = IN_T * IN_STRIDE;  // one array (ts or val), one buffer
  constexpr bool BULK = enc_bulk<IN>();  // one 2-D tensor copy per array and tile where the arrays allow it
  // the point-major batch stage checks the hot tier's slow-changing preconditions once per input tile (below)
  constexpr bool GROUPS = IN == 1 && !APPEND;
  constexpr size_t WARP_SMEM = enc_warp_smem<IN>();
  uint8_t *wbase = reinterpret_cast<uint8_t *>(smem) + warp * WARP_SMEM;
  // in_tiles: [buffer][array (0 ts, 1 val)][row][lane]
  uint64_t *in_tiles = reinterpret_cast<uint64_t *>(wbase);
  uint32_t *out_tile = STAGED ? reinterpret_cast<uint32_t *>(in_tiles + 2 * NSTAGE * IN_TILE_DW)
                              : reinterpret_cast<uint32_t *>(wbase);

  // BULK: one mbarrier per tile buffer behind the output tile; `bulk_seq` counts the tiles this warp has requested
  // through them (buffer = seq % NSTAGE, phase parity = (seq / NSTAGE) & 1), across batches
  const uint32_t mbar0 = BULK ? enc_smem_addr(out_tile + ENC_OUT_TILE_WORDS) : 0u;
  uint32_t bulk_seq = 0;
  // the tiles come by tensor copy (they zero-fill what is out of range, so they serve every batch) unless the
  // host could not describe the arrays
  const bool bulk = BULK && tmaps.ok != 0;
  if (BULK) {
    if (lane == 0) {
      for (uint32_t b = 0; b < NSTAGE; b++) enc_mbar_init(mbar0 + 8u * b, 1);
      enc_mbar_init_fence();
    }
    __syncwarp();
  }

  const uint64_t n_batches = (p.n_series + 31) >> 5;
  const uint64_t warp_slot = (uint64_t)blockIdx.x * ENC_WARPS + warp;  // PACKED: scratch slot set
  for (uint64_t batch_iter = 0;; batch_iter++) {
  uint64_t batch;
  if (PACKED) {
    unsigned long long b = 0;
    if (lane == 0) b = atomicAdd(p.batch_counter, 1ull);
    batch = __shfl_sync(FULL_MASK, b, 0);
  } else if (IN == 3) {
    // grid-stride: the overflow pass launches a bounded grid over as many lanes as records could have been touched,
    // and a warp stops at its first batch past the touched ones (below)
    batch = warp_slot + batch_iter * ((uint64_t)gridDim.x * ENC_WARPS);
  } else {
    if (batch_iter) break;
    batch = warp_slot;
  }
  if (batch >= n_batches) break;
  const uint64_t warp_s0 = batch * 32ull;
  const uint64_t sidx = warp_s0 + lane;
  const bool valid = sidx < p.n_series && (IN != 3 || !p.route_touched || sidx < *p.route_n_touched);
  // the lane's input series and encoder record, and (IN = 3) the encoder index whose datapoints it takes
  uint64_t in_s = sidx, rec = sidx;
  uint32_t lane_enc = 0;
  if constexpr (IN == 3) {
    if (p.route_touched && !__any_sync(FULL_MASK, valid)) break;  // (overflow pass: past the touched records)
    if (p.route_touched && valid) {
      const RouteTouched e = p.route_touched[sidx];
      rec = e.rec;
      in_s = e.series;
      lane_enc = e.enc;
    }
  }

  EncLane s;
  s.carry = 0;
  s.sh = 0;
  s.k = 0;
  s.words_out = 0;
  s.prev_time = 0;
  s.prev_delta = 0;
  s.prev_bits = 0;
  s.plz = 64;
  s.ptz = 0;
  s.int_val = 0.0;
  s.unit = 0;
  s.num_sig = 0;
  s.hi_lower_sig = 0;
  s.n_lower_sig = 0;
  s.max_mult = 0;
  s.err = 0;
  s.n_enc = 0;
  s.is_float = false;

  uint32_t n_pts = 0;
  uint64_t ann_i = 0, ann_end = 0;
  uint64_t last_ann_off = 0;
  uint32_t last_ann_len = 0;  // 0 = no annotation written yet
  const uint32_t slot_words = (uint32_t)(p.out_stride >> 2);
  // APPEND only (nothing of it exists in the batch instantiations, whose code stays as it was)
  std::conditional_t<APPEND, EncAppendVars, EncNoVars> av;
  // IN = 4 only: the series' transformation state (this lane's slot behind the output tile), and the Reset datapoint
  // of the window loaded last
  bool xf_reset = false;
  m3tsz_transform_state *xs = nullptr;
  int64_t xf_extra_t = 0;
  if constexpr (IN == 4) {
    for (int k = 0; k < M3TSZ_MAX_TRANSFORMS; k++) xf_reset |= ((p.xf_ops >> (4 * k)) & 0xfu) == M3TSZ_TRANSFORM_RESET;
    xs = &(reinterpret_cast<XfSlot *>(wbase + ENC_OUT_TILE_WORDS * 4) + lane)->st;
    if (valid && p.xf_state)
      *xs = p.xf_state[sidx];
    else
      memset(xs, 0, sizeof(*xs));
  }
  // IN = 5 only: the lane's element record, source series and type (its slot behind the output tile)
  XfElemSlot *xe = nullptr;
  if constexpr (ELEM) {
    xe = reinterpret_cast<XfElemSlot *>(wbase + ENC_OUT_TILE_WORDS * 4) + lane;
    bool all = false;
    for (int k = 0; k < M3TSZ_MAX_TRANSFORMS; k++) {
      const uint32_t op = (p.xf_ops >> (4 * k)) & 0xfu;
      xf_reset |= op == M3TSZ_TRANSFORM_RESET;
      all |= op == M3TSZ_TRANSFORM_ADD;
    }
    uint32_t ty = 0;
    uint64_t src = sidx;
    if (valid) {
      ty = (uint32_t)(sidx / p.tile_n_src);
      src = sidx - (uint64_t)ty * p.tile_n_src;
    }
    if (valid && p.xf_elem) {
      const m3tsz_element_state &r = p.xf_elem[src];
      xe->e.w = r.head;
      xe->e.pv[0] = r.head.prev_v;
      for (int j = 1; j < M3TSZ_MAX_ELEMENT_TYPES; j++) xe->e.pv[j] = r.prev_v_more[j - 1];
      xe->reserved = r.reserved;
    } else {
      memset(xe, 0, sizeof(*xe));
    }
    xe->src = src;
    xe->ty = ty;
    xe->all = all ? 1u : 0u;
  }
  if constexpr (APPEND) {
    if (valid) {
      n_pts = p.n_points ? p.n_points[in_s] : (uint32_t)p.points_stride;
      if (n_pts > p.points_stride) s.err = M3TSZ_ERR_INVALID_ARG;
      if (p.ann_series_off) {
        ann_i = p.ann_series_off[in_s];
        ann_end = p.ann_series_off[in_s + 1];
      }
      // a series without datapoints (or with bad arguments) loads nothing and keeps its state and slot
      if (n_pts > 0 && s.err == 0) s.err = enc_state_load<INT_OPT>(p.state[rec], s, out_tile, lane, av.ann_cs);
      if (s.err) n_pts = 0;
      av.n_enc0 = s.n_enc;
      if (n_pts > 0 && s.n_enc == 0) put64(s, out_tile, lane, (uint64_t)s.prev_time, 64);  // WriteFirstTime :89-102
    }
  } else if (valid) {
    n_pts = (!TILES && p.n_points) ? p.n_points[sidx] : (uint32_t)p.points_stride;
    // failed source stream: no tiles
    if constexpr (ELEM) {
      if (p.tile_src_status && p.tile_src_status[xe->src] != 0) n_pts = 0;
    } else if (TILES && p.tile_src_status && p.tile_src_status[sidx] != 0) {
      n_pts = 0;
    }
    if (n_pts > p.points_stride) {
      s.err = M3TSZ_ERR_INVALID_ARG;
      n_pts = 0;
    }
    if ((IN == 4 || ELEM) && xf_reset) n_pts *= 2;  // two rows per window
    const int64_t start = p.start[sidx];
    s.prev_time = start;
    s.unit = initial_time_unit(start, p.default_unit);  // encoder.reset :268-272
    if (p.ann_series_off) {
      ann_i = p.ann_series_off[sidx];
      ann_end = p.ann_series_off[sidx + 1];
    }
    if (n_pts > 0 && s.err == 0) {
      if (slot_words < (uint32_t)ENC_GUARD + 4u) {
        s.err = M3TSZ_ERR_CAPACITY;
      } else {
        put64(s, out_tile, lane, (uint64_t)start, 64);  // WriteFirstTime :89-102
      }
    }
  }
  const uint32_t max_pts = __reduce_max_sync(FULL_MASK, n_pts);

  // Paired flush: every lane decides how many 16-byte groups of ITS OWN column leave the tile (the complete 32-byte
  // sectors, keeping the <= 7 leftover words; the last flush also writes the final 16-byte group, which the tail
  // pads the stream to), and lanes l and l ^ 4 write their two columns together: first column A = l & ~4, then
  // column B = l | 4, one sector per round, the lane with bit 2 clear writing its first half and the other lane its
  // second half (big-endian byte order).  So a store instruction writes 16 whole sectors, where one 16-byte group
  // per lane left 32 half-written ones, and a flush takes no more rounds than its fullest column has groups
  // (ceil(gA / 2) + ceil(gB / 2) per pair).  Tile reads: in lockstep, the lanes of a round read rows 4q + i of
  // columns whose bit 2 is clear (A) or set (B), with q even for one lane of a pair and odd for the other, so the
  // banks (4q + i + column) % 32 are distinct.  The sectors are whole in memory when out_stride is a multiple of 32
  // bytes, as the bench's is.
  uint8_t *my_out = PACKED ? p.out + (warp_slot * 32ull + (uint64_t)lane) * p.out_stride
                           : p.out + rec * p.out_stride;
  const uint32_t par = (lane >> 2) & 1u;  // 0: this lane's column is its pair's column A, 1: column B
  // the partner's slot (lane l ^ 4 is 4 slots away in both output modes; the overflow records of IN = 3 lie anywhere)
  uint8_t *o_out = par ? my_out - 4ull * p.out_stride : my_out + 4ull * p.out_stride;
  if constexpr (IN == 3)
    o_out = reinterpret_cast<uint8_t *>(__shfl_xor_sync(FULL_MASK, reinterpret_cast<unsigned long long>(my_out), 4));
  auto flush_out = [&](bool last) {
    __syncwarp();
    const uint32_t grp = last ? s.k >> 2 : (s.k >> 3) << 1;  // 16-byte groups of this lane's column (<= 7)
    // every flush before the last moves whole sectors, so words_out is a multiple of 8 here and its low 3 bits
    // can carry grp: one shuffle tells a lane where its partner's stream stands and how much it writes
    const uint32_t wg_o = __shfl_xor_sync(FULL_MASK, s.words_out | grp, 4);
    const uint32_t grp_o = wg_o & 7u;
    uint8_t *const d_me = my_out + (uint64_t)s.words_out * 4ull;
    uint8_t *const d_o = o_out + (uint64_t)(wg_o & ~7u) * 4ull;
    const uint32_t gA = par ? grp_o : grp, gB = par ? grp : grp_o;
    const uint32_t nA = (gA + 1) >> 1;  // rounds of column A
    const uint32_t rounds = __reduce_max_sync(FULL_MASK, nA + ((gB + 1) >> 1));
    for (uint32_t r = 0; r < rounds; r++) {
      const bool in_a = r < nA;
      const uint32_t q = 2 * (in_a ? r : r - nA) + par;  // group of the column this round writes
      if (q < (in_a ? gA : gB)) {  // (q <= 6: rows 4q .. 4q + 3 lie inside the tile)
        const uint32_t *tp = out_tile + (4 * q) * ENC_STRIDE + (in_a ? (lane & ~4u) : (lane | 4u));
        uint4 v;
        v.x = __byte_perm(tp[0], 0, 0x0123);
        v.y = __byte_perm(tp[ENC_STRIDE], 0, 0x0123);
        v.z = __byte_perm(tp[2 * ENC_STRIDE], 0, 0x0123);
        v.w = __byte_perm(tp[3 * ENC_STRIDE], 0, 0x0123);
        *reinterpret_cast<uint4 *>(((in_a == (par == 0)) ? d_me : d_o) + 16ull * q) = v;
      }
    }
    __syncwarp();  // the partner is done reading this lane's column before its leftover moves up
    // move the leftover words to the top of the lane's column: the rows do not overlap, because a flush that
    // writes anything writes at least a sector (done >= 8 > rem), and the last flush leaves nothing
    const uint32_t done = 4 * grp, rem = s.k - done;
    if (done)
      for (uint32_t i = 0; i < rem; i++) out_tile[i * ENC_STRIDE + lane] = out_tile[(done + i) * ENC_STRIDE + lane];
    s.words_out += done;
    s.k = rem;
    __syncwarp();
  };

  // asynchronous staging of input tile `tile` (rows tile*IN_T ..) into buffer (tile_base + tile) % NSTAGE:
  // lanes 0-7 / 8-15: ts / value rows of series 2i, lanes 16-23 / 24-31: of series 2i+1
  const int st_r = lane & (IN_T - 1);
  const int st_arr = (lane >> 3) & 1;
  const int st_jo = lane >> 4;
  const bool uniform_n = __all_sync(FULL_MASK, !valid || n_pts == max_pts) && __all_sync(FULL_MASK, valid);
  const uint32_t tile_base = bulk ? bulk_seq : 0u;  // buffer of tile t: (tile_base + t) % NSTAGE
  auto stage = [&](uint32_t tile) {
    const uint32_t row0 = tile * IN_T;
    if (row0 >= max_pts) return;
    const uint32_t buf = (tile_base + tile) % NSTAGE;
    if (bulk) {
      if (lane == 0) {
        const uint32_t bar = mbar0 + buf * 8u;
        enc_mbar_expect_tx(bar, 2u * (uint32_t)IN_TILE_DW * 8u);  // the whole box counts, in range or not
        const uint32_t d0 = enc_smem_addr(in_tiles + (buf * 2u) * IN_TILE_DW);
        enc_tma_2d(d0, &tmaps.ts, (int)warp_s0, (int)row0, bar);
        enc_tma_2d(d0 + (uint32_t)IN_TILE_DW * 8u, &tmaps.val, (int)warp_s0, (int)row0, bar);
      }
      return;
    }
    if (IN == 1) {
      // point-major inputs: a row of the tile is 32 consecutive elements of the array -- every lane
      // copies its own column (IN_T rows x 2 arrays), sources coalesced across the warp, no shuffles
      const uint64_t *st = reinterpret_cast<const uint64_t *>(p.ts) + (uint64_t)row0 * p.n_series + sidx;
      const uint64_t *sv = reinterpret_cast<const uint64_t *>(p.val) + (uint64_t)row0 * p.n_series + sidx;
      const uint32_t d0 = enc_smem_addr(in_tiles + (buf * 2u) * IN_TILE_DW + lane);
      const uint32_t lim = s.err == 0 ? n_pts : 0u;  // (0 for a lane without a series)
#pragma unroll
      for (int r = 0; r < IN_T; r++) {
        if (row0 + (uint32_t)r < lim) {
          enc_cp_async8(d0 + (uint32_t)(r * IN_STRIDE) * 8u, st);
          enc_cp_async8(d0 + (uint32_t)(IN_TILE_DW + r * IN_STRIDE) * 8u, sv);
        }
        st += p.n_series;
        sv += p.n_series;
      }
      return;
    }
    const uint64_t *src = (st_arr ? reinterpret_cast<const uint64_t *>(p.val)
                                  : reinterpret_cast<const uint64_t *>(p.ts)) +
                          (warp_s0 + st_jo) * p.points_stride + row0 + st_r;
    const uint32_t dst0 = enc_smem_addr(in_tiles + (buf * 2u + (uint32_t)st_arr) * IN_TILE_DW +
                                        st_r * IN_STRIDE + st_jo);
    const uint64_t step = 2ull * p.points_stride;
    if (uniform_n && row0 + IN_T <= max_pts) {
#pragma unroll
      for (int i = 0; i < 16; i++) {
        enc_cp_async8(dst0 + (uint32_t)i * 16u, src);
        src += step;
      }
    } else {
      for (int i = 0; i < 16; i++) {
        const uint32_t nj = __shfl_sync(FULL_MASK, (valid && s.err == 0) ? n_pts : 0u, 2 * i + st_jo);
        if (row0 + (uint32_t)st_r < nj) enc_cp_async8(dst0 + (uint32_t)i * 16u, src);
        src += step;
      }
    }
  };

  if (STAGED) {  // the first NSTAGE - 1 tiles; the loop requests each next one as it starts a tile
    for (uint32_t t = 0; t + 1 < NSTAGE; t++) {
      stage(t);
      if (!bulk) asm volatile("cp.async.commit_group;\n" ::: "memory");
    }
  }
  // direct input stages: element `row` of this lane's series
  auto load_row = [&](uint32_t row, int64_t &t_o, uint64_t &v_o, bool &skip_o) {
    skip_o = false;
    t_o = 0;
    v_o = 0;
    if (!valid || row >= n_pts) return;
    if constexpr (IN == 3) {  // the inputs' own layout (in_mode 1: point-major)
      const uint64_t o = p.in_mode ? (uint64_t)row * p.route_n_in + in_s : in_s * p.points_stride + row;
      t_o = __ldg(p.ts + o);
      v_o = (uint64_t)__double_as_longlong(__ldg(p.val + o));
      return;
    }
    if constexpr (IN == 4 || ELEM) {
      if (xf_reset && (row & 1u)) {  // the Reset datapoint of window row / 2 (0: none, or its window was skipped)
        skip_o = xf_extra_t == 0;
        t_o = xf_extra_t;  // (value +0)
        return;
      }
      if (xf_reset) row >>= 1;
    }
    if constexpr (ELEM) {
      const uint64_t o = (uint64_t)row * p.tile_n_src + xe->src;  // the lane's source series
      const int64_t c = __ldg(p.tile_count + o);
      skip_o = (c == 0);
      t_o = p.tile_start + (int64_t)(row + 1) * p.tile_step;  // the window's end boundary
      double v = 0.0;
      xf_extra_t = 0;
      if (!skip_o) {
        const bool counter = p.metric_type == M3TSZ_METRIC_COUNTER;
        const uint32_t ty = xe->ty;
        xf_element_window(
            p.xf_ops, p.tile_step, xe->e, xe->all ? 0u : ty, xe->all ? p.tile_n_types : ty + 1, t_o,
            [&](uint32_t i) {
              // (o laundered per type: hoisting the eight arrays' addresses out of the loop spilled registers)
              uint64_t oi;
              asm volatile("mov.b64 %0, %1;" : "=l"(oi) : "l"(o));
              return tile_value_of(p, counter, (int)((p.tile_types >> (4 * i)) & 0xfu), oi, c);
            },
            [&](uint32_t i, double r, int64_t extra_t) {
              if (i == ty) {
                v = r;
                xf_extra_t = extra_t;
              }
            });
        if (p.xf_discard_nan && xf_isnan(v)) {  // DiscardNaNAggregatedValues: nothing of this type's window
          skip_o = true;
          xf_extra_t = 0;
        }
      }
      v_o = (uint64_t)__double_as_longlong(v);
    } else if (TILES) {
      const uint64_t o = (uint64_t)row * p.n_series + sidx;
      const int64_t c = __ldg(p.tile_count + o);
      skip_o = (c == 0);
      t_o = p.tile_start + (int64_t)(row + 1) * p.tile_step;  // the window's end boundary
      double v = 0.0;
      v = tile_value_of(p, p.metric_type == M3TSZ_METRIC_COUNTER, p.agg_type, o, c);
      if constexpr (IN == 4) {
        xf_extra_t = 0;
        if (!skip_o) {
          xf_window(p.xf_ops, p.tile_step, *xs, t_o, v, xf_extra_t);
          if (p.xf_discard_nan && xf_isnan(v)) {  // DiscardNaNAggregatedValues: nothing of the window
            skip_o = true;
            xf_extra_t = 0;
          }
        }
      }
      v_o = (uint64_t)__double_as_longlong(v);
    }
  };
  int64_t t_pf1 = 0;
  uint64_t fb_pf1 = 0;
  bool sk_pf = false, sk_pf1 = false;

  int64_t t_pf = 0;
  uint64_t fb_pf = 0;
  if (!STAGED) {  // two rows in flight
    load_row(0, t_pf, fb_pf, sk_pf);
    load_row(1, t_pf1, fb_pf1, sk_pf1);
  }
  bool steady = false;  // same s/ms/us/ns unit as the batch's and not the first datapoint
  bool hot_ok = false;  // steady, and float mode when int-optimised: both only change on the slow path
  if constexpr (APPEND) {  // the loaded encoder's
    steady = !p.units && p.unit == s.unit && (s.unit >= 1 && s.unit <= 4) && s.n_enc > 0;
    hot_ok = steady && (!INT_OPT || s.is_float);
  }
  const uint64_t *in_next = in_tiles + lane;  // this lane's ts cell of the row to fetch next (value: + one tile)

  // ---- input pipeline: request tile t+NSTAGE-1, wait for tile t (the one starting at row `iter`) ----
  auto begin_tile = [&](uint32_t iter) {
    __syncwarp();  // everyone is done reading the buffer about to be overwritten (tile t-1's)
    stage(iter / IN_T + NSTAGE - 1);
    const uint32_t g = tile_base + iter / IN_T;  // (tile_base is 0 unless this batch is bulk-filled)
    const uint32_t buf = g % NSTAGE;
    if (bulk) {
      enc_mbar_wait(mbar0 + buf * 8u, (g / NSTAGE) & 1u);  // every lane: the tile's bytes have landed
    } else {
      asm volatile("cp.async.commit_group;\n" ::: "memory");
      asm volatile("cp.async.wait_group %0;\n" ::"n"(NSTAGE - 1) : "memory");
    }
    __syncwarp();
    // row 0 of the tile that just landed; rows 1..IN_T-1 are fetched one datapoint ahead below
    const uint64_t *tile = in_tiles + (buf * 2u) * IN_TILE_DW + lane;
    t_pf = (int64_t)tile[0];
    fb_pf = tile[IN_TILE_DW];
    in_next = tile + IN_STRIDE;
  };

  // ---- the hot tier's code: '0' (zero DoD) [+ '1' no-update] + XOR code, one merge ----
  // The state update is unconditional (upd) where an inactive lane is a FINISHED lane (IN 0 / 1); with IN = 2 / 4 a
  // lane may sit out one row (an empty window) and must keep its state, and so must every lane in append mode,
  // whose state outlives the call.
  auto hot_commit = [&](int64_t t, uint64_t fb, bool upd, bool emit) {
    if (upd) s.prev_time = t;
    const uint32_t pre = INT_OPT ? 1u : 0u;  // '0' zero DoD [+ '1' no-update]
    const int pb = INT_OPT ? 2 : 1;
    const uint64_t x = s.prev_bits ^ fb;
    int cl, ct;
    lz_tz(x, cl, ct);  // (64, 0) for x == 0
    const bool zero = !INT_OPT && (x == 0);  // int-optimised: a repeat is not a hot datapoint (fb != prev_bits)
    const bool cont = !zero && cl >= s.plz && ct >= s.ptz;
    const int nm = 64 - cl - ct;
    // payload left-aligned: (x >> ptz) << (64 - plen) == x << plz, (x >> ct) << (64 - nm) == x << cl
    const uint64_t P = shl64_clamp(x, (uint32_t)(cont ? s.plz : cl));  // (x == 0: cl = 64 shifts everything out)
    const int plen = zero ? 0 : (cont ? 64 - s.plz - s.ptz : nm);
    const uint32_t hdr = zero ? (pre << 1)
                              : (cont ? ((pre << 2) | 2u)
                                      : ((pre << 14) | (3u << 12) | ((uint32_t)cl << 6) | (uint32_t)(nm - 1)));
    const int hb = pb + (zero ? 1 : (cont ? 2 : 14));
    if (upd) {
      s.plz = cl;  // PrevXOR := x
      s.ptz = ct;
      s.prev_bits = fb;
    }
    if (emit) {
      emit_code_p(s, out_tile, lane, hdr, hb, P, plen);
      s.n_enc++;
    }
  };

  // one datapoint, every tier, with every per-datapoint check (the tile of row `iter` has landed)
  auto row_active = [&](uint32_t iter) {
    return s.err == 0 && iter < n_pts && !(TILES && sk_pf);  // (n_pts is 0 without a series)
  };
  auto encode_row = [&](uint32_t iter, bool tile_last, bool active) {

    // ---- append mode: check the datapoint before any of it (annotation included) is written ----
    if constexpr (APPEND) {
      if constexpr (IN == 3) {
        // only the datapoints routed to this lane's encoder; the annotations of the others are passed over
        if (active) active = p.route_target[p.in_mode ? (uint64_t)iter * p.route_n_in + in_s
                                                      : in_s * p.points_stride + iter] == lane_enc;
        if (p.ann_series_off)
          while (ann_i < ann_end && p.ann_entries[ann_i].dp_index < iter) ann_i++;
      }
      if (active) {
        const int u = p.units ? (int)p.units[in_s * p.points_stride + iter] : p.unit;
        // room for the datapoint's worst case, its annotation (marker + varint + bytes) and a snapshot's tail
        uint64_t need = (uint64_t)s.words_out + s.k + ENC_GUARD + 4;
        if (p.ann_series_off && ann_i < ann_end) {
          const m3tsz_annotation_entry e = p.ann_entries[ann_i];
          if (e.dp_index == iter && e.length > 0) need += (e.length + 3) / 4 + 4;
        }
        s.err = enc_check_time(s, t_pf, u);
        if (s.err == 0 && need > slot_words) s.err = M3TSZ_ERR_CAPACITY;
        active = s.err == 0;
      }
    }

    // ---- make room in the output tile ----
    const bool tight = active && (s.k > (uint32_t)(ENC_OUT_W - ENC_GUARD));
    if (__any_sync(FULL_MASK, tight)) flush_out(false);

    // ---- annotations (warp-cooperative; timestamp_encoder.go:166-195) ----
    bool want_ann = false;
    uint64_t a_off = 0;
    uint32_t a_len = 0;
    // byte i of the annotation at a_off: the annotation inputs' bytes, or (IN = 6) the source stream's, bit-aligned
    // at bit a_off of the batch (inside the source stream, which the decode checked: the next byte is there too
    // whenever the annotation does not start on a byte)
    auto ann_byte = [&](uint64_t off, uint32_t i) -> uint32_t {
      if constexpr (TANN) {
        const uint64_t b = off + 8ull * i;
        const uint32_t sh = (uint32_t)(b & 7u);
        const uint8_t *q = p.tile_src_streams + (b >> 3);
        return sh ? (((uint32_t)q[0] << sh) | ((uint32_t)q[1] >> (8u - sh))) & 0xffu : (uint32_t)q[0];
      } else {
        return p.ann_bytes[off + i];
      }
    };
    if (TANN || p.ann_series_off) {
      if constexpr (TANN) {
        // the window's annotation (every row of the window carries it, the Reset row included), rewritten only when
        // its bytes differ from the last one written
        if (active) {
          const uint32_t w = xf_reset ? iter >> 1 : iter;
          const uint64_t ref = __ldg(p.tile_ann + (uint64_t)w * p.tile_n_src + xe->src);
          if (ref) {
            if constexpr (TBLK) {
              a_off = ref >> kBlockAnnLenBits;
              a_len = (uint32_t)(ref & ((1ull << kBlockAnnLenBits) - 1));
            } else {
              a_off = __ldg(p.tile_src_off + xe->src) * 8ull + (ref >> 32);
              a_len = (uint32_t)ref;
            }
            bool same = a_len == last_ann_len;
            if (same && a_off != last_ann_off)
              for (uint32_t i = 0; same && i < a_len; i++) same = ann_byte(a_off, i) == ann_byte(last_ann_off, i);
            want_ann = !same;
          }
        }
      } else if (active && ann_i < ann_end) {
        const m3tsz_annotation_entry e = p.ann_entries[ann_i];
        if (e.dp_index == iter) {
          ann_i++;
          a_off = e.byte_offset;
          a_len = e.length;
          if (a_len > 0) {
            if constexpr (APPEND) {
              // the last annotation written may belong to an earlier call: compare checksums, as the reference does
              const uint64_t h = xxh64(p.ann_bytes + a_off, a_len);
              want_ann = h != av.ann_cs;
              av.ann_cs = h;
            } else {
              // rewritten only when it differs from the last annotation written
              // (xxhash64 inequality in the reference == byte inequality here)
              bool same = (a_len == last_ann_len);
              for (uint32_t i = 0; same && i < a_len; i++)
                same = p.ann_bytes[a_off + i] == p.ann_bytes[last_ann_off + i];
              want_ann = !same;
            }
          }
        }
      }
      if (__any_sync(FULL_MASK, want_ann)) {
        uint32_t rem = 0, done_bytes = 0;
        if (want_ann) {
          put32(s, out_tile, lane, (kMarkerOpcode << 2) | (uint32_t)kMarkerAnnotation, kMarkerBits);
          uint64_t ux = ((uint64_t)(a_len - 1)) << 1;  // binary.PutVarint(len-1), len >= 1
          while (ux >= 0x80) {
            put32(s, out_tile, lane, (uint32_t)(ux & 0x7f) | 0x80u, 8);
            ux >>= 7;
          }
          put32(s, out_tile, lane, (uint32_t)ux, 8);
          rem = a_len;
          last_ann_off = a_off;
          last_ann_len = a_len;
        }
        for (;;) {
          if (rem > 0) {
            // capacity: stop this series rather than overrun its slot
            const uint64_t need_words = (uint64_t)s.words_out + s.k + (rem + 3) / 4 + ENC_GUARD + 4;
            if (need_words > slot_words) {
              s.err = M3TSZ_ERR_CAPACITY;
              rem = 0;
            }
          }
          while (rem > 0 && s.k < (uint32_t)(ENC_OUT_W - ENC_GUARD)) {
            put32(s, out_tile, lane, ann_byte(a_off, done_bytes), 8);
            done_bytes++;
            rem--;
          }
          if (!__any_sync(FULL_MASK, rem > 0)) break;
          flush_out(false);
        }
      }
    }

    // ---- encode one datapoint ----
    {
      // this datapoint was fetched from shared memory one datapoint ago (the load latency
      // hides behind the previous bit packing); fetch the next row of the tile now
      const int64_t t = t_pf;
      const uint64_t fb = fb_pf;
      if (STAGED) {
        if (!tile_last) {
          t_pf = (int64_t)in_next[0];
          fb_pf = in_next[IN_TILE_DW];
          in_next += IN_STRIDE;
        }
      } else {  // rotate the two-deep prefetch; request row iter + 2
        t_pf = t_pf1;
        fb_pf = fb_pf1;
        sk_pf = sk_pf1;
        load_row(iter + 2, t_pf1, fb_pf1, sk_pf1);
      }
      const double v = __longlong_as_double((long long)fb);
      const bool room = s.words_out + s.k + (uint32_t)(ENC_GUARD + 4) <= slot_words;  // < 2^31 words
      // hot candidate: same (valid s/ms/us/ns) unit, zero delta-of-delta, not the
      // first datapoint, a float-mode XOR code (value is certainly not int-like)
      const int64_t delta = (int64_t)((uint64_t)t - (uint64_t)s.prev_time);
      // (the int-likeness filter runs on the FP64 pipe for every lane: no divergent region around it)
      const bool not_int = !INT_OPT || !maybe_int(v);
      bool hot = (active & room & hot_ok & not_int) && delta == s.prev_delta;
      if (INT_OPT) hot = hot && fb != s.prev_bits;
      Tier2 c2;
      if (__all_sync(FULL_MASK, hot || !active)) {
        hot_commit(t, fb, (!TILES && !APPEND) || active, active);  // every live lane
      } else if (__all_sync(FULL_MASK, tier2_candidate<INT_OPT>(s, active && room && steady, delta, fb, v, c2) ||
                                           !active)) {
        // second tier: small delta-of-delta + (float XOR | float repeat | int diff | int
        // repeat) without a mode / header update, still one merge per lane
        if (active) {
          s.prev_time = t;
          s.prev_delta = delta;
          tier2_commit<INT_OPT>(s, out_tile, lane, fb, c2);
          s.n_enc++;
        }
      } else if (active && s.err == 0) {
        if (!room) {
          s.err = M3TSZ_ERR_CAPACITY;
        } else {
          const int u = p.units ? (int)p.units[in_s * p.points_stride + iter] : p.unit;
          uint32_t hdr;
          int hb;
          encode_time(s, out_tile, lane, t, u, hdr, hb);
          if (s.err == 0) {
            uint64_t payload;
            int plen;
            encode_value<INT_OPT>(s, v, hdr, hb, payload, plen);
            emit_code(s, out_tile, lane, hdr, hb, payload, plen);
            s.n_enc++;
          }
          // the fast tiers' slow-changing preconditions: the unit only changes here
          steady = !p.units && p.unit == s.unit && (s.unit >= 1 && s.unit <= 4) && s.n_enc > 0;
          hot_ok = steady && (!INT_OPT || s.is_float);
        }
      }
    }
  };

  if constexpr (GROUPS) {
    // Tile -> row.  What only changes every few rows or on the slow path is checked once per input tile, with
    // margins for IN_T hot datapoints of at most 2 + 14 + 64 bits (3 words) each: every live lane has all IN_T rows
    // (no lane ends inside the tile), room in its slot for them, and the hot tier's preconditions; there are no
    // annotations.  Inside such a tile the per-datapoint vote only looks at the data.  The first datapoint that
    // fails it, and every later row of the tile, takes encode_row with all of its checks.  A lane that is not
    // live is finished or failed for the whole tile and votes yes, as it does in encode_row.
    for (uint32_t row0 = 0; row0 < max_pts; row0 += IN_T) {  // warp-uniform
      begin_tile(row0);
      uint32_t iter = row0;
      const bool live = s.err == 0 && row0 < n_pts;
      const bool pre = hot_ok && row0 + IN_T <= n_pts &&
                       s.words_out + s.k + (uint32_t)(3 * (IN_T - 1) + ENC_GUARD + 4) <= slot_words;
      if (!p.ann_series_off && row0 + IN_T <= max_pts && __all_sync(FULL_MASK, pre || !live)) {
        // room in the output tile for IN_T hot codes: at most 10 words past a column of <= ENC_OUT_W - ENC_GUARD
        if (__any_sync(FULL_MASK, live && s.k > (uint32_t)(ENC_OUT_W - ENC_GUARD))) flush_out(false);
#pragma unroll 1
        for (; iter < row0 + IN_T; iter++) {
          const int64_t t = t_pf;
          const uint64_t fb = fb_pf;
          const bool more = iter + 1 < row0 + IN_T;
          if (more) {  // fetch the next row
            t_pf = (int64_t)in_next[0];
            fb_pf = in_next[IN_TILE_DW];
            in_next += IN_STRIDE;
          }
          const int64_t delta = (int64_t)((uint64_t)t - (uint64_t)s.prev_time);
          bool hot = delta == s.prev_delta;
          if (INT_OPT) hot = hot && fb != s.prev_bits && !maybe_int(__longlong_as_double((long long)fb));
          if (!__all_sync(FULL_MASK, hot || !live)) {  // this row and the rest of the tile: encode_row
            t_pf = t;
            fb_pf = fb;
            if (more) in_next -= IN_STRIDE;
            break;
          }
          hot_commit(t, fb, true, live);
        }
      }
      const uint32_t row_end = min(row0 + (uint32_t)IN_T, max_pts);
#pragma unroll 1
      for (; iter < row_end; iter++) encode_row(iter, iter == row0 + IN_T - 1, row_active(iter));
    }
  } else {
    for (uint32_t iter = 0; iter < max_pts; iter++) {  // warp-uniform (n_pts is 0 for lanes without a series)
      const bool tile_last = (iter & (IN_T - 1)) == IN_T - 1;
      const bool active = row_active(iter);
      if (STAGED && (iter & (IN_T - 1)) == 0) begin_tile(iter);
      encode_row(iter, tile_last, active);
    }
  }
  if (STAGED) asm volatile("cp.async.wait_all;\n" ::: "memory");
  if (bulk) bulk_seq += (max_pts + (uint32_t)IN_T - 1u) / (uint32_t)IN_T;  // every requested tile was waited for

  if constexpr (APPEND) {
    // ---- whole sectors to the slot, the rest (<= 7 words + the partial word) into the state ----
    flush_out(false);
    if (valid) {
      if (s.n_enc != av.n_enc0) enc_state_save<INT_OPT>(p.state[rec], s, out_tile, lane, av.ann_cs);
      // A routed lane reports nothing: route_series already gave every datapoint its result, and its room bound
      // (each earlier datapoint of the call at its worst case) implies the check above, as its time checks are
      // encode_time's, so s.err stays 0 here.  A change to either check must keep that implication;
      // tests/test_device_route_on_host.py asserts it for every routed datapoint.
      if (IN != 3) {
        p.n_appended[sidx] = s.n_enc - av.n_enc0;
        p.status[sidx] = s.err;
      }
    }
    continue;  // (one batch per warp)
  }

  // ---- tail: end-of-stream marker + zero padding (scheme.go:198-211) ----
  uint64_t total_bits = 0;
  if (valid && s.n_enc > 0) {
    put32(s, out_tile, lane, (kMarkerOpcode << 2) | (uint32_t)kMarkerEOS, kMarkerBits);
    total_bits = ((uint64_t)s.words_out + s.k) * 32ull + s.sh;
    if (s.sh > 0) {  // flush the partial word (zero padded)
      out_tile[s.k * ENC_STRIDE + lane] = s.carry;
      s.k++;
      s.carry = 0;
      s.sh = 0;
    }
    // pad to a whole 16-byte group (zeros; bytes past out_len are unspecified)
    while (s.k & 3u) {
      out_tile[s.k * ENC_STRIDE + lane] = 0u;
      s.k++;
    }
  } else if (valid) {
    s.k = 0;  // nothing encoded: empty stream (encoder.go:285-289)
    s.words_out = 0;
  } else {
    s.k = 0;
  }
  flush_out(true);
  const uint64_t my_len = (total_bits + 7) >> 3;
  if (valid && TILES && p.n_tiles_out) p.n_tiles_out[sidx] = s.n_enc;
  if (valid && p.out_bits) p.out_bits[sidx] = total_bits;  // incl. the end-of-stream marker, before padding
  if (valid && p.last_value) {
    // Encoder.LastEncoded().Value (encoder.go:305-319): the float when the encoder is in float
    // mode, else its intVal -- the SCALED integer in int mode, and 0 without the int optimisation
    // (isFloat is never set there)
    p.last_value[sidx] = (INT_OPT && s.is_float) ? __longlong_as_double((long long)s.prev_bits)
                                                 : (INT_OPT ? s.int_val : 0.0);
  }
  if (!PACKED) {
    if (valid) {
      if (p.out_len) p.out_len[sidx] = my_len;
      if (p.status) p.status[sidx] = s.err;
    }
  } else {
    // ---- allocate exact space and move the batch's streams into the packed buffer ----
    const uint64_t amask = (uint64_t)p.align - 1;
    const uint64_t alen = valid ? ((my_len + amask) & ~amask) : 0ull;
    uint64_t incl = alen;  // inclusive warp scan
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint64_t o = __shfl_up_sync(FULL_MASK, incl, d);
      if (lane >= d) incl += o;
    }
    const uint64_t total = __shfl_sync(FULL_MASK, incl, 31);
    unsigned long long base = 0;
    if (lane == 0 && total) base = atomicAdd(p.packed_cursor, (unsigned long long)total);
    base = __shfl_sync(FULL_MASK, base, 0);
    const bool fits = base + total <= p.packed_capacity;
    const uint64_t my_off = base + incl - alen;
    if (valid) {
      p.packed_off[sidx] = my_off;
      if (p.out_len) p.out_len[sidx] = fits ? my_len : 0ull;
      if (p.status) p.status[sidx] = (!fits && s.err == 0) ? M3TSZ_ERR_CAPACITY : s.err;
      // the transformation state moves on only with a written series (status OK: no source error, no CAPACITY)
      if (IN == 4 && p.xf_state && fits && s.err == 0 && !(p.tile_src_status && p.tile_src_status[sidx] != 0))
        p.xf_state[sidx] = *xs;
      // IN = 5: this lane's part of its series' new record (launch_tiles_types_status commits it when the source and
      // every type's row are OK).  Type 0's lane writes the element's fields and the inputs of types the call does
      // not have; type j's lane its own input
      if constexpr (ELEM) {
        if (p.xf_elem_out) {
          m3tsz_element_state &r = p.xf_elem_out[xe->src];
          const uint32_t ty = xe->ty;
          if (ty == 0) {
            r.head = xe->e.w;
            r.head.prev_v = xe->e.pv[0];
            for (uint32_t j = p.tile_n_types; j < M3TSZ_MAX_ELEMENT_TYPES; j++) r.prev_v_more[j - 1] = xe->e.pv[j];
            r.reserved = xe->reserved;
          } else {
            r.prev_v_more[ty - 1] = xe->e.pv[ty];
          }
        }
      }
    }
    __syncwarp();  // the flushes' stores to the slots are visible to the whole warp's copy below
    if (fits && total) {
      const uint8_t *slot0 = p.out + warp_slot * 32ull * p.out_stride;
      if (p.align >= 16) {
        // series after series, 32 lanes x 16 bytes, sixteen loads in flight per lane; the flush
        // above zero-padded every stream to a whole 16-byte group inside its slot
        for (int j = 0; j < 32; j++) {
          const uint64_t lj = __shfl_sync(FULL_MASK, my_len, j);
          const uint64_t oj = __shfl_sync(FULL_MASK, my_off, j);
          if (lj == 0) continue;
          const uint4 *src = reinterpret_cast<const uint4 *>(slot0 + (uint64_t)j * p.out_stride);
          uint4 *dst = reinterpret_cast<uint4 *>(p.packed + oj);
          const uint32_t nv = (uint32_t)((lj + 15) >> 4);
          uint32_t i = lane;
          for (; i + 480 < nv; i += 512) {  // 16 loads in flight per lane: 8 KB per warp
            uint4 r[16];
#pragma unroll
            for (int u = 0; u < 16; u++) r[u] = __ldcg(src + i + 32 * u);
#pragma unroll
            for (int u = 0; u < 16; u++) __stcs(dst + i + 32 * u, r[u]);
          }
          for (; i + 96 < nv; i += 128) {
            uint4 r[4];
#pragma unroll
            for (int u = 0; u < 4; u++) r[u] = __ldcg(src + i + 32 * u);
#pragma unroll
            for (int u = 0; u < 4; u++) __stcs(dst + i + 32 * u, r[u]);
          }
          for (; i < nv; i += 32) __stcs(dst + i, __ldcg(src + i));
        }
      } else {
        for (int j = 0; j < 32; j++) {
          const uint64_t lj = __shfl_sync(FULL_MASK, my_len, j);
          const uint64_t oj = __shfl_sync(FULL_MASK, my_off, j);
          const uint8_t *src = slot0 + (uint64_t)j * p.out_stride;
          uint8_t *dst = p.packed + oj;
          for (uint64_t i = lane; i < lj; i += 32) dst[i] = __ldcg(src + i);
        }
      }
    }
    __syncwarp();  // the next batch overwrites the slots
  }
  }  // batch loop
}

template <int IN>
constexpr size_t enc_block_smem() {
  return enc_warp_smem<IN>() * ENC_WARPS;
}

// Shared-memory carveout of the encode kernels (the rest of the SM's 256 KB of L1 + shared memory is L1).
// At 132 KB (124 KB of L1) the point-major stage holds 4 blocks (31 KB each: 16 warps per SM), the series-major
// stage 2 (48 KB each) and the Gauge stage 5 (register-limited).  Point-major encode of 500 k x 1440,
// int-optimised, on an H100 SXM (400 W power limit, 1980 MHz max SM clock), median of 3:
// * with 16-byte flushes and 8-row tiles (8 warps): 10.39 / 10.38 / 11.94 / 14.10 ms at 100 / 132 / 164 / 228 KB;
//   4-row tiles, 4 blocks at 132 KB (16 warps, the same L1): 12.93 ms.  More warps at equal L1 were slower, so
//   L1 size was not the cause.  Without the flush's global stores (wrong bytes, a diagnostic build) 8 and 16
//   warps took 7.43 and 6.06 ms: half-written sectors were what made more warps slower.
// * with whole-sector flushes: 10.29 ms at 8 warps; 8.46 ms with 4-row tiles at 16 warps (132 KB), 9.31 at
//   100 KB (3 blocks); 2-row tiles at 20 warps 8.52; 4-row x 3 stages at 164 KB (16 warps, 92 KB of L1) 8.57.
// * with paired flushes (16 whole sectors per store), 4-row tiles at 16 warps (132 KB), 30 launches: 7.97 / 7.90 ms
//   against 8.25 / 8.30 for whole-sector lane-local flushes in the same session.
constexpr int ENC_CARVEOUT_KB = 132;

// Tensor maps of the point-major input arrays: ts / val as [points_stride][n_series] tensors of 8-byte elements,
// box = enc_in_t<1>() rows x 32 series, no swizzle, zero fill outside.  ok = 0 when the arrays cannot be described
// (then the kernel keeps its cp.async fills).
static void enc_build_tensor_maps(const EncodeParams &p, EncTensorMaps &tm) {
  memset(&tm, 0, sizeof(tm));
  typedef CUresult (*encode_tiled_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                      const cuuint64_t *, const cuuint32_t *, const cuuint32_t *,
                                      CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                      CUtensorMapFloatOOBfill);
  static encode_tiled_fn fn = [] {
    void *f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      f = nullptr;
    return reinterpret_cast<encode_tiled_fn>(f);
  }();
  if (!fn) return;
  if (p.in_mode != 1 || !p.ts || !p.val) return;
  if ((((uintptr_t)p.ts | (uintptr_t)p.val) & 15u) != 0) return;
  if ((p.n_series & 1ull) != 0 || p.n_series >= (1ull << 31) || p.points_stride == 0 ||
      p.points_stride >= (1ull << 31))
    return;
  const cuuint64_t dims[2] = {(cuuint64_t)p.n_series, (cuuint64_t)p.points_stride};
  const cuuint64_t strides[1] = {(cuuint64_t)p.n_series * 8ull};
  const cuuint32_t box[2] = {32u, (cuuint32_t)enc_in_t<1>()};
  const cuuint32_t estr[2] = {1u, 1u};
  const CUresult a = fn(&tm.ts, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, const_cast<int64_t *>(p.ts), dims, strides, box,
                        estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                        CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  const CUresult b = fn(&tm.val, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, const_cast<double *>(p.val), dims, strides, box,
                        estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                        CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  tm.ok = (a == CUDA_SUCCESS && b == CUDA_SUCCESS) ? 1 : 0;
}

template <bool INT_OPT, bool PACKED, int IN, bool APPEND = false>
static cudaError_t launch_encode_one(const EncodeParams &p, cudaStream_t stream) {
  constexpr size_t smem = enc_block_smem<IN>();
  const uint64_t per_block = (uint64_t)ENC_WARPS * 32ull;
  uint64_t blocks = (p.n_series + per_block - 1) / per_block;
  if (blocks == 0) return cudaSuccess;
  if (blocks > 0x7fffffffull) return cudaErrorInvalidValue;
  if (IN == 3 && p.route_touched) {  // the overflow pass: a grid-stride loop over a grid of a few blocks per SM
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev))
      return cudaErrorInvalidValue;
    if (blocks > 8ull * (uint64_t)sms) blocks = 8ull * (uint64_t)sms;
  }
  cudaError_t e = cudaFuncSetAttribute(encode_kernel<INT_OPT, PACKED, IN, APPEND>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(encode_kernel<INT_OPT, PACKED, IN, APPEND>, cudaFuncAttributePreferredSharedMemoryCarveout,
                           ENC_CARVEOUT_KB * 100 / 228);
  if (e != cudaSuccess) return e;
  if (PACKED) {
    const uint64_t resident = encode_packed_resident_blocks();
    if (resident == 0) return cudaErrorInvalidValue;
    if (blocks > resident) blocks = resident;
  }
  EncTensorMaps tm;
  if (IN == 3)
    memset(&tm, 0, sizeof(tm));  // (in_mode names the routed stage's input layout; it reads no tiles)
  else
    enc_build_tensor_maps(p, tm);  // (ok = 0 for the other input stages)
  encode_kernel<INT_OPT, PACKED, IN, APPEND><<<(unsigned)blocks, ENC_WARPS * 32, smem, stream>>>(p, tm);
  return cudaGetLastError();
}

// Persistent grid of the packed mode: resident blocks on the current device (also the number
// of scratch slot sets: resident blocks x ENC_WARPS x 32 slots of out_stride bytes).
uint64_t encode_packed_resident_blocks() {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
  int best = 0;
  auto probe = [&](auto kernel, size_t sm) {
    int n = 0;
    cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, ENC_CARVEOUT_KB * 100 / 228);
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm) == cudaSuccess &&
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, ENC_WARPS * 32, sm) == cudaSuccess && n > best)
      best = n;
  };
  probe(encode_kernel<true, true, 0>, enc_block_smem<0>());
  probe(encode_kernel<false, true, 0>, enc_block_smem<0>());
  probe(encode_kernel<true, true, 1>, enc_block_smem<1>());
  probe(encode_kernel<false, true, 1>, enc_block_smem<1>());
  probe(encode_kernel<true, true, 2>, enc_block_smem<2>());
  probe(encode_kernel<false, true, 2>, enc_block_smem<2>());
  return (uint64_t)sms * (uint64_t)best;
}
uint64_t encode_packed_scratch_slots(uint64_t n_series) {
  const uint64_t per_block = (uint64_t)ENC_WARPS * 32ull;
  uint64_t blocks = (n_series + per_block - 1) / per_block;
  const uint64_t resident = encode_packed_resident_blocks();
  if (blocks > resident) blocks = resident;
  return blocks * per_block;
}

// in_mode 0: series-major inputs; 1: point-major inputs; 2: Gauge aggregates; 4: the aggregates through the
// transformations; 5: an element's several types through them; 6: 5 with the windows' annotations; 7: 6 over
// several source blocks per series (2, 4, 5, 6 and 7: packed output only)
cudaError_t launch_encode(const EncodeParams &p, bool int_optimized, cudaStream_t stream) {
  if (p.in_mode == 2) {
    if (!p.packed) return cudaErrorInvalidValue;
    return int_optimized ? launch_encode_one<true, true, 2>(p, stream) : launch_encode_one<false, true, 2>(p, stream);
  }
  if (p.in_mode == 4) {
    if (!p.packed) return cudaErrorInvalidValue;
    return int_optimized ? launch_encode_one<true, true, 4>(p, stream) : launch_encode_one<false, true, 4>(p, stream);
  }
  if (p.in_mode == 5) {
    if (!p.packed || p.tile_n_src == 0) return cudaErrorInvalidValue;
    return int_optimized ? launch_encode_one<true, true, 5>(p, stream) : launch_encode_one<false, true, 5>(p, stream);
  }
  if (p.in_mode == 6) {
    if (!p.packed || p.tile_n_src == 0 || !p.tile_ann || !p.tile_src_streams || !p.tile_src_off)
      return cudaErrorInvalidValue;
    return int_optimized ? launch_encode_one<true, true, 6>(p, stream) : launch_encode_one<false, true, 6>(p, stream);
  }
  if (p.in_mode == 7) {
    if (!p.packed || p.tile_n_src == 0 || !p.tile_ann || !p.tile_src_streams) return cudaErrorInvalidValue;
    return int_optimized ? launch_encode_one<true, true, 7>(p, stream) : launch_encode_one<false, true, 7>(p, stream);
  }
  if (p.in_mode == 1) {
    if (p.packed)
      return int_optimized ? launch_encode_one<true, true, 1>(p, stream) : launch_encode_one<false, true, 1>(p, stream);
    return int_optimized ? launch_encode_one<true, false, 1>(p, stream)
                         : launch_encode_one<false, false, 1>(p, stream);
  }
  if (p.packed) {
    return int_optimized ? launch_encode_one<true, true, 0>(p, stream) : launch_encode_one<false, true, 0>(p, stream);
  }
  return int_optimized ? launch_encode_one<true, false, 0>(p, stream) : launch_encode_one<false, false, 0>(p, stream);
}

// ---------------------------------------------------------------------------
// encoder sets (DESIGN.md §4.6)
// ---------------------------------------------------------------------------
cudaError_t launch_encode_append(const EncodeParams &p, bool int_optimized, cudaStream_t stream) {
  if (p.in_mode == 1)
    return int_optimized ? launch_encode_one<true, false, 1, true>(p, stream)
                         : launch_encode_one<false, false, 1, true>(p, stream);
  return int_optimized ? launch_encode_one<true, false, 0, true>(p, stream)
                       : launch_encode_one<false, false, 0, true>(p, stream);
}

cudaError_t launch_encode_routed(const EncodeParams &p, bool int_optimized, cudaStream_t stream) {
  return int_optimized ? launch_encode_one<true, false, 3, true>(p, stream)
                       : launch_encode_one<false, false, 3, true>(p, stream);
}

// one thread per bucket (route_series); a 7-row tile column per lane for enc_state_load's leftover words
constexpr int ROUTE_THREADS = 128;
template <bool INT_OPT>
__global__ void __launch_bounds__(ROUTE_THREADS) route_kernel(const RouteParams p) {
  __shared__ uint32_t tile[ROUTE_THREADS / 32][7 * ENC_STRIDE];
  const uint64_t s = (uint64_t)blockIdx.x * ROUTE_THREADS + threadIdx.x;
  if (s >= p.n_series) return;
  route_series<INT_OPT>(p, s, tile[threadIdx.x >> 5], threadIdx.x & 31);
}

cudaError_t launch_route(const RouteParams &p, bool int_optimized, cudaStream_t stream) {
  const uint64_t blocks = (p.n_series + ROUTE_THREADS - 1) / ROUTE_THREADS;
  if (blocks == 0) return cudaSuccess;
  if (blocks > 0x7fffffffull) return cudaErrorInvalidValue;
  if (int_optimized)
    route_kernel<true><<<(unsigned)blocks, ROUTE_THREADS, 0, stream>>>(p);
  else
    route_kernel<false><<<(unsigned)blocks, ROUTE_THREADS, 0, stream>>>(p);
  return cudaGetLastError();
}

__global__ void encoder_set_reset_kernel(m3tsz_encoder_state *state, uint64_t n, const int64_t *start,
                                         int default_unit, bool int_opt) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  m3tsz_encoder_state st;
  enc_state_reset(st, start[i], default_unit, int_opt);
  state[i] = st;
}

// one thread per encoder: its tail (<= 3 16-byte groups) at the committed position of its slot
__global__ void encoder_set_stream_kernel(const m3tsz_encoder_state *state, uint64_t n, uint8_t *buf,
                                          uint64_t stride, uint64_t *len) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const m3tsz_encoder_state st = state[i];
  uint32_t w[12];
  uint64_t at = 0;
  const uint32_t nw = enc_snapshot_words(st, w, at);
  if (nw) {
    uint4 *dst = reinterpret_cast<uint4 *>(buf + i * stride + at * 4ull);
    for (uint32_t g = 0; g < nw / 4; g++)
      dst[g] = make_uint4(__byte_perm(w[4 * g], 0, 0x0123), __byte_perm(w[4 * g + 1], 0, 0x0123),
                          __byte_perm(w[4 * g + 2], 0, 0x0123), __byte_perm(w[4 * g + 3], 0, 0x0123));
  }
  len[i] = st.num_encoded ? (st.bits + kMarkerBits + 7) >> 3 : 0ull;
}

cudaError_t launch_encoder_set_reset(m3tsz_encoder_state *state, uint64_t n, const int64_t *start, int default_unit,
                                     bool int_optimized, cudaStream_t stream) {
  const unsigned tb = 256;
  if ((n + tb - 1) / tb > 0x7fffffffull) return cudaErrorInvalidValue;
  encoder_set_reset_kernel<<<(unsigned)((n + tb - 1) / tb), tb, 0, stream>>>(state, n, start, default_unit,
                                                                             int_optimized);
  return cudaGetLastError();
}

cudaError_t launch_encoder_set_stream(const m3tsz_encoder_state *state, uint64_t n, uint8_t *buf, uint64_t stride,
                                      uint64_t *len, cudaStream_t stream) {
  const unsigned tb = 256;
  if ((n + tb - 1) / tb > 0x7fffffffull) return cudaErrorInvalidValue;
  encoder_set_stream_kernel<<<(unsigned)((n + tb - 1) / tb), tb, 0, stream>>>(state, n, buf, stride, len);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------
// tile aggregation through a rollup (DESIGN.md §4.8): forward stage, then the fold into the group element's windows
// ---------------------------------------------------------------------------
// One window of a rollup element: every value AddUnique gives it arrives at the same timestamp (the source windows'
// common end), so Gauge.updateTotals (gauge.go:74-101) keeps the FIRST value as Last (timestamp.After(lastAt) is
// false for equal times), counts NaNs and skips them in sum / min / max / sumSq; min and max start as math.NaN()
// and keep the first of +-0.  Counter.Update (counter.go:52-78) takes int64(value) (amd64's conversion) and wraps.
struct RollupGaugeAcc {
  double sum, mn, mx, last, sq;
  int64_t cnt;
};
struct RollupCounterAcc {
  int64_t sum, mn, mx, sq, cnt;
};
__device__ __forceinline__ void rollup_gauge_init(RollupGaugeAcc &a) {  // NewGauge, gauge.go:45-51
  a.sum = 0.0;
  a.mn = xf_bits(kXfEmptyNaN);
  a.mx = xf_bits(kXfEmptyNaN);
  a.last = 0.0;
  a.sq = 0.0;
  a.cnt = 0;
}
__device__ __forceinline__ void rollup_counter_init(RollupCounterAcc &a) {  // NewCounter, counter.go:44-50
  a.sum = 0;
  a.mn = (int64_t)0x7fffffffffffffffull;
  a.mx = (int64_t)0x8000000000000000ull;
  a.sq = 0;
  a.cnt = 0;
}
// amd64's ADDSD of a running total and a non-NaN value: a NaN total keeps its payload (quieted), Inf + -Inf gives
// the default NaN
__device__ __forceinline__ double rollup_add(double a, double x) {
  const double r = __dadd_rn(a, x);
  if (!xf_isnan(r)) return r;
  return xf_isnan(a) ? xf_bits((uint64_t)__double_as_longlong(a) | 0x0008000000000000ull) : xf_bits(kXfOpNaN);
}
__device__ __forceinline__ void rollup_gauge_add(RollupGaugeAcc &a, double x) {
  if (a.cnt == 0) a.last = x;
  a.cnt++;
  if (xf_isnan(x)) return;
  a.sum = rollup_add(a.sum, x);
  if (xf_isnan(a.mx) || a.mx < x) a.mx = x;
  if (xf_isnan(a.mn) || a.mn > x) a.mn = x;
  a.sq = rollup_add(a.sq, __dmul_rn(x, x));
}
__device__ __forceinline__ void rollup_counter_add(RollupCounterAcc &a, double x) {
  const int64_t v = go_f64_to_i64(x);
  a.sum = (int64_t)((uint64_t)a.sum + (uint64_t)v);
  a.cnt++;
  if (a.mx < v) a.mx = v;
  if (a.mn > v) a.mn = v;
  a.sq = (int64_t)((uint64_t)a.sq + (uint64_t)v * (uint64_t)v);
}

// The annotated forward stage's step for a window of source s with datapoints: the fused decode's reference `ref`
// (0: none) in the batch-addressed form the multi-type stage's IN = 7 reads, (bit offset from the batch's first bit)
// << kBlockAnnLenBits | length.  src_off NULL: the decode over source blocks already wrote it so.  false: a payload
// of 2^27 bytes or more, which rejects the source (the limit of that form, as over source blocks)
__device__ __forceinline__ bool rollup_ann_ref(uint64_t &ref, const uint64_t *src_off, uint64_t s) {
  if (!ref || !src_off) return true;
  const uint64_t len = ref & 0xffffffffull;
  if (len >> kBlockAnnLenBits) return false;
  ref = ((src_off[s] * 8ull + (ref >> 32)) << kBlockAnnLenBits) | len;
  return true;
}
// The annotated fold's step for one member (MaybeReplaceAnnotation in Gauge / Counter Update, reached through
// AddUnique): a window the member forwarded with a non-empty annotation (its ann_present bit) replaces the group's
// reference, and any other keeps it
__device__ __forceinline__ void rollup_ann_add(uint64_t &g, uint32_t ann_bits, uint32_t lane, const uint64_t *ref) {
  if ((ann_bits >> lane) & 1u) g = *ref;
}

// Forward stage: one lane per source series, windows in order (the chain is a recurrence over them), 32 windows at a
// time staged in shared memory so that the series-major rows are written as whole 256-byte runs; the presence words
// of those 32 windows are one word-major row, written by the warp as 128-byte runs.  ANN: also the ann_present row
// the same way; the references stay window-major where the decode wrote them (a lane's read of window w is one
// 256-byte run per warp), rewritten in place only where a forwarded window has one.
constexpr int ROLLUP_FWD_WARPS = 4;
template <bool ANN>
__global__ void __launch_bounds__(ROLLUP_FWD_WARPS * 32) rollup_forward_kernel(const RollupForwardParams p) {
  __shared__ double tile[ROLLUP_FWD_WARPS][32][33];
  const uint32_t lane = threadIdx.x & 31u, wi = threadIdx.x >> 5;
  const uint64_t s0 = ((uint64_t)blockIdx.x * ROLLUP_FWD_WARPS + wi) * 32ull, s = s0 + lane;
  const bool valid = s < p.n_src;
  const bool ok = valid && p.src_status[s] == M3TSZ_OK;
  const bool counter = p.tiles.metric_type == M3TSZ_METRIC_COUNTER;
  m3tsz_transform_state st;
  if (valid && p.state)
    st = p.state[s];
  else
    memset(&st, 0, sizeof(st));
  double(*const tl)[33] = tile[wi];
  bool too_large = false;  // (ANN)
  for (uint32_t w0 = 0; w0 < p.n_windows; w0 += 32) {
    uint32_t bits = 0, abits = 0;
#pragma unroll 1
    for (uint32_t i = 0; i < 32; i++) {
      const uint32_t w = w0 + i;
      double v = 0.0;
      if (ok && w < p.n_windows) {
        const uint64_t o = (uint64_t)w * p.n_src + s;
        const int64_t c = __ldg(p.tiles.tile_count + o);
        if (c != 0) {
          v = tile_value_of(p.tiles, counter, p.src_type, o, c);
          int64_t extra_t = 0;  // (a Reset datapoint is not forwarded)
          xf_window(p.ops, p.tiles.tile_step, st, p.tiles.tile_start + (int64_t)(w + 1) * p.tiles.tile_step, v,
                    extra_t);
          if (!(p.discard_nan && xf_isnan(v))) bits |= 1u << i;
          if constexpr (ANN) {
            uint64_t ref = p.ann[o];
            if (!rollup_ann_ref(ref, p.src_off, s)) {
              too_large = true;
            } else if (ref && ((bits >> i) & 1u)) {
              abits |= 1u << i;
              if (p.src_off) p.ann[o] = ref;
            }
          }
        }
      }
      tl[lane][i] = v;
    }
    __syncwarp();
    const uint32_t w = w0 + lane;
    for (uint32_t j = 0; j < 32; j++)
      if (s0 + j < p.n_src && w < p.n_windows) p.fwd[(s0 + j) * p.n_windows + w] = tl[j][lane];
    if (valid) p.present[(uint64_t)(w0 >> 5) * p.n_src + s] = bits;
    if constexpr (ANN)
      if (valid) p.ann_present[(uint64_t)(w0 >> 5) * p.n_src + s] = abits;
    __syncwarp();
  }
  if (valid) p.state_out[s] = st;
  if constexpr (ANN)
    if (too_large) p.src_status_out[s] = M3TSZ_ERR_STREAM_TOO_LARGE;  // (the fold then fails every group listing s)
}

// Fold: one warp per group, lane l over windows w0 + l; members in listed order (each lane folds its own window, so
// the order is the same in every window), their present words read once per 32 windows, their values as 256-byte
// runs.  A block's groups write their window rows through shared memory, ROLLUP_FOLD_WARPS adjacent slots at a time.
// ANN: also each group window's annotation reference, a seventh row; a member's ann_present word is read with its
// present word, and its window-major reference only where that bit is set.
constexpr int ROLLUP_FOLD_WARPS = 8;
template <bool ANN>
__global__ void __launch_bounds__(ROLLUP_FOLD_WARPS * 32) rollup_fold_kernel(const RollupFoldParams p) {
  constexpr int NR = ANN ? 7 : 6;
  __shared__ uint64_t out[NR][32][ROLLUP_FOLD_WARPS];
  const uint32_t lane = threadIdx.x & 31u, wi = threadIdx.x >> 5;
  const uint64_t g0 = (uint64_t)blockIdx.x * ROLLUP_FOLD_WARPS, g = g0 + wi;
  const bool valid = g < p.n_groups;
  // the group's status: its range, then its members in listed order (the first failing one)
  int32_t gst = M3TSZ_OK;
  uint64_t lo = 0, hi = 0;
  if (valid) {
    lo = p.group_off[g];
    hi = p.group_off[g + 1];
    if (lo > hi || hi > p.n_members) {
      gst = M3TSZ_ERR_INVALID_ARG;
    } else {
      for (uint64_t i0 = lo; i0 < hi && gst == M3TSZ_OK; i0 += 32) {
        int32_t e = M3TSZ_OK;
        if (i0 + lane < hi) {
          const uint32_t m = p.members[i0 + lane];
          e = m >= p.n_src ? M3TSZ_ERR_INVALID_ARG : p.src_status[m];
        }
        const uint32_t bad = __ballot_sync(FULL_MASK, e != M3TSZ_OK);
        if (bad) gst = __shfl_sync(FULL_MASK, e, __ffs(bad) - 1);
      }
    }
    if (lane == 0) p.group_status[g] = gst;
  }
  const bool fold = valid && gst == M3TSZ_OK;
  for (uint32_t w0 = 0; w0 < p.n_windows; w0 += 32) {
    const uint32_t w = w0 + lane, word = w0 >> 5;  // (a window past the range has no present bit)
    uint64_t r[NR];
    uint64_t gann = 0;  // (ANN)
    if (p.counter) {
      RollupCounterAcc a;
      rollup_counter_init(a);
      if (fold) {
        for (uint64_t i = lo; i < hi; i++) {
          const uint64_t m = __ldg(p.members + i);
          const uint32_t bits = __ldg(p.present + (uint64_t)word * p.n_src + m);
          if ((bits >> lane) & 1u) rollup_counter_add(a, __ldg(p.fwd + m * p.n_windows + w));
          if constexpr (ANN)
            rollup_ann_add(gann, __ldg(p.ann_present + (uint64_t)word * p.n_src + m), lane,
                           p.ann + (uint64_t)w * p.n_src + m);
        }
      }
      r[0] = (uint64_t)a.sum;
      r[1] = (uint64_t)a.cnt;
      r[2] = (uint64_t)a.mn;
      r[3] = (uint64_t)a.mx;
      r[4] = 0;
      r[5] = (uint64_t)a.sq;
    } else {
      RollupGaugeAcc a;
      rollup_gauge_init(a);
      if (fold) {
        for (uint64_t i = lo; i < hi; i++) {
          const uint64_t m = __ldg(p.members + i);
          const uint32_t bits = __ldg(p.present + (uint64_t)word * p.n_src + m);
          if ((bits >> lane) & 1u) rollup_gauge_add(a, __ldg(p.fwd + m * p.n_windows + w));
          if constexpr (ANN)
            rollup_ann_add(gann, __ldg(p.ann_present + (uint64_t)word * p.n_src + m), lane,
                           p.ann + (uint64_t)w * p.n_src + m);
        }
      }
      r[0] = (uint64_t)__double_as_longlong(a.sum);
      r[1] = (uint64_t)a.cnt;
      r[2] = (uint64_t)__double_as_longlong(a.mn);
      r[3] = (uint64_t)__double_as_longlong(a.mx);
      r[4] = (uint64_t)__double_as_longlong(a.last);
      r[5] = (uint64_t)__double_as_longlong(a.sq);
    }
    if constexpr (ANN) r[6] = gann;
#pragma unroll
    for (int k = 0; k < NR; k++) out[k][lane][wi] = r[k];
    __syncthreads();
    // row rr of this window block, group column c: ROLLUP_FOLD_WARPS adjacent 8-byte slots of one window row
    for (uint32_t t = threadIdx.x; t < 32u * ROLLUP_FOLD_WARPS; t += blockDim.x) {
      const uint32_t rr = t / ROLLUP_FOLD_WARPS, c = t % ROLLUP_FOLD_WARPS;
      if (w0 + rr >= p.n_windows || g0 + c >= p.n_groups) continue;
      const uint64_t o = (uint64_t)(w0 + rr) * p.n_groups + g0 + c;
      reinterpret_cast<uint64_t *>(p.sum)[o] = out[0][rr][c];
      p.count[o] = (int64_t)out[1][rr][c];
      reinterpret_cast<uint64_t *>(p.min)[o] = out[2][rr][c];
      reinterpret_cast<uint64_t *>(p.max)[o] = out[3][rr][c];
      if (!p.counter) reinterpret_cast<uint64_t *>(p.last)[o] = out[4][rr][c];
      if (p.sum_sq) reinterpret_cast<uint64_t *>(p.sum_sq)[o] = out[5][rr][c];
      if constexpr (ANN) p.group_ann[o] = out[6][rr][c];
    }
    __syncthreads();
  }
}

cudaError_t launch_rollup_forward(const RollupForwardParams &p, bool annotated, cudaStream_t stream) {
  if (p.n_src == 0 || p.n_windows == 0) return cudaSuccess;
  const uint64_t per_block = 32ull * ROLLUP_FWD_WARPS, blocks = (p.n_src + per_block - 1) / per_block;
  if (blocks > 0x7fffffffull) return cudaErrorInvalidValue;
  if (annotated) {
    if (!p.ann || !p.ann_present || !p.src_status_out) return cudaErrorInvalidValue;
    rollup_forward_kernel<true><<<(unsigned)blocks, ROLLUP_FWD_WARPS * 32, 0, stream>>>(p);
  } else {
    rollup_forward_kernel<false><<<(unsigned)blocks, ROLLUP_FWD_WARPS * 32, 0, stream>>>(p);
  }
  return cudaGetLastError();
}

cudaError_t launch_rollup_fold(const RollupFoldParams &p, bool annotated, cudaStream_t stream) {
  if (p.n_groups == 0) return cudaSuccess;
  const uint64_t blocks = (p.n_groups + ROLLUP_FOLD_WARPS - 1) / ROLLUP_FOLD_WARPS;
  if (blocks > 0x7fffffffull) return cudaErrorInvalidValue;
  if (annotated) {
    if (!p.group_ann) return cudaErrorInvalidValue;  // (ann / ann_present: read only where a bit is set)
    rollup_fold_kernel<true><<<(unsigned)blocks, ROLLUP_FOLD_WARPS * 32, 0, stream>>>(p);
  } else {
    rollup_fold_kernel<false><<<(unsigned)blocks, ROLLUP_FOLD_WARPS * 32, 0, stream>>>(p);
  }
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------
// element sets (DESIGN.md §4.12): the aggregator's elements fed datapoint by datapoint, one lane per element
// ---------------------------------------------------------------------------
// t.Truncate(resolution) of Go's time.Time, which truncates the time since the zero time (year 1): the start of t's
// window, with off = that origin's distance to the Unix epoch modulo the resolution.  false: the start would lie
// below INT64_MIN.
__device__ __forceinline__ bool elem_window_start(int64_t t, int64_t res, int64_t off, int64_t &ws) {
  int64_t r = t % res;
  if (r < 0) r += res;
  r += off;
  if (r >= res) r -= res;
  if (t < (int64_t)0x8000000000000000ull + r) return false;
  ws = t - r;
  return true;
}
// a window starting at ws ends at or before `at` (ws + res <= at without the overflow of ws + res)
__device__ __forceinline__ bool elem_ends_by(int64_t ws, int64_t res, int64_t at) {
  return ws < at && (uint64_t)at - (uint64_t)ws >= (uint64_t)res;
}

// The open window a lane holds in registers: its start and the aggregates of the fused decode's windows (the Gauge's
// min / max as its running form, +inf / -inf with no value yet; the Counter's int64)
template <bool CTR>
struct ElemAcc {
  using V = std::conditional_t<CTR, int64_t, double>;
  int64_t start, cnt;
  V sum, mn, mx, sq;
  double last;  // Gauge only
  int64_t last_at;
  // an annotated set's window annotation to slot o (ElementParams::store_ann)
  __device__ static __forceinline__ void store_ann(const ElementParams &p, uint64_t o, uint64_t a_off, uint32_t a_len) {
    p.store_ann(o, a_off, a_len);
  }
};
template <bool CTR>
__device__ __forceinline__ void elem_init(ElemAcc<CTR> &a, int64_t ws) {  // NewGauge / NewCounter
  a.start = ws;
  a.cnt = 0;
  if constexpr (CTR) {
    a.sum = 0;
    a.mn = (int64_t)0x7fffffffffffffffull;
    a.mx = (int64_t)0x8000000000000000ull;
    a.sq = 0;
  } else {
    a.sum = 0.0;
    a.mn = xf_bits(0x7ff0000000000000ull);
    a.mx = xf_bits(0xfff0000000000000ull);
    a.sq = 0.0;
  }
  a.last = 0.0;
  a.last_at = 0;
}
// slots hold what the fused decode publishes: a Gauge window without a non-NaN value has min = max = math.NaN()
template <bool CTR>
__device__ __forceinline__ void elem_load(const ElementParams &p, uint64_t o, ElemAcc<CTR> &a) {
  using V = typename ElemAcc<CTR>::V;
  a.start = p.start[o];
  a.cnt = p.count[o];
  a.sum = static_cast<const V *>(p.sum)[o];
  a.mn = static_cast<const V *>(p.min)[o];
  a.mx = static_cast<const V *>(p.max)[o];
  a.sq = static_cast<const V *>(p.sum_sq)[o];
  if constexpr (!CTR) {
    if (xf_isnan(a.mn)) {
      a.mn = xf_bits(0x7ff0000000000000ull);
      a.mx = xf_bits(0xfff0000000000000ull);
    }
    a.last = p.last[o];
    a.last_at = p.last_at[o];
  }
}
template <bool CTR>
__device__ __forceinline__ void elem_store(const ElementParams &p, uint64_t o, const ElemAcc<CTR> &a) {
  using V = typename ElemAcc<CTR>::V;
  p.start[o] = a.start;
  p.count[o] = a.cnt;
  static_cast<V *>(p.sum)[o] = a.sum;
  static_cast<V *>(p.sum_sq)[o] = a.sq;
  if constexpr (CTR) {
    static_cast<V *>(p.min)[o] = a.mn;
    static_cast<V *>(p.max)[o] = a.mx;
  } else {
    const bool none = a.mn == xf_bits(0x7ff0000000000000ull) && a.mx == xf_bits(0xfff0000000000000ull);
    static_cast<V *>(p.min)[o] = none ? xf_bits(kXfEmptyNaN) : a.mn;
    static_cast<V *>(p.max)[o] = none ? xf_bits(kXfEmptyNaN) : a.mx;
    p.last[o] = a.last;
    p.last_at[o] = a.last_at;
  }
}
// Gauge.Update (gauge.go:74-106) / Counter.Update (counter.go:52-78) as the fused decode runs them
template <bool CTR>
__device__ __forceinline__ void elem_update(ElemAcc<CTR> &a, int64_t t, double v) {
  if constexpr (CTR) {  // int64(value), int64 arithmetic that wraps
    const int64_t x = go_f64_to_i64(v);
    a.sum = (int64_t)((uint64_t)a.sum + (uint64_t)x);
    if (a.mx < x) a.mx = x;
    if (a.mn > x) a.mn = x;
    a.sq = (int64_t)((uint64_t)a.sq + (uint64_t)x * (uint64_t)x);
  } else {
    if (a.cnt == 0 || t > a.last_at) {  // lastAt.IsZero() || timestamp.After(lastAt), NaN values included
      a.last_at = t;
      a.last = v;
    }
    if (v == v) {
      a.sum = __dadd_rn(a.sum, v);
      a.sq = __dadd_rn(a.sq, __dmul_rn(v, v));
    }
    if (v > a.mx) a.mx = v;
    if (v < a.mn) a.mn = v;
  }
  a.cnt++;
}

// AddUnion of element s's datapoints in row order.  The window the last datapoint went to stays in registers (in-order
// data almost never leaves it) and goes back to its slot when a datapoint needs another one, and at the end.
// ANN: so does the window's annotation, as a reference (a_off, a_len) into the call's annotation bytes: the last
// non-empty one of the window's accepted datapoints (MaybeReplaceAnnotation, aggregation/common.go:47-61).  It goes to
// the slot with the window, and only when it changed (a_dirty): a window opened here always writes its length, 0
// without an annotation, so a slot never keeps the length of a window it held before.
template <bool CTR, bool ANN = false>
__device__ __forceinline__ void elem_add_lane(const ElementParams &p, uint64_t s) {
  const uint32_t n_pts = p.n_points ? p.n_points[s] : (uint32_t)p.points_stride;
  if (n_pts > p.points_stride) {
    p.status[s] = M3TSZ_ERR_INVALID_ARG;
    return;
  }
  const int64_t wm = p.watermark[s];
  ElemAcc<CTR> a;
  elem_init(a, 0);
  int cur = -1;  // the slot `a` belongs to, -1: none
  int32_t status = M3TSZ_OK;
  uint64_t a_off = 0, ann_i = 0, ann_end = 0;
  uint32_t a_len = 0;
  bool a_dirty = false;
  if (ANN && p.ann_series_off) {
    ann_i = p.ann_series_off[s];
    ann_end = p.ann_series_off[s + 1];
  }
  for (uint32_t i = 0; i < n_pts; i++) {
    const uint64_t at = (uint64_t)i * p.n + s;
    int res = M3TSZ_ERR_CAPACITY;  // (after a CAPACITY, the rest of the element's datapoints)
    if (status == M3TSZ_OK) {
      const int64_t t = p.ts[at];
      const double v = p.val[at];
      int64_t ws = 0;
      uint64_t d_off = 0;  // this datapoint's annotation, d_len 0: none
      uint32_t d_len = 0;
      if constexpr (ANN) {
        while (ann_i < ann_end && p.ann_entries[ann_i].dp_index < i) ann_i++;
        if (ann_i < ann_end && p.ann_entries[ann_i].dp_index == i) {
          d_off = p.ann_entries[ann_i].byte_offset;
          d_len = p.ann_entries[ann_i].length;
        }
      }
      if (!elem_window_start(t, p.resolution, p.trunc_off, ws)) {
        res = M3TSZ_ERR_INVALID_ARG;
      } else if (elem_ends_by(ws, p.resolution, wm)) {
        res = M3TSZ_ERR_AGGREGATION_CLOSED;
      } else if (ANN && d_len > p.ann_cap) {
        status = res = M3TSZ_ERR_CAPACITY;
      } else {
        res = M3TSZ_OK;
        if (cur < 0 || ws != a.start) {  // the window's slot, or a free one
          int hit = -1, fr = -1;
          for (uint32_t r = 0; r < p.n_slots; r++) {
            if ((int)r == cur) continue;
            const uint64_t o = (uint64_t)r * p.n + s;
            if (p.count[o] == 0) {
              if (fr < 0) fr = (int)r;
            } else if (p.start[o] == ws) {
              hit = (int)r;
              break;
            }
          }
          if (hit < 0 && fr < 0) {
            status = res = M3TSZ_ERR_CAPACITY;
          } else {
            if (cur >= 0) {
              elem_store(p, (uint64_t)cur * p.n + s, a);
              if (ANN && a_dirty) ElemAcc<CTR>::store_ann(p, (uint64_t)cur * p.n + s, a_off, a_len);
            }
            cur = hit >= 0 ? hit : fr;
            if (hit >= 0)
              elem_load(p, (uint64_t)hit * p.n + s, a);
            else
              elem_init(a, ws);
            a_len = 0;
            a_dirty = hit < 0;
          }
        }
        if (res == M3TSZ_OK) {
          elem_update(a, t, v);
          if (ANN && d_len) {
            a_off = d_off;
            a_len = d_len;
            a_dirty = true;
          }
        }
      }
    }
    p.result[at] = (int8_t)res;
  }
  if (cur >= 0) {
    elem_store(p, (uint64_t)cur * p.n + s, a);
    if (ANN && a_dirty) ElemAcc<CTR>::store_ann(p, (uint64_t)cur * p.n + s, a_off, a_len);
  }
  p.status[s] = status;
}

// Consume(target) of element s: its windows ending at or before p.target, in start order, through the multi-type
// stage's element step (xf_element_window over tile_value_of of the slot), staged as rows for the encoder-set append:
// type j's datapoints in rows j * n + s of p.row_ts / p.row_val ([p.rows_stride][n_types * n]), their count in
// p.row_n.  An element whose output rows lack room changes nothing and gets CAPACITY.  `e` is the lane's element record
// while it runs (the kernel's is in shared memory: xf_element_window indexes its inputs by type).
// ANN: every staged datapoint of a window also gets an entry for the append, row i's at row_ann_off[i] =
// i * rows_stride, referring to the window's slot bytes (length 0 without an annotation, which the append takes as
// none); an entry past a row's count is never read.
template <bool CTR, bool ANN = false>
__device__ __forceinline__ void elem_consume_lane(const ElementParams &p, uint64_t s, XfElem &e) {
  const uint64_t kn = (uint64_t)p.n_types * p.n;
  // a slot's annotation length (ElementParams::slot_ann_len)
  auto ann_len = [&](uint64_t o) -> uint32_t { return p.slot_ann_len(o); };
  if constexpr (ANN) {  // (ElementParams::stage_ann_offsets, kept as written here so that this kernel's SASS stays)
    for (uint32_t j = 0; j < p.n_types; j++) p.row_ann_off[(uint64_t)j * p.n + s] = ((uint64_t)j * p.n + s) * p.rows_stride;
    if (s + 1 == p.n) p.row_ann_off[kn] = kn * p.rows_stride;
  }
  uint32_t m = 0;
  uint64_t ann_words = 0;  // ANN: the flushed windows' annotations as the append's room check counts them
  for (uint32_t r = 0; r < p.n_slots; r++) {
    const uint64_t o = (uint64_t)r * p.n + s;
    if (p.count[o] != 0 && elem_ends_by(p.start[o], p.resolution, p.target)) {
      m++;
      if constexpr (ANN) {
        const uint32_t l = ann_len(o);
        if (l) ann_words += (l + 3u) / 4u + 4u;
      }
    }
  }
  bool reset = false;
  for (int k = 0; k < M3TSZ_MAX_TRANSFORMS; k++) reset |= ((p.ops >> (4 * k)) & 0xfu) == M3TSZ_TRANSFORM_RESET;
  int32_t status = M3TSZ_OK;
  if (m) {
    // the append's room check before a row's last datapoint, every earlier one at its worst case (163 bits with a
    // time-unit change, m3tsz_encode_bound_units) after an empty encoder's 64-bit start: stream words so far +
    // ENC_GUARD + 4 <= slot words.  ANN: each datapoint's annotation adds (len + 3) / 4 + 4 words to its own check
    // and at most that much to the stream (marker, varint and bytes), so the last check, with every datapoint's
    // annotation words added, bounds all of them.
    const uint64_t per_row = (uint64_t)m * (reset ? 2u : 1u);
    for (uint32_t j = 0; j < p.n_types; j++) {
      const m3tsz_encoder_state &e = p.out_state[(uint64_t)j * p.n + s];
      const uint64_t bits = e.bits + (e.num_encoded ? 0u : 64u) + (per_row - 1) * 163u;
      uint64_t words = (bits >> 5) + ENC_GUARD + 4;
      if constexpr (ANN) words += ann_words * (reset ? 2u : 1u);
      if (words > p.out_slot_words) status = M3TSZ_ERR_CAPACITY;
    }
  }
  if (m == 0 || status != M3TSZ_OK) {
    for (uint32_t j = 0; j < p.n_types; j++) p.row_n[(uint64_t)j * p.n + s] = 0;
    p.status[s] = status;
    return;
  }
  {
    const m3tsz_element_state &r = p.elem[s];
    e.w = r.head;
    e.pv[0] = r.head.prev_v;
    for (int j = 1; j < M3TSZ_MAX_ELEMENT_TYPES; j++) e.pv[j] = r.prev_v_more[j - 1];
  }
  uint64_t rows = 0;  // type j's datapoints so far in bits 8j .. 8j + 7 (at most 2 * M3TSZ_MAX_ELEMENT_WINDOWS)
  int64_t prev = 0;
  for (uint32_t q = 0; q < m; q++) {
    int best = -1;  // the next window in start order (starts are distinct)
    int64_t bs = 0;
    for (uint32_t r = 0; r < p.n_slots; r++) {
      const uint64_t o = (uint64_t)r * p.n + s;
      if (p.count[o] == 0) continue;
      const int64_t ws = p.start[o];
      if (!elem_ends_by(ws, p.resolution, p.target) || (q && ws <= prev)) continue;
      if (best < 0 || ws < bs) {
        best = (int)r;
        bs = ws;
      }
    }
    prev = bs;
    const uint64_t o = (uint64_t)best * p.n + s;
    const int64_t c = p.count[o];
    const int64_t t = bs + p.resolution;  // the window's end
    uint32_t a_len = 0;
    if constexpr (ANN) a_len = ann_len(o);
    // ANN: the entry of staged datapoint d of row `row` (the same window annotation for the Reset datapoint)
    auto stage_ann = [&](uint64_t row, uint64_t d) {
      if constexpr (ANN) p.stage_ann(row, d, o, a_len);
    };
    xf_element_window(
        p.ops, p.resolution, e, 0u, p.n_types, t,
        [&](uint32_t i) {
          uint64_t oi;  // (laundered per type, as in the IN = 5 stage)
          asm volatile("mov.b64 %0, %1;" : "=l"(oi) : "l"(o));
          return tile_value_of(p.tiles, CTR, (int)((p.types >> (4 * i)) & 0xfu), oi, c);
        },
        [&](uint32_t i, double v, int64_t extra_t) {
          if (p.discard_nan && xf_isnan(v)) return;  // nothing of this type's window, its Reset datapoint included
          const uint64_t d = (rows >> (8 * i)) & 0xffu;
          uint64_t at = d * kn + (uint64_t)i * p.n + s;
          p.row_ts[at] = t;
          p.row_val[at] = v;
          stage_ann((uint64_t)i * p.n + s, d);
          if (extra_t != 0) {
            at += kn;
            p.row_ts[at] = extra_t;
            p.row_val[at] = 0.0;
            stage_ann((uint64_t)i * p.n + s, d + 1);
          }
          rows += (uint64_t)(extra_t != 0 ? 2u : 1u) << (8 * i);
        });
    p.count[o] = 0;  // the slot is free
  }
  p.watermark[s] = prev + p.resolution;
  m3tsz_element_state &r = p.elem[s];
  r.head = e.w;
  r.head.prev_v = e.pv[0];
  for (int j = 1; j < M3TSZ_MAX_ELEMENT_TYPES; j++) r.prev_v_more[j - 1] = e.pv[j];
  for (uint32_t j = 0; j < p.n_types; j++) p.row_n[(uint64_t)j * p.n + s] = (uint32_t)((rows >> (8 * j)) & 0xffu);
  p.status[s] = M3TSZ_OK;
}

constexpr int ELEM_THREADS = 256;
template <bool CTR, bool ANN>
__global__ void __launch_bounds__(ELEM_THREADS) element_add_kernel(const ElementParams p) {
  const uint64_t s = (uint64_t)blockIdx.x * ELEM_THREADS + threadIdx.x;
  if (s < p.n) elem_add_lane<CTR, ANN>(p, s);
}
template <bool CTR, bool ANN>
__global__ void __launch_bounds__(ELEM_THREADS) element_consume_kernel(const ElementParams p) {
  __shared__ XfElem rec[ELEM_THREADS];
  const uint64_t s = (uint64_t)blockIdx.x * ELEM_THREADS + threadIdx.x;
  if (s < p.n) elem_consume_lane<CTR, ANN>(p, s, rec[threadIdx.x]);
}
__global__ void element_status_kernel(const int32_t *row_status, uint64_t n, uint32_t n_types, int32_t *status) {
  const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n || status[s] != M3TSZ_OK) return;
  for (uint32_t j = 0; j < n_types; j++) {
    const int32_t st = row_status[(uint64_t)j * n + s];
    if (st != M3TSZ_OK) {
      status[s] = st;
      return;
    }
  }
}

static unsigned elem_blocks(uint64_t n) { return (unsigned)((n + ELEM_THREADS - 1) / ELEM_THREADS); }

cudaError_t launch_element_add(const ElementParams &p, cudaStream_t stream) {
  if (p.n == 0) return cudaSuccess;
  if ((p.n + ELEM_THREADS - 1) / ELEM_THREADS > 0x7fffffffull) return cudaErrorInvalidValue;
  const bool ann = p.ann_len != nullptr;
  if (p.counter && ann)
    element_add_kernel<true, true><<<elem_blocks(p.n), ELEM_THREADS, 0, stream>>>(p);
  else if (p.counter)
    element_add_kernel<true, false><<<elem_blocks(p.n), ELEM_THREADS, 0, stream>>>(p);
  else if (ann)
    element_add_kernel<false, true><<<elem_blocks(p.n), ELEM_THREADS, 0, stream>>>(p);
  else
    element_add_kernel<false, false><<<elem_blocks(p.n), ELEM_THREADS, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_element_consume(const ElementParams &p, cudaStream_t stream) {
  if (p.n == 0) return cudaSuccess;
  if ((p.n + ELEM_THREADS - 1) / ELEM_THREADS > 0x7fffffffull) return cudaErrorInvalidValue;
  const bool ann = p.ann_len != nullptr;
  if (ann && (!p.row_ann_off || !p.row_ann)) return cudaErrorInvalidValue;
  if (p.counter && ann)
    element_consume_kernel<true, true><<<elem_blocks(p.n), ELEM_THREADS, 0, stream>>>(p);
  else if (p.counter)
    element_consume_kernel<true, false><<<elem_blocks(p.n), ELEM_THREADS, 0, stream>>>(p);
  else if (ann)
    element_consume_kernel<false, true><<<elem_blocks(p.n), ELEM_THREADS, 0, stream>>>(p);
  else
    element_consume_kernel<false, false><<<elem_blocks(p.n), ELEM_THREADS, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_element_status(const int32_t *row_status, uint64_t n, uint32_t n_types, int32_t *status,
                                  cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  if ((n + ELEM_THREADS - 1) / ELEM_THREADS > 0x7fffffffull) return cudaErrorInvalidValue;
  element_status_kernel<<<elem_blocks(n), ELEM_THREADS, 0, stream>>>(row_status, n, n_types, status);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------
// Timer element sets (DESIGN.md §4.12): aggregation.Timer over cm.Stream, one lane per element
// ---------------------------------------------------------------------------
// One window slot's cm.Stream (aggregation/quantile/cm/stream.go), its header in registers and its entries in the
// slot's arena: entry i at at(i) = base + i * n.  The list (sampleList) is linked by index; its arena and free list
// are not observable, only the logical list is.  The two pending minHeaps (heap.go) are kept as the reference's
// arrays, pushed and sorted exactly as written there, since where -0 / +0 and NaN land depends on both.  Every
// float -> int64 conversion is Go's (go_f64_to_i64) and every operation is rounded on its own.
struct CmStream {
  m3tsz_timer_stream_header h;
  double *value, *ha, *hb;
  int64_t *nr, *dl;
  int32_t *prv, *nxt;
  uint64_t base, n;
  double eps;
  int32_t every;
  const double *q;
  uint32_t nq;

  __device__ __forceinline__ uint64_t at(int32_t i) const { return base + (uint64_t)i * n; }
  __device__ __forceinline__ double *less() const { return h.less_is_b ? hb : ha; }
  __device__ __forceinline__ double *more() const { return h.less_is_b ? ha : hb; }
  __device__ __forceinline__ int32_t &n_less() { return h.less_is_b ? h.n_b : h.n_a; }
  __device__ __forceinline__ int32_t &n_more() { return h.less_is_b ? h.n_a : h.n_b; }

  // NewStream + ResetSetData: an empty stream
  __device__ __forceinline__ void init() {
    h.num_values = 0;
    h.compress_min_rank = 0;
    h.head = h.tail = h.insert_cursor = h.compress_cursor = -1;
    h.n_samples = h.n_used = 0;
    h.free_head = -1;
    h.counter = 0;
    h.n_a = h.n_b = 0;
    h.less_is_b = 0;
    h.reserved = 0;
  }
  __device__ __forceinline__ int32_t size() const { return h.n_samples + h.n_a + h.n_b; }
  // minHeap.Push: append, then sift up
  __device__ __forceinline__ static void heap_push(double *hp, uint64_t base, uint64_t n, int32_t &len, double v) {
    int32_t i = len++;
    hp[base + (uint64_t)i * n] = v;
    while (i > 0) {
      const int32_t parent = (i - 1) / 2;
      const double pv = hp[base + (uint64_t)parent * n], iv = hp[base + (uint64_t)i * n];
      if (pv <= iv) break;
      hp[base + (uint64_t)parent * n] = iv;
      hp[base + (uint64_t)i * n] = pv;
      i = parent;
    }
  }
  // minHeap.SortDesc: the in-place heapsort (Pop in a loop)
  __device__ __forceinline__ void sort_desc(double *hp, int32_t len) const {
    for (int32_t m = len - 1; m > 0; m--) {
      double t = hp[at(0)];
      hp[at(0)] = hp[at(m)];
      hp[at(m)] = t;
      int32_t i = 0, smallest = 0;
      for (;;) {
        const int32_t left = smallest * 2 + 1, right = left + 1;
        if (left < m && hp[at(left)] < hp[at(smallest)]) smallest = left;
        if (right < m && hp[at(right)] < hp[at(smallest)]) smallest = right;
        if (smallest == i) break;
        t = hp[at(i)];
        hp[at(i)] = hp[at(smallest)];
        hp[at(smallest)] = t;
        i = smallest;
      }
    }
  }
  __device__ __forceinline__ int32_t acquire(double v, int64_t delta) {
    int32_t k;
    if (h.free_head >= 0) {
      k = h.free_head;
      h.free_head = nxt[at(k)];
    } else {
      k = h.n_used++;
    }
    value[at(k)] = v;
    nr[at(k)] = 1;
    dl[at(k)] = delta;
    h.n_samples++;
    return k;
  }
  __device__ __forceinline__ void push_back(int32_t k) {
    prv[at(k)] = h.tail;
    nxt[at(k)] = -1;
    if (h.head < 0)
      h.head = k;
    else
      nxt[at(h.tail)] = k;
    h.tail = k;
  }
  __device__ __forceinline__ void insert_before(int32_t k, int32_t mark) {
    const int32_t p = prv[at(mark)];
    if (p < 0)
      h.head = k;
    else
      nxt[at(p)] = k;
    prv[at(mark)] = k;
    nxt[at(k)] = mark;
    prv[at(k)] = p;
  }
  __device__ __forceinline__ void remove(int32_t k) {
    const int32_t p = prv[at(k)], x = nxt[at(k)];
    nxt[at(k)] = h.free_head;
    h.free_head = k;
    h.n_samples--;
    if (p < 0)
      h.head = x;
    else
      nxt[at(p)] = x;
    if (x < 0)
      h.tail = p;
    else
      prv[at(x)] = p;
  }
  __device__ __forceinline__ void reset_insert_cursor() {
    h.less_is_b ^= 1;
    h.insert_cursor = h.head;
  }
  // the smallest allowed error over the quantile list at `rank` (threshold(); compress's inner loop at maxRank)
  __device__ __forceinline__ int64_t min_threshold(int64_t rank) const {
    int64_t mn = INT64_MAX;
    const int64_t num = h.num_values;
    const double e2 = __dmul_rn(2.0, eps);
    for (uint32_t i = 0; i < nq; i++) {
      int64_t qm;
      if (rank >= go_f64_to_i64(__dmul_rn(q[i], (double)num)))
        qm = go_f64_to_i64(__ddiv_rn(__dmul_rn(e2, (double)rank), q[i]));
      else
        qm = go_f64_to_i64(__ddiv_rn(__dmul_rn(e2, (double)(num - rank)), __dsub_rn(1.0, q[i])));
      if (qm < mn) mn = qm;
    }
    return mn;
  }
  __device__ __forceinline__ void insert() {
    const int32_t cc = h.compress_cursor;
    const double comp_value = cc >= 0 ? value[at(cc)] : xf_bits(0x7ff8000000000001ull);
    double *vals = more();
    const int32_t len = n_more();
    sort_desc(vals, len);
    int32_t idx = len - 1;
    while (h.insert_cursor >= 0 && idx >= 0) {  // (idx < 0 only walks the rest of the list)
      const int32_t curr = h.insert_cursor;
      const double ipv = value[at(curr)];
      while (idx >= 0 && vals[at(idx)] <= ipv) {
        const double v = vals[at(idx)];
        idx--;
        const int32_t k = acquire(v, nr[at(curr)] + dl[at(curr)] - 1);
        insert_before(k, curr);
        if (comp_value >= v) h.compress_min_rank++;
        h.num_values++;
      }
      h.insert_cursor = nxt[at(curr)];
    }
    if (h.insert_cursor < 0) {
      while (idx >= 0 && vals[at(idx)] >= value[at(h.tail)]) {
        const int32_t k = acquire(vals[at(idx)], 0);
        idx--;
        push_back(k);
        h.num_values++;
      }
    }
    n_more() = 0;  // (values left over, a NaN's, are dropped)
    reset_insert_cursor();
  }
  __device__ __forceinline__ void compress() {
    if (h.n_samples < 3) return;
    if (h.compress_cursor < 0) {
      const int32_t c = prv[at(h.tail)];
      h.compress_min_rank = h.num_values - 1 - nr[at(c)];
      h.compress_cursor = prv[at(c)];
    }
    while (h.compress_cursor != h.head) {
      const int32_t curr = h.compress_cursor, next = nxt[at(curr)], prev = prv[at(curr)];
      const int64_t c_nr = nr[at(curr)];
      const int64_t threshold = min_threshold(h.compress_min_rank + c_nr + dl[at(curr)]);
      h.compress_min_rank -= c_nr;
      const int64_t n_nr = nr[at(next)];
      if (c_nr + n_nr + dl[at(next)] <= threshold) {
        if (h.insert_cursor == curr) h.insert_cursor = next;
        nr[at(next)] = n_nr + c_nr;
        remove(curr);
      }
      h.compress_cursor = prev;
    }
    h.compress_cursor = -1;
  }
  // AddBatch of the values v(0) .. v(len - 1)
  template <class V>
  __device__ __forceinline__ void add_batch(uint32_t len, V v) {
    uint32_t i = 0;
    if (h.n_samples == 0) {
      push_back(acquire(v(0), 0));
      h.insert_cursor = h.head;
      h.num_values++;
      i = 1;
    }
    const double ipv = value[at(h.insert_cursor)];  // (read once: stale after an insert inside the batch)
    int32_t counter = h.counter;
    for (; i < len; i++) {
      const double x = v(i);
      if (x < ipv)
        heap_push(less(), base, n, n_less(), x);
      else
        heap_push(more(), base, n, n_more(), x);
      if (counter == every) {
        insert();
        compress();
        counter = 0;
      }
      counter++;
    }
    h.counter = counter;
  }
  // Flush, then calcQuantiles into cq[0 .. nq) (0 where it sets nothing, as a new stream's buffer)
  __device__ __forceinline__ void flush(double *cq, int64_t *rank, int64_t *thr) {
    while (h.n_a > 0 || h.n_b > 0) {
      if (n_more() == 0) reset_insert_cursor();
      insert();
      compress();
    }
    for (uint32_t i = 0; i < nq; i++) cq[i] = 0.0;
    if (nq == 0 || h.num_values == 0) return;
    if (h.num_values <= 3) {  // quantilesFromBuf
      double buf[3];
      int32_t m = 0;
      for (int32_t c = h.head; c >= 0 && m < 3; c = nxt[at(c)]) buf[m++] = value[at(c)];
      for (uint32_t i = 0; i < nq; i++) {
        int64_t k = go_f64_to_i64(__dmul_rn(q[i], (double)m));
        if (k >= m) k = m - 1;
        cq[i] = buf[k];
      }
      return;
    }
    for (uint32_t i = 0; i < nq; i++) {
      rank[i] = go_f64_to_i64(ceil(__dmul_rn(q[i], (double)h.num_values)));
      thr[i] = go_f64_to_i64(ceil(__ddiv_rn((double)min_threshold(rank[i]), 2.0)));
    }
    int64_t min_rank = 0, max_rank = 0;
    uint32_t idx = 0;
    int32_t curr = h.head, prev = h.head;
    while (curr >= 0 && idx < nq) {
      max_rank = min_rank + nr[at(curr)] + dl[at(curr)];
      if (max_rank > rank[idx] + thr[idx] || min_rank > rank[idx]) cq[idx++] = value[at(prev)];
      min_rank += nr[at(curr)];
      prev = curr;
      curr = nxt[at(curr)];
    }
    for (uint32_t i = idx; i < nq; i++)
      if (max_rank >= rank[i] + thr[i] || min_rank > rank[i]) cq[i] = value[at(prev)];
  }
};

__device__ __forceinline__ CmStream timer_stream(const ElementTimerParams &p, uint32_t r, uint64_t s) {
  CmStream c;
  c.value = p.value;
  c.ha = p.heap_a;
  c.hb = p.heap_b;
  c.nr = p.num_ranks;
  c.dl = p.delta;
  c.prv = p.prev;
  c.nxt = p.next;
  c.base = (uint64_t)r * p.cap * p.e.n + s;
  c.n = p.e.n;
  c.eps = p.eps;
  c.every = p.every;
  c.q = p.q;
  c.nq = p.n_q;
  return c;
}

// One amd64 SSE operation's result r = a op b as Go's Timer sees it (its sums take NaN samples, unlike the Gauge's):
// a NaN operand comes through quieted, the first one when both are; an invalid operation on other operands gives
// the default NaN 0xFFF8000000000000.  (The GPU would write its canonical NaN instead.)
__device__ __forceinline__ double amd64_op(double r, double a, double b) {
  if (r == r) return r;
  if (a != a) return __longlong_as_double(__double_as_longlong(a) | 0x0008000000000000ll);
  if (b != b) return __longlong_as_double(__double_as_longlong(b) | 0x0008000000000000ll);
  return __longlong_as_double((long long)0xFFF8000000000000ull);
}
// aggregation.stdev over a Timer's sums, with amd64_op's NaN rule (math.Sqrt of a negative is the default NaN)
__device__ __forceinline__ double timer_stdev(int64_t count, double sum_sq, double sum) {
  const int64_t div = (int64_t)((uint64_t)count * (uint64_t)(count - 1));
  if (div == 0) return 0.0;
  const double cf = __ll2double_rn(count), df = __ll2double_rn(div);
  const double a = amd64_op(__dmul_rn(cf, sum_sq), cf, sum_sq), b = amd64_op(__dmul_rn(sum, sum), sum, sum);
  const double num = amd64_op(__dsub_rn(a, b), a, b);
  const double x = amd64_op(__ddiv_rn(num, df), num, df);
  if (x != x) return x;
  return x < 0.0 ? __longlong_as_double((long long)0xFFF8000000000000ull) : __dsqrt_rn(x);
}

// aggregation.Type.Quantile(): the quantile of a quantile type, 0 for the others
__device__ __forceinline__ double timer_type_quantile(int32_t t) {
  switch (t) {
    case M3TSZ_AGG_P10: return 0.1;
    case M3TSZ_AGG_P20: return 0.2;
    case M3TSZ_AGG_P25: return 0.25;
    case M3TSZ_AGG_P30: return 0.3;
    case M3TSZ_AGG_P40: return 0.4;
    case M3TSZ_AGG_P50: case M3TSZ_AGG_MEDIAN: return 0.5;
    case M3TSZ_AGG_P60: return 0.6;
    case M3TSZ_AGG_P70: return 0.7;
    case M3TSZ_AGG_P75: return 0.75;
    case M3TSZ_AGG_P80: return 0.8;
    case M3TSZ_AGG_P90: return 0.9;
    case M3TSZ_AGG_P95: return 0.95;
    case M3TSZ_AGG_P99: return 0.99;
    case M3TSZ_AGG_P999: return 0.999;
    case M3TSZ_AGG_P9999: return 0.9999;
    default: return 0.0;
  }
}

// Timer.ValueOf of a flushed window: count values, their sum / sumSq, the stream's ends and its quantiles cq
__device__ __forceinline__ double timer_value_of(const ElementTimerParams &p, int32_t t, int64_t cnt, double sum,
                                                 double sq, double front, double back, const double *cq) {
  const double qt = timer_type_quantile(t);
  if (qt > 0.0) {  // Quantile(q): the first listed quantile >= q
    for (uint32_t i = 0; i < p.n_q; i++)
      if (p.q[i] >= qt) return cq[i];
    return xf_bits(0x7ff8000000000001ull);
  }
  switch (t) {
    case M3TSZ_AGG_MIN: return front;
    case M3TSZ_AGG_MAX: return back;
    case M3TSZ_AGG_MEAN: return amd64_op(__ddiv_rn(sum, (double)cnt), sum, (double)cnt);
    case M3TSZ_AGG_COUNT: return (double)cnt;
    case M3TSZ_AGG_SUM: return sum;
    case M3TSZ_AGG_SUMSQ: return sq;
    case M3TSZ_AGG_STDEV: return timer_stdev(cnt, sq, sum);
    default: return 0.0;
  }
}

// Timer.AddBatch of element s's batches in row order (m3tsz_element_set_add_timer).  A first pass checks the batch
// marks; each batch then finds its window's slot (or a free one), checks the slot's room and adds to it.
// ANN (m3tsz_element_set_add_timer_annotated): a batch's annotation is its first row's entry (a BatchTimer has one);
// an entry with a length on a continuation row breaks the batch rule.  An accepted batch with one replaces its
// window's annotation (MaybeReplaceAnnotation, aggregation/timer.go:57-76), kept as in elem_add_lane: a reference
// (a_off, a_len) into the call's bytes for the slot `cur`, copied to the slot when the batches leave it, and only when
// it changed (a window opened here always writes its length).  A batch whose annotation is longer than ann_cap gets
// CAPACITY after the closed and invalid-start checks.
template <bool ANN = false>
__device__ __forceinline__ void elem_timer_add_lane(const ElementTimerParams &tp, uint64_t s) {
  const ElementParams &p = tp.e;
  const uint32_t n_pts = p.n_points ? p.n_points[s] : (uint32_t)p.points_stride;
  if (n_pts > p.points_stride) {
    p.status[s] = M3TSZ_ERR_INVALID_ARG;
    return;
  }
  auto cont = [&](uint32_t i) { return tp.batch && tp.batch[(uint64_t)i * p.n + s] != 0; };
  bool bad = n_pts && cont(0);
  int64_t t0 = 0;
  for (uint32_t i = 0; i < n_pts && !bad; i++) {
    const int64_t t = p.ts[(uint64_t)i * p.n + s];
    if (!cont(i))
      t0 = t;
    else if (t != t0)
      bad = true;
  }
  uint64_t ann_i = 0, ann_end = 0;
  if (ANN && p.ann_series_off) {
    ann_i = p.ann_series_off[s];
    ann_end = p.ann_series_off[s + 1];
    for (uint64_t k = ann_i; k < ann_end && !bad; k++) {
      const m3tsz_annotation_entry &en = p.ann_entries[k];
      bad = en.length != 0 && en.dp_index < n_pts && cont(en.dp_index);
    }
  }
  if (bad) {
    for (uint32_t i = 0; i < n_pts; i++) p.result[(uint64_t)i * p.n + s] = (int8_t)M3TSZ_ERR_INVALID_ARG;
    p.status[s] = M3TSZ_ERR_INVALID_ARG;
    return;
  }
  const int64_t wm = p.watermark[s];
  int32_t status = M3TSZ_OK;
  int cur = -1;  // ANN: the slot whose annotation (a_off, a_len) is held, -1: none
  uint64_t a_off = 0;
  uint32_t a_len = 0;
  bool a_dirty = false;
  uint32_t i = 0;
  while (i < n_pts) {
    uint32_t j = i + 1;
    while (j < n_pts && cont(j)) j++;
    const uint32_t len = j - i;
    int res = M3TSZ_ERR_CAPACITY;
    if (status == M3TSZ_OK) {
      const int64_t t = p.ts[(uint64_t)i * p.n + s];
      int64_t ws = 0;
      uint64_t d_off = 0;  // ANN: this batch's annotation, d_len 0: none
      uint32_t d_len = 0;
      if constexpr (ANN) {
        while (ann_i < ann_end && p.ann_entries[ann_i].dp_index < i) ann_i++;
        if (ann_i < ann_end && p.ann_entries[ann_i].dp_index == i) {
          d_off = p.ann_entries[ann_i].byte_offset;
          d_len = p.ann_entries[ann_i].length;
        }
      }
      if (!elem_window_start(t, p.resolution, p.trunc_off, ws)) {
        res = M3TSZ_ERR_INVALID_ARG;
      } else if (elem_ends_by(ws, p.resolution, wm)) {
        res = M3TSZ_ERR_AGGREGATION_CLOSED;
      } else if (ANN && d_len > p.ann_cap) {
        status = res = M3TSZ_ERR_CAPACITY;
      } else {
        int hit = -1, fr = -1;
        for (uint32_t r = 0; r < p.n_slots; r++) {
          const uint64_t o = (uint64_t)r * p.n + s;
          if (p.count[o] == 0) {
            if (fr < 0) fr = (int)r;
          } else if (p.start[o] == ws) {
            hit = (int)r;
            break;
          }
        }
        const int r = hit >= 0 ? hit : fr;
        CmStream c;
        if (r >= 0) {
          c = timer_stream(tp, (uint32_t)r, s);
          if (hit >= 0)
            c.h = tp.hdr[(uint64_t)r * p.n + s];
          else
            c.init();
        }
        if (r < 0 || (uint64_t)c.size() + len > tp.cap) {
          status = res = M3TSZ_ERR_CAPACITY;
        } else {
          const uint64_t o = (uint64_t)r * p.n + s;
          int64_t cnt = 0;
          double sum = 0.0, sq = 0.0;
          if (hit >= 0) {
            cnt = p.count[o];
            sum = static_cast<const double *>(p.sum)[o];
            sq = static_cast<const double *>(p.sum_sq)[o];
          }
          for (uint32_t k = i; k < j; k++) {
            const double v = p.val[(uint64_t)k * p.n + s];
            sum = amd64_op(__dadd_rn(sum, v), sum, v);
            const double v2 = amd64_op(__dmul_rn(v, v), v, v);
            sq = amd64_op(__dadd_rn(sq, v2), sq, v2);
          }
          c.add_batch(len, [&](uint32_t k) { return p.val[(uint64_t)(i + k) * p.n + s]; });
          p.start[o] = ws;
          p.count[o] = cnt + len;
          static_cast<double *>(p.sum)[o] = sum;
          static_cast<double *>(p.sum_sq)[o] = sq;
          tp.hdr[o] = c.h;
          res = M3TSZ_OK;
          if constexpr (ANN) {
            if (r != cur) {
              if (cur >= 0 && a_dirty) p.store_ann((uint64_t)cur * p.n + s, a_off, a_len);
              cur = r;
              a_len = 0;
              a_dirty = hit < 0;
            }
            if (d_len) {
              a_off = d_off;
              a_len = d_len;
              a_dirty = true;
            }
          }
        }
      }
    }
    for (uint32_t k = i; k < j; k++) p.result[(uint64_t)k * p.n + s] = (int8_t)res;
    i = j;
  }
  if (ANN && cur >= 0 && a_dirty) p.store_ann((uint64_t)cur * p.n + s, a_off, a_len);
  p.status[s] = status;
}

// Consume(target) of Timer element s, as elem_consume_lane: the same room check, window order, staging and commit;
// each due window's stream is flushed and its quantiles computed here.  More than M3TSZ_MAX_ELEMENT_TYPES types come
// without ops: each type's row takes every window's value, and the record is not touched.
// ANN (m3tsz_element_set_consume_timer_annotated): every staged datapoint also gets its window's entry, and the room
// check counts the annotations, both as elem_consume_lane<CTR, true> does.
template <bool ANN = false>
__device__ __forceinline__ void elem_timer_consume_lane(const ElementTimerParams &tp, uint64_t s, XfElem &e) {
  const ElementParams &p = tp.e;
  const uint64_t kn = (uint64_t)tp.n_types * p.n;
  if constexpr (ANN) p.stage_ann_offsets(s, tp.n_types);
  uint32_t m = 0;
  uint64_t ann_words = 0;  // ANN: the flushed windows' annotations as the append's room check counts them
  for (uint32_t r = 0; r < p.n_slots; r++) {
    const uint64_t o = (uint64_t)r * p.n + s;
    if (p.count[o] != 0 && elem_ends_by(p.start[o], p.resolution, p.target)) {
      m++;
      if constexpr (ANN) {
        const uint32_t l = p.slot_ann_len(o);
        if (l) ann_words += (l + 3u) / 4u + 4u;
      }
    }
  }
  bool reset = false;
  for (int k = 0; k < M3TSZ_MAX_TRANSFORMS; k++) reset |= ((p.ops >> (4 * k)) & 0xfu) == M3TSZ_TRANSFORM_RESET;
  int32_t status = M3TSZ_OK;
  if (m) {  // (elem_consume_lane's room check)
    const uint64_t per_row = (uint64_t)m * (reset ? 2u : 1u);
    for (uint32_t j = 0; j < tp.n_types; j++) {
      const m3tsz_encoder_state &oe = p.out_state[(uint64_t)j * p.n + s];
      const uint64_t bits = oe.bits + (oe.num_encoded ? 0u : 64u) + (per_row - 1) * 163u;
      uint64_t words = (bits >> 5) + ENC_GUARD + 4;
      if constexpr (ANN) words += ann_words * (reset ? 2u : 1u);
      if (words > p.out_slot_words) status = M3TSZ_ERR_CAPACITY;
    }
  }
  if (m == 0 || status != M3TSZ_OK) {
    for (uint32_t j = 0; j < tp.n_types; j++) p.row_n[(uint64_t)j * p.n + s] = 0;
    p.status[s] = status;
    return;
  }
  const bool xf = tp.n_types <= M3TSZ_MAX_ELEMENT_TYPES;
  if (xf) {
    const m3tsz_element_state &r = p.elem[s];
    e.w = r.head;
    e.pv[0] = r.head.prev_v;
    for (int j = 1; j < M3TSZ_MAX_ELEMENT_TYPES; j++) e.pv[j] = r.prev_v_more[j - 1];
  }
  uint64_t rows = 0;  // type j's datapoints so far in bits 8j .. 8j + 7 (xf)
  int64_t prev = 0;
  for (uint32_t w = 0; w < m; w++) {
    int best = -1;
    int64_t bs = 0;
    for (uint32_t r = 0; r < p.n_slots; r++) {
      const uint64_t o = (uint64_t)r * p.n + s;
      if (p.count[o] == 0) continue;
      const int64_t ws = p.start[o];
      if (!elem_ends_by(ws, p.resolution, p.target) || (w && ws <= prev)) continue;
      if (best < 0 || ws < bs) {
        best = (int)r;
        bs = ws;
      }
    }
    prev = bs;
    const uint64_t o = (uint64_t)best * p.n + s;
    const int64_t cnt = p.count[o];
    const double sum = static_cast<const double *>(p.sum)[o], sq = static_cast<const double *>(p.sum_sq)[o];
    const int64_t t = bs + p.resolution;
    uint32_t a_len = 0;
    if constexpr (ANN) a_len = p.slot_ann_len(o);
    CmStream c = timer_stream(tp, (uint32_t)best, s);
    c.h = tp.hdr[o];
    double cq[M3TSZ_MAX_TIMER_QUANTILES];
    int64_t rank[M3TSZ_MAX_TIMER_QUANTILES], thr[M3TSZ_MAX_TIMER_QUANTILES];
    c.flush(cq, rank, thr);
    const double front = c.value[c.at(c.h.head)], back = c.value[c.at(c.h.tail)];
    auto value_of = [&](uint32_t i) { return timer_value_of(tp, tp.type[i], cnt, sum, sq, front, back, cq); };
    if (xf) {
      xf_element_window(p.ops, p.resolution, e, 0u, tp.n_types, t, value_of, [&](uint32_t i, double v, int64_t extra_t) {
        if (p.discard_nan && xf_isnan(v)) return;
        const uint64_t d = (rows >> (8 * i)) & 0xffu;
        uint64_t a = d * kn + (uint64_t)i * p.n + s;
        p.row_ts[a] = t;
        p.row_val[a] = v;
        if constexpr (ANN) p.stage_ann((uint64_t)i * p.n + s, d, o, a_len);
        if (extra_t != 0) {
          a += kn;
          p.row_ts[a] = extra_t;
          p.row_val[a] = 0.0;
          if constexpr (ANN) p.stage_ann((uint64_t)i * p.n + s, d + 1, o, a_len);
        }
        rows += (uint64_t)(extra_t != 0 ? 2u : 1u) << (8 * i);
      });
    } else {
      for (uint32_t i = 0; i < tp.n_types; i++) {
        const uint64_t a = (uint64_t)w * kn + (uint64_t)i * p.n + s;
        p.row_ts[a] = t;
        p.row_val[a] = value_of(i);
        if constexpr (ANN) p.stage_ann((uint64_t)i * p.n + s, w, o, a_len);
      }
    }
    p.count[o] = 0;  // the slot is free; its stream is made anew when an add opens it
  }
  p.watermark[s] = prev + p.resolution;
  if (xf) {
    m3tsz_element_state &r = p.elem[s];
    r.head = e.w;
    r.head.prev_v = e.pv[0];
    for (int j = 1; j < M3TSZ_MAX_ELEMENT_TYPES; j++) r.prev_v_more[j - 1] = e.pv[j];
  }
  for (uint32_t j = 0; j < tp.n_types; j++)
    p.row_n[(uint64_t)j * p.n + s] = xf ? (uint32_t)((rows >> (8 * j)) & 0xffu) : m;
  p.status[s] = M3TSZ_OK;
}

// (__maxnreg__ rather than __launch_bounds__: under the latter ptxas held these two at 80 registers and spilled around
// the double-division calls of the stream's thresholds; with 128 neither spills)
template <bool ANN>
__global__ void __maxnreg__(128) element_timer_add_kernel(const ElementTimerParams p) {
  const uint64_t s = (uint64_t)blockIdx.x * ELEM_THREADS + threadIdx.x;
  if (s < p.e.n) elem_timer_add_lane<ANN>(p, s);
}
template <bool ANN>
__global__ void __maxnreg__(128) element_timer_consume_kernel(const ElementTimerParams p) {
  __shared__ XfElem rec[ELEM_THREADS];
  const uint64_t s = (uint64_t)blockIdx.x * ELEM_THREADS + threadIdx.x;
  if (s < p.e.n) elem_timer_consume_lane<ANN>(p, s, rec[threadIdx.x]);
}

cudaError_t launch_element_timer_add(const ElementTimerParams &p, cudaStream_t stream) {
  if (p.e.n == 0) return cudaSuccess;
  if ((p.e.n + ELEM_THREADS - 1) / ELEM_THREADS > 0x7fffffffull) return cudaErrorInvalidValue;
  if (p.e.ann_len)
    element_timer_add_kernel<true><<<elem_blocks(p.e.n), ELEM_THREADS, 0, stream>>>(p);
  else
    element_timer_add_kernel<false><<<elem_blocks(p.e.n), ELEM_THREADS, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_element_timer_consume(const ElementTimerParams &p, cudaStream_t stream) {
  if (p.e.n == 0) return cudaSuccess;
  if ((p.e.n + ELEM_THREADS - 1) / ELEM_THREADS > 0x7fffffffull) return cudaErrorInvalidValue;
  const bool ann = p.e.ann_len != nullptr;
  if (ann && (!p.e.row_ann_off || !p.e.row_ann)) return cudaErrorInvalidValue;
  if (ann)
    element_timer_consume_kernel<true><<<elem_blocks(p.e.n), ELEM_THREADS, 0, stream>>>(p);
  else
    element_timer_consume_kernel<false><<<elem_blocks(p.e.n), ELEM_THREADS, 0, stream>>>(p);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------
// element sets through a rollup (DESIGN.md §4.12): forward, fold, commit
// ---------------------------------------------------------------------------
// Consume(target) of source s of a rollup pipeline (generic_elem.go:912-937): its windows ending at or before
// p.src.target, in start order as elem_consume_lane selects them, each through tile_value_of of the source's one type
// and the pre-ops on the record's head (xf_element_window with one type is xf_window on it; a Reset forwards nothing
// extra).  The q-th window's start and value go to fwd_start / fwd_val at q * n + s, and bit q of fwd_present says
// the value is forwarded (discard_nan drops a NaN with or without ops, as processValue does).  The slots, record and
// watermark stay as they are: the commit frees the due slots (fwd_due) and saves the record (rec) unless a failed
// group holds the source back.
// ANN: a forwarded window whose slot holds an annotation (a length of 1 .. src.ann_cap; above the capacity reads as
// none, as the annotated consume reads it) sets bit q of fwd_ann_present and writes its reference to fwd_ann; the
// slot's bytes stay where they are for the fold to copy.
template <bool CTR, bool ANN = false>
__device__ __forceinline__ void elem_forward_lane(const ElementRollupParams &p, uint64_t s) {
  const ElementParams &e = p.src;
  uint32_t m = 0;
  uint64_t due = 0;
  for (uint32_t r = 0; r < e.n_slots; r++) {
    const uint64_t o = (uint64_t)r * e.n + s;
    if (e.count[o] != 0 && elem_ends_by(e.start[o], e.resolution, e.target)) {
      m++;
      due |= 1ull << r;
    }
  }
  m3tsz_transform_state st = e.elem[s].head;
  uint64_t present = 0;
  int64_t prev = 0;
  for (uint32_t q = 0; q < m; q++) {
    int best = -1;  // the next due window in start order (starts are distinct)
    int64_t bs = 0;
    for (uint32_t r = 0; r < e.n_slots; r++) {
      if (!((due >> r) & 1u)) continue;
      const int64_t ws = e.start[(uint64_t)r * e.n + s];
      if (q && ws <= prev) continue;
      if (best < 0 || ws < bs) {
        best = (int)r;
        bs = ws;
      }
    }
    prev = bs;
    const uint64_t o = (uint64_t)best * e.n + s;
    double v = tile_value_of(e.tiles, CTR, (int)(e.types & 0xfu), o, e.count[o]);
    int64_t extra_t = 0;
    xf_window(e.ops, e.resolution, st, bs + e.resolution, v, extra_t);
    if (!(p.discard_nan && xf_isnan(v))) present |= 1ull << q;
    p.fwd_start[(uint64_t)q * e.n + s] = bs;
    p.fwd_val[(uint64_t)q * e.n + s] = v;
  }
  if constexpr (ANN) {  // (after the windows' loop, so that nothing more lives across xf_window's calls; the pass of
                        // ElementRollupParams::forward_ann, kept as written here so that this kernel's SASS stays)
    uint64_t ann = 0;
    for (uint32_t r = 0; r < e.n_slots; r++) {
      if (!((due >> r) & 1u)) continue;
      const uint64_t o = (uint64_t)r * e.n + s;
      const uint32_t l = e.ann_len[o];
      if (l == 0 || l > e.ann_cap) continue;
      const int64_t ws = e.start[o];
      uint32_t q = 0;  // the window's place in start order
      for (uint32_t r2 = 0; r2 < e.n_slots; r2++) q += ((due >> r2) & 1u) && e.start[(uint64_t)r2 * e.n + s] < ws;
      if (!((present >> q) & 1u)) continue;
      ann |= 1ull << q;
      p.fwd_ann[(uint64_t)q * e.n + s] = (o << 17) | l;
    }
    p.fwd_ann_present[s] = ann;
  }
  p.fwd_n[s] = m;
  p.fwd_present[s] = present;
  p.fwd_due[s] = due;
  p.rec[s] = st;
}

// A group window while the fold holds it: its start and the rollup fold's accumulator (every value arrives at one
// timestamp, so rollup_gauge_add / rollup_counter_add: the first value is Last, NaNs are counted, sums wrap), loaded
// from and stored to the slot form elem_store writes (a Gauge window without a non-NaN value has min = max =
// math.NaN(), which is the fold's own empty form; last_at is the window's end, where the values arrive)
template <bool CTR>
struct ElemFoldAcc {
  using A = std::conditional_t<CTR, RollupCounterAcc, RollupGaugeAcc>;
  int64_t start;
  A a;
  // the annotated fold's group window annotation to group slot o (ElementRollupParams::store_group_ann)
  __device__ static __forceinline__ void store_ann(const ElementRollupParams &p, uint64_t o, uint64_t ref,
                                                   uint32_t lane, uint32_t n_lanes) {
    p.store_group_ann(o, ref, lane, n_lanes);
  }
};
template <bool CTR>
__device__ __forceinline__ void elem_fold_load(const ElementRollupParams &p, uint64_t o, ElemFoldAcc<CTR> &f) {
  f.start = p.g_start[o];
  f.a.cnt = p.g_count[o];
  if constexpr (CTR) {
    f.a.sum = static_cast<const int64_t *>(p.g_sum)[o];
    f.a.mn = static_cast<const int64_t *>(p.g_min)[o];
    f.a.mx = static_cast<const int64_t *>(p.g_max)[o];
    f.a.sq = static_cast<const int64_t *>(p.g_sum_sq)[o];
  } else {
    f.a.sum = static_cast<const double *>(p.g_sum)[o];
    f.a.mn = static_cast<const double *>(p.g_min)[o];
    f.a.mx = static_cast<const double *>(p.g_max)[o];
    f.a.sq = static_cast<const double *>(p.g_sum_sq)[o];
    f.a.last = p.g_last[o];
  }
}
template <bool CTR>
__device__ __forceinline__ void elem_fold_store(const ElementRollupParams &p, uint64_t o, const ElemFoldAcc<CTR> &f) {
  using V = std::conditional_t<CTR, int64_t, double>;
  p.g_start[o] = f.start;
  p.g_count[o] = f.a.cnt;
  static_cast<V *>(p.g_sum)[o] = f.a.sum;
  static_cast<V *>(p.g_min)[o] = f.a.mn;
  static_cast<V *>(p.g_max)[o] = f.a.mx;
  static_cast<V *>(p.g_sum_sq)[o] = f.a.sq;
  if constexpr (!CTR) {
    p.g_last[o] = f.a.last;
    p.g_last_at[o] = (int64_t)((uint64_t)f.start + (uint64_t)p.src.resolution);
  }
}

// What the fold reads of the member at one listed position: its source index, its due windows, which of them are
// forwarded, and its first due window's start and value (later ones are read from fwd_start / fwd_val); ANN: which
// forwarded windows carry an annotation (their references are read from fwd_ann, those windows' only)
struct FwdMember {
  uint64_t m;  // >= src.n: an invalid index (n = 0)
  uint32_t n;
  uint64_t present;
  int64_t start0;
  double val0;
  uint64_t ann;
};
template <bool ANN = false>
__device__ __forceinline__ FwdMember fwd_member(const ElementRollupParams &p, uint64_t i) {
  FwdMember a;
  a.m = p.members[i];
  a.n = 0;
  a.present = 0;
  a.start0 = 0;
  a.val0 = 0.0;
  a.ann = 0;
  if (a.m < p.src.n) {
    a.n = p.fwd_n[a.m];
    a.present = p.fwd_present[a.m];
    if constexpr (ANN) a.ann = p.fwd_ann_present[a.m];
    if (a.n) {
      a.start0 = p.fwd_start[a.m];
      a.val0 = p.fwd_val[a.m];
    }
  }
  return a;
}

// AddUnique of group g's members in listed order (generic_elem.go:246-281), each member's forwarded windows in start
// order, into the group window with the source window's start.  member(i) gives listed position i (lo <= i < hi),
// asked for in order.  First a pass that checks the range and the indices (INVALID_ARG) and counts the group's new
// windows against its free slots (CAPACITY): a failed group changes nothing.  Then the fold, the current window in
// registers (it goes back to its slot when a value needs another one, and at the end); a window that ends at or
// before the group's watermark is dropped (AGGREGATION_CLOSED, the other windows still fold).  fresh: room for
// g_slots starts.  Returns the group's status (also written to group_status[g]).
// ANN: MaybeReplaceAnnotation through AddUnique (generic_elem.go:278-281): each folded value whose window carries an
// annotation makes it its group window's, kept in registers as the forward's reference beside the accumulator.  It goes
// to the slot with the window when it changed: a window opened here always writes its length (0 without one), one
// already open keeps its annotation unless a value replaced it.  The first pass also fails the group with CAPACITY
// for an annotation longer than g_ann_cap on a value that would fold.  The lanes lane .. of n_lanes split a copy.
template <bool CTR, bool ANN = false, class Member>
__device__ __forceinline__ int32_t elem_fold_group(const ElementRollupParams &p, uint64_t g, int64_t *fresh,
                                                   Member member, uint32_t lane = 0, uint32_t n_lanes = 1) {
  const uint64_t lo = p.group_off[g], hi = p.group_off[g + 1], G = p.n_groups;
  const int64_t res = p.src.resolution, wm = p.g_watermark[g];
  int32_t status = M3TSZ_OK;
  // ANN: the reference of member a's q-th window (its bit of a.ann set)
  auto ann_ref = [&](const FwdMember &a, uint32_t q) { return p.fwd_ann[(uint64_t)q * p.src.n + a.m]; };
  auto window = [&](const FwdMember &a, uint32_t q, int64_t &ws, double &v) {
    if (q == 0) {
      ws = a.start0;
      v = a.val0;
    } else {
      ws = p.fwd_start[(uint64_t)q * p.src.n + a.m];
      v = p.fwd_val[(uint64_t)q * p.src.n + a.m];
    }
  };
  if (lo > hi || hi > p.n_members) {
    status = M3TSZ_ERR_INVALID_ARG;
  } else {
    uint32_t n_free = 0, n_fresh = 0;
    for (uint32_t r = 0; r < p.g_slots; r++) n_free += p.g_count[(uint64_t)r * G + g] == 0;
    bool bad = false, full = false, seen = false;
    int64_t last = 0;  // the last start checked (a group's values mostly go to one window)
    for (uint64_t i = lo; i < hi; i++) {
      const FwdMember a = member(i);
      if (a.m >= p.src.n) bad = true;
      for (uint32_t q = 0; q < a.n; q++) {
        if (!((a.present >> q) & 1u)) continue;
        int64_t ws;
        double v;
        window(a, q, ws, v);
        if constexpr (ANN) {
          if (((a.ann >> q) & 1u) && !elem_ends_by(ws, res, wm) && (ann_ref(a, q) & 0x1ffffu) > p.g_ann_cap)
            full = true;
        }
        if ((seen && ws == last) || elem_ends_by(ws, res, wm)) continue;
        seen = true;
        last = ws;
        bool known = false;
        for (uint32_t r = 0; r < p.g_slots && !known; r++) {
          const uint64_t o = (uint64_t)r * G + g;
          known = p.g_count[o] != 0 && p.g_start[o] == ws;
        }
        for (uint32_t k = 0; k < n_fresh && !known; k++) known = fresh[k] == ws;
        if (known) continue;
        if (n_fresh < n_free)
          fresh[n_fresh++] = ws;
        else
          full = true;
      }
    }
    status = bad ? M3TSZ_ERR_INVALID_ARG : full ? M3TSZ_ERR_CAPACITY : M3TSZ_OK;
  }
  if (status == M3TSZ_OK) {
    ElemFoldAcc<CTR> f;
    int cur = -1;  // the slot `f` belongs to, -1: none
    bool closed = false;
    uint64_t a_ref = 0;  // ANN: the window's annotation taken in this call (0: none), and whether its slot needs it
    bool a_dirty = false;
    for (uint64_t i = lo; i < hi; i++) {
      const FwdMember a = member(i);
      for (uint32_t q = 0; q < a.n; q++) {
        if (!((a.present >> q) & 1u)) continue;
        int64_t ws;
        double v;
        window(a, q, ws, v);
        if (elem_ends_by(ws, res, wm)) {
          closed = true;
          continue;
        }
        if (cur < 0 || ws != f.start) {  // the window's slot, or a free one (the first pass counted them)
          if (cur >= 0) {
            elem_fold_store(p, (uint64_t)cur * G + g, f);
            if (ANN && a_dirty) ElemFoldAcc<CTR>::store_ann(p, (uint64_t)cur * G + g, a_ref, lane, n_lanes);
          }
          int hit = -1, fr = -1;
          for (uint32_t r = 0; r < p.g_slots; r++) {
            const uint64_t o = (uint64_t)r * G + g;
            if (p.g_count[o] == 0) {
              if (fr < 0) fr = (int)r;
            } else if (p.g_start[o] == ws) {
              hit = (int)r;
              break;
            }
          }
          cur = hit >= 0 ? hit : fr;
          if (hit >= 0) {
            elem_fold_load(p, (uint64_t)hit * G + g, f);
          } else {
            f.start = ws;
            if constexpr (CTR)
              rollup_counter_init(f.a);
            else
              rollup_gauge_init(f.a);
          }
          a_ref = 0;
          a_dirty = hit < 0;
        }
        if constexpr (CTR)
          rollup_counter_add(f.a, v);
        else
          rollup_gauge_add(f.a, v);
        if (ANN && ((a.ann >> q) & 1u)) {
          a_ref = ann_ref(a, q);
          a_dirty = true;
        }
      }
    }
    if (cur >= 0) {
      elem_fold_store(p, (uint64_t)cur * G + g, f);
      if (ANN && a_dirty) ElemFoldAcc<CTR>::store_ann(p, (uint64_t)cur * G + g, a_ref, lane, n_lanes);
    }
    if (closed) status = M3TSZ_ERR_AGGREGATION_CLOSED;
  }
  p.group_status[g] = status;
  return status;
}

// The commit of source s: a source that a failed group holds back (mark[s], that group's status) keeps its windows,
// record and watermark; every other one frees its due slots, saves its new record and moves its watermark to the last
// due window's end
__device__ __forceinline__ void elem_commit_lane(const ElementRollupParams &p, uint64_t s) {
  const int32_t mk = p.mark[s];
  p.src_status[s] = mk;
  const uint32_t m = p.fwd_n[s];
  if (mk != 0 || m == 0) return;
  const uint64_t due = p.fwd_due[s];
  for (uint32_t r = 0; r < p.src.n_slots; r++)
    if ((due >> r) & 1u) p.src.count[(uint64_t)r * p.src.n + s] = 0;
  p.src.watermark[s] = p.fwd_start[(uint64_t)(m - 1) * p.src.n + s] + p.src.resolution;
  p.src.elem[s].head = p.rec[s];
}

template <bool CTR, bool ANN>
__global__ void __launch_bounds__(ELEM_THREADS) element_forward_kernel(const ElementRollupParams p) {
  const uint64_t s = (uint64_t)blockIdx.x * ELEM_THREADS + threadIdx.x;
  if (s < p.src.n) elem_forward_lane<CTR, ANN>(p, s);
}

// One warp per group.  The lanes gather 32 listed members at a time (their indices as one coalesced load, their due
// counts, presence words and first forwarded windows as one gather); every lane then runs the group's fold on the
// same values, shuffled from the lane that loaded them, so the fold is in listed order and its branches are uniform.
// The lanes' stores to the group's slots are of equal values.  A group that failed with CAPACITY or INVALID_ARG marks
// the members its range names for the commit.  ANN: the presence words carry the annotation words with them, and the
// lanes split each annotation copy.
constexpr int ELEM_FOLD_WARPS = 8;
template <bool CTR, bool ANN>
__global__ void __launch_bounds__(ELEM_FOLD_WARPS * 32) element_fold_kernel(const ElementRollupParams p) {
  __shared__ int64_t fresh[ELEM_FOLD_WARPS][M3TSZ_MAX_ELEMENT_WINDOWS];
  const uint32_t lane = threadIdx.x & 31u, wi = threadIdx.x >> 5;
  const uint64_t g = (uint64_t)blockIdx.x * ELEM_FOLD_WARPS + wi;
  if (g >= p.n_groups) return;
  const uint64_t lo = p.group_off[g], hi = p.group_off[g + 1];
  uint64_t base = ~0ull;
  FwdMember mine;
  auto member = [&](uint64_t i) {
    const uint64_t b = lo + ((i - lo) & ~31ull);
    if (b != base) {
      base = b;
      mine.m = ~0ull;
      mine.n = 0;
      mine.present = 0;
      mine.start0 = 0;
      mine.val0 = 0.0;
      mine.ann = 0;
      if (b + lane < hi) mine = fwd_member<ANN>(p, b + lane);
    }
    const int j = (int)((i - lo) & 31u);
    FwdMember a;
    a.m = __shfl_sync(FULL_MASK, mine.m, j);
    a.n = __shfl_sync(FULL_MASK, mine.n, j);
    a.present = __shfl_sync(FULL_MASK, mine.present, j);
    a.start0 = __shfl_sync(FULL_MASK, mine.start0, j);
    a.val0 = __shfl_sync(FULL_MASK, mine.val0, j);
    a.ann = 0;
    if constexpr (ANN) a.ann = __shfl_sync(FULL_MASK, mine.ann, j);
    return a;
  };
  const int32_t st = elem_fold_group<CTR, ANN>(p, g, fresh[wi], member, lane, 32u);
  if ((st == M3TSZ_ERR_CAPACITY || st == M3TSZ_ERR_INVALID_ARG) && lo <= hi) {
    const uint64_t end = hi < p.n_members ? hi : p.n_members;
    for (uint64_t i = lo + lane; i < end; i += 32) {
      const uint32_t m = p.members[i];
      if (m < p.src.n) atomicMax(p.mark + m, st);
    }
  }
}

__global__ void __launch_bounds__(ELEM_THREADS) element_commit_kernel(const ElementRollupParams p) {
  const uint64_t s = (uint64_t)blockIdx.x * ELEM_THREADS + threadIdx.x;
  if (s < p.src.n) elem_commit_lane(p, s);
}

cudaError_t launch_element_forward(const ElementRollupParams &p, cudaStream_t stream) {
  if (p.src.n == 0) return cudaSuccess;
  if ((p.src.n + ELEM_THREADS - 1) / ELEM_THREADS > 0x7fffffffull) return cudaErrorInvalidValue;
  const bool ann = p.src.ann_len != nullptr;
  if (ann && (!p.fwd_ann_present || !p.fwd_ann)) return cudaErrorInvalidValue;
  if (p.src.counter && ann)
    element_forward_kernel<true, true><<<elem_blocks(p.src.n), ELEM_THREADS, 0, stream>>>(p);
  else if (p.src.counter)
    element_forward_kernel<true, false><<<elem_blocks(p.src.n), ELEM_THREADS, 0, stream>>>(p);
  else if (ann)
    element_forward_kernel<false, true><<<elem_blocks(p.src.n), ELEM_THREADS, 0, stream>>>(p);
  else
    element_forward_kernel<false, false><<<elem_blocks(p.src.n), ELEM_THREADS, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_element_fold(const ElementRollupParams &p, cudaStream_t stream) {
  if (p.n_groups == 0) return cudaSuccess;
  const uint64_t blocks = (p.n_groups + ELEM_FOLD_WARPS - 1) / ELEM_FOLD_WARPS;
  if (blocks > 0x7fffffffull) return cudaErrorInvalidValue;
  const bool ann = p.src.ann_len != nullptr;
  if (ann && (!p.fwd_ann_present || !p.fwd_ann || !p.g_ann_len || !p.g_ann_slot)) return cudaErrorInvalidValue;
  if (p.src.counter && ann)
    element_fold_kernel<true, true><<<(unsigned)blocks, ELEM_FOLD_WARPS * 32, 0, stream>>>(p);
  else if (p.src.counter)
    element_fold_kernel<true, false><<<(unsigned)blocks, ELEM_FOLD_WARPS * 32, 0, stream>>>(p);
  else if (ann)
    element_fold_kernel<false, true><<<(unsigned)blocks, ELEM_FOLD_WARPS * 32, 0, stream>>>(p);
  else
    element_fold_kernel<false, false><<<(unsigned)blocks, ELEM_FOLD_WARPS * 32, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_element_commit(const ElementRollupParams &p, cudaStream_t stream) {
  if (p.src.n == 0) return cudaSuccess;
  if ((p.src.n + ELEM_THREADS - 1) / ELEM_THREADS > 0x7fffffffull) return cudaErrorInvalidValue;
  element_commit_kernel<<<elem_blocks(p.src.n), ELEM_THREADS, 0, stream>>>(p);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------
// element-set rollups across shards (DESIGN.md §4.12): the forwarded writer and AddUnique of its records
// ---------------------------------------------------------------------------
// The smallest forwarded window start of group g's members above `prev` (have: a start was found before); each
// member's forwarded starts ascend with q, so a member's first start above prev is its candidate
__device__ __forceinline__ bool fw_next_start(const ElementRollupParams &p, uint64_t lo, uint64_t hi, bool have,
                                              int64_t prev, int64_t &next) {
  bool found = false;
  for (uint64_t i = lo; i < hi; i++) {
    const uint64_t m = p.members[i];
    const uint32_t n = p.fwd_n[m];
    const uint64_t pr = p.fwd_present[m];
    for (uint32_t q = 0; q < n; q++) {
      if (!((pr >> q) & 1u)) continue;
      const int64_t ws = p.fwd_start[(uint64_t)q * p.src.n + m];
      if (have && ws <= prev) continue;
      if (!found || ws < next) next = ws;
      found = true;
      break;
    }
  }
  return found;
}

// Group g's range and member checks (INVALID_ARG: no records), its record count (distinct forwarded starts) and value
// count (forwarded values)
__device__ __forceinline__ void fw_count_group(const ElementForwardedParams &p, uint64_t g) {
  const ElementRollupParams &rp = p.rp;
  const uint64_t lo = rp.group_off[g], hi = rp.group_off[g + 1];
  bool bad = lo > hi || hi > rp.n_members;
  uint64_t nv = 0;
  for (uint64_t i = lo; i < hi && !bad; i++) {
    const uint64_t m = rp.members[i];
    if (m >= rp.src.n) {
      bad = true;
    } else {
      const uint32_t n = rp.fwd_n[m];
      nv += __popcll(rp.fwd_present[m] & (n >= 64 ? ~0ull : ((1ull << n) - 1)));
    }
  }
  uint64_t nr = 0;
  if (!bad) {
    int64_t ws = 0, nx = 0;
    while (fw_next_start(rp, lo, hi, nr != 0, ws, nx)) {
      ws = nx;
      nr++;
    }
  } else {
    nv = 0;
  }
  p.n_rec[g] = nr;
  p.n_val[g] = nv;
  rp.group_status[g] = bad ? M3TSZ_ERR_INVALID_ARG : M3TSZ_OK;
}
__global__ void __launch_bounds__(ELEM_THREADS) forward_write_count_kernel(const ElementForwardedParams p) {
  const uint64_t g = (uint64_t)blockIdx.x * ELEM_THREADS + threadIdx.x;
  if (g < p.rp.n_groups) fw_count_group(p, g);
}

// A valid group that fits (its records and values end within the capacities) writes them at its scanned offsets; a
// later one gets CAPACITY.  The last group that fits writes the written counts, the last group the needed ones (the
// caller zeroes `counts`).  Returns the group's status (also written to group_status[g]).
__device__ __forceinline__ int32_t fw_write_group(const ElementForwardedParams &p, uint64_t g) {
  const ElementRollupParams &rp = p.rp;
  const uint64_t G = rp.n_groups;
  const uint64_t rec_end = p.rec_off[g] + p.n_rec[g], val_end = p.val_off[g] + p.n_val[g];
  const bool fit = rec_end <= p.rec_cap && val_end <= p.val_cap;
  // (the next group's offsets are this group's ends: it fits when its own ends do)
  if (fit && (g + 1 == G || p.rec_off[g + 1] + p.n_rec[g + 1] > p.rec_cap ||
              p.val_off[g + 1] + p.n_val[g + 1] > p.val_cap)) {
    p.counts[0] = rec_end;
    p.counts[1] = val_end;
  }
  if (g + 1 == G) {
    p.counts[2] = rec_end;
    p.counts[3] = val_end;
  }
  const uint64_t lo = rp.group_off[g], hi = rp.group_off[g + 1];
  int32_t st = rp.group_status[g];
  if (st == M3TSZ_OK && !fit) st = M3TSZ_ERR_CAPACITY;
  if (st == M3TSZ_OK) {
    uint64_t r = p.rec_off[g], v = p.val_off[g];
    int64_t ws = 0, nx = 0;
    bool have = false;
    while (fw_next_start(rp, lo, hi, have, ws, nx)) {
      ws = nx;
      have = true;
      const uint64_t v0 = v;
      for (uint64_t i = lo; i < hi; i++) {
        const uint64_t m = rp.members[i];
        const uint32_t n = rp.fwd_n[m];
        const uint64_t pr = rp.fwd_present[m];
        for (uint32_t q = 0; q < n; q++) {
          const int64_t s = rp.fwd_start[(uint64_t)q * rp.src.n + m];
          if (s > ws) break;
          if (s == ws && ((pr >> q) & 1u)) p.out_val[v++] = rp.fwd_val[(uint64_t)q * rp.src.n + m];
        }
      }
      m3tsz_forwarded_metric &f = p.out_rec[r++];
      f.key = p.group_key ? p.group_key[g] : g;
      f.time_ns = (int64_t)((uint64_t)ws + (uint64_t)rp.src.resolution);
      f.value_off = v0;
      f.n_values = (uint32_t)(v - v0);
      f.source_id = p.source_id;
      f.version = 0;
      f.reserved = 0;
    }
  }
  rp.group_status[g] = st;
  return st;
}
// A failed group marks its members for the commit.
__global__ void __launch_bounds__(ELEM_THREADS) forward_write_kernel(const ElementForwardedParams p) {
  const uint64_t g = (uint64_t)blockIdx.x * ELEM_THREADS + threadIdx.x;
  const ElementRollupParams &rp = p.rp;
  if (g >= rp.n_groups) return;
  const int32_t st = fw_write_group(p, g);
  const uint64_t lo = rp.group_off[g], hi = rp.group_off[g + 1];
  if (st != M3TSZ_OK && lo <= hi) {
    const uint64_t end = hi < rp.n_members ? hi : rp.n_members;
    for (uint64_t i = lo; i < end; i++) {
      const uint32_t m = rp.members[i];
      if (m < rp.src.n) atomicMax(rp.mark + m, st);
    }
  }
}

// The radix sort's inputs: record i's element (n for an invalid key) and its index
__global__ void __launch_bounds__(ELEM_THREADS) add_forwarded_prep_kernel(const ElementForwardedParams p) {
  const uint64_t i = (uint64_t)blockIdx.x * ELEM_THREADS + threadIdx.x;
  if (i >= p.n_recs) return;
  const uint64_t k = p.rec[i].key, n = p.rp.n_groups;
  p.sort_key[i] = k < n ? k : n;
  p.sort_idx[i] = i;
}

// AddUnique of element e's records (sorted positions j .. while the key is e), in array order.  The window the last
// record went to stays in registers (elem_fold_load / elem_fold_store), as in the fold; a new window's source bits are
// zeroed when it is opened.
template <bool CTR>
__device__ __forceinline__ void add_forwarded_lane(const ElementForwardedParams &p, uint64_t j) {
  const ElementRollupParams &rp = p.rp;
  const uint64_t e = p.sorted_key[j], G = rp.n_groups;
  if (e >= G) {
    for (; j < p.n_recs && p.sorted_key[j] == e; j++) p.result[p.sorted_idx[j]] = (int8_t)M3TSZ_ERR_INVALID_ARG;
    return;
  }
  const int64_t res = rp.src.resolution, wm = rp.g_watermark[e];
  const uint32_t W = p.bit_words;
  ElemFoldAcc<CTR> f;
  int cur = -1;
  int32_t status = M3TSZ_OK;
  for (; j < p.n_recs && p.sorted_key[j] == e; j++) {
    const uint64_t i = p.sorted_idx[j];
    const m3tsz_forwarded_metric m = p.rec[i];
    int r = M3TSZ_ERR_CAPACITY;  // (after a CAPACITY, the rest of the element's records)
    if (status == M3TSZ_OK) {
      int64_t t0 = 0;
      if (m.n_values == 0 || m.value_off > p.n_vals || m.n_values > p.n_vals - m.value_off || m.version != 0 ||
          m.reserved != 0 || !elem_window_start(m.time_ns, res, p.trunc_off, t0) ||
          t0 < (int64_t)0x8000000000000000ull + res) {
        r = M3TSZ_ERR_INVALID_ARG;
      } else if (elem_ends_by(t0 - res, res, wm)) {
        r = M3TSZ_ERR_AGGREGATION_CLOSED;
      } else if (m.source_id >= W * 32u) {
        status = r = M3TSZ_ERR_CAPACITY;
      } else {
        const int64_t ws = t0 - res;
        r = M3TSZ_OK;
        if (cur < 0 || ws != f.start) {  // the window's slot, or a free one
          int hit, fr;
          rp.group_slot(e, cur, ws, hit, fr);
          if (hit < 0 && fr < 0) {
            status = r = M3TSZ_ERR_CAPACITY;
          } else {
            if (cur >= 0) elem_fold_store(rp, (uint64_t)cur * G + e, f);
            cur = hit >= 0 ? hit : fr;
            if (hit >= 0) {
              elem_fold_load(rp, (uint64_t)hit * G + e, f);
            } else {
              f.start = ws;
              if constexpr (CTR)
                rollup_counter_init(f.a);
              else
                rollup_gauge_init(f.a);
              for (uint32_t w = 0; w < W; w++) p.bits[((uint64_t)cur * W + w) * G + e] = 0u;
            }
          }
        }
        if (r == M3TSZ_OK) {
          uint32_t *word = p.bits + ((uint64_t)cur * W + (m.source_id >> 5)) * G + e;
          const uint32_t bit = 1u << (m.source_id & 31u);
          if (*word & bit) {
            r = M3TSZ_ERR_DUPLICATE_SOURCE;
          } else {
            *word |= bit;
            for (uint32_t k = 0; k < m.n_values; k++) {
              const double v = p.val[m.value_off + k];
              if constexpr (CTR)
                rollup_counter_add(f.a, v);
              else
                rollup_gauge_add(f.a, v);
            }
          }
        }
      }
    }
    p.result[i] = (int8_t)r;
  }
  if (cur >= 0) elem_fold_store(rp, (uint64_t)cur * G + e, f);
  p.status[e] = status;
}

template <bool CTR>
__global__ void __launch_bounds__(ELEM_THREADS) add_forwarded_kernel(const ElementForwardedParams p) {
  const uint64_t j = (uint64_t)blockIdx.x * ELEM_THREADS + threadIdx.x;
  if (j >= p.n_recs || (j && p.sorted_key[j - 1] == p.sorted_key[j])) return;  // one lane per element with records
  add_forwarded_lane<CTR>(p, j);
}

cudaError_t launch_forward_write_count(const ElementForwardedParams &p, cudaStream_t stream) {
  if (p.rp.n_groups == 0) return cudaSuccess;
  if ((p.rp.n_groups + ELEM_THREADS - 1) / ELEM_THREADS > 0x7fffffffull) return cudaErrorInvalidValue;
  forward_write_count_kernel<<<elem_blocks(p.rp.n_groups), ELEM_THREADS, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_forward_write(const ElementForwardedParams &p, cudaStream_t stream) {
  if (p.rp.n_groups == 0) return cudaSuccess;
  if ((p.rp.n_groups + ELEM_THREADS - 1) / ELEM_THREADS > 0x7fffffffull) return cudaErrorInvalidValue;
  forward_write_kernel<<<elem_blocks(p.rp.n_groups), ELEM_THREADS, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_add_forwarded_prep(const ElementForwardedParams &p, cudaStream_t stream) {
  if (p.n_recs == 0) return cudaSuccess;
  if ((p.n_recs + ELEM_THREADS - 1) / ELEM_THREADS > 0x7fffffffull) return cudaErrorInvalidValue;
  add_forwarded_prep_kernel<<<elem_blocks(p.n_recs), ELEM_THREADS, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_add_forwarded(const ElementForwardedParams &p, cudaStream_t stream) {
  if (p.n_recs == 0) return cudaSuccess;
  if ((p.n_recs + ELEM_THREADS - 1) / ELEM_THREADS > 0x7fffffffull) return cudaErrorInvalidValue;
  if (p.rp.src.counter)
    add_forwarded_kernel<true><<<elem_blocks(p.n_recs), ELEM_THREADS, 0, stream>>>(p);
  else
    add_forwarded_kernel<false><<<elem_blocks(p.n_recs), ELEM_THREADS, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t forward_write_scan(void *tmp, size_t &bytes, const uint64_t *in, uint64_t *out, uint64_t n,
                               cudaStream_t stream) {
  return cub::DeviceScan::ExclusiveSum(tmp, bytes, in, out, n, stream);
}

cudaError_t add_forwarded_sort(void *tmp, size_t &bytes, const uint64_t *key_in, uint64_t *key_out,
                               const uint64_t *idx_in, uint64_t *idx_out, uint64_t n, int end_bit,
                               cudaStream_t stream) {
  return cub::DeviceRadixSort::SortPairs(tmp, bytes, key_in, key_out, idx_in, idx_out, n, 0, end_bit, stream);
}

// ---------------------------------------------------------------------------
// Timer element sets through a rollup (DESIGN.md §4.12): the Timer forward and fold; the commit is the one above
// ---------------------------------------------------------------------------
// elem_forward_lane for Timer source s (tp: the source set's streams, tp.e = p.src): the same due windows in start
// order and scratch, each window's value Flush + ValueOf(tp.type[0]) as elem_timer_consume_lane computes it, through
// the pre-ops on the record's head.  Each flushed header goes back to its slot: the flush rewrote the slot's arena, and
// a source held back keeps the flushed stream (a second Flush, its heaps empty, gives the same quantiles).
// ANN: the annotated forward's reference pass (ElementRollupParams::forward_ann), after the windows' loop.
template <bool ANN = false>
__device__ __forceinline__ void elem_timer_forward_lane(const ElementRollupParams &p, const ElementTimerParams &tp,
                                                        uint64_t s) {
  const ElementParams &e = p.src;
  uint32_t m = 0;
  uint64_t due = 0;
  for (uint32_t r = 0; r < e.n_slots; r++) {
    const uint64_t o = (uint64_t)r * e.n + s;
    if (e.count[o] != 0 && elem_ends_by(e.start[o], e.resolution, e.target)) {
      m++;
      due |= 1ull << r;
    }
  }
  m3tsz_transform_state st = e.elem[s].head;
  uint64_t present = 0;
  int64_t prev = 0;
  for (uint32_t q = 0; q < m; q++) {
    int best = -1;
    int64_t bs = 0;
    for (uint32_t r = 0; r < e.n_slots; r++) {
      if (!((due >> r) & 1u)) continue;
      const int64_t ws = e.start[(uint64_t)r * e.n + s];
      if (q && ws <= prev) continue;
      if (best < 0 || ws < bs) {
        best = (int)r;
        bs = ws;
      }
    }
    prev = bs;
    const uint64_t o = (uint64_t)best * e.n + s;
    CmStream c = timer_stream(tp, (uint32_t)best, s);
    c.h = tp.hdr[o];
    double cq[M3TSZ_MAX_TIMER_QUANTILES];
    int64_t rank[M3TSZ_MAX_TIMER_QUANTILES], thr[M3TSZ_MAX_TIMER_QUANTILES];
    c.flush(cq, rank, thr);
    tp.hdr[o] = c.h;
    double v = timer_value_of(tp, tp.type[0], e.count[o], static_cast<const double *>(e.sum)[o],
                              static_cast<const double *>(e.sum_sq)[o], c.value[c.at(c.h.head)],
                              c.value[c.at(c.h.tail)], cq);
    int64_t extra_t = 0;
    xf_window(e.ops, e.resolution, st, bs + e.resolution, v, extra_t);
    if (!(p.discard_nan && xf_isnan(v))) present |= 1ull << q;
    p.fwd_start[(uint64_t)q * e.n + s] = bs;
    p.fwd_val[(uint64_t)q * e.n + s] = v;
  }
  if constexpr (ANN) p.forward_ann(s, due, present);
  p.fwd_n[s] = m;
  p.fwd_present[s] = present;
  p.fwd_due[s] = due;
  p.rec[s] = st;
}

// elem_fold_group for a Timer group set (gt: its streams, gt.e.n = p.n_groups): the same checks, order and closed
// rule, each value one Timer.Add into the group window (count + 1, the sums with amd64's NaN rule as
// elem_timer_add_lane takes them, then AddBatch of the one value: k values are k batches, each reading the insertion
// point afresh).  The first pass also counts each touched window's values, n_add[r] for group slot r and
// n_add[g_slots + k] for fresh[k], and fails the group with CAPACITY where its list + pending + those values exceed
// gt.cap (an upper bound: the fold's compressions only free room).
// ANN: elem_fold_group's annotation rule: the first pass also fails the group with CAPACITY for an annotation longer
// than g_ann_cap on a value that would fold, and the group window's reference stays in registers beside its stream and
// sums, resolved into the slot (ElementRollupParams::store_group_ann, this lane copying every word) only when changed.
template <bool ANN = false, class Member>
__device__ __forceinline__ int32_t elem_timer_fold_group(const ElementRollupParams &p, const ElementTimerParams &gt,
                                                         uint64_t g, int64_t *fresh, uint32_t *n_add, Member member) {
  const uint64_t lo = p.group_off[g], hi = p.group_off[g + 1], G = p.n_groups;
  const int64_t res = p.src.resolution, wm = p.g_watermark[g];
  int32_t status = M3TSZ_OK;
  auto window = [&](const FwdMember &a, uint32_t q, int64_t &ws, double &v) {
    if (q == 0) {
      ws = a.start0;
      v = a.val0;
    } else {
      ws = p.fwd_start[(uint64_t)q * p.src.n + a.m];
      v = p.fwd_val[(uint64_t)q * p.src.n + a.m];
    }
  };
  if (lo > hi || hi > p.n_members) {
    status = M3TSZ_ERR_INVALID_ARG;
  } else {
    for (uint32_t r = 0; r < 2 * p.g_slots; r++) n_add[r] = 0;
    uint32_t n_free = 0, n_fresh = 0;
    for (uint32_t r = 0; r < p.g_slots; r++) n_free += p.g_count[(uint64_t)r * G + g] == 0;
    bool bad = false, full = false;
    int last = -1;  // the n_add entry of the last window counted (a group's values mostly go to one window)
    int64_t last_ws = 0;
    for (uint64_t i = lo; i < hi; i++) {
      const FwdMember a = member(i);
      if (a.m >= p.src.n) bad = true;
      for (uint32_t q = 0; q < a.n; q++) {
        if (!((a.present >> q) & 1u)) continue;
        int64_t ws;
        double v;
        window(a, q, ws, v);
        if (elem_ends_by(ws, res, wm)) continue;
        if constexpr (ANN) {
          if (((a.ann >> q) & 1u) && (p.fwd_ann[(uint64_t)q * p.src.n + a.m] & 0x1ffffu) > p.g_ann_cap) full = true;
        }
        int at = -1;
        if (last >= 0 && ws == last_ws) {
          at = last;
        } else {
          for (uint32_t r = 0; r < p.g_slots && at < 0; r++) {
            const uint64_t o = (uint64_t)r * G + g;
            if (p.g_count[o] != 0 && p.g_start[o] == ws) at = (int)r;
          }
          for (uint32_t k = 0; k < n_fresh && at < 0; k++)
            if (fresh[k] == ws) at = (int)(p.g_slots + k);
          if (at < 0 && n_fresh < n_free) {
            fresh[n_fresh] = ws;
            at = (int)(p.g_slots + n_fresh++);
          }
        }
        if (at < 0) {
          full = true;
          continue;
        }
        last = at;
        last_ws = ws;
        n_add[at]++;
      }
    }
    if (!bad && !full) {
      for (uint32_t r = 0; r < p.g_slots; r++) {
        const uint64_t o = (uint64_t)r * G + g;
        uint64_t size = 0;
        if (p.g_count[o] != 0) {
          const m3tsz_timer_stream_header &h = gt.hdr[o];
          size = (uint64_t)h.n_samples + (uint64_t)h.n_a + (uint64_t)h.n_b;
        }
        if (size + n_add[r] > gt.cap) full = true;
      }
      for (uint32_t k = 0; k < n_fresh; k++) full |= n_add[p.g_slots + k] > gt.cap;
    }
    status = bad ? M3TSZ_ERR_INVALID_ARG : full ? M3TSZ_ERR_CAPACITY : M3TSZ_OK;
  }
  if (status == M3TSZ_OK) {
    int cur = -1;  // the group slot the registers hold, -1: none
    int64_t w_start = 0, cnt = 0;
    double sum = 0.0, sq = 0.0;
    CmStream c = timer_stream(gt, 0u, g);  // (set again for the slot whenever `cur` changes)
    bool closed = false;
    uint64_t a_ref = 0;  // ANN: the window's annotation taken in this call (0: none), and whether its slot needs it
    bool a_dirty = false;
    auto store = [&]() {
      const uint64_t o = (uint64_t)cur * G + g;
      p.g_start[o] = w_start;
      p.g_count[o] = cnt;
      static_cast<double *>(p.g_sum)[o] = sum;
      static_cast<double *>(p.g_sum_sq)[o] = sq;
      gt.hdr[o] = c.h;
      if (ANN && a_dirty) p.store_group_ann(o, a_ref, 0u, 1u);
    };
    for (uint64_t i = lo; i < hi; i++) {
      const FwdMember a = member(i);
      for (uint32_t q = 0; q < a.n; q++) {
        if (!((a.present >> q) & 1u)) continue;
        int64_t ws;
        double v;
        window(a, q, ws, v);
        if (elem_ends_by(ws, res, wm)) {
          closed = true;
          continue;
        }
        if (cur < 0 || ws != w_start) {  // the window's slot, or a free one (the first pass counted them)
          if (cur >= 0) store();
          int hit, fr;
          p.group_slot(g, -1, ws, hit, fr);
          cur = hit >= 0 ? hit : fr;
          const uint64_t o = (uint64_t)cur * G + g;
          w_start = ws;
          cnt = 0;
          sum = sq = 0.0;
          if (hit >= 0) {
            cnt = p.g_count[o];
            sum = static_cast<const double *>(p.g_sum)[o];
            sq = static_cast<const double *>(p.g_sum_sq)[o];
          }
          c = timer_stream(gt, (uint32_t)cur, g);
          if (hit >= 0)
            c.h = gt.hdr[o];
          else
            c.init();
          a_ref = 0;
          a_dirty = hit < 0;
        }
        cnt++;
        sum = amd64_op(__dadd_rn(sum, v), sum, v);
        const double v2 = amd64_op(__dmul_rn(v, v), v, v);
        sq = amd64_op(__dadd_rn(sq, v2), sq, v2);
        c.add_batch(1u, [&](uint32_t) { return v; });
        if (ANN && ((a.ann >> q) & 1u)) {
          a_ref = p.fwd_ann[(uint64_t)q * p.src.n + a.m];
          a_dirty = true;
        }
      }
    }
    if (cur >= 0) store();
    if (closed) status = M3TSZ_ERR_AGGREGATION_CLOSED;
  }
  p.group_status[g] = status;
  return status;
}

// (__maxnreg__ as the other Timer kernels: the stream's code is the same)
template <bool ANN>
__global__ void __maxnreg__(128) element_timer_forward_kernel(const ElementRollupParams p,
                                                              const ElementTimerParams tp) {
  const uint64_t s = (uint64_t)blockIdx.x * ELEM_THREADS + threadIdx.x;
  if (s < p.src.n) elem_timer_forward_lane<ANN>(p, tp, s);
}

// One lane per group, unlike element_fold_kernel's warp per group: a group's values go through the serial stream one
// Timer.Add at a time, so a warp that ran one group would leave 31 lanes idle; with a lane per group the warp runs 32
// groups' folds at once (DESIGN.md §4.12 has both mappings measured).  The fresh-window starts and per-window tallies
// are the lane's own (local memory; a group touches few of the entries).
template <bool ANN>
__global__ void __maxnreg__(128) element_timer_fold_kernel(const ElementRollupParams p, const ElementTimerParams gt) {
  const uint64_t g = (uint64_t)blockIdx.x * ELEM_THREADS + threadIdx.x;
  if (g >= p.n_groups) return;
  int64_t fresh[M3TSZ_MAX_ELEMENT_WINDOWS];
  uint32_t n_add[2 * M3TSZ_MAX_ELEMENT_WINDOWS];
  const int32_t st =
      elem_timer_fold_group<ANN>(p, gt, g, fresh, n_add, [&](uint64_t i) { return fwd_member<ANN>(p, i); });
  const uint64_t lo = p.group_off[g], hi = p.group_off[g + 1];
  if ((st == M3TSZ_ERR_CAPACITY || st == M3TSZ_ERR_INVALID_ARG) && lo <= hi) {
    const uint64_t end = hi < p.n_members ? hi : p.n_members;
    for (uint64_t i = lo; i < end; i++) {
      const uint32_t m = p.members[i];
      if (m < p.src.n) atomicMax(p.mark + m, st);
    }
  }
}

cudaError_t launch_element_timer_forward(const ElementRollupParams &p, const ElementTimerParams &src,
                                         cudaStream_t stream) {
  if (p.src.n == 0) return cudaSuccess;
  if ((p.src.n + ELEM_THREADS - 1) / ELEM_THREADS > 0x7fffffffull) return cudaErrorInvalidValue;
  const bool ann = p.src.ann_len != nullptr;
  if (ann && (!p.fwd_ann_present || !p.fwd_ann)) return cudaErrorInvalidValue;
  if (ann)
    element_timer_forward_kernel<true><<<elem_blocks(p.src.n), ELEM_THREADS, 0, stream>>>(p, src);
  else
    element_timer_forward_kernel<false><<<elem_blocks(p.src.n), ELEM_THREADS, 0, stream>>>(p, src);
  return cudaGetLastError();
}

cudaError_t launch_element_timer_fold(const ElementRollupParams &p, const ElementTimerParams &groups,
                                      cudaStream_t stream) {
  if (p.n_groups == 0) return cudaSuccess;
  if ((p.n_groups + ELEM_THREADS - 1) / ELEM_THREADS > 0x7fffffffull) return cudaErrorInvalidValue;
  const bool ann = p.src.ann_len != nullptr;
  if (ann && (!p.fwd_ann_present || !p.fwd_ann || !p.g_ann_len || !p.g_ann_slot)) return cudaErrorInvalidValue;
  if (ann)
    element_timer_fold_kernel<true><<<elem_blocks(p.n_groups), ELEM_THREADS, 0, stream>>>(p, groups);
  else
    element_timer_fold_kernel<false><<<elem_blocks(p.n_groups), ELEM_THREADS, 0, stream>>>(p, groups);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------
// Timer element-set rollups across shards (DESIGN.md §4.12): the writer is forward_write's kernels after
// element_timer_forward_kernel; AddUnique into a Timer group set is the lane below
// ---------------------------------------------------------------------------
// add_forwarded_lane for Timer element e (gt: the group set's streams): the same record loop, checks, slot search and
// source bits, with one check after the duplicate one: a record whose values would take its window past gt.cap
// samples (list, pending and the record's values) stops the element with CAPACITY, its bit clear (a slot opened for it
// stays free).  Each value is then one Timer.Add as elem_timer_fold_group makes it.  The window the last record went
// to (its count, sums and stream header) stays in registers.  (The record checks and the Timer.Add are copies of
// add_forwarded_lane's and elem_timer_fold_group's; tests/test_device_element_timer_forwarded_on_host.py pins them.)
__device__ __forceinline__ void add_forwarded_timer_lane(const ElementForwardedParams &p, const ElementTimerParams &gt,
                                                         uint64_t j) {
  const ElementRollupParams &rp = p.rp;
  const uint64_t e = p.sorted_key[j], G = rp.n_groups;
  if (e >= G) {
    for (; j < p.n_recs && p.sorted_key[j] == e; j++) p.result[p.sorted_idx[j]] = (int8_t)M3TSZ_ERR_INVALID_ARG;
    return;
  }
  const int64_t res = rp.src.resolution, wm = rp.g_watermark[e];
  const uint32_t W = p.bit_words;
  int cur = -1;  // the group slot the registers hold, -1: none
  int64_t w_start = 0, cnt = 0;
  double sum = 0.0, sq = 0.0;
  CmStream c = timer_stream(gt, 0u, e);  // (set again for the slot whenever `cur` changes)
  auto store = [&]() {
    if (cnt == 0) return;  // (a slot opened for a refused record)
    const uint64_t o = (uint64_t)cur * G + e;
    rp.g_start[o] = w_start;
    rp.g_count[o] = cnt;
    static_cast<double *>(rp.g_sum)[o] = sum;
    static_cast<double *>(rp.g_sum_sq)[o] = sq;
    gt.hdr[o] = c.h;
  };
  int32_t status = M3TSZ_OK;
  for (; j < p.n_recs && p.sorted_key[j] == e; j++) {
    const uint64_t i = p.sorted_idx[j];
    const m3tsz_forwarded_metric m = p.rec[i];
    int r = M3TSZ_ERR_CAPACITY;  // (after a CAPACITY, the rest of the element's records)
    if (status == M3TSZ_OK) {
      int64_t t0 = 0;
      if (m.n_values == 0 || m.value_off > p.n_vals || m.n_values > p.n_vals - m.value_off || m.version != 0 ||
          m.reserved != 0 || !elem_window_start(m.time_ns, res, p.trunc_off, t0) ||
          t0 < (int64_t)0x8000000000000000ull + res) {
        r = M3TSZ_ERR_INVALID_ARG;
      } else if (elem_ends_by(t0 - res, res, wm)) {
        r = M3TSZ_ERR_AGGREGATION_CLOSED;
      } else if (m.source_id >= W * 32u) {
        status = r = M3TSZ_ERR_CAPACITY;
      } else {
        const int64_t ws = t0 - res;
        r = M3TSZ_OK;
        if (cur < 0 || ws != w_start) {  // the window's slot, or a free one
          int hit, fr;
          rp.group_slot(e, cur, ws, hit, fr);
          if (hit < 0 && fr < 0) {
            status = r = M3TSZ_ERR_CAPACITY;
          } else {
            if (cur >= 0) store();
            cur = hit >= 0 ? hit : fr;
            const uint64_t o = (uint64_t)cur * G + e;
            w_start = ws;
            c = timer_stream(gt, (uint32_t)cur, e);
            if (hit >= 0) {
              cnt = rp.g_count[o];
              sum = static_cast<const double *>(rp.g_sum)[o];
              sq = static_cast<const double *>(rp.g_sum_sq)[o];
              c.h = gt.hdr[o];
            } else {
              cnt = 0;
              sum = sq = 0.0;
              c.init();
              for (uint32_t w = 0; w < W; w++) p.bits[((uint64_t)cur * W + w) * G + e] = 0u;
            }
          }
        }
        if (r == M3TSZ_OK) {
          uint32_t *word = p.bits + ((uint64_t)cur * W + (m.source_id >> 5)) * G + e;
          const uint32_t bit = 1u << (m.source_id & 31u);
          if (*word & bit) {
            r = M3TSZ_ERR_DUPLICATE_SOURCE;
          } else if ((uint64_t)c.size() + m.n_values > gt.cap) {
            status = r = M3TSZ_ERR_CAPACITY;
          } else {
            *word |= bit;
            for (uint32_t k = 0; k < m.n_values; k++) {
              const double v = p.val[m.value_off + k];
              cnt++;
              sum = amd64_op(__dadd_rn(sum, v), sum, v);
              const double v2 = amd64_op(__dmul_rn(v, v), v, v);
              sq = amd64_op(__dadd_rn(sq, v2), sq, v2);
              c.add_batch(1u, [&](uint32_t) { return v; });
            }
          }
        }
      }
    }
    p.result[i] = (int8_t)r;
  }
  if (cur >= 0) store();
  p.status[e] = status;
}

// (__maxnreg__ as the other Timer kernels: the stream's code is the same)
__global__ void __maxnreg__(128) add_forwarded_timer_kernel(const ElementForwardedParams p,
                                                            const ElementTimerParams gt) {
  const uint64_t j = (uint64_t)blockIdx.x * ELEM_THREADS + threadIdx.x;
  if (j >= p.n_recs || (j && p.sorted_key[j - 1] == p.sorted_key[j])) return;  // one lane per element with records
  add_forwarded_timer_lane(p, gt, j);
}

cudaError_t launch_add_forwarded_timer(const ElementForwardedParams &p, const ElementTimerParams &groups,
                                       cudaStream_t stream) {
  if (p.n_recs == 0) return cudaSuccess;
  if ((p.n_recs + ELEM_THREADS - 1) / ELEM_THREADS > 0x7fffffffull) return cudaErrorInvalidValue;
  add_forwarded_timer_kernel<<<elem_blocks(p.n_recs), ELEM_THREADS, 0, stream>>>(p, groups);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------
// compaction: slots -> packed buffer with CSR offsets
// ---------------------------------------------------------------------------
__global__ void compact_lens_kernel(const uint64_t *len, uint64_t n, uint64_t mask, uint64_t *out) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (len[i] + mask) & ~mask;
  if (i == n) out[i] = 0;
}

__global__ void compact_gather_kernel(const uint8_t *slots, uint64_t slot_stride, const uint64_t *len,
                                      uint64_t n, uint8_t *packed, uint64_t cap,
                                      const uint64_t *offsets, int32_t *overflow) {
  const uint64_t w = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const uint64_t o = offsets[w], l = len[w];
  if (o + l > cap) {
    if (lane == 0) atomicExch(overflow, 1);
    return;
  }
  const uint8_t *src = slots + w * slot_stride;
  uint8_t *dst = packed + o;
  if ((((uintptr_t)dst | (uintptr_t)src) & 15u) == 0) {
    // 16-byte vector copies, four in flight per lane
    const uint64_t nv = l >> 4;
    const uint4 *s4 = reinterpret_cast<const uint4 *>(src);
    uint4 *d4 = reinterpret_cast<uint4 *>(dst);
    uint64_t i = lane;
    for (; i + 96 < nv; i += 128) {
      const uint4 a = __ldg(s4 + i), b = __ldg(s4 + i + 32), c = __ldg(s4 + i + 64), d = __ldg(s4 + i + 96);
      d4[i] = a;
      d4[i + 32] = b;
      d4[i + 64] = c;
      d4[i + 96] = d;
    }
    for (; i < nv; i += 32) d4[i] = __ldg(s4 + i);
    for (uint64_t j = (nv << 4) + lane; j < l; j += 32) dst[j] = src[j];
  } else if ((((uintptr_t)dst | (uintptr_t)src) & 3u) == 0) {
    const uint64_t nw = l >> 2;
    for (uint64_t i = lane; i < nw; i += 32)
      reinterpret_cast<uint32_t *>(dst)[i] = reinterpret_cast<const uint32_t *>(src)[i];
    for (uint64_t i = (nw << 2) + lane; i < l; i += 32) dst[i] = src[i];
  } else {
    for (uint64_t i = lane; i < l; i += 32) dst[i] = src[i];
  }
}

size_t compact_scan_tmp_bytes(uint64_t n_series) {
  size_t tmp = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tmp, (uint64_t *)nullptr, (uint64_t *)nullptr,
                                (int)(n_series + 1));
  return tmp + (n_series + 1) * sizeof(uint64_t);
}

cudaError_t launch_compact(const uint8_t *slots, uint64_t slot_stride, const uint64_t *len,
                           uint64_t n_series, uint32_t align, uint8_t *packed,
                           uint64_t packed_capacity, uint64_t *offsets, void *scan_tmp,
                           size_t scan_tmp_bytes, int32_t *overflow_flag, cudaStream_t stream) {
  if (n_series + 1 > 0x7fffffffull) return cudaErrorInvalidValue;
  uint64_t *alen = reinterpret_cast<uint64_t *>(scan_tmp);
  void *cub_tmp = reinterpret_cast<uint8_t *>(scan_tmp) + (n_series + 1) * sizeof(uint64_t);
  size_t cub_bytes = scan_tmp_bytes - (n_series + 1) * sizeof(uint64_t);
  const uint64_t mask = (uint64_t)align - 1;
  const unsigned tb = 256;
  compact_lens_kernel<<<(unsigned)((n_series + 1 + tb - 1) / tb), tb, 0, stream>>>(len, n_series, mask, alen);
  cudaError_t e = cub::DeviceScan::ExclusiveSum(cub_tmp, cub_bytes, alen, offsets, (int)(n_series + 1), stream);
  if (e != cudaSuccess) return e;
  if (n_series == 0) return cudaGetLastError();
  const uint64_t threads = n_series * 32ull;
  compact_gather_kernel<<<(unsigned)((threads + tb - 1) / tb), tb, 0, stream>>>(
      slots, slot_stride, len, n_series, packed, packed_capacity, offsets, overflow_flag);
  return cudaGetLastError();
}

}  // namespace m3tsz
