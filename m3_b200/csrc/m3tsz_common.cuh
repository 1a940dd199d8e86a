// m3tsz_common.cuh -- shared device helpers for the sm_90a M3TSZ kernels.
//
// Format constants follow the reference (paths under
// /root/reference/src/dbnode/encoding): scheme.go:30-62 (marker + time buckets),
// m3tsz/m3tsz.go:28-62 (value opcodes), SURVEY.md Appendix A (normative summary).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "../../include/m3tsz_b200.h"

namespace m3tsz {

constexpr unsigned FULL_MASK = 0xffffffffu;

// marker scheme (scheme.go:30-38): 9-bit opcode 0x100 + 2-bit value
constexpr uint32_t kMarkerOpcode = 0x100;
constexpr int kMarkerBits = 11;
constexpr int kMarkerEOS = 0, kMarkerAnnotation = 1, kMarkerTimeUnit = 2;

constexpr int kMaxMult = 6;  // m3tsz.go:60

// Time-encoding scheme kinds (scheme.go:40-53,109-120,160-165)
enum SchemeKind : int {
  kSchemeNone = 0,  // nil scheme (errNoTimeSchemaForUnit)
  kScheme32 = 1,    // s, ms: buckets 7/9/12, default 32 bits
  kScheme64 = 2,    // us, ns: buckets 7/9/12, default 64 bits
  kSchemeZero = 3   // m, h, d, y: the all-zero scheme left in the table
};

__host__ __device__ __forceinline__ bool unit_is_valid(int u) { return u > 0 && u < 9; }

__host__ __device__ __forceinline__ int64_t unit_nanos(int u) {  // unit.go:185-195
  switch (u) {
    case 1: return 1000000000LL;
    case 2: return 1000000LL;
    case 3: return 1000LL;
    case 4: return 1LL;
    case 5: return 60LL * 1000000000LL;
    case 6: return 3600LL * 1000000000LL;
    case 7: return 86400LL * 1000000000LL;
    case 8: return 365LL * 86400LL * 1000000000LL;
    default: return 0;
  }
}

__host__ __device__ __forceinline__ int scheme_kind_for_unit(int u) {
  if (!unit_is_valid(u)) return kSchemeNone;
  if (u <= 2) return kScheme32;
  if (u <= 4) return kScheme64;
  return kSchemeZero;
}

// initialTimeUnit, m3tsz/timestamp_encoder.go:248-259
__host__ __device__ __forceinline__ int initial_time_unit(int64_t start, int unit) {
  if (!unit_is_valid(unit)) return 0;
  return (start % unit_nanos(unit) == 0) ? unit : 0;
}

// Go shift semantics: x >> n == 0 and x << n == 0 for n >= 64.
__device__ __forceinline__ uint64_t shr64(uint64_t x, int n) { return n >= 64 ? 0ull : x >> n; }
__device__ __forceinline__ uint64_t shl64(uint64_t x, int n) { return n >= 64 ? 0ull : x << n; }
// PTX shifts: amounts above 63 (incl. "negative" ones read as unsigned) are clamped and shift everything
// out -- defined behaviour, so no guard compare + select around the hot path's shifts
__device__ __forceinline__ uint64_t shr64_clamp(uint64_t x, uint32_t n) {
  uint64_t r;
  asm("shr.b64 %0, %1, %2;" : "=l"(r) : "l"(x), "r"(n));
  return r;
}
__device__ __forceinline__ uint64_t shl64_clamp(uint64_t x, uint32_t n) {
  uint64_t r;
  asm("shl.b64 %0, %1, %2;" : "=l"(r) : "l"(x), "r"(n));
  return r;
}

// encoding.SignExtend (encoding.go:45-49) for 1 <= n <= 64
__device__ __forceinline__ int64_t sign_extend(uint64_t v, int n) {
  int sh = 64 - n;
  return ((int64_t)(v << sh)) >> sh;
}

// encoding.LeadingAndTrailingZeros (encoding.go:33-43): (64, 0) for v == 0
__device__ __forceinline__ void lz_tz(uint64_t v, int &lz, int &tz) {
  uint32_t hi, lo;  // unpacked in PTX: "hi != 0" must stay a 32-bit test (not v >= 2^32: two compares)
  asm("mov.b64 {%0, %1}, %2;" : "=r"(lo), "=r"(hi) : "l"(v));
  lz = hi ? __clz((int)hi) : 32 + __clz((int)lo);  // 64 for v == 0
  const int tlo = __clz((int)__brev(lo)), thi = 32 + __clz((int)__brev(hi));
  tz = lo ? tlo : (hi ? thi : 0);
}

__device__ __forceinline__ int num_sig(uint64_t v) { return 64 - __clzll((long long)v); }  // encoding.go:29-31

// multipliers[], m3tsz/m3tsz.go:131-140 (exact powers of ten)
__device__ __forceinline__ double mult_pow10(int m) {
  switch (m) {
    case 0: return 1.0;
    case 1: return 10.0;
    case 2: return 100.0;
    case 3: return 1000.0;
    case 4: return 10000.0;
    case 5: return 100000.0;
    default: return 1000000.0;
  }
}

// Go int64(float64) on amd64 (CVTTSD2SQ): truncation toward zero; out of range / NaN -> MinInt64.  The
// Counter aggregation takes its values this way (int64(dp.Value), m3coordinator ingest/write.go:560-567).  The
// encoder's classifier has the same conversion as go_f64_to_u64_via_i64 (m3tsz_encode.cu), where the host tests
// of the encoder compile it from; tests/test_independent_aggregations.py checks that the two agree.
__device__ __forceinline__ int64_t go_f64_to_i64(double a) {
  if (!(a >= -9223372036854775808.0 && a < 9223372036854775808.0)) return (int64_t)0x8000000000000000ull;
  return (int64_t)__double2ll_rz(a);
}

// aggregation.stdev (src/aggregator/aggregation/common.go:29-37): div = count*(count-1) in int64 (0: result 0),
// num = float64(count)*sumSq - sum*sum as two roundings each (no fusion), sqrt(num / float64(div)).  Every NaN this
// arithmetic can make on amd64 is the invalid-operation default 0xFFF8000000000000 (Inf - Inf, sqrt of a negative,
// or one carried in `sum` from +Inf + -Inf), so a NaN result is written as that.
__device__ __forceinline__ double agg_stdev(int64_t count, double sum_sq, double sum) {
  const int64_t div = (int64_t)((uint64_t)count * (uint64_t)(count - 1));
  if (div == 0) return 0.0;
  const double num = __dsub_rn(__dmul_rn(__ll2double_rn(count), sum_sq), __dmul_rn(sum, sum));
  const double r = __dsqrt_rn(__ddiv_rn(num, __ll2double_rn(div)));
  return r == r ? r : __longlong_as_double((long long)0xFFF8000000000000ull);
}

// XXH64, seed 0 (cespare/xxhash/v2 Sum64, go.mod:10): TimestampEncoder keeps the checksum of the last annotation
// written (timestamp_encoder.go:56,166-195) and rewrites an annotation only when its checksum differs; Encoder.
// LastAnnotationChecksum() exposes it (encoder.go:321-327).  One definition for the streaming handles (host) and the
// encoder sets' append kernel (device).  Little-endian byte order: x86-64 / aarch64 hosts and the GPU.
__host__ __device__ inline uint64_t xxh64(const uint8_t *d, size_t n) {
  const uint64_t P1 = 11400714785074694791ull, P2 = 14029467366897019727ull, P3 = 1609587929392839161ull,
                 P4 = 9650029242287828579ull, P5 = 2870177450012600261ull;
  auto rotl = [](uint64_t x, int r) { return (x << r) | (x >> (64 - r)); };
  auto xround = [&](uint64_t acc, uint64_t in) { return rotl(acc + in * P2, 31) * P1; };
  auto rd64 = [](const uint8_t *p) {
    uint64_t v;
    memcpy(&v, p, 8);
    return v;
  };
  auto rd32 = [](const uint8_t *p) {
    uint32_t v;
    memcpy(&v, p, 4);
    return v;
  };
  const uint8_t *p = d, *end = d + n;
  uint64_t h;
  if (n >= 32) {
    uint64_t v1 = P1 + P2, v2 = P2, v3 = 0, v4 = 0 - P1;
    while (p + 32 <= end) {
      v1 = xround(v1, rd64(p));
      v2 = xround(v2, rd64(p + 8));
      v3 = xround(v3, rd64(p + 16));
      v4 = xround(v4, rd64(p + 24));
      p += 32;
    }
    h = rotl(v1, 1) + rotl(v2, 7) + rotl(v3, 12) + rotl(v4, 18);
    h = (h ^ xround(0, v1)) * P1 + P4;
    h = (h ^ xround(0, v2)) * P1 + P4;
    h = (h ^ xround(0, v3)) * P1 + P4;
    h = (h ^ xround(0, v4)) * P1 + P4;
  } else {
    h = P5;
  }
  h += (uint64_t)n;
  while (p + 8 <= end) {
    h = rotl(h ^ xround(0, rd64(p)), 27) * P1 + P4;
    p += 8;
  }
  if (p + 4 <= end) {
    h = rotl(h ^ ((uint64_t)rd32(p) * P1), 23) * P2 + P3;
    p += 4;
  }
  while (p < end) {
    h = rotl(h ^ ((uint64_t)*p * P5), 11) * P1;
    p++;
  }
  h ^= h >> 33;
  h *= P2;
  h ^= h >> 29;
  h *= P3;
  h ^= h >> 32;
  return h;
}

// Big-endian 32-bit word `widx` of a byte buffer whose base is 4-byte aligned.
// Words (partly) past `nbytes` are zero-filled, never read out of bounds.
__device__ __forceinline__ uint32_t load_be32(const uint8_t *base, uint64_t nbytes, uint64_t widx) {
  uint64_t b = widx << 2;
  if (b + 4 <= nbytes) {
    uint32_t v = __ldg(reinterpret_cast<const uint32_t *>(base + b));
    return __byte_perm(v, 0, 0x0123);
  }
  uint32_t v = 0;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    uint32_t x = (b + i < nbytes) ? (uint32_t)base[b + i] : 0u;
    v = (v << 8) | x;
  }
  return v;
}

}  // namespace m3tsz
