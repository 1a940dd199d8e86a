// m3tsz_decode.cu -- batch M3TSZ decode for sm_90a (+ fused downsample).
//
// Mapping (DESIGN.md §3): one LANE per series, 32 series per warp.  A stream is
// a serial bit-dependency chain (every field width depends on decoded state),
// so the per-series state machine runs on one lane while the WARP cooperates
// on memory: each lane's compressed words are staged into a shared-memory ring
// of 16-byte quads ([quad][lane]) by asynchronous 16-byte copies (cp.async /
// LDGSTS, conflict-free, 64-byte chunks per lane) issued one refill ahead of
// consumption, every datapoint is parsed branch-free from two LDS.128 (eight
// words, no bank conflicts wherever the lanes stand) with selects and funnel
// shifts, and a group of four decoded (ts, value) pairs stays in registers until
// the lane stores it as one whole 32-byte sector per array (two STG.128).
//
// Format: SURVEY.md Appendix A; reference decode path
//   m3tsz/iterator.go:81-219, m3tsz/timestamp_iterator.go:80-326,
//   m3tsz/float_encoder_iterator.go:105-165, istream.go:73-115.
#include <type_traits>

#include "m3tsz_common.cuh"
#include "m3tsz_kernels.h"

namespace m3tsz {

// <= this many requested words ahead: the lane triggers a refill event.  It has to leave DEC_CHK * 80 bits + the
// fast path's window landed after a group.
constexpr int DEC_TRIGGER = 24;
constexpr int DEC_CHK = 4;        // datapoints per ring bookkeeping / group pre-check
constexpr int DEC_SAFE_MIN = 12;  // fewer landed words ahead than this: confirm the copy in flight
constexpr int DEC_MIN_BLOCKS = 4;     // 4 x 4 warps with ~110 registers beat 5 blocks squeezed into 96
constexpr int DEC_MIN_BLOCKS_DS = 5;  // fused-downsample kernels: 5 x 4 warps at 96 registers beat 4 blocks
constexpr int DEC_WARPS = 4;      // warps per block
constexpr int DEC_RING = 64;      // staged words per lane (ring buffer, power of two)
constexpr int DEC_FILL = 16;      // words per lane per asynchronous refill chunk
constexpr int DEC_ACCEPT = DEC_RING - DEC_FILL;  // lanes with <= this many words ahead take a chunk
constexpr int DEC_GROUP = 4;      // datapoints per output group (one 32-byte sector per array)
constexpr int DEC_FAST_WORDS = 4; // the fast path reads 4 consecutive words

constexpr int DEC_QUADS = DEC_RING / 4;  // + 1 mirror quad (copy of quad 0) so quad q+1 is always at +1
constexpr int DEC_IN_TILE_WORDS = (DEC_QUADS + 1) * 32 * 4;
static_assert(DEC_CHK == DEC_GROUP, "ring bookkeeping runs once per output group");
constexpr size_t DEC_WARP_SMEM_PLAIN = (size_t)DEC_IN_TILE_WORDS * 4;
static_assert(DEC_WARP_SMEM_PLAIN % 16 == 0, "every warp's ring must stay 16-byte aligned");

constexpr uint64_t kGoNaNBits = 0x7FF8000000000001ull;  // math.NaN()

struct DecState {
  uint64_t wbase;  // global word index of this stream's 4-byte-aligned base
  uint32_t pos;    // current bit position relative to wbase
  uint32_t end;    // end-of-stream bit position (exclusive)
  int64_t prev_time, prev_delta;
  uint64_t prev_bits, prev_xor;
  double int_val;
  int64_t unit_ns;
  int sig, mult, unit, scheme;
  int emit_unit;   // time unit in force at the last datapoint produced
  int first_unit;  // ... at the first datapoint produced
  int err;
  uint32_t n;
  bool is_float, done;
  uint32_t ann_count, ann_len;
  uint32_t ann_bit;
};

// ---------------------------------------------------------------------------
// generic bit reader over global memory (slow path: first datapoint, markers,
// annotations, unit changes, 32/64-bit delta-of-delta, int-mode headers)
// ---------------------------------------------------------------------------
// Where the slow path reads from: the lane's ring column while the words it
// needs have landed there (words [.., ring_safe) relative to wbase), global
// memory otherwise (first datapoint before the first refill, annotations that
// run past the ring, lanes that ran dry).
struct SlowSrc {
  const uint8_t *base;
  uint64_t nbytes;
  const uint32_t *ring_lane;  // the lane's 16-byte cell of quad 0 (ring + lane * 4 words)
  uint32_t ring_safe;
};

// per-datapoint unit / annotation event table (optional; include/m3tsz_b200.h m3tsz_dp_event)
struct EventSink {
  m3tsz_dp_event *events;
  uint64_t capacity;
  unsigned long long *count;
  uint64_t series;
  uint32_t pos0;  // bit position of the stream's first bit (relative to wbase)
};

__device__ __forceinline__ void push_event(const EventSink &ev, uint32_t dp_index, uint32_t kind, uint32_t unit,
                                           uint64_t bit_offset, uint32_t length) {
  if (!ev.count) return;
  const unsigned long long i = atomicAdd(ev.count, 1ull);
  if (i < ev.capacity) {
    m3tsz_dp_event e;
    e.series = ev.series;
    e.dp_index = dp_index;
    e.kind = (uint16_t)kind;
    e.unit = (uint16_t)unit;
    e.bit_offset = bit_offset;
    e.length = length;
    e.reserved = 0;
    ev.events[i] = e;
  }
}

__device__ __forceinline__ uint64_t gpeek64(const SlowSrc &src, uint64_t wbase, uint32_t pos) {
  const uint32_t wr = pos >> 5;
  uint32_t w0, w1, w2;
  if (wr + 3u <= src.ring_safe) {
    // ring_lane = ring + lane * 4 (words); word w lives at quad (w >> 2) & 15, element w & 3
    const uint32_t a0 = wr, a1 = wr + 1, a2 = wr + 2;
    w0 = __byte_perm(src.ring_lane[((a0 >> 2) & (DEC_QUADS - 1)) * 128 + (a0 & 3)], 0, 0x0123);
    w1 = __byte_perm(src.ring_lane[((a1 >> 2) & (DEC_QUADS - 1)) * 128 + (a1 & 3)], 0, 0x0123);
    w2 = __byte_perm(src.ring_lane[((a2 >> 2) & (DEC_QUADS - 1)) * 128 + (a2 & 3)], 0, 0x0123);
  } else {
    const uint64_t w = wbase + wr;
    w0 = load_be32(src.base, src.nbytes, w);
    w1 = load_be32(src.base, src.nbytes, w + 1);
    w2 = load_be32(src.base, src.nbytes, w + 2);
  }
  const uint32_t hi = __funnelshift_l(w1, w0, pos);
  const uint32_t lo = __funnelshift_l(w2, w1, pos);
  return ((uint64_t)hi << 32) | lo;
}

#define M3_RD(nbits, var)                                                        \
  uint64_t var;                                                                  \
  {                                                                              \
    const int _n = (nbits);                                                      \
    if (s.pos + (uint32_t)_n > s.end) {                                          \
      s.err = M3TSZ_ERR_EOF;                                                     \
      return false;                                                              \
    }                                                                            \
    var = _n ? (gpeek64(src, s.wbase, s.pos) >> (64 - _n)) : 0ull;               \
    s.pos += (uint32_t)_n;                                                       \
  }

// Decodes exactly one datapoint with the complete grammar.  Returns true when a
// datapoint was produced (iterator.Next() == true *or* the value was read
// without error); false on end-of-stream (s.done) or error (s.err).
template <bool INT_OPT>
__device__ __noinline__ bool decode_dp_slow(DecState &s, const SlowSrc src, int default_unit,
                                            int64_t &out_t, uint64_t &out_v, const EventSink *evp) {
  const EventSink &ev = *evp;
  // ---- ReadTimestamp, timestamp_iterator.go:80-113 ----
  const bool first = (s.prev_time == 0);
  int64_t nt = 0;
  if (first) {  // readFirstTimestamp :136-162
    M3_RD(64, x);
    nt = (int64_t)x;
    if (s.unit == 0) {
      s.unit = initial_time_unit(nt, default_unit);
      s.unit_ns = unit_nanos(s.unit);
    }
    int k = scheme_kind_for_unit(s.unit);
    if (k != kSchemeNone) s.scheme = k;
  }
  bool unit_changed = false;
  int64_t dod = 0;
  // readMarkerOrDeltaOfDelta :233-244 / tryReadMarker :175-231 (recursion unrolled)
  for (;;) {
    if (s.pos + kMarkerBits <= s.end) {
      uint32_t p = (uint32_t)(gpeek64(src, s.wbase, s.pos) >> 53);
      if ((p >> 2) == kMarkerOpcode) {
        int m = (int)(p & 3);
        if (m == kMarkerEOS) {
          s.pos += kMarkerBits;
          s.done = true;
          return false;
        }
        if (m == kMarkerAnnotation) {  // readAnnotation :328-356
          s.pos += kMarkerBits;
          uint64_t ux = 0;
          int shift = 0;
          bool fin = false;
          for (int i = 0; i < 10; i++) {  // binary.ReadUvarint
            if (s.pos + 8 > s.end) {
              s.err = (i > 0) ? M3TSZ_ERR_UNEXPECTED_EOF : M3TSZ_ERR_EOF;
              return false;
            }
            uint32_t b = (uint32_t)(gpeek64(src, s.wbase, s.pos) >> 56);
            s.pos += 8;
            if (b < 0x80) {
              if (i == 9 && b > 1) {
                s.err = M3TSZ_ERR_VARINT_OVERFLOW;
                return false;
              }
              ux |= shl64((uint64_t)b, shift);
              fin = true;
              break;
            }
            ux |= shl64((uint64_t)(b & 0x7f), shift);
            shift += 7;
          }
          if (!fin) {
            s.err = M3TSZ_ERR_VARINT_OVERFLOW;
            return false;
          }
          int64_t alen = (int64_t)(ux >> 1);
          if (ux & 1) alen = ~alen;
          alen += 1;
          if (alen <= 0) {
            s.err = M3TSZ_ERR_ANNOTATION_LEN;
            return false;
          }
          if ((uint64_t)alen * 8ull > (uint64_t)(s.end - s.pos)) {
            s.err = M3TSZ_ERR_EOF;
            return false;
          }
          if (s.ann_count == 0) {
            s.ann_bit = s.pos;
            s.ann_len = (uint32_t)alen;
          }
          s.ann_count++;
          push_event(ev, s.n, M3TSZ_EVENT_ANNOTATION, 0, (uint64_t)(s.pos - ev.pos0), (uint32_t)alen);
          s.pos += (uint32_t)alen * 8u;
          continue;
        }
        if (m == kMarkerTimeUnit) {  // ReadTimeUnit :118-134
          s.pos += kMarkerBits;
          M3_RD(8, tub);
          int tu = (int)tub;
          if (unit_is_valid(tu) && tu != s.unit) {
            unit_changed = true;
            s.scheme = scheme_kind_for_unit(tu);
          }
          if (tu != s.unit && s.n > 0) push_event(ev, s.n, M3TSZ_EVENT_TIME_UNIT, (uint32_t)tu, 0, 0);
          s.unit = tu;
          s.unit_ns = unit_nanos(tu);
          continue;
        }
        // marker value 3: not a marker, parse as delta-of-delta
      }
    }
    break;
  }
  // readDeltaOfDelta :246-305
  if (unit_changed) {  // readFullTimestamp :307-326
    int k = scheme_kind_for_unit(s.unit);
    if (k == kSchemeNone) {
      s.err = M3TSZ_ERR_NO_TIME_SCHEME;
      return false;
    }
    s.scheme = k;
    M3_RD(64, x);
    dod = (int64_t)x;
  } else if (s.scheme == kSchemeNone) {
    s.err = M3TSZ_ERR_NO_TIME_SCHEME;
    return false;
  } else {
    M3_RD(1, cb);
    if (cb != 0 && s.scheme != kSchemeZero) {
      int nb = (s.scheme == kScheme32) ? 32 : 64;
      bool swallowed = false;
      for (int i = 0; i < 3; i++) {
        if (s.pos + 1 > s.end) {  // error swallowed by the reference (:271-274)
          swallowed = true;
          break;
        }
        uint64_t b = gpeek64(src, s.wbase, s.pos) >> 63;
        s.pos += 1;
        if (b == 0) {
          nb = (i == 0) ? 7 : (i == 1 ? 9 : 12);
          break;
        }
      }
      if (!swallowed) {
        M3_RD(nb, bits);
        int64_t d = sign_extend(bits, nb);
        dod = unit_is_valid(s.unit) ? (int64_t)((uint64_t)d * (uint64_t)s.unit_ns) : 0;
      }
    }
    // kSchemeZero: no buckets, default bucket has 0 value bits => dod = 0
  }
  s.prev_delta = (int64_t)((uint64_t)s.prev_delta + (uint64_t)dod);
  if (first)
    s.prev_time = (int64_t)((uint64_t)nt + (uint64_t)s.prev_delta);
  else
    s.prev_time = (int64_t)((uint64_t)s.prev_time + (uint64_t)s.prev_delta);
  if (unit_changed) s.prev_delta = 0;

  // ---- value: iterator.go:108-219 ----
  bool full_float = false, next_float = false, int_hdr = false, int_diff = false;
  if (!INT_OPT) {
    full_float = first;
    next_float = !first;
  } else if (first) {
    M3_RD(1, b);
    if (b == 1) {
      full_float = true;
      s.is_float = true;
    } else {
      int_hdr = true;
      int_diff = true;
    }
  } else {
    M3_RD(1, b);
    if (b == 0) {  // opcodeUpdate
      M3_RD(1, r);
      if (r == 1) {
        // repeat: value unchanged
      } else {
        M3_RD(1, f);
        if (f == 1) {
          full_float = true;
          s.is_float = true;
        } else {
          int_hdr = true;
          int_diff = true;
          // isFloat = false is applied after the diff is read (iterator.go:148)
        }
      }
    } else if (s.is_float) {
      next_float = true;
    } else {
      int_diff = true;
    }
  }
  if (full_float) {  // readFullFloat float_encoder_iterator.go:105-115
    M3_RD(64, vb);
    s.prev_bits = vb;
    s.prev_xor = vb;
  }
  if (next_float) {  // readNextFloat :117-165
    M3_RD(1, cb);
    if (cb == 0) {
      s.prev_xor = 0;
    } else {
      M3_RD(1, c2);
      if (c2 == 0) {
        int pl, pt;
        lz_tz(s.prev_xor, pl, pt);
        int nm = 64 - pl - pt;
        M3_RD(nm, mb);
        s.prev_xor = shl64(mb, pt);
        s.prev_bits ^= s.prev_xor;
      } else {
        M3_RD(12, hdr);
        int nlz = (int)((hdr >> 6) & 63);
        int nm = (int)(hdr & 63) + 1;
        M3_RD(nm, mb);
        int ntz = 64 - nlz - nm;
        s.prev_xor = (ntz < 0) ? 0ull : shl64(mb, ntz);
        s.prev_bits ^= s.prev_xor;
      }
    }
  }
  if (int_hdr) {  // readIntSigMult iterator.go:178-193
    M3_RD(1, us);
    if (us == 1) {
      M3_RD(1, nz);
      if (nz == 0) {
        s.sig = 0;
      } else {
        M3_RD(6, sb);
        s.sig = (int)sb + 1;
      }
    }
    M3_RD(1, um);
    if (um == 1) {
      M3_RD(3, mb);
      s.mult = (int)mb;
      if (s.mult > kMaxMult) {
        s.err = M3TSZ_ERR_INVALID_MULT;
        return false;
      }
    }
  }
  if (int_diff) {  // readIntValDiff(+Slow) iterator.go:195-219
    uint64_t neg, mag;
    if (s.sig == 64) {
      M3_RD(1, sg);
      M3_RD(64, mg);
      neg = sg;
      mag = mg;
    } else {
      M3_RD(s.sig + 1, bits);
      neg = bits >> s.sig;
      mag = bits & ((1ull << s.sig) - 1ull);
    }
    double m = __ull2double_rn(mag);
    s.int_val = neg ? __dadd_rn(s.int_val, m) : __dsub_rn(s.int_val, m);
    if (int_hdr) s.is_float = false;
  }
  out_t = s.prev_time;
  s.emit_unit = s.unit;
  if (s.n == 0) s.first_unit = s.unit;
  if (!INT_OPT || s.is_float) {
    out_v = s.prev_bits;
  } else {
    double v = s.mult ? __ddiv_rn(s.int_val, mult_pow10(s.mult)) : s.int_val;  // m3tsz.go:121-127
    out_v = (uint64_t)__double_as_longlong(v);
  }
  return true;
}
#undef M3_RD

// The annotation a datapoint carries when decode_dp_slow read `count` > 1 annotation markers before it (it keeps the
// first in *bit / *len): the last of them, as Current() reports it (readAnnotation replaces PrevAnt,
// timestamp_iterator.go:328-356).  The slow path has checked every marker, varint and payload up to the datapoint,
// which are annotation and time-unit markers only, so the walk reads them without checks.
__device__ __forceinline__ void dec_last_annotation(const SlowSrc src, uint64_t wbase, uint32_t count, uint32_t *bit,
                                                    uint32_t *len) {
  uint32_t pos = *bit + *len * 8u;
  for (uint32_t k = 1; k < count;) {
    const int m = (int)((gpeek64(src, wbase, pos) >> 53) & 3u);
    pos += kMarkerBits;
    if (m == kMarkerTimeUnit) {
      pos += 8;
      continue;
    }
    uint64_t ux = 0;
    for (int i = 0, shift = 0; i < 10; i++, shift += 7) {  // binary.ReadUvarint
      const uint32_t b = (uint32_t)(gpeek64(src, wbase, pos) >> 56);
      pos += 8;
      ux |= shl64((uint64_t)(b & 0x7f), shift);
      if (b < 0x80) break;
    }
    int64_t alen = (int64_t)(ux >> 1);
    if (ux & 1) alen = ~alen;
    *bit = pos;
    *len = (uint32_t)(alen + 1);
    pos += *len * 8u;
    k++;
  }
}

__device__ __forceinline__ uint32_t smem_addr(const void *p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }

// The fills ask L2 for the whole 128-byte line (.L2::128B) of every 16-byte request: a 64-byte chunk is half a
// line, and the lane fetches the other half about 9 datapoints later, long after its DRAM row has closed -- with
// the hint, that half is already in L2 (DESIGN.md §3.2(c)).
__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src, uint32_t src_bytes) {
  asm volatile("cp.async.ca.shared.global.L2::128B [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async16_full(uint32_t dst, const void *src) {
  asm volatile("cp.async.ca.shared.global.L2::128B [%0], [%1], 16;\n" ::"r"(dst), "l"(src) : "memory");
}
// Lane-local refill: the lane copies the 64-byte chunk at global word index gw
// (a multiple of 16) of ITS OWN stream into quads slot_q0..slot_q0+3 of its own
// column with four 16-byte cp.async (a warp instruction writes 32 x 16 B =
// 4 conflict-free wavefronts; no shuffles).  Quad 0 is mirrored to quad 16.
__device__ __forceinline__ void ring_fill(uint32_t ring_lane_addr, const uint8_t *streams, uint64_t nbytes,
                                               bool take, uint32_t gw, uint32_t slot_q0) {
  if (take && ((uint64_t)gw * 4ull + 64ull <= nbytes)) {
    // whole chunk inside the buffer (every chunk but the batch's last): constant-size copies
    const uint8_t *src = streams + (uint64_t)gw * 4ull;
    const uint32_t dst = ring_lane_addr + slot_q0 * 512u;
    cp_async16_full(dst, src);
    cp_async16_full(dst + 512u, src + 16);
    cp_async16_full(dst + 1024u, src + 32);
    cp_async16_full(dst + 1536u, src + 48);
    if (slot_q0 == 0) cp_async16_full(ring_lane_addr + DEC_QUADS * 512u, src);
  } else if (take) {
#pragma unroll
    for (uint32_t k = 0; k < 4; k++) {
      const uint64_t b = ((uint64_t)gw + 4u * k) * 4ull;
      const uint32_t nb = (b + 16 <= nbytes) ? 16u : (b < nbytes ? (uint32_t)(nbytes - b) : 0u);
      const uint8_t *src = nb ? (streams + b) : streams;
      const uint32_t dst = ring_lane_addr + (slot_q0 + k) * 512u;
      cp_async16(dst, src, nb);
      if (k == 0 && slot_q0 == 0) cp_async16(ring_lane_addr + DEC_QUADS * 512u, src, nb);
    }
  }
}

// The fused-downsample modes: 1 Gauge (sum, count, min, max), 2 + last / lastAt, 4 + sumSq (the Gauge with
// expensive aggregations), 5 Counter (int64 sum, count, min, max, sumSq); 6, 7, 8: modes 2, 4, 5 that also write
// each window's annotation reference (ds_ann).
__host__ __device__ constexpr bool dec_ds_mode(int mode) {
  return mode == 1 || mode == 2 || mode == 4 || mode == 5 || mode == 6 || mode == 7 || mode == 8;
}
__host__ __device__ constexpr int dec_base_mode(int mode) {
  return mode == 6 ? 2 : (mode == 7 ? 4 : (mode == 8 ? 5 : mode));
}
// 4 and 5 carry two more 64-bit accumulators than mode 2 and start from the same budget (-Xptxas -v reports no
// spills at 96 registers).  6-8 add the window's annotation reference and the walk to a datapoint's last annotation:
// at 96 registers mode 7 spilled, so they take the plain decode's 4 blocks.  The block loop (BLK) keeps its
// counterpart's budget, except mode 4, whose int-optimised kernel spilled at 96 registers
__host__ __device__ constexpr int dec_min_blocks(int mode, bool blk = false) {
  return (dec_ds_mode(mode) && mode < 6 && !(blk && mode == 4)) ? DEC_MIN_BLOCKS_DS : DEC_MIN_BLOCKS;
}

// window accumulator type: the Gauge's float64, the Counter's int64 (counter.go:31-41)
template <bool COUNTER> struct DsVal { using T = double; };
template <> struct DsVal<true> { using T = int64_t; };

// Fused-downsample per-lane accumulator: aggregation.Gauge of the open window
// (/root/reference/src/aggregator/aggregation/gauge.go:31-106), or aggregation.Counter (counter.go:31-78) in mode 5.
template <typename V>
struct DsAcc {
  int64_t d;      // hot path: (time of the last datapoint) - w_end while the group's pre-check holds
  int64_t w_end;  // exclusive end of the open window
  int32_t cur_w, hi_w;  // open window (-1: none) / highest window initialised so far
  uint64_t o;     // element index of the open window in the window-major outputs: cur_w * n_series + sidx
  bool in_open;   // the last datapoint produced lies in the open window (false after an ignored one)
  // sum as gauge.go:92; min / max start at +inf / -inf instead of NaN: with `v < mn` / `v > mx`
  // that takes the same decisions as gauge.go:93-99 on every sequence of values (a NaN value never
  // compares true, signed zeros keep the first one seen), and "no value seen" is the one state
  // mn == +inf && mx == -inf, written out as NaN / NaN.  Counter: min / max start at MaxInt64 / MinInt64 and are
  // written as they are (counter.go:44-78)
  V sum, mn, mx;
  V sq;              // modes 4, 5: sumSq (gauge.go:101-103, counter.go:72-74)
  uint32_t cnt;      // datapoints in the open window (NaNs counted, gauge.go:85)
  uint32_t n_sync;   // s.n when cnt was last brought up to date: s.n - n_sync = hot datapoints since (all of
                     // them in the open window), folded into cnt at the next commit / general-path visit
  int64_t last_t;    // MODE 2: lastAt / last (gauge.go:74-81)
  uint64_t last_v;
};
// Modes 6-8: the open window's annotation, the last one a datapoint of the window carried (MaybeReplaceAnnotation,
// aggregation/common.go:47-61), as a packed reference (m3tsz_aggregate_tiles_annotated): 0 none
struct DsAnn {
  uint64_t ref;
};
struct DsNoAnn {};

// MODE 0: plain decode (ts, value) ; 1: fused 5-tuple-less downsample (sum, count, min, max);
// 2: downsample + last (+ lastAt scratch); 4: + sumSq; 5: Counter downsample.
// BLK (modes 2 and 4-8): the lane decodes its series' source blocks, segments [block_off[s], block_off[s + 1]), one
// after another into the same windows (m3tsz_aggregate_tiles_blocks).
template <bool INT_OPT, int MODE, bool BLK = false>
__global__ void __launch_bounds__(DEC_WARPS * 32, dec_min_blocks(MODE, BLK))
    decode_kernel(const DecodeParams p) {
  // MODE 0: plain decode, series-major output [series][point]; 3: plain decode, point-major output
  // [point][series] (every step's 32 lanes store 32 consecutive elements: coalesced 256-byte rows);
  // 1: fused downsample (sum, count, min, max); 2: + last / lastAt; 4: + sumSq (Gauge with expensive
  // aggregations); 5: Counter (int64(value): sum, count, min, max, sumSq; no last, no NaN vote)
  // The fused-downsample and point-major kernels read the ring as 8-byte pairs; series-major decode keeps the
  // 16-byte reads (the pairs cost more shared-memory wavefronts, see the parse).
  constexpr int BASE = dec_base_mode(MODE);
  constexpr bool ANN = BASE != MODE;  // modes 6-8: + each window's annotation reference
  constexpr bool RING64 = (MODE != 0);
  constexpr bool DS = dec_ds_mode(MODE), LAST = (BASE == 2 || BASE == 4), PLAIN = (MODE == 0 || MODE == 3),
                 PM = (MODE == 3);
  constexpr bool SQ = (BASE == 4), CTR = (BASE == 5);  // Gauge sumSq / Counter
  using V = typename DsVal<CTR>::T;
  extern __shared__ __align__(16) uint32_t smem[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  constexpr size_t warp_smem = DEC_WARP_SMEM_PLAIN;
  uint32_t *ring = reinterpret_cast<uint32_t *>(reinterpret_cast<uint8_t *>(smem) + warp * warp_smem);
  const uint32_t *ring_lane = ring + lane * 4;  // this lane's 16-byte cell of quad 0
  const uint32_t ring_lane_addr = smem_addr(ring_lane);

  const uint64_t warp_s0 = ((uint64_t)blockIdx.x * DEC_WARPS + warp) * 32ull;
  if (warp_s0 >= p.n_series) return;
  const uint64_t sidx = warp_s0 + lane;
  const bool valid = sidx < p.n_series;

  DecState s;
  s.wbase = 0;
  s.pos = 0;
  s.end = 0;
  s.prev_time = 0;
  s.prev_delta = 0;
  s.prev_bits = 0;
  s.prev_xor = 0;
  s.int_val = 0.0;
  s.unit_ns = 0;
  s.sig = 0;
  s.mult = 0;
  s.unit = 0;
  s.scheme = kSchemeNone;
  s.emit_unit = 0;
  s.first_unit = 0;
  s.err = 0;
  s.n = 0;
  s.is_float = false;
  s.done = !valid;
  s.ann_count = 0;
  s.ann_len = 0;
  s.ann_bit = 0;
  uint32_t pos0 = 0;
  // BLK: the series' next segment and the end of its range
  uint64_t blk = 0, blk_end = 0;
  // BLK: opens the series' next non-empty segment with a fresh stream state (the window accumulator carries on);
  // false when none is left, or with s.err on a segment outside the buffer or too large
  auto next_block = [&]() -> bool {
    while (blk < blk_end) {
      const uint64_t q = blk++;
      const uint64_t o0 = p.offsets[q];
      const uint64_t o1 = p.lengths ? o0 + p.lengths[q] : p.offsets[q + 1];
      if (o1 < o0 || o1 > p.streams_bytes) {
        s.err = M3TSZ_ERR_INVALID_ARG;
        return false;
      }
      if (o1 - o0 >= (1ull << 28)) {
        s.err = M3TSZ_ERR_STREAM_TOO_LARGE;
        return false;
      }
      if (o1 == o0) continue;  // an empty segment adds no datapoints
      const uint64_t w = o0 >> 2;
      s.wbase = w & ~(uint64_t)(DEC_FILL - 1);
      s.pos = (uint32_t)(w - s.wbase) * 32u + (uint32_t)(o0 & 3) * 8u;
      s.end = s.pos + (uint32_t)(o1 - o0) * 8u;
      pos0 = s.pos;
      s.prev_time = 0;  // the block's first timestamp, unit and int / float state come from its own stream
      s.prev_delta = 0;
      s.prev_bits = 0;
      s.prev_xor = 0;
      s.int_val = 0.0;
      s.unit_ns = 0;
      s.sig = 0;
      s.mult = 0;
      s.unit = 0;
      s.scheme = kSchemeNone;
      s.is_float = false;
      s.done = false;
      s.ann_count = 0;
      s.ann_len = 0;
      s.ann_bit = 0;
      return true;
    }
    return false;
  };
  if (valid) {
    if constexpr (BLK) {
      blk = p.block_off[sidx];
      blk_end = p.block_off[sidx + 1];
      if (blk > blk_end || blk_end > p.n_segments)
        s.err = M3TSZ_ERR_INVALID_ARG;
      else if (!next_block() && s.err == 0)
        s.done = true;  // no datapoints: every window empty, status OK
    } else {
      const uint64_t o0 = p.offsets[sidx];
      const uint64_t o1 = p.lengths ? o0 + p.lengths[sidx] : p.offsets[sidx + 1];
      if (o1 < o0 || o1 > p.streams_bytes) {
        s.err = M3TSZ_ERR_INVALID_ARG;
      } else if (o1 - o0 >= (1ull << 28)) {
        s.err = M3TSZ_ERR_STREAM_TOO_LARGE;
      } else {
        // base = the stream's first word rounded down to a DEC_FILL-word boundary
        const uint64_t w = o0 >> 2;
        s.wbase = w & ~(uint64_t)(DEC_FILL - 1);
        s.pos = (uint32_t)(w - s.wbase) * 32u + (uint32_t)(o0 & 3) * 8u;
        s.end = s.pos + (uint32_t)(o1 - o0) * 8u;
        pos0 = s.pos;
      }
    }
  }
  // rejected before its first datapoint (BLK: or without any): publish now (see the sink)
  if (DS && valid && (s.err != 0 || (BLK && s.done))) {
    if (p.n_points) p.n_points[sidx] = 0;
    if (p.status) p.status[sidx] = s.err;
  }
  uint32_t gbase = (uint32_t)s.wbase;  // streams_bytes < 16 GiB (checked by the host); BLK: the current block's
  // previous XOR's leading / trailing zero counts, kept eagerly (float path)
  int plz = 64, ptz = 0;

  const double kNaN = __longlong_as_double((long long)kGoNaNBits);
  constexpr int64_t kMaxI64 = 0x7fffffffffffffffll, kMinI64 = (int64_t)0x8000000000000000ull;
  DsAcc<V> acc;
  acc.d = 0;
  acc.w_end = 0;
  acc.cur_w = -1;
  acc.hi_w = -1;
  acc.o = 0;
  acc.in_open = false;
  if constexpr (CTR) {
    acc.sum = 0;
    acc.mn = kMaxI64;
    acc.mx = kMinI64;
    acc.sq = 0;
  } else {
    acc.sum = 0.0;
    acc.mn = __longlong_as_double(0x7ff0000000000000ll);
    acc.mx = __longlong_as_double((long long)0xfff0000000000000ull);
    if constexpr (SQ) acc.sq = 0.0;
  }
  acc.cnt = 0;
  acc.n_sync = 0;
  acc.last_t = 0;
  acc.last_v = 0;
  std::conditional_t<ANN, DsAnn, DsNoAnn> wa;  // (modes 6-8 only)
  if constexpr (ANN) wa.ref = 0;
  const int64_t range_end = p.range_start + (int64_t)p.n_windows * p.window;
  (void)range_end;

  // ---- fused-downsample helpers (per lane) ----
  const double kPosInf = __longlong_as_double(0x7ff0000000000000ll);
  const double kNegInf = __longlong_as_double((long long)0xfff0000000000000ull);
  auto ds_store = [&]() {  // commit the open window's aggregate
    const uint64_t o = acc.o;
    if constexpr (CTR) {
      p.ds_isum[o] = acc.sum;
      p.ds_count[o] = (int64_t)acc.cnt;
      p.ds_imin[o] = acc.mn;
      p.ds_imax[o] = acc.mx;
      p.ds_isum_sq[o] = acc.sq;
    } else {
      const bool none = acc.mn == kPosInf && acc.mx == kNegInf;  // no non-NaN value in the window
      p.ds_sum[o] = acc.sum;
      p.ds_count[o] = (int64_t)acc.cnt;
      p.ds_min[o] = none ? kNaN : acc.mn;
      p.ds_max[o] = none ? kNaN : acc.mx;
      if (LAST) {
        p.ds_last[o] = __longlong_as_double((long long)acc.last_v);
        p.ds_last_at[o] = acc.last_t;
      }
      if constexpr (SQ) p.ds_sum_sq[o] = acc.sq;
    }
    if constexpr (ANN) p.ds_ann[o] = wa.ref;
  };
  auto ds_store_empty = [&](int32_t w) {  // NewGauge: sum 0, count 0, min/max NaN, last 0 (gauge.go:45-51)
    const uint64_t o = (uint64_t)(uint32_t)w * p.n_series + sidx;
    if constexpr (CTR) {  // NewCounter: sum 0, count 0, min MaxInt64, max MinInt64, sumSq 0 (counter.go:44-50)
      p.ds_isum[o] = 0;
      p.ds_count[o] = 0;
      p.ds_imin[o] = kMaxI64;
      p.ds_imax[o] = kMinI64;
      p.ds_isum_sq[o] = 0;
    } else {
      p.ds_sum[o] = 0.0;
      p.ds_count[o] = 0;
      p.ds_min[o] = kNaN;
      p.ds_max[o] = kNaN;
      if (LAST) {
        p.ds_last[o] = 0.0;
        p.ds_last_at[o] = 0;
      }
      if constexpr (SQ) p.ds_sum_sq[o] = 0.0;
    }
    if constexpr (ANN) p.ds_ann[o] = 0;
  };
  auto ds_reset = [&]() {
    if constexpr (ANN) wa.ref = 0;
    if constexpr (CTR) {
      acc.sum = 0;
      acc.cnt = 0;
      acc.mn = kMaxI64;
      acc.mx = kMinI64;
      acc.sq = 0;
    } else {
      acc.sum = 0.0;
      acc.cnt = 0;
      acc.mn = kPosInf;
      acc.mx = kNegInf;
      if constexpr (SQ) acc.sq = 0.0;
    }
  };
  // Counter.Update without lastAt and count (counter.go:52-78): x = int64(value), int64 arithmetic that wraps
  auto ctr_add = [&](uint64_t vbits) {
    const int64_t x = go_f64_to_i64(__longlong_as_double((long long)vbits));
    acc.sum = (int64_t)((uint64_t)acc.sum + (uint64_t)x);
    if (acc.mx < x) acc.mx = x;
    if (acc.mn > x) acc.mn = x;
    acc.sq = (int64_t)((uint64_t)acc.sq + (uint64_t)x * (uint64_t)x);
  };
  auto ds_add = [&](uint64_t vbits) {  // Gauge.updateTotals without `last` and `count` (gauge.go:85-101)
    if constexpr (CTR) {
      ctr_add(vbits);
    } else {
      const double dv = __longlong_as_double((long long)vbits);
      if (dv == dv) acc.sum = __dadd_rn(acc.sum, dv);
      if (dv > acc.mx) acc.mx = dv;
      if (dv < acc.mn) acc.mn = dv;
      if constexpr (SQ) {  // after the NaN check, a separate multiply and add (gauge.go:101-103)
        if (dv == dv) acc.sq = __dadd_rn(acc.sq, __dmul_rn(dv, dv));
      }
    }
  };
  auto ds_add_no_nan = [&](uint64_t vbits) {  // ... when no lane of the warp holds a NaN
    if constexpr (CTR) {
      ctr_add(vbits);
    } else {
      const double dv = __longlong_as_double((long long)vbits);
      acc.sum = __dadd_rn(acc.sum, dv);
      if (dv > acc.mx) acc.mx = dv;
      if (dv < acc.mn) acc.mn = dv;
      if constexpr (SQ) acc.sq = __dadd_rn(acc.sq, __dmul_rn(dv, dv));
    }
  };

  // refills are DEC_FILL-word aligned: start at the stream's first word rounded down
  uint32_t filled = (s.pos >> 5) & ~(uint32_t)(DEC_FILL - 1);  // words [.., filled) requested
  uint32_t safe = filled;                                       // words [.., safe) have landed
  uint32_t group_row0 = 0;  // datapoint index of the output group's row 0 (warp-uniform)
  uint64_t o_t[4] = {0, 0, 0, 0}, o_v[4] = {0, 0, 0, 0};  // the group's datapoints
  // row 0 of every group is 32-byte aligned when the arrays are and cap is a multiple of 4
  const bool out_aligned =
      MODE == 0 && (((uintptr_t)p.ts | (uintptr_t)p.val) & 31u) == 0 && (p.cap & 3u) == 0;  // series-major only
  // running output pointers of this lane's series (MODE 0)
  uint64_t *dt = nullptr, *dv = nullptr;
  if (MODE == 0) {
    dt = reinterpret_cast<uint64_t *>(p.ts) + sidx * p.cap;
    dv = reinterpret_cast<uint64_t *>(p.val) + sidx * p.cap;
  }
  if (PM) {  // row `r` of series s lives at r * n_series + s: the pointers advance one row per step
    dt = reinterpret_cast<uint64_t *>(p.ts) + sidx;
    dv = reinterpret_cast<uint64_t *>(p.val) + sidx;
  }
  // scheme/unit admit the fast path (they only change on the slow path)
  bool su_ok = false;
  // maintained flags: `live` = lane still decoding; they change on the general path only
  bool live = !s.done && s.err == 0;
  bool fast_en = false;  // live && su_ok

  for (;;) {  // one group of DEC_GROUP datapoints per iteration
    if (!__any_sync(FULL_MASK, live)) break;

    // ---- ring maintenance (every DEC_CHK datapoints) ----
    // A refill EVENT is warp-wide: it first waits for the previous event's copies
    // (issued many datapoints ago, so normally landed), then every lane with room
    // takes another 16-word chunk.  Lanes that nevertheless run dry fall back to
    // the slow path (reads global memory), so the thresholds only tune speed.
    {
      const bool active = live;
      const uint32_t cw = s.pos >> 5;
      int avail = (int)(filled - cw);
      if (__any_sync(FULL_MASK, active && (avail <= DEC_TRIGGER ||
                                           ((int)(safe - cw) < DEC_SAFE_MIN && filled > safe)))) {
        cp_async_wait_all();
        __syncwarp();
        if (avail < 0) {  // the slow path skipped past the ring (annotation): restart at cw
          filled = cw & ~(uint32_t)(DEC_FILL - 1);
          avail = (int)(filled - cw);
        }
        safe = filled;
#pragma unroll 1
        for (int rep = 0; rep < 3; rep++) {
          // first pass: everyone with room tops up when someone is at the trigger level;
          // later passes only serve lanes that are still short (start-up / restart)
          const bool trig = __any_sync(FULL_MASK, active && avail <= DEC_TRIGGER);
          if (!trig) break;
          const uint32_t fmask =
              __ballot_sync(FULL_MASK, active && avail <= (rep == 0 ? DEC_ACCEPT : DEC_TRIGGER));
          if (!fmask) break;
          ring_fill(ring_lane_addr, p.streams, p.streams_bytes, (fmask >> lane) & 1u, gbase + filled,
                    (filled >> 2) & (DEC_QUADS - 1));
          if ((fmask >> lane) & 1u) {
            filled += DEC_FILL;
            avail += DEC_FILL;
          }
        }
        if (__any_sync(FULL_MASK, active && cw + DEC_FAST_WORDS > safe && filled > safe)) {
          cp_async_wait_all();  // start-up / restart only: nothing landed yet
          __syncwarp();
          safe = filled;
        }
      }
    }

    // Hot-path conditions that cannot change while the group stays on the hot path,
    // checked once with margins for DEC_CHK datapoints of <= 80 bits each: words
    // landed, distance to the end of the stream, not the first datapoint and no
    // wrap of prev_time to 0 (first <=> PrevTime == 0, timestamp_iterator.go:89),
    // float mode.
    bool pre_ok = fast_en && (((s.pos + 80u * (DEC_CHK - 1)) >> 5) + DEC_FAST_WORDS <= safe) &&
                  (s.pos + 80u * DEC_CHK <= s.end) && (s.prev_time > 0) &&
                  ((uint64_t)s.prev_delta < (1ull << 60)) && (!INT_OPT || s.is_float);
    if (DS) {
      // fused downsample, additionally: timestamps strictly increasing in steps of at most one
      // window (so a datapoint is in the open window or opens the next one), the last datapoint
      // inside the open window, the open window is the newest one (no committed window ahead that
      // would have to be re-opened), and at least four more windows before the end of the range
      // (four datapoints advance at most four windows).  Only the last compare is per group: the
      // rest is a flag maintained where it can change (general path, window advance).
      // (a finished lane keeps d < 0 and delta == 0: the hot path's advance test needs no `active`)
      acc.d = live ? (int64_t)((uint64_t)s.prev_time - (uint64_t)acc.w_end) : -1ll;
      pre_ok = pre_ok && acc.in_open && acc.cur_w == acc.hi_w && s.prev_delta > 0 && s.prev_delta <= p.window &&
               (uint32_t)acc.cur_w + (uint32_t)DEC_CHK < p.n_windows;
    }
    // one vote per group: the per-datapoint vote below then only looks at the header bits.  The flag is
    // warp-uniform: a general-path datapoint (taken by the whole warp) clears it for the rest of the group.
    bool group_ok = __all_sync(FULL_MASK, pre_ok || !live);

#pragma unroll
    for (int rr = 0; rr < DEC_CHK; rr++) {
      const bool active = live;
      const uint32_t cw = s.pos >> 5;
      int64_t t = 0;
      uint64_t v = 0;
      bool emitted = false;
      uint64_t dp_ann = 0;  // modes 6-8: the annotation reference this datapoint carries (slow path only)
      (void)dp_ann;
      // ---------------- parse: the 128-bit window at the current word ----------------
      const uint32_t sh = s.pos & 31u;
      // the window = words cw .. cw+3 of the lane's ring column (16-byte cells, [quad][lane]), as the five
      // words u0..u4 from the even word e = cw & ~1 on; the byte swap then picks word e+i or e+i+1 (PRMT
      // on its first or its second operand).  Selector and addresses come from the bit position with
      // multiply-adds (FMA pipe): the kernels are ALU-pipe-bound (rt 2 cycles per warp instruction).
      const uint32_t r3 = s.pos >> 3;
      const uint32_t psel = 0x0123u + (r3 & 4u) * 0x1111u;  // 0x0123: swap(a), 0x4567: swap(b)
      uint32_t u0, u1, u2, u3, u4;
      if (RING64) {
        // two 8-byte pairs + one word (pair p = cw >> 1 sits at quad p >> 1, half p & 1: pair p+1 is 8 bytes
        // on, or 504 on in the next quad's cell; pair p+2 is always one quad = 512 bytes on, the mirror quad
        // covering the wrap): no selects (6 ALU instructions fewer per datapoint), but 12 shared-memory
        // wavefronts instead of 8 (2-way / 4-way bank conflicts) -- pays where the L1 pipe has room: the fused
        // downsample and point-major decode with 92 KB of L1; not series-major decode, whose sector stores
        // already fill that pipe
        const uint32_t t8 = r3 & 8u;  // (p & 1) * 8
        const uint32_t a0 = ring_lane_addr + ((s.pos << 2) & ((DEC_QUADS - 1) * 512u)) + t8;
        const uint32_t a1 = a0 + t8 * 62u;  // + 8 below: +8 or +504
        asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(u0), "=r"(u1) : "r"(a0));
        asm volatile("ld.shared.v2.u32 {%0, %1}, [%2+8];" : "=r"(u2), "=r"(u3) : "r"(a1));
        asm volatile("ld.shared.u32 %0, [%1+512];" : "=r"(u4) : "r"(a0));
      } else {
        // two conflict-free LDS.128 (quads q, q+1) and one select level on (cw & 2)
        const uint4 *qp = reinterpret_cast<const uint4 *>(ring_lane) + ((cw >> 2) & (DEC_QUADS - 1)) * 32;
        const uint4 qa = qp[0], qb = qp[32];
        const bool j2 = (cw & 2u) != 0;
        u0 = j2 ? qa.z : qa.x, u1 = j2 ? qa.w : qa.y, u2 = j2 ? qb.x : qa.z, u3 = j2 ? qb.y : qa.w,
        u4 = j2 ? qb.z : qb.x;
      }
      // (prmt.b32 directly: __byte_perm would mask the selector with 0x7777 first)
      uint32_t w0, w1, w2, w3;
      asm("prmt.b32 %0, %1, %2, %3;" : "=r"(w0) : "r"(u0), "r"(u1), "r"(psel));
      asm("prmt.b32 %0, %1, %2, %3;" : "=r"(w1) : "r"(u1), "r"(u2), "r"(psel));
      asm("prmt.b32 %0, %1, %2, %3;" : "=r"(w2) : "r"(u2), "r"(u3), "r"(psel));
      asm("prmt.b32 %0, %1, %2, %3;" : "=r"(w3) : "r"(u3), "r"(u4), "r"(psel));
      // 96-bit window at the bit position: (h, h1, h2); a field at offset c <= 32 is two more funnels
      const uint32_t h = __funnelshift_l(w1, w0, sh), h1 = __funnelshift_l(w2, w1, sh),
                     h2 = __funnelshift_l(w3, w2, sh);
#define M3_FIELD64(c_) \
  (((uint64_t)__funnelshift_lc(h1, h, (c_)) << 32) | (uint64_t)__funnelshift_lc(h2, h1, (c_)))

      // ---- hot candidate: zero delta-of-delta, float XOR code (skipped once the group left the hot path) ----
      if (group_ok) {
        uint32_t x = h << 1;
        uint32_t c = 1;
        // '0' zero DoD [+ '1' no update]: top bits 01 <=> signed h >= 0x40000000 (one compare)
        const bool hot = INT_OPT ? ((int32_t)h >= 0x40000000) : ((int32_t)h >= 0);
        if (INT_OPT) {
          x <<= 1;
          c = 2;
        }
        const bool zero = !(x >> 31);
        const bool cont = (x >> 30) == 2u;
        const int lz = (int)((x >> 24) & 63u);
        const int nunc = (int)((x >> 18) & 63u) + 1;
        int n = cont ? (64 - plz - ptz) : nunc;
        const int tz = cont ? ptz : (64 - lz - nunc);
        c += cont ? 2u : 14u;
        if (zero) {
          n = 0;
          c -= cont ? 1u : 13u;
        }
        const uint64_t field = M3_FIELD64(c);
        c += (uint32_t)n;
        const bool take = __all_sync(FULL_MASK, hot || !active);
        if (take) {
          // every live lane: unconditional update (finished lanes compute garbage
          // they never read again)
          s.pos += c;
          // xor = (top n bits of the field) << tz; nothing for the zero code, an empty contained
          // window (previous XOR zero) or a malformed uncontained header (lz + n > 64: the
          // reference shifts everything out)
          // (clamping PTX shifts: n == 0 shifts right by 64, tz < 0 shifts left by > 63 -- both give 0)
          const uint64_t xr = shl64_clamp(shr64_clamp(field, 64u - (uint32_t)n), (uint32_t)tz);
          if (PLAIN) {
            s.prev_time = (int64_t)((uint64_t)s.prev_time + (uint64_t)s.prev_delta);
            s.prev_xor = xr;
            s.prev_bits ^= xr;
            lz_tz(xr, plz, ptz);
            if (PM) {
              if (active && group_row0 + (uint32_t)rr < (uint32_t)p.cap) {
                dt[0] = (uint64_t)s.prev_time;
                dv[0] = s.prev_bits;
              }
              dt += p.n_series;
              dv += p.n_series;
            } else {
              o_t[rr] = (uint64_t)s.prev_time;
              o_v[rr] = s.prev_bits;
            }
            s.n += (uint32_t)active;
            continue;
          } else {
            // this datapoint's time relative to the end of the open window; a lane whose datapoint opens
            // the next window (adv: d >= 0, the sign of the high word) commits in place.  NaN values ride on
            // the same vote: without one in the warp the accumulate needs no NaN select (gauge.go:85-101).
            acc.d = (int64_t)((uint64_t)acc.d + (uint64_t)s.prev_delta);
            int32_t d_lo, d_hi;  // (unpacked in PTX: a 64-bit compare would be two instructions)
            asm("mov.b64 {%0, %1}, %2;" : "=r"(d_lo), "=r"(d_hi) : "l"(acc.d));
            const bool adv = d_hi >= 0;
            const uint64_t nb = s.prev_bits ^ xr;
            const double nbd = __longlong_as_double((long long)nb);
            if (__any_sync(FULL_MASK, adv || (!CTR && nbd != nbd))) {  // (a Counter needs no NaN vote)
              if (adv) {  // it opens the next window: commit the one it leaves
                const uint32_t hot_n = s.n - acc.n_sync;  // hot datapoints since cnt was last updated
                if (LAST && hot_n) {  // `last` of in-order datapoints = the previous one
                  acc.last_t = (int64_t)((uint64_t)acc.d - (uint64_t)s.prev_delta + (uint64_t)acc.w_end);
                  acc.last_v = s.prev_bits;
                }
                acc.cnt += hot_n;
                acc.n_sync = s.n;
                ds_store();
                acc.cur_w++;
                acc.hi_w = acc.cur_w;
                acc.o += p.n_series;
                acc.w_end += p.window;
                acc.d -= p.window;
                ds_reset();
              }
              ds_add(nb);
            } else {
              ds_add_no_nan(nb);
            }
            s.prev_xor = xr;
            s.prev_bits = nb;
            lz_tz(xr, plz, ptz);
            // (finished lanes committed their window when they stopped: what they add here is never read)
            s.n++;  // also this window's count: cnt += s.n - n_sync at the next commit / general visit
            continue;
          }
        }
      }

      // ---------------- general path (any mix of cases) ----------------
      {
        if (DS && group_ok && live)  // leaving the hot path: prev_time was carried in acc.d
          s.prev_time = (int64_t)((uint64_t)acc.d + (uint64_t)acc.w_end);
        group_ok = false;  // the group's pre-check does not survive a general-path datapoint
        if (DS) {  // fold the hot datapoints since the last visit into the open window's count
          const uint32_t hot_n = s.n - acc.n_sync;
          if (LAST && hot_n) {  // ... and the newest of them is `last`
            acc.last_t = s.prev_time;
            acc.last_v = s.prev_bits;
          }
          acc.cnt += hot_n;
        }
        bool ok = fast_en && (cw + DEC_FAST_WORDS <= safe) && (s.prev_time != 0);
        uint32_t c = 1;  // bits consumed before the payload
        int64_t dod = 0;
        if (h >> 31) {
          const bool m9 = (h >> 30) == 2u, m12 = (h >> 29) == 6u, m16 = (h >> 28) == 14u;
          const bool marker = (h >> 23) == kMarkerOpcode;
          const int32_t f = m9 ? (((int32_t)(h << 2)) >> 25)
                               : (m12 ? (((int32_t)(h << 3)) >> 23) : (((int32_t)(h << 4)) >> 20));
          c = m9 ? 9u : (m12 ? 12u : 16u);
          ok = ok && (m9 || m12 || m16) && !marker;
          dod = (int64_t)((uint64_t)(int64_t)f * (uint64_t)s.unit_ns);
        }
        uint32_t x = h << c;
        // value grammar (iterator.go:128-176); kinds: float-next / int-diff / repeat /
        // update to float mode (full 64-bit value) / update of the int header + diff
        bool k_float = true, k_int = false, k_full = false, k_hdr = false;
        int nsig = s.sig, nmult = s.mult;
        if (INT_OPT) {
          const bool b0 = (x >> 31) != 0;
          const bool rep = !b0 && ((x >> 30) & 1u);
          k_float = b0 && s.is_float;
          k_int = b0 && !s.is_float;
          c += b0 ? 1u : 2u;
          x <<= 1;
          if (!b0 && !rep) {  // opcodeUpdate, not a repeat (divergent, infrequent)
            c += 1;           // float / int mode flag
            if ((x >> 30) & 1u) {
              k_full = true;
            } else {  // readIntSigMult, iterator.go:178-193; <= 12 more header bits
              k_hdr = true;
              k_int = true;
              uint32_t y = x << 2;
              if (y >> 31) {
                if ((y >> 30) & 1u) {
                  nsig = (int)((y >> 24) & 63u) + 1;
                  y <<= 8;
                  c += 8;
                } else {
                  nsig = 0;
                  y <<= 2;
                  c += 2;
                }
              } else {
                y <<= 1;
                c += 1;
              }
              if (y >> 31) {
                nmult = (int)((y >> 28) & 7u);
                c += 4;
              } else {
                c += 1;
              }
              ok = ok && (nmult <= kMaxMult);  // the error case is the slow path's
            }
          }
          ok = ok && !(k_int && nsig == 64);
        }
        const bool zero = !(x >> 31);
        const bool cont = (x >> 30) == 2u;
        const int lz = (int)((x >> 24) & 63u);
        const int nunc = (int)((x >> 18) & 63u) + 1;
        int n = cont ? (64 - plz - ptz) : nunc;
        int tz = cont ? ptz : (64 - lz - nunc);
        uint32_t hb = cont ? 2u : 14u;
        if (zero) {
          n = 0;
          hb = 1;
        }
        if (INT_OPT && !k_float) {
          hb = 0;
          n = k_int ? nsig + 1 : (k_full ? 64 : 0);
        }
        c += hb;
        const uint64_t field = M3_FIELD64(c);
        const uint64_t payload = n ? (field >> (64 - n)) : 0ull;
        c += (uint32_t)n;
        if (ok) {
          if (s.pos + c > s.end) {
            s.err = M3TSZ_ERR_EOF;  // truncated stream: the datapoint is not produced
          } else {
            s.pos += c;
            s.prev_delta = (int64_t)((uint64_t)s.prev_delta + (uint64_t)dod);
            s.prev_time = (int64_t)((uint64_t)s.prev_time + (uint64_t)s.prev_delta);
            if (k_float) {
              const uint64_t xr = (tz < 0) ? 0ull : (payload << tz);
              s.prev_xor = xr;
              s.prev_bits ^= xr;
              lz_tz(xr, plz, ptz);
            }
            if (INT_OPT && k_full) {  // readFullFloat, float_encoder_iterator.go:105-115
              s.prev_bits = payload;
              s.prev_xor = payload;
              lz_tz(payload, plz, ptz);
              s.is_float = true;
            }
            if (INT_OPT && k_hdr) {
              s.sig = nsig;
              s.mult = nmult;
              s.is_float = false;
            }
            t = s.prev_time;
            v = s.prev_bits;
            emitted = true;
            if (INT_OPT && !s.is_float) {  // int mode: diff or repeat
              if (k_int) {
                const uint64_t neg = payload >> s.sig;
                const uint64_t mag = payload & ((1ull << s.sig) - 1ull);
                const double m = __ull2double_rn(mag);
                s.int_val = neg ? __dadd_rn(s.int_val, m) : __dsub_rn(s.int_val, m);
              }
              const double dvv = s.mult ? __ddiv_rn(s.int_val, mult_pow10(s.mult)) : s.int_val;
              v = (uint64_t)__double_as_longlong(dvv);
            }
          }
        } else if (active) {  // complete grammar, from global memory
          DecState tmp = s;   // copy-in / copy-out keeps the lane state in registers
          int64_t st = 0;
          uint64_t sv = 0;
          SlowSrc src;
          src.base = p.streams;
          src.nbytes = p.streams_bytes;
          src.ring_lane = ring_lane;
          src.ring_safe = ((int)(filled - cw) >= 0) ? safe : 0u;  // ring abandoned after a skip
          EventSink evs;
          evs.events = p.events;
          evs.capacity = p.events_capacity;
          evs.count = p.event_count;
          evs.series = sidx;
          evs.pos0 = pos0;
          if constexpr (ANN) tmp.ann_count = 0;  // (no per-series annotation output in these modes)
          bool em = decode_dp_slow<INT_OPT>(tmp, src, p.default_unit, st, sv, &evs);
          if constexpr (ANN) {
            // the annotation of this datapoint, the last marker before it, as (bit offset from the stream's first
            // bit) << 32 | length in bytes: the stream limit of 2^28 bytes keeps both in 32 bits, and a length is at
            // least 1.  BLK: (bit offset from the first bit of the batch) << kBlockAnnLenBits | length, so that the
            // encoder needs no block table; a longer annotation rejects the series
            if (em && tmp.ann_count) {
              uint32_t abit = tmp.ann_bit, alen = tmp.ann_len;
              if (tmp.ann_count > 1) dec_last_annotation(src, tmp.wbase, tmp.ann_count, &abit, &alen);
              if constexpr (BLK) {
                if (alen >> kBlockAnnLenBits) {
                  tmp.err = M3TSZ_ERR_STREAM_TOO_LARGE;
                  em = false;
                } else {
                  dp_ann = ((tmp.wbase * 32ull + abit) << kBlockAnnLenBits) | alen;
                }
              } else {
                dp_ann = ((uint64_t)(abit - pos0) << 32) | alen;
              }
            }
          }
          s = tmp;
          t = st;
          v = sv;
          emitted = em;
          lz_tz(s.prev_xor, plz, ptz);
          su_ok = (s.scheme == kScheme32 || s.scheme == kScheme64) && (s.unit >= 1 && s.unit <= 4);
          if constexpr (BLK) {
            // the end of a block opens the next one in this step; its first datapoint takes the slow path (prev_time
            // 0), which reads global memory until the next refill event fills the ring from the new block (that
            // event first waits for the copies still in flight from the old one)
            if (s.done && s.err == 0 && next_block()) {
              plz = 64;
              ptz = 0;
              su_ok = false;
              gbase = (uint32_t)s.wbase;
              filled = (s.pos >> 5) & ~(uint32_t)(DEC_FILL - 1);
              safe = filled;
            }
          }
        }
        live = !s.done && s.err == 0;
        fast_en = live && su_ok;
      }

      // ---------------- sink (general path) ----------------
      if (PLAIN) {
        if (emitted) {
          // (a live lane produces exactly one datapoint per step: this one is row group_row0 + rr)
          if (PM) {
            if (group_row0 + (uint32_t)rr < (uint32_t)p.cap) {
              dt[0] = (uint64_t)t;
              dv[0] = v;
            }
          } else {
            o_t[rr] = (uint64_t)t;
            o_v[rr] = v;
          }
          s.n++;
        }
        if (PM) {
          dt += p.n_series;
          dv += p.n_series;
        }
      } else {
        if (emitted) {
          s.n++;
          // inside the open window (one unsigned compare covers both bounds; an open window
          // lies inside the range)?  Otherwise: inside the range at all?
          bool in_win = acc.cur_w >= 0 && (uint64_t)(t - (acc.w_end - p.window)) < (uint64_t)p.window;
          const bool in_range = t >= p.range_start && t < range_end;
          if (!in_win && in_range) {
            // commit the window we are leaving
            if (acc.cur_w >= 0) ds_store();
            int64_t nw;
            if (acc.cur_w >= 0 && t >= acc.w_end && t - acc.w_end < p.window)
              nw = (int64_t)acc.cur_w + 1;
            else
              nw = (int64_t)((uint64_t)(t - p.range_start) / (uint64_t)p.window);
            acc.o = (uint64_t)nw * p.n_series + sidx;
            if (nw > (int64_t)acc.hi_w) {
              for (int64_t w = (int64_t)acc.hi_w + 1; w < nw; w++) ds_store_empty((int32_t)w);
              acc.hi_w = (int32_t)nw;
              ds_reset();
            } else {  // out-of-order timestamp: reopen a committed window
              const uint64_t o = acc.o;
              if constexpr (CTR) {
                acc.sum = p.ds_isum[o];
                acc.cnt = (uint32_t)p.ds_count[o];
                acc.mn = p.ds_imin[o];
                acc.mx = p.ds_imax[o];
                acc.sq = p.ds_isum_sq[o];
              } else {
                acc.sum = p.ds_sum[o];
                acc.cnt = (uint32_t)p.ds_count[o];
                acc.mn = p.ds_min[o];
                acc.mx = p.ds_max[o];
                if (acc.mn != acc.mn) {  // stored as NaN / NaN: no value yet
                  acc.mn = kPosInf;
                  acc.mx = kNegInf;
                }
                if (LAST) {
                  acc.last_v = (uint64_t)__double_as_longlong(p.ds_last[o]);
                  acc.last_t = p.ds_last_at[o];
                }
                if constexpr (SQ) acc.sq = p.ds_sum_sq[o];
              }
              if constexpr (ANN) wa.ref = p.ds_ann[o];
            }
            acc.cur_w = (int32_t)nw;
            acc.w_end = p.range_start + (nw + 1) * p.window;
            in_win = true;
          }
          acc.in_open = in_win;
          if (in_win) {
            if constexpr (ANN)
              if (dp_ann) wa.ref = dp_ann;  // an empty annotation keeps the window's earlier one
            // lastAt.IsZero() || timestamp.After(lastAt), gauge.go:74-81 (NaN values included)
            if (LAST && (acc.cnt == 0 || t > acc.last_t)) {
              acc.last_t = t;
              acc.last_v = v;
            }
            acc.cnt++;
            ds_add(v);
          }
        }
        acc.n_sync = s.n;  // everything up to here is accounted for
        if (!live && active) {
          // this lane is done: commit its open window and publish its counters now, so that the
          // hot path may run its unconditional updates on finished lanes without harm
          if (acc.cur_w >= 0) ds_store();
          acc.cur_w = -1;
          acc.in_open = false;
          acc.d = -1;
          s.prev_delta = 0;
          if (p.n_points) p.n_points[sidx] = s.n;
          if (p.status) p.status[sidx] = s.err;
        }
      }
    }
    if (DS && group_ok && live)  // the group stayed hot: materialise prev_time for the next pre-check
      s.prev_time = (int64_t)((uint64_t)acc.d + (uint64_t)acc.w_end);

    // ---------------- store the group: each lane writes its own series ----------------
    // Every live lane emits exactly one datapoint per step until it stops, so the group's
    // rows are o_t/o_v[0 .. my_rows).  4 rows = one 32-byte sector per array, written as two
    // 16-byte stores (STG.128, the widest sm_90 has) when the row is 32-byte aligned.
    if (MODE == 0 && valid) {
      const uint32_t lim = s.n < (uint32_t)p.cap ? s.n : (uint32_t)p.cap;
      const uint32_t my_rows = lim > group_row0 ? min(lim - group_row0, 4u) : 0u;
      if (my_rows == 4u && out_aligned) {
        asm volatile("st.global.v2.b64 [%0], {%1, %2};\n\tst.global.v2.b64 [%0+16], {%3, %4};" ::"l"(dt),
                     "l"(o_t[0]), "l"(o_t[1]), "l"(o_t[2]), "l"(o_t[3])
                     : "memory");
        asm volatile("st.global.v2.b64 [%0], {%1, %2};\n\tst.global.v2.b64 [%0+16], {%3, %4};" ::"l"(dv),
                     "l"(o_v[0]), "l"(o_v[1]), "l"(o_v[2]), "l"(o_v[3])
                     : "memory");
      } else {
#pragma unroll
        for (int r = 0; r < 4; r++)
          if ((uint32_t)r < my_rows) {
            dt[r] = o_t[r];
            dv[r] = o_v[r];
          }
      }
      dt += DEC_GROUP;
      dv += DEC_GROUP;
    }
    group_row0 += DEC_CHK;
  }
  cp_async_wait_all();

  // ---------------- epilogue ----------------
  if (DS && valid) {
    if (acc.cur_w >= 0) ds_store();
    for (int64_t w = (int64_t)acc.hi_w + 1; w < (int64_t)p.n_windows; w++) ds_store_empty((int32_t)w);
  }
  if (valid) {
    int st = s.err;
    if (PLAIN) {
      if (p.n_points) p.n_points[sidx] = s.n;
      if (st == 0 && s.n > p.cap) st = M3TSZ_ERR_CAPACITY;
      if (p.status) p.status[sidx] = st;
    }
    if (p.unit_out) p.unit_out[sidx] = (uint8_t)(s.n ? s.emit_unit : s.unit);
    if (p.unit_first_out) p.unit_first_out[sidx] = (uint8_t)(s.n ? s.first_unit : s.unit);
    if (p.ann_out) {
      m3tsz_annotation_ref a;
      a.bit_offset = s.ann_count ? (uint64_t)(s.ann_bit - pos0) : 0ull;
      a.length = s.ann_len;
      a.count = s.ann_count;
      p.ann_out[sidx] = a;
    }
  }
}

#undef M3_FIELD64

template <bool INT_OPT, int MODE, bool BLK = false>
static cudaError_t launch_one(const DecodeParams &p, cudaStream_t stream) {
  constexpr size_t smem = DEC_WARP_SMEM_PLAIN * DEC_WARPS;
  cudaError_t e = cudaFuncSetAttribute(decode_kernel<INT_OPT, MODE, BLK>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  // Shared-memory carveout = resident blocks x 35.8 KB; the rest of the SM's 256 KB of L1 + shared memory is
  // L1, which holds the fills in flight (cp.async.ca allocates a line per request).  Measured on an H100 SXM (700 W, 1980 MHz) at
  // 500 k x 1440, int-optimised (ms, carveout 100 / 132 / 164 / 196 / 228 KB): point-major decode 8.22 / 7.59 /
  // 7.60 / 7.58 / 8.57, fused downsample 6.36 / 5.37 / 5.00 / 4.98 / 5.78.  So: plain decode 4 blocks + 92 KB
  // of L1, fused downsample 5 blocks + 60 KB.
  constexpr int carveout_kb = dec_ds_mode(MODE) ? 196 : 164;
  e = cudaFuncSetAttribute(decode_kernel<INT_OPT, MODE, BLK>, cudaFuncAttributePreferredSharedMemoryCarveout,
                           carveout_kb * 100 / 228);
  if (e != cudaSuccess) return e;
  const uint64_t per_block = (uint64_t)DEC_WARPS * 32ull;
  const uint64_t blocks = (p.n_series + per_block - 1) / per_block;
  if (blocks == 0) return cudaSuccess;
  if (blocks > 0x7fffffffull) return cudaErrorInvalidValue;
  decode_kernel<INT_OPT, MODE, BLK><<<(unsigned)blocks, DEC_WARPS * 32, smem, stream>>>(p);
  return cudaGetLastError();
}

// mode: 0 plain decode (series-major), 1 fused downsample (sum/count/min/max), 2 + last, 3 plain decode (point-major),
// 4 fused downsample + last + sumSq, 5 fused Counter downsample, 6 / 7 / 8: 2 / 4 / 5 + window annotations
cudaError_t launch_decode(const DecodeParams &p, bool int_optimized, int mode, cudaStream_t stream) {
  if (p.block_off) {  // several source blocks per series: the tile calls' modes only
    switch (mode) {
      case 2: return int_optimized ? launch_one<true, 2, true>(p, stream) : launch_one<false, 2, true>(p, stream);
      case 4: return int_optimized ? launch_one<true, 4, true>(p, stream) : launch_one<false, 4, true>(p, stream);
      case 5: return int_optimized ? launch_one<true, 5, true>(p, stream) : launch_one<false, 5, true>(p, stream);
      case 6: return int_optimized ? launch_one<true, 6, true>(p, stream) : launch_one<false, 6, true>(p, stream);
      case 7: return int_optimized ? launch_one<true, 7, true>(p, stream) : launch_one<false, 7, true>(p, stream);
      case 8: return int_optimized ? launch_one<true, 8, true>(p, stream) : launch_one<false, 8, true>(p, stream);
      default: return cudaErrorInvalidValue;
    }
  }
  switch (mode) {
    case 0: return int_optimized ? launch_one<true, 0>(p, stream) : launch_one<false, 0>(p, stream);
    case 1: return int_optimized ? launch_one<true, 1>(p, stream) : launch_one<false, 1>(p, stream);
    case 2: return int_optimized ? launch_one<true, 2>(p, stream) : launch_one<false, 2>(p, stream);
    case 3: return int_optimized ? launch_one<true, 3>(p, stream) : launch_one<false, 3>(p, stream);
    case 4: return int_optimized ? launch_one<true, 4>(p, stream) : launch_one<false, 4>(p, stream);
    case 5: return int_optimized ? launch_one<true, 5>(p, stream) : launch_one<false, 5>(p, stream);
    case 6: return int_optimized ? launch_one<true, 6>(p, stream) : launch_one<false, 6>(p, stream);
    case 7: return int_optimized ? launch_one<true, 7>(p, stream) : launch_one<false, 7>(p, stream);
    case 8: return int_optimized ? launch_one<true, 8>(p, stream) : launch_one<false, 8>(p, stream);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace m3tsz
