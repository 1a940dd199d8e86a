// m3tsz_kernels.h -- internal launch interface between the C-ABI layer
// (m3tsz_capi.cu) and the kernels (m3tsz_decode.cu, m3tsz_encode.cu).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/m3tsz_b200.h"

namespace m3tsz {

struct DecodeParams {
  const uint8_t *streams;
  uint64_t streams_bytes;
  const uint64_t *offsets;
  const uint64_t *lengths;  // optional [n_series]: stream s = [offsets[s], offsets[s] + lengths[s])
  uint64_t n_series;
  int default_unit;
  // plain decode outputs (series-major [n_series][cap])
  int64_t *ts;
  double *val;
  uint64_t cap;
  // fused downsample outputs (window-major [n_windows][n_series])
  int64_t range_start, window;
  uint32_t n_windows;
  double *ds_sum;
  int64_t *ds_count;
  double *ds_min;
  double *ds_max;
  double *ds_last;      // mode 2
  int64_t *ds_last_at;  // mode 2 (lastAt of every window; needed to re-open a window)
  // per-series outputs
  uint32_t *n_points;
  int32_t *status;
  uint8_t *unit_out;
  m3tsz_annotation_ref *ann_out;
  uint8_t *unit_first_out;
  // per-datapoint unit / annotation events (optional)
  m3tsz_dp_event *events;
  uint64_t events_capacity;
  unsigned long long *event_count;
  // modes 4 and 5 (after every older field, which keep their parameter offsets; window-major like the above)
  double *ds_sum_sq;    // mode 4: Gauge sumSq (+ the mode 2 outputs)
  int64_t *ds_isum, *ds_imin, *ds_imax, *ds_isum_sq;  // mode 5: Counter (+ ds_count)
  // modes 6-8 (after every older field): window-major annotation references, (bit offset of the payload from the
  // stream's first bit) << 32 | length in bytes, 0 for a window without one
  uint64_t *ds_ann;
  // several source blocks per series (m3tsz_aggregate_tiles_blocks; modes 2 and 4-8, after every older field):
  // offsets / lengths address n_segments segments, and series s decodes segments [block_off[s], block_off[s + 1])
  // one after another as one datapoint sequence.  ds_ann then holds (bit offset of the payload from the first bit of
  // `streams`) << kBlockAnnLenBits | length in bytes.
  const uint64_t *block_off;
  uint64_t n_segments;
};

// The length field of a block-mode annotation reference: an annotation of 2^27 bytes or more is refused
// (M3TSZ_ERR_STREAM_TOO_LARGE), so that a 37-bit bit offset (streams_bytes < 16 GiB) fits above it.
constexpr int kBlockAnnLenBits = 27;

// mode: 0 plain decode, 1 fused downsample (sum/count/min/max), 2 fused downsample + last, 3 point-major decode,
// 4 fused downsample + last + sumSq, 5 fused Counter downsample; 6 / 7 / 8: modes 2 / 4 / 5 + ds_ann.  With
// p.block_off (modes 2 and 4-8 only) the kernels that decode several source blocks per series.
cudaError_t launch_decode(const DecodeParams &p, bool int_optimized, int mode, cudaStream_t stream);

// The layout stays what it was before the tile stage's Counter and sumSq inputs: the kernel's second parameter (the
// tensor maps) follows this one, and every other encode_kernel keeps its parameter offsets and SASS.  The tile
// stage (IN = 2) reads no ts / val, so its window sumSq shares that first pointer, and a Counter's int64 sum / min /
// max share the Gauge's pointers.
struct EncodeParams {
  union {
    const int64_t *ts;
    const void *tile_sum_sq;  // IN = 2, SumSq / Stdev: window-major sumSq, double (Gauge) or int64 (Counter)
  };
  // IN = 6 (the multi-type stage with annotations) reads no val / n_points / annotation entries: the source streams,
  // their offsets and the window-major annotation references of the fused decode (DecodeParams::ds_ann) share them.
  // IN = 7 (the same over source blocks) reads the streams and the references only
  union {
    const double *val;
    const uint8_t *tile_src_streams;
  };
  uint64_t n_series;
  uint64_t points_stride;
  union {
    const uint32_t *n_points;  // optional
    const uint64_t *tile_src_off;
  };
  const int64_t *start;
  int unit;
  // IN = 4 (tile stage with transformations): the op list, op k in bits 4k .. 4k + 3, 0 ends it (in the padding
  // after `unit`, so no other field moves)
  uint32_t xf_ops;
  const uint8_t *units;  // optional per-datapoint units
  const uint64_t *ann_series_off;
  union {
    const m3tsz_annotation_entry *ann_entries;
    const uint64_t *tile_ann;  // [points_stride][tile_n_src]
  };
  const uint8_t *ann_bytes;
  int default_unit;
  int xf_discard_nan;  // IN = 4: a NaN result writes nothing of its window (in the padding after default_unit)
  uint8_t *out;
  uint64_t out_stride;
  uint64_t *out_len;
  int32_t *status;
  uint64_t *out_bits;   // optional [n_series]: stream length in bits (incl. the EOS marker)
  double *last_value;  // optional [n_series]: Encoder.LastEncoded().Value incl. the scaled-int quirk
  // packed mode (out = per-warp scratch slot sets, see encode_kernel)
  uint8_t *packed;
  uint64_t packed_capacity;
  uint64_t *packed_off;                // [n_series] start of every stream in `packed`
  unsigned long long *packed_cursor;   // bytes allocated so far (zero on entry)
  unsigned long long *batch_counter;   // work counter (zero on entry)
  uint32_t align;
  // input stage (see encode_kernel): 0 series-major ts/val, 1 point-major ts/val, 2 Gauge aggregates, 4 the
  // aggregates through the transformations, 5 an element's several types through them, 6 the same with the
  // windows' annotations
  int in_mode;
  // window-major [points_stride][n_series]; a Counter's (metric_type M3TSZ_METRIC_COUNTER) are int64
  union { const double *tile_sum; const int64_t *tile_isum; };
  union { const double *tile_min; const int64_t *tile_imin; };
  union { const double *tile_max; const int64_t *tile_imax; };
  // bucket writes (launch_encode_routed, IN = 3) share the tile stage's fields: the target encoder of every
  // datapoint, in the inputs' layout; lane j of the overflow pass continues record route_touched[j].rec (NULL: the
  // primary pass, lane s continues encoder 0 of series s); route_n_in is the number of input series
  union { const double *tile_last; const uint8_t *route_target; };
  union { const int64_t *tile_count; const struct RouteTouched *route_touched; };
  union { const int32_t *tile_src_status; const uint32_t *route_n_touched; };  // tile_src_status: optional [n_series]
  union { int64_t tile_start; uint64_t route_n_in; };
  int64_t tile_step;
  int agg_type;
  int metric_type;        // M3TSZ_METRIC_COUNTER, or the Gauge (M3TSZ_METRIC_GAUGE, or 0)
  uint32_t *n_tiles_out;  // optional [n_series]
  // encoder-set append (launch_encode_append): per-series state in, updated in place; datapoints taken.  The tile
  // stage with transformations (IN = 4) keeps its per-series transformation state (optional) in the same pointer,
  // and the multi-type stage (IN = 5) reads its per-series element state (optional) from it.
  union {
    m3tsz_encoder_state *state;
    m3tsz_transform_state *xf_state;
    const m3tsz_element_state *xf_elem;
  };
  // IN = 5: xf_elem_out (optional, [tile_n_src]) takes each lane's part of its series' new element record, which
  // launch_tiles_types_status commits
  union {
    uint32_t *n_appended;
    m3tsz_element_state *xf_elem_out;
  };
  // IN = 5 (an element's several aggregation types; after every older field, which keep their parameter offsets,
  // and inside the alignment gap before the tensor maps, which keep theirs): the launch's n_series rows are
  // tile_n_types * tile_n_src, row r is source series r % tile_n_src and type r / tile_n_src, type j's id is
  // (tile_types >> 4j) & 0xf
  uint64_t tile_n_src;
  uint32_t tile_types;
  uint32_t tile_n_types;
};

// an overflow record that a bucket write gave datapoints: pool record, its series, its encoder index (1..K-1)
struct RouteTouched {
  uint32_t rec, series, enc, reserved;
};

// what the route kernel reads and writes (launch_route, m3tsz_encode.cu)
struct RouteParams {
  m3tsz_encoder_state *state;  // [n_series]: encoder 0 of every bucket
  uint64_t n_series;
  uint64_t slot_words;  // words per primary slot
  m3tsz_encoder_state *pool_state;  // [pool_capacity]: encoders 1..K-1
  uint64_t pool_capacity;
  uint64_t pool_slot_words;
  uint32_t *pool_count;  // records in use
  int32_t *table;        // [n_series][K - 1] pool record of encoder i + 1, -1 = not open
  int n_encoders;        // K
  int default_unit;
  const int64_t *ts;
  const double *val;
  uint64_t points_stride;
  const uint32_t *n_points;
  int unit;
  int point_major;
  const uint8_t *units;
  const uint64_t *ann_series_off;
  const m3tsz_annotation_entry *ann_entries;
  const uint8_t *ann_bytes;
  uint8_t *target;  // per datapoint: encoder index, 0xff = not written
  int8_t *result;
  int32_t *status;
  RouteTouched *touched;  // [pool_capacity]
  uint32_t *n_touched;
};
// The tensor maps follow EncodeParams at the next 64-byte boundary of the constant bank, whose parameters start at
// 0x210: 304 bytes is the most EncodeParams can take without moving them (and every kernel's SASS with them).
static_assert(sizeof(EncodeParams) == 304, "the tensor maps follow EncodeParams: its size fixes their offset");

uint64_t encode_packed_resident_blocks();
// encoder sets (m3tsz_encode.cu): append runs encode_kernel's append mode over p.state / p.out (the slots)
cudaError_t launch_encode_append(const EncodeParams &p, bool int_optimized, cudaStream_t stream);
cudaError_t launch_encoder_set_reset(m3tsz_encoder_state *state, uint64_t n, const int64_t *start, int default_unit,
                                     bool int_optimized, cudaStream_t stream);
cudaError_t launch_encoder_set_stream(const m3tsz_encoder_state *state, uint64_t n, uint8_t *buf, uint64_t stride,
                                      uint64_t *len, cudaStream_t stream);
// bucket writes: route every datapoint to an encoder of its bucket, then append each encoder's share (encode_kernel's
// routed mode, once over the primary set and once over the overflow records the route touched)
cudaError_t launch_route(const RouteParams &p, bool int_optimized, cudaStream_t stream);
cudaError_t launch_encode_routed(const EncodeParams &p, bool int_optimized, cudaStream_t stream);
uint64_t encode_packed_scratch_slots(uint64_t n_series);  // slots of out_stride bytes the packed mode needs
cudaError_t launch_encode(const EncodeParams &p, bool int_optimized, cudaStream_t stream);

// iterator layer above the codec (m3tsz_merge.cu)
struct MergeParams {
  const int64_t *ts;  // decoded reader sequences [n_seq][cap]
  const double *val;
  uint64_t cap;
  const uint32_t *n_points;   // [n_seq]
  const int32_t *seq_status;  // optional [n_seq]
  const uint64_t *slice_off, *replica_off, *series_off;
  uint64_t n_series;
  int64_t start, end;
  int strategy;
  int64_t *ts_out;  // [n_series][out_cap]
  double *val_out;
  uint64_t out_cap;
  uint32_t *n_out;
  int32_t *status;
  // element strides: series-major [seq][cap] = (cap, 1); point-major [cap][n_seq] = (1, n_seq)
  uint64_t in_seq_stride, in_pt_stride, out_seq_stride, out_pt_stride;
};
cudaError_t launch_merge(const MergeParams &p, cudaStream_t stream);

struct ChecksumParams {
  const uint8_t *streams;
  uint64_t streams_bytes;
  const uint64_t *offsets;  // CSR [n_series + 1]
  const uint64_t *lengths;  // optional [n_series]: exact sizes when the starts are padded
  uint64_t n_series;
  const uint32_t *expected;  // optional: index-entry DataChecksum per stream
  uint32_t *out;             // optional: Adler-32 per stream
  int32_t *status;           // optional: OK / CHECKSUM_MISMATCH / INVALID_ARG / STREAM_TOO_LARGE
};
cudaError_t launch_checksum(const ChecksumParams &p, cudaStream_t stream);

// Prometheus conversion epilogue (m3tsz_query.cu)
struct PromParams {
  const int64_t *ts;  // [n_series][cap]
  const double *val;
  uint64_t cap;
  const uint32_t *n_points;
  uint64_t n_series;
  int64_t resolution;
  const uint8_t *handle_resets;  // optional [n_series]
  double tolerance;
  int64_t tolerance_until;
  int64_t *ts_out;  // [n_series][out_cap] milliseconds
  double *val_out;
  uint64_t out_cap;
  uint32_t *n_out;
  int32_t *status;  // optional
};
cudaError_t launch_prom(const PromParams &p, cudaStream_t stream);

// tile aggregation glue (m3tsz_query.cu)
cudaError_t launch_fill_i64(int64_t *dst, int64_t v, uint64_t n, cudaStream_t stream);
// the longest stream of a batch (offsets + lengths, or CSR offsets) into *out (zeroed by the caller); streams the
// decode refuses (outside the buffer, 2^28 bytes or more) are left out.  With block_off, over source blocks: the
// largest sum, over series s, of the lengths of segments [block_off[s], block_off[s + 1]) (a series with an invalid
// range counts 0); without, segment s is series s.
cudaError_t launch_max_stream_len(const uint64_t *offsets, const uint64_t *lengths, const uint64_t *block_off,
                                  uint64_t n_series, uint64_t n_segments, uint64_t streams_bytes,
                                  unsigned long long *out, cudaStream_t stream);
// The same room for the rollup's group rows: the largest sum, over groups g, of the segment lengths above of each
// member m < n_series listed in members[group_off[g] .. group_off[g + 1]) (a group with an invalid range counts 0)
cudaError_t launch_group_max_stream_len(const uint64_t *offsets, const uint64_t *lengths, const uint64_t *block_off,
                                        uint64_t n_series, uint64_t n_segments, uint64_t streams_bytes,
                                        const uint64_t *group_off, const uint32_t *members, uint64_t n_members,
                                        uint64_t n_groups, unsigned long long *out, cudaStream_t stream);
// a failed source's error goes to all n_types rows of its series; with `state`, a series whose source and rows are
// all OK takes its new record from `scratch`
cudaError_t launch_tiles_types_status(const int32_t *src_status, int32_t *status, uint64_t n, uint32_t n_types,
                                      const m3tsz_element_state *scratch, m3tsz_element_state *state,
                                      cudaStream_t stream);

// tile aggregation through a rollup (m3tsz_aggregate_tiles_rollup; m3tsz_encode.cu).  The forward stage: the lane
// that owns source series s runs its non-empty windows' values through the op list and writes the forwarded values
// series-major, fwd[s][w], with a presence bit per window, present[w / 32][s] bit w % 32 (NaN payloads are values).
struct RollupForwardParams {
  // the fused decode's window-major [n_windows][n_src] aggregates, in the fields the tile stages read them from
  // (tile_sum .. tile_count, tile_sum_sq, metric_type, tile_start, tile_step); tile_value_of takes them from here
  EncodeParams tiles;
  const int32_t *src_status;  // [n_src]: a failed source forwards nothing
  uint64_t n_src;
  uint32_t n_windows;
  uint32_t n_words;  // presence rows, ceil(n_windows / 32), of n_src words each
  int src_type;
  uint32_t ops;  // as EncodeParams::xf_ops
  int discard_nan;
  const m3tsz_transform_state *state;  // optional [n_src]
  m3tsz_transform_state *state_out;    // [n_src]: each source's new record (committed by launch_rollup_commit)
  double *fwd;
  uint32_t *present;
  // the annotated variant (after every older field, which keep their offsets): `ann` is the fused decode's window-major
  // [n_windows][n_src] references.  Without a block table (src_off = the sources' byte offsets) a reference holds
  // (bit offset from the stream's first bit) << 32 | length, and the stage rewrites a forwarded window's in place as
  // (bit offset from the batch's first bit) << kBlockAnnLenBits | length; with one it already has that form.  A
  // source with a window annotation of 2^27 bytes or more gets src_status_out[s] = M3TSZ_ERR_STREAM_TOO_LARGE.
  // ann_present[w / 32][s] bit w % 32: window w was forwarded and carries an annotation.
  uint64_t *ann;
  const uint64_t *src_off;
  int32_t *src_status_out;
  uint32_t *ann_present;
};
// The fold: window w of group g takes the forwarded values of its members, in listed order, and writes the aggregate
// slots of the fused decode over n_groups "series" (window-major [n_windows][n_groups], the same representation)
struct RollupFoldParams {
  const double *fwd;
  const uint32_t *present;
  const int32_t *src_status;
  uint64_t n_src;
  uint32_t n_windows;
  uint32_t n_words;
  const uint64_t *group_off;  // [n_groups + 1]
  const uint32_t *members;    // [n_members]
  uint64_t n_members;
  uint64_t n_groups;
  int counter;  // Counter.Update(int64(v)) into int64 slots, else Gauge.Update into double slots
  void *sum, *min, *max, *sum_sq;  // sum_sq optional
  int64_t *count;
  double *last;           // Gauge only
  int32_t *group_status;  // [n_groups]: INVALID_ARG for a bad range or index, else the first failing member's error
  // the annotated variant (after every older field): the forward stage's ann_present words and batch-addressed
  // references, and each group window's reference, window-major [n_windows][n_groups]: the last non-zero one of the
  // members, in listed order, whose window was forwarded (0: none, or the group failed)
  const uint32_t *ann_present;
  const uint64_t *ann;
  uint64_t *group_ann;
};
// annotated: the variants that carry the annotation references (p.ann / ann_present / group_ann)
cudaError_t launch_rollup_forward(const RollupForwardParams &p, bool annotated, cudaStream_t stream);
cudaError_t launch_rollup_fold(const RollupFoldParams &p, bool annotated, cudaStream_t stream);
// The source records (m3tsz_query.cu): a source takes its new record from `scratch` when it decoded and every group
// that lists it has all n_types rows OK; src_status_out (optional) takes each source's decode status.  `mark` is
// [n_src] bytes of scratch.
cudaError_t launch_rollup_commit(const uint64_t *group_off, const uint32_t *members, uint64_t n_members,
                                 uint64_t n_groups, const int32_t *status, uint32_t n_types, const int32_t *src_status,
                                 uint64_t n_src, uint8_t *mark, const m3tsz_transform_state *scratch,
                                 m3tsz_transform_state *state, int32_t *src_status_out, cudaStream_t stream);

// element sets (m3tsz_element_set_*; m3tsz_encode.cu): one lane per element over its open-window slots, window-slot
// major [n_slots][n] (slot r of element s at r * n + s)
struct ElementParams {
  uint64_t n;
  uint32_t n_slots;
  int counter;          // Counter: int64 sum / min / max / sumSq, no last; else the Gauge
  int64_t resolution;
  int64_t trunc_off;    // Go's Truncate origin: (the zero time's distance to the Unix epoch) % resolution
  int64_t *start, *count;
  void *sum, *min, *max, *sum_sq;
  double *last;
  int64_t *last_at;
  m3tsz_element_state *elem;
  int64_t *watermark;
  // add: point-major datapoints [points_stride][n]
  const int64_t *ts;
  const double *val;
  uint64_t points_stride;
  const uint32_t *n_points;  // optional
  int8_t *result;
  int32_t *status;
  // consume: the windows ending at or before `target` go to rows staged point-major [rows_stride][n_types * n]
  int64_t target;
  uint32_t types, n_types;  // type j's id in bits 4j .. 4j + 3
  uint32_t ops;             // as EncodeParams::xf_ops
  int discard_nan;          // (only with ops, as the tile calls)
  const m3tsz_encoder_state *out_state;  // [n_types * n]: the output rows' encoders (their room)
  uint64_t out_slot_words;
  int64_t *row_ts;
  double *row_val;
  uint32_t *row_n;
  uint64_t rows_stride;
  // the slots as tile_value_of reads them (tile_sum .. tile_count, tile_sum_sq, metric_type)
  EncodeParams tiles;
  // the annotated calls (ann_len set): each slot's annotation, its length in ann_len [n_slots][n] and slot r of
  // element s's bytes at (r * n + s) * ann_cap
  uint32_t *ann_len;
  uint8_t *ann_slot;
  uint64_t ann_cap;
  // add: the call's sparse annotation list (optional; dp_index counts rows of the element's column)
  const uint64_t *ann_series_off;
  const m3tsz_annotation_entry *ann_entries;
  const uint8_t *ann_bytes;
  // consume: the staged rows' annotations for the append, row i's entries from row_ann_off[i] = i * rows_stride
  uint64_t *row_ann_off;
  m3tsz_annotation_entry *row_ann;

  // The annotated lanes' slot helpers (the Gauge / Counter lanes and the Timer lanes share them).
  // add: a window annotation to slot o, the a_len bytes at ann_bytes + a_off (the add's inputs) as whole 8-byte words,
  // the last one zero-padded (a_len <= ann_cap, a multiple of 8)
  __device__ __forceinline__ void store_ann(uint64_t o, uint64_t a_off, uint32_t a_len) const {
    ann_len[o] = a_len;
    uint64_t *dst = reinterpret_cast<uint64_t *>(ann_slot + o * ann_cap);
    const uint8_t *src = ann_bytes + a_off;
    for (uint32_t w = 0; w < (a_len + 7u) / 8u; w++) {
      uint64_t x = 0;
      for (uint32_t b = 0; b < 8u && w * 8u + b < a_len; b++) x |= (uint64_t)src[w * 8u + b] << (8u * b);
      dst[w] = x;
    }
  }
  // consume / forward: slot o's annotation length (one above the capacity, which the library never stores, reads as
  // none)
  __device__ __forceinline__ uint32_t slot_ann_len(uint64_t o) const {
    const uint32_t l = ann_len[o];
    return l <= ann_cap ? l : 0u;
  }
  // consume: element s's k rows' entry lists, row i's at row_ann_off[i] = i * rows_stride (the last element also
  // writes the end)
  __device__ __forceinline__ void stage_ann_offsets(uint64_t s, uint32_t k) const {
    for (uint32_t j = 0; j < k; j++) row_ann_off[(uint64_t)j * n + s] = ((uint64_t)j * n + s) * rows_stride;
    if (s + 1 == n) row_ann_off[(uint64_t)k * n] = (uint64_t)k * n * rows_stride;
  }
  // consume: the entry of staged datapoint d of row `row`, slot o's a_len bytes (length 0, which the append takes as
  // none, without an annotation); an entry past a row's count is never read
  __device__ __forceinline__ void stage_ann(uint64_t row, uint64_t d, uint64_t o, uint32_t a_len) const {
    m3tsz_annotation_entry en;
    en.dp_index = (uint32_t)d;
    en.length = a_len;
    en.byte_offset = o * ann_cap;
    row_ann[row * rows_stride + d] = en;
  }
};
// (the annotated kernels when p.ann_len is set)
cudaError_t launch_element_add(const ElementParams &p, cudaStream_t stream);
cudaError_t launch_element_consume(const ElementParams &p, cudaStream_t stream);
// an element consumed with status OK takes the first failing status of its n_types rows
cudaError_t launch_element_status(const int32_t *row_status, uint64_t n, uint32_t n_types, int32_t *status,
                                  cudaStream_t stream);

// Timer element sets (m3tsz_element_set_*_timer; m3tsz_encode.cu): the set's slots and rows in `e` (its types and
// n_types unused; e.ops / e.discard_nan as in the other sets), each slot's CM stream in the m3tsz_element_timer_streams
// arrays (slot o = r * n + s, its entry i at (r * cap + i) * n + s), and the element's types and quantile list here
#define M3TSZ_MAX_TIMER_TYPES 23
#define M3TSZ_MAX_TIMER_QUANTILES 15
struct ElementTimerParams {
  ElementParams e;
  m3tsz_timer_stream_header *hdr;
  double *value;
  int64_t *num_ranks, *delta;
  int32_t *prev, *next;
  double *heap_a, *heap_b;
  uint32_t cap;
  int32_t every;  // insertAndCompressEvery
  double eps;
  const int8_t *batch;  // add: optional [points_stride][n], nonzero continues the previous row's batch
  uint32_t n_types, n_q;
  int32_t type[M3TSZ_MAX_TIMER_TYPES];
  double q[M3TSZ_MAX_TIMER_QUANTILES];  // Types.PooledQuantiles of type[]
};
// (the annotated kernels when p.e.ann_len is set, as for the other sets)
cudaError_t launch_element_timer_add(const ElementTimerParams &p, cudaStream_t stream);
cudaError_t launch_element_timer_consume(const ElementTimerParams &p, cudaStream_t stream);

// element sets through a rollup (m3tsz_element_set_forward; m3tsz_encode.cu): the source set's forward (one lane per
// source), the fold into the group set's windows (one warp per group) and the sources' commit (one lane per source)
struct ElementRollupParams {
  ElementParams src;  // the source set: its slots, records and watermarks, target, ops and its one type (types)
  int discard_nan;    // the source side drops a NaN forwarded value with or without ops
  // the forward's output: the q-th due window of source s (start order) at q * src.n + s, window-major
  // [src.n_slots][src.n]; per source the number of due windows, which of them forward a value (bit q), which slots
  // they are in (bit r) and the new record
  int64_t *fwd_start;
  double *fwd_val;
  uint32_t *fwd_n;
  uint64_t *fwd_present, *fwd_due;
  m3tsz_transform_state *rec;
  // the groups: group g is the sources members[group_off[g] .. group_off[g + 1])
  const uint64_t *group_off;
  const uint32_t *members;
  uint64_t n_members, n_groups;
  // the group set's slots, window-slot major [g_slots][n_groups], and watermarks
  uint32_t g_slots;
  int64_t *g_start, *g_count;
  void *g_sum, *g_min, *g_max, *g_sum_sq;
  double *g_last;
  int64_t *g_last_at;
  const int64_t *g_watermark;
  int32_t *group_status;
  // the commit: mark[s] is the largest status of a failed group listing s (0: none)
  int32_t *mark;
  int32_t *src_status;
  // the annotated forward (src.ann_len set; src.ann_len / ann_slot / ann_cap are the source slots' annotations): per
  // source, bit q of fwd_ann_present says the q-th due window is forwarded and carries an annotation, and for those
  // windows only fwd_ann[q * src.n + s] refers to it as (its slot r * src.n + s) << 17 | its length (1 .. 65536);
  // the group slots' annotations, laid out as the source slots'
  uint64_t *fwd_ann_present;
  uint64_t *fwd_ann;
  uint32_t *g_ann_len;
  uint8_t *g_ann_slot;
  uint64_t g_ann_cap;

  // The annotated forward's and fold's helpers (the Gauge / Counter lanes and the Timer lanes share them).
  // forward, after its windows' loop: source s's forwarded windows (bit q of `present`, due slots the bits of `due`)
  // whose slot holds an annotation (a length of 1 .. src.ann_cap; above the capacity reads as none, as the annotated
  // consume reads it) set bit q of fwd_ann_present and write their reference to fwd_ann; the slot's bytes stay where
  // they are for the fold to copy
  __device__ __forceinline__ void forward_ann(uint64_t s, uint64_t due, uint64_t present) const {
    const ElementParams &e = src;
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
      fwd_ann[(uint64_t)q * e.n + s] = (o << 17) | l;
    }
    fwd_ann_present[s] = ann;
  }
  // fold: a group window's annotation to group slot o.  ref is the forward's reference to a source slot (0: none),
  // whose bytes go over as whole 8-byte words (the annotated add zero-pads a slot's last word), lane `lane` of n_lanes
  // copying words lane, lane + n_lanes, ...; every lane writes the length
  __device__ __forceinline__ void store_group_ann(uint64_t o, uint64_t ref, uint32_t lane, uint32_t n_lanes) const {
    const uint32_t len = (uint32_t)(ref & 0x1ffffu);
    g_ann_len[o] = len;
    const uint64_t *from = reinterpret_cast<const uint64_t *>(src.ann_slot + (ref >> 17) * src.ann_cap);
    uint64_t *dst = reinterpret_cast<uint64_t *>(g_ann_slot + o * g_ann_cap);
    for (uint32_t w = lane; w < (len + 7u) / 8u; w += n_lanes) dst[w] = from[w];
  }
  // AddUnique's and the Timer fold's slot search: group g's slot holding window ws (hit), else its first free slot
  // (fr), -1 for none; slot `skip` (the one a lane holds in registers, -1: none) is passed over
  __device__ __forceinline__ void group_slot(uint64_t g, int skip, int64_t ws, int &hit, int &fr) const {
    hit = fr = -1;
    for (uint32_t s = 0; s < g_slots; s++) {
      if ((int)s == skip) continue;
      const uint64_t o = (uint64_t)s * n_groups + g;
      if (g_count[o] == 0) {
        if (fr < 0) fr = (int)s;
      } else if (g_start[o] == ws) {
        hit = (int)s;
        break;
      }
    }
  }
};
// (the annotated kernels when p.src.ann_len is set)
cudaError_t launch_element_forward(const ElementRollupParams &p, cudaStream_t stream);
// (p.mark must be zero)
cudaError_t launch_element_fold(const ElementRollupParams &p, cudaStream_t stream);
cudaError_t launch_element_commit(const ElementRollupParams &p, cudaStream_t stream);
// element-set rollups across shards (m3tsz_element_set_forward_write / _add_forwarded; m3tsz_encode.cu).
// forward_write: p.fwd_* from launch_element_forward; the count pass writes each group's record and value counts (and
// INVALID_ARG / OK to group_status), the caller scans them into rec_off / val_off, and the write pass writes the groups
// that fit, the statuses, the commit marks and `counts`.  add_forwarded: the records' element keys (key, or n for an
// invalid key) and indices for the caller's radix sort, then one lane per element over the sorted indices.
struct ElementForwardedParams {
  ElementRollupParams rp;  // forward_write: the forward's; add_forwarded: the group set as rp.g_* / rp.n_groups
  const uint64_t *group_key;
  uint32_t source_id;
  m3tsz_forwarded_metric *out_rec;
  double *out_val;
  uint64_t rec_cap, val_cap;
  uint64_t *n_rec, *n_val, *rec_off, *val_off;
  uint64_t *counts;
  // add_forwarded
  const m3tsz_forwarded_metric *rec;
  const double *val;
  uint64_t n_recs, n_vals;
  uint64_t *sort_key, *sort_idx;          // prep: key / index in record order
  const uint64_t *sorted_key, *sorted_idx;  // the lanes: after the sort
  uint32_t *bits;
  uint32_t bit_words;  // capacity / 32
  int64_t trunc_off;
  int8_t *result;
  int32_t *status;
};
cudaError_t launch_forward_write_count(const ElementForwardedParams &p, cudaStream_t stream);
cudaError_t launch_forward_write(const ElementForwardedParams &p, cudaStream_t stream);
cudaError_t launch_add_forwarded_prep(const ElementForwardedParams &p, cudaStream_t stream);
cudaError_t launch_add_forwarded(const ElementForwardedParams &p, cudaStream_t stream);
// cub scratch sizes and calls for the two passes (tmp NULL: *bytes gets the size)
cudaError_t forward_write_scan(void *tmp, size_t &bytes, const uint64_t *in, uint64_t *out, uint64_t n,
                               cudaStream_t stream);
cudaError_t add_forwarded_sort(void *tmp, size_t &bytes, const uint64_t *key_in, uint64_t *key_out,
                               const uint64_t *idx_in, uint64_t *idx_out, uint64_t n, int end_bit,
                               cudaStream_t stream);

// Timer sets through a rollup (m3tsz_element_set_forward_timer): p as above (its g_min / g_max / g_last unused), with
// the source set's streams and one type in `src` and the group set's streams and quantile list in `groups`; the commit
// is launch_element_commit's.  (p.mark must be zero for the fold.)  The annotated kernels when p.src.ann_len is set, with
// the annotated forward's fields of p.
cudaError_t launch_element_timer_forward(const ElementRollupParams &p, const ElementTimerParams &src,
                                         cudaStream_t stream);
cudaError_t launch_element_timer_fold(const ElementRollupParams &p, const ElementTimerParams &groups,
                                      cudaStream_t stream);
// Timer sets across shards (m3tsz_element_set_forward_write_timer / _add_forwarded_timer): the writer runs
// launch_element_timer_forward in place of launch_element_forward; the add runs the prep kernel and the sort as
// add_forwarded does, then one lane per element with `groups` the group set's streams and quantile list.
cudaError_t launch_add_forwarded_timer(const ElementForwardedParams &p, const ElementTimerParams &groups,
                                       cudaStream_t stream);

// exclusive scan of aligned lengths + gather into a packed buffer
cudaError_t launch_compact(const uint8_t *slots, uint64_t slot_stride, const uint64_t *len,
                           uint64_t n_series, uint32_t align, uint8_t *packed,
                           uint64_t packed_capacity, uint64_t *offsets, void *scan_tmp,
                           size_t scan_tmp_bytes, int32_t *overflow_flag, cudaStream_t stream);
size_t compact_scan_tmp_bytes(uint64_t n_series);

}  // namespace m3tsz
