// m3tsz_capi.cu -- the C ABI declared in include/m3tsz_b200.h.
//
// Thin host layer: argument validation, launch bookkeeping, and the *_host
// variants (H2D copy -> kernel -> D2H copy through context-owned scratch).
// There is deliberately no CPU codec in this library: without a CUDA device
// m3tsz_ctx_create fails with M3TSZ_ERR_NO_DEVICE.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>

#include "m3tsz_common.cuh"
#include "m3tsz_kernels.h"

#include "m3tsz_ctx.h"

using namespace m3tsz;

using namespace m3tsz::host;

static bool valid_align(uint32_t align) {
  return align == 1 || align == 4 || align == 8 || align == 16 || align == 32 || align == 64;
}

// The stream addressing both decode entry points check, and the DecodeParams fields they share.
static bool decode_params(const m3tsz_options *opts, const uint8_t *d_streams, uint64_t streams_bytes,
                          const uint64_t *d_offsets, const uint64_t *d_lengths, uint64_t n_series,
                          uint32_t *d_n_points, int32_t *d_status, DecodeParams &p) {
  if (!d_streams || !d_offsets || ((uintptr_t)d_streams & 15u) ||
      streams_bytes >= (1ull << 34))  // 32-bit word / byte offsets inside the kernel; split larger batches
    return false;
  memset(&p, 0, sizeof(p));
  p.streams = d_streams;
  p.streams_bytes = streams_bytes;
  p.offsets = d_offsets;
  p.lengths = d_lengths;
  p.n_series = n_series;
  p.default_unit = opts->default_time_unit;
  p.n_points = d_n_points;
  p.status = d_status;
  return true;
}

// The inputs the encode entry points check (pointers, alignments, the annotation triple, and
// point-major input, which takes no units or annotations), and the EncodeParams fields they share.
// The batch encoders need d_start and d_out_len; an encoder-set append takes both from its states.
static bool encode_params(const m3tsz_options *opts, const int64_t *d_ts, const double *d_val, uint64_t n_series,
                          uint64_t points_stride, const uint32_t *d_n_points, const int64_t *d_start, int32_t unit,
                          const uint8_t *d_units, const uint64_t *d_ann_series_off,
                          const m3tsz_annotation_entry *d_ann_entries, const uint8_t *d_ann_bytes,
                          uint64_t *d_out_len, int32_t *d_status, const m3tsz_encode_extras *extras,
                          EncodeParams &p, bool append = false) {
  if (!d_ts || !d_val || (!append && (!d_start || !d_out_len)) || points_stride > 0xffffffffull ||
      ((uintptr_t)d_ts & 7u) || ((uintptr_t)d_val & 7u))
    return false;
  if (d_ann_series_off && (!d_ann_entries || !d_ann_bytes)) return false;
  const bool point_major = extras && extras->point_major_input;
  if (point_major && (d_units || d_ann_series_off)) return false;
  memset(&p, 0, sizeof(p));
  p.ts = d_ts;
  p.val = d_val;
  p.n_series = n_series;
  p.points_stride = points_stride;
  p.n_points = d_n_points;
  p.start = d_start;
  p.unit = unit;
  p.units = d_units;
  p.ann_series_off = d_ann_series_off;
  p.ann_entries = d_ann_entries;
  p.ann_bytes = d_ann_bytes;
  p.default_unit = opts->default_time_unit;
  p.out_len = d_out_len;
  p.status = d_status;
  if (extras) {
    p.last_value = extras->d_last_value;
    p.out_bits = extras->d_out_bits;
  }
  p.in_mode = point_major ? 1 : 0;
  return true;
}

// Packed mode: the kernel encodes into a set of context slots of slot_bytes each and appends
// every finished stream at an `align`ed cursor (*d_total_bytes, zeroed by the caller) in d_packed.
static int packed_params(m3tsz_ctx *ctx, const ScratchFence &fence, uint64_t n_series, uint64_t slot_bytes,
                         uint32_t align,
                         uint8_t *d_packed, uint64_t packed_capacity, uint64_t *d_offsets,
                         uint64_t *d_total_bytes, cudaStream_t st, EncodeParams &p) {
  const uint64_t slots = encode_packed_scratch_slots(n_series);
  if (slots == 0) return set_cuda_error(ctx, cudaGetLastError(), "encode_packed_scratch_slots");
  void *scratch = nullptr, *ctr = nullptr;
  int rc;
  if ((rc = ensure(ctx, fence, kSlotPackedSlots, slots * slot_bytes, &scratch))) return rc;
  if ((rc = ensure(ctx, fence, kSlotBatchCounter, 64, &ctr))) return rc;
  CK(cudaMemsetAsync(ctr, 0, 64, st));
  p.out = (uint8_t *)scratch;
  p.out_stride = slot_bytes;
  p.packed = d_packed;
  p.packed_capacity = packed_capacity;
  p.packed_off = d_offsets;
  p.packed_cursor = reinterpret_cast<unsigned long long *>(d_total_bytes);
  p.batch_counter = reinterpret_cast<unsigned long long *>(ctr);
  p.align = align;
  return M3TSZ_OK;
}

extern "C" {

int m3tsz_version(void) { return M3TSZ_B200_VERSION; }

const char *m3tsz_status_string(int st) {
  switch (st) {
    case M3TSZ_OK: return "ok";
    case M3TSZ_ERR_EOF: return "EOF";
    case M3TSZ_ERR_ENCODER_CLOSED: return "encoder is closed";
    case M3TSZ_ERR_NO_DATAPOINTS: return "encoder has no encoded datapoints";
    case M3TSZ_ERR_DOD_OVERFLOW: return "deltaOfDelta value overflows 32 bits";
    case M3TSZ_ERR_NO_TIME_SCHEME: return "time encoding scheme doesn't exist for unit";
    case M3TSZ_ERR_UNRECOGNIZED_UNIT: return "unrecognized time unit";
    case M3TSZ_ERR_INVALID_MULT: return "supplied multiplier is invalid";
    case M3TSZ_ERR_ANNOTATION_LEN: return "expected annotation length to be >= 0";
    case M3TSZ_ERR_ANNOTATION_SHORT: return "expected to read annotation bytes, but got end of stream";
    case M3TSZ_ERR_ITER_CLOSED: return "iterator is closed";
    case M3TSZ_ERR_VARINT_OVERFLOW: return "binary: varint overflows a 64-bit integer";
    case M3TSZ_ERR_UNEXPECTED_EOF: return "unexpected EOF";
    case M3TSZ_ERR_OUT_OF_ORDER: return "values are out of order from inner iterator";
    case M3TSZ_ERR_TOO_MANY_ITERATORS: return "too many replicas / readers for one series";
    case M3TSZ_ERR_TOO_MANY_ENCODERS: return "too many encoders per block";
    case M3TSZ_ERR_AGGREGATION_CLOSED: return "aggregation is closed";
    case M3TSZ_ERR_DUPLICATE_SOURCE: return "duplicate forwarding source";
    case M3TSZ_ERR_CHECKSUM_MISMATCH: return "checksum does not match expected checksum";
    case M3TSZ_ERR_CAPACITY: return "output capacity exceeded";
    case M3TSZ_ERR_INVALID_ARG: return "invalid argument";
    case M3TSZ_ERR_CUDA: return "CUDA error";
    case M3TSZ_ERR_NO_DEVICE: return "no CUDA device (this library has no CPU fallback)";
    case M3TSZ_ERR_STREAM_TOO_LARGE: return "stream too large";
    default: return "unknown status";
  }
}

int m3tsz_ctx_create(int device, m3tsz_ctx **out) {
  if (!out) return M3TSZ_ERR_INVALID_ARG;
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0) {
    (void)cudaGetLastError();
    return M3TSZ_ERR_NO_DEVICE;
  }
  if (device < 0 || device >= n) return M3TSZ_ERR_INVALID_ARG;
  m3tsz_ctx *ctx = new (std::nothrow) m3tsz_ctx();
  if (!ctx) return M3TSZ_ERR_INVALID_ARG;
  ctx->device = device;
  if (cudaSetDevice(device) != cudaSuccess ||
      cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithFlags(&ctx->stream2, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreateWithFlags(&ctx->ev, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&ctx->scratch_ev, cudaEventDisableTiming) != cudaSuccess ||
      cudaMalloc(&ctx->d_flag, 2 * sizeof(int32_t)) != cudaSuccess) {
    (void)cudaGetLastError();
    delete ctx;
    return M3TSZ_ERR_CUDA;
  }
  *out = ctx;
  return M3TSZ_OK;
}

void m3tsz_ctx_destroy(m3tsz_ctx *ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  for (auto &sc : ctx->s)
    if (sc.ptr) cudaFree(sc.ptr);
  if (ctx->d_flag) cudaFree(ctx->d_flag);
  for (int i = 0; i < 2; i++)
    if (ctx->h_stage[i]) cudaFreeHost(ctx->h_stage[i]);
  if (ctx->ev) cudaEventDestroy(ctx->ev);
  if (ctx->scratch_ev) cudaEventDestroy(ctx->scratch_ev);
  if (ctx->stream2) cudaStreamDestroy(ctx->stream2);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}

const char *m3tsz_last_cuda_error(const m3tsz_ctx *ctx) { return ctx ? ctx->last_error : ""; }
uint64_t m3tsz_ctx_launch_count(const m3tsz_ctx *ctx) { return ctx ? ctx->launches : 0; }

uint64_t m3tsz_encode_bound_units(uint64_t n, int per_datapoint_units) {
  // 64-bit start + per datapoint <= 68 (timestamp: '1111' + 64-bit delta-of-delta) + 80 (value:
  // 3 control bits + 13-bit int header + 64 bits) bits + 11-bit end-of-stream marker, plus the
  // write-ahead guard the kernel keeps.  With per-datapoint units a datapoint may also carry a
  // time-unit marker (11 + 8 bits) and then a raw 64-bit delta-of-delta: 83 bits of timestamp.
  const uint64_t per_dp = per_datapoint_units ? (83 + 80) : (68 + 80);
  uint64_t bits = 64 + n * per_dp + 11;
  uint64_t bytes = (bits + 7) / 8 + 64;
  return (bytes + 15) & ~15ull;
}
uint64_t m3tsz_encode_bound(uint64_t n) { return m3tsz_encode_bound_units(n, 0); }

// --------------------------------------------------------------------------
int m3tsz_decode_batch_ex(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams,
                          uint64_t streams_bytes, const uint64_t *d_offsets, uint64_t n_series,
                          int64_t *d_ts, double *d_val, uint64_t max_points, uint32_t *d_n_points,
                          int32_t *d_status, uint8_t *d_unit, m3tsz_annotation_ref *d_ann,
                          const m3tsz_decode_extras *ex, void *stream) {
  if (!ctx || !valid_opts(opts)) return M3TSZ_ERR_INVALID_ARG;
  if (n_series == 0) return M3TSZ_OK;
  DecodeParams p;
  if (!decode_params(opts, d_streams, streams_bytes, d_offsets, ex ? ex->d_lengths : nullptr, n_series,
                     d_n_points, d_status, p) ||
      !d_ts || !d_val || max_points == 0 || max_points >= (1ull << 27))
    return M3TSZ_ERR_INVALID_ARG;
  if (ex && ex->d_events && (!ex->d_event_count || ex->events_capacity == 0)) return M3TSZ_ERR_INVALID_ARG;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  p.ts = d_ts;
  p.val = d_val;
  p.cap = max_points;
  p.unit_out = d_unit;
  p.ann_out = d_ann;
  if (ex) {
    p.unit_first_out = ex->d_unit_first;
    if (ex->d_events) {
      p.events = ex->d_events;
      p.events_capacity = ex->events_capacity;
      p.event_count = reinterpret_cast<unsigned long long *>(ex->d_event_count);
    }
  }
  CK(launch_decode(p, opts->int_optimized != 0, (ex && ex->point_major) ? 3 : 0, (cudaStream_t)stream));
  ctx->launches++;
  return M3TSZ_OK;
}

int m3tsz_decode_batch(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams,
                       uint64_t streams_bytes, const uint64_t *d_offsets, uint64_t n_series,
                       int64_t *d_ts, double *d_val, uint64_t max_points, uint32_t *d_n_points,
                       int32_t *d_status, uint8_t *d_unit, m3tsz_annotation_ref *d_ann,
                       void *stream) {
  return m3tsz_decode_batch_ex(ctx, opts, d_streams, streams_bytes, d_offsets, n_series, d_ts, d_val,
                               max_points, d_n_points, d_status, d_unit, d_ann, nullptr, stream);
}

// The window range of every downsample and tile call: 1 .. 2^31 - 1 windows of step > 0 ns, and
// start + n_windows * step inside int64
static bool valid_windows(int64_t start_ns, int64_t step_ns, uint32_t n_windows) {
  return step_ns > 0 && n_windows != 0 && n_windows <= 0x7fffffffu &&
         (__int128)start_ns + (__int128)n_windows * (__int128)step_ns <= (__int128)INT64_MAX;
}

static int downsample_impl(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams,
                           uint64_t streams_bytes, const uint64_t *d_offsets, const uint64_t *d_lengths,
                           uint64_t n_series,
                           int64_t range_start_ns, int64_t window_ns, uint32_t n_windows, double *d_sum,
                           int64_t *d_count, double *d_min, double *d_max, double *d_last,
                           int64_t *d_last_at, bool want_last, uint32_t *d_n_points, int32_t *d_status,
                           void *stream) {
  if (!ctx || !valid_opts(opts)) return M3TSZ_ERR_INVALID_ARG;
  if (n_series == 0) return M3TSZ_OK;
  DecodeParams p;
  if (!decode_params(opts, d_streams, streams_bytes, d_offsets, d_lengths, n_series, d_n_points, d_status, p) ||
      !d_sum || !d_count || !d_min || !d_max || !valid_windows(range_start_ns, window_ns, n_windows) ||
      (want_last && !d_last))
    return M3TSZ_ERR_INVALID_ARG;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  ScratchFence fence(ctx, (cudaStream_t)stream, want_last && !d_last_at);
  if (want_last && !d_last_at) {  // lastAt lives in context scratch
    void *sc = nullptr;
    int rc = ensure(ctx, fence, kSlotWinLastAt, (size_t)n_series * n_windows * 8, &sc);
    if (rc) return rc;
    d_last_at = (int64_t *)sc;
  }
  p.range_start = range_start_ns;
  p.window = window_ns;
  p.n_windows = n_windows;
  p.ds_sum = d_sum;
  p.ds_count = d_count;
  p.ds_min = d_min;
  p.ds_max = d_max;
  p.ds_last = d_last;
  p.ds_last_at = d_last_at;
  CK(launch_decode(p, opts->int_optimized != 0, want_last ? 2 : 1, (cudaStream_t)stream));
  ctx->launches++;
  return M3TSZ_OK;
}

// A Gauge without sumSq is downsample_impl (modes 1 / 2); a Gauge with sumSq is mode 4, a Counter mode 5.
int m3tsz_decode_downsample_ex(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams,
                               uint64_t streams_bytes, const uint64_t *d_offsets, const uint64_t *d_lengths,
                               uint64_t n_series, int64_t range_start_ns, int64_t window_ns, uint32_t n_windows,
                               const m3tsz_downsample_outputs *o, void *stream) {
  if (!ctx || !valid_opts(opts) || !o || o->reserved != 0) return M3TSZ_ERR_INVALID_ARG;
  const bool gauge = o->metric_type == M3TSZ_METRIC_GAUGE, counter = o->metric_type == M3TSZ_METRIC_COUNTER;
  if (gauge) {
    if (o->d_counter_sum || o->d_counter_min || o->d_counter_max || o->d_counter_sum_sq ||
        (o->d_last_at && !o->d_last && !o->d_sum_sq))
      return M3TSZ_ERR_INVALID_ARG;
    if (!o->d_sum_sq)
      return downsample_impl(ctx, opts, d_streams, streams_bytes, d_offsets, d_lengths, n_series, range_start_ns,
                             window_ns, n_windows, o->d_sum, o->d_count, o->d_min, o->d_max, o->d_last,
                             o->d_last_at, o->d_last != nullptr, o->d_n_points, o->d_status, stream);
  } else if (counter) {
    if (o->d_sum || o->d_min || o->d_max || o->d_sum_sq || o->d_last || o->d_last_at) return M3TSZ_ERR_INVALID_ARG;
  } else {
    return M3TSZ_ERR_INVALID_ARG;
  }
  if (n_series == 0) return M3TSZ_OK;
  DecodeParams p;
  if (!decode_params(opts, d_streams, streams_bytes, d_offsets, d_lengths, n_series, o->d_n_points, o->d_status,
                     p) ||
      !o->d_count || !valid_windows(range_start_ns, window_ns, n_windows) ||
      (gauge && (!o->d_sum || !o->d_min || !o->d_max)) ||
      (counter && (!o->d_counter_sum || !o->d_counter_min || !o->d_counter_max)))
    return M3TSZ_ERR_INVALID_ARG;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  ScratchFence fence(ctx, (cudaStream_t)stream,
                     gauge ? (!o->d_last || !o->d_last_at) : !o->d_counter_sum_sq);
  // what the caller leaves out but the kernel keeps (to re-open a committed window exactly) lives in scratch
  const size_t wb = (size_t)n_series * n_windows * 8;
  void *sc = nullptr;
  int rc;
  p.range_start = range_start_ns;
  p.window = window_ns;
  p.n_windows = n_windows;
  p.ds_count = o->d_count;
  if (gauge) {
    p.ds_sum = o->d_sum;
    p.ds_min = o->d_min;
    p.ds_max = o->d_max;
    p.ds_sum_sq = o->d_sum_sq;
    p.ds_last = o->d_last;
    p.ds_last_at = o->d_last_at;
    if (!p.ds_last) {
      if ((rc = ensure(ctx, fence, kSlotWinLast, wb, &sc))) return rc;
      p.ds_last = (double *)sc;
    }
    if (!p.ds_last_at) {
      if ((rc = ensure(ctx, fence, kSlotWinLastAt, wb, &sc))) return rc;
      p.ds_last_at = (int64_t *)sc;
    }
  } else {
    p.ds_isum = o->d_counter_sum;
    p.ds_imin = o->d_counter_min;
    p.ds_imax = o->d_counter_max;
    p.ds_isum_sq = o->d_counter_sum_sq;
    if (!p.ds_isum_sq) {
      if ((rc = ensure(ctx, fence, kSlotWinSumSq, wb, &sc))) return rc;
      p.ds_isum_sq = (int64_t *)sc;
    }
  }
  CK(launch_decode(p, opts->int_optimized != 0, gauge ? 4 : 5, (cudaStream_t)stream));
  ctx->launches++;
  return M3TSZ_OK;
}

int m3tsz_decode_downsample_batch(m3tsz_ctx *ctx, const m3tsz_options *opts,
                                  const uint8_t *d_streams, uint64_t streams_bytes,
                                  const uint64_t *d_offsets, uint64_t n_series,
                                  int64_t range_start_ns, int64_t window_ns, uint32_t n_windows,
                                  double *d_sum, int64_t *d_count, double *d_min, double *d_max,
                                  uint32_t *d_n_points, int32_t *d_status, void *stream) {
  return downsample_impl(ctx, opts, d_streams, streams_bytes, d_offsets, nullptr, n_series, range_start_ns,
                         window_ns, n_windows, d_sum, d_count, d_min, d_max, nullptr, nullptr, false,
                         d_n_points, d_status, stream);
}

int m3tsz_decode_downsample_last_batch(m3tsz_ctx *ctx, const m3tsz_options *opts,
                                       const uint8_t *d_streams, uint64_t streams_bytes,
                                       const uint64_t *d_offsets, uint64_t n_series,
                                       int64_t range_start_ns, int64_t window_ns, uint32_t n_windows,
                                       double *d_sum, int64_t *d_count, double *d_min, double *d_max,
                                       double *d_last, int64_t *d_last_at, uint32_t *d_n_points,
                                       int32_t *d_status, void *stream) {
  return downsample_impl(ctx, opts, d_streams, streams_bytes, d_offsets, nullptr, n_series, range_start_ns,
                         window_ns, n_windows, d_sum, d_count, d_min, d_max, d_last, d_last_at, true,
                         d_n_points, d_status, stream);
}

int m3tsz_encode_batch_ex(m3tsz_ctx *ctx, const m3tsz_options *opts, const int64_t *d_ts,
                          const double *d_val, uint64_t n_series, uint64_t points_stride,
                          const uint32_t *d_n_points, const int64_t *d_start, int32_t unit,
                          const uint8_t *d_units, const uint64_t *d_ann_series_off,
                          const m3tsz_annotation_entry *d_ann_entries, const uint8_t *d_ann_bytes,
                          uint8_t *d_out, uint64_t out_stride, uint64_t *d_out_len, int32_t *d_status,
                          const m3tsz_encode_extras *extras, void *stream) {
  if (!ctx || !valid_opts(opts)) return M3TSZ_ERR_INVALID_ARG;
  if (n_series == 0) return M3TSZ_OK;
  EncodeParams p;
  if (!encode_params(opts, d_ts, d_val, n_series, points_stride, d_n_points, d_start, unit, d_units,
                     d_ann_series_off, d_ann_entries, d_ann_bytes, d_out_len, d_status, extras, p) ||
      !d_out || (out_stride & 15u) || out_stride == 0 || out_stride > (1ull << 33) || ((uintptr_t)d_out & 15u))
    return M3TSZ_ERR_INVALID_ARG;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  p.out = d_out;
  p.out_stride = out_stride;
  CK(launch_encode(p, opts->int_optimized != 0, (cudaStream_t)stream));
  ctx->launches++;
  return M3TSZ_OK;
}

int m3tsz_encode_batch(m3tsz_ctx *ctx, const m3tsz_options *opts, const int64_t *d_ts,
                       const double *d_val, uint64_t n_series, uint64_t points_stride,
                       const uint32_t *d_n_points, const int64_t *d_start, int32_t unit,
                       const uint8_t *d_units, const uint64_t *d_ann_series_off,
                       const m3tsz_annotation_entry *d_ann_entries, const uint8_t *d_ann_bytes,
                       uint8_t *d_out, uint64_t out_stride, uint64_t *d_out_len, int32_t *d_status,
                       void *stream) {
  return m3tsz_encode_batch_ex(ctx, opts, d_ts, d_val, n_series, points_stride, d_n_points, d_start, unit,
                               d_units, d_ann_series_off, d_ann_entries, d_ann_bytes, d_out, out_stride,
                               d_out_len, d_status, nullptr, stream);
}

int m3tsz_encoder_set_reset(m3tsz_ctx *ctx, const m3tsz_options *opts, m3tsz_encoder_state *d_state,
                            uint64_t n_series, const int64_t *d_start, void *stream) {
  if (!ctx || !valid_opts(opts)) return M3TSZ_ERR_INVALID_ARG;
  if (n_series == 0) return M3TSZ_OK;
  if (!d_state || !d_start || ((uintptr_t)d_state & 15u)) return M3TSZ_ERR_INVALID_ARG;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  CK(launch_encoder_set_reset(d_state, n_series, d_start, opts->default_time_unit, opts->int_optimized != 0,
                              (cudaStream_t)stream));
  ctx->launches++;
  return M3TSZ_OK;
}

int m3tsz_encoder_set_append(m3tsz_ctx *ctx, const m3tsz_options *opts, m3tsz_encoder_state *d_state,
                             uint64_t n_series, const int64_t *d_ts, const double *d_val, uint64_t points_stride,
                             const uint32_t *d_n_points, int32_t unit, const uint8_t *d_units,
                             const uint64_t *d_ann_series_off, const m3tsz_annotation_entry *d_ann_entries,
                             const uint8_t *d_ann_bytes, int32_t point_major_input, uint8_t *d_buf,
                             uint64_t buf_stride, uint32_t *d_n_appended, int32_t *d_status, void *stream) {
  if (!ctx || !valid_opts(opts)) return M3TSZ_ERR_INVALID_ARG;
  if (n_series == 0) return M3TSZ_OK;
  m3tsz_encode_extras ex;
  memset(&ex, 0, sizeof(ex));
  ex.point_major_input = point_major_input;
  EncodeParams p;
  if (!encode_params(opts, d_ts, d_val, n_series, points_stride, d_n_points, nullptr, unit, d_units,
                     d_ann_series_off, d_ann_entries, d_ann_bytes, nullptr, d_status, &ex, p, true) ||
      !d_state || ((uintptr_t)d_state & 15u) || !d_n_appended || !d_status || !d_buf || (buf_stride & 15u) ||
      buf_stride == 0 || buf_stride > (1ull << 33) || ((uintptr_t)d_buf & 15u))
    return M3TSZ_ERR_INVALID_ARG;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  p.out = d_buf;
  p.out_stride = buf_stride;
  p.state = d_state;
  p.n_appended = d_n_appended;
  CK(launch_encode_append(p, opts->int_optimized != 0, (cudaStream_t)stream));
  ctx->launches++;
  return M3TSZ_OK;
}

int m3tsz_encoder_set_stream(m3tsz_ctx *ctx, const m3tsz_encoder_state *d_state, uint64_t n_series,
                             uint8_t *d_buf, uint64_t buf_stride, uint64_t *d_len, void *stream) {
  if (!ctx) return M3TSZ_ERR_INVALID_ARG;
  if (n_series == 0) return M3TSZ_OK;
  if (!d_state || ((uintptr_t)d_state & 15u) || !d_buf || !d_len || (buf_stride & 15u) || buf_stride == 0 ||
      ((uintptr_t)d_buf & 15u))
    return M3TSZ_ERR_INVALID_ARG;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  CK(launch_encoder_set_stream(d_state, n_series, d_buf, buf_stride, d_len, (cudaStream_t)stream));
  ctx->launches++;
  return M3TSZ_OK;
}

int m3tsz_encoder_set_write(m3tsz_ctx *ctx, const m3tsz_options *opts, m3tsz_encoder_state *d_state, uint8_t *d_buf,
                            uint64_t buf_stride, uint64_t n_series, m3tsz_encoder_state *d_pool_state,
                            uint8_t *d_pool_buf, uint64_t pool_stride, uint64_t pool_capacity, uint32_t *d_pool_count,
                            int32_t *d_table, int32_t n_encoders, const int64_t *d_ts, const double *d_val,
                            uint64_t points_stride, const uint32_t *d_n_points, int32_t unit, const uint8_t *d_units,
                            const uint64_t *d_ann_series_off, const m3tsz_annotation_entry *d_ann_entries,
                            const uint8_t *d_ann_bytes, int32_t point_major_input, int8_t *d_result,
                            int32_t *d_status, void *stream) {
  if (!ctx || !valid_opts(opts) || n_encoders < 1 || n_encoders > M3TSZ_MAX_BUCKET_ENCODERS)
    return M3TSZ_ERR_INVALID_ARG;
  if (n_series == 0) return M3TSZ_OK;
  m3tsz_encode_extras ex;
  memset(&ex, 0, sizeof(ex));
  ex.point_major_input = point_major_input;
  EncodeParams p;
  auto bad_slots = [](const void *st, const uint8_t *buf, uint64_t stride) {
    return !st || ((uintptr_t)st & 15u) || !buf || ((uintptr_t)buf & 15u) || (stride & 15u) || stride == 0 ||
           stride > (1ull << 33);
  };
  if (!encode_params(opts, d_ts, d_val, n_series, points_stride, d_n_points, nullptr, unit, d_units,
                     d_ann_series_off, d_ann_entries, d_ann_bytes, nullptr, d_status, &ex, p, true) ||
      !d_result || !d_status || bad_slots(d_state, d_buf, buf_stride) || n_series >= (1ull << 31) ||
      points_stride == 0)
    return M3TSZ_ERR_INVALID_ARG;
  if (n_encoders > 1 && (bad_slots(d_pool_state, d_pool_buf, pool_stride) || !d_pool_count || !d_table ||
                         pool_capacity == 0 || pool_capacity >= (1ull << 31)))
    return M3TSZ_ERR_INVALID_ARG;
  if (n_encoders == 1) pool_capacity = 0;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  const cudaStream_t st = (cudaStream_t)stream;
  ScratchFence fence(ctx, st);
  void *target = nullptr, *touched = nullptr, *count = nullptr;
  int rc;
  if ((rc = ensure(ctx, fence, kSlotRouteTarget, n_series * points_stride, &target))) return rc;
  if ((rc = ensure(ctx, fence, kSlotRouteTouched, pool_capacity * sizeof(RouteTouched), &touched))) return rc;
  if ((rc = ensure(ctx, fence, kSlotRouteCount, sizeof(uint32_t), &count))) return rc;
  CK(cudaMemsetAsync(count, 0, sizeof(uint32_t), st));
  RouteParams r;
  memset(&r, 0, sizeof(r));
  r.state = d_state;
  r.n_series = n_series;
  r.slot_words = buf_stride >> 2;
  r.pool_state = d_pool_state;
  r.pool_capacity = pool_capacity;
  r.pool_slot_words = pool_stride >> 2;
  r.pool_count = d_pool_count;
  r.table = d_table;
  r.n_encoders = n_encoders;
  r.default_unit = opts->default_time_unit;
  r.ts = d_ts;
  r.val = d_val;
  r.points_stride = points_stride;
  r.n_points = d_n_points;
  r.unit = unit;
  r.point_major = point_major_input ? 1 : 0;
  r.units = d_units;
  r.ann_series_off = d_ann_series_off;
  r.ann_entries = d_ann_entries;
  r.ann_bytes = d_ann_bytes;
  r.target = (uint8_t *)target;
  r.result = d_result;
  r.status = d_status;
  r.touched = (RouteTouched *)touched;
  r.n_touched = (uint32_t *)count;
  const bool int_opt = opts->int_optimized != 0;
  CK(launch_route(r, int_opt, st));
  ctx->launches++;
  // encoder 0 of every bucket over the original inputs, then the overflow records the route gave datapoints
  p.route_target = (const uint8_t *)target;
  p.route_n_in = n_series;
  p.out = d_buf;
  p.out_stride = buf_stride;
  p.state = d_state;
  p.status = nullptr;
  CK(launch_encode_routed(p, int_opt, st));
  ctx->launches++;
  if (n_encoders > 1) {
    const uint64_t most = n_series * (uint64_t)(n_encoders - 1);
    p.n_series = most < pool_capacity ? most : pool_capacity;
    p.out = d_pool_buf;
    p.out_stride = pool_stride;
    p.state = d_pool_state;
    p.route_touched = (const RouteTouched *)touched;
    p.route_n_touched = (const uint32_t *)count;
    CK(launch_encode_routed(p, int_opt, st));
    ctx->launches++;
  }
  return M3TSZ_OK;
}

int m3tsz_encode_batch_packed(m3tsz_ctx *ctx, const m3tsz_options *opts, const int64_t *d_ts,
                              const double *d_val, uint64_t n_series, uint64_t points_stride,
                              const uint32_t *d_n_points, const int64_t *d_start, int32_t unit,
                              const uint8_t *d_units, const uint64_t *d_ann_series_off,
                              const m3tsz_annotation_entry *d_ann_entries, const uint8_t *d_ann_bytes,
                              uint64_t slot_bytes, uint32_t align, uint8_t *d_packed,
                              uint64_t packed_capacity, uint64_t *d_offsets, uint64_t *d_out_len,
                              int32_t *d_status, uint64_t *d_total_bytes, void *stream) {
  return m3tsz_encode_batch_packed_ex(ctx, opts, d_ts, d_val, n_series, points_stride, d_n_points, d_start, unit,
                                      d_units, d_ann_series_off, d_ann_entries, d_ann_bytes, slot_bytes, align,
                                      d_packed, packed_capacity, d_offsets, d_out_len, d_status, d_total_bytes,
                                      nullptr, stream);
}

int m3tsz_encode_batch_packed_ex(m3tsz_ctx *ctx, const m3tsz_options *opts, const int64_t *d_ts,
                                 const double *d_val, uint64_t n_series, uint64_t points_stride,
                                 const uint32_t *d_n_points, const int64_t *d_start, int32_t unit,
                                 const uint8_t *d_units, const uint64_t *d_ann_series_off,
                                 const m3tsz_annotation_entry *d_ann_entries, const uint8_t *d_ann_bytes,
                                 uint64_t slot_bytes, uint32_t align, uint8_t *d_packed,
                                 uint64_t packed_capacity, uint64_t *d_offsets, uint64_t *d_out_len,
                                 int32_t *d_status, uint64_t *d_total_bytes, const m3tsz_encode_extras *extras,
                                 void *stream) {
  if (!ctx || !valid_opts(opts) || !d_total_bytes || !valid_align(align)) return M3TSZ_ERR_INVALID_ARG;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  cudaStream_t st = (cudaStream_t)stream;
  ScratchFence fence(ctx, st);
  CK(cudaMemsetAsync(d_total_bytes, 0, sizeof(uint64_t), st));
  if (n_series == 0) return M3TSZ_OK;
  EncodeParams p;
  if (!encode_params(opts, d_ts, d_val, n_series, points_stride, d_n_points, d_start, unit, d_units,
                     d_ann_series_off, d_ann_entries, d_ann_bytes, d_out_len, d_status, extras, p) ||
      !d_packed || !d_offsets || ((uintptr_t)d_packed & 63u))
    return M3TSZ_ERR_INVALID_ARG;
  if (slot_bytes == 0) slot_bytes = m3tsz_encode_bound_units(points_stride, d_units != nullptr);
  slot_bytes = (slot_bytes + 15) & ~15ull;
  if (slot_bytes > (1ull << 33)) return M3TSZ_ERR_INVALID_ARG;
  int rc = packed_params(ctx, fence, n_series, slot_bytes, align, d_packed, packed_capacity, d_offsets, d_total_bytes,
                         st, p);
  if (rc) return rc;
  CK(launch_encode(p, opts->int_optimized != 0, st));
  ctx->launches++;
  return M3TSZ_OK;
}

int m3tsz_compact_streams(m3tsz_ctx *ctx, const uint8_t *d_slots, uint64_t slot_stride,
                          const uint64_t *d_len, uint64_t n_series, uint32_t align,
                          uint8_t *d_packed, uint64_t packed_capacity, uint64_t *d_offsets,
                          void *stream) {
  if (!ctx || !d_offsets || (n_series && (!d_slots || !d_len || !d_packed))) return M3TSZ_ERR_INVALID_ARG;
  if (!valid_align(align)) return M3TSZ_ERR_INVALID_ARG;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  cudaStream_t st = (cudaStream_t)stream;
  ScratchFence fence(ctx, st);  // (scratch, and d_flag)
  size_t tmp_bytes = compact_scan_tmp_bytes(n_series);
  void *tmp = nullptr;
  int rc = ensure(ctx, fence, kSlotCompactTmp, tmp_bytes, &tmp);
  if (rc) return rc;
  CK(cudaMemsetAsync(ctx->d_flag, 0, sizeof(int32_t), st));
  CK(launch_compact(d_slots, slot_stride, d_len, n_series, align, d_packed, packed_capacity,
                    d_offsets, tmp, tmp_bytes, ctx->d_flag, st));
  ctx->launches += 3;
  int32_t flag = 0;
  CK(cudaMemcpyAsync(&flag, ctx->d_flag, sizeof(flag), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return flag ? M3TSZ_ERR_CAPACITY : M3TSZ_OK;
}

int m3tsz_prom_convert_batch(m3tsz_ctx *ctx, const int64_t *d_ts, const double *d_val, uint64_t cap,
                             const uint32_t *d_n_points, uint64_t n_series, int64_t resolution_ns,
                             const uint8_t *d_handle_resets, double value_decrease_tolerance,
                             int64_t tolerance_until_ns, int64_t *d_ts_ms_out, double *d_val_out,
                             uint64_t out_cap, uint32_t *d_n_out, int32_t *d_status, void *stream) {
  if (!ctx) return M3TSZ_ERR_INVALID_ARG;
  if (n_series == 0) return M3TSZ_OK;
  if (!d_ts || !d_val || !d_n_points || !d_ts_ms_out || !d_val_out || !d_n_out || cap == 0 || out_cap == 0 ||
      resolution_ns < 0 || (d_handle_resets && resolution_ns == 0) ||
      value_decrease_tolerance != value_decrease_tolerance)
    return M3TSZ_ERR_INVALID_ARG;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  PromParams p;
  memset(&p, 0, sizeof(p));
  p.ts = d_ts;
  p.val = d_val;
  p.cap = cap;
  p.n_points = d_n_points;
  p.n_series = n_series;
  p.resolution = resolution_ns;
  p.handle_resets = d_handle_resets;
  p.tolerance = value_decrease_tolerance;
  p.tolerance_until = tolerance_until_ns;
  p.ts_out = d_ts_ms_out;
  p.val_out = d_val_out;
  p.out_cap = out_cap;
  p.n_out = d_n_out;
  p.status = d_status;
  CK(launch_prom(p, (cudaStream_t)stream));
  ctx->launches++;
  return M3TSZ_OK;
}

// The element a tile call writes, as the tile stages read it, and how its sources are addressed.  The
// transformations: op k in bits 4k .. 4k + 3 of one word, 0 ending the list (a non-empty list is never 0).
struct TileTransforms {
  const int32_t *types = nullptr;  // output row j * n_src + s is source s under types[j]
  uint32_t n_types = 0;
  // the multi-type stage (m3tsz_aggregate_tiles_types and the calls built on it) with its element records, whatever
  // n_types is; else the single-type stage of m3tsz_aggregate_tiles_ex / _transform
  bool multi = false;
  uint32_t ops = 0;
  bool reset = false;  // a Reset op: two rows per window
  // a NaN result writes nothing of its window.  The single-element calls discard only with a non-empty op list,
  // which keeps m3tsz_aggregate_tiles_ex's bytes; the rollup whatever its lists are (DESIGN.md §4.8).
  bool discard = false;
  m3tsz_transform_state *state = nullptr;     // the single-type stage's records
  m3tsz_element_state *elem_state = nullptr;  // the multi-type stage's records
  bool annotated = false;                     // (multi-type stage only) each window's annotation
  // over source blocks: offsets / lengths address n_segments segments, and series s is segments
  // [block_off[s], block_off[s + 1])
  const uint64_t *block_off = nullptr;
  uint64_t n_segments = 0;
};

// The packed outputs of a tile call (m3tsz_aggregate_tiles_batch's align .. d_total_bytes)
struct TileOutputs {
  uint32_t align;
  uint8_t *packed;
  uint64_t capacity;
  uint64_t *offsets, *len;
  int32_t *status;
  uint32_t *n_tiles;
  uint64_t *total_bytes;
};

static bool valid_packing(const TileOutputs &o) {
  return valid_align(o.align) && o.packed && o.offsets && o.len && !((uintptr_t)o.packed & 63u);
}

// Window-major aggregates ([n_windows][n_src] each) in context scratch: the fused decode's of the sources, or the
// rollup's of its groups, in the same representation.  sst: each source's status.
struct TileWindows {
  void *sum = nullptr, *cnt = nullptr, *min = nullptr, *max = nullptr, *last = nullptr, *lat = nullptr;
  void *sst = nullptr, *np = nullptr, *sq = nullptr, *ann = nullptr;
};

// the windows keep sumSq for SumSq / Stdev, and always for the Counter
static bool needs_sum_sq(bool counter, const int32_t *types, uint32_t n) {
  bool sq = counter;
  for (uint32_t j = 0; j < n; j++) sq |= types[j] == M3TSZ_AGG_SUMSQ || types[j] == M3TSZ_AGG_STDEV;
  return sq;
}

// Step 1 of every tile call: the fused decode + windows of the sources: the Gauge with `last` (mode 2), + sumSq if a
// type needs it (mode 4), or the Counter (mode 5, its int64 sum / min / max in the Gauge's slots); xf.annotated:
// + each window's annotation reference (modes 6-8).
static int tiles_decode(m3tsz_ctx *ctx, const ScratchFence &fence, const m3tsz_options *opts,
                        const uint8_t *d_streams, uint64_t streams_bytes,
                        const uint64_t *d_offsets, const uint64_t *d_lengths, uint64_t n_series, int64_t start_ns,
                        int64_t step_ns, uint32_t n_windows, bool counter, const TileTransforms &xf, cudaStream_t st,
                        TileWindows &w) {
  DecodeParams p;
  if (!decode_params(opts, d_streams, streams_bytes, d_offsets, d_lengths, n_series, nullptr, nullptr, p))
    return M3TSZ_ERR_INVALID_ARG;
  const bool sq = needs_sum_sq(counter, xf.types, xf.n_types);
  const size_t wb = (size_t)n_series * n_windows * 8;
  int rc;
  if ((rc = ensure(ctx, fence, kSlotWinSum, wb, &w.sum))) return rc;
  if ((rc = ensure(ctx, fence, kSlotWinCount, wb, &w.cnt))) return rc;
  if ((rc = ensure(ctx, fence, kSlotWinMin, wb, &w.min))) return rc;
  if ((rc = ensure(ctx, fence, kSlotWinMax, wb, &w.max))) return rc;
  if ((rc = ensure(ctx, fence, kSlotWinLastAt, wb, &w.lat))) return rc;
  if ((rc = ensure(ctx, fence, kSlotWinLast, wb, &w.last))) return rc;
  if ((rc = ensure(ctx, fence, kSlotNPoints, n_series * 4, &w.np))) return rc;
  if ((rc = ensure(ctx, fence, kSlotStatus, n_series * 4, &w.sst))) return rc;
  if (xf.annotated && (rc = ensure(ctx, fence, kSlotWinAnn, wb, &w.ann))) return rc;
  if (sq && (rc = ensure(ctx, fence, kSlotWinSumSq, wb, &w.sq))) return rc;
  p.n_points = (uint32_t *)w.np;
  p.status = (int32_t *)w.sst;
  p.range_start = start_ns;
  p.window = step_ns;
  p.n_windows = n_windows;
  p.ds_count = (int64_t *)w.cnt;
  if (counter) {
    p.ds_isum = (int64_t *)w.sum;
    p.ds_imin = (int64_t *)w.min;
    p.ds_imax = (int64_t *)w.max;
    p.ds_isum_sq = (int64_t *)w.sq;
  } else {
    p.ds_sum = (double *)w.sum;
    p.ds_min = (double *)w.min;
    p.ds_max = (double *)w.max;
    p.ds_sum_sq = (double *)w.sq;
    p.ds_last = (double *)w.last;
    p.ds_last_at = (int64_t *)w.lat;
  }
  p.ds_ann = (uint64_t *)w.ann;
  p.block_off = xf.block_off;
  p.n_segments = xf.n_segments;
  const int mode = xf.annotated ? (counter ? 8 : sq ? 7 : 6) : (counter ? 5 : sq ? 4 : 2);
  CK(launch_decode(p, opts->int_optimized != 0, mode, st));
  ctx->launches++;
  return M3TSZ_OK;
}

// The window aggregates as the tile stages read them: window-major [n_windows][n_src] (IN = 2 / 4 read
// n_src = p.n_series, the multi-type stage p.tile_n_src)
static void tile_inputs(EncodeParams &p, bool counter, const TileWindows &w) {
  p.tile_count = (const int64_t *)w.cnt;
  if (counter) {
    p.tile_isum = (const int64_t *)w.sum;
    p.tile_imin = (const int64_t *)w.min;
    p.tile_imax = (const int64_t *)w.max;
  } else {
    p.tile_sum = (const double *)w.sum;
    p.tile_min = (const double *)w.min;
    p.tile_max = (const double *)w.max;
    p.tile_last = (const double *)w.last;
  }
  p.tile_sum_sq = w.sq;  // (NULL unless SumSq / Stdev / Counter)
}

// The room a row's slot adds for its annotations with xf.annotated: `launch` writes the bound (launch_max_stream_len
// or launch_group_max_stream_len) into a zeroed device word, which is read back.
extern "C++" {
template <typename Launch>
static int annotation_room(m3tsz_ctx *ctx, const ScratchFence &fence, cudaStream_t st, const Launch &launch,
                           uint64_t &room) {
  void *d_mx = nullptr;
  int rc;
  if ((rc = ensure(ctx, fence, kSlotSrcMaxLen, 8, &d_mx))) return rc;
  CK(cudaMemsetAsync(d_mx, 0, 8, st));
  CK(launch((unsigned long long *)d_mx));
  ctx->launches++;
  CK(cudaMemcpyAsync(&room, d_mx, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return M3TSZ_OK;
}
}

// Step 2 of every tile call: the element xf over the windows w of n_src sources, re-encoded straight into the packed
// outputs (the encoder's input stage skips empty windows, stamps the window end and takes Gauge.ValueOf(type)), then
// the status pass: a failed source's error goes to all its rows.  With xf.annotated the rows copy annotations of the
// streams d_streams, and every slot adds ann_room bytes for them (annotation_room).  The references w.ann hold the
// payload's bit offset in its stream, whose byte offset is d_offsets[source], or, with xf.block_off or a NULL
// d_offsets, in the whole batch.
static int tiles_encode(m3tsz_ctx *ctx, const ScratchFence &fence, const m3tsz_options *opts, const TileWindows &w,
                        uint64_t n_src,
                        int64_t start_ns, int64_t step_ns, uint32_t n_windows, int32_t metric_type, int32_t out_unit,
                        const TileTransforms &xf, const uint8_t *d_streams, const uint64_t *d_offsets,
                        uint64_t ann_room, const TileOutputs &out, cudaStream_t st) {
  CK(cudaMemsetAsync(out.total_bytes, 0, sizeof(uint64_t), st));
  const uint64_t n_rows = (uint64_t)xf.n_types * n_src;
  if (n_rows == 0) return M3TSZ_OK;  // (a rollup without groups)
  int rc;
  // (a Reset op writes up to two datapoints per window)
  uint64_t slot_bytes = m3tsz_encode_bound(xf.reset ? 2ull * n_windows : (uint64_t)n_windows);
  // a row's annotations are copies of different annotations of its source streams
  if (xf.annotated) slot_bytes = (slot_bytes + ann_room + 15) & ~15ull;
  EncodeParams p;
  memset(&p, 0, sizeof(p));
  if ((rc = packed_params(ctx, fence, n_rows, slot_bytes, out.align, out.packed, out.capacity, out.offsets,
                          out.total_bytes, st, p)))
    return rc;
  // every row's encoder starts at the tile range's start (the target block's start)
  void *d_es = nullptr, *d_rec = nullptr;
  if ((rc = ensure(ctx, fence, kSlotTileStarts, n_rows * 8, &d_es))) return rc;
  CK(launch_fill_i64((int64_t *)d_es, start_ns, n_rows, st));
  // lanes write their parts of each source's new element record to scratch; the status pass commits whole records
  if (xf.elem_state && (rc = ensure(ctx, fence, kSlotElementScratch, n_src * sizeof(m3tsz_element_state), &d_rec)))
    return rc;
  p.n_series = n_rows;
  p.points_stride = n_windows;
  p.start = (const int64_t *)d_es;
  p.unit = out_unit;
  p.default_unit = opts->default_time_unit;
  p.out_len = out.len;
  p.status = out.status;
  tile_inputs(p, metric_type == M3TSZ_METRIC_COUNTER, w);
  p.tile_src_status = (const int32_t *)w.sst;
  p.tile_start = start_ns;
  p.tile_step = step_ns;
  p.agg_type = xf.types[0];
  p.metric_type = metric_type;
  p.n_tiles_out = out.n_tiles;
  p.xf_ops = xf.ops;
  p.xf_discard_nan = xf.discard ? 1 : 0;
  if (xf.multi) {
    p.in_mode = 5;
    if (xf.annotated) {
      p.tile_src_off = xf.block_off ? nullptr : d_offsets;
      p.in_mode = p.tile_src_off ? 6 : 7;  // (7: the references hold the payload's bit offset in the whole batch)
      p.tile_ann = (const uint64_t *)w.ann;
      p.tile_src_streams = d_streams;
    }
    p.xf_elem = xf.elem_state;
    p.xf_elem_out = (m3tsz_element_state *)d_rec;
    p.tile_n_src = n_src;
    p.tile_n_types = xf.n_types;
    for (uint32_t j = 0; j < xf.n_types; j++) p.tile_types |= (uint32_t)xf.types[j] << (4 * j);
  } else if (xf.ops) {
    p.in_mode = 4;
    p.xf_state = xf.state;
  } else {
    p.in_mode = 2;
  }
  CK(launch_encode(p, opts->int_optimized != 0, st));
  ctx->launches += 2;
  CK(launch_tiles_types_status((const int32_t *)w.sst, out.status, n_src, xf.n_types,
                               (const m3tsz_element_state *)d_rec, xf.elem_state, st));
  ctx->launches++;
  return M3TSZ_OK;
}

// Every tile call but the rollup, after the caller checked its element: the fused decode, then the element stage.
static int aggregate_tiles_impl(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams,
                                uint64_t streams_bytes, const uint64_t *d_offsets, const uint64_t *d_lengths,
                                uint64_t n_series, int64_t start_ns, int64_t step_ns, uint32_t n_windows,
                                int32_t metric_type, int32_t out_unit, const TileTransforms &xf,
                                const TileOutputs &out, void *stream) {
  if (!ctx || !valid_opts(opts) || !out.total_bytes || !out.status) return M3TSZ_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  if (n_series == 0) {
    DeviceGuard guard(ctx->device);
    CK(cudaMemsetAsync(out.total_bytes, 0, sizeof(uint64_t), st));
    return M3TSZ_OK;
  }
  if (!valid_packing(out) || !valid_windows(start_ns, step_ns, n_windows)) return M3TSZ_ERR_INVALID_ARG;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  ScratchFence fence(ctx, st);
  TileWindows win;
  int rc;
  if ((rc = tiles_decode(ctx, fence, opts, d_streams, streams_bytes, d_offsets, d_lengths, n_series, start_ns, step_ns,
                         n_windows, metric_type == M3TSZ_METRIC_COUNTER, xf, st, win)))
    return rc;
  // the longest source stream of the call (over source blocks: the largest sum of a series' block lengths)
  uint64_t room = 0;
  if (xf.annotated && (rc = annotation_room(ctx, fence, st, [&](unsigned long long *mx) {
        return launch_max_stream_len(d_offsets, d_lengths, xf.block_off, n_series, xf.n_segments, streams_bytes, mx,
                                     st);
      }, room)))
    return rc;
  return tiles_encode(ctx, fence, opts, win, n_series, start_ns, step_ns, n_windows, metric_type, out_unit, xf,
                      d_streams, d_offsets, room, out, st);
}

// aggregation.Type.IsValidForGauge / IsValidForCounter, src/metrics/aggregation/type.go:178-196
static bool valid_tile_pair(int32_t metric_type, int32_t agg_type) {
  switch (agg_type) {
    case M3TSZ_AGG_LAST: return metric_type == M3TSZ_METRIC_GAUGE;
    case M3TSZ_AGG_MIN: case M3TSZ_AGG_MAX: case M3TSZ_AGG_MEAN: case M3TSZ_AGG_COUNT: case M3TSZ_AGG_SUM:
    case M3TSZ_AGG_SUMSQ: case M3TSZ_AGG_STDEV:
      return metric_type == M3TSZ_METRIC_GAUGE || metric_type == M3TSZ_METRIC_COUNTER;
    default: return false;
  }
}

// newParsedPipeline (aggregator/elem_base.go:682-752): known types, derivative order <= 1
static bool parse_transforms(const int32_t *ops, uint32_t n_ops, TileTransforms &xf) {
  if (n_ops > M3TSZ_MAX_TRANSFORMS || (n_ops && !ops)) return false;
  int binary = 0;
  for (uint32_t k = 0; k < n_ops; k++) {
    if (ops[k] < M3TSZ_TRANSFORM_ABSOLUTE || ops[k] > M3TSZ_TRANSFORM_RESET) return false;
    binary += ops[k] == M3TSZ_TRANSFORM_PERSECOND || ops[k] == M3TSZ_TRANSFORM_INCREASE;
    xf.reset |= ops[k] == M3TSZ_TRANSFORM_RESET;
    xf.ops |= (uint32_t)ops[k] << (4 * k);
  }
  return binary <= 1;
}

// An element of the multi-type stage: its types strictly ascending (idDecompressor.Decompress walks a bitset), each
// valid for the metric, its transformations, and its records
static bool parse_element(int32_t metric_type, const int32_t *types, uint32_t n_types, const int32_t *ops,
                          uint32_t n_ops, m3tsz_element_state *state, TileTransforms &xf) {
  if (!types || n_types == 0 || n_types > M3TSZ_MAX_ELEMENT_TYPES) return false;
  for (uint32_t j = 0; j < n_types; j++)
    if (!valid_tile_pair(metric_type, types[j]) || (j && types[j] <= types[j - 1])) return false;
  xf.types = types;
  xf.n_types = n_types;
  xf.multi = true;
  xf.elem_state = state;
  return parse_transforms(ops, n_ops, xf);
}

int m3tsz_aggregate_tiles_batch(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams,
                                uint64_t streams_bytes, const uint64_t *d_offsets,
                                const uint64_t *d_lengths, uint64_t n_series, int64_t start_ns,
                                int64_t step_ns, uint32_t n_windows, int32_t agg_type, int32_t out_unit,
                                uint32_t align, uint8_t *d_packed, uint64_t packed_capacity,
                                uint64_t *d_out_offsets, uint64_t *d_out_len, int32_t *d_status,
                                uint32_t *d_n_tiles, uint64_t *d_total_bytes, void *stream) {
  if (!(agg_type == M3TSZ_AGG_LAST || agg_type == M3TSZ_AGG_MIN || agg_type == M3TSZ_AGG_MAX ||
        agg_type == M3TSZ_AGG_MEAN || agg_type == M3TSZ_AGG_COUNT || agg_type == M3TSZ_AGG_SUM))
    return M3TSZ_ERR_INVALID_ARG;
  TileTransforms xf;
  xf.types = &agg_type;
  xf.n_types = 1;
  return aggregate_tiles_impl(ctx, opts, d_streams, streams_bytes, d_offsets, d_lengths, n_series, start_ns, step_ns,
                              n_windows, M3TSZ_METRIC_GAUGE, out_unit, xf,
                              {align, d_packed, packed_capacity, d_out_offsets, d_out_len, d_status, d_n_tiles,
                               d_total_bytes},
                              stream);
}

int m3tsz_aggregate_tiles_ex(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams,
                             uint64_t streams_bytes, const uint64_t *d_offsets, const uint64_t *d_lengths,
                             uint64_t n_series, int64_t start_ns, int64_t step_ns, uint32_t n_windows,
                             int32_t metric_type, int32_t agg_type, int32_t out_unit, uint32_t align,
                             uint8_t *d_packed, uint64_t packed_capacity, uint64_t *d_out_offsets,
                             uint64_t *d_out_len, int32_t *d_status, uint32_t *d_n_tiles,
                             uint64_t *d_total_bytes, void *stream) {
  if (!valid_tile_pair(metric_type, agg_type)) return M3TSZ_ERR_INVALID_ARG;
  TileTransforms xf;
  xf.types = &agg_type;
  xf.n_types = 1;
  return aggregate_tiles_impl(ctx, opts, d_streams, streams_bytes, d_offsets, d_lengths, n_series, start_ns, step_ns,
                              n_windows, metric_type, out_unit, xf,
                              {align, d_packed, packed_capacity, d_out_offsets, d_out_len, d_status, d_n_tiles,
                               d_total_bytes},
                              stream);
}

int m3tsz_aggregate_tiles_transform(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams,
                                    uint64_t streams_bytes, const uint64_t *d_offsets, const uint64_t *d_lengths,
                                    uint64_t n_series, int64_t start_ns, int64_t step_ns, uint32_t n_windows,
                                    int32_t metric_type, int32_t agg_type, int32_t out_unit, uint32_t align,
                                    uint8_t *d_packed, uint64_t packed_capacity, uint64_t *d_out_offsets,
                                    uint64_t *d_out_len, int32_t *d_status, uint32_t *d_n_tiles,
                                    uint64_t *d_total_bytes, const int32_t *ops, uint32_t n_ops,
                                    int32_t discard_nan, m3tsz_transform_state *d_state, void *stream) {
  TileTransforms xf;
  if (!valid_tile_pair(metric_type, agg_type) || !parse_transforms(ops, n_ops, xf)) return M3TSZ_ERR_INVALID_ARG;
  xf.types = &agg_type;
  xf.n_types = 1;
  xf.discard = xf.ops && discard_nan;
  xf.state = d_state;
  return aggregate_tiles_impl(ctx, opts, d_streams, streams_bytes, d_offsets, d_lengths, n_series, start_ns, step_ns,
                              n_windows, metric_type, out_unit, xf,
                              {align, d_packed, packed_capacity, d_out_offsets, d_out_len, d_status, d_n_tiles,
                               d_total_bytes},
                              stream);
}

int m3tsz_aggregate_tiles_types(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams,
                                uint64_t streams_bytes, const uint64_t *d_offsets, const uint64_t *d_lengths,
                                uint64_t n_series, int64_t start_ns, int64_t step_ns, uint32_t n_windows,
                                int32_t metric_type, const int32_t *agg_types, uint32_t n_types,
                                int32_t out_unit, uint32_t align, uint8_t *d_packed, uint64_t packed_capacity,
                                uint64_t *d_out_offsets, uint64_t *d_out_len, int32_t *d_status,
                                uint32_t *d_n_tiles, uint64_t *d_total_bytes, const int32_t *ops,
                                uint32_t n_ops, int32_t discard_nan, m3tsz_element_state *d_state,
                                void *stream) {
  TileTransforms xf;
  if (!parse_element(metric_type, agg_types, n_types, ops, n_ops, d_state, xf)) return M3TSZ_ERR_INVALID_ARG;
  xf.discard = xf.ops && discard_nan;
  return aggregate_tiles_impl(ctx, opts, d_streams, streams_bytes, d_offsets, d_lengths, n_series, start_ns, step_ns,
                              n_windows, metric_type, out_unit, xf,
                              {align, d_packed, packed_capacity, d_out_offsets, d_out_len, d_status, d_n_tiles,
                               d_total_bytes},
                              stream);
}

int m3tsz_aggregate_tiles_annotated(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams,
                                    uint64_t streams_bytes, const uint64_t *d_offsets, const uint64_t *d_lengths,
                                    uint64_t n_series, int64_t start_ns, int64_t step_ns, uint32_t n_windows,
                                    int32_t metric_type, const int32_t *agg_types, uint32_t n_types,
                                    int32_t out_unit, uint32_t align, uint8_t *d_packed, uint64_t packed_capacity,
                                    uint64_t *d_out_offsets, uint64_t *d_out_len, int32_t *d_status,
                                    uint32_t *d_n_tiles, uint64_t *d_total_bytes, const int32_t *ops,
                                    uint32_t n_ops, int32_t discard_nan, m3tsz_element_state *d_state,
                                    void *stream) {
  TileTransforms xf;
  if (!parse_element(metric_type, agg_types, n_types, ops, n_ops, d_state, xf)) return M3TSZ_ERR_INVALID_ARG;
  xf.discard = xf.ops && discard_nan;
  xf.annotated = true;
  return aggregate_tiles_impl(ctx, opts, d_streams, streams_bytes, d_offsets, d_lengths, n_series, start_ns, step_ns,
                              n_windows, metric_type, out_unit, xf,
                              {align, d_packed, packed_capacity, d_out_offsets, d_out_len, d_status, d_n_tiles,
                               d_total_bytes},
                              stream);
}

int m3tsz_aggregate_tiles_blocks(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams,
                                 uint64_t streams_bytes, const uint64_t *d_offsets, const uint64_t *d_lengths,
                                 uint64_t n_segments, const uint64_t *d_block_off, uint64_t n_series, int64_t start_ns,
                                 int64_t step_ns, uint32_t n_windows, int32_t metric_type, const int32_t *agg_types,
                                 uint32_t n_types, int32_t out_unit, uint32_t align, uint8_t *d_packed,
                                 uint64_t packed_capacity, uint64_t *d_out_offsets, uint64_t *d_out_len,
                                 int32_t *d_status, uint32_t *d_n_tiles, uint64_t *d_total_bytes, const int32_t *ops,
                                 uint32_t n_ops, int32_t discard_nan, m3tsz_element_state *d_state,
                                 int32_t annotations, void *stream) {
  // (the block table's ranges are checked per series on the device: a bad one is that series' INVALID_ARG)
  TileTransforms xf;
  if (!d_block_off || !parse_element(metric_type, agg_types, n_types, ops, n_ops, d_state, xf))
    return M3TSZ_ERR_INVALID_ARG;
  xf.discard = xf.ops && discard_nan;
  xf.annotated = annotations != 0;
  xf.block_off = d_block_off;
  xf.n_segments = n_segments;
  return aggregate_tiles_impl(ctx, opts, d_streams, streams_bytes, d_offsets, d_lengths, n_series, start_ns, step_ns,
                              n_windows, metric_type, out_unit, xf,
                              {align, d_packed, packed_capacity, d_out_offsets, d_out_len, d_status, d_n_tiles,
                               d_total_bytes},
                              stream);
}

// Tile aggregation through a rollup (DESIGN.md §4.8): the fused decode of the sources under src_type, the forward
// stage (each source's pre_ops chain), the fold into the groups' windows, then the multi-type element stage over
// n_rollup_types * n_groups rows, its status pass, and the source records.  annotated: the annotated decode, forward
// and fold variants carry each group window's annotation to its rows.
static int aggregate_tiles_rollup_impl(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams,
                                       uint64_t streams_bytes, const uint64_t *d_offsets, const uint64_t *d_lengths,
                                       uint64_t n_segments, const uint64_t *d_block_off, uint64_t n_series,
                                       int64_t start_ns, int64_t step_ns, uint32_t n_windows, int32_t metric_type,
                                       int32_t src_type, const int32_t *pre_ops, uint32_t n_pre_ops,
                                       const uint64_t *d_group_off, const uint32_t *d_members, uint64_t n_members,
                                       uint64_t n_groups, const int32_t *rollup_types, uint32_t n_rollup_types,
                                       const int32_t *post_ops, uint32_t n_post_ops, int32_t discard_nan,
                                       m3tsz_transform_state *d_src_state, m3tsz_element_state *d_group_state,
                                       int32_t out_unit, const TileOutputs &out, int32_t *d_src_status, bool annotated,
                                       void *stream) {
  TileTransforms pre, post;  // the sources' element and the groups'
  if (!ctx || !valid_opts(opts) || !out.total_bytes || !valid_tile_pair(metric_type, src_type) ||
      (!d_block_off && n_segments != n_series) || (n_groups && (!d_group_off || !out.status)) ||
      (n_members && !d_members) || !parse_transforms(pre_ops, n_pre_ops, pre) ||
      !parse_element(metric_type, rollup_types, n_rollup_types, post_ops, n_post_ops, d_group_state, post))
    return M3TSZ_ERR_INVALID_ARG;
  if (((uint64_t)n_rollup_types * n_groups != 0 && !valid_packing(out)) || !valid_windows(start_ns, step_ns, n_windows))
    return M3TSZ_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  ScratchFence fence(ctx, st);
  const bool counter = metric_type == M3TSZ_METRIC_COUNTER;
  int rc;
  // 1. fused decode + windows of the sources under their one type
  pre.types = &src_type;
  pre.n_types = 1;
  pre.block_off = d_block_off;
  pre.n_segments = n_segments;
  pre.annotated = annotated;
  TileWindows win;
  if (n_series && (rc = tiles_decode(ctx, fence, opts, d_streams, streams_bytes, d_offsets, d_lengths, n_series,
                                     start_ns, step_ns, n_windows, counter, pre, st, win)))
    return rc;
  // 2. forward stage: series-major forwarded values and presence words, each source's new record to scratch
  const uint32_t n_words = (n_windows + 31) / 32;
  void *d_fwd, *d_pres, *d_srec, *d_mark;
  if ((rc = ensure(ctx, fence, kSlotFwdVal, (size_t)n_series * n_windows * 8, &d_fwd))) return rc;
  if ((rc = ensure(ctx, fence, kSlotFwdPresent, (size_t)n_series * n_words * 4, &d_pres))) return rc;
  if ((rc = ensure(ctx, fence, kSlotSrcRecScratch, n_series * sizeof(m3tsz_transform_state), &d_srec))) return rc;
  if ((rc = ensure(ctx, fence, kSlotSrcMark, n_series, &d_mark))) return rc;
  RollupForwardParams fp;
  memset(&fp, 0, sizeof(fp));
  tile_inputs(fp.tiles, counter, win);
  fp.tiles.metric_type = metric_type;
  fp.tiles.tile_start = start_ns;
  fp.tiles.tile_step = step_ns;
  fp.src_status = (const int32_t *)win.sst;
  fp.n_src = n_series;
  fp.n_windows = n_windows;
  fp.n_words = n_words;
  fp.src_type = src_type;
  fp.ops = pre.ops;
  fp.discard_nan = discard_nan ? 1 : 0;  // (generic_elem.go:892-894: with or without transformations)
  fp.state = d_src_state;
  fp.state_out = (m3tsz_transform_state *)d_srec;
  fp.fwd = (double *)d_fwd;
  fp.present = (uint32_t *)d_pres;
  void *d_apres = nullptr;
  if (annotated) {
    if ((rc = ensure(ctx, fence, kSlotFwdAnnPresent, (size_t)n_series * n_words * 4, &d_apres))) return rc;
    fp.ann = (uint64_t *)win.ann;
    fp.src_off = d_block_off ? nullptr : d_offsets;  // (the block decode's references are batch-addressed already)
    fp.src_status_out = (int32_t *)win.sst;
    fp.ann_present = (uint32_t *)d_apres;
  }
  CK(launch_rollup_forward(fp, annotated, st));
  ctx->launches++;
  // 3. fold: the groups' window-major aggregates, in the fused decode's representation, and their statuses
  const size_t gb = (size_t)n_groups * n_windows * 8;
  TileWindows grp;
  if ((rc = ensure(ctx, fence, kSlotGroupSum, gb, &grp.sum))) return rc;
  if ((rc = ensure(ctx, fence, kSlotGroupCount, gb, &grp.cnt))) return rc;
  if ((rc = ensure(ctx, fence, kSlotGroupMin, gb, &grp.min))) return rc;
  if ((rc = ensure(ctx, fence, kSlotGroupMax, gb, &grp.max))) return rc;
  if (!counter && (rc = ensure(ctx, fence, kSlotGroupLast, gb, &grp.last))) return rc;
  if (needs_sum_sq(counter, rollup_types, n_rollup_types) && (rc = ensure(ctx, fence, kSlotGroupSumSq, gb, &grp.sq)))
    return rc;
  if ((rc = ensure(ctx, fence, kSlotGroupStatus, n_groups * 4, &grp.sst))) return rc;
  if (annotated && (rc = ensure(ctx, fence, kSlotGroupAnn, gb, &grp.ann))) return rc;
  RollupFoldParams gp;
  memset(&gp, 0, sizeof(gp));
  gp.fwd = (const double *)d_fwd;
  gp.present = (const uint32_t *)d_pres;
  gp.src_status = (const int32_t *)win.sst;
  gp.n_src = n_series;
  gp.n_windows = n_windows;
  gp.n_words = n_words;
  gp.group_off = d_group_off;
  gp.members = d_members;
  gp.n_members = n_members;
  gp.n_groups = n_groups;
  gp.counter = counter ? 1 : 0;
  gp.sum = grp.sum;
  gp.count = (int64_t *)grp.cnt;
  gp.min = grp.min;
  gp.max = grp.max;
  gp.last = (double *)grp.last;
  gp.sum_sq = grp.sq;
  gp.group_status = (int32_t *)grp.sst;
  gp.ann_present = (const uint32_t *)d_apres;
  gp.ann = (const uint64_t *)win.ann;
  gp.group_ann = (uint64_t *)grp.ann;
  CK(launch_rollup_fold(gp, annotated, st));
  ctx->launches++;
  // 4. the rollup element over n_rollup_types * n_groups rows, the groups as its sources.  With annotations a group
  // row copies annotations of its members' streams (batch-addressed references: IN = 7), so its slot adds the largest
  // sum, over groups, of the members' source lengths
  post.discard = discard_nan != 0;
  post.annotated = annotated;
  uint64_t room = 0;
  if (annotated && (uint64_t)n_rollup_types * n_groups != 0 &&
      (rc = annotation_room(ctx, fence, st, [&](unsigned long long *mx) {
         return launch_group_max_stream_len(d_offsets, d_lengths, d_block_off, n_series, n_segments, streams_bytes,
                                            d_group_off, d_members, n_members, n_groups, mx, st);
       }, room)))
    return rc;
  if ((rc = tiles_encode(ctx, fence, opts, grp, n_groups, start_ns, step_ns, n_windows, metric_type, out_unit, post,
                         d_streams, nullptr, room, out, st)))
    return rc;
  // 5. the source records: a source is saved when it decoded and every group that lists it was saved
  CK(launch_rollup_commit(d_group_off, d_members, n_members, n_groups, out.status, n_rollup_types,
                          (const int32_t *)win.sst, n_series, (uint8_t *)d_mark, (const m3tsz_transform_state *)d_srec,
                          d_src_state, d_src_status, st));
  ctx->launches += 2;
  return M3TSZ_OK;
}

int m3tsz_aggregate_tiles_rollup(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams,
                                 uint64_t streams_bytes, const uint64_t *d_offsets, const uint64_t *d_lengths,
                                 uint64_t n_segments, const uint64_t *d_block_off, uint64_t n_series, int64_t start_ns,
                                 int64_t step_ns, uint32_t n_windows, int32_t metric_type, int32_t src_type,
                                 const int32_t *pre_ops, uint32_t n_pre_ops, const uint64_t *d_group_off,
                                 const uint32_t *d_members, uint64_t n_members, uint64_t n_groups,
                                 const int32_t *rollup_types, uint32_t n_rollup_types, const int32_t *post_ops,
                                 uint32_t n_post_ops, int32_t discard_nan, m3tsz_transform_state *d_src_state,
                                 m3tsz_element_state *d_group_state, int32_t out_unit, uint32_t align,
                                 uint8_t *d_packed, uint64_t packed_capacity, uint64_t *d_out_offsets,
                                 uint64_t *d_out_len, int32_t *d_status, uint32_t *d_n_tiles, uint64_t *d_total_bytes,
                                 int32_t *d_src_status, void *stream) {
  return aggregate_tiles_rollup_impl(
      ctx, opts, d_streams, streams_bytes, d_offsets, d_lengths, n_segments, d_block_off, n_series, start_ns, step_ns,
      n_windows, metric_type, src_type, pre_ops, n_pre_ops, d_group_off, d_members, n_members, n_groups, rollup_types,
      n_rollup_types, post_ops, n_post_ops, discard_nan, d_src_state, d_group_state, out_unit,
      {align, d_packed, packed_capacity, d_out_offsets, d_out_len, d_status, d_n_tiles, d_total_bytes}, d_src_status,
      false, stream);
}

int m3tsz_aggregate_tiles_rollup_annotated(
    m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams, uint64_t streams_bytes,
    const uint64_t *d_offsets, const uint64_t *d_lengths, uint64_t n_segments, const uint64_t *d_block_off,
    uint64_t n_series, int64_t start_ns, int64_t step_ns, uint32_t n_windows, int32_t metric_type, int32_t src_type,
    const int32_t *pre_ops, uint32_t n_pre_ops, const uint64_t *d_group_off, const uint32_t *d_members,
    uint64_t n_members, uint64_t n_groups, const int32_t *rollup_types, uint32_t n_rollup_types,
    const int32_t *post_ops, uint32_t n_post_ops, int32_t discard_nan, m3tsz_transform_state *d_src_state,
    m3tsz_element_state *d_group_state, int32_t out_unit, uint32_t align, uint8_t *d_packed, uint64_t packed_capacity,
    uint64_t *d_out_offsets, uint64_t *d_out_len, int32_t *d_status, uint32_t *d_n_tiles, uint64_t *d_total_bytes,
    int32_t *d_src_status, void *stream) {
  return aggregate_tiles_rollup_impl(
      ctx, opts, d_streams, streams_bytes, d_offsets, d_lengths, n_segments, d_block_off, n_series, start_ns, step_ns,
      n_windows, metric_type, src_type, pre_ops, n_pre_ops, d_group_off, d_members, n_members, n_groups, rollup_types,
      n_rollup_types, post_ops, n_post_ops, discard_nan, d_src_state, d_group_state, out_unit,
      {align, d_packed, packed_capacity, d_out_offsets, d_out_len, d_status, d_n_tiles, d_total_bytes}, d_src_status,
      true, stream);
}

// ---- element sets (DESIGN.md §4.12) ----
// The checks every element-set call makes on the set (its element as m3tsz_aggregate_tiles_types checks one, its
// arrays' presence and alignment), and the parameters the kernels read; xf takes the parsed lists.
static bool element_set_no_output(const m3tsz_element_set *set) {
  return !set->d_out_state && !set->d_out_buf && set->out_stride == 0;
}
// A Timer's type list (IsValidForTimer: all but Last), strictly ascending, up to M3TSZ_MAX_TIMER_TYPES without ops
static bool parse_timer_element(const int32_t *types, uint32_t n_types, const int32_t *ops, uint32_t n_ops,
                                TileTransforms &xf) {
  if (!types || n_types == 0 || n_types > (n_ops ? M3TSZ_MAX_ELEMENT_TYPES : M3TSZ_MAX_TIMER_TYPES)) return false;
  for (uint32_t j = 0; j < n_types; j++)
    if (types[j] < M3TSZ_AGG_MIN || types[j] > M3TSZ_AGG_P75 || (j && types[j] <= types[j - 1])) return false;
  xf.types = types;
  xf.n_types = n_types;
  xf.multi = true;
  return parse_transforms(ops, n_ops, xf);
}

// timer: the set must be a Timer set (the Timer calls), else it must not be one (every other call but the reset)
static bool element_params(const m3tsz_options *opts, const m3tsz_element_set *set, ElementParams &p,
                           TileTransforms &xf, bool timer = false) {
  if (!valid_opts(opts) || !set || set->reserved != 0) return false;
  const m3tsz_element_set &e = *set;
  const bool counter = e.metric_type == M3TSZ_METRIC_COUNTER;
  if (timer != (e.metric_type == M3TSZ_METRIC_TIMER)) return false;
  if (e.n_windows == 0 || e.n_windows > M3TSZ_MAX_ELEMENT_WINDOWS || e.resolution_ns <= 0 ||
      e.n_elements > (1ull << 40) ||
      !(timer ? parse_timer_element(e.agg_types, e.n_types, e.ops, e.n_ops, xf)
              : parse_element(e.metric_type, e.agg_types, e.n_types, e.ops, e.n_ops, e.d_elem, xf)))
    return false;
  auto a8 = [](const void *q) { return q && !((uintptr_t)q & 7u); };
  auto a16 = [](const void *q) { return q && !((uintptr_t)q & 15u); };
  if (timer) {  // (a Timer's slots: start, count, sum, sum_sq)
    if (!a8(e.d_win_start) || !a8(e.d_win_count) || !a8(e.d_win_sum) || !a8(e.d_win_sum_sq) || !a16(e.d_elem) ||
        !a8(e.d_watermark))
      return false;
    for (const void *q : {(const void *)e.d_win_min, (const void *)e.d_win_max, (const void *)e.d_win_last,
                          (const void *)e.d_win_last_at})
      if ((uintptr_t)q & 7u) return false;
  } else if (!a8(e.d_win_start) || !a8(e.d_win_count) || !a8(e.d_win_sum) || !a8(e.d_win_min) ||
             !a8(e.d_win_max) || !a8(e.d_win_sum_sq) || (!counter && (!a8(e.d_win_last) || !a8(e.d_win_last_at))) ||
             !a16(e.d_elem) || !a8(e.d_watermark)) {
    return false;
  }
  // a set without output (NULL output arrays, out_stride 0) is a rollup's source set: every call but the consume
  // takes it
  if (!element_set_no_output(set) && (!a16(e.d_out_state) || !a16(e.d_out_buf) || (e.out_stride & 15u) ||
                                      e.out_stride == 0 || e.out_stride > (1ull << 33)))
    return false;
  memset(&p, 0, sizeof(p));
  p.n = e.n_elements;
  p.n_slots = e.n_windows;
  p.counter = counter ? 1 : 0;
  p.resolution = e.resolution_ns;
  // time.Time.Truncate counts from the zero time, 62135596800 s before the Unix epoch
  p.trunc_off = (int64_t)((unsigned __int128)62135596800ull * 1000000000ull % (unsigned __int128)e.resolution_ns);
  p.start = e.d_win_start;
  p.count = e.d_win_count;
  p.sum = e.d_win_sum;
  p.min = e.d_win_min;
  p.max = e.d_win_max;
  p.sum_sq = e.d_win_sum_sq;
  p.last = e.d_win_last;
  p.last_at = e.d_win_last_at;
  p.elem = e.d_elem;
  p.watermark = e.d_watermark;
  if (!timer)
    for (uint32_t j = 0; j < xf.n_types; j++) p.types |= (uint32_t)xf.types[j] << (4 * j);
  p.n_types = xf.n_types;
  p.ops = xf.ops;
  p.discard_nan = (xf.ops && e.discard_nan) ? 1 : 0;  // (as m3tsz_aggregate_tiles_types)
  p.out_state = e.d_out_state;
  p.out_slot_words = e.out_stride >> 2;
  memset(&p.tiles, 0, sizeof(p.tiles));
  TileWindows w;
  w.sum = e.d_win_sum;
  w.cnt = e.d_win_count;
  w.min = e.d_win_min;
  w.max = e.d_win_max;
  w.last = e.d_win_last;
  w.sq = e.d_win_sum_sq;
  tile_inputs(p.tiles, counter, w);
  p.tiles.metric_type = e.metric_type;
  return true;
}

int m3tsz_element_set_reset(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                            const int64_t *d_start, void *stream) {
  ElementParams p;
  TileTransforms xf;
  if (!ctx || !set || !element_params(opts, set, p, xf, set->metric_type == M3TSZ_METRIC_TIMER) ||
      (p.n && !d_start && !element_set_no_output(set)))
    return M3TSZ_ERR_INVALID_ARG;
  if (p.n == 0) return M3TSZ_OK;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  cudaStream_t st = (cudaStream_t)stream;
  ScratchFence fence(ctx, st, !element_set_no_output(set));  // (the output rows' starts)
  const size_t wb = (size_t)p.n * p.n_slots * 8;
  for (void *a : {(void *)p.start, (void *)p.count, p.sum, p.min, p.max, p.sum_sq, (void *)p.last, (void *)p.last_at})
    if (a) CK(cudaMemsetAsync(a, 0, wb, st));
  CK(cudaMemsetAsync(p.elem, 0, p.n * sizeof(m3tsz_element_state), st));
  CK(launch_fill_i64(p.watermark, INT64_MIN, p.n, st));
  ctx->launches++;
  if (element_set_no_output(set)) return M3TSZ_OK;
  // row j * n + s of the output starts at element s's start
  const uint64_t kn = (uint64_t)p.n_types * p.n;
  void *d_rs = nullptr;
  int rc;
  if ((rc = ensure(ctx, fence, kSlotElemRowTs, kn * 8, &d_rs))) return rc;
  for (uint32_t j = 0; j < p.n_types; j++)
    CK(cudaMemcpyAsync((int64_t *)d_rs + (uint64_t)j * p.n, d_start, p.n * 8, cudaMemcpyDeviceToDevice, st));
  CK(launch_encoder_set_reset(set->d_out_state, kn, (const int64_t *)d_rs, opts->default_time_unit,
                              opts->int_optimized != 0, st));
  ctx->launches++;
  return M3TSZ_OK;
}

// The annotated calls' slot arrays (m3tsz_element_annotations), checked as element_params checks the others; p gets
// them.  The lengths and bytes cover R * n_elements slots: a capacity of at most 2^16 keeps every offset in 64 bits.
static bool element_ann_params(const m3tsz_element_annotations *ann, ElementParams &p) {
  if (!ann || ann->reserved != 0 || ann->capacity == 0 || (ann->capacity & 7u) ||
      ann->capacity > M3TSZ_MAX_ELEMENT_ANNOTATION || !ann->d_len || ((uintptr_t)ann->d_len & 3u) || !ann->d_bytes ||
      ((uintptr_t)ann->d_bytes & 7u))
    return false;
  p.ann_len = ann->d_len;
  p.ann_slot = ann->d_bytes;
  p.ann_cap = ann->capacity;
  return true;
}

// m3tsz_element_set_add(_annotated): ann NULL is the plain add
static int element_set_add(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                           const m3tsz_element_annotations *ann, const int64_t *d_ts, const double *d_val,
                           uint64_t points_stride, const uint32_t *d_n_points, const uint64_t *d_ann_series_off,
                           const m3tsz_annotation_entry *d_ann_entries, const uint8_t *d_ann_bytes, int8_t *d_result,
                           int32_t *d_status, void *stream, bool annotated) {
  ElementParams p;
  TileTransforms xf;
  if (!ctx || !element_params(opts, set, p, xf) || points_stride > 0xffffffffull) return M3TSZ_ERR_INVALID_ARG;
  if (annotated && (!element_ann_params(ann, p) || ((uintptr_t)d_ann_series_off & 7u) ||
                    (d_ann_series_off && (!d_ann_entries || !d_ann_bytes || ((uintptr_t)d_ann_entries & 7u)))))
    return M3TSZ_ERR_INVALID_ARG;
  if (p.n == 0) return M3TSZ_OK;
  if (!d_ts || !d_val || !d_result || !d_status || ((uintptr_t)d_ts & 7u) || ((uintptr_t)d_val & 7u) ||
      ((uintptr_t)d_n_points & 3u) || ((uintptr_t)d_status & 3u))
    return M3TSZ_ERR_INVALID_ARG;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  p.ts = d_ts;
  p.val = d_val;
  p.points_stride = points_stride;
  p.n_points = d_n_points;
  p.result = d_result;
  p.status = d_status;
  if (annotated) {
    p.ann_series_off = d_ann_series_off;
    p.ann_entries = d_ann_entries;
    p.ann_bytes = d_ann_bytes;
  }
  CK(launch_element_add(p, (cudaStream_t)stream));
  ctx->launches++;
  return M3TSZ_OK;
}

int m3tsz_element_set_add(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                          const int64_t *d_ts, const double *d_val, uint64_t points_stride,
                          const uint32_t *d_n_points, int8_t *d_result, int32_t *d_status, void *stream) {
  return element_set_add(ctx, opts, set, nullptr, d_ts, d_val, points_stride, d_n_points, nullptr, nullptr, nullptr,
                         d_result, d_status, stream, false);
}

int m3tsz_element_set_add_annotated(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                                    const m3tsz_element_annotations *ann, const int64_t *d_ts, const double *d_val,
                                    uint64_t points_stride, const uint32_t *d_n_points,
                                    const uint64_t *d_ann_series_off, const m3tsz_annotation_entry *d_ann_entries,
                                    const uint8_t *d_ann_bytes, int8_t *d_result, int32_t *d_status, void *stream) {
  return element_set_add(ctx, opts, set, ann, d_ts, d_val, points_stride, d_n_points, d_ann_series_off,
                         d_ann_entries, d_ann_bytes, d_result, d_status, stream, true);
}

// The consume kernel stages each element's flushed datapoints as rows, the encoder-set append writes them, and the
// status pass folds each element's rows into its status.  Annotated: the kernel also stages each row's annotation
// entries (a fixed-stride list over the slots' bytes), which the append reads as it reads an encoder set's sparse
// list; its lane code takes that list in the point-major stage too (dp_index counts a series' rows in either layout).
static int element_set_consume(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                               const m3tsz_element_annotations *ann, int64_t target_ns, int32_t out_unit,
                               int32_t *d_status, void *stream, bool annotated) {
  ElementParams p;
  TileTransforms xf;
  if (!ctx || !element_params(opts, set, p, xf) || element_set_no_output(set) || !unit_is_valid(out_unit))
    return M3TSZ_ERR_INVALID_ARG;
  if (annotated && !element_ann_params(ann, p)) return M3TSZ_ERR_INVALID_ARG;
  if (p.n == 0) return M3TSZ_OK;
  if (!d_status || ((uintptr_t)d_status & 3u)) return M3TSZ_ERR_INVALID_ARG;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  cudaStream_t st = (cudaStream_t)stream;
  ScratchFence fence(ctx, st);
  const uint64_t kn = (uint64_t)p.n_types * p.n;
  const uint64_t rows = (uint64_t)p.n_slots * (xf.reset ? 2u : 1u);  // a Reset op writes two datapoints per window
  void *d_ts = nullptr, *d_val = nullptr, *d_n = nullptr, *d_rst = nullptr, *d_app = nullptr;
  int rc;
  if ((rc = ensure(ctx, fence, kSlotElemRowTs, kn * rows * 8, &d_ts))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemRowVal, kn * rows * 8, &d_val))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemRowN, kn * 4, &d_n))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemRowStatus, kn * 4, &d_rst))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemRowAppended, kn * 4, &d_app))) return rc;
  if (annotated) {
    void *d_aoff = nullptr, *d_aent = nullptr;
    if ((rc = ensure(ctx, fence, kSlotElemRowAnnOff, (kn + 1) * 8, &d_aoff))) return rc;
    if ((rc = ensure(ctx, fence, kSlotElemRowAnn, kn * rows * sizeof(m3tsz_annotation_entry), &d_aent))) return rc;
    p.row_ann_off = (uint64_t *)d_aoff;
    p.row_ann = (m3tsz_annotation_entry *)d_aent;
  }
  p.target = target_ns;
  p.row_ts = (int64_t *)d_ts;
  p.row_val = (double *)d_val;
  p.row_n = (uint32_t *)d_n;
  p.rows_stride = rows;
  p.status = d_status;
  CK(launch_element_consume(p, st));
  m3tsz_encode_extras ex;
  memset(&ex, 0, sizeof(ex));
  ex.point_major_input = 1;
  EncodeParams ep;
  if (!encode_params(opts, p.row_ts, p.row_val, kn, rows, p.row_n, nullptr, out_unit, nullptr, nullptr, nullptr,
                     nullptr, nullptr, (int32_t *)d_rst, &ex, ep, true))
    return M3TSZ_ERR_INVALID_ARG;
  if (annotated) {  // (the public calls take no annotations with point-major input; this list is the library's own)
    ep.ann_series_off = p.row_ann_off;
    ep.ann_entries = p.row_ann;
    ep.ann_bytes = p.ann_slot;
  }
  ep.out = set->d_out_buf;
  ep.out_stride = set->out_stride;
  ep.state = set->d_out_state;
  ep.n_appended = (uint32_t *)d_app;
  CK(launch_encode_append(ep, opts->int_optimized != 0, st));
  CK(launch_element_status((const int32_t *)d_rst, p.n, p.n_types, d_status, st));
  ctx->launches += 3;
  return M3TSZ_OK;
}

int m3tsz_element_set_consume(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                              int64_t target_ns, int32_t out_unit, int32_t *d_status, void *stream) {
  return element_set_consume(ctx, opts, set, nullptr, target_ns, out_unit, d_status, stream, false);
}

int m3tsz_element_set_consume_annotated(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                                        const m3tsz_element_annotations *ann, int64_t target_ns, int32_t out_unit,
                                        int32_t *d_status, void *stream) {
  return element_set_consume(ctx, opts, set, ann, target_ns, out_unit, d_status, stream, true);
}

// ---- Timer element sets ----
// aggregation.Type.Quantile()
static double timer_quantile(int32_t t) {
  static const double q[] = {0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9, 0.95, 0.99, 0.999, 0.9999, 0.25, 0.75};
  if (t == M3TSZ_AGG_MEDIAN) return 0.5;
  return t >= M3TSZ_AGG_P10 && t <= M3TSZ_AGG_P75 ? q[t - M3TSZ_AGG_P10] : 0.0;
}

// The Timer calls' checks: the set's (element_params), the streams' arrays and options; tp takes the set's
// parameters, the streams, the types and their PooledQuantiles list (listed order, Median and P50 once)
static bool timer_params(const m3tsz_options *opts, const m3tsz_element_set *set,
                         const m3tsz_element_timer_streams *ts, ElementTimerParams &tp, TileTransforms &xf) {
  memset(&tp, 0, sizeof(tp));
  if (!element_params(opts, set, tp.e, xf, true) || !ts || ts->reserved != 0 || ts->sample_capacity == 0 ||
      ts->sample_capacity > (1u << 30) || !std::isfinite(ts->eps) || !(ts->eps > 0.0) ||
      ts->insert_and_compress_every == 0 || ts->insert_and_compress_every > 0x7fffffffu)
    return false;
  auto a = [](const void *q, uintptr_t m) { return q && !((uintptr_t)q & m); };
  if (!a(ts->d_header, 7) || !a(ts->d_value, 7) || !a(ts->d_num_ranks, 7) || !a(ts->d_delta, 7) ||
      !a(ts->d_prev, 3) || !a(ts->d_next, 3) || !a(ts->d_heap_a, 7) || !a(ts->d_heap_b, 7))
    return false;
  tp.hdr = ts->d_header;
  tp.value = ts->d_value;
  tp.num_ranks = ts->d_num_ranks;
  tp.delta = ts->d_delta;
  tp.prev = ts->d_prev;
  tp.next = ts->d_next;
  tp.heap_a = ts->d_heap_a;
  tp.heap_b = ts->d_heap_b;
  tp.cap = ts->sample_capacity;
  tp.every = (int32_t)ts->insert_and_compress_every;
  tp.eps = ts->eps;
  tp.n_types = xf.n_types;
  bool median = false;
  for (uint32_t j = 0; j < xf.n_types; j++) {
    const int32_t t = xf.types[j];
    tp.type[j] = t;
    const double q = timer_quantile(t);
    if (q == 0.0) continue;
    if (t == M3TSZ_AGG_P50 || t == M3TSZ_AGG_MEDIAN) {
      if (median) continue;
      median = true;
    }
    tp.q[tp.n_q++] = q;
  }
  return true;
}

// m3tsz_element_set_add_timer(_annotated): ann NULL is the plain add
static int element_set_add_timer(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                                 const m3tsz_element_timer_streams *streams, const m3tsz_element_annotations *ann,
                                 const int64_t *d_ts, const double *d_val, uint64_t points_stride,
                                 const uint32_t *d_n_points, const int8_t *d_batch, const uint64_t *d_ann_series_off,
                                 const m3tsz_annotation_entry *d_ann_entries, const uint8_t *d_ann_bytes,
                                 int8_t *d_result, int32_t *d_status, void *stream, bool annotated) {
  ElementTimerParams tp;
  TileTransforms xf;
  if (!ctx || !timer_params(opts, set, streams, tp, xf) || points_stride > 0xffffffffull) return M3TSZ_ERR_INVALID_ARG;
  if (annotated && (!element_ann_params(ann, tp.e) || ((uintptr_t)d_ann_series_off & 7u) ||
                    (d_ann_series_off && (!d_ann_entries || !d_ann_bytes || ((uintptr_t)d_ann_entries & 7u)))))
    return M3TSZ_ERR_INVALID_ARG;
  if (tp.e.n == 0) return M3TSZ_OK;
  if (!d_ts || !d_val || !d_result || !d_status || ((uintptr_t)d_ts & 7u) || ((uintptr_t)d_val & 7u) ||
      ((uintptr_t)d_n_points & 3u) || ((uintptr_t)d_status & 3u))
    return M3TSZ_ERR_INVALID_ARG;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  tp.e.ts = d_ts;
  tp.e.val = d_val;
  tp.e.points_stride = points_stride;
  tp.e.n_points = d_n_points;
  tp.e.result = d_result;
  tp.e.status = d_status;
  tp.batch = d_batch;
  if (annotated) {
    tp.e.ann_series_off = d_ann_series_off;
    tp.e.ann_entries = d_ann_entries;
    tp.e.ann_bytes = d_ann_bytes;
  }
  CK(launch_element_timer_add(tp, (cudaStream_t)stream));
  ctx->launches++;
  return M3TSZ_OK;
}

int m3tsz_element_set_add_timer(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                                const m3tsz_element_timer_streams *streams, const int64_t *d_ts, const double *d_val,
                                uint64_t points_stride, const uint32_t *d_n_points, const int8_t *d_batch,
                                int8_t *d_result, int32_t *d_status, void *stream) {
  return element_set_add_timer(ctx, opts, set, streams, nullptr, d_ts, d_val, points_stride, d_n_points, d_batch,
                               nullptr, nullptr, nullptr, d_result, d_status, stream, false);
}

int m3tsz_element_set_add_timer_annotated(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                                          const m3tsz_element_timer_streams *streams,
                                          const m3tsz_element_annotations *ann, const int64_t *d_ts,
                                          const double *d_val, uint64_t points_stride, const uint32_t *d_n_points,
                                          const int8_t *d_batch, const uint64_t *d_ann_series_off,
                                          const m3tsz_annotation_entry *d_ann_entries, const uint8_t *d_ann_bytes,
                                          int8_t *d_result, int32_t *d_status, void *stream) {
  return element_set_add_timer(ctx, opts, set, streams, ann, d_ts, d_val, points_stride, d_n_points, d_batch,
                               d_ann_series_off, d_ann_entries, d_ann_bytes, d_result, d_status, stream, true);
}

// element_set_consume with the Timer's consume kernel: the same scratch rows, annotation entries, append and status
// pass.  m3tsz_element_set_consume_timer(_annotated): ann NULL is the plain consume
static int element_set_consume_timer(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                                     const m3tsz_element_timer_streams *streams, const m3tsz_element_annotations *ann,
                                     int64_t target_ns, int32_t out_unit, int32_t *d_status, void *stream,
                                     bool annotated) {
  ElementTimerParams tp;
  TileTransforms xf;
  if (!ctx || !timer_params(opts, set, streams, tp, xf) || element_set_no_output(set) || !unit_is_valid(out_unit))
    return M3TSZ_ERR_INVALID_ARG;
  ElementParams &p = tp.e;
  if (annotated && !element_ann_params(ann, p)) return M3TSZ_ERR_INVALID_ARG;
  if (p.n == 0) return M3TSZ_OK;
  if (!d_status || ((uintptr_t)d_status & 3u)) return M3TSZ_ERR_INVALID_ARG;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  cudaStream_t st = (cudaStream_t)stream;
  ScratchFence fence(ctx, st);
  const uint64_t kn = (uint64_t)tp.n_types * p.n;
  const uint64_t rows = (uint64_t)p.n_slots * (xf.reset ? 2u : 1u);
  void *d_ts = nullptr, *d_val = nullptr, *d_n = nullptr, *d_rst = nullptr, *d_app = nullptr;
  int rc;
  if ((rc = ensure(ctx, fence, kSlotElemRowTs, kn * rows * 8, &d_ts))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemRowVal, kn * rows * 8, &d_val))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemRowN, kn * 4, &d_n))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemRowStatus, kn * 4, &d_rst))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemRowAppended, kn * 4, &d_app))) return rc;
  if (annotated) {
    void *d_aoff = nullptr, *d_aent = nullptr;
    if ((rc = ensure(ctx, fence, kSlotElemRowAnnOff, (kn + 1) * 8, &d_aoff))) return rc;
    if ((rc = ensure(ctx, fence, kSlotElemRowAnn, kn * rows * sizeof(m3tsz_annotation_entry), &d_aent))) return rc;
    p.row_ann_off = (uint64_t *)d_aoff;
    p.row_ann = (m3tsz_annotation_entry *)d_aent;
  }
  p.target = target_ns;
  p.row_ts = (int64_t *)d_ts;
  p.row_val = (double *)d_val;
  p.row_n = (uint32_t *)d_n;
  p.rows_stride = rows;
  p.status = d_status;
  CK(launch_element_timer_consume(tp, st));
  m3tsz_encode_extras ex;
  memset(&ex, 0, sizeof(ex));
  ex.point_major_input = 1;
  EncodeParams ep;
  if (!encode_params(opts, p.row_ts, p.row_val, kn, rows, p.row_n, nullptr, out_unit, nullptr, nullptr, nullptr,
                     nullptr, nullptr, (int32_t *)d_rst, &ex, ep, true))
    return M3TSZ_ERR_INVALID_ARG;
  if (annotated) {  // (as element_set_consume)
    ep.ann_series_off = p.row_ann_off;
    ep.ann_entries = p.row_ann;
    ep.ann_bytes = p.ann_slot;
  }
  ep.out = set->d_out_buf;
  ep.out_stride = set->out_stride;
  ep.state = set->d_out_state;
  ep.n_appended = (uint32_t *)d_app;
  CK(launch_encode_append(ep, opts->int_optimized != 0, st));
  CK(launch_element_status((const int32_t *)d_rst, p.n, tp.n_types, d_status, st));
  ctx->launches += 3;
  return M3TSZ_OK;
}

int m3tsz_element_set_consume_timer(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                                    const m3tsz_element_timer_streams *streams, int64_t target_ns, int32_t out_unit,
                                    int32_t *d_status, void *stream) {
  return element_set_consume_timer(ctx, opts, set, streams, nullptr, target_ns, out_unit, d_status, stream, false);
}

int m3tsz_element_set_consume_timer_annotated(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                                              const m3tsz_element_timer_streams *streams,
                                              const m3tsz_element_annotations *ann, int64_t target_ns,
                                              int32_t out_unit, int32_t *d_status, void *stream) {
  return element_set_consume_timer(ctx, opts, set, streams, ann, target_ns, out_unit, d_status, stream, true);
}

// The forward calls' status arrays: present and aligned where there are sources / groups
static bool forward_statuses_ok(uint64_t S, uint64_t n_groups, const int32_t *d_src_status,
                                const int32_t *d_group_status) {
  return !((S && (!d_src_status || ((uintptr_t)d_src_status & 3u))) ||
           (n_groups && (!d_group_status || ((uintptr_t)d_group_status & 3u))));
}

// The forward calls' scratch (the forwarded windows, records and commit marks) and the rest of rp: the call's
// groups and the group set gp's slots
static int element_forward_scratch(m3tsz_ctx *ctx, ScratchFence &fence, ElementRollupParams &rp,
                                   const ElementParams &gp, int64_t target_ns, const uint64_t *d_group_off,
                                   const uint32_t *d_members, uint64_t n_members, uint64_t n_groups,
                                   int32_t *d_src_status, int32_t *d_group_status, int32_t discard_nan) {
  const uint64_t sn = rp.src.n ? rp.src.n : 1;  // (the fold reads nothing of the sources when there are none)
  void *d_fs, *d_fv, *d_fn, *d_fp, *d_fd, *d_rec, *d_mark;
  int rc;
  if ((rc = ensure(ctx, fence, kSlotElemFwdStart, (size_t)sn * rp.src.n_slots * 8, &d_fs))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemFwdVal, (size_t)sn * rp.src.n_slots * 8, &d_fv))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemFwdN, sn * 4, &d_fn))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemFwdPresent, sn * 8, &d_fp))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemFwdDue, sn * 8, &d_fd))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemFwdRec, sn * sizeof(m3tsz_transform_state), &d_rec))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemFwdMark, sn * 4, &d_mark))) return rc;
  rp.src.target = target_ns;
  rp.discard_nan = discard_nan ? 1 : 0;  // (generic_elem.go:892-894: with or without transformations)
  rp.fwd_start = (int64_t *)d_fs;
  rp.fwd_val = (double *)d_fv;
  rp.fwd_n = (uint32_t *)d_fn;
  rp.fwd_present = (uint64_t *)d_fp;
  rp.fwd_due = (uint64_t *)d_fd;
  rp.rec = (m3tsz_transform_state *)d_rec;
  rp.group_off = d_group_off;
  rp.members = d_members;
  rp.n_members = n_members;
  rp.n_groups = n_groups;
  rp.g_slots = gp.n_slots;
  rp.g_start = gp.start;
  rp.g_count = gp.count;
  rp.g_sum = gp.sum;
  rp.g_min = gp.min;
  rp.g_max = gp.max;
  rp.g_sum_sq = gp.sum_sq;
  rp.g_last = gp.last;
  rp.g_last_at = gp.last_at;
  rp.g_watermark = gp.watermark;
  rp.group_status = d_group_status;
  rp.mark = (int32_t *)d_mark;
  rp.src_status = d_src_status;
  return M3TSZ_OK;
}

// The annotated forward calls' annotation structs: both checked (element_ann_params) into the source and group set
// parameters, and the source and group arrays must not overlap (the fold copies source slot bytes into group slots)
static bool forward_ann_params(const m3tsz_element_annotations *src_ann, ElementParams &sp,
                               const m3tsz_element_annotations *group_ann, ElementParams &gp) {
  if (!element_ann_params(src_ann, sp) || !element_ann_params(group_ann, gp)) return false;
  auto overlap = [](const void *a, uint64_t na, const void *b, uint64_t nb) {
    return na && nb && (uintptr_t)a < (uintptr_t)b + nb && (uintptr_t)b < (uintptr_t)a + na;
  };
  const uint64_t sl = (uint64_t)sp.n_slots * sp.n, gl = (uint64_t)gp.n_slots * gp.n;
  const void *sa[2] = {sp.ann_len, sp.ann_slot}, *ga[2] = {gp.ann_len, gp.ann_slot};
  const uint64_t sb[2] = {sl * 4, sl * sp.ann_cap}, gb[2] = {gl * 4, gl * gp.ann_cap};
  for (int i = 0; i < 2; i++)
    for (int j = 0; j < 2; j++)
      if (overlap(sa[i], sb[i], ga[j], gb[j])) return false;
  return true;
}

// The annotated forward calls' scratch: which forwarded windows carry an annotation and their references; rp takes
// them and the group set gp's annotation arrays
static int forward_ann_scratch(m3tsz_ctx *ctx, ScratchFence &fence, ElementRollupParams &rp, const ElementParams &gp) {
  void *d_fap, *d_fa;
  const uint64_t sn = rp.src.n ? rp.src.n : 1;
  int rc;
  if ((rc = ensure(ctx, fence, kSlotElemFwdAnnPresent, sn * 8, &d_fap))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemFwdAnn, (size_t)sn * rp.src.n_slots * 8, &d_fa))) return rc;
  rp.fwd_ann_present = (uint64_t *)d_fap;
  rp.fwd_ann = (uint64_t *)d_fa;
  rp.g_ann_len = gp.ann_len;
  rp.g_ann_slot = gp.ann_slot;
  rp.g_ann_cap = gp.ann_cap;
  return M3TSZ_OK;
}

// The forward kernel writes each source's due windows to scratch, the fold kernel folds them into the groups' windows
// and marks the members of the groups that failed, and the commit kernel frees the other sources' due windows.
// m3tsz_element_set_forward(_annotated): annotated, the forward also writes which forwarded windows carry an
// annotation and their references, and the fold copies each group window's into its slot.
static int element_set_forward(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *src,
                               const m3tsz_element_annotations *src_ann, int64_t target_ns,
                               const uint64_t *d_group_off, const uint32_t *d_members, uint64_t n_members,
                               uint64_t n_groups, const m3tsz_element_set *groups,
                               const m3tsz_element_annotations *group_ann, int32_t *d_src_status,
                               int32_t *d_group_status, void *stream, bool annotated) {
  ElementRollupParams rp;
  memset(&rp, 0, sizeof(rp));
  ElementParams gp;
  TileTransforms sx, gx;
  if (!ctx || !element_params(opts, src, rp.src, sx) || !element_params(opts, groups, gp, gx)) return M3TSZ_ERR_INVALID_ARG;
  if (src->metric_type != groups->metric_type || src->resolution_ns != groups->resolution_ns || sx.n_types != 1 ||
      src->d_win_start == groups->d_win_start || n_groups != groups->n_elements || n_members > (1ull << 40) ||
      (n_groups && !d_group_off) || (n_members && !d_members) || ((uintptr_t)d_group_off & 7u) ||
      ((uintptr_t)d_members & 3u))
    return M3TSZ_ERR_INVALID_ARG;
  if (annotated && !forward_ann_params(src_ann, rp.src, group_ann, gp)) return M3TSZ_ERR_INVALID_ARG;
  if (!forward_statuses_ok(rp.src.n, n_groups, d_src_status, d_group_status)) return M3TSZ_ERR_INVALID_ARG;
  if (rp.src.n == 0 && n_groups == 0) return M3TSZ_OK;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  cudaStream_t st = (cudaStream_t)stream;
  ScratchFence fence(ctx, st);
  int rc = element_forward_scratch(ctx, fence, rp, gp, target_ns, d_group_off, d_members, n_members, n_groups,
                                   d_src_status, d_group_status, src->discard_nan);
  if (rc != M3TSZ_OK) return rc;
  if (annotated && (rc = forward_ann_scratch(ctx, fence, rp, gp)) != M3TSZ_OK) return rc;
  CK(cudaMemsetAsync(rp.mark, 0, (rp.src.n ? rp.src.n : 1) * 4, st));
  CK(launch_element_forward(rp, st));
  CK(launch_element_fold(rp, st));
  CK(launch_element_commit(rp, st));
  ctx->launches += 3;
  return M3TSZ_OK;
}

int m3tsz_element_set_forward(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *src,
                              int64_t target_ns, const uint64_t *d_group_off, const uint32_t *d_members,
                              uint64_t n_members, uint64_t n_groups, const m3tsz_element_set *groups,
                              int32_t *d_src_status, int32_t *d_group_status, void *stream) {
  return element_set_forward(ctx, opts, src, nullptr, target_ns, d_group_off, d_members, n_members, n_groups, groups,
                             nullptr, d_src_status, d_group_status, stream, false);
}

int m3tsz_element_set_forward_annotated(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *src,
                                        const m3tsz_element_annotations *src_ann, int64_t target_ns,
                                        const uint64_t *d_group_off, const uint32_t *d_members, uint64_t n_members,
                                        uint64_t n_groups, const m3tsz_element_set *groups,
                                        const m3tsz_element_annotations *group_ann, int32_t *d_src_status,
                                        int32_t *d_group_status, void *stream) {
  return element_set_forward(ctx, opts, src, src_ann, target_ns, d_group_off, d_members, n_members, n_groups, groups,
                             group_ann, d_src_status, d_group_status, stream, true);
}

// ---- element-set rollups across shards ----
// The forward kernel writes each source's due windows to scratch (element_forward_scratch, with no group set), the
// count pass counts each group's records and values, two scans place them, the write pass writes the groups that fit
// and marks the members of the others, and the commit kernel frees the other sources' due windows.
// m3tsz_element_set_forward_write(_timer): `timer` selects the source check (timer_params on src and src_streams, or
// element_params) and the source forward (element_timer_forward_kernel, or element_forward_kernel).
static int element_set_forward_write(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *src,
                                     const m3tsz_element_timer_streams *src_streams, int64_t target_ns,
                                     const uint64_t *d_group_off, const uint32_t *d_members, uint64_t n_members,
                                     uint64_t n_groups, const uint64_t *d_group_key, uint32_t source_id,
                                     m3tsz_forwarded_metric *d_metrics, uint64_t metric_capacity, double *d_values,
                                     uint64_t value_capacity, uint64_t *d_counts, int32_t *d_src_status,
                                     int32_t *d_group_status, void *stream, bool timer) {
  ElementForwardedParams fp;
  memset(&fp, 0, sizeof(fp));
  ElementRollupParams &rp = fp.rp;
  ElementTimerParams sp;
  TileTransforms sx;
  if (!ctx || !(timer ? timer_params(opts, src, src_streams, sp, sx) : element_params(opts, src, rp.src, sx)))
    return M3TSZ_ERR_INVALID_ARG;
  if (timer) rp.src = sp.e;
  if (sx.n_types != 1 || n_groups > (1ull << 40) || n_members > (1ull << 40) || metric_capacity > (1ull << 40) ||
      value_capacity > (1ull << 40) || (n_groups && !d_group_off) || (n_members && !d_members) ||
      ((uintptr_t)d_group_off & 7u) || ((uintptr_t)d_members & 3u) || ((uintptr_t)d_group_key & 7u) || !d_counts ||
      ((uintptr_t)d_counts & 7u) || (metric_capacity && (!d_metrics || ((uintptr_t)d_metrics & 7u))) ||
      (value_capacity && (!d_values || ((uintptr_t)d_values & 7u))))
    return M3TSZ_ERR_INVALID_ARG;
  if (!forward_statuses_ok(rp.src.n, n_groups, d_src_status, d_group_status)) return M3TSZ_ERR_INVALID_ARG;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  cudaStream_t st = (cudaStream_t)stream;
  CK(cudaMemsetAsync(d_counts, 0, 4 * 8, st));
  if (rp.src.n == 0 && n_groups == 0) return M3TSZ_OK;
  ScratchFence fence(ctx, st);
  ElementParams none;  // (no group set: the fold's fields stay unused)
  memset(&none, 0, sizeof(none));
  int rc = element_forward_scratch(ctx, fence, rp, none, target_ns, d_group_off, d_members, n_members, n_groups,
                                   d_src_status, d_group_status, src->discard_nan);
  if (rc != M3TSZ_OK) return rc;
  const uint64_t gn = n_groups ? n_groups : 1;
  void *d_nr, *d_nv, *d_ro, *d_vo, *d_tmp;
  size_t tmp_bytes = 0;
  CK(forward_write_scan(nullptr, tmp_bytes, nullptr, nullptr, gn, st));
  if ((rc = ensure(ctx, fence, kSlotElemFwdRecN, gn * 8, &d_nr))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemFwdValN, gn * 8, &d_nv))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemFwdRecOff, gn * 8, &d_ro))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemFwdValOff, gn * 8, &d_vo))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemFwdScanTmp, tmp_bytes ? tmp_bytes : 1, &d_tmp))) return rc;
  fp.group_key = d_group_key;
  fp.source_id = source_id;
  fp.out_rec = d_metrics;
  fp.out_val = d_values;
  fp.rec_cap = metric_capacity;
  fp.val_cap = value_capacity;
  fp.n_rec = (uint64_t *)d_nr;
  fp.n_val = (uint64_t *)d_nv;
  fp.rec_off = (uint64_t *)d_ro;
  fp.val_off = (uint64_t *)d_vo;
  fp.counts = d_counts;
  CK(cudaMemsetAsync(rp.mark, 0, (rp.src.n ? rp.src.n : 1) * 4, st));
  if (timer) {
    sp.e = rp.src;
    CK(launch_element_timer_forward(rp, sp, st));
  } else {
    CK(launch_element_forward(rp, st));
  }
  CK(launch_forward_write_count(fp, st));
  if (n_groups) {
    CK(forward_write_scan(d_tmp, tmp_bytes, fp.n_rec, fp.rec_off, n_groups, st));
    CK(forward_write_scan(d_tmp, tmp_bytes, fp.n_val, fp.val_off, n_groups, st));
  }
  CK(launch_forward_write(fp, st));
  CK(launch_element_commit(rp, st));
  ctx->launches += 6;
  return M3TSZ_OK;
}

int m3tsz_element_set_forward_write(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *src,
                                    int64_t target_ns, const uint64_t *d_group_off, const uint32_t *d_members,
                                    uint64_t n_members, uint64_t n_groups, const uint64_t *d_group_key,
                                    uint32_t source_id, m3tsz_forwarded_metric *d_metrics, uint64_t metric_capacity,
                                    double *d_values, uint64_t value_capacity, uint64_t *d_counts,
                                    int32_t *d_src_status, int32_t *d_group_status, void *stream) {
  return element_set_forward_write(ctx, opts, src, nullptr, target_ns, d_group_off, d_members, n_members, n_groups,
                                   d_group_key, source_id, d_metrics, metric_capacity, d_values, value_capacity,
                                   d_counts, d_src_status, d_group_status, stream, false);
}

int m3tsz_element_set_forward_write_timer(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *src,
                                          const m3tsz_element_timer_streams *src_streams, int64_t target_ns,
                                          const uint64_t *d_group_off, const uint32_t *d_members, uint64_t n_members,
                                          uint64_t n_groups, const uint64_t *d_group_key, uint32_t source_id,
                                          m3tsz_forwarded_metric *d_metrics, uint64_t metric_capacity,
                                          double *d_values, uint64_t value_capacity, uint64_t *d_counts,
                                          int32_t *d_src_status, int32_t *d_group_status, void *stream) {
  return element_set_forward_write(ctx, opts, src, src_streams, target_ns, d_group_off, d_members, n_members,
                                   n_groups, d_group_key, source_id, d_metrics, metric_capacity, d_values,
                                   value_capacity, d_counts, d_src_status, d_group_status, stream, true);
}

// The prep kernel writes each record's element key and index, the radix sort orders them by key (stable, so each
// element's records stay in array order), and one lane per element takes its records.
// m3tsz_element_set_add_forwarded(_timer): `timer` selects the set check (timer_params on set and set_streams, or
// element_params) and the lane (add_forwarded_timer_kernel, or add_forwarded_kernel).
static int element_set_add_forwarded(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                                     const m3tsz_element_timer_streams *set_streams,
                                     const m3tsz_element_sources *sources, const m3tsz_forwarded_metric *d_metrics,
                                     uint64_t n_metrics, const double *d_values, uint64_t n_values, int8_t *d_result,
                                     int32_t *d_status, void *stream, bool timer) {
  ElementForwardedParams fp;
  memset(&fp, 0, sizeof(fp));
  ElementTimerParams gt;
  ElementParams &gp = gt.e;
  TileTransforms gx;
  if (!ctx || !(timer ? timer_params(opts, set, set_streams, gt, gx) : element_params(opts, set, gp, gx)))
    return M3TSZ_ERR_INVALID_ARG;
  if (!sources || sources->reserved != 0 || sources->capacity == 0 || (sources->capacity & 31u) ||
      sources->capacity > M3TSZ_MAX_FORWARD_SOURCES || !sources->d_bits || ((uintptr_t)sources->d_bits & 3u) ||
      n_metrics > (1ull << 40) || n_values > (1ull << 40) || (n_metrics && (!d_metrics || !d_result)) ||
      ((uintptr_t)d_metrics & 7u) || (n_values && !d_values) || ((uintptr_t)d_values & 7u) ||
      (gp.n && (!d_status || ((uintptr_t)d_status & 3u))))
    return M3TSZ_ERR_INVALID_ARG;
  if (gp.n == 0 && n_metrics == 0) return M3TSZ_OK;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  cudaStream_t st = (cudaStream_t)stream;
  if (gp.n) CK(cudaMemsetAsync(d_status, 0, gp.n * 4, st));
  if (n_metrics == 0) return M3TSZ_OK;
  ScratchFence fence(ctx, st);
  int end_bit = 1;  // the key bits: elements 0 .. n - 1, and n for an invalid key
  while (end_bit < 64 && (gp.n >> end_bit) != 0) end_bit++;
  size_t tmp_bytes = 0;
  CK(add_forwarded_sort(nullptr, tmp_bytes, nullptr, nullptr, nullptr, nullptr, n_metrics, end_bit, st));
  void *d_k, *d_i, *d_sk, *d_si, *d_tmp;
  int rc;
  if ((rc = ensure(ctx, fence, kSlotElemAddFwdKey, n_metrics * 8, &d_k))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemAddFwdIdx, n_metrics * 8, &d_i))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemAddFwdSortedKey, n_metrics * 8, &d_sk))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemAddFwdSortedIdx, n_metrics * 8, &d_si))) return rc;
  if ((rc = ensure(ctx, fence, kSlotElemAddFwdSortTmp, tmp_bytes ? tmp_bytes : 1, &d_tmp))) return rc;
  ElementRollupParams &rp = fp.rp;
  rp.src.n = gp.n;
  rp.src.counter = gp.counter;
  rp.src.resolution = gp.resolution;
  rp.n_groups = gp.n;
  rp.g_slots = gp.n_slots;
  rp.g_start = gp.start;
  rp.g_count = gp.count;
  rp.g_sum = gp.sum;
  rp.g_min = gp.min;
  rp.g_max = gp.max;
  rp.g_sum_sq = gp.sum_sq;
  rp.g_last = gp.last;
  rp.g_last_at = gp.last_at;
  rp.g_watermark = gp.watermark;
  fp.rec = d_metrics;
  fp.val = d_values;
  fp.n_recs = n_metrics;
  fp.n_vals = n_values;
  fp.sort_key = (uint64_t *)d_k;
  fp.sort_idx = (uint64_t *)d_i;
  fp.sorted_key = (const uint64_t *)d_sk;
  fp.sorted_idx = (const uint64_t *)d_si;
  fp.bits = sources->d_bits;
  fp.bit_words = sources->capacity / 32u;
  fp.trunc_off = gp.trunc_off;
  fp.result = d_result;
  fp.status = d_status;
  CK(launch_add_forwarded_prep(fp, st));
  CK(add_forwarded_sort(d_tmp, tmp_bytes, fp.sort_key, (uint64_t *)d_sk, fp.sort_idx, (uint64_t *)d_si, n_metrics,
                        end_bit, st));
  CK(timer ? launch_add_forwarded_timer(fp, gt, st) : launch_add_forwarded(fp, st));
  ctx->launches += 3;
  return M3TSZ_OK;
}

int m3tsz_element_set_add_forwarded(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                                    const m3tsz_element_sources *sources, const m3tsz_forwarded_metric *d_metrics,
                                    uint64_t n_metrics, const double *d_values, uint64_t n_values, int8_t *d_result,
                                    int32_t *d_status, void *stream) {
  return element_set_add_forwarded(ctx, opts, set, nullptr, sources, d_metrics, n_metrics, d_values, n_values,
                                   d_result, d_status, stream, false);
}

int m3tsz_element_set_add_forwarded_timer(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                                          const m3tsz_element_timer_streams *set_streams,
                                          const m3tsz_element_sources *sources,
                                          const m3tsz_forwarded_metric *d_metrics, uint64_t n_metrics,
                                          const double *d_values, uint64_t n_values, int8_t *d_result,
                                          int32_t *d_status, void *stream) {
  return element_set_add_forwarded(ctx, opts, set, set_streams, sources, d_metrics, n_metrics, d_values, n_values,
                                   d_result, d_status, stream, true);
}

// element_set_forward with the Timer forward and fold kernels: the same groups, scratch, annotation scratch and
// commit.  m3tsz_element_set_forward_timer(_annotated): src_ann / group_ann NULL is the plain forward
static int element_set_forward_timer(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *src,
                                     const m3tsz_element_timer_streams *src_streams,
                                     const m3tsz_element_annotations *src_ann, int64_t target_ns,
                                     const uint64_t *d_group_off, const uint32_t *d_members, uint64_t n_members,
                                     uint64_t n_groups, const m3tsz_element_set *groups,
                                     const m3tsz_element_timer_streams *group_streams,
                                     const m3tsz_element_annotations *group_ann, int32_t *d_src_status,
                                     int32_t *d_group_status, void *stream, bool annotated) {
  ElementTimerParams sp, gt;
  TileTransforms sx, gx;
  if (!ctx || !timer_params(opts, src, src_streams, sp, sx) || !timer_params(opts, groups, group_streams, gt, gx))
    return M3TSZ_ERR_INVALID_ARG;
  if (src->resolution_ns != groups->resolution_ns || sx.n_types != 1 || n_groups != groups->n_elements ||
      n_members > (1ull << 40) || (n_groups && !d_group_off) || (n_members && !d_members) ||
      ((uintptr_t)d_group_off & 7u) || ((uintptr_t)d_members & 3u))
    return M3TSZ_ERR_INVALID_ARG;
  // the two sets share no slot or stream array: the forward rewrites the source streams and the fold the group ones
  const uint64_t sl = (uint64_t)sp.e.n_slots * sp.e.n, gl = (uint64_t)gt.e.n_slots * gt.e.n;
  const uint64_t se = sl * sp.cap, ge = gl * gt.cap;
  const void *sa[] = {sp.e.start, sp.e.count, sp.e.sum, sp.e.sum_sq, sp.hdr, sp.value, sp.num_ranks, sp.delta,
                      sp.prev, sp.next, sp.heap_a, sp.heap_b};
  const void *ga[] = {gt.e.start, gt.e.count, gt.e.sum, gt.e.sum_sq, gt.hdr, gt.value, gt.num_ranks, gt.delta,
                      gt.prev, gt.next, gt.heap_a, gt.heap_b};
  const uint64_t sb[] = {sl * 8, sl * 8, sl * 8, sl * 8, sl * 64, se * 8, se * 8, se * 8, se * 4, se * 4, se * 8, se * 8};
  const uint64_t gb[] = {gl * 8, gl * 8, gl * 8, gl * 8, gl * 64, ge * 8, ge * 8, ge * 8, ge * 4, ge * 4, ge * 8, ge * 8};
  for (int i = 0; i < 12; i++)
    for (int j = 0; j < 12; j++)
      if (sb[i] && gb[j] && (uintptr_t)sa[i] < (uintptr_t)ga[j] + gb[j] && (uintptr_t)ga[j] < (uintptr_t)sa[i] + sb[i])
        return M3TSZ_ERR_INVALID_ARG;
  if (annotated && !forward_ann_params(src_ann, sp.e, group_ann, gt.e)) return M3TSZ_ERR_INVALID_ARG;
  if (!forward_statuses_ok(sp.e.n, n_groups, d_src_status, d_group_status)) return M3TSZ_ERR_INVALID_ARG;
  if (sp.e.n == 0 && n_groups == 0) return M3TSZ_OK;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  cudaStream_t st = (cudaStream_t)stream;
  ScratchFence fence(ctx, st);
  ElementRollupParams rp;
  memset(&rp, 0, sizeof(rp));
  rp.src = sp.e;
  int rc = element_forward_scratch(ctx, fence, rp, gt.e, target_ns, d_group_off, d_members, n_members, n_groups,
                                   d_src_status, d_group_status, src->discard_nan);
  if (rc != M3TSZ_OK) return rc;
  if (annotated && (rc = forward_ann_scratch(ctx, fence, rp, gt.e)) != M3TSZ_OK) return rc;
  sp.e = rp.src;
  CK(cudaMemsetAsync(rp.mark, 0, (rp.src.n ? rp.src.n : 1) * 4, st));
  CK(launch_element_timer_forward(rp, sp, st));
  CK(launch_element_timer_fold(rp, gt, st));
  CK(launch_element_commit(rp, st));
  ctx->launches += 3;
  return M3TSZ_OK;
}

int m3tsz_element_set_forward_timer(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *src,
                                    const m3tsz_element_timer_streams *src_streams, int64_t target_ns,
                                    const uint64_t *d_group_off, const uint32_t *d_members, uint64_t n_members,
                                    uint64_t n_groups, const m3tsz_element_set *groups,
                                    const m3tsz_element_timer_streams *group_streams, int32_t *d_src_status,
                                    int32_t *d_group_status, void *stream) {
  return element_set_forward_timer(ctx, opts, src, src_streams, nullptr, target_ns, d_group_off, d_members,
                                   n_members, n_groups, groups, group_streams, nullptr, d_src_status, d_group_status,
                                   stream, false);
}

int m3tsz_element_set_forward_timer_annotated(
    m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *src,
    const m3tsz_element_timer_streams *src_streams, const m3tsz_element_annotations *src_ann, int64_t target_ns,
    const uint64_t *d_group_off, const uint32_t *d_members, uint64_t n_members, uint64_t n_groups,
    const m3tsz_element_set *groups, const m3tsz_element_timer_streams *group_streams,
    const m3tsz_element_annotations *group_ann, int32_t *d_src_status, int32_t *d_group_status, void *stream) {
  return element_set_forward_timer(ctx, opts, src, src_streams, src_ann, target_ns, d_group_off, d_members,
                                   n_members, n_groups, groups, group_streams, group_ann, d_src_status,
                                   d_group_status, stream, true);
}

int m3tsz_merge_series_batch_ex(m3tsz_ctx *ctx, const int64_t *d_ts, const double *d_val, uint64_t cap,
                                const uint32_t *d_n_points, const int32_t *d_seq_status,
                                const uint64_t *d_slice_off, const uint64_t *d_replica_off,
                                const uint64_t *d_series_off, uint64_t n_series, int64_t start_ns,
                                int64_t end_ns, int32_t strategy, int64_t *d_ts_out, double *d_val_out,
                                uint64_t out_cap, uint32_t *d_n_out, int32_t *d_status, uint64_t n_seq,
                                int32_t point_major_in, int32_t point_major_out, void *stream) {
  if (!ctx) return M3TSZ_ERR_INVALID_ARG;
  if (n_series == 0) return M3TSZ_OK;
  if (!d_ts || !d_val || !d_n_points || !d_slice_off || !d_replica_off || !d_series_off || !d_ts_out ||
      !d_val_out || !d_n_out || !d_status || cap == 0 || out_cap == 0 || out_cap > 0xffffffffull ||
      strategy < 0 || strategy > 3)
    return M3TSZ_ERR_INVALID_ARG;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  MergeParams p;
  memset(&p, 0, sizeof(p));
  p.ts = d_ts;
  p.val = d_val;
  p.cap = cap;
  p.n_points = d_n_points;
  p.seq_status = d_seq_status;
  p.slice_off = d_slice_off;
  p.replica_off = d_replica_off;
  p.series_off = d_series_off;
  p.n_series = n_series;
  p.start = start_ns;
  p.end = end_ns;
  p.strategy = strategy;
  p.ts_out = d_ts_out;
  p.val_out = d_val_out;
  p.out_cap = out_cap;
  p.n_out = d_n_out;
  p.status = d_status;
  if (point_major_in && n_seq == 0) return M3TSZ_ERR_INVALID_ARG;
  p.in_seq_stride = point_major_in ? 1 : cap;
  p.in_pt_stride = point_major_in ? n_seq : 1;
  p.out_seq_stride = point_major_out ? 1 : out_cap;
  p.out_pt_stride = point_major_out ? n_series : 1;
  CK(launch_merge(p, (cudaStream_t)stream));
  ctx->launches++;
  return M3TSZ_OK;
}

int m3tsz_merge_series_batch(m3tsz_ctx *ctx, const int64_t *d_ts, const double *d_val, uint64_t cap,
                             const uint32_t *d_n_points, const int32_t *d_seq_status,
                             const uint64_t *d_slice_off, const uint64_t *d_replica_off,
                             const uint64_t *d_series_off, uint64_t n_series, int64_t start_ns,
                             int64_t end_ns, int32_t strategy, int64_t *d_ts_out, double *d_val_out,
                             uint64_t out_cap, uint32_t *d_n_out, int32_t *d_status, void *stream) {
  return m3tsz_merge_series_batch_ex(ctx, d_ts, d_val, cap, d_n_points, d_seq_status, d_slice_off, d_replica_off,
                                     d_series_off, n_series, start_ns, end_ns, strategy, d_ts_out, d_val_out,
                                     out_cap, d_n_out, d_status, 0, 0, 0, stream);
}

int m3tsz_checksum_batch(m3tsz_ctx *ctx, const uint8_t *d_streams, uint64_t streams_bytes,
                         const uint64_t *d_offsets, const uint64_t *d_lengths, uint64_t n_series,
                         const uint32_t *d_expected, uint32_t *d_checksums, int32_t *d_status,
                         void *stream) {
  if (!ctx) return M3TSZ_ERR_INVALID_ARG;
  if (n_series == 0) return M3TSZ_OK;
  if (!d_streams || !d_offsets || (!d_checksums && !d_status) || (d_expected && !d_status))
    return M3TSZ_ERR_INVALID_ARG;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  ChecksumParams p;
  memset(&p, 0, sizeof(p));
  p.streams = d_streams;
  p.streams_bytes = streams_bytes;
  p.offsets = d_offsets;
  p.lengths = d_lengths;
  p.n_series = n_series;
  p.expected = d_expected;
  p.out = d_checksums;
  p.status = d_status;
  CK(launch_checksum(p, (cudaStream_t)stream));
  ctx->launches++;
  return M3TSZ_OK;
}

// --------------------------------------------------------------------------
// host-buffer variants
// --------------------------------------------------------------------------
int m3tsz_decode_batch_host(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *h_streams,
                            uint64_t streams_bytes, const uint64_t *h_offsets, uint64_t n_series,
                            int64_t *h_ts, double *h_val, uint64_t max_points,
                            uint32_t *h_n_points, int32_t *h_status, uint8_t *h_unit,
                            m3tsz_annotation_ref *h_ann) {
  if (!ctx || !valid_opts(opts)) return M3TSZ_ERR_INVALID_ARG;
  if (n_series == 0) return M3TSZ_OK;
  if (!h_streams || !h_offsets || !h_ts || !h_val || max_points == 0) return M3TSZ_ERR_INVALID_ARG;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  ScratchFence fence(ctx);  // (after earlier device calls on this context, whatever their streams)
  DrainStreams drain{ctx};
  void *d_streams, *d_off, *d_ts, *d_val, *d_n, *d_st, *d_unit = nullptr, *d_ann = nullptr;
  int rc;
  if ((rc = ensure(ctx, fence, kSlotStreams, streams_bytes + 16, &d_streams))) return rc;
  if ((rc = ensure(ctx, fence, kSlotSeriesIndex, (n_series + 1) * 8, &d_off))) return rc;
  if ((rc = ensure(ctx, fence, kSlotTs, n_series * max_points * 8, &d_ts))) return rc;
  if ((rc = ensure(ctx, fence, kSlotVal, n_series * max_points * 8, &d_val))) return rc;
  if ((rc = ensure(ctx, fence, kSlotNPoints, n_series * 4, &d_n))) return rc;
  if ((rc = ensure(ctx, fence, kSlotStatus, n_series * 4, &d_st))) return rc;
  if (h_unit && (rc = ensure(ctx, fence, kSlotUnit, n_series, &d_unit))) return rc;
  if (h_ann && (rc = ensure(ctx, fence, kSlotAnnRefs, n_series * sizeof(m3tsz_annotation_ref), &d_ann))) return rc;
  // Chunked pipeline over two streams: the H2D copy of chunk c+1 overlaps the
  // kernel and the D2H copy of chunk c (PCIe is full duplex).
  cudaStream_t sts[2] = {ctx->stream, ctx->stream2};
  CK(cudaMemcpyAsync(d_off, h_offsets, (n_series + 1) * 8, cudaMemcpyHostToDevice, sts[0]));
  CK(cudaEventRecord(ctx->ev, sts[0]));
  CK(cudaStreamWaitEvent(sts[1], ctx->ev, 0));
  const uint64_t per_series = streams_bytes / n_series + max_points * 16;
  const uint64_t ch = pick_chunk(n_series, per_series);
  int k = 0;
  for (uint64_t c0 = 0; c0 < n_series; c0 += ch, k++) {
    const uint64_t c1 = (c0 + ch < n_series) ? c0 + ch : n_series, n = c1 - c0;
    cudaStream_t st = sts[k & 1];
    const uint64_t b0 = h_offsets[c0], b1 = h_offsets[c1];
    if (b1 < b0 || b1 > streams_bytes) return M3TSZ_ERR_INVALID_ARG;
    if (b1 > b0)
      CK(cudaMemcpyAsync((uint8_t *)d_streams + b0, h_streams + b0, b1 - b0, cudaMemcpyHostToDevice, st));
    rc = m3tsz_decode_batch(ctx, opts, (const uint8_t *)d_streams, streams_bytes,
                            (const uint64_t *)d_off + c0, n, (int64_t *)d_ts + c0 * max_points,
                            (double *)d_val + c0 * max_points, max_points, (uint32_t *)d_n + c0,
                            (int32_t *)d_st + c0, d_unit ? (uint8_t *)d_unit + c0 : nullptr,
                            d_ann ? (m3tsz_annotation_ref *)d_ann + c0 : nullptr, st);
    if (rc) return rc;
    CK(cudaMemcpyAsync(h_ts + c0 * max_points, (int64_t *)d_ts + c0 * max_points, n * max_points * 8,
                       cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(h_val + c0 * max_points, (double *)d_val + c0 * max_points, n * max_points * 8,
                       cudaMemcpyDeviceToHost, st));
    if (h_n_points) CK(cudaMemcpyAsync(h_n_points + c0, (uint32_t *)d_n + c0, n * 4, cudaMemcpyDeviceToHost, st));
    if (h_status) CK(cudaMemcpyAsync(h_status + c0, (int32_t *)d_st + c0, n * 4, cudaMemcpyDeviceToHost, st));
    if (h_unit) CK(cudaMemcpyAsync(h_unit + c0, (uint8_t *)d_unit + c0, n, cudaMemcpyDeviceToHost, st));
    if (h_ann)
      CK(cudaMemcpyAsync(h_ann + c0, (m3tsz_annotation_ref *)d_ann + c0, n * sizeof(m3tsz_annotation_ref),
                         cudaMemcpyDeviceToHost, st));
  }
  CK(cudaStreamSynchronize(sts[0]));
  CK(cudaStreamSynchronize(sts[1]));
  return M3TSZ_OK;
}

int m3tsz_decode_downsample_batch_host(m3tsz_ctx *ctx, const m3tsz_options *opts,
                                       const uint8_t *h_streams, uint64_t streams_bytes,
                                       const uint64_t *h_offsets, uint64_t n_series,
                                       int64_t range_start_ns, int64_t window_ns,
                                       uint32_t n_windows, double *h_sum, int64_t *h_count,
                                       double *h_min, double *h_max, uint32_t *h_n_points,
                                       int32_t *h_status) {
  if (!ctx || !valid_opts(opts)) return M3TSZ_ERR_INVALID_ARG;
  if (n_series == 0) return M3TSZ_OK;
  if (!h_streams || !h_offsets || !h_sum || !h_count || !h_min || !h_max) return M3TSZ_ERR_INVALID_ARG;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  ScratchFence fence(ctx);  // (after earlier device calls on this context, whatever their streams)
  DrainStreams drain{ctx};
  cudaStream_t st = ctx->stream;
  const size_t wb = (size_t)n_series * n_windows * 8;
  void *d_streams, *d_off, *d_sum, *d_cnt, *d_min, *d_max, *d_n, *d_st;
  int rc;
  if ((rc = ensure(ctx, fence, kSlotStreams, streams_bytes + 16, &d_streams))) return rc;
  if ((rc = ensure(ctx, fence, kSlotSeriesIndex, (n_series + 1) * 8, &d_off))) return rc;
  if ((rc = ensure(ctx, fence, kSlotWinSum, wb, &d_sum))) return rc;
  if ((rc = ensure(ctx, fence, kSlotWinCount, wb, &d_cnt))) return rc;
  if ((rc = ensure(ctx, fence, kSlotWinMin, wb, &d_min))) return rc;
  if ((rc = ensure(ctx, fence, kSlotWinMax, wb, &d_max))) return rc;
  if ((rc = ensure(ctx, fence, kSlotNPoints, n_series * 4, &d_n))) return rc;
  if ((rc = ensure(ctx, fence, kSlotStatus, n_series * 4, &d_st))) return rc;
  CK(cudaMemcpyAsync(d_streams, h_streams, streams_bytes, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_off, h_offsets, (n_series + 1) * 8, cudaMemcpyHostToDevice, st));
  rc = m3tsz_decode_downsample_batch(ctx, opts, (const uint8_t *)d_streams, streams_bytes,
                                     (const uint64_t *)d_off, n_series, range_start_ns, window_ns,
                                     n_windows, (double *)d_sum, (int64_t *)d_cnt, (double *)d_min,
                                     (double *)d_max, (uint32_t *)d_n, (int32_t *)d_st, st);
  if (rc) return rc;
  CK(cudaMemcpyAsync(h_sum, d_sum, wb, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(h_count, d_cnt, wb, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(h_min, d_min, wb, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(h_max, d_max, wb, cudaMemcpyDeviceToHost, st));
  if (h_n_points) CK(cudaMemcpyAsync(h_n_points, d_n, n_series * 4, cudaMemcpyDeviceToHost, st));
  if (h_status) CK(cudaMemcpyAsync(h_status, d_st, n_series * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return M3TSZ_OK;
}

int m3tsz_encode_batch_host(m3tsz_ctx *ctx, const m3tsz_options *opts, const int64_t *h_ts,
                            const double *h_val, uint64_t n_series, uint64_t points_stride,
                            const uint32_t *h_n_points, const int64_t *h_start, int32_t unit,
                            const uint8_t *h_units, const uint64_t *h_ann_series_off,
                            const m3tsz_annotation_entry *h_ann_entries,
                            const uint8_t *h_ann_bytes, uint64_t ann_bytes_len, uint32_t align,
                            uint8_t *h_packed, uint64_t packed_capacity, uint64_t *h_offsets,
                            uint64_t *h_out_len, int32_t *h_status) {
  if (!ctx || !valid_opts(opts)) return M3TSZ_ERR_INVALID_ARG;
  if (!h_offsets) return M3TSZ_ERR_INVALID_ARG;
  h_offsets[0] = 0;
  if (n_series == 0) return M3TSZ_OK;
  if (!h_ts || !h_val || !h_start || !h_packed) return M3TSZ_ERR_INVALID_ARG;
  if (!valid_align(align)) return M3TSZ_ERR_INVALID_ARG;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  ScratchFence fence(ctx);  // (after earlier device calls on this context, whatever their streams)
  DrainStreams drain{ctx};
  cudaStream_t sts[2] = {ctx->stream, ctx->stream2};
  const uint64_t ann_total = h_ann_series_off ? ann_bytes_len + 16 * h_ann_series_off[n_series] : 0;
  const uint64_t out_stride = m3tsz_encode_bound_units(points_stride, h_units != nullptr) + ((ann_total + 15) & ~15ull);
  const uint64_t ch = pick_chunk(n_series, points_stride * 16 + points_stride * 8);
  const size_t row_bytes = (size_t)points_stride * 8;
  int rc;
  // whole-batch device inputs that are small: start, n_points, annotations
  void *d_start, *d_np = nullptr, *d_aoff = nullptr, *d_aent = nullptr, *d_abytes = nullptr;
  if ((rc = ensure(ctx, fence, kSlotSeriesIndex, (n_series + 1) * 8, &d_start))) return rc;
  CK(cudaMemcpyAsync(d_start, h_start, n_series * 8, cudaMemcpyHostToDevice, sts[0]));
  if (h_n_points) {
    if ((rc = ensure(ctx, fence, kSlotNPoints, n_series * 4, &d_np))) return rc;
    CK(cudaMemcpyAsync(d_np, h_n_points, n_series * 4, cudaMemcpyHostToDevice, sts[0]));
  }
  if (h_ann_series_off) {
    if (!h_ann_entries || (!h_ann_bytes && ann_bytes_len)) return M3TSZ_ERR_INVALID_ARG;
    const uint64_t n_ent = h_ann_series_off[n_series];
    if ((rc = ensure(ctx, fence, kSlotAnnSeriesOff, (n_series + 1) * 8, &d_aoff))) return rc;
    if ((rc = ensure(ctx, fence, kSlotAnnEntries, n_ent * sizeof(m3tsz_annotation_entry), &d_aent))) return rc;
    if ((rc = ensure(ctx, fence, kSlotAnnBytes, ann_bytes_len, &d_abytes))) return rc;
    CK(cudaMemcpyAsync(d_aoff, h_ann_series_off, (n_series + 1) * 8, cudaMemcpyHostToDevice, sts[0]));
    if (n_ent)
      CK(cudaMemcpyAsync(d_aent, h_ann_entries, n_ent * sizeof(m3tsz_annotation_entry),
                         cudaMemcpyHostToDevice, sts[0]));
    if (ann_bytes_len) CK(cudaMemcpyAsync(d_abytes, h_ann_bytes, ann_bytes_len, cudaMemcpyHostToDevice, sts[0]));
  }
  CK(cudaEventRecord(ctx->ev, sts[0]));
  CK(cudaStreamWaitEvent(sts[1], ctx->ev, 0));

  // per-stream chunk buffers
  struct Lane {
    void *ts, *val, *units, *out, *len, *st, *packed, *off, *tmp;
    uint64_t c0, c1;
    bool busy;
  } ln[2];
  const size_t tmp_bytes = compact_scan_tmp_bytes(ch);
  // every start is rounded up to `align`: budget the aligned worst case per stream
  const uint64_t packed_stride = (out_stride + align - 1) & ~(uint64_t)(align - 1);
  for (int i = 0; i < 2; i++) {
    ln[i].units = nullptr;
    ln[i].busy = false;
    if ((rc = ensure(ctx, fence, lane_slot(i, 0), ch * row_bytes, &ln[i].ts))) return rc;
    if ((rc = ensure(ctx, fence, lane_slot(i, 1), ch * row_bytes, &ln[i].val))) return rc;
    if (h_units && (rc = ensure(ctx, fence, lane_slot(i, 2), ch * points_stride, &ln[i].units))) return rc;
    if ((rc = ensure(ctx, fence, lane_slot(i, 3), ch * out_stride, &ln[i].out))) return rc;
    if ((rc = ensure(ctx, fence, lane_slot(i, 4), ch * 8, &ln[i].len))) return rc;
    if ((rc = ensure(ctx, fence, lane_slot(i, 5), ch * 4, &ln[i].st))) return rc;
    if ((rc = ensure(ctx, fence, lane_slot(i, 6), ch * packed_stride + 64, &ln[i].packed))) return rc;
    if ((rc = ensure(ctx, fence, lane_slot(i, 7), (ch + 1) * 8, &ln[i].off))) return rc;
    if ((rc = ensure(ctx, fence, lane_slot(i, 8), tmp_bytes, &ln[i].tmp))) return rc;
    if ((rc = ensure_stage(ctx, i, (ch + 1) * 8 + 8))) return rc;
  }
  CK(cudaMemsetAsync(ctx->d_flag, 0, 2 * sizeof(int32_t), sts[0]));
  CK(cudaStreamSynchronize(sts[0]));  // the flags are zero before either lane's kernels can set them

  auto issue = [&](int i, uint64_t c0) -> int {
    Lane &L = ln[i];
    cudaStream_t st = sts[i];
    L.c0 = c0;
    L.c1 = (c0 + ch < n_series) ? c0 + ch : n_series;
    L.busy = true;
    const uint64_t n = L.c1 - c0;
    CK(cudaMemcpyAsync(L.ts, h_ts + c0 * points_stride, n * row_bytes, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(L.val, h_val + c0 * points_stride, n * row_bytes, cudaMemcpyHostToDevice, st));
    if (h_units)
      CK(cudaMemcpyAsync(L.units, h_units + c0 * points_stride, n * points_stride, cudaMemcpyHostToDevice, st));
    int r = m3tsz_encode_batch(ctx, opts, (const int64_t *)L.ts, (const double *)L.val, n, points_stride,
                               d_np ? (const uint32_t *)d_np + c0 : nullptr, (const int64_t *)d_start + c0,
                               unit, (const uint8_t *)L.units, d_aoff ? (const uint64_t *)d_aoff + c0 : nullptr,
                               (const m3tsz_annotation_entry *)d_aent, (const uint8_t *)d_abytes,
                               (uint8_t *)L.out, out_stride, (uint64_t *)L.len, (int32_t *)L.st, st);
    if (r) return r;
    CK(launch_compact((const uint8_t *)L.out, out_stride, (const uint64_t *)L.len, n, align,
                      (uint8_t *)L.packed, ch * packed_stride + 64, (uint64_t *)L.off, L.tmp, tmp_bytes,
                      ctx->d_flag + i, st));
    ctx->launches += 3;
    CK(cudaMemcpyAsync(ctx->h_stage[i], L.off, (n + 1) * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync((uint8_t *)ctx->h_stage[i] + (ch + 1) * 8, ctx->d_flag + i, 4, cudaMemcpyDeviceToHost, st));
    if (h_out_len) CK(cudaMemcpyAsync(h_out_len + c0, L.len, n * 8, cudaMemcpyDeviceToHost, st));
    if (h_status) CK(cudaMemcpyAsync(h_status + c0, L.st, n * 4, cudaMemcpyDeviceToHost, st));
    return M3TSZ_OK;
  };
  uint64_t host_base = 0;
  auto finish = [&](int i) -> int {
    Lane &L = ln[i];
    if (!L.busy) return M3TSZ_OK;
    L.busy = false;
    CK(cudaStreamSynchronize(sts[i]));  // offsets of this chunk are on the host now
    const uint64_t n = L.c1 - L.c0;
    const uint64_t *co = (const uint64_t *)ctx->h_stage[i];
    const uint64_t total = co[n];
    int32_t overflow = 0;
    memcpy(&overflow, (const uint8_t *)ctx->h_stage[i] + (ch + 1) * 8, 4);
    if (overflow || host_base + total > packed_capacity) return M3TSZ_ERR_CAPACITY;
    if (total)
      CK(cudaMemcpyAsync(h_packed + host_base, L.packed, total, cudaMemcpyDeviceToHost, sts[i]));
    for (uint64_t j = 0; j <= n; j++) h_offsets[L.c0 + j] = host_base + co[j];
    host_base += total;
    host_base = (host_base + align - 1) & ~(uint64_t)(align - 1);
    return M3TSZ_OK;
  };
  int k = 0;
  if ((rc = issue(0, 0))) return rc;
  for (uint64_t c0 = 0; c0 < n_series; c0 += ch, k++) {
    const uint64_t next = c0 + ch;
    if (next < n_series) {
      // the other lane's previous chunk has been finished already (its D2H is queued
      // on its own stream, so reusing its buffers is ordered)
      if ((rc = issue((k + 1) & 1, next))) return rc;
    }
    if ((rc = finish(k & 1))) return rc;
  }
  CK(cudaStreamSynchronize(sts[0]));
  CK(cudaStreamSynchronize(sts[1]));
  // CSR convention: offsets[n] is the end of the last stream; un-pad the final alignment
  return M3TSZ_OK;
}


// --------------------------------------------------------------------------
// Fetch path with host buffers: only compressed bytes go up, only the merged result
// comes back (the decoded replicas never cross PCIe).
int m3tsz_fetch_batch_host(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *h_streams,
                           uint64_t streams_bytes, const uint64_t *h_offsets, uint64_t n_seq,
                           const uint64_t *h_slice_off, const uint64_t *h_replica_off,
                           const uint64_t *h_series_off, uint64_t n_series, uint64_t max_points,
                           int64_t start_ns, int64_t end_ns, int32_t strategy, int64_t *h_ts_out,
                           double *h_val_out, uint64_t out_cap, uint32_t *h_n_out, int32_t *h_status) {
  if (!ctx || !valid_opts(opts)) return M3TSZ_ERR_INVALID_ARG;
  if (n_series == 0) return M3TSZ_OK;
  if (!h_streams || !h_offsets || !h_slice_off || !h_replica_off || !h_series_off || !h_ts_out || !h_val_out ||
      !h_n_out || !h_status || max_points == 0 || out_cap == 0 || n_seq == 0 || strategy < 0 || strategy > 3)
    return M3TSZ_ERR_INVALID_ARG;
  const uint64_t n_rep = h_series_off[n_series], n_slice = h_replica_off[n_rep];
  if (h_slice_off[n_slice] != n_seq || h_series_off[0] != 0 || h_replica_off[0] != 0 || h_slice_off[0] != 0)
    return M3TSZ_ERR_INVALID_ARG;
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  ScratchFence fence(ctx);  // (after earlier device calls on this context, whatever their streams)
  DrainStreams drain{ctx};
  cudaStream_t sts[2] = {ctx->stream, ctx->stream2};
  // series per chunk: ~8 chunks, whole sequences of whole series
  uint64_t ch = (n_series + 7) / 8;
  {
    const uint64_t per_series = (streams_bytes + (n_seq * max_points * 16)) / n_series + out_cap * 16;
    uint64_t min_ch = (32ull << 20) / (per_series ? per_series : 1);
    if (min_ch < 1024) min_ch = 1024;
    if (ch < min_ch) ch = min_ch;
    if (ch > n_series) ch = n_series;
  }
  // the largest chunk in sequences / slices / replicas
  uint64_t max_q = 0, max_k = 0, max_r = 0;
  for (uint64_t s0 = 0; s0 < n_series; s0 += ch) {
    const uint64_t s1 = s0 + ch < n_series ? s0 + ch : n_series;
    const uint64_t r0 = h_series_off[s0], r1 = h_series_off[s1];
    if (r1 < r0 || r1 > n_rep) return M3TSZ_ERR_INVALID_ARG;
    const uint64_t k0 = h_replica_off[r0], k1 = h_replica_off[r1];
    if (k1 < k0 || k1 > n_slice) return M3TSZ_ERR_INVALID_ARG;
    const uint64_t q0 = h_slice_off[k0], q1 = h_slice_off[k1];
    if (q1 < q0 || q1 > n_seq) return M3TSZ_ERR_INVALID_ARG;
    if (q1 - q0 > max_q) max_q = q1 - q0;
    if (k1 - k0 > max_k) max_k = k1 - k0;
    if (r1 - r0 > max_r) max_r = r1 - r0;
  }
  void *d_streams, *d_off;
  int rc;
  if ((rc = ensure(ctx, fence, kSlotStreams, streams_bytes + 16, &d_streams))) return rc;
  if ((rc = ensure(ctx, fence, kSlotSeriesIndex, (n_seq + 1) * 8, &d_off))) return rc;
  struct Lane {
    void *ts, *val, *n, *st, *meta, *ots, *oval, *on, *ost;
  } ln[2];
  const size_t meta_words = (max_k + 1) + (max_r + 1) + (ch + 1);
  for (int i = 0; i < 2; i++) {
    if ((rc = ensure(ctx, fence, lane_slot(i, 0), max_q * max_points * 8, &ln[i].ts))) return rc;
    if ((rc = ensure(ctx, fence, lane_slot(i, 1), max_q * max_points * 8, &ln[i].val))) return rc;
    if ((rc = ensure(ctx, fence, lane_slot(i, 2), max_q * 4, &ln[i].n))) return rc;
    if ((rc = ensure(ctx, fence, lane_slot(i, 3), max_q * 4, &ln[i].st))) return rc;
    if ((rc = ensure(ctx, fence, lane_slot(i, 4), meta_words * 8, &ln[i].meta))) return rc;
    if ((rc = ensure(ctx, fence, lane_slot(i, 5), ch * out_cap * 8, &ln[i].ots))) return rc;
    if ((rc = ensure(ctx, fence, lane_slot(i, 6), ch * out_cap * 8, &ln[i].oval))) return rc;
    if ((rc = ensure(ctx, fence, lane_slot(i, 7), ch * 4, &ln[i].on))) return rc;
    if ((rc = ensure(ctx, fence, lane_slot(i, 8), ch * 4, &ln[i].ost))) return rc;
    if ((rc = ensure_stage(ctx, i, meta_words * 8))) return rc;
  }
  CK(cudaMemcpyAsync(d_off, h_offsets, (n_seq + 1) * 8, cudaMemcpyHostToDevice, sts[0]));
  CK(cudaEventRecord(ctx->ev, sts[0]));
  CK(cudaStreamWaitEvent(sts[1], ctx->ev, 0));
  int k = 0;
  for (uint64_t s0 = 0; s0 < n_series; s0 += ch, k++) {
    const int i = k & 1;
    cudaStream_t st = sts[i];
    Lane &L = ln[i];
    const uint64_t s1 = s0 + ch < n_series ? s0 + ch : n_series, ns = s1 - s0;
    const uint64_t r0 = h_series_off[s0], r1 = h_series_off[s1];
    const uint64_t k0 = h_replica_off[r0], k1 = h_replica_off[r1];
    const uint64_t q0 = h_slice_off[k0], q1 = h_slice_off[k1], nq = q1 - q0;
    const uint64_t b0 = h_offsets[q0], b1 = h_offsets[q1];
    if (b1 < b0 || b1 > streams_bytes) return M3TSZ_ERR_INVALID_ARG;
    CK(cudaStreamSynchronize(st));  // lane buffers + staging are free again
    // iterator structure of the chunk, rebased to the chunk's first sequence / slice / replica
    uint64_t *m = (uint64_t *)ctx->h_stage[i];
    uint64_t *m_slice = m, *m_rep = m + (max_k + 1), *m_ser = m_rep + (max_r + 1);
    for (uint64_t j = k0; j <= k1; j++) m_slice[j - k0] = h_slice_off[j] - q0;
    for (uint64_t j = r0; j <= r1; j++) m_rep[j - r0] = h_replica_off[j] - k0;
    for (uint64_t j = s0; j <= s1; j++) m_ser[j - s0] = h_series_off[j] - r0;
    CK(cudaMemcpyAsync(L.meta, m, meta_words * 8, cudaMemcpyHostToDevice, st));
    if (b1 > b0)
      CK(cudaMemcpyAsync((uint8_t *)d_streams + b0, h_streams + b0, b1 - b0, cudaMemcpyHostToDevice, st));
    if (nq) {
      rc = m3tsz_decode_batch(ctx, opts, (const uint8_t *)d_streams, streams_bytes, (const uint64_t *)d_off + q0, nq,
                              (int64_t *)L.ts, (double *)L.val, max_points, (uint32_t *)L.n, (int32_t *)L.st,
                              nullptr, nullptr, st);
      if (rc) return rc;
    }
    const uint64_t *dm = (const uint64_t *)L.meta;
    rc = m3tsz_merge_series_batch(ctx, (const int64_t *)L.ts, (const double *)L.val, max_points,
                                  (const uint32_t *)L.n, (const int32_t *)L.st, dm, dm + (max_k + 1),
                                  dm + (max_k + 1) + (max_r + 1), ns, start_ns, end_ns, strategy, (int64_t *)L.ots,
                                  (double *)L.oval, out_cap, (uint32_t *)L.on, (int32_t *)L.ost, st);
    if (rc) return rc;
    CK(cudaMemcpyAsync(h_ts_out + s0 * out_cap, L.ots, ns * out_cap * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(h_val_out + s0 * out_cap, L.oval, ns * out_cap * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(h_n_out + s0, L.on, ns * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(h_status + s0, L.ost, ns * 4, cudaMemcpyDeviceToHost, st));
  }
  CK(cudaStreamSynchronize(sts[0]));
  CK(cudaStreamSynchronize(sts[1]));
  return M3TSZ_OK;
}

}  // extern "C"
