// m3tsz_query.cu -- the two consumers directly after the decode path (SURVEY.md §8f N3/N4):
//
//  * Prometheus conversion epilogue: iteratorToPromResult,
//    /root/reference/src/query/storage/prom_converter.go:42-120 (ns -> ms timestamps,
//    valueDecreaseTolerance, counter-reset cumulativeSum per resolution window), over the
//    decoded / merged (ts, value) arrays that m3tsz_decode_batch / m3tsz_merge_series_batch
//    leave in HBM -- the last per-datapoint host loop of a fetch.
//  * Tile aggregation glue (storage.TileAggregator, src/dbnode/storage/types.go:1444-1472): the
//    fused decode+downsample kernel leaves window-major Gauge aggregates, the encoder's IN = 2 input
//    stage (m3tsz_encode.cu) turns them into (window end, Gauge.ValueOf(type)) datapoints on the fly;
//    only small helper kernels live here.
#include "m3tsz_common.cuh"
#include "m3tsz_kernels.h"

namespace m3tsz {

// ---------------------------------------------------------------------------
// Prometheus epilogue
// ---------------------------------------------------------------------------
// A count larger than the row (decode or merge output that hit its capacity) is refused like the
// encoder refuses it: nothing of the row is read, nothing of the output row is written, n_out = 0 and
// INVALID_ARG.  Converting only the stored prefix would hand back e.g. a counter's cumulative sum over
// part of its datapoints with status OK.
__device__ __forceinline__ void prom_refuse_row(const PromParams &p, uint64_t s) {
  p.n_out[s] = 0;
  if (p.status) p.status[s] = M3TSZ_ERR_INVALID_ARG;
}

// Plain conversion (no tolerance, no counter normalisation): every datapoint is
// independent -- one warp per series, lanes stride over the datapoints (coalesced).
__global__ void prom_simple_kernel(const PromParams p) {
  const uint64_t w = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= p.n_series) return;
  const uint32_t n = p.n_points[w];
  if (n > p.cap) {
    if (lane == 0) prom_refuse_row(p, w);
    return;
  }
  const uint32_t m = n < p.out_cap ? n : (uint32_t)p.out_cap;
  const int64_t *ts = p.ts + w * p.cap;
  const double *val = p.val + w * p.cap;
  int64_t *to = p.ts_out + w * p.out_cap;
  double *vo = p.val_out + w * p.out_cap;
  for (uint32_t i = lane; i < m; i += 32) {
    to[i] = ts[i] / 1000000;  // TimeToPromTimestamp, converter.go:388-391 (truncating)
    vo[i] = val[i];
  }
  if (lane == 0) {
    p.n_out[w] = n;
    if (p.status) p.status[w] = n > p.out_cap ? M3TSZ_ERR_CAPACITY : M3TSZ_OK;
  }
}

// General form: the tolerance clamp and the cumulative sum are sequential recurrences in
// floating point (order matters bit for bit), so one thread walks one series.
__global__ void prom_general_kernel(const PromParams p) {
  const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= p.n_series) return;
  const uint32_t n = p.n_points[s];
  if (n > p.cap) {
    prom_refuse_row(p, s);
    return;
  }
  const int64_t *ts = p.ts + s * p.cap;
  const double *val = p.val + s * p.cap;
  int64_t *to = p.ts_out + s * p.out_cap;
  double *vo = p.val_out + s * p.out_cap;
  const bool handle = p.handle_resets && p.handle_resets[s] != 0;
  const double tol = p.tolerance;
  bool first = true;
  double cumulative = 0.0, prev_v = 0.0;
  int64_t prev_t = 0;
  uint64_t k = 0;
  for (uint32_t i = 0; i < n; i++) {
    const int64_t t = ts[i];
    double v = val[i];
    if (tol > 0 && t < p.tolerance_until) {  // prom_converter.go:68-72
      if (!first && v < prev_v && v > __dmul_rn(prev_v, __dsub_rn(1.0, tol))) v = prev_v;
    }
    if (handle) {  // :84-98
      if (p.resolution != 0 && t / p.resolution != prev_t / p.resolution && !first) {
        if (k < p.out_cap) {
          to[k] = prev_t / 1000000;
          vo[k] = cumulative;
        }
        k++;
      }
      if (v < prev_v)
        cumulative = __dadd_rn(cumulative, v);  // counter reset
      else
        cumulative = __dadd_rn(cumulative, __dsub_rn(v, prev_v));
    } else {
      if (k < p.out_cap) {
        to[k] = t / 1000000;
        vo[k] = v;
      }
      k++;
    }
    prev_t = t;
    prev_v = v;
    first = false;
  }
  if (handle && !first) {  // :113-118
    if (k < p.out_cap) {
      to[k] = prev_t / 1000000;
      vo[k] = cumulative;
    }
    k++;
  }
  p.n_out[s] = (uint32_t)k;
  if (p.status) p.status[s] = k > p.out_cap ? M3TSZ_ERR_CAPACITY : M3TSZ_OK;
}

cudaError_t launch_prom(const PromParams &p, cudaStream_t stream) {
  if (p.n_series == 0) return cudaSuccess;
  const unsigned tb = 256;
  if (!(p.tolerance > 0) && !p.handle_resets) {
    const uint64_t threads = p.n_series * 32ull;
    const uint64_t blocks = (threads + tb - 1) / tb;
    if (blocks > 0x7fffffffull) return cudaErrorInvalidValue;
    prom_simple_kernel<<<(unsigned)blocks, tb, 0, stream>>>(p);
  } else {
    const uint64_t blocks = (p.n_series + tb - 1) / tb;
    if (blocks > 0x7fffffffull) return cudaErrorInvalidValue;
    prom_general_kernel<<<(unsigned)blocks, tb, 0, stream>>>(p);
  }
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------
// Tile aggregation glue (the re-encode itself is the encoder's IN = 2 input stage, m3tsz_encode.cu)
// ---------------------------------------------------------------------------
__global__ void fill_i64_kernel(int64_t *dst, int64_t v, uint64_t n) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = v;
}
cudaError_t launch_fill_i64(int64_t *dst, int64_t v, uint64_t n, cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  const unsigned tb = 256;
  fill_i64_kernel<<<(unsigned)((n + tb - 1) / tb), tb, 0, stream>>>(dst, v, n);
  return cudaGetLastError();
}

// Every tile call's status merge, and the multi-type stage's state commit (one thread per source series): a failed
// source's error goes to all n_types rows of the series; a series whose source and rows are all OK takes the record
// its lanes wrote to `scratch` (the encode kernel's IN = 5 epilogue)
__global__ void tiles_types_status_kernel(const int32_t *src_status, int32_t *status, uint64_t n, uint32_t n_types,
                                          const m3tsz_element_state *scratch, m3tsz_element_state *state) {
  const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const int32_t e = src_status[s];
  bool ok = e == 0;
  for (uint32_t j = 0; j < n_types; j++) {
    int32_t *row = status + (uint64_t)j * n + s;
    if (e != 0)
      *row = e;
    else
      ok = ok && *row == M3TSZ_OK;
  }
  if (state && ok) state[s] = scratch[s];
}
cudaError_t launch_tiles_types_status(const int32_t *src_status, int32_t *status, uint64_t n, uint32_t n_types,
                                      const m3tsz_element_state *scratch, m3tsz_element_state *state,
                                      cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  const unsigned tb = 256;
  tiles_types_status_kernel<<<(unsigned)((n + tb - 1) / tb), tb, 0, stream>>>(src_status, status, n, n_types, scratch,
                                                                              state);
  return cudaGetLastError();
}

// The rollup's source records.  First every group that was not saved (a row not OK: its members failed, its range or
// an index was invalid, or a row hit CAPACITY) marks the members its range names inside d_members; then a source that
// decoded and is unmarked takes its new record.  (Concurrent marks store the same byte.)
__global__ void rollup_mark_kernel(const uint64_t *group_off, const uint32_t *members, uint64_t n_members,
                                   uint64_t n_groups, const int32_t *status, uint32_t n_types, uint64_t n_src,
                                   uint8_t *mark) {
  // one warp per group, its lanes over the members: a large group costs its length / 32 steps
  const uint64_t g = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31u;
  if (g >= n_groups) return;
  bool ok = true;
  for (uint32_t j = 0; j < n_types; j++) ok = ok && status[(uint64_t)j * n_groups + g] == M3TSZ_OK;
  if (ok) return;
  const uint64_t lo = group_off[g], hi = group_off[g + 1] < n_members ? group_off[g + 1] : n_members;
  for (uint64_t i = lo + lane; i < hi; i += 32) {
    const uint32_t m = members[i];
    if (m < n_src) mark[m] = 1;
  }
}
__global__ void rollup_commit_kernel(const int32_t *src_status, const uint8_t *mark, uint64_t n,
                                     const m3tsz_transform_state *scratch, m3tsz_transform_state *state,
                                     int32_t *src_status_out) {
  const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const int32_t e = src_status[s];
  if (src_status_out) src_status_out[s] = e;
  if (state && e == M3TSZ_OK && !mark[s]) state[s] = scratch[s];
}
cudaError_t launch_rollup_commit(const uint64_t *group_off, const uint32_t *members, uint64_t n_members,
                                 uint64_t n_groups, const int32_t *status, uint32_t n_types, const int32_t *src_status,
                                 uint64_t n_src, uint8_t *mark, const m3tsz_transform_state *scratch,
                                 m3tsz_transform_state *state, int32_t *src_status_out, cudaStream_t stream) {
  if (n_src == 0) return cudaSuccess;
  const unsigned tb = 256;
  if ((n_groups * 32 + tb - 1) / tb > 0x7fffffffull || (n_src + tb - 1) / tb > 0x7fffffffull)
    return cudaErrorInvalidValue;
  cudaError_t e = cudaMemsetAsync(mark, 0, n_src, stream);
  if (e != cudaSuccess) return e;
  if (n_groups)
    rollup_mark_kernel<<<(unsigned)((n_groups * 32 + tb - 1) / tb), tb, 0, stream>>>(group_off, members, n_members,
                                                                                    n_groups, status, n_types, n_src,
                                                                                    mark);
  rollup_commit_kernel<<<(unsigned)((n_src + tb - 1) / tb), tb, 0, stream>>>(src_status, mark, n_src, scratch, state,
                                                                            src_status_out);
  return cudaGetLastError();
}

// The room of a tile call with annotations: a row's annotations are copies of different annotations of its source
// stream, or of any of its series' source blocks, so its bound adds the largest sum of a series' segment lengths (one
// warp-wide max and one atomic per warp)
__device__ __forceinline__ unsigned long long series_stream_len(const uint64_t *offsets, const uint64_t *lengths,
                                                                const uint64_t *block_off, uint64_t s,
                                                                uint64_t n_segments, uint64_t streams_bytes) {
  unsigned long long len = 0;
  uint64_t q0 = s, q1 = s + 1;
  if (block_off) {
    q0 = block_off[s];
    q1 = block_off[s + 1];
    if (q0 > q1 || q1 > n_segments) q1 = q0;
  }
  for (uint64_t q = q0; q < q1; q++) {
    const uint64_t o0 = offsets[q], o1 = lengths ? o0 + lengths[q] : offsets[q + 1];
    if (o1 >= o0 && o1 <= streams_bytes && o1 - o0 < (1ull << 28)) len += o1 - o0;
  }
  return len;
}
__global__ void max_stream_len_kernel(const uint64_t *offsets, const uint64_t *lengths, const uint64_t *block_off,
                                      uint64_t n, uint64_t n_segments, uint64_t streams_bytes,
                                      unsigned long long *out) {
  const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long len = 0;
  if (s < n) len = series_stream_len(offsets, lengths, block_off, s, n_segments, streams_bytes);
  for (int d = 16; d > 0; d >>= 1) {
    const unsigned long long o = __shfl_xor_sync(0xffffffffu, len, d);
    len = o > len ? o : len;
  }
  if ((threadIdx.x & 31) == 0 && len) atomicMax(out, len);
}
cudaError_t launch_max_stream_len(const uint64_t *offsets, const uint64_t *lengths, const uint64_t *block_off,
                                  uint64_t n_series, uint64_t n_segments, uint64_t streams_bytes,
                                  unsigned long long *out, cudaStream_t stream) {
  if (n_series == 0) return cudaSuccess;
  const unsigned tb = 256;
  max_stream_len_kernel<<<(unsigned)((n_series + tb - 1) / tb), tb, 0, stream>>>(
      offsets, lengths, block_off, n_series, n_segments, streams_bytes, out);
  return cudaGetLastError();
}

// The same for the rollup's group rows, whose annotations are copies of annotations of any member's stream: one warp
// per group, its lanes over the members, then a warp-wide sum and one atomic per group
__global__ void group_max_stream_len_kernel(const uint64_t *offsets, const uint64_t *lengths, const uint64_t *block_off,
                                            uint64_t n_series, uint64_t n_segments, uint64_t streams_bytes,
                                            const uint64_t *group_off, const uint32_t *members, uint64_t n_members,
                                            uint64_t n_groups, unsigned long long *out) {
  const uint64_t g = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31u;
  if (g >= n_groups) return;
  const uint64_t lo = group_off[g], hi = group_off[g + 1];
  if (lo > hi || hi > n_members) return;
  unsigned long long len = 0;
  for (uint64_t i = lo + lane; i < hi; i += 32) {
    const uint32_t m = members[i];
    if (m < n_series) len += series_stream_len(offsets, lengths, block_off, m, n_segments, streams_bytes);
  }
  for (int d = 16; d > 0; d >>= 1) len += __shfl_xor_sync(0xffffffffu, len, d);
  if (lane == 0 && len) atomicMax(out, len);
}
cudaError_t launch_group_max_stream_len(const uint64_t *offsets, const uint64_t *lengths, const uint64_t *block_off,
                                        uint64_t n_series, uint64_t n_segments, uint64_t streams_bytes,
                                        const uint64_t *group_off, const uint32_t *members, uint64_t n_members,
                                        uint64_t n_groups, unsigned long long *out, cudaStream_t stream) {
  if (n_groups == 0 || n_series == 0) return cudaSuccess;
  const unsigned tb = 256;
  if ((n_groups * 32 + tb - 1) / tb > 0x7fffffffull) return cudaErrorInvalidValue;
  group_max_stream_len_kernel<<<(unsigned)((n_groups * 32 + tb - 1) / tb), tb, 0, stream>>>(
      offsets, lengths, block_off, n_series, n_segments, streams_bytes, group_off, members, n_members, n_groups, out);
  return cudaGetLastError();
}

}  // namespace m3tsz
