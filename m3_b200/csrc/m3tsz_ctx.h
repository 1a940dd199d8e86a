// m3tsz_ctx.h -- internal: the context object and host helpers shared by the C-ABI
// translation units (m3tsz_capi.cu, m3tsz_stream.cu).  Not installed.
#pragma once

#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "m3tsz_common.cuh"
#include "m3tsz_kernels.h"

struct Scratch {
  void *ptr = nullptr;
  size_t bytes = 0;
};

// Context scratch slots: grow-only device buffers that live as long as the context (see
// ensure()).  Calls that name the same slot share its memory:
//
//   slot          holds                                          used by
//   0             streams                                        decode_host, downsample_host, fetch
//   1             offsets, or the encoder starts                 decode_host, downsample_host, fetch; encode_host
//   2, 3          decoded ts, val                                decode_host
//   4, 5          n_points, status                               decode_host, downsample_host, tiles,
//                                                                encode_host (4)
//   6             unit                                           decode_host
//   7             annotation refs, or annotation series offsets  decode_host; encode_host
//   8-11          window sum / count / min / max                 downsample_host, tiles
//                 (a Counter's int64 sum / count / min / max:    tiles
//                 the same 8 bytes per window)
//   12            lastAt                                         downsample_last / downsample_ex with a NULL
//                                                                d_last_at, tiles
//   13, 14        annotation entries, annotation bytes           encode_host
//   15            compaction scan temp                           compact_streams
//   16-24, 26-34  pipeline lane 0 / 1, buffers 0-8 (lane_slot)   encode_host, fetch
//   25            window sumSq (Gauge float64 / Counter int64)   downsample_ex with a NULL sum_sq, tiles
//   36, 37        packed slot sets, batch counter                packed encode, tiles
//   38, 39        window last, tile encoder starts               tiles, downsample_ex (38, NULL d_last); tiles
//   40-47         streaming handles, under handle_mu             m3tsz_stream.cu
//   35            element records of the multi-type tile stage   tiles (aggregate_tiles_types)
//   48-50         route targets, touched records, their count    encoder_set_write
//   51, 52        window annotation references, the longest     tiles (aggregate_tiles_annotated)
//                 source stream
//   53-56         forwarded values, presence words, source      tiles (aggregate_tiles_rollup)
//                 records, source marks
//   57-63         group window sum / count / min / max / last   tiles (aggregate_tiles_rollup)
//                 / sumSq, group statuses
//   64, 65        forwarded-annotation words, group annotation   tiles (aggregate_tiles_rollup_annotated)
//                 references
//   66-70         staged row ts / values / counts, row statuses, element_set_consume; element_set_reset (66: the
//                 datapoints appended                            output rows' starts)
//   71, 72        staged rows' annotation offsets and entries    element_set_consume_annotated
//   73-79         forwarded window starts / values, due-window   element_set_forward
//                 counts, presence and slot words, source
//                 records, source marks
enum Slot : int {
  kSlotStreams = 0,
  kSlotSeriesIndex = 1,  // per-series index input: stream offsets, or the encoder starts
  kSlotTs = 2,
  kSlotVal = 3,
  kSlotNPoints = 4,
  kSlotStatus = 5,
  kSlotUnit = 6,
  kSlotAnnRefs = 7,       // decode output
  kSlotAnnSeriesOff = 7,  // encode input
  kSlotWinSum = 8,
  kSlotWinCount = 9,
  kSlotWinMin = 10,
  kSlotWinMax = 11,
  kSlotWinLastAt = 12,
  kSlotAnnEntries = 13,
  kSlotAnnBytes = 14,
  kSlotCompactTmp = 15,
  kSlotLaneBase = 16,
  kSlotWinSumSq = 25,  // between the two pipeline lanes' slot ranges
  kSlotElementScratch = 35,
  kSlotPackedSlots = 36,
  kSlotBatchCounter = 37,
  kSlotWinLast = 38,
  kSlotTileStarts = 39,
  // streaming handles: an encoder's buffers, or an iterator's
  kSlotEncTs = 40,
  kSlotEncVal = 41,
  kSlotEncUnit = 42,
  kSlotHandleMeta = 43,  // both: small per-call results
  kSlotEncOut = 44,
  kSlotEncAnnOff = 45,
  kSlotEncAnnEntries = 46,
  kSlotEncAnnBytes = 47,
  kSlotIterStream = 40,
  kSlotIterTs = 41,
  kSlotIterVal = 42,
  kSlotIterEvents = 44,
  // bucket writes
  kSlotRouteTarget = 48,
  kSlotRouteTouched = 49,
  kSlotRouteCount = 50,
  // tile aggregation with annotations
  kSlotWinAnn = 51,
  kSlotSrcMaxLen = 52,
  // tile aggregation through a rollup
  kSlotFwdVal = 53,
  kSlotFwdPresent = 54,
  kSlotSrcRecScratch = 55,
  kSlotSrcMark = 56,
  kSlotGroupSum = 57,
  kSlotGroupCount = 58,
  kSlotGroupMin = 59,
  kSlotGroupMax = 60,
  kSlotGroupLast = 61,
  kSlotGroupSumSq = 62,
  kSlotGroupStatus = 63,
  // the rollup that keeps annotations
  kSlotFwdAnnPresent = 64,
  kSlotGroupAnn = 65,
  // element sets
  kSlotElemRowTs = 66,
  kSlotElemRowVal = 67,
  kSlotElemRowN = 68,
  kSlotElemRowStatus = 69,
  kSlotElemRowAppended = 70,
  kSlotElemRowAnnOff = 71,
  kSlotElemRowAnn = 72,
  // element sets through a rollup
  kSlotElemFwdStart = 73,
  kSlotElemFwdVal = 74,
  kSlotElemFwdN = 75,
  kSlotElemFwdPresent = 76,
  kSlotElemFwdDue = 77,
  kSlotElemFwdRec = 78,
  kSlotElemFwdMark = 79,
  // ... that keep annotations
  kSlotElemFwdAnnPresent = 80,
  kSlotElemFwdAnn = 81,
  // element-set rollups across shards: the writer's per-group counts, their scans and the scan's scratch; the
  // AddUnique's sort keys and indices before and after the sort, and the sort's scratch
  kSlotElemFwdRecN = 82,
  kSlotElemFwdValN = 83,
  kSlotElemFwdRecOff = 84,
  kSlotElemFwdValOff = 85,
  kSlotElemFwdScanTmp = 86,
  kSlotElemAddFwdKey = 87,
  kSlotElemAddFwdIdx = 88,
  kSlotElemAddFwdSortedKey = 89,
  kSlotElemAddFwdSortedIdx = 90,
  kSlotElemAddFwdSortTmp = 91,
  kNumSlots = 92
};

// Buffer k (0-8) of pipeline lane `lane` (0 or 1): slots 16-24 and 26-34.
inline Slot lane_slot(int lane, int k) { return Slot(kSlotLaneBase + 10 * lane + k); }

struct m3tsz_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;   // used by the *_host entry points
  cudaStream_t stream2 = nullptr;  // second lane of the chunked H2D / kernel / D2H pipeline
  cudaEvent_t ev = nullptr;
  // recorded by every call that uses the scratch below or d_flag, on the stream it ran on (ScratchFence)
  cudaEvent_t scratch_ev = nullptr;
  uint64_t launches = 0;
  char last_error[256] = {0};
  Scratch s[kNumSlots];
  int32_t *d_flag = nullptr;  // [2]
  void *h_stage[2] = {nullptr, nullptr};  // pinned staging for per-chunk offsets
  size_t h_stage_bytes[2] = {0, 0};
  std::mutex handle_mu;  // serialises the streaming handles' use of the scratch below
};

namespace m3tsz {
namespace host {

inline int set_cuda_error(m3tsz_ctx *ctx, cudaError_t e, const char *where) {
  if (ctx) snprintf(ctx->last_error, sizeof(ctx->last_error), "%s: %s", where, cudaGetErrorString(e));
  return M3TSZ_ERR_CUDA;
}

#define CK(call)                                                 \
  do {                                                           \
    cudaError_t _e = (call);                                     \
    if (_e != cudaSuccess) return set_cuda_error(ctx, _e, #call); \
  } while (0)

inline int ensure_stage(m3tsz_ctx *ctx, int i, size_t bytes) {
  if (ctx->h_stage_bytes[i] >= bytes) return M3TSZ_OK;
  if (ctx->h_stage[i]) CK(cudaFreeHost(ctx->h_stage[i]));
  ctx->h_stage[i] = nullptr;
  ctx->h_stage_bytes[i] = 0;
  CK(cudaMallocHost(&ctx->h_stage[i], bytes));
  ctx->h_stage_bytes[i] = bytes;
  return M3TSZ_OK;
}

// Series per pipeline chunk: ~8 chunks per call, but never tiny ones.
inline uint64_t pick_chunk(uint64_t n_series, uint64_t bytes_per_series) {
  uint64_t ch = (n_series + 7) / 8;
  uint64_t min_ch = (16ull << 20) / (bytes_per_series ? bytes_per_series : 1);
  if (min_ch < 2048) min_ch = 2048;
  if (ch < min_ch) ch = min_ch;
  if (ch > n_series) ch = n_series;
  ch = (ch + 127) & ~127ull;  // whole thread blocks
  return ch;
}

// Entry points run on the context's device and restore the caller's current device on
// return (a process that drives several GPUs must not be retargeted by a library call).
struct DeviceGuard {
  int prev = -1;
  bool ok = true;
  cudaError_t err = cudaSuccess;
  explicit DeviceGuard(int device) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != device) {
      err = cudaSetDevice(device);
      ok = (err == cudaSuccess);
    } else {
      prev = -1;
    }
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

// Declared right after the DeviceGuard of every call that uses context scratch or d_flag.  The scratch belongs to
// the context, not to a stream, so these calls are ordered in the order they are issued, whatever streams they run
// on: the call's stream (for the *_host calls and the streaming handles, both context streams) waits for the last
// such call's work, and on every exit path the call's own work is recorded as the new last.  Neither this nor
// ensure() is locked: batch calls on one context come from one host thread at a time.  `active` false: the call
// uses no scratch this time (e.g. the caller passed every output), and the fence does nothing.
struct ScratchFence {
  m3tsz_ctx *ctx;
  cudaStream_t st, st2 = nullptr;
  bool active;
  ScratchFence(m3tsz_ctx *c, cudaStream_t s, bool use = true) : ctx(c), st(s), active(use) {
    if (active) cudaStreamWaitEvent(st, ctx->scratch_ev, 0);
  }
  explicit ScratchFence(m3tsz_ctx *c) : ctx(c), st(c->stream), st2(c->stream2), active(true) {
    cudaStreamWaitEvent(st, ctx->scratch_ev, 0);
    cudaStreamWaitEvent(st2, ctx->scratch_ev, 0);
  }
  ~ScratchFence() {
    if (!active) return;
    if (st2) {  // one event, two streams: the second joins the first
      cudaEventRecord(ctx->ev, st2);
      cudaStreamWaitEvent(st, ctx->ev, 0);
    }
    cudaEventRecord(ctx->scratch_ev, st);
  }
  ScratchFence(const ScratchFence &) = delete;
  ScratchFence &operator=(const ScratchFence &) = delete;
};

// A scratch slot of at least `bytes`, under the call's fence.  Growing a slot frees the old buffer, so it first waits
// for the last scratch-using call to finish.
inline int ensure(m3tsz_ctx *ctx, const ScratchFence &fence, Slot slot, size_t bytes, void **out) {
  if (!fence.active) {
    snprintf(ctx->last_error, sizeof(ctx->last_error), "scratch slot %d used without its fence", (int)slot);
    return M3TSZ_ERR_CUDA;
  }
  Scratch &sc = ctx->s[slot];
  if (bytes == 0) bytes = 16;
  if (sc.bytes < bytes) {
    CK(cudaEventSynchronize(ctx->scratch_ev));
    if (sc.ptr) CK(cudaFree(sc.ptr));
    sc.ptr = nullptr;
    sc.bytes = 0;
    size_t want = bytes + bytes / 8;  // grow-only with slack
    cudaError_t e = cudaMalloc(&sc.ptr, want);
    if (e != cudaSuccess) {
      (void)cudaGetLastError();
      want = bytes;
      CK(cudaMalloc(&sc.ptr, want));
    }
    sc.bytes = want;
  }
  *out = sc.ptr;
  return M3TSZ_OK;
}

// Declared right after a *_host call's ScratchFence: however the call returns, it does not
// leave copies from or into the caller's buffers in flight on the context's streams.
struct DrainStreams {
  m3tsz_ctx *ctx;
  ~DrainStreams() {
    cudaStreamSynchronize(ctx->stream);
    cudaStreamSynchronize(ctx->stream2);
  }
};

inline bool valid_opts(const m3tsz_options *o) {
  return o && (o->int_optimized == 0 || o->int_optimized == 1) && o->default_time_unit >= 0 &&
         o->default_time_unit <= 8;
}

}  // namespace host
}  // namespace m3tsz

