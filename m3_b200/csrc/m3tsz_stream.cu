// m3tsz_stream.cu -- per-series streaming handles of the C ABI (include/m3tsz_b200.h):
// opaque m3tsz_encoder / m3tsz_iter objects a cgo shim binds method for method to
//   encoding.Encoder         /root/reference/src/dbnode/encoding/types.go:39-91
//   encoding.ReaderIterator  types.go:180-203        encoding.Decoder types.go:342-345
// plus EncoderPool / ReaderIteratorPool (encoder_pool.go:27-48, iterator_pool.go:27-47).
//
// The handles hold only HOST state: an encoder buffers (time, value, unit,
// annotation) and validates every Encode() call the way TimestampEncoder does
// (m3tsz/timestamp_encoder.go:104-246); the bitstream is produced by the batch ENCODE
// KERNEL (one series per launch) when Len/Stream/Discard/LastEncoded need it, and an
// iterator decodes its whole stream with the batch DECODE KERNEL on the first Next().
// There is no CPU codec here: without the GPU the handles cannot be created.
// A launch per series costs far more than the reference spends on a stream; the
// handles exist so that the reference's per-series call sites keep working unchanged
// while the batch sites (SURVEY.md §3.2/§3.3) move to the batch entry points.
#include <cuda_runtime.h>

#include <new>
#include <string>
#include <vector>

#include "m3tsz_ctx.h"

using namespace m3tsz;
using namespace m3tsz::host;

// ---------------------------------------------------------------------------
struct m3tsz_encoder {
  m3tsz_ctx *ctx = nullptr;
  m3tsz_options opts{};
  int64_t start = 0;
  bool closed = false;
  // buffered datapoints
  std::vector<int64_t> ts;
  std::vector<double> val;
  std::vector<uint8_t> unit;
  std::vector<m3tsz_annotation_entry> ann;
  std::vector<uint8_t> ann_bytes;
  // TimestampEncoder state mirrored for Encode()'s validation
  int cur_unit = 0;
  int64_t prev_time = 0, prev_delta = 0;
  uint64_t ann_checksum = 0;
  bool has_ann_checksum = false;
  // lazily produced stream
  bool fresh = false;
  int enc_status = 0;
  std::vector<uint8_t> stream;
  uint64_t stream_bits = 0;
  double last_value = 0.0;
  int64_t failed_dod = 0;  // delta-of-delta (in time units) of the last Encode that overflowed
  struct m3tsz_encoder_pool *pool = nullptr;
};

struct m3tsz_iter {
  m3tsz_ctx *ctx = nullptr;
  m3tsz_options opts{};
  bool closed = false;
  std::vector<uint8_t> data;
  bool decoded = false;
  int status = 0;
  int64_t pos = -1;  // index of the current datapoint
  std::vector<int64_t> ts;
  std::vector<double> val;
  std::vector<uint8_t> unit;                         // per datapoint
  std::vector<std::pair<uint32_t, uint32_t>> ann;    // per datapoint: (offset into ann_bytes, length)
  std::vector<uint8_t> ann_bytes;
  struct m3tsz_iter_pool *pool = nullptr;
};

struct m3tsz_encoder_pool {
  m3tsz_ctx *ctx;
  m3tsz_options opts;
  std::mutex mu;
  std::vector<m3tsz_encoder *> free_list;
};
struct m3tsz_iter_pool {
  m3tsz_ctx *ctx;
  m3tsz_options opts;
  std::mutex mu;
  std::vector<m3tsz_iter *> free_list;
};

namespace {

void encoder_reset_state(m3tsz_encoder *e, int64_t start) {  // encoder.reset, encoder.go:266-279
  e->start = start;
  e->ts.clear();
  e->val.clear();
  e->unit.clear();
  e->ann.clear();
  e->ann_bytes.clear();
  e->cur_unit = initial_time_unit(start, e->opts.default_time_unit);
  e->prev_time = start;
  e->prev_delta = 0;
  e->ann_checksum = 0;
  e->has_ann_checksum = false;
  e->fresh = false;
  e->enc_status = 0;
  e->stream.clear();
  e->stream_bits = 0;
  e->last_value = 0.0;
  e->closed = false;
}

// Runs the encode kernel over the buffered series (one launch) and brings back the stream,
// its bit length and the encoder's last value.
int encoder_materialise(m3tsz_encoder *e) {
  if (e->fresh) return e->enc_status;
  m3tsz_ctx *ctx = e->ctx;
  const size_t n = e->ts.size();
  e->stream.clear();
  e->stream_bits = 0;
  e->last_value = 0.0;
  e->enc_status = 0;
  if (n == 0) {
    e->fresh = true;
    return M3TSZ_OK;
  }
  std::lock_guard<std::mutex> lock(ctx->handle_mu);
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  ScratchFence fence(ctx);
  cudaStream_t st = ctx->stream;
  const uint64_t stride = m3tsz_encode_bound_units(n, 1) + ((e->ann_bytes.size() + 16 * e->ann.size() + 15) & ~15ull);
  void *d_ts, *d_val, *d_unit, *d_start, *d_out, *d_len, *d_st, *d_bits, *d_last, *d_aoff = nullptr,
       *d_aent = nullptr, *d_ab = nullptr;
  int rc;
  if ((rc = ensure(ctx, fence, kSlotEncTs, n * 8, &d_ts))) return rc;
  if ((rc = ensure(ctx, fence, kSlotEncVal, n * 8, &d_val))) return rc;
  if ((rc = ensure(ctx, fence, kSlotEncUnit, n, &d_unit))) return rc;
  if ((rc = ensure(ctx, fence, kSlotHandleMeta, 64, &d_start))) return rc;
  if ((rc = ensure(ctx, fence, kSlotEncOut, stride, &d_out))) return rc;
  d_len = (uint8_t *)d_start + 8;
  d_st = (uint8_t *)d_start + 16;
  d_bits = (uint8_t *)d_start + 24;
  d_last = (uint8_t *)d_start + 32;
  CK(cudaMemcpyAsync(d_ts, e->ts.data(), n * 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_val, e->val.data(), n * 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_unit, e->unit.data(), n, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_start, &e->start, 8, cudaMemcpyHostToDevice, st));
  uint64_t aoff[2] = {0, e->ann.size()};
  if (!e->ann.empty()) {
    if ((rc = ensure(ctx, fence, kSlotEncAnnOff, 16, &d_aoff))) return rc;
    if ((rc = ensure(ctx, fence, kSlotEncAnnEntries, e->ann.size() * sizeof(m3tsz_annotation_entry), &d_aent)))
      return rc;
    if ((rc = ensure(ctx, fence, kSlotEncAnnBytes, e->ann_bytes.size(), &d_ab))) return rc;
    CK(cudaMemcpyAsync(d_aoff, aoff, 16, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_aent, e->ann.data(), e->ann.size() * sizeof(m3tsz_annotation_entry),
                       cudaMemcpyHostToDevice, st));
    if (!e->ann_bytes.empty())
      CK(cudaMemcpyAsync(d_ab, e->ann_bytes.data(), e->ann_bytes.size(), cudaMemcpyHostToDevice, st));
  }
  m3tsz_encode_extras ex;
  memset(&ex, 0, sizeof(ex));
  ex.d_last_value = (double *)d_last;
  ex.d_out_bits = (uint64_t *)d_bits;
  rc = m3tsz_encode_batch_ex(ctx, &e->opts, (const int64_t *)d_ts, (const double *)d_val, 1, n, nullptr,
                             (const int64_t *)d_start, M3TSZ_UNIT_SECOND, (const uint8_t *)d_unit,
                             (const uint64_t *)d_aoff, (const m3tsz_annotation_entry *)d_aent,
                             (const uint8_t *)d_ab, (uint8_t *)d_out, stride, (uint64_t *)d_len,
                             (int32_t *)d_st, &ex, st);
  if (rc) return rc;
  struct {
    uint64_t len;
    int32_t status, pad;
    uint64_t bits;
    double last;
  } res;
  CK(cudaMemcpyAsync(&res, d_len, sizeof(res), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  e->enc_status = res.status;
  e->stream.resize(res.len);
  if (res.len) {
    CK(cudaMemcpyAsync(e->stream.data(), d_out, res.len, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  }
  e->stream_bits = res.bits;
  e->last_value = res.last;
  e->fresh = true;
  return e->enc_status;
}

// ts.Segment split of the stream (encoder.go:394-457): the tail is the last raw byte's used
// bits + the end-of-stream marker + padding (scheme.go:198-211).
size_t tail_len_of(uint64_t total_bits) {
  if (total_bits < 12) return 0;
  const uint64_t raw_bits = total_bits - kMarkerBits;       // bits the ostream held
  const unsigned pos = (unsigned)((raw_bits - 1) % 8) + 1;  // bits used in its last byte
  return (pos + kMarkerBits + 7) / 8;
}

int copy_out(const std::vector<uint8_t> &src, uint8_t *buf, size_t cap, size_t *len) {
  if (len) *len = src.size();
  if (src.size() > cap) return M3TSZ_ERR_CAPACITY;
  if (!src.empty()) {
    if (!buf) return M3TSZ_ERR_INVALID_ARG;
    memcpy(buf, src.data(), src.size());
  }
  return M3TSZ_OK;
}

uint8_t bits_at(const std::vector<uint8_t> &d, uint64_t bit) {  // 8 bits starting at `bit`
  const uint64_t i = bit >> 3;
  const unsigned sh = (unsigned)(bit & 7);
  const unsigned w = ((unsigned)d[i] << 8) | (i + 1 < d.size() ? d[i + 1] : 0u);
  return (uint8_t)(w >> (8 - sh));
}

// Decodes the iterator's stream with the batch kernel (one launch; re-run when the
// datapoint or event capacity was too small).
int iter_materialise(m3tsz_iter *it) {
  if (it->decoded) return M3TSZ_OK;
  m3tsz_ctx *ctx = it->ctx;
  it->ts.clear();
  it->val.clear();
  it->unit.clear();
  it->ann.clear();
  it->ann_bytes.clear();
  it->status = 0;
  if (it->data.empty()) {  // an empty reader: the first read hits io.EOF (istream.go:86-92)
    it->status = M3TSZ_ERR_EOF;
    it->decoded = true;
    return M3TSZ_OK;
  }
  std::lock_guard<std::mutex> lock(ctx->handle_mu);
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return set_cuda_error(ctx, guard.err, "cudaSetDevice");
  ScratchFence fence(ctx);
  cudaStream_t st = ctx->stream;
  const size_t nbytes = it->data.size();
  uint64_t cap = 1024, ev_cap = 64;
  void *d_stream, *d_meta;
  int rc;
  if ((rc = ensure(ctx, fence, kSlotIterStream, nbytes + 16, &d_stream))) return rc;
  if ((rc = ensure(ctx, fence, kSlotHandleMeta, 64, &d_meta))) return rc;
  CK(cudaMemcpyAsync(d_stream, it->data.data(), nbytes, cudaMemcpyHostToDevice, st));
  struct Meta {
    uint64_t off[2];
    uint64_t ev_count;
    uint32_t n;
    int32_t status;
    uint8_t unit_first, unit_last;
  } meta;
  std::vector<m3tsz_dp_event> events;
  for (int attempt = 0; attempt < 8; attempt++) {
    void *d_ts, *d_val, *d_ev;
    if ((rc = ensure(ctx, fence, kSlotIterTs, cap * 8, &d_ts))) return rc;
    if ((rc = ensure(ctx, fence, kSlotIterVal, cap * 8, &d_val))) return rc;
    if ((rc = ensure(ctx, fence, kSlotIterEvents, ev_cap * sizeof(m3tsz_dp_event), &d_ev))) return rc;
    memset(&meta, 0, sizeof(meta));
    meta.off[1] = nbytes;
    CK(cudaMemcpyAsync(d_meta, &meta, sizeof(meta), cudaMemcpyHostToDevice, st));
    uint8_t *m = (uint8_t *)d_meta;
    m3tsz_decode_extras ex;
    memset(&ex, 0, sizeof(ex));
    ex.d_unit_first = m + offsetof(Meta, unit_first);
    ex.d_events = (m3tsz_dp_event *)d_ev;
    ex.events_capacity = ev_cap;
    ex.d_event_count = (uint64_t *)(m + offsetof(Meta, ev_count));
    rc = m3tsz_decode_batch_ex(ctx, &it->opts, (const uint8_t *)d_stream, nbytes, (const uint64_t *)m, 1,
                               (int64_t *)d_ts, (double *)d_val, cap, (uint32_t *)(m + offsetof(Meta, n)),
                               (int32_t *)(m + offsetof(Meta, status)), m + offsetof(Meta, unit_last), nullptr,
                               &ex, st);
    if (rc) return rc;
    CK(cudaMemcpyAsync(&meta, d_meta, sizeof(meta), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (meta.status == M3TSZ_ERR_CAPACITY || meta.ev_count > ev_cap) {
      if (meta.n > cap) cap = meta.n;
      if (meta.ev_count > ev_cap) ev_cap = meta.ev_count;
      continue;
    }
    const size_t n = meta.n;
    it->ts.resize(n);
    it->val.resize(n);
    events.resize(meta.ev_count);
    if (n) {
      CK(cudaMemcpyAsync(it->ts.data(), d_ts, n * 8, cudaMemcpyDeviceToHost, st));
      CK(cudaMemcpyAsync(it->val.data(), d_val, n * 8, cudaMemcpyDeviceToHost, st));
    }
    if (meta.ev_count)
      CK(cudaMemcpyAsync(events.data(), d_ev, meta.ev_count * sizeof(m3tsz_dp_event), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    it->status = meta.status;
    // Current()'s (unit, annotation) of every datapoint from the event table
    it->unit.assign(n, meta.unit_first);
    it->ann.assign(n, std::make_pair(0u, 0u));
    size_t from = 0;
    uint8_t u = meta.unit_first;
    for (const m3tsz_dp_event &e : events) {  // stream order within the one series
      if (e.dp_index >= n) continue;
      if (e.kind == M3TSZ_EVENT_TIME_UNIT) {
        for (size_t i = from; i < e.dp_index; i++) it->unit[i] = u;
        from = e.dp_index;
        u = (uint8_t)e.unit;
      } else if (e.kind == M3TSZ_EVENT_ANNOTATION) {
        const uint32_t o = (uint32_t)it->ann_bytes.size();
        for (uint32_t k = 0; k < e.length; k++) it->ann_bytes.push_back(bits_at(it->data, e.bit_offset + 8ull * k));
        it->ann[e.dp_index] = std::make_pair(o, e.length);  // a later annotation of the same datapoint wins
      }
    }
    for (size_t i = from; i < n; i++) it->unit[i] = u;
    it->decoded = true;
    return M3TSZ_OK;
  }
  return M3TSZ_ERR_CAPACITY;
}

}  // namespace

extern "C" {

// ------------------------------------------------------------------ encoder
int m3tsz_encoder_create(m3tsz_ctx *ctx, const m3tsz_options *opts, int64_t start_ns, m3tsz_encoder **out) {
  if (!ctx || !valid_opts(opts) || !out) return M3TSZ_ERR_INVALID_ARG;
  m3tsz_encoder *e = new (std::nothrow) m3tsz_encoder();
  if (!e) return M3TSZ_ERR_INVALID_ARG;
  e->ctx = ctx;
  e->opts = *opts;
  encoder_reset_state(e, start_ns);
  *out = e;
  return M3TSZ_OK;
}

void m3tsz_encoder_destroy(m3tsz_encoder *e) { delete e; }

int m3tsz_encoder_reset(m3tsz_encoder *e, int64_t start_ns, uint64_t capacity) {
  if (!e) return M3TSZ_ERR_INVALID_ARG;
  encoder_reset_state(e, start_ns);
  if (capacity) {
    e->ts.reserve(capacity / 2);  // capacity is a byte hint in the reference (ostream buffer)
    e->val.reserve(capacity / 2);
  }
  return M3TSZ_OK;
}

int m3tsz_encoder_encode(m3tsz_encoder *e, int64_t ts_ns, double value, int32_t unit, const uint8_t *annotation,
                         uint64_t annotation_len) {
  if (!e) return M3TSZ_ERR_INVALID_ARG;
  if (e->closed) return M3TSZ_ERR_ENCODER_CLOSED;  // encoder.go:91-93
  if (annotation_len && !annotation) return M3TSZ_ERR_INVALID_ARG;
  if (e->ts.size() >= (1ull << 27) - 1) return M3TSZ_ERR_CAPACITY;
  // TimestampEncoder.WriteNextTime validation (timestamp_encoder.go:104-246): an invalid unit
  // fails in maybeWriteTimeUnitChange / the scheme lookup; a second / millisecond
  // delta-of-delta must fit 32 bits.  A failing datapoint is dropped as a whole (DESIGN.md §6).
  const bool tu_valid = unit_is_valid(unit);
  const bool changed = tu_valid && unit != e->cur_unit;
  const int64_t delta = (int64_t)((uint64_t)ts_ns - (uint64_t)e->prev_time);
  if (!changed) {
    if (!tu_valid) return M3TSZ_ERR_UNRECOGNIZED_UNIT;
    const int64_t dod_ns = (int64_t)((uint64_t)delta - (uint64_t)e->prev_delta);
    const int64_t dod = dod_ns / unit_nanos(unit);  // Go's truncating division
    if ((unit == M3TSZ_UNIT_SECOND || unit == M3TSZ_UNIT_MILLISECOND) && (dod > INT32_MAX || dod < INT32_MIN)) {
      e->failed_dod = dod;
      return M3TSZ_ERR_DOD_OVERFLOW;
    }
  }
  if (annotation_len) {
    const uint64_t cs = xxh64(annotation, annotation_len);
    e->ann_checksum = cs;  // rewritten only when it differs, but the checksum is the same either way
    e->has_ann_checksum = true;
    m3tsz_annotation_entry a;
    a.dp_index = (uint32_t)e->ts.size();
    a.length = (uint32_t)annotation_len;
    a.byte_offset = e->ann_bytes.size();
    e->ann.push_back(a);
    e->ann_bytes.insert(e->ann_bytes.end(), annotation, annotation + annotation_len);
  }
  e->prev_time = ts_ns;
  if (changed) {
    e->cur_unit = unit;
    e->prev_delta = 0;
  } else {
    e->prev_delta = delta;
  }
  e->ts.push_back(ts_ns);
  e->val.push_back(value);
  e->unit.push_back((uint8_t)unit);
  e->fresh = false;
  return M3TSZ_OK;
}

int64_t m3tsz_encoder_failed_dod(const m3tsz_encoder *e) { return e ? e->failed_dod : 0; }

uint64_t m3tsz_encoder_num_encoded(const m3tsz_encoder *e) { return e ? e->ts.size() : 0; }  // encoder.go:299-302

int m3tsz_encoder_last_encoded(m3tsz_encoder *e, int64_t *ts_ns, double *value) {  // encoder.go:305-319
  if (!e) return M3TSZ_ERR_INVALID_ARG;
  if (e->ts.empty()) return M3TSZ_ERR_NO_DATAPOINTS;
  int rc = encoder_materialise(e);
  if (rc) return rc;
  if (ts_ns) *ts_ns = e->prev_time;
  if (value) *value = e->last_value;
  return M3TSZ_OK;
}

int m3tsz_encoder_last_annotation_checksum(const m3tsz_encoder *e, uint64_t *checksum) {  // encoder.go:321-327
  if (!e) return M3TSZ_ERR_INVALID_ARG;
  if (e->ts.empty()) return M3TSZ_ERR_NO_DATAPOINTS;
  // NewTimestampEncoder starts from the checksum of the empty annotation
  static const uint64_t empty = xxh64(nullptr, 0);
  if (checksum) *checksum = e->has_ann_checksum ? e->ann_checksum : empty;
  return M3TSZ_OK;
}

int m3tsz_encoder_empty(const m3tsz_encoder *e) { return !e || e->ts.empty(); }  // encoder.go:330-332

int m3tsz_encoder_len(m3tsz_encoder *e, uint64_t *len) {  // encoder.go:336-354
  if (!e || !len) return M3TSZ_ERR_INVALID_ARG;
  int rc = encoder_materialise(e);
  *len = e->stream.size();
  return rc;
}

int m3tsz_encoder_stream(m3tsz_encoder *e, uint8_t *buf, uint64_t cap, uint64_t *len, uint64_t *tail_len) {
  if (!e) return M3TSZ_ERR_INVALID_ARG;  // Stream(ctx), encoder.go:282-297: (nil, false) <=> *len == 0
  int rc = encoder_materialise(e);
  if (rc) return rc;
  if (tail_len) *tail_len = tail_len_of(e->stream_bits);
  size_t l = 0;
  rc = copy_out(e->stream, buf, cap, &l);
  if (len) *len = l;
  return rc;
}

int m3tsz_encoder_close(m3tsz_encoder *e) {  // encoder.go:357-370 (idempotent; returns to its pool)
  if (!e) return M3TSZ_ERR_INVALID_ARG;
  if (e->closed) return M3TSZ_OK;
  encoder_reset_state(e, e->start);
  e->closed = true;
  if (e->pool) {
    std::lock_guard<std::mutex> lock(e->pool->mu);
    e->pool->free_list.push_back(e);
  }
  return M3TSZ_OK;
}

int m3tsz_encoder_discard(m3tsz_encoder *e, uint8_t *buf, uint64_t cap, uint64_t *len, uint64_t *tail_len) {
  int rc = m3tsz_encoder_stream(e, buf, cap, len, tail_len);  // encoder.go:374-381
  if (rc) return rc;
  return m3tsz_encoder_close(e);
}

int m3tsz_encoder_discard_reset(m3tsz_encoder *e, int64_t start_ns, uint64_t capacity, uint8_t *buf, uint64_t cap,
                                uint64_t *len, uint64_t *tail_len) {
  int rc = m3tsz_encoder_stream(e, buf, cap, len, tail_len);  // encoder.go:385-392
  if (rc) return rc;
  return m3tsz_encoder_reset(e, start_ns, capacity);
}

// ------------------------------------------------------------------ iterator
int m3tsz_iter_create(m3tsz_ctx *ctx, const m3tsz_options *opts, m3tsz_iter **out) {
  if (!ctx || !valid_opts(opts) || !out) return M3TSZ_ERR_INVALID_ARG;
  m3tsz_iter *it = new (std::nothrow) m3tsz_iter();
  if (!it) return M3TSZ_ERR_INVALID_ARG;
  it->ctx = ctx;
  it->opts = *opts;
  *out = it;
  return M3TSZ_OK;
}

void m3tsz_iter_destroy(m3tsz_iter *it) { delete it; }

int m3tsz_iter_reset(m3tsz_iter *it, const uint8_t *data, uint64_t len) {  // iterator.go:253-263
  if (!it || (len && !data) || len >= (1ull << 28)) return M3TSZ_ERR_INVALID_ARG;
  it->data.assign(data, data + len);
  it->decoded = false;
  it->closed = false;
  it->status = 0;
  it->pos = -1;
  return M3TSZ_OK;
}

int m3tsz_iter_next(m3tsz_iter *it) {  // iterator.go:81-106; 1 = a datapoint is current, 0 = done / error
  if (!it || it->closed) return 0;
  if (iter_materialise(it) != M3TSZ_OK) {
    it->status = M3TSZ_ERR_CUDA;
    it->decoded = true;
    it->ts.clear();
  }
  if (it->pos + 1 < (int64_t)it->ts.size()) {
    it->pos++;
    return 1;
  }
  it->pos = (int64_t)it->ts.size();  // past the end: Err() now reports the stream's status
  return 0;
}

int m3tsz_iter_current(const m3tsz_iter *it, int64_t *ts_ns, double *value, int32_t *unit,
                       const uint8_t **annotation, uint64_t *annotation_len) {  // iterator.go:229-231
  if (!it || it->pos < 0 || it->pos >= (int64_t)it->ts.size()) return M3TSZ_ERR_INVALID_ARG;
  const size_t i = (size_t)it->pos;
  if (ts_ns) *ts_ns = it->ts[i];
  if (value) *value = it->val[i];
  if (unit) *unit = it->unit[i];
  if (annotation) *annotation = it->ann[i].second ? it->ann_bytes.data() + it->ann[i].first : nullptr;
  if (annotation_len) *annotation_len = it->ann[i].second;
  return M3TSZ_OK;
}

int m3tsz_iter_err(const m3tsz_iter *it) {  // iterator.go:234-236: set by the Next() that failed
  if (!it) return M3TSZ_ERR_INVALID_ARG;
  if (it->closed) return M3TSZ_ERR_ITER_CLOSED;
  if (!it->decoded || it->pos < (int64_t)it->ts.size()) return M3TSZ_OK;
  return it->status;
}

int m3tsz_iter_close(m3tsz_iter *it) {  // iterator.go:267-278
  if (!it) return M3TSZ_ERR_INVALID_ARG;
  if (it->closed) return M3TSZ_OK;
  it->closed = true;
  it->data.clear();
  it->ts.clear();
  it->val.clear();
  if (it->pool) {
    std::lock_guard<std::mutex> lock(it->pool->mu);
    it->pool->free_list.push_back(it);
  }
  return M3TSZ_OK;
}

// ------------------------------------------------------------------ pools (encoder_pool.go, iterator_pool.go)
int m3tsz_encoder_pool_create(m3tsz_ctx *ctx, const m3tsz_options *opts, uint64_t size, m3tsz_encoder_pool **out) {
  if (!ctx || !valid_opts(opts) || !out) return M3TSZ_ERR_INVALID_ARG;
  m3tsz_encoder_pool *p = new (std::nothrow) m3tsz_encoder_pool();
  if (!p) return M3TSZ_ERR_INVALID_ARG;
  p->ctx = ctx;
  p->opts = *opts;
  for (uint64_t i = 0; i < size; i++) {  // Init(alloc): the pool is filled up front
    m3tsz_encoder *e = nullptr;
    if (m3tsz_encoder_create(ctx, opts, 0, &e) != M3TSZ_OK) break;
    e->pool = p;
    e->closed = true;
    p->free_list.push_back(e);
  }
  *out = p;
  return M3TSZ_OK;
}
int m3tsz_encoder_pool_get(m3tsz_encoder_pool *p, m3tsz_encoder **out) {  // Get(): the caller Reset()s it
  if (!p || !out) return M3TSZ_ERR_INVALID_ARG;
  {
    std::lock_guard<std::mutex> lock(p->mu);
    if (!p->free_list.empty()) {
      *out = p->free_list.back();
      p->free_list.pop_back();
      return M3TSZ_OK;
    }
  }
  int rc = m3tsz_encoder_create(p->ctx, &p->opts, 0, out);  // pool exhausted: allocate (pool.ObjectPool does)
  if (rc == M3TSZ_OK) {
    (*out)->pool = p;
    (*out)->closed = true;
  }
  return rc;
}
void m3tsz_encoder_pool_destroy(m3tsz_encoder_pool *p) {
  if (!p) return;
  for (m3tsz_encoder *e : p->free_list) delete e;
  delete p;
}

int m3tsz_iter_pool_create(m3tsz_ctx *ctx, const m3tsz_options *opts, uint64_t size, m3tsz_iter_pool **out) {
  if (!ctx || !valid_opts(opts) || !out) return M3TSZ_ERR_INVALID_ARG;
  m3tsz_iter_pool *p = new (std::nothrow) m3tsz_iter_pool();
  if (!p) return M3TSZ_ERR_INVALID_ARG;
  p->ctx = ctx;
  p->opts = *opts;
  for (uint64_t i = 0; i < size; i++) {  // alloc(nil, nil), iterator_pool.go:37-41
    m3tsz_iter *it = nullptr;
    if (m3tsz_iter_create(ctx, opts, &it) != M3TSZ_OK) break;
    it->pool = p;
    p->free_list.push_back(it);
  }
  *out = p;
  return M3TSZ_OK;
}
int m3tsz_iter_pool_get(m3tsz_iter_pool *p, m3tsz_iter **out) {
  if (!p || !out) return M3TSZ_ERR_INVALID_ARG;
  {
    std::lock_guard<std::mutex> lock(p->mu);
    if (!p->free_list.empty()) {
      *out = p->free_list.back();
      p->free_list.pop_back();
      (*out)->closed = false;
      return M3TSZ_OK;
    }
  }
  int rc = m3tsz_iter_create(p->ctx, &p->opts, out);
  if (rc == M3TSZ_OK) (*out)->pool = p;
  return rc;
}
void m3tsz_iter_pool_destroy(m3tsz_iter_pool *p) {
  if (!p) return;
  for (m3tsz_iter *it : p->free_list) delete it;
  delete p;
}

}  // extern "C"
