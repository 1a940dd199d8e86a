/*
 * m3tsz_b200.h -- C ABI of the H100-native M3TSZ batch codec (libm3tsz_b200.so).
 *
 * This is the drop-in boundary for the reference's M3TSZ path.  The reference
 * (m3db/m3, 100 % Go) has no FFI today: the codec sits behind the Go interfaces
 *   encoding.Encoder         src/dbnode/encoding/types.go:39-91
 *   encoding.ReaderIterator  src/dbnode/encoding/types.go:180-203
 *   encoding.Decoder         src/dbnode/encoding/types.go:342-345
 * installed through the pool allocator closures at
 *   src/dbnode/server/server.go:1780-1800 (and the sites in SURVEY.md §1).
 * A cgo shim (INTEGRATION.md) implements those interfaces over the entry points
 * below; each entry point cites the reference function(s) it replaces.
 *
 * Conventions: plain pointers and sizes, no C++/torch types; every function
 * returns an int status (M3TSZ_OK == 0) and never throws or aborts; the caller
 * owns every buffer; the library owns only scratch held by an explicit
 * m3tsz_ctx.  "d_" pointers are CUDA device pointers, "h_" pointers are host
 * pointers.  `stream` is a cudaStream_t passed as void* (NULL = default stream).
 * Device entry points are asynchronous on `stream`: every launch and copy of the
 * call is on `stream`, and the call returns before it runs, except as listed
 * below.  Host entry points synchronise before returning.
 *
 * Streams and one context.  One context may serve device calls on several
 * streams.  The context's scratch belongs to the context, not to a stream, so
 * the calls that use it (the tile calls, m3tsz_decode_downsample_ex and
 * m3tsz_decode_downsample_last_batch with a NULL lastAt / sumSq / last output,
 * m3tsz_encode_batch_packed(_ex), m3tsz_compact_streams,
 * m3tsz_encoder_set_write, m3tsz_element_set_reset of a set with output rows,
 * m3tsz_element_set_consume(_annotated), m3tsz_element_set_forward(_annotated),
 * m3tsz_element_set_forward_write(_timer), m3tsz_element_set_add_forwarded(_timer)) are
 * ordered in the order they are issued: each one's stream waits on the device
 * for the context's previous such call, whatever stream that was on.  Two such
 * calls on one context therefore never overlap; a caller who wants them to
 * overlap uses two contexts.  A *_host call (and a streaming handle's call)
 * waits for the context's earlier device calls of this kind before it touches
 * the scratch.  The other device calls take no part in this ordering.
 * Batch calls on one context must still come from one host thread at a time:
 * the scratch and this ordering are not locked.
 *
 * Device entry points that block the host until their stream reaches a point of
 * the call (each one's comment says so too): m3tsz_compact_streams,
 * m3tsz_aggregate_tiles_annotated, m3tsz_aggregate_tiles_blocks (with
 * annotations) and m3tsz_aggregate_tiles_rollup_annotated.
 *
 * Besides those, a scratch-using call that has to grow a scratch slot (the first
 * call at a larger size) waits on the host for the context's previous
 * scratch-using call to finish before it frees the smaller buffer.
 *
 * Bit-exactness contract: encoded streams are byte-identical to what the
 * reference m3tsz encoder produces for the same (start, datapoints, units,
 * annotations); decoded (timestamp, value) pairs are bit-identical to the
 * reference iterator's.  See DESIGN.md for the (documented) behaviour on
 * corrupt / truncated streams.
 */
#ifndef M3TSZ_B200_H
#define M3TSZ_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define M3TSZ_B200_VERSION 100 /* 0.1.0 */

/* xtime.Unit, src/x/time/unit.go:30-42 */
enum {
  M3TSZ_UNIT_NONE = 0,
  M3TSZ_UNIT_SECOND = 1,
  M3TSZ_UNIT_MILLISECOND = 2,
  M3TSZ_UNIT_MICROSECOND = 3,
  M3TSZ_UNIT_NANOSECOND = 4,
  M3TSZ_UNIT_MINUTE = 5,
  M3TSZ_UNIT_HOUR = 6,
  M3TSZ_UNIT_DAY = 7,
  M3TSZ_UNIT_YEAR = 8
};

/* Status codes.  1..12 mirror the reference's error values for this path. */
enum {
  M3TSZ_OK = 0,
  M3TSZ_ERR_EOF = 1,               /* io.EOF from IStream (istream.go:86-92): truncated stream */
  M3TSZ_ERR_ENCODER_CLOSED = 2,    /* errEncoderClosed, m3tsz/encoder.go:37 */
  M3TSZ_ERR_NO_DATAPOINTS = 3,     /* errNoEncodedDatapoints, m3tsz/encoder.go:38 */
  M3TSZ_ERR_DOD_OVERFLOW = 4,      /* "deltaOfDelta value %d %s overflows 32 bits", timestamp_encoder.go:219 */
  M3TSZ_ERR_NO_TIME_SCHEME = 5,    /* errNoTimeSchemaForUnit, timestamp_iterator.go:33 */
  M3TSZ_ERR_UNRECOGNIZED_UNIT = 6, /* errUnrecognizedTimeUnit, src/x/time/unit.go:45 */
  M3TSZ_ERR_INVALID_MULT = 7,      /* errInvalidMultiplier, m3tsz/m3tsz.go:69 */
  M3TSZ_ERR_ANNOTATION_LEN = 8,    /* errUnexpectedAnnotationLength, timestamp_iterator.go:34 */
  M3TSZ_ERR_ANNOTATION_SHORT = 9,  /* errAnnotationTooFewBytes, timestamp_iterator.go:35 */
  M3TSZ_ERR_ITER_CLOSED = 10,      /* errClosed, m3tsz/iterator.go:33 */
  M3TSZ_ERR_VARINT_OVERFLOW = 11,  /* Go encoding/binary errOverflow */
  M3TSZ_ERR_UNEXPECTED_EOF = 12,   /* io.ErrUnexpectedEOF */
  M3TSZ_ERR_OUT_OF_ORDER = 13,     /* errOutOfOrderIterator, encoding/iterators.go:229-236 */
  M3TSZ_ERR_TOO_MANY_ITERATORS = 14, /* > 12 replicas per series or readers per block slice */
  M3TSZ_ERR_CHECKSUM_MISMATCH = 15, /* errSeekChecksumMismatch, persist/fs/seek.go:50-51, read.go:395-397 */
  M3TSZ_ERR_TOO_MANY_ENCODERS = 16, /* errTooManyEncoders, storage/series/buffer.go:57 */
  M3TSZ_ERR_AGGREGATION_CLOSED = 17, /* errAggregationClosed, aggregator/elem_base.go:72 */
  M3TSZ_ERR_DUPLICATE_SOURCE = 18, /* errDuplicateForwardingSource, aggregator/elem_base.go:74 */
  /* library-level conditions */
  M3TSZ_ERR_CAPACITY = 100,        /* more datapoints / bytes than the caller's buffer holds */
  M3TSZ_ERR_INVALID_ARG = 101,
  M3TSZ_ERR_CUDA = 102,            /* a CUDA runtime call failed; see m3tsz_last_cuda_error */
  M3TSZ_ERR_NO_DEVICE = 103,       /* no usable CUDA device: the library has NO CPU fallback */
  M3TSZ_ERR_STREAM_TOO_LARGE = 104 /* a single stream exceeds 256 MiB */
};

/* encoding.Options subset that changes the bitstream (encoding/options.go:31-73)
 * + the intOptimized constructor flag (m3tsz/encoder.go:64-69, iterator.go:67-71). */
typedef struct m3tsz_options {
  int32_t int_optimized;     /* m3tsz.DefaultIntOptimizationEnabled = 1 (m3tsz/m3tsz.go:30) */
  int32_t default_time_unit; /* encoding.Options.DefaultTimeUnit(), default M3TSZ_UNIT_SECOND */
} m3tsz_options;

typedef struct m3tsz_ctx m3tsz_ctx;

/* Library / context ------------------------------------------------------ */
int m3tsz_version(void);
const char *m3tsz_status_string(int status);
/* Creates a context bound to CUDA device `device`.  Fails with
 * M3TSZ_ERR_NO_DEVICE when there is no GPU: there is no CPU code path. */
int m3tsz_ctx_create(int device, m3tsz_ctx **out);
void m3tsz_ctx_destroy(m3tsz_ctx *ctx);
const char *m3tsz_last_cuda_error(const m3tsz_ctx *ctx);
/* Number of kernel launches this context has issued (bench "gpu_launches"). */
uint64_t m3tsz_ctx_launch_count(const m3tsz_ctx *ctx);

/* First annotation seen in a stream (ReaderIterator.Current()'s ts.Annotation,
 * encoding/types.go:184-187): bit offset of its first payload byte from the
 * start of the stream, its length in bytes, and how many annotations the
 * stream holds in total. */
typedef struct m3tsz_annotation_ref {
  uint64_t bit_offset;
  uint32_t length;
  uint32_t count;
} m3tsz_annotation_ref;

/* Per-datapoint unit and annotation (ReaderIterator.Current() returns
 * (datapoint, unit, annotation) for EVERY datapoint, encoding/types.go:184-187,
 * m3tsz/iterator.go:229-231).  Both change rarely, so the decoder reports them as
 * an event table instead of two dense [n_series][max_points] arrays:
 *   M3TSZ_EVENT_TIME_UNIT  : from datapoint dp_index on, the unit in force is `unit`
 *                            (a time-unit marker, timestamp_iterator.go:118-134; the unit of
 *                            datapoint 0 is reported per series in d_unit_first)
 *   M3TSZ_EVENT_ANNOTATION : datapoint dp_index carries an annotation of `length` bytes whose
 *                            first payload bit is `bit_offset` bits after the start of the stream
 *                            (timestamp_iterator.go:328-356); datapoints without an event have none.
 * Events of one series appear in stream order but interleaved with other series';
 * events whose dp_index >= n_points[series] belong to a datapoint that failed to decode. */
enum { M3TSZ_EVENT_TIME_UNIT = 1, M3TSZ_EVENT_ANNOTATION = 2 };
typedef struct m3tsz_dp_event {
  uint64_t series;
  uint32_t dp_index;
  uint16_t kind;
  uint16_t unit;
  uint64_t bit_offset;
  uint32_t length;
  uint32_t reserved;
} m3tsz_dp_event;

/* Optional inputs / outputs of m3tsz_decode_batch_ex (all may be NULL / 0). */
typedef struct m3tsz_decode_extras {
  const uint64_t *d_lengths; /* [n_series] exact stream sizes: stream s = [d_offsets[s], +d_lengths[s]);
                                lets the streams sit anywhere in d_streams (index-entry (Offset, Size),
                                persist/schema/types.go:70-78); d_offsets then needs n_series entries */
  uint8_t *d_unit_first;     /* [n_series] unit in force at the first datapoint */
  m3tsz_dp_event *d_events;  /* event table, events_capacity entries */
  uint64_t events_capacity;
  uint64_t *d_event_count;   /* required with d_events; must be zero on entry; receives the number of
                                events produced (may exceed events_capacity: re-run with a larger table) */
  int32_t point_major;       /* != 0: d_ts / d_val are POINT-major, [max_points][n_series] (datapoint i of
                                series s at i * n_series + s) -- the step-major layout the query engine's
                                step iterators consume (src/query/storage/m3/encoded_step_iterator_generic.go),
                                like the downsample outputs.  Every decode step then stores 32 consecutive
                                elements per warp (coalesced 256-byte rows) instead of 32 separate 32-byte
                                sectors; rows >= n_points[s] of a series are left untouched. */
  int32_t reserved;
} m3tsz_decode_extras;

/* ------------------------------------------------------------------------
 * Batch decode.  Replaces, for n_series independent streams, the loop
 *   it := m3tsz.NewReaderIterator(reader, intOptimized, opts)   m3tsz/iterator.go:67-78
 *   for it.Next() { dp, unit, ann := it.Current() }             m3tsz/iterator.go:81-106,229-231
 * i.e. the per-series bodies of src/query/storage/prom_converter.go:65-110 and
 * src/query/storage/m3/encoded_series_iterator.go:94-120.
 *
 * d_streams : all streams concatenated (16-byte aligned base); stream s is
 *             bytes [d_offsets[s], d_offsets[s+1]) = ts.Segment head||tail.
 * d_ts/d_val: [n_series][max_points] (series-major); d_val receives float64.
 * d_n_points: datapoints decoded per series (may exceed max_points =>
 *             status M3TSZ_ERR_CAPACITY, first max_points are stored).
 * d_status  : per-series iterator Err() (M3TSZ_OK on a clean end-of-stream).
 * d_unit    : optional [n_series], time unit in force at the last datapoint.
 * d_ann     : optional [n_series], first annotation reference.
 * Limits (M3TSZ_ERR_INVALID_ARG beyond): streams_bytes < 2^34, max_points < 2^27,
 * one stream < 2^28 bytes (M3TSZ_ERR_STREAM_TOO_LARGE for that series); split
 * larger batches.  Stream starts may have any alignment; 64-byte aligned starts
 * (m3tsz_compact_streams with align = 64) decode fastest.  Outputs are stored as
 * whole 32-byte sectors when d_ts / d_val are 32-byte aligned and max_points is a
 * multiple of 4 (any other shape is stored row by row: same result, slower).
 * ---------------------------------------------------------------------- */
int m3tsz_decode_batch(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams,
                       uint64_t streams_bytes, const uint64_t *d_offsets, uint64_t n_series,
                       int64_t *d_ts, double *d_val, uint64_t max_points, uint32_t *d_n_points,
                       int32_t *d_status, uint8_t *d_unit, m3tsz_annotation_ref *d_ann,
                       void *stream);

/* m3tsz_decode_batch + the optional per-datapoint unit / annotation events and
 * non-CSR stream placement (extras may be NULL). */
int m3tsz_decode_batch_ex(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams,
                          uint64_t streams_bytes, const uint64_t *d_offsets, uint64_t n_series,
                          int64_t *d_ts, double *d_val, uint64_t max_points, uint32_t *d_n_points,
                          int32_t *d_status, uint8_t *d_unit, m3tsz_annotation_ref *d_ann,
                          const m3tsz_decode_extras *extras, void *stream);

/* Same call with HOST buffers (pageable or pinned): copies the streams and
 * offsets to the device, decodes, copies the results back, synchronises. */
int m3tsz_decode_batch_host(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *h_streams,
                            uint64_t streams_bytes, const uint64_t *h_offsets, uint64_t n_series,
                            int64_t *h_ts, double *h_val, uint64_t max_points,
                            uint32_t *h_n_points, int32_t *h_status, uint8_t *h_unit,
                            m3tsz_annotation_ref *h_ann);

/* ------------------------------------------------------------------------
 * Batch encode.  Replaces, for n_series independent series, the loop
 *   enc.Reset(start, capacity, schema)                          m3tsz/encoder.go:262-279
 *   for each dp { enc.Encode(dp, unit, annotation) }            m3tsz/encoder.go:90-110
 *   seg := enc.Discard()                                        m3tsz/encoder.go:374-381
 * at the batch re-encode sites src/dbnode/storage/series/buffer.go:1543-1573,
 * 583-610, src/dbnode/persist/fs/merger.go:333-356.
 *
 * d_ts/d_val : [n_series][points_stride] series-major inputs.
 * d_n_points : optional [n_series]; NULL => every series has points_stride points.
 * d_start    : [n_series] encoder start (block start), ns.
 * unit       : time unit passed to every Encode call; d_units (optional,
 *              [n_series][points_stride] bytes) overrides it per datapoint.
 * annotations: optional sparse list: entries [d_ann_series_off[s], d_ann_series_off[s+1])
 *              belong to series s, sorted by dp_index; bytes in d_ann_bytes.
 * d_out      : [n_series][out_stride] bytes (out_stride % 16 == 0); series s
 *              gets its final stream (head||tail incl. end-of-stream marker)
 *              at d_out + s*out_stride, length d_out_len[s].
 * d_status   : per-series first Encode() error (encoding stops at that point;
 *              d_out_len then covers the datapoints before the error, like the
 *              reference's numEncoded), or M3TSZ_ERR_CAPACITY.
 * ---------------------------------------------------------------------- */
typedef struct m3tsz_annotation_entry {
  uint32_t dp_index;
  uint32_t length;
  uint64_t byte_offset; /* into d_ann_bytes */
} m3tsz_annotation_entry;

int m3tsz_encode_batch(m3tsz_ctx *ctx, const m3tsz_options *opts, const int64_t *d_ts,
                       const double *d_val, uint64_t n_series, uint64_t points_stride,
                       const uint32_t *d_n_points, const int64_t *d_start, int32_t unit,
                       const uint8_t *d_units, const uint64_t *d_ann_series_off,
                       const m3tsz_annotation_entry *d_ann_entries, const uint8_t *d_ann_bytes,
                       uint8_t *d_out, uint64_t out_stride, uint64_t *d_out_len, int32_t *d_status,
                       void *stream);

/* m3tsz_encode_batch + optional per-series encoder state that the reference's accessors
 * expose (extras may be NULL):
 *   d_last_value: Encoder.LastEncoded().Value (encoder.go:305-319) -- the float in float mode,
 *                 else the encoder's intVal: the SCALED integer in int mode and 0 when
 *                 int_optimized == 0 (the reference never sets isFloat there);
 *   point_major_input: see the struct;
 *   d_out_bits  : stream length in bits incl. the end-of-stream marker, before the zero
 *                 padding (splits the bytes into ts.Segment head / tail: the tail is the
 *                 last ceil((pos + 11) / 8) bytes, pos = ((bits - 12) mod 8) + 1,
 *                 scheme.go:198-211). */
typedef struct m3tsz_encode_extras {
  double *d_last_value;
  uint64_t *d_out_bits;
  int32_t point_major_input; /* != 0: d_ts / d_val are POINT-major, [points_stride][n_series] (datapoint i of
                                series s at i * n_series + s; the layout m3tsz_decode_batch_ex writes with
                                extras.point_major): every encode step reads 32 consecutive elements per warp,
                                no shared-memory staging.  Per-datapoint units and annotations are not
                                supported with it (M3TSZ_ERR_INVALID_ARG). */
  int32_t reserved;
} m3tsz_encode_extras;
int m3tsz_encode_batch_ex(m3tsz_ctx *ctx, const m3tsz_options *opts, const int64_t *d_ts,
                          const double *d_val, uint64_t n_series, uint64_t points_stride,
                          const uint32_t *d_n_points, const int64_t *d_start, int32_t unit,
                          const uint8_t *d_units, const uint64_t *d_ann_series_off,
                          const m3tsz_annotation_entry *d_ann_entries, const uint8_t *d_ann_bytes,
                          uint8_t *d_out, uint64_t out_stride, uint64_t *d_out_len, int32_t *d_status,
                          const m3tsz_encode_extras *extras, void *stream);

/* Worst-case stream bytes for n points without annotations (rounded up to 16),
 * for a batch-wide unit (m3tsz_encode_bound) or with per-datapoint units
 * (d_units given: every datapoint may add a time-unit marker and a raw 64-bit
 * delta-of-delta, timestamp_encoder.go:130-164,197-205). */
uint64_t m3tsz_encode_bound(uint64_t n_points);
uint64_t m3tsz_encode_bound_units(uint64_t n_points, int per_datapoint_units);

/* ------------------------------------------------------------------------
 * Encoder sets: n_series OPEN encoders that live on the device and take datapoints over many calls -- the write
 * path BufferBucket.write -> encoder.Encode(dp, unit, annotation) (src/dbnode/storage/series/buffer.go:1261-1364)
 * for thousands of series per call, plus Stream() snapshots for readers of the open block (buffer.go:1366-1391,
 * m3tsz/encoder.go:282-297).
 *
 * One open encoder = one 128-byte m3tsz_encoder_state in caller-owned device memory (16-byte aligned) plus one
 * slot of buf_stride bytes in a caller-owned [n_series][buf_stride] buffer (buf_stride % 16 == 0; a multiple of
 * 32 makes every write a whole 32-byte sector).  The state holds positions, never pointers, so a caller whose
 * slots are full copies [n][stride] into a larger [n][stride2] buffer (each slot's first stride bytes) and goes on
 * appending with stride2.
 *
 * The slot only ever receives whole 32-byte sectors of the stream (at most 7 words plus the partial word wait in
 * the state); a snapshot writes the rest at the committed position.
 * ---------------------------------------------------------------------- */
typedef struct m3tsz_encoder_state {
  int64_t start_ns;      /* Reset(start), encoder.go:262-279 */
  uint64_t num_encoded;  /* NumEncoded(), encoder.go:299-302 */
  int64_t last_ts;       /* LastEncoded().TimestampNanos (valid when num_encoded > 0) */
  double last_value;     /* LastEncoded().Value incl. the scaled-int / 0 quirk (as m3tsz_encode_extras.d_last_value) */
  uint64_t ann_checksum; /* LastAnnotationChecksum(): XXH64 of the last annotation written, encoder.go:321-327 */
  uint64_t bits;         /* stream bits so far, before the tail: Len() = num_encoded ? ceil((bits + 11) / 8) : 0 */
  uint64_t internal[10]; /* codec state, opaque */
} m3tsz_encoder_state;

/* Reset(start) of every encoder of the set (encoder.go:262-279): empty streams, d_start [n_series] ns.  The state
 * records opts->int_optimized; the other calls refuse a state reset in the other mode. */
int m3tsz_encoder_set_reset(m3tsz_ctx *ctx, const m3tsz_options *opts, m3tsz_encoder_state *d_state,
                            uint64_t n_series, const int64_t *d_start, void *stream);

/* Appends d_n_points[s] (NULL: points_stride each; 0 leaves the encoder and its slot untouched) datapoints to
 * encoder s, one launch for the whole set.  Inputs as m3tsz_encode_batch_ex: series-major [n][points_stride], or
 * point-major [points_stride][n] when point_major_input != 0 (then d_units and annotations must be NULL), unit /
 * d_units, the sparse annotation list (dp_index counts within this call).  An annotation is written when its
 * XXH64 differs from the state's ann_checksum, as the reference decides.
 *
 * A series stops at its first datapoint that fails: d_status[s] = M3TSZ_ERR_DOD_OVERFLOW,
 * M3TSZ_ERR_UNRECOGNIZED_UNIT, M3TSZ_ERR_CAPACITY (the slot cannot hold 56 bytes past the stream so far -- the
 * datapoint's worst case plus a snapshot tail -- and its annotation rounded up to 4 bytes + 16) or
 * M3TSZ_ERR_INVALID_ARG (a state reset with the
 * other int_optimized, or n_points > points_stride).  d_n_appended[s] counts the datapoints taken; state and
 * slot are then exactly as after the last one taken (nothing of the failing datapoint is written), so dropping
 * it and appending the rest gives the stream of the sequence without it. */
int m3tsz_encoder_set_append(m3tsz_ctx *ctx, const m3tsz_options *opts, m3tsz_encoder_state *d_state,
                             uint64_t n_series, const int64_t *d_ts, const double *d_val, uint64_t points_stride,
                             const uint32_t *d_n_points, int32_t unit, const uint8_t *d_units,
                             const uint64_t *d_ann_series_off, const m3tsz_annotation_entry *d_ann_entries,
                             const uint8_t *d_ann_bytes, int32_t point_major_input, uint8_t *d_buf,
                             uint64_t buf_stride, uint32_t *d_n_appended, int32_t *d_status, void *stream);

/* Stream() of every encoder without closing it: writes the tail (the state's leftover words, end-of-stream marker,
 * zero pad) at the committed position, so that d_buf[s * buf_stride, + d_len[s]) is the reference's head || tail,
 * d_len[s] = 0 for an empty encoder.  The state is unchanged; the next append overwrites the tail.  The snapshot
 * decodes with m3tsz_decode_batch_ex (d_offsets[s] = s * buf_stride, extras.d_lengths = d_len) and packs with
 * m3tsz_compact_streams (slot_stride = buf_stride). */
int m3tsz_encoder_set_stream(m3tsz_ctx *ctx, const m3tsz_encoder_state *d_state, uint64_t n_series,
                             uint8_t *d_buf, uint64_t buf_stride, uint64_t *d_len, void *stream);

/* ------------------------------------------------------------------------
 * Buffer buckets: BufferBucket.write (src/dbnode/storage/series/buffer.go:1261-1364) for n_series buckets per call.
 * A bucket holds up to n_encoders (K, 1..M3TSZ_MAX_BUCKET_ENCODERS) in-order encoders; K plays the role of
 * EncodersPerBlockLimit.  Encoder 0 of series s is record s of an encoder set (d_state / d_buf, reset with
 * m3tsz_encoder_set_reset; append / stream keep working on it).  Encoders 1..K-1 are opened on demand from an
 * overflow pool: d_pool_state [pool_capacity] + d_pool_buf [pool_capacity][pool_stride], *d_pool_count records in
 * use, and d_table [n_series][K-1] (int32) naming the pool record of encoder i + 1 (-1: not open).  Resetting the
 * pool is *d_pool_count = 0 and d_table = -1; all of it holds positions, not pointers, so growing is a copy.  With
 * K = 1 the pool arguments may be NULL / 0.
 *
 * The datapoints of one call are processed in call order, one write each: the first encoder whose last write is
 * before the datapoint takes it; a datapoint equal to an encoder's last write (timestamp, LastEncoded().Value --
 * the scaled int in int-optimised mode, 0 without it -- and the checksum of the last annotation written) is a
 * no-op; otherwise a new encoder is opened (start = encoder 0's start_ns), or the write fails with
 * M3TSZ_ERR_TOO_MANY_ENCODERS when K are open.  A t == 0 datapoint on an empty encoder 0 fails with
 * M3TSZ_ERR_NO_DATAPOINTS (LastEncoded errors); DOD_OVERFLOW / UNRECOGNIZED_UNIT are decided against the target
 * encoder.  A failed write changes nothing and later datapoints of the call go on.
 *
 * Inputs as m3tsz_encoder_set_append.  d_result (int8, the inputs' layout): 0 written, -1 unchanged, else the
 * failed write's status (3, 4, 6, 16, or 100 = M3TSZ_ERR_CAPACITY).  d_status[s]: M3TSZ_OK; M3TSZ_ERR_CAPACITY when
 * the target's slot lacks room for the datapoint (the bound of m3tsz_encoder_set_append, with every earlier
 * datapoint of the call counted at its worst case: a slot of m3tsz_encode_bound_units(P, 1) bytes takes P) or no
 * pool record is free -- that datapoint and every later one of the series get CAPACITY and nothing of them is
 * written, so growing and re-sending exactly those gives the unstopped result; or M3TSZ_ERR_INVALID_ARG (encoder 0
 * reset in the other mode, or n_points > points_stride): the series is untouched and its d_result not written.
 * ---------------------------------------------------------------------- */
#define M3TSZ_MAX_BUCKET_ENCODERS 12
int m3tsz_encoder_set_write(m3tsz_ctx *ctx, const m3tsz_options *opts, m3tsz_encoder_state *d_state, uint8_t *d_buf,
                            uint64_t buf_stride, uint64_t n_series, m3tsz_encoder_state *d_pool_state,
                            uint8_t *d_pool_buf, uint64_t pool_stride, uint64_t pool_capacity, uint32_t *d_pool_count,
                            int32_t *d_table, int32_t n_encoders, const int64_t *d_ts, const double *d_val,
                            uint64_t points_stride, const uint32_t *d_n_points, int32_t unit, const uint8_t *d_units,
                            const uint64_t *d_ann_series_off, const m3tsz_annotation_entry *d_ann_entries,
                            const uint8_t *d_ann_bytes, int32_t point_major_input, int8_t *d_result,
                            int32_t *d_status, void *stream);

/* ------------------------------------------------------------------------
 * Batch encode straight into ONE packed buffer (the fileset data-file layout,
 * src/dbnode/persist/fs/write.go: concatenated segments + index entries that
 * carry (Offset, Size), persist/schema/types.go:70-78) -- no per-series slots,
 * no separate compaction pass.  Same inputs as m3tsz_encode_batch.  Stream s is
 *   d_packed[d_offsets[s] .. d_offsets[s] + d_out_len[s])
 * with every start rounded up to `align` bytes (1,4,8,16,32,64; >= 16 copies
 * fastest, 64 decodes fastest).  Streams are placed in completion order, NOT in
 * series order: d_offsets has n_series entries and is not monotonic; decode with
 * m3tsz_decode_batch_ex (extras.d_lengths = d_out_len).  *d_total_bytes (device)
 * receives the bytes used; a series that does not fit packed_capacity gets
 * M3TSZ_ERR_CAPACITY and length 0.  slot_bytes = per-series staging bound (0 =
 * m3tsz_encode_bound_units(points_stride, d_units != NULL); add the annotation
 * bytes of the largest series when annotations are given).  d_packed must be
 * 64-byte aligned.  The context keeps the staging slots (resident warps x 32 x
 * slot_bytes: proportional to the SM count), reused by every call.
 * ---------------------------------------------------------------------- */
int m3tsz_encode_batch_packed(m3tsz_ctx *ctx, const m3tsz_options *opts, const int64_t *d_ts,
                              const double *d_val, uint64_t n_series, uint64_t points_stride,
                              const uint32_t *d_n_points, const int64_t *d_start, int32_t unit,
                              const uint8_t *d_units, const uint64_t *d_ann_series_off,
                              const m3tsz_annotation_entry *d_ann_entries, const uint8_t *d_ann_bytes,
                              uint64_t slot_bytes, uint32_t align, uint8_t *d_packed,
                              uint64_t packed_capacity, uint64_t *d_offsets, uint64_t *d_out_len,
                              int32_t *d_status, uint64_t *d_total_bytes, void *stream);
/* ... with the optional extras of m3tsz_encode_batch_ex: point-major inputs
 * (extras->point_major_input: d_ts / d_val are [points_stride][n_series], no per-datapoint
 * units / annotations), LastEncoded values, stream bit lengths. */
int m3tsz_encode_batch_packed_ex(m3tsz_ctx *ctx, const m3tsz_options *opts, const int64_t *d_ts,
                                 const double *d_val, uint64_t n_series, uint64_t points_stride,
                                 const uint32_t *d_n_points, const int64_t *d_start, int32_t unit,
                                 const uint8_t *d_units, const uint64_t *d_ann_series_off,
                                 const m3tsz_annotation_entry *d_ann_entries, const uint8_t *d_ann_bytes,
                                 uint64_t slot_bytes, uint32_t align, uint8_t *d_packed,
                                 uint64_t packed_capacity, uint64_t *d_offsets, uint64_t *d_out_len,
                                 int32_t *d_status, uint64_t *d_total_bytes,
                                 const m3tsz_encode_extras *extras, void *stream);

/* Packs the per-series slots written by m3tsz_encode_batch into one contiguous
 * buffer (the fileset data-file layout, src/dbnode/persist/fs/write.go): fills
 * d_offsets[n_series+1] (exclusive prefix sum of d_out_len, each start rounded
 * up to `align` bytes, align in {1,4,8,16,32,64}) and copies the bytes.  64-byte
 * aligned starts let the decoder's lanes read their staging rings in phase (fewer
 * shared-memory bank conflicts); any alignment decodes to the same result.
 * Blocks the host: it reads the capacity flag back, so it returns once `stream`
 * has run the whole call. */
int m3tsz_compact_streams(m3tsz_ctx *ctx, const uint8_t *d_slots, uint64_t slot_stride,
                          const uint64_t *d_len, uint64_t n_series, uint32_t align,
                          uint8_t *d_packed, uint64_t packed_capacity, uint64_t *d_offsets,
                          void *stream);

/* Host-buffer encode: copies the inputs to the device, encodes, packs the
 * streams on the device (m3tsz_compact_streams, `align`-byte aligned starts)
 * and copies back ONE contiguous buffer + CSR offsets -- the fileset data-file
 * layout -- so that only compressed bytes cross PCIe.  h_offsets has
 * n_series+1 entries; stream s is h_packed[h_offsets[s] .. +h_out_len[s]). */
int m3tsz_encode_batch_host(m3tsz_ctx *ctx, const m3tsz_options *opts, const int64_t *h_ts,
                            const double *h_val, uint64_t n_series, uint64_t points_stride,
                            const uint32_t *h_n_points, const int64_t *h_start, int32_t unit,
                            const uint8_t *h_units, const uint64_t *h_ann_series_off,
                            const m3tsz_annotation_entry *h_ann_entries,
                            const uint8_t *h_ann_bytes, uint64_t ann_bytes_len, uint32_t align,
                            uint8_t *h_packed, uint64_t packed_capacity, uint64_t *h_offsets,
                            uint64_t *h_out_len, int32_t *h_status);

/* ------------------------------------------------------------------------
 * Fused decode + downsample (BASELINE config 4).  Decodes every stream and
 * folds each datapoint into fixed windows with the reference aggregator's
 * Gauge arithmetic: aggregation.Gauge.updateTotals
 * (src/aggregator/aggregation/gauge.go:73-106: count++ always; NaN skipped for
 * sum/min/max; min/max start NaN; sum added in arrival order), window index =
 * floor((ts - range_start) / window) as timestamp.Truncate(resolution) does
 * (src/aggregator/aggregator/generic_elem.go:220).  Datapoints outside
 * [range_start, range_start + n_windows*window) are ignored.
 *
 * Outputs are WINDOW-major: element (series s, window w) at [w*n_series + s]
 * (step-major, the layout the query engine's step iterators consume,
 * src/query/storage/m3/encoded_step_iterator_generic.go).
 * ---------------------------------------------------------------------- */
int m3tsz_decode_downsample_batch(m3tsz_ctx *ctx, const m3tsz_options *opts,
                                  const uint8_t *d_streams, uint64_t streams_bytes,
                                  const uint64_t *d_offsets, uint64_t n_series,
                                  int64_t range_start_ns, int64_t window_ns, uint32_t n_windows,
                                  double *d_sum, int64_t *d_count, double *d_min, double *d_max,
                                  uint32_t *d_n_points, int32_t *d_status, void *stream);

/* Same, plus Gauge.Last() per window (gauge.go:73-84: the value with the latest
 * timestamp, first arrival among equal timestamps; 0 for an empty window) in
 * d_last, and optionally Gauge.LastAt() (ns; 0 for an empty window) in d_last_at
 * (NULL: the context keeps it in scratch -- it is what lets an out-of-order
 * datapoint re-open a committed window exactly).  Gauge.Mean() = sum / count
 * (0 when count == 0) is left to the consumer (gauge.go:117-122). */
int m3tsz_decode_downsample_last_batch(m3tsz_ctx *ctx, const m3tsz_options *opts,
                                       const uint8_t *d_streams, uint64_t streams_bytes,
                                       const uint64_t *d_offsets, uint64_t n_series,
                                       int64_t range_start_ns, int64_t window_ns, uint32_t n_windows,
                                       double *d_sum, int64_t *d_count, double *d_min, double *d_max,
                                       double *d_last, int64_t *d_last_at, uint32_t *d_n_points,
                                       int32_t *d_status, void *stream);

/* ------------------------------------------------------------------------
 * Fused decode + downsample for either metric type the aggregator keeps per
 * window (src/aggregator/aggregation): the same decode, windows and
 * out-of-order handling as m3tsz_decode_downsample_last_batch, one outputs
 * struct.  metric_type is the reference's metric.Type id
 * (src/metrics/metric/types.go:35-38):
 *
 *   M3TSZ_METRIC_GAUGE: aggregation.Gauge (gauge.go:73-106).  d_sum, d_count,
 *     d_min, d_max are required.  d_sum_sq asks for the Gauge with expensive
 *     aggregations: sumSq += v*v after the NaN check, multiply and add rounded
 *     separately, 0 for an empty window.  d_last / d_last_at as in
 *     m3tsz_decode_downsample_last_batch (with d_sum_sq, a NULL d_last or
 *     d_last_at is kept in context scratch).  The counter_* fields must be NULL.
 *   M3TSZ_METRIC_COUNTER: aggregation.Counter (counter.go:44-78) fed
 *     int64(value) with Go/amd64 semantics (truncation toward zero; NaN, +-Inf
 *     and values outside [-2^63, 2^63) give MinInt64), as the coordinator's
 *     ingest does (src/cmd/services/m3coordinator/ingest/write.go:560-567).
 *     int64 sum / min / max / sumSq, wrapping like Go; an empty window has sum 0,
 *     sumSq 0, count 0, min MaxInt64, max MinInt64.  d_count, d_counter_sum,
 *     d_counter_min, d_counter_max are required, d_counter_sum_sq is optional
 *     (context scratch when NULL); the Gauge fields must be NULL.
 *
 * Every output is window-major [n_windows][n_series].  d_n_points / d_status
 * are optional, as in the other downsample calls.  d_lengths may be NULL (CSR
 * offsets) or give stream s = [d_offsets[s], d_offsets[s] + d_lengths[s]).
 * Missing, mixed or unknown fields / metric types: M3TSZ_ERR_INVALID_ARG
 * before any launch.
 * ---------------------------------------------------------------------- */
enum { /* metric.Type ids, src/metrics/metric/types.go:35-38 */
  M3TSZ_METRIC_COUNTER = 1,
  M3TSZ_METRIC_TIMER = 2, /* element sets only (m3tsz_element_set_add_timer); every other call refuses it */
  M3TSZ_METRIC_GAUGE = 3
};
typedef struct m3tsz_downsample_outputs {
  int32_t metric_type;
  int32_t reserved;     /* 0 */
  /* Gauge */
  double *d_sum;
  double *d_min;
  double *d_max;
  double *d_sum_sq;
  double *d_last;
  int64_t *d_last_at;
  /* both */
  int64_t *d_count;
  /* Counter */
  int64_t *d_counter_sum;
  int64_t *d_counter_min;
  int64_t *d_counter_max;
  int64_t *d_counter_sum_sq;
  /* per series */
  uint32_t *d_n_points;
  int32_t *d_status;
} m3tsz_downsample_outputs;
int m3tsz_decode_downsample_ex(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams,
                               uint64_t streams_bytes, const uint64_t *d_offsets, const uint64_t *d_lengths,
                               uint64_t n_series, int64_t range_start_ns, int64_t window_ns, uint32_t n_windows,
                               const m3tsz_downsample_outputs *out, void *stream);

int m3tsz_decode_downsample_batch_host(m3tsz_ctx *ctx, const m3tsz_options *opts,
                                       const uint8_t *h_streams, uint64_t streams_bytes,
                                       const uint64_t *h_offsets, uint64_t n_series,
                                       int64_t range_start_ns, int64_t window_ns,
                                       uint32_t n_windows, double *h_sum, int64_t *h_count,
                                       double *h_min, double *h_max, uint32_t *h_n_points,
                                       int32_t *h_status);

/* ------------------------------------------------------------------------
 * Segment checksums (SURVEY.md §8f N2: fileset ingestion).  The fileset data file
 * is the concatenated streams and every index entry carries (Offset, Size,
 * DataChecksum) (src/dbnode/persist/schema/types.go:70-78) -- i.e. this library's
 * CSR layout plus the Adler-32 that the reference verifies on every read:
 *   ts.Segment.CalculateChecksum  src/dbnode/ts/segment.go:60-76  (head then tail)
 *   digest.Checksum               src/dbnode/digest/digest.go:36-38
 *   check                         src/dbnode/persist/fs/read.go:395-397, seek.go:370-373
 * Computes the Adler-32 of every stream [d_offsets[s], d_offsets[s+1]) -- or
 * [d_offsets[s], d_offsets[s] + d_lengths[s]) when d_lengths is given (index-entry
 * (Offset, Size) addressing: any placement and order, d_offsets then needs only
 * n_series entries) -- into d_checksums (optional) and, when d_expected (the index entries'
 * DataChecksum) is given, sets d_status[s] to M3TSZ_ERR_CHECKSUM_MISMATCH where
 * it differs.  One of d_checksums / d_status is required.
 * ---------------------------------------------------------------------- */
int m3tsz_checksum_batch(m3tsz_ctx *ctx, const uint8_t *d_streams, uint64_t streams_bytes,
                         const uint64_t *d_offsets, const uint64_t *d_lengths, uint64_t n_series,
                         const uint32_t *d_expected, uint32_t *d_checksums, int32_t *d_status,
                         void *stream);

/* ------------------------------------------------------------------------
 * Series merge: the iterator layer directly above the codec (SURVEY.md §8f N1).
 * For every series, merges the DECODED streams of its replicas / blocks exactly
 * like the reference's seriesIterator over multiReaderIterators:
 *   iterators            src/dbnode/encoding/iterators.go:56-262
 *   multiReaderIterator  src/dbnode/encoding/multi_reader_iterator.go:62-155
 *   seriesIterator       src/dbnode/encoding/series_iterator.go:74-83,129-215
 * i.e. k-way timestamp merge, equal-timestamp strategy (0 last-pushed = default,
 * 1 highest value, 2 lowest value, 3 highest frequency; encoding/iterators_types.go),
 * removal of consecutive equal timestamps, [start_ns, end_ns) filter (both 0 = no
 * filter), errOutOfOrderIterator, propagation of reader (decode) errors.
 *
 * Inputs are the outputs of m3tsz_decode_batch over n_seq streams:
 *   sequence q = (d_ts + q*cap, d_val + q*cap, d_n_points[q], d_seq_status[q])
 *   slice k    = sequences [d_slice_off[k], d_slice_off[k+1])  readers of one block
 *   replica r  = slices    [d_replica_off[r], d_replica_off[r+1])  in block order
 *   series s   = replicas  [d_series_off[s], d_series_off[s+1])
 * Outputs: merged datapoints [n_series][out_cap], count, status per series.
 * ---------------------------------------------------------------------- */
int m3tsz_merge_series_batch(m3tsz_ctx *ctx, const int64_t *d_ts, const double *d_val, uint64_t cap,
                             const uint32_t *d_n_points, const int32_t *d_seq_status,
                             const uint64_t *d_slice_off, const uint64_t *d_replica_off,
                             const uint64_t *d_series_off, uint64_t n_series, int64_t start_ns,
                             int64_t end_ns, int32_t strategy, int64_t *d_ts_out, double *d_val_out,
                             uint64_t out_cap, uint32_t *d_n_out, int32_t *d_status, void *stream);

/* ------------------------------------------------------------------------
 * Fetch with HOST buffers: decode + series merge in one call, so that only the
 * COMPRESSED replica streams go up over PCIe and only the MERGED series come back
 * (the decoded replicas, 16 B per datapoint and replica, never leave the device).
 * Same structure arguments as m3tsz_merge_series_batch, over the streams
 * h_offsets[q] .. h_offsets[q+1] of sequence q (sequences of one series must be
 * consecutive: the call works through chunks of whole series on two CUDA streams,
 * H2D / decode / merge / D2H overlapped).  max_points = decode capacity per
 * sequence; outputs [n_series][out_cap] + h_n_out + h_status as m3tsz_merge_series_batch.
 * ---------------------------------------------------------------------- */
int m3tsz_fetch_batch_host(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *h_streams,
                           uint64_t streams_bytes, const uint64_t *h_offsets, uint64_t n_seq,
                           const uint64_t *h_slice_off, const uint64_t *h_replica_off,
                           const uint64_t *h_series_off, uint64_t n_series, uint64_t max_points,
                           int64_t start_ns, int64_t end_ns, int32_t strategy, int64_t *h_ts_out,
                           double *h_val_out, uint64_t out_cap, uint32_t *h_n_out, int32_t *h_status);

/* ------------------------------------------------------------------------
 * Prometheus conversion epilogue (SURVEY.md §8f N4): iteratorToPromResult,
 * src/query/storage/prom_converter.go:42-120, over decoded / merged series that are
 * already in HBM -- the last per-datapoint host loop of a fetch:
 *   - timestamps ns -> ms (TimeToPromTimestamp, converter.go:388-391, truncating);
 *   - value_decrease_tolerance > 0: a value that dips below its predecessor by less
 *     than the tolerance, before tolerance_until_ns, is replaced by the predecessor
 *     (the replaced value is the next predecessor), :68-72;
 *   - d_handle_resets[s] != 0 (the host sets it when the series' first annotation says
 *     OpenMetricsHandleValueResets and maxResolution >= the normalisation threshold,
 *     :74-82): one sample per resolution_ns window holding the reset-aware cumulative
 *     sum, stamped with the window's last datapoint, :84-98,113-118.
 * Inputs [n_series][cap] + d_n_points; outputs [n_series][out_cap] + d_n_out (the
 * number of samples; > out_cap => d_status M3TSZ_ERR_CAPACITY, first out_cap stored).
 * A series with d_n_points[s] > cap (a decode or merge row that hit its capacity) is
 * refused: d_status M3TSZ_ERR_INVALID_ARG, d_n_out 0, nothing of its input row read and
 * nothing of its output row written; the other series are converted as usual.
 * d_handle_resets and d_status may be NULL.  In-place (outputs == inputs, out_cap ==
 * cap) is allowed.
 * ---------------------------------------------------------------------- */
int m3tsz_prom_convert_batch(m3tsz_ctx *ctx, const int64_t *d_ts, const double *d_val, uint64_t cap,
                             const uint32_t *d_n_points, uint64_t n_series, int64_t resolution_ns,
                             const uint8_t *d_handle_resets, double value_decrease_tolerance,
                             int64_t tolerance_until_ns, int64_t *d_ts_ms_out, double *d_val_out,
                             uint64_t out_cap, uint32_t *d_n_out, int32_t *d_status, void *stream);

/* ------------------------------------------------------------------------
 * Tile aggregation (SURVEY.md §8f N3): the compute of a storage.TileAggregator
 * (src/dbnode/storage/types.go:1444-1472, AggregateTilesOptions{Start, End, Step};
 * the open-source default is a no-op, storage/options.go:949-951).  For every
 * source stream: decode, fold the datapoints of [start_ns, start_ns + n_windows *
 * step_ns) into step-sized windows with the aggregator's Gauge
 * (aggregation/gauge.go:73-106), emit one datapoint per NON-EMPTY window --
 * timestamp = the window's end boundary (aggregator/list.go:541-543), value =
 * Gauge.ValueOf(agg_type) (gauge.go:144-165) -- and re-encode them as the target
 * namespace's M3TSZ stream (encoder start = start_ns, unit = out_unit), straight
 * into one packed buffer (layout of m3tsz_encode_batch_packed: d_out_offsets[s],
 * d_out_len[s], *d_total_bytes).  d_lengths may be NULL (CSR offsets).
 * d_status[s]: the source stream's decode error if any (no output for that series),
 * else the encoder's status.  d_n_tiles (optional): datapoints written per series.
 * ---------------------------------------------------------------------- */
enum { /* aggregation.Type ids, src/metrics/aggregation/type.go:31-38 */
  M3TSZ_AGG_LAST = 1,
  M3TSZ_AGG_MIN = 2,
  M3TSZ_AGG_MAX = 3,
  M3TSZ_AGG_MEAN = 4,
  M3TSZ_AGG_MEDIAN = 5, /* Timer element sets only, as are the quantile types below */
  M3TSZ_AGG_COUNT = 6,
  M3TSZ_AGG_SUM = 7,
  M3TSZ_AGG_SUMSQ = 8, /* m3tsz_aggregate_tiles_ex only */
  M3TSZ_AGG_STDEV = 9, /* m3tsz_aggregate_tiles_ex only */
  M3TSZ_AGG_P10 = 10,
  M3TSZ_AGG_P20 = 11,
  M3TSZ_AGG_P30 = 12,
  M3TSZ_AGG_P40 = 13,
  M3TSZ_AGG_P50 = 14,
  M3TSZ_AGG_P60 = 15,
  M3TSZ_AGG_P70 = 16,
  M3TSZ_AGG_P80 = 17,
  M3TSZ_AGG_P90 = 18,
  M3TSZ_AGG_P95 = 19,
  M3TSZ_AGG_P99 = 20,
  M3TSZ_AGG_P999 = 21,
  M3TSZ_AGG_P9999 = 22,
  M3TSZ_AGG_P25 = 23,
  M3TSZ_AGG_P75 = 24
};
/* Gauge with the six types above; SumSq / Stdev are rejected here (m3tsz_aggregate_tiles_ex has them). */
int m3tsz_aggregate_tiles_batch(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams,
                                uint64_t streams_bytes, const uint64_t *d_offsets,
                                const uint64_t *d_lengths, uint64_t n_series, int64_t start_ns,
                                int64_t step_ns, uint32_t n_windows, int32_t agg_type, int32_t out_unit,
                                uint32_t align, uint8_t *d_packed, uint64_t packed_capacity,
                                uint64_t *d_out_offsets, uint64_t *d_out_len, int32_t *d_status,
                                uint32_t *d_n_tiles, uint64_t *d_total_bytes, void *stream);

/* The same for either metric type (M3TSZ_METRIC_*; one call per type: the caller groups series the way
 * AggregateTilesOptions.MetricTypeByName does).  Valid pairs (metrics/aggregation/type.go:178-196):
 *   Gauge: Last, Min, Max, Mean, Count, Sum, SumSq, Stdev -- Gauge.ValueOf, gauge.go:144-165;
 *   Counter: Min, Max, Mean, Count, Sum, SumSq, Stdev -- Counter.ValueOf, counter.go:112-134, over the
 *   windows of m3tsz_decode_downsample_ex's Counter (float64() of the int64 aggregates).
 * Stdev = aggregation.stdev (common.go:29-37): 0 when count*(count-1) == 0, else
 * sqrt((count*sumSq - sum*sum) / (count*(count-1))) with every operation rounded on its own.
 * Gauge with one of the six types above gives exactly m3tsz_aggregate_tiles_batch's bytes.
 * Any other pair: M3TSZ_ERR_INVALID_ARG before any launch. */
int m3tsz_aggregate_tiles_ex(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams,
                             uint64_t streams_bytes, const uint64_t *d_offsets, const uint64_t *d_lengths,
                             uint64_t n_series, int64_t start_ns, int64_t step_ns, uint32_t n_windows,
                             int32_t metric_type, int32_t agg_type, int32_t out_unit, uint32_t align,
                             uint8_t *d_packed, uint64_t packed_capacity, uint64_t *d_out_offsets,
                             uint64_t *d_out_len, int32_t *d_status, uint32_t *d_n_tiles,
                             uint64_t *d_total_bytes, void *stream);

/* Tile aggregation with the aggregator's transformations (GenericElem.processValue,
 * src/aggregator/aggregator/generic_elem.go:804-950): each non-empty window's value
 * ValueOf(agg_type) at t = the window's end runs through `ops` in order before it is
 * written.  `ops` is the parsed transformation list of a pipeline without a rollup
 * (newParsedPipeline, aggregator/elem_base.go:682-752), transformation.Type ids:
 *   ABSOLUTE  math.Abs (the sign bit cleared, a NaN keeps its payload);
 *   PERSECOND (v - prev_v) * 1e9 / (t - prev_t), two roundings; prev = the previous
 *             non-empty window's binary-op input and end, (0, NaN) when there is none;
 *             math.NaN() if prev_t >= t, either value is NaN or the difference is < 0;
 *   INCREASE  v - prev_v, a NaN prev_v counting as 0; math.NaN() if prev_t >= t, v is
 *             NaN or the difference is < 0 (so -0 passes);
 *   ADD       a running sum over the element's life that skips NaN (one per Add op);
 *   RESET     v passes; also writes (t + max(step_ns / 2, 1), 0) after it (only the
 *             last Reset's; not written at timestamp 0).
 * NaN results: math.NaN() is 0x7FF8000000000001; a NaN made by arithmetic (Inf - Inf) is
 * amd64's 0xFFF8000000000000; a NaN carried from one input keeps its payload.
 * discard_nan != 0 (DiscardNaNAggregatedValues, the reference default): a window whose
 * result is NaN writes nothing, its Reset datapoint included; its binary-op input and
 * Add sums still count.  At most M3TSZ_MAX_TRANSFORMS ops (the reference has no limit),
 * at most one PerSecond / Increase (maxSupportedTransformationDerivativeOrder = 1), no
 * unknown id: else M3TSZ_ERR_INVALID_ARG before any launch.
 * d_state (optional, [n_series], caller-owned, all zeros = a new element) carries the
 * previous window and the Add sums from one call to the next: splitting the windows into
 * consecutive calls writes the same datapoints as one call.  A series' record is written
 * only when its d_status is M3TSZ_OK: after a source decode error or M3TSZ_ERR_CAPACITY it
 * is left as it was, so re-running those series with a larger buffer gives the unstopped
 * result.  NULL: every series starts new and nothing is saved.
 * d_n_tiles counts every datapoint written, Reset datapoints included; with a Reset op the
 * series' slot bound is m3tsz_encode_bound(2 * n_windows).  n_ops == 0 gives exactly
 * m3tsz_aggregate_tiles_ex's bytes.  One aggregation type per call: the reference's Add
 * op is one closure shared by all of an element's aggregation types; here each call's
 * type keeps its own sums (m3tsz_aggregate_tiles_types runs an element's types together
 * and shares them). */
enum { /* transformation.Type ids, src/metrics/transformation/type.go:36-43 */
  M3TSZ_TRANSFORM_ABSOLUTE = 1,
  M3TSZ_TRANSFORM_PERSECOND = 2,
  M3TSZ_TRANSFORM_INCREASE = 3,
  M3TSZ_TRANSFORM_ADD = 4,
  M3TSZ_TRANSFORM_RESET = 5
};
#define M3TSZ_MAX_TRANSFORMS 8
typedef struct m3tsz_transform_state {
  int32_t has_prev;                   /* a non-empty window has been through the binary op */
  int32_t reserved0;
  int64_t prev_t;                     /* its end */
  double prev_v;                      /* the binary op's input there (consumedValues) */
  double sum[M3TSZ_MAX_TRANSFORMS];   /* sum[k]: the running sum of the Add op at position k */
  uint64_t reserved1;
} m3tsz_transform_state;              /* 96 bytes */
int m3tsz_aggregate_tiles_transform(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams,
                                    uint64_t streams_bytes, const uint64_t *d_offsets, const uint64_t *d_lengths,
                                    uint64_t n_series, int64_t start_ns, int64_t step_ns, uint32_t n_windows,
                                    int32_t metric_type, int32_t agg_type, int32_t out_unit, uint32_t align,
                                    uint8_t *d_packed, uint64_t packed_capacity, uint64_t *d_out_offsets,
                                    uint64_t *d_out_len, int32_t *d_status, uint32_t *d_n_tiles,
                                    uint64_t *d_total_bytes, const int32_t *ops, uint32_t n_ops,
                                    int32_t discard_nan, m3tsz_transform_state *d_state, void *stream);

/* Tile aggregation of an element with several aggregation types (GenericElem.processValue's
 * loop over e.aggTypes, generic_elem.go:830-889): one decode + windows for the whole set,
 * one output stream per (type, series).  agg_types (host, 1 .. M3TSZ_MAX_ELEMENT_TYPES
 * entries) must be strictly ascending, as idDecompressor.Decompress returns an element's
 * types (metrics/aggregation/id_compress.go:110-135), and every entry must be valid for
 * metric_type as in m3tsz_aggregate_tiles_ex; `ops` is checked as in
 * m3tsz_aggregate_tiles_transform.  Else M3TSZ_ERR_INVALID_ARG before any launch.
 * Per non-empty window, for type j = 0 .. n_types - 1 in order, ValueOf(agg_types[j]) runs
 * through `ops` exactly as in m3tsz_aggregate_tiles_transform, except that:
 *   - the Add op at position i updates one sum shared by every type (the reference's one
 *     transformAdd closure, transformation/unary.go:46-54): type 0 adds before type 1;
 *   - the binary op's previous value is type j's own input in the previous non-empty
 *     window (consumedValues[j]); the previous window's end is the element's;
 *   - discard_nan drops type j's datapoint (and its Reset datapoint) only.
 * Output row j * n_series + s is series s, type j: d_out_offsets, d_out_len, d_status and
 * d_n_tiles have n_types * n_series entries, the rows packed into d_packed as
 * m3tsz_encode_batch_packed packs streams (slot bound as in m3tsz_aggregate_tiles_transform).
 * A source decode error goes to all n_types rows of its series, with no output.
 * d_state (optional, [n_series], caller-owned, all zeros = a new element) carries the
 * element from one call to the next.  A series' record is written only when its source
 * decoded and all n_types rows are M3TSZ_OK, so re-running the series after an error or
 * M3TSZ_ERR_CAPACITY gives the unstopped result for every type.  NULL: every series starts
 * new and nothing is saved.  With n_types == 1 the call writes the bytes, lengths, tile
 * counts, status and (in the first 96 bytes of the record) the state of
 * m3tsz_aggregate_tiles_transform (m3tsz_aggregate_tiles_ex when n_ops == 0).  Without an
 * Add op, row j equals m3tsz_aggregate_tiles_transform's for agg_types[j]. */
#define M3TSZ_MAX_ELEMENT_TYPES 8
typedef struct m3tsz_element_state {
  m3tsz_transform_state head; /* has_prev, prev_t, prev_v = type 0's binary-op input, sum[8] (shared) */
  double prev_v_more[M3TSZ_MAX_ELEMENT_TYPES - 1]; /* the binary op's input of types 1..7 */
  uint64_t reserved;
} m3tsz_element_state;        /* 160 bytes */
int m3tsz_aggregate_tiles_types(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams,
                                uint64_t streams_bytes, const uint64_t *d_offsets, const uint64_t *d_lengths,
                                uint64_t n_series, int64_t start_ns, int64_t step_ns, uint32_t n_windows,
                                int32_t metric_type, const int32_t *agg_types, uint32_t n_types,
                                int32_t out_unit, uint32_t align, uint8_t *d_packed, uint64_t packed_capacity,
                                uint64_t *d_out_offsets, uint64_t *d_out_len, int32_t *d_status,
                                uint32_t *d_n_tiles, uint64_t *d_total_bytes, const int32_t *ops,
                                uint32_t n_ops, int32_t discard_nan, m3tsz_element_state *d_state,
                                void *stream);

/* m3tsz_aggregate_tiles_types that keeps annotations, as the aggregator's flush does: the
 * same parameters, contract and outputs, plus each window's annotation.  A window keeps the
 * last non-empty annotation it was given (MaybeReplaceAnnotation, aggregation/common.go:47-61)
 * and is flushed with it alone (consumeState.annotation, aggregator/generic_elem.go:567 and
 * 915-931); nothing carries over from earlier windows or calls.  So the annotation of series s
 * in window w is that of the last datapoint, in stream order, whose timestamp lies in window w
 * and that carries one (an annotation marker directly before it: Current() reports it on that
 * datapoint only); none if there is no such datapoint.  Out-of-order datapoints count for the
 * window they fall in; datapoints outside [start_ns, start_ns + n_windows * step_ns) count for
 * nothing.  Every datapoint a window writes carries the window's annotation, in every type's
 * row and the Reset datapoint included; the encoder writes it only when it is non-empty and its
 * bytes differ from the last annotation written to that row (timestamp_encoder.go:164-195), so
 * the Reset datapoint and later windows with the same annotation add no marker.  A window that
 * discard_nan drops writes nothing, its annotation included.
 * Room: every annotation a row writes is a copy of a different annotation of its source stream,
 * so a row takes at most m3tsz_encode_bound(rows) + its source stream's length; the scratch
 * slots are sized for the longest source stream of the call (one 8-byte read back to the host).
 * A row that does not fit gets M3TSZ_ERR_CAPACITY, never a truncated stream.
 * Limits: a window's annotation is kept on the device as (bit offset from the stream's first
 * bit) << 32 | length in bytes; a stream of 2^28 bytes or more, whose offsets would not fit, is
 * already refused by the decode (M3TSZ_ERR_STREAM_TOO_LARGE on all of its rows).
 * Sources without annotations give exactly m3tsz_aggregate_tiles_types' outputs.
 * Blocks the host: it waits for `stream` to reach the 8-byte read of the longest source
 * stream (after the fused decode), then issues the encode stage and returns. */
int m3tsz_aggregate_tiles_annotated(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams,
                                    uint64_t streams_bytes, const uint64_t *d_offsets, const uint64_t *d_lengths,
                                    uint64_t n_series, int64_t start_ns, int64_t step_ns, uint32_t n_windows,
                                    int32_t metric_type, const int32_t *agg_types, uint32_t n_types,
                                    int32_t out_unit, uint32_t align, uint8_t *d_packed, uint64_t packed_capacity,
                                    uint64_t *d_out_offsets, uint64_t *d_out_len, int32_t *d_status,
                                    uint32_t *d_n_tiles, uint64_t *d_total_bytes, const int32_t *ops,
                                    uint32_t n_ops, int32_t discard_nan, m3tsz_element_state *d_state,
                                    void *stream);

/* Tile aggregation of a range inside one target block that spans many source blocks
 * (AggregateTiles, dbnode/storage/namespace.go:1775-1786): each series has one stream per
 * source block, and comes out as one stream per aggregation type.
 * Addressing: segment q is [d_offsets[q], d_offsets[q] + d_lengths[q]), or, with d_lengths
 * NULL, [d_offsets[q], d_offsets[q + 1]).  Series s is segments [d_block_off[s],
 * d_block_off[s + 1]) (n_series + 1 entries), in the order listed (block-start order).  A
 * series whose range decreases or runs past n_segments gets M3TSZ_ERR_INVALID_ARG on all its
 * rows; the other series are unaffected.
 * Each segment is decoded on its own (its own first timestamp, time unit, int / float state
 * and annotation markers), and series s's datapoints are those of its segments, concatenated
 * in the listed order.  From there every rule is m3tsz_aggregate_tiles_types' (annotations
 * == 0) or m3tsz_aggregate_tiles_annotated's (annotations != 0) on that sequence: windows,
 * out-of-order datapoints, datapoints outside the range, types, ops, discard_nan, d_state, the
 * row layout j * n_series + s and d_n_tiles.  Equal timestamps in different segments are not
 * deduplicated.  With one segment per series the outputs are exactly those calls' outputs.
 * With annotations, a segment's stream writes its first annotation even when it equals the
 * previous segment's last, so a window whose only annotated datapoint is a segment's first
 * keeps that annotation, where one stream re-encoding the concatenation would not carry it.
 * Errors: a decode error of any segment, the first in listed order, is the series' error on
 * all its rows, with no output and no record saved.  An empty segment adds no datapoints, and
 * a series with no segments, or only empty ones, has every window empty and status M3TSZ_OK
 * (where the single-stream calls report an empty stream as M3TSZ_ERR_EOF, as the reference
 * iterator does).
 * Room: a row takes at most m3tsz_encode_bound(rows), plus, with annotations, the sum of its
 * series' segment lengths; the slots are sized for the largest such sum of the call (one
 * 8-byte read back).  A row that does not fit gets M3TSZ_ERR_CAPACITY.
 * Limits: with annotations, a window's annotation is kept on the device as (bit offset of the
 * payload from d_streams' first bit) << 27 | length in bytes, so a series in which a datapoint
 * carries an annotation of 2^27 bytes or more gets M3TSZ_ERR_STREAM_TOO_LARGE on all its rows.
 * d_block_off NULL, or any check of m3tsz_aggregate_tiles_types: M3TSZ_ERR_INVALID_ARG before
 * any launch.
 * With annotations this call blocks the host, as m3tsz_aggregate_tiles_annotated does (the
 * read of the largest sum); without, it does not. */
int m3tsz_aggregate_tiles_blocks(m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams,
                                 uint64_t streams_bytes, const uint64_t *d_offsets, const uint64_t *d_lengths,
                                 uint64_t n_segments, const uint64_t *d_block_off, uint64_t n_series, int64_t start_ns,
                                 int64_t step_ns, uint32_t n_windows, int32_t metric_type, const int32_t *agg_types,
                                 uint32_t n_types, int32_t out_unit, uint32_t align, uint8_t *d_packed,
                                 uint64_t packed_capacity, uint64_t *d_out_offsets, uint64_t *d_out_len,
                                 int32_t *d_status, uint32_t *d_n_tiles, uint64_t *d_total_bytes, const int32_t *ops,
                                 uint32_t n_ops, int32_t discard_nan, m3tsz_element_state *d_state,
                                 int32_t annotations, void *stream);

/* Tile aggregation through a rollup (the pipeline "transformations, Rollup, remainder" of
 * newParsedPipeline, aggregator/elem_base.go:682-752): each group's source series are folded
 * into one element per group, which writes one stream per rollup type.
 * Sources: as in m3tsz_aggregate_tiles_blocks with d_block_off; with d_block_off NULL, one
 * stream per series (n_segments must then equal n_series).  Every source series is one element
 * of (metric_type, src_type): its non-empty windows' values Gauge/Counter.ValueOf(src_type)
 * run through pre_ops (d_src_state [n_series], optional, carries the chain from call to call)
 * and are forwarded with the window's end as timestamp; only the value is forwarded (a Reset
 * op here forwards no extra datapoint, generic_elem.go:912-937).
 * Groups: group g is the sources d_members[d_group_off[g] .. d_group_off[g + 1]) (n_groups + 1
 * offsets, n_members members), folded in that listed order: a source may be in several groups,
 * in none, or twice in one.  Window w of group g takes every forwarded value of window w of
 * its members, all at one timestamp, through AddUnique (generic_elem.go:246-281):
 *   - Gauge: Gauge.Update (gauge.go:74-101); Last is the first member's value, count counts
 *     NaNs, sum / min / max / sumSq skip them, min and max keep the first of +-0;
 *   - Counter: Counter.Update(int64(value)) with amd64's conversion (NaN and out of range give
 *     MinInt64), int64 sum / sumSq that wrap.
 * From there the group is the element of m3tsz_aggregate_tiles_types with rollup_types (1..8,
 * strictly ascending, each valid for metric_type), post_ops and d_group_state [n_groups]
 * (optional): output row j * n_groups + g is group g under rollup_types[j], with the tile
 * timestamps of the other calls (start_ns + (w + 1) * step_ns).  A window that no member
 * forwarded a value to writes nothing.
 * discard_nan (DiscardNaNAggregatedValues) applies on both sides whether or not that side
 * has ops, as processValue does (generic_elem.go:892-894): a source window whose value is NaN
 * after pre_ops is not forwarded (so it adds nothing to the group's window, Count included),
 * and a rollup row value that is NaN after post_ops is not written.  (The single-element tile
 * calls discard only with ops, to keep m3tsz_aggregate_tiles_ex's bytes.)
 * Statuses: d_status / d_n_tiles / d_out_offsets / d_out_len have n_rollup_types * n_groups
 * entries.  A group whose range decreases or runs past n_members, or that lists a source index
 * >= n_series, gets M3TSZ_ERR_INVALID_ARG on its rows; a member that fails to decode gives its
 * error to every group that lists it (the first failing member in listed order).  A group
 * without members, or without values, writes empty rows with M3TSZ_OK.  d_src_status
 * (optional, [n_series]) takes each source's decode status.  Room: a row takes at most
 * m3tsz_encode_bound(n_windows), twice that with a Reset in post_ops; a row that does not fit
 * gets M3TSZ_ERR_CAPACITY.
 * Records: a group's record is saved when its rows are all OK and all its members decoded; a
 * source's when it decoded and every group that lists it was saved (a source in no group: when
 * it decoded).  So re-running exactly the failed groups with their members gives the result of
 * one unstopped call, and consecutive calls over a split window range give one call's bytes.
 * A rollup in post_ops (a chained rollup) is not taken: run the next level as another call.
 * Invalid metric / source type pair, type list, op lists (parse as in
 * m3tsz_aggregate_tiles_transform), or NULL d_group_off / d_members where needed:
 * M3TSZ_ERR_INVALID_ARG before any launch. */
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
                                 int32_t *d_src_status, void *stream);

/* Tile aggregation through a rollup that keeps annotations: the parameters and every rule of
 * m3tsz_aggregate_tiles_rollup, plus the annotations the reference's rollup element keeps
 * (Gauge / Counter Update's MaybeReplaceAnnotation, reached through AddUnique with the
 * annotation each source window forwards).
 *   - A source window forwards the annotation of m3tsz_aggregate_tiles_annotated (over source
 *     blocks, of m3tsz_aggregate_tiles_blocks with annotations): the last one among its
 *     datapoints, none if they carry none.
 *   - The annotation of window w of group g is the last non-empty one, in listed member order,
 *     among the members whose value for w was forwarded (a NaN that discard_nan drops is not;
 *     one forwarded with discard_nan 0 is).  Every row of the group, a Reset op's extra
 *     datapoint included, writes its datapoints of w with that annotation, which the encoder
 *     writes only when it differs from the last one written.  No annotation crosses calls.
 *   - Values, counts, statuses and records are those of m3tsz_aggregate_tiles_rollup; with no
 *     annotated source the bytes are too.
 *   - A source window annotation of 2^27 bytes or more gives that source
 *     M3TSZ_ERR_STREAM_TOO_LARGE, which goes to every group that lists it.
 *   - Room: a row also takes, for copies of its members' annotations, the largest sum over
 *     groups of the members' source stream lengths (summed over their blocks); a row that does
 *     not fit gets M3TSZ_ERR_CAPACITY.  Every encode scratch slot takes that room, so one wide
 *     group raises the call's device scratch (DESIGN.md §4.8); a call that cannot allocate it
 *     returns M3TSZ_ERR_CUDA.
 *   - Blocks the host: with rows to write it waits for `stream` to reach the read of that room
 *     (after the fold), then issues the encode stage and returns. */
int m3tsz_aggregate_tiles_rollup_annotated(
    m3tsz_ctx *ctx, const m3tsz_options *opts, const uint8_t *d_streams, uint64_t streams_bytes,
    const uint64_t *d_offsets, const uint64_t *d_lengths, uint64_t n_segments, const uint64_t *d_block_off,
    uint64_t n_series, int64_t start_ns, int64_t step_ns, uint32_t n_windows, int32_t metric_type, int32_t src_type,
    const int32_t *pre_ops, uint32_t n_pre_ops, const uint64_t *d_group_off, const uint32_t *d_members,
    uint64_t n_members, uint64_t n_groups, const int32_t *rollup_types, uint32_t n_rollup_types,
    const int32_t *post_ops, uint32_t n_post_ops, int32_t discard_nan, m3tsz_transform_state *d_src_state,
    m3tsz_element_state *d_group_state, int32_t out_unit, uint32_t align, uint8_t *d_packed, uint64_t packed_capacity,
    uint64_t *d_out_offsets, uint64_t *d_out_len, int32_t *d_status, uint32_t *d_n_tiles, uint64_t *d_total_bytes,
    int32_t *d_src_status, void *stream);

/* ------------------------------------------------------------------------
 * Element sets: the aggregator's elements fed datapoint by datapoint (DESIGN.md §4.12).  GenericElem.AddUnion /
 * AddValue add a datapoint to the open window it falls in (src/aggregator/aggregator/generic_elem.go:193-240);
 * Consume(target) flushes every window whose end is at or before target, in order, through ValueOf of each aggregation
 * type and the transformations, at the window's end (generic_elem.go:291-358, 804-950, list.go:531-543).  A set is
 * n_elements Gauge or Counter elements with one resolution, one type list and one transformation list.
 *
 * The caller owns every array (device memory):
 *   - open windows: n_windows (R) slots per element, window-slot-major [R][n_elements] (slot r of element s at
 *     r * n_elements + s), 8-byte aligned: the window start, its datapoint count (0: the slot is free) and the
 *     aggregates the fused decode keeps: Gauge sum, min, max, sumSq (float64), last (float64) and lastAt (int64 ns);
 *     Counter sum, min, max, sumSq (int64; d_win_last / d_win_last_at unused, may be NULL);
 *   - d_elem: one m3tsz_element_state per element (the record the tile calls carry), 16-byte aligned;
 *   - d_watermark: one int64 per element, the end of the last window consumed (INT64_MIN: none yet);
 *   - the output: an encoder set (m3tsz_encoder_set_*) of n_types * n_elements records, row j * n_elements + s
 *     being element s under agg_types[j] (as m3tsz_aggregate_tiles_types numbers its rows); stream / grow / the
 *     accessors work on it unchanged.
 * agg_types (1 .. M3TSZ_MAX_ELEMENT_TYPES, strictly ascending, valid for metric_type) and ops / discard_nan are
 * checked and applied as in m3tsz_aggregate_tiles_types.  Every call checks all of its arguments on the host before
 * any launch (M3TSZ_ERR_INVALID_ARG).  Resetting or growing is a copy of these arrays: they hold no pointers.
 * ---------------------------------------------------------------------- */
#define M3TSZ_MAX_ELEMENT_WINDOWS 64
typedef struct m3tsz_element_set {
  uint64_t n_elements;
  uint32_t n_windows;       /* R: open-window slots per element, 1 .. M3TSZ_MAX_ELEMENT_WINDOWS */
  int32_t metric_type;      /* M3TSZ_METRIC_GAUGE, M3TSZ_METRIC_COUNTER or M3TSZ_METRIC_TIMER (the Timer calls) */
  int64_t resolution_ns;    /* > 0 */
  const int32_t *agg_types; /* host */
  uint32_t n_types;
  uint32_t n_ops;
  const int32_t *ops;       /* host */
  int32_t discard_nan;
  int32_t reserved;         /* 0 */
  int64_t *d_win_start, *d_win_count;
  void *d_win_sum, *d_win_min, *d_win_max, *d_win_sum_sq;
  double *d_win_last;
  int64_t *d_win_last_at;
  m3tsz_element_state *d_elem;
  int64_t *d_watermark;
  m3tsz_encoder_state *d_out_state;
  uint8_t *d_out_buf;
  uint64_t out_stride;      /* bytes per output slot, a multiple of 16 */
} m3tsz_element_set;
/* A set without output (d_out_state and d_out_buf NULL, out_stride 0) has no encoder set: it is a rollup's source set
 * (m3tsz_element_set_forward).  reset, add, add_annotated and forward take it and never touch an output;
 * consume and consume_annotated refuse it (M3TSZ_ERR_INVALID_ARG). */

/* Frees every window, zeroes every record, sets every watermark to INT64_MIN, and resets the output encoder set with
 * d_start [n_elements] (element s's start for all of its rows; a set without output reads nothing of d_start, which
 * may then be NULL). */
int m3tsz_element_set_reset(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                            const int64_t *d_start, void *stream);

/* Adds datapoints to the elements' open windows, point-major d_ts / d_val [points_stride][n_elements]: element s
 * takes d_n_points[s] (NULL: points_stride) of them, in row order.  Per datapoint, in that order:
 *   - its window starts at t.Truncate(resolution_ns), Go's time.Time truncation (from the zero time, so negative times
 *     round down);
 *   - a window whose end is at or before the element's watermark is closed: M3TSZ_ERR_AGGREGATION_CLOSED, nothing
 *     changes (the reference closes only the last window it consumed, DESIGN.md §6);
 *   - else the datapoint updates its open window, or opens one: Gauge.Update / Counter.Update as the fused decode
 *     runs them (gauge.go:74-106, counter.go:52-78);
 *   - a new window with all R slots open is M3TSZ_ERR_CAPACITY for that datapoint and every later one of the element
 *     in this call: nothing of them is added, so adding exactly those again after growing R gives the unstopped
 *     result.
 * d_result (int8, [points_stride][n_elements]): 0 added, else the status above (M3TSZ_ERR_INVALID_ARG for a time
 * whose window start lies below INT64_MIN); rows past the element's count are not written.  d_status [n_elements]:
 * M3TSZ_OK, M3TSZ_ERR_CAPACITY, or M3TSZ_ERR_INVALID_ARG (n_points > points_stride: the element is untouched). */
int m3tsz_element_set_add(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                          const int64_t *d_ts, const double *d_val, uint64_t points_stride,
                          const uint32_t *d_n_points, int8_t *d_result, int32_t *d_status, void *stream);

/* Consume(target_ns) of every element: the open windows whose end is at or before target_ns, in ascending start
 * order, each as one window of m3tsz_aggregate_tiles_types: every type's ValueOf, the transformations on the element
 * record, the NaN discard and the Reset datapoint, appended to the type's output row at the window's end with unit
 * out_unit (as m3tsz_encoder_set_append).  The flushed slots are freed and the watermark moves to the last one's end.
 * d_status [n_elements]: M3TSZ_OK; M3TSZ_ERR_CAPACITY when a row's slot lacks room for the flush with every datapoint
 * at its worst case (the append's bound: a slot of m3tsz_encode_bound_units(P, 1) bytes takes P datapoints) -- the element
 * then keeps its windows, record and watermark and nothing is appended, so consuming again after growing the output
 * gives the unstopped result; else the first failing row's append status (the element is consumed, and that row
 * stops as m3tsz_encoder_set_append stops a series). */
int m3tsz_element_set_consume(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                              int64_t target_ns, int32_t out_unit, int32_t *d_status, void *stream);

/* Element sets that keep annotations (DESIGN.md §4.12): each open window holds the last non-empty annotation of the
 * datapoints added to it, as Gauge.Update / Counter.Update keep it (aggregation/common.go:47-61), and every datapoint a
 * consume flushes for the window carries it (generic_elem.go:567, 923-931), the Reset datapoint included.
 *
 * The window slots' annotations live in caller-owned device memory beside the other slot arrays, pointer-free like
 * them (growing R or the capacity is a copy):
 *   - d_len [R][n_elements], 4-byte aligned: the byte length of slot r's annotation, 0 for none;
 *   - d_bytes, 8-byte aligned: slot r of element s's bytes at (r * n_elements + s) * capacity.
 * capacity: bytes per slot, a multiple of 8 in 8 .. M3TSZ_MAX_ELEMENT_ANNOTATION.
 *
 * The lengths need no initial value.  The annotated add writes a slot's length whenever it opens a window there (0
 * until a datapoint with an annotation arrives) and stores at most `capacity`; the annotated consume reads the lengths
 * of open slots only, and takes a length above `capacity` as none.  The plain calls neither read nor write these
 * arrays, so a window the plain add opened keeps whatever length its slot held, and an annotated consume writes it
 * with that slot's stale annotation.  A set should therefore use one kind of call; to switch a set to the annotated
 * calls, zero d_len after its last plain add.  The annotated calls write the same bytes as the plain calls where no
 * datapoint carries an annotation. */
#define M3TSZ_MAX_ELEMENT_ANNOTATION 65536
typedef struct m3tsz_element_annotations {
  uint32_t *d_len;   /* [R][n_elements]: bytes of window slot r's annotation, 0 = none */
  uint8_t *d_bytes;  /* slot r of element s at (r * n_elements + s) * capacity */
  uint32_t capacity; /* bytes per slot: a multiple of 8, 8 .. M3TSZ_MAX_ELEMENT_ANNOTATION */
  uint32_t reserved; /* 0 */
} m3tsz_element_annotations;

/* m3tsz_element_set_add with annotations: the sparse list of m3tsz_encoder_set_append (entries
 * [d_ann_series_off[s], d_ann_series_off[s+1]) belong to element s, sorted by dp_index, which counts rows of the
 * element's point-major column in this call; length 0 is no annotation; d_ann_series_off NULL: none in this call).
 * A datapoint the add accepts (d_result 0) with a non-empty annotation makes it its window's annotation, whatever its
 * value (NaN included); a refused datapoint changes no annotation.  A datapoint that would be accepted but whose
 * annotation is longer than `capacity` gets M3TSZ_ERR_CAPACITY under the rule of a new window with all R slots open:
 * nothing of it or of the element's later datapoints in this call is added, so growing the capacity and adding exactly
 * those again gives the unstopped result. */
int m3tsz_element_set_add_annotated(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                                    const m3tsz_element_annotations *ann, const int64_t *d_ts, const double *d_val,
                                    uint64_t points_stride, const uint32_t *d_n_points,
                                    const uint64_t *d_ann_series_off, const m3tsz_annotation_entry *d_ann_entries,
                                    const uint8_t *d_ann_bytes, int8_t *d_result, int32_t *d_status, void *stream);

/* m3tsz_element_set_consume where every datapoint flushed for a window carries the window's annotation; the output row
 * writes it when its XXH64 differs from the row's last one written (as m3tsz_encoder_set_append does).  The room check
 * also counts each flushed datapoint's annotation as the append's own check does, (len + 3) / 4 + 4 words for a
 * non-empty one.  The flushed slots' bytes stay where they are until the next add. */
int m3tsz_element_set_consume_annotated(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                                        const m3tsz_element_annotations *ann, int64_t target_ns, int32_t out_unit,
                                        int32_t *d_status, void *stream);

/* Element sets through a rollup (the pipeline "transformations, Rollup, remainder", DESIGN.md §4.12): each source's
 * Consume(target_ns) forwards its windows' values to the groups that list it, and each group takes them through its
 * rollup element's AddUnique (generic_elem.go:246-281, 912-937).
 *   - src: the source set, of metric type M, with exactly one aggregation type (the rollup's source type, valid for M
 *     as in m3tsz_aggregate_tiles_rollup: Counter Sum and Gauge Last are the usual ones), its ops the pipeline's
 *     transformations before the rollup and its discard_nan the pipeline's.  It needs no output (see above).
 *   - groups: an element set of the same M and resolution_ns with n_elements == n_groups, its type list the rollup's
 *     types and its ops the remainder's; m3tsz_element_set_consume consumes it as any other set.
 *   - group g is the sources d_members[d_group_off[g] .. d_group_off[g + 1]) (n_groups + 1 offsets, n_members
 *     members), as in m3tsz_aggregate_tiles_rollup: a source may be in several groups, in none, or twice in one.
 * Rules:
 *   1. Forward: every source takes its open windows that end at or before target_ns, in ascending start order; each
 *      window's value is ValueOf(the source type) through the ops on the source's record (a Reset forwards nothing
 *      extra).  discard_nan drops a NaN value with or without ops (generic_elem.go:892-894): it is not forwarded.
 *   2. Fold: every group takes its members in listed order, and each member's forwarded windows in start order, into
 *      the group window with the same start as the source window, opening a slot if needed.  Every value of a window
 *      arrives at one timestamp, so the fold is m3tsz_aggregate_tiles_rollup's: Gauge Last is the first value, count
 *      counts NaNs, sum / min / max / sumSq skip them; Counter int64(value) with sums that wrap.  The slot holds the
 *      result as an add leaves it (a Gauge's last_at is the window's end).  A member listed twice is folded twice.
 *   3. A group window that ends at or before the group's watermark is closed: its values are dropped and the group
 *      gets M3TSZ_ERR_AGGREGATION_CLOSED; its other windows still fold.
 *   4. A group with fewer free slots than new windows gets M3TSZ_ERR_CAPACITY, and nothing is folded into it.
 *   5. A group whose range decreases or runs past n_members, or that lists a source >= src->n_elements, gets
 *      M3TSZ_ERR_INVALID_ARG (over CAPACITY), and nothing is folded into it.
 *   6. Commit: a group that failed with CAPACITY or INVALID_ARG holds back every member its range names (up to
 *      n_members): such a source keeps its windows, record and watermark, and d_src_status[s] is that group's status
 *      (INVALID_ARG when groups of both kinds list it).  Every other source frees its due windows, saves its record
 *      and moves its watermark to the last due window's end, with d_src_status[s] = M3TSZ_OK; a source in no group
 *      drops its values.  So after growing the groups' open windows, calling again with exactly the failed groups
 *      (d_group_off / d_members listing only them, the same group set) gives the result of one unstopped call.
 * d_group_status [n_groups]: M3TSZ_OK or the status above.  The call reads and writes no annotation arrays (an
 * annotated group set's new windows get no annotation lengths: consume it with the plain consume, or forward with
 * m3tsz_element_set_forward_annotated).  A metric type or
 * resolution mismatch, a source type list of other than one type, an invalid type or op list, n_groups other than
 * groups->n_elements, n_members above 2^40, src and groups sharing their slots, or NULL d_group_off / d_members /
 * statuses where they are needed: M3TSZ_ERR_INVALID_ARG before any launch. */
int m3tsz_element_set_forward(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *src,
                              int64_t target_ns, const uint64_t *d_group_off, const uint32_t *d_members,
                              uint64_t n_members, uint64_t n_groups, const m3tsz_element_set *groups,
                              int32_t *d_src_status, int32_t *d_group_status, void *stream);

/* m3tsz_element_set_forward for sets that keep annotations: src_ann holds the source set's window annotations and
 * group_ann the group set's (m3tsz_element_annotations, both required).  Values, counts, statuses, records, watermarks
 * and the commit rule are those of m3tsz_element_set_forward; in addition:
 *   1. A forwarded source window carries its slot's annotation: src_ann->d_len and the slot's bytes, a length of 0 or
 *      above src_ann->capacity being none (as m3tsz_element_set_consume_annotated reads it).
 *   2. A group window's annotation follows MaybeReplaceAnnotation through AddUnique (generic_elem.go:278-281,
 *      aggregation/common.go:47-61): members in listed order, each member's forwarded windows in start order, every
 *      forwarded value with a non-empty annotation replaces its group window's annotation.  A NaN that discard_nan
 *      drops is not forwarded, so its annotation is not taken; a NaN forwarded without discard_nan carries its
 *      annotation; a value dropped because its group window is closed changes nothing.  The order is the listed
 *      member order, not arrival order (DESIGN.md §6).
 *   3. A group window already open keeps its annotation unless a forwarded value replaces it; a window the call opens
 *      writes its length (the annotation it took, or 0), so the group set's lengths need no initial value either.
 *   4. A group one of whose values that would fold (its group window not closed) carries an annotation longer than
 *      group_ann->capacity gets M3TSZ_ERR_CAPACITY under rule 4 above: nothing is folded into it and its members are
 *      held back (INVALID_ARG over CAPACITY), so growing the group set's capacity and calling again with exactly the
 *      failed groups gives the unstopped result.
 *   5. The source annotation arrays are read, never written: a committed source's slot bytes stay until its next add.
 * Besides the checks of m3tsz_element_set_forward: a NULL src_ann or group_ann, a capacity that is not a multiple of 8
 * in 8 .. M3TSZ_MAX_ELEMENT_ANNOTATION, a non-zero reserved, misaligned pointers, or source and group annotation
 * arrays that overlap: M3TSZ_ERR_INVALID_ARG before any launch.  Consume the group set with
 * m3tsz_element_set_consume_annotated. */
int m3tsz_element_set_forward_annotated(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *src,
                                        const m3tsz_element_annotations *src_ann, int64_t target_ns,
                                        const uint64_t *d_group_off, const uint32_t *d_members, uint64_t n_members,
                                        uint64_t n_groups, const m3tsz_element_set *groups,
                                        const m3tsz_element_annotations *group_ann, int32_t *d_src_status,
                                        int32_t *d_group_status, void *stream);

/* Element-set rollups across shards (DESIGN.md §4.12): the reference splits a rollup whose sources live on other
 * shards in two.  The source shard's forwarded writer (aggregator/forwarded_writer.go) collects, per rollup key and
 * window, the values of its local sources and sends one aggregated.ForwardedMetric with ForwardMetadata.SourceID; the
 * group shard takes it through GenericElem.AddUnique (generic_elem.go:241-288), which refuses a (source, version) its
 * window has already seen.  m3tsz_element_set_forward_write is the first half, m3tsz_element_set_add_forwarded the
 * second, for Gauge and Counter sets; m3tsz_element_set_forward_write_timer and m3tsz_element_set_add_forwarded_timer
 * (after the Timer calls below) are the pair for Timer sets.  Without annotations.
 *
 * One forwarded metric, pointer-free so that a batch (records + one float64 values array) can be copied, concatenated
 * or sent as bytes (40 bytes, 8-byte aligned): */
typedef struct m3tsz_forwarded_metric {
  uint64_t key;       /* the receiving group set's element index */
  int64_t time_ns;    /* ForwardedMetric.TimeNanos: the source window's end */
  uint64_t value_off; /* its first value in the batch's values array */
  uint32_t n_values;  /* >= 1 */
  uint32_t source_id; /* ForwardMetadata.SourceID: the writing shard */
  uint32_t version;   /* ForwardedMetric.Version: 0 (a resend is not taken) */
  uint32_t reserved;  /* 0 */
} m3tsz_forwarded_metric;

/* The sources a group set's windows have seen: `capacity` bits per window slot, one per source id, in caller-owned
 * device memory beside the slot arrays, word-interleaved across elements (word w of slot r of element s at
 * (r * (capacity / 32) + w) * n_elements + s), 4-byte aligned.  capacity: a multiple of 32 in 32 ..
 * M3TSZ_MAX_FORWARD_SOURCES.  Pointer-free: growing R or the capacity is a copy.
 * The bits need no initial value: m3tsz_element_set_add_forwarded zeroes a slot's bits when it opens a window there.
 * Only m3tsz_element_set_add_forwarded reads or writes them, so a window opened by add or forward has stale bits: a
 * group set fed by add_forwarded takes all of its values that way, the shard's own sources included (through its own
 * forward_write records, as the reference's shard reaches its own groups through its client). */
#define M3TSZ_MAX_FORWARD_SOURCES 65536
typedef struct m3tsz_element_sources {
  uint32_t *d_bits;
  uint32_t capacity; /* bits per slot: a multiple of 32, 32 .. M3TSZ_MAX_FORWARD_SOURCES */
  uint32_t reserved; /* 0 */
} m3tsz_element_sources;

/* The source shard's forwarded writer.  src, target_ns, d_group_off, d_members, n_members and n_groups are those of
 * m3tsz_element_set_forward (there is no group set here: n_groups is the call's group count), and every source
 * forwards its due windows by that call's rule 1.  Nothing is folded: for each group, in group order, one record per
 * distinct forwarded window start, in ascending start order, with
 *   key = d_group_key[g] (d_group_key NULL: g), time_ns = the window start + resolution, source_id as given,
 *   version 0, and as values the window's forwarded values of the group's members in listed member order (a member
 *   listed twice contributes twice).  A window to which no member forwards a value gets no record (onDone skips an
 *   empty bucket).
 * The records go to d_metrics [metric_capacity] and their values to d_values [value_capacity], groups in order.  A
 * group whose range decreases or runs past n_members, or that lists a source >= src->n_elements, gets
 * M3TSZ_ERR_INVALID_ARG and writes nothing.  The others' record and value counts are exclusive-scanned: the groups
 * that fit inside metric_capacity and value_capacity are written, and every later group gets M3TSZ_ERR_CAPACITY (a
 * prefix rule).  The commit is rule 6 of m3tsz_element_set_forward: a failed group holds back its members.  So
 * calling again after growing, with exactly the failed groups, gives the remaining records; the two calls' records
 * together are the unstopped call's.
 * d_counts [4] (uint64): metrics written, values written, metrics needed, values needed (all groups but the invalid
 * ones).  d_src_status [src->n_elements], d_group_status [n_groups]: as in m3tsz_element_set_forward.
 * Host checks (M3TSZ_ERR_INVALID_ARG before any launch): those of m3tsz_element_set_forward on src, a Timer set, a
 * source type list of other than one type, n_groups or n_members above 2^40, capacities above 2^40, NULL or
 * misaligned required pointers. */
int m3tsz_element_set_forward_write(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *src,
                                    int64_t target_ns, const uint64_t *d_group_off, const uint32_t *d_members,
                                    uint64_t n_members, uint64_t n_groups, const uint64_t *d_group_key,
                                    uint32_t source_id, m3tsz_forwarded_metric *d_metrics, uint64_t metric_capacity,
                                    double *d_values, uint64_t value_capacity, uint64_t *d_counts,
                                    int32_t *d_src_status, int32_t *d_group_status, void *stream);

/* AddUnique of forwarded metrics into a group set (Entry.addForwardedWithLock -> GenericElem.AddUnique, entry.go:
 * 1177-1191, generic_elem.go:241-288).  Each element takes its records in array order (which stands in for arrival
 * order); per record, in that order:
 *   1. key >= n_elements, n_values 0, a value range past n_values, version != 0 or reserved != 0:
 *      M3TSZ_ERR_INVALID_ARG, nothing changes;
 *   2. the group window starts at Truncate(time_ns, resolution) - resolution (Go's truncation, as in add): the slot
 *      m3tsz_element_set_forward folds the same source window into.  A start below INT64_MIN is INVALID_ARG;
 *   3. a window ending at or before the element's watermark: M3TSZ_ERR_AGGREGATION_CLOSED, nothing changes;
 *   4. source_id >= sources->capacity, or a new window with all R slots open: M3TSZ_ERR_CAPACITY for the record and
 *      every later record of the element in this call (add's stop rule);
 *   5. the window has seen source_id: M3TSZ_ERR_DUPLICATE_SOURCE, nothing changes, later records continue;
 *   6. else the source's bit is set and each value is folded in order with m3tsz_element_set_forward's fold (Gauge
 *      Last = the first value; Counter int64(value), sums that wrap).
 * d_result (int8 [n_metrics], input order): 0 or the status above.  d_status [n_elements]: M3TSZ_OK or
 * M3TSZ_ERR_CAPACITY.  After a CAPACITY stop and a grow, sending exactly the refused records again gives the unstopped
 * result, and so does sending the whole batch again: the accepted records come back DUPLICATE_SOURCE (at-least-once
 * delivery).  The call reads and writes no annotation arrays and needs no output rows.
 * Host checks (M3TSZ_ERR_INVALID_ARG before any launch): the set's (a Timer set is refused), a NULL or bad sources
 * struct, n_metrics or n_values above 2^40, NULL or misaligned required pointers. */
int m3tsz_element_set_add_forwarded(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                                    const m3tsz_element_sources *sources, const m3tsz_forwarded_metric *d_metrics,
                                    uint64_t n_metrics, const double *d_values, uint64_t n_values, int8_t *d_result,
                                    int32_t *d_status, void *stream);

/* Timer element sets (DESIGN.md §4.12): an element set of metric_type M3TSZ_METRIC_TIMER, whose windows are
 * aggregation.Timer (aggregation/timer.go) over the CM stream (aggregation/quantile/cm/stream.go).
 *   - Types: strictly ascending, any but Last (IsValidForTimer); 1 .. 23 of them without ops, 1 ..
 *     M3TSZ_MAX_ELEMENT_TYPES with ops.  The stream's quantile list is Types.PooledQuantiles over them: the quantile
 *     types in the listed order (ascending id), Median and P50 one 0.5.  It is not sorted: P25 / P75 (ids 23 / 24)
 *     come after P9999, and "first listed quantile >= q" is what Quantile(q) returns.
 *   - Slots: d_win_start, d_win_count (values added; 0: the slot is free), d_win_sum, d_win_sum_sq (float64, summed
 *     in add order, NaN included, no FMA); d_win_min / d_win_max / d_win_last / d_win_last_at are unused (may be NULL).
 *   - ValueOf: Min / Max the flushed stream's first / last sample, Mean sum / count, Count, Sum, SumSq, Stdev as in
 *     m3tsz_aggregate_tiles_ex, and each quantile type Quantile(q) of the stream after Flush.  A quantile that
 *     calcQuantiles leaves unset reads 0, as a freshly made stream holds it.
 *   - A set of more than M3TSZ_MAX_ELEMENT_TYPES types has no ops and leaves its records untouched; up to that many,
 *     the records are kept as for the other sets.
 * m3tsz_element_set_reset takes a Timer set as any other; add, consume, their annotated forms, forward and
 * forward_annotated refuse it (M3TSZ_ERR_INVALID_ARG before any launch), as the tile and downsample calls refuse metric
 * type 2; a Timer rollup forwards with m3tsz_element_set_forward_timer.  A Timer set that keeps annotations takes
 * m3tsz_element_set_add_timer_annotated, m3tsz_element_set_consume_timer_annotated and
 * m3tsz_element_set_forward_timer_annotated, which refuse Gauge and Counter sets.
 *
 * Each window slot's stream lives in caller-owned device memory, pointer-free (growing R or the capacity is a copy).
 * Slot o = r * n_elements + s; its sample i (list sample or pending heap entry) at (r * sample_capacity + i) *
 * n_elements + s, so a warp's lanes touch adjacent words.  The header is written when an add opens the window, so
 * nothing needs an initial value. */
typedef struct m3tsz_timer_stream_header {
  int64_t num_values;        /* numValues: values inserted into the sorted list */
  int64_t compress_min_rank; /* compressMinRank */
  int32_t head, tail;        /* the list's ends (sample indices), -1: none */
  int32_t insert_cursor;     /* insertCursor, -1: nil */
  int32_t compress_cursor;   /* compressCursor, -1: nil */
  int32_t n_samples;         /* samples in the list */
  int32_t n_used;            /* sample entries ever taken; freed ones are chained through d_next from free_head */
  int32_t free_head;
  int32_t counter;           /* insertAndCompressCounter */
  int32_t n_a, n_b;          /* the pending heaps' lengths */
  int32_t less_is_b;         /* bufLess is heap b (resetInsertCursor swaps the two) */
  int32_t reserved;
} m3tsz_timer_stream_header; /* 64 bytes */
typedef struct m3tsz_element_timer_streams {
  m3tsz_timer_stream_header *d_header; /* [R][n_elements], 8-byte aligned */
  double *d_value;                     /* list samples: value, numRanks, delta, prev / next links (-1: none) */
  int64_t *d_num_ranks;
  int64_t *d_delta;
  int32_t *d_prev, *d_next;
  double *d_heap_a, *d_heap_b;         /* the pending minHeaps, as the reference's arrays */
  uint32_t sample_capacity;            /* >= 1: values a slot holds, list samples and pending values together */
  uint32_t insert_and_compress_every;  /* >= 1 (StreamOptions: 1024) */
  double eps;                          /* finite, > 0 (StreamOptions: 1e-3) */
  uint64_t reserved;                   /* 0 */
} m3tsz_element_timer_streams;

/* Timer.AddBatch of the elements' samples, point-major d_ts / d_val [points_stride][n_elements] with d_n_points as
 * in m3tsz_element_set_add.  d_batch (optional, int8 [points_stride][n_elements]): a nonzero entry continues the
 * previous row's batch (BatchTimer); NULL: every row is its own batch (AppendTimerSample).  Per batch, in order:
 *   - its window is that of its first row's timestamp; a window at or before the watermark refuses the whole batch
 *     (M3TSZ_ERR_AGGREGATION_CLOSED), a start below INT64_MIN too (M3TSZ_ERR_INVALID_ARG);
 *   - capacity: a slot holds at most sample_capacity values, list samples and pending values together.  A batch that
 *     would exceed it, or that needs a new window when all R slots are open, gets M3TSZ_ERR_CAPACITY, and so does
 *     every later row of the element in this call: nothing of them is added, so adding exactly those rows again
 *     after growing gives the unstopped result.  No insert and no consume-time Flush can then run out of room;
 *   - else count += len, sum += v and sumSq += v * v in order, and the stream's AddBatch (the first value of a new
 *     window straight into the list; the pending heaps; insert + compress every insert_and_compress_every values).
 * d_result [points_stride][n_elements]: each row its batch's status.  d_status: M3TSZ_OK, M3TSZ_ERR_CAPACITY, or
 * M3TSZ_ERR_INVALID_ARG when n_points > points_stride (nothing written) or when a continuation is in row 0 or has
 * another timestamp than its batch's first row (every row M3TSZ_ERR_INVALID_ARG; the element is untouched).
 * Host checks (M3TSZ_ERR_INVALID_ARG before any launch): the set's, NULL streams, sample_capacity of 0 or above 2^30,
 * eps not finite or <= 0, insert_and_compress_every of 0 or above 2^31 - 1, a non-zero reserved, misaligned arrays. */
int m3tsz_element_set_add_timer(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                                const m3tsz_element_timer_streams *streams, const int64_t *d_ts, const double *d_val,
                                uint64_t points_stride, const uint32_t *d_n_points, const int8_t *d_batch,
                                int8_t *d_result, int32_t *d_status, void *stream);

/* m3tsz_element_set_consume of a Timer set: each due window, in start order, is flushed (Flush: insert + compress
 * until both pending heaps are empty, then calcQuantiles), and ValueOf of each type goes through the ops, the NaN
 * discard and the Reset row, onto the output rows, with the plain consume's room check and commit rule. */
int m3tsz_element_set_consume_timer(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                                    const m3tsz_element_timer_streams *streams, int64_t target_ns, int32_t out_unit,
                                    int32_t *d_status, void *stream);

/* Timer element sets through a rollup (DESIGN.md §4.12): m3tsz_element_set_forward for Timer sets.  A Timer source
 * with a rollup pipeline forwards ValueOf(its type) through its pre-rollup ops (generic_elem.go:860-937); the forwarded
 * metric keeps its type, so each group window is a Timer and AddUnique is Timer.Add of each value
 * (generic_elem.go:276-281, aggregation/timer.go:52-76).
 *   - src: a Timer set with exactly one type (any but Last, e.g. P99, Max or Mean), its ops the pre-rollup ops and its
 *     discard_nan the pipeline's; it usually has no output.  src_streams: its streams.
 *   - groups: a Timer set of the same resolution_ns with n_elements == n_groups, the rollup's types and the
 *     remainder's ops; m3tsz_element_set_consume_timer consumes it.  group_streams: its streams.
 *   - group g is the sources d_members[d_group_off[g] .. d_group_off[g + 1]), as in m3tsz_element_set_forward.
 * Rules:
 *   1. Forward: every source takes its open windows that end at or before target_ns, in start order.  Each window's
 *      stream is Flushed and gives ValueOf(the source type), which goes through the ops on the source's record as
 *      m3tsz_element_set_consume_timer computes a type's value (a Reset forwards nothing extra).  discard_nan drops a
 *      NaN value with or without ops.  Each flushed stream header is written back to its slot, since the flush
 *      rewrote the slot's samples; a Flush with empty heaps only recomputes the quantiles, so a held-back source
 *      forwards the same bits when called again.
 *   2. Fold: every group takes its members in listed order, and each member's forwarded windows in start order, into
 *      the group window with the same start as the source window, opening a slot if needed.  Each value is one
 *      Timer.Add: count + 1, sum and sumSq in order (NaN included, as m3tsz_element_set_add_timer sums them), then
 *      AddBatch of that one value.  k values into one window are k one-value batches, not one batch of k (each reads
 *      the insertion point afresh, which changes the quantiles).  A member listed twice is folded twice.
 *   3. A group window that ends at or before the group's watermark is closed: its values are dropped and the group
 *      gets M3TSZ_ERR_AGGREGATION_CLOSED; its other windows still fold.
 *   4. Capacity: a group with fewer free slots than new windows, or with a window this call touches whose list
 *      samples + pending values + the values this call folds into it (0 + n for a new window) exceed
 *      group_streams->sample_capacity, gets M3TSZ_ERR_CAPACITY, and nothing is folded into it.  The sample bound
 *      ignores the room the fold's compressions free, so it is deterministic: growing and calling again gives the
 *      unstopped result.
 *   5. Invalid group and 6. commit: rules 5 and 6 of m3tsz_element_set_forward.  A held-back source keeps its
 *      windows, counts, sums, record and watermark; its due streams stay flushed in place (rule 1).  So after
 *      growing the group set's open windows and / or sample capacity, calling again with exactly the failed groups
 *      gives the result of one unstopped call.
 * Host checks (M3TSZ_ERR_INVALID_ARG before any launch): those of m3tsz_element_set_forward, those of
 * m3tsz_element_set_add_timer for both sets and stream structs, either set not a Timer set, a source type list other
 * than one type, and source and group sets sharing slot or stream arrays.  m3tsz_element_set_forward and
 * m3tsz_element_set_forward_annotated keep refusing Timer sets. */
int m3tsz_element_set_forward_timer(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *src,
                                    const m3tsz_element_timer_streams *src_streams, int64_t target_ns,
                                    const uint64_t *d_group_off, const uint32_t *d_members, uint64_t n_members,
                                    uint64_t n_groups, const m3tsz_element_set *groups,
                                    const m3tsz_element_timer_streams *group_streams, int32_t *d_src_status,
                                    int32_t *d_group_status, void *stream);

/* Timer element sets that keep annotations (DESIGN.md §4.12): the Timer calls with the set's window annotations in
 * `ann` (m3tsz_element_annotations, laid out and checked as for the other sets; the lengths need no initial value).
 * Each Timer window keeps one annotation, as aggregation.Timer does (MaybeReplaceAnnotation, timer.go:57-76).
 *
 * m3tsz_element_set_add_timer with annotations: the sparse list of m3tsz_element_set_add_annotated (dp_index counts
 * rows of the element's column).  A batch has one annotation, its first row's entry, as a BatchTimer has one; with
 * d_batch NULL every row is its own batch with its own annotation (AppendTimerSample).  An entry with a length on a
 * continuation row breaks the batch rule: every row of the element gets M3TSZ_ERR_INVALID_ARG and it is untouched.  Per
 * batch, after the closed and invalid-start checks (a closed batch is M3TSZ_ERR_AGGREGATION_CLOSED whatever its
 * annotation), an annotation longer than ann->capacity gets M3TSZ_ERR_CAPACITY under the R rule: nothing of the batch
 * or of the element's later rows in this call is added.  Then the slot and sample-room checks.  An accepted batch with
 * a non-empty annotation replaces its window's annotation, NaN samples included; a refused batch changes none.  A
 * window this call opens writes its slot's length (0 until an annotation arrives). */
int m3tsz_element_set_add_timer_annotated(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                                          const m3tsz_element_timer_streams *streams,
                                          const m3tsz_element_annotations *ann, const int64_t *d_ts,
                                          const double *d_val, uint64_t points_stride, const uint32_t *d_n_points,
                                          const int8_t *d_batch, const uint64_t *d_ann_series_off,
                                          const m3tsz_annotation_entry *d_ann_entries, const uint8_t *d_ann_bytes,
                                          int8_t *d_result, int32_t *d_status, void *stream);

/* m3tsz_element_set_consume_timer where every datapoint staged for a window carries the window's annotation: every
 * type's datapoint, the Reset datapoint, and the rows of a set of more than M3TSZ_MAX_ELEMENT_TYPES types.  The room
 * check counts each flushed datapoint's annotation as m3tsz_element_set_consume_annotated does. */
int m3tsz_element_set_consume_timer_annotated(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                                              const m3tsz_element_timer_streams *streams,
                                              const m3tsz_element_annotations *ann, int64_t target_ns,
                                              int32_t out_unit, int32_t *d_status, void *stream);

/* m3tsz_element_set_forward_timer for Timer sets that keep annotations: src_ann and group_ann as in
 * m3tsz_element_set_forward_annotated (both required).  Values, statuses, records, watermarks, the stream write-back
 * and the commit are those of m3tsz_element_set_forward_timer; the annotations follow rules 1-5 of
 * m3tsz_element_set_forward_annotated: a forwarded window carries its slot's annotation (a length of 0 or above
 * src_ann->capacity being none); each folded value with one replaces its group window's (MaybeReplaceAnnotation
 * through AddUnique), members in listed order and each member's windows in start order; a value that discard_nan drops
 * carries nothing and one dropped at a closed group window changes nothing; a window the fold opens writes its length;
 * a value that would fold with an annotation longer than group_ann->capacity fails its group with M3TSZ_ERR_CAPACITY
 * beside the slot and sample counts (nothing folded, members held back; INVALID_ARG still wins); the source annotation
 * arrays are only read.  Host checks: those of m3tsz_element_set_forward_timer and of
 * m3tsz_element_set_forward_annotated's annotation structs. */
int m3tsz_element_set_forward_timer_annotated(
    m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *src,
    const m3tsz_element_timer_streams *src_streams, const m3tsz_element_annotations *src_ann, int64_t target_ns,
    const uint64_t *d_group_off, const uint32_t *d_members, uint64_t n_members, uint64_t n_groups,
    const m3tsz_element_set *groups, const m3tsz_element_timer_streams *group_streams,
    const m3tsz_element_annotations *group_ann, int32_t *d_src_status, int32_t *d_group_status, void *stream);

/* Timer element-set rollups across shards (DESIGN.md §4.12): the cross-shard pair above for Timer sets, without
 * annotations.  A latency timer rolled up with its host or pod tag dropped has members on every shard, and arrival
 * order changes the group's quantiles, not only its Last.
 *
 * The source shard's writer: m3tsz_element_set_forward_write with the source's streams.  src is a Timer set of one
 * type (any but Last); each source forwards its due windows as m3tsz_element_set_forward_timer does (rule 1: Flush,
 * ValueOf of the type through the pre-rollup ops, the flushed headers written back).  Records, the prefix capacity
 * rule, d_counts, held-back members and statuses are m3tsz_element_set_forward_write's.
 * Host checks: those of m3tsz_element_set_forward_write, with src checked as m3tsz_element_set_add_timer checks a set
 * and its streams; a set that is not a Timer set is refused.  m3tsz_element_set_forward_write keeps refusing Timer
 * sets. */
int m3tsz_element_set_forward_write_timer(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *src,
                                          const m3tsz_element_timer_streams *src_streams, int64_t target_ns,
                                          const uint64_t *d_group_off, const uint32_t *d_members, uint64_t n_members,
                                          uint64_t n_groups, const uint64_t *d_group_key, uint32_t source_id,
                                          m3tsz_forwarded_metric *d_metrics, uint64_t metric_capacity,
                                          double *d_values, uint64_t value_capacity, uint64_t *d_counts,
                                          int32_t *d_src_status, int32_t *d_group_status, void *stream);

/* AddUnique of forwarded metrics into a Timer group set (its streams in set_streams).  Each element takes its records
 * in array order, which stands in for arrival order and for a Timer also fixes the quantiles.  Per record, rules 1-5
 * of m3tsz_element_set_add_forwarded, then:
 *   6. the window's list samples + pending values + the record's n_values exceed set_streams->sample_capacity:
 *      M3TSZ_ERR_CAPACITY for the record and every later record of the element in this call; the source's bit stays
 *      clear, and a slot opened for the record stays free;
 *   7. else the source's bit is set and each value, in the record's order, is one Timer.Add into the window (count +
 *      1, sum and sumSq as m3tsz_element_set_add_timer sums them, then AddBatch of that one value), as
 *      m3tsz_element_set_forward_timer folds a value.
 * d_result and d_status as in m3tsz_element_set_add_forwarded.  After a CAPACITY stop and
 * m3tsz_element_set_forward_timer's grow (open windows and / or sample capacity), sending the refused records again,
 * or the whole batch, gives the unstopped result.
 * Host checks: those of m3tsz_element_set_add_forwarded, with the set checked as m3tsz_element_set_add_timer checks a
 * set and its streams; a set that is not a Timer set is refused.  m3tsz_element_set_add_forwarded keeps refusing
 * Timer sets. */
int m3tsz_element_set_add_forwarded_timer(m3tsz_ctx *ctx, const m3tsz_options *opts, const m3tsz_element_set *set,
                                          const m3tsz_element_timer_streams *set_streams,
                                          const m3tsz_element_sources *sources,
                                          const m3tsz_forwarded_metric *d_metrics, uint64_t n_metrics,
                                          const double *d_values, uint64_t n_values, int8_t *d_result,
                                          int32_t *d_status, void *stream);

/* ------------------------------------------------------------------------
 * Per-series streaming handles: what a cgo shim binds METHOD FOR METHOD to the
 * reference's interfaces (INTEGRATION.md §2 is that shim):
 *   encoding.Encoder         src/dbnode/encoding/types.go:39-91   -> m3tsz_encoder_*
 *   encoding.ReaderIterator  types.go:180-203, Decoder :342-345   -> m3tsz_iter_*
 *   EncoderPool / ReaderIteratorPool  encoder_pool.go:27-48, iterator_pool.go:27-47 -> *_pool_*
 * The handles keep host state only; bitstreams are produced / consumed by the
 * batch kernels (one series per launch) lazily: an encoder when Len / Stream /
 * Discard / LastEncoded is called, an iterator on its first Next().  Handles of one
 * context serialise on the context's scratch; a handle itself is single-threaded like
 * the reference's objects.  Error conventions are the reference's:
 *   Encode on a closed encoder -> M3TSZ_ERR_ENCODER_CLOSED; a second/millisecond
 *   delta-of-delta that overflows 32 bits -> M3TSZ_ERR_DOD_OVERFLOW; invalid unit ->
 *   M3TSZ_ERR_UNRECOGNIZED_UNIT (the failing datapoint is dropped as a whole, DESIGN.md §6);
 *   LastEncoded / LastAnnotationChecksum on an empty encoder -> M3TSZ_ERR_NO_DATAPOINTS;
 *   iterator Err(): sticky status, visible after the Next() that failed; closed ->
 *   M3TSZ_ERR_ITER_CLOSED.
 * ---------------------------------------------------------------------- */
typedef struct m3tsz_encoder m3tsz_encoder;
typedef struct m3tsz_iter m3tsz_iter;
typedef struct m3tsz_encoder_pool m3tsz_encoder_pool;
typedef struct m3tsz_iter_pool m3tsz_iter_pool;

/* m3tsz.NewEncoder(start, nil, intOptimized, opts), m3tsz/encoder.go:64-85 */
int m3tsz_encoder_create(m3tsz_ctx *ctx, const m3tsz_options *opts, int64_t start_ns, m3tsz_encoder **out);
void m3tsz_encoder_destroy(m3tsz_encoder *enc);
/* Reset(start, capacity, schema), encoder.go:262-279 (re-opens a closed encoder) */
int m3tsz_encoder_reset(m3tsz_encoder *enc, int64_t start_ns, uint64_t capacity);
/* Encode(dp, unit, annotation), encoder.go:90-110 */
int m3tsz_encoder_encode(m3tsz_encoder *enc, int64_t ts_ns, double value, int32_t unit,
                         const uint8_t *annotation, uint64_t annotation_len);
/* the delta-of-delta (in time units) of the last Encode that returned M3TSZ_ERR_DOD_OVERFLOW: the
 * value the reference formats into its error ("deltaOfDelta value %d %s overflows 32 bits") */
int64_t m3tsz_encoder_failed_dod(const m3tsz_encoder *enc);
uint64_t m3tsz_encoder_num_encoded(const m3tsz_encoder *enc); /* NumEncoded, :299-302 */
/* LastEncoded, :305-319: PrevTime and -- the reference's quirk, kept -- the float value in
 * float mode, else the encoder's intVal: the SCALED integer in int mode, 0 when int_optimized == 0 */
int m3tsz_encoder_last_encoded(m3tsz_encoder *enc, int64_t *ts_ns, double *value);
/* LastAnnotationChecksum, :321-327: XXH64 (cespare/xxhash/v2) of the last annotation written */
int m3tsz_encoder_last_annotation_checksum(const m3tsz_encoder *enc, uint64_t *checksum);
int m3tsz_encoder_empty(const m3tsz_encoder *enc);              /* Empty, :330-332 */
int m3tsz_encoder_len(m3tsz_encoder *enc, uint64_t *len);        /* Len, :336-354 (with the tail) */
/* Stream(ctx), :282-297: copies head||tail into buf; *len == 0 <=> (nil, false).  *tail_len
 * (optional) = bytes of the ts.Segment tail, so head = buf[0 .. len - tail_len). */
int m3tsz_encoder_stream(m3tsz_encoder *enc, uint8_t *buf, uint64_t cap, uint64_t *len, uint64_t *tail_len);
int m3tsz_encoder_close(m3tsz_encoder *enc);                    /* Close, :357-370 (idempotent) */
/* Discard, :374-381 (segment + Close) / DiscardReset, :385-392 (segment + Reset) */
int m3tsz_encoder_discard(m3tsz_encoder *enc, uint8_t *buf, uint64_t cap, uint64_t *len, uint64_t *tail_len);
int m3tsz_encoder_discard_reset(m3tsz_encoder *enc, int64_t start_ns, uint64_t capacity, uint8_t *buf,
                                uint64_t cap, uint64_t *len, uint64_t *tail_len);

/* m3tsz.NewReaderIterator(nil, intOptimized, opts), m3tsz/iterator.go:67-78 */
int m3tsz_iter_create(m3tsz_ctx *ctx, const m3tsz_options *opts, m3tsz_iter **out);
void m3tsz_iter_destroy(m3tsz_iter *it);
/* Reset(reader, schema), iterator.go:253-263: the handle copies the stream bytes */
int m3tsz_iter_reset(m3tsz_iter *it, const uint8_t *data, uint64_t len);
int m3tsz_iter_next(m3tsz_iter *it); /* Next, :81-106: 1 while a datapoint is current, else 0 */
/* Current, :229-231: datapoint, the unit in force AT THIS datapoint, and its annotation
 * (valid until the next call on this iterator; NULL / 0 when the datapoint has none) */
int m3tsz_iter_current(const m3tsz_iter *it, int64_t *ts_ns, double *value, int32_t *unit,
                       const uint8_t **annotation, uint64_t *annotation_len);
int m3tsz_iter_err(const m3tsz_iter *it); /* Err, :234-236 */
int m3tsz_iter_close(m3tsz_iter *it);     /* Close, :267-278 */

/* EncoderPool.Init(alloc) / Get() / Put via Close(), encoder_pool.go:27-48 */
int m3tsz_encoder_pool_create(m3tsz_ctx *ctx, const m3tsz_options *opts, uint64_t size,
                              m3tsz_encoder_pool **out);
int m3tsz_encoder_pool_get(m3tsz_encoder_pool *pool, m3tsz_encoder **out);
void m3tsz_encoder_pool_destroy(m3tsz_encoder_pool *pool);
/* ReaderIteratorPool, iterator_pool.go:27-47 (the pooled iterators are created with a nil reader) */
int m3tsz_iter_pool_create(m3tsz_ctx *ctx, const m3tsz_options *opts, uint64_t size, m3tsz_iter_pool **out);
int m3tsz_iter_pool_get(m3tsz_iter_pool *pool, m3tsz_iter **out);
void m3tsz_iter_pool_destroy(m3tsz_iter_pool *pool);

/* ------------------------------------------------------------------------
 * Fetch-side exchange (SURVEY.md §8e, BASELINE config 5): series shard trivially, so
 * encode / decode need no collective; only a query that spans shards needs every
 * shard's DECODED blocks on every GPU.  m3tsz_allgather_decoded decodes the first
 * gather_series streams of the local shard chunk by chunk and all-gathers chunk k-1
 * over NCCL / NVLink while chunk k+1 is decoded: every chunk is decoded straight into this
 * rank's block of the gathered arrays and gathered IN PLACE (one grouped ncclAllGather per
 * chunk, no staging copies).  Every rank passes the same gather_series / max_points /
 * chunk_series (gather_series a multiple of chunk_series; 0 = 32768).  Outputs (on every
 * rank); the datapoint arrays are CHUNK-major, the layout the collective writes without a
 * second pass:
 *   d_ts_all / d_val_all : [n_chunks][n_ranks][chunk_series][max_points]; series s of rank r
 *                          sits at (((s / C) * n_ranks + r) * C + s % C) * max_points, C = chunk_series
 *   d_n_points_all / d_status_all : [n_ranks][gather_series]
 * nccl_comm is an ncclComm_t of n_ranks ranks (the caller's, or one made with
 * m3tsz_nccl_comm_create from an id broadcast out of band).  NCCL is resolved at run
 * time (dlopen of the libnccl.so.2 the process has loaded); without it the calls
 * return M3TSZ_ERR_NO_DEVICE.  d_lengths may be NULL (CSR offsets).  Asynchronous:
 * `stream` continues after the pipeline has finished.
 * ---------------------------------------------------------------------- */
int m3tsz_nccl_unique_id(uint8_t *out128);
int m3tsz_nccl_comm_create(m3tsz_ctx *ctx, const uint8_t *unique_id128, int n_ranks, int rank, void **comm);
int m3tsz_nccl_comm_destroy(void *comm);
int m3tsz_allgather_decoded(m3tsz_ctx *ctx, const m3tsz_options *opts, void *nccl_comm, int n_ranks,
                            const uint8_t *d_streams, uint64_t streams_bytes, const uint64_t *d_offsets,
                            const uint64_t *d_lengths, uint64_t n_series, uint64_t gather_series,
                            uint64_t max_points, uint64_t chunk_series, int64_t *d_ts_all, double *d_val_all,
                            uint32_t *d_n_points_all, int32_t *d_status_all, void *stream);

/* m3tsz_merge_series_batch with POINT-major arrays: point_major_in: d_ts / d_val are
 * [cap][n_seq] (datapoint i of sequence q at i * n_seq + q, what m3tsz_decode_batch_ex writes with
 * extras.point_major); point_major_out: outputs are [out_cap][n_series].  With replicas that
 * advance in step (the normal RF = 3 fetch) the threads of a warp then read and write
 * consecutive elements. */
int m3tsz_merge_series_batch_ex(m3tsz_ctx *ctx, const int64_t *d_ts, const double *d_val, uint64_t cap,
                                const uint32_t *d_n_points, const int32_t *d_seq_status,
                                const uint64_t *d_slice_off, const uint64_t *d_replica_off,
                                const uint64_t *d_series_off, uint64_t n_series, int64_t start_ns,
                                int64_t end_ns, int32_t strategy, int64_t *d_ts_out, double *d_val_out,
                                uint64_t out_cap, uint32_t *d_n_out, int32_t *d_status, uint64_t n_seq,
                                int32_t point_major_in, int32_t point_major_out, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* M3TSZ_B200_H */
