"""ctypes binding of the C ABI in include/m3tsz_b200.h (libm3tsz_b200.so).

There is no CPU fallback anywhere in this package: if the shared library has
not been built, or no CUDA device is present, the calls below raise.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# M3TSZ_B200_LIB names another build of the library to load instead, so that two builds can be compared
# run for run on the same machine
LIB_PATH = os.environ.get("M3TSZ_B200_LIB") or os.path.join(_HERE, "libm3tsz_b200.so")

OK = 0
ERR_EOF = 1
ERR_DOD_OVERFLOW = 4
ERR_NO_TIME_SCHEME = 5
ERR_UNRECOGNIZED_UNIT = 6
ERR_INVALID_MULT = 7
ERR_OUT_OF_ORDER = 13
ERR_TOO_MANY_ITERATORS = 14
ERR_TOO_MANY_ENCODERS = 16
ERR_AGGREGATION_CLOSED = 17
ERR_DUPLICATE_SOURCE = 18
ERR_CAPACITY = 100
ERR_INVALID_ARG = 101
ERR_CUDA = 102
ERR_NO_DEVICE = 103

AGG_LAST, AGG_MIN, AGG_MAX, AGG_MEAN, AGG_COUNT, AGG_SUM = 1, 2, 3, 4, 6, 7  # aggregation.Type ids
AGG_SUMSQ, AGG_STDEV = 8, 9  # the expensive aggregations (m3tsz_aggregate_tiles_ex only)
METRIC_COUNTER, METRIC_TIMER, METRIC_GAUGE = 1, 2, 3  # metric.Type ids (the Timer: element sets only)
# the Timer's further aggregation.Type ids (Timer element sets)
AGG_MEDIAN = 5
AGG_P10, AGG_P20, AGG_P30, AGG_P40, AGG_P50, AGG_P60, AGG_P70, AGG_P80, AGG_P90 = range(10, 19)
AGG_P95, AGG_P99, AGG_P999, AGG_P9999, AGG_P25, AGG_P75 = range(19, 25)
# the aggregator's default Timer types (types_options.go): Sum, SumSq, Mean, Min, Max, Count, Stdev, Median, P50, P95,
# P99, in ascending id order
DEFAULT_TIMER_TYPES = (AGG_MIN, AGG_MAX, AGG_MEAN, AGG_MEDIAN, AGG_COUNT, AGG_SUM, AGG_SUMSQ, AGG_STDEV, AGG_P50,
                       AGG_P95, AGG_P99)
MAX_TIMER_TYPES = 23  # a Timer set without transformations: every type but Last
# transformation.Type ids (m3tsz_aggregate_tiles_transform)
TRANSFORM_ABSOLUTE, TRANSFORM_PERSECOND, TRANSFORM_INCREASE, TRANSFORM_ADD, TRANSFORM_RESET = 1, 2, 3, 4, 5
MAX_TRANSFORMS = 8  # M3TSZ_MAX_TRANSFORMS
TRANSFORM_STATE_BYTES = 96  # sizeof(m3tsz_transform_state)
MAX_ELEMENT_TYPES = 8  # M3TSZ_MAX_ELEMENT_TYPES (m3tsz_aggregate_tiles_types)
ELEMENT_STATE_BYTES = 160  # sizeof(m3tsz_element_state)
MAX_ELEMENT_WINDOWS = 64  # M3TSZ_MAX_ELEMENT_WINDOWS (element sets)
MAX_ELEMENT_ANNOTATION = 65536  # M3TSZ_MAX_ELEMENT_ANNOTATION (bytes per window slot of an annotated element set)
MAX_FORWARD_SOURCES = 65536  # M3TSZ_MAX_FORWARD_SOURCES (source ids per window slot of m3tsz_element_sources)

UNIT_NONE, UNIT_S, UNIT_MS, UNIT_US, UNIT_NS, UNIT_MIN, UNIT_HOUR, UNIT_DAY, UNIT_YEAR = range(9)


class Options(C.Structure):
    """m3tsz_options: intOptimized flag + encoding.Options.DefaultTimeUnit."""
    _fields_ = [("int_optimized", C.c_int32), ("default_time_unit", C.c_int32)]


class AnnotationRef(C.Structure):
    _fields_ = [("bit_offset", C.c_uint64), ("length", C.c_uint32), ("count", C.c_uint32)]


class DpEvent(C.Structure):
    """m3tsz_dp_event: per-datapoint unit change / annotation (include/m3tsz_b200.h)."""
    _fields_ = [("series", C.c_uint64), ("dp_index", C.c_uint32), ("kind", C.c_uint16),
                ("unit", C.c_uint16), ("bit_offset", C.c_uint64), ("length", C.c_uint32),
                ("reserved", C.c_uint32)]


EVENT_TIME_UNIT, EVENT_ANNOTATION = 1, 2


class ElementSet(C.Structure):
    """m3tsz_element_set: an element set's settings (host lists) and its device arrays (include/m3tsz_b200.h)."""
    _fields_ = [("n_elements", C.c_uint64), ("n_windows", C.c_uint32), ("metric_type", C.c_int32),
                ("resolution_ns", C.c_int64), ("agg_types", C.POINTER(C.c_int32)), ("n_types", C.c_uint32),
                ("n_ops", C.c_uint32), ("ops", C.POINTER(C.c_int32)), ("discard_nan", C.c_int32),
                ("reserved", C.c_int32)] + [(f, C.c_void_p) for f in (
                    "d_win_start", "d_win_count", "d_win_sum", "d_win_min", "d_win_max", "d_win_sum_sq", "d_win_last",
                    "d_win_last_at", "d_elem", "d_watermark", "d_out_state", "d_out_buf")] + [
                ("out_stride", C.c_uint64)]


class ForwardedMetric(C.Structure):
    """m3tsz_forwarded_metric: one record of a forwarded batch, 40 bytes (include/m3tsz_b200.h)."""
    _fields_ = [("key", C.c_uint64), ("time_ns", C.c_int64), ("value_off", C.c_uint64), ("n_values", C.c_uint32),
                ("source_id", C.c_uint32), ("version", C.c_uint32), ("reserved", C.c_uint32)]


FORWARDED_METRIC_BYTES = 40


class ElementSources(C.Structure):
    """m3tsz_element_sources: the source ids each window slot of a group set has seen (include/m3tsz_b200.h)."""
    _fields_ = [("d_bits", C.c_void_p), ("capacity", C.c_uint32), ("reserved", C.c_uint32)]


class ElementAnnotations(C.Structure):
    """m3tsz_element_annotations: the window slots' annotation lengths and bytes (include/m3tsz_b200.h)."""
    _fields_ = [("d_len", C.c_void_p), ("d_bytes", C.c_void_p), ("capacity", C.c_uint32), ("reserved", C.c_uint32)]


class ElementTimerStreams(C.Structure):
    """m3tsz_element_timer_streams: the window slots' CM streams (include/m3tsz_b200.h)."""
    _fields_ = [(f, C.c_void_p) for f in ("d_header", "d_value", "d_num_ranks", "d_delta", "d_prev", "d_next",
                                          "d_heap_a", "d_heap_b")] + [
        ("sample_capacity", C.c_uint32), ("insert_and_compress_every", C.c_uint32), ("eps", C.c_double),
        ("reserved", C.c_uint64)]


TIMER_STREAM_HEADER_BYTES = 64  # sizeof(m3tsz_timer_stream_header)


class DecodeExtras(C.Structure):
    """m3tsz_decode_extras."""
    _fields_ = [("d_lengths", C.c_void_p), ("d_unit_first", C.c_void_p), ("d_events", C.c_void_p),
                ("events_capacity", C.c_uint64), ("d_event_count", C.c_void_p), ("point_major", C.c_int32),
                ("reserved", C.c_int32)]


class EncodeExtras(C.Structure):
    """m3tsz_encode_extras."""
    _fields_ = [("d_last_value", C.c_void_p), ("d_out_bits", C.c_void_p), ("point_major_input", C.c_int32),
                ("reserved", C.c_int32)]


class DownsampleOutputs(C.Structure):
    """m3tsz_downsample_outputs (device pointers; 0 = not wanted)."""
    _fields_ = [("metric_type", C.c_int32), ("reserved", C.c_int32),
                ("d_sum", C.c_void_p), ("d_min", C.c_void_p), ("d_max", C.c_void_p), ("d_sum_sq", C.c_void_p),
                ("d_last", C.c_void_p), ("d_last_at", C.c_void_p), ("d_count", C.c_void_p),
                ("d_counter_sum", C.c_void_p), ("d_counter_min", C.c_void_p), ("d_counter_max", C.c_void_p),
                ("d_counter_sum_sq", C.c_void_p), ("d_n_points", C.c_void_p), ("d_status", C.c_void_p)]


class AnnotationEntry(C.Structure):
    _fields_ = [("dp_index", C.c_uint32), ("length", C.c_uint32), ("byte_offset", C.c_uint64)]


class M3tszError(RuntimeError):
    def __init__(self, status, what=""):
        self.status = status
        msg = status_string(status)
        super().__init__("m3tsz_b200: %s (status %d)%s" % (msg, status, (": " + what) if what else ""))


_lib = None

# every symbol include/m3tsz_b200.h declares (tests check the .so exports all of them)
EXPORTED_SYMBOLS = [
    "m3tsz_version", "m3tsz_status_string", "m3tsz_ctx_create", "m3tsz_ctx_destroy",
    "m3tsz_last_cuda_error", "m3tsz_ctx_launch_count", "m3tsz_decode_batch",
    "m3tsz_decode_batch_host", "m3tsz_encode_batch", "m3tsz_encode_bound",
    "m3tsz_compact_streams", "m3tsz_encode_batch_host", "m3tsz_decode_downsample_batch",
    "m3tsz_decode_downsample_batch_host", "m3tsz_merge_series_batch", "m3tsz_checksum_batch",
    "m3tsz_decode_batch_ex", "m3tsz_decode_downsample_last_batch", "m3tsz_encode_bound_units",
    "m3tsz_encode_batch_packed", "m3tsz_encode_batch_packed_ex", "m3tsz_prom_convert_batch", "m3tsz_aggregate_tiles_batch",
    "m3tsz_encode_batch_ex", "m3tsz_fetch_batch_host", "m3tsz_merge_series_batch_ex", "m3tsz_nccl_unique_id", "m3tsz_nccl_comm_create",
    "m3tsz_nccl_comm_destroy", "m3tsz_allgather_decoded",
    "m3tsz_encoder_create", "m3tsz_encoder_destroy", "m3tsz_encoder_reset", "m3tsz_encoder_encode",
    "m3tsz_encoder_num_encoded", "m3tsz_encoder_failed_dod", "m3tsz_encoder_last_encoded", "m3tsz_encoder_last_annotation_checksum",
    "m3tsz_encoder_empty", "m3tsz_encoder_len", "m3tsz_encoder_stream", "m3tsz_encoder_close",
    "m3tsz_encoder_discard", "m3tsz_encoder_discard_reset",
    "m3tsz_iter_create", "m3tsz_iter_destroy", "m3tsz_iter_reset", "m3tsz_iter_next", "m3tsz_iter_current",
    "m3tsz_iter_err", "m3tsz_iter_close",
    "m3tsz_encoder_pool_create", "m3tsz_encoder_pool_get", "m3tsz_encoder_pool_destroy",
    "m3tsz_iter_pool_create", "m3tsz_iter_pool_get", "m3tsz_iter_pool_destroy",
    "m3tsz_encoder_set_reset", "m3tsz_encoder_set_append", "m3tsz_encoder_set_stream",
    "m3tsz_decode_downsample_ex", "m3tsz_aggregate_tiles_ex", "m3tsz_encoder_set_write",
    "m3tsz_aggregate_tiles_transform", "m3tsz_aggregate_tiles_types", "m3tsz_aggregate_tiles_annotated",
    "m3tsz_aggregate_tiles_blocks", "m3tsz_aggregate_tiles_rollup", "m3tsz_aggregate_tiles_rollup_annotated",
    "m3tsz_element_set_reset", "m3tsz_element_set_add", "m3tsz_element_set_consume",
    "m3tsz_element_set_add_annotated", "m3tsz_element_set_consume_annotated", "m3tsz_element_set_forward",
    "m3tsz_element_set_forward_annotated", "m3tsz_element_set_add_timer", "m3tsz_element_set_consume_timer",
    "m3tsz_element_set_forward_timer", "m3tsz_element_set_add_timer_annotated",
    "m3tsz_element_set_consume_timer_annotated", "m3tsz_element_set_forward_timer_annotated",
    "m3tsz_element_set_forward_write", "m3tsz_element_set_add_forwarded",
    "m3tsz_element_set_forward_write_timer", "m3tsz_element_set_add_forwarded_timer",
]

ENCODER_STATE_BYTES = 128  # sizeof(m3tsz_encoder_state)
MAX_BUCKET_ENCODERS = 12  # M3TSZ_MAX_BUCKET_ENCODERS


def lib():
    """Loads libm3tsz_b200.so.  Fails loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "m3_b200: %s is missing - build it with `python -c 'import __graft_entry__ as g; "
            "g.build()'` (nvcc, sm_90a).  This package has no CPU fallback." % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp, u64, i64, i32, u32 = C.c_void_p, C.c_uint64, C.c_int64, C.c_int32, C.c_uint32
    po = C.POINTER(Options)
    L.m3tsz_version.restype = C.c_int
    L.m3tsz_version.argtypes = []
    L.m3tsz_status_string.restype = C.c_char_p
    L.m3tsz_status_string.argtypes = [C.c_int]
    L.m3tsz_ctx_create.restype = C.c_int
    L.m3tsz_ctx_create.argtypes = [C.c_int, C.POINTER(vp)]
    L.m3tsz_ctx_destroy.restype = None
    L.m3tsz_ctx_destroy.argtypes = [vp]
    L.m3tsz_last_cuda_error.restype = C.c_char_p
    L.m3tsz_last_cuda_error.argtypes = [vp]
    L.m3tsz_ctx_launch_count.restype = u64
    L.m3tsz_ctx_launch_count.argtypes = [vp]
    L.m3tsz_encode_bound.restype = u64
    L.m3tsz_encode_bound.argtypes = [u64]
    L.m3tsz_decode_batch.restype = C.c_int
    L.m3tsz_decode_batch.argtypes = [vp, po, vp, u64, vp, u64, vp, vp, u64, vp, vp, vp, vp, vp]
    L.m3tsz_encode_bound_units.restype = u64
    L.m3tsz_encode_bound_units.argtypes = [u64, C.c_int]
    L.m3tsz_encode_batch_packed.restype = C.c_int
    L.m3tsz_encode_batch_packed.argtypes = [vp, po, vp, vp, u64, u64, vp, vp, i32, vp, vp, vp, vp, u64, u32,
                                            vp, u64, vp, vp, vp, vp, vp]
    pv, pu64 = C.POINTER(vp), C.POINTER(u64)
    L.m3tsz_encode_batch_ex.restype = C.c_int
    L.m3tsz_encode_batch_ex.argtypes = [vp, po, vp, vp, u64, u64, vp, vp, i32, vp, vp, vp, vp, vp, u64,
                                        vp, vp, C.POINTER(EncodeExtras), vp]
    L.m3tsz_encode_batch_packed_ex.restype = C.c_int
    L.m3tsz_encode_batch_packed_ex.argtypes = [vp, po, vp, vp, u64, u64, vp, vp, i32, vp, vp, vp, vp, u64, u32,
                                               vp, u64, vp, vp, vp, vp, C.POINTER(EncodeExtras), vp]
    L.m3tsz_encoder_create.restype = C.c_int
    L.m3tsz_encoder_create.argtypes = [vp, po, i64, pv]
    L.m3tsz_encoder_destroy.restype = None
    L.m3tsz_encoder_destroy.argtypes = [vp]
    L.m3tsz_encoder_reset.restype = C.c_int
    L.m3tsz_encoder_reset.argtypes = [vp, i64, u64]
    L.m3tsz_encoder_encode.restype = C.c_int
    L.m3tsz_encoder_encode.argtypes = [vp, i64, C.c_double, i32, C.c_char_p, u64]
    L.m3tsz_encoder_failed_dod.restype = i64
    L.m3tsz_encoder_failed_dod.argtypes = [vp]
    L.m3tsz_encoder_num_encoded.restype = u64
    L.m3tsz_encoder_num_encoded.argtypes = [vp]
    L.m3tsz_encoder_last_encoded.restype = C.c_int
    L.m3tsz_encoder_last_encoded.argtypes = [vp, C.POINTER(i64), C.POINTER(C.c_double)]
    L.m3tsz_encoder_last_annotation_checksum.restype = C.c_int
    L.m3tsz_encoder_last_annotation_checksum.argtypes = [vp, pu64]
    L.m3tsz_encoder_empty.restype = C.c_int
    L.m3tsz_encoder_empty.argtypes = [vp]
    L.m3tsz_encoder_len.restype = C.c_int
    L.m3tsz_encoder_len.argtypes = [vp, pu64]
    for f in ("m3tsz_encoder_stream", "m3tsz_encoder_discard"):
        getattr(L, f).restype = C.c_int
        getattr(L, f).argtypes = [vp, vp, u64, pu64, pu64]
    L.m3tsz_encoder_discard_reset.restype = C.c_int
    L.m3tsz_encoder_discard_reset.argtypes = [vp, i64, u64, vp, u64, pu64, pu64]
    L.m3tsz_encoder_close.restype = C.c_int
    L.m3tsz_encoder_close.argtypes = [vp]
    L.m3tsz_iter_create.restype = C.c_int
    L.m3tsz_iter_create.argtypes = [vp, po, pv]
    L.m3tsz_iter_destroy.restype = None
    L.m3tsz_iter_destroy.argtypes = [vp]
    L.m3tsz_iter_reset.restype = C.c_int
    L.m3tsz_iter_reset.argtypes = [vp, C.c_char_p, u64]
    L.m3tsz_iter_next.restype = C.c_int
    L.m3tsz_iter_next.argtypes = [vp]
    L.m3tsz_iter_current.restype = C.c_int
    L.m3tsz_iter_current.argtypes = [vp, C.POINTER(i64), C.POINTER(C.c_double), C.POINTER(i32), pv, pu64]
    L.m3tsz_iter_err.restype = C.c_int
    L.m3tsz_iter_err.argtypes = [vp]
    L.m3tsz_iter_close.restype = C.c_int
    L.m3tsz_iter_close.argtypes = [vp]
    for f in ("m3tsz_encoder_pool_create", "m3tsz_iter_pool_create"):
        getattr(L, f).restype = C.c_int
        getattr(L, f).argtypes = [vp, po, u64, pv]
    for f in ("m3tsz_encoder_pool_get", "m3tsz_iter_pool_get"):
        getattr(L, f).restype = C.c_int
        getattr(L, f).argtypes = [vp, pv]
    for f in ("m3tsz_encoder_pool_destroy", "m3tsz_iter_pool_destroy"):
        getattr(L, f).restype = None
        getattr(L, f).argtypes = [vp]
    L.m3tsz_nccl_unique_id.restype = C.c_int
    L.m3tsz_nccl_unique_id.argtypes = [vp]
    L.m3tsz_nccl_comm_create.restype = C.c_int
    L.m3tsz_nccl_comm_create.argtypes = [vp, vp, C.c_int, C.c_int, C.POINTER(vp)]
    L.m3tsz_nccl_comm_destroy.restype = C.c_int
    L.m3tsz_nccl_comm_destroy.argtypes = [vp]
    L.m3tsz_allgather_decoded.restype = C.c_int
    L.m3tsz_allgather_decoded.argtypes = [vp, po, vp, C.c_int, vp, u64, vp, vp, u64, u64, u64, u64, vp, vp, vp,
                                          vp, vp]
    L.m3tsz_fetch_batch_host.restype = C.c_int
    L.m3tsz_fetch_batch_host.argtypes = [vp, po, vp, u64, vp, u64, vp, vp, vp, u64, u64, i64, i64, i32, vp, vp,
                                         u64, vp, vp]
    L.m3tsz_prom_convert_batch.restype = C.c_int
    L.m3tsz_prom_convert_batch.argtypes = [vp, vp, vp, u64, vp, u64, i64, vp, C.c_double, i64, vp, vp, u64,
                                           vp, vp, vp]
    L.m3tsz_aggregate_tiles_batch.restype = C.c_int
    L.m3tsz_aggregate_tiles_batch.argtypes = [vp, po, vp, u64, vp, vp, u64, i64, i64, u32, i32, i32, u32, vp,
                                              u64, vp, vp, vp, vp, vp, vp]
    L.m3tsz_decode_batch_ex.restype = C.c_int
    L.m3tsz_decode_batch_ex.argtypes = [vp, po, vp, u64, vp, u64, vp, vp, u64, vp, vp, vp, vp,
                                        C.POINTER(DecodeExtras), vp]
    L.m3tsz_decode_downsample_last_batch.restype = C.c_int
    L.m3tsz_decode_downsample_last_batch.argtypes = [vp, po, vp, u64, vp, u64, i64, i64, u32, vp, vp, vp,
                                                     vp, vp, vp, vp, vp, vp]
    L.m3tsz_decode_batch_host.restype = C.c_int
    L.m3tsz_decode_batch_host.argtypes = [vp, po, vp, u64, vp, u64, vp, vp, u64, vp, vp, vp, vp]
    L.m3tsz_encode_batch.restype = C.c_int
    L.m3tsz_encode_batch.argtypes = [vp, po, vp, vp, u64, u64, vp, vp, i32, vp, vp, vp, vp, vp, u64,
                                     vp, vp, vp]
    L.m3tsz_encode_batch_host.restype = C.c_int
    L.m3tsz_encode_batch_host.argtypes = [vp, po, vp, vp, u64, u64, vp, vp, i32, vp, vp, vp, vp, u64,
                                          u32, vp, u64, vp, vp, vp]
    L.m3tsz_compact_streams.restype = C.c_int
    L.m3tsz_compact_streams.argtypes = [vp, vp, u64, vp, u64, u32, vp, u64, vp, vp]
    L.m3tsz_decode_downsample_batch.restype = C.c_int
    L.m3tsz_decode_downsample_batch.argtypes = [vp, po, vp, u64, vp, u64, i64, i64, u32, vp, vp, vp,
                                                vp, vp, vp, vp]
    L.m3tsz_decode_downsample_batch_host.restype = C.c_int
    L.m3tsz_decode_downsample_batch_host.argtypes = [vp, po, vp, u64, vp, u64, i64, i64, u32, vp, vp,
                                                     vp, vp, vp, vp]
    L.m3tsz_merge_series_batch.restype = C.c_int
    L.m3tsz_merge_series_batch.argtypes = [vp, vp, vp, u64, vp, vp, vp, vp, vp, u64, i64, i64, i32, vp, vp,
                                           u64, vp, vp, vp]
    L.m3tsz_merge_series_batch_ex.restype = C.c_int
    L.m3tsz_merge_series_batch_ex.argtypes = [vp, vp, vp, u64, vp, vp, vp, vp, vp, u64, i64, i64, i32, vp, vp,
                                              u64, vp, vp, u64, i32, i32, vp]
    L.m3tsz_checksum_batch.restype = C.c_int
    L.m3tsz_checksum_batch.argtypes = [vp, vp, u64, vp, vp, u64, vp, vp, vp, vp]
    L.m3tsz_encoder_set_reset.restype = C.c_int
    L.m3tsz_encoder_set_reset.argtypes = [vp, po, vp, u64, vp, vp]
    L.m3tsz_encoder_set_append.restype = C.c_int
    L.m3tsz_encoder_set_append.argtypes = [vp, po, vp, u64, vp, vp, u64, vp, i32, vp, vp, vp, vp, i32, vp, u64,
                                           vp, vp, vp]
    L.m3tsz_encoder_set_write.restype = C.c_int
    L.m3tsz_encoder_set_write.argtypes = [vp, po, vp, vp, u64, u64, vp, vp, u64, u64, vp, vp, i32, vp, vp, u64, vp,
                                          i32, vp, vp, vp, vp, i32, vp, vp, vp]
    L.m3tsz_encoder_set_stream.restype = C.c_int
    L.m3tsz_encoder_set_stream.argtypes = [vp, vp, u64, vp, u64, vp, vp]
    L.m3tsz_decode_downsample_ex.restype = C.c_int
    L.m3tsz_decode_downsample_ex.argtypes = [vp, po, vp, u64, vp, vp, u64, i64, i64, u32,
                                             C.POINTER(DownsampleOutputs), vp]
    L.m3tsz_aggregate_tiles_ex.restype = C.c_int
    L.m3tsz_aggregate_tiles_ex.argtypes = [vp, po, vp, u64, vp, vp, u64, i64, i64, u32, i32, i32, i32, u32, vp,
                                           u64, vp, vp, vp, vp, vp, vp]
    L.m3tsz_aggregate_tiles_transform.restype = C.c_int
    L.m3tsz_aggregate_tiles_transform.argtypes = [vp, po, vp, u64, vp, vp, u64, i64, i64, u32, i32, i32, i32, u32,
                                                  vp, u64, vp, vp, vp, vp, vp, C.POINTER(C.c_int32), u32, i32, vp,
                                                  vp]
    L.m3tsz_aggregate_tiles_types.restype = C.c_int
    L.m3tsz_aggregate_tiles_types.argtypes = [vp, po, vp, u64, vp, vp, u64, i64, i64, u32, i32, C.POINTER(C.c_int32),
                                              u32, i32, u32, vp, u64, vp, vp, vp, vp, vp, C.POINTER(C.c_int32), u32,
                                              i32, vp, vp]
    L.m3tsz_aggregate_tiles_annotated.restype = C.c_int
    L.m3tsz_aggregate_tiles_annotated.argtypes = L.m3tsz_aggregate_tiles_types.argtypes
    L.m3tsz_aggregate_tiles_blocks.restype = C.c_int
    L.m3tsz_aggregate_tiles_blocks.argtypes = [vp, po, vp, u64, vp, vp, u64, vp, u64, i64, i64, u32, i32,
                                               C.POINTER(C.c_int32), u32, i32, u32, vp, u64, vp, vp, vp, vp, vp,
                                               C.POINTER(C.c_int32), u32, i32, vp, i32, vp]
    pi32 = C.POINTER(C.c_int32)
    L.m3tsz_aggregate_tiles_rollup.restype = C.c_int
    L.m3tsz_aggregate_tiles_rollup.argtypes = [vp, po, vp, u64, vp, vp, u64, vp, u64, i64, i64, u32, i32, i32,
                                               pi32, u32, vp, vp, u64, u64, pi32, u32, pi32, u32, i32, vp, vp,
                                               i32, u32, vp, u64, vp, vp, vp, vp, vp, vp, vp]
    L.m3tsz_aggregate_tiles_rollup_annotated.restype = C.c_int
    L.m3tsz_aggregate_tiles_rollup_annotated.argtypes = L.m3tsz_aggregate_tiles_rollup.argtypes
    pes = C.POINTER(ElementSet)
    L.m3tsz_element_set_reset.restype = C.c_int
    L.m3tsz_element_set_reset.argtypes = [vp, po, pes, vp, vp]
    L.m3tsz_element_set_add.restype = C.c_int
    L.m3tsz_element_set_add.argtypes = [vp, po, pes, vp, vp, u64, vp, vp, vp, vp]
    L.m3tsz_element_set_consume.restype = C.c_int
    L.m3tsz_element_set_consume.argtypes = [vp, po, pes, i64, i32, vp, vp]
    pea = C.POINTER(ElementAnnotations)
    L.m3tsz_element_set_add_annotated.restype = C.c_int
    L.m3tsz_element_set_add_annotated.argtypes = [vp, po, pes, pea, vp, vp, u64, vp, vp, vp, vp, vp, vp, vp]
    L.m3tsz_element_set_consume_annotated.restype = C.c_int
    L.m3tsz_element_set_consume_annotated.argtypes = [vp, po, pes, pea, i64, i32, vp, vp]
    L.m3tsz_element_set_forward.restype = C.c_int
    L.m3tsz_element_set_forward.argtypes = [vp, po, pes, i64, vp, vp, u64, u64, pes, vp, vp, vp]
    L.m3tsz_element_set_forward_annotated.restype = C.c_int
    L.m3tsz_element_set_forward_annotated.argtypes = [vp, po, pes, pea, i64, vp, vp, u64, u64, pes, pea, vp, vp, vp]
    L.m3tsz_element_set_forward_write.restype = C.c_int
    L.m3tsz_element_set_forward_write.argtypes = [vp, po, pes, i64, vp, vp, u64, u64, vp, C.c_uint32, vp, u64, vp,
                                                  u64, vp, vp, vp, vp]
    L.m3tsz_element_set_add_forwarded.restype = C.c_int
    L.m3tsz_element_set_add_forwarded.argtypes = [vp, po, pes, C.POINTER(ElementSources), vp, u64, vp, u64, vp, vp,
                                                  vp]
    pts = C.POINTER(ElementTimerStreams)
    L.m3tsz_element_set_add_timer.restype = C.c_int
    L.m3tsz_element_set_add_timer.argtypes = [vp, po, pes, pts, vp, vp, u64, vp, vp, vp, vp, vp]
    L.m3tsz_element_set_consume_timer.restype = C.c_int
    L.m3tsz_element_set_consume_timer.argtypes = [vp, po, pes, pts, i64, i32, vp, vp]
    L.m3tsz_element_set_forward_timer.restype = C.c_int
    L.m3tsz_element_set_forward_timer.argtypes = [vp, po, pes, pts, i64, vp, vp, u64, u64, pes, pts, vp, vp, vp]
    L.m3tsz_element_set_add_timer_annotated.restype = C.c_int
    L.m3tsz_element_set_add_timer_annotated.argtypes = [vp, po, pes, pts, pea, vp, vp, u64, vp, vp, vp, vp, vp, vp,
                                                        vp, vp]
    L.m3tsz_element_set_consume_timer_annotated.restype = C.c_int
    L.m3tsz_element_set_consume_timer_annotated.argtypes = [vp, po, pes, pts, pea, i64, i32, vp, vp]
    L.m3tsz_element_set_forward_timer_annotated.restype = C.c_int
    L.m3tsz_element_set_forward_timer_annotated.argtypes = [vp, po, pes, pts, pea, i64, vp, vp, u64, u64, pes, pts,
                                                            pea, vp, vp, vp]
    L.m3tsz_element_set_forward_write_timer.restype = C.c_int
    L.m3tsz_element_set_forward_write_timer.argtypes = [vp, po, pes, pts, i64, vp, vp, u64, u64, vp, C.c_uint32, vp,
                                                        u64, vp, u64, vp, vp, vp, vp]
    L.m3tsz_element_set_add_forwarded_timer.restype = C.c_int
    L.m3tsz_element_set_add_forwarded_timer.argtypes = [vp, po, pes, pts, C.POINTER(ElementSources), vp, u64, vp,
                                                        u64, vp, vp, vp]
    _lib = L
    return L


def status_string(status):
    try:
        return lib().m3tsz_status_string(int(status)).decode()
    except Exception:  # library missing: still produce a message
        return "status %d" % status


class Context:
    """m3tsz_ctx: owns the device binding and the scratch used by *_host calls."""

    def __init__(self, device=0):
        self._h = C.c_void_p()
        rc = lib().m3tsz_ctx_create(int(device), C.byref(self._h))
        if rc != OK:
            raise M3tszError(rc, "m3tsz_ctx_create(device=%d)" % device)
        self.device = device

    @property
    def handle(self):
        return self._h

    def launch_count(self):
        return int(lib().m3tsz_ctx_launch_count(self._h))

    def last_cuda_error(self):
        return lib().m3tsz_last_cuda_error(self._h).decode()

    def check(self, rc, what=""):
        if rc != OK:
            extra = what
            if rc == ERR_CUDA:
                extra = (what + " " + self.last_cuda_error()).strip()
            raise M3tszError(rc, extra)

    def close(self):
        if self._h:
            lib().m3tsz_ctx_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
