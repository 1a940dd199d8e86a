"""ctypes binding of the transformation oracle (tests/xf_oracle.c -> tests/libm3tsz_xf_oracle.so): what the
aggregator's transformations do to a flushed window's value, src/metrics/transformation and GenericElem.processValue.
Test infrastructure only, like agg_oracle_lib.py; __graft_entry__.build() compiles the library, and
build_c_oracle() rebuilds it when the source is newer.  The tile path (decode -> downsample -> ValueOf ->
transformations) composes this oracle with the aggregation oracle (agg_oracle_lib.aggregate_tiles_series_ex)."""
import ctypes as C

import numpy as np

import agg_oracle_lib as A
from host_build import build_c_oracle

XF_ABSOLUTE, XF_PERSECOND, XF_INCREASE, XF_ADD, XF_RESET = 1, 2, 3, 4, 5  # transformation.Type ids
# m3tsz_transform_state: has_prev, reserved, prev_t, prev_v, sum[8], reserved (96 bytes)
XF_STATE_DTYPE = np.dtype([("has_prev", "<i4"), ("reserved0", "<i4"), ("prev_t", "<i8"), ("prev_v", "<f8"),
                           ("sum", "<f8", (8,)), ("reserved1", "<u8")])
assert XF_STATE_DTYPE.itemsize == 96


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


_lib = None


def _xf_lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build_c_oracle("xf"))
        vp = C.c_void_p
        L.m3o_transform_series.restype = C.c_size_t
        L.m3o_transform_series.argtypes = [vp, C.c_size_t, C.c_int, C.c_int64, vp, vp, vp, C.c_size_t, vp, vp]
        _lib = L
    return _lib


def new_transform_state():
    """one zeroed state record (a new element), a numpy structured array of shape (1,), updated in place"""
    return np.zeros(1, dtype=XF_STATE_DTYPE)


def transform_series(ops, discard_nan, step_ns, state, t, v):
    """the flush of non-empty windows (t[i], v[i]) through `ops`; `state` (new_transform_state()) is updated.
    -> (ts, values) written, Reset datapoints included"""
    ops_a = np.ascontiguousarray(ops, dtype=np.int32)
    t = np.ascontiguousarray(t, dtype=np.int64)
    v = np.ascontiguousarray(v, dtype=np.float64)
    to = np.zeros(max(1, 2 * len(t)), dtype=np.int64)
    vo = np.zeros(max(1, 2 * len(t)), dtype=np.float64)
    n = _xf_lib().m3o_transform_series(_ptr(ops_a), len(ops_a), int(bool(discard_nan)), int(step_ns), _ptr(state),
                                       _ptr(t), _ptr(v), len(t), _ptr(to), _ptr(vo))
    return to[:n].copy(), vo[:n].copy()


def aggregate_tiles_transform_series(ts, vals, start_ns, step_ns, n_windows, metric_type, agg_type, ops, discard_nan,
                                     state):
    """decode -> downsample -> ValueOf (the aggregation oracle's tiles: one datapoint per non-empty window) ->
    transformations, for one series; `state` is updated in place"""
    wt, wv = A.aggregate_tiles_series_ex(ts, vals, start_ns, step_ns, n_windows, metric_type, agg_type)
    return transform_series(ops, discard_nan, step_ns, state, wt, wv)
