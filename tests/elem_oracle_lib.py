"""ctypes binding of the multi-type element oracle (tests/elem_oracle.c -> tests/libm3tsz_elem_oracle.so): what an
element with several aggregation types writes for its flushed windows, GenericElem.processValue's loop over
e.aggTypes.  Test infrastructure only, like xf_oracle_lib.py; __graft_entry__.build() compiles the library, and
build_c_oracle() rebuilds it when the source is newer.  The tile path (decode -> downsample -> ValueOf of every
type -> the element) composes this oracle with the aggregation oracle (agg_oracle_lib.aggregate_tiles_series_ex)."""
import ctypes as C

import numpy as np

import agg_oracle_lib as A
from host_build import build_c_oracle

# m3tsz_element_state: m3tsz_transform_state (type 0's binary-op input in prev_v), then types 1..7's (160 bytes)
ELEM_STATE_DTYPE = np.dtype([("has_prev", "<i4"), ("reserved0", "<i4"), ("prev_t", "<i8"), ("prev_v", "<f8"),
                             ("sum", "<f8", (8,)), ("reserved1", "<u8"), ("prev_v_more", "<f8", (7,)),
                             ("reserved", "<u8")])
assert ELEM_STATE_DTYPE.itemsize == 160


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


_lib = None


def _elem_lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build_c_oracle("elem"))
        vp = C.c_void_p
        L.m3o_element_series.restype = None
        L.m3o_element_series.argtypes = [vp, C.c_size_t, C.c_int, C.c_int64, C.c_size_t, vp, vp, vp, C.c_size_t,
                                         vp, vp, vp]
        _lib = L
    return _lib


def new_element_state():
    """one zeroed record (a new element), a numpy structured array of shape (1,), updated in place"""
    return np.zeros(1, dtype=ELEM_STATE_DTYPE)


def element_series(ops, discard_nan, step_ns, n_types, state, t, v):
    """the flush of non-empty windows: t[i] the window's end, v[i][j] type j's value there; `state`
    (new_element_state()) is updated.  -> [(ts, values) written by type j, Reset datapoints included]"""
    ops_a = np.ascontiguousarray(ops, dtype=np.int32)
    t = np.ascontiguousarray(t, dtype=np.int64)
    v = np.ascontiguousarray(np.asarray(v, dtype=np.float64).reshape(len(t), n_types))
    n = len(t)
    to = np.zeros(max(1, n_types * 2 * n), dtype=np.int64)
    vo = np.zeros(max(1, n_types * 2 * n), dtype=np.float64)
    cnt = np.zeros(max(1, n_types), dtype=np.uint64)
    _elem_lib().m3o_element_series(_ptr(ops_a), len(ops_a), int(bool(discard_nan)), int(step_ns), n_types,
                                   _ptr(state), _ptr(t), _ptr(v), n, _ptr(to), _ptr(vo), _ptr(cnt))
    return [(to[j * 2 * n: j * 2 * n + int(cnt[j])].copy(), vo[j * 2 * n: j * 2 * n + int(cnt[j])].copy())
            for j in range(n_types)]


def element_windows(ts, vals, start_ns, step_ns, n_windows, metric_type, agg_types):
    """decode -> downsample -> ValueOf of every type (the aggregation oracle's tiles) for one series:
    (window ends, values [n, k])"""
    wt, cols = None, []
    for a in agg_types:
        t, v = A.aggregate_tiles_series_ex(ts, vals, start_ns, step_ns, n_windows, metric_type, a)
        assert wt is None or np.array_equal(wt, t)
        wt = t
        cols.append(np.asarray(v, dtype=np.float64))
    return np.asarray(wt, dtype=np.int64), np.stack(cols, axis=1) if cols else np.zeros((0, 0))


def aggregate_tiles_types_series(ts, vals, start_ns, step_ns, n_windows, metric_type, agg_types, ops, discard_nan,
                                 state):
    """the tile path of one series for an element's types; `state` is updated in place -> [(ts, values)] per type"""
    wt, wv = element_windows(ts, vals, start_ns, step_ns, n_windows, metric_type, agg_types)
    return element_series(ops, discard_nan, step_ns, len(agg_types), state, wt, wv)
