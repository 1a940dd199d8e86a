"""ctypes binding of the aggregation oracle (tests/agg_oracle.c -> tests/libm3tsz_agg_oracle.so): the aggregator's
Gauge with expensive aggregations (sumSq, Stdev), its Counter and stdev, src/aggregator/aggregation/{gauge,counter,
common}.go.  Test infrastructure only, like oracle_lib.py; __graft_entry__.build() compiles the library, and
build_c_oracle() rebuilds it when the source is newer."""
import ctypes as C

import numpy as np

from host_build import build_c_oracle


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


_lib = None


AGG_SUMSQ, AGG_STDEV = 8, 9
AGG_LAST, AGG_MIN, AGG_MAX, AGG_MEAN, AGG_COUNT, AGG_SUM = 1, 2, 3, 4, 6, 7  # aggregation.Type ids
METRIC_COUNTER, METRIC_GAUGE = 1, 3  # metric.Type ids


def _agg_lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build_c_oracle("agg"))
        vp = C.c_void_p
        sigs = {
            "m3o_go_int64": (C.c_int64, [C.c_double]),
            "m3o_stdev": (C.c_double, [C.c_int64, C.c_double, C.c_double]),
            "m3o_downsample_gauge_ex": (None, [vp, vp, C.c_size_t, C.c_int64, C.c_int64, C.c_size_t] + [vp] * 7),
            "m3o_downsample_counter": (None, [vp, vp, C.c_size_t, C.c_int64, C.c_int64, C.c_size_t] + [vp] * 5),
            "m3o_gauge_value_of_ex": (C.c_double, [C.c_int, C.c_double, C.c_int64, C.c_double, C.c_double,
                                                   C.c_double, C.c_double]),
            "m3o_counter_value_of": (C.c_double, [C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int64]),
            "m3o_aggregate_tiles_series_ex": (C.c_size_t, [vp, vp, C.c_size_t, C.c_int64, C.c_int64, C.c_size_t,
                                                           C.c_int, C.c_int, vp, vp]),
        }
        for name, (res, args) in sigs.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def go_int64(v):
    return int(_agg_lib().m3o_go_int64(float(v)))


def stdev(count, sum_sq, sum_):
    return float(_agg_lib().m3o_stdev(int(count), float(sum_sq), float(sum_)))


def downsample_gauge_ex(ts, vals, range_start_ns, window_ns, n_windows):
    """-> (sum, count, min, max, last, last_at, sum_sq), one entry per window."""
    ts = np.ascontiguousarray(ts, dtype=np.int64)
    vals = np.ascontiguousarray(vals, dtype=np.float64)
    f = [np.empty(n_windows, dtype=np.float64) for _ in range(5)]
    c = np.empty(n_windows, dtype=np.int64)
    la = np.empty(n_windows, dtype=np.int64)
    _agg_lib().m3o_downsample_gauge_ex(_ptr(ts), _ptr(vals), len(ts), int(range_start_ns), int(window_ns), n_windows,
                                       _ptr(f[0]), _ptr(c), _ptr(f[1]), _ptr(f[2]), _ptr(f[3]), _ptr(la), _ptr(f[4]))
    return f[0], c, f[1], f[2], f[3], la, f[4]


def downsample_counter(ts, vals, range_start_ns, window_ns, n_windows):
    """-> (sum, count, min, max, sum_sq) int64, one entry per window."""
    ts = np.ascontiguousarray(ts, dtype=np.int64)
    vals = np.ascontiguousarray(vals, dtype=np.float64)
    o = [np.empty(n_windows, dtype=np.int64) for _ in range(5)]
    _agg_lib().m3o_downsample_counter(_ptr(ts), _ptr(vals), len(ts), int(range_start_ns), int(window_ns), n_windows,
                                      *[_ptr(a) for a in o])
    return tuple(o)


def gauge_value_of_ex(agg_type, s, c, mn, mx, last, sum_sq):
    return float(_agg_lib().m3o_gauge_value_of_ex(int(agg_type), float(s), int(c), float(mn), float(mx),
                                                  float(last), float(sum_sq)))


def counter_value_of(agg_type, s, c, mn, mx, sum_sq):
    return float(_agg_lib().m3o_counter_value_of(int(agg_type), int(s), int(c), int(mn), int(mx), int(sum_sq)))


def aggregate_tiles_series_ex(ts, vals, start_ns, step_ns, n_windows, metric_type, agg_type):
    ts = np.ascontiguousarray(ts, dtype=np.int64)
    vals = np.ascontiguousarray(vals, dtype=np.float64)
    to = np.zeros(max(1, n_windows), dtype=np.int64)
    vo = np.zeros(max(1, n_windows), dtype=np.float64)
    n = _agg_lib().m3o_aggregate_tiles_series_ex(_ptr(ts), _ptr(vals), len(ts), int(start_ns), int(step_ns),
                                                 int(n_windows), int(metric_type), int(agg_type), _ptr(to), _ptr(vo))
    return to[:n].copy(), vo[:n].copy()
