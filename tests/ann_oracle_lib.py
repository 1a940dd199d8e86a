"""ctypes binding of the window-annotation oracle (tests/ann_oracle.c -> tests/libm3tsz_ann_oracle.so), and the tile
path of m3tsz_aggregate_tiles_annotated composed from the oracles: the reference iterator's per-datapoint annotations
(oracle_lib), the window rule (ann_oracle.c), the element (elem_oracle_lib over the aggregation oracle's windows) and
the reference encoder writing every datapoint of a window with the window's annotation.  Test infrastructure only,
like elem_oracle_lib.py; __graft_entry__.build() compiles the library, and build_c_oracle() rebuilds it when the
source is newer."""
import ctypes as C

import numpy as np

import elem_oracle_lib as E
import oracle_lib as O
from host_build import build_c_oracle

TRANSFORM_RESET = 5


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


_lib = None


def _ann_lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build_c_oracle("ann"))
        vp = C.c_void_p
        L.m3o_window_annotations.restype = None
        L.m3o_window_annotations.argtypes = [vp, vp, C.c_size_t, C.c_int64, C.c_int64, C.c_size_t, vp]
        _lib = L
    return _lib


def window_annotations(ts, ann_ids, start_ns, step_ns, n_windows):
    """the id (ann_ids[i], -1 for none) of the annotation each window keeps: the last datapoint in stream order that
    falls in the window and carries one; -1 when there is none"""
    ts = np.ascontiguousarray(ts, dtype=np.int64)
    ids = np.ascontiguousarray(ann_ids, dtype=np.int64)
    out = np.empty(max(1, n_windows), dtype=np.int64)
    _ann_lib().m3o_window_annotations(_ptr(ts), _ptr(ids), len(ts), int(start_ns), int(step_ns), int(n_windows),
                                      _ptr(out))
    return out[:n_windows].copy()


def decode_annotated(stream, int_optimized, default_unit=O.UNIT_S):
    """the reference iterator over one stream (oracle/m3tsz_oracle.c): (ts, values, the annotation Current() reports
    on each datapoint (b"" for none), err)"""
    it = O.Iterator(bytes(stream), int_optimized, default_unit)
    ts, vals, anns = [], [], []
    while it.next():
        t, v, _, a = it.current()
        ts.append(t)
        vals.append(v)
        anns.append(a)
    return np.array(ts, dtype=np.int64), np.array(vals, dtype=np.float64), anns, it.err()


def aggregate_tiles_annotated_series(stream, int_optimized, start_ns, step_ns, n_windows, metric_type, agg_types,
                                     ops, discard_nan, state, out_unit=O.UNIT_S, default_unit=O.UNIT_S):
    """m3tsz_aggregate_tiles_annotated for one source stream; `state` (elem_oracle_lib.new_element_state()) is
    updated in place unless the source fails.  -> (stream bytes per type, datapoints per type, source error)"""
    ts, vals, anns, err = decode_annotated(stream, int_optimized, default_unit)
    k = len(agg_types)
    if err:
        return [b""] * k, [0] * k, err
    ids = np.array([i if a else -1 for i, a in enumerate(anns)], dtype=np.int64)
    win = window_annotations(ts, ids, start_ns, step_ns, n_windows)
    wt, wv = E.element_windows(ts, vals, start_ns, step_ns, n_windows, metric_type, agg_types)
    res = E.element_series(ops, discard_nan, step_ns, k, state, wt, wv)
    reset = TRANSFORM_RESET in [int(o) for o in ops]
    rw = int(max(float(int(step_ns) // 2), 1.0))
    streams, counts = [], []
    for j in range(k):
        to, vo = res[j]
        enc = O.Encoder(int(start_ns), int_optimized, default_unit)
        i = 0
        for t in wt.tolist():  # a type writes a window's datapoint, then its Reset datapoint, or neither
            if i < len(to) and int(to[i]) == t:
                w = (t - int(start_ns)) // int(step_ns) - 1
                a = anns[win[w]] if win[w] >= 0 else b""
                for _ in range(2 if (reset and t + rw != 0) else 1):
                    rc = enc.encode(int(to[i]), float(vo[i]), out_unit, a)
                    assert rc == 0, rc
                    i += 1
        assert i == len(to)
        streams.append(enc.stream() or b"")
        counts.append(len(to))
    return streams, counts, 0
