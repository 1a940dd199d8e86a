"""ctypes binding of the Timer oracle (tests/timer_oracle.c -> tests/libm3tsz_timer_oracle.so): aggregation.Timer over
cm.Stream for one window or many.  Test infrastructure only; __graft_entry__.build() compiles the library."""
import ctypes as C

import numpy as np

from host_build import build_c_oracle

_lib = None


def _timer_lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build_c_oracle("timer"))
        vp = C.c_void_p
        L.m3o_timer_window.restype = None
        L.m3o_timer_window.argtypes = [vp, vp, C.c_size_t, vp, C.c_size_t, C.c_double, C.c_int64, vp, vp]
        L.m3o_timer_windows.restype = None
        L.m3o_timer_windows.argtypes = [vp, vp, vp, vp, C.c_size_t, C.c_size_t, vp, C.c_size_t, C.c_double,
                                        C.c_int64, vp, vp]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def timer_window(batches, types, eps=1e-3, every=1024):
    """ValueOf of every type after AddBatch of each batch (a list of value lists) -> (values [k], peak list + pending
    count after a batch)"""
    v = np.ascontiguousarray(np.concatenate([np.asarray(b, dtype=np.float64) for b in batches])
                             if batches else np.zeros(0), dtype=np.float64)
    bl = np.array([len(b) for b in batches], dtype=np.uint32)
    ty = np.ascontiguousarray(types, dtype=np.int32)
    out = np.zeros(max(1, len(ty)), dtype=np.float64)
    peak = np.zeros(1, dtype=np.int64)
    _timer_lib().m3o_timer_window(_ptr(v), _ptr(bl), len(bl), _ptr(ty), len(ty), float(eps), int(every), _ptr(out),
                                  _ptr(peak))
    return out[: len(ty)], int(peak[0])


def timer_windows(values, v_off, batch_len, b_off, types, eps=1e-3, every=1024, w0=0, w1=None, out=None, peak=None):
    """m3o_timer_windows over windows [w0, w1) of the CSR arrays (numpy); out [W, k] float64, peak [W] int64"""
    W = len(v_off) - 1
    w1 = W if w1 is None else w1
    ty = np.ascontiguousarray(types, dtype=np.int32)
    if out is None:
        out = np.zeros((W, len(ty)), dtype=np.float64)
    if peak is None:
        peak = np.zeros(W, dtype=np.int64)
    _timer_lib().m3o_timer_windows(_ptr(values), _ptr(v_off), _ptr(batch_len), _ptr(b_off), w0, w1, _ptr(ty),
                                   len(ty), float(eps), int(every), _ptr(out), _ptr(peak))
    return out, peak
