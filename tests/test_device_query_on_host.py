"""The Prometheus-epilogue kernels (m3_b200/csrc/m3tsz_query.cu: `prom_simple_kernel`, one warp per series, and
`prom_general_kernel`, one thread per series) compiled for the host from the CUDA source and run thread by thread
the way `launch_prom` picks and shapes them; compared with the oracle's iteratorToPromResult restatement and the
independent Python one (tests/test_independent_query_rows.py) on random batches: counters with resets, tolerance
clamps, NaN, empty series, output capacity overflow, and rows whose count exceeds their capacity (refused unread)."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O
from host_build import compile, cut, source_text
from test_independent_query_rows import prom_convert

SEC = 10 ** 9

DRIVER = r"""
extern "C" int dev_prom(const int64_t *ts, const double *val, uint64_t cap, const uint32_t *n_points, uint64_t n_series,
                        int64_t resolution, const uint8_t *handle_resets, double tolerance, int64_t tolerance_until,
                        int64_t *ts_out, double *val_out, uint64_t out_cap, uint32_t *n_out, int32_t *status) {
  using namespace m3tsz;
  PromParams p;
  memset(&p, 0, sizeof(p));
  p.ts = ts; p.val = val; p.cap = cap; p.n_points = n_points; p.n_series = n_series; p.resolution = resolution;
  p.handle_resets = handle_resets; p.tolerance = tolerance; p.tolerance_until = tolerance_until;
  p.ts_out = ts_out; p.val_out = val_out; p.out_cap = out_cap; p.n_out = n_out; p.status = status;
  blockDim.x = 256;
  const bool simple = !(p.tolerance > 0) && !p.handle_resets;  // launch_prom
  const uint64_t threads = simple ? n_series * 32ull : n_series;
  for (uint64_t t = 0; t < threads; t++) {
    blockIdx.x = (unsigned)(t / 256);
    threadIdx.x = (unsigned)(t % 256);
    if (simple) prom_simple_kernel(p); else prom_general_kernel(p);
  }
  return simple ? 1 : 0;
}
"""


@pytest.fixture(scope="module")
def dev():
    src = source_text("m3tsz_query.cu")
    body = src[src.index("namespace m3tsz {"): src.index("cudaError_t launch_prom")] + "\n}  // namespace m3tsz\n"
    params = "namespace m3tsz {\n" + cut(source_text("m3tsz_kernels.h"), r"struct PromParams") + "\n}\n"
    assert "<<<" not in body
    lib = compile("dev_query_host", params + body, DRIVER)
    lib.dev_prom.restype = C.c_int
    return lib


def _batch(rng, S, cap):
    ts = np.zeros((S, cap), dtype=np.int64)
    vals = np.zeros((S, cap), dtype=np.float64)
    n = rng.integers(0, cap + 1, size=S).astype(np.uint32)
    n[:3] = [0, 1, cap]
    for s in range(S):
        k = int(n[s])
        t0 = 1599955200 * SEC + int(rng.integers(0, 10 ** 9))
        ts[s, :k] = t0 + np.cumsum(rng.integers(1, 120, size=k)) * SEC // 2
        kind = s % 3
        if kind == 0 and k:
            inc = np.abs(np.round(rng.normal(size=k) * 10, 1))
            v = np.cumsum(inc)
            for r in rng.integers(0, k, size=max(1, k // 30)):
                v[r:] -= v[r] - inc[r]
            vals[s, :k] = v
        elif kind == 1 and k:
            v = 1000.0 + np.cumsum(np.abs(rng.normal(size=k)))
            v[rng.integers(0, k, size=max(1, k // 10))] *= (1 - 10.0 ** -rng.integers(2, 7))
            vals[s, :k] = v
        elif k:
            v = rng.normal(size=k) * 100
            v[rng.integers(0, k, size=max(1, k // 20))] = np.nan
            vals[s, :k] = v
    return ts, vals, n


@pytest.mark.parametrize("mode", ["simple", "tolerance", "resets", "both", "small_cap"])
def test_prom_kernels_on_host_match_oracle_and_model(dev, mode):
    rng = np.random.default_rng({"simple": 1, "tolerance": 2, "resets": 3, "both": 4, "small_cap": 5}[mode])
    S, cap = 90, 70
    ts, vals, n = _batch(rng, S, cap)
    resolution = 300 * SEC
    tol = 1e-3 if mode in ("tolerance", "both", "small_cap") else 0.0
    until = int(ts[:, : cap // 2].max()) if tol else 0
    handle = None
    if mode in ("resets", "both", "small_cap"):
        handle = (rng.random(S) < 0.6).astype(np.uint8)
    out_cap = cap + 1 if mode != "small_cap" else 20
    t_out, v_out, n_out, st, was_simple = _convert(dev, ts, vals, n, S, cap, resolution, handle, tol, until, out_cap)
    assert was_simple == (1 if mode == "simple" else 0)
    for s in range(S):
        _assert_series(ts, vals, n, s, resolution, handle, tol, until, out_cap, t_out, v_out, n_out, st)


T_FILL, V_FILL = -777, np.uint64(0x7FF4DEADBEEF0001)  # output prefill: an int and a NaN bit pattern nobody computes


def _convert(dev, ts, vals, n, S, cap, resolution, handle, tol, until, out_cap):
    """runs the epilogue over the first S rows of ts / vals (which may have more rows) into prefilled outputs"""
    t_out = np.full((S, out_cap), T_FILL, dtype=np.int64)
    v_out = np.full((S, out_cap), V_FILL, dtype=np.uint64).view(np.float64)
    n_out = np.full(S, 12345, dtype=np.uint32)
    st = np.full(S, -1, dtype=np.int32)
    p = lambda a: C.c_void_p(a.ctypes.data)
    was_simple = dev.dev_prom(p(ts), p(vals), C.c_uint64(cap), p(n), C.c_uint64(S), C.c_int64(resolution),
                              None if handle is None else p(handle), C.c_double(tol), C.c_int64(until), p(t_out),
                              p(v_out), C.c_uint64(out_cap), p(n_out), p(st))
    return t_out, v_out, n_out, st, was_simple


def _assert_series(ts, vals, n, s, resolution, handle, tol, until, out_cap, t_out, v_out, n_out, st):
    """series s equals the oracle's and the independent model's conversion of its n[s] datapoints"""
    k = int(n[s])
    h = bool(handle[s]) if handle is not None else False
    o_ts, o_v = O.prom_convert_series(ts[s, :k], vals[s, :k], resolution, h, tol, until)
    ref = prom_convert(ts[s, :k].tolist(), vals[s, :k].tolist(), resolution, h, tol, until)
    assert len(ref) == len(o_ts) == int(n_out[s]), (s, len(ref), len(o_ts), int(n_out[s]))
    assert int(st[s]) == (100 if len(ref) > out_cap else 0), s  # M3TSZ_ERR_CAPACITY
    m = min(len(ref), out_cap)
    assert t_out[s, :m].tolist() == o_ts[:m].tolist() == [r[0] for r in ref[:m]], s
    assert (v_out[s, :m].view(np.uint64) == o_v[:m].view(np.uint64)).all(), s


@pytest.mark.parametrize("mode", ["simple", "tolerance", "resets"])
def test_prom_kernels_on_host_refuse_rows_shorter_than_their_count(dev, mode):
    """n_points[s] > cap is what decode and merge report for a row that hit its capacity.  Such a series gets
    INVALID_ARG and n_out 0, and its output row keeps what was there; its input row is not read (the rows after the
    last series hold sentinels that would be converted otherwise).  A series with n_points == cap right before it and
    every other series convert as usual."""
    rng = np.random.default_rng({"simple": 11, "tolerance": 12, "resets": 13}[mode])
    S, cap, extra = 40, 24, 2
    ts, vals, n = _batch(rng, S + extra, cap)  # rows S.. are memory after the last series
    ts[S:] = 1599955200 * SEC
    vals[S:] = 4321.0
    n = n[:S].copy()
    mid, last = S // 2, S - 1
    n[mid - 1], n[mid], n[last] = cap, cap + 3, cap + cap // 2
    resolution = 300 * SEC
    tol = 1e-3 if mode == "tolerance" else 0.0
    until = int(ts[:S].max()) if tol else 0
    handle = (np.arange(S) % 3 != 1).astype(np.uint8) if mode == "resets" else None
    out_cap = cap + 1
    t_out, v_out, n_out, st, was_simple = _convert(dev, ts, vals, n, S, cap, resolution, handle, tol, until, out_cap)
    assert was_simple == (1 if mode == "simple" else 0)
    for s in range(S):
        if s in (mid, last):
            assert int(st[s]) == 101 and int(n_out[s]) == 0, (s, int(st[s]), int(n_out[s]))  # M3TSZ_ERR_INVALID_ARG
            assert (t_out[s] == T_FILL).all() and (v_out[s].view(np.uint64) == V_FILL).all(), s
        else:
            _assert_series(ts, vals, n, s, resolution, handle, tol, until, out_cap, t_out, v_out, n_out, st)
