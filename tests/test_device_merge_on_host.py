"""The series-merge kernels (m3_b200/csrc/m3tsz_merge.cu: `merge_fast_kernel` and the general `merge_kernel`, one
thread per series) compiled for the host from the CUDA source text -- everything between `namespace m3tsz {` and the
launcher, with `MergeParams` cut out of m3tsz_kernels.h -- and run series by series with threadIdx / blockIdx set
the way the launcher would (`launch_merge`: the fast kernel first for the last-pushed strategy, then the general
kernel on the series it gave up on).  Compared with the merge oracle AND with the independent Python object model
of tests/test_independent_merge.py on random fetch shapes (reader errors, out-of-order blocks, empty slices, range
filters, all four strategies), series-major and point-major strides."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O
import test_independent_merge as M
from host_build import compile, cut, source_text

DRIVER = r"""
extern "C" void dev_merge(const int64_t *ts, const double *val, uint64_t cap, const uint32_t *n_points,
                          const int32_t *seq_status, const uint64_t *slice_off, const uint64_t *replica_off,
                          const uint64_t *series_off, uint64_t n_series, int64_t start, int64_t end, int strategy,
                          int64_t *ts_out, double *val_out, uint64_t out_cap, uint32_t *n_out, int32_t *status,
                          uint64_t in_seq_stride, uint64_t in_pt_stride, uint64_t out_seq_stride,
                          uint64_t out_pt_stride, int *n_fast) {
  using namespace m3tsz;
  MergeParams p;
  memset(&p, 0, sizeof(p));
  p.ts = ts; p.val = val; p.cap = cap; p.n_points = n_points; p.seq_status = seq_status;
  p.slice_off = slice_off; p.replica_off = replica_off; p.series_off = series_off; p.n_series = n_series;
  p.start = start; p.end = end; p.strategy = strategy;
  p.ts_out = ts_out; p.val_out = val_out; p.out_cap = out_cap; p.n_out = n_out; p.status = status;
  p.in_seq_stride = in_seq_stride; p.in_pt_stride = in_pt_stride;
  p.out_seq_stride = out_seq_stride; p.out_pt_stride = out_pt_stride;
  blockDim.x = 128;
  const bool fast = (strategy == 0);  // launch_merge
  *n_fast = 0;
  for (int pass = fast ? 0 : 1; pass < 2; pass++)
    for (uint64_t s = 0; s < n_series; s++) {
      blockIdx.x = (unsigned)(s / 128);
      threadIdx.x = (unsigned)(s % 128);
      if (pass == 0) {
        merge_fast_kernel(p);
        if (status[s] != MRG_REDO) (*n_fast)++;
      } else {
        merge_kernel(p, fast);
      }
    }
}
"""


@pytest.fixture(scope="module")
def dev():
    src = source_text("m3tsz_merge.cu")
    body = src[src.index("namespace m3tsz {"): src.index("cudaError_t launch_merge")] + "\n}  // namespace m3tsz\n"
    params = "namespace m3tsz {\n" + cut(source_text("m3tsz_kernels.h"), r"struct MergeParams") + "\n}\n"
    assert "<<<" not in body
    lib = compile("dev_merge_host", params + body, DRIVER)
    lib.dev_merge.restype = None
    return lib


def _run(dev, ts, vals, n_points, status, slice_off, replica_off, series_off, start, end, strategy, point_major):
    n_series = len(series_off) - 1
    n_seq, cap = ts.shape
    out_cap = max(1, int(n_points.sum()))
    so = np.ascontiguousarray(slice_off, dtype=np.uint64)
    ro = np.ascontiguousarray(replica_off, dtype=np.uint64)
    se = np.ascontiguousarray(series_off, dtype=np.uint64)
    if point_major:  # [cap][n_seq] inputs, [out_cap][n_series] outputs
        tin, vin = np.ascontiguousarray(ts.T), np.ascontiguousarray(vals.T)
        t_out = np.zeros((out_cap, n_series), dtype=np.int64)
        v_out = np.zeros((out_cap, n_series), dtype=np.float64)
        strides = (1, n_seq, 1, n_series)
    else:
        tin, vin = np.ascontiguousarray(ts), np.ascontiguousarray(vals)
        t_out = np.zeros((n_series, out_cap), dtype=np.int64)
        v_out = np.zeros((n_series, out_cap), dtype=np.float64)
        strides = (cap, 1, out_cap, 1)
    n_out = np.zeros(n_series, dtype=np.uint32)
    st = np.zeros(n_series, dtype=np.int32)
    n_fast = C.c_int()
    p = lambda a: C.c_void_p(a.ctypes.data)
    dev.dev_merge(p(tin), p(vin), C.c_uint64(cap), p(n_points), p(status), p(so), p(ro), p(se), C.c_uint64(n_series),
                  C.c_int64(start), C.c_int64(end), C.c_int(strategy), p(t_out), p(v_out), C.c_uint64(out_cap),
                  p(n_out), p(st), *[C.c_uint64(x) for x in strides], C.byref(n_fast))
    if point_major:
        t_out, v_out = t_out.T, v_out.T
    return t_out, v_out, n_out, st, n_fast.value


@pytest.mark.parametrize("seed", range(5))
@pytest.mark.parametrize("strategy", [0, 1, 2, 3])
def test_merge_kernels_on_host_match_oracle(dev, seed, strategy):
    rng = np.random.default_rng(900 + seed * 5 + strategy)
    n_series = 150
    seqs, ts, vals, n_points, status, slice_off, replica_off, series_off, base = M._random_case(rng, n_series)
    fast_total = 0
    for flt in (False, True):
        start, end = (base + 15 * 10 ** 9, base + 95 * 10 ** 9) if flt else (0, 0)
        o_ts, o_val, o_n, o_st = O.series_merge_batch(ts, vals, n_points, status, slice_off, replica_off, series_off,
                                                      start=start, end=end, strategy=strategy,
                                                      out_cap=max(1, int(n_points.sum())))
        for point_major in (False, True):
            d_ts, d_val, d_n, d_st, n_fast = _run(dev, ts, vals, n_points, status, slice_off, replica_off, series_off,
                                                  start, end, strategy, point_major)
            assert (d_st == o_st).all(), np.nonzero(d_st != o_st)[0][:5]
            assert (d_n == o_n).all()
            for s in range(n_series):
                k = int(o_n[s])
                assert (d_ts[s, :k] == o_ts[s, :k]).all(), s
                assert (d_val[s, :k].view(np.uint64) == o_val[s, :k].view(np.uint64)).all(), s
            fast_total += n_fast
    if strategy == 0:
        assert fast_total > 0  # the register-resident fast kernel handled part of the batch itself


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("strategy", [0, 1, 2, 3])
def test_merge_kernels_on_host_special_values(dev, seed, strategy):
    """the special-value batches of test_independent_merge (NaN payloads, +-Inf, +-0 at equal timestamps, 1-12
    replicas, 1-4 readers per slice; and 1-4 replicas of single-reader slices, the fast kernel's shape), filter on
    and off, both layouts: every value bit for bit against the oracle"""
    from test_merge_oracle import build
    rng = np.random.default_rng(1300 + seed * 5 + strategy)
    series = M.special_value_series(rng, 60) + M.special_value_series(rng, 60, replicas=(1, 4), readers=(1, 1))
    ts, vals, npts, st, slice_off, replica_off, series_off = build(series)
    fast_total = 0
    for start, end in ((0, 0), M.SPECIAL_RANGE):
        o_ts, o_val, o_n, o_st = O.series_merge_batch(ts, vals, npts, st, slice_off, replica_off, series_off,
                                                      start=start, end=end, strategy=strategy,
                                                      out_cap=max(1, int(npts.sum())))
        for point_major in (False, True):
            d_ts, d_val, d_n, d_st, n_fast = _run(dev, ts, vals, npts, st, slice_off, replica_off, series_off,
                                                  start, end, strategy, point_major)
            assert (d_st == o_st).all() and (d_n == o_n).all()
            for s in range(len(series)):
                k = int(o_n[s])
                assert (d_ts[s, :k] == o_ts[s, :k]).all(), s
                assert (d_val[s, :k].view(np.uint64) == o_val[s, :k].view(np.uint64)).all(), s
            fast_total += n_fast
    if strategy == 0:
        assert fast_total > 0


def test_merge_kernels_on_host_rf3_fetch_shape(dev):
    """the shape a fetch normally has (and the bench measures): 3 replicas x 1 block x 1 reader, identical
    timestamps, replica values that differ now and then -- all of it on the fast kernel"""
    rng = np.random.default_rng(77)
    S, P = 200, 64
    base = 1_600_000_000 * 10 ** 9
    ts = np.tile(base + np.arange(P, dtype=np.int64) * 60 * 10 ** 9, (S * 3, 1))
    vals = np.repeat(np.round(rng.normal(size=(S, P)) * 10), 3, axis=0)
    flip = rng.random(vals.shape) < 0.05
    vals[flip] += 1.0
    n_points = np.full(S * 3, P, dtype=np.uint32)
    n_points[rng.integers(0, S * 3, size=20)] = rng.integers(0, P, size=20)
    status = np.zeros(S * 3, dtype=np.int32)
    ar = lambda step: np.arange(0, S * 3 + 1, step, dtype=np.uint64)
    o = O.series_merge_batch(ts, vals, n_points, status, ar(1), ar(1), ar(3), out_cap=P)
    for pm in (False, True):
        d_ts, d_val, d_n, d_st, n_fast = _run(dev, ts, vals, n_points, status, ar(1), ar(1), ar(3), 0, 0, 0, pm)
        assert n_fast == S
        assert (d_st == o[3]).all() and (d_n == o[2]).all()
        for s in range(S):
            k = int(o[2][s])
            assert (d_ts[s, :k] == o[0][s, :k]).all() and (d_val[s, :k] == o[1][s, :k]).all()


def test_merge_kernels_on_host_last_failing_replica_wins(dev):
    """series_iterator.go:157-168: every failing replica overwrites the error of the ones before it (see
    tests/test_merge_oracle.py::test_series_last_failing_replica_sets_the_error) -- fast and general kernel."""
    from test_merge_oracle import START, at, build
    a = [(1.0, at(1)), (2.0, at(2)), (3.0, at(3))]
    for strategy in (0, 1):
        for series, want in (([[[[([], 55)]], [[([], 66)]], [[a]]]], 66), ([[[[([], 66)]], [[a]], [[([], 55)]]]], 55),
                             ([[[[a]], [[([], 55)]], [[([], 66)]]]], 66)):
            ts, val, npts, st, slice_off, replica_off, series_off = build(series)
            for pm in (False, True):
                d = _run(dev, np.ascontiguousarray(ts, dtype=np.int64), np.ascontiguousarray(val, dtype=np.float64),
                         np.ascontiguousarray(npts, dtype=np.uint32), np.ascontiguousarray(st, dtype=np.int32),
                         slice_off, replica_off, series_off, START, START + 60 * 10 ** 9, strategy, pm)
                assert d[3].tolist() == [want] and d[2].tolist() == [0], (strategy, want, d[3], d[2])
