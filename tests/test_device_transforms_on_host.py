"""The tile stage's transformation chain, compiled for the host from the .cu source text: `xf_isnan`, `xf_bits`,
`xf_per_second`, `xf_increase` and `xf_window` (m3tsz_encode.cu) with `m3tsz_transform_state` and the
M3TSZ_TRANSFORM_* ids (include/m3tsz_b200.h).  A driver runs a series' non-empty windows through it the way the
kernel's IN = 4 stage does (a discarded NaN writes nothing, the Reset datapoint follows its window unless its
timestamp is 0) and must equal the oracle (tests/xf_oracle.c) bit for bit, state included, on the goldens and on
the random sequences of test_independent_transforms.py, calls split at random.  A CPU regression harness for the
device source; nothing of it ships."""
import ctypes as C

import numpy as np
import pytest

import xf_oracle_lib as X
from host_build import compile, constants, cut, fn, source_text
from test_independent_transforms import _goldens, _oracle_state, _splits, _val, random_pipeline, random_windows

DRIVER = r"""
// the kernel's IN = 4 rows for n non-empty windows of one series: the window's datapoint unless a discarded NaN,
// then the Reset datapoint unless there is none (extra_t == 0)
extern "C" size_t dev_transform_series(const int32_t *ops, size_t n_ops, int discard_nan, int64_t step,
                                       m3tsz_transform_state *st, const int64_t *t, const double *v, size_t n,
                                       int64_t *t_out, double *v_out) {
  uint32_t word = 0;
  for (size_t k = 0; k < n_ops; k++) word |= (uint32_t)ops[k] << (4 * k);
  size_t k = 0;
  for (size_t i = 0; i < n; i++) {
    double x = v[i];
    int64_t extra_t = 0;
    xf_window(word, step, *st, t[i], x, extra_t);
    if (discard_nan && xf_isnan(x)) continue;
    t_out[k] = t[i];
    v_out[k++] = x;
    if (extra_t != 0) {
      t_out[k] = extra_t;
      v_out[k++] = 0.0;
    }
  }
  return k;
}
"""


@pytest.fixture(scope="module")
def dev():
    enc = source_text("m3tsz_encode.cu")
    parts = [constants(enc, r"kXf\w*")]
    for name in ("xf_isnan", "xf_bits", "xf_per_second", "xf_increase", "xf_window"):
        parts.append(cut(enc, fn(name)))
    lib = compile("dev_xf_host", "\n".join(parts), DRIVER)
    vp = C.c_void_p
    lib.dev_transform_series.restype = C.c_size_t
    lib.dev_transform_series.argtypes = [vp, C.c_size_t, C.c_int, C.c_int64, vp, vp, vp, C.c_size_t, vp, vp]
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _dev_series(lib, ops, discard, step, st, t, v):
    ops_a = np.ascontiguousarray(ops, dtype=np.int32)
    t = np.ascontiguousarray(t, dtype=np.int64)
    v = np.ascontiguousarray(v, dtype=np.float64)
    to = np.zeros(max(1, 2 * len(t)), dtype=np.int64)
    vo = np.zeros(max(1, 2 * len(t)), dtype=np.float64)
    n = lib.dev_transform_series(_p(ops_a), len(ops_a), int(discard), int(step), _p(st), _p(t), _p(v), len(t),
                                 _p(to), _p(vo))
    return to[:n], vo[:n]


@pytest.mark.parametrize("case", _goldens(), ids=lambda c: c["name"])
def test_goldens_device_chain(dev, case):
    st = _oracle_state(case)
    for call in case["calls"]:
        t = np.array([w[0] for w in call["windows"]], dtype=np.int64)
        v = np.array([_val(w[1]) for w in call["windows"]], dtype=np.uint64).view(np.float64)
        to, vo = _dev_series(dev, case["ops"], case["discard_nan"], case["step_ns"], st, t, v)
        assert list(zip(to.tolist(), vo.view(np.uint64).tolist())) == [(t, _val(v)) for t, v in call["want"]]


def test_random_device_chain_matches_oracle(dev):
    rng = np.random.default_rng(90210)
    for it in range(3000):
        ops = random_pipeline(rng)
        discard = bool(rng.random() < 0.5)
        step, ts, vs = random_windows(rng, int(rng.integers(0, 25)))
        sd, so = X.new_transform_state(), X.new_transform_state()
        for a, b in _splits(rng, len(ts)):
            t = np.array(ts[a:b], dtype=np.int64)
            v = np.array(vs[a:b], dtype=np.uint64).view(np.float64)
            gt, gv = _dev_series(dev, ops, discard, step, sd, t, v)
            et, ev = X.transform_series(ops, discard, step, so, t, v)
            assert (gt == et).all() and (gv.view(np.uint64) == ev.view(np.uint64)).all(), (it, ops, discard, step)
        assert sd.tobytes() == so.tobytes(), (it, ops)
