"""The multi-type tile stage's element step, compiled for the host from the .cu source text: `xf_isnan`, `xf_bits`,
`xf_per_second`, `xf_increase`, `xf_window`, `struct XfElem` and `xf_element_window` (m3tsz_encode.cu) with the
state records and ids of include/m3tsz_b200.h.  A driver runs each type's lane the way the kernel's IN = 5 stage does
(its own record loaded from the series' m3tsz_element_state; every type when the list has an Add op, else its own;
a discarded NaN writes nothing; the Reset datapoint follows unless its timestamp is 0), then assembles the saved
record from the lanes' parts as the epilogue does.  Datapoints and record must equal the oracle (tests/elem_oracle.c)
bit for bit, on the goldens and on random type sets, op lists and call splits.  A CPU regression harness for the
device source; nothing of it ships."""
import ctypes as C

import numpy as np
import pytest

import elem_oracle_lib as E
from host_build import compile, constants, cut, fn, source_text
from test_independent_element import _element_windows, _goldens, random_element_pipeline
from test_independent_transforms import _splits, _val

DRIVER = r"""
// lane j of the IN = 5 stage for n non-empty windows (v: [n][k]) of one series, from record `rec`; its datapoints go
// to t_out / v_out (2n entries), and its part of the new record into `out` (type 0: the element's fields and the
// inputs of types >= k; type j: prev_v_more[j - 1])
static size_t lane(const int32_t *ops, size_t n_ops, int discard_nan, int64_t step, uint32_t k, uint32_t j,
                   const m3tsz_element_state &rec, const int64_t *t, const double *v, size_t n, int64_t *t_out,
                   double *v_out, m3tsz_element_state &out) {
  uint32_t word = 0;
  bool all = false;
  for (size_t i = 0; i < n_ops; i++) {
    word |= (uint32_t)ops[i] << (4 * i);
    all |= ops[i] == M3TSZ_TRANSFORM_ADD;
  }
  XfElem e;
  e.w = rec.head;
  e.pv[0] = rec.head.prev_v;
  for (int i = 1; i < M3TSZ_MAX_ELEMENT_TYPES; i++) e.pv[i] = rec.prev_v_more[i - 1];
  size_t m = 0;
  for (size_t w = 0; w < n; w++) {
    double x = 0.0;
    int64_t extra_t = 0;
    xf_element_window(word, step, e, all ? 0u : j, all ? k : j + 1, t[w],
                      [&](uint32_t i) { return v[w * k + i]; },
                      [&](uint32_t i, double r, int64_t et) {
                        if (i == j) {
                          x = r;
                          extra_t = et;
                        }
                      });
    if (n_ops && discard_nan && xf_isnan(x)) continue;
    t_out[m] = t[w];
    v_out[m++] = x;
    if (extra_t != 0) {
      t_out[m] = extra_t;
      v_out[m++] = 0.0;
    }
  }
  if (j == 0) {
    out.head = e.w;
    out.head.prev_v = e.pv[0];
    for (uint32_t i = k; i < M3TSZ_MAX_ELEMENT_TYPES; i++) out.prev_v_more[i - 1] = e.pv[i];
    out.reserved = rec.reserved;
  } else {
    out.prev_v_more[j - 1] = e.pv[j];
  }
  return m;
}

extern "C" void dev_element_series(const int32_t *ops, size_t n_ops, int discard_nan, int64_t step, size_t k,
                                   m3tsz_element_state *st, const int64_t *t, const double *v, size_t n,
                                   int64_t *t_out, double *v_out, size_t *n_out) {
  m3tsz_element_state next;
  memset(&next, 0xA5, sizeof(next));  // every byte must come from some lane
  for (uint32_t j = 0; j < k; j++)
    n_out[j] = lane(ops, n_ops, discard_nan, step, (uint32_t)k, j, *st, t, v, n, t_out + j * 2 * n,
                    v_out + j * 2 * n, next);
  *st = next;
}
"""


@pytest.fixture(scope="module")
def dev():
    enc = source_text("m3tsz_encode.cu")
    parts = [constants(enc, r"kXf\w*"), cut(enc, r"struct XfElem \{")]
    for name in ("xf_isnan", "xf_bits", "xf_per_second", "xf_increase", "xf_window", "xf_element_window"):
        parts.append(cut(enc, fn(name)))
    lib = compile("dev_elem_host", "\n".join(parts), DRIVER)
    vp = C.c_void_p
    lib.dev_element_series.restype = None
    lib.dev_element_series.argtypes = [vp, C.c_size_t, C.c_int, C.c_int64, C.c_size_t, vp, vp, vp, C.c_size_t, vp,
                                       vp, vp]
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _dev_series(lib, ops, discard, step, k, st, t, v):
    ops_a = np.ascontiguousarray(ops if len(ops) else [0], dtype=np.int32)
    t = np.ascontiguousarray(t, dtype=np.int64)
    v = np.ascontiguousarray(np.asarray(v, dtype=np.float64).reshape(len(t), k))
    n = len(t)
    to = np.zeros(max(1, k * 2 * n), dtype=np.int64)
    vo = np.zeros(max(1, k * 2 * n), dtype=np.float64)
    cnt = np.zeros(k, dtype=np.uint64)
    lib.dev_element_series(_p(ops_a), len(ops), int(discard), int(step), k, _p(st), _p(t), _p(v), n, _p(to), _p(vo),
                           _p(cnt))
    return [(to[j * 2 * n: j * 2 * n + int(cnt[j])], vo[j * 2 * n: j * 2 * n + int(cnt[j])]) for j in range(k)]


@pytest.mark.parametrize("case", _goldens(), ids=lambda c: c["name"])
def test_goldens_device_element(dev, case):
    k = len(case["agg_types"])
    st = E.new_element_state()
    for call in case["calls"]:
        t = np.array([w[0] for w in call["windows"]], dtype=np.int64)
        v = np.array([[_val(x) for x in w[1]] for w in call["windows"]], dtype=np.uint64).reshape(len(t), k)
        res = _dev_series(dev, case["ops"], case["discard_nan"], case["step_ns"], k, st, t, v.view(np.float64))
        for j in range(k):
            got = list(zip(res[j][0].tolist(), res[j][1].view(np.uint64).tolist()))
            assert got == [(a, _val(b)) for a, b in call["want"][j]]


def test_random_device_element_matches_oracle(dev):
    rng = np.random.default_rng(4242)
    for it in range(2000):
        k = int(rng.integers(1, 9))
        ops = random_element_pipeline(rng) if rng.random() < 0.9 else []
        discard = bool(rng.random() < 0.5)
        step, ts, vs = _element_windows(rng, int(rng.integers(0, 20)), k)
        sd, so = E.new_element_state(), E.new_element_state()
        for a, b in _splits(rng, len(ts)):
            t = np.array(ts[a:b], dtype=np.int64)
            v = np.array(vs[a:b], dtype=np.uint64).reshape(b - a, k).view(np.float64)
            got = _dev_series(dev, ops, discard, step, k, sd, t, v)
            # (the oracle discards with any list; the device applies discard_nan only with ops, as tiles_ex)
            exp = E.element_series(ops, discard and len(ops) > 0, step, k, so, t, v)
            for j in range(k):
                assert (got[j][0] == exp[j][0]).all() and \
                    (got[j][1].view(np.uint64) == exp[j][1].view(np.uint64)).all(), (it, ops, discard, j)
        assert sd.tobytes() == so.tobytes(), (it, ops, k)
