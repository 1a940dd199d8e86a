"""The Timer element sets' device steps compiled for the host from the .cu source text (tests/host_build.py): the add
lane (`elem_timer_add_lane`: the batch rule, windows, the capacity rule, Timer.AddBatch into the slot's CM stream,
`struct CmStream`) and the consume lane (`elem_timer_consume_lane`: Flush, calcQuantiles, ValueOf of each type through
xf_element_window, staged as rows).  A driver runs every element's lane the way the kernels do; results, statuses,
staged rows, records and watermarks must equal the CPU model (tests/element_timer_model.py) bit for bit on random
sequences: both capacity stops followed by grow and resend, closed windows, invalid batch continuations, windows that
cross insert_and_compress_every inside a batch, +-0 and NaN samples.  A CPU regression harness; nothing of it ships."""
import ctypes as C

import numpy as np
import pytest

import elem_oracle_lib as E
from element_timer_model import TimerElementModel
from host_build import compile, constants, cut, fn, source_text
from indep_timer import pooled_quantiles

SEC = 1_000_000_000
RES = 60 * SEC

PRE = r"""
#include <type_traits>
#include <climits>
"""

DRIVER = r"""
static ElementTimerParams params(uint64_t n, uint32_t R, int64_t res, int64_t off, int64_t *start, int64_t *count,
                                 double *sum, double *sq, int64_t *wm, m3tsz_timer_stream_header *hdr, double *value,
                                 int64_t *nr, int64_t *dl, int32_t *prv, int32_t *nxt, double *ha, double *hb,
                                 uint32_t cap, int32_t every, double eps, const int32_t *types, uint32_t k,
                                 const double *q, uint32_t nq) {
  ElementTimerParams p;
  memset(&p, 0, sizeof(p));
  p.e.n = n; p.e.n_slots = R; p.e.resolution = res; p.e.trunc_off = off;
  p.e.start = start; p.e.count = count; p.e.sum = sum; p.e.sum_sq = sq; p.e.watermark = wm;
  p.hdr = hdr; p.value = value; p.num_ranks = nr; p.delta = dl; p.prev = prv; p.next = nxt; p.heap_a = ha;
  p.heap_b = hb; p.cap = cap; p.every = every; p.eps = eps; p.n_types = k; p.n_q = nq;
  for (uint32_t j = 0; j < k; j++) p.type[j] = types[j];
  for (uint32_t j = 0; j < nq; j++) p.q[j] = q[j];
  return p;
}
#define ARGS uint64_t n, uint32_t R, int64_t res, int64_t off, int64_t *start, int64_t *count, double *sum, \
  double *sq, int64_t *wm, m3tsz_timer_stream_header *hdr, double *value, int64_t *nr, int64_t *dl, int32_t *prv, \
  int32_t *nxt, double *ha, double *hb, uint32_t cap, int32_t every, double eps, const int32_t *types, uint32_t k, \
  const double *q, uint32_t nq
#define PASS n, R, res, off, start, count, sum, sq, wm, hdr, value, nr, dl, prv, nxt, ha, hb, cap, every, eps, types, \
  k, q, nq
extern "C" void dev_add(ARGS, const int64_t *ts, const double *val, uint64_t P, const uint32_t *n_points,
                        const int8_t *batch, int8_t *result, int32_t *status) {
  ElementTimerParams p = params(PASS);
  p.e.ts = ts; p.e.val = val; p.e.points_stride = P; p.e.n_points = n_points; p.e.result = result;
  p.e.status = status; p.batch = batch;
  for (uint64_t s = 0; s < n; s++) elem_timer_add_lane(p, s);
}
extern "C" void dev_consume(ARGS, m3tsz_element_state *elem, int64_t target, uint32_t ops, int discard,
                            const m3tsz_encoder_state *out_state, uint64_t slot_words, int64_t *row_ts,
                            double *row_val, uint32_t *row_n, uint64_t rows_stride, int32_t *status) {
  ElementTimerParams p = params(PASS);
  p.e.elem = elem; p.e.target = target; p.e.ops = ops; p.e.discard_nan = discard;
  p.e.out_state = out_state; p.e.out_slot_words = slot_words; p.e.row_ts = row_ts; p.e.row_val = row_val;
  p.e.row_n = row_n; p.e.rows_stride = rows_stride; p.e.status = status;
  for (uint64_t s = 0; s < n; s++) {
    XfElem e;
    elem_timer_consume_lane(p, s, e);
  }
}
"""


@pytest.fixture(scope="module")
def dev():
    enc, com, ker = source_text("m3tsz_encode.cu"), source_text("m3tsz_common.cuh"), source_text("m3tsz_kernels.h")
    parts = [PRE, constants(enc, r"kXf\w*|ENC_GUARD"), cut(ker, r"struct EncodeParams\b"),
             cut(ker, r"struct ElementParams\b"), "#define M3TSZ_MAX_TIMER_TYPES 23\n#define M3TSZ_MAX_TIMER_QUANTILES 15",
             cut(ker, r"struct ElementTimerParams\b"), cut(enc, r"struct XfElem \{"), cut(com, fn("go_f64_to_i64")),
             cut(com, fn("agg_stdev"))]
    for name in ("xf_isnan", "xf_bits", "xf_per_second", "xf_increase", "xf_window", "xf_element_window",
                 "elem_window_start", "elem_ends_by"):
        parts.append(cut(enc, fn(name)))
    parts.append(cut(enc, r"struct CmStream\b"))
    for name in ("timer_stream", "amd64_op", "timer_stdev", "timer_type_quantile", "timer_value_of", "elem_timer_add_lane",
                 "elem_timer_consume_lane"):
        parts.append(cut(enc, fn(name)))
    lib = compile("dev_elem_timer_host", "\n".join(parts), DRIVER)
    vp, i64, u64, u32, i32 = C.c_void_p, C.c_int64, C.c_uint64, C.c_uint32, C.c_int32
    head = [u64, u32, i64, i64] + [vp] * 5 + [vp] * 8 + [u32, i32, C.c_double, vp, u32, vp, u32]
    lib.dev_add.restype = None
    lib.dev_add.argtypes = head + [vp, vp, u64, vp, vp, vp, vp]
    lib.dev_consume.restype = None
    lib.dev_consume.argtypes = head + [vp, i64, u32, C.c_int, vp, u64, vp, vp, vp, u64, vp]
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class DevTimerSet:
    """N Timer elements in host arrays laid out as the device's"""

    def __init__(self, lib, N, R, types, ops, discard, cap, every, eps):
        self.lib, self.N, self.types, self.ops, self.discard = lib, N, list(types), list(ops), discard
        self.every, self.eps = every, eps
        self.w = {f: np.zeros((R, N), dtype=d) for f, d in (("start", np.int64), ("count", np.int64),
                                                            ("sum", np.float64), ("sum_sq", np.float64))}
        self.wm = np.full(N, -(1 << 63), dtype=np.int64)
        self.elem = np.zeros(N, dtype=E.ELEM_STATE_DTYPE)
        self.hdr = np.zeros((R, N, 64), dtype=np.uint8)
        self.arr = {f: np.zeros((R, cap, N), dtype=d) for f, d in (
            ("value", np.float64), ("nr", np.int64), ("dl", np.int64), ("prv", np.int32), ("nxt", np.int32),
            ("ha", np.float64), ("hb", np.float64))}
        self.q = np.array(pooled_quantiles(types) or [0.0], dtype=np.float64)
        self.nq = len(pooled_quantiles(types))
        self.ty = np.array(types, dtype=np.int32)
        self.off = (62135596800 * SEC) % RES

    @property
    def R(self):
        return self.w["start"].shape[0]

    @property
    def cap(self):
        return self.arr["value"].shape[1]

    def grow(self, R=None, cap=None):
        R, cap = R or self.R, cap or self.cap
        for f, a in self.w.items():
            b = np.zeros((R, self.N), dtype=a.dtype)
            b[: a.shape[0]] = a
            self.w[f] = b
        h = np.zeros((R, self.N, 64), dtype=np.uint8)
        h[: self.hdr.shape[0]] = self.hdr
        self.hdr = h
        for f, a in self.arr.items():
            b = np.zeros((R, cap, self.N), dtype=a.dtype)
            b[: a.shape[0], : a.shape[1]] = a
            self.arr[f] = b

    def _head(self):
        w, a = self.w, self.arr
        return [self.N, self.R, RES, self.off, _p(w["start"]), _p(w["count"]), _p(w["sum"]), _p(w["sum_sq"]),
                _p(self.wm), _p(self.hdr)] + [_p(a[f]) for f in ("value", "nr", "dl", "prv", "nxt", "ha", "hb")] + [
                self.cap, self.every, self.eps, _p(self.ty), len(self.types), _p(self.q), self.nq]

    def add(self, cols):
        """cols: per element [(t, v, continues)] -> (results, statuses)"""
        P = max([len(c) for c in cols] + [1])
        ts = np.zeros((P, self.N), dtype=np.int64)
        vs = np.zeros((P, self.N), dtype=np.float64)
        bt = np.zeros((P, self.N), dtype=np.int8)
        for s, c in enumerate(cols):
            for i, (t, v, b) in enumerate(c):
                ts[i, s], vs[i, s], bt[i, s] = t, v, b
        n = np.array([len(c) for c in cols], dtype=np.uint32)
        res = np.zeros((P, self.N), dtype=np.int8)
        st = np.zeros(self.N, dtype=np.int32)
        self.lib.dev_add(*self._head(), _p(ts), _p(vs), P, _p(n), _p(bt), _p(res), _p(st))
        return [res[: len(c), s].tolist() for s, c in enumerate(cols)], st.tolist()

    def consume(self, target):
        k = len(self.types)
        rows = self.R * (2 if 5 in self.ops else 1)
        rt = np.zeros((rows, k * self.N), dtype=np.int64)
        rv = np.zeros((rows, k * self.N), dtype=np.float64)
        rn = np.zeros(k * self.N, dtype=np.uint32)
        st = np.zeros(self.N, dtype=np.int32)
        out_state = np.zeros((k * self.N, 128), dtype=np.uint8)
        ops = sum(o << (4 * j) for j, o in enumerate(self.ops))
        self.lib.dev_consume(*self._head(), _p(self.elem), int(target), ops, int(self.discard and len(self.ops) > 0),
                             _p(out_state), 1 << 20, _p(rt), _p(rv), _p(rn), rows, _p(st))
        out = [[(rt[: rn[j * self.N + s], j * self.N + s], rv[: rn[j * self.N + s], j * self.N + s])
                for j in range(k)] for s in range(self.N)]
        return out, st.tolist()


TYPES = [[2, 3, 4, 5, 6, 7, 8, 9, 14, 19, 20], [5, 10, 18], [14, 20, 23, 24], [3, 6], [2, 3, 4, 5, 6, 7, 8, 9] +
         list(range(10, 25)), [3, 14, 20]]
OPS = [[], [], [], [4, 3, 5], [], [3]]


def _value(rng, pool):
    r = rng.random()
    if r < 0.05:
        return float("nan")
    if r < 0.15:
        return -0.0 if r < 0.1 else 0.0
    if r < 0.4 and pool:
        return pool[int(rng.integers(0, len(pool)))]
    return float(np.round(rng.normal() * 100, 1))


def _rows(rng, clock, pool):
    rows = []
    for _ in range(int(rng.integers(0, 4))):
        t = clock + int(rng.integers(-2 * RES, RES)) // SEC * SEC
        n = int(rng.integers(1, 4)) if rng.random() < 0.7 else int(rng.integers(4, 40))
        for i in range(n):
            v = _value(rng, pool)
            pool.append(v)
            rows.append((t, v, 1 if i else 0))
    if rows and rng.random() < 0.03:  # a broken continuation
        i = int(rng.integers(0, len(rows)))
        rows[i] = (rows[i][0] + (SEC if rows[i][2] else 0), rows[i][1], 1)
    return rows


def _check(out, want):
    for j in range(len(want)):
        assert np.array_equal(out[j][0], want[j][0])
        assert np.array_equal(out[j][1].view(np.uint64), np.asarray(want[j][1], dtype=np.float64).view(np.uint64))


@pytest.mark.parametrize("variant", range(len(TYPES)))
def test_random_sequences_equal_the_model(dev, variant):
    rng = np.random.default_rng(77 + variant)
    types, ops = TYPES[variant], OPS[variant]
    for it in range(12):
        N, R, cap = 12, int(rng.integers(1, 4)), int(rng.choice([4, 16, 64]))
        every = int(rng.choice([1, 2, 3, 7, 64]))
        eps = float(rng.choice([1e-3, 0.05]))
        d = DevTimerSet(dev, N, R, types, ops, bool(it % 2), cap, every, eps)
        models = [TimerElementModel(types, RES, ops, bool(it % 2), R, cap, eps, every) for _ in range(N)]
        pools = [[] for _ in range(N)]
        clock = 10 * RES
        for step in range(8):
            cols = [_rows(rng, clock, pools[s]) for s in range(N)]
            got_r, got_s = d.add(cols)
            for s, m in enumerate(models):
                want_r, want_s = m.add([(t, v) for t, v, _ in cols[s]], [b for _, _, b in cols[s]])
                assert (got_r[s], got_s[s]) == (want_r, want_s), (it, step, s)
            if 100 in got_s:  # grow both limits and resend exactly the refused rows
                d.grow(R=d.R + 1, cap=d.cap * 2)
                again = [[r for i, r in enumerate(c) if got_r[s][i] == 100] for s, c in enumerate(cols)]
                for m in models:
                    m.R, m.cap = d.R, d.cap
                got_r, got_s = d.add(again)
                for s, m in enumerate(models):
                    assert (got_r[s], got_s[s]) == m.add([(t, v) for t, v, _ in again[s]],
                                                         [b for _, _, b in again[s]]), (it, step, s)
            clock += int(rng.integers(0, 2)) * RES
            if rng.random() < 0.6:
                target = clock - int(rng.integers(0, 2)) * RES
                out, st = d.consume(target)
                assert st == [0] * N
                for s, m in enumerate(models):
                    _check(out[s], m.consume(target))
                    assert d.elem[s].tobytes() == m.state.tobytes()
                    assert d.wm[s] == m.watermark


def test_insert_and_compress_inside_one_batch(dev):
    """a 3000-value batch with every = 64 runs the periodic insert + compress mid-batch, with the stale insertion
    point the reference keeps"""
    rng = np.random.default_rng(5)
    types = [2, 3, 5, 10, 18, 20]
    d = DevTimerSet(dev, 2, 1, types, [], False, 4096, 64, 1e-3)
    models = [TimerElementModel(types, RES, [], False, 1, 4096, 1e-3, 64) for _ in range(2)]
    cols = [[(RES + SEC, float(v), 1 if i else 0) for i, v in enumerate(rng.normal(size=3000).round(2))]
            for _ in range(2)]
    got_r, got_s = d.add(cols)
    assert got_s == [0, 0]
    for s, m in enumerate(models):
        assert m.add([(t, v) for t, v, _ in cols[s]], [b for _, _, b in cols[s]])[1] == 0
    out, st = d.consume(2 * RES)
    for s, m in enumerate(models):
        _check(out[s], m.consume(2 * RES))
