"""The element sets' device steps compiled for the host from the .cu source text (tests/host_build.py): the add lane
(`elem_add_lane`: Go truncation, the closed-window and capacity rules, Gauge / Counter Update into the slots) and the
consume lane (`elem_consume_lane`: the windows in start order through tile_value_of and xf_element_window, staged as
rows), with `struct EncodeParams` / `struct ElementParams` of m3tsz_kernels.h.  A driver runs every element's lane
the way the kernels do; results, statuses, staged rows and records must equal the CPU model
(tests/element_set_model.py) bit for bit on random sequences: out-of-order datapoints inside open windows, late ones
into closed windows, NaN / +-Inf, the Counter's int64 wrap, capacity.  A CPU regression harness; nothing of it
ships."""
import ctypes as C

import numpy as np
import pytest

import agg_oracle_lib as A
import elem_oracle_lib as E
from element_set_model import ElementModel
from host_build import compile, constants, cut, fn, source_text

SEC = 1_000_000_000

PRE = r"""
#include <type_traits>
static inline double __ldg(const double *p) { return *p; }
static inline int64_t __ldg(const int64_t *p) { return *p; }
"""

DRIVER = r"""
static ElementParams params(int counter, uint64_t n, uint32_t R, int64_t res, int64_t off, int64_t *start,
                            int64_t *count, void *sum, void *mn, void *mx, void *sq, double *last, int64_t *last_at,
                            int64_t *wm) {
  ElementParams p;
  memset(&p, 0, sizeof(p));
  p.n = n; p.n_slots = R; p.counter = counter; p.resolution = res; p.trunc_off = off;
  p.start = start; p.count = count; p.sum = sum; p.min = mn; p.max = mx; p.sum_sq = sq; p.last = last;
  p.last_at = last_at; p.watermark = wm;
  p.tiles.tile_count = count;
  p.tiles.tile_sum = (const double *)sum; p.tiles.tile_min = (const double *)mn; p.tiles.tile_max = (const double *)mx;
  p.tiles.tile_last = last; p.tiles.tile_sum_sq = sq;
  return p;
}
extern "C" void dev_add(int counter, uint64_t n, uint32_t R, int64_t res, int64_t off, int64_t *start, int64_t *count,
                        void *sum, void *mn, void *mx, void *sq, double *last, int64_t *last_at, int64_t *wm,
                        const int64_t *ts, const double *val, uint64_t P, const uint32_t *n_points, int8_t *result,
                        int32_t *status) {
  ElementParams p = params(counter, n, R, res, off, start, count, sum, mn, mx, sq, last, last_at, wm);
  p.ts = ts; p.val = val; p.points_stride = P; p.n_points = n_points; p.result = result; p.status = status;
  for (uint64_t s = 0; s < n; s++) counter ? elem_add_lane<true>(p, s) : elem_add_lane<false>(p, s);
}
extern "C" void dev_consume(int counter, uint64_t n, uint32_t R, int64_t res, int64_t off, int64_t *start,
                            int64_t *count, void *sum, void *mn, void *mx, void *sq, double *last, int64_t *last_at,
                            int64_t *wm, m3tsz_element_state *elem, int64_t target, uint32_t types, uint32_t k,
                            uint32_t ops, int discard, const m3tsz_encoder_state *out_state, uint64_t slot_words,
                            int64_t *row_ts, double *row_val, uint32_t *row_n, uint64_t rows_stride,
                            int32_t *status) {
  ElementParams p = params(counter, n, R, res, off, start, count, sum, mn, mx, sq, last, last_at, wm);
  p.elem = elem; p.target = target; p.types = types; p.n_types = k; p.ops = ops; p.discard_nan = discard;
  p.out_state = out_state; p.out_slot_words = slot_words; p.row_ts = row_ts; p.row_val = row_val; p.row_n = row_n;
  p.rows_stride = rows_stride; p.status = status;
  p.tiles.metric_type = counter ? M3TSZ_METRIC_COUNTER : M3TSZ_METRIC_GAUGE;
  for (uint64_t s = 0; s < n; s++) {
    XfElem e;
    counter ? elem_consume_lane<true>(p, s, e) : elem_consume_lane<false>(p, s, e);
  }
}
"""


@pytest.fixture(scope="module")
def dev():
    enc, com, ker = source_text("m3tsz_encode.cu"), source_text("m3tsz_common.cuh"), source_text("m3tsz_kernels.h")
    parts = [PRE, constants(enc, r"kXf\w*|ENC_GUARD"), cut(ker, r"struct EncodeParams\b"),
             cut(ker, r"struct ElementParams\b"), cut(enc, r"struct XfElem \{"), cut(com, fn("go_f64_to_i64")),
             cut(com, fn("agg_stdev"))]
    for name in ("xf_isnan", "xf_bits", "xf_per_second", "xf_increase", "xf_window", "xf_element_window",
                 "tile_value_of", "elem_window_start", "elem_ends_by"):
        parts.append(cut(enc, fn(name)))
    parts.append(cut(enc, r"struct ElemAcc\b"))
    for name in ("elem_init", "elem_load", "elem_store", "elem_update", "elem_add_lane", "elem_consume_lane"):
        parts.append(cut(enc, fn(name)))
    body = "\n".join(parts)
    body = body.replace('asm volatile("mov.b64 %0, %1;" : "=l"(oi) : "l"(o));', "oi = o;")
    lib = compile("dev_elem_set_host", body, DRIVER)
    vp, i64, u64, u32 = C.c_void_p, C.c_int64, C.c_uint64, C.c_uint32
    lib.dev_add.restype = None
    lib.dev_add.argtypes = [C.c_int, u64, u32, i64, i64] + [vp] * 9 + [vp, vp, u64, vp, vp, vp]
    lib.dev_consume.restype = None
    lib.dev_consume.argtypes = [C.c_int, u64, u32, i64, i64] + [vp] * 9 + [vp, i64, u32, u32, u32, C.c_int, vp, u64,
                                                                           vp, vp, vp, u64, vp]
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class DevSet:
    """N elements in host arrays laid out as the device's"""

    def __init__(self, lib, N, R, metric, types, res, ops, discard):
        self.lib, self.N, self.R, self.res = lib, N, R, res
        self.counter = metric == A.METRIC_COUNTER
        self.types, self.ops, self.discard = types, ops, discard
        t = np.int64 if self.counter else np.float64
        self.w = {f: np.zeros((R, N), dtype=d) for f, d in (
            ("start", np.int64), ("count", np.int64), ("sum", t), ("min", t), ("max", t), ("sum_sq", t),
            ("last", np.float64), ("last_at", np.int64))}
        self.wm = np.full(N, -(1 << 63), dtype=np.int64)
        self.elem = np.zeros(N, dtype=E.ELEM_STATE_DTYPE)
        self.off = (62135596800 * SEC) % res

    def _arrays(self):
        w = self.w
        return [_p(w[f]) for f in ("start", "count", "sum", "min", "max", "sum_sq", "last", "last_at")] + [_p(self.wm)]

    def add(self, cols):
        P = max([len(c) for c in cols] + [1])
        ts = np.zeros((P, self.N), dtype=np.int64)
        vb = np.zeros((P, self.N), dtype=np.uint64)
        for s, c in enumerate(cols):
            for i, (t, v) in enumerate(c):
                ts[i, s], vb[i, s] = t, v
        n = np.array([len(c) for c in cols], dtype=np.uint32)
        res = np.zeros((P, self.N), dtype=np.int8)
        st = np.zeros(self.N, dtype=np.int32)
        self.lib.dev_add(int(self.counter), self.N, self.R, self.res, self.off, *self._arrays(), _p(ts),
                         _p(vb.view(np.float64)), P, _p(n), _p(res), _p(st))
        return [res[: len(c), s].tolist() for s, c in enumerate(cols)], st.tolist()

    def consume(self, target, slot_words=1 << 20):
        k = len(self.types)
        reset = 5 in self.ops
        rows = self.R * (2 if reset else 1)
        rt = np.zeros((rows, k * self.N), dtype=np.int64)
        rv = np.zeros((rows, k * self.N), dtype=np.float64)
        rn = np.zeros(k * self.N, dtype=np.uint32)
        st = np.zeros(self.N, dtype=np.int32)
        out_state = np.zeros((k * self.N, 128), dtype=np.uint8)
        types = sum(t << (4 * j) for j, t in enumerate(self.types))
        ops = sum(o << (4 * j) for j, o in enumerate(self.ops))
        self.lib.dev_consume(int(self.counter), self.N, self.R, self.res, self.off, *self._arrays(), _p(self.elem),
                             int(target), types, k, ops, int(self.discard and len(self.ops) > 0), _p(out_state),
                             slot_words, _p(rt), _p(rv), _p(rn), rows, _p(st))
        out = [[(rt[: rn[j * self.N + s], j * self.N + s], rv[: rn[j * self.N + s], j * self.N + s])
                for j in range(k)] for s in range(self.N)]
        return out, st.tolist()


def _value(rng, counter):
    if counter:
        return float(rng.choice([rng.integers(-1000, 1000), 9.0e18, -9.1e18, 2.0 ** 63, np.nan, 3.7e9]))
    return float(rng.choice([rng.normal() * 100, np.nan, np.inf, -np.inf, 0.0, -0.0]))


def _bits(v):
    return int(np.array([v], dtype=np.float64).view(np.uint64)[0])


@pytest.mark.parametrize("metric", [A.METRIC_GAUGE, A.METRIC_COUNTER])
def test_random_sequences_equal_the_model(dev, metric):
    rng = np.random.default_rng(31 + metric)
    counter = metric == A.METRIC_COUNTER
    menu = [2, 3, 4, 6, 7, 8, 9] + ([] if counter else [1])
    for it in range(40):
        N, R = 16, int(rng.integers(1, 5))
        res = int(rng.choice([10, 60, 7])) * SEC
        types = sorted(rng.choice(menu, int(rng.integers(1, 4)), replace=False).tolist())
        ops = [[], [3], [1, 2], [4], [5], [4, 3, 5]][it % 6]
        discard = bool(it % 2)
        d = DevSet(dev, N, R, metric, types, res, ops, discard)
        models = [ElementModel(metric, types, res, ops, discard, open_windows=R) for _ in range(N)]
        clock = int(rng.integers(-5, 5)) * res
        for step in range(8):
            cols = []
            for s in range(N):
                n = int(rng.integers(0, 5))
                cols.append([(clock + int(rng.integers(-3 * res, res)) // SEC * SEC
                              + (int(rng.integers(0, SEC)) if rng.random() < 0.1 else 0),
                              _bits(_value(rng, counter))) for _ in range(n)])
            got_r, got_s = d.add(cols)
            for s, m in enumerate(models):
                want_r, want_s = m.add(cols[s])
                assert (got_r[s], got_s[s]) == (want_r, want_s), (it, step, s)
            clock += int(rng.integers(0, 2)) * res
            if rng.random() < 0.6:
                target = clock - int(rng.integers(0, 2)) * res
                out, st = d.consume(target)
                assert st == [0] * N
                for s, m in enumerate(models):
                    want = m.consume(target)
                    for j in range(len(types)):
                        assert np.array_equal(out[s][j][0], want[j][0]), (it, step, s, j)
                        assert np.array_equal(out[s][j][1].view(np.uint64), want[j][1].view(np.uint64)), \
                            (it, step, s, j)
                    assert d.elem[s].tobytes() == m.state.tobytes()
                    assert d.wm[s] == m.watermark


def test_output_room_refuses_the_whole_element(dev):
    d = DevSet(dev, 2, 4, A.METRIC_GAUGE, [1, 2], 60 * SEC, [5], False)
    d.add([[(5 * SEC, _bits(1.0)), (65 * SEC, _bits(2.0))], []])
    before = {f: a.copy() for f, a in d.w.items()}
    out, st = d.consume(120 * SEC, slot_words=(64 + 3 * 163) // 32 + 14 - 1)  # a word short of 4 datapoints
    assert st == [100, 0] and all(len(t) == 0 for t, _ in out[0])
    assert all(np.array_equal(before[f], d.w[f]) for f in before) and d.wm[0] == -(1 << 63)
    out, st = d.consume(120 * SEC, slot_words=(64 + 3 * 163) // 32 + 14)
    assert st == [0, 0] and [len(t) for t, _ in out[0]] == [4, 4]
