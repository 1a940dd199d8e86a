"""The annotated element-set device steps compiled for the host from the .cu source text (tests/host_build.py): the add
lane `elem_add_lane<CTR, true>` (each window's last non-empty annotation kept in registers and written to its slot,
the capacity stop), and the consume lane `elem_consume_lane<CTR, true>` (each staged datapoint's
annotation entry, the room check counting the annotations).  A driver runs every element's lane the way the kernels
do; on random sequences -- annotated and bare datapoints, NaN values, late datapoints to older open windows, closed
windows, R and annotation-capacity stops followed by a resend -- results, statuses, staged rows and the annotation of
every staged datapoint must equal the CPU model (tests/element_set_ann_model.py), and for every staged datapoint the
consume's room bound must imply the encoder-set append's own check.  A CPU regression harness; nothing of it ships."""
import ctypes as C

import numpy as np
import pytest

import agg_oracle_lib as A
import elem_oracle_lib as E
from element_set_ann_model import AnnotatedElementModel, annotation_words, sparse_annotations
from element_set_model import ERR_CAPACITY
from host_build import compile, constants, cut, fn, source_text

SEC = 1_000_000_000
ENC_GUARD = 10  # (checked against the source below)

PRE = r"""
#include <type_traits>
static inline double __ldg(const double *p) { return *p; }
static inline int64_t __ldg(const int64_t *p) { return *p; }
"""

DRIVER = r"""
static ElementParams params(int counter, uint64_t n, uint32_t R, int64_t res, int64_t off, int64_t *start,
                            int64_t *count, void *sum, void *mn, void *mx, void *sq, double *last, int64_t *last_at,
                            int64_t *wm, uint32_t *ann_len, uint8_t *ann_slot, uint64_t cap) {
  ElementParams p;
  memset(&p, 0, sizeof(p));
  p.n = n; p.n_slots = R; p.counter = counter; p.resolution = res; p.trunc_off = off;
  p.start = start; p.count = count; p.sum = sum; p.min = mn; p.max = mx; p.sum_sq = sq; p.last = last;
  p.last_at = last_at; p.watermark = wm;
  p.tiles.tile_count = count;
  p.tiles.tile_sum = (const double *)sum; p.tiles.tile_min = (const double *)mn; p.tiles.tile_max = (const double *)mx;
  p.tiles.tile_last = last; p.tiles.tile_sum_sq = sq;
  p.ann_len = ann_len; p.ann_slot = ann_slot; p.ann_cap = cap;
  return p;
}
extern "C" void dev_add(int counter, uint64_t n, uint32_t R, int64_t res, int64_t off, int64_t *start, int64_t *count,
                        void *sum, void *mn, void *mx, void *sq, double *last, int64_t *last_at, int64_t *wm,
                        uint32_t *ann_len, uint8_t *ann_slot, uint64_t cap, const int64_t *ts, const double *val,
                        uint64_t P, const uint32_t *n_points, const uint64_t *a_off,
                        const m3tsz_annotation_entry *a_ent, const uint8_t *a_bytes, int8_t *result,
                        int32_t *status) {
  ElementParams p = params(counter, n, R, res, off, start, count, sum, mn, mx, sq, last, last_at, wm, ann_len,
                           ann_slot, cap);
  p.ts = ts; p.val = val; p.points_stride = P; p.n_points = n_points; p.result = result; p.status = status;
  p.ann_series_off = a_off; p.ann_entries = a_ent; p.ann_bytes = a_bytes;
  for (uint64_t s = 0; s < n; s++) counter ? elem_add_lane<true, true>(p, s) : elem_add_lane<false, true>(p, s);
}
extern "C" void dev_consume(int counter, uint64_t n, uint32_t R, int64_t res, int64_t off, int64_t *start,
                            int64_t *count, void *sum, void *mn, void *mx, void *sq, double *last, int64_t *last_at,
                            int64_t *wm, uint32_t *ann_len, uint8_t *ann_slot, uint64_t cap,
                            m3tsz_element_state *elem, int64_t target, uint32_t types, uint32_t k,
                            uint32_t ops, int discard, const m3tsz_encoder_state *out_state, uint64_t slot_words,
                            int64_t *row_ts, double *row_val, uint32_t *row_n, uint64_t rows_stride,
                            uint64_t *row_ann_off, m3tsz_annotation_entry *row_ann, int32_t *status) {
  ElementParams p = params(counter, n, R, res, off, start, count, sum, mn, mx, sq, last, last_at, wm, ann_len,
                           ann_slot, cap);
  p.elem = elem; p.target = target; p.types = types; p.n_types = k; p.ops = ops; p.discard_nan = discard;
  p.out_state = out_state; p.out_slot_words = slot_words; p.row_ts = row_ts; p.row_val = row_val; p.row_n = row_n;
  p.rows_stride = rows_stride; p.row_ann_off = row_ann_off; p.row_ann = row_ann; p.status = status;
  p.tiles.metric_type = counter ? M3TSZ_METRIC_COUNTER : M3TSZ_METRIC_GAUGE;
  for (uint64_t s = 0; s < n; s++) {
    XfElem e;
    counter ? elem_consume_lane<true, true>(p, s, e) : elem_consume_lane<false, true>(p, s, e);
  }
}
"""

ENTRY = np.dtype([("dp_index", "<u4"), ("length", "<u4"), ("byte_offset", "<u8")])


@pytest.fixture(scope="module")
def dev():
    enc, com, ker = source_text("m3tsz_encode.cu"), source_text("m3tsz_common.cuh"), source_text("m3tsz_kernels.h")
    assert "constexpr int ENC_GUARD = %d;" % ENC_GUARD in enc
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
    lib = compile("dev_elem_ann_host", body, DRIVER)
    vp, i64, u64, u32 = C.c_void_p, C.c_int64, C.c_uint64, C.c_uint32
    lib.dev_add.restype = None
    lib.dev_add.argtypes = [C.c_int, u64, u32, i64, i64] + [vp] * 9 + [vp, vp, u64] + [vp, vp, u64, vp, vp, vp, vp,
                                                                                        vp, vp]
    lib.dev_consume.restype = None
    lib.dev_consume.argtypes = [C.c_int, u64, u32, i64, i64] + [vp] * 9 + [vp, vp, u64] + [
        vp, i64, u32, u32, u32, C.c_int, vp, u64, vp, vp, vp, u64, vp, vp, vp]
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class DevSet:
    """N annotated elements in host arrays laid out as the device's"""

    def __init__(self, lib, N, R, metric, types, res, ops, discard, cap):
        self.lib, self.N, self.R, self.res, self.cap = lib, N, R, res, cap
        self.counter = metric == A.METRIC_COUNTER
        self.types, self.ops, self.discard = types, ops, discard
        t = np.int64 if self.counter else np.float64
        self.w = {f: np.zeros((R, N), dtype=d) for f, d in (
            ("start", np.int64), ("count", np.int64), ("sum", t), ("min", t), ("max", t), ("sum_sq", t),
            ("last", np.float64), ("last_at", np.int64))}
        self.wm = np.full(N, -(1 << 63), dtype=np.int64)
        self.elem = np.zeros(N, dtype=E.ELEM_STATE_DTYPE)
        self.off = (62135596800 * SEC) % res
        # lengths start as garbage: the add writes a slot's length when it opens a window there
        self.ann_len = np.full((R, N), 0xffffffff, dtype=np.uint32)
        self.ann_slot = np.zeros((R, N, cap), dtype=np.uint8)

    def grow(self, R=None, cap=None):
        if R is not None and R > self.R:
            for f, a in self.w.items():
                b = np.zeros((R, self.N), dtype=a.dtype)
                b[: self.R] = a
                self.w[f] = b
            ln = np.zeros((R, self.N), dtype=np.uint32)
            ln[: self.R] = self.ann_len
            sl = np.zeros((R, self.N, self.cap), dtype=np.uint8)
            sl[: self.R] = self.ann_slot
            self.ann_len, self.ann_slot, self.R = ln, sl, R
        if cap is not None and cap > self.cap:
            sl = np.zeros((self.R, self.N, cap), dtype=np.uint8)
            sl[:, :, : self.cap] = self.ann_slot
            self.ann_slot, self.cap = sl, cap

    def _arrays(self):
        w = self.w
        return [_p(w[f]) for f in ("start", "count", "sum", "min", "max", "sum_sq", "last", "last_at")] + [
            _p(self.wm), _p(self.ann_len), _p(self.ann_slot), self.cap]

    def add(self, cols):
        P = max([len(c) for c in cols] + [1])
        ts = np.zeros((P, self.N), dtype=np.int64)
        vb = np.zeros((P, self.N), dtype=np.uint64)
        for s, c in enumerate(cols):
            for i, (t, v, _) in enumerate(c):
                ts[i, s], vb[i, s] = t, v
        n = np.array([len(c) for c in cols], dtype=np.uint32)
        a_off, a_ent, a_bytes = sparse_annotations(cols)
        a_off = a_off.astype(np.uint64)
        res = np.zeros((P, self.N), dtype=np.int8)
        st = np.zeros(self.N, dtype=np.int32)
        self.lib.dev_add(int(self.counter), self.N, self.R, self.res, self.off, *self._arrays(), _p(ts),
                         _p(vb.view(np.float64)), P, _p(n), _p(a_off), _p(a_ent), _p(a_bytes), _p(res), _p(st))
        return [res[: len(c), s].tolist() for s, c in enumerate(cols)], st.tolist()

    def consume(self, target, slot_words):
        k = len(self.types)
        reset = 5 in self.ops
        rows = self.R * (2 if reset else 1)
        rt = np.zeros((rows, k * self.N), dtype=np.int64)
        rv = np.zeros((rows, k * self.N), dtype=np.float64)
        rn = np.zeros(k * self.N, dtype=np.uint32)
        r_off = np.zeros(k * self.N + 1, dtype=np.uint64)
        r_ann = np.zeros(k * self.N * rows, dtype=ENTRY)
        st = np.zeros(self.N, dtype=np.int32)
        out_state = np.zeros((k * self.N, 128), dtype=np.uint8)
        types = sum(t << (4 * j) for j, t in enumerate(self.types))
        ops = sum(o << (4 * j) for j, o in enumerate(self.ops))
        self.lib.dev_consume(int(self.counter), self.N, self.R, self.res, self.off, *self._arrays(), _p(self.elem),
                             int(target), types, k, ops, int(self.discard and len(self.ops) > 0), _p(out_state),
                             slot_words, _p(rt), _p(rv), _p(rn), rows, _p(r_off), _p(r_ann), _p(st))
        assert r_off.tolist() == [i * rows for i in range(k * self.N + 1)]
        arena = self.ann_slot.reshape(-1)
        out = []
        for s in range(self.N):
            per = []
            for j in range(k):
                row = j * self.N + s
                m = rn[row]
                anns = []
                for d in range(m):
                    e = r_ann[row * rows + d]
                    assert e["dp_index"] == d
                    anns.append(arena[e["byte_offset"]: e["byte_offset"] + e["length"]].tobytes())
                per.append((rt[:m, row], rv[:m, row], anns))
            out.append(per)
        return out, st.tolist()


def _bits(v):
    return int(np.array([v], dtype=np.float64).view(np.uint64)[0])


PAYLOADS = [b"", b"", b"a", b"prom", b"0123456789abcdef", b"p" * 40]


def _append_check_holds(anns, slot_words):
    """the encoder-set append's room check for every datapoint of a row written to an empty encoder, each earlier
    datapoint at its worst case (163 bits, and its annotation's words at most): floor(bits / 32) + ENC_GUARD + 4 +
    annotation words <= slot words"""
    bits = 64
    for a in anns:
        if (bits >> 5) + ENC_GUARD + 4 + annotation_words(len(a)) > slot_words:
            return False
        bits += 163 + 32 * annotation_words(len(a))
    return True


@pytest.mark.parametrize("metric", [A.METRIC_GAUGE, A.METRIC_COUNTER])
def test_random_sequences_equal_the_model(dev, metric):
    rng = np.random.default_rng(71 + metric)
    counter = metric == A.METRIC_COUNTER
    menu = [2, 3, 4, 6, 7, 8, 9] + ([] if counter else [1])
    refused = resent = 0
    for it in range(40):
        N, R, cap = 16, int(rng.integers(1, 5)), int(rng.choice([8, 16, 48]))
        res = int(rng.choice([10, 60, 7])) * SEC
        types = sorted(rng.choice(menu, int(rng.integers(1, 4)), replace=False).tolist())
        ops = [[], [3], [1, 2], [4], [5], [4, 3, 5]][it % 6]
        discard = bool(it % 2)
        d = DevSet(dev, N, R, metric, types, res, ops, discard, cap)
        models = [AnnotatedElementModel(metric, types, res, ops, discard, open_windows=R, capacity=cap)
                  for _ in range(N)]
        clock = int(rng.integers(-5, 5)) * res
        for step in range(10):
            cols = []
            for s in range(N):
                pts = []
                for _ in range(int(rng.integers(0, 6))):
                    t = clock + int(rng.integers(-3 * res, res)) // SEC * SEC
                    v = float(rng.choice([rng.integers(-1000, 1000), np.nan, 2.5]) if counter else
                              rng.choice([rng.normal() * 100, np.nan, np.inf, -0.0]))
                    pts.append((t, _bits(v), PAYLOADS[int(rng.integers(0, len(PAYLOADS)))]))
                cols.append(pts)
            got_r, got_s = d.add(cols)
            for s, m in enumerate(models):
                assert (got_r[s], got_s[s]) == m.add(cols[s]), (it, step, s)
            if ERR_CAPACITY in got_s and rng.random() < 0.7:
                # grow and resend exactly the datapoints that got CAPACITY
                d.grow(R=min(d.R + 2, 64), cap=64)
                for m in models:
                    m.m.R, m.capacity = d.R, d.cap
                again = [[p for p, r in zip(c, got_r[s]) if r == ERR_CAPACITY] for s, c in enumerate(cols)]
                got_r, got_s = d.add(again)
                for s, m in enumerate(models):
                    assert (got_r[s], got_s[s]) == m.add(again[s]), (it, step, s)
                resent += 1
            clock += int(rng.integers(0, 2)) * res
            if rng.random() < 0.6:
                target = clock - int(rng.integers(0, 2)) * res
                slot_words = int(rng.choice([1 << 20, 40, 60, 90]))
                out, st = d.consume(target, slot_words)
                for s, m in enumerate(models):
                    if st[s] == ERR_CAPACITY:
                        refused += 1
                        assert all(len(t) == 0 for t, _, _ in out[s])
                        continue
                    assert st[s] == 0
                    want = m.consume(target)
                    for j in range(len(types)):
                        got_t, got_v, got_a = out[s][j]
                        assert np.array_equal(got_t, want[j][0]), (it, step, s, j)
                        assert np.array_equal(got_v.view(np.uint64), want[j][1].view(np.uint64)), (it, step, s, j)
                        assert got_a == want[j][2], (it, step, s, j)
                        assert _append_check_holds(got_a, slot_words), (it, step, s, j)
                    assert d.elem[s].tobytes() == m.state.tobytes()
                    assert d.wm[s] == m.watermark
    assert refused and resent  # both stops were exercised


def test_annotation_room_alone_refuses_the_element(dev):
    d = DevSet(dev, 2, 4, A.METRIC_GAUGE, [1], 60 * SEC, [], False, 64)
    assert d.add([[(5 * SEC, _bits(1.0), b"z" * 64)], [(5 * SEC, _bits(1.0), b"")]]) == ([[0], [0]], [0, 0])
    # one datapoint: 2 words + ENC_GUARD + 4 without its annotation, (64 + 3) / 4 + 4 = 20 more with it
    out, st = d.consume(60 * SEC, 2 + ENC_GUARD + 4 + 20 - 1)
    assert st == [ERR_CAPACITY, 0] and out[1][0][2] == [b""]
    assert d.w["count"][:, 0].sum() == 1 and d.ann_len[0, 0] == 64
    out, st = d.consume(60 * SEC, 2 + ENC_GUARD + 4 + 20)
    assert st == [0, 0] and out[0][0][2] == [b"z" * 64]
