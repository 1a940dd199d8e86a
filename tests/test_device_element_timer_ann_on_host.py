"""The annotated Timer element-set lanes compiled for the host from the .cu source text (tests/host_build.py):
`elem_timer_add_lane<true>` (a batch's annotation from its first row, the broken-batch rule, the capacity stop, the
window's annotation kept as a reference and copied to its slot) and `elem_timer_consume_lane<true>` (each staged
datapoint's entry, the room check counting the annotations).  A driver runs every element's lane the way the kernels
do; on random sequences -- single samples and batches, annotations on some batches and now and then on a continuation
row, NaN samples, closed windows, annotation-length / open-window / sample-room stops (each tallied on its own) each
followed by grow and resend, consumes stopped by annotation room alone -- results, statuses, staged rows and every
staged datapoint's annotation must equal the CPU model (tests/element_timer_ann_model.py), and the consume's room
bound must imply the encoder-set append's own check.  A CPU regression harness; nothing of it ships."""
import ctypes as C

import numpy as np
import pytest

from element_set_ann_model import sparse_annotations
from element_set_model import ERR_CAPACITY
from element_timer_ann_model import AnnotatedTimerModel
from host_build import compile, constants, cut, fn, source_text
from test_device_element_ann_on_host import ENTRY, _append_check_holds
from test_device_element_timer_on_host import DRIVER as TIMER_DRIVER
from test_device_element_timer_on_host import PRE, RES, SEC, DevTimerSet, _p, _value

DRIVER = TIMER_DRIVER + r"""
extern "C" void dev_add_ann(ARGS, uint32_t *ann_len, uint8_t *ann_slot, uint64_t acap, const int64_t *ts,
                            const double *val, uint64_t P, const uint32_t *n_points, const int8_t *batch,
                            const uint64_t *a_off, const m3tsz_annotation_entry *a_ent, const uint8_t *a_bytes,
                            int8_t *result, int32_t *status) {
  ElementTimerParams p = params(PASS);
  p.e.ts = ts; p.e.val = val; p.e.points_stride = P; p.e.n_points = n_points; p.e.result = result;
  p.e.status = status; p.batch = batch;
  p.e.ann_len = ann_len; p.e.ann_slot = ann_slot; p.e.ann_cap = acap;
  p.e.ann_series_off = a_off; p.e.ann_entries = a_ent; p.e.ann_bytes = a_bytes;
  for (uint64_t s = 0; s < n; s++) elem_timer_add_lane<true>(p, s);
}
extern "C" void dev_consume_ann(ARGS, uint32_t *ann_len, uint8_t *ann_slot, uint64_t acap, m3tsz_element_state *elem,
                                int64_t target, uint32_t ops, int discard, const m3tsz_encoder_state *out_state,
                                uint64_t slot_words, int64_t *row_ts, double *row_val, uint32_t *row_n,
                                uint64_t rows_stride, uint64_t *row_ann_off, m3tsz_annotation_entry *row_ann,
                                int32_t *status) {
  ElementTimerParams p = params(PASS);
  p.e.elem = elem; p.e.target = target; p.e.ops = ops; p.e.discard_nan = discard;
  p.e.out_state = out_state; p.e.out_slot_words = slot_words; p.e.row_ts = row_ts; p.e.row_val = row_val;
  p.e.row_n = row_n; p.e.rows_stride = rows_stride; p.e.status = status;
  p.e.ann_len = ann_len; p.e.ann_slot = ann_slot; p.e.ann_cap = acap; p.e.row_ann_off = row_ann_off;
  p.e.row_ann = row_ann;
  for (uint64_t s = 0; s < n; s++) {
    XfElem e;
    elem_timer_consume_lane<true>(p, s, e);
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
    lib = compile("dev_elem_timer_ann_host", "\n".join(parts), DRIVER)
    vp, i64, u64, u32, i32 = C.c_void_p, C.c_int64, C.c_uint64, C.c_uint32, C.c_int32
    head = [u64, u32, i64, i64] + [vp] * 5 + [vp] * 8 + [u32, i32, C.c_double, vp, u32, vp, u32] + [vp, vp, u64]
    lib.dev_add_ann.restype = None
    lib.dev_add_ann.argtypes = head + [vp, vp, u64, vp, vp, vp, vp, vp, vp, vp]
    lib.dev_consume_ann.restype = None
    lib.dev_consume_ann.argtypes = head + [vp, i64, u32, C.c_int, vp, u64, vp, vp, vp, u64, vp, vp, vp]
    return lib


class DevAnnTimerSet(DevTimerSet):
    """DevTimerSet with each slot's annotation (lengths start as garbage: an add writes a length when it opens a
    window)"""

    def __init__(self, lib, N, R, types, ops, discard, cap, every, eps, acap):
        super().__init__(lib, N, R, types, ops, discard, cap, every, eps)
        self.ann_len = np.full((R, N), 0xffffffff, dtype=np.uint32)
        self.ann_slot = np.zeros((R, N, acap), dtype=np.uint8)

    @property
    def acap(self):
        return self.ann_slot.shape[2]

    def grow(self, R=None, cap=None, acap=None):
        R0 = self.R
        super().grow(R, cap)
        R, acap = self.R, acap or self.acap
        ln = np.zeros((R, self.N), dtype=np.uint32)
        ln[:R0] = self.ann_len
        sl = np.zeros((R, self.N, acap), dtype=np.uint8)
        sl[:R0, :, : self.acap] = self.ann_slot
        self.ann_len, self.ann_slot = ln, sl

    def _head(self):
        return super()._head() + [_p(self.ann_len), _p(self.ann_slot), self.acap]

    def add(self, cols):
        """cols: per element [(t, v, continues, annotation)] -> (results, statuses)"""
        P = max([len(c) for c in cols] + [1])
        ts = np.zeros((P, self.N), dtype=np.int64)
        vs = np.zeros((P, self.N), dtype=np.float64)
        bt = np.zeros((P, self.N), dtype=np.int8)
        for s, c in enumerate(cols):
            for i, (t, v, b, _) in enumerate(c):
                ts[i, s], vs[i, s], bt[i, s] = t, v, b
        n = np.array([len(c) for c in cols], dtype=np.uint32)
        a_off, a_ent, a_bytes = sparse_annotations([[(0, 0, a) for *_, a in c] for c in cols])
        a_off = a_off.astype(np.uint64)
        res = np.zeros((P, self.N), dtype=np.int8)
        st = np.zeros(self.N, dtype=np.int32)
        self.lib.dev_add_ann(*self._head(), _p(ts), _p(vs), P, _p(n), _p(bt), _p(a_off), _p(a_ent), _p(a_bytes),
                             _p(res), _p(st))
        return [res[: len(c), s].tolist() for s, c in enumerate(cols)], st.tolist()

    def consume(self, target, slot_words=1 << 20):
        k = len(self.types)
        rows = self.R * (2 if 5 in self.ops else 1)
        rt = np.zeros((rows, k * self.N), dtype=np.int64)
        rv = np.zeros((rows, k * self.N), dtype=np.float64)
        rn = np.zeros(k * self.N, dtype=np.uint32)
        r_off = np.zeros(k * self.N + 1, dtype=np.uint64)
        r_ann = np.zeros(k * self.N * rows, dtype=ENTRY)
        st = np.zeros(self.N, dtype=np.int32)
        out_state = np.zeros((k * self.N, 128), dtype=np.uint8)
        ops = sum(o << (4 * j) for j, o in enumerate(self.ops))
        self.lib.dev_consume_ann(*self._head(), _p(self.elem), int(target), ops,
                                 int(self.discard and len(self.ops) > 0), _p(out_state), slot_words, _p(rt), _p(rv),
                                 _p(rn), rows, _p(r_off), _p(r_ann), _p(st))
        assert r_off.tolist() == [i * rows for i in range(k * self.N + 1)]
        arena = self.ann_slot.reshape(-1)
        out = []
        for s in range(self.N):
            per = []
            for j in range(k):
                row, m = j * self.N + s, rn[j * self.N + s]
                anns = []
                for d in range(m):
                    e = r_ann[row * rows + d]
                    assert e["dp_index"] == d
                    anns.append(arena[e["byte_offset"]: e["byte_offset"] + e["length"]].tobytes())
                per.append((rt[:m, row], rv[:m, row], anns))
            out.append(per)
        return out, st.tolist()


PAYLOADS = [b"a", b"prom", b"0123456789abcdef", b"p" * 40]
TYPES = [[3, 14, 20], [2, 3, 4, 5, 6, 7, 8, 9] + list(range(10, 25)), [3, 6]]
OPS = [[], [], [4, 3, 5]]


def _rows(rng, clock, pool):
    rows = []
    for _ in range(int(rng.integers(0, 4))):
        t = clock + int(rng.integers(-2 * RES, RES)) // SEC * SEC
        a = PAYLOADS[int(rng.integers(0, len(PAYLOADS)))] if rng.random() < 0.5 else b""
        for i in range(int(rng.integers(1, 4)) if rng.random() < 0.7 else int(rng.integers(4, 20))):
            v = _value(rng, pool)
            pool.append(v)
            rows.append((t, v, 1 if i else 0, b"" if i else a))
    if rows and rng.random() < 0.03:  # an annotation on a continuation row
        i = int(rng.integers(0, len(rows)))
        rows[i] = rows[i][:2] + (1, b"late")
    return rows


def _model_add(m, col):
    return m.add([(t, v) for t, v, _, _ in col], [b for _, _, b, _ in col], [a for *_, a in col])


@pytest.mark.parametrize("variant", range(len(TYPES)))
def test_random_sequences_equal_the_model(dev, variant):
    rng = np.random.default_rng(131 + variant)
    types, ops = TYPES[variant], OPS[variant]
    stops, refused = set(), 0
    for it in range(12):
        N, R, cap, acap = 12, int(rng.integers(1, 4)), int(rng.choice([4, 16, 64])), int(rng.choice([8, 16, 48]))
        every, eps = int(rng.choice([1, 3, 64])), float(rng.choice([1e-3, 0.05]))
        d = DevAnnTimerSet(dev, N, R, types, ops, bool(it % 2), cap, every, eps, acap)
        models = [AnnotatedTimerModel(types, RES, ops, bool(it % 2), R, cap, eps, every, capacity=acap)
                  for _ in range(N)]
        pools = [[] for _ in range(N)]
        clock = 10 * RES
        for step in range(8):
            cols = [_rows(rng, clock, pools[s]) for s in range(N)]
            got_r, got_s = d.add(cols)
            for s, m in enumerate(models):
                assert (got_r[s], got_s[s]) == _model_add(m, cols[s]), (it, step, s)
            if ERR_CAPACITY in got_s:  # grow every limit and resend exactly the refused rows
                for s, c in enumerate(cols):  # which stop: the model holds the windows as they were at the stop
                    if got_s[s] == ERR_CAPACITY:
                        t, _, _, a = c[got_r[s].index(ERR_CAPACITY)]
                        ws, m = t - t % RES, models[s].m
                        stops.add("ann" if len(a) > d.acap else
                                  "slots" if ws not in m.windows and len(m.windows) >= m.R else "samples")
                d.grow(R=d.R + 1, cap=d.cap * 2, acap=64)
                for m in models:
                    m.m.R, m.m.cap, m.capacity = d.R, d.cap, d.acap
                again = [[r for i, r in enumerate(c) if got_r[s][i] == ERR_CAPACITY] for s, c in enumerate(cols)]
                got_r, got_s = d.add(again)
                for s, m in enumerate(models):
                    assert (got_r[s], got_s[s]) == _model_add(m, again[s]), (it, step, s)
            clock += int(rng.integers(0, 2)) * RES
            if rng.random() < 0.6:
                target = clock - int(rng.integers(0, 2)) * RES
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
                    assert d.elem[s].tobytes() == m.state.tobytes() and d.wm[s] == m.watermark
    assert stops == {"ann", "slots", "samples"} and refused


def test_annotation_room_alone_refuses_the_element(dev):
    d = DevAnnTimerSet(dev, 2, 4, [3], [], False, 16, 1024, 1e-3, 64)
    assert d.add([[(5 * SEC, 1.0, 0, b"z" * 64)], [(5 * SEC, 1.0, 0, b"")]]) == ([[0], [0]], [0, 0])
    # one datapoint: 2 words + ENC_GUARD + 4 without its annotation, (64 + 3) / 4 + 4 = 20 more with it
    out, st = d.consume(RES, 2 + 10 + 4 + 20 - 1)
    assert st == [ERR_CAPACITY, 0] and out[1][0][2] == [b""]
    assert d.w["count"][:, 0].sum() == 1 and d.ann_len[0, 0] == 64
    out, st = d.consume(RES, 2 + 10 + 4 + 20)
    assert st == [0, 0] and out[0][0][2] == [b"z" * 64]
