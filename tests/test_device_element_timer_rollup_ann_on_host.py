"""The annotated Timer element rollup's device steps compiled for the host from the .cu source text
(tests/host_build.py): the forward lane `elem_timer_forward_lane<true>` (its windows' flush and values, then
ElementRollupParams::forward_ann: which forwarded windows carry an annotation, and their references), the group fold
`elem_timer_fold_group<true>` (the annotation capacity check beside the slot and sample counts in the first pass; each
group window's reference kept beside its stream, cleared when the fold moves to another window and written to the slot
only when it changed) and the commit lane.  The annotated Timer add and consume lanes feed the source set and drain the
group set, as tests/test_device_element_timer_ann_on_host.py drives them.  A driver runs the steps the way the kernels
do; statuses, staged group rows and their annotations, records, watermarks and the annotations of both sets' open slots
must equal the CPU model (tests/element_timer_ann_model.py) on random sequences: several due windows per source and
forward, group windows left and returned to within one fold, members listed twice, discard_nan on and off, annotation
/ open-window / sample-room stops each followed by grow and a re-run of exactly the failed groups (the held-back sources
forwarding the same bits and references again), closed and invalid groups.

ElementRollupParams::forward_ann and ElementParams::stage_ann_offsets restate passes that elem_forward_lane<CTR, true>
and elem_consume_lane<CTR, true> keep written out (calling the helpers there changes those kernels' SASS); two tests
run each pair on the same inputs and require the same output.  A CPU regression harness; nothing of it ships."""
import ctypes as C

import numpy as np
import pytest

from element_timer_ann_model import AnnotatedTimerGroup, AnnotatedTimerSource, forward
from element_timer_rollup_model import ERR_CAPACITY, ERR_CLOSED, ERR_INVALID_ARG, OK
from host_build import compile, constants, cut, fn, source_text
from test_device_element_timer_ann_on_host import DRIVER as ANN_DRIVER
from test_device_element_timer_ann_on_host import PRE as TIMER_PRE
from test_device_element_timer_ann_on_host import DevAnnTimerSet, _rows
from test_device_element_timer_on_host import RES, SEC, _p
from test_device_element_timer_rollup_on_host import PIPES, _memberships

PRE = TIMER_PRE + r"""
static inline double __ldg(const double *p) { return *p; }
static inline int64_t __ldg(const int64_t *p) { return *p; }
"""

DRIVER = ANN_DRIVER + r"""
extern "C" size_t params_size() { return sizeof(ElementTimerParams); }
extern "C" void make_params(ARGS, uint32_t *ann_len, uint8_t *ann_slot, uint64_t acap, m3tsz_element_state *elem,
                            uint32_t ops, ElementTimerParams *out) {
  *out = params(PASS);
  out->e.elem = elem;
  out->e.ops = ops;
  out->e.ann_len = ann_len; out->e.ann_slot = ann_slot; out->e.ann_cap = acap;
}
extern "C" void dev_forward(const ElementTimerParams *sp, const ElementTimerParams *gp, int64_t target, int discard,
                            const uint64_t *group_off, const uint32_t *members, uint64_t n_members, int64_t *fs,
                            double *fv, uint32_t *fnn, uint64_t *fp, uint64_t *fd, m3tsz_transform_state *rec,
                            uint64_t *fap, uint64_t *fa, int32_t *mark, int32_t *src_status, int32_t *group_status) {
  ElementRollupParams p;
  memset(&p, 0, sizeof(p));
  p.src = sp->e;
  p.src.target = target;
  p.discard_nan = discard;
  p.fwd_start = fs; p.fwd_val = fv; p.fwd_n = fnn; p.fwd_present = fp; p.fwd_due = fd; p.rec = rec;
  p.fwd_ann_present = fap; p.fwd_ann = fa;
  p.group_off = group_off; p.members = members; p.n_members = n_members; p.n_groups = gp->e.n;
  p.g_slots = gp->e.n_slots; p.g_start = gp->e.start; p.g_count = gp->e.count; p.g_sum = gp->e.sum;
  p.g_sum_sq = gp->e.sum_sq; p.g_watermark = gp->e.watermark;
  p.g_ann_len = gp->e.ann_len; p.g_ann_slot = gp->e.ann_slot; p.g_ann_cap = gp->e.ann_cap;
  p.group_status = group_status; p.mark = mark; p.src_status = src_status;
  ElementTimerParams s = *sp;
  s.e = p.src;
  for (uint64_t i = 0; i < p.src.n; i++) elem_timer_forward_lane<true>(p, s, i);
  for (uint64_t i = 0; i < p.src.n; i++) mark[i] = 0;
  for (uint64_t g = 0; g < p.n_groups; g++) {
    int64_t fresh[M3TSZ_MAX_ELEMENT_WINDOWS];
    uint32_t n_add[2 * M3TSZ_MAX_ELEMENT_WINDOWS];
    auto member = [&](uint64_t i) { return fwd_member<true>(p, i); };
    const int32_t st = elem_timer_fold_group<true>(p, *gp, g, fresh, n_add, member);
    const uint64_t lo = group_off[g], hi = group_off[g + 1];
    if ((st == M3TSZ_ERR_CAPACITY || st == M3TSZ_ERR_INVALID_ARG) && lo <= hi)  // (the kernel's atomicMax)
      for (uint64_t i = lo; i < (hi < n_members ? hi : n_members); i++)
        if (members[i] < p.src.n && mark[members[i]] < st) mark[members[i]] = st;
  }
  for (uint64_t i = 0; i < p.src.n; i++) elem_commit_lane(p, i);
}
// elem_forward_lane<false, true> (a Gauge Sum source) writes fap / fa with its own pass; forward_ann then writes
// fap2 / fa2 from the lane's due and presence words
extern "C" void pin_forward(uint64_t n, uint32_t R, int64_t res, int64_t *start, int64_t *count, double *sum,
                            m3tsz_element_state *elem, uint32_t *ann_len, uint64_t acap, int64_t target, int discard,
                            int64_t *fs, double *fv, uint32_t *fnn, uint64_t *fp, uint64_t *fd,
                            m3tsz_transform_state *rec, uint64_t *fap, uint64_t *fa, uint64_t *fap2, uint64_t *fa2) {
  ElementRollupParams p;
  memset(&p, 0, sizeof(p));
  p.src.n = n; p.src.n_slots = R; p.src.resolution = res; p.src.start = start; p.src.count = count; p.src.sum = sum;
  p.src.elem = elem; p.src.target = target; p.src.types = M3TSZ_AGG_SUM; p.src.n_types = 1;
  p.src.tiles.tile_sum = sum; p.src.tiles.tile_count = count; p.src.tiles.metric_type = M3TSZ_METRIC_GAUGE;
  p.src.ann_len = ann_len; p.src.ann_cap = acap;
  p.discard_nan = discard;
  p.fwd_start = fs; p.fwd_val = fv; p.fwd_n = fnn; p.fwd_present = fp; p.fwd_due = fd; p.rec = rec;
  p.fwd_ann_present = fap; p.fwd_ann = fa;
  for (uint64_t s = 0; s < n; s++) elem_forward_lane<false, true>(p, s);
  p.fwd_ann_present = fap2; p.fwd_ann = fa2;
  for (uint64_t s = 0; s < n; s++) p.forward_ann(s, fd[s], fp[s]);
}
// elem_consume_lane<false, true> on elements with no due window writes only its entry offsets (off), then
// stage_ann_offsets writes off2
extern "C" void pin_offsets(uint64_t n, uint32_t R, uint32_t k, uint64_t rows_stride, int64_t *count, uint32_t *row_n,
                            int32_t *status, uint64_t *off, uint64_t *off2) {
  ElementParams p;
  memset(&p, 0, sizeof(p));
  p.n = n; p.n_slots = R; p.n_types = k; p.types = M3TSZ_AGG_SUM; p.count = count; p.start = count;
  p.rows_stride = rows_stride; p.row_n = row_n; p.status = status; p.row_ann_off = off;
  p.tiles.metric_type = M3TSZ_METRIC_GAUGE;
  for (uint64_t s = 0; s < n; s++) {
    XfElem e;
    elem_consume_lane<false, true>(p, s, e);
  }
  p.row_ann_off = off2;
  for (uint64_t s = 0; s < n; s++) p.stage_ann_offsets(s, k);
}
"""


@pytest.fixture(scope="module")
def dev():
    enc, com, ker = source_text("m3tsz_encode.cu"), source_text("m3tsz_common.cuh"), source_text("m3tsz_kernels.h")
    parts = [PRE, constants(enc, r"kXf\w*|ENC_GUARD"), cut(ker, r"struct EncodeParams\b"),
             cut(ker, r"struct ElementParams\b"), "#define M3TSZ_MAX_TIMER_TYPES 23\n#define M3TSZ_MAX_TIMER_QUANTILES 15",
             cut(ker, r"struct ElementTimerParams\b"), cut(ker, r"struct ElementRollupParams\b"),
             cut(enc, r"struct XfElem \{"), cut(com, fn("go_f64_to_i64")), cut(com, fn("agg_stdev"))]
    for name in ("xf_isnan", "xf_bits", "xf_per_second", "xf_increase", "xf_window", "xf_element_window",
                 "tile_value_of", "elem_window_start", "elem_ends_by"):
        parts.append(cut(enc, fn(name)))
    parts.append(cut(enc, r"struct CmStream\b"))
    for name in ("timer_stream", "amd64_op", "timer_stdev", "timer_type_quantile", "timer_value_of", "elem_timer_add_lane",
                 "elem_timer_consume_lane", "elem_consume_lane", "elem_forward_lane"):
        parts.append(cut(enc, fn(name)))
    parts.append(cut(enc, r"struct FwdMember\b"))
    for name in ("fwd_member", "elem_commit_lane", "elem_timer_forward_lane", "elem_timer_fold_group"):
        parts.append(cut(enc, fn(name)))
    body = "\n".join(parts).replace('asm volatile("mov.b64 %0, %1;" : "=l"(oi) : "l"(o));', "oi = o;")
    lib = compile("dev_elem_timer_rollup_ann_host", body, DRIVER)
    vp, i64, u64, u32, i32 = C.c_void_p, C.c_int64, C.c_uint64, C.c_uint32, C.c_int32
    head = [u64, u32, i64, i64] + [vp] * 5 + [vp] * 8 + [u32, i32, C.c_double, vp, u32, vp, u32] + [vp, vp, u64]
    lib.dev_add_ann.restype = None
    lib.dev_add_ann.argtypes = head + [vp, vp, u64, vp, vp, vp, vp, vp, vp, vp]
    lib.dev_consume_ann.restype = None
    lib.dev_consume_ann.argtypes = head + [vp, i64, u32, C.c_int, vp, u64, vp, vp, vp, u64, vp, vp, vp]
    lib.params_size.restype = C.c_size_t
    lib.make_params.restype = None
    lib.make_params.argtypes = head + [vp, u32, vp]
    lib.dev_forward.restype = None
    lib.dev_forward.argtypes = [vp, vp, i64, C.c_int, vp, vp, u64] + [vp] * 11
    lib.pin_forward.restype = None
    lib.pin_forward.argtypes = [u64, u32, i64, vp, vp, vp, vp, vp, u64, i64, C.c_int] + [vp] * 10
    lib.pin_offsets.restype = None
    lib.pin_offsets.argtypes = [u64, u32, u32, u64, vp, vp, vp, vp, vp]
    return lib


def _params(lib, d):
    buf = C.create_string_buffer(lib.params_size())
    lib.make_params(*d._head(), _p(d.elem), sum(o << (4 * j) for j, o in enumerate(d.ops)), buf)
    return buf


def dev_forward(lib, src, grp, target, group_off, members):
    """one annotated forward of DevAnnTimerSet src into DevAnnTimerSet grp -> (source statuses, group statuses)"""
    S, G = src.N, grp.N
    fs = np.zeros((src.R, S), dtype=np.int64)
    fv = np.zeros((src.R, S), dtype=np.float64)
    fnn = np.zeros(S, dtype=np.uint32)
    fp, fd, fap = (np.zeros(S, dtype=np.uint64) for _ in range(3))
    fa = np.full((src.R, S), 0xdeadbeef, dtype=np.uint64)  # (read only where fap's bit is set)
    rec = np.zeros((S, 96), dtype=np.uint8)
    mark, sst, gst = np.zeros(S, dtype=np.int32), np.zeros(S, dtype=np.int32), np.zeros(G, dtype=np.int32)
    off = np.ascontiguousarray(group_off, dtype=np.uint64)
    mem = np.ascontiguousarray(members, dtype=np.uint32)
    lib.dev_forward(_params(lib, src), _params(lib, grp), int(target), int(src.discard), _p(off), _p(mem), len(mem),
                    _p(fs), _p(fv), _p(fnn), _p(fp), _p(fd), _p(rec), _p(fap), _p(fa), _p(mark), _p(sst), _p(gst))
    return sst.tolist(), gst.tolist()


def _open_annotations(d):
    """{(element, window start): annotation} of a DevAnnTimerSet's open slots (above the capacity reads as b"")"""
    out = {}
    for r in range(d.R):
        for s in range(d.N):
            if d.w["count"][r, s]:
                ln = int(d.ann_len[r, s])
                out[(s, int(d.w["start"][r, s]))] = d.ann_slot[r, s, :ln].tobytes() if ln <= d.acap else b""
    return out


def _model_annotations(models):
    out = {}
    for s, m in enumerate(models):
        for ws in m.m.windows:
            a = m.ann[ws]
            out[(s, ws)] = b"" if m.capacity is not None and len(a) > m.capacity else a
    return out


def _stops(sms, gms, target, off, mem):
    """per group, which capacity rules the forward would break: "ann" (an annotation longer than the group slots),
    "slots" (more new windows than free slots), "samples" (a window past sample_capacity)"""
    fw = [s.forwarded(target) for s in sms]
    out = []
    for g, grp in enumerate(gms):
        lo, hi = int(off[g]), int(off[g + 1])
        stop = set()
        if lo <= hi <= len(mem) and all(int(mem[i]) < len(sms) for i in range(lo, hi)):
            vals = [(ws, a) for i in range(lo, hi) for ws, _, a in fw[int(mem[i])] if not grp.m.closed(ws)]
            if any(len(a) > grp.capacity for _, a in vals):
                stop.add("ann")
            starts = [ws for ws, _ in vals]
            if len(grp.m.windows) + len(set(starts) - set(grp.m.windows)) > grp.m.R:
                stop.add("slots")
            if any((grp.m.windows[ws].stream.size() if ws in grp.m.windows else 0) + starts.count(ws) > grp.m.cap
                   for ws in set(starts)):
                stop.add("samples")
        out.append(stop)
    return out


@pytest.mark.parametrize("pipe", range(len(PIPES)))
def test_random_sequences_equal_the_model(dev, pipe):
    src_type, pre, types, post = PIPES[pipe]
    rng = np.random.default_rng(211 + pipe)
    seen, stops, retried, multi, long_src = set(), set(), 0, 0, 0
    for it in range(14):
        S, G, R, RG = 12, 6, int(rng.integers(2, 5)), int(rng.integers(1, 4))
        cap, gcap, acap, gacap = 64, int(rng.choice([2, 3, 6, 64])), 48, int(rng.choice([8, 16, 48]))
        every, eps = int(rng.choice([1, 2, 3, 1024])), float(rng.choice([1e-3, 0.05]))
        discard = bool(it % 2)
        src = DevAnnTimerSet(dev, S, R, [src_type], pre, discard, cap, every, eps, acap)
        grp = DevAnnTimerSet(dev, G, RG, types, post, discard, gcap, every, eps, gacap)
        sms = [AnnotatedTimerSource(src_type, RES, pre, discard, R, cap, eps, every, capacity=acap) for _ in range(S)]
        gms = [AnnotatedTimerGroup(types, RES, post, discard, RG, gcap, eps, every, capacity=gacap) for _ in range(G)]
        off, mem = _memberships(rng, S, G)
        if len(mem) > 1:
            mem[int(rng.integers(1, len(mem)))] = mem[0]  # a member listed twice (in one group or in two)
        pools = [[] for _ in range(S)]
        clock = 10 * RES
        for step in range(8):
            cols = [_rows(rng, clock, pools[s]) for s in range(S)]
            got_r, got_s = src.add(cols)
            for s, m in enumerate(sms):
                c = cols[s]
                want = m.add([(t, v) for t, v, _, _ in c], [b for _, _, b, _ in c], [a for *_, a in c])
                assert (got_r[s], got_s[s]) == want, (it, step, s)
            if rng.random() < 0.3:  # a source slot whose length reads above the capacity
                r, s = int(rng.integers(0, src.R)), int(rng.integers(0, S))
                if src.w["count"][r, s]:
                    src.ann_len[r, s] = acap + 8
                    sms[s].set_length_above_capacity(int(src.w["start"][r, s]))
                    long_src += 1
            clock += int(rng.integers(0, 2)) * RES
            if rng.random() < 0.75:
                target = clock - int(rng.integers(0, 2)) * RES
                multi += sum(len(m.forwarded(target)) > 1 for m in sms)
                why = _stops(sms, gms, target, off, mem)
                sst, gst = dev_forward(dev, src, grp, target, off, mem)
                assert (sst, gst) == forward(sms, gms, target, off, mem), (it, step)
                seen.update(gst)
                failed = [g for g in range(G) if gst[g] == ERR_CAPACITY]
                for g in failed:
                    assert why[g], (it, step, g)
                    stops.update(why[g])
                if failed:  # grow every limit and re-run exactly the failed groups
                    grp.grow(R=grp.R + 2, cap=grp.cap * 4, acap=64)
                    for m in gms:
                        m.m.R, m.m.cap, m.capacity = grp.R, grp.cap, grp.acap
                    lens = [int(off[g + 1] - off[g]) if g in failed else 0 for g in range(G)]
                    off2 = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
                    mem2 = np.concatenate([mem[int(off[g]): int(off[g + 1])] for g in failed]).astype(np.uint32)
                    got = dev_forward(dev, src, grp, target, off2, mem2)
                    assert got == forward(sms, gms, target, off2, mem2), (it, step, "retry")
                    retried += 1
                for s, m in enumerate(sms):
                    assert src.elem[s].tobytes() == m.state.tobytes() and src.wm[s] == m.watermark, (it, step, s)
                assert _open_annotations(src) == _model_annotations(sms), (it, step)
                assert _open_annotations(grp) == _model_annotations(gms), (it, step)
                if rng.random() < 0.6:
                    out, st = grp.consume(target)
                    assert st == [OK] * G
                    for g, m in enumerate(gms):
                        want = m.consume(target)
                        for j in range(len(types)):
                            got_t, got_v, got_a = out[g][j]
                            assert np.array_equal(got_t, want[j][0]), (it, step, g, j)
                            assert np.array_equal(got_v.view(np.uint64), want[j][1].view(np.uint64)), (it, step, g, j)
                            assert got_a == want[j][2], (it, step, g, j)
                        assert grp.elem[g].tobytes() == m.state.tobytes() and grp.wm[g] == m.watermark
    assert seen == {OK, ERR_CLOSED, ERR_CAPACITY, ERR_INVALID_ARG}
    assert stops == {"ann", "slots", "samples"} and retried and multi and long_src


def test_fold_leaves_and_returns_to_a_group_window(dev):
    """one group fed windows A, B, A in listed order: the fold leaves A's slot, takes B's (whose reference starts
    cleared), and returns to A; each window keeps the last annotation of its own values"""
    src = DevAnnTimerSet(dev, 3, 2, [20], [], False, 16, 1024, 1e-3, 16)
    grp = DevAnnTimerSet(dev, 1, 2, [3, 20], [], False, 16, 1024, 1e-3, 16)
    sms = [AnnotatedTimerSource(20, RES, capacity=16) for _ in range(3)]
    gms = [AnnotatedTimerGroup([3, 20], RES, capacity=16)]
    cols = [[(SEC, 1.0, 0, b"A1")], [(RES + SEC, 2.0, 0, b"")], [(SEC, 3.0, 0, b"A3")]]
    src.add(cols)
    for m, c in zip(sms, cols):
        m.add([(t, v) for t, v, _, _ in c], None, [a for *_, a in c])
    assert dev_forward(dev, src, grp, 2 * RES, [0, 3], [0, 1, 2]) == forward(sms, gms, 2 * RES, [0, 3], [0, 1, 2])
    assert _open_annotations(grp) == _model_annotations(gms) == {(0, 0): b"A3", (0, RES): b""}


def test_forward_ann_equals_the_forward_lanes_pass(dev):
    rng = np.random.default_rng(5)
    for it in range(40):
        N, R, acap = 16, int(rng.integers(1, 9)), 16
        start = np.zeros((R, N), dtype=np.int64)
        for s in range(N):
            start[:, s] = rng.permutation(np.arange(-3, 9))[:R] * RES
        count = (rng.random((R, N)) < 0.7).astype(np.int64) * rng.integers(1, 5, (R, N))
        sm = np.where(rng.random((R, N)) < 0.2, np.nan, rng.normal(size=(R, N)))
        ann_len = rng.choice([0, 0, 3, 8, 16, 17, 0xffffffff], (R, N)).astype(np.uint32)
        elem = np.zeros((N, 160), dtype=np.uint8)
        fs, fv = np.zeros((R, N), dtype=np.int64), np.zeros((R, N), dtype=np.float64)
        fnn = np.zeros(N, dtype=np.uint32)
        fp, fd, fap, fap2 = (np.zeros(N, dtype=np.uint64) for _ in range(4))
        fa, fa2 = np.zeros((R, N), dtype=np.uint64), np.zeros((R, N), dtype=np.uint64)
        rec = np.zeros((N, 96), dtype=np.uint8)
        dev.pin_forward(N, R, RES, _p(start), _p(count), _p(sm), _p(elem), _p(ann_len), acap, 6 * RES, it % 2,
                        _p(fs), _p(fv), _p(fnn), _p(fp), _p(fd), _p(rec), _p(fap), _p(fa), _p(fap2), _p(fa2))
        assert np.array_equal(fap, fap2), it
        for s in range(N):
            for q in range(R):
                if (int(fap[s]) >> q) & 1:
                    assert fa[q, s] == fa2[q, s], (it, s, q)


def test_stage_ann_offsets_equals_the_consume_lanes_loop(dev):
    for n, R, k, stride in ((1, 1, 1, 1), (7, 3, 4, 6), (33, 2, 23, 4)):
        count = np.zeros((R, n), dtype=np.int64)
        row_n = np.zeros(k * n, dtype=np.uint32)
        st = np.zeros(n, dtype=np.int32)
        off, off2 = np.full(k * n + 1, 7, dtype=np.uint64), np.full(k * n + 1, 9, dtype=np.uint64)
        dev.pin_offsets(n, R, k, stride, _p(count), _p(row_n), _p(st), _p(off), _p(off2))
        assert off.tolist() == off2.tolist() == [i * stride for i in range(k * n + 1)]

