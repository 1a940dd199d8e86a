"""The annotated element rollup's device steps compiled for the host from the .cu source text (tests/host_build.py):
the forward lane `elem_forward_lane<CTR, true>` (which forwarded windows carry an annotation, and their references),
the group fold `elem_fold_group<CTR, true>` (each group window's annotation in listed member order, written to its slot
when it changed; the annotation capacity check in the first pass) and the commit lane, with the annotated add and
consume lanes feeding the source set and draining the group set, as tests/test_device_element_ann_on_host.py drives
them.  A driver runs the steps the way the kernels do, as tests/test_device_element_rollup_on_host.py's does; statuses,
staged group rows and their annotations, the records, the watermarks and the annotations of both sets' open slots must
equal the CPU model (tests/element_rollup_ann_model.py) on random sequences: annotation-capacity and open-window stops
followed by re-runs of exactly the failed groups, closed and invalid groups, NaNs with and without discard_nan, a
member listed twice, source slot lengths above the capacity, and group windows open across forwards.  A CPU
regression harness; nothing of it ships."""
import ctypes as C

import numpy as np
import pytest

import agg_oracle_lib as A
from element_rollup_ann_model import (ERR_CAPACITY, ERR_CLOSED, ERR_INVALID_ARG, OK, AnnotatedGroup,
                                       AnnotatedSource, forward)
from host_build import compile, constants, cut, fn, source_text
from test_device_element_ann_on_host import DRIVER as ANN_DRIVER
from test_device_element_ann_on_host import PRE, DevSet, _bits, _p
from test_device_element_rollup_on_host import PIPES, _memberships

SEC = 1_000_000_000

DRIVER = ANN_DRIVER + r"""
extern "C" void dev_forward(int counter, uint64_t n, uint32_t R, int64_t res, int64_t off, int64_t *start,
                            int64_t *count, void *sum, void *mn, void *mx, void *sq, double *last, int64_t *last_at,
                            int64_t *wm, uint32_t *ann_len, uint8_t *ann_slot, uint64_t cap,
                            m3tsz_element_state *elem, int64_t target, uint32_t type, uint32_t ops, int discard,
                            uint64_t G, uint32_t RG, int64_t *g_start, int64_t *g_count, void *g_sum, void *g_min,
                            void *g_max, void *g_sq, double *g_last, int64_t *g_last_at, int64_t *g_wm,
                            uint32_t *g_ann_len, uint8_t *g_ann_slot, uint64_t g_cap, const uint64_t *group_off,
                            const uint32_t *members, uint64_t n_members, int64_t *fs, double *fv, uint32_t *fnn,
                            uint64_t *fp, uint64_t *fd, m3tsz_transform_state *rec, uint64_t *fap, uint64_t *fa,
                            int32_t *mark, int32_t *src_status, int32_t *group_status) {
  ElementRollupParams p;
  memset(&p, 0, sizeof(p));
  p.src = params(counter, n, R, res, off, start, count, sum, mn, mx, sq, last, last_at, wm, ann_len, ann_slot, cap);
  p.src.elem = elem; p.src.target = target; p.src.types = type; p.src.n_types = 1; p.src.ops = ops;
  p.src.tiles.metric_type = counter ? M3TSZ_METRIC_COUNTER : M3TSZ_METRIC_GAUGE;
  p.discard_nan = discard;
  p.fwd_start = fs; p.fwd_val = fv; p.fwd_n = fnn; p.fwd_present = fp; p.fwd_due = fd; p.rec = rec;
  p.fwd_ann_present = fap; p.fwd_ann = fa;
  p.group_off = group_off; p.members = members; p.n_members = n_members; p.n_groups = G;
  p.g_slots = RG; p.g_start = g_start; p.g_count = g_count; p.g_sum = g_sum; p.g_min = g_min; p.g_max = g_max;
  p.g_sum_sq = g_sq; p.g_last = g_last; p.g_last_at = g_last_at; p.g_watermark = g_wm;
  p.g_ann_len = g_ann_len; p.g_ann_slot = g_ann_slot; p.g_ann_cap = g_cap;
  p.group_status = group_status; p.mark = mark; p.src_status = src_status;
  for (uint64_t s = 0; s < n; s++) counter ? elem_forward_lane<true, true>(p, s) : elem_forward_lane<false, true>(p, s);
  for (uint64_t s = 0; s < n; s++) mark[s] = 0;
  for (uint64_t g = 0; g < G; g++) {
    int64_t fresh[M3TSZ_MAX_ELEMENT_WINDOWS];
    auto member = [&](uint64_t i) { return fwd_member<true>(p, i); };
    const int32_t st = counter ? elem_fold_group<true, true>(p, g, fresh, member)
                               : elem_fold_group<false, true>(p, g, fresh, member);
    const uint64_t lo = group_off[g], hi = group_off[g + 1];
    if ((st == M3TSZ_ERR_CAPACITY || st == M3TSZ_ERR_INVALID_ARG) && lo <= hi)  // (the kernel's atomicMax)
      for (uint64_t i = lo; i < (hi < n_members ? hi : n_members); i++)
        if (members[i] < n && mark[members[i]] < st) mark[members[i]] = st;
  }
  for (uint64_t s = 0; s < n; s++) elem_commit_lane(p, s);
}
"""


@pytest.fixture(scope="module")
def dev():
    enc, com, ker = source_text("m3tsz_encode.cu"), source_text("m3tsz_common.cuh"), source_text("m3tsz_kernels.h")
    parts = [PRE, constants(enc, r"kXf\w*|ENC_GUARD"), cut(ker, r"struct EncodeParams\b"),
             cut(ker, r"struct ElementParams\b"), cut(ker, r"struct ElementRollupParams\b"),
             cut(enc, r"struct XfElem \{"), cut(com, fn("go_f64_to_i64")), cut(com, fn("agg_stdev"))]
    for name in ("xf_isnan", "xf_bits", "xf_per_second", "xf_increase", "xf_window", "xf_element_window",
                 "tile_value_of", "elem_window_start", "elem_ends_by"):
        parts.append(cut(enc, fn(name)))
    parts += [cut(enc, r"struct ElemAcc\b"), cut(enc, r"struct RollupGaugeAcc\b"), cut(enc, r"struct RollupCounterAcc\b")]
    for name in ("elem_init", "elem_load", "elem_store", "elem_update", "elem_add_lane", "elem_consume_lane",
                 "rollup_gauge_init", "rollup_counter_init", "rollup_add", "rollup_gauge_add", "rollup_counter_add",
                 "elem_forward_lane"):
        parts.append(cut(enc, fn(name)))
    parts.append(cut(enc, r"struct ElemFoldAcc\b"))
    for name in ("elem_fold_load", "elem_fold_store"):
        parts.append(cut(enc, fn(name)))
    parts.append(cut(enc, r"struct FwdMember\b"))
    for name in ("fwd_member", "elem_fold_group", "elem_commit_lane"):
        parts.append(cut(enc, fn(name)))
    body = "\n".join(parts)
    body = body.replace('asm volatile("mov.b64 %0, %1;" : "=l"(oi) : "l"(o));', "oi = o;")
    lib = compile("dev_elem_rollup_ann_host", body, DRIVER)
    vp, i64, u64, u32 = C.c_void_p, C.c_int64, C.c_uint64, C.c_uint32
    lib.dev_add.restype = None
    lib.dev_add.argtypes = [C.c_int, u64, u32, i64, i64] + [vp] * 9 + [vp, vp, u64] + [vp, vp, u64, vp, vp, vp, vp,
                                                                                        vp, vp]
    lib.dev_consume.restype = None
    lib.dev_consume.argtypes = [C.c_int, u64, u32, i64, i64] + [vp] * 9 + [vp, vp, u64] + [
        vp, i64, u32, u32, u32, C.c_int, vp, u64, vp, vp, vp, u64, vp, vp, vp]
    lib.dev_forward.restype = None
    lib.dev_forward.argtypes = ([C.c_int, u64, u32, i64, i64] + [vp] * 9 + [vp, vp, u64] +
                                [vp, i64, u32, u32, C.c_int, u64, u32] + [vp] * 9 + [vp, vp, u64] + [vp, vp, u64] +
                                [vp] * 11)
    return lib


def dev_forward(lib, src, grp, src_type, target, group_off, members):
    """one annotated forward of DevSet src into DevSet grp -> (source statuses, group statuses)"""
    S, G = src.N, grp.N
    fs = np.zeros((src.R, S), dtype=np.int64)
    fv = np.zeros((src.R, S), dtype=np.float64)
    fnn = np.zeros(S, dtype=np.uint32)
    fp = np.zeros(S, dtype=np.uint64)
    fd = np.zeros(S, dtype=np.uint64)
    rec = np.zeros((S, 96), dtype=np.uint8)
    fap = np.zeros(S, dtype=np.uint64)
    fa = np.full((src.R, S), 0xdeadbeef, dtype=np.uint64)  # (read only where fap's bit is set)
    mark = np.zeros(S, dtype=np.int32)
    sst = np.zeros(S, dtype=np.int32)
    gst = np.zeros(G, dtype=np.int32)
    off = np.ascontiguousarray(group_off, dtype=np.uint64)
    mem = np.ascontiguousarray(members, dtype=np.uint32)
    ops = sum(o << (4 * j) for j, o in enumerate(src.ops))
    lib.dev_forward(int(src.counter), S, src.R, src.res, src.off, *src._arrays(), _p(src.elem), int(target), src_type,
                    ops, int(src.discard), G, grp.R, *grp._arrays(), _p(off), _p(mem), len(mem), _p(fs), _p(fv),
                    _p(fnn), _p(fp), _p(fd), _p(rec), _p(fap), _p(fa), _p(mark), _p(sst), _p(gst))
    return sst.tolist(), gst.tolist()


def _open_annotations(d):
    """{(element, window start): annotation} of a DevSet's open slots (a length above the capacity reads as b"")"""
    out = {}
    for r in range(d.R):
        for s in range(d.N):
            if d.w["count"][r, s]:
                ln = int(d.ann_len[r, s])
                out[(s, int(d.w["start"][r, s]))] = d.ann_slot[r, s, :ln].tobytes() if ln <= d.cap else b""
    return out


def _model_annotations(models):
    out = {}
    for s, m in enumerate(models):
        for ws in m.m.windows:
            a = m.ann[ws]
            out[(s, ws)] = b"" if m.capacity is not None and len(a) > m.capacity else a
    return out


PAYLOADS = [b"", b"", b"", b"a", b"prom", b"0123456789abcdef", b"p" * 40]


@pytest.mark.parametrize("pipe", range(len(PIPES)))
def test_random_sequences_equal_the_model(dev, pipe):
    metric, src_type, pre, types, post = PIPES[pipe]
    counter = metric == A.METRIC_COUNTER
    rng = np.random.default_rng(171 + pipe)
    seen, retried, long_src, kept_open = set(), 0, 0, 0
    for it in range(25):
        S, G, R, RG = 14, 6, int(rng.integers(2, 5)), int(rng.integers(1, 4))
        cap, gcap = 48, int(rng.choice([8, 16, 48]))
        res = int(rng.choice([10, 60])) * SEC
        discard = bool(it % 2)
        src = DevSet(dev, S, R, metric, [src_type], res, pre, discard, cap)
        grp = DevSet(dev, G, RG, metric, types, res, post, discard, gcap)
        sms = [AnnotatedSource(metric, src_type, res, pre, discard, open_windows=R, capacity=cap) for _ in range(S)]
        gms = [AnnotatedGroup(metric, types, res, post, discard, open_windows=RG, capacity=gcap) for _ in range(G)]
        off, mem = _memberships(rng, S, G)
        if len(mem) > 1:
            mem[int(rng.integers(1, len(mem)))] = mem[0]  # a member listed twice (in one group or in two)
        clock = int(rng.integers(-5, 5)) * res
        for step in range(8):
            cols = []
            for s in range(S):
                pts = []
                for _ in range(int(rng.integers(0, 4))):
                    t = clock + int(rng.integers(-3 * res, res)) // SEC * SEC
                    v = float(rng.choice([rng.integers(-1000, 1000), np.nan]) if counter else
                              rng.choice([rng.normal() * 100, np.nan, np.inf]))
                    pts.append((t, _bits(v), PAYLOADS[int(rng.integers(0, len(PAYLOADS)))]))
                cols.append(pts)
            got_r, got_s = src.add(cols)
            for s, m in enumerate(sms):
                assert (got_r[s], got_s[s]) == m.add(cols[s]), (it, step, s)
            if rng.random() < 0.3:  # a source slot whose length reads above the capacity
                r, s = int(rng.integers(0, R)), int(rng.integers(0, S))
                if src.w["count"][r, s]:
                    src.ann_len[r, s] = cap + 8
                    sms[s].set_length_above_capacity(int(src.w["start"][r, s]))
                    long_src += 1
            clock += int(rng.integers(0, 2)) * res
            if rng.random() < 0.7:
                target = clock - int(rng.integers(0, 2)) * res
                sst, gst = dev_forward(dev, src, grp, src_type, target, off, mem)
                wst, wgst = forward(sms, gms, target, off, mem)
                assert (sst, gst) == (wst, wgst), (it, step)
                seen.update(gst)
                failed = [g for g in range(G) if gst[g] == ERR_CAPACITY]
                if failed and rng.random() < 0.8:
                    # grow the group set (open windows and annotation bytes), re-run exactly the failed groups
                    grp.grow(R=RG + 4, cap=64)
                    RG += 4
                    for m in gms:
                        m.m.R, m.capacity = RG, 64
                    lens = [int(off[g + 1] - off[g]) if g in failed else 0 for g in range(G)]
                    off2 = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
                    mem2 = np.concatenate([mem[int(off[g]): int(off[g + 1])] for g in failed]).astype(np.uint32)
                    sst, gst = dev_forward(dev, src, grp, src_type, target, off2, mem2)
                    wst, wgst = forward(sms, gms, target, off2, mem2)
                    assert (sst, gst) == (wst, wgst), (it, step, "retry")
                    retried += 1
                for s, m in enumerate(sms):
                    assert src.elem[s].tobytes() == m.state.tobytes(), (it, step, s)
                    assert src.wm[s] == m.watermark
                assert _open_annotations(src) == _model_annotations(sms), (it, step)
                g_ann = _open_annotations(grp)
                assert g_ann == _model_annotations(gms), (it, step)
                kept_open += sum(1 for a in g_ann.values() if a)
                if rng.random() < 0.5:
                    out, st = grp.consume(target, 1 << 20)
                    assert st == [OK] * G
                    for g, m in enumerate(gms):
                        want = m.consume(target)
                        for j in range(len(types)):
                            got_t, got_v, got_a = out[g][j]
                            assert np.array_equal(got_t, want[j][0]), (it, step, g, j)
                            assert np.array_equal(got_v.view(np.uint64), want[j][1].view(np.uint64)), (it, step, g, j)
                            assert got_a == want[j][2], (it, step, g, j)
                        assert grp.elem[g].tobytes() == m.state.tobytes()
                        assert grp.wm[g] == m.watermark
    assert seen == {OK, ERR_CLOSED, ERR_CAPACITY, ERR_INVALID_ARG} and retried > 0 and long_src > 0 and kept_open > 0


def test_annotation_capacity_alone_stops_the_group(dev):
    """one group, room for its window, an annotation one word too long: CAPACITY with nothing folded and the source
    held back; a closed window's long annotation does not count; growing the capacity and re-running folds it"""
    res = 10 * SEC
    src = DevSet(dev, 2, 2, A.METRIC_GAUGE, [1], res, [], False, 32)
    grp = DevSet(dev, 1, 2, A.METRIC_GAUGE, [7], res, [], False, 8)
    assert src.add([[(5 * SEC, _bits(1.0), b"x" * 9)], [(5 * SEC, _bits(2.0), b"y" * 8)]]) == ([[0], [0]], [0, 0])
    assert dev_forward(dev, src, grp, 1, res, [0, 2], [1, 0]) == ([ERR_CAPACITY, ERR_CAPACITY], [ERR_CAPACITY])
    assert grp.w["count"].sum() == 0 and src.w["count"].sum() == 2
    grp.grow(cap=16)
    assert dev_forward(dev, src, grp, 1, res, [0, 2], [1, 0]) == ([OK, OK], [OK])
    assert _open_annotations(grp) == {(0, 0): b"x" * 9}
    out, st = grp.consume(res, 1 << 20)
    assert st == [OK] and out[0][0][2] == [b"x" * 9]
    # the group window [0, res) is closed now: a late source value with a long annotation gets CLOSED, not CAPACITY
    late = DevSet(dev, 1, 2, A.METRIC_GAUGE, [1], res, [], False, 32)
    late.add([[(5 * SEC, _bits(3.0), b"z" * 30)]])
    assert dev_forward(dev, late, grp, 1, res, [0, 1], [0]) == ([OK], [ERR_CLOSED])
