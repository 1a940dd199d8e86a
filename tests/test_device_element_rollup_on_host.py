"""The element rollup's device steps compiled for the host from the .cu source text (tests/host_build.py): the forward
lane (`elem_forward_lane`: the due windows in start order through tile_value_of and xf_window, the source-side NaN
discard), the group fold (`elem_fold_group`: the range and index checks, the capacity count, the fold in listed order
into the window with the source window's start, closed group windows) and the commit lane (`elem_commit_lane`), with
`struct ElementRollupParams` of m3tsz_kernels.h.  The source set is fed by the add lane and the group set consumed by
the consume lane, as in tests/test_device_element_set_on_host.py.  A driver runs the steps the way the kernels do (every
source's forward, every group's fold with its failed groups marking their members, every source's commit); statuses,
group rows and records, source records and watermarks must equal the CPU model (tests/element_rollup_model.py) on
random sequences: CAPACITY stops followed by re-runs of exactly the failed groups, closed group windows, invalid
groups, sources in several groups or in none, NaN / +-Inf.  A CPU regression harness; nothing of it ships."""
import ctypes as C

import numpy as np
import pytest

import agg_oracle_lib as A
from element_rollup_model import ERR_CAPACITY, ERR_CLOSED, ERR_INVALID_ARG, OK, GroupModel, SourceModel, forward
from host_build import compile, constants, cut, fn, source_text
from test_device_element_set_on_host import DRIVER as SET_DRIVER
from test_device_element_set_on_host import PRE, DevSet, _bits, _p, _value

SEC = 1_000_000_000

DRIVER = SET_DRIVER + r"""
extern "C" void dev_forward(int counter, uint64_t n, uint32_t R, int64_t res, int64_t off, int64_t *start,
                            int64_t *count, void *sum, void *mn, void *mx, void *sq, double *last, int64_t *last_at,
                            int64_t *wm, m3tsz_element_state *elem, int64_t target, uint32_t type, uint32_t ops,
                            int discard, uint64_t G, uint32_t RG, int64_t *g_start, int64_t *g_count, void *g_sum,
                            void *g_min, void *g_max, void *g_sq, double *g_last, int64_t *g_last_at, int64_t *g_wm,
                            const uint64_t *group_off, const uint32_t *members, uint64_t n_members, int64_t *fs,
                            double *fv, uint32_t *fnn, uint64_t *fp, uint64_t *fd, m3tsz_transform_state *rec,
                            int32_t *mark, int32_t *src_status, int32_t *group_status) {
  ElementRollupParams p;
  memset(&p, 0, sizeof(p));
  p.src = params(counter, n, R, res, off, start, count, sum, mn, mx, sq, last, last_at, wm);
  p.src.elem = elem; p.src.target = target; p.src.types = type; p.src.n_types = 1; p.src.ops = ops;
  p.src.tiles.metric_type = counter ? M3TSZ_METRIC_COUNTER : M3TSZ_METRIC_GAUGE;
  p.discard_nan = discard;
  p.fwd_start = fs; p.fwd_val = fv; p.fwd_n = fnn; p.fwd_present = fp; p.fwd_due = fd; p.rec = rec;
  p.group_off = group_off; p.members = members; p.n_members = n_members; p.n_groups = G;
  p.g_slots = RG; p.g_start = g_start; p.g_count = g_count; p.g_sum = g_sum; p.g_min = g_min; p.g_max = g_max;
  p.g_sum_sq = g_sq; p.g_last = g_last; p.g_last_at = g_last_at; p.g_watermark = g_wm;
  p.group_status = group_status; p.mark = mark; p.src_status = src_status;
  for (uint64_t s = 0; s < n; s++) counter ? elem_forward_lane<true>(p, s) : elem_forward_lane<false>(p, s);
  for (uint64_t s = 0; s < n; s++) mark[s] = 0;
  for (uint64_t g = 0; g < G; g++) {
    int64_t fresh[M3TSZ_MAX_ELEMENT_WINDOWS];
    auto member = [&](uint64_t i) { return fwd_member(p, i); };
    const int32_t st = counter ? elem_fold_group<true>(p, g, fresh, member) : elem_fold_group<false>(p, g, fresh, member);
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
    lib = compile("dev_elem_rollup_host", body, DRIVER)
    vp, i64, u64, u32 = C.c_void_p, C.c_int64, C.c_uint64, C.c_uint32
    lib.dev_add.restype = None
    lib.dev_add.argtypes = [C.c_int, u64, u32, i64, i64] + [vp] * 9 + [vp, vp, u64, vp, vp, vp]
    lib.dev_consume.restype = None
    lib.dev_consume.argtypes = [C.c_int, u64, u32, i64, i64] + [vp] * 9 + [vp, i64, u32, u32, u32, C.c_int, vp, u64,
                                                                           vp, vp, vp, u64, vp]
    lib.dev_forward.restype = None
    lib.dev_forward.argtypes = ([C.c_int, u64, u32, i64, i64] + [vp] * 9 + [vp, i64, u32, u32, C.c_int, u64, u32]
                                + [vp] * 9 + [vp, vp, u64] + [vp] * 9)
    return lib


def dev_forward(lib, src, grp, src_type, target, group_off, members):
    """one forward of DevSet src into DevSet grp -> (source statuses, group statuses)"""
    S, G = src.N, grp.N
    fs = np.zeros((src.R, S), dtype=np.int64)
    fv = np.zeros((src.R, S), dtype=np.float64)
    fnn = np.zeros(S, dtype=np.uint32)
    fp = np.zeros(S, dtype=np.uint64)
    fd = np.zeros(S, dtype=np.uint64)
    rec = np.zeros((S, 96), dtype=np.uint8)
    mark = np.zeros(S, dtype=np.int32)
    sst = np.zeros(S, dtype=np.int32)
    gst = np.zeros(G, dtype=np.int32)
    off = np.ascontiguousarray(group_off, dtype=np.uint64)
    mem = np.ascontiguousarray(members, dtype=np.uint32)
    ops = sum(o << (4 * j) for j, o in enumerate(src.ops))
    lib.dev_forward(int(src.counter), S, src.R, src.res, src.off, *src._arrays(), _p(src.elem), int(target), src_type,
                    ops, int(src.discard), G, grp.R, *grp._arrays(), _p(off), _p(mem), len(mem), _p(fs), _p(fv),
                    _p(fnn), _p(fp), _p(fd), _p(rec), _p(mark), _p(sst), _p(gst))
    return sst.tolist(), gst.tolist()


PIPES = [(A.METRIC_COUNTER, 7, [3], [7], [4]), (A.METRIC_GAUGE, 1, [], [2, 3, 7], []),
         (A.METRIC_GAUGE, 4, [1, 2], [1, 6, 7], [5]), (A.METRIC_COUNTER, 2, [], [2, 9], [])]


def _memberships(rng, S, G):
    """random CSR groups: duplicates, sources in several groups or none, and now and then an invalid group"""
    lens = rng.integers(0, 5, G)
    mem = rng.integers(0, S, int(lens.sum())).astype(np.uint32)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    if rng.random() < 0.3 and len(mem):
        mem[int(rng.integers(0, len(mem)))] = S + 3  # an index past the sources
    if rng.random() < 0.3 and G > 2:
        g = int(rng.integers(1, G))
        off[g] = off[g + 1] + 1 if off[g + 1] + 1 <= off[-1] else off[g]  # a decreasing range
    return off, mem


@pytest.mark.parametrize("pipe", range(len(PIPES)))
def test_random_sequences_equal_the_model(dev, pipe):
    metric, src_type, pre, types, post = PIPES[pipe]
    counter = metric == A.METRIC_COUNTER
    rng = np.random.default_rng(71 + pipe)
    seen, retried = set(), 0
    for it in range(25):
        S, G, R, RG = 14, 6, int(rng.integers(2, 5)), int(rng.integers(1, 4))
        res = int(rng.choice([10, 60])) * SEC
        discard = bool(it % 2)
        src = DevSet(dev, S, R, metric, [src_type], res, pre, discard)
        grp = DevSet(dev, G, RG, metric, types, res, post, discard)
        sms = [SourceModel(metric, src_type, res, pre, discard, open_windows=R) for _ in range(S)]
        gms = [GroupModel(metric, types, res, post, discard, open_windows=RG) for _ in range(G)]
        off, mem = _memberships(rng, S, G)
        clock = int(rng.integers(-5, 5)) * res
        for step in range(8):
            cols = [[(clock + int(rng.integers(-3 * res, res)) // SEC * SEC, _bits(_value(rng, counter)))
                     for _ in range(int(rng.integers(0, 4)))] for _ in range(S)]
            got_r, got_s = src.add(cols)
            for s, m in enumerate(sms):
                assert (got_r[s], got_s[s]) == m.add(cols[s]), (it, step, s)
            clock += int(rng.integers(0, 2)) * res
            if rng.random() < 0.7:
                target = clock - int(rng.integers(0, 2)) * res
                sst, gst = dev_forward(dev, src, grp, src_type, target, off, mem)
                wst, wgst = forward(sms, gms, target, off, mem)
                assert (sst, gst) == (wst, wgst), (it, step)
                seen.update(gst)
                failed = [g for g in range(G) if gst[g] == ERR_CAPACITY]
                if failed and rng.random() < 0.7:
                    # grow the group set and re-run exactly the failed groups (the others' ranges empty)
                    grp_big = DevSet(dev, G, RG + 4, metric, types, res, post, discard)
                    for f in grp.w:
                        grp_big.w[f][:RG] = grp.w[f]
                    grp_big.wm[:], grp_big.elem[:] = grp.wm, grp.elem
                    grp, RG = grp_big, RG + 4
                    for m in gms:
                        m.R = RG
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
                if rng.random() < 0.7:
                    out, st = grp.consume(target)
                    assert st == [OK] * G
                    for g, m in enumerate(gms):
                        want = m.consume(target)
                        for j in range(len(types)):
                            assert np.array_equal(out[g][j][0], want[j][0]), (it, step, g, j)
                            assert np.array_equal(out[g][j][1].view(np.uint64), want[j][1].view(np.uint64)), \
                                (it, step, g, j)
                        assert grp.elem[g].tobytes() == m.state.tobytes()
                        assert grp.wm[g] == m.watermark
    assert seen == {OK, ERR_CLOSED, ERR_CAPACITY, ERR_INVALID_ARG} and retried > 0
