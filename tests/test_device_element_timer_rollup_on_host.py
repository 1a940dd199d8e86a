"""The Timer element rollup's device steps compiled for the host from the .cu source text (tests/host_build.py): the
forward lane (`elem_timer_forward_lane`: the due windows in start order, each stream flushed and its header written
back, ValueOf of the source type through xf_window, the source-side NaN discard), the group fold
(`elem_timer_fold_group`: the range and index checks, the slot and sample-capacity counts, one Timer.Add per value in
listed order, closed group windows) and the plain rollup's commit lane (`elem_commit_lane`).  The source set is fed by
the Timer add lane and the group set consumed by the Timer consume lane, as in
tests/test_device_element_timer_on_host.py.  A driver runs the steps the way the kernels do; statuses, group rows,
records and watermarks must equal the CPU model (tests/element_timer_rollup_model.py) bit for bit on random sequences:
both CAPACITY stops followed by grow and re-runs of exactly the failed groups, closed and invalid groups, NaN with and
without discard_nan, members listed twice, several due windows per source, group windows open across forwards, and
held-back sources forwarding the same bits again.  A CPU regression harness; nothing of it ships."""
import ctypes as C

import numpy as np
import pytest

from element_timer_rollup_model import (ERR_CAPACITY, ERR_CLOSED, ERR_INVALID_ARG, OK, TimerGroupModel,
                                        TimerSourceModel, forward)
from host_build import compile, constants, cut, fn, source_text
from test_device_element_timer_on_host import DRIVER as TIMER_DRIVER
from test_device_element_timer_on_host import PRE, RES, SEC, DevTimerSet, _check, _p, _rows

DRIVER = TIMER_DRIVER + r"""
extern "C" size_t params_size() { return sizeof(ElementTimerParams); }
extern "C" void make_params(ARGS, m3tsz_element_state *elem, uint32_t ops, ElementTimerParams *out) {
  *out = params(PASS);
  out->e.elem = elem;
  out->e.ops = ops;
}
extern "C" void dev_forward(const ElementTimerParams *sp, const ElementTimerParams *gp, int64_t target, int discard,
                            const uint64_t *group_off, const uint32_t *members, uint64_t n_members, int64_t *fs,
                            double *fv, uint32_t *fnn, uint64_t *fp, uint64_t *fd, m3tsz_transform_state *rec,
                            int32_t *mark, int32_t *src_status, int32_t *group_status) {
  ElementRollupParams p;
  memset(&p, 0, sizeof(p));
  p.src = sp->e;
  p.src.target = target;
  p.discard_nan = discard;
  p.fwd_start = fs; p.fwd_val = fv; p.fwd_n = fnn; p.fwd_present = fp; p.fwd_due = fd; p.rec = rec;
  p.group_off = group_off; p.members = members; p.n_members = n_members; p.n_groups = gp->e.n;
  p.g_slots = gp->e.n_slots; p.g_start = gp->e.start; p.g_count = gp->e.count; p.g_sum = gp->e.sum;
  p.g_sum_sq = gp->e.sum_sq; p.g_watermark = gp->e.watermark;
  p.group_status = group_status; p.mark = mark; p.src_status = src_status;
  ElementTimerParams s = *sp;
  s.e = p.src;
  for (uint64_t i = 0; i < p.src.n; i++) elem_timer_forward_lane(p, s, i);
  for (uint64_t i = 0; i < p.src.n; i++) mark[i] = 0;
  for (uint64_t g = 0; g < p.n_groups; g++) {
    int64_t fresh[M3TSZ_MAX_ELEMENT_WINDOWS];
    uint32_t n_add[2 * M3TSZ_MAX_ELEMENT_WINDOWS];
    auto member = [&](uint64_t i) { return fwd_member(p, i); };
    const int32_t st = elem_timer_fold_group(p, *gp, g, fresh, n_add, member);
    const uint64_t lo = group_off[g], hi = group_off[g + 1];
    if ((st == M3TSZ_ERR_CAPACITY || st == M3TSZ_ERR_INVALID_ARG) && lo <= hi)  // (the kernel's atomicMax)
      for (uint64_t i = lo; i < (hi < n_members ? hi : n_members); i++)
        if (members[i] < p.src.n && mark[members[i]] < st) mark[members[i]] = st;
  }
  for (uint64_t i = 0; i < p.src.n; i++) elem_commit_lane(p, i);
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
                 "elem_window_start", "elem_ends_by"):
        parts.append(cut(enc, fn(name)))
    parts.append(cut(enc, r"struct CmStream\b"))
    for name in ("timer_stream", "amd64_op", "timer_stdev", "timer_type_quantile", "timer_value_of", "elem_timer_add_lane",
                 "elem_timer_consume_lane"):
        parts.append(cut(enc, fn(name)))
    parts.append(cut(enc, r"struct FwdMember\b"))
    for name in ("fwd_member", "elem_commit_lane", "elem_timer_forward_lane", "elem_timer_fold_group"):
        parts.append(cut(enc, fn(name)))
    lib = compile("dev_elem_timer_rollup_host", "\n".join(parts), DRIVER)
    vp, i64, u64, u32, i32 = C.c_void_p, C.c_int64, C.c_uint64, C.c_uint32, C.c_int32
    head = [u64, u32, i64, i64] + [vp] * 5 + [vp] * 8 + [u32, i32, C.c_double, vp, u32, vp, u32]
    lib.dev_add.restype = None
    lib.dev_add.argtypes = head + [vp, vp, u64, vp, vp, vp, vp]
    lib.dev_consume.restype = None
    lib.dev_consume.argtypes = head + [vp, i64, u32, C.c_int, vp, u64, vp, vp, vp, u64, vp]
    lib.params_size.restype = C.c_size_t
    lib.make_params.restype = None
    lib.make_params.argtypes = head + [vp, u32, vp]
    lib.dev_forward.restype = None
    lib.dev_forward.argtypes = [vp, vp, i64, C.c_int, vp, vp, u64] + [vp] * 9
    return lib


def _params(lib, d):
    buf = C.create_string_buffer(lib.params_size())
    ops = sum(o << (4 * j) for j, o in enumerate(d.ops))
    lib.make_params(*d._head(), _p(d.elem), ops, buf)
    return buf


def dev_forward(lib, src, grp, target, group_off, members):
    """one forward of DevTimerSet src into DevTimerSet grp -> (source statuses, group statuses)"""
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
    sp, gp = _params(lib, src), _params(lib, grp)
    lib.dev_forward(sp, gp, int(target), int(src.discard), _p(off), _p(mem), len(mem), _p(fs), _p(fv), _p(fnn),
                    _p(fp), _p(fd), _p(rec), _p(mark), _p(sst), _p(gst))
    return sst.tolist(), gst.tolist()


# (source type, pre-ops, group types, remainder ops)
PIPES = [(20, [], [3, 14, 20], []), (3, [1], [2, 3, 4, 5, 6, 7, 8, 9, 14, 19, 20], []), (4, [2], [7, 18], [3]),
         (2, [], [6, 9, 23, 24], [])]


def _memberships(rng, S, G):
    """random CSR groups: members listed twice, sources in several groups or none, now and then an invalid group"""
    lens = rng.integers(0, 6, G)
    mem = rng.integers(0, S, int(lens.sum())).astype(np.uint32)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    if rng.random() < 0.3 and len(mem):
        mem[int(rng.integers(0, len(mem)))] = S + 3  # an index past the sources
    if rng.random() < 0.2 and G > 2:
        g = int(rng.integers(1, G))
        off[g] = off[g + 1] + 1 if off[g + 1] + 1 <= off[-1] else off[g]  # a decreasing range
    return off, mem


def _rerun_failed(lib, src, grp, gms, sms, target, off, mem, gst, G):
    """grow the group set past the stop and forward exactly the failed groups again (the others' ranges empty)"""
    failed = [g for g in range(G) if gst[g] == ERR_CAPACITY]
    grp.grow(R=grp.R + 2, cap=grp.cap * 4)
    for m in gms:
        m.R, m.cap = grp.R, grp.cap
    lens = [int(off[g + 1] - off[g]) if g in failed else 0 for g in range(G)]
    off2 = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    mem2 = np.concatenate([mem[int(off[g]): int(off[g + 1])] for g in failed] + [np.zeros(0)]).astype(np.uint32)
    got = dev_forward(lib, src, grp, target, off2, mem2)
    want = forward(sms, gms, target, off2, mem2)
    return got, want


@pytest.mark.parametrize("pipe", range(len(PIPES)))
def test_random_sequences_equal_the_model(dev, pipe):
    src_type, pre, types, post = PIPES[pipe]
    rng = np.random.default_rng(91 + pipe)
    seen, retried = set(), 0
    for it in range(14):
        S, G, R, RG = 12, 6, int(rng.integers(2, 5)), int(rng.integers(1, 4))
        cap, gcap = 64, int(rng.choice([3, 6, 64]))
        every, eps = int(rng.choice([1, 2, 3, 1024])), float(rng.choice([1e-3, 0.05]))
        discard = bool(it % 2)
        src = DevTimerSet(dev, S, R, [src_type], pre, discard, cap, every, eps)
        grp = DevTimerSet(dev, G, RG, types, post, discard, gcap, every, eps)
        sms = [TimerSourceModel(src_type, RES, pre, discard, R, cap, eps, every) for _ in range(S)]
        gms = [TimerGroupModel(types, RES, post, discard, RG, gcap, eps, every) for _ in range(G)]
        off, mem = _memberships(rng, S, G)
        pools = [[] for _ in range(S)]
        clock = 10 * RES
        for step in range(8):
            cols = [_rows(rng, clock, pools[s]) for s in range(S)]
            got_r, got_s = src.add(cols)
            for s, m in enumerate(sms):
                want = m.add([(t, v) for t, v, _ in cols[s]], [b for _, _, b in cols[s]])
                assert (got_r[s], got_s[s]) == want, (it, step, s)
            clock += int(rng.integers(0, 2)) * RES
            if rng.random() < 0.75:
                target = clock - int(rng.integers(0, 2)) * RES
                sst, gst = dev_forward(dev, src, grp, target, off, mem)
                assert (sst, gst) == forward(sms, gms, target, off, mem), (it, step)
                seen.update(gst)
                if ERR_CAPACITY in gst and rng.random() < 0.7:
                    got, want = _rerun_failed(dev, src, grp, gms, sms, target, off, mem, gst, G)
                    assert got == want, (it, step, "retry")
                    retried += 1
                for s, m in enumerate(sms):
                    assert src.elem[s].tobytes() == m.state.tobytes(), (it, step, s)
                    assert src.wm[s] == m.watermark
                if rng.random() < 0.6:
                    out, st = grp.consume(target)
                    assert st == [OK] * G
                    for g, m in enumerate(gms):
                        _check(out[g], m.consume(target))
                        assert grp.elem[g].tobytes() == m.state.tobytes()
                        assert grp.wm[g] == m.watermark
    assert seen == {OK, ERR_CLOSED, ERR_CAPACITY, ERR_INVALID_ARG} and retried > 0


def test_both_capacity_stops_then_grow(dev):
    """a group short of slots, then one short of samples: each fails whole, and grow + re-run gives the values of
    one unstopped forward"""
    types = [3, 14, 20]
    for R, cap in ((1, 64), (4, 3)):
        src = DevTimerSet(dev, 4, 4, [20], [], False, 16, 1024, 1e-3)
        grp = DevTimerSet(dev, 1, R, types, [], False, cap, 1024, 1e-3)
        sms = [TimerSourceModel(20, RES, [], False, 4, 16) for _ in range(4)]
        gms = [TimerGroupModel(types, RES, [], False, R, cap)]
        cols = [[(RES + SEC * s, float(s), 0), (2 * RES + SEC, float(-s), 0)] for s in range(4)]
        src.add(cols)
        for s, m in enumerate(sms):
            m.add([(t, v) for t, v, _ in cols[s]])
        off, mem = np.array([0, 4], dtype=np.uint64), np.arange(4, dtype=np.uint32)
        got = dev_forward(dev, src, grp, 3 * RES, off, mem)
        assert got == forward(sms, gms, 3 * RES, off, mem) == ([ERR_CAPACITY] * 4, [ERR_CAPACITY])
        got, want = _rerun_failed(dev, src, grp, gms, sms, 3 * RES, off, mem, got[1], 1)
        assert got == want == ([OK] * 4, [OK])
        out, _ = grp.consume(3 * RES)
        _check(out[0], gms[0].consume(3 * RES))
