"""The Timer cross-shard rollup's device steps compiled for the host from the .cu source text (tests/host_build.py):
the writer (`elem_timer_forward_lane`, then `fw_count_group` / `fw_write_group` over `fw_next_start` and
`elem_commit_lane`) and AddUnique into a Timer group set (`add_forwarded_timer_lane`, with
`ElementRollupParams::group_slot`).  A driver runs the steps the way the kernels do: every source's forward, every
group's count, the exclusive scans, every group's write with its failed groups marking their members, every source's
commit; and for the add, the records' keys sorted stably (the radix sort) and one lane per element that has records.
Records, counts, statuses, source records and watermarks, AddUnique results and statuses, and the group sets' consumed
rows must equal the CPU model (tests/element_timer_forwarded_model.py) on random two-shard sequences, with both
capacity stops reached, then grown and resent; and the reference's TimerElem.AddUnique golden runs through the lane.
Two tests pin the lane's copies of code it shares with other lanes: its record checks give add_forwarded_lane's
results, and its Timer.Add gives the slots, streams and bytes elem_timer_fold_group folds.  A CPU regression harness;
nothing of it ships."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from element_timer_forwarded_model import (ERR_CAPACITY, ERR_CLOSED, ERR_DUPLICATE_SOURCE, ERR_INVALID_ARG, OK,
                                           TimerForwardedGroupModel, TimerSourceModel, add_forwarded_timer,
                                           forward_write)
from host_build import compile, constants, cut, fn, source_text
from test_device_element_forwarded_on_host import REC_DTYPE, _same_records
from test_device_element_timer_on_host import PRE, RES, SEC, DevTimerSet, _check, _p, _rows
from test_device_element_timer_rollup_on_host import DRIVER as ROLLUP_DRIVER
from test_device_element_timer_rollup_on_host import _params, dev_forward

DRIVER = ROLLUP_DRIVER + r"""
#include <algorithm>
#include <vector>
// the prep kernel and the radix sort: the records' element keys (n for an invalid key), stably sorted
static void sort_records(const m3tsz_forwarded_metric *recs, uint64_t n_recs, uint64_t n, std::vector<uint64_t> &sk,
                         std::vector<uint64_t> &si) {
  std::vector<uint64_t> key(n_recs + 1), order(n_recs);
  for (uint64_t i = 0; i < n_recs; i++) {
    key[i] = recs[i].key < n ? recs[i].key : n;
    order[i] = i;
  }
  std::stable_sort(order.begin(), order.end(), [&](uint64_t x, uint64_t y) { return key[x] < key[y]; });
  sk.assign(n_recs + 1, 0);
  si.assign(n_recs + 1, 0);
  for (uint64_t j = 0; j < n_recs; j++) {
    sk[j] = key[order[j]];
    si[j] = order[j];
  }
}
extern "C" void dev_forward_write_timer(const ElementTimerParams *sp, int64_t target, int discard, uint64_t G,
                                        const uint64_t *group_off, const uint32_t *members, uint64_t n_members,
                                        const uint64_t *group_key, uint32_t source_id, m3tsz_forwarded_metric *out_rec,
                                        uint64_t rec_cap, double *out_val, uint64_t val_cap, uint64_t *counts,
                                        int32_t *src_status, int32_t *group_status) {
  ElementForwardedParams fp;
  memset(&fp, 0, sizeof(fp));
  ElementRollupParams &p = fp.rp;
  p.src = sp->e;
  p.src.target = target;
  p.discard_nan = discard;
  const uint64_t n = p.src.n, R = p.src.n_slots;
  std::vector<int64_t> fs(n * R + 1);
  std::vector<double> fv(n * R + 1);
  std::vector<uint32_t> fnn(n + 1);
  std::vector<uint64_t> fpr(n + 1), fd(n + 1), nr(G + 1), nv(G + 1), ro(G + 1), vo(G + 1);
  std::vector<m3tsz_transform_state> rec(n + 1);
  std::vector<int32_t> mark(n + 1, 0);
  p.fwd_start = fs.data(); p.fwd_val = fv.data(); p.fwd_n = fnn.data(); p.fwd_present = fpr.data();
  p.fwd_due = fd.data(); p.rec = rec.data();
  p.group_off = group_off; p.members = members; p.n_members = n_members; p.n_groups = G;
  p.group_status = group_status; p.mark = mark.data(); p.src_status = src_status;
  fp.group_key = group_key; fp.source_id = source_id; fp.out_rec = out_rec; fp.out_val = out_val;
  fp.rec_cap = rec_cap; fp.val_cap = val_cap; fp.n_rec = nr.data(); fp.n_val = nv.data(); fp.rec_off = ro.data();
  fp.val_off = vo.data(); fp.counts = counts;
  ElementTimerParams s = *sp;
  s.e = p.src;
  for (uint64_t i = 0; i < n; i++) elem_timer_forward_lane(p, s, i);
  for (uint64_t g = 0; g < G; g++) fw_count_group(fp, g);
  uint64_t a = 0, b = 0;  // (the two cub exclusive scans)
  for (uint64_t g = 0; g < G; g++) {
    ro[g] = a; vo[g] = b; a += nr[g]; b += nv[g];
  }
  for (int i = 0; i < 4; i++) counts[i] = 0;
  for (uint64_t g = 0; g < G; g++) {
    const int32_t st = fw_write_group(fp, g);
    const uint64_t lo = group_off[g], hi = group_off[g + 1];
    if (st != M3TSZ_OK && lo <= hi)  // (the kernel's atomicMax)
      for (uint64_t i = lo; i < (hi < n_members ? hi : n_members); i++)
        if (members[i] < n && mark[members[i]] < st) mark[members[i]] = st;
  }
  for (uint64_t i = 0; i < n; i++) elem_commit_lane(p, i);
}
static ElementForwardedParams add_params(uint64_t n, uint32_t R, int64_t res, int64_t off, int64_t *start,
                                         int64_t *count, void *sum, void *sq, const int64_t *wm, uint32_t *bits,
                                         uint32_t bit_words, const m3tsz_forwarded_metric *recs, uint64_t n_recs,
                                         const double *vals, uint64_t n_vals, int8_t *result, int32_t *status) {
  ElementForwardedParams fp;
  memset(&fp, 0, sizeof(fp));
  ElementRollupParams &p = fp.rp;
  p.src.n = n; p.src.resolution = res;
  p.n_groups = n; p.g_slots = R; p.g_start = start; p.g_count = count; p.g_sum = sum; p.g_sum_sq = sq;
  p.g_watermark = wm;
  fp.rec = recs; fp.val = vals; fp.n_recs = n_recs; fp.n_vals = n_vals;
  fp.bits = bits; fp.bit_words = bit_words; fp.trunc_off = off; fp.result = result; fp.status = status;
  for (uint64_t e = 0; e < n; e++) status[e] = 0;
  return fp;
}
extern "C" void dev_add_forwarded_timer(const ElementTimerParams *gp, uint32_t *bits, uint32_t bit_words,
                                        const m3tsz_forwarded_metric *recs, uint64_t n_recs, const double *vals,
                                        uint64_t n_vals, int8_t *result, int32_t *status) {
  const ElementParams &e = gp->e;
  ElementForwardedParams fp = add_params(e.n, e.n_slots, e.resolution, e.trunc_off, e.start, e.count, e.sum,
                                         e.sum_sq, e.watermark, bits, bit_words, recs, n_recs, vals, n_vals, result,
                                         status);
  std::vector<uint64_t> sk, si;
  sort_records(recs, n_recs, e.n, sk, si);
  fp.sorted_key = sk.data(); fp.sorted_idx = si.data();
  for (uint64_t j = 0; j < n_recs; j++)
    if (j == 0 || sk[j - 1] != sk[j]) add_forwarded_timer_lane(fp, *gp, j);
}
// add_forwarded_lane<false> (a Gauge group set) over the same records: its results, statuses and source bits
extern "C" void dev_add_forwarded_gauge(uint64_t n, uint32_t R, int64_t res, int64_t off, int64_t *start,
                                        int64_t *count, double *sum, double *mn, double *mx, double *sq, double *last,
                                        int64_t *last_at, const int64_t *wm, uint32_t *bits, uint32_t bit_words,
                                        const m3tsz_forwarded_metric *recs, uint64_t n_recs, const double *vals,
                                        uint64_t n_vals, int8_t *result, int32_t *status) {
  ElementForwardedParams fp = add_params(n, R, res, off, start, count, sum, sq, wm, bits, bit_words, recs, n_recs,
                                         vals, n_vals, result, status);
  fp.rp.g_min = mn; fp.rp.g_max = mx; fp.rp.g_last = last; fp.rp.g_last_at = last_at;
  std::vector<uint64_t> sk, si;
  sort_records(recs, n_recs, n, sk, si);
  fp.sorted_key = sk.data(); fp.sorted_idx = si.data();
  for (uint64_t j = 0; j < n_recs; j++)
    if (j == 0 || sk[j - 1] != sk[j]) add_forwarded_lane<false>(fp, j);
}
"""


@pytest.fixture(scope="module")
def dev():
    enc, com, ker = source_text("m3tsz_encode.cu"), source_text("m3tsz_common.cuh"), source_text("m3tsz_kernels.h")
    parts = [PRE + "static inline int __popcll(unsigned long long v) { return __builtin_popcountll(v); }\n",
             constants(enc, r"kXf\w*|ENC_GUARD"), cut(ker, r"struct EncodeParams\b"),
             cut(ker, r"struct ElementParams\b"), "#define M3TSZ_MAX_TIMER_TYPES 23\n#define M3TSZ_MAX_TIMER_QUANTILES 15",
             cut(ker, r"struct ElementTimerParams\b"), cut(ker, r"struct ElementRollupParams\b"),
             cut(ker, r"struct ElementForwardedParams\b"),
             cut(enc, r"struct XfElem \{"), cut(com, fn("go_f64_to_i64")), cut(com, fn("agg_stdev"))]
    for name in ("xf_isnan", "xf_bits", "xf_per_second", "xf_increase", "xf_window", "xf_element_window",
                 "elem_window_start", "elem_ends_by"):
        parts.append(cut(enc, fn(name)))
    parts.append(cut(enc, r"struct CmStream\b"))
    for name in ("timer_stream", "amd64_op", "timer_stdev", "timer_type_quantile", "timer_value_of", "elem_timer_add_lane",
                 "elem_timer_consume_lane"):
        parts.append(cut(enc, fn(name)))
    parts += [cut(enc, r"struct RollupGaugeAcc\b"), cut(enc, r"struct RollupCounterAcc\b")]
    for name in ("rollup_gauge_init", "rollup_counter_init", "rollup_add", "rollup_gauge_add", "rollup_counter_add"):
        parts.append(cut(enc, fn(name)))
    parts += [cut(enc, r"struct ElemFoldAcc\b"), cut(enc, r"struct FwdMember\b")]
    for name in ("elem_fold_load", "elem_fold_store", "fwd_member", "elem_commit_lane", "elem_timer_forward_lane",
                 "elem_timer_fold_group", "fw_next_start", "fw_count_group", "fw_write_group", "add_forwarded_lane",
                 "add_forwarded_timer_lane"):
        parts.append(cut(enc, fn(name)))
    lib = compile("dev_elem_timer_forwarded_host", "\n".join(parts), DRIVER)
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
    lib.dev_forward_write_timer.restype = None
    lib.dev_forward_write_timer.argtypes = [vp, i64, C.c_int, u64, vp, vp, u64, vp, u32, vp, u64, vp, u64, vp, vp,
                                            vp]
    lib.dev_add_forwarded_timer.restype = None
    lib.dev_add_forwarded_timer.argtypes = [vp, vp, u32, vp, u64, vp, u64, vp, vp]
    lib.dev_add_forwarded_gauge.restype = None
    lib.dev_add_forwarded_gauge.argtypes = [u64, u32, i64, i64] + [vp] * 9 + [vp, u32, vp, u64, vp, u64, vp, vp]
    return lib


def dev_forward_write_timer(lib, src, target, group_off, members, source_id, keys=None, rec_cap=1 << 12,
                            val_cap=1 << 12):
    """one writer call of DevTimerSet src -> (records [(key, time_ns, [values], source_id, version, reserved)],
    source statuses, group statuses, counts)"""
    S, G = src.N, len(group_off) - 1
    out_rec = np.zeros(max(1, rec_cap), dtype=REC_DTYPE)
    out_val = np.zeros(max(1, val_cap), dtype=np.float64)
    counts = np.zeros(4, dtype=np.uint64)
    sst = np.zeros(max(1, S), dtype=np.int32)
    gst = np.zeros(max(1, G), dtype=np.int32)
    off = np.ascontiguousarray(group_off, dtype=np.uint64)
    mem = np.ascontiguousarray(members, dtype=np.uint32) if len(members) else np.zeros(1, dtype=np.uint32)
    k = None if keys is None else np.ascontiguousarray(keys, dtype=np.uint64)
    lib.dev_forward_write_timer(_params(lib, src), int(target), int(src.discard), G, _p(off), _p(mem), len(members),
                                None if k is None else _p(k), source_id, _p(out_rec), rec_cap, _p(out_val), val_cap,
                                _p(counts), _p(sst), _p(gst))
    recs = [(int(r["key"]), int(r["time_ns"]), out_val[r["value_off"]: r["value_off"] + r["n_values"]].tolist(),
             int(r["source_id"]), int(r["version"]), int(r["reserved"])) for r in out_rec[: int(counts[0])]]
    return recs, sst[:S].tolist(), gst[:G].tolist(), tuple(int(c) for c in counts)


def _pack(records):
    rec = np.zeros(max(1, len(records)), dtype=REC_DTYPE)
    vals = []
    for i, (key, t, vs, sid, ver, rsv) in enumerate(records):
        rec[i] = (key, t, len(vals), len(vs), sid, ver, rsv)
        vals += vs
    return rec, np.array(vals + [0.0], dtype=np.float64), len(vals)


class DevTimerGroups(DevTimerSet):
    """a Timer group DevTimerSet with its source bits [R, capacity / 32, N]"""

    def __init__(self, lib, N, R, types, ops, discard, cap, every, eps, source_capacity=64):
        super().__init__(lib, N, R, types, ops, discard, cap, every, eps)
        self.bits = np.zeros((R, source_capacity // 32, N), dtype=np.uint32)

    def grow(self, R=None, cap=None, source_capacity=None):
        super().grow(R, cap)
        bits = self.bits
        self.bits = np.zeros((self.R, (source_capacity or bits.shape[1] * 32) // 32, self.N), dtype=np.uint32)
        self.bits[: bits.shape[0], : bits.shape[1]] = bits

    def add_forwarded(self, records):
        rec, v, nv = _pack(records)
        result = np.zeros(max(1, len(records)), dtype=np.int8)
        st = np.zeros(self.N, dtype=np.int32)
        self.lib.dev_add_forwarded_timer(_params(self.lib, self), _p(self.bits), self.bits.shape[1], _p(rec),
                                         len(records), _p(v), nv, _p(result), _p(st))
        return result[: len(records)].tolist(), st.tolist()


def _models(grp, types, **k):
    return [TimerForwardedGroupModel(types, RES, grp.ops, grp.discard, grp.R, grp.cap, grp.eps, grp.every, **k)
            for _ in range(grp.N)]


# (source type, pre-ops, group types, remainder ops)
PIPES = [(20, [], [3, 14, 20], []), (3, [1], [2, 3, 4, 5, 6, 7, 8, 9, 14, 19, 20], []), (4, [2], [7, 18], [3])]


def _memberships(rng, S, G):
    """random CSR groups: members listed twice, sources in several groups or none, now and then an invalid group"""
    lens = rng.integers(0, 5, G)
    mem = rng.integers(0, S, int(lens.sum())).astype(np.uint32)
    if len(mem) > 1:
        mem[1] = mem[0]
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    if rng.random() < 0.3 and len(mem):
        mem[int(rng.integers(0, len(mem)))] = S + 3  # an index past the sources
    if rng.random() < 0.2 and G > 2:
        g = int(rng.integers(1, G))
        off[g] = off[g + 1] + 1 if off[g + 1] + 1 <= off[-1] else off[g]  # a decreasing range
    return off, mem


def _noise(rng, recs, G, clock):
    """redeliveries, invalid records, late records and source ids past a small capacity, mixed into a batch"""
    out = list(recs)
    for _ in range(int(rng.integers(0, 6))):
        kind = int(rng.integers(0, 5))
        if kind == 0 and recs:
            out.insert(int(rng.integers(0, len(out) + 1)), recs[int(rng.integers(0, len(recs)))])
        elif kind == 1:
            out.append((int(rng.integers(0, G + 2)), clock, [1.0], 1, int(rng.integers(0, 2)), 0))
        elif kind == 2:
            out.append((int(rng.integers(0, G)), clock, [], 1, 0, 0))
        elif kind == 3:
            out.append((int(rng.integers(0, G)), clock - 6 * RES, [2.0], 3, 0, 0))
        else:
            out.append((int(rng.integers(0, G)), clock, [3.0, float("nan")], 70, 0, 0))
    return out


@pytest.mark.parametrize("pipe", range(len(PIPES)))
def test_random_sequences_equal_the_model(dev, pipe):
    src_type, pre, types, post = PIPES[pipe]
    rng = np.random.default_rng(431 + pipe)
    seen_w, seen_a, stops = set(), set(), set()
    for it in range(12):
        S, G, R, RG, K = 8, 5, int(rng.integers(2, 5)), int(rng.integers(1, 4)), 2
        gcap = int(rng.choice([3, 6, 64]))
        every, eps = int(rng.choice([1, 3, 1024])), float(rng.choice([1e-3, 0.05]))
        discard = bool(it % 2)
        srcs = [DevTimerSet(dev, S, R, [src_type], pre, discard, 64, every, eps) for _ in range(K)]
        sms = [[TimerSourceModel(src_type, RES, pre, discard, R, 64, eps, every) for _ in range(S)] for _ in range(K)]
        grp = DevTimerGroups(dev, G, RG, types, post, discard, gcap, every, eps)
        gms = _models(grp, types, source_capacity=64)
        memb = [_memberships(rng, S, G) for _ in range(K)]
        keys = rng.permutation(G).astype(np.uint64) if it % 3 else None
        pools = [[[] for _ in range(S)] for _ in range(K)]
        clock = 10 * RES
        for step in range(6):
            for k in range(K):
                cols = [_rows(rng, clock, pools[k][s]) for s in range(S)]
                got_r, got_s = srcs[k].add(cols)
                for s, m in enumerate(sms[k]):
                    want = m.add([(t, v) for t, v, _ in cols[s]], [b for _, _, b in cols[s]])
                    assert (got_r[s], got_s[s]) == want, (it, step, k, s)
            clock += int(rng.integers(0, 2)) * RES
            target = clock - int(rng.integers(0, 2)) * RES
            batch = []
            for k in range(K):
                off, mem = memb[k]
                rc, vc = int(rng.integers(0, 12)), int(rng.integers(0, 24))
                got = dev_forward_write_timer(dev, srcs[k], target, off, mem, k, keys, rc, vc)
                want = forward_write(sms[k], target, off, mem, k, keys, rc, vc)
                _same_records(got[0], want[0])
                assert got[1:] == want[1:], (it, step, k)
                seen_w.update(got[2])
                batch += got[0]
                failed = [g for g in range(G) if got[2][g] == ERR_CAPACITY]
                if failed:  # the failed groups again, with room for all (the others' ranges empty)
                    lens = [int(off[g + 1] - off[g]) if g in failed else 0 for g in range(G)]
                    off2 = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
                    mem2 = np.concatenate([mem[int(off[g]): int(off[g + 1])] for g in failed]).astype(np.uint32)
                    got = dev_forward_write_timer(dev, srcs[k], target, off2, mem2, k, keys)
                    want = forward_write(sms[k], target, off2, mem2, k, keys)
                    _same_records(got[0], want[0])
                    assert got[1:] == want[1:], (it, step, k, "retry")
                    batch += got[0]
                for s, m in enumerate(sms[k]):
                    assert srcs[k].elem[s].tobytes() == m.state.tobytes() and srcs[k].wm[s] == m.watermark
            batch = _noise(rng, batch, G, clock)
            r, st = grp.add_forwarded(batch)
            assert (r, st) == add_forwarded_timer(gms, batch), (it, step)
            seen_a.update(r)
            if ERR_CAPACITY in st:  # note which limit stopped, grow both and resend the refused records or all
                for g in range(G):
                    if st[g] == ERR_CAPACITY:
                        i = next(i for i, b in enumerate(batch) if b[0] == g and r[i] == ERR_CAPACITY)
                        ws = batch[i][1] // RES * RES - RES
                        if batch[i][3] >= 64:
                            stops.add("source id")
                        elif ws in gms[g].windows:
                            stops.add("samples")
                        else:
                            stops.add("samples" if len(gms[g].windows) < gms[g].R else "windows")
                grp.grow(R=grp.R + 3, cap=grp.cap * 8, source_capacity=128)
                for m in gms:
                    m.R, m.cap, m.source_capacity = grp.R, grp.cap, 128
                again = [b for b, x in zip(batch, r) if x == ERR_CAPACITY] if rng.random() < 0.5 else batch
                r2, st2 = grp.add_forwarded(again)
                assert (r2, st2) == add_forwarded_timer(gms, again), (it, step, "resend")
            if rng.random() < 0.7:
                out, st = grp.consume(target)
                assert st == [OK] * G
                for g, m in enumerate(gms):
                    _check(out[g], m.consume(target))
                    assert grp.elem[g].tobytes() == m.state.tobytes() and grp.wm[g] == m.watermark
    assert seen_w == {OK, ERR_CAPACITY, ERR_INVALID_ARG}
    assert seen_a == {OK, ERR_CAPACITY, ERR_INVALID_ARG, ERR_CLOSED, ERR_DUPLICATE_SOURCE}
    assert {"samples", "windows"} <= stops, stops


def test_golden_through_the_lane(dev):
    """TimerElem.AddUnique's steps; the golden's 10 s windows are scaled to this harness' 60 s resolution (every time
    times 6: the same windows, as 60 s and 10 s both divide the zero time's offset)"""
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                           "m3tsz_timer_forwarded_goldens.json")) as f:
        cases = json.load(f)["add_unique"]
    for c in cases:
        assert 6 * c["resolution_s"] * SEC == RES
        grp = DevTimerGroups(dev, 1, 4, c["types"], [], False, 64, c["every"], c["eps"])
        model = _models(grp, c["types"])
        for at_s, vals, sid, want_r, windows_s, window_s, want in c["steps"]:
            rec = [(0, 6 * at_s * SEC + RES, list(vals), sid, 0, 0)]
            r, st = grp.add_forwarded(rec)
            assert (r, st) == add_forwarded_timer(model, rec)
            assert r == [OK if want_r == "ok" else ERR_DUPLICATE_SOURCE] and st == [OK], c["name"]
            live = grp.w["count"][:, 0] != 0
            assert sorted(grp.w["start"][live, 0].tolist()) == [6 * w * SEC for w in windows_s]
            slot = int(np.nonzero(live & (grp.w["start"][:, 0] == 6 * window_s * SEC))[0][0])
            if "count" in want:
                assert grp.w["count"][slot, 0] == want["count"]
            for k in ("sum", "sum_sq"):
                if k in want:
                    assert abs(grp.w[k][slot, 0] - want[k]) <= 1e-10 * abs(want[k]), k
            for sid_seen in want.get("seen", []):
                assert grp.bits[slot, sid_seen // 32, 0] >> (sid_seen % 32) & 1
        out, _ = grp.consume(6 * 300 * SEC)
        want = model[0].consume(6 * 300 * SEC)
        _check(out[0], want)
        assert out[0][c["types"].index(14)][1][0] == 12.2  # (P50 of window 210: 11.1, 12.2, 13.3, 14.4)


def test_record_checks_match_the_gauge_lane(dev):
    """the lane's copy of add_forwarded_lane's record checks and slot rule: with room for every sample, a Timer group
    set and a Gauge group set given the same records return the same results, statuses, source bits and windows"""
    rng = np.random.default_rng(5)
    G = 6
    for it in range(20):
        R, cap = int(rng.integers(1, 4)), 32 * int(rng.integers(1, 3))
        tg = DevTimerGroups(dev, G, R, [3, 14], [], False, 1 << 10, 1024, 1e-3, cap)
        w = {f: np.zeros((R, G), dtype=d) for f, d in (("start", np.int64), ("count", np.int64), ("sum", np.float64),
                                                      ("min", np.float64), ("max", np.float64),
                                                      ("sum_sq", np.float64), ("last", np.float64),
                                                      ("last_at", np.int64))}
        wm = np.full(G, -(1 << 63), dtype=np.int64)
        bits = np.zeros((R, cap // 32, G), dtype=np.uint32)
        clock = 10 * RES
        for step in range(4):
            recs = [(int(rng.integers(0, G + 1)), clock + int(rng.integers(-2, 3)) * RES,
                     [float(x) for x in rng.normal(size=int(rng.integers(0, 3)))], int(rng.integers(0, cap + 8)),
                     int(rng.random() < 0.05), 0) for _ in range(40)]
            if step == 2:
                wm[:] = clock - RES
                tg.wm[:] = wm
            rt, stt = tg.add_forwarded(recs)
            rec, v, nv = _pack(recs)
            rg = np.zeros(len(recs), dtype=np.int8)
            stg = np.zeros(G, dtype=np.int32)
            dev.dev_add_forwarded_gauge(G, R, RES, tg.off, *[_p(w[f]) for f in w], _p(wm), _p(bits), cap // 32,
                                        _p(rec), len(recs), _p(v), nv, _p(rg), _p(stg))
            assert rt == rg.tolist() and stt == stg.tolist(), (it, step)
            assert np.array_equal(tg.bits, bits)
            assert np.array_equal(tg.w["count"] != 0, w["count"] != 0)
            assert np.array_equal(np.where(w["count"] != 0, tg.w["start"], 0), np.where(w["count"] != 0, w["start"], 0))
            assert np.array_equal(tg.w["count"], w["count"])
            clock += RES


def test_timer_adds_match_the_fold(dev):
    """the lane's copy of elem_timer_fold_group's Timer.Add: two shards' records, concatenated in shard order, leave
    the group set's slots, headers and stream arrays byte for byte as one Timer forward over a single set whose groups
    list the members shard by shard"""
    rng = np.random.default_rng(9)
    S, G, K = 6, 4, 2
    types = [3, 14, 20]
    for it in range(8):
        every = int(rng.choice([1, 3, 1024]))
        srcs = [DevTimerSet(dev, S, 4, [20], [], False, 64, every, 1e-3) for _ in range(K)]
        single = DevTimerSet(dev, K * S, 4, [20], [], False, 64, every, 1e-3)
        pools = [[] for _ in range(K * S)]
        cols = [_rows(rng, 10 * RES, pools[i]) for i in range(K * S)]
        cols = [[(t, v, 0) for t, v, _ in c] for c in cols]
        for k in range(K):
            srcs[k].add(cols[k * S: (k + 1) * S])
        single.add(cols)
        memb = [_memberships(rng, S, G) for _ in range(K)]
        memb = [(off, np.minimum(mem, S - 1)) for off, mem in memb]
        lists = [[k * S + int(m) for k in range(K) for m in memb[k][1][int(memb[k][0][g]): int(memb[k][0][g + 1])]]
                 if all(memb[k][0][g] <= memb[k][0][g + 1] for k in range(K)) else [] for g in range(G)]
        off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.uint64)
        mem = np.array([m for x in lists for m in x] + [0], dtype=np.uint32)[: int(off[-1])]
        target = 12 * RES
        ga = DevTimerGroups(dev, G, 8, types, [], False, 256, every, 1e-3)
        gb = DevTimerSet(dev, G, 8, types, [], False, 256, every, 1e-3)
        batch = []
        for k in range(K):
            recs, _, gst, _ = dev_forward_write_timer(dev, srcs[k], target, memb[k][0], memb[k][1], k)
            batch += [r for r in recs if lists[r[0]]]
        r, st = ga.add_forwarded(batch)
        assert set(r) <= {OK} and st == [OK] * G
        sst, gst = dev_forward(dev, single, gb, target, off, mem)
        assert gst == [OK] * G
        for g in range(G):  # (the two may open a group's windows in other slots: matched by start)
            sa = {int(ga.w["start"][r, g]): r for r in range(ga.R) if ga.w["count"][r, g]}
            sb = {int(gb.w["start"][r, g]): r for r in range(gb.R) if gb.w["count"][r, g]}
            assert sa.keys() == sb.keys(), (it, g)
            for ws, a in sa.items():
                b = sb[ws]
                for f in ("count", "sum", "sum_sq"):
                    assert ga.w[f][a, g].tobytes() == gb.w[f][b, g].tobytes(), (it, g, f)
                assert ga.hdr[a, g].tobytes() == gb.hdr[b, g].tobytes(), (it, g)
                for f in ga.arr:
                    assert ga.arr[f][a, :, g].tobytes() == gb.arr[f][b, :, g].tobytes(), (it, g, f)
