"""The cross-shard rollup's device steps compiled for the host from the .cu source text (tests/host_build.py): the
writer's count and write passes (`fw_count_group`, `fw_write_group`, over `fw_next_start`) between the element
rollup's forward and commit lanes, and AddUnique's lane (`add_forwarded_lane`), with `struct ElementForwardedParams`
of m3tsz_kernels.h.  A driver runs the steps the way the kernels do: every source's forward, every group's count, the
exclusive scans, every group's write with its failed groups marking their members, every source's commit; and for
the add, the records' keys sorted stably (the radix sort) and one lane per element that has records.  Records,
counts, statuses, source records and watermarks, AddUnique results and statuses, and the group sets' consumed rows
must equal the CPU model (tests/element_forwarded_model.py) on random sequences over two source shards: members listed
twice, invalid groups, keys permuted, NaN with and without discard_nan, closed, duplicate, invalid and capacity
records (open windows, source ids and the writer's buffers), each capacity stop followed by a grow and a resend; and
the reference's AddUnique goldens through the lane.  A CPU regression harness; nothing of it ships."""
import ctypes as C
import json
import math
import os

import numpy as np
import pytest

import agg_oracle_lib as A
from element_forwarded_model import (ERR_CAPACITY, ERR_CLOSED, ERR_DUPLICATE_SOURCE, ERR_INVALID_ARG, OK,
                                     ForwardedGroupModel, SourceModel, add_forwarded, forward_write)
from host_build import compile, constants, cut, fn, source_text
from test_device_element_rollup_on_host import DRIVER as ROLLUP_DRIVER
from test_device_element_set_on_host import PRE, DevSet, _bits, _p, _value

SEC = 1_000_000_000

DRIVER = ROLLUP_DRIVER + r"""
#include <algorithm>
extern "C" void dev_forward_write(int counter, uint64_t n, uint32_t R, int64_t res, int64_t off, int64_t *start,
                                  int64_t *count, void *sum, void *mn, void *mx, void *sq, double *last,
                                  int64_t *last_at, int64_t *wm, m3tsz_element_state *elem, int64_t target,
                                  uint32_t type, uint32_t ops, int discard, uint64_t G, const uint64_t *group_off,
                                  const uint32_t *members, uint64_t n_members, const uint64_t *group_key,
                                  uint32_t source_id, m3tsz_forwarded_metric *out_rec, uint64_t rec_cap,
                                  double *out_val, uint64_t val_cap, uint64_t *counts, int32_t *src_status,
                                  int32_t *group_status) {
  ElementForwardedParams fp;
  memset(&fp, 0, sizeof(fp));
  ElementRollupParams &p = fp.rp;
  p.src = params(counter, n, R, res, off, start, count, sum, mn, mx, sq, last, last_at, wm);
  p.src.elem = elem; p.src.target = target; p.src.types = type; p.src.n_types = 1; p.src.ops = ops;
  p.src.tiles.metric_type = counter ? M3TSZ_METRIC_COUNTER : M3TSZ_METRIC_GAUGE;
  p.discard_nan = discard;
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
  for (uint64_t s = 0; s < n; s++) counter ? elem_forward_lane<true>(p, s) : elem_forward_lane<false>(p, s);
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
  for (uint64_t s = 0; s < n; s++) elem_commit_lane(p, s);
}
extern "C" void dev_add_forwarded(int counter, uint64_t n, uint32_t R, int64_t res, int64_t off, int64_t *start,
                                  int64_t *count, void *sum, void *mn, void *mx, void *sq, double *last,
                                  int64_t *last_at, int64_t *wm, uint32_t *bits, uint32_t bit_words,
                                  const m3tsz_forwarded_metric *recs, uint64_t n_recs, const double *vals,
                                  uint64_t n_vals, int8_t *result, int32_t *status) {
  ElementForwardedParams fp;
  memset(&fp, 0, sizeof(fp));
  ElementRollupParams &p = fp.rp;
  p.src.n = n; p.src.counter = counter; p.src.resolution = res;
  p.n_groups = n; p.g_slots = R; p.g_start = start; p.g_count = count; p.g_sum = sum; p.g_min = mn; p.g_max = mx;
  p.g_sum_sq = sq; p.g_last = last; p.g_last_at = last_at; p.g_watermark = wm;
  std::vector<uint64_t> key(n_recs + 1), idx(n_recs + 1), sk(n_recs + 1), si(n_recs + 1);
  fp.rec = recs; fp.val = vals; fp.n_recs = n_recs; fp.n_vals = n_vals;
  fp.sort_key = key.data(); fp.sort_idx = idx.data(); fp.sorted_key = sk.data(); fp.sorted_idx = si.data();
  fp.bits = bits; fp.bit_words = bit_words; fp.trunc_off = off; fp.result = result; fp.status = status;
  for (uint64_t e = 0; e < n; e++) status[e] = 0;
  for (uint64_t i = 0; i < n_recs; i++) {  // (the prep kernel)
    const uint64_t k = recs[i].key;
    key[i] = k < n ? k : n;
    idx[i] = i;
  }
  std::vector<uint64_t> order(idx.begin(), idx.begin() + n_recs);  // (the radix sort: stable on the key)
  std::stable_sort(order.begin(), order.end(), [&](uint64_t x, uint64_t y) { return key[x] < key[y]; });
  for (uint64_t j = 0; j < n_recs; j++) {
    sk[j] = key[order[j]];
    si[j] = order[j];
  }
  for (uint64_t j = 0; j < n_recs; j++)
    if (j == 0 || sk[j - 1] != sk[j]) counter ? add_forwarded_lane<true>(fp, j) : add_forwarded_lane<false>(fp, j);
}
"""

REC_DTYPE = np.dtype([("key", "<u8"), ("time_ns", "<i8"), ("value_off", "<u8"), ("n_values", "<u4"),
                      ("source_id", "<u4"), ("version", "<u4"), ("reserved", "<u4")])


@pytest.fixture(scope="module")
def dev():
    enc, com, ker = source_text("m3tsz_encode.cu"), source_text("m3tsz_common.cuh"), source_text("m3tsz_kernels.h")
    parts = [PRE + "static inline int __popcll(unsigned long long v) { return __builtin_popcountll(v); }\n",
             constants(enc, r"kXf\w*|ENC_GUARD"), cut(ker, r"struct EncodeParams\b"),
             cut(ker, r"struct ElementParams\b"), cut(ker, r"struct ElementRollupParams\b"),
             cut(ker, r"struct ElementForwardedParams\b"),
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
    for name in ("fwd_member", "elem_fold_group", "elem_commit_lane", "fw_next_start", "fw_count_group",
                 "fw_write_group", "add_forwarded_lane"):
        parts.append(cut(enc, fn(name)))
    body = "\n".join(parts)
    body = body.replace('asm volatile("mov.b64 %0, %1;" : "=l"(oi) : "l"(o));', "oi = o;")
    lib = compile("dev_elem_forwarded_host", body, DRIVER)
    vp, i64, u64, u32 = C.c_void_p, C.c_int64, C.c_uint64, C.c_uint32
    lib.dev_add.restype = None
    lib.dev_add.argtypes = [C.c_int, u64, u32, i64, i64] + [vp] * 9 + [vp, vp, u64, vp, vp, vp]
    lib.dev_consume.restype = None
    lib.dev_consume.argtypes = [C.c_int, u64, u32, i64, i64] + [vp] * 9 + [vp, i64, u32, u32, u32, C.c_int, vp, u64,
                                                                           vp, vp, vp, u64, vp]
    lib.dev_forward_write.restype = None
    lib.dev_forward_write.argtypes = ([C.c_int, u64, u32, i64, i64] + [vp] * 9 + [vp, i64, u32, u32, C.c_int, u64,
                                                                                  vp, vp, u64, vp, u32, vp, u64, vp,
                                                                                  u64, vp, vp, vp])
    lib.dev_add_forwarded.restype = None
    lib.dev_add_forwarded.argtypes = ([C.c_int, u64, u32, i64, i64] + [vp] * 9 + [vp, u32, vp, u64, vp, u64, vp, vp])
    return lib


def dev_forward_write(lib, src, src_type, target, group_off, members, source_id, keys=None, rec_cap=1 << 12,
                      val_cap=1 << 12):
    """one writer call of DevSet src -> (records [(key, time_ns, [values], source_id, version, reserved)], source
    statuses, group statuses, counts)"""
    S, G = src.N, len(group_off) - 1
    out_rec = np.zeros(max(1, rec_cap), dtype=REC_DTYPE)
    out_val = np.zeros(max(1, val_cap), dtype=np.float64)
    counts = np.zeros(4, dtype=np.uint64)
    sst = np.zeros(max(1, S), dtype=np.int32)
    gst = np.zeros(max(1, G), dtype=np.int32)
    off = np.ascontiguousarray(group_off, dtype=np.uint64)
    mem = np.ascontiguousarray(members, dtype=np.uint32) if len(members) else np.zeros(1, dtype=np.uint32)
    k = None if keys is None else np.ascontiguousarray(keys, dtype=np.uint64)
    ops = sum(o << (4 * j) for j, o in enumerate(src.ops))
    lib.dev_forward_write(int(src.counter), S, src.R, src.res, src.off, *src._arrays(), _p(src.elem), int(target),
                          src_type, ops, int(src.discard), G, _p(off), _p(mem), len(members),
                          None if k is None else _p(k), source_id, _p(out_rec), rec_cap, _p(out_val), val_cap,
                          _p(counts), _p(sst), _p(gst))
    recs = [(int(r["key"]), int(r["time_ns"]), out_val[r["value_off"]: r["value_off"] + r["n_values"]].tolist(),
             int(r["source_id"]), int(r["version"]), int(r["reserved"])) for r in out_rec[: int(counts[0])]]
    return recs, sst[:S].tolist(), gst[:G].tolist(), tuple(int(c) for c in counts)


class DevGroups(DevSet):
    """a group DevSet with its source bits [R, capacity / 32, N]"""

    def __init__(self, lib, N, R, metric, types, res, ops, discard, cap):
        super().__init__(lib, N, R, metric, types, res, ops, discard)
        self.bits = np.zeros((R, cap // 32, N), dtype=np.uint32)

    def grow(self, R, cap):
        w, bits = self.w, self.bits
        for f in w:
            b = np.zeros((R, self.N), dtype=w[f].dtype)
            b[: w[f].shape[0]] = w[f]
            w[f] = b
        self.bits = np.zeros((R, cap // 32, self.N), dtype=np.uint32)
        self.bits[: bits.shape[0], : bits.shape[1]] = bits
        self.R = R

    def add_forwarded(self, records):
        rec = np.zeros(max(1, len(records)), dtype=REC_DTYPE)
        vals = []
        for i, (key, t, vs, sid, ver, rsv) in enumerate(records):
            rec[i] = (key, t, len(vals), len(vs), sid, ver, rsv)
            vals += vs
        v = np.array(vals + [0.0], dtype=np.float64)
        result = np.zeros(max(1, len(records)), dtype=np.int8)
        st = np.zeros(self.N, dtype=np.int32)
        self.lib.dev_add_forwarded(int(self.counter), self.N, self.R, self.res, self.off, *self._arrays(),
                                   _p(self.bits), self.bits.shape[1], _p(rec), len(records), _p(v), len(vals),
                                   _p(result), _p(st))
        return result[: len(records)].tolist(), st.tolist()


def _same_values(a, b):
    return len(a) == len(b) and all(np.float64(x).tobytes() == np.float64(y).tobytes() for x, y in zip(a, b))


def _same_records(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g[:2] == w[:2] and g[3:] == w[3:] and _same_values(g[2], w[2]), (g, w)


PIPES = [(A.METRIC_COUNTER, 7, [3], [7], [4]), (A.METRIC_GAUGE, 1, [], [2, 3, 7], []),
         (A.METRIC_GAUGE, 4, [1, 2], [1, 6, 7], [5]), (A.METRIC_COUNTER, 2, [], [2, 9], [])]


def _memberships(rng, S, G):
    """random CSR groups: duplicates, sources in several groups or none, and now and then an invalid group"""
    lens = rng.integers(0, 5, G)
    mem = rng.integers(0, S, int(lens.sum())).astype(np.uint32)
    if len(mem) > 1:
        mem[1] = mem[0]
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    if rng.random() < 0.3 and len(mem):
        mem[int(rng.integers(0, len(mem)))] = S + 3  # an index past the sources
    if rng.random() < 0.3 and G > 2:
        g = int(rng.integers(1, G))
        off[g] = off[g + 1] + 1 if off[g + 1] + 1 <= off[-1] else off[g]  # a decreasing range
    return off, mem


def _noise(rng, recs, G, clock, res):
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
            out.append((int(rng.integers(0, G)), clock - 6 * res, [2.0], 3, 0, 0))
        else:
            out.append((int(rng.integers(0, G)), clock, [3.0, np.nan], 40, 0, 0))
    return out


@pytest.mark.parametrize("pipe", range(len(PIPES)))
def test_random_sequences_equal_the_model(dev, pipe):
    metric, src_type, pre, types, post = PIPES[pipe]
    counter = metric == A.METRIC_COUNTER
    rng = np.random.default_rng(171 + pipe)
    seen_w, seen_a, grown = set(), set(), 0
    for it in range(20):
        S, G, R, RG, K = 10, 6, int(rng.integers(2, 5)), int(rng.integers(1, 4)), 2
        res = int(rng.choice([10, 60])) * SEC
        discard = bool(it % 2)
        cap = 32
        srcs = [DevSet(dev, S, R, metric, [src_type], res, pre, discard) for _ in range(K)]
        sms = [[SourceModel(metric, src_type, res, pre, discard, open_windows=R) for _ in range(S)] for _ in range(K)]
        grp = DevGroups(dev, G, RG, metric, types, res, post, discard, cap)
        gms = [ForwardedGroupModel(metric, types, res, post, discard, open_windows=RG, source_capacity=cap)
               for _ in range(G)]
        memb = [_memberships(rng, S, G) for _ in range(K)]
        keys = rng.permutation(G).astype(np.uint64) if it % 3 else None
        clock = int(rng.integers(-5, 5)) * res
        for step in range(6):
            for k in range(K):
                cols = [[(clock + int(rng.integers(-3 * res, res)) // SEC * SEC, _bits(_value(rng, counter)))
                         for _ in range(int(rng.integers(0, 4)))] for _ in range(S)]
                got = srcs[k].add(cols)
                for s, m in enumerate(sms[k]):
                    assert (got[0][s], got[1][s]) == m.add(cols[s]), (it, step, k, s)
            clock += int(rng.integers(0, 2)) * res
            if rng.random() > 0.8:
                continue
            target = clock - int(rng.integers(0, 2)) * res
            batch = []
            for k in range(K):
                off, mem = memb[k]
                rc, vc = int(rng.integers(0, 12)), int(rng.integers(0, 24))
                got = dev_forward_write(dev, srcs[k], src_type, target, off, mem, k, keys, rc, vc)
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
                    got = dev_forward_write(dev, srcs[k], src_type, target, off2, mem2, k, keys)
                    want = forward_write(sms[k], target, off2, mem2, k, keys)
                    _same_records(got[0], want[0])
                    assert got[1:] == want[1:], (it, step, k, "retry")
                    batch += got[0]
                for s, m in enumerate(sms[k]):
                    assert srcs[k].elem[s].tobytes() == m.state.tobytes() and srcs[k].wm[s] == m.watermark
            batch = _noise(rng, batch, G, clock, res)
            r, st = grp.add_forwarded(batch)
            wr, wst = add_forwarded(gms, batch)
            assert (r, st) == (wr, wst), (it, step)
            seen_a.update(r)
            if ERR_CAPACITY in st:  # grow and resend exactly the refused records, or the whole batch
                grp.grow(grp.R + 4, 64)
                for m in gms:
                    m.R, m.source_capacity = grp.R, 64
                again = [b for b, x in zip(batch, r) if x == ERR_CAPACITY] if rng.random() < 0.5 else batch
                r, st = grp.add_forwarded(again)
                assert (r, st) == add_forwarded(gms, again), (it, step, "resend")
                grown += 1
            if rng.random() < 0.7:
                out, st = grp.consume(target)
                assert st == [OK] * G
                for g, m in enumerate(gms):
                    want = m.consume(target)
                    for j in range(len(types)):
                        assert np.array_equal(out[g][j][0], want[j][0]), (it, step, g, j)
                        assert np.array_equal(out[g][j][1].view(np.uint64), want[j][1].view(np.uint64)), \
                            (it, step, g, j)
                    assert grp.elem[g].tobytes() == m.state.tobytes() and grp.wm[g] == m.watermark
    assert seen_w == {OK, ERR_CAPACITY, ERR_INVALID_ARG}
    assert seen_a == {OK, ERR_CAPACITY, ERR_INVALID_ARG, ERR_CLOSED, ERR_DUPLICATE_SOURCE} and grown > 0


def test_add_unique_goldens_through_the_lane(dev):
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "m3tsz_forwarded_goldens.json")) as f:
        cases = json.load(f)["add_unique"]
    for c in cases:
        res = c["resolution_s"] * SEC
        metric = A.METRIC_COUNTER if c["metric"] == "counter" else A.METRIC_GAUGE
        grp = DevGroups(dev, 1, 4, metric, [7], res, [], False, 5696)
        for at_s, vals, sid, want_r, windows_s, window_s, want in c["steps"]:
            r, st = grp.add_forwarded([(0, at_s * SEC + res, list(vals), sid, 0, 0)])
            assert r == [OK if want_r == "ok" else ERR_DUPLICATE_SOURCE] and st == [OK], c["name"]
            live = grp.w["count"][:, 0] != 0
            assert sorted(grp.w["start"][live, 0].tolist()) == [w * SEC for w in windows_s], c["name"]
            slot = int(np.nonzero(live & (grp.w["start"][:, 0] == window_s * SEC))[0][0])
            for k, w in want.items():
                if k == "eps":
                    continue
                got = grp.w[k][slot, 0]
                if k == "sum" and "eps" in want:
                    assert math.isclose(float(got), w, rel_tol=want["eps"]), c["name"]
                else:
                    assert got == w, (c["name"], k)
