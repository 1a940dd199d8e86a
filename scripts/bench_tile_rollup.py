#!/usr/bin/env python3
"""Times tile aggregation through a rollup (m3tsz_aggregate_tiles_rollup) against the calls around it.

  500 k sources x 1440 datapoints, 5-minute windows (288).  Workloads:
    counter: the counter-shaped batch of bench_aggregations.py through the documented Prometheus pipeline
             Sum + [Increase] -> Rollup [Sum] -> [Add];
    gauge:   the int-optimised Gaussian-walk batch through Last -> Rollup [Min, Max, Sum].
  Memberships:
    contiguous: 5 000 groups of 100 contiguous members;
    random:     50 000 groups of 10 random members; a random half of the sources is in 2 groups each, the other
                half in none (500 k memberships).

Alternating within every round: (a) the rollup call; (b) the same sources through aggregate_tiles_transform with the
same pre-ops (aggregate_tiles without them): the same decode, S rows encoded instead of k x G; (d) the fused decode
alone (decode_downsample_ex, the same mode), so that (a) - (d) is the share of the forward stage, the fold and the
group element.  Calls with records zero them in the timed region (every round starts new elements).  Each call is
timed with CUDA events; the median over the rounds is reported, with the algorithmic bytes of the forward array and
the fold.  Prints the card, its power limit and SM clocks, read in the same run, and checks a seeded sample of groups
(rows, tile counts, statuses and group records) against the composed oracle.

    python scripts/bench_tile_rollup.py [--series 500000] [--points 1440] [--rounds 10] [--sample 6]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import elem_oracle_lib as E  # noqa: E402
import rollup_oracle_lib as R  # noqa: E402
import xf_oracle_lib as X  # noqa: E402
from bench_aggregations import card, counter_batch, timed  # noqa: E402
from m3_b200 import capi, synth  # noqa: E402
from m3_b200.codec import BatchCodec  # noqa: E402

SEC = 1_000_000_000


def memberships(S, seed):
    rng = np.random.default_rng(seed)
    out = {}
    g = 5_000
    out["contiguous"] = (np.arange(0, S + 1, S // g, dtype=np.int64)[: g + 1], np.arange(S, dtype=np.int32))
    half = rng.permutation(S)[: S // 2]
    mem = np.concatenate([rng.permutation(half), rng.permutation(half)]).astype(np.int32)
    g = len(mem) // 10
    out["random"] = (np.arange(0, g * 10 + 1, 10, dtype=np.int64), mem[: g * 10])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=500_000)
    ap.add_argument("--points", type=int, default=1440)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--sample", type=int, default=6)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_tile_rollup.py needs a CUDA device")
    S, P, W, step = a.series, a.points, 288, 300 * SEC
    info = card()
    print("card (name, power limit, max SM clock, SM clock):", info)
    codec = BatchCodec(0, int_optimized=True)
    ts, gvals, start = synth.gaussian_walk(S, P, "cuda", seed=42)
    cvals = counter_batch(S, P, 43)
    s0 = int(start[0].item())
    batches = {}
    for name, vals in (("gauge", gvals), ("counter", cvals)):
        enc = codec.encode(ts, vals, start, unit=capi.UNIT_S)
        assert int((enc.status != 0).sum()) == 0
        packed, off = codec.compact(enc, align=16)
        del enc
        batches[name] = (packed, off)
    del gvals, cvals, ts
    torch.cuda.empty_cache()

    GA, CO = capi.METRIC_GAUGE, capi.METRIC_COUNTER
    INC, ADD = capi.TRANSFORM_INCREASE, capi.TRANSFORM_ADD
    LAST, MIN, MAX, SUM = capi.AGG_LAST, capi.AGG_MIN, capi.AGG_MAX, capi.AGG_SUM
    # name: (batch, metric, source type, pre-ops, rollup types, post-ops)
    workloads = {
        "counter Sum+[Increase] -> Rollup[Sum] -> [Add]": ("counter", CO, SUM, [INC], [SUM], [ADD]),
        "gauge Last -> Rollup[Min, Max, Sum]": ("gauge", GA, LAST, [], [MIN, MAX, SUM], []),
    }
    mships = {k: (torch.from_numpy(o).cuda(), torch.from_numpy(m).cuda(), o, m)
              for k, (o, m) in memberships(S, 7).items()}
    xs = codec.transform_state(S)
    words = (W + 31) // 32
    t, results, checks = {}, {}, {}
    rng = np.random.default_rng(1234)
    for wname, (b, metric, src, pre, types, post) in workloads.items():
        p_, o_ = batches[b]
        for mname, (d_off, d_mem, h_off, h_mem) in mships.items():
            G, n_mem = len(h_off) - 1, len(h_mem)
            gs = codec.element_state(G)
            keys = ["(a) rollup", "(b) tiles_transform", "(d) decode only"]
            keys = ["%s | %s | %s" % (wname, mname, k) for k in keys]
            out = {}

            def rollup():
                xs.zero_()
                gs.zero_()
                out.pop("a", None)
                out["a"] = codec.aggregate_tiles_rollup(p_, o_, s0, step, W, src, d_off, d_mem, types,
                                                        metric_type=metric, pre_transforms=pre, post_transforms=post,
                                                        src_state=xs, group_state=gs)

            def transform():
                out.pop("b", None)
                if pre:
                    xs.zero_()
                    out["b"] = codec.aggregate_tiles(p_, o_, s0, step, W, agg_type=src, metric_type=metric,
                                                     transforms=pre, state=xs)
                else:
                    out["b"] = codec.aggregate_tiles(p_, o_, s0, step, W, agg_type=src, metric_type=metric)

            def decode_only():
                out.pop("d", None)
                out["d"] = codec.decode_downsample(p_, o_, s0, step, W, want_last=metric == GA, metric=metric)

            fns = dict(zip(keys, (rollup, transform, decode_only)))
            for k in keys:
                fns[k]()
                fns[k]()
            torch.cuda.synchronize()
            t.update(timed(lambda k: fns[k](), a.rounds, keys))
            fns[keys[0]]()
            torch.cuda.synchronize()
            # the stages' algorithmic bytes: the forward stage writes S x W values and presence words; the fold reads
            # every membership's row and presence words and writes the groups' five window aggregates
            fwd_bytes = S * W * 8 + S * words * 4
            fold_bytes = n_mem * (W * 8 + words * 4) + G * W * 8 * 5 + (G + 1) * 8 + n_mem * 4
            results["%s | %s" % (wname, mname)] = {"fwd_array_bytes": fwd_bytes, "fold_bytes": fold_bytes,
                                                   "groups": G, "memberships": n_mem}
            # a seeded sample of groups against the composed oracle
            r, nt, sst = out["a"]
            sample = sorted(rng.choice(G, a.sample, replace=False).tolist())
            srcs = sorted({int(m) for g in sample for m in h_mem[h_off[g]: h_off[g + 1]]})
            idx = {s: i for i, s in enumerate(srcs)}
            sub_mem = np.array([idx[int(m)] for g in sample for m in h_mem[h_off[g]: h_off[g + 1]]], dtype=np.int32)
            sub_off = np.zeros(len(sample) + 1, dtype=np.int64)
            sub_off[1:] = np.cumsum([h_off[g + 1] - h_off[g] for g in sample])
            ho = o_.cpu().numpy()
            hp = p_[: int(ho[-1])].cpu().numpy()
            dec = R.decode_sources([hp[ho[s]: ho[s + 1]].tobytes() for s in srcs], True, False)
            es, eg = np.zeros(len(srcs), X.XF_STATE_DTYPE), np.zeros(len(sample), E.ELEM_STATE_DTYPE)
            rows, src_st = R.aggregate_tiles_rollup(dec, True, s0, step, W, metric, src, pre, sub_off, sub_mem, types,
                                                    post, True, es, eg)
            of, ln, st = r.offsets.cpu().numpy(), r.out_len.cpu().numpy(), r.status.cpu().numpy()
            ntc, gsh = nt.cpu().numpy(), gs.cpu().numpy().copy().view(E.ELEM_STATE_DTYPE).reshape(-1)
            bad = 0
            for i, g in enumerate(sample):
                for j in range(len(types)):
                    e_st, e_b, e_n = rows[j][i]
                    got = r.packed[int(of[j, g]): int(of[j, g]) + int(ln[j, g])].cpu().numpy().tobytes()
                    bad += int(st[j, g] != e_st or ntc[j, g] != e_n or got != e_b)
                bad += int(gsh[g].tobytes() != eg[i].tobytes())
            bad += int(sst.cpu().numpy()[srcs].tolist() != src_st)
            checks["%s | %s" % (wname, mname)] = bad
            out.clear()
            del gs
            torch.cuda.empty_cache()

    res = {"card": info, "series": S, "points": P, "windows": W, "rounds": a.rounds, "results": {}}
    for key, ms in t.items():
        res["results"][key] = {"ms": ms}
        print("%-80s %8.3f ms" % (key, ms))
    for key, v in results.items():
        a_ms, d_ms = t[key + " | (a) rollup"], t[key + " | (d) decode only"]
        v["rollup_stages_ms"] = a_ms - d_ms
        res["results"][key] = v
        print("%-80s (a)-(d) %7.3f ms, forward array %.1f MB, fold %.1f MB, sample mismatches %d" %
              (key, a_ms - d_ms, v["fwd_array_bytes"] / 1e6, v["fold_bytes"] / 1e6, checks[key]))
    res["sample_mismatches"] = checks
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)
    if any(checks.values()):
        sys.exit("sampled outputs differ from the oracle")


if __name__ == "__main__":
    main()
