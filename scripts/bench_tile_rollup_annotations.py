#!/usr/bin/env python3
"""Times tile aggregation through a rollup that keeps annotations (m3tsz_aggregate_tiles_rollup_annotated) against
the plain rollup (m3tsz_aggregate_tiles_rollup) on the workloads of bench_tile_rollup.py.

  500 k sources x 1440 datapoints, 5-minute windows (288).  Workloads:
    counter: Sum + [Increase] -> Rollup [Sum] -> [Add] over the counter-shaped batch;
    gauge:   Last -> Rollup [Min, Max, Sum] over the int-optimised Gaussian-walk batch;
  each with the contiguous and the random membership of bench_tile_rollup.py, on two encodings of the same values:
    annotated: the OpenMetrics counter payload on the first datapoint of every 120 (a 2-hour source block at the
               synthetic one-minute spacing), as a Prometheus-written series carries it;
    plain:     no annotation.
Within every round the annotated call and the plain call alternate; each is timed with CUDA events and the median
over the rounds is reported.  Prints the card, its power limit and SM clocks, read in the same run, and checks a
seeded sample of groups of the annotated call (rows, tile counts, statuses, group records) against the composed
oracle (tests/rollup_ann_oracle_lib.py).

    python scripts/bench_tile_rollup_annotations.py [--series 500000] [--points 1440] [--rounds 10] [--sample 6]
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
import rollup_ann_oracle_lib as RA  # noqa: E402
import xf_oracle_lib as X  # noqa: E402
from bench_aggregations import card, counter_batch, timed  # noqa: E402
from bench_tile_rollup import memberships  # noqa: E402
from m3_b200 import capi, synth  # noqa: E402
from m3_b200.codec import BatchCodec  # noqa: E402

SEC = 1_000_000_000
PAYLOAD = bytes([0x08, 0x01, 0x10, 0x01])  # annotation.Payload{COUNTER, HandleValueResets}
EVERY = 120


def block_annotations(S, P, dev):
    """(series_off, entries, bytes): PAYLOAD on datapoints 0, EVERY, 2 * EVERY, ... of every series"""
    per = (P + EVERY - 1) // EVERY
    ent = np.zeros(S * per, dtype=[("dp", "<u4"), ("len", "<u4"), ("off", "<u8")])
    ent["dp"] = np.tile(np.arange(0, P, EVERY, dtype=np.uint32), S)
    ent["len"] = len(PAYLOAD)
    off = np.arange(0, S * per + 1, per, dtype=np.int64)
    return (torch.from_numpy(off).to(dev), torch.from_numpy(ent.view(np.uint8).reshape(-1, 16).copy()).to(dev),
            torch.tensor(list(PAYLOAD), dtype=torch.uint8, device=dev))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=500_000)
    ap.add_argument("--points", type=int, default=1440)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--sample", type=int, default=6)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_tile_rollup_annotations.py needs a CUDA device")
    S, P, W, step = a.series, a.points, 288, 300 * SEC
    info = card()
    print("card (name, power limit, max SM clock, SM clock):", info)
    codec = BatchCodec(0, int_optimized=True)
    ts, gvals, start = synth.gaussian_walk(S, P, "cuda", seed=42)
    cvals = counter_batch(S, P, 43)
    s0 = int(start[0].item())
    anns = block_annotations(S, P, "cuda")
    batches = {}
    for name, vals in (("gauge", gvals), ("counter", cvals)):
        for kind, ann in (("annotated", anns), ("plain", None)):
            enc = codec.encode(ts, vals, start, unit=capi.UNIT_S, annotations=ann,
                               out_stride=codec.encode_bound(P) + 16 * ((P + EVERY - 1) // EVERY) * 8)
            assert int((enc.status != 0).sum()) == 0
            batches[(name, kind)] = codec.compact(enc, align=16)
            del enc
    del gvals, cvals, ts, anns
    torch.cuda.empty_cache()

    GA, CO = capi.METRIC_GAUGE, capi.METRIC_COUNTER
    INC, ADD = capi.TRANSFORM_INCREASE, capi.TRANSFORM_ADD
    LAST, MIN, MAX, SUM = capi.AGG_LAST, capi.AGG_MIN, capi.AGG_MAX, capi.AGG_SUM
    workloads = {
        "counter Sum+[Increase] -> Rollup[Sum] -> [Add]": ("counter", CO, SUM, [INC], [SUM], [ADD]),
        "gauge Last -> Rollup[Min, Max, Sum]": ("gauge", GA, LAST, [], [MIN, MAX, SUM], []),
    }
    mships = {k: (torch.from_numpy(o).cuda(), torch.from_numpy(m).cuda(), o, m)
              for k, (o, m) in memberships(S, 7).items()}
    xs = codec.transform_state(S)
    t, checks = {}, {}
    rng = np.random.default_rng(1234)
    for wname, (b, metric, src, pre, types, post) in workloads.items():
        for mname, (d_off, d_mem, h_off, h_mem) in mships.items():
            G = len(h_off) - 1
            gs = codec.element_state(G)
            for kind in ("annotated", "plain"):
                p_, o_ = batches[(b, kind)]
                keys = ["%s | %s | %s sources | %s" % (wname, mname, kind, c)
                        for c in ("rollup_annotated", "rollup")]
                out = {}

                def call(ann, tag):
                    def f():
                        xs.zero_()
                        gs.zero_()
                        out.pop(tag, None)
                        out[tag] = codec.aggregate_tiles_rollup(p_, o_, s0, step, W, src, d_off, d_mem, types,
                                                                metric_type=metric, pre_transforms=pre,
                                                                post_transforms=post, src_state=xs, group_state=gs,
                                                                annotations=ann)
                    return f

                fns = dict(zip(keys, (call(True, "ann"), call(False, "plain"))))
                for k in keys:
                    fns[k]()
                    fns[k]()
                torch.cuda.synchronize()
                t.update(timed(lambda k: fns[k](), a.rounds, keys))
                fns[keys[0]]()
                torch.cuda.synchronize()
                r, nt, sst = out["ann"]
                sample = sorted(rng.choice(G, a.sample, replace=False).tolist())
                srcs = sorted({int(m) for g in sample for m in h_mem[h_off[g]: h_off[g + 1]]})
                idx = {s: i for i, s in enumerate(srcs)}
                sub_mem = np.array([idx[int(m)] for g in sample for m in h_mem[h_off[g]: h_off[g + 1]]],
                                   dtype=np.int32)
                sub_off = np.zeros(len(sample) + 1, dtype=np.int64)
                sub_off[1:] = np.cumsum([h_off[g + 1] - h_off[g] for g in sample])
                ho = o_.cpu().numpy()
                hp = p_[: int(ho[-1])].cpu().numpy()
                dec = RA.decode_sources([hp[ho[s]: ho[s + 1]].tobytes() for s in srcs], True, False)
                es, eg = np.zeros(len(srcs), X.XF_STATE_DTYPE), np.zeros(len(sample), E.ELEM_STATE_DTYPE)
                rows, src_st = RA.aggregate_tiles_rollup_annotated(dec, True, s0, step, W, metric, src, pre, sub_off,
                                                                   sub_mem, types, post, True, es, eg)
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
                checks["%s | %s | %s sources" % (wname, mname, kind)] = bad
                out.clear()
            del gs
            torch.cuda.empty_cache()

    res = {"card": info, "series": S, "points": P, "windows": W, "rounds": a.rounds, "results": {}}
    for key, ms in t.items():
        res["results"][key] = {"ms": ms}
        print("%-100s %8.3f ms" % (key, ms))
    for key, bad in checks.items():
        ratio = t[key + " | rollup_annotated"] / t[key + " | rollup"]
        res["results"][key] = {"ratio": ratio, "sample_mismatches": bad}
        print("%-100s annotated / plain call %.3f, sample mismatches %d" % (key, ratio, bad))
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)
    if any(checks.values()):
        sys.exit("sampled outputs differ from the oracle")


if __name__ == "__main__":
    main()
