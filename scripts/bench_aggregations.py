#!/usr/bin/env python3
"""Times the fused decode + downsample modes and the tile aggregation per metric type at the bench shape.

  500 k series x 1440 datapoints (int-optimised Gaussian walk, the bench.py batch), 5-minute windows (288), plus a
  counter-shaped batch of the same size: monotone integer counters that reset now and then, and in every 1000th
  series a few values (3e18, 4e9) that make the int64 sum / sumSq wrap.

Downsample: Gauge (sum/count/min/max), Gauge + last, Gauge + last + sumSq (expensive aggregations), Counter --
alternating, one call each per round.  Tiles: Gauge Last, Gauge Stdev, Counter Sum.  Each call is timed with CUDA
events; the median over the rounds is reported with G datapoints/s and the algorithmic GB/s: the stream bytes read
plus the window arrays written (8 bytes per window, series and array), counted from the shapes; for tiles also the
window arrays read back by the re-encode and the packed bytes written.  Prints the card, its power limit and SM
clocks, read in the same run, and checks a seeded sample of every output against the CPU oracle.

    python scripts/bench_aggregations.py [--series 500000] [--points 1440] [--rounds 10] [--sample 48]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import agg_oracle_lib as A  # noqa: E402
import oracle_lib as O  # noqa: E402
from m3_b200 import capi, synth  # noqa: E402
from m3_b200.codec import BatchCodec  # noqa: E402

SEC = 1_000_000_000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def counter_batch(S, P, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    incr = torch.randint(0, 50, (S, P), device="cuda", generator=g, dtype=torch.int64)
    period = torch.randint(20_000, 1_000_000, (S, 1), device="cuda", generator=g, dtype=torch.int64)
    vals = (torch.cumsum(incr, dim=1) % period).to(torch.float64)  # monotone, reset at every wrap of `period`
    big = torch.arange(0, S, 1000, device="cuda")
    vals[big, 100:104] = 3.0e18   # the int64 sum wraps
    vals[big, 700:702] = 4.0e9    # x*x wraps
    return vals


def timed(fn, n_rounds, names):
    ms = {k: [] for k in names}
    for _ in range(n_rounds):
        for k in names:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn(k)
            b.record()
            b.synchronize()
            ms[k].append(a.elapsed_time(b))
    return {k: float(np.median(v)) for k, v in ms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=500_000)
    ap.add_argument("--points", type=int, default=1440)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--sample", type=int, default=48)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_aggregations.py needs a CUDA device")
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
        batches[name] = (packed, off, int(off[-1].item()))
    del gvals, cvals
    del ts
    torch.cuda.empty_cache()

    gp, go, gbytes = batches["gauge"]
    cp, co, cbytes = batches["counter"]
    outs = {}
    ds = {
        "gauge (mode 1)": lambda o: codec.decode_downsample(gp, go, s0, step, W, out=o),
        "gauge+last (mode 2)": lambda o: codec.decode_downsample(gp, go, s0, step, W, out=o, want_last=True),
        "gauge+last+sumSq (mode 4)": lambda o: codec.decode_downsample(gp, go, s0, step, W, out=o, want_sum_sq=True),
        "counter (mode 5)": lambda o: codec.decode_downsample(cp, co, s0, step, W, out=o,
                                                              metric=capi.METRIC_COUNTER),
    }
    arrays = {"gauge (mode 1)": 4, "gauge+last (mode 2)": 6, "gauge+last+sumSq (mode 4)": 7, "counter (mode 5)": 5}
    for k, f in ds.items():  # allocate + warm up
        outs[k] = f(None)
        f(outs[k])
    torch.cuda.synchronize()
    t_ds = timed(lambda k: ds[k](outs[k]), a.rounds, list(ds))

    tiles = {
        "tiles gauge Last": (gp, go, capi.METRIC_GAUGE, capi.AGG_LAST),
        "tiles gauge Stdev": (gp, go, capi.METRIC_GAUGE, capi.AGG_STDEV),
        "tiles counter Sum": (cp, co, capi.METRIC_COUNTER, capi.AGG_SUM),
    }
    t_out = {}
    for k, (p_, o_, m, agg) in tiles.items():
        t_out[k] = codec.aggregate_tiles(p_, o_, s0, step, W, agg_type=agg, metric_type=m)
        codec.aggregate_tiles(p_, o_, s0, step, W, agg_type=agg, metric_type=m, out=t_out[k][0])
    torch.cuda.synchronize()

    def run_tile(k):
        p_, o_, m, agg = tiles[k]
        res, n_t = codec.aggregate_tiles(p_, o_, s0, step, W, agg_type=agg, metric_type=m, out=t_out[k][0])
        t_out[k] = (res, n_t)
    t_tl = timed(run_tile, a.rounds, list(tiles))

    res = {"card": info, "series": S, "points": P, "windows": W, "rounds": a.rounds, "results": {}}
    dp = S * P
    for k, ms in t_ds.items():
        nbytes = (cbytes if k.startswith("counter") else gbytes) + arrays[k] * W * S * 8
        res["results"][k] = {"ms": ms, "G_dp_per_s": dp / ms / 1e6, "alg_GB_per_s": nbytes / ms / 1e6}
    for k, ms in t_tl.items():
        sb = cbytes if "counter" in k else gbytes
        na = 5 if "counter" in k else (7 if "Stdev" in k else 6)
        out_b = int(t_out[k][0].total.item())
        nbytes = sb + 2 * na * W * S * 8 + out_b
        res["results"][k] = {"ms": ms, "G_dp_per_s": dp / ms / 1e6, "alg_GB_per_s": nbytes / ms / 1e6,
                             "packed_bytes": out_b}
    for k, r in res["results"].items():
        print("%-28s %8.3f ms  %6.2f G dp/s  %7.1f GB/s (algorithmic)" % (k, r["ms"], r["G_dp_per_s"],
                                                                        r["alg_GB_per_s"]))

    # ---- a seeded sample of every output against the oracle ----
    rng = np.random.default_rng(1234)
    sample = np.unique(np.concatenate([rng.integers(0, S, a.sample), np.arange(0, S, 1000)[:8]]))
    bad = 0
    host = {}
    for name, (p_, o_, _) in batches.items():
        ho = o_.cpu().numpy()
        hp = p_[: int(ho[-1])].cpu().numpy()
        host[name] = [O.decode_series(hp[ho[s]: ho[s + 1]].tobytes(), True, cap=P + 1) for s in sample]
    t_idx = torch.from_numpy(sample).cuda()
    col = lambda x: None if x is None else x[:, t_idx].cpu().numpy()  # [W, len(sample)]
    h = {k: [col(x) for x in (o.sum, o.count, o.min, o.max, o.last, o.sum_sq)] for k, o in outs.items()}
    for i, s in enumerate(sample):
        gts, gv, gn, gerr = host["gauge"][i]
        cts, cv, cn, cerr = host["counter"][i]
        bad += int(gerr != 0 or cerr != 0)
        eg = A.downsample_gauge_ex(gts, gv, s0, step, W)
        ec = A.downsample_counter(cts, cv, s0, step, W)
        for k, arr in h.items():
            if k.startswith("counter"):
                exp = [ec[0], ec[1], ec[2], ec[3], None, ec[4]]
            else:
                exp = [eg[0], eg[1], eg[2], eg[3], eg[4], eg[6]]
            for got, e in zip(arr, exp):
                if got is not None and e is not None:
                    bad += int(not (got[:, i].view(np.uint64) == np.asarray(e).view(np.uint64)).all())
        for k, (p_, o_, m, agg) in tiles.items():
            src = host["counter" if m == capi.METRIC_COUNTER else "gauge"][i]
            tts, tv = A.aggregate_tiles_series_ex(src[0], src[1], s0, step, W, m, agg)
            exp = O.encode_series(tts, tv, s0, O.UNIT_S, True) if len(tts) else b""
            r, _ = t_out[k]
            a0, ln = int(r.offsets[s].item()), int(r.out_len[s].item())
            bad += int(r.packed[a0: a0 + ln].cpu().numpy().tobytes() != exp or int(r.status[s].item()) != 0)
    res["sampled_series"] = int(len(sample))
    res["sample_mismatches"] = bad
    print("oracle check on %d sampled series x every output: %s" %
          (len(sample), "all sampled outputs equal the oracle" if bad == 0 else "%d MISMATCHES" % bad))
    print(json.dumps(res))
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
