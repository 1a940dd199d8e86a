#!/usr/bin/env python3
"""Times tile aggregation with and without the aggregator's transformations at the bench shape.

  500 k series x 1440 datapoints, 5-minute windows (288): the counter-shaped batch of bench_aggregations.py
  (monotone integer counters that reset now and then) and its int-optimised Gaussian-walk batch.

Alternating within every round: tiles Counter Sum against Counter Sum + PerSecond (the rate series) and against
Counter Sum + Absolute (the counters' sums are >= 0, so the same bytes: the cost of the transformation stage
itself), and tiles Gauge Last against Gauge Last + Reset (twice the datapoints written).  A transformed call
includes zeroing its 48 MB of state (every round starts new elements).  Each call is timed with CUDA events;
the median over the rounds is reported with the packed bytes written.  Prints the card, its power limit and SM
clocks, read in the same run, and checks a seeded sample of every output (bytes and saved state) against the CPU
oracle.

    python scripts/bench_transforms.py [--series 500000] [--points 1440] [--rounds 10] [--sample 48]
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

import agg_oracle_lib as A  # noqa: E402
import oracle_lib as O  # noqa: E402
import xf_oracle_lib as X  # noqa: E402
from bench_aggregations import card, counter_batch, timed  # noqa: E402
from m3_b200 import capi, synth  # noqa: E402
from m3_b200.codec import BatchCodec  # noqa: E402

SEC = 1_000_000_000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=500_000)
    ap.add_argument("--points", type=int, default=1440)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--sample", type=int, default=48)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_transforms.py needs a CUDA device")
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

    runs = {
        "tiles counter Sum": ("counter", capi.METRIC_COUNTER, capi.AGG_SUM, ()),
        "tiles counter Sum + PerSecond": ("counter", capi.METRIC_COUNTER, capi.AGG_SUM, (capi.TRANSFORM_PERSECOND,)),
        # the counters' sums are >= 0: the same bytes as Sum alone, so this row is the transformation stage's cost
        "tiles counter Sum + Absolute": ("counter", capi.METRIC_COUNTER, capi.AGG_SUM, (capi.TRANSFORM_ABSOLUTE,)),
        "tiles gauge Last": ("gauge", capi.METRIC_GAUGE, capi.AGG_LAST, ()),
        "tiles gauge Last + Reset": ("gauge", capi.METRIC_GAUGE, capi.AGG_LAST, (capi.TRANSFORM_RESET,)),
    }
    outs, states = {}, {}

    def run(k, out=None):
        b, m, agg, ops = runs[k]
        p_, o_ = batches[b]
        if ops:
            states[k].zero_()  # every round the same call: a new element
        return codec.aggregate_tiles(p_, o_, s0, step, W, agg_type=agg, metric_type=m, transforms=ops,
                                     state=states.get(k), out=out)

    for k in runs:
        if runs[k][3]:
            states[k] = codec.transform_state(S)
        outs[k] = run(k)
        outs[k] = run(k, outs[k][0])
    torch.cuda.synchronize()

    def step_fn(k):
        outs[k] = run(k, outs[k][0])
    t = timed(step_fn, a.rounds, list(runs))

    res = {"card": info, "series": S, "points": P, "windows": W, "rounds": a.rounds, "results": {}}
    for k, ms in t.items():
        out_b = int(outs[k][0].total.item())
        res["results"][k] = {"ms": ms, "G_dp_per_s": S * P / ms / 1e6, "packed_bytes": out_b,
                             "datapoints_written": int(outs[k][1].sum().item())}
        print("%-32s %8.3f ms  %6.2f G dp/s  %12d packed bytes" % (k, ms, S * P / ms / 1e6, out_b))

    # ---- a seeded sample of every output against the oracle ----
    rng = np.random.default_rng(1234)
    sample = np.unique(rng.integers(0, S, a.sample))
    bad = 0
    host = {}
    for name, (p_, o_) in batches.items():
        ho = o_.cpu().numpy()
        hp = p_[: int(ho[-1])].cpu().numpy()
        host[name] = [O.decode_series(hp[ho[s]: ho[s + 1]].tobytes(), True, cap=P + 1) for s in sample]
    for k, (b, m, agg, ops) in runs.items():
        r, nt = outs[k]
        st = states[k].cpu().numpy().view(X.XF_STATE_DTYPE).reshape(-1) if ops else None
        for i, s in enumerate(sample):
            src = host[b][i]
            bad += int(src[3] != 0)
            est = X.new_transform_state()
            tts, tv = X.aggregate_tiles_transform_series(src[0][:src[2]], src[1][:src[2]], s0, step, W, m, agg,
                                                         list(ops), True, est)
            exp = O.encode_series(tts, tv, s0, O.UNIT_S, True) if len(tts) else b""
            a0, ln = int(r.offsets[s].item()), int(r.out_len[s].item())
            bad += int(r.packed[a0: a0 + ln].cpu().numpy().tobytes() != exp or int(r.status[s].item()) != 0)
            bad += int(int(nt[s].item()) != len(tts))
            if st is not None:
                bad += int(st[s: s + 1].tobytes() != est.tobytes())
    res["sampled_series"] = int(len(sample))
    res["sample_mismatches"] = bad
    print("oracle check on %d sampled series x every output: %s" %
          (len(sample), "all sampled outputs equal the oracle" if bad == 0 else "%d MISMATCHES" % bad))
    print(json.dumps(res))
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
