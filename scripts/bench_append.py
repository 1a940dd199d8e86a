#!/usr/bin/env python3
"""Encoder-set append timings, one JSON line (card name and power limit read in the same run).

(a) ingest shape: 1 M open encoders, one datapoint each per call (synth.gaussian_walk), 360 calls; median
    call time from CUDA events, datapoints/s, and the bytes a call must move: state read + write (2 x 128 B per
    series), 16 B of input per series and the committed output, with their share of 3.35 TB/s (H100 SXM HBM3).
(b) 500 k x 1440 appended in chunks of 1, 60 and 1440 points next to encode() of the same data; the snapshots
    are compared with encode()'s bytes.

    python scripts/bench_append.py [--series-a N] [--calls-a N] [--series-b N] [--points-b N]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from m3_b200 import synth  # noqa: E402
from m3_b200.codec import BatchCodec  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def ingest(codec, S, calls):
    ts, vals, start = synth.gaussian_walk(S, calls, "cuda", seed=1)
    tsp, vap = ts.t().contiguous(), vals.t().contiguous()  # one row per call: [1][S] point-major
    del ts, vals
    es = codec.encoder_set(start, codec.encode_bound(calls))
    for i in range(3):  # warm-up, then back to empty encoders
        es.append(tsp[i: i + 1], vap[i: i + 1], point_major=True)
    es.reset(start)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(calls)]
    committed = []
    prev_bits = torch.zeros(S, dtype=torch.int64, device="cuda")
    for i in range(calls):
        ev[i][0].record()
        es.append(tsp[i: i + 1], vap[i: i + 1], point_major=True)
        ev[i][1].record()
        if i % 36 == 0:  # committed output bytes of this call (whole sectors moved to the slots)
            torch.cuda.synchronize()
            bits = es.state.view(torch.int64)[:, 5]
            committed.append(int(((bits >> 8) - (prev_bits >> 8)).clamp(min=0).sum().item()) * 32)
        prev_bits = es.state.view(torch.int64)[:, 5].clone()
    torch.cuda.synchronize()
    ms = [a.elapsed_time(b) for a, b in ev]
    med = median(ms)
    out_b = sum(committed) / max(1, len(committed))
    algo = S * (2 * 128 + 16) + out_b
    return {"series": S, "calls": calls, "median_call_ms": round(med, 4), "p10_ms": round(sorted(ms)[calls // 10], 4),
            "p90_ms": round(sorted(ms)[calls * 9 // 10], 4), "dp_per_s": round(S / (med / 1e3)),
            "bytes_per_call": int(algo), "committed_bytes_per_call_sampled": int(out_b),
            "share_of_3.35TBps": round(algo / (med / 1e3) / HBM_BYTES_PER_S, 3)}


def chunks(codec, S, P):
    ts, vals, start = synth.gaussian_walk(S, P, "cuda", seed=2)
    tsp, vap = ts.t().contiguous(), vals.t().contiguous()
    ref = codec.encode(ts, vals, start)
    codec.encode(ts, vals, start, out=ref)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    codec.encode(ts, vals, start, out=ref)
    b.record()
    torch.cuda.synchronize()
    res = {"series": S, "points": P, "encode_ms": round(a.elapsed_time(b), 3)}
    es = codec.encoder_set(start, ref.out.shape[1])
    for c in (1, 60, P):
        es.reset(start)
        a.record()
        for i in range(0, P, c):
            es.append(tsp[i: i + c], vap[i: i + c], point_major=True)
        b.record()
        snap = es.stream()
        torch.cuda.synchronize()
        same = torch.equal(snap.out_len, ref.out_len)
        col = torch.arange(ref.out.shape[1], device="cuda")
        for r0 in range(0, S, 20_000):  # byte-compare the streams (bytes past each length are not part of them)
            if not same:
                break
            keep = col[None, :] < ref.out_len[r0: r0 + 20_000, None]
            same = bool(torch.equal(snap.out[r0: r0 + 20_000] * keep, ref.out[r0: r0 + 20_000] * keep))
        res["chunk_%d" % c] = {"total_ms": round(a.elapsed_time(b), 3), "calls": (P + c - 1) // c,
                               "identical_to_encode": same}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series-a", type=int, default=1_000_000)
    ap.add_argument("--calls-a", type=int, default=360)
    ap.add_argument("--series-b", type=int, default=500_000)
    ap.add_argument("--points-b", type=int, default=1440)
    args = ap.parse_args()
    codec = BatchCodec(0, int_optimized=True)
    out = {"card": card(), "ingest": ingest(codec, args.series_a, args.calls_a)}
    torch.cuda.empty_cache()
    out["chunks"] = chunks(codec, args.series_b, args.points_b)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
