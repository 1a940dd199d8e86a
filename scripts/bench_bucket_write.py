#!/usr/bin/env python3
"""Bucket writes (BucketSet.write, m3tsz_encoder_set_write) against the plain encoder-set append, one JSON line.

(a) 1 M buckets, one datapoint per call, 360 calls, all in order: write (K = 4) and append alternating, median ms
    per call -- what routing costs on the common path;
(b) the same, but each call also sends, for 1 % of the series, a datapoint up to 10 steps late and, for 0.5 %, a
    rewrite of their last timestamp with a new value (append is timed on the same inputs, as a cost reference only);
(c) read() of the block written in (b), next to snapshot + decode of the plain encoder set of (b).

The card's name, power limit and max SM clock are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from m3_b200 import capi  # noqa: E402
from m3_b200.codec import BatchCodec  # noqa: E402

SEC = 10 ** 9
START = 1599955200 * SEC


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b), out


def traffic(S, c, mixed, g):
    """call c: (ts [S, 2], vals [S, 2], n_points [S]); column 1 is a late datapoint or a rewrite where n = 2"""
    t = START + (c + 1) * 10 * SEC
    ts = torch.full((S, 2), t, dtype=torch.int64, device="cuda")
    vals = torch.round(torch.randn((S, 2), generator=g, device="cuda", dtype=torch.float64) * 50, decimals=2)
    n = torch.ones(S, dtype=torch.int32, device="cuda")
    if mixed:
        u = torch.rand((S,), generator=g, device="cuda")
        late = u < 0.01
        rewrite = (u >= 0.01) & (u < 0.015)
        steps = torch.randint(1, 11, (S,), generator=g, device="cuda")
        ts[:, 1] = torch.where(late, t - steps * 10 * SEC, ts[:, 1])
        n = torch.where(late | rewrite, 2, 1).to(torch.int32)
    return ts, vals, n


def call_bytes(state, ts, res, n, status):
    """bytes per series that one call of one datapoint per series moves, from the shapes: the append loads and saves
    a state and reads the inputs, n_points and writes its count and status; the route reads the state and the same
    inputs again and writes a target byte, the result and a status; the routed append reads the target byte"""
    row = state.shape[1] * state.element_size()
    inputs = 2 * ts.element_size() + n.element_size()  # (ts and value of one datapoint)
    append = 2 * row + inputs + 2 * status.element_size()
    route = row + inputs + 1 + res.element_size() + status.element_size() + 1
    return append, route


def run(S, calls, mixed, K, seed):
    codec = BatchCodec(int_optimized=True)
    start = torch.full((S,), START, dtype=torch.int64, device="cuda")
    stride = codec.encode_bound(calls) + 64
    bs = codec.bucket_set(start, stride, encoders=K, pool_records=(2 * S if mixed else 1024), pool_stride=512)
    es = codec.encoder_set(start, stride)
    g = torch.Generator(device="cuda").manual_seed(seed)
    tw, ta = [], []
    capacity = 0
    sizes = None
    for c in range(calls):
        ts, vals, n = traffic(S, c, mixed, g)
        order = (0, 1) if c % 2 == 0 else (1, 0)  # alternate which of the two goes first
        for k in order:
            if k == 0:
                ms, (res, st) = timed(lambda: bs.write(ts, vals, n_points=n))
                tw.append(ms)
                capacity += int((st == capi.ERR_CAPACITY).sum().item())
                sizes = call_bytes(bs.primary.state, ts[:, :1], res[:, :1], n, st)
            else:
                ms, _ = timed(lambda: es.append(ts, vals, n_points=n))
                ta.append(ms)
    med = lambda x: sorted(x[10:])[len(x[10:]) // 2]  # (the first calls warm up)
    return codec, bs, es, med(tw), med(ta), capacity, sizes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1 << 20)
    ap.add_argument("--calls", type=int, default=360)
    a = ap.parse_args()
    S, K = a.series, 4
    out = {"card": card(), "series": S, "calls": a.calls, "encoders": K}
    _, bs, es, w, ap_, cap, sizes = run(S, a.calls, False, K, 1)
    out["a_write_ms"], out["a_append_ms"], out["a_ratio"], out["a_capacity"] = w, ap_, w / ap_, cap
    # bytes per series and call besides the committed stream bytes, from the shapes of the call
    out["append_bytes_per_series"], out["route_added_bytes_per_series"] = sizes
    del bs, es
    torch.cuda.empty_cache()
    codec, bs, es, w, ap_, cap, _ = run(S, a.calls, True, K, 2)
    out["b_write_ms"], out["b_append_ms"], out["b_ratio"], out["b_capacity"] = w, ap_, w / ap_, cap
    out["b_pool_records_used"] = int(bs.pool_count.item())
    cap_pts = a.calls + 32  # (a bucket takes a second datapoint in 1.5 % of the calls)
    r_ms, r = timed(lambda: bs.read(cap_pts))
    out["c_read_status_nonzero"] = int((r[3] != 0).sum().item())
    del r
    torch.cuda.empty_cache()
    r_ms, r = timed(lambda: bs.read(cap_pts))  # (the first read allocated its buffers)
    del r
    torch.cuda.empty_cache()

    def plain():
        enc = es.stream()
        return codec.decode(enc.out.reshape(-1), es.offsets(), cap_pts, lengths=enc.out_len)

    plain()  # warm-up
    p_ms, _ = timed(plain)
    out["c_read_ms"], out["c_snapshot_decode_ms"] = r_ms, p_ms
    print(json.dumps(out))


if __name__ == "__main__":
    main()
