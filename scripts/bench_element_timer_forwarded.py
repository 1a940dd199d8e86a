#!/usr/bin/env python3
"""Timer element-set rollups across shards (m3tsz_element_set_forward_write_timer / _add_forwarded_timer), one JSON line
(card name, power limit and max SM clock read in the same run).

Shape: bench_element_timer_rollup.py's Timer shape split over 8 source sets standing for shards: 1 M Timer sources of
type P99, one sample per source every 10 s, 1-minute resolution, R = 2 open windows of 8 samples; the rollup [Max, P50,
P99].  Two memberships with members drawn across all shards: 100 000 groups of 10 and 10 000 groups of 100.  Per
minute: forward_write_timer on each shard, add_forwarded_timer of all shards' batches in shard order into the group
set (the order the single set lists each group's members in, so both give the same windows), and as the reference
point one forward_timer of the same data from a single set holding every source.  CUDA events around each Python
call; reported: median ms of each, over --minutes minutes after one warm-up minute.

    python scripts/bench_element_timer_forwarded.py [--sources N] [--shards K] [--minutes M]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from m3_b200 import capi  # noqa: E402
from m3_b200.codec import BatchCodec, ForwardedBatch  # noqa: E402

SEC = 1_000_000_000
RES = 60 * SEC
T0 = 1_600_000_020 * SEC
TYPES = [capi.AGG_MAX, capi.AGG_P50, capi.AGG_P99]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2] if xs else None


def split(off, mem, K):
    """members by shard (source s on shard s % K, local index s // K), in order; and the single set's lists"""
    G = len(off) - 1
    gid = np.repeat(np.arange(G), np.diff(off))
    sh = mem % K
    parts = []
    for k in range(K):
        sel = sh == k
        o = np.zeros(G + 1, dtype=np.int64)
        o[1:] = np.cumsum(np.bincount(gid[sel], minlength=G))
        parts.append((o, (mem[sel] // K).astype(np.int32)))
    order = np.lexsort((sh, gid))  # stable: by group, then shard, listed order kept
    return parts, off, mem[order].astype(np.int32)


def timer_set(codec, N, types, R, cap, source_capacity=0):
    return codec.element_set(torch.full((N,), T0, dtype=torch.int64, device="cuda"), capi.METRIC_TIMER, types, RES,
                             open_windows=R, sample_capacity=cap, stride=0, source_capacity=source_capacity)


def run(codec, S, K, G, per, minutes, rng):
    dev = "cuda"
    one = timer_set(codec, S, [capi.AGG_P99], 2, 8)
    shards = [timer_set(codec, len(range(k, S, K)), [capi.AGG_P99], 2, 8) for k in range(K)]
    ref = timer_set(codec, G, TYPES, 2, 2 * per)
    grp = timer_set(codec, G, TYPES, 2, 2 * per, source_capacity=32)
    off = np.arange(0, G * per + 1, per, dtype=np.int64)
    mem = rng.integers(0, S, G * per).astype(np.int64)
    parts, o1, m1 = split(off, mem, K)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    parts = [(d(o), d(m)) for o, m in parts]
    o1, m1 = d(o1), d(m1)
    phase = (torch.arange(S, device=dev) % 10) * SEC  # each source's phase inside its 10 s cadence
    gen = torch.Generator(device=dev).manual_seed(3)
    t_write, t_add, t_fwd = [], [], []
    ev = lambda: torch.cuda.Event(enable_timing=True)
    same = True
    for minute in range(minutes + 1):
        base = T0 + minute * RES
        ts = torch.stack([base + i * 10 * SEC + phase for i in range(6)]).contiguous()
        vals = (torch.round(torch.rand((6, S), generator=gen, device=dev, dtype=torch.float64) * 5000) / 10)
        one.add(ts, vals)
        for k, sh in enumerate(shards):
            sh.add(ts[:, k::K].contiguous(), vals[:, k::K].contiguous())
        target = base + RES
        torch.cuda.synchronize()
        a, b = ev(), ev()
        a.record()
        one.forward_timer(target, o1, m1, ref)
        b.record()
        torch.cuda.synchronize()
        fwd_ms = a.elapsed_time(b)
        batches, w_ms = [], []
        for k, sh in enumerate(shards):
            a, b = ev(), ev()
            a.record()
            bt, _, gst = sh.forward_write_timer(target, parts[k][0], parts[k][1], k, metric_capacity=G,
                                                value_capacity=G * per)
            b.record()
            torch.cuda.synchronize()
            w_ms.append(a.elapsed_time(b))
            batches.append(bt)
        cat = ForwardedBatch.concat(batches)
        torch.cuda.synchronize()
        a, b = ev(), ev()
        a.record()
        res, st = grp.add_forwarded_timer(cat)
        b.record()
        torch.cuda.synchronize()
        assert int(res.abs().sum()) == 0 and int(st.abs().sum()) == 0
        # (each group's one window this minute, in its first free slot: count and sum as the single-set forward's)
        same &= all(bool(torch.equal(ref.win[f].view(torch.int64), grp.win[f].view(torch.int64)))
                    for f in ("count", "sum", "sum_sq"))
        # free the group windows, so that the next minute opens new ones
        ref.win["count"].zero_()
        grp.win["count"].zero_()
        if minute:
            t_fwd.append(fwd_ms)
            t_write.append(median(w_ms))
            t_add.append(a.elapsed_time(b))
    return {"groups": G, "members": per, "records": int(cat.metrics.shape[0]), "values": int(cat.values.numel()),
            "forward_write_timer_per_shard_ms": median(t_write), "add_forwarded_timer_ms": median(t_add),
            "single_set_forward_timer_ms": median(t_fwd), "group_sums_equal": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sources", type=int, default=1_000_000)
    ap.add_argument("--shards", type=int, default=8)
    ap.add_argument("--minutes", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_element_timer_forwarded.py needs a CUDA device")
    codec = BatchCodec(0)
    rng = np.random.default_rng(1)
    out = {"card": card(), "sources": a.sources, "shards": a.shards, "shapes": []}
    for G, per in ((100_000, 10), (10_000, 100)):
        out["shapes"].append(run(codec, a.sources, a.shards, G, per, a.minutes, rng))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
