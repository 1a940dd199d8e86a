#!/usr/bin/env python3
"""Element sets through a rollup (m3tsz_element_set_forward), one JSON line (card name, power limit and max SM clock
read in the same run).

The ingest shape of an aggregator shard with a rollup rule: 1 M source elements, one datapoint per source per add
call at a 10 s cadence, 1-minute resolution; a minute of ingest is 6 adds, 1 forward into the group set and 1 consume
of the group set.  Two memberships, as scripts/bench_tile_rollup.py: 5 000 contiguous groups of 100, and 50 000 groups
of 10 random sources.  Two pipelines: Counter Sum + [Increase] -> Rollup [Sum] -> [Add], and Gauge Last -> Rollup
[Min, Max, Sum].  Beside each, in the same run and alternating call by call, the route without element sets:
EncoderSet.append of the same datapoints, and at each flush stream() + aggregate_tiles_rollup over the minute that
ended (a decode of every source stream so far, the forward, the fold and the groups' encode).

Reported: median ms per add, forward, group consume and per call of the other route; the algorithmic bytes of the add,
the forward and the fold (from the shapes, the formulas below); and, from one more minute under torch.profiler, the
device time of each kernel of a forward.

    python scripts/bench_element_rollup.py [--sources N] [--calls N]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from m3_b200 import capi  # noqa: E402
from m3_b200.codec import BatchCodec  # noqa: E402

SEC = 1_000_000_000
RES = 60 * SEC
CADENCE = 10 * SEC
T0 = 1_600_000_020 * SEC  # a whole minute
HBM_BYTES_PER_S = 3.35e12
PIPES = {  # name: (metric, source type, pre-ops, rollup types, post-ops)
    "counter_increase_sum_add": (capi.METRIC_COUNTER, capi.AGG_SUM, [capi.TRANSFORM_INCREASE], [capi.AGG_SUM],
                                 [capi.TRANSFORM_ADD]),
    "gauge_last_min_max_sum": (capi.METRIC_GAUGE, capi.AGG_LAST, [], [capi.AGG_MIN, capi.AGG_MAX, capi.AGG_SUM], []),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2] if xs else None


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    return a, b


def membership(kind, S, dev):
    if kind == "contiguous":
        off = torch.arange(0, 500_000 + 1, 100, dtype=torch.int64, device=dev)
        return off, torch.arange(500_000, dtype=torch.int32, device=dev)
    gen = torch.Generator(device=dev).manual_seed(11)
    off = torch.arange(0, 500_000 + 1, 10, dtype=torch.int64, device=dev)
    return off, torch.randint(0, S, (500_000,), dtype=torch.int32, device=dev, generator=gen)


def run(codec, S, calls, pipe_name, kind):
    dev = "cuda"
    metric, src_type, pre, types, post = PIPES[pipe_name]
    gauge = metric == capi.METRIC_GAUGE
    k = len(types)
    off, mem = membership(kind, S, dev)
    G = off.numel() - 1
    start = torch.full((S,), T0, dtype=torch.int64, device=dev)
    offs = (torch.arange(S, device=dev) % 10) * SEC  # each source's phase inside its 10 s cadence
    gen = torch.Generator(device=dev).manual_seed(3)
    flushes = calls // 6
    src = codec.element_set(start, metric, [src_type], RES, transforms=pre, open_windows=2, stride=0)
    grp = codec.element_set(torch.full((G,), T0, dtype=torch.int64, device=dev), metric, types, RES,
                            transforms=post, open_windows=2,
                            stride=int(capi.lib().m3tsz_encode_bound_units(flushes + 2, 1)))
    enc = codec.encoder_set(start, codec.encode_bound(calls + 6))
    xs, gs = codec.transform_state(S), codec.element_state(G)
    t_add, t_fwd, t_cons, t_app, t_tile = [], [], [], [], []
    level = torch.zeros(S, dtype=torch.float64, device=dev)
    for i in range(calls):
        ts = (T0 + i * CADENCE + offs).view(1, S).contiguous()
        step = torch.randn(S, dtype=torch.float64, device=dev, generator=gen)
        level = level + (step if gauge else step.abs().round())
        vals = level.view(1, S).contiguous()
        t_add.append(timed(lambda: src.add(ts, vals)))
        t_app.append(timed(lambda: enc.append(ts, vals, point_major=True)))
        if (i + 1) % 6 == 0:
            target = T0 + (i + 1) // 6 * RES
            t_fwd.append(timed(lambda: src.forward(target, off, mem, grp)))
            t_cons.append(timed(lambda: grp.consume(target)))

            def tiles():
                snap = enc.stream()
                codec.aggregate_tiles_rollup(snap.out.view(-1), enc.offsets(), target - RES, RES, 1, src_type, off,
                                             mem, types, metric_type=metric, pre_transforms=pre, post_transforms=post,
                                             discard_nan=False, src_state=xs, group_state=gs, lengths=snap.out_len)
            t_tile.append(timed(tiles))
    torch.cuda.synchronize()
    ms = lambda evs: [a.elapsed_time(b) for a, b in evs[1:]]  # (the first of each: warm-up)
    add_ms, fwd_ms, cons_ms, app_ms, tile_ms = ms(t_add), ms(t_fwd), ms(t_cons), ms(t_app), ms(t_tile)

    # one more minute, its forward under the profiler: device time per kernel
    for i in range(calls, calls + 6):
        src.add((T0 + i * CADENCE + offs).view(1, S).contiguous(), level.view(1, S).contiguous())
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        src.forward(T0 + (calls + 6) // 6 * RES, off, mem, grp)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            name = e.name.split("<")[0].split("(")[0].replace("void ", "").replace("m3tsz::", "")
            kern[name] = round(kern.get(name, 0.0) + e.device_time_total / 1e3, 4)

    # algorithmic bytes.  add: as scripts/bench_elements.py (R = 2 slots)
    fields = 8 if gauge else 6
    add_b = S * (16 + 8 + 16 * 2 + 2 * 8 * fields + 1 + 4)
    # forward, per source: its slots' start and count (16 R), the due window's ValueOf input (8) and count (8), the
    # record's head read (96) and written to scratch (96), the forwarded start / value (16), its count, presence and
    # due words (20); the commit: the mark (4), the count / due words, start and new head read back (4 + 8 + 8 + 96),
    # the freed count, watermark and record written (8 + 8 + 96) and the status (4).  Per listed member: its index (4)
    # and its count, presence word, start and value (28).  Per group: its slots' start and count (16 R), the window's
    # aggregates read and written (2 x 8 x fields, last_at included for the Gauge) and its status (4).
    fwd_b = (S * (16 * 2 + 16 + 2 * 96 + 16 + 20 + 4 + 4 + 8 + 8 + 96 + 8 + 8 + 96 + 4)
             + mem.numel() * (4 + 28) + G * (16 * 2 + 2 * 8 * fields + 4))
    r = lambda x: None if x is None else round(x, 4)
    share = lambda b, m: None if m is None else round(b / (m / 1e3) / HBM_BYTES_PER_S, 3)
    return {"pipeline": pipe_name, "membership": kind, "sources": S, "groups": G, "members": mem.numel(),
            "rollup_types": k, "calls": calls,
            "add_median_ms": r(median(add_ms)), "add_bytes": add_b,
            "forward_median_ms": r(median(fwd_ms)), "forward_bytes": fwd_b,
            "forward_share_of_3.35TBps": share(fwd_b, median(fwd_ms)), "forward_kernels_ms": kern,
            "group_consume_median_ms": r(median(cons_ms)),
            "route_append_median_ms": r(median(app_ms)), "route_flush_median_ms": r(median(tile_ms)),
            "per_minute_ms": {"element_sets": r(6 * median(add_ms) + median(fwd_ms) + median(cons_ms)),
                              "append_then_tile_rollup": r(6 * median(app_ms) + median(tile_ms))}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sources", type=int, default=1_000_000)
    ap.add_argument("--calls", type=int, default=42)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_element_rollup: no CUDA device")
    codec = BatchCodec(0, int_optimized=True)
    runs = [run(codec, args.sources, args.calls, p, kind) for p in PIPES for kind in ("contiguous", "random")]
    print(json.dumps({"card": card(), "runs": runs}))


if __name__ == "__main__":
    main()
