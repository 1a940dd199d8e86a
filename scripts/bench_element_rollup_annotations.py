#!/usr/bin/env python3
"""Element sets through a rollup that keep annotations (m3tsz_element_set_forward_annotated), one JSON line (card
name, power limit and max SM clock read in the same run).

The shape of scripts/bench_element_rollup.py: 1 M source elements, one datapoint per source per add call at a 10 s
cadence, 1-minute resolution, the same two pipelines and two memberships; every datapoint carries the 4-byte
OpenMetrics counter payload.  A minute of ingest is 6 annotated adds, 1 annotated forward and 1 annotated group
consume.  Alternating call by call in the same run with it: the plain element rollup on the same datapoints without
annotations, and the route without element sets, annotated EncoderSet.append of the same datapoints and at each flush
stream() + aggregate_tiles_rollup(annotations=True) over the minute that ended.

Reported: median ms per call of each route, the algorithmic bytes of the annotated forward (from the shapes, the
formula below), and from one more minute under torch.profiler the device time of each kernel of an annotated and of a
plain forward.

    python scripts/bench_element_rollup_annotations.py [--sources N] [--calls N]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_element_rollup import (CADENCE, HBM_BYTES_PER_S, PIPES, RES, SEC, T0, card, median,  # noqa: E402
                                  membership, timed)
from m3_b200 import capi  # noqa: E402
from m3_b200.codec import BatchCodec  # noqa: E402

PROM = bytes([0x08, 0x01, 0x10, 0x01])  # annotation.Payload{OpenMetricsFamilyType: COUNTER, HandleValueResets: true}


def annotations(S, dev):
    """the sparse list of one datapoint per element, each carrying PROM (dp_index 0, one copy of the bytes)"""
    off = torch.arange(S + 1, dtype=torch.int64, device=dev)
    ent = torch.zeros((S, 4), dtype=torch.int32, device=dev)
    ent[:, 1] = len(PROM)  # dp_index 0, length, byte_offset 0
    return off, ent.view(torch.uint8).view(S, 16), torch.tensor(list(PROM), dtype=torch.uint8, device=dev)


def forward_kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            name = e.name.split("<")[0].split("(")[0].replace("void ", "").replace("m3tsz::", "")
            kern[name] = round(kern.get(name, 0.0) + e.device_time_total / 1e3, 4)
    return kern


def run(codec, S, calls, pipe_name, kind):
    dev = "cuda"
    metric, src_type, pre, types, post = PIPES[pipe_name]
    gauge = metric == capi.METRIC_GAUGE
    off, mem = membership(kind, S, dev)
    G = off.numel() - 1
    start = torch.full((S,), T0, dtype=torch.int64, device=dev)
    gstart = torch.full((G,), T0, dtype=torch.int64, device=dev)
    offs = (torch.arange(S, device=dev) % 10) * SEC
    gen = torch.Generator(device=dev).manual_seed(3)
    flushes = calls // 6
    stride = int(capi.lib().m3tsz_encode_bound_units(flushes + 2, 1)) + 32 * (flushes + 2)  # (+ the annotation words)
    ann = annotations(S, dev)
    a_src = codec.element_set(start, metric, [src_type], RES, transforms=pre, open_windows=2, stride=0,
                              annotation_capacity=8)
    a_grp = codec.element_set(gstart, metric, types, RES, transforms=post, open_windows=2, stride=stride,
                              annotation_capacity=8)
    p_src = codec.element_set(start, metric, [src_type], RES, transforms=pre, open_windows=2, stride=0)
    p_grp = codec.element_set(gstart, metric, types, RES, transforms=post, open_windows=2, stride=stride)
    enc = codec.encoder_set(start, codec.encode_bound(calls + 6) + 32 * (calls + 6))
    xs, gs = codec.transform_state(S), codec.element_state(G)
    t = {k: [] for k in ("a_add", "a_fwd", "a_cons", "p_add", "p_fwd", "p_cons", "app", "tile")}
    level = torch.zeros(S, dtype=torch.float64, device=dev)
    for i in range(calls):
        ts = (T0 + i * CADENCE + offs).view(1, S).contiguous()
        step = torch.randn(S, dtype=torch.float64, device=dev, generator=gen)
        level = level + (step if gauge else step.abs().round())
        vals = level.view(1, S).contiguous()
        t["a_add"].append(timed(lambda: a_src.add(ts, vals, annotations=ann)))
        t["p_add"].append(timed(lambda: p_src.add(ts, vals)))
        t["app"].append(timed(lambda: enc.append(ts.view(S, 1), vals.view(S, 1), annotations=ann)))
        if (i + 1) % 6 == 0:
            target = T0 + (i + 1) // 6 * RES
            t["a_fwd"].append(timed(lambda: a_src.forward(target, off, mem, a_grp)))
            t["p_fwd"].append(timed(lambda: p_src.forward(target, off, mem, p_grp)))
            t["a_cons"].append(timed(lambda: a_grp.consume(target)))
            t["p_cons"].append(timed(lambda: p_grp.consume(target)))

            def tiles():
                snap = enc.stream()
                codec.aggregate_tiles_rollup(snap.out.view(-1), enc.offsets(), target - RES, RES, 1, src_type, off,
                                             mem, types, metric_type=metric, pre_transforms=pre, post_transforms=post,
                                             discard_nan=False, src_state=xs, group_state=gs, lengths=snap.out_len,
                                             annotations=True)
            t["tile"].append(timed(tiles))
    torch.cuda.synchronize()
    ms = {k: median([a.elapsed_time(b) for a, b in v[1:]]) for k, v in t.items()}  # (the first of each: warm-up)

    # one more minute, each forward under the profiler: device time per kernel
    for i in range(calls, calls + 6):
        ts, vals = (T0 + i * CADENCE + offs).view(1, S).contiguous(), level.view(1, S).contiguous()
        a_src.add(ts, vals, annotations=ann)
        p_src.add(ts, vals)
    torch.cuda.synchronize()
    target = T0 + (calls + 6) // 6 * RES
    a_kern = forward_kernels(lambda: a_src.forward(target, off, mem, a_grp))
    p_kern = forward_kernels(lambda: p_src.forward(target, off, mem, p_grp))

    # algorithmic bytes of the annotated forward: the plain forward's (scripts/bench_element_rollup.py, R = 2 slots,
    # one due window per source) and, per source, its due window's length read (4), the slots' starts read again by
    # the reference pass (8 R), the annotation word and the reference written (8 + 8); per listed member its
    # annotation word (8) and its reference (8); per group the length written (4) and the payload word read from a
    # source slot and written to the group slot (8 + 8)
    fields = 8 if gauge else 6
    plain_b = (S * (16 * 2 + 16 + 2 * 96 + 16 + 20 + 4 + 4 + 8 + 8 + 96 + 8 + 8 + 96 + 4)
               + mem.numel() * (4 + 28) + G * (16 * 2 + 2 * 8 * fields + 4))
    fwd_b = plain_b + S * (4 + 8 * 2 + 8 + 8) + mem.numel() * (8 + 8) + G * (4 + 8 + 8)
    r = lambda x: None if x is None else round(x, 4)
    minute = lambda add, fwd, cons: r(6 * ms[add] + ms[fwd] + ms[cons])
    return {"pipeline": pipe_name, "membership": kind, "sources": S, "groups": G, "members": mem.numel(),
            "calls": calls,
            "annotated": {"add_ms": r(ms["a_add"]), "forward_ms": r(ms["a_fwd"]), "consume_ms": r(ms["a_cons"]),
                          "forward_kernels_ms": a_kern, "forward_bytes": fwd_b,
                          "forward_share_of_3.35TBps": round(fwd_b / (ms["a_fwd"] / 1e3) / HBM_BYTES_PER_S, 3)},
            "plain": {"add_ms": r(ms["p_add"]), "forward_ms": r(ms["p_fwd"]), "consume_ms": r(ms["p_cons"]),
                      "forward_kernels_ms": p_kern, "forward_bytes": plain_b},
            "append_then_tile_rollup": {"append_ms": r(ms["app"]), "flush_ms": r(ms["tile"])},
            "per_minute_ms": {"annotated_element_sets": minute("a_add", "a_fwd", "a_cons"),
                              "plain_element_sets": minute("p_add", "p_fwd", "p_cons"),
                              "annotated_append_then_tile_rollup": r(6 * ms["app"] + ms["tile"])}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sources", type=int, default=1_000_000)
    ap.add_argument("--calls", type=int, default=42)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_element_rollup_annotations: no CUDA device")
    codec = BatchCodec(0, int_optimized=True)
    runs = [run(codec, args.sources, args.calls, p, kind) for p in PIPES for kind in ("contiguous", "random")]
    print(json.dumps({"card": card(), "runs": runs}))


if __name__ == "__main__":
    main()
