#!/usr/bin/env python3
"""Timer element sets through a rollup (m3tsz_element_set_forward_timer), one JSON line (card name, power limit and
max SM clock read in the same run).

The shape of an aggregator shard with a timer rollup rule: 1 M Timer sources, one sample per source per add call at a
10 s cadence, 1-minute resolution, R = 2 open windows; a minute is 6 add_timer calls, 1 forward_timer into the group
set and 1 consume of the group set.  Source types: P99 without ops, and Max with one pre-op (Absolute).  Memberships:
10 000 contiguous groups of 100, and 100 000 groups of 10 random sources.  Group types: {Max, P50, P99} and the default
11.  Beside each, in the same run and alternating call by call, the route available without the forward: a source
set with output rows, its consume, a decode of the rows (and a reset of its encoders), a torch gather of each group's
members into point-major [members, groups] arrays, add_timer of those into the group set (one row, one Timer.Add, per
value in listed order) and its consume.  Both routes write the same group bytes; that is checked, and a sample of
groups of the last minute is checked against the CPU model (tests/element_timer_rollup_model.py).

Reported: median ms per minute of both routes and of each call; the algorithmic bytes of the forward (the formulas
below, from the shapes); and, from one more minute under torch.profiler, the device time of the forward's kernels.

    python scripts/bench_element_timer_rollup.py [--sources N] [--minutes N]
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
from m3_b200 import capi  # noqa: E402
from m3_b200.codec import BatchCodec  # noqa: E402

SEC = 1_000_000_000
RES = 60 * SEC
CADENCE = 10 * SEC
T0 = 1_600_000_020 * SEC  # a whole minute
SRC = {"p99": (capi.AGG_P99, []), "max_absolute": (capi.AGG_MAX, [capi.TRANSFORM_ABSOLUTE])}
TYPES = {"max_p50_p99": [capi.AGG_MAX, capi.AGG_P50, capi.AGG_P99], "default11": list(capi.DEFAULT_TIMER_TYPES)}


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
    if kind == "contiguous":  # 10 000 x 100
        G, k = S // 100, 100
        return torch.arange(0, G * k + 1, k, dtype=torch.int64, device=dev), \
            torch.arange(G * k, dtype=torch.int32, device=dev), k
    G, k = S // 10, 10  # 100 000 x 10, random
    gen = torch.Generator(device=dev).manual_seed(11)
    return torch.arange(0, G * k + 1, k, dtype=torch.int64, device=dev), \
        torch.randint(0, S, (G * k,), dtype=torch.int32, device=dev, generator=gen), k


def timer_set(codec, N, types, ops, R, cap, stride):
    return codec.element_set(torch.full((N,), T0, dtype=torch.int64, device="cuda"), capi.METRIC_TIMER, types, RES,
                             transforms=ops, open_windows=R, sample_capacity=cap, stride=stride)


def run(codec, S, minutes, src_name, kind, types_name):
    dev = "cuda"
    src_type, pre = SRC[src_name]
    types = TYPES[types_name]
    off, mem, k = membership(kind, S, dev)
    G = off.numel() - 1
    stride = int(capi.lib().m3tsz_encode_bound_units(minutes + 3, 1))
    src = timer_set(codec, S, [src_type], pre, 2, 8, 0)
    grp = timer_set(codec, G, types, [], 2, 2 * k, stride)
    src_b = timer_set(codec, S, [src_type], pre, 2, 8, int(capi.lib().m3tsz_encode_bound_units(4, 1)))
    grp_b = timer_set(codec, G, types, [], 2, 2 * k, stride)
    start = torch.full((S,), T0, dtype=torch.int64, device=dev)
    offs = (torch.arange(S, device=dev) % 10) * SEC  # each source's phase inside its 10 s cadence
    gen = torch.Generator(device=dev).manual_seed(3)
    t_add, t_fwd, t_cons, t_add_b, t_route_b = [], [], [], [], []
    last_minute = []
    for m in range(minutes + 1):
        last_minute = []
        for c in range(6):
            i = m * 6 + c
            ts = (T0 + i * CADENCE + offs).view(1, S).contiguous()
            vals = (torch.round(torch.rand(S, generator=gen, device=dev, dtype=torch.float64) * 5000) / 10
                    - (50.0 if pre else 0.0)).view(1, S).contiguous()
            last_minute.append((ts, vals))
            t_add.append(timed(lambda: src.add(ts, vals)))
            t_add_b.append(timed(lambda: src_b.add(ts, vals)))
        target = T0 + (m + 1) * RES

        def route_a():
            src.forward_timer(target, off, mem, grp)

        def route_b():
            src_b.consume(target)
            snap = src_b.stream()
            dec = codec.decode(snap.out.view(-1), src_b.out.offsets(), 2, lengths=snap.out_len)
            v = dec.values[:, 0]  # (one window per source and minute)
            src_b.out.reset(start)
            pts = v[mem.long()].view(G, k).t().contiguous()
            tss = torch.full((k, G), target - RES, dtype=torch.int64, device=dev)
            grp_b.add(tss, pts)
            grp_b.consume(target)

        t_fwd.append(timed(route_a))
        t_cons.append(timed(lambda: grp.consume(target)))
        t_route_b.append(timed(route_b))
    torch.cuda.synchronize()
    ms = lambda evs, skip: [a.elapsed_time(b) for a, b in evs[skip:]]  # (the first minute: warm-up)
    add_ms, add_b_ms = ms(t_add, 6), ms(t_add_b, 6)
    fwd_ms, cons_ms, route_b_ms = ms(t_fwd, 1), ms(t_cons, 1), ms(t_route_b, 1)

    # both routes wrote the same group bytes
    sa, sb = grp.stream(), grp_b.stream()
    same_bytes = bool(torch.equal(sa.out_len, sb.out_len) and torch.equal(sa.out, sb.out))
    # a sample of groups' last minute against the CPU model
    from element_timer_rollup_model import TimerGroupModel, TimerSourceModel, forward
    dec = codec.decode(sa.out.view(-1), grp.out.offsets(), minutes + 2, lengths=sa.out_len)
    dn, dv = dec.n_points.cpu().numpy(), dec.values.cpu().numpy()
    offc, memc = off.cpu().numpy(), mem.cpu().numpy()
    tsc = [t.cpu().numpy()[0] for t, _ in last_minute]
    vsc = [v.cpu().numpy()[0] for _, v in last_minute]
    model_ok = True
    for g in np.random.default_rng(1).choice(G, 16, replace=False).tolist():
        sms = []
        for s in memc[offc[g]: offc[g + 1]].tolist():
            sm = TimerSourceModel(src_type, RES, pre, False, 2, 8)
            sm.add([(int(tsc[c][s]), float(vsc[c][s])) for c in range(6)])
            sms.append(sm)
        gm = TimerGroupModel(types, RES, [], False, 2, 2 * k)
        target = T0 + (minutes + 1) * RES
        forward(sms, [gm], target, [0, len(sms)], list(range(len(sms))))
        for j, (_, v) in enumerate(gm.consume(target)):
            row = j * G + g
            model_ok &= bool(dv[row, dn[row] - 1] == v[0])  # (no NaN in these samples)

    # one more minute, its forward under the profiler: device time per kernel
    for c in range(6):
        i = (minutes + 1) * 6 + c
        src.add((T0 + i * CADENCE + offs).view(1, S).contiguous(), last_minute[c][1])
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        src.forward_timer(T0 + (minutes + 2) * RES, off, mem, grp)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            name = e.name.split("<")[0].split("(")[0].replace("void ", "").replace("m3tsz::", "")
            kern[name] = round(kern.get(name, 0.0) + e.device_time_total / 1e3, 4)

    # algorithmic bytes of a forward.  Per source (one due window of n = 6 samples): its slots' start and count
    # (16 R), the window's count / sum / sumSq (24), its header read and written (128), the flush's list (value,
    # numRanks, delta, prev, next: 32 B per sample) read and written and its pending heap read (8 B per value: n - 1),
    # the record's head read (96) and written to scratch (96), the forwarded start / value (16), count, presence and
    # due words (20); the commit as the plain forward's (4 + 8 + 8 + 96 read, 8 + 8 + 96 + 4 written).  Per listed
    # member: its index (4) and its count, presence word, start and value (28).  Per group: its slots' start and count
    # (16 R), the window's slot read and written (2 x 32), its header (128), and per value one pending-heap write
    # (8; the periodic insert runs at the consume for these sizes) and the status (4).
    n, R = 6, 2
    fwd_b = (S * (16 * R + 24 + 128 + 2 * 32 * n + 8 * (n - 1) + 2 * 96 + 16 + 20 + 4 + 8 + 8 + 96 + 8 + 8 + 96 + 4)
             + mem.numel() * (4 + 28 + 8) + G * (16 * R + 2 * 32 + 128 + 4))
    r = lambda x: None if x is None else round(x, 4)
    return {"source": src_name, "membership": kind, "group_types": types_name, "sources": S, "groups": G,
            "members": mem.numel(), "minutes": minutes,
            "add_median_ms": r(median(add_ms)), "forward_median_ms": r(median(fwd_ms)), "forward_bytes": fwd_b,
            "forward_kernels_ms": kern, "group_consume_median_ms": r(median(cons_ms)),
            "route_b_add_median_ms": r(median(add_b_ms)), "route_b_flush_median_ms": r(median(route_b_ms)),
            "per_minute_ms": {"forward_timer": r(6 * median(add_ms) + median(fwd_ms) + median(cons_ms)),
                              "consume_decode_gather_add": r(6 * median(add_b_ms) + median(route_b_ms))},
            "same_group_bytes": same_bytes, "sampled_groups_equal_model": model_ok}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sources", type=int, default=1_000_000)
    ap.add_argument("--minutes", type=int, default=6)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_element_timer_rollup: no CUDA device")
    codec = BatchCodec(0, int_optimized=False)
    runs = []
    for src_name in SRC:
        for kind in ("contiguous", "random"):
            for types_name in TYPES:
                runs.append(run(codec, args.sources, args.minutes, src_name, kind, types_name))
                torch.cuda.empty_cache()
    print(json.dumps({"card": card(), "runs": runs}))


if __name__ == "__main__":
    main()
