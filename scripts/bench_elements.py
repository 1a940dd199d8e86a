#!/usr/bin/env python3
"""Element-set timings (m3tsz_element_set_add / _consume), one JSON line (card name and power limit read in the same
run).

The ingest shape of an aggregator shard: 1 M elements, one datapoint per element per add call at a 10 s cadence,
1-minute resolution, a consume at every 6th call (each flushes the minute that just ended).  Two sets: Counter {Sum}
and Gauge {Last, Min, Max}.  Beside each, in the same run and alternating call by call, the route without element
sets: EncoderSet.append of the same datapoints, and at each flush stream() + aggregate_tiles_types over the snapshot
for the minute that ended (a decode of every stream so far, then the element step and a fresh encode).

Reported: median ms per add, per consume, and per call of the other route; the algorithmic bytes each moves (from
the shapes, the formulas below); and, from one more flush under torch.profiler, the device time of each kernel of a
consume (the staging kernel against the encoder-set append it feeds).

    python scripts/bench_elements.py [--elements N] [--calls N]
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


def run(codec, N, calls, metric, types):
    dev = "cuda"
    k = len(types)
    gauge = metric == capi.METRIC_GAUGE
    start = torch.full((N,), T0, dtype=torch.int64, device=dev)
    offs = (torch.arange(N, device=dev) % 10) * SEC  # each element's phase inside its 10 s cadence
    gen = torch.Generator(device=dev).manual_seed(3)
    flushes = calls // 6
    stride = int(capi.lib().m3tsz_encode_bound_units(2 * flushes + 2, 1))
    es = codec.element_set(start, metric, types, RES, open_windows=2, stride=stride)
    enc = codec.encoder_set(start, codec.encode_bound(calls))
    state = codec.element_state(N)
    t_add, t_cons, t_app, t_tile = [], [], [], []
    level = torch.zeros(N, dtype=torch.float64, device=dev)
    for i in range(calls):
        ts = (T0 + i * CADENCE + offs).view(1, N).contiguous()
        step = torch.randn(N, dtype=torch.float64, device=dev, generator=gen)
        level = level + (step if gauge else step.abs().round())
        vals = level.view(1, N).contiguous()
        t_add.append(timed(lambda: es.add(ts, vals)))
        t_app.append(timed(lambda: enc.append(ts, vals, point_major=True)))
        if (i + 1) % 6 == 0:
            target = T0 + (i + 1) // 6 * RES
            t_cons.append(timed(lambda: es.consume(target)))

            def tiles():
                snap = enc.stream()
                codec.aggregate_tiles_types(snap.out.view(-1), enc.offsets(), target - RES, RES, 1, types,
                                            metric_type=metric, lengths=snap.out_len, state=state,
                                            discard_nan=False)
            t_tile.append(timed(tiles))
    torch.cuda.synchronize()
    ms = lambda evs: [a.elapsed_time(b) for a, b in evs[1:]]  # (the first of each: warm-up)
    add_ms, cons_ms, app_ms, tile_ms = ms(t_add), ms(t_cons), ms(t_app), ms(t_tile)

    # one more minute, its consume under the profiler: device time per kernel
    for i in range(calls, calls + 6):
        ts = (T0 + i * CADENCE + offs).view(1, N).contiguous()
        es.add(ts, level.view(1, N).contiguous())
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        es.consume(T0 + (calls + 6) // 6 * RES)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            name = e.name.split("<")[0].split("(")[0].replace("void ", "").replace("m3tsz::", "")
            kern[name] = round(kern.get(name, 0.0) + e.device_time_total / 1e3, 4)

    # algorithmic bytes.  add: the datapoint (16 B), the element's watermark (8), its R slots' start and count to
    # find the window (16 R), the window's aggregates read and written (2 x 8 B x fields), result (1) and status (4).
    fields = 8 if gauge else 6
    add_b = N * (16 + 8 + 16 * 2 + 2 * 8 * fields + 1 + 4)
    # consume: the slots' start and count (16 R), the flushed window's aggregates (8 x fields) and its freed count (8),
    # the element record read and written (2 x 160), the watermark (16), per type the staged row written and read back
    # (2 x 16), its count (2 x 4), the output encoder's state read and written (2 x 128), the row's status (2 x 4) and
    # about 8 bytes of stream, and the element status (2 x 4)
    cons_b = N * (16 * 2 + 8 * fields + 8 + 2 * 160 + 16 + k * (32 + 8 + 256 + 8 + 8) + 8)
    # the other route per call: the encoder-set append (state read and written, 2 x 128, input 16, ~4 B of stream)
    app_b = N * (2 * 128 + 16 + 4)
    r = lambda x: None if x is None else round(x, 4)
    share = lambda b, m: None if m is None else round(b / (m / 1e3) / HBM_BYTES_PER_S, 3)
    return {"metric": "counter" if not gauge else "gauge", "types": types, "elements": N, "calls": calls,
            "add_median_ms": r(median(add_ms)), "add_bytes": add_b, "add_share_of_3.35TBps": share(add_b, median(add_ms)),
            "consume_median_ms": r(median(cons_ms)), "consume_bytes": cons_b,
            "consume_share_of_3.35TBps": share(cons_b, median(cons_ms)),
            "consume_kernels_ms": kern,
            "route_append_median_ms": r(median(app_ms)), "route_append_bytes": app_b,
            "route_flush_median_ms": r(median(tile_ms)),
            "per_minute_ms": {"element_set": r(6 * median(add_ms) + median(cons_ms)),
                              "append_then_tiles": r(6 * median(app_ms) + median(tile_ms))}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--elements", type=int, default=1_000_000)
    ap.add_argument("--calls", type=int, default=42)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_elements: no CUDA device")
    codec = BatchCodec(0, int_optimized=True)
    out = {"card": card(), "runs": [run(codec, args.elements, args.calls, capi.METRIC_COUNTER, [capi.AGG_SUM]),
                                    run(codec, args.elements, args.calls, capi.METRIC_GAUGE,
                                        [capi.AGG_LAST, capi.AGG_MIN, capi.AGG_MAX])]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
