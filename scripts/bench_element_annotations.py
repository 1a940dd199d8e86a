#!/usr/bin/env python3
"""Element sets that keep annotations (m3tsz_element_set_add_annotated / _consume_annotated) against the plain calls
and against the route the library offered before them, one JSON line (card name and power limit read in the same
run).

The shape of scripts/bench_elements.py: 1 M elements, one datapoint per element per add call at a 10 s cadence,
1-minute resolution, a consume at every 6th call.  Every datapoint carries a Prometheus-sized annotation (the 4-byte
annotation.Payload of a counter that handles value resets, the 2-byte one of a gauge), as the downsampler passes one
with every sample.  Three flows run alternating call by call in one process:
  - plain: an element set without annotations (the datapoints only);
  - annotated: an element set with an annotation capacity of 8 bytes per window slot, given the annotations;
  - route: EncoderSet.append of the same datapoints with their annotations, and at each flush stream() +
    aggregate_tiles_types(annotations=True) over the snapshot for the minute that ended.

Reported: median ms per add and per consume of each flow, per call of the route, per minute (six adds and one
consume), and the algorithmic bytes each call moves (from the shapes, the formulas below).

    python scripts/bench_element_annotations.py [--elements N] [--calls N]
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
from m3_b200.codec import BatchCodec  # noqa: E402

SEC = 1_000_000_000
RES = 60 * SEC
CADENCE = 10 * SEC
T0 = 1_600_000_020 * SEC  # a whole minute
PAYLOAD = {capi.METRIC_COUNTER: bytes([0x08, 0x01, 0x10, 0x01]), capi.METRIC_GAUGE: bytes([0x08, 0x02])}


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


def every_datapoint(N, payload, dev):
    """the sparse annotation list of one datapoint per element, each carrying `payload`"""
    off = torch.arange(N + 1, dtype=torch.int64, device=dev)
    ent = np.zeros(N, dtype=[("dp_index", "<u4"), ("length", "<u4"), ("byte_offset", "<u8")])
    ent["length"] = len(payload)
    ent = torch.from_numpy(ent.view(np.uint8).reshape(N, 16)).to(dev)
    return off, ent, torch.tensor(list(payload), dtype=torch.uint8, device=dev)


def run(codec, N, calls, metric, types):
    dev = "cuda"
    k = len(types)
    gauge = metric == capi.METRIC_GAUGE
    payload = PAYLOAD[metric]
    start = torch.full((N,), T0, dtype=torch.int64, device=dev)
    offs = (torch.arange(N, device=dev) % 10) * SEC
    gen = torch.Generator(device=dev).manual_seed(3)
    flushes = calls // 6
    # room for every flush with its annotation at the append's own count ((len + 3) / 4 + 4 words per datapoint)
    stride = int(capi.lib().m3tsz_encode_bound_units(2 * flushes + 2, 1)) + 16 * (2 * flushes + 2) * 4
    plain = codec.element_set(start, metric, types, RES, open_windows=2, stride=stride)
    ann = codec.element_set(start, metric, types, RES, open_windows=2, stride=stride, annotation_capacity=8)
    enc = codec.encoder_set(start, codec.encode_bound(calls) + 32 * calls)
    state = codec.element_state(N)
    a_in = every_datapoint(N, payload, dev)
    t = {f: [] for f in ("plain_add", "ann_add", "plain_consume", "ann_consume", "route_append", "route_flush")}
    level = torch.zeros(N, dtype=torch.float64, device=dev)
    for i in range(calls):
        ts = (T0 + i * CADENCE + offs).view(1, N).contiguous()
        step = torch.randn(N, dtype=torch.float64, device=dev, generator=gen)
        level = level + (step if gauge else step.abs().round())
        vals = level.view(1, N).contiguous()
        # (one datapoint per element: [1, N] point-major is [N, 1] series-major, which the public append takes with
        # annotations)
        t["plain_add"].append(timed(lambda: plain.add(ts, vals)))
        t["ann_add"].append(timed(lambda: ann.add(ts, vals, annotations=a_in)))
        t["route_append"].append(timed(lambda: enc.append(ts.view(N, 1), vals.view(N, 1), annotations=a_in)))
        if (i + 1) % 6 == 0:
            target = T0 + (i + 1) // 6 * RES
            t["plain_consume"].append(timed(lambda: plain.consume(target)))
            t["ann_consume"].append(timed(lambda: ann.consume(target)))

            def tiles():
                snap = enc.stream()
                codec.aggregate_tiles_types(snap.out.view(-1), enc.offsets(), target - RES, RES, 1, types,
                                            metric_type=metric, lengths=snap.out_len, state=state,
                                            discard_nan=False, annotations=True)
            t["route_flush"].append(timed(tiles))
    torch.cuda.synchronize()
    for es in (plain, ann):
        assert int(es.watermark.min()) == T0 + flushes * RES, "a consume was refused"
    assert torch.equal(plain.elem, ann.elem)
    med = {f: median([a.elapsed_time(b) for a, b in evs[1:]]) for f, evs in t.items()}  # (first of each: warm-up)

    # algorithmic bytes.  plain add: as scripts/bench_elements.py.  The annotated add adds the list's offsets (2 x 8)
    # and entry (16), the payload read, and the slot's length (4) and bytes (8) written once per call.
    fields = 8 if gauge else 6
    plain_add_b = N * (16 + 8 + 16 * 2 + 2 * 8 * fields + 1 + 4)
    ann_add_b = plain_add_b + N * (16 + 16 + len(payload) + 4 + 8)
    # consume: as scripts/bench_elements.py; annotated, also the slot's length (4), per type the row's offset and
    # entry written and read back (2 x 24) and the slot's bytes read by the append (8)
    plain_cons_b = N * (16 * 2 + 8 * fields + 8 + 2 * 160 + 16 + k * (32 + 8 + 256 + 8 + 8) + 8)
    ann_cons_b = plain_cons_b + N * (4 + k * (2 * 24 + 8))
    route_app_b = N * (2 * 128 + 16 + 4 + 16 + 16 + len(payload))
    r = lambda x: None if x is None else round(x, 4)
    return {"metric": "gauge" if gauge else "counter", "types": types, "elements": N, "calls": calls,
            "payload_bytes": len(payload),
            "median_ms": {f: r(v) for f, v in med.items()},
            "bytes": {"plain_add": plain_add_b, "ann_add": ann_add_b, "plain_consume": plain_cons_b,
                      "ann_consume": ann_cons_b, "route_append": route_app_b},
            "per_minute_ms": {"plain": r(6 * med["plain_add"] + med["plain_consume"]),
                              "annotated": r(6 * med["ann_add"] + med["ann_consume"]),
                              "route_annotated": r(6 * med["route_append"] + med["route_flush"])}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--elements", type=int, default=1_000_000)
    ap.add_argument("--calls", type=int, default=42)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_element_annotations: no CUDA device")
    codec = BatchCodec(0, int_optimized=True)
    out = {"card": card(), "runs": [run(codec, args.elements, args.calls, capi.METRIC_COUNTER, [capi.AGG_SUM]),
                                    run(codec, args.elements, args.calls, capi.METRIC_GAUGE,
                                        [capi.AGG_LAST, capi.AGG_MIN, capi.AGG_MAX])]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
