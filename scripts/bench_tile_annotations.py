#!/usr/bin/env python3
"""Times tile aggregation that keeps annotations (m3tsz_aggregate_tiles_annotated) against the call without them.

  500 k series x 1440 datapoints, 5-minute windows (288): a Counter {Sum} (the counter-shaped batch of
  bench_aggregations.py) and a Gauge {Last, Min, Max} (the Gaussian walk), int-optimised.

Every series of the annotated sources carries an annotation.Payload on datapoint 0 only, as a Prometheus writer
leaves it (COUNTER with open_metrics_handle_value_resets / GAUGE); the plain sources are the same datapoints without
it.  Alternating within every round: the annotated sources through the new call and through
m3tsz_aggregate_tiles_types, and the plain sources through both.  Each call is timed with CUDA events; the median over
the rounds is reported.  Prints the card, its power limit and SM clocks, read in the same run, and checks a seeded
sample of the new call's outputs against the CPU oracle, and that on the plain sources both calls write the same rows.

    python scripts/bench_tile_annotations.py [--series 500000] [--points 1440] [--rounds 10] [--sample 32]
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

import ann_oracle_lib as N  # noqa: E402
import elem_oracle_lib as E  # noqa: E402
from bench_aggregations import card, counter_batch, timed  # noqa: E402
from m3_b200 import capi, synth  # noqa: E402
from m3_b200.codec import BatchCodec  # noqa: E402

SEC = 1_000_000_000
# annotation.Payload (fields 1 open_metrics_family_type, 2 open_metrics_handle_value_resets)
PAYLOAD = {"counter": bytes([0x08, 0x01, 0x10, 0x01]), "gauge": bytes([0x08, 0x02])}


def annotations_on_first(S, payload):
    """one annotation per series, on datapoint 0: (series_off, entries, bytes) for BatchCodec.encode"""
    off = torch.arange(S + 1, dtype=torch.int64, device="cuda")
    ent = np.zeros(1, dtype=[("dp", "<u4"), ("len", "<u4"), ("off", "<u8")])
    ent["len"] = len(payload)
    ent = torch.from_numpy(np.repeat(ent, S).view(np.uint8).reshape(S, 16)).cuda()
    return off, ent, torch.tensor(list(payload), dtype=torch.uint8, device="cuda")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=500_000)
    ap.add_argument("--points", type=int, default=1440)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--sample", type=int, default=32)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_tile_annotations.py needs a CUDA device")
    S, P, W, step = a.series, a.points, 288, 300 * SEC
    info = card()
    print("card (name, power limit, max SM clock, SM clock):", info)
    codec = BatchCodec(0, int_optimized=True)
    ts, gvals, start = synth.gaussian_walk(S, P, "cuda", seed=42)
    cvals = counter_batch(S, P, 43)
    s0 = int(start[0].item())
    batches = {}
    for name, vals in (("gauge", gvals), ("counter", cvals)):
        for ann in (True, False):
            enc = codec.encode(ts, vals, start, unit=capi.UNIT_S,
                               annotations=annotations_on_first(S, PAYLOAD[name]) if ann else None)
            assert int((enc.status != 0).sum()) == 0
            batches[(name, ann)] = codec.compact(enc, align=16)
            del enc
    del gvals, cvals, ts
    torch.cuda.empty_cache()

    cases = {"counter {Sum}": ("counter", capi.METRIC_COUNTER, [7]),
             "gauge {Last, Min, Max}": ("gauge", capi.METRIC_GAUGE, [1, 2, 3])}
    runs = {"annotated sources, annotated call": (True, True), "annotated sources, types call": (True, False),
            "plain sources, types call": (False, False), "plain sources, annotated call": (False, True)}
    out = {}

    def run(k, key):
        b, m, types = cases[k]
        src_ann, call_ann = runs[key]
        p_, o_ = batches[(b, src_ann)]
        out.clear()  # (the previous output back to the allocator first: one output of up to ~25 GB at a time)
        out[key] = codec.aggregate_tiles_types(p_, o_, s0, step, W, types, metric_type=m, annotations=call_ann)

    rng = np.random.default_rng(1234)
    sample = np.unique(rng.integers(0, S, a.sample))
    t, bad = {}, 0
    row = lambda r, j, s: r.packed[int(r.offsets[j, s]): int(r.offsets[j, s]) + int(r.out_len[j, s])].cpu() \
        .numpy().tobytes()
    for k, (b, m, types) in cases.items():
        keys = list(runs)
        for key in keys:  # warm-up: allocations, scratch, module load
            run(k, key)
            run(k, key)
        torch.cuda.synchronize()
        tk = timed(lambda key: run(k, key), a.rounds, keys)
        t.update({k + " | " + key: v for key, v in tk.items()})
        # ---- a seeded sample against the oracle; plain sources: both calls write the same rows ----
        p_, o_ = batches[(b, True)]
        ho = o_.cpu().numpy()
        run(k, "annotated sources, annotated call")
        r, nt = out["annotated sources, annotated call"]
        bad += int((r.status != 0).sum())
        for s in sample:
            src = p_[int(ho[s]): int(ho[s + 1])].cpu().numpy().tobytes()
            rows, counts, err = N.aggregate_tiles_annotated_series(src, True, s0, step, W, m, types, [], False,
                                                                   E.new_element_state())
            bad += int(err != 0)
            for j in range(len(types)):
                bad += int(row(r, j, s) != rows[j] or int(nt[j, s]) != counts[j])
        run(k, "plain sources, annotated call")
        ra = [[row(out["plain sources, annotated call"][0], j, s) for s in sample] for j in range(len(types))]
        run(k, "plain sources, types call")
        rb = [[row(out["plain sources, types call"][0], j, s) for s in sample] for j in range(len(types))]
        bad += int(ra != rb)
        out.clear()
        torch.cuda.empty_cache()

    res = {"card": info, "series": S, "points": P, "windows": W, "rounds": a.rounds, "results": {}}
    for key, ms in t.items():
        res["results"][key] = {"ms": ms}
        print("%-70s %8.3f ms" % (key, ms))
    res["sampled_series"] = int(len(sample))
    res["sample_mismatches"] = bad
    print("oracle check on %d sampled series: %s" %
          (len(sample), "all sampled outputs equal the oracle" if bad == 0 else "%d MISMATCHES" % bad))
    print(json.dumps(res))
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
