#!/usr/bin/env python3
"""Times tile aggregation across source blocks (m3tsz_aggregate_tiles_blocks) against the ways to get the same
outputs without it.

  500 k series, 1 datapoint a minute over 24 h as 12 two-hour source blocks of 120 datapoints, 5-minute windows
  (288), int-optimised: a Counter {Sum} (the counter-shaped batch of bench_aggregations.py) and a Gauge {Last, Min,
  Max} (the Gaussian walk), each without and with annotations (an annotation.Payload on every block's first
  datapoint, as each block's Prometheus writer leaves it).

  (a) the blocks call over the 12 block streams of every series;
  (b) m3tsz_aggregate_tiles_types on one pre-concatenated stream per series that encodes the blocks' decoded
      datapoints (the payload on datapoint 0, which is what one stream holds of twelve equal payloads).  It is made
      from the decoded blocks, not from the generator's values: the int-optimised value diffs are float64 sums, so a
      stream over 1440 datapoints can decode the Counter batch's 3e18 values differently from twelve 120-datapoint
      streams;
  (c) without annotations only, the route without the blocks call: decode the 12 blocks, merge_series with one
      replica of 12 slices, encode one stream per series, then m3tsz_aggregate_tiles_types.

One process, alternating within every round; each call is timed with CUDA events and the median over the rounds is
reported.  Prints the card, its power limit and SM clocks, read in the same run.  Checks that without annotations (a),
(b) and (c) write the same bytes on every row, and with annotations (a) against (b) on every row (equal here: all
payloads of a series are the same bytes).

    python scripts/bench_tile_blocks.py [--series 500000] [--rounds 10]
"""
import argparse
import json
import os
import sys
from types import SimpleNamespace

# route (c) allocates and frees tens of GB per round: keep the allocator from fragmenting
os.environ.setdefault("PYTORCH_CUDA_ALLOC_CONF", "expandable_segments:True")
import torch  # noqa: E402

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_aggregations import card, counter_batch, timed  # noqa: E402
from bench_tile_annotations import PAYLOAD, annotations_on_first  # noqa: E402
from m3_b200 import capi, synth  # noqa: E402
from m3_b200.codec import BatchCodec  # noqa: E402

SEC = 1_000_000_000
NB, PB = 12, 120


def block_inputs(codec, ts, vals, payload):
    """the 12 block streams of every series -> (blob, offsets, lengths, blocks), segment s * 12 + b"""
    S = ts.shape[0]
    parts = []
    for b in range(NB):
        sl = slice(b * PB, (b + 1) * PB)
        enc = codec.encode(ts[:, sl].contiguous(), vals[:, sl].contiguous(), ts[:, b * PB].contiguous(),
                           unit=capi.UNIT_S, annotations=annotations_on_first(S, payload) if payload else None)
        assert int((enc.status != 0).sum()) == 0
        parts.append(codec.compact(enc, align=16))
        del enc
    base, pos = [], 0
    for p_, _ in parts:
        base.append(pos)
        pos += (p_.numel() + 15) // 16 * 16
    blob = torch.zeros(pos + 16, dtype=torch.uint8, device="cuda")
    for (p_, _), b0 in zip(parts, base):
        blob[b0: b0 + p_.numel()] = p_
    off = torch.stack([o[:-1] + b0 for (_, o), b0 in zip(parts, base)], dim=1).reshape(-1).contiguous()
    lengths = torch.stack([o[1:] - o[:-1] for _, o in parts], dim=1).reshape(-1).contiguous()
    blocks = torch.arange(S + 1, dtype=torch.int64, device="cuda") * NB
    return blob, off, lengths, blocks


def concat_stream(codec, blocks_input, S, start, payload=None):
    """route (c) up to the tile call: decode the 12 blocks, merge them (one replica of 12 slices), encode one stream
    per series -> (packed, offsets)"""
    blob, off, lengths, _ = blocks_input
    d = codec.decode(blob, off, PB, lengths=lengths)
    one = torch.arange(S * NB + 1, dtype=torch.int64, device="cuda")
    t_m, v_m, n_m, _ = codec.merge_series(d.ts, d.values, d.n_points, d.status, one, one[::NB].contiguous(),
                                          torch.arange(S + 1, dtype=torch.int64, device="cuda"), NB * PB)
    del d
    enc = codec.encode(t_m, v_m, start, unit=capi.UNIT_S, n_points=n_m,
                       annotations=annotations_on_first(S, payload) if payload else None)
    del t_m, v_m
    assert int((enc.status != 0).sum()) == 0
    return codec.compact(enc, align=16)


def first_different_row(ra, rb, chunk=65536):
    """the first row whose bytes differ (the packed layouts may differ), compared a chunk of rows at a time; -1: none"""
    la, lb = ra.out_len.reshape(-1), rb.out_len.reshape(-1)
    if not torch.equal(la, lb):
        return int(torch.nonzero(la != lb)[0].item())
    oa, ob = ra.offsets.reshape(-1), rb.offsets.reshape(-1)
    for i in range(0, la.numel(), chunk):
        ln = la[i: i + chunk]
        n = int(ln.sum().item())
        row = torch.repeat_interleave(torch.arange(ln.numel(), device="cuda"), ln)
        within = torch.arange(n, device="cuda") - torch.repeat_interleave(torch.cumsum(ln, 0) - ln, ln)
        ne = ra.packed[torch.repeat_interleave(oa[i: i + chunk], ln) + within] != \
            rb.packed[torch.repeat_interleave(ob[i: i + chunk], ln) + within]
        if bool(ne.any()):
            return i + int(row[torch.nonzero(ne)[0]].item())
    return -1


def row_bytes(r, q):
    o, n = int(r.offsets.reshape(-1)[q]), int(r.out_len.reshape(-1)[q])
    return r.packed[o: o + n].cpu().numpy().tobytes()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=500_000)
    ap.add_argument("--rounds", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_tile_blocks.py needs a CUDA device")
    S, P, W, step = a.series, NB * PB, 288, 300 * SEC
    info = card()
    print("card (name, power limit, max SM clock, SM clock):", info)
    codec = BatchCodec(0, int_optimized=True)
    ts, gvals, start = synth.gaussian_walk(S, P, "cuda", seed=42)
    cvals = counter_batch(S, P, 43)
    s0 = int(start[0].item())
    inputs = {}
    for name, vals in (("gauge", gvals), ("counter", cvals)):
        for ann in (False, True):
            pl = PAYLOAD[name] if ann else None
            inputs[(name, ann, "blocks")] = block_inputs(codec, ts, vals, pl)
    del gvals, cvals
    torch.cuda.empty_cache()
    for name in ("gauge", "counter"):
        for ann in (False, True):
            inputs[(name, ann, "concat")] = concat_stream(codec, inputs[(name, ann, "blocks")], S, start,
                                                          PAYLOAD[name] if ann else None)
    del ts
    torch.cuda.empty_cache()

    cases = {"counter {Sum}": ("counter", capi.METRIC_COUNTER, [7]),
             "gauge {Last, Min, Max}": ("gauge", capi.METRIC_GAUGE, [1, 2, 3])}
    out = {}

    def run(case, ann, way):
        name, m, types = cases[case]
        out.clear()  # (the previous output back to the allocator first)
        if way == "a":
            blob, off, lengths, blocks = inputs[(name, ann, "blocks")]
            out[way] = codec.aggregate_tiles_types(blob, off, s0, step, W, types, metric_type=m, lengths=lengths,
                                                   annotations=ann, blocks=blocks)
        elif way == "b":
            p_, o_ = inputs[(name, ann, "concat")]
            out[way] = codec.aggregate_tiles_types(p_, o_, s0, step, W, types, metric_type=m, annotations=ann)
        else:
            p_, o_ = concat_stream(codec, inputs[(name, False, "blocks")], S, start)
            out[way] = codec.aggregate_tiles_types(p_, o_, s0, step, W, types, metric_type=m)

    t, bad = {}, 0
    for case in cases:
        for ann in (False, True):
            ways = ["a", "b"] + ([] if ann else ["c"])
            for w in ways:  # warm-up: allocations, scratch, module load
                run(case, ann, w)
                run(case, ann, w)
            torch.cuda.synchronize()
            tk = timed(lambda w: run(case, ann, w), a.rounds, ways)
            label = "%s, %s" % (case, "annotations" if ann else "no annotations")
            t.update({label + " | " + w: v for w, v in tk.items()})
            run(case, ann, "a")
            r, nt_a = out.pop("a")
            # (a)'s rows, moved out of its packed buffer (sized for the bound) so that route (c) has room
            ref = SimpleNamespace(packed=r.packed[: int(r.total.item())].clone(), offsets=r.offsets.clone(),
                                  out_len=r.out_len.clone(), status=r.status.clone())
            del r
            bad += int((ref.status != 0).sum())
            for w in ways[1:]:
                run(case, ann, w)
                r, nt = out[w]
                q = first_different_row(ref, r)
                ok = bool((r.status == 0).all()) and torch.equal(nt, nt_a) and q < 0
                print("%s: (a) and (%s) write %s" % (label, w, "the same rows" if ok else "DIFFERENT rows"))
                if not ok:
                    print("  status (a) %s, (%s) %s; n_tiles equal: %s; first different row %d" % (
                        torch.unique(ref.status).tolist(), w, torch.unique(r.status).tolist(),
                        torch.equal(nt, nt_a), q))
                    if q >= 0:
                        print("  (a) %s\n  (%s) %s" % (row_bytes(ref, q).hex(), w, row_bytes(r, q).hex()))
                bad += int(not ok)
            out.clear()
            del ref
            torch.cuda.empty_cache()

    res = {"card": info, "series": S, "blocks": NB, "points_per_block": PB, "windows": W, "rounds": a.rounds,
           "results": {}}
    for key, ms in t.items():
        res["results"][key] = {"ms": ms}
        print("%-75s %8.3f ms" % (key, ms))
    res["mismatches"] = bad
    print(json.dumps(res))
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
