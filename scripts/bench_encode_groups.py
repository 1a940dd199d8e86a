#!/usr/bin/env python3
"""Times the point-major encode at the bench shape (500 k series x 1440 points, Gaussian walk, int-optimised,
out_stride as bench.py sizes it) three ways, and prints one JSON line:

  seq_encode_ms   encode inside a sustained encode -> decode sequence (30 pairs, CUDA events around each encode)
  b2b_encode_ms   30 encodes back to back
  decode_ms       the point-major decode inside the same sequence

beside the card's name, its power limit and the SM clock sampled during the runs.  One build per process: pick it
with M3TSZ_B200_LIB, and alternate the builds from the shell to compare them.

    M3TSZ_B200_LIB=/path/to/libm3tsz_b200.so python scripts/bench_encode_groups.py [--series N] [--reps 30]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def smi(query):
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + query, "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=500_000)
    ap.add_argument("--points", type=int, default=1440)
    ap.add_argument("--reps", type=int, default=30)
    a = ap.parse_args()

    import torch
    from bench import ClockSampler
    from m3_b200 import capi, synth
    from m3_b200.codec import BatchCodec, DecodeResult, EncodeResult

    S, P = a.series, a.points
    dev = torch.device("cuda", 0)
    codec = BatchCodec(0, int_optimized=True)
    ts, vals, start = synth.gaussian_walk(S, P, dev, seed=1000)
    ts_pm, vals_pm = ts.t().contiguous(), vals.t().contiguous()
    del ts, vals
    stride = ((64 + 9 * P) + 63) // 64 * 64
    enc = EncodeResult(out=torch.empty((S, stride), dtype=torch.uint8, device=dev),
                       out_len=torch.empty(S, dtype=torch.int64, device=dev),
                       status=torch.empty(S, dtype=torch.int32, device=dev))
    seg_off = torch.arange(S, dtype=torch.int64, device=dev) * stride
    dec = DecodeResult(ts=torch.empty((P, S), dtype=torch.int64, device=dev),
                       values=torch.empty((P, S), dtype=torch.float64, device=dev),
                       n_points=torch.empty(S, dtype=torch.int32, device=dev),
                       status=torch.empty(S, dtype=torch.int32, device=dev),
                       unit=torch.empty(S, dtype=torch.uint8, device=dev), annotations=None)
    encode = lambda: codec.encode(ts_pm, vals_pm, start, unit=1, out=enc, point_major=True)
    decode = lambda: codec.decode(enc.out.view(-1), seg_off, P, out=dec, lengths=enc.out_len, point_major=True)
    ev = lambda: torch.cuda.Event(enable_timing=True)

    for _ in range(3):
        encode()
        decode()
    torch.cuda.synchronize()
    assert int((enc.status != 0).sum()) == 0 and int((dec.status != 0).sum()) == 0
    assert torch.equal(dec.ts, ts_pm)
    out_bytes = int(enc.out_len.sum().item())

    sampler = ClockSampler(0)
    sampler.start()
    pairs = []
    for _ in range(a.reps):
        e = [ev() for _ in range(3)]
        e[0].record()
        encode()
        e[1].record()
        decode()
        e[2].record()
        pairs.append(e)
    torch.cuda.synchronize()
    seq_enc = sorted(x[0].elapsed_time(x[1]) for x in pairs)
    seq_dec = sorted(x[1].elapsed_time(x[2]) for x in pairs)
    b0, b1 = ev(), ev()
    b0.record()
    for _ in range(a.reps):
        encode()
    b1.record()
    torch.cuda.synchronize()
    clocks = sampler.stop()

    med = lambda xs: xs[len(xs) // 2]
    print(json.dumps({
        "lib": capi.LIB_PATH, "gpu": torch.cuda.get_device_name(0), "power_limit": smi("power.limit"),
        "sm_mhz_median": clocks.get("sm_mhz"), "sm_max_mhz": clocks.get("sm_max_mhz"),
        "throttle": clocks.get("reasons"), "series": S, "points": P, "out_bytes": out_bytes,
        "seq_encode_ms": round(sum(seq_enc) / len(seq_enc), 3), "seq_encode_median_ms": round(med(seq_enc), 3),
        "b2b_encode_ms": round(b0.elapsed_time(b1) / a.reps, 3),
        "decode_ms": round(sum(seq_dec) / len(seq_dec), 3)}))


if __name__ == "__main__":
    main()
