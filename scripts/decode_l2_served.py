"""Point-major decode at the bench shape (500 k x 1440, int-optimised, Gaussian walk), timed twice with the library
named by M3TSZ_B200_LIB (default: the in-tree build):

  normal     every series decodes its own segment, as bench.py's step does (streams read from HBM);
  l2_served  every series' (offset, length) points at one of the first N_HOT segments (N_HOT = 3000 by default,
             ~32 MB of streams, which stay resident in the 50 MB L2), so the reads are served from L2 while the
             11.5 GB of outputs are still written.

If l2_served is not clearly faster than normal, reading the streams is not what the decode kernel waits on.
Prints one JSON line with both times (CUDA events, mean of ROUNDS alternated windows of N launches) and the
card's name and power limit."""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from m3_b200 import capi, synth  # noqa: E402
from m3_b200.codec import BatchCodec, DecodeResult, EncodeResult  # noqa: E402

S = int(os.environ.get("S", 500_000))
P = 1440
N_HOT = int(os.environ.get("N_HOT", 3000))
N, ROUNDS = 10, 3


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "unknown (%s)" % e


def main():
    dev = torch.device("cuda", 0)
    codec = BatchCodec(0, int_optimized=True)
    ts, vals, start = synth.gaussian_walk(S, P, dev, seed=1000)
    stride = ((64 + 9 * P) + 63) // 64 * 64  # bench.py's segment stride
    enc = EncodeResult(out=torch.empty((S, stride), dtype=torch.uint8, device=dev),
                       out_len=torch.empty(S, dtype=torch.int64, device=dev),
                       status=torch.empty(S, dtype=torch.int32, device=dev))
    ts_pm, vals_pm = ts.t().contiguous(), vals.t().contiguous()
    del ts, vals
    codec.encode(ts_pm, vals_pm, start, unit=1, out=enc, point_major=True)
    del vals_pm
    seg_flat = enc.out.view(-1)
    seg_off = torch.arange(S, dtype=torch.int64, device=dev) * stride
    hot = torch.arange(S, dtype=torch.int64, device=dev) % N_HOT
    hot_off, hot_len = seg_off[hot].contiguous(), enc.out_len[hot].contiguous()
    dec = DecodeResult(ts=torch.empty((P, S), dtype=torch.int64, device=dev),
                       values=torch.empty((P, S), dtype=torch.float64, device=dev),
                       n_points=torch.empty(S, dtype=torch.int32, device=dev),
                       status=torch.empty(S, dtype=torch.int32, device=dev),
                       unit=torch.empty(S, dtype=torch.uint8, device=dev), annotations=None)
    runs = {
        "normal": lambda: codec.decode(seg_flat, seg_off, P, out=dec, lengths=enc.out_len, point_major=True),
        "l2_served": lambda: codec.decode(seg_flat, hot_off, P, out=dec, lengths=hot_len, point_major=True),
    }
    for fn in runs.values():
        fn()
        fn()
    torch.cuda.synchronize()
    ok = bool(torch.equal(dec.ts[:, :N_HOT], ts_pm[:, :N_HOT])) and int((dec.status != 0).sum()) == 0
    ms = {k: [] for k in runs}
    for _ in range(ROUNDS):
        for k, fn in runs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(N):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1) / N)
    print(json.dumps({"lib": capi.LIB_PATH, "card": card(), "series": S, "points": P, "hot_segments": N_HOT,
                      "hot_stream_bytes": int(hot_len[:N_HOT].sum().item()),
                      "stream_bytes": int(enc.out_len.sum().item()), "l2_run_decodes_ok": ok,
                      "normal_ms": [round(x, 4) for x in ms["normal"]],
                      "l2_served_ms": [round(x, 4) for x in ms["l2_served"]]}))


if __name__ == "__main__":
    main()
