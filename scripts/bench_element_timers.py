#!/usr/bin/env python3
"""Timer element sets on the GPU (m3tsz_element_set_*_timer, DESIGN.md §4.12): ms per add, per consume and per minute of
ingest, in two shapes, with the C oracle (tests/timer_oracle.c, a CPU restatement of the reference's Timer, not the Go
reference) timed on every usable host core over the same windows.

  (a) downsampler-like: N timers, 1-minute windows, one sample per element per 10-second add, a consume every 6 adds,
      R = 2, for {Max, P50, P99} and for the default 11 types;
  (b) high-rate: 10 k timers, 6000 samples per window added as 60 batches of 100 (so the 1024-value insert / compress
      runs), R = 2; the largest list + pending count a slot reached is the sample_capacity a caller needs.

Sampled outputs are checked against the oracle.  Prints one JSON object; the card, its power limit and SM clock come
from the same run.

    python scripts/bench_element_timers.py [--n 1000000] [--minutes 3] [--out results/bench_element_timers.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from m3_b200 import capi  # noqa: E402
from m3_b200.codec import BatchCodec  # noqa: E402
import timer_oracle_lib as T  # noqa: E402

SEC = 1_000_000_000
RES = 60 * SEC
START = 1_600_000_020 * SEC


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def oracle_minute(vals, batch_len, types, eps, every, n_threads):
    """the C oracle over every window of one minute (vals [N, n] and batch_len [N, b]), on n_threads host threads
    -> (values [N, k], peaks [N], seconds)"""
    N, n = vals.shape
    v = np.ascontiguousarray(vals, dtype=np.float64).reshape(-1)
    v_off = np.arange(N + 1, dtype=np.uint64) * n
    bl = np.ascontiguousarray(batch_len, dtype=np.uint32).reshape(-1)
    b_off = np.arange(N + 1, dtype=np.uint64) * batch_len.shape[1]
    out = np.zeros((N, len(types)), dtype=np.float64)
    peak = np.zeros(N, dtype=np.int64)
    chunks = np.linspace(0, N, n_threads * 4 + 1).astype(int)
    t0 = time.perf_counter()
    with ThreadPoolExecutor(n_threads) as ex:  # (ctypes releases the GIL around each call)
        list(ex.map(lambda i: T.timer_windows(v, v_off, bl, b_off, types, eps, every, int(chunks[i]),
                                              int(chunks[i + 1]), out, peak), range(len(chunks) - 1)))
    return out, peak, time.perf_counter() - t0


def decoded_values(codec, es, N, k, cap):
    snap = es.stream()
    dec = codec.decode(snap.out.view(-1), es.out.offsets(), cap, lengths=snap.out_len)
    return dec.values.cpu().numpy().view(np.uint64), dec.n_points.cpu().numpy()


def shape_a(codec, N, types, minutes, n_threads):
    gen = torch.Generator(device="cuda").manual_seed(7)
    es = codec.element_set(torch.full((N,), START, dtype=torch.int64, device="cuda"), capi.METRIC_TIMER, types, RES,
                           open_windows=2, sample_capacity=8, stride=int(capi.lib().m3tsz_encode_bound_units(4, 1)))
    k = len(types)
    adds, cons, vals_all = [], [], []
    for mi in range(minutes + 1):  # minute 0 warms up
        es.reset(torch.full((N,), START + mi * RES, dtype=torch.int64, device="cuda"))
        mv = []
        for a in range(6):
            ts = torch.full((1, N), START + mi * RES + a * 10 * SEC, dtype=torch.int64, device="cuda")
            vs = torch.round(torch.rand((1, N), generator=gen, device="cuda", dtype=torch.float64) * 5000) / 10
            mv.append(vs)
            ms = timed(lambda: es.add(ts, vs))
            if mi:
                adds.append(ms)
        ms = timed(lambda: es.consume(START + (mi + 1) * RES))
        if mi:
            cons.append(ms)
            vals_all = torch.cat(mv, 0).t().contiguous().cpu().numpy()
    # the last minute: the oracle over the same windows, and sampled outputs against it
    bl = np.ones((N, 6), dtype=np.uint32)
    want, _, secs = oracle_minute(vals_all, bl, types, 1e-3, 1024, n_threads)
    got, npts = decoded_values(codec, es, N, k, 2)
    sample = np.random.default_rng(0).choice(N, min(N, 20000), replace=False)
    for j in range(k):
        rows = j * N + sample
        assert (npts[rows] == 1).all()
        assert (got[rows, 0] == want[sample, j].view(np.uint64)).all(), j
    add_ms, con_ms = float(np.median(adds)), float(np.median(cons))
    slot_bytes = 8 * (4 + 0) + 64 + 1 * 48  # per window: start, count, sum, sum_sq, header, one sample's entries
    return {"n": N, "types": types, "ms_per_add": add_ms, "ms_per_consume": con_ms,
            "ms_per_minute": 6 * add_ms + con_ms,
            "add_bytes": N * (16 + 2 * 32 + 64 * 2 + 48),  # inputs, slot scan of R = 2, header r/w, one entry
            "consume_bytes": N * (2 * 32 + 64 + 6 * 48 + k * 8 * 3),
            "oracle_s_per_minute": secs, "oracle_threads": n_threads, "sampled": int(len(sample)),
            "slot_bytes_approx": slot_bytes}


def shape_b(codec, types, n_threads, N=10_000, per_window=6000, batch=100, cap=8192):
    gen = torch.Generator(device="cuda").manual_seed(9)
    es = codec.element_set(torch.full((N,), START, dtype=torch.int64, device="cuda"), capi.METRIC_TIMER, types, RES,
                           open_windows=2, sample_capacity=cap, stride=int(capi.lib().m3tsz_encode_bound_units(4, 1)))
    k = len(types)
    marks = torch.ones((batch, N), dtype=torch.int8, device="cuda")
    marks[0] = 0
    adds, cons, peak = [], [], 0
    for mi in range(2):
        mv = []
        for a in range(per_window // batch):
            ts = torch.full((batch, N), START + mi * RES + a * SEC // 2, dtype=torch.int64, device="cuda")
            vs = torch.round(torch.rand((batch, N), generator=gen, device="cuda", dtype=torch.float64) ** 3 * 1e5) / 10
            mv.append(vs)
            ms = timed(lambda: es.add(ts, vs, batch=marks))
            if mi:
                adds.append(ms)
            h = es.streams["header"].view(torch.int32)  # n_samples at word 8, n_a / n_b at 12 / 13
            peak = max(peak, int((h[..., 8] + h[..., 12] + h[..., 13]).max()))
        ms = timed(lambda: es.consume(START + (mi + 1) * RES))
        if mi:
            cons.append(ms)
    vals = torch.cat(mv, 0).t().contiguous().cpu().numpy()
    bl = np.full((N, per_window // batch), batch, dtype=np.uint32)
    want, opeak, secs = oracle_minute(vals, bl, types, 1e-3, 1024, n_threads)
    got, npts = decoded_values(codec, es, N, k, 2)
    sample = np.random.default_rng(1).choice(N, 2000, replace=False)
    for j in range(k):
        rows = j * N + sample
        assert (got[rows, 1] == want[sample, j].view(np.uint64)).all(), j
    add_ms, con_ms = float(np.median(adds)), float(np.median(cons))
    return {"n": N, "types": types, "samples_per_window": per_window, "batch": batch,
            "ms_per_add": add_ms, "ms_per_consume": con_ms, "ms_per_minute": len(adds) * add_ms + con_ms,
            "peak_list_plus_pending": peak, "oracle_peak": int(opeak.max()),
            "input_bytes_per_minute": N * per_window * 17, "oracle_s_per_minute": secs, "oracle_threads": n_threads}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--minutes", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    codec = BatchCodec(0, int_optimized=False)  # (float encoding: the decoded values are the bits written)
    n_threads = len(os.sched_getaffinity(0))
    res = {"card": card(), "host_threads": n_threads}
    res["a_max_p50_p99"] = shape_a(codec, a.n, [capi.AGG_MAX, capi.AGG_P50, capi.AGG_P99], a.minutes, n_threads)
    res["a_default"] = shape_a(codec, a.n, list(capi.DEFAULT_TIMER_TYPES), a.minutes, n_threads)
    res["b_default"] = shape_b(codec, list(capi.DEFAULT_TIMER_TYPES), n_threads)
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
