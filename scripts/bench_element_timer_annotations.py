#!/usr/bin/env python3
"""Timer element sets that keep annotations against the plain Timer calls, one JSON line (card name, power limit and
max SM clock read in the same run).

Shapes: (a) of bench_element_timers.py, 1 M timers, one sample per timer per add call at a 10 s cadence, 1-minute
resolution, {Max, P50, P99}, R = 2 (a minute: 6 add calls and 1 consume); and the P99 -> {Max, P50, P99} rollups of
bench_element_timer_rollup.py, 10 000 groups x 100 contiguous sources and 100 000 groups x 10 random sources (a minute:
6 adds, 1 forward, 1 consume of the groups).  The annotated flow carries a 4-byte annotation on every sample; the plain
flow none.  The two flows alternate call by call in one process.

Reported: median ms per call of both flows; the device time per kernel over one more minute of each under
torch.profiler; the annotated flow's extra algorithmic bytes (formulas below); and, for every shape, a sample of the
output rows (elements' or groups') checked against the CPU model (tests/element_timer_ann_model.py).

    python scripts/bench_element_timer_annotations.py [--timers N] [--minutes N]
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
T0 = 1_600_000_020 * SEC
TYPES = [capi.AGG_MAX, capi.AGG_P50, capi.AGG_P99]
ANN = b"rt=1"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2] if xs else None


def every_sample_annotated(N, dev):
    """the sparse list with entry (0, 4, 0) for every element's one row, all pointing at the same 4 bytes"""
    off = torch.arange(N + 1, dtype=torch.int64, device=dev)
    ent = torch.zeros((N, 16), dtype=torch.uint8, device=dev)
    ent.view(torch.int32)[:, 1] = len(ANN)
    by = torch.tensor(list(ANN) + [0] * 4, dtype=torch.uint8, device=dev)
    return off, ent, by


class Flow:
    """one flow (annotated or plain): a set of N Timer elements fed one sample each per add call; with groups, a
    source set without output forwarded into a group set every minute"""

    def __init__(self, codec, N, annotated, groups=None):
        dev = codec.device
        self.annotated, self.N, self.groups = annotated, N, groups
        cap = 8 if annotated else 0
        start = torch.full((N,), T0, dtype=torch.int64, device=dev)
        if groups is None:
            self.es = codec.element_set(start, capi.METRIC_TIMER, TYPES, RES, open_windows=2, sample_capacity=16,
                                        annotation_capacity=cap)
        else:
            off, mem = groups
            self.off, self.mem = off, mem
            self.es = codec.element_set(start, capi.METRIC_TIMER, [capi.AGG_P99], RES, open_windows=2,
                                        sample_capacity=16, annotation_capacity=cap, stride=0)
            G = off.numel() - 1
            self.grp = codec.element_set(torch.full((G,), T0, dtype=torch.int64, device=dev), capi.METRIC_TIMER,
                                         TYPES, RES, open_windows=2, sample_capacity=int(N // G) * 2 + 8,
                                         annotation_capacity=cap)
        self.ann = every_sample_annotated(N, dev) if annotated else None
        g = torch.Generator(device=dev).manual_seed(7)
        self.vals = [torch.rand((1, N), generator=g, device=dev, dtype=torch.float64) * 100 for _ in range(6)]

    def add(self, minute, k):
        ts = torch.full((1, self.N), T0 + minute * RES + k * CADENCE, dtype=torch.int64, device=self.vals[0].device)
        return self.es.add(ts, self.vals[k], annotations=self.ann)

    def flush(self, minute):
        target = T0 + (minute + 1) * RES
        if self.groups is None:
            return self.es.consume(target)
        self.es.forward_timer(target, self.off, self.mem, self.grp)
        return self.grp.consume(target)


def time_call(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    return a, b


def run_shape(codec, name, N, minutes, groups=None):
    flows = {"annotated": Flow(codec, N, True, groups), "plain": Flow(codec, N, False, groups)}
    ev = {f: {"add": [], "flush": []} for f in flows}
    for minute in range(minutes):
        for k in range(6):
            for f, fl in flows.items():
                ev[f]["add"].append(time_call(lambda: fl.add(minute, k)))
        for f, fl in flows.items():
            ev[f]["flush"].append(time_call(lambda: fl.flush(minute)))
    torch.cuda.synchronize()
    out = {}
    for f in flows:
        for c, xs in ev[f].items():
            ms = [a.elapsed_time(b) for a, b in xs[6 if c == "add" else 1:]]  # (the first minute warms up)
            out["%s_%s_ms" % (f, c)] = median(ms)
        out["%s_minute_ms" % f] = 6 * out["%s_add_ms" % f] + out["%s_flush_ms" % f]
    # one more minute of each under the profiler: device time per kernel
    from torch.profiler import ProfilerActivity, profile
    for f, fl in flows.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for k in range(6):
                fl.add(minutes, k)
            fl.flush(minutes)
            torch.cuda.synchronize()
        out["%s_kernels_us" % f] = {e.key: round(e.device_time_total, 1) for e in prof.key_averages()
                                    if e.device_time_total > 0 and "element" in e.key}
    # extra algorithmic bytes of the annotated flow per minute: each add reads one 16-byte entry and its 8-byte series
    # offset and 4 annotation bytes per sample, and writes each open window's length (4) and one 8-byte word; each flush
    # reads a length per due window and stages one 16-byte entry per datapoint (+ 8-byte row offsets)
    rows = N if groups is None else groups[0].numel() - 1
    out["annotated_extra_bytes_per_minute"] = 6 * N * (16 + 8 + 4 + 4 + 8) + rows * len(TYPES) * (4 + 16 + 8)
    if groups is not None:
        out["annotated_extra_bytes_per_minute"] += N * (8 + 8) + rows * (4 + 8)  # forward refs, group slot copies
    out["checked"] = check_sample(flows["annotated"], minutes + 1)
    return {name: out}


def check_sample(flow, minutes):
    """a sample of the annotated flow's output rows against the CPU model, fed every sample of the run: 16 elements'
    rows, or for a rollup 4 groups' rows (their member sources modelled, forwarded into the group every minute)"""
    from element_timer_ann_model import AnnotatedTimerGroup, AnnotatedTimerModel, AnnotatedTimerSource, forward
    int_opt = flow.es.codec.int_optimized
    out_set = flow.es if flow.groups is None else flow.grp
    snap = out_set.stream()
    out, ln = snap.out.cpu().numpy(), snap.out_len.cpu().numpy()
    R = out_set.n_elements
    vals = [v.cpu().numpy()[0] for v in flow.vals]
    rng = np.random.default_rng(3)
    picks = rng.choice(R, 16 if flow.groups is None else 4, replace=False).tolist()
    off = mem = None
    if flow.groups is not None:
        off, mem = flow.off.cpu().numpy(), flow.mem.cpu().numpy()
    for e in picks:
        if flow.groups is None:
            m = AnnotatedTimerModel(TYPES, RES, (), False, 2, 16, capacity=8, start_ns=T0, int_optimized=int_opt)
            srcs, ids = [m], [e]
        else:
            members = mem[off[e]: off[e + 1]].tolist()
            ids = sorted(set(members))
            srcs = [AnnotatedTimerSource(capi.AGG_P99, RES, (), False, 2, 16, capacity=8) for _ in ids]
            m = AnnotatedTimerGroup(TYPES, RES, (), False, 2, flow.grp.sample_capacity, capacity=8, start_ns=T0,
                                    int_optimized=int_opt)
            local = [ids.index(x) for x in members]
        for minute in range(minutes):
            for k in range(6):
                for sm, x in zip(srcs, ids):
                    sm.add([(T0 + minute * RES + k * CADENCE, float(vals[k][x]))], None, [ANN])
            target = T0 + (minute + 1) * RES
            if flow.groups is not None:
                assert forward(srcs, [m], target, [0, len(local)], local) == ([0] * len(srcs), [0])
            m.consume(target)
        for j, want in enumerate(m.streams()):
            assert out[j * R + e, : ln[j * R + e]].tobytes() == want, (e, j)
    return len(picks)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--timers", type=int, default=1_000_000)
    ap.add_argument("--minutes", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    codec = BatchCodec(0, int_optimized=True)
    dev = codec.device
    N = a.timers
    res = {"card": card(), "timers": N, "minutes": a.minutes}
    res.update(run_shape(codec, "a_1M_max_p50_p99", N, a.minutes))
    G = N // 100
    contiguous = (torch.arange(G + 1, dtype=torch.int64, device=dev) * 100,
                  torch.arange(G * 100, dtype=torch.int32, device=dev))
    res.update(run_shape(codec, "rollup_%dx100_contiguous" % G, N, a.minutes, contiguous))
    G = N // 10
    g = torch.Generator(device=dev).manual_seed(5)
    rand = (torch.arange(G + 1, dtype=torch.int64, device=dev) * 10,
            torch.randint(0, N, (G * 10,), generator=g, device=dev, dtype=torch.int64).to(torch.int32))
    res.update(run_shape(codec, "rollup_%dx10_random" % G, N, a.minutes, rand))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
