#!/usr/bin/env python3
"""Times tile aggregation of an element with several aggregation types against the single-type calls it replaces.

  500 k series x 1440 datapoints, 5-minute windows (288): the int-optimised Gaussian-walk batch and the
  counter-shaped batch of bench_aggregations.py.

Alternating within every round: one m3tsz_aggregate_tiles_types call (one decode + windows, one encode launch over
k x S rows) against the k single-type calls (m3tsz_aggregate_tiles_ex, or m3tsz_aggregate_tiles_transform with ops)
that write the same rows.  Cases: Gauge {Last, Min, Max, Mean, Sum}; Counter {Min, Max, Sum}; Gauge {Min, Max, Sum}
with [Add], where the single-type calls keep one sum per type and so write different values: only the time compares.
A call with ops includes zeroing its state (every round starts new elements).  Each call is timed with CUDA events;
the median over the rounds is reported.  Prints the card, its power limit and SM clocks, read in the same run, and
checks a seeded sample of every multi-type output (bytes, tile counts, status and saved record) against the CPU
oracle, and of the single-type calls without Add against the multi-type rows.

    python scripts/bench_tile_types.py [--series 500000] [--points 1440] [--rounds 10] [--sample 32]
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

import elem_oracle_lib as E  # noqa: E402
import oracle_lib as O  # noqa: E402
from bench_aggregations import card, counter_batch, timed  # noqa: E402
from m3_b200 import capi, synth  # noqa: E402
from m3_b200.codec import BatchCodec  # noqa: E402

SEC = 1_000_000_000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=500_000)
    ap.add_argument("--points", type=int, default=1440)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--sample", type=int, default=32)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_tile_types.py needs a CUDA device")
    S, P, W, step = a.series, a.points, 288, 300 * SEC
    info = card()
    print("card (name, power limit, max SM clock, SM clock):", info)
    codec = BatchCodec(0, int_optimized=True)
    ts, gvals, start = synth.gaussian_walk(S, P, "cuda", seed=42)
    cvals = counter_batch(S, P, 43)
    s0 = int(start[0].item())
    batches = {}
    for name, vals in (("gauge", gvals), ("counter", cvals)):
        enc = codec.encode(ts, vals, start, unit=capi.UNIT_S)
        assert int((enc.status != 0).sum()) == 0
        packed, off = codec.compact(enc, align=16)
        del enc
        batches[name] = (packed, off)
    del gvals, cvals, ts
    torch.cuda.empty_cache()

    G, C_ = capi.METRIC_GAUGE, capi.METRIC_COUNTER
    cases = {
        "gauge {Last, Min, Max, Mean, Sum}": ("gauge", G, [1, 2, 3, 4, 7], []),
        "counter {Min, Max, Sum}": ("counter", C_, [2, 3, 7], []),
        "gauge {Min, Max, Sum} + [Add]": ("gauge", G, [2, 3, 7], [capi.TRANSFORM_ADD]),
    }
    res_multi, res_single = {}, {}
    el_state = {k: codec.element_state(S) for k, c in cases.items() if c[3]}
    xf_state = {k: [codec.transform_state(S) for _ in c[2]] for k, c in cases.items() if c[3]}

    def copy_sample(k, sample):
        """the sampled series' rows of both ways, on the host"""
        types = cases[k][2]
        r, nt = res_multi[k]
        of, ln = r.offsets.cpu().numpy(), r.out_len.cpu().numpy()
        st, ntc = r.status.cpu().numpy(), nt.cpu().numpy()
        row = lambda pk, o, n: pk[int(o): int(o) + int(n)].cpu().numpy().tobytes()
        multi_rows = [[(row(r.packed, of[j, s], ln[j, s]), int(st[j, s]), int(ntc[j, s])) for s in sample]
                      for j in range(len(types))]
        single_rows = []
        for rs, _ in res_single[k]:
            os_, ls = rs.offsets.cpu().numpy(), rs.out_len.cpu().numpy()
            single_rows.append([row(rs.packed, os_[s], ls[s]) for s in sample])
        return multi_rows, single_rows

    def multi(k):
        b, m, types, ops = cases[k]
        p_, o_ = batches[b]
        st = el_state.get(k)
        if st is not None:
            st.zero_()
        res_multi.pop(k, None)  # (its buffer back to the allocator first)
        res_multi[k] = codec.aggregate_tiles_types(p_, o_, s0, step, W, types, metric_type=m, transforms=ops,
                                                   state=st)

    def single(k):
        b, m, types, ops = cases[k]
        p_, o_ = batches[b]
        prev = res_single.get(k)
        outs = []
        for j, agg in enumerate(types):
            st = xf_state[k][j] if ops else None
            if st is not None:
                st.zero_()
            outs.append(codec.aggregate_tiles(p_, o_, s0, step, W, agg_type=agg, metric_type=m, transforms=ops,
                                              state=st, out=prev[j][0] if prev else None))
        res_single[k] = outs

    # one case at a time (its outputs take up to ~25 GB), the two ways alternating within every round
    fns, t = {}, {}
    rng = np.random.default_rng(1234)
    sample = np.unique(rng.integers(0, S, a.sample))
    checked = {}
    for k in cases:
        keys = [k + " | one call", k + " | k single calls"]
        fns[keys[0]] = (lambda k=k: multi(k))
        fns[keys[1]] = (lambda k=k: single(k))
        for key in keys:  # warm-up: allocations, scratch, module load
            fns[key]()
            fns[key]()
        torch.cuda.synchronize()
        t.update(timed(lambda key: fns[key](), a.rounds, keys))
        checked[k] = copy_sample(k, sample)
        res_multi.pop(k)
        res_single.pop(k)
        torch.cuda.empty_cache()

    res = {"card": info, "series": S, "points": P, "windows": W, "rounds": a.rounds, "results": {}}
    for key, ms in t.items():
        res["results"][key] = {"ms": ms, "G_dp_per_s": S * P / ms / 1e6}
        print("%-50s %8.3f ms  %6.2f G source dp/s" % (key, ms, S * P / ms / 1e6))
    for k in cases:
        r = t[k + " | k single calls"] / t[k + " | one call"]
        res["results"][k + " | speedup"] = r
        print("%-50s %8.2fx" % (k + " | one call vs k calls", r))

    # ---- a seeded sample of every output against the oracle ----
    bad = 0
    host = {}
    for name, (p_, o_) in batches.items():
        ho = o_.cpu().numpy()
        hp = p_[: int(ho[-1])].cpu().numpy()
        host[name] = [O.decode_series(hp[ho[s]: ho[s + 1]].tobytes(), True, cap=P + 1) for s in sample]
    for k, (b, m, types, ops) in cases.items():
        multi_rows, single_rows = checked[k]
        rec = el_state[k].cpu().numpy().view(E.ELEM_STATE_DTYPE).reshape(-1) if ops else None
        for i, s in enumerate(sample):
            src = host[b][i]
            bad += int(src[3] != 0)
            est = E.new_element_state()
            rows = E.aggregate_tiles_types_series(src[0][:src[2]], src[1][:src[2]], s0, step, W, m, types, ops,
                                                  len(ops) > 0, est)
            for j, (tts, tv) in enumerate(rows):
                exp = O.encode_series(tts, tv, s0, O.UNIT_S, True) if len(tts) else b""
                got, st_, nt_ = multi_rows[j][i]
                bad += int(got != exp or st_ != 0 or nt_ != len(tts))
                if not ops:  # the single-type calls write the same rows
                    bad += int(single_rows[j][i] != got)
            if rec is not None:
                bad += int(rec[s: s + 1].tobytes() != est.tobytes())
    res["sampled_series"] = int(len(sample))
    res["sample_mismatches"] = bad
    print("oracle check on %d sampled series x every output: %s" %
          (len(sample), "all sampled outputs equal the oracle" if bad == 0 else "%d MISMATCHES" % bad))
    print(json.dumps(res))
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
