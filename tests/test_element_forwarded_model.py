"""The cross-shard rollup model (tests/element_forwarded_model.py): it reproduces the reference's AddUnique and
forwarded-writer goldens (tests/golden/m3tsz_forwarded_goldens.json); with one shard and its records in group order
it is the element rollup model's forward; split over several shards whose records arrive in any order it gives the same
group windows; a redelivered batch changes nothing; and both capacity stops recover by grow-and-resend, of exactly
the refused records or of the whole batch."""
import copy
import json
import math
import os

import numpy as np
import pytest

import agg_oracle_lib as A
from element_forwarded_model import (ERR_CAPACITY, ERR_CLOSED, ERR_DUPLICATE_SOURCE, ERR_INVALID_ARG, OK,
                                     ForwardedGroupModel, SourceModel, add_forwarded, forward_write, write_buckets)
from element_rollup_model import GroupModel, forward

SEC = 1_000_000_000
RES = 60 * SEC
START = 1_600_000_020 * SEC
GAUGE, COUNTER = A.METRIC_GAUGE, A.METRIC_COUNTER
LAST, SUM = 1, 7


def _bits(v):
    return int(np.array([v], dtype=np.float64).view(np.uint64)[0])


def _world(rng, metric, S=30, G=7, W=4, nan=False):
    src_type = SUM if metric == COUNTER else LAST
    srcs = [SourceModel(metric, src_type, RES, open_windows=8) for _ in range(S)]
    for s in srcs:
        pts = []
        for w in range(W):
            if rng.random() < 0.3:
                continue
            v = float("nan") if nan and rng.random() < 0.2 else float(rng.integers(0, 100))
            pts.append((START + w * RES + int(rng.integers(0, 60)) * SEC, _bits(v)))
        s.add(pts)
    n = G * 5
    off = list(range(0, n + 1, 5))
    mem = [int(m) for m in rng.integers(0, S, n)]
    return srcs, off, mem, W


def _groups(metric, G, R=8, cap=64, fwd=True):
    cls = ForwardedGroupModel if fwd else GroupModel
    kw = {"source_capacity": cap} if fwd else {}
    return [cls(metric, [SUM], RES, open_windows=R, **kw) for _ in range(G)]


def _windows(groups):
    return [{ws: list(map(repr, v)) for ws, v in g.windows.items()} for g in groups]


def _shards(srcs, off, mem, K):
    """source s on shard s % K; each shard's sources renumbered, its groups listing its own members in order"""
    local = [[s for s in range(len(srcs)) if s % K == k] for k in range(K)]
    idx = {s: i for k in range(K) for i, s in enumerate(local[k])}
    parts = []
    for k in range(K):
        o, m = [0], []
        for g in range(len(off) - 1):
            m += [idx[x] for x in mem[off[g]:off[g + 1]] if x % K == k]
            o.append(len(m))
        parts.append(([srcs[s] for s in local[k]], o, m))
    return parts


@pytest.mark.parametrize("metric", [GAUGE, COUNTER])
@pytest.mark.parametrize("K", [1, 2, 5])
def test_shards_compose_to_forward(metric, K):
    rng = np.random.default_rng(K + metric * 10)
    srcs, off, mem, W = _world(rng, metric, nan=True)
    G = len(off) - 1
    one = copy.deepcopy(srcs)
    want = _groups(metric, G, fwd=False)
    # the single-set forward over members listed shard by shard
    o2, m2 = [0], []
    for g in range(G):
        m2 += [x for k in range(K) for x in mem[off[g]:off[g + 1]] if x % K == k]
        o2.append(len(m2))
    forward(one, want, START + W * RES, o2, m2)
    got = _groups(metric, G)
    recs = []
    for k, (ss, o, m) in enumerate(_shards(srcs, off, mem, K)):
        r, st, gst, _ = forward_write(ss, START + W * RES, o, m, k)
        assert set(st) == {0} and set(gst) == {OK}
        recs += r
    res, est = add_forwarded(got, recs)
    assert set(res) == {OK} and set(est) == {OK}
    assert _windows(got) == _windows(want)
    # shuffled arrival changes only the order each window's shards arrive in: sums and counts stay
    perm = rng.permutation(len(recs))
    again = _groups(metric, G)
    res, _ = add_forwarded(again, [recs[i] for i in perm])
    assert set(res) == {OK}
    for a, b in zip(again, got):
        assert sorted(a.windows) == sorted(b.windows)
        assert all(len(a.windows[w]) == len(b.windows[w]) for w in a.windows)


def test_redelivery_changes_nothing():
    rng = np.random.default_rng(3)
    srcs, off, mem, W = _world(rng, COUNTER)
    recs, _, _, _ = forward_write(srcs, START + W * RES, off, mem, 4)
    g = _groups(COUNTER, len(off) - 1)
    add_forwarded(g, recs)
    before = _windows(g)
    res, st = add_forwarded(g, recs)
    assert set(res) == {ERR_DUPLICATE_SOURCE} and set(st) == {OK}
    assert _windows(g) == before


@pytest.mark.parametrize("resend", ["refused", "whole"])
@pytest.mark.parametrize("limit", ["windows", "sources"])
def test_add_capacity_stop_and_resend(resend, limit):
    rng = np.random.default_rng(5)
    srcs, off, mem, W = _world(rng, GAUGE)
    recs, _, _, _ = forward_write(srcs, START + W * RES, off, mem, 40)
    G = len(off) - 1
    want = _groups(GAUGE, G)
    add_forwarded(want, recs)
    small = _groups(GAUGE, G, R=2 if limit == "windows" else 8, cap=32 if limit == "sources" else 64)
    res, st = add_forwarded(small, recs)
    assert ERR_CAPACITY in res and ERR_CAPACITY in st
    for g in small:
        g.R, g.source_capacity = 8, 64
    again = [r for r, x in zip(recs, res) if x == ERR_CAPACITY] if resend == "refused" else recs
    res2, st2 = add_forwarded(small, again)
    assert set(st2) == {OK} and ERR_CAPACITY not in res2
    if resend == "whole":
        assert [x for x, y in zip(res2, res) if y == OK] == [ERR_DUPLICATE_SOURCE] * res.count(OK)
    assert _windows(small) == _windows(want)


def test_write_capacity_prefix_and_retry():
    rng = np.random.default_rng(9)
    srcs, off, mem, W = _world(rng, COUNTER)
    full_srcs = copy.deepcopy(srcs)
    want, _, _, counts = forward_write(full_srcs, START + W * RES, off, mem, 1)
    cap = counts[2] // 2
    got, st, gst, c = forward_write(srcs, START + W * RES, off, mem, 1, metric_capacity=cap)
    k = gst.index(ERR_CAPACITY)
    assert set(gst[:k]) == {OK} and set(gst[k:]) == {ERR_CAPACITY} and c[0] <= cap and c[2] == counts[2]
    # the failed groups again (the others' ranges empty)
    o = [0] * (k + 1)
    m = []
    for g in range(k, len(off) - 1):
        m += mem[off[g]:off[g + 1]]
        o.append(len(m))
    more, st2, gst2, _ = forward_write(srcs, START + W * RES, o, m, 1)
    assert set(gst2) == {OK}
    assert got + more == want


def test_closed_and_invalid_records():
    g = _groups(COUNTER, 2)
    t = START + RES
    res, _ = add_forwarded(g, [(0, t, [1.0], 0, 0, 0), (5, t, [1.0], 0, 0, 0), (0, t, [], 1, 0, 0),
                               (0, t, [1.0], 1, 1, 0), (0, t, [1.0], 1, 0, 2)])
    assert res == [OK, ERR_INVALID_ARG, ERR_INVALID_ARG, ERR_INVALID_ARG, ERR_INVALID_ARG]
    g[0].consume(START + RES)
    g[0].watermark = START + RES
    res, _ = add_forwarded(g, [(0, t, [2.0], 2, 0, 0)])
    assert res == [ERR_CLOSED]


def test_records_after_a_stop_are_capacity_whatever_they_hold():
    """add's stop rule: after a CAPACITY stop every later record of the element is CAPACITY, an invalid one too; other
    elements and invalid keys go on"""
    g = _groups(COUNTER, 2, R=1)
    t = START + RES
    recs = [(0, t, [1.0], 0, 0, 0), (0, t + RES, [1.0], 0, 0, 0), (0, t, [1.0], 1, 1, 0), (0, t, [], 1, 0, 0),
            (1, t, [1.0], 0, 0, 1), (9, t, [1.0], 0, 0, 0)]
    res, st = add_forwarded(g, recs)
    assert res == [OK, ERR_CAPACITY, ERR_CAPACITY, ERR_CAPACITY, ERR_INVALID_ARG, ERR_INVALID_ARG]
    assert st == [ERR_CAPACITY, OK]


def goldens():
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "m3tsz_forwarded_goldens.json")) as f:
        return json.load(f)


RESULT = {"ok": OK, "duplicate": ERR_DUPLICATE_SOURCE}


def golden_record(step, res):
    """an AddUnique step as a record: the reference's timestamp t falls in window Truncate(t); a record carries the
    source window's end, so time_ns = t + resolution keys the same window"""
    at_s, vals, sid = step[:3]
    return (0, at_s * SEC + res, list(vals), sid, 0, 0)


def check_window(got, want, case):
    for k, w in want.items():
        if k == "eps":
            continue
        if k == "sum" and "eps" in want:
            assert math.isclose(got[k], w, rel_tol=want["eps"]), case
        else:
            assert got[k] == w, (case, k)


@pytest.mark.parametrize("case", [c["name"] for c in goldens()["add_unique"]])
def test_add_unique_goldens(case):
    c = next(c for c in goldens()["add_unique"] if c["name"] == case)
    res = c["resolution_s"] * SEC
    metric = COUNTER if c["metric"] == "counter" else GAUGE
    g = ForwardedGroupModel(metric, [SUM], res, open_windows=4, source_capacity=5696)
    for step in c["steps"]:
        r, st = add_forwarded([g], [golden_record(step, res)])
        assert r == [RESULT[step[3]]] and st == [OK], case
        assert sorted(g.windows) == [w * SEC for w in step[4]], case
        check_window(g.aggregates(step[5] * SEC), step[6], case)


def test_writer_golden():
    c = goldens()["writer"][0]
    got = write_buckets([tuple(w) for w in c["writes"]])
    assert [list(r[:2]) + [r[2]] for r in got] == c["want"]
