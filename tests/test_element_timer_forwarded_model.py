"""The Timer cross-shard rollup model (tests/element_timer_forwarded_model.py): it reproduces the reference's
TimerElem.AddUnique golden (tests/golden/m3tsz_timer_forwarded_goldens.json); K shards written in shard order and
concatenated give, window by window and on the quantiles too, the Timer rollup model's forward over one set whose
groups list the members shard by shard; a redelivered batch changes nothing; and a sample-capacity stop and an
open-window stop each recover by grow and resend."""
import json
import os

import numpy as np
import pytest

from element_timer_forwarded_model import (ERR_CAPACITY, ERR_CLOSED, ERR_DUPLICATE_SOURCE, OK,
                                           TimerForwardedGroupModel, TimerSourceModel, add_forwarded_timer,
                                           forward_write)
from element_timer_rollup_model import TimerGroupModel, forward
from test_element_timer_rollup_model import check_add_unique_want

SEC = 1_000_000_000
RES = 60 * SEC
START = 1_600_000_020 * SEC
TYPES = [3, 14, 20]  # Max, P50, P99


def _f64(x):
    return np.float64(x).tobytes()


def timer_world(rng, K, S=6, G=4, W=3, src_type=20, pre=(), twice=True):
    """K shards of S Timer source models each, with random samples over W windows, and per shard G groups of its own
    sources (a member listed twice when `twice`).  -> (shards [[TimerSourceModel]], single [TimerSourceModel] (shard k's
    source s at k * S + s, the same samples), memberships [(off, mem)] per shard, single set's (off, mem): group g
    lists shard 0's members, then shard 1's, ...)"""
    def src():
        return TimerSourceModel(src_type, RES, list(pre), False, open_windows=W + 1, sample_capacity=64)
    shards = [[src() for _ in range(S)] for _ in range(K)]
    single = [src() for _ in range(K * S)]
    for k in range(K):
        for s in range(S):
            rows = [(START + w * RES + int(rng.integers(0, 60)) * SEC, float(np.round(rng.normal() * 100, 1)))
                    for w in range(W) for _ in range(int(rng.integers(0, 4)))]
            shards[k][s].add(rows)
            single[k * S + s].add(rows)
    memb = []
    for k in range(K):
        lens = rng.integers(0, 4, G)
        mem = [int(m) for m in rng.integers(0, S, int(lens.sum()))]
        if twice and len(mem) > 1:
            mem[1] = mem[0]
        memb.append((np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64), mem))
    lists = [[k * S + m for k in range(K) for m in memb[k][1][int(memb[k][0][g]): int(memb[k][0][g + 1])]]
             for g in range(G)]
    off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.uint64)
    return shards, single, memb, (off, [m for x in lists for m in x])


def same_windows(a, b):
    """two Timer group models hold the same windows: count, sum, sum_sq and every type's value, bit for bit"""
    assert sorted(a.windows) == sorted(b.windows)
    for ws in a.windows:
        x, y = a.windows[ws], b.windows[ws]
        assert x.count == y.count and _f64(x.sum) == _f64(y.sum) and _f64(x.sum_sq) == _f64(y.sum_sq), ws
        assert [_f64(v) for v in x.values()] == [_f64(v) for v in y.values()], ws


def test_golden():
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                           "m3tsz_timer_forwarded_goldens.json")) as f:
        cases = json.load(f)["add_unique"]
    for c in cases:
        res = c["resolution_s"] * SEC
        g = TimerForwardedGroupModel(c["types"], res, (), False, 4, 64, c["eps"], c["every"], source_capacity=64)
        for at_s, vals, sid, want_r, windows_s, window_s, want in c["steps"]:
            r, st = add_forwarded_timer([g], [(0, at_s * SEC + res, vals, sid, 0, 0)])
            assert r == [OK if want_r == "ok" else ERR_DUPLICATE_SOURCE] and st == [OK], c["name"]
            assert sorted(g.windows) == [w * SEC for w in windows_s]
            check_add_unique_want(g.windows[window_s * SEC], want)
            assert set(want.get("seen", [])) <= g.seen_by(window_s * SEC)


@pytest.mark.parametrize("K", [1, 2, 5])
@pytest.mark.parametrize("pre", [(), (2,)])
def test_shards_equal_one_forward(K, pre):
    rng = np.random.default_rng(7 * K + len(pre))
    for it in range(6):
        shards, single, memb, (off, mem) = timer_world(rng, K, pre=pre)
        G = len(off) - 1
        target = START + 3 * RES
        batch = []
        for k in range(K):
            recs, sst, gst, _ = forward_write(shards[k], target, memb[k][0], memb[k][1], k)
            assert set(gst) <= {OK} and set(sst) <= {0}
            batch += recs
        ga = [TimerForwardedGroupModel(TYPES, RES, open_windows=8, sample_capacity=256) for _ in range(G)]
        gb = [TimerGroupModel(TYPES, RES, open_windows=8, sample_capacity=256) for _ in range(G)]
        r, st = add_forwarded_timer(ga, batch)
        assert set(r) <= {OK} and st == [OK] * G
        sst, gst = forward(single, gb, target, off, mem)
        assert gst == [OK] * G and sst == [0] * len(single)
        for a, b in zip(ga, gb):
            same_windows(a, b)
        for k in range(K):
            for s, m in enumerate(shards[k]):
                b = single[k * len(shards[k]) + s]
                assert m.state.tobytes() == b.state.tobytes() and m.watermark == b.watermark


def test_redelivery_changes_nothing():
    rng = np.random.default_rng(3)
    shards, _, memb, _ = timer_world(rng, 2)
    batch = []
    for k in range(2):
        batch += forward_write(shards[k], START + 3 * RES, memb[k][0], memb[k][1], k)[0]
    ga = [TimerForwardedGroupModel(TYPES, RES, open_windows=8) for _ in range(4)]
    gb = [TimerForwardedGroupModel(TYPES, RES, open_windows=8) for _ in range(4)]
    add_forwarded_timer(ga, batch)
    add_forwarded_timer(gb, batch)
    r, st = add_forwarded_timer(ga, batch[::-1])
    assert set(r) == {ERR_DUPLICATE_SOURCE} and st == [OK] * 4
    for a, b in zip(ga, gb):
        same_windows(a, b)


def test_closed_records():
    g = TimerForwardedGroupModel(TYPES, RES)
    g.watermark = START + RES
    r, _ = add_forwarded_timer([g], [(0, START + RES, [1.0], 0, 0, 0), (0, START + 2 * RES, [1.0], 0, 0, 0)])
    assert r == [ERR_CLOSED, OK] and list(g.windows) == [START + RES]


@pytest.mark.parametrize("stop", ["samples", "windows"])
def test_capacity_stop_recovers_by_grow_and_resend(stop):
    """a sample-capacity stop (a window short of room) and an open-window stop: the element stops at the record,
    nothing of it is taken, a window it would open stays closed, and grow + resend gives the unstopped result"""
    rng = np.random.default_rng(11)
    shards, _, memb, _ = timer_world(rng, 2, S=8, G=2)
    batch = []
    for k in range(2):
        batch += forward_write(shards[k], START + 3 * RES, memb[k][0], memb[k][1], k)[0]
    R, cap = (8, 2) if stop == "samples" else (1, 256)
    ga = [TimerForwardedGroupModel(TYPES, RES, open_windows=R, sample_capacity=cap) for _ in range(2)]
    gb = [TimerForwardedGroupModel(TYPES, RES, open_windows=8, sample_capacity=256) for _ in range(2)]
    r, st = add_forwarded_timer(ga, batch)
    assert ERR_CAPACITY in st
    first = r.index(ERR_CAPACITY)
    key = batch[first][0]
    ws = batch[first][1] - RES
    assert ga[key].seen_by(ws) == ({k for (kk, t, _, k, _, _), x in zip(batch, r) if kk == key and t - RES == ws
                                    and x == OK})
    for m in ga:
        m.R, m.cap = 8, 256
    again = [b for b, x in zip(batch, r) if x == ERR_CAPACITY]
    r2, st2 = add_forwarded_timer(ga, again)
    assert set(r2) == {OK} and st2 == [OK] * 2
    add_forwarded_timer(gb, batch)
    for a, b in zip(ga, gb):
        same_windows(a, b)
