"""Element sets on the GPU (m3tsz_element_set_*, DESIGN.md §4.12), in both int_optimized modes: datapoints added over
several calls and consumed at flush ticks give byte for byte the streams, and the element records, of
m3tsz_aggregate_tiles_types over streams of the same datapoints; the reference's element tables through the call;
closed windows, capacity on windows and on output slots with grow-and-resend, argument checks, and a large set sampled
against the CPU model (tests/element_set_model.py)."""
import json
import os

import numpy as np
import pytest
import torch

import agg_oracle_lib as A
from element_set_model import ElementModel
from m3_b200 import capi
from test_element_set_model import _bits, add_case_datapoints, random_series

pytestmark = pytest.mark.gpu

SEC = 1_000_000_000
RES = 60 * SEC
START = 1_600_000_020 * SEC  # a whole minute
DEV = "cuda"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "m3tsz_element_consume_goldens.json")


@pytest.fixture(scope="module")
def codecs():
    from m3_b200.codec import BatchCodec
    return {True: BatchCodec(0, int_optimized=True), False: BatchCodec(0, int_optimized=False)}


def _point_major(cols, P=None):
    """per-element lists [(t, value bits)] -> (ts [P, N], values [P, N], n_points [N]) on the device"""
    N = len(cols)
    P = max([len(c) for c in cols] + [1]) if P is None else P
    ts = np.zeros((P, N), dtype=np.int64)
    vb = np.zeros((P, N), dtype=np.uint64)
    for s, c in enumerate(cols):
        for i, (t, v) in enumerate(c):
            ts[i, s], vb[i, s] = t, v
    n = np.array([len(c) for c in cols], dtype=np.int32)
    return (torch.from_numpy(ts).to(DEV), torch.from_numpy(vb.view(np.float64)).to(DEV), torch.from_numpy(n).to(DEV))


def _rows(es):
    """the output snapshot as bytes per row"""
    snap = es.stream()
    out, ln = snap.out.cpu().numpy(), snap.out_len.cpu().numpy()
    return [out[r, : ln[r]].tobytes() for r in range(len(ln))]


def _decoded_rows(codec, es, cap=64):
    """each output row's datapoints [(t, value bits)]"""
    snap = es.stream()
    dec = codec.decode(snap.out.view(-1), es.out.offsets(), cap, lengths=snap.out_len)
    ts, vals, n = dec.ts.cpu().numpy(), dec.values.cpu().numpy().view(np.uint64), dec.n_points.cpu().numpy()
    ln = snap.out_len.cpu().numpy()
    return [list(zip(ts[r, : n[r]].tolist(), vals[r, : n[r]].tolist())) if ln[r] else [] for r in range(len(ln))]


def _tiles(codec, cols, metric, types, ops, discard, n_windows):
    """aggregate_tiles_types over streams of the same datapoints -> (bytes per row, element records)"""
    N = len(cols)
    P = max([len(c) for c in cols] + [1])
    ts = np.zeros((N, P), dtype=np.int64)
    vb = np.zeros((N, P), dtype=np.uint64)
    for s, c in enumerate(cols):
        for i, (t, v) in enumerate(c):
            ts[s, i], vb[s, i] = t, v
    n = torch.tensor([len(c) for c in cols], dtype=torch.int32, device=DEV)
    start = torch.full((N,), START, dtype=torch.int64, device=DEV)
    enc = codec.encode(torch.from_numpy(ts).to(DEV), torch.from_numpy(vb.view(np.float64)).to(DEV), start,
                       n_points=n)
    assert int(enc.status.abs().sum()) == 0
    offs = torch.arange(N, dtype=torch.int64, device=DEV) * enc.out.shape[1]
    state = codec.element_state(N)
    out, _ = codec.aggregate_tiles_types(enc.out.view(-1), offs, START, RES, n_windows, types, metric_type=metric,
                                         lengths=enc.out_len, transforms=ops, discard_nan=discard, state=state)
    assert int(out.status.abs().sum()) == 0
    packed = out.packed.cpu().numpy()
    o, ln = out.offsets.reshape(-1).cpu().numpy(), out.out_len.reshape(-1).cpu().numpy()
    return [packed[o[r]: o[r] + ln[r]].tobytes() for r in range(len(ln))], state


CASES = [
    (A.METRIC_GAUGE, [1, 2, 3], []),
    (A.METRIC_GAUGE, [1, 2, 3, 4, 6, 7, 8, 9], [4, 3, 5]),
    (A.METRIC_GAUGE, [4, 7], [1, 2]),
    (A.METRIC_COUNTER, [7], []),
    (A.METRIC_COUNTER, [2, 3, 4, 6, 7, 8, 9], [3]),
    (A.METRIC_COUNTER, [7, 9], [4, 5]),
]


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("n_calls", [1, 2, 5, 17])
def test_equals_aggregate_tiles_types(codecs, int_opt, case, n_calls):
    metric, types, ops = CASES[case]
    codec = codecs[int_opt]
    rng = np.random.default_rng(100 * case + n_calls + int_opt)
    N, W = 70, 8
    discard = bool(case % 2)
    cols = [random_series(rng, START, RES, W, metric) for _ in range(N)]
    es = codec.element_set(torch.full((N,), START, dtype=torch.int64, device=DEV), metric, types, RES,
                           transforms=ops, discard_nan=discard, open_windows=W)
    cuts = [np.sort(rng.integers(0, len(c) + 1, n_calls - 1)).tolist() for c in cols]
    for call in range(n_calls):
        parts = []
        for s, c in enumerate(cols):
            b = [0] + cuts[s] + [len(c)]
            parts.append(c[b[call]: b[call + 1]])
        ts, vals, n = _point_major(parts)
        res, st = es.add(ts, vals, n)
        assert int(st.abs().sum()) == 0 and int(res.abs().sum()) == 0
        # a flush tick that closes no window a later datapoint falls in
        pending = [c[([0] + cuts[s] + [len(c)])[call + 1]:] for s, c in enumerate(cols)]
        firsts = [p[0][0] - (p[0][0] - START) % RES for p in pending if p]
        if call + 1 < n_calls and firsts:
            assert int(es.consume(min(firsts)).abs().sum()) == 0
    assert int(es.consume(START + W * RES).abs().sum()) == 0
    want, state = _tiles(codec, cols, metric, types, ops, discard, W)
    assert _rows(es) == want
    assert torch.equal(es.elem, state)


@pytest.mark.parametrize("int_opt", [True, False])
def test_goldens_through_the_call(codecs, int_opt):
    codec = codecs[int_opt]
    with open(GOLDEN) as f:
        g = json.load(f)
    for case in g["adds"]:
        es = codec.element_set(torch.zeros(1, dtype=torch.int64, device=DEV), case["metric_type"], case["agg_types"],
                               case["resolution_ns"])
        for (t, v), want in zip(add_case_datapoints(case), case["want_windows"]):
            res, st = es.add(*_point_major([[(t, _bits(v))]])[:2])
            assert int(res.abs().sum()) == 0 and int(st.abs().sum()) == 0
            w = {f: a[:, 0].cpu() for f, a in es.win.items()}
            open_ = {int(w["start"][r]): r for r in range(es.open_windows) if int(w["count"][r]) > 0}
            assert sorted(open_) == [x["start_ns"] for x in want]
            for x in want:
                r = open_[x["start_ns"]]
                got = {f: w[f][r].item() for f in w}
                got["mean"] = got["sum"] / got["count"]
                for f, val in x.items():
                    if f != "start_ns":
                        assert got[f] == val, (case["name"], f)
    for case in g["consumes"]:
        es = codec.element_set(torch.zeros(1, dtype=torch.int64, device=DEV), case["metric_type"], case["agg_types"],
                               case["resolution_ns"])
        ts, vals, _ = _point_major([[(t, _bits(v)) for t, v in case["windows"]]])
        es.add(ts, vals)
        seen = 0
        for step in case["steps"]:
            assert int(es.consume(step["target_ns"]).abs().sum()) == 0
            rows = _decoded_rows(codec, es)
            assert [[(t, float(np.uint64(v).view(np.float64))) for t, v in r[seen:]] for r in rows] == \
                [[tuple(x) for x in w] for w in step["want"]]
            seen = len(rows[0])


@pytest.mark.parametrize("int_opt", [True, False])
def test_closed_windows(codecs, int_opt):
    codec = codecs[int_opt]
    es = codec.element_set(torch.full((2,), START, dtype=torch.int64, device=DEV), A.METRIC_GAUGE, [1], RES)
    ts, vals, _ = _point_major([[(START + 5 * SEC, _bits(1.0)), (START + RES, _bits(2.0))], []])
    es.add(ts, vals, torch.tensor([2, 0], dtype=torch.int32, device=DEV))
    assert es.consume(START + RES).tolist() == [0, 0]
    assert es.watermark.tolist() == [START + RES, -(1 << 63)]
    late = [(START + 7 * SEC, _bits(3.0)), (START + RES + SEC, _bits(4.0)), (START - SEC, _bits(5.0))]
    ts, vals, n = _point_major([late, late])
    res, st = es.add(ts, vals, n)
    assert res[:, 0].tolist() == [capi.ERR_AGGREGATION_CLOSED, 0, capi.ERR_AGGREGATION_CLOSED]
    assert res[:, 1].tolist() == [0, 0, 0]  # nothing consumed yet
    assert st.tolist() == [0, 0]
    assert capi.status_string(capi.ERR_AGGREGATION_CLOSED) == "aggregation is closed"


def _sequence(rng, N, W, metric):
    return [random_series(rng, START, RES, W, metric) for _ in range(N)]


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("metric", [A.METRIC_GAUGE, A.METRIC_COUNTER])
def test_capacity_grow_and_resend(codecs, int_opt, metric):
    codec = codecs[int_opt]
    rng = np.random.default_rng(5 + int_opt)
    N, W = 96, 6
    cols = _sequence(rng, N, W, metric)
    start = torch.full((N,), START, dtype=torch.int64, device=DEV)
    types, ops = ([1, 8] if metric == A.METRIC_GAUGE else [7, 8]), [4, 5]
    full = codec.element_set(start, metric, types, RES, transforms=ops, open_windows=W)
    full.add(*_point_major(cols))
    assert int(full.consume(START + W * RES).abs().sum()) == 0
    # windows: two slots, then grow and send again exactly the datapoints that got CAPACITY
    es = codec.element_set(start, metric, types, RES, transforms=ops, open_windows=2, stride=64)
    res, st = es.add(*_point_major(cols))
    res = res.cpu().numpy()
    assert (st.cpu().numpy() == capi.ERR_CAPACITY).any()
    again = [[p for i, p in enumerate(c) if res[i, s] == capi.ERR_CAPACITY] for s, c in enumerate(cols)]
    assert all(res[i, s] in (0, capi.ERR_CAPACITY) for s, c in enumerate(cols) for i in range(len(c)))
    es.grow(open_windows=W)
    res2, st2 = es.add(*_point_major(again))
    assert int(st2.abs().sum()) == 0 and int(res2.abs().sum()) == 0
    # output slots: 64 bytes take no flush; the elements keep everything until the slots grow
    st = es.consume(START + W * RES).cpu().numpy()
    busy = np.array([len(c) > 0 for c in cols])
    assert (st[busy] == capi.ERR_CAPACITY).all() and (st[~busy] == 0).all()
    assert (es.watermark.cpu().numpy()[busy] == -(1 << 63)).all()
    es.grow(stride=full.out.stride)
    assert int(es.consume(START + W * RES).abs().sum()) == 0
    assert _rows(es) == _rows(full)
    assert torch.equal(es.elem, full.elem) and torch.equal(es.watermark, full.watermark)


@pytest.mark.parametrize("int_opt", [True, False])
def test_argument_checks_and_ragged_points(codecs, int_opt):
    codec = codecs[int_opt]
    start = torch.full((4,), START, dtype=torch.int64, device=DEV)
    bad = [dict(agg_types=[3, 2]), dict(agg_types=[1], metric_type=A.METRIC_COUNTER), dict(resolution_ns=0),
           dict(open_windows=capi.MAX_ELEMENT_WINDOWS + 1), dict(transforms=[2, 3]), dict(transforms=[9])]
    for kw in bad:
        args = dict(metric_type=A.METRIC_GAUGE, agg_types=[1], resolution_ns=RES)
        args.update(kw)
        with pytest.raises(capi.M3tszError) as e:
            codec.element_set(start, **args)
        assert e.value.status == capi.ERR_INVALID_ARG
    es = codec.element_set(start, A.METRIC_GAUGE, [1], RES)
    es.out_unit = 0
    with pytest.raises(capi.M3tszError):
        es.consume(START)
    es.out_unit = capi.UNIT_S
    cols = [[(START + j * SEC, _bits(float(j))) for j in range(i)] for i in range(4)]
    ts, vals, n = _point_major(cols, P=3)
    n[3] = 4  # more than the rows given: that element is refused, the others go on
    res, st = es.add(ts, vals, n)
    assert st.tolist() == [0, 0, 0, capi.ERR_INVALID_ARG]
    assert es.win["count"].sum(0).tolist() == [0, 1, 2, 0]
    assert res[:, 3].tolist() == [0, 0, 0]


@pytest.mark.parametrize("int_opt", [True, False])
def test_100k_elements_sampled_against_the_model(codecs, int_opt):
    codec = codecs[int_opt]
    rng = np.random.default_rng(11 + int_opt)
    N, W, metric, types, ops = 100_000, 5, A.METRIC_GAUGE, [1, 2, 3], [3]
    es = codec.element_set(torch.full((N,), START, dtype=torch.int64, device=DEV), metric, types, RES,
                           transforms=ops, discard_nan=True, open_windows=3, stride=codec.encode_bound(32))
    sample = rng.choice(N, 300, replace=False)
    models = {int(s): ElementModel(metric, types, RES, ops, True, open_windows=3) for s in sample}
    results = {int(s): [] for s in sample}
    for step in range(3 * W):
        # one tick: up to three datapoints per element around the tick, some late, some NaN / Inf
        n = rng.integers(0, 4, N).astype(np.int32)
        t = START + step * 20 * SEC + rng.integers(-90, 30, (3, N)) * SEC
        v = rng.normal(size=(3, N)) * 100
        v[rng.random((3, N)) < 0.02] = np.nan
        v[rng.random((3, N)) < 0.01] = np.inf
        res, _ = es.add(torch.from_numpy(t).to(DEV).contiguous(), torch.from_numpy(v).to(DEV).contiguous(),
                        torch.from_numpy(n).to(DEV))
        res = res.cpu().numpy()
        for s, m in models.items():
            pts = [(int(t[i, s]), _bits(v[i, s])) for i in range(n[s])]
            r, _ = m.add(pts)
            assert res[: n[s], s].tolist() == r, (step, s)
        if step % 3 == 2:
            target = START + (step // 3) * RES
            es.consume(target)
            for s, m in models.items():
                results[s].append(m.consume(target))
    rows = _decoded_rows(codec, es)
    for s, m in models.items():
        for j in range(len(types)):
            want = [p for out in results[s] for p in zip(out[j][0].tolist(), out[j][1].view(np.uint64).tolist())]
            assert rows[j * N + s] == want, (s, j)
    got = es.elem.cpu().numpy()
    for s, m in models.items():
        assert got[s].tobytes() == m.state.tobytes()
