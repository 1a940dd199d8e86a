"""GPU encode: the point-major stage's per-tile check of the hot tier.

The point-major encode reads its inputs in tiles of 4 rows and checks once per tile that every live lane has all 4
rows, room in its slot for 4 worst-case hot datapoints and the hot tier's preconditions; inside such a tile the
per-datapoint vote only looks at the data.  These tests put every way of leaving the hot tier at every row of a
tile (0, 1, 2 and 3): a delta-of-delta change, an int-like value (int-optimised), a repeat, a series that runs out
of slot, a series that ends there.  Every stream, its `out_len` and its status are compared with the oracle, with
tensor-copy input fills (even n_series) and lane-local ones (odd n_series, whose last warp is ragged).  Per-datapoint
units and annotations, which the point-major stage does not take, are run through the series-major stage the same
way."""
import numpy as np
import pytest

import oracle_lib as O

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
SEC = 1_000_000_000
START = 1599955200 * SEC
P = 67  # 16 whole tiles and a partial one of 3 rows
SLOT_WORDS_MARGIN = 14  # words the encoder keeps free in a slot before each datapoint (worst case + tail)


@pytest.fixture(scope="module")
def codecs():
    from m3_b200.codec import BatchCodec
    return {True: BatchCodec(0, True), False: BatchCodec(0, False)}


def _base(S, seed):
    """Regular 10 s cadence and random-walk floats at several scales: every datapoint after the first is a hot
    one.  n_points is ragged (P, and every length down to P - 7); a few series have none."""
    rng = np.random.default_rng(seed)
    ts = START + np.arange(1, P + 1, dtype=np.int64)[None, :].repeat(S, 0) * 10 * SEC
    scale = 10.0 ** (np.arange(S) % 5 - 2)
    vals = 100 + np.cumsum(rng.normal(size=(S, P)), axis=1) * scale[:, None]
    n_pts = (P - np.arange(S) % 8).astype(np.int32)
    n_pts[5::29] = 0
    return ts, vals, n_pts


def _event_rows(S, seed):
    """Per series, one datapoint index 4k + r with r = s % 4 (every row of a tile) inside the first 60 rows."""
    rng = np.random.default_rng(seed)
    return 4 * rng.integers(1, 15, size=S) + np.arange(S) % 4


def _expected(ts, vals, n, int_opt, slot_words, units=None, anns=None):
    """The oracle's stream of the first n datapoints and the status, stopping with a capacity error at the first
    datapoint before which the slot has fewer than SLOT_WORDS_MARGIN words left; and the datapoints encoded."""
    from m3_b200 import capi
    if n == 0:
        return b"", 0, 0
    e = O.Encoder(START, int_opt)
    for i in range(n):
        data, pos = e.raw()
        bits = (len(data) - 1) * 8 + pos if data else 64
        if bits // 32 + SLOT_WORDS_MARGIN > slot_words:
            return (e.stream() or b""), capi.ERR_CAPACITY, i
        u = O.UNIT_S if units is None else int(units[i])
        assert e.encode(int(ts[i]), float(vals[i]), u, (anns or {}).get(i, b"")) == 0
    return e.stream() or b"", 0, n


def _encode(codec, ts, vals, n_pts, stride, point_major, units=None, annotations=None):
    S = ts.shape[0]
    t, v = torch.from_numpy(ts).cuda(), torch.from_numpy(vals).cuda()
    if point_major:
        t, v = t.t().contiguous(), v.t().contiguous()
    out = codec.encode(t, v, torch.full((S,), START, dtype=torch.int64, device="cuda"), unit=O.UNIT_S,
                       n_points=torch.from_numpy(n_pts).cuda(), out_stride=stride, point_major=point_major,
                       units=None if units is None else torch.from_numpy(units).cuda(), annotations=annotations)
    torch.cuda.synchronize()
    return out.out.cpu().numpy(), out.out_len.cpu().numpy(), out.status.cpu().numpy()


def _check(got, expected):
    buf, out_len, status = got
    for s, (exp, st, _) in enumerate(expected):
        assert (int(status[s]), int(out_len[s])) == (st, len(exp)), s
        assert buf[s, :len(exp)].tobytes() == exp, s


def _case(case, S, int_opt, seed):
    ts, vals, n_pts = _base(S, seed)
    rows = _event_rows(S, seed + 1)
    for s, i in enumerate(rows):
        if case == "dod":  # the delta changes at i (and changes back after it)
            ts[s, i:] += 7 * SEC
        elif case == "int_like":
            vals[s, i] = float(round(vals[s, i]))
        elif case == "repeat":
            vals[s, i] = vals[s, i - 1]
        elif case == "ends":  # the series' last datapoint is row r of its tile
            n_pts[s] = i + 1
    return ts, vals, n_pts, rows


@pytest.mark.parametrize("S", [96, 95])  # even: tensor-copy fills; odd: lane-local fills, ragged last warp
@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("case", ["dod", "int_like", "repeat", "ends"])
def test_leaving_the_hot_tier_at_every_row(codecs, case, S, int_opt):
    codec = codecs[int_opt]
    ts, vals, n_pts, _ = _case(case, S, int_opt, seed=S * 7 + len(case))
    stride = codec.encode_bound(P)
    expected = [_expected(ts[s], vals[s], int(n_pts[s]), int_opt, stride // 4) for s in range(S)]
    assert all(st == 0 for _, st, _ in expected)
    got = _encode(codec, ts, vals, n_pts, stride, True)
    _check(got, expected)
    _check(_encode(codec, ts, vals, n_pts, stride, False), expected)  # the series-major stage agrees


@pytest.mark.parametrize("S", [96, 95])
@pytest.mark.parametrize("int_opt", [True, False])
def test_capacity_at_every_row(codecs, S, int_opt):
    """A slot that runs out part-way: every series stops at the same datapoint, with the same out_len and status,
    as the per-datapoint check makes it; the stops fall on every row of a tile."""
    from m3_b200 import capi
    codec = codecs[int_opt]
    ts, vals, n_pts = _base(S, seed=S + int_opt)
    rng = np.random.default_rng(3)
    vals[::3] = rng.normal(size=(S, P))[::3] * 1e9  # full-width XOR codes next to cheaper walks
    stride = 240
    expected = [_expected(ts[s], vals[s], int(n_pts[s]), int_opt, stride // 4) for s in range(S)]
    stops = [k for _, st, k in expected if st == capi.ERR_CAPACITY]  # the datapoints the series stopped at
    assert {k % 4 for k in stops} == {0, 1, 2, 3}, stops
    got = _encode(codec, ts, vals, n_pts, stride, True)
    _check(got, expected)
    _check(_encode(codec, ts, vals, n_pts, stride, False), expected)  # the series-major stage agrees


@pytest.mark.parametrize("int_opt", [True, False])
def test_units_and_annotations_at_every_row(codecs, int_opt):
    """Per-datapoint unit changes and annotations (series-major stage: the point-major one does not take them) at
    every row of a tile."""
    S = 64
    codec = codecs[int_opt]
    ts, vals, n_pts, rows = _case("none", S, int_opt, seed=21)
    units = np.full((S, P), O.UNIT_S, dtype=np.uint8)
    entries, series_off, blob, anns = [], [0], bytearray(), []
    for s, i in enumerate(rows):
        a = {}
        if s % 2:
            units[s, i:] = O.UNIT_MS
        else:
            a[int(i)] = bytes([s, s + 1, s + 2])
        for j, b in a.items():
            entries.append((j, len(b), len(blob)))
            blob += b
        series_off.append(len(entries))
        anns.append(a)
    ent = np.zeros(len(entries), dtype=[("dp", "<u4"), ("len", "<u4"), ("off", "<u8")])
    for k, e in enumerate(entries):
        ent[k] = e
    ann = (torch.tensor(series_off, dtype=torch.int64, device="cuda"),
           torch.from_numpy(ent.view(np.uint8).reshape(-1, 16).copy()).cuda(),
           torch.frombuffer(bytearray(bytes(blob) + b"\0"), dtype=torch.uint8).cuda())
    stride = _bound_units(P) + 64
    expected = [_expected(ts[s], vals[s], int(n_pts[s]), int_opt, stride // 4, units[s], anns[s]) for s in range(S)]
    assert all(st == 0 for _, st, _ in expected)
    _check(_encode(codec, ts, vals, n_pts, stride, False, units=units, annotations=ann), expected)


def _bound_units(n):
    from m3_b200 import capi
    return (int(capi.lib().m3tsz_encode_bound_units(n, 1)) + 15) // 16 * 16
