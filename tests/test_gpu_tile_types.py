"""Tile aggregation of an element with several aggregation types on the GPU (m3tsz_aggregate_tiles_types, the tile
stage's IN = 5 instantiation): bytes, out_len, n_tiles, status and the saved per-series element record against the
oracle (decode -> downsample -> ValueOf of every type -> the element, tests/elem_oracle.c -> oracle encode), in both
int_optimized modes and both stream addressings; and the call's equivalences with the single-type calls."""
import numpy as np
import pytest
import torch

import agg_oracle_lib as A
import elem_oracle_lib as E
import oracle_lib as O
from m3_b200 import capi
from test_gpu_transforms import N_WIN, R0, WIN, _batch, _csr, _padded, codecs  # noqa: F401

pytestmark = pytest.mark.gpu

AB, PS, INC, ADD, RST = 1, 2, 3, 4, 5
GAUGE_ALL = [1, 2, 3, 4, 6, 7, 8, 9]
COUNTER_ALL = [2, 3, 4, 6, 7, 8, 9]

# (metric, types, ops)
ELEMENTS = [
    (A.METRIC_GAUGE, GAUGE_ALL, [ADD]),
    (A.METRIC_COUNTER, COUNTER_ALL, [PS, ADD]),
    (A.METRIC_GAUGE, [4, 7], []),
    (A.METRIC_GAUGE, [2, 3, 7], [ADD, RST]),
    (A.METRIC_COUNTER, [2, 3, 7], [INC]),
    (A.METRIC_GAUGE, [1], [AB, ADD, PS, ADD, RST, AB, ADD, RST]),
    (A.METRIC_COUNTER, [6, 9], [RST, AB]),
    (A.METRIC_GAUGE, [1, 2, 8], [ADD, INC, ADD]),
]


def _state_host(st):
    return st.cpu().numpy().copy().view(E.ELEM_STATE_DTYPE).reshape(-1)


class Expect:
    """the oracle's view of a batch: each stream's datapoints (or its decode error) and each series' record"""

    def __init__(self, streams, int_opt, state=None):
        self.int_opt = int_opt
        self.src = [O.decode_series(b, int_opt, cap=4096) for b in streams]
        self.state = state if state is not None else np.zeros(len(streams), dtype=E.ELEM_STATE_DTYPE)

    def call(self, r0, step, n_win, metric, types, ops, discard, save=None):
        """-> [type][series] (status, bytes, n_tiles); advances the records of the series in `save` (default: every
        series that decodes)"""
        k = len(types)
        out = [[None] * len(self.src) for _ in range(k)]
        for s, (ts, vals, n, err) in enumerate(self.src):
            if err != 0:
                for j in range(k):
                    out[j][s] = (err, b"", 0)
                continue
            st = self.state[s: s + 1].copy()
            res = E.aggregate_tiles_types_series(ts[:n], vals[:n], r0, step, n_win, metric, types, ops,
                                                 discard and len(ops) > 0, st)
            if save is None or s in save:
                self.state[s] = st[0]
            for j, (tt, tv) in enumerate(res):
                out[j][s] = (0, O.encode_series(tt, tv, r0, O.UNIT_S, self.int_opt) if len(tt) else b"", len(tt))
        return out


def _check(r, n_tiles, exp, only=None):
    st, ln, of = r.status.cpu().numpy(), r.out_len.cpu().numpy(), r.offsets.cpu().numpy()
    packed, nt = r.packed.cpu().numpy(), n_tiles.cpu().numpy()
    for j, row in enumerate(exp):
        for s, (e_st, e_bytes, e_n) in enumerate(row):
            if only is not None and s not in only:
                continue
            assert st[j, s] == e_st, (j, s, st[j, s], e_st)
            if e_st:
                assert ln[j, s] == 0 and nt[j, s] == 0, (j, s)
                continue
            assert nt[j, s] == e_n, (j, s, nt[j, s], e_n)
            assert ln[j, s] == len(e_bytes) and packed[of[j, s]: of[j, s] + ln[j, s]].tobytes() == e_bytes, (j, s)


def _run(codec, blob, off, lengths, r0, n_win, metric, types, ops, discard, state, capacity=None):
    return codec.aggregate_tiles_types(blob, off, r0, WIN, n_win, types, metric_type=metric, lengths=lengths,
                                       capacity=capacity, transforms=ops, discard_nan=discard, state=state)


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("addressing", ["csr", "lengths"])
@pytest.mark.parametrize("discard", [True, False])
def test_elements_against_oracle(codecs, int_opt, addressing, discard):
    """every element, two consecutive calls carrying the record; damaged sources keep theirs untouched"""
    codec = codecs[int_opt]
    streams = _batch(int_opt, both_inf=not discard)
    blob, off, lengths = _csr(streams) if addressing == "csr" else _padded(streams)
    S = len(streams)
    for metric, types, ops in ELEMENTS:
        state = codec.element_state(S)
        exp = Expect(streams, int_opt)
        half = N_WIN // 2
        for r0, n_win in ((R0, half), (R0 + half * WIN, N_WIN - half)):
            r, nt = _run(codec, blob, off, lengths, r0, n_win, metric, types, ops, discard, state)
            torch.cuda.synchronize()
            _check(r, nt, exp.call(r0, WIN, n_win, metric, types, ops, discard))
            assert _state_host(state).tobytes() == exp.state.tobytes(), (metric, types, ops)


@pytest.mark.parametrize("int_opt", [True, False])
def test_call_splits_and_null_state(codecs, int_opt):
    """1 / 2 / 5 calls with the record give one call's datapoints; without a record every call starts new"""
    codec = codecs[int_opt]
    streams = _batch(int_opt, S=70, seed=9)
    blob, off, lengths = _csr(streams)
    S = len(streams)
    metric, types, ops = A.METRIC_GAUGE, [2, 4, 7], [ADD, PS]
    one = Expect(streams, int_opt).call(R0, WIN, N_WIN, metric, types, ops, True)
    for parts in (1, 2, 5):
        bounds = np.linspace(0, N_WIN, parts + 1).astype(int)
        state = codec.element_state(S)
        exp = Expect(streams, int_opt)
        for a, b in zip(bounds[:-1], bounds[1:]):
            r, nt = _run(codec, blob, off, lengths, R0 + int(a) * WIN, int(b - a), metric, types, ops, True, state)
            torch.cuda.synchronize()
            _check(r, nt, exp.call(R0 + int(a) * WIN, WIN, int(b - a), metric, types, ops, True))
        assert _state_host(state).tobytes() == exp.state.tobytes(), parts
        if parts == 1:
            _check(r, nt, one)
    r, nt = _run(codec, blob, off, lengths, R0 + 4 * WIN, 5, metric, types, ops, True, None)
    torch.cuda.synchronize()
    _check(r, nt, Expect(streams, int_opt).call(R0 + 4 * WIN, WIN, 5, metric, types, ops, True))


def test_capacity_on_one_row_then_retry(codecs):
    """a buffer too small for the batch: rows that did not fit report CAPACITY and their series keep their records;
    re-running with a larger buffer gives the unstopped result"""
    codec = codecs[True]
    streams = _batch(True, S=64, seed=13, damage=False)
    blob, off, lengths = _csr(streams)
    S = len(streams)
    metric, types, ops = A.METRIC_GAUGE, [1, 3, 7], [ADD, RST]
    r, _ = _run(codec, blob, off, lengths, R0, N_WIN, metric, types, ops, True, None)
    cap = int(r.total.item()) // 2 // 64 * 64  # about half the rows' warps fit
    state = codec.element_state(S)
    r, nt = _run(codec, blob, off, lengths, R0, N_WIN, metric, types, ops, True, state, capacity=cap)
    torch.cuda.synchronize()
    st = r.status.cpu().numpy()
    assert set(np.unique(st).tolist()) == {0, capi.ERR_CAPACITY}
    bad = set(int(s) for s in np.nonzero((st != 0).any(axis=0))[0])
    good = set(range(S)) - bad
    # a series with one row that did not fit and another that did
    assert any((st[:, s] == 0).any() for s in bad)
    e_full = Expect(streams, True).call(R0, WIN, N_WIN, metric, types, ops, True)
    exp = Expect(streams, True)
    e_rows = exp.call(R0, WIN, N_WIN, metric, types, ops, True, save=good)
    rec = _state_host(state)
    z = np.zeros(1, dtype=E.ELEM_STATE_DTYPE).tobytes()
    for s in range(S):
        assert rec[s].tobytes() == (exp.state[s].tobytes() if s in good else z), s
    for j in range(len(types)):
        for s in good:
            assert st[j, s] == 0
    _check(r, nt, e_rows, only=good)
    r2, nt2 = _run(codec, blob, off, lengths, R0, N_WIN, metric, types, ops, True, state)
    torch.cuda.synchronize()
    exp2 = Expect(streams, True, state=exp.state.copy())
    e2 = exp2.call(R0, WIN, N_WIN, metric, types, ops, True)
    assert int((r2.status != 0).sum()) == 0
    _check(r2, nt2, e2)
    assert _state_host(state).tobytes() == exp2.state.tobytes()
    # the retried series wrote what one unstopped call writes
    _check(r2, nt2, e_full, only=bad)


@pytest.mark.parametrize("int_opt", [True, False])
def test_single_type_equals_transform_call(codecs, int_opt):
    """k = 1: aggregate_tiles' bytes, lengths, tile counts and status, and its 96-byte state in the record's prefix"""
    codec = codecs[int_opt]
    streams = _batch(int_opt, S=80, seed=21)
    blob, off, lengths = _padded(streams)
    S = len(streams)
    for metric, agg, ops in ((A.METRIC_COUNTER, 7, [PS, ADD]), (A.METRIC_GAUGE, 1, [ADD, RST]),
                             (A.METRIC_GAUGE, 9, [INC]), (A.METRIC_GAUGE, 8, [])):
        el = codec.element_state(S)
        xs = codec.transform_state(S)
        for r0, n in ((R0, 5), (R0 + 5 * WIN, 7)):
            a, na = _run(codec, blob, off, lengths, r0, n, metric, [agg], ops, True, el)
            b, nb = codec.aggregate_tiles(blob, off, r0, WIN, n, agg, metric_type=metric, lengths=lengths,
                                          transforms=ops, discard_nan=True, state=xs if ops else None)
            torch.cuda.synchronize()
            assert torch.equal(a.status[0], b.status) and torch.equal(a.out_len[0], b.out_len)
            assert torch.equal(na[0], nb)
            pa, pb = a.packed.cpu().numpy(), b.packed.cpu().numpy()
            oa, ob, ln = a.offsets[0].cpu().numpy(), b.offsets.cpu().numpy(), b.out_len.cpu().numpy()
            for s in range(S):
                assert pa[oa[s]: oa[s] + ln[s]].tobytes() == pb[ob[s]: ob[s] + ln[s]].tobytes(), (agg, s)
        if ops:
            e = el.cpu().numpy()
            assert (e[:, :96] == xs.cpu().numpy()).all() and (e[:, 96:] == 0).all()


@pytest.mark.parametrize("int_opt", [True, False])
def test_rows_equal_single_type_calls_without_add(codecs, int_opt):
    """no ops: row j is aggregate_tiles_ex's for type j; a list without Add: row j is aggregate_tiles_transform's"""
    codec = codecs[int_opt]
    streams = _batch(int_opt, S=90, seed=31)
    blob, off, lengths = _csr(streams)
    S = len(streams)
    for metric, types, ops in ((A.METRIC_GAUGE, GAUGE_ALL, []), (A.METRIC_COUNTER, COUNTER_ALL, []),
                               (A.METRIC_GAUGE, [1, 4, 9], [PS, RST]), (A.METRIC_COUNTER, [2, 6, 7], [AB, INC])):
        r, nt = _run(codec, blob, off, lengths, R0, N_WIN, metric, types, ops, True, None)
        for j, agg in enumerate(types):
            b, nb = codec.aggregate_tiles(blob, off, R0, WIN, N_WIN, agg, metric_type=metric, transforms=ops,
                                          discard_nan=True)
            torch.cuda.synchronize()
            assert torch.equal(r.status[j], b.status) and torch.equal(r.out_len[j], b.out_len)
            assert torch.equal(nt[j], nb)
            pa, pb = r.packed.cpu().numpy(), b.packed.cpu().numpy()
            oa, ob, ln = r.offsets[j].cpu().numpy(), b.offsets.cpu().numpy(), b.out_len.cpu().numpy()
            for s in range(S):
                assert pa[oa[s]: oa[s] + ln[s]].tobytes() == pb[ob[s]: ob[s] + ln[s]].tobytes(), (agg, s)


def test_add_rows_differ_from_single_type_calls(codecs):
    """with Add the types share the sums: row 1 is not the single-type call's"""
    codec = codecs[True]
    streams = _batch(True, S=40, seed=3, damage=False)
    blob, off, lengths = _csr(streams)
    r, nt = _run(codec, blob, off, lengths, R0, N_WIN, A.METRIC_GAUGE, [2, 3], [ADD], True, None)
    b, nb = codec.aggregate_tiles(blob, off, R0, WIN, N_WIN, 3, transforms=[ADD])
    torch.cuda.synchronize()
    assert int((r.status != 0).sum()) == 0 and int((b.status != 0).sum()) == 0
    pa, pb = r.packed.cpu().numpy(), b.packed.cpu().numpy()
    oa, la = r.offsets[1].cpu().numpy(), r.out_len[1].cpu().numpy()
    ob, lb = b.offsets.cpu().numpy(), b.out_len.cpu().numpy()
    differ = [s for s in range(len(streams)) if pa[oa[s]: oa[s] + la[s]].tobytes() != pb[ob[s]: ob[s] + lb[s]].tobytes()]
    # Max's sum includes Min's values; a series without windows in the range, or whose sums are NaN / Inf either
    # way, writes the same
    assert len(differ) > len(streams) // 2


@pytest.mark.parametrize("types,metric", [
    ([3, 2], A.METRIC_GAUGE), ([2, 2], A.METRIC_GAUGE), ([1, 2], A.METRIC_COUNTER), ([5], A.METRIC_GAUGE),
    (list(range(1, 10)), A.METRIC_GAUGE), ([], A.METRIC_GAUGE), ([2, 7], 2)])
def test_invalid_type_lists(codecs, types, metric):
    from m3_b200.capi import M3tszError as M3Error
    codec = codecs[True]
    streams = _batch(True, S=8, seed=1)
    blob, off, lengths = _csr(streams)
    with pytest.raises(M3Error):
        _run(codec, blob, off, lengths, R0, N_WIN, metric, types, [], True, None)


def test_invalid_ops(codecs):
    from m3_b200.capi import M3tszError as M3Error
    codec = codecs[True]
    streams = _batch(True, S=8, seed=1)
    blob, off, lengths = _csr(streams)
    for ops in ([PS, INC], [6], [ADD] * 9, [0]):
        with pytest.raises(M3Error):
            _run(codec, blob, off, lengths, R0, N_WIN, A.METRIC_GAUGE, [2, 3], ops, True, None)


def test_100k_series_sampled(codecs):
    codec = codecs[True]
    S = 100_000
    base = _batch(True, S=200, seed=77)
    streams = [base[i % len(base)] for i in range(S)]
    blob, off, lengths = _csr(streams)
    metric, types, ops = A.METRIC_GAUGE, [1, 2, 3, 4, 7], [ADD, RST]
    state = codec.element_state(S)
    r, nt = _run(codec, blob, off, lengths, R0, N_WIN, metric, types, ops, True, state)
    torch.cuda.synchronize()
    sample = sorted(set([0, 1, 31, 32, 4097, S - 1] + list(np.random.default_rng(5).integers(0, S, 40))))
    exp = Expect([streams[s] for s in sample], True)
    e_rows = exp.call(R0, WIN, N_WIN, metric, types, ops, True)
    st, ln, of = r.status.cpu().numpy(), r.out_len.cpu().numpy(), r.offsets.cpu().numpy()
    packed, ntc = r.packed.cpu().numpy(), nt.cpu().numpy()
    rec = _state_host(state)
    for i, s in enumerate(sample):
        for j in range(len(types)):
            e_st, e_bytes, e_n = e_rows[j][i]
            assert st[j, s] == e_st, (j, s)
            if e_st == 0:
                assert ntc[j, s] == e_n and packed[of[j, s]: of[j, s] + ln[j, s]].tobytes() == e_bytes, (j, s)
        assert rec[s].tobytes() == exp.state[i].tobytes(), s
