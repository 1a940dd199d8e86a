"""Tile aggregation with the aggregator's transformations on the GPU (m3tsz_aggregate_tiles_transform, the tile
stage's IN = 4 instantiation): bytes, out_len, n_tiles, status and the saved per-series state against the oracle
(decode -> downsample -> ValueOf -> transformations -> oracle encode, tests/xf_oracle.c), in both int_optimized
modes and both stream addressings."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import agg_oracle_lib as A
import xf_oracle_lib as X
import oracle_lib as O

pytestmark = pytest.mark.gpu

SEC = 1_000_000_000
WIN = 60 * SEC
N_WIN = 12
R0 = 1_700_000_040 * SEC  # range start (window-aligned)
START = R0 - 10 * WIN     # source encoder start
AB, PS, INC, ADD, RST = 1, 2, 3, 4, 5

# (metric, aggregation type, ops)
PIPELINES = [
    (A.METRIC_COUNTER, A.AGG_SUM, [PS]),
    (A.METRIC_GAUGE, A.AGG_LAST, [INC]),
    (A.METRIC_GAUGE, A.AGG_SUM, [RST]),
    (A.METRIC_GAUGE, A.AGG_MAX, [AB, PS]),
    (A.METRIC_GAUGE, A.AGG_MIN, [INC, ADD]),
    (A.METRIC_COUNTER, A.AGG_MEAN, [ADD, ADD]),
    (A.METRIC_GAUGE, A.AGG_STDEV, [ADD, RST, AB]),
    (A.METRIC_COUNTER, A.AGG_COUNT, [RST, INC, RST]),
    (A.METRIC_GAUGE, A.AGG_LAST, [AB, ADD, PS, ADD, RST, AB, ADD, RST]),
]


@pytest.fixture(scope="module")
def codecs():
    from m3_b200.codec import BatchCodec
    return {True: BatchCodec(0, int_optimized=True), False: BatchCodec(0, int_optimized=False)}


def _series(rng, n, both_inf):
    """n datapoints in order with gaps of empty windows; values: ordinary, decreasing runs and specials (NaN
    payloads, one or both infinity signs, +-0)"""
    t = R0 - int(rng.integers(0, 3)) * WIN + int(rng.integers(0, 60)) * SEC
    inf = [math.inf, -math.inf] if both_inf else [math.inf if rng.random() < 0.5 else -math.inf]
    specials = [math.nan, -0.0, 0.0, 2.0 ** 63, -1.5, 4.0e9] + inf
    ts, vals, x = [], [], float(rng.integers(0, 1000))
    for _ in range(n):
        ts.append(t)
        r = rng.random()
        if r < 0.15:
            vals.append(specials[int(rng.integers(0, len(specials)))])
        else:
            x += float(rng.integers(0, 300)) if r < 0.8 else -float(rng.integers(0, 500))
            vals.append(x if rng.random() < 0.7 else x + 0.25)
        t += int(rng.integers(1, 91)) * SEC
        if rng.random() < 0.04:
            t += 3 * WIN  # empty windows
    return np.array(ts, dtype=np.int64), np.array(vals, dtype=np.float64)


def _batch(int_opt, S=96, seed=5, both_inf=False, damage=True, n_max=200):
    rng = np.random.default_rng(seed)
    streams = []
    for s in range(S):
        ts, vals = _series(rng, int(rng.integers(1, n_max)), both_inf)
        b = O.encode_series(ts, vals, START, O.UNIT_S, int_opt)
        if damage and s % 17 == 4:
            b = b[: max(1, len(b) * 3 // 5)]  # truncated: a source decode error
        streams.append(b)
    return streams


def _csr(streams):
    off = np.zeros(len(streams) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(b) for b in streams])
    blob = np.frombuffer(b"".join(streams) + b"\0" * 16, dtype=np.uint8).copy()
    return torch.from_numpy(blob).cuda(), torch.from_numpy(off).cuda(), None


def _padded(streams):
    starts, pos = [], 0
    for b in streams:
        starts.append(pos)
        pos += (len(b) + 63) // 64 * 64
    blob = np.zeros(pos + 16, dtype=np.uint8)
    for p, b in zip(starts, streams):
        blob[p: p + len(b)] = np.frombuffer(b, dtype=np.uint8)
    t = lambda a: torch.tensor(a, dtype=torch.int64, device="cuda")
    return torch.from_numpy(blob).cuda(), t(starts), t([len(b) for b in streams])


def _state_host(st):
    return st.cpu().numpy().copy().view(X.XF_STATE_DTYPE).reshape(-1)


class Expect:
    """the oracle's view of a batch: each stream's datapoints (or its decode error) and each series' state"""

    def __init__(self, streams, int_opt, state=None):
        self.int_opt = int_opt
        self.src = [O.decode_series(b, int_opt, cap=4096) for b in streams]
        self.state = state if state is not None else np.zeros(len(streams), dtype=X.XF_STATE_DTYPE)

    def call(self, r0, step, n_win, metric, agg, ops, discard):
        """-> per series (status, bytes, n_tiles); advances the states of the series that succeed and keeps the
        datapoints each series writes in self.dps"""
        out = []
        self.dps = [[] for _ in self.src]
        for s, (ts, vals, n, err) in enumerate(self.src):
            if err != 0:
                out.append((err, b"", 0))
                continue
            st = self.state[s: s + 1].copy()
            tt, tv = X.aggregate_tiles_transform_series(ts[:n], vals[:n], r0, step, n_win, metric, agg, ops,
                                                        discard, st)
            self.state[s] = st[0]
            self.dps[s] = list(zip(tt.tolist(), tv.view(np.uint64).tolist()))
            out.append((0, O.encode_series(tt, tv, r0, O.UNIT_S, self.int_opt) if len(tt) else b"", len(tt)))
        return out


def _check(r, n_tiles, exp, only=None):
    st, ln, of = r.status.cpu().numpy(), r.out_len.cpu().numpy(), r.offsets.cpu().numpy()
    packed, nt = r.packed.cpu().numpy(), n_tiles.cpu().numpy()
    for s, (e_st, e_bytes, e_n) in enumerate(exp):
        if only is not None and s not in only:
            continue
        assert st[s] == e_st, (s, st[s], e_st)
        if e_st:
            assert ln[s] == 0 and nt[s] == 0, s
            continue
        assert nt[s] == e_n, (s, nt[s], e_n)
        assert ln[s] == len(e_bytes) and packed[of[s]: of[s] + ln[s]].tobytes() == e_bytes, s


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("addressing", ["csr", "lengths"])
@pytest.mark.parametrize("discard", [True, False])
def test_pipelines_against_oracle(codecs, int_opt, addressing, discard):
    """every pipeline, two consecutive calls carrying the state; damaged sources keep their state untouched"""
    codec = codecs[int_opt]
    streams = _batch(int_opt)
    blob, off, lengths = _csr(streams) if addressing == "csr" else _padded(streams)
    S = len(streams)
    for metric, agg, ops in PIPELINES:
        exp = Expect(streams, int_opt)
        state = codec.transform_state(S)
        # a state that is not new: an arbitrary earlier history for every series (the damaged ones too)
        init = np.zeros(S, dtype=X.XF_STATE_DTYPE)
        init["has_prev"][::3] = 1
        init["prev_t"][::3] = R0 - WIN
        init["prev_v"][::3] = 5.0
        init["sum"][::2, :] = 1.5
        exp.state[:] = init
        state.copy_(torch.from_numpy(init.view(np.uint8).reshape(S, 96)).cuda())
        for k in range(2):
            r0 = R0 + k * (N_WIN // 2) * WIN
            r, nt = codec.aggregate_tiles(blob, off, r0, WIN, N_WIN // 2, agg_type=agg, metric_type=metric,
                                          lengths=lengths, transforms=ops, discard_nan=discard, state=state)
            torch.cuda.synchronize()
            _check(r, nt, exp.call(r0, WIN, N_WIN // 2, metric, agg, ops, discard))
            assert _state_host(state).tobytes() == exp.state.tobytes(), (metric, agg, ops)
        assert (np.array([e[3] for e in exp.src]) != 0).any()  # damaged sources are in the batch


@pytest.mark.parametrize("int_opt", [True, False])
def test_both_infinities_and_nan_payloads(codecs, int_opt):
    """+Inf and -Inf in one series: Last / Min / Max carry the values' own bits (a window's NaN sum would be the
    hardware's), so Increase and Add meet Inf - Inf and write amd64's NaN"""
    codec = codecs[int_opt]
    streams = _batch(int_opt, S=64, seed=9, both_inf=True, damage=False)
    blob, off, _ = _csr(streams)
    for agg, ops in ((A.AGG_LAST, [INC]), (A.AGG_LAST, [ADD]), (A.AGG_MAX, [ADD, PS]), (A.AGG_MIN, [AB, ADD, RST])):
        for discard in (True, False):
            exp = Expect(streams, int_opt)
            state = codec.transform_state(len(streams))
            r, nt = codec.aggregate_tiles(blob, off, R0, WIN, N_WIN, agg_type=agg, transforms=ops,
                                          discard_nan=discard, state=state)
            torch.cuda.synchronize()
            _check(r, nt, exp.call(R0, WIN, N_WIN, A.METRIC_GAUGE, agg, ops, discard))
            assert _state_host(state).tobytes() == exp.state.tobytes()


@pytest.mark.parametrize("int_opt", [True, False])
def test_split_invariance(codecs, int_opt):
    """1, 2 and 7 consecutive calls carrying the state write the same datapoints as one call.  Every call's bytes
    equal the oracle's encoding of the datapoints it writes, and those datapoints, concatenated over the calls, are
    the same for every split.  In float mode the decoded streams show that directly; an int-optimised stream is
    not lossless for integers beyond 2^53 (the reference encoder's own recurrence, DESIGN.md §6), and a Counter's
    int64(NaN) = MinInt64 makes such rates, so there the decoded values depend on where a stream starts."""
    codec = codecs[int_opt]
    streams = _batch(int_opt, S=64, seed=13, damage=False, n_max=400)
    blob, off, _ = _csr(streams)
    S, n_win = len(streams), 14
    for metric, agg, ops in PIPELINES:
        results = {}
        for n_calls in (1, 2, 7):
            cuts = np.linspace(0, n_win, n_calls + 1).astype(int)
            state = codec.transform_state(S)
            exp = Expect(streams, int_opt)
            dps = [[] for _ in range(S)]
            decoded = [[] for _ in range(S)]
            for a, b in zip(cuts[:-1], cuts[1:]):
                r0 = R0 + int(a) * WIN
                r, nt = codec.aggregate_tiles(blob, off, r0, WIN, int(b - a), agg_type=agg, metric_type=metric,
                                              transforms=ops, discard_nan=False, state=state)
                torch.cuda.synchronize()
                _check(r, nt, exp.call(r0, WIN, int(b - a), metric, agg, ops, False))
                packed, of, ln = r.packed.cpu().numpy(), r.offsets.cpu().numpy(), r.out_len.cpu().numpy()
                for s in range(S):
                    dps[s] += exp.dps[s]
                    if ln[s] == 0:  # no non-empty window in this call: an empty stream
                        continue
                    ts, vals, n, err = O.decode_series(packed[of[s]: of[s] + ln[s]].tobytes(), int_opt, cap=64)
                    assert err == 0
                    decoded[s] += list(zip(ts[:n].tolist(), vals[:n].view(np.uint64).tolist()))
            assert _state_host(state).tobytes() == exp.state.tobytes()
            if not int_opt:
                assert decoded == dps
            results[n_calls] = (dps, exp.state.tobytes())
        assert results[1] == results[2] == results[7], (metric, agg, ops)


@pytest.mark.parametrize("int_opt", [True, False])
def test_capacity_then_grow_and_retry(codecs, int_opt):
    """a packed buffer too small for every warp: the series that got CAPACITY keep their state; re-running exactly
    those with a larger buffer gives the unstopped bytes and state"""
    codec = codecs[int_opt]
    streams = _batch(int_opt, S=160, seed=21, damage=False)
    blob, off, _ = _csr(streams)
    S = len(streams)
    ops = [INC, RST]
    state0 = codec.transform_state(S)
    codec.aggregate_tiles(blob, off, R0, WIN, 6, metric_type=A.METRIC_COUNTER, agg_type=A.AGG_SUM, transforms=ops,
                          state=state0)  # a history first
    full_state = state0.clone()
    full, full_nt = codec.aggregate_tiles(blob, off, R0 + 6 * WIN, WIN, 6, metric_type=A.METRIC_COUNTER,
                                          agg_type=A.AGG_SUM, transforms=ops, state=full_state)
    torch.cuda.synchronize()
    need = int(full.total.item())
    state = state0.clone()
    small, small_nt = codec.aggregate_tiles(blob, off, R0 + 6 * WIN, WIN, 6, metric_type=A.METRIC_COUNTER,
                                            agg_type=A.AGG_SUM, transforms=ops, state=state, capacity=need // 2)
    torch.cuda.synchronize()
    st = small.status.cpu().numpy()
    from m3_b200 import capi
    bad = np.nonzero(st == capi.ERR_CAPACITY)[0]
    good = np.nonzero(st == 0)[0]
    assert len(bad) > 0 and len(good) > 0 and len(bad) + len(good) == S
    sh, s0h, sfh = state.cpu().numpy(), state0.cpu().numpy(), full_state.cpu().numpy()
    assert (sh[bad] == s0h[bad]).all() and (sh[good] == sfh[good]).all()
    _check(small, small_nt, _as_exp(full, full_nt), only=set(good.tolist()))
    # retry the CAPACITY series, streams addressed in place through (offset, length)
    idx = torch.from_numpy(bad).cuda()
    o = off[:-1][idx].contiguous()
    ln = (off[1:] - off[:-1])[idx].contiguous()
    sub = state[idx].contiguous()
    r, nt = codec.aggregate_tiles(blob, o, R0 + 6 * WIN, WIN, 6, metric_type=A.METRIC_COUNTER, agg_type=A.AGG_SUM,
                                  transforms=ops, state=sub, lengths=ln)
    state[idx] = sub
    torch.cuda.synchronize()
    assert torch.equal(state, full_state)
    fe = _as_exp(full, full_nt)
    _check(r, nt, [fe[s] for s in bad.tolist()])


def _as_exp(r, nt):
    st, ln, of = r.status.cpu().numpy(), r.out_len.cpu().numpy(), r.offsets.cpu().numpy()
    packed, n = r.packed.cpu().numpy(), nt.cpu().numpy()
    return [(int(st[s]), packed[of[s]: of[s] + ln[s]].tobytes(), int(n[s])) for s in range(len(st))]


@pytest.mark.parametrize("int_opt", [True, False])
def test_reset_half_step_truncated_and_at_zero(codecs, int_opt):
    """a step of 61 s puts the Reset datapoint 30.5 s after the window's end, which a seconds stream truncates as the
    reference's encoder does; with windows ending at -1 s and a 2 s step one Reset datapoint falls on 0 and is not
    written"""
    codec = codecs[int_opt]
    rng = np.random.default_rng(4)
    for r0, step, n_win, start in ((R0, 61 * SEC, 10, START), (-11 * SEC, 2 * SEC, 10, -20 * SEC)):
        streams = []
        for s in range(40):
            pool = np.arange(start, r0 + step * n_win + 5 * SEC, SEC)
            ts = np.sort(rng.choice(pool, size=int(rng.integers(1, min(40, len(pool)))), replace=False))
            n = len(ts)
            vals = np.round(rng.normal(100, 50, size=n), 1)
            streams.append(O.encode_series(ts.astype(np.int64), vals, start, O.UNIT_S, int_opt))
        blob, off, _ = _csr(streams)
        for ops in ([RST], [PS, RST]):
            exp = Expect(streams, int_opt)
            state = codec.transform_state(len(streams))
            r, nt = codec.aggregate_tiles(blob, off, r0, step, n_win, agg_type=A.AGG_LAST, transforms=ops,
                                          discard_nan=False, state=state)
            torch.cuda.synchronize()
            e = exp.call(r0, step, n_win, A.METRIC_GAUGE, A.AGG_LAST, ops, False)
            _check(r, nt, e)
            assert _state_host(state).tobytes() == exp.state.tobytes()
            if r0 < 0:  # some series had a non-empty window ending at -1 s: fewer Reset datapoints than windows
                assert any(n_ % 2 == 1 for _, _, n_ in e)


def _raw(codec, blob, off, S, ops, n_ops, metric=A.METRIC_GAUGE, agg=A.AGG_LAST, state=None):
    from m3_b200 import capi
    from m3_b200.codec import PackedResult
    dev = codec.device
    cap = S * codec.encode_bound(2 * N_WIN)
    out = PackedResult(packed=torch.empty(cap, dtype=torch.uint8, device=dev),
                       offsets=torch.empty(S, dtype=torch.int64, device=dev),
                       out_len=torch.empty(S, dtype=torch.int64, device=dev),
                       status=torch.empty(S, dtype=torch.int32, device=dev),
                       total=torch.zeros(1, dtype=torch.int64, device=dev))
    n_tiles = torch.empty(S, dtype=torch.int32, device=dev)
    ops_a = (C.c_int32 * max(1, len(ops)))(*ops) if ops is not None else None
    rc = capi.lib().m3tsz_aggregate_tiles_transform(
        codec.ctx.handle, C.byref(codec.opts), blob.data_ptr(), blob.numel(), off.data_ptr(), None, S, R0, WIN,
        N_WIN, metric, agg, O.UNIT_S, 64, out.packed.data_ptr(), cap, out.offsets.data_ptr(), out.out_len.data_ptr(),
        out.status.data_ptr(), n_tiles.data_ptr(), out.total.data_ptr(), ops_a, n_ops, 1,
        state.data_ptr() if state is not None else None, None)
    return (out, n_tiles) if rc == 0 else rc


@pytest.mark.parametrize("int_opt", [True, False])
def test_no_ops_is_tiles_ex(codecs, int_opt):
    from test_gpu_aggregations import _tiles_ex_raw
    codec = codecs[int_opt]
    streams = _batch(int_opt, S=64, seed=2)
    blob, off, _ = _csr(streams)
    S = len(streams)
    for metric, agg in ((A.METRIC_GAUGE, A.AGG_LAST), (A.METRIC_COUNTER, A.AGG_SUM), (A.METRIC_GAUGE, A.AGG_STDEV)):
        state = codec.transform_state(S)
        a, na = _raw(codec, blob, off, S, [], 0, metric, agg, state)
        b, nb = _tiles_ex_raw(codec, blob, off, S, metric, agg)
        torch.cuda.synchronize()
        assert torch.equal(a.status, b.status) and torch.equal(na, nb) and torch.equal(a.out_len, b.out_len)
        assert int((state != 0).sum()) == 0  # no ops: no state written
        pa, pb = a.packed.cpu().numpy(), b.packed.cpu().numpy()
        oa, ob, ln = a.offsets.cpu().numpy(), b.offsets.cpu().numpy(), a.out_len.cpu().numpy()
        for s in range(S):
            assert (pa[oa[s]: oa[s] + ln[s]] == pb[ob[s]: ob[s] + ln[s]]).all(), (s, agg)


def test_invalid_pipelines_launch_nothing(codecs):
    from m3_b200 import capi
    codec = codecs[True]
    streams = _batch(True, S=8, damage=False)
    blob, off, _ = _csr(streams)
    S = len(streams)
    n0 = codec.launch_count()
    bad = [([PS, INC], 2), ([PS, PS], 2), ([INC, ADD, INC], 3), ([6], 1), ([0], 1), ([-1], 1), ([AB] * 9, 9),
           (None, 1)]
    for ops, n in bad:
        assert _raw(codec, blob, off, S, ops, n) == capi.ERR_INVALID_ARG, ops
    assert _raw(codec, blob, off, S, [PS], 1, A.METRIC_COUNTER, A.AGG_LAST) == capi.ERR_INVALID_ARG
    assert codec.launch_count() == n0
    with pytest.raises(capi.M3tszError):
        codec.aggregate_tiles(blob, off, R0, WIN, N_WIN, transforms=[INC, PS])
    assert codec.launch_count() == n0


@pytest.mark.parametrize("int_opt", [True, False])
def test_large_batch_sample(codecs, int_opt):
    """100 k series, a sample of them checked against the oracle"""
    from m3_b200 import synth
    S, P = 100_000, 240
    codec = codecs[int_opt]
    ts, vals, start = synth.gaussian_walk(S, P, "cuda", seed=5)
    vals = torch.round(vals * 4) / 4
    enc = codec.encode(ts, vals, start, unit=O.UNIT_S)
    packed, offsets = codec.compact(enc, align=64)
    s0 = int(start[0].item())
    step, n_win = 300 * SEC, 12
    hts, hvals = ts.cpu().numpy(), vals.cpu().numpy()
    for metric, agg, ops in ((A.METRIC_COUNTER, A.AGG_SUM, [PS]), (A.METRIC_GAUGE, A.AGG_LAST, [RST])):
        state = codec.transform_state(S)
        r, nt = codec.aggregate_tiles(packed, offsets, s0, step, n_win, agg_type=agg, metric_type=metric,
                                      transforms=ops, state=state)
        torch.cuda.synchronize()
        assert int((r.status != 0).sum()) == 0
        st = _state_host(state)
        pk, of, ln, n = r.packed.cpu().numpy(), r.offsets.cpu().numpy(), r.out_len.cpu().numpy(), nt.cpu().numpy()
        for s in np.random.default_rng(1).choice(S, size=300, replace=False).tolist() + [0, S - 1]:
            est = X.new_transform_state()
            tt, tv = X.aggregate_tiles_transform_series(hts[s], hvals[s], s0, step, n_win, metric, agg, ops, True,
                                                        est)
            assert n[s] == len(tt) and st[s: s + 1].tobytes() == est.tobytes(), s
            assert pk[of[s]: of[s] + ln[s]].tobytes() == O.encode_series(tt, tv, s0, O.UNIT_S, int_opt), s
