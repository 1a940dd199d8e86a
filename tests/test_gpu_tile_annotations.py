"""Tile aggregation that keeps annotations on the GPU (m3tsz_aggregate_tiles_annotated: the fused decode's modes 6-8
and the tile stage's IN = 6 instantiation): bytes, out_len, n_tiles, status and the saved element record against the
oracle (the reference iterator's annotations, the window rule, the element, the reference encoder with annotations;
ann_oracle_lib.aggregate_tiles_annotated_series), in both int_optimized modes and both stream addressings; the
equivalence with m3tsz_aggregate_tiles_types on sources without annotations; and the round trip through decode."""
import math

import numpy as np
import pytest
import torch

import agg_oracle_lib as A
import ann_oracle_lib as N
import elem_oracle_lib as E
import oracle_lib as O
from m3_b200 import capi
from test_gpu_transforms import R0, START, WIN, _csr, _padded, codecs  # noqa: F401

pytestmark = pytest.mark.gpu

SEC = 10 ** 9
N_WIN = 12
AB, PS, INC, ADD, RST = 1, 2, 3, 4, 5
# annotation.Payload{OpenMetricsFamilyType: COUNTER, OpenMetricsHandleValueResets: true}
PROM_COUNTER_PAYLOAD = bytes([0x08, 0x01, 0x10, 0x01])
ERR_STREAM_TOO_LARGE = 104  # M3TSZ_ERR_STREAM_TOO_LARGE

# (metric, types, ops): modes 6 / 7 / 8 of the decode, k = 1 and k = 3 with and without Add, a Reset op
ELEMENTS = [
    (A.METRIC_GAUGE, [1], []),
    (A.METRIC_COUNTER, [7], [RST]),
    (A.METRIC_GAUGE, [2, 3, 7], [ADD]),
    (A.METRIC_GAUGE, [1, 2, 3], []),
    (A.METRIC_GAUGE, [8, 9], [RST, AB]),
    (A.METRIC_COUNTER, [2, 3, 7], [INC, ADD]),
]


def _blob(rng, n):
    return bytes(rng.integers(0, 256, size=n).astype(np.uint8))


def _encode(dps, int_opt):
    enc = O.Encoder(START, int_opt)
    for t, v, a in dps:
        assert enc.encode(int(t), float(v), O.UNIT_S, a) == 0
    return enc.stream() or b""


def _in_order(rng, n=80, gap=13):
    """n datapoints from two windows before the range to past its end, values with a NaN run"""
    t0 = R0 - 2 * WIN + int(rng.integers(1, 30)) * SEC
    out = []
    for i in range(n):
        v = math.nan if 30 <= i < 34 else float(rng.integers(0, 500)) / (1 if i % 3 else 4)
        out.append([t0 + i * gap * SEC, v, b""])
    return out


def annotated_batch(int_opt, seed=5):
    """the cases of the issue, one per series (41 series: a ragged last warp), and their sources' bytes"""
    rng = np.random.default_rng(seed)
    cases = []

    def add(dps):
        cases.append([tuple(d) for d in dps])

    d = [[t + 2 * WIN, v, a] for t, v, a in _in_order(rng)]  # (inside the range from datapoint 0 on)
    d[0][2] = PROM_COUNTER_PAYLOAD  # the Prometheus case: datapoint 0 only
    add(d)
    d = _in_order(rng)  # changes mid-block; several in one window (the last wins); an empty one keeps the window's
    for i, a in ((12, b"a"), (13, b"bb"), (14, b""), (15, b"ccc"), (40, b"a"), (41, b"a"), (60, b"zz")):
        d[i][2] = a
    add(d)
    d = _in_order(rng)  # an out-of-order datapoint carries an annotation into an earlier window
    d[25][2] = b"early"
    late = [d[40][0] - 3 * WIN + 7 * SEC, 11.0, b"late-into-an-earlier-window"]
    d.insert(50, late)
    d[52][2] = b"x"
    add(d)
    d = _in_order(rng, n=120)  # annotations outside the range only
    d[0][2] = b"before"
    d[1][2] = b"before2"
    d[-1][2] = b"after"
    add(d)
    d = _in_order(rng)  # an annotated NaN window (discard_nan drops it, its annotation with it)
    d[31][2] = b"nan-window"
    add(d)
    for n in (1, 63, 64, 200, 4100, 5000):  # lengths; the long ones cross the decoder's ring
        d = _in_order(rng)
        d[10][2] = _blob(rng, n)
        d[11][2] = _blob(rng, n)
        d[50][2] = d[10][2]
        add(d)
    add(_in_order(rng))  # none
    for _ in range(41 - len(cases) - 1):  # random positions, repeats, out-of-order
        d = _in_order(rng, n=int(rng.integers(5, 120)), gap=int(rng.integers(5, 40)))
        pool = [_blob(rng, int(rng.choice([1, 7, 64, 300]))) for _ in range(3)]
        for i in range(len(d)):
            if rng.random() < 0.2:
                d[i][2] = pool[int(rng.integers(0, 3))]
        if len(d) > 6 and rng.random() < 0.5:
            j = int(rng.integers(1, len(d) - 3))
            d[j], d[j + 2] = d[j + 2], d[j]
        add(d)
    streams = [_encode(c, int_opt) for c in cases]
    # a source truncated inside an annotation: the 4100-byte one of series 9's datapoint 10, cut 1000 bytes in
    # (what precedes it is about as long as the stream of datapoints 0-9)
    assert len(cases[9][10][2]) == 4100
    streams.append(streams[9][: len(_encode(cases[9][:10], int_opt)) + 1000])
    return streams


class Expect:
    """the oracle over a batch: [type][series] (status, bytes, n_tiles) and each series' record"""

    def __init__(self, streams, int_opt):
        self.streams, self.int_opt = streams, int_opt
        self.state = np.zeros(len(streams), dtype=E.ELEM_STATE_DTYPE)

    def call(self, r0, n_win, metric, types, ops, discard, save=None):
        k = len(types)
        out = [[None] * len(self.streams) for _ in range(k)]
        for s, src in enumerate(self.streams):
            st = self.state[s: s + 1].copy()
            res, counts, err = N.aggregate_tiles_annotated_series(src, self.int_opt, r0, WIN, n_win, metric, types,
                                                                  ops, discard and len(ops) > 0, st)
            if err == 0 and (save is None or s in save):
                self.state[s] = st[0]
            for j in range(k):
                out[j][s] = (err, res[j], counts[j])
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


def _state_host(st):
    return st.cpu().numpy().copy().view(E.ELEM_STATE_DTYPE).reshape(-1)


def _run(codec, blob, off, lengths, r0, n_win, metric, types, ops, discard, state, capacity=None, annotations=True):
    return codec.aggregate_tiles_types(blob, off, r0, WIN, n_win, types, metric_type=metric, lengths=lengths,
                                       capacity=capacity, transforms=ops, discard_nan=discard, state=state,
                                       annotations=annotations)


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("addressing", ["csr", "lengths"])
def test_annotated_elements_against_oracle(codecs, int_opt, addressing):
    """every element, discard on and off, two consecutive calls carrying the record (nothing of the annotations
    carries over: the second call starts without one)"""
    codec = codecs[int_opt]
    streams = annotated_batch(int_opt)
    blob, off, lengths = _csr(streams) if addressing == "csr" else _padded(streams)
    S = len(streams)
    exp0 = Expect(streams, int_opt).call(R0, N_WIN, A.METRIC_GAUGE, [1], [], True)
    assert exp0[0][S - 1][0] != 0  # the truncated source fails
    for discard in (True, False):
        for metric, types, ops in ELEMENTS:
            state = codec.element_state(S)
            exp = Expect(streams, int_opt)
            half = N_WIN // 2
            for r0, n_win in ((R0, half), (R0 + half * WIN, N_WIN - half)):
                r, nt = _run(codec, blob, off, lengths, r0, n_win, metric, types, ops, discard, state)
                torch.cuda.synchronize()
                _check(r, nt, exp.call(r0, n_win, metric, types, ops, discard))
                assert _state_host(state).tobytes() == exp.state.tobytes(), (metric, types, ops)


@pytest.mark.parametrize("int_opt", [True, False])
def test_without_annotations_equals_tiles_types(codecs, int_opt):
    """sources without annotations: the outputs of m3tsz_aggregate_tiles_types, record included"""
    codec = codecs[int_opt]
    rng = np.random.default_rng(3)
    streams = [_encode(_in_order(rng, n=int(rng.integers(1, 120)), gap=int(rng.integers(5, 40))), int_opt)
               for _ in range(300)]
    blob, off, lengths = _csr(streams)
    S = len(streams)
    for metric, types, ops in ELEMENTS:
        outs = []
        for ann in (False, True):
            state = codec.element_state(S)
            r, nt = _run(codec, blob, off, lengths, R0, N_WIN, metric, types, ops, True, state, annotations=ann)
            torch.cuda.synchronize()
            rows = [[r.packed[int(r.offsets[j, s]): int(r.offsets[j, s]) + int(r.out_len[j, s])].cpu().numpy()
                     .tobytes() for s in range(S)] for j in range(len(types))]
            outs.append((rows, r.out_len.cpu(), r.status.cpu(), nt.cpu(), state.cpu()))
        (a, la, sa, ta, za), (b, lb, sb, tb, zb) = outs
        assert a == b and torch.equal(la, lb) and torch.equal(sa, sb) and torch.equal(ta, tb) and torch.equal(za, zb)


def _first_annotation(codec, tiles, s, j=0):
    """decode(..., want_annotations=True) of one tile stream: (bytes of its first annotation, count)"""
    o, n = int(tiles.offsets[j, s]), int(tiles.out_len[j, s])
    seg = tiles.packed[o: o + n].contiguous()
    d = codec.decode(seg, torch.tensor([0, n], dtype=torch.int64, device="cuda"), 4 * N_WIN, want_annotations=True)
    torch.cuda.synchronize()
    ref = d.annotations[0].cpu().numpy().view(np.uint64)
    bit, ln, cnt = int(ref[0]), int(ref[1] & 0xffffffff), int(ref[1] >> 32)
    bits = np.unpackbits(seg.cpu().numpy())
    return np.packbits(bits[bit: bit + 8 * ln]).tobytes(), cnt


@pytest.mark.parametrize("int_opt", [True, False])
def test_round_trip_first_annotation(codecs, int_opt):
    """the tiles' first annotation, as the Prometheus conversion's FirstAnnotation() reads it, is the source's"""
    codec = codecs[int_opt]
    streams = annotated_batch(int_opt)
    blob, off, lengths = _csr(streams)
    tiles, _ = _run(codec, blob, off, lengths, R0, N_WIN, A.METRIC_COUNTER, [7], [], True, None)
    torch.cuda.synchronize()
    assert _first_annotation(codec, tiles, 0) == (PROM_COUNTER_PAYLOAD, 1)
    # the series with an annotation per size: its first tile's window holds the datapoints 10 and 11 (the last wins)
    for s in range(5, 11):
        src_anns = N.decode_annotated(streams[s], int_opt)[2]
        got, cnt = _first_annotation(codec, tiles, s)
        assert got == src_anns[11] and cnt >= 1, s


@pytest.mark.parametrize("int_opt", [True, False])
def test_capacity_then_retry(codecs, int_opt):
    """a packed buffer too small for every row: CAPACITY on some rows and no record for their series; the same call
    over those series with a larger buffer gives the unstopped result"""
    codec = codecs[int_opt]
    streams = annotated_batch(int_opt, seed=8)[:-1]
    blob, off, lengths = _padded(streams)
    S = len(streams)
    metric, types, ops = A.METRIC_GAUGE, [7], [ADD]
    state = codec.element_state(S)
    exp = Expect(streams, int_opt)
    full = exp.call(R0, N_WIN, metric, types, ops, True, save=set())
    # 40 rows, two warps: room for one warp's rows (the first one holds the long annotations), not for both
    need = sum(len(full[0][s][1]) + 64 for s in range(S))
    r, nt = _run(codec, blob, off, lengths, R0, N_WIN, metric, types, ops, True, state, capacity=int(need * 0.6))
    torch.cuda.synchronize()
    st = r.status.cpu().numpy()
    failed = sorted({s for s in range(S) if (st[:, s] == capi.ERR_CAPACITY).any()})
    ok = [s for s in range(S) if s not in failed]
    assert failed and ok
    _check(r, nt, full, only=set(ok))
    host = _state_host(state)
    for s in failed:
        assert host[s].tobytes() == bytes(E.ELEM_STATE_DTYPE.itemsize), s
    # retry the failed series alone (their records are still new)
    sub = [streams[s] for s in failed]
    b2, o2, l2 = _padded(sub)
    st2 = codec.element_state(len(sub))
    r2, nt2 = _run(codec, b2, o2, l2, R0, N_WIN, metric, types, ops, True, st2)
    torch.cuda.synchronize()
    _check(r2, nt2, Expect(sub, int_opt).call(R0, N_WIN, metric, types, ops, True))


def test_stream_too_large_status(codecs):
    """a source of 2^28 bytes, whose annotation offsets would not fit the packed reference: STREAM_TOO_LARGE on all
    of its rows, nothing written; the other series are unaffected"""
    codec = codecs[True]
    good = _encode([(R0 + 5 * SEC, 1.0, b"ok")], True)
    n_big = 1 << 28
    blob = torch.zeros(n_big + 4096, dtype=torch.uint8, device="cuda")
    blob[:len(good)] = torch.tensor(list(good), dtype=torch.uint8, device="cuda")
    off = torch.tensor([0, 2048], dtype=torch.int64, device="cuda")
    lengths = torch.tensor([len(good), n_big], dtype=torch.int64, device="cuda")
    r, nt = codec.aggregate_tiles_types(blob, off, R0, WIN, N_WIN, [2, 7], lengths=lengths, annotations=True,
                                        capacity=1 << 20)
    torch.cuda.synchronize()
    st = r.status.cpu().numpy()
    assert (st[:, 1] == ERR_STREAM_TOO_LARGE).all() and (st[:, 0] == 0).all()
    assert (r.out_len.cpu().numpy()[:, 1] == 0).all() and (nt.cpu().numpy()[:, 1] == 0).all()
    del blob
    torch.cuda.empty_cache()


def test_invalid_arguments(codecs):
    codec = codecs[True]
    blob, off, lengths = _csr([_encode([(R0 + 5 * SEC, 1.0, b"a")], True)])
    for types in ([], [3, 2], [1] * 9):
        with pytest.raises(Exception):
            codec.aggregate_tiles_types(blob, off, R0, WIN, N_WIN, types, annotations=True)
    with pytest.raises(Exception):
        codec.aggregate_tiles_types(blob, off, R0, WIN, N_WIN, [1], metric_type=A.METRIC_COUNTER, annotations=True)


def _encode_gpu_annotated(codec, S, P, seed):
    """S series x P datapoints from the synthetic walk, annotations (1-80 bytes) at 0-3 random datapoints of each
    series, encoded on the device -> (blob, offsets, lengths) with lengths addressing"""
    from m3_b200 import synth
    rng = np.random.default_rng(seed)
    ts, vals, start = synth.gaussian_walk(S, P, "cuda", seed=seed)
    n_ann = rng.integers(0, 4, size=S)
    series_off = np.zeros(S + 1, dtype=np.int64)
    series_off[1:] = np.cumsum(n_ann)
    E_ = int(series_off[-1])
    dp = np.concatenate([np.sort(rng.choice(P, size=k, replace=False)) for k in n_ann]).astype(np.uint32) \
        if E_ else np.zeros(0, dtype=np.uint32)
    ln = rng.integers(1, 81, size=E_).astype(np.uint32)
    boff = np.zeros(E_, dtype=np.uint64)
    boff[1:] = np.cumsum(ln[:-1])
    ann_bytes = rng.integers(0, 256, size=max(1, int(ln.sum()))).astype(np.uint8)
    ent = np.zeros(E_, dtype=[("dp", "<u4"), ("len", "<u4"), ("off", "<u8")])
    ent["dp"], ent["len"], ent["off"] = dp, ln, boff
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    enc = codec.encode(ts, vals, start, annotations=(to(series_off), to(ent.view(np.uint8).reshape(-1, 16)),
                                                     to(ann_bytes)))
    torch.cuda.synchronize()
    assert int((enc.status != 0).sum()) == 0
    stride = enc.out.shape[1]
    offsets = torch.arange(S, dtype=torch.int64, device="cuda") * stride
    return enc.out.view(-1), offsets, enc.out_len, int(start[0].item())


@pytest.mark.parametrize("int_opt", [True, False])
def test_large_batch_random_positions(codecs, int_opt):
    """64 k series x 1440 datapoints, annotations at random positions: sampled rows against the oracle"""
    codec = codecs[int_opt]
    S, P = 65536, 1440
    blob, off, lengths, start = _encode_gpu_annotated(codec, S, P, seed=21 + int(int_opt))
    step = 300 * SEC
    r0 = start
    types, ops = [1, 2, 3], [ADD]
    r, nt = codec.aggregate_tiles_types(blob, off, r0, step, 288, types, lengths=lengths, transforms=ops,
                                        annotations=True)
    torch.cuda.synchronize()
    assert int((r.status != 0).sum()) == 0
    host_blob, host_off, host_len = blob.cpu().numpy(), off.cpu().numpy(), lengths.cpu().numpy()
    rng = np.random.default_rng(4)
    sample = sorted(set(rng.choice(S, size=48, replace=False).tolist()) | {0, 31, 32, S - 1})
    packed, of, ln, ntt = r.packed.cpu().numpy(), r.offsets.cpu().numpy(), r.out_len.cpu().numpy(), nt.cpu().numpy()
    for s in sample:
        src = host_blob[host_off[s]: host_off[s] + host_len[s]].tobytes()
        st = E.new_element_state()
        rows, counts, err = N.aggregate_tiles_annotated_series(src, int_opt, r0, step, 288, A.METRIC_GAUGE, types, ops,
                                                               True, st)
        assert err == 0
        for j in range(len(types)):
            assert ntt[j, s] == counts[j] and packed[of[j, s]: of[j, s] + ln[j, s]].tobytes() == rows[j], (s, j)
