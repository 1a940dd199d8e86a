"""Encoder sets on the GPU (m3tsz_encoder_set_*): appends in any split give the bytes of one encode() and of the
oracle, snapshots at call boundaries are the oracle's Stream() of the prefix and decode to it, the state's public
prefix answers the reference's accessors, untouched series stay bit-identical, failing datapoints are dropped
whole, full slots grow, and the block flush (snapshot -> compact -> checksum) matches encode() at size."""
import numpy as np
import pytest
import torch

import oracle_lib as O
from m3_b200 import capi
from m3_b200.codec import BatchCodec

pytestmark = pytest.mark.gpu
SEC = 10 ** 9
START = 1599955200 * SEC


def _data(S, P, seed, int_opt):
    rng = np.random.default_rng(seed)
    ts = START + np.cumsum(rng.choice([10, 10, 10, 60, 1, 300], size=(S, P)), axis=1).astype(np.int64) * SEC
    kind = np.arange(S) % 5
    vals = np.where(kind[:, None] == 0, 100.0 + np.cumsum(rng.normal(size=(S, P)), axis=1),
                    np.round(rng.normal(size=(S, P)) * 1000, 2))
    vals[kind == 2] = np.round(np.cumsum(rng.normal(size=(int((kind == 2).sum()), P)), axis=1))  # int-like
    sp = [np.nan, np.inf, -np.inf, -0.0, 2.0 ** 63, -2.0 ** 63, 1e300, 3.0, 0.1 + 0.2]
    vals[kind == 3, ::17] = (sp * P)[: vals[kind == 3, ::17].shape[1]]
    return ts, vals


def _schedules(P, seed):
    r = np.random.default_rng(seed)
    chunks, left = [], P
    while left:
        c = int(min(left, r.choice([0, 1, 5, 8, 31, 64, 100])))
        chunks.append(c)
        left -= c
    return {"one": [P], "per_point": [1] * P, "ragged": chunks}


def _oracle_stream(ts, vals, int_opt):
    return O.encode_series(ts, vals, START, O.UNIT_S, int_opt) if len(ts) else b""


def _snapshot_bytes(es):
    r = es.stream()
    torch.cuda.synchronize()
    buf, ln = r.out.cpu().numpy(), r.out_len.cpu().numpy()
    return [buf[s, : ln[s]].tobytes() for s in range(es.n_series)], r


@pytest.mark.parametrize("S", [37, 64, 1000])
@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("point_major", [False, True])
def test_any_split_equals_encode_and_oracle(S, int_opt, point_major):
    P = 300
    codec = BatchCodec(0, int_optimized=int_opt)
    ts, vals = _data(S, P, S + 7 * int_opt, int_opt)
    t_ts, t_v = torch.from_numpy(ts).cuda(), torch.from_numpy(vals).cuda()
    start = torch.full((S,), START, dtype=torch.int64, device="cuda")
    ref = codec.encode(t_ts, t_v, start)
    torch.cuda.synchronize()
    r_out, r_len = ref.out.cpu().numpy(), ref.out_len.cpu().numpy()
    check = list(range(0, S, max(1, S // 12)))
    for name, sched in _schedules(P, S).items():
        if name == "per_point" and S == 1000:
            sched = [1] * 40 + [P - 40]
        es = codec.encoder_set(start, codec.encode_bound(P))
        i = 0
        snap_at = {1, len(sched) // 2}
        for k, c in enumerate(sched):
            a, b = t_ts[:, i: i + c], t_v[:, i: i + c]
            if point_major:
                a, b = a.t().contiguous(), b.t().contiguous()
            n_app, st = es.append(a.contiguous(), b.contiguous(), point_major=point_major)
            torch.cuda.synchronize()
            assert (st.cpu().numpy() == 0).all() and (n_app.cpu().numpy() == c).all(), (name, k)
            i += c
            if k in snap_at:
                got, _ = _snapshot_bytes(es)
                for s in check:
                    assert got[s] == _oracle_stream(ts[s, :i], vals[s, :i], int_opt), (name, k, s)
        got, _ = _snapshot_bytes(es)
        for s in range(S):
            assert got[s] == r_out[s, : r_len[s]].tobytes(), (name, s)
        for s in check:
            assert got[s] == _oracle_stream(ts[s], vals[s], int_opt), (name, s)


@pytest.mark.parametrize("int_opt", [True, False])
def test_snapshots_decode_accessors_and_untouched_series(int_opt):
    S, P = 64, 120
    codec = BatchCodec(0, int_optimized=int_opt)
    ts, vals = _data(S, P, 3, int_opt)
    t_ts, t_v = torch.from_numpy(ts).cuda(), torch.from_numpy(vals).cuda()
    es = codec.encoder_set(torch.full((S,), START, dtype=torch.int64, device="cuda"), codec.encode_bound(P))
    oracles = [O.Encoder(START, int_opt) for _ in range(S)]
    taken = np.zeros(S, dtype=np.int64)
    rng = np.random.default_rng(9)
    while taken.min() < P:
        n = np.minimum(rng.integers(0, 9, size=S), P - taken)
        n[rng.random(S) < 0.3] = 0  # untouched series this call
        C = int(n.max()) if n.max() > 0 else 1
        a = np.zeros((S, C), dtype=np.int64)
        b = np.zeros((S, C))
        for s in range(S):
            a[s, : n[s]] = ts[s, taken[s]: taken[s] + n[s]]
            b[s, : n[s]] = vals[s, taken[s]: taken[s] + n[s]]
        state0, buf0 = es.state.clone(), es.buf.clone()
        n_app, st = es.append(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda(),
                              n_points=torch.from_numpy(n.astype(np.int32)).cuda())
        torch.cuda.synchronize()
        assert (st.cpu().numpy() == 0).all() and (n_app.cpu().numpy() == n).all()
        idle = torch.from_numpy(n == 0).cuda()
        assert torch.equal(es.state[idle], state0[idle]) and torch.equal(es.buf[idle], buf0[idle])
        for s in range(S):
            for j in range(n[s]):
                assert oracles[s].encode(int(a[s, j]), float(b[s, j]), O.UNIT_S, b"") == 0
        taken += n
        got, snap = _snapshot_bytes(es)
        num = es.num_encoded.cpu().numpy()
        lt, lv = [x.cpu().numpy() for x in es.last_encoded]
        ln = es.len.cpu().numpy()
        cs = es.ann_checksum.cpu().numpy().view(np.uint64)
        for s in range(S):
            o = oracles[s]
            assert got[s] == (o.stream() or b""), s
            assert num[s] == o.num_encoded() and ln[s] == o.len()
            if num[s]:
                t, v, _ = o.last_encoded()
                assert lt[s] == t and np.float64(lv[s]).view(np.uint64) == np.float64(v).view(np.uint64)
                assert cs[s] == o.last_annotation_checksum()[0]
        # the snapshot decodes to the prefix, bit for bit as the oracle decodes it (int-optimised mode rounds values
        # such as 0.1 + 0.2 to their decimal, as the reference does)
        dec = codec.decode(snap.out.view(-1), es.offsets(), P, lengths=snap.out_len)
        torch.cuda.synchronize()
        dn = dec.n_points.cpu().numpy()
        for s in range(0, S, 7):
            k = int(taken[s])
            assert dn[s] == k
            if k == 0:
                continue
            e_ts, e_v, e_n, _ = O.decode_series(got[s], int_opt, cap=P)
            assert e_n == k and (e_ts == ts[s, :k]).all()
            assert (dec.ts[s, :k].cpu().numpy() == e_ts).all()
            assert (dec.values[s, :k].cpu().numpy().view(np.uint64) == e_v.view(np.uint64)).all()


@pytest.mark.parametrize("int_opt", [True, False])
def test_annotations_across_calls(int_opt):
    S, P = 40, 30
    codec = BatchCodec(0, int_optimized=int_opt)
    ts, vals = _data(S, P, 21, int_opt)
    anns = {}
    for s in range(S):
        for j in range(P):
            if (s + j) % 4 == 0:
                anns[(s, j)] = b"same-annotation" if s % 2 else bytes(range(s, s + 40))  # long: XXH64 32-byte path
    es = codec.encoder_set(torch.full((S,), START, dtype=torch.int64, device="cuda"), codec.encode_bound(P) + 4096)
    for c0 in range(0, P, 10):
        off, ent, blob = [0], [], b""
        for s in range(S):
            for j in range(c0, c0 + 10):
                if (s, j) in anns:
                    ent.append((j - c0, len(anns[(s, j)]), len(blob)))
                    blob += anns[(s, j)]
            off.append(len(ent))
        e = np.zeros(len(ent), dtype=[("i", "<u4"), ("l", "<u4"), ("o", "<u8")])
        for k, x in enumerate(ent):
            e[k] = x
        a_off = torch.tensor(off, dtype=torch.int64, device="cuda")
        a_ent = torch.from_numpy(e.view(np.uint8).reshape(-1, 16).copy()).cuda()
        a_b = torch.from_numpy(np.frombuffer(blob, dtype=np.uint8).copy()).cuda()
        n_app, st = es.append(torch.from_numpy(ts[:, c0: c0 + 10].copy()).cuda(),
                              torch.from_numpy(vals[:, c0: c0 + 10].copy()).cuda(), annotations=(a_off, a_ent, a_b))
        torch.cuda.synchronize()
        assert (st.cpu().numpy() == 0).all() and (n_app.cpu().numpy() == 10).all()
    got, _ = _snapshot_bytes(es)
    cs = es.ann_checksum.cpu().numpy().view(np.uint64)
    for s in range(S):
        o = O.Encoder(START, int_opt)
        for j in range(P):
            assert o.encode(int(ts[s, j]), float(vals[s, j]), O.UNIT_S, anns.get((s, j), b"")) == 0
        assert got[s] == o.stream(), s
        assert cs[s] == o.last_annotation_checksum()[0]


@pytest.mark.parametrize("int_opt", [True, False])
def test_errors_capacity_mode_and_reset(int_opt):
    S, P = 64, 60
    codec = BatchCodec(0, int_optimized=int_opt)
    ts, vals = _data(S, P, 33, int_opt)
    bad = 5
    ts[bad, 25:] += (1 << 33) * SEC  # second-unit delta-of-delta overflow at datapoint 25 of series 5
    start = torch.full((S,), START, dtype=torch.int64, device="cuda")
    es = codec.encoder_set(start, codec.encode_bound(P))
    n_app, st = es.append(torch.from_numpy(ts[:, :40].copy()).cuda(), torch.from_numpy(vals[:, :40].copy()).cuda())
    torch.cuda.synchronize()
    n_app, st = n_app.cpu().numpy(), st.cpu().numpy()
    assert st[bad] == capi.ERR_DOD_OVERFLOW and n_app[bad] == 25
    assert (np.delete(st, bad) == 0).all() and (np.delete(n_app, bad) == 40).all()
    # drop the failing datapoint, append the rest (shifted back so that they fit the series)
    rest = ts[:, 40:].copy()
    rest[bad] -= (1 << 33) * SEC
    fix = ts[bad, 26:40] - (1 << 33) * SEC
    n = np.where(np.arange(S) == bad, 14, 0).astype(np.int32)
    a = np.zeros((S, 14), dtype=np.int64)
    a[bad] = fix
    b = np.zeros((S, 14))
    b[bad] = vals[bad, 26:40]
    es.append(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda(), n_points=torch.from_numpy(n).cuda())
    es.append(torch.from_numpy(rest).cuda(), torch.from_numpy(vals[:, 40:].copy()).cuda())
    got, _ = _snapshot_bytes(es)
    keep = np.r_[0:25, 26:P]
    fixed = ts[bad].copy()
    fixed[25:] -= (1 << 33) * SEC
    assert got[bad] == _oracle_stream(fixed[keep], vals[bad, keep], int_opt)
    assert got[0] == _oracle_stream(ts[0], vals[0], int_opt)
    # capacity: a small slot stops each series where the rule says; grow and finish gives the one-shot bytes
    ts, vals = _data(S, P, 34, int_opt)
    t_ts, t_v = torch.from_numpy(ts).cuda(), torch.from_numpy(vals).cuda()
    small = 256
    es = codec.encoder_set(start, small)
    n_app, st = es.append(t_ts, t_v)
    torch.cuda.synchronize()
    n_app, st = n_app.cpu().numpy(), st.cpu().numpy()
    for s in range(S):
        o = O.Encoder(START, int_opt)
        exp = 0
        for j in range(P):
            raw, pos = o.raw()
            bits = (len(raw) - 1) * 8 + pos if raw else 0
            words = (bits >> 5) + (2 if j == 0 else 0)  # the first datapoint follows the 64-bit start
            if words + 14 > small // 4:
                break
            o.encode(int(ts[s, j]), float(vals[s, j]), O.UNIT_S, b"")
            exp += 1
        assert n_app[s] == exp and st[s] == (capi.ERR_CAPACITY if exp < P else 0), s
    es.grow(codec.encode_bound(P))
    n_rest = torch.from_numpy((P - n_app).astype(np.int32)).cuda()
    a = np.zeros_like(ts)
    b = np.zeros_like(vals)
    for s in range(S):
        a[s, : P - n_app[s]] = ts[s, n_app[s]:]
        b[s, : P - n_app[s]] = vals[s, n_app[s]:]
    n2, st2 = es.append(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda(), n_points=n_rest)
    ref = codec.encode(t_ts, t_v, start)
    torch.cuda.synchronize()
    assert (st2.cpu().numpy() == 0).all()
    got, _ = _snapshot_bytes(es)
    r_out, r_len = ref.out.cpu().numpy(), ref.out_len.cpu().numpy()
    for s in range(S):
        assert got[s] == r_out[s, : r_len[s]].tobytes(), s
    # mode mismatch: a state reset with the other int_optimized is refused and stays untouched
    other = BatchCodec(0, int_optimized=not int_opt)
    before = es.state.clone()
    es.codec = other
    n3, st3 = es.append(t_ts[:, :3].contiguous(), t_v[:, :3].contiguous())
    torch.cuda.synchronize()
    assert (st3.cpu().numpy() == capi.ERR_INVALID_ARG).all() and (n3.cpu().numpy() == 0).all()
    assert torch.equal(es.state, before)
    # reset re-arms: fresh streams from the new start
    es.codec = codec
    start2 = start + 7200 * SEC
    es.reset(start2)
    assert int(es.len.sum().item()) == 0
    t2 = t_ts[:, :20] + 7200 * SEC
    es.append(t2.contiguous(), t_v[:, :20].contiguous())
    got, _ = _snapshot_bytes(es)
    for s in (0, 17, S - 1):
        assert got[s] == O.encode_series(t2[s].cpu().numpy(), vals[s, :20], START + 7200 * SEC, O.UNIT_S, int_opt)


def test_at_size_block_flush_matches_encode():
    """200 k encoders x 720 datapoints appended one per call (720 launches), then snapshot -> compact ->
    checksum: the lengths and Adler-32 checksums of encode() on the same data"""
    from m3_b200 import synth
    S, P = 200_000, 720
    codec = BatchCodec(0, int_optimized=True)
    ts, vals, start = synth.gaussian_walk(S, P, "cuda", seed=5)
    tsp, vap = ts.t().contiguous(), vals.t().contiguous()
    es = codec.encoder_set(start, codec.encode_bound(P))
    for i in range(P):
        n_app, st = es.append(tsp[i: i + 1], vap[i: i + 1], point_major=True)
    torch.cuda.synchronize()
    assert int((st != 0).sum()) == 0 and int((n_app != 1).sum()) == 0
    snap = es.stream()
    packed, offsets = codec.compact(snap, align=16)
    c_app, s_app = codec.segment_checksums(packed, offsets)
    ref = codec.encode(ts, vals, start)
    packed_r, offsets_r = codec.compact(ref, align=16)
    c_ref, s_ref = codec.segment_checksums(packed_r, offsets_r)
    torch.cuda.synchronize()
    assert torch.equal(snap.out_len, ref.out_len)
    assert torch.equal(c_app, c_ref) and int((s_app != 0).sum()) == 0 and int((s_ref != 0).sum()) == 0
