"""Bucket writes on the GPU (BatchCodec.bucket_set, m3tsz_encoder_set_write) against the BufferBucket.write model
over the ORACLE encoder (bucket_model.py): every per-datapoint result, every encoder's snapshot bytes and public
prefix, and read() against the oracle merge of the model's streams, in both modes, for both input layouts, for
series counts off a multiple of 32 and K = 1, 2, 4, 12, over many calls.  Also CAPACITY from a full slot and from an
exhausted pool followed by grow and re-send, untouched buckets, K = 1 in-order traffic against append, and one
at-size batch."""
import json
import os

import numpy as np
import pytest
import torch

import oracle_lib as O
from bucket_model import ERR_CAPACITY, SEC, Bucket, random_calls
from m3_b200 import capi
from m3_b200.codec import BatchCodec

pytestmark = pytest.mark.gpu
START = 1599955200 * SEC


def _inputs(calls, S, point_major, units, anns):
    """one call of every series -> (ts, vals, n_points, units, annotations) device tensors"""
    P = max(1, max(len(c) for c in calls))
    ts = np.zeros((S, P), np.int64)
    vals = np.zeros((S, P), np.float64)
    un = np.full((S, P), O.UNIT_S, np.uint8)
    n = np.array([len(c) for c in calls], np.int32)
    off, ents, blob = [0], [], b""
    for s, c in enumerate(calls):
        for j, (t, v, u, a) in enumerate(c):
            ts[s, j], vals[s, j], un[s, j] = t, v, u
            if a:
                ents.append((j | (len(a) << 32), len(blob)))
                blob += a
        off.append(len(ents))
    if point_major:
        ts, vals = ts.T.copy(), vals.T.copy()
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    ann = None
    if anns:
        e = np.array(ents or [(0, 0)], np.uint64).view(np.uint8).reshape(-1, 16)
        ann = (d(np.array(off, np.int64)), d(e), d(np.frombuffer(blob + b"\0", np.uint8).copy()))
    return d(ts), d(vals), d(n), (d(un) if units else None), ann


def _check_encoders(bs, models, what):
    prim, pool = bs.stream()
    pb, pl = prim.out.cpu().numpy(), prim.out_len.cpu().numpy()
    qb, ql = pool.out.cpu().numpy(), pool.out_len.cpu().numpy()
    table = bs.table.cpu().numpy()
    n_open = bs.open_encoders().cpu().numpy()
    for s, m in enumerate(models):
        assert n_open[s] == len(m.encs), (what, s)
        for i, e in enumerate(m.encs):
            exp = e.stream() or b""
            if i == 0:
                got = pb[s, : pl[s]].tobytes()
            else:
                r = table[s, i - 1]
                got = qb[r, : ql[r]].tobytes()
            assert got == exp, (what, s, i)
    for i in range(bs.encoders):
        num = bs.num_encoded(i).cpu().numpy()
        lt, lv = (x.cpu().numpy() for x in bs.last_encoded(i))
        cs = bs.ann_checksum(i).cpu().numpy().view(np.uint64)
        for s, m in enumerate(models):
            if i >= len(m.encs):
                assert num[s] == 0
                continue
            e = m.encs[i]
            assert num[s] == e.num_encoded(), (what, s, i)
            if num[s]:
                t, v, err = e.last_encoded()
                assert (t, np.float64(v).view(np.uint64)) == (lt[s], np.float64(lv[s]).view(np.uint64)), (what, s, i)
                assert e.last_annotation_checksum()[0] == cs[s], (what, s, i)


def _check_untouched(bs, before, idle):
    """buckets without datapoints in a call keep every byte of their encoders and table row; pool records past the
    counter stay as they were"""
    state, buf, pool, pool_buf, table, _ = before
    idle = torch.tensor(idle, dtype=torch.int64, device="cuda")
    assert torch.equal(bs.primary.state[idle], state[idle]) and torch.equal(bs.primary.buf[idle], buf[idle])
    assert torch.equal(bs.table[idle], table[idle])
    recs = table[idle].flatten()
    recs = recs[recs >= 0].long()
    assert torch.equal(bs.pool[recs], pool[recs]) and torch.equal(bs.pool_buf[recs], pool_buf[recs])
    now = int(bs.pool_count.item())
    assert torch.equal(bs.pool[now:], pool[now:]) and torch.equal(bs.pool_buf[now:], pool_buf[now:])


def _check_read(bs, models, what):
    cap = max(1, max(sum(e.num_encoded() for e in m.encs) for m in models))
    ts, vals, n, st = (x.cpu().numpy() for x in bs.read(cap))
    for s, m in enumerate(models):
        et, ev, est = m.read()  # (a stream the reference's iterator ends with an error carries it into the read)
        assert st[s] == est, (what, s)
        assert n[s] == len(et), (what, s)
        assert (ts[s, : n[s]] == et).all(), (what, s)
        assert (vals[s, : n[s]].view(np.uint64) == ev.view(np.uint64)).all(), (what, s)


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("K", [1, 2, 4, 12])
@pytest.mark.parametrize("point_major", [False, True])
def test_bucket_write_matches_the_model(int_opt, K, point_major):
    S = 45
    codec = BatchCodec(int_optimized=int_opt)
    units = anns = not point_major  # (point-major input takes neither)
    per = [random_calls(97 * s + K + 7 * int_opt, START, 12, 5, int_opt, units=units and s % 3 == 1,
                        anns=anns and s % 2 == 0) for s in range(S)]
    models = [Bucket(START, int_opt, K) for _ in range(S)]
    bs = codec.bucket_set(torch.full((S,), START, dtype=torch.int64, device="cuda"), 4096, encoders=K,
                          pool_records=S * max(1, K - 1), pool_stride=2048)
    for c in range(12):
        calls = [per[s][c] for s in range(S)]
        ts, vals, n, un, ann = _inputs(calls, S, point_major, units, anns)
        before = (bs.primary.state.clone(), bs.primary.buf.clone(), bs.pool.clone(), bs.pool_buf.clone(),
                  bs.table.clone(), int(bs.pool_count.item()))
        res, status = bs.write(ts, vals, n_points=n, units=un, annotations=ann, point_major=point_major)
        _check_untouched(bs, before, [s for s in range(S) if not calls[s]])
        res = res.cpu().numpy()
        if point_major:
            res = res.T
        assert (status.cpu().numpy() == 0).all()
        for s in range(S):
            exp = [models[s].write(*dp) for dp in calls[s]]
            assert list(res[s, : len(exp)]) == exp, (c, s, calls[s])
        if c % 4 == 3:
            _check_encoders(bs, models, c)
    _check_encoders(bs, models, "end")
    _check_read(bs, models, "end")


def test_bucket_read_of_the_reference_tables():
    """the write tables of buffer_test.go (tests/golden/m3tsz_buffer_goldens.json): each write's wasWritten and
    error, the encoders opened, LastEncoded of each, and the read the reference asserts"""
    gold = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                                       "m3tsz_buffer_goldens.json")))
    codec = BatchCodec(int_optimized=True)
    for case in gold["cases"]:
        K = case["limit"] or capi.MAX_BUCKET_ENCODERS  # (a limit of 0 is the reference's "no limit")
        ws = case["writes"]
        bs = codec.bucket_set(torch.tensor([START], dtype=torch.int64, device="cuda"), 1024, encoders=K,
                              pool_records=16, pool_stride=1024)
        ts = torch.tensor([[START + w["offset_ns"] for w in ws]], dtype=torch.int64, device="cuda")
        vals = torch.tensor([[w["value"] for w in ws]], dtype=torch.float64, device="cuda")
        units = torch.tensor([[w["unit"] for w in ws]], dtype=torch.uint8, device="cuda")
        res, st = bs.write(ts, vals, units=units)
        exp = [0 if w["written"] else (capi.ERR_TOO_MANY_ENCODERS if w["error"] else -1) for w in ws]
        assert res.cpu().tolist()[0] == exp and st.item() == 0, case["name"]
        if "encoders" in case:
            assert bs.open_encoders().item() == case["encoders"], case["name"]
        if "last_encoded_offsets_ns" in case:
            last = [bs.last_encoded(i)[0].item() - START for i in range(case["encoders"])]
            assert last == case["last_encoded_offsets_ns"], case["name"]
        rt, rv, rn, rs = bs.read(16)
        assert rs.item() == 0, case["name"]
        got = list(zip(rt[0, : rn.item()].cpu().tolist(), rv[0, : rn.item()].cpu().tolist()))
        assert got == [(START + o, v) for o, v in case["read"]], case["name"]


def test_decode_of_a_first_write_far_before_the_block_start_matches_the_oracle():
    """a t == 0 write that opened an encoder of a bucket ~1.6e9 s after it: the reference's iterator returns the
    datapoint and then EOF; the device decode does the same, and read() carries the EOF"""
    for int_opt in (True, False):
        codec = BatchCodec(int_optimized=int_opt)
        bs = codec.bucket_set(torch.tensor([START], dtype=torch.int64, device="cuda"), 1024, encoders=2,
                              pool_records=4, pool_stride=1024)
        res, _ = bs.write(torch.tensor([[START + 10 * SEC, 0]], dtype=torch.int64, device="cuda"),
                          torch.tensor([[1.0, 2.5]], dtype=torch.float64, device="cuda"))
        assert res.cpu().tolist() == [[0, 0]]
        _, pool = bs.stream()
        stream = pool.out[0, : pool.out_len[0]]
        dps, err = O.decode_all(stream.cpu().numpy().tobytes(), int_opt)
        d = codec.decode(stream.contiguous(), torch.tensor([0, stream.numel()], dtype=torch.int64, device="cuda"), 8)
        assert (d.n_points.item(), d.status.item()) == (len(dps), err) == (1, 1)
        assert (d.ts[0, 0].item(), d.values[0, 0].item()) == (0, 2.5)
        m = Bucket(START, int_opt, 2)
        m.write(START + 10 * SEC, 1.0)
        m.write(0, 2.5)
        _check_read(bs, [m], "t0")


def test_bucket_upserts_in_one_call():
    """rewrites, exact duplicates and late writes of the same few timestamps in one call: the results and the read
    (the last write of every timestamp) as the model gives them"""
    codec = BatchCodec(int_optimized=True)
    t = [START + k * SEC for k in range(1, 7)]
    call = [(t[0], 1.0), (t[1], 2.0), (t[2], 3.0), (t[0], 1.0), (t[0], 4.0), (t[1], 5.0), (t[3], 6.0), (t[0], 7.0),
            (t[4], 8.0), (t[1], 9.0), (t[1], 9.0), (t[4], 8.0)]
    bs = codec.bucket_set(torch.tensor([START], dtype=torch.int64, device="cuda"), 1024, encoders=12,
                          pool_records=16, pool_stride=1024)
    ts = torch.tensor([[x[0] for x in call]], dtype=torch.int64, device="cuda")
    vals = torch.tensor([[x[1] for x in call]], dtype=torch.float64, device="cuda")
    res, st = bs.write(ts, vals)
    m = Bucket(START, True, 12)
    assert res.cpu().tolist()[0] == [m.write(a, b) for a, b in call]
    assert -1 in res.cpu().tolist()[0]
    _check_encoders(bs, [m], "upserts")
    _check_read(bs, [m], "upserts")
    et, ev, _ = m.read()
    assert list(et) == t[:5] and list(ev) == [7.0, 9.0, 3.0, 6.0, 8.0]


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("what", ["slot", "pool"])
def test_bucket_capacity_then_grow_and_resend(int_opt, what):
    """CAPACITY from a full slot or an exhausted pool stops the series at that datapoint; growing and sending exactly
    the stopped datapoints again gives the unstopped result"""
    S, K = 40, 4
    codec = BatchCodec(int_optimized=int_opt)
    per = [random_calls(31 * s + 3, START, 10, 8, int_opt, rare=False) for s in range(S)]
    models = [Bucket(START, int_opt, K) for _ in range(S)]
    stride, records = (96, 4 * S) if what == "slot" else (4096, 3)
    bs = codec.bucket_set(torch.full((S,), START, dtype=torch.int64, device="cuda"), stride, encoders=K,
                          pool_records=records, pool_stride=stride)
    stopped = 0
    for c in range(10):
        calls = [per[s][c] for s in range(S)]
        while True:
            ts, vals, n, _, _ = _inputs(calls, S, False, False, False)
            res, status = bs.write(ts, vals, n_points=n)
            res, status = res.cpu().numpy(), status.cpu().numpy()
            rest = [[] for _ in range(S)]
            for s in range(S):
                m = len(calls[s])
                if status[s] == ERR_CAPACITY:
                    j = int(np.argmax(res[s, :m] == ERR_CAPACITY))
                    assert (res[s, j:m] == ERR_CAPACITY).all()
                    rest[s] = calls[s][j:]
                    m = j
                    stopped += 1
                else:
                    assert status[s] == 0
                assert list(res[s, :m]) == [models[s].write(*dp) for dp in calls[s][:m]], (c, s)
            if not any(rest):
                break
            bs.grow(stride=bs.stride * 2, pool_stride=bs.pool_stride * 2, pool_records=bs.pool.shape[0] * 2)
            calls = rest
    assert stopped > 0
    _check_encoders(bs, models, what)
    _check_read(bs, models, what)


@pytest.mark.parametrize("point_major", [False, True])
def test_bucket_k1_in_order_is_append_and_leaves_idle_buckets_untouched(point_major):
    S, P = 70, 6
    codec = BatchCodec(int_optimized=True)
    start = torch.full((S,), START, dtype=torch.int64, device="cuda")
    bs = codec.bucket_set(start, 2048, encoders=1)
    es = codec.encoder_set(start, 2048)
    g = torch.Generator().manual_seed(3)
    for c in range(5):
        t = START + (torch.arange(P, dtype=torch.int64) + 1 + c * P) * 10 * SEC
        ts = t[None, :].repeat(S, 1)
        vals = torch.round(torch.randn((S, P), generator=g, dtype=torch.float64) * 100, decimals=1)
        n = torch.randint(0, P + 1, (S,), generator=g, dtype=torch.int32)
        n[5] = 0
        if point_major:
            ts, vals = ts.T.contiguous(), vals.T.contiguous()
        before = (bs.primary.state[5].clone(), bs.primary.buf[5].clone())
        ts, vals, n = ts.cuda(), vals.cuda(), n.cuda()
        res, status = bs.write(ts, vals, n_points=n, point_major=point_major)
        _, st2 = es.append(ts, vals, n_points=n, point_major=point_major)
        assert (status == 0).all() and (st2 == 0).all()
        assert (bs.primary.state[5] == before[0]).all() and (bs.primary.buf[5] == before[1]).all()
        assert torch.equal(bs.primary.state, es.state)
        a, b = bs.primary.stream(), es.stream()
        assert torch.equal(a.out_len, b.out_len)
        for s in range(S):
            assert torch.equal(a.out[s, : a.out_len[s]], b.out[s, : b.out_len[s]])


def test_bucket_write_at_size():
    """1 M buckets, 6 calls of mixed traffic (1 % late, 0.5 % rewrites of the last timestamp), a sample against the
    model"""
    S, K = 1 << 20, 4
    codec = BatchCodec(int_optimized=True)
    bs = codec.bucket_set(torch.full((S,), START, dtype=torch.int64, device="cuda"), 256, encoders=K,
                          pool_records=S // 8, pool_stride=128)
    g = torch.Generator(device="cuda").manual_seed(5)
    sample = torch.randint(0, S, (300,), generator=g, device="cuda").unique().cpu().numpy()
    models = {int(s): Bucket(START, True, K) for s in sample}
    for c in range(6):
        t = START + (c + 1) * 10 * SEC
        ts = torch.full((S, 2), t, dtype=torch.int64, device="cuda")
        u = torch.rand((S,), generator=g, device="cuda")
        late = u < 0.01
        rewrite = (u >= 0.01) & (u < 0.015)
        ts[:, 1] = torch.where(late, t - torch.randint(1, 11, (S,), generator=g, device="cuda") * 10 * SEC,
                               torch.full_like(ts[:, 1], t))
        vals = torch.round(torch.randn((S, 2), generator=g, device="cuda", dtype=torch.float64) * 50, decimals=2)
        n = torch.where(late | rewrite, 2, 1).to(torch.int32)
        res, status = bs.write(ts, vals, n_points=n)
        assert (status == 0).all()
        tsh, vh, nh, rh = ts.cpu().numpy(), vals.cpu().numpy(), n.cpu().numpy(), res.cpu().numpy()
        for s, m in models.items():
            exp = [m.write(int(tsh[s, j]), float(vh[s, j])) for j in range(nh[s])]
            assert list(rh[s, : nh[s]]) == exp, (c, s)
    prim, pool = bs.stream()
    table = bs.table.cpu().numpy()
    for s, m in models.items():
        for i, e in enumerate(m.encs):
            enc, r = (prim, s) if i == 0 else (pool, table[s, i - 1])
            got = enc.out[r, : enc.out_len[r]].cpu().numpy().tobytes()
            assert got == (e.stream() or b""), (s, i)
