"""Tile aggregation across source blocks on the GPU (m3tsz_aggregate_tiles_blocks: the fused decode's block loop and
the tile stage's IN = 7 instantiation): bytes, out_len, n_tiles, status and the element record against the composed
oracle (blocks_oracle_lib), in both int_optimized modes, both segment addressings and with and without annotations;
one block per series against the existing calls; the equivalence with the existing call on one concatenated stream
per series; errors, room and the annotation packing's limit; and the fileset path end to end."""
import ctypes as C

import numpy as np
import pytest
import torch

import blocks_oracle_lib as B
import elem_oracle_lib as E
import oracle_lib as O
from m3_b200 import capi, fileset
from test_gpu_tile_annotations import ELEMENTS, PROM_COUNTER_PAYLOAD, _check, _state_host, annotated_batch
from test_gpu_transforms import _csr, _padded, codecs  # noqa: F401
from test_tile_blocks_oracle import (B0, BS, COUNTER, GAUGE, N_WIN, R0, SEC, STEP, boundary_annotation_case, encode,
                                     plain_series, random_series)

pytestmark = pytest.mark.gpu

ERR_STREAM_TOO_LARGE = 104
ADD, RST = 4, 5


def layout(series, addressing):
    """series = [[block bytes, ...], ...] -> (blob, offsets, lengths, blocks) with one segment per (series, block)"""
    segs = [b for blocks in series for b in blocks]
    blob, off, lengths = _csr(segs) if addressing == "csr" else _padded(segs)
    bo = np.zeros(len(series) + 1, dtype=np.int64)
    bo[1:] = np.cumsum([len(blocks) for blocks in series])
    return blob, off, lengths, torch.from_numpy(bo).cuda()


def run(codec, inputs, r0, n_win, metric, types, ops, discard, state, annotations, capacity=None):
    blob, off, lengths, blocks = inputs
    return codec.aggregate_tiles_types(blob, off, r0, STEP, n_win, types, metric_type=metric, lengths=lengths,
                                       capacity=capacity, transforms=ops, discard_nan=discard, state=state,
                                       annotations=annotations, blocks=blocks)


class Expect:
    """the composed oracle over a batch of series given as block lists: [type][series] (status, bytes, n_tiles)"""

    def __init__(self, series, int_opt, annotations):
        self.series, self.int_opt, self.ann = series, int_opt, annotations
        self.state = np.zeros(len(series), dtype=E.ELEM_STATE_DTYPE)

    def call(self, r0, n_win, metric, types, ops, discard, save=None):
        out = [[None] * len(self.series) for _ in types]
        for s, blocks in enumerate(self.series):
            st = self.state[s: s + 1].copy()
            rows, counts, err = B.aggregate_tiles_blocks_series(blocks, self.int_opt, r0, STEP, n_win, metric, types,
                                                                ops, discard and len(ops) > 0, st, self.ann)
            if err == 0 and (save is None or s in save):
                self.state[s] = st[0]
            for j in range(len(types)):
                out[j][s] = (err, rows[j], counts[j])
        return out


def rows_of(r, k, S):
    return [[r.packed[int(r.offsets[j, s]): int(r.offsets[j, s]) + int(r.out_len[j, s])].cpu().numpy().tobytes()
             for s in range(S)] for j in range(k)]


def mixed_batch(int_opt, annotations, seed=11):
    """45 series (a ragged last warp): 0, 1, 2, 5 and 12 blocks with empty and missing blocks, unit and int / float
    changes, NaN runs, out-of-order and stray datapoints, equal timestamps across blocks; the hand-built boundary
    annotation case; a truncated and a corrupted middle block"""
    rng = np.random.default_rng(seed)
    series = [random_series(rng, (0, 1, 2, 5, 12)[i % 5], int_opt, annotations) for i in range(41)]
    series.append(boundary_annotation_case(int_opt)[0])
    good = plain_series(rng, 5, int_opt)
    series.append(good[:2] + [good[2][: len(good[2]) // 2]] + good[3:])            # truncated middle block
    bad = bytearray(good[2])
    bad[8] ^= 0xff
    series.append(good[:2] + [bytes(bad)] + good[3:])                              # corrupted middle block
    series.append([b"", b""])                                                      # only empty segments
    return series


@pytest.mark.parametrize("annotations", [False, True])
@pytest.mark.parametrize("addressing", ["csr", "lengths"])
@pytest.mark.parametrize("int_opt", [True, False])
def test_one_block_equals_the_existing_calls(codecs, int_opt, addressing, annotations):
    codec = codecs[int_opt]
    streams = annotated_batch(int_opt)
    S = len(streams)
    blob, off, lengths = _csr(streams) if addressing == "csr" else _padded(streams)
    blocks = torch.arange(S + 1, dtype=torch.int64, device="cuda")
    for metric, types, ops in ELEMENTS:
        outs = []
        for use_blocks in (False, True):
            state = codec.element_state(S)
            r, nt = codec.aggregate_tiles_types(blob, off, R0, STEP, N_WIN, types, metric_type=metric,
                                                lengths=lengths, transforms=ops, state=state, annotations=annotations,
                                                blocks=blocks if use_blocks else None)
            torch.cuda.synchronize()
            outs.append((rows_of(r, len(types), S), r.out_len.cpu(), r.status.cpu(), nt.cpu(), state.cpu()))
        (a, la, sa, ta, za), (b, lb, sb, tb, zb) = outs
        assert a == b and torch.equal(la, lb) and torch.equal(sa, sb) and torch.equal(ta, tb) and torch.equal(za, zb)


@pytest.mark.parametrize("annotations", [False, True])
@pytest.mark.parametrize("addressing", ["csr", "lengths"])
@pytest.mark.parametrize("int_opt", [True, False])
def test_blocks_against_oracle(codecs, int_opt, addressing, annotations):
    """every element, discard on and off, two consecutive calls carrying the record"""
    codec = codecs[int_opt]
    series = mixed_batch(int_opt, annotations)
    S = len(series)
    inputs = layout(series, addressing)
    for discard in (True, False):
        for metric, types, ops in ELEMENTS:
            state = codec.element_state(S)
            exp = Expect(series, int_opt, annotations)
            half = N_WIN // 2
            for r0, n_win in ((R0, half), (R0 + half * STEP, N_WIN - half)):
                r, nt = run(codec, inputs, r0, n_win, metric, types, ops, discard, state, annotations)
                torch.cuda.synchronize()
                e = exp.call(r0, n_win, metric, types, ops, discard)
                _check(r, nt, e)
                assert _state_host(state).tobytes() == exp.state.tobytes(), (metric, types, ops)
            st = r.status.cpu().numpy()
            assert (st[:, S - 3] != 0).all() and (st[:, S - 1] == 0).all()  # the truncated block; only empty ones


@pytest.mark.parametrize("int_opt", [True, False])
def test_two_calls_equal_one(codecs, int_opt):
    """consecutive window ranges write the datapoints of one call over the whole range, and the same final record"""
    codec = codecs[int_opt]
    rng = np.random.default_rng(12)
    series = [plain_series(rng, int(rng.integers(1, 13)), int_opt) for _ in range(70)]
    S = len(series)
    inputs = layout(series, "csr")
    metric, types, ops = GAUGE, [1, 2, 3], [ADD]
    one = codec.element_state(S)
    r, _ = run(codec, inputs, R0, N_WIN, metric, types, ops, True, one, False)
    whole = rows_of(r, 3, S)
    two = codec.element_state(S)
    parts = []
    for r0, n_win in ((R0, 7), (R0 + 7 * STEP, N_WIN - 7)):
        r, _ = run(codec, inputs, r0, n_win, metric, types, ops, True, two, False)
        parts.append(rows_of(r, 3, S))
    torch.cuda.synchronize()
    assert torch.equal(one.cpu(), two.cpu())
    dec = lambda b: list(zip(*_datapoints(b, int_opt)))
    for j in range(3):
        for s in range(S):
            assert dec(whole[j][s]) == dec(parts[0][j][s]) + dec(parts[1][j][s]), (j, s)


def _datapoints(b, int_opt):
    if not b:
        return [], []
    it = O.Iterator(b, int_opt, O.UNIT_S)
    ts, vs = [], []
    while it.next():
        t, v, _, _ = it.current()
        ts.append(t)
        vs.append(np.float64(v).view(np.int64))
    assert it.err() == 0
    return ts, vs


@pytest.mark.parametrize("int_opt", [True, False])
def test_without_annotations_equals_the_concatenated_call(codecs, int_opt):
    """GPU against GPU: the blocks call equals m3tsz_aggregate_tiles_types on one stream per series that encodes the
    concatenation, with transformations and the record over two calls"""
    codec = codecs[int_opt]
    rng = np.random.default_rng(13)
    series = [plain_series(rng, int(rng.integers(1, 13)), int_opt) for _ in range(300)]
    S = len(series)
    inputs = layout(series, "lengths")
    blob1, off1, _ = _csr([B.concat_stream(b, int_opt, B0) for b in series])
    for metric, types, ops in ELEMENTS:
        sa, sb = codec.element_state(S), codec.element_state(S)
        for r0, n_win in ((R0, 9), (R0 + 9 * STEP, N_WIN - 9)):
            ra, ta = run(codec, inputs, r0, n_win, metric, types, ops, True, sa, False)
            rb, tb = codec.aggregate_tiles_types(blob1, off1, r0, STEP, n_win, types, metric_type=metric,
                                                 transforms=ops, state=sb)
            torch.cuda.synchronize()
            assert rows_of(ra, len(types), S) == rows_of(rb, len(types), S)
            assert torch.equal(ra.status.cpu(), rb.status.cpu()) and torch.equal(ta.cpu(), tb.cpu())
            assert torch.equal(ra.out_len.cpu(), rb.out_len.cpu())
        assert torch.equal(sa.cpu(), sb.cpu())


def test_bad_block_range_is_that_series_error(codecs):
    codec = codecs[True]
    rng = np.random.default_rng(14)
    series = [plain_series(rng, 2, True) for _ in range(4)]
    blob, off, lengths, _ = layout(series, "csr")
    # series 1: a decreasing range; series 3: past n_segments (8); series 0 and 2 as listed
    blocks = torch.tensor([0, 2, 1, 6, 9], dtype=torch.int64, device="cuda")
    r, nt = codec.aggregate_tiles_types(blob, off, R0, STEP, N_WIN, [1, 2], blocks=blocks, annotations=True)
    torch.cuda.synchronize()
    st = r.status.cpu().numpy()
    assert (st[:, 1] == capi.ERR_INVALID_ARG).all() and (st[:, 3] == capi.ERR_INVALID_ARG).all()
    segs = [b for s in series for b in s]
    exp = Expect([segs[0:2], [], segs[1:6], []], True, True).call(R0, N_WIN, GAUGE, [1, 2], [], True)
    _check(r, nt, exp, only={0, 2})
    # no block table: refused before any launch
    rc = capi.lib().m3tsz_aggregate_tiles_blocks(codec.ctx.handle, C.byref(codec.opts), None, 0, None, None, 0, None,
                                                 1, R0, STEP, N_WIN, 1, (C.c_int32 * 1)(1), 1, 1, 64, None, 0, None,
                                                 None, None, None, None, None, 0, 0, None, 0, None)
    assert rc == capi.ERR_INVALID_ARG


@pytest.mark.parametrize("int_opt", [True, False])
def test_capacity_then_retry(codecs, int_opt):
    codec = codecs[int_opt]
    series = mixed_batch(int_opt, True, seed=15)[:40]
    S = len(series)
    inputs = layout(series, "lengths")
    metric, types, ops = GAUGE, [7], [ADD]
    state = codec.element_state(S)
    full = Expect(series, int_opt, True).call(R0, N_WIN, metric, types, ops, True, save=set())
    need = sum(len(full[0][s][1]) + 64 for s in range(S))
    r, nt = run(codec, inputs, R0, N_WIN, metric, types, ops, True, state, True, capacity=int(need * 0.6))
    torch.cuda.synchronize()
    st = r.status.cpu().numpy()
    failed = sorted({s for s in range(S) if (st[:, s] == capi.ERR_CAPACITY).any()})
    ok = [s for s in range(S) if s not in failed]
    assert failed and ok
    _check(r, nt, full, only=set(ok))
    host = _state_host(state)
    for s in failed:
        assert host[s].tobytes() == bytes(E.ELEM_STATE_DTYPE.itemsize), s
    sub = [series[s] for s in failed]
    st2 = codec.element_state(len(sub))
    r2, nt2 = run(codec, layout(sub, "csr"), R0, N_WIN, metric, types, ops, True, st2, True)
    torch.cuda.synchronize()
    _check(r2, nt2, Expect(sub, int_opt, True).call(R0, N_WIN, metric, types, ops, True))


def _annotations_of(b, int_opt):
    it = O.Iterator(b, int_opt, O.UNIT_S)
    out = []
    while it.next():
        out.append(it.current()[3])
    return out


@pytest.mark.parametrize("int_opt", [True, False])
def test_prometheus_payload_on_every_block(codecs, int_opt):
    """the payload on every block's first datapoint: each row writes it once"""
    codec = codecs[int_opt]
    series = []
    for _ in range(33):
        blocks = []
        for b in range(12):
            dps = [[t, v, u, a] for t, v, u, a in
                   [(B0 + b * BS + (3 + 20 * i) * SEC, float(i + b), O.UNIT_S, b"") for i in range(20)]]
            dps[0][3] = PROM_COUNTER_PAYLOAD
            blocks.append(encode(dps, int_opt, B0 + b * BS))
        series.append(blocks)
    inputs = layout(series, "csr")
    r, nt = run(codec, inputs, R0, N_WIN, COUNTER, [7], [RST], True, None, True)
    torch.cuda.synchronize()
    assert int((r.status != 0).sum()) == 0
    _check(r, nt, Expect(series, int_opt, True).call(R0, N_WIN, COUNTER, [7], [RST], True))
    for row in rows_of(r, 1, len(series))[0]:
        anns = _annotations_of(row, int_opt)
        assert [a for a in anns if a] == [PROM_COUNTER_PAYLOAD]


def test_annotation_packing_limit(codecs):
    """an annotation of 2^27 bytes does not fit the block-mode reference: STREAM_TOO_LARGE on all of its series' rows;
    one byte shorter fits; the other series are unaffected"""
    codec = codecs[True]
    small = encode([[B0 + 5 * SEC, 1.0, O.UNIT_S, b"a"], [R0 + 5 * SEC, 2.0, O.UNIT_S, b""]], True, B0)
    series = [[small]]
    for n in ((1 << 27) - 1, 1 << 27):
        big = encode([[R0 + 5 * SEC, 1.0, O.UNIT_S, b"\x5a" * n], [R0 + 65 * SEC, 2.0, O.UNIT_S, b""]], True, R0)
        series.append([small, big])
    inputs = layout(series, "csr")
    r, nt = codec.aggregate_tiles_types(inputs[0], inputs[1], R0, STEP, N_WIN, [2, 7], blocks=inputs[3],
                                        annotations=True)
    torch.cuda.synchronize()
    st = r.status.cpu().numpy()
    assert (st[:, 0] == 0).all() and (st[:, 1] == 0).all() and (st[:, 2] == ERR_STREAM_TOO_LARGE).all()
    assert (r.out_len.cpu().numpy()[:, 2] == 0).all() and (nt.cpu().numpy()[:, 2] == 0).all()
    # the fitting one carries its annotation into window 0
    o, n = int(r.offsets[0, 1]), int(r.out_len[0, 1])
    anns = _annotations_of(r.packed[o: o + n].cpu().numpy().tobytes(), True)
    assert anns[0] == b"\x5a" * ((1 << 27) - 1)
    del r, inputs
    torch.cuda.empty_cache()


@pytest.mark.parametrize("annotations", [False, True])
def test_fileset_end_to_end(codecs, tmp_path, annotations):
    """12 block volumes -> read_block_range -> upload -> segment_checksums -> the blocks call -> the oracle"""
    codec = codecs[True]
    rng = np.random.default_rng(17)
    ids = [b"series-%03d" % i for i in range(50)]
    per = {i: random_series(rng, 12, True, annotations) for i in ids}
    for b in range(12):
        present = [i for i in ids if per[i][b]]
        blob = b"".join(per[i][b] for i in present)
        off = np.cumsum([0] + [len(per[i][b]) for i in present[:-1]])
        fileset.write_fileset(str(tmp_path), "src", 0, B0 + b * BS, BS, present, blob, off,
                              [len(per[i][b]) for i in present])
    br = fileset.read_block_range(str(tmp_path), "src", 0, [B0 + b * BS for b in range(12)])
    d_data = torch.from_numpy(br.data.copy()).cuda()
    d_off, d_len = torch.from_numpy(br.offsets).cuda(), torch.from_numpy(br.sizes).cuda()
    _, cst = codec.segment_checksums(d_data, d_off, lengths=d_len,
                                     expected=torch.from_numpy(br.data_checksums.view(np.int32)).cuda())
    assert int((cst != 0).sum()) == 0
    blocks = torch.from_numpy(br.block_off).cuda()
    state = codec.element_state(len(br.ids))
    r, nt = codec.aggregate_tiles_types(d_data, d_off, R0, STEP, N_WIN, [2, 3, 7], lengths=d_len, transforms=[ADD],
                                        state=state, annotations=annotations, blocks=blocks)
    torch.cuda.synchronize()
    series = [[blk for blk in per[i] if blk] for i in br.ids]
    exp = Expect(series, True, annotations)
    _check(r, nt, exp.call(R0, N_WIN, GAUGE, [2, 3, 7], [ADD], True))
    assert _state_host(state).tobytes() == exp.state.tobytes()


@pytest.mark.parametrize("int_opt", [True, False])
def test_large_batch_12_blocks(codecs, int_opt):
    """100 k series x 12 blocks of 120 datapoints: every row equals the call on one concatenated stream per series
    (no annotations), sampled rows equal the oracle (with annotations: none in these sources)"""
    from m3_b200 import synth
    codec = codecs[int_opt]
    S, NB, PB = 100_000, 12, 120
    ts, vals, start = synth.gaussian_walk(S, NB * PB, "cuda", seed=31 + int(int_opt))
    whole = codec.encode(ts, vals, start)
    parts = [codec.encode(ts[:, b * PB:(b + 1) * PB].contiguous(), vals[:, b * PB:(b + 1) * PB].contiguous(),
                          ts[:, b * PB].contiguous()) for b in range(NB)]
    torch.cuda.synchronize()
    assert int((whole.status != 0).sum()) == 0 and all(int((p.status != 0).sum()) == 0 for p in parts)
    stride = parts[0].out.shape[1]
    blob = torch.cat([p.out.reshape(-1) for p in parts] + [torch.zeros(16, dtype=torch.uint8, device="cuda")])
    sidx = torch.arange(S, dtype=torch.int64, device="cuda")
    off = torch.stack([b * S * stride + sidx * stride for b in range(NB)], dim=1).reshape(-1)
    lengths = torch.stack([p.out_len for p in parts], dim=1).reshape(-1).to(torch.int64)
    blocks = torch.arange(S + 1, dtype=torch.int64, device="cuda") * NB
    wstride = whole.out.shape[1]
    w_off = sidx * wstride
    r0, step, W = int(start[0].item()), 300 * SEC, 288
    types, ops = [1, 2, 3], [ADD]
    ra, ta = codec.aggregate_tiles_types(blob, off, r0, step, W, types, lengths=lengths, transforms=ops, blocks=blocks)
    rb, tb = codec.aggregate_tiles_types(whole.out.reshape(-1), w_off, r0, step, W, types,
                                         lengths=whole.out_len.to(torch.int64), transforms=ops)
    torch.cuda.synchronize()
    assert int((ra.status != 0).sum()) == 0
    assert torch.equal(ra.out_len, rb.out_len) and torch.equal(ta, tb) and torch.equal(ra.status, rb.status)
    # every row's bytes: gather both packed buffers row by row in the same order
    def gathered(r):
        ln, of = r.out_len.reshape(-1), r.offsets.reshape(-1)
        idx = torch.repeat_interleave(of, ln) + (torch.arange(int(ln.sum().item()), device="cuda") -
                                                  torch.repeat_interleave(torch.cumsum(ln, 0) - ln, ln))
        return r.packed[idx]
    assert torch.equal(gathered(ra), gathered(rb))
    rc, tc = codec.aggregate_tiles_types(blob, off, r0, step, W, types, lengths=lengths, transforms=ops,
                                         blocks=blocks, annotations=True)
    torch.cuda.synchronize()
    assert torch.equal(gathered(rc), gathered(ra)) and torch.equal(tc, ta)
    host_blob, host_off, host_len = blob.cpu().numpy(), off.cpu().numpy(), lengths.cpu().numpy()
    rng = np.random.default_rng(5)
    sample = sorted(set(rng.choice(S, size=24, replace=False).tolist()) | {0, 31, 32, S - 1})
    packed, of, ln = ra.packed.cpu().numpy(), ra.offsets.cpu().numpy(), ra.out_len.cpu().numpy()
    for s in sample:
        segs = [host_blob[host_off[q]: host_off[q] + host_len[q]].tobytes() for q in range(s * NB, (s + 1) * NB)]
        rows, counts, err = B.aggregate_tiles_blocks_series(segs, int_opt, r0, step, W, GAUGE, types, ops, True,
                                                            E.new_element_state(), False)
        assert err == 0
        for j in range(len(types)):
            assert packed[of[j, s]: of[j, s] + ln[j, s]].tobytes() == rows[j], (s, j)
    del ra, rb, rc, blob, whole, parts, ts, vals
    torch.cuda.empty_cache()
