"""Every decode kernel on malformed streams, and under every default time unit, against the oracle and the decoder's
own complete grammar.

The corpus is `test_device_malformed_on_host.corpus`: well-formed base streams, most at a steady cadence, each followed
by its damaged variants (flipped bits, overwritten bytes, truncations, markers and headers spliced in at a datapoint
boundary).  Lanes keep a base's variants together, so that a warp is on the hot path when the damage arrives, with
the clean base between them.  Expected values: the oracle in float mode, the complete grammar (`decode_dp_slow` run on
the host) in int mode, where the CPU test pins it against the oracle (identical, or a prefix with an error status).

Then the default time units 0-8 and the units 5-8 (minute .. year, the all-zero time scheme): decode and encode
against the oracle under `default_unit=u`, whatever it gives, M3TSZ_ERR_NO_TIME_SCHEME included."""
import functools

import numpy as np
import pytest

import agg_oracle_lib as A
import oracle_lib as O
from test_device_malformed_on_host import START, corpus, grammar, oracle_batch

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
capi = pytest.importorskip("m3_b200.capi")
SEC = 10 ** 9
WIN = 60 * SEC
N_WIN = 48  # the steady streams' 240 datapoints every 10 s fill 40 windows
UNIT_NS = [0, SEC, 10 ** 6, 10 ** 3, 1, 60 * SEC, 3600 * SEC, 86400 * SEC, 365 * 86400 * SEC]


@pytest.fixture(scope="module")
def codecs():
    from m3_b200.codec import BatchCodec
    return {True: BatchCodec(0, True), False: BatchCodec(0, False)}


class Expected:
    """per lane: datapoints (ts, value bits), n, status, and the grammar's units / annotation / events"""

    def __init__(self, streams, int_opt, default_unit=O.UNIT_S):
        self.g = [grammar(b, int_opt, default_unit) for b in streams]
        self.n = np.array([len(g.dps) for g in self.g], dtype=np.int64)
        self.status = np.array([g.status for g in self.g], dtype=np.int32)
        cap = int(self.n.max()) + 4
        self.ts = np.zeros((len(streams), cap), dtype=np.int64)
        self.vals = np.zeros((len(streams), cap), dtype=np.uint64)
        for s, g in enumerate(self.g):
            self.ts[s, : len(g.ts)] = g.ts
            self.vals[s, : len(g.vals)] = g.vals
        o_ts, o_v, o_n, o_st = oracle_batch(streams, int_opt, default_unit, cap=cap)
        o_v = o_v.view(np.uint64)
        for s in range(len(streams)):
            k = int(self.n[s])
            if not int_opt:  # float mode: the oracle itself, status included
                assert o_n[s] == k and o_st[s] == self.status[s], s
            else:  # int mode: the grammar; difference 1 is a prefix with an error status
                assert o_n[s] == k and o_st[s] == self.status[s] or (self.status[s] != 0 and o_n[s] > k), s
            assert (o_ts[s, :k] == self.ts[s, :k]).all() and (o_v[s, :k] == self.vals[s, :k]).all(), s

    def prefix(self, s):
        k = int(self.n[s])
        return self.ts[s, :k], self.vals[s, :k].view(np.float64)


def _lanes(int_opt):
    """The corpus as lanes: each variant, with the clean base of its group before every third variant, and one more
    clean lane if the count is a multiple of 32 (a ragged last warp).  Returns (streams, clean_of, healthy)."""
    cases = corpus(int_opt)
    base = {bi: b for bi, kind, b in cases if kind == "clean"}
    streams, clean_of, healthy = [], [], []
    for i, (bi, kind, b) in enumerate(cases):
        if kind != "clean" and i % 3 == 0:
            streams.append(base[bi])
            clean_of.append(base[bi])
            healthy.append(True)
        streams.append(b)
        clean_of.append(base[bi])
        healthy.append(kind == "clean")
    if len(streams) % 32 == 0:
        streams.append(base[0])
        clean_of.append(base[0])
        healthy.append(True)
    return streams, clean_of, np.array(healthy)


@functools.lru_cache(maxsize=None)
def _case(int_opt):
    streams, clean_of, healthy = _lanes(int_opt)
    return streams, clean_of, healthy, Expected(streams, int_opt)


def _csr(streams):
    """one contiguous buffer that ends at the last stream's last byte"""
    off = np.zeros(len(streams) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(b) for b in streams])
    blob = np.frombuffer(b"".join(streams), dtype=np.uint8).copy()
    return torch.from_numpy(blob).cuda(), torch.from_numpy(off).cuda(), None


def _scattered(streams, seed=3):
    """offsets + lengths: the i-th stream at byte (37 i + 5) mod 128 of its own stretch, random bytes between the
    streams, the buffer ending at the last stream's last byte"""
    rng = np.random.default_rng(seed)
    starts, pos = [], 0
    for i, b in enumerate(streams):
        pos += (37 * i + 5 - pos) % 128
        starts.append(pos)
        pos += len(b)
    buf = rng.integers(0, 256, size=pos, dtype=np.uint8)
    for st, b in zip(starts, streams):
        buf[st: st + len(b)] = np.frombuffer(b, dtype=np.uint8)
    t = lambda a: torch.tensor(a, dtype=torch.int64, device="cuda")
    return torch.from_numpy(buf).cuda(), t(starts), t([len(b) for b in streams])


SENT_TS, SENT_V = -0x5A5A5A5A5A5A5A5B, 0x7FF4DEADBEEF0001


def _decode(codec, inputs, cap, point_major, want_events=0):
    from m3_b200.codec import DecodeResult
    blob, off, lengths = inputs
    S = off.numel() - 1 if lengths is None else lengths.numel()
    shape = (cap, S) if point_major else (S, cap)
    out = DecodeResult(ts=torch.full(shape, SENT_TS, dtype=torch.int64, device="cuda"),
                       values=torch.full(shape, SENT_V, dtype=torch.int64, device="cuda").view(torch.float64),
                       n_points=torch.empty(S, dtype=torch.int32, device="cuda"),
                       status=torch.empty(S, dtype=torch.int32, device="cuda"),
                       unit=torch.empty(S, dtype=torch.uint8, device="cuda"),
                       annotations=torch.empty((S, 16), dtype=torch.uint8, device="cuda"))
    r = codec.decode(blob, off, cap, want_annotations=True, out=out, lengths=lengths, want_events=want_events,
                     point_major=point_major)
    torch.cuda.synchronize()
    return r


def _host(r, point_major):
    ts, v = r.ts.cpu().numpy(), r.values.cpu().numpy().view(np.uint64)
    return (ts.T, v.T) if point_major else (ts, v)


def _check_decode(r, e, point_major, idx=None):
    """n_points, status, datapoints, the rows after them (the sentinel), the unit, the first annotation"""
    idx = np.arange(len(e.g)) if idx is None else idx
    n, st = r.n_points.cpu().numpy(), r.status.cpu().numpy()
    assert (n[idx] == e.n[idx]).all(), np.nonzero(n[idx] != e.n[idx])[0][:10]
    assert (st[idx] == e.status[idx]).all(), np.nonzero(st[idx] != e.status[idx])[0][:10]
    ts, v = _host(r, point_major)
    unit = r.unit.cpu().numpy()
    ann = r.annotations.cpu().numpy().view(np.uint64).reshape(-1, 2)
    for s in idx:
        k, g = int(e.n[s]), e.g[s]
        assert (ts[s, :k] == e.ts[s, :k]).all() and (v[s, :k] == e.vals[s, :k]).all(), s
        assert (ts[s, k:] == SENT_TS).all() and (v[s, k:] == np.uint64(SENT_V)).all(), s
        assert unit[s] == (g.emit_unit if k else g.unit), s
        a_bit, a_len, a_count = g.ann
        assert int(ann[s, 0]) == a_bit and int(ann[s, 1]) == a_len | (a_count << 32), s


def _events(e, idx):
    rows = []
    for s in idx:
        ev = e.g[s].events.copy()
        ev[:, :8] = np.frombuffer(np.uint64(s).tobytes(), dtype=np.uint8)
        rows.append(ev)
    return np.concatenate(rows) if rows else np.zeros((0, 32), dtype=np.uint8)


def _sorted_rows(a):
    return a[np.lexsort(a.T[::-1])] if len(a) else a


@pytest.mark.parametrize("int_opt", [False, True])
@pytest.mark.parametrize("point_major", [False, True])
@pytest.mark.parametrize("addressing", ["csr", "scattered"])
def test_decode_on_malformed_streams(codecs, int_opt, point_major, addressing):
    streams, clean_of, healthy, e = _case(int_opt)
    S = len(streams)
    cap = e.ts.shape[1]
    place = _csr if addressing == "csr" else _scattered
    exp_ev = _events(e, range(S))
    r = _decode(codecs[int_opt], place(streams), cap, point_major, want_events=len(exp_ev) + 64)
    _check_decode(r, e, point_major)
    # the event table: the grammar's events, as a multiset; the unit at the first datapoint
    assert int(r.event_count.item()) == len(exp_ev)
    got_ev = r.events.cpu().numpy()[: len(exp_ev)]
    assert (_sorted_rows(got_ev) == _sorted_rows(exp_ev)).all()
    uf = r.unit_first.cpu().numpy()
    assert all(uf[s] == (e.g[s].first_unit if e.n[s] else e.g[s].unit) for s in range(S))
    # healthy lanes decode as in a batch where every damaged lane is its clean original
    r2 = _decode(codecs[int_opt], place(clean_of), cap, point_major)
    a, b = _host(r, point_major), _host(r2, point_major)
    assert (a[0][healthy] == b[0][healthy]).all() and (a[1][healthy] == b[1][healthy]).all()
    for x, y in ((r.n_points, r2.n_points), (r.status, r2.status), (r.unit, r2.unit), (r.annotations, r2.annotations)):
        assert torch.equal(x[torch.from_numpy(healthy).cuda()], y[torch.from_numpy(healthy).cuda()])
    n_bad = int((e.status != 0).sum())
    print("decode int_opt=%s point_major=%s %s: %d lanes, %d with an error status, %d events" %
          (int_opt, point_major, addressing, S, n_bad, len(exp_ev)))


@pytest.mark.parametrize("int_opt", [False, True])
def test_decode_bench_shape_with_damaged_lanes(codecs, int_opt):
    """the bench's workload (a Gaussian batch of 1440 points per series through (offset, size) into point-major
    outputs) on 131072 series, 300 of them replaced by damaged corpus streams"""
    from m3_b200 import synth
    codec = codecs[int_opt]
    S, P = 131072, 1440
    ts, vals, start = synth.gaussian_walk(S, P, "cuda", seed=11)
    enc = codec.encode(ts, vals, start, unit=1)
    stride = enc.out.shape[1]
    cases = [c[2] for c in corpus(int_opt) if c[1] != "clean"]
    rng = np.random.default_rng(5)
    lanes = np.sort(rng.choice(S, size=300, replace=False))
    streams = [cases[j][:stride] for j in rng.choice(len(cases), size=len(lanes), replace=False)]
    off = torch.arange(S, dtype=torch.int64, device="cuda") * stride
    # (the undamaged batch: an int-optimised Gaussian series may decode to other bits than its inputs, as the
    # reference's does, so the healthy lanes are compared with this decode)
    r0 = codec.decode(enc.out.view(-1), off, P, lengths=enc.out_len, point_major=True)
    for s, b in zip(lanes, streams):
        enc.out[s, : len(b)] = torch.from_numpy(np.frombuffer(b, dtype=np.uint8).copy()).cuda()
        enc.out_len[s] = len(b)
    e = Expected(streams, int_opt)
    assert int(e.n.max()) <= P
    r = codec.decode(enc.out.view(-1), off, P, lengths=enc.out_len, point_major=True)
    torch.cuda.synchronize()
    healthy = torch.ones(S, dtype=torch.bool, device="cuda")
    healthy[torch.from_numpy(lanes).cuda()] = False
    assert bool((r.status[healthy] == 0).all()) and bool((r.n_points[healthy] == P).all())
    assert torch.equal(r.ts.t()[healthy], r0.ts.t()[healthy])
    assert torch.equal(r.values.t()[healthy].view(torch.int64), r0.values.t()[healthy].view(torch.int64))
    assert torch.equal(r0.ts.t()[healthy], ts[healthy])
    n, st = r.n_points.cpu().numpy()[lanes], r.status.cpu().numpy()[lanes]
    assert (n == e.n).all() and (st == e.status).all()
    idx = torch.from_numpy(lanes).cuda()
    g_ts = r.ts[:, idx].t().cpu().numpy()
    g_v = r.values[:, idx].t().contiguous().view(torch.int64).cpu().numpy().view(np.uint64)
    for i in range(len(lanes)):
        k = int(e.n[i])
        assert (g_ts[i, :k] == e.ts[i, :k]).all() and (g_v[i, :k] == e.vals[i, :k]).all(), i
    assert int((st != 0).sum()) > 20


def _ds_expected(e, kind):
    """the oracle's windows over each lane's expected datapoints"""
    S = len(e.g)
    rows = []
    for s in range(S):
        ts, v = e.prefix(s)
        if kind in ("plain", "last"):
            rows.append(O.downsample_series(ts, v, START, WIN, N_WIN))
        elif kind == "sum_sq":
            rows.append(A.downsample_gauge_ex(ts, v, START, WIN, N_WIN))
        else:
            rows.append(A.downsample_counter(ts, v, START, WIN, N_WIN))
    return [np.stack([r[j] for r in rows], axis=1) for j in range(len(rows[0]))]


def _same_f64(got, exp):
    g, x = got.view(np.uint64), exp.view(np.uint64)
    return bool(((g == x) | (np.isnan(got) & np.isnan(exp))).all())


@pytest.mark.parametrize("int_opt", [False, True])
@pytest.mark.parametrize("kind", ["plain", "last", "sum_sq", "counter"])
def test_fused_downsample_on_malformed_streams(codecs, int_opt, kind):
    streams, _, _, e = _case(int_opt)
    codec = codecs[int_opt]
    inputs = [_csr(streams)] + ([_scattered(streams)] if kind in ("sum_sq", "counter") else [])
    exp = _ds_expected(e, kind)
    for blob, off, lengths in inputs:
        kw = dict(lengths=lengths)
        if kind == "last":
            kw["want_last"] = True
        elif kind == "sum_sq":
            kw["want_sum_sq"] = True
        elif kind == "counter":
            kw["metric"] = capi.METRIC_COUNTER
        r = codec.decode_downsample(blob, off, START, WIN, N_WIN, **kw)
        torch.cuda.synchronize()
        assert (r.n_points.cpu().numpy() == e.n).all() and (r.status.cpu().numpy() == e.status).all()
        h = lambda t: t.cpu().numpy()
        if kind == "counter":
            for g, x in zip((r.sum, r.count, r.min, r.max, r.sum_sq), exp):
                assert (h(g) == x).all()
            continue
        assert _same_f64(h(r.sum), exp[0])  # +Inf and -Inf in one window: any NaN
        assert (h(r.count) == exp[1]).all()
        for g, x in ((r.min, exp[2]), (r.max, exp[3])):
            assert (h(g).view(np.uint64) == x.view(np.uint64)).all()
        if kind == "last":
            assert (h(r.last).view(np.uint64) == exp[4].view(np.uint64)).all()
        if kind == "sum_sq":
            assert (h(r.last).view(np.uint64) == exp[4].view(np.uint64)).all() and (h(r.last_at) == exp[5]).all()
            assert (h(r.sum_sq).view(np.uint64) == exp[6].view(np.uint64)).all()


def _rows(r, nt):
    """every (type, series) row of a tile call: (status, n_tiles, bytes)"""
    packed = r.packed.cpu().numpy()
    off, ln, st, n = (x.cpu().numpy() for x in (r.offsets, r.out_len, r.status, nt))
    k, S = st.shape
    return [[(int(st[j, s]), int(n[j, s]), packed[off[j, s]: off[j, s] + ln[j, s]].tobytes() if st[j, s] == 0
              else int(ln[j, s])) for s in range(S)] for j in range(k)]


def _tile_streams(int_opt, n=2400):
    """the first 2400 lanes (a few dozen base groups, each with its variants) and their expected statuses"""
    streams, _, _, e = _case(int_opt)
    S = min(n, len(streams))
    return streams[:S], e.status[:S]


@pytest.mark.parametrize("int_opt", [False, True])
@pytest.mark.parametrize("call", ["types", "annotated", "blocks", "blocks_annotated"])
def test_tiles_on_malformed_sources(codecs, int_opt, call):
    codec = codecs[int_opt]
    streams, st = _tile_streams(int_opt)
    if call.startswith("blocks"):  # an empty segment is no datapoints and M3TSZ_OK (DESIGN.md §6, item 8)
        st = np.where([len(b) == 0 for b in streams], 0, st)
    bad = st != 0
    assert bad.sum() > 20
    types = [1, 2, 7]  # Last, Min, Sum

    def run(ids):
        srcs = [streams[i] for i in ids]
        ann = call.endswith("annotated")
        if call.startswith("blocks"):  # every odd series: its stream after a well-formed block
            segs, blocks = [], [0]
            for i, b in zip(ids, srcs):
                segs += [streams[0], b] if i % 2 else [b]
                blocks.append(len(segs))
            blob, off, lengths = _scattered(segs)
            blk = torch.tensor(blocks, dtype=torch.int64, device="cuda")
            r, nt = codec.aggregate_tiles_types(blob, off, START, WIN, N_WIN, types, lengths=lengths,
                                                annotations=ann, blocks=blk)
        else:
            blob, off, lengths = _scattered(srcs)
            r, nt = codec.aggregate_tiles_types(blob, off, START, WIN, N_WIN, types, lengths=lengths, annotations=ann)
        torch.cuda.synchronize()
        return _rows(r, nt)

    got = run(range(len(streams)))
    keep = np.nonzero(~bad)[0]
    ref = run(keep)
    for j in range(len(types)):
        for s in np.nonzero(bad)[0]:  # the decode status, no tiles, no bytes
            assert got[j][s] == (int(st[s]), 0, 0), (j, s)
        for i, s in enumerate(keep):
            assert got[j][s] == ref[j][i], (j, s)


@pytest.mark.parametrize("int_opt", [False, True])
@pytest.mark.parametrize("annotations", [False, True])
def test_rollup_on_malformed_sources(codecs, int_opt, annotations):
    codec = codecs[int_opt]
    streams, st = _tile_streams(int_opt)
    S = len(streams)
    # groups of three consecutive sources, odd groups listed backwards; a trailing group of one
    groups = [list(range(g, min(g + 3, S))) for g in range(0, S, 3)]
    groups = [m[::-1] if i % 2 else m for i, m in enumerate(groups)]

    def run(srcs, grp):
        blob, off, lengths = _scattered(srcs)
        go = np.zeros(len(grp) + 1, dtype=np.int64)
        go[1:] = np.cumsum([len(m) for m in grp])
        mem = np.array([x for m in grp for x in m], dtype=np.int32)
        r, nt, sst = codec.aggregate_tiles_rollup(blob, off, START, WIN, N_WIN, 1, torch.from_numpy(go).cuda(),
                                                  torch.from_numpy(mem).cuda(), [2, 3, 7], lengths=lengths,
                                                  annotations=annotations)
        torch.cuda.synchronize()
        return _rows(r, nt), sst.cpu().numpy()

    got, sst = run(streams, groups)
    assert (sst == st).all()
    clean = [g for g, m in enumerate(groups) if all(st[x] == 0 for x in m)]
    keep = sorted({x for g in clean for x in groups[g]})
    new = {x: i for i, x in enumerate(keep)}
    ref, _ = run([streams[x] for x in keep], [[new[x] for x in groups[g]] for g in clean])
    assert len(clean) < len(groups)
    for j in range(3):
        for g, m in enumerate(groups):
            first = next((int(st[x]) for x in m if st[x] != 0), 0)
            if first:
                assert got[j][g] == (first, 0, 0), (j, g)
        for i, g in enumerate(clean):
            assert got[j][g] == ref[j][i], (j, g)


# ---------------------------------------------------------------------------------------------------------------
# default time units 0-8, units 5-8
# ---------------------------------------------------------------------------------------------------------------
def _unit_streams(int_opt, du):
    """streams for default unit du: encoded under du (every unit 1-8, starts aligned and misaligned to it), written
    under seconds, and whose first datapoint changes the unit"""
    rng = np.random.default_rng(40 + du)
    out = []
    P = 64
    for u in range(1, 9):
        for misalign in (0, 7 * SEC + 3):
            start = START - START % UNIT_NS[u] + misalign
            steps = rng.integers(1, 4, size=P) * UNIT_NS[u]
            steps[rng.random(P) < 0.7] = UNIT_NS[u]
            ts = start + np.cumsum(steps).astype(np.int64)
            vals = np.round(100 + np.cumsum(rng.normal(size=P)), 2 if u % 2 else 9)
            o, ln, stat = O.encode_batch(ts[None], vals[None], start, u, int_opt, default_unit=du)
            if stat[0] == 0:
                out.append(o[0, : ln[0]].tobytes())
    cases = corpus(int_opt)
    out += [b for bi, kind, b in cases if kind == "clean"][:12]
    for u in range(1, 9):
        e = O.Encoder(START, int_opt, du)
        t = START
        for i in range(40):
            t += 10 * SEC
            assert e.encode(t, float(i % 7) * 1.5, u if i == 0 else (u if i < 20 else O.UNIT_S)) == 0
        out.append(e.stream())
    return out


@pytest.mark.parametrize("int_opt", [False, True])
@pytest.mark.parametrize("du", range(9))
def test_decode_under_default_unit(int_opt, du):
    from m3_b200.codec import BatchCodec
    codec = BatchCodec(0, int_opt, default_unit=du)
    streams = _unit_streams(int_opt, du)
    S = len(streams)
    e = Expected(streams, int_opt, du)
    cap = e.ts.shape[1]
    for place in (_csr, _scattered):
        for pm in (False, True):
            _check_decode(_decode(codec, place(streams), cap, pm), e, pm)
    blob, off, _ = _csr(streams)
    for kind, kw in (("plain", {}), ("last", {"want_last": True}), ("sum_sq", {"want_sum_sq": True}),
                     ("counter", {"metric": capi.METRIC_COUNTER})):
        r = codec.decode_downsample(blob, off, START, WIN, N_WIN, **kw)
        torch.cuda.synchronize()
        assert (r.n_points.cpu().numpy() == e.n).all() and (r.status.cpu().numpy() == e.status).all()
        exp = _ds_expected(e, kind)
        if kind == "counter":
            assert (r.sum.cpu().numpy() == exp[0]).all() and (r.count.cpu().numpy() == exp[1]).all()
        else:
            assert _same_f64(r.sum.cpu().numpy(), exp[0]) and (r.count.cpu().numpy() == exp[1]).all()
    print("default unit %d int_opt=%s: %d streams, statuses %s" % (du, int_opt, S, np.unique(e.status).tolist()))


def _unit_inputs(P=48, seed=0):
    """8 whole warps, warp w encoding under unit w + 1; timestamps on that unit's grid"""
    rng = np.random.default_rng(seed)
    S = 8 * 32 + 5
    unit_of = np.minimum(np.arange(S) // 32 + 1, 8)
    ts = np.zeros((S, P), dtype=np.int64)
    for s in range(S):
        u = UNIT_NS[unit_of[s]]
        ts[s] = START - START % u + np.cumsum(np.where(rng.random(P) < 0.8, 1, rng.integers(1, 5, size=P))) * u
    vals = np.where(rng.random((S, P)) < 0.5, np.round(rng.normal(size=(S, P)) * 100, 2),
                    100 + np.cumsum(rng.normal(size=(S, P)), axis=1))
    return ts, vals, unit_of


def _oracle_encode(ts, vals, units, int_opt, du):
    """(stream, status) per series through O.Encoder, a unit per datapoint"""
    out = []
    for s in range(ts.shape[0]):
        e = O.Encoder(START, int_opt, du)
        err = 0
        for i in range(ts.shape[1]):
            err = e.encode(int(ts[s, i]), float(vals[s, i]), int(units[s, i]))
            if err:
                break
        out.append((e.stream() or b"", err))
    return out


@pytest.mark.parametrize("int_opt", [False, True])
@pytest.mark.parametrize("du", range(9))
def test_encode_under_default_unit(int_opt, du):
    from m3_b200.codec import BatchCodec
    from m3_b200.encoding import Encoder
    codec = BatchCodec(0, int_opt, default_unit=du)
    ts, vals, unit_of = _unit_inputs(seed=du)
    S, P = ts.shape
    start = torch.full((S,), START, dtype=torch.int64, device="cuda")
    d_ts, d_v = torch.from_numpy(ts).cuda(), torch.from_numpy(vals).cuda()
    for u in range(1, 9):  # one unit per call; warp u - 1 has timestamps on its grid
        e_out, e_len, e_st = O.encode_batch(ts, vals, START, u, int_opt, default_unit=du, n_threads=8)
        enc = codec.encode(d_ts, d_v, start, unit=u)
        pm = codec.encode(d_ts.t().contiguous(), d_v.t().contiguous(), start, unit=u, point_major=True)
        pk = codec.encode_packed(d_ts, d_v, start, unit=u)
        torch.cuda.synchronize()
        for r in (enc, pm):
            g_len, g_st, g_out = r.out_len.cpu().numpy(), r.status.cpu().numpy(), r.out.cpu().numpy()
            assert (g_st == e_st).all() and (g_len[e_st == 0] == e_len[e_st == 0].astype(np.int64)).all(), u
            for s in np.nonzero(e_st == 0)[0]:
                assert g_out[s, : g_len[s]].tobytes() == e_out[s, : e_len[s]].tobytes(), (u, s)
        p_out, p_off, p_len, p_st = (x.cpu().numpy() for x in (pk.packed, pk.offsets, pk.out_len, pk.status))
        assert (p_st == e_st).all()
        for s in np.nonzero(e_st == 0)[0]:
            assert p_out[p_off[s]: p_off[s] + p_len[s]].tobytes() == e_out[s, : e_len[s]].tobytes(), (u, s)
        # what the device encoded decodes as the oracle decodes it
        ok = np.nonzero(e_st == 0)[0]
        streams = [e_out[s, : e_len[s]].tobytes() for s in ok]
        if streams:
            ex = Expected(streams, int_opt, du)
            _check_decode(_decode(codec, _csr(streams), ex.ts.shape[1], False), ex, False)
    # a unit per datapoint, mixing 1-8 (a change every few datapoints)
    rng = np.random.default_rng(60 + du)
    units = np.repeat(rng.integers(1, 9, size=(S, P // 4)), 4, axis=1).astype(np.uint8)
    units[:, 0] = unit_of
    exp = _oracle_encode(ts, vals, units, int_opt, du)
    enc = codec.encode(d_ts, d_v, start, units=torch.from_numpy(units).cuda())
    torch.cuda.synchronize()
    g_len, g_st, g_out = enc.out_len.cpu().numpy(), enc.status.cpu().numpy(), enc.out.cpu().numpy()
    for s, (b, err) in enumerate(exp):
        assert g_st[s] == err, s
        if not err:
            assert g_out[s, : g_len[s]].tobytes() == b, s
    # an encoder set: reset, then two appends
    es = codec.encoder_set(start, codec.encode_bound(P))
    es.reset(start)
    h = P // 2
    for a in (slice(0, h), slice(h, P)):
        es.append(d_ts[:, a].contiguous(), d_v[:, a].contiguous(), unit=5 + du % 4)
    res = es.stream()
    e_out, e_len, e_st = O.encode_batch(ts, vals, START, 5 + du % 4, int_opt, default_unit=du, n_threads=8)
    torch.cuda.synchronize()
    assert (e_st == 0).sum() > S // 2
    g_len, g_out = res.out_len.cpu().numpy(), res.out.cpu().numpy()
    for s in np.nonzero(e_st == 0)[0]:
        assert g_out[s, : g_len[s]].tobytes() == e_out[s, : e_len[s]].tobytes(), s
    # the Encoder facade, one series per unit
    for u in range(1, 9):
        s = (u - 1) * 32
        f = Encoder(START, int_opt, du)
        o = O.Encoder(START, int_opt, du)
        for i in range(P):
            err = o.encode(int(ts[s, i]), float(vals[s, i]), u)
            try:
                f.encode(int(ts[s, i]), float(vals[s, i]), u)
                got = 0
            except capi.M3tszError as x:
                got = x.status
            assert got == err, (u, i)
            if err:
                break
        assert (f.stream() or b"") == (o.stream() or b""), u
