"""The host-buffer entry points (m3tsz_*_batch_host) over batches large enough for several
pipeline chunks, compared exactly with the device entry points on the same inputs (those are
checked against the oracle elsewhere), and their error exits taken with the copies of earlier
chunks still in flight: each must return its status and leave the codec usable."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

SEC = 1_000_000_000
S, P = 6500, 1440  # 4 chunks of 2048 series in the encode and decode pipelines
SF = 3500          # fetch series at RF = 3: 4 chunks of 1024 series


@pytest.fixture(scope="module")
def batch():
    from m3_b200 import capi, synth
    from m3_b200.codec import BatchCodec
    codec = BatchCodec(0, True)
    ts, vals, start = synth.gaussian_walk(S, P, "cuda", seed=11)
    enc = codec.encode(ts, vals, start, unit=capi.UNIT_S)
    packed, off = codec.compact(enc, align=1)
    torch.cuda.synchronize()
    assert int((enc.status != 0).sum()) == 0
    return {"codec": codec, "ts": ts, "vals": vals, "start": start, "enc": enc,
            "streams": packed[: int(off[-1])], "off": off}


def first_n_equal(a, b, n):
    """Rows of a and b agree bit for bit on their first n[s] entries (nothing writes the rest)."""
    mask = torch.arange(a.shape[1]).unsqueeze(0) < n.long().unsqueeze(1)
    return torch.equal(a.view(torch.int64)[mask], b.view(torch.int64)[mask])


def status_of(call):
    from m3_b200 import capi
    with pytest.raises(capi.M3tszError) as e:
        call()
    return e.value.status


# ------------------------------------------------------------------ encode_host
def encode_host(b, capacity=None, align=1):
    from m3_b200 import capi
    out = {"packed": torch.empty(capacity, dtype=torch.uint8).pin_memory(),
           "off": torch.empty(S + 1, dtype=torch.int64).pin_memory(),
           "len": torch.empty(S, dtype=torch.int64).pin_memory(),
           "st": torch.empty(S, dtype=torch.int32).pin_memory()}
    b["codec"].encode_host(b["h_ts"], b["h_vals"], b["h_start"], capi.UNIT_S, out["packed"], out["off"],
                           out["len"], out["st"], align=align)
    return out


def check_encode_host(out, enc, packed, off):
    """h_out_len / h_status / h_offsets equal the device encode + compact, and so does every stream's
    bytes (the alignment padding between streams is not written, so it is not compared)."""
    assert torch.equal(out["len"], enc.out_len.cpu()) and torch.equal(out["st"], enc.status.cpu())
    h_off = off.cpu()
    assert torch.equal(out["off"], h_off)
    o, n = h_off[:-1].numpy(), enc.out_len.cpu().numpy()
    total = int(h_off[-1])
    edge = np.zeros(total + 1, dtype=np.int8)
    np.add.at(edge, o, 1)
    np.add.at(edge, o + n, -1)
    covered = np.cumsum(edge[:total]) > 0
    assert (out["packed"][:total].numpy()[covered] == packed[:total].cpu().numpy()[covered]).all()


@pytest.fixture(scope="module")
def host_inputs(batch):
    batch["h_ts"] = batch["ts"].cpu().pin_memory()
    batch["h_vals"] = batch["vals"].cpu().pin_memory()
    batch["h_start"] = batch["start"].cpu()
    return batch


@pytest.mark.parametrize("align", [1, 64])
def test_encode_host_matches_device(host_inputs, align):
    b = host_inputs
    packed, off = b["codec"].compact(b["enc"], align=align)
    torch.cuda.synchronize()
    out = encode_host(b, capacity=int(off[-1]), align=align)
    check_encode_host(out, b["enc"], packed, off)


def test_encode_host_capacity_in_later_chunk(host_inputs):
    from m3_b200 import capi
    b = host_inputs
    off = b["off"].cpu()
    # the first two chunks (4 096 series) fit, the third does not
    assert status_of(lambda: encode_host(b, capacity=int(off[5000]))) == capi.ERR_CAPACITY
    out = encode_host(b, capacity=int(off[-1]))
    check_encode_host(out, b["enc"], b["streams"], b["off"])


# ------------------------------------------------------------------ decode_host / decode_downsample_host
def decode_host(b, h_off):
    out = {"ts": torch.empty((S, P), dtype=torch.int64).pin_memory(),
           "vals": torch.empty((S, P), dtype=torch.float64).pin_memory(),
           "n": torch.empty(S, dtype=torch.int32).pin_memory(),
           "st": torch.empty(S, dtype=torch.int32).pin_memory()}
    b["codec"].decode_host(b["h_streams"], h_off, P, out["ts"], out["vals"], out["n"], out["st"])
    return out


def check_decode_host(b, out):
    dec = b["codec"].decode(b["streams"], b["off"], P)
    torch.cuda.synchronize()
    n = dec.n_points.cpu()
    assert torch.equal(out["n"], n) and torch.equal(out["st"], dec.status.cpu())
    assert first_n_equal(out["ts"], dec.ts.cpu(), n) and first_n_equal(out["vals"], dec.values.cpu(), n)


@pytest.fixture(scope="module")
def host_streams(batch):
    batch["h_streams"] = batch["streams"].cpu().pin_memory()
    batch["h_off"] = batch["off"].cpu().pin_memory()
    return batch


def test_decode_host_matches_device(host_streams):
    check_decode_host(host_streams, decode_host(host_streams, host_streams["h_off"]))


def test_decode_host_bad_last_offset(host_streams):
    from m3_b200 import capi
    b = host_streams
    bad = b["h_off"].clone()
    bad[-1] = b["h_streams"].numel() + 1  # only the last chunk reads it
    assert status_of(lambda: decode_host(b, bad)) == capi.ERR_INVALID_ARG
    check_decode_host(b, decode_host(b, b["h_off"]))


def test_decode_downsample_host_matches_device(host_streams):
    b = host_streams
    t0, step, W = int(b["start"][0]), 300 * SEC, 288
    outs = [torch.empty((W, S), dtype=dt).pin_memory()
            for dt in (torch.float64, torch.int64, torch.float64, torch.float64)]
    h_n = torch.empty(S, dtype=torch.int32).pin_memory()
    h_st = torch.empty(S, dtype=torch.int32).pin_memory()
    b["codec"].decode_downsample_host(b["h_streams"], b["h_off"], t0, step, W, *outs, h_n, h_st)
    ds = b["codec"].decode_downsample(b["streams"], b["off"], t0, step, W)
    torch.cuda.synchronize()
    assert torch.equal(h_n, ds.n_points.cpu()) and torch.equal(h_st, ds.status.cpu())
    for h, d in zip(outs, (ds.sum, ds.count, ds.min, ds.max)):
        assert torch.equal(h.view(torch.int64), d.cpu().view(torch.int64))


# ------------------------------------------------------------------ fetch_host
@pytest.fixture(scope="module")
def replicas(host_streams):
    """SF series x 3 replicas; replica r of series s is stream (s + r) % S of the batch, so the
    replicas share timestamps and disagree on values (the merge strategy matters)."""
    b = host_streams
    off = b["off"].cpu().numpy()
    blob = b["h_streams"].numpy()
    src = (np.arange(SF)[:, None] + np.arange(3)[None, :]).reshape(-1) % S
    ln = off[src + 1] - off[src]
    seq_off = np.zeros(3 * SF + 1, dtype=np.int64)
    seq_off[1:] = np.cumsum(ln)
    h_streams = torch.zeros(int(seq_off[-1]), dtype=torch.uint8).pin_memory()
    hs = h_streams.numpy()
    for q, s in enumerate(src):
        hs[seq_off[q]: seq_off[q + 1]] = blob[off[s]: off[s + 1]]
    ar = torch.arange(3 * SF + 1, dtype=torch.int64)
    return {"codec": b["codec"], "start": int(b["start"][0]), "h_streams": h_streams,
            "h_off": torch.from_numpy(seq_off).pin_memory(), "slice": ar, "rep": ar.clone(),
            "ser": torch.arange(0, 3 * SF + 1, 3, dtype=torch.int64)}


def fetch_host(f, h_off, **kw):
    out = {"ts": torch.empty((SF, P), dtype=torch.int64).pin_memory(),
           "vals": torch.empty((SF, P), dtype=torch.float64).pin_memory(),
           "n": torch.empty(SF, dtype=torch.int32).pin_memory(),
           "st": torch.empty(SF, dtype=torch.int32).pin_memory()}
    f["codec"].fetch_host(f["h_streams"], h_off, f["slice"], f["rep"], f["ser"], P, P, out["ts"], out["vals"],
                          out["n"], out["st"], **kw)
    return out


def check_fetch_host(f, out, start_ns=0, end_ns=0, strategy=0):
    codec = f["codec"]
    dec = codec.decode(f["h_streams"].cuda(), f["h_off"].cuda(), P)
    ts, vals, n, st = codec.merge_series(dec.ts, dec.values, dec.n_points, dec.status, f["slice"].cuda(),
                                         f["rep"].cuda(), f["ser"].cuda(), P, start_ns, end_ns, strategy)
    torch.cuda.synchronize()
    n = n.cpu()
    assert torch.equal(out["n"], n) and torch.equal(out["st"], st.cpu())
    assert first_n_equal(out["ts"], ts.cpu(), n) and first_n_equal(out["vals"], vals.cpu(), n)


@pytest.mark.parametrize("filtered", [False, True])
def test_fetch_host_matches_device(replicas, filtered):
    f = replicas
    kw = {}
    if filtered:  # a range filter and the highest-value strategy
        kw = {"start_ns": f["start"] + 100 * 60 * SEC, "end_ns": f["start"] + 1000 * 60 * SEC, "strategy": 1}
    out = fetch_host(f, f["h_off"], **kw)
    if filtered:
        assert bool((out["n"] == 900).all())
    check_fetch_host(f, out, **kw)


def test_fetch_host_bad_last_offset(replicas):
    from m3_b200 import capi
    f = replicas
    bad = f["h_off"].clone()
    bad[-1] = f["h_streams"].numel() + 1  # only the last chunk reads it
    assert status_of(lambda: fetch_host(f, bad)) == capi.ERR_INVALID_ARG
    check_fetch_host(f, fetch_host(f, f["h_off"]))
