"""The M3TSZ grammar at its edges, on the CPU: the corpus of tests/grammar_edges.py through the oracle, the
independent Python encoder and decoder, and the encoder's and decoder's device code compiled for the host.

- Coverage: every cell of the corpus' table occurs where the corpus says, as a tracing reader sees the oracle's
  bytes, on every row of a 4-row input tile.
- The independent encoder and decoder equal the oracle on the whole corpus (bytes, datapoints, status).
- The device encoder's functions equal the oracle through both host drivers (the general path only, and the second
  tier wherever `tier2_candidate` accepts), and the second tier takes the in-bucket delta-of-delta edges and never
  one past +-2047.
- The decoder's complete grammar equals the oracle."""
import ctypes as C
import struct
from collections import defaultdict

import numpy as np
import pytest

import grammar_edges as G
import indep_m3tsz as I
import oracle_lib as O
from host_build import DevDecode, build_dev_decoder, build_dev_encoder

LANES = (0, 1)  # lane 1 negates the int series


def oracle_encode(s):
    """(the oracle's Stream() of the datapoints before the first failing one, status, datapoints encoded)"""
    e = O.Encoder(int(s.start), s.int_opt, s.unit)
    for i in range(len(s.ts)):
        err = e.encode(int(s.ts[i]), float(s.vals[i]), s.unit)
        if err:
            return e.stream() or b"", err, i
    return e.stream() or b"", 0, len(s.ts)


@pytest.fixture(scope="module")
def cases():
    out = []
    for lane in LANES:
        for s in G.corpus(lane):
            out.append((s,) + oracle_encode(s))
    return out


def _bits(v):
    return struct.unpack("<Q", struct.pack("<d", v))[0]


def test_every_cell_occurs_on_every_row(cases):
    rows = defaultdict(set)
    n_ovf = 0
    for s, stream, status, n_ok in cases:
        tr = []
        I.decode(stream, s.int_opt, s.unit, trace=tr)
        assert len(tr) == n_ok, s.name
        n_ovf += status != 0
        for key, i in s.cells:
            assert G.check_cell(key, s, tr, i, status), (s.name, key, i, tr[i] if i < len(tr) else None)
            rows[key].add(i % G.ROWS)
    table = G.cell_table()
    assert set(rows) == table, (sorted(table - set(rows), key=str)[:20], sorted(set(rows) - table, key=str)[:20])
    first_only = {"dod1", "overflow1", "start", "int_first_sig"}
    for key, r in rows.items():
        if key[0] not in first_only:
            assert r == {0, 1, 2, 3}, (key, r)
    # s / ms, both modes, each overflow edge on the first datapoint and on every row of a tile later
    assert n_ovf == len(LANES) * 2 * 2 * len(G.OVERFLOW_DODS) * (G.ROWS + 1)
    print("grammar edges: %d cells, %d series (%d lanes), %d ending in a delta-of-delta overflow" %
          (len(table), len(cases), len(LANES), n_ovf))


def test_independent_encoder_and_decoder_equal_the_oracle(cases):
    for s, stream, status, n_ok in cases:
        dps = [(int(t), float(v), s.unit, b"") for t, v in zip(s.ts[:n_ok], s.vals[:n_ok])]
        # (a first datapoint that fails leaves the oracle's stream holding the start time alone)
        assert I.encode(int(s.start), dps, s.int_opt, s.unit) == (stream if n_ok else b""), s.name
        if status:  # the model asserts where the oracle returns the overflow
            with pytest.raises(AssertionError, match="overflows"):
                I.encode(int(s.start), dps + [(int(s.ts[n_ok]), float(s.vals[n_ok]), s.unit, b"")], s.int_opt, s.unit)
        got = I.decode(stream, s.int_opt, s.unit)
        exp, err = O.decode_all(stream, s.int_opt, s.unit)
        assert err == 0 and len(exp) == n_ok, s.name
        assert [(t, b) for t, b, _, _ in got] == [(d[0], _bits(d[1])) for d in exp], s.name


@pytest.fixture(scope="module")
def dev_enc():
    return build_dev_encoder()


def _dev_encode(lib, s, n, use_tier2):
    ts = np.ascontiguousarray(s.ts[:n], dtype=np.int64)
    vals = np.ascontiguousarray(s.vals[:n], dtype=np.float64)
    out = np.zeros(64 + 24 * max(n, 1), dtype=np.uint8)
    tiers = np.zeros(max(n, 1), dtype=np.uint8)
    nt = C.c_int()
    r = lib.dev_encode_series(ts.ctypes.data, vals.ctypes.data, None, n, int(s.start), s.unit, int(s.int_opt), s.unit,
                              int(use_tier2), out.ctypes.data, len(out), C.byref(nt), tiers.ctypes.data)
    return (out[:r].tobytes() if r >= 0 else int(-r)), tiers[:n]


def test_device_encoder_equals_the_oracle_through_both_drivers(cases, dev_enc):
    n_t2 = n_edges = n_e13 = 0
    for s, stream, status, n_ok in cases:
        general, _ = _dev_encode(dev_enc, s, len(s.ts), False)
        mixed, tiers = _dev_encode(dev_enc, s, len(s.ts), True)
        if status:  # the same status, and the prefix before the failing datapoint gives the oracle's bytes
            assert general == status and mixed == status, s.name
            exp = stream if n_ok else b""
            assert _dev_encode(dev_enc, s, n_ok, False)[0] == exp and _dev_encode(dev_enc, s, n_ok, True)[0] == exp
            continue
        assert general == stream, s.name
        assert mixed == stream, s.name
        n_t2 += int((tiers == 2).sum())
        for key, i in s.cells:
            if key[0] == "dod":  # an edge after the first datapoint: the second tier exactly inside +-2047
                n_edges += 1
                assert tiers[i] == (2 if -2048 <= key[3] <= 2047 else 1), (s.name, key, tiers)
            if key[0] in ("mult", "mult7", "int_diff_overflow", "float_changed", "int_newsig0"):
                assert tiers[i] == 1, (s.name, key)  # a multiplier or mode change: the general path
            if key[0] == "e13":  # 10^13 at the multiplier in force: a switch to float mode (general path), or not
                to_float = I.convert_to_int_float(abs(float(s.vals[i])), key[1])[2]
                assert tiers[i] == (1 if to_float else 2), (s.name, key)
                n_e13 += to_float
    assert n_edges > 1000 and n_t2 > 10000 and n_e13 >= 6 * 4 * len(LANES)


@pytest.fixture(scope="module")
def dev_dec():
    return build_dev_decoder()


def test_complete_grammar_decodes_like_the_oracle(cases, dev_dec):
    for s, stream, status, n_ok in cases:
        exp, err = O.decode_all(stream, s.int_opt, s.unit)
        r = DevDecode(dev_dec, stream, s.int_opt, lead=len(s.name) % 7, default_unit=s.unit)
        assert r.status == err == 0, s.name
        assert r.dps == [(d[0], _bits(d[1])) for d in exp], s.name
