"""A deterministic corpus of malformed M3TSZ streams, and the decoder's complete grammar (`decode_dp_slow`, compiled for
the host by `host_build.build_dev_decoder`) against the oracle on every stream of it.

The corpus (`corpus(int_opt)`) starts from well-formed base streams, most of them 240 datapoints at a steady cadence
so that a warp of their variants is on the decoder's hot path when the damage arrives: the goldens and production
fixtures, the value families of the ring-fill tests (constants, full-width doubles, a walk, counters, decimals,
repeats), unit changes across s / ms / us / ns, annotations longer than the 256-byte ring, int / float switches,
+-2^63 (a 64-bit significand) and six-decimal values (multiplier 6).  Every base stream yields variants with one and
three flipped bits, four overwritten bytes, a truncation plus a flip, and bits spliced in at a datapoint boundary (the
grammar's bit position after each datapoint): a time-unit marker carrying 0, 5-9 or 255, marker value 3, annotation
markers with a zero or negative length, an overflowing 10-byte varint, a length past the end or a long in-bounds
payload, and int-mode headers with multiplier 7 or a 64-bit significand.  A few long streams add every
byte-truncation, cuts inside varints and annotation payloads included.

The CPU test pins the grammar against the oracle over the whole corpus: identical in float mode (datapoints, value
bits and status); in int mode identical or a prefix with an error status, the documented difference 1 (DESIGN.md §6).
The GPU tests (tests/test_gpu_malformed_streams.py) then compare every decode kernel with that grammar."""
import base64
import functools
import json
import os

import numpy as np
import pytest

import oracle_lib as O
from host_build import DevDecode, build_dev_decoder

G = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "m3tsz_goldens.json")))
SEC = 10 ** 9
START = 1599955200 * SEC
STEP = 10 * SEC  # the steady cadence of most base streams
P = 240
CAP = 4096  # more datapoints than any corpus stream holds

MARKER = 0x100  # 9-bit marker opcode, then a 2-bit marker value
M_ANN, M_UNIT = 1, 2


def _bits(b):
    return np.unpackbits(np.frombuffer(bytes(b), dtype=np.uint8))


def _pack(bits):
    return np.packbits(np.concatenate([bits, np.zeros((-len(bits)) % 8, dtype=np.uint8)])).tobytes()


def _field(v, n):
    return np.array([(int(v) >> (n - 1 - i)) & 1 for i in range(n)], dtype=np.uint8)


def _bytes_bits(bs):
    return _bits(bytes(bs)) if bs else np.zeros(0, dtype=np.uint8)


def _marker(value):
    return np.concatenate([_field(MARKER, 9), _field(value, 2)])


def _uvarint(x):
    out = bytearray()
    while x >= 0x80:
        out.append((x & 0x7F) | 0x80)
        x >>= 7
    out.append(x)
    return bytes(out)


def _ann_len_varint(alen):
    """binary.PutVarint(alen - 1), as the encoder writes an annotation's length"""
    v = alen - 1
    return _uvarint((v << 1) if v >= 0 else ((~v << 1) | 1))


def _splices(rng):
    """(name, bits) inserted at a datapoint boundary"""
    out = [("unit%d" % u, np.concatenate([_marker(M_UNIT), _field(u, 8)])) for u in (0, 5, 6, 7, 8, 9, 255)]
    out.append(("marker3", _marker(3)))
    out.append(("ann_len0", np.concatenate([_marker(M_ANN), _bytes_bits(_ann_len_varint(0))])))
    out.append(("ann_len_neg", np.concatenate([_marker(M_ANN), _bytes_bits(_ann_len_varint(-5))])))
    out.append(("ann_varint_overflow", np.concatenate([_marker(M_ANN), _bytes_bits(b"\xff" * 9 + b"\x02")])))
    out.append(("ann_past_end", np.concatenate([_marker(M_ANN), _bytes_bits(_ann_len_varint(1 << 20))])))
    payload = bytes(rng.integers(0, 256, size=700, dtype=np.uint8))
    out.append(("ann_long", np.concatenate([_marker(M_ANN), _bytes_bits(_ann_len_varint(700) + payload)])))
    # a datapoint with a zero delta-of-delta and an int-mode header update: '0' dod, '0' update, '0' no repeat,
    # '0' int mode, then readIntSigMult
    head = _field(0, 4)
    out.append(("int_mult7", np.concatenate([head, _field(1, 1), _field(1, 1), _field(9, 6), _field(1, 1),
                                             _field(7, 3), _field(0x2A5, 11)])))
    out.append(("int_sig64", np.concatenate([head, _field(1, 1), _field(1, 1), _field(63, 6), _field(0, 1),
                                             _field(1, 1), _field(0x0123456789ABCDEF, 64)])))
    return out


def _enc(ts, vals, int_opt, units=None, anns=None):
    e = O.Encoder(START, int_opt)
    for i in range(len(ts)):
        u = O.UNIT_S if units is None else int(units[i])
        a = b"" if anns is None else anns.get(i, b"")
        assert e.encode(int(ts[i]), float(vals[i]), u, a) == 0
    return e.stream()


def _base_streams(int_opt):
    """[(name, stream)]: goldens / fixtures first, then generated families (two seeds each)."""
    out = []
    if not int_opt:
        out += [("golden%d" % i, bytes.fromhex(s["bytes"])) for i, s in enumerate(G["streams"])]
    else:
        out += [("fixture%d" % i, base64.b64decode(b)) for i, b in enumerate(G["fixtures_b64"]["streams"])]
        out.append(("regression", base64.b64decode(G["regression_b64"]["stream"])))
    steady = START + np.arange(1, P + 1, dtype=np.int64) * STEP
    for seed in range(2):
        rng = np.random.default_rng(100 * seed + 7 + int(int_opt))
        walk = np.cumsum(rng.normal(size=P))
        irregular = START + np.cumsum(rng.integers(1, 5000, size=P)).astype(np.int64) * SEC
        fam = [
            ("constants", steady, np.full(P, 42.0)),
            ("doubles", steady, np.ldexp(rng.random(P) - 0.5, rng.integers(-900, 900, size=P))),
            ("doubles_irregular", irregular, np.ldexp(rng.random(P) - 0.5, rng.integers(-900, 900, size=P))),
            ("walk", steady, 100 + walk),
            ("counters", steady, np.cumsum(rng.integers(0, 50, size=P)).astype(np.float64)),
            ("decimals", steady, np.round(walk, 2)),
            ("repeats", steady, rng.integers(0, 3, size=P) * 0.5),
            ("switches", steady, np.where((np.arange(P) // 20) % 2 == 0, np.round(walk * 10), 100 + walk)),
            ("pm2_63", steady, np.where(np.arange(P) % 2 == 0, 9.2e18, -2.0 ** 63)),
            ("six_decimals", steady, np.round(walk, 6)),
        ]
        for name, ts, vals in fam:
            out.append(("%s%d" % (name, seed), O.encode_series(ts, vals, START, O.UNIT_S, int_opt)))
        units = np.full(P, O.UNIT_S)
        for i0, u in ((0, O.UNIT_MS), (40, O.UNIT_US), (90, O.UNIT_NS), (150, O.UNIT_S), (200, O.UNIT_MS)):
            units[i0:] = u
        out.append(("units%d" % seed, _enc(steady, 100 + walk, int_opt, units=units)))
        anns = {i: bytes(rng.integers(0, 256, size=300 + 300 * (j % 3), dtype=np.uint8))
                for j, i in enumerate((2, 60, 61, 130))}
        anns.update({i: b"ab%d" % i for i in (5, 100, 101, 180)})
        out.append(("annotations%d" % seed, _enc(steady, 100 + walk, int_opt, anns=anns)))
    return out


def grammar(stream, int_opt, default_unit=O.UNIT_S):
    """the complete grammar's decode of one stream (a DevDecode)"""
    return DevDecode(build_dev_decoder(), stream, int_opt, cap=CAP, default_unit=default_unit, ev_cap=1024)


@functools.lru_cache(maxsize=None)
def corpus(int_opt):
    """[(base index, kind, stream)]: every base stream's variants follow it, the clean base first (kind 'clean');
    the base list is `_base_streams(int_opt)`.  Deterministic."""
    bases = _base_streams(int_opt)
    rng = np.random.default_rng(31 + int(int_opt))
    splices = _splices(rng)
    out = []
    for bi, (name, b) in enumerate(bases):
        out.append((bi, "clean", b))
        nbits = 8 * len(b)
        for k in range(6):
            a = _bits(b).copy()
            a[int(rng.integers(0, nbits))] ^= 1
            out.append((bi, "flip1", _pack(a)))
        for k in range(4):
            a = _bits(b).copy()
            a[rng.choice(nbits, size=3, replace=False)] ^= 1
            out.append((bi, "flip3", _pack(a)))
        for k in range(4):
            a = bytearray(b)
            at = int(rng.integers(0, max(1, len(b) - 4)))
            a[at: at + 4] = bytes(rng.integers(0, 256, size=4, dtype=np.uint8))[: len(a) - at]
            out.append((bi, "bytes4", bytes(a)))
        for k in range(4):
            cut = int(rng.integers(1, len(b)))
            a = _bits(b[:cut]).copy()
            a[int(rng.integers(0, 8 * cut))] ^= 1
            out.append((bi, "cut_flip", _pack(a)))
        g = grammar(b, int_opt)
        assert g.status == 0
        if len(g.bitpos) >= 16:
            for sname, sb in splices:
                i = int(rng.integers(len(g.bitpos) // 4, len(g.bitpos) - 4))
                a = _bits(b)
                at = int(g.bitpos[i])
                out.append((bi, "splice_" + sname, _pack(np.concatenate([a[:at], sb, a[at:]]))))
    for name in ("annotations0", "units1", "walk0"):
        bi = [n for n, _ in bases].index(name)
        b = bases[bi][1]
        out += [(bi, "cut", b[:cut]) for cut in range(len(b))]
    return out


def oracle_batch(streams, int_opt, default_unit=O.UNIT_S, cap=CAP):
    """O.decode_batch over a list of streams: (ts, vals, n, status)"""
    off = np.zeros(len(streams) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(b) for b in streams])
    blob = np.frombuffer(b"".join(streams) + b"\0", dtype=np.uint8)
    return O.decode_batch(blob, off, cap, int_opt, default_unit, n_threads=8)


@pytest.mark.parametrize("int_opt", [False, True])
def test_grammar_matches_the_oracle_on_malformed_streams(int_opt):
    cases = corpus(int_opt)
    streams = [c[2] for c in cases]
    e_ts, e_v, e_n, e_st = oracle_batch(streams, int_opt)
    same = prefix = 0
    kinds = {}
    for i, b in enumerate(streams):
        g = grammar(b, int_opt)
        k = int(e_n[i])
        exp = list(zip(e_ts[i, :k].tolist(), e_v[i, :k].view(np.uint64).tolist()))
        if (g.dps, g.status) == (exp, int(e_st[i])):
            same += 1
        else:
            # int mode only: the kernel stops at the first failed read, the reference may overwrite that error
            assert int_opt, (i, cases[i][:2], len(g.dps), k, g.status, int(e_st[i]))
            assert g.status != 0 and len(g.dps) < k and g.dps == exp[: len(g.dps)], (i, cases[i][:2])
            prefix += 1
        kinds[cases[i][1]] = kinds.get(cases[i][1], 0) + (int(e_st[i]) != 0)
    print("malformed corpus int_opt=%s: %d streams, %d identical to the oracle (status included), %d a prefix with an "
          "error status; failing streams per kind: %s" % (int_opt, len(cases), same, prefix, kinds))
    assert len(cases) > 3000
    assert same + prefix == len(cases)
    # the damage reaches the error paths (an invalid unit marker, or a long in-bounds annotation, may leave a
    # well-formed stream)
    assert all(kinds[k] > 0 for k in ("flip1", "flip3", "bytes4", "cut_flip", "cut", "splice_unit5", "splice_unit8",
                                      "splice_marker3", "splice_ann_len0", "splice_ann_len_neg",
                                      "splice_ann_varint_overflow", "splice_ann_past_end", "splice_int_mult7",
                                      "splice_int_sig64")), kinds
