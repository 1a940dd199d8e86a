"""The decoder's complete-grammar path -- `decode_dp_slow<INT_OPT>` with `DecState`, `SlowSrc`, `EventSink`,
`push_event`, `gpeek64`, the `M3_RD` read macro (m3_b200/csrc/m3tsz_decode.cu) and `load_be32` / `sign_extend`
(m3tsz_common.cuh) -- cut out of the CUDA sources at test time, compiled for the host and driven like one lane that
never leaves the slow path (global-memory source, `ring_safe = 0`).  Only the CUDA intrinsics and the three PTX
helpers of the common header are restated in C++.

Checks against the oracle: every stream family decodes to the same (timestamp, value bits) in both modes from any
byte offset of a packed buffer; the event table carries every unit change and annotation; and on EVERY
byte-truncation the device code's sticky status is compared with the reference semantics the oracle implements --
identical in float mode (datapoints and error), and in int mode never more datapoints than the reference, every
difference being the documented one (DESIGN.md §6, difference 1: the reference's `readBits` may overwrite an earlier
error and carry on; the kernel stops at the first failed read)."""
import base64
import json
import os
import random
import struct

import numpy as np
import pytest

import oracle_lib as O
from host_build import DevDecode, build_dev_decoder

G = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "m3tsz_goldens.json")))
SEC = 10 ** 9


@pytest.fixture(scope="module")
def dev():
    return build_dev_decoder()


def _dev_decode(dev, stream, int_opt, lead=0, cap=4096, want_events=False):
    """the stream placed `lead` bytes into a zero-padded buffer (any byte offset, like a packed data file)"""
    r = DevDecode(dev, stream, int_opt, lead=lead, cap=cap)
    if want_events:
        return r.dps, r.status, r.events, r.emit_unit, r.first_unit
    return r.dps, r.status


def _oracle(stream, int_opt):
    dps, err = O.decode_all(stream, int_opt)
    return [(d[0], struct.unpack("<Q", struct.pack("<d", d[1]))[0]) for d in dps], err, dps


def _streams(int_opt):
    out = []
    if not int_opt:
        out += [bytes.fromhex(s["bytes"]) for s in G["streams"]]
    else:
        out += [base64.b64decode(b) for b in G["fixtures_b64"]["streams"]]
        out.append(base64.b64decode(G["regression_b64"]["stream"]))
    r = random.Random(5 + int(int_opt))
    rng = np.random.default_rng(6 + int(int_opt))
    start = 1599955200 * SEC
    for k in range(12):
        P = 60
        ts = start + np.cumsum(rng.choice([1, 10, 60, 300, 4000, 10 ** 6], size=P)).astype(np.int64) * SEC
        if k % 3 == 0:
            vals = 100.0 + np.cumsum(rng.normal(size=P))
        elif k % 3 == 1:
            vals = np.round(rng.normal(size=P) * 10.0 ** r.randrange(0, 8), r.randrange(0, 5))
        else:
            vals = np.round(rng.normal(size=P) * 5, 2)
            vals[::7] = [np.nan, 2.0 ** 63, -2.0 ** 63, 1e300, 0.5, 12.0, -0.0, np.inf, 5e-324][: len(vals[::7])]
        out.append(O.encode_series(ts, vals, start, O.UNIT_S, int_opt))
    e = O.Encoder(1427162400 * SEC, int_opt)
    t = 1427162462 * SEC
    for i in range(40):
        unit = O.UNIT_MS if i == 0 else (O.UNIT_US if i == 10 else (O.UNIT_NS if i == 25 else O.UNIT_S))
        ann = b"foo" if i < 5 else (b"bar" if i < 7 else (b"x" * 300 if i == 10 else b""))
        assert e.encode(t, float(r.randrange(1000)) / 4, unit, ann) == 0
        t += SEC * r.randrange(1, 500)
    out.append(e.stream())
    return out


@pytest.mark.parametrize("int_opt", [False, True])
def test_device_slow_path_decodes_like_the_oracle(dev, int_opt):
    n = 0
    for stream in _streams(int_opt):
        exp, err, dps = _oracle(stream, int_opt)
        assert err == 0
        for lead in (0, 1, 2, 3, 7, 61, 64):
            got, derr = _dev_decode(dev, stream, int_opt, lead=lead)
            assert derr == 0 and got == exp, (n, lead)
        got, derr, events, last_unit, first_unit = _dev_decode(dev, stream, int_opt, want_events=True)
        # event table: every annotation, and every unit change after the first datapoint
        ev = events.view(np.uint8).reshape(-1, 32)
        kinds = ev[:, 12:14].copy().view(np.uint16).ravel()
        n_ann = sum(1 for d in dps if len(d) > 3 and d[3])
        n_unit = sum(1 for i in range(1, len(dps)) if len(dps[i]) > 2 and dps[i][2] != dps[i - 1][2])
        assert int((kinds == 2).sum()) == n_ann and int((kinds == 1).sum()) == n_unit, n
        if dps and len(dps[0]) > 2:
            assert first_unit == dps[0][2] and last_unit == dps[-1][2]
        n += 1
    assert n >= 17


@pytest.mark.parametrize("int_opt", [False, True])
def test_device_slow_path_on_every_truncation(dev, int_opt):
    cases = same = fewer = 0
    for stream in _streams(int_opt)[:14]:
        for cut in range(len(stream)):
            got, derr = _dev_decode(dev, stream[:cut], int_opt)
            exp, err, _ = _oracle(stream[:cut], int_opt)
            cases += 1
            if not int_opt:
                assert (got, derr != 0) == (exp, err != 0), (cut, len(stream), derr, err)
                if derr in (1, 12) and err in (1, 12):
                    pass  # io.EOF / io.ErrUnexpectedEOF both mean "ran out of bytes"
                else:
                    assert derr == err, (cut, derr, err)
                same += 1
                continue
            # int mode: sticky status -- a prefix of what the reference returns, never more
            assert got == exp[: len(got)], (cut, len(stream))
            if (got, derr != 0) == (exp, err != 0):
                same += 1
            else:
                fewer += 1
                assert derr != 0, (cut, len(stream))  # the kernel stopped at a failed read the reference overwrote
    print("truncations int_opt=%s: %d cases, %d identical to the reference semantics, %d where the device code "
          "stops at an earlier failed read" % (int_opt, cases, same, fewer))
    assert cases > 3000
    if int_opt:
        assert same > 0.9 * cases  # the documented difference is the rare case
    else:
        assert same == cases
