"""The ENCODER's device functions, compiled for the host from the .cu source text and driven one series at a time
the way a lane of the kernel drives them: `EncLane`, `put32` / `put64`, the value classifier, `track_new_sig`,
`sig_mult_hdr`, `xor_code`, `encode_value<INT_OPT>`, `encode_time`, `tier2_candidate<INT_OPT>` /
`tier2_commit<INT_OPT>` are cut out of m3_b200/csrc/m3tsz_encode.cu (and the constants / unit helpers out of
m3tsz_common.cuh) at test time.  Only what is PTX is replaced by a plain C++ statement of the same contract: the
predicated-store merge `emit_code_p` (here: put32 + put64 of the same bits), `lz_tz` / `shl64_clamp`, the CUDA
intrinsics.  Two drivers -- every datapoint through the general path, and the second tier wherever
`tier2_candidate` says so (the kernel picks per warp vote, so any mix has to give the same bytes) -- must both
reproduce the ORACLE's bytes on the reference's families, unit changes, jittered timestamps, special values and
Gaussian walks, in both modes.  A CPU regression harness for the device source; nothing of it ships."""
import ctypes as C
import random

import numpy as np
import pytest

import oracle_lib as O
from host_build import build_dev_encoder

SEC = 10 ** 9


@pytest.fixture(scope="module")
def dev():
    return build_dev_encoder()


def _dev_encode(dev, ts, vals, start, unit, int_opt, use_tier2, units=None):
    ts = np.ascontiguousarray(ts, dtype=np.int64)
    vals = np.ascontiguousarray(vals, dtype=np.float64)
    un = None if units is None else np.ascontiguousarray(units, dtype=np.uint8)
    out = np.zeros(64 + 24 * len(ts), dtype=np.uint8)
    nt = C.c_int()
    n = dev.dev_encode_series(ts.ctypes.data, vals.ctypes.data, None if un is None else un.ctypes.data, len(ts),
                              int(start), int(unit), int(int_opt), 1, int(use_tier2), out.ctypes.data, len(out),
                              C.byref(nt), None)
    assert n >= 0, n
    return out[:n].tobytes(), nt.value


def _gen(r, num_dig, num_dec):
    dig = r.getrandbits(62) % 10 ** num_dig
    return float(dig) if num_dec == 0 else float("%d.%d" % (dig, r.getrandbits(62) % 10 ** num_dec))


def _series(int_opt):
    r = random.Random(71 + int(int_opt))
    rng = np.random.default_rng(73 + int(int_opt))
    start = 1599955200 * SEC
    fams = [(12, 0), (7, 6), (0, 1), (2, 16), (5, 3), (3, 0), (18, 0), (1, 2), (0, 6), (4, 4), (9, 2), (0, 0)]
    for num_dig, num_dec in fams:
        for rep in range(3):
            P = 250
            ts = start + np.cumsum(rng.choice([1, 10, 60, 60, 60, 300, 4000, 10 ** 6], size=P)).astype(np.int64) * SEC
            if rep == 0:
                ts = start + np.arange(1, P + 1, dtype=np.int64) * 60 * SEC
            vals = np.array([_gen(r, num_dig, num_dec) for _ in range(P)])
            if rep == 1:
                vals *= rng.choice([-1.0, 1.0], size=P)
            if rep == 2:
                idx = rng.integers(1, P, size=P // 4)
                vals[idx] = vals[idx - 1]
                oth = rng.integers(0, P, size=P // 8)
                vals[oth] = [_gen(r, *fams[r.randrange(len(fams))]) for _ in oth]
            yield ts, vals, start
    for k in range(12):
        P = 300
        ts = start + np.arange(1, P + 1, dtype=np.int64) * 60 * SEC
        if k % 3 == 0:
            vals = 100.0 + np.cumsum(rng.normal(size=P))
        elif k % 3 == 1:
            vals = np.round(np.cumsum(rng.normal(size=P) * 10.0 ** rng.integers(0, 12)))
        else:
            vals = np.round(rng.normal(size=P) * 5, int(rng.integers(0, 7)))
            sp = [np.nan, np.inf, -np.inf, -0.0, 2.0 ** 63, -2.0 ** 63, 1e300, -1e300, 5e-324, 0.0, 9.2e18, 1e13]
            vals[::23] = (sp * 2)[: len(vals[::23])]
        yield ts, vals, start


@pytest.mark.parametrize("int_opt", [True, False])
def test_device_encoder_functions_reproduce_oracle_bytes(dev, int_opt):
    n = n_t2 = n_dp = 0
    for ts, vals, start in _series(int_opt):
        exp = O.encode_series(ts, vals, start, O.UNIT_S, int_opt)
        general, zero = _dev_encode(dev, ts, vals, start, O.UNIT_S, int_opt, use_tier2=False)
        mixed, t2 = _dev_encode(dev, ts, vals, start, O.UNIT_S, int_opt, use_tier2=True)
        assert zero == 0
        assert general == exp, n
        assert mixed == exp, n
        n += 1
        n_t2 += t2
        n_dp += len(ts)
    assert n == 48 and n_t2 > 0.3 * n_dp  # the second tier really carried a large share of the datapoints


@pytest.mark.parametrize("int_opt", [True, False])
def test_device_encoder_time_units_and_unit_changes(dev, int_opt):
    """all four scheme units as the series' unit, and per-datapoint unit changes (marker + 64-bit delta-of-delta)"""
    rng = np.random.default_rng(91)
    start = 1599955200 * SEC
    for unit, step in ((O.UNIT_S, SEC), (O.UNIT_MS, 10 ** 6), (O.UNIT_US, 10 ** 3), (O.UNIT_NS, 1)):
        P = 200
        ts = start + np.cumsum(rng.integers(1, 5000, size=P)).astype(np.int64) * step
        vals = np.round(rng.normal(size=P) * 100, 2)
        e = O.Encoder(start, int_opt)
        for t, v in zip(ts.tolist(), vals.tolist()):
            assert e.encode(t, v, unit, b"") == 0
        for tier2 in (False, True):
            got, _ = _dev_encode(dev, ts, vals, start, unit, int_opt, tier2)
            assert got == e.stream(), (unit, tier2)
    P = 240
    ts = start + np.cumsum(rng.integers(1, 5000, size=P)).astype(np.int64) * 10 ** 6
    vals = np.round(rng.normal(size=P) * 100, 1)
    units = np.full(P, O.UNIT_S, dtype=np.uint8)
    units[40:80] = O.UNIT_MS
    units[80:120] = O.UNIT_US
    units[120:121] = O.UNIT_NS
    units[200:] = O.UNIT_MS
    e = O.Encoder(start, int_opt)
    for t, v, u in zip(ts.tolist(), vals.tolist(), units.tolist()):
        assert e.encode(t, v, u, b"") == 0
    for tier2 in (False, True):
        got, _ = _dev_encode(dev, ts, vals, start, O.UNIT_S, int_opt, tier2, units=units)
        assert got == e.stream(), tier2
