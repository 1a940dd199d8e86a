"""The encoder sets' APPEND path, compiled for the host from the .cu source text and driven one open encoder at a
time the way a lane of the append kernel drives it: the encoder functions of the encoder harness plus
`EncStateInternal`, `enc_state_reset`, `enc_state_load<INT_OPT>` / `enc_state_save<INT_OPT>`, `enc_check_time`,
`enc_snapshot_words` (m3tsz_encode.cu) and `xxh64` (m3tsz_common.cuh) are cut out of the source at test time.
Between two calls only the 128-byte state and the slot's whole sectors survive, as on the device.

Every series is appended in several schedules (one call, one datapoint per call, random chunks with empty ones)
and snapshotted at every call boundary: each snapshot must equal the ORACLE encoder's Stream() of the prefix, the
state's public prefix its NumEncoded / LastEncoded / LastAnnotationChecksum / Len, in both modes, over the
reference's value families, Gaussian walks, special values, unit changes at call boundaries, annotations
repeated across a boundary (not rewritten) and long annotations (XXH64's 32-byte path).  A CPU regression
harness for the device source; nothing of it ships."""
import ctypes as C
import random

import numpy as np
import pytest

import oracle_lib as O
from host_build import build_dev_append
from test_device_encoder_on_host import SEC, _series


@pytest.fixture(scope="module")
def dev():
    return build_dev_append()


class HostEncoder:
    """One open encoder: a 128-byte state and a slot, nothing else kept between calls."""

    def __init__(self, dev, start, int_opt, n_max, ann_bytes=0):
        self.dev, self.int_opt = dev, int_opt
        self.state = np.zeros(16, dtype=np.uint64)
        self.slot = np.zeros(64 + 40 * n_max + 2 * ann_bytes, dtype=np.uint8)
        dev.dev_reset(self.state.ctypes.data, int(start), O.UNIT_S, int(int_opt))

    def append(self, ts, vals, units=None, unit=O.UNIT_S, anns=None, tier2=True):
        n = len(ts)
        ts = np.ascontiguousarray(ts, dtype=np.int64)
        vals = np.ascontiguousarray(vals, dtype=np.float64)
        un = None if units is None else np.ascontiguousarray(units, dtype=np.uint8)
        anns = anns or [b""] * n
        off = np.zeros(max(1, n), dtype=np.uint32)
        ln = np.zeros(max(1, n), dtype=np.uint32)
        blob = b""
        for i, a in enumerate(anns):
            off[i], ln[i] = len(blob), len(a)
            blob += a
        ab = np.frombuffer(blob + b"\0", dtype=np.uint8).copy()
        err = C.c_int()
        got = self.dev.dev_append(self.state.ctypes.data, self.slot.ctypes.data, ts.ctypes.data, vals.ctypes.data,
                                  None if un is None else un.ctypes.data, int(unit), n, off.ctypes.data,
                                  ln.ctypes.data, ab.ctypes.data, int(self.int_opt), int(tier2), C.byref(err))
        return got, err.value

    def snapshot(self):
        slot = self.slot.copy()  # a snapshot writes past the committed bytes; the next append overwrites them
        n = self.dev.dev_snapshot(self.state.ctypes.data, slot.ctypes.data)
        return slot[:n].tobytes()

    def public(self):
        st = self.state
        return (int(st[1]), int(st[2].view(np.int64)), float(st[3:4].view(np.float64)[0]), int(st[4]), int(st[5]))


def _schedules(n, seed):
    r = random.Random(seed)
    chunks = []
    left = n
    while left > 0:
        c = r.choice([0, 0, 1, 2, 3, 7, 8, 9, 31, 33, 64])
        c = min(c, left)
        chunks.append(c)
        left -= c
    return {"one_call": [n], "per_point": [1] * n, "random": chunks}


def _check_prefix(enc, oracle, int_opt, what):
    exp = oracle.stream() or b""
    assert enc.snapshot() == exp, what
    num, last_ts, last_val, ann_cs, bits = enc.public()
    assert num == oracle.num_encoded(), what
    exp_len = oracle.len()
    assert (((bits + 11 + 7) // 8) if num else 0) == exp_len, what
    if num:
        t, v, err = oracle.last_encoded()
        assert err == 0 and t == last_ts, what
        assert np.float64(v).view(np.uint64) == np.float64(last_val).view(np.uint64), what
        cs, err = oracle.last_annotation_checksum()
        assert cs == ann_cs, what


def _run(dev, ts, vals, start, int_opt, sched, units=None, anns=None, tier2=True, what=""):
    n = len(ts)
    enc = HostEncoder(dev, start, int_opt, n, sum(len(a) for a in anns) if anns else 0)
    oracle = O.Encoder(start, int_opt)
    i = 0
    for k, c in enumerate(sched):
        got, err = enc.append(ts[i: i + c], vals[i: i + c], None if units is None else units[i: i + c],
                              anns=None if anns is None else anns[i: i + c], tier2=tier2)
        assert (got, err) == (c, 0), (what, k, got, err)
        for j in range(i, i + c):
            u = O.UNIT_S if units is None else int(units[j])
            assert oracle.encode(int(ts[j]), float(vals[j]), u, anns[j] if anns else b"") == 0
        i += c
        _check_prefix(enc, oracle, int_opt, (what, k))
    return enc.snapshot()


@pytest.mark.parametrize("int_opt", [True, False])
def test_append_any_split_gives_the_oracle_stream(dev, int_opt):
    n = 0
    for idx, (ts, vals, start) in enumerate(_series(int_opt)):
        exp = O.encode_series(ts, vals, start, O.UNIT_S, int_opt)
        for name, sched in _schedules(len(ts), 1000 * idx + int_opt).items():
            if name == "per_point" and idx % 4:  # the slowest schedule on a quarter of the series
                continue
            assert _run(dev, ts, vals, start, int_opt, sched, tier2=bool(idx % 2), what=(idx, name)) == exp
            n += 1
    assert n >= 48 * 2


@pytest.mark.parametrize("int_opt", [True, False])
def test_append_unit_changes_at_call_boundaries(dev, int_opt):
    rng = np.random.default_rng(5)
    start = 1599955200 * SEC
    P = 240
    ts = start + np.cumsum(rng.integers(1, 5000, size=P)).astype(np.int64) * 10 ** 6
    vals = np.round(rng.normal(size=P) * 100, 1)
    units = np.full(P, O.UNIT_S, dtype=np.uint8)
    units[40:80] = O.UNIT_MS
    units[80:120] = O.UNIT_US
    units[120:121] = O.UNIT_NS
    units[200:] = O.UNIT_MS
    bounds = [0, 40, 80, 120, 121, 200, P]
    at_changes = [b - a for a, b in zip(bounds, bounds[1:])]
    straddling = [30, 20, 45, 30, 1, 84, 30]
    for sched in (at_changes, straddling, [1] * P):
        assert sum(sched) == P
        _run(dev, ts, vals, start, int_opt, sched, units=units, what=sched[:3])


@pytest.mark.parametrize("int_opt", [True, False])
def test_append_annotations_across_calls(dev, int_opt):
    """an annotation repeated in the next call is not rewritten (its checksum is in the state); a changed one is;
    short and long (>= 32 bytes: XXH64's four-lane path) annotations"""
    rng = np.random.default_rng(11)
    start = 1599955200 * SEC
    P = 120
    ts = start + np.arange(1, P + 1, dtype=np.int64) * 10 * SEC
    vals = 100.0 + np.cumsum(rng.normal(size=P))
    long_a = bytes(range(40))
    longer = bytes(rng.integers(0, 256, size=200).tolist())
    anns = [b""] * P
    for i in range(0, 30):
        anns[i] = b"proto-v1"  # the same annotation on every datapoint of several calls
    for i in range(30, 60, 3):
        anns[i] = long_a
    anns[61] = longer
    anns[62] = longer
    anns[90] = b"x"
    anns[91] = b"proto-v1"
    for sched in ([P], [10] * 12, [1] * P, [7, 0, 23, 1, 30, 29, 30]):
        _run(dev, ts, vals, start, int_opt, sched, anns=anns, what=sched[:3])
    # an annotation written in one call and repeated as the first datapoint of the next is not written again
    enc = HostEncoder(dev, start, int_opt, P, 64)
    enc.append(ts[:1], vals[:1], anns=[b"abc"])
    enc.append(ts[1:2], vals[1:2], anns=[b"abc"])
    o = O.Encoder(start, int_opt)
    o.encode(int(ts[0]), float(vals[0]), O.UNIT_S, b"abc")
    o.encode(int(ts[1]), float(vals[1]), O.UNIT_S, b"abc")
    assert enc.snapshot() == o.stream()


@pytest.mark.parametrize("int_opt", [True, False])
def test_append_failing_datapoint_is_dropped_whole(dev, int_opt):
    """a second-unit delta-of-delta overflow stops the call at that datapoint: state and stream stay as after the
    last datapoint taken, annotation included; dropping it and appending the rest gives the oracle's stream of the
    sequence without it"""
    start = 1599955200 * SEC
    P = 50
    ts = start + np.arange(1, P + 1, dtype=np.int64) * 10 * SEC
    ts[20:] += (1 << 33) * SEC  # datapoint 20: delta-of-delta 2^33 s
    vals = np.arange(P, dtype=np.float64) * 1.5
    anns = [b""] * P
    anns[20] = b"dropped-with-its-datapoint"
    enc = HostEncoder(dev, start, int_opt, P, 64)
    got, err = enc.append(ts[:30], vals[:30], anns=anns[:30])
    assert (got, err) == (20, O.ERR_DOD_OVERFLOW)
    assert enc.snapshot() == O.encode_series(ts[:20], vals[:20], start, O.UNIT_S, int_opt)
    got, err = enc.append(ts[21:], vals[21:])  # datapoint 21 follows datapoint 19: an overflow again
    assert (got, err) == (0, O.ERR_DOD_OVERFLOW)
    keep = np.r_[0:20, 21:P]
    ts2 = ts.copy()
    ts2[20:] -= (1 << 33) * SEC
    enc2 = HostEncoder(dev, start, int_opt, P, 64)
    assert enc2.append(ts2[:20], vals[:20]) == (20, 0)
    assert enc2.append(ts2[21:], vals[21:]) == (P - 21, 0)
    assert enc2.snapshot() == O.encode_series(ts2[keep], vals[keep], start, O.UNIT_S, int_opt)
    # an unrecognised unit is refused the same way
    enc3 = HostEncoder(dev, start, int_opt, P)
    units = np.full(10, O.UNIT_S, dtype=np.uint8)
    units[4] = 0
    assert enc3.append(ts2[:10], vals[:10], units=units) == (4, 6)
    assert enc3.snapshot() == O.encode_series(ts2[:4], vals[:4], start, O.UNIT_S, int_opt)


def test_append_refuses_a_state_of_the_other_mode(dev):
    start = 1599955200 * SEC
    enc = HostEncoder(dev, start, True, 8)
    before = enc.state.copy()
    enc.int_opt = False
    ts = start + np.arange(1, 5, dtype=np.int64) * SEC
    assert enc.append(ts, np.ones(4)) == (0, 101)
    assert (enc.state == before).all()
