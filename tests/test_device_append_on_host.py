"""The encoder sets' APPEND path, compiled for the host from the .cu source text and driven one open encoder at a
time the way a lane of the append kernel drives it: the encoder functions of test_device_encoder_on_host plus
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
import os
import random
import re
import subprocess
import tempfile

import numpy as np
import pytest

import oracle_lib as O
from test_device_encoder_on_host import CSRC, EMIT, ROOT, SEC, SHIM, _cut, _fn, _series

ERRS = "enum { M3TSZ_ERR_CAPACITY = 100, M3TSZ_ERR_INVALID_ARG = 101 };\n"

DRIVER = r"""
// one append call on one encoder: what a lane of encode_kernel<., false, ., true> does with its series
template <bool INT_OPT>
static long long append_call(m3tsz_encoder_state *st, uint8_t *slot, const int64_t *ts, const double *vals,
                             const uint8_t *units, int unit, size_t n, const uint32_t *ann_off,
                             const uint32_t *ann_len, const uint8_t *ann_bytes, int use_tier2, int *err) {
  std::vector<uint32_t> tile((n * 40 + 64) * ENC_STRIDE, 0u);
  EncLane s;
  memset(&s, 0, sizeof(s));
  uint64_t ann_cs = 0;
  *err = enc_state_load<INT_OPT>(*st, s, tile.data(), 0, ann_cs);
  if (*err) return 0;
  const uint32_t n0 = s.n_enc;
  if (n && s.n_enc == 0) put64(s, tile.data(), 0, (uint64_t)s.prev_time, 64);
  for (size_t i = 0; i < n; i++) {
    const int64_t t = ts[i];
    const double v = vals[i];
    const int u = units ? (int)units[i] : unit;
    *err = enc_check_time(s, t, u);
    if (*err) break;
    if (ann_len[i]) {  // timestamp_encoder.go:166-195 with the checksum carried in the state
      const uint64_t h = xxh64(ann_bytes + ann_off[i], ann_len[i]);
      if (h != ann_cs) {
        put32(s, tile.data(), 0, (kMarkerOpcode << 2) | (uint32_t)kMarkerAnnotation, kMarkerBits);
        uint64_t ux = ((uint64_t)(ann_len[i] - 1)) << 1;
        while (ux >= 0x80) {
          put32(s, tile.data(), 0, (uint32_t)(ux & 0x7f) | 0x80u, 8);
          ux >>= 7;
        }
        put32(s, tile.data(), 0, (uint32_t)ux, 8);
        for (uint32_t b = 0; b < ann_len[i]; b++) put32(s, tile.data(), 0, ann_bytes[ann_off[i] + b], 8);
      }
      ann_cs = h;
    }
    const bool steady = (u == s.unit) && (s.unit >= 1 && s.unit <= 4) && s.n_enc > 0;
    uint64_t fb;
    memcpy(&fb, &v, 8);
    const int64_t delta = (int64_t)((uint64_t)t - (uint64_t)s.prev_time);
    Tier2 c2;
    if (use_tier2 && tier2_candidate<INT_OPT>(s, steady, delta, fb, v, c2)) {
      s.prev_time = t;
      s.prev_delta = delta;
      tier2_commit<INT_OPT>(s, tile.data(), 0, fb, c2);
    } else {
      uint32_t hdr;
      int hb;
      encode_time(s, tile.data(), 0, t, u, hdr, hb);
      if (s.err) {  // enc_check_time let through a datapoint encode_time refuses
        *err = -1;
        return -1;
      }
      uint64_t payload;
      int plen;
      encode_value<INT_OPT>(s, v, hdr, hb, payload, plen);
      emit_code(s, tile.data(), 0, hdr, hb, payload, plen);
    }
    s.n_enc++;
  }
  // the epilogue's flush: whole sectors to the slot, <= 7 words stay
  const uint32_t done = s.k & ~7u;
  for (uint32_t w = 0; w < done; w++)
    for (int b = 0; b < 4; b++) slot[(s.words_out + w) * 4ull + b] = (uint8_t)(tile[w * ENC_STRIDE] >> (24 - 8 * b));
  for (uint32_t w = done; w < s.k; w++) tile[(w - done) * ENC_STRIDE] = tile[w * ENC_STRIDE];
  s.words_out += done;
  s.k -= done;
  if (s.n_enc != n0) enc_state_save<INT_OPT>(*st, s, tile.data(), 0, ann_cs);
  return (long long)(s.n_enc - n0);
}
extern "C" long long dev_append(m3tsz_encoder_state *st, uint8_t *slot, const int64_t *ts, const double *vals,
                                const uint8_t *units, int unit, size_t n, const uint32_t *ann_off,
                                const uint32_t *ann_len, const uint8_t *ann_bytes, int int_opt, int use_tier2,
                                int *err) {
  return int_opt ? append_call<true>(st, slot, ts, vals, units, unit, n, ann_off, ann_len, ann_bytes, use_tier2, err)
                 : append_call<false>(st, slot, ts, vals, units, unit, n, ann_off, ann_len, ann_bytes, use_tier2, err);
}
extern "C" void dev_reset(m3tsz_encoder_state *st, int64_t start, int default_unit, int int_opt) {
  enc_state_reset(*st, start, default_unit, int_opt != 0);
}
// the snapshot kernel's work for one encoder; returns Len()
extern "C" uint64_t dev_snapshot(const m3tsz_encoder_state *st, uint8_t *slot) {
  uint32_t w[12];
  uint64_t at = 0;
  const uint32_t n = enc_snapshot_words(*st, w, at);
  for (uint32_t i = 0; i < n; i++)
    for (int b = 0; b < 4; b++) slot[(at + i) * 4 + b] = (uint8_t)(w[i] >> (24 - 8 * b));
  return st->num_encoded ? (st->bits + kMarkerBits + 7) / 8 : 0;
}
"""


@pytest.fixture(scope="module")
def dev():
    enc = open(os.path.join(CSRC, "m3tsz_encode.cu")).read()
    com = open(os.path.join(CSRC, "m3tsz_common.cuh")).read()
    hdr = open(os.path.join(ROOT, "include", "m3tsz_b200.h")).read()
    state = re.search(r"typedef struct m3tsz_encoder_state \{.*?\} m3tsz_encoder_state;", hdr, flags=re.S).group(0)
    consts = "\n".join(re.findall(r"^constexpr [^\n]*\bk(?:Marker|MaxMult)[^\n]*$", com, flags=re.M))
    parts = [ERRS, state, consts, _cut(com, r"enum SchemeKind"),
             _cut(com, r"__host__ __device__[^\n{;]*\bunit_is_valid\s*\("),
             _cut(com, r"__host__ __device__[^\n{;]*\bunit_nanos\s*\("),
             _cut(com, r"__host__ __device__[^\n{;]*\bscheme_kind_for_unit\s*\("),
             _cut(com, r"__host__ __device__[^\n{;]*\binitial_time_unit\s*\("),
             _cut(com, r"__host__ __device__[^\n{;]*\bxxh64\s*\("),
             _cut(com, _fn("num_sig")), _cut(com, _fn("mult_pow10")),
             _cut(enc, r"struct EncLane"), _cut(enc, _fn("put32")), _cut(enc, _fn("put64")), EMIT,
             _cut(enc, _fn("emit_code"))]
    for name in ("maybe_int", "go_f64_to_u64_via_i64", "convert_to_int_float", "track_new_sig", "sig_mult_hdr",
                 "xor_code", "encode_value", "encode_time"):
        parts.append(_cut(enc, _fn(name)))
    parts += [_cut(enc, r"struct Tier2"), _cut(enc, _fn("div_unit")), _cut(enc, _fn("tier2_candidate")),
              _cut(enc, _fn("tier2_commit")), _cut(enc, r"struct EncStateInternal")]
    for name in ("enc_state_tag", "enc_state_reset", "enc_state_load", "enc_state_save", "enc_check_time",
                 "enc_snapshot_words"):
        parts.append(_cut(enc, _fn(name)))
    body = "\n".join(parts)
    assert "asm" not in body, "a PTX block slipped into the host build"
    d = tempfile.mkdtemp(prefix="m3dev_append_host_")
    path = os.path.join(d, "dev_append_host.cpp")
    open(path, "w").write(SHIM + body + DRIVER)
    so = os.path.join(d, "dev_append_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-w", path, "-o", so])
    lib = C.CDLL(so)
    vp = C.c_void_p
    lib.dev_append.restype = C.c_longlong
    lib.dev_append.argtypes = [vp, vp, vp, vp, vp, C.c_int, C.c_size_t, vp, vp, vp, C.c_int, C.c_int,
                               C.POINTER(C.c_int)]
    lib.dev_reset.restype = None
    lib.dev_reset.argtypes = [vp, C.c_int64, C.c_int, C.c_int]
    lib.dev_snapshot.restype = C.c_uint64
    lib.dev_snapshot.argtypes = [vp, vp]
    return lib


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
