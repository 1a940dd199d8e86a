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
import ctypes as C
import json
import os
import random
import re
import struct
import subprocess
import tempfile

import numpy as np
import pytest

import oracle_lib as O
from test_device_encoder_on_host import _cut, _fn

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
CSRC = os.path.join(ROOT, "m3_b200", "csrc")
G = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "m3tsz_goldens.json")))
SEC = 10 ** 9

SHIM = r"""
#include <cmath>
#include <cstdint>
#include <cstring>
#include "%s"
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
static inline double __dsub_rn(double a, double b) { return a - b; }
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline double __ddiv_rn(double a, double b) { return a / b; }
static inline double __ull2double_rn(unsigned long long a) { return (double)a; }
static inline long long __double_as_longlong(double a) { long long r; memcpy(&r, &a, 8); return r; }
static inline uint32_t __ldg(const uint32_t *p) { return *p; }
static inline uint32_t __byte_perm(uint32_t v, uint32_t, uint32_t sel) {  // only the byte swap is used
  if (sel != 0x0123) __builtin_trap();
  return __builtin_bswap32(v);
}
// funnel shift left by (sh & 31): the high word of (hi:lo) << sh  (PTX shf.l.wrap)
static inline uint32_t __funnelshift_l(uint32_t lo, uint32_t hi, uint32_t sh) {
  sh &= 31;
  return sh ? ((hi << sh) | (lo >> (32 - sh))) : hi;
}
static inline unsigned long long atomicAdd(unsigned long long *p, unsigned long long v) {
  const unsigned long long o = *p;
  *p += v;
  return o;
}
constexpr int DEC_QUADS = 16;
// ---- PTX helpers of m3tsz_common.cuh restated ----
static inline uint64_t shl64(uint64_t x, int n) { return n >= 64 ? 0ull : x << n; }
static inline void lz_tz(uint64_t v, int &lz, int &tz) {
  if (!v) { lz = 64; tz = 0; return; }
  lz = __builtin_clzll(v);
  tz = __builtin_ctzll(v);
}
"""

DRIVER = r"""
template <bool INT_OPT>
static int drive(const uint8_t *buf, uint64_t nbytes, uint64_t o0, uint64_t o1, int default_unit, int64_t *ts,
                 uint64_t *vals, uint32_t *bitpos, uint32_t cap, uint32_t *n_out, m3tsz_dp_event *events,
                 uint64_t ev_cap, unsigned long long *ev_count, int *units, uint32_t *ann) {
  DecState s;
  memset(&s, 0, sizeof(s));
  s.scheme = kSchemeNone;
  // the kernel's addressing: base = the stream's first word rounded down to a 16-word boundary
  const uint64_t w = o0 >> 2;
  s.wbase = w & ~(uint64_t)15;
  s.pos = (uint32_t)(w - s.wbase) * 32u + (uint32_t)(o0 & 3) * 8u;
  s.end = s.pos + (uint32_t)(o1 - o0) * 8u;
  const uint32_t pos0 = s.pos;
  SlowSrc src;
  src.base = buf;
  src.nbytes = nbytes;
  src.ring_lane = nullptr;
  src.ring_safe = 0;
  EventSink ev;
  ev.events = events;
  ev.capacity = ev_cap;
  ev.count = ev_count;
  ev.series = 0;
  ev.pos0 = pos0;
  while (!s.done && s.err == 0 && s.n < cap) {
    int64_t t = 0;
    uint64_t v = 0;
    if (decode_dp_slow<INT_OPT>(s, src, default_unit, t, v, &ev)) {
      ts[s.n] = t;
      vals[s.n] = v;
      bitpos[s.n] = s.pos - pos0;  // the stream bit after the datapoint
      s.n++;
    }
  }
  *n_out = s.n;
  units[0] = s.emit_unit;  // unit at the last datapoint produced
  units[1] = s.first_unit;  // ... at the first
  units[2] = s.unit;        // unit in force when the decode stopped
  // the first annotation, as the kernel's m3tsz_annotation_ref holds it
  ann[0] = s.ann_count ? s.ann_bit - pos0 : 0u;
  ann[1] = s.ann_len;
  ann[2] = s.ann_count;
  return s.err;
}
extern "C" int dev_decode(const uint8_t *buf, uint64_t nbytes, uint64_t o0, uint64_t o1, int int_opt, int default_unit,
                          int64_t *ts, uint64_t *vals, uint32_t *bitpos, uint32_t cap, uint32_t *n_out,
                          m3tsz_dp_event *events, uint64_t ev_cap, unsigned long long *ev_count, int *units,
                          uint32_t *ann) {
  return int_opt ? drive<true>(buf, nbytes, o0, o1, default_unit, ts, vals, bitpos, cap, n_out, events, ev_cap,
                               ev_count, units, ann)
                 : drive<false>(buf, nbytes, o0, o1, default_unit, ts, vals, bitpos, cap, n_out, events, ev_cap,
                                ev_count, units, ann);
}
"""


def build_dev_decoder():
    """Compiles the decoder's complete grammar for the host (g++ only) and returns the loaded library."""
    dec = open(os.path.join(CSRC, "m3tsz_decode.cu")).read()
    com = open(os.path.join(CSRC, "m3tsz_common.cuh")).read()
    consts = "\n".join(re.findall(r"^constexpr [^\n]*\bk(?:Marker|MaxMult)[^\n]*$", com, flags=re.M))
    m = re.search(r"#define M3_RD\(nbits, var\).*?\n  \}\n", dec, flags=re.S)
    assert m
    parts = [consts, _cut(com, r"enum SchemeKind"),
             _cut(com, r"__host__ __device__[^\n{;]*\bunit_is_valid\s*\("),
             _cut(com, r"__host__ __device__[^\n{;]*\bunit_nanos\s*\("),
             _cut(com, r"__host__ __device__[^\n{;]*\bscheme_kind_for_unit\s*\("),
             _cut(com, r"__host__ __device__[^\n{;]*\binitial_time_unit\s*\("),
             _cut(com, _fn("sign_extend")), _cut(com, _fn("mult_pow10")), _cut(com, _fn("load_be32")),
             _cut(dec, r"struct DecState"), _cut(dec, r"struct SlowSrc"), _cut(dec, r"struct EventSink"),
             _cut(dec, _fn("push_event")), _cut(dec, _fn("gpeek64")), m.group(0), _cut(dec, _fn("decode_dp_slow"))]
    body = "\n".join(parts)
    assert "asm" not in body
    d = tempfile.mkdtemp(prefix="m3dev_dec_host_")
    path = os.path.join(d, "dev_dec_host.cpp")
    open(path, "w").write(SHIM % os.path.join(ROOT, "include", "m3tsz_b200.h") + body + DRIVER)
    so = os.path.join(d, "dev_dec_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-w", path, "-o", so])
    lib = C.CDLL(so)
    lib.dev_decode.restype = C.c_int
    return lib


@pytest.fixture(scope="module")
def dev():
    return build_dev_decoder()


class DevDecode:
    """One stream through the complete grammar: `status`, `dps` [(ts, value bits)], `bitpos` (the stream bit after
    each datapoint), `emit_unit` / `first_unit` / `unit` (at the last and first datapoint, and when the decode
    stopped), `ann` (the first annotation: bit offset from the stream's first bit, length, count) and `events`
    (uint8 [E, 32] rows of m3tsz_dp_event, series 0)."""

    def __init__(self, dev, stream, int_opt, lead=0, cap=4096, default_unit=1, ev_cap=256):
        buf = np.zeros(lead + len(stream) + 64, dtype=np.uint8)
        buf[lead: lead + len(stream)] = np.frombuffer(stream, dtype=np.uint8)
        ts = np.zeros(cap, dtype=np.int64)
        vals = np.zeros(cap, dtype=np.uint64)
        bitpos = np.zeros(cap, dtype=np.uint32)
        n = C.c_uint32()
        events = np.zeros((ev_cap, 32), dtype=np.uint8)
        evc = C.c_ulonglong(0)
        units = np.zeros(3, dtype=np.int32)
        ann = np.zeros(3, dtype=np.uint32)
        p = lambda a: C.c_void_p(a.ctypes.data)
        self.status = dev.dev_decode(p(buf), C.c_uint64(lead + len(stream)), C.c_uint64(lead),
                                     C.c_uint64(lead + len(stream)), int(int_opt), int(default_unit), p(ts), p(vals),
                                     p(bitpos), C.c_uint32(cap), C.byref(n), p(events), C.c_uint64(ev_cap),
                                     C.byref(evc), p(units), p(ann))
        k = n.value
        self.ts, self.vals, self.bitpos = ts[:k], vals[:k], bitpos[:k]
        self.dps = list(zip(self.ts.tolist(), self.vals.tolist()))
        self.emit_unit, self.first_unit, self.unit = (int(u) for u in units)
        self.ann = tuple(int(a) for a in ann)
        assert evc.value <= ev_cap
        self.events = events[: evc.value]


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
