"""A deterministic corpus of series that sit on the edges of the M3TSZ grammar -- test infrastructure only.

Random data reaches the grammar's edges only by chance: the last and first value of each delta-of-delta bucket, an
XOR that exactly fills or just misses the previous window, a significant-bit drop held for exactly as many
datapoints as the tracker counts, a value that reaches 10^13 after a multiplier is in force.  The codec has several
copies of that grammar (the encoder's general path, second tier, hot tier and point-major tile stage, the encoder
state record, the decoder's hot candidate, fast path and complete grammar), so every copy has to agree at exactly
these points.

`corpus(lane)` returns `Series(name, ts, vals, start, unit, int_opt, cells)`, all of P datapoints.  Each series is
built to hit named CELLS at known datapoint indices (`cells`: [(key, index)]); `check_cell` says whether a
datapoint, as `indep_m3tsz.decode(..., trace=...)` read it from the stream, is that cell.  `cell_table()` is the
table of every cell the corpus claims.  Every series starts with two lead datapoints (the same value at the base
cadence) and the variants of a series prepend 0-3 more of them, so each cell lands on rows 4k, 4k + 1, 4k + 2 and
4k + 3 of a point-major input tile (a cell on the first datapoint stays at row 0).

`lane` varies the values and the start inside each cell (other lead values and walks, a shifted start, int series
negated on odd lanes), so that 32 lanes of one series template take the same cell at the same datapoint with
different data: the layout that makes the kernels' warp-voted tiers take it."""
import math
import struct
import zlib
from collections import namedtuple

import numpy as np

import indep_m3tsz as I

SEC = 10 ** 9
UNIT_NS = {1: SEC, 2: 10 ** 6, 3: 10 ** 3, 4: 1}
START0 = 1599955200 * SEC  # a multiple of every unit 1-4
P = 16  # datapoints per series (tails are steady repeats)
ROWS = 4  # rows of the point-major encode stage's input tile

Series = namedtuple("Series", "name ts vals start unit int_opt cells")

DODS = [0, 1, -1, 63, 64, -64, -65, 255, 256, -256, -257, 2047, 2048, -2048, -2049, 2 ** 31 - 1, -2 ** 31]
# 64-bit buckets (us / ns).  2^62 us is past int64 nanoseconds: the microsecond series stop at 2^52.
DODS_WIDE = {3: [2 ** 31, -2 ** 31 - 1, 2 ** 40, -2 ** 40, 2 ** 52, -2 ** 52],
             4: [2 ** 31, -2 ** 31 - 1, 2 ** 40, -2 ** 40, 2 ** 62, -2 ** 62]}
OVERFLOW_DODS = [2 ** 31, -2 ** 31 - 1]  # s / ms: M3TSZ_ERR_DOD_OVERFLOW


def dods(u):
    return DODS + DODS_WIDE.get(u, [])


def rems(u):
    """sub-unit remainders of the delta-of-delta, by magnitude (the sign follows the delta-of-delta: the division
    truncates toward zero)"""
    un = UNIT_NS[u]
    return {"0": 0} if un == 1 else {"0": 0, "1": 1, "u-1": un - 1, "half": un // 2}


def _rem_kind(r, un):
    r = abs(r)
    return {0: "0", 1: "1", un - 1: "u-1", un // 2: "half"}.get(r, "other") if un > 1 else ("0" if r == 0 else "other")


def f64(bits):
    return struct.unpack("<d", struct.pack("<Q", bits & (2 ** 64 - 1)))[0]


def bits(v):
    return struct.unpack("<Q", struct.pack("<d", v))[0]


def _lz_tz(x):
    return (64, 0) if x == 0 else (64 - x.bit_length(), (x & -x).bit_length() - 1)


def _window(lz, tz):
    """an XOR with exactly lz leading and tz trailing zeros (its two end bits set, and every fourth bit between)"""
    n = 64 - lz - tz
    body = (1 << (n - 1)) | 1 if n > 1 else 1
    body |= sum(1 << i for i in range(0, n, 4)) & ((1 << n) - 1)
    return body << tz


# ---------------------------------------------------------------------------------------------------------------
# building blocks
# ---------------------------------------------------------------------------------------------------------------
def _seed(*a):
    return zlib.crc32(repr(a).encode())


def _walk(lane, n, seed):
    """n non-integral values (never int-like at any multiplier): a walk around 100 with 15-digit mantissas"""
    rng = np.random.default_rng([seed, lane])
    return list(100.0 + 0.123456789012345 * (lane + 1) + np.cumsum(rng.normal(size=n)) * 1.000000007)


def _make(name, deltas, vals, start, unit, int_opt, cells, extra, pad_value=None):
    """`deltas` / `vals` of the probe after its two lead datapoints; `extra` more leads in front.  Cell indices are
    given relative to the probe's first datapoint after the leads; the tail repeats the last delta and value."""
    un = UNIT_NS[unit]
    base = 10 * un
    lead_v = vals[0] if pad_value is None else pad_value
    d = [base] * (2 + extra) + list(deltas)
    v = [lead_v] * (2 + extra) + list(vals)
    assert len(d) <= P, name
    while len(d) < P:
        d.append(base)
        v.append(v[-1])
    ts = np.array(start + np.cumsum(np.array(d, dtype=object)), dtype=np.int64)
    off = 2 + extra
    return Series(name, ts, np.array(v, dtype=np.float64), start, unit, int_opt,
                  [(k, i + off) for k, i in cells])


def _rows(name, deltas, vals, start, unit, int_opt, cells, pad_value=None):
    return [_make("%s/r%d" % (name, r), deltas, vals, start, unit, int_opt, cells, r, pad_value) for r in range(ROWS)]


# ---------------------------------------------------------------------------------------------------------------
# time
# ---------------------------------------------------------------------------------------------------------------
def _time(lane):
    out = []
    for int_opt in (False, True):
        for u in (1, 2, 3, 4):
            un = UNIT_NS[u]
            base = 10 * un
            start = START0 + lane * 2 * un
            for d in dods(u):
                for rk, rm in rems(u).items():
                    dd = d * un + (rm if d >= 0 else -rm)
                    w = _walk(lane, 4, _seed(u, d, rk))
                    # an edge delta-of-delta, then back to the base cadence in two halves (each inside 32 bits)
                    half = (dd // 2) // un * un
                    key = ("dod", int_opt, u, d, rk)
                    out += _rows("dod/%d/%d/%s/%d" % (u, d, rk, int_opt), [base + dd, base + half, base],
                                 w[:3], start, u, int_opt, [(key, 0)], pad_value=w[3])
                    # the same edge on the first datapoint (delta from start, previous delta 0)
                    ts = [start + dd, start + dd + dd // 2 // un * un]
                    ts += [ts[-1] + base * (i + 1) for i in range(P - 2)]
                    vals = _walk(lane, P, _seed(7, u, d, rk))
                    out.append(Series("dod1/%d/%d/%s/%d" % (u, d, rk, int_opt), np.array(ts, dtype=np.int64),
                                      np.array(vals), start, u, int_opt, [(("dod1", int_opt, u, d, rk), 0)]))
            if u <= 2:
                for d in OVERFLOW_DODS:
                    w = _walk(lane, 3, 5)
                    out += _rows("ovf/%d/%d/%d" % (u, d, int_opt), [base + d * un, base], w[:2], start, u, int_opt,
                                 [(("overflow", int_opt, u), 0)], pad_value=w[2])
                    ts = [start + d * un + base * i for i in range(P)]
                    out.append(Series("ovf1/%d/%d/%d" % (u, d, int_opt), np.array(ts, dtype=np.int64),
                                      np.array(_walk(lane, P, 6)), start, u, int_opt,
                                      [(("overflow1", int_opt, u), 0)]))
            # equal timestamps and negative deltas
            w = _walk(lane, 6, 8)
            out += _rows("delta/%d/%d" % (u, int_opt), [0, 0, -base, -base, -3 * base, base], w[:6], start, u,
                         int_opt, [(("delta0", int_opt, u), 0), (("delta0", int_opt, u), 1),
                                   (("delta_neg", int_opt, u), 2), (("delta_neg", int_opt, u), 4)])
            # start 0, negative, and not a multiple of the unit (no unit in force: the first datapoint changes it)
            for kind, st in (("zero", 0), ("negative", -START0 - lane * un), ("misaligned", START0 + 3 + lane)):
                if kind == "misaligned" and un == 1:
                    continue
                ts = [st + base * (i + 1) for i in range(P)]
                out.append(Series("start/%s/%d/%d" % (kind, u, int_opt), np.array(ts, dtype=np.int64),
                                  np.array(_walk(lane, P, 9)), st, u, int_opt, [(("start", int_opt, u, kind), 0)]))
    return out


# ---------------------------------------------------------------------------------------------------------------
# float XOR (float mode, and int-optimised series in float mode)
# ---------------------------------------------------------------------------------------------------------------
WINDOWS = [(0, 0), (11, 0), (0, 17), (20, 20), (31, 32), (1, 52), (12, 1)]
SPECIALS = {"nan_payload": [0x7FF0000000000001, 0x7FF8000000000001, 0xFFF8000000000000, 0x7FFFFFFFFFFFFFFF],
            "zero": [0x0000000000000000, 0x8000000000000000],
            "inf": [0x7FF0000000000000, 0xFFF0000000000000],
            "subnormal": [0x0000000000000001, 0x000FFFFFFFFFFFFF, 0x8000000000000001]}


def _xor_series(name, v0, xs, int_opt, unit, lane, cells):
    vals, b = [], v0
    for x in xs:
        b ^= x
        vals.append(f64(b))
    return _rows(name, [10 * UNIT_NS[unit]] * len(xs), vals, START0 + lane * SEC, unit, int_opt, cells,
                 pad_value=f64(v0))


def _xor(lane):
    out = []
    for int_opt in (False, True):
        v0 = bits(100.0 + 0.123456789012345 * (lane + 1))
        unit = 1
        m = int_opt
        for kind, x in (("zero", 0), ("lz63", 1), ("tz63", 1 << 63), ("ones", 2 ** 64 - 1)):
            out += _xor_series("xor/%s/%d" % (kind, m), v0, [_window(8, 8), x, x], int_opt, unit, lane,
                               [(("xor", m, kind), 1), (("xor", m, kind), 2)])
        for lz, tz in WINDOWS:
            # a window, the same window exactly (contained), one bit wider on each side in turn (new windows), back
            # to the window and one bit narrower on both sides (contained)
            w = _window(lz, tz)
            n = 64 - lz - tz
            xs = [w, w ^ (1 << (tz + n // 2)) if n > 2 else w]
            cells = [(("xor", m, "exact"), 1)]
            if lz > 0:
                xs += [_window(lz - 1, tz), w]
                cells.append((("xor", m, "wider_lead"), len(xs) - 2))
            if tz > 0:
                xs += [_window(lz, tz - 1), w]
                cells.append((("xor", m, "wider_trail"), len(xs) - 2))
            if n > 2:
                xs.append(_window(lz + 1, tz + 1))
                cells.append((("xor", m, "narrower"), len(xs) - 1))
            out += _xor_series("xor/win%d_%d/%d" % (lz, tz, m), v0, xs, int_opt, unit, lane, cells)
        # the widest codes: a full-width XOR alternating with a narrower one (78-bit new window, 66-bit contained)
        xs = [_window(4, 4)] + [2 ** 64 - 1, _window(3, 5)] * 4
        out += _xor_series("xor/alt/%d" % m, v0, xs, int_opt, unit, lane,
                           [(("xor", m, "alt78"), i) for i in range(1, 9, 2)] +
                           [(("xor", m, "alt66"), i) for i in range(2, 9, 2)])
        for kind, bs in SPECIALS.items():
            vals = []
            for b in bs:
                vals += [f64(b), f64(v0 ^ (lane << 3))]
            out += _rows("special/%s/%d" % (kind, m), [10 * SEC] * len(vals), vals, START0 + lane * SEC, unit,
                         int_opt, [(("special", m, kind), i) for i in range(0, len(vals), 2)],
                         pad_value=f64(v0 ^ (lane << 3)))
    return out


# ---------------------------------------------------------------------------------------------------------------
# int mode
# ---------------------------------------------------------------------------------------------------------------
def _below(k):
    """the largest double below 2^k (2^k - 1 while that is exact)"""
    return float(2 ** k - 1) if k <= 53 else math.nextafter(2.0 ** k, 0.0)


def _int(lane):
    out = []
    sg = -1.0 if lane % 2 else 1.0
    base = 10 * SEC
    start = START0 + lane * SEC

    def rows(name, vals, cells, pad=None):
        neg = lambda v: sg * v if v else 0.0
        return _rows(name, [base] * len(vals), [neg(v) for v in vals], start, 1, True, cells,
                     pad_value=None if pad is None else neg(pad))

    # |diff| = 2^k - 1 and 2^k, both signs: num_sig 1..63
    for k in range(0, 64):
        for mag in ([_below(k)] if k else []) + ([2.0 ** k] if k <= 62 else []):
            n = int(mag).bit_length()
            out += rows("sig/%d/%d" % (k, n), [mag, 0.0, -mag, 0.0],
                        [(("int_sig", n, "+" if sg > 0 else "-"), 0), (("int_sig", n, "-" if sg > 0 else "+"), 1),
                         (("int_sig", n, "-" if sg > 0 else "+"), 2), (("int_sig", n, "+" if sg > 0 else "-"), 3)],
                        pad=0.0)
    # the first value's 64-bit payload: -2^63 (|value| 2^63, num_sig 64); and a diff of 2^63 or more (float)
    ts = np.array([START0 + (i + 1) * base for i in range(P)], dtype=np.int64)
    out.append(Series("sig64_first", ts, np.array([-2.0 ** 63] + [-2.0 ** 63 + 2 ** 20] * (P - 1)), START0, 1, True,
                      [(("int_first_sig", 64), 0)]))
    big = _below(63)
    out += rows("diff_overflow", [big, -big, 5.0], [(("int_diff_overflow",), 1)], pad=0.0)
    # new_sig = 0: the same integer at rising multipliers, five times (the tracker's highest lower value is 0)
    out += rows("newsig0", [0.8, 0.08, 0.008, 0.0008, 0.00008, 0.00009], [(("int_newsig0",), 4)], pad=8.0)
    # tracker: drops of exactly 2, 3 and 4 bits held for 4, 5 and 6 datapoints (a higher lower value in a 4-bit run)
    S = 20
    for drop in (2, 3, 4):
        for held in (4, 5, 6):
            vals, v = [], 0.0
            v += 2.0 ** (S - 1)
            vals.append(v)
            for j in range(held):
                ns = S - drop + (1 if (drop == 4 and j == 1) else 0)
                v += (2.0 ** (ns - 1)) * (1 if j % 2 else -1)
                vals.append(v)
            v += 2.0 ** (S - 1)
            vals.append(v)
            out += rows("track/%d/%d" % (drop, held), vals, [(("track", drop, held), 1)], pad=0.0)
    # multipliers 0..6 one at a time, jumping, and 7 decimals (float)
    out += rows("mult/step", [1.0, 1.1, 1.12, 1.123, 1.1234, 1.12345, 1.123456, 1.1234567],
                [(("mult", m, "step"), m) for m in range(1, 7)] + [(("mult7",), 7)], pad=3.0)
    for m in range(1, 7):
        v = round(1.0 + sum(10.0 ** -j * ((j % 9) + 1) for j in range(1, m + 1)), m)
        out += rows("mult/jump%d" % m, [2.0, v, 2.0], [(("mult", m, "jump"), 1)], pad=3.0)
    # float -> int: max_mult is written again (the float_changed branch), and re-established at 2
    out += rows("float_changed/0", [5.0, 6.0, 1.2345678, 7.0], [(("float_changed", 0), 3)], pad=4.0)
    out += rows("float_changed/2", [1.25, 1.5, 1.2345678, 1.75], [(("float_changed", 2), 3)], pad=1.0)
    # 10^13 reached after multiplier m is in force: v * 10^m = 10^13, and its neighbours
    for m in range(1, 7):
        first = 10.0 ** -m
        at = 10.0 ** (13 - m)
        for which, v in (("at", at), ("below", math.nextafter(at, 0.0)), ("above", math.nextafter(at, math.inf)),
                         ("int_below", (10.0 ** 13 - 1) / 10.0 ** m)):
            out += rows("e13/%d/%s" % (m, which), [first, 2 * first, v, 3 * first], [(("e13", m, which), 2)],
                        pad=first)
    # within 1-2 ulps of k / 10^m (the r < 0.1 / r > 0.9 rounding at the multiplier in force)
    for m in range(0, 7):
        for k in (3, 1234567):
            c = k / 10.0 ** m
            first = 10.0 ** -m
            for off in (-2, -1, 1, 2):
                v = c
                for _ in range(abs(off)):
                    v = math.nextafter(v, math.inf if off > 0 else -math.inf)
                out += rows("round/%d/%d/%d" % (m, k, off), [first, v, c + first], [(("round", m, off), 1)],
                            pad=first)
    # int repeats and float repeats
    out += rows("repeat/int", [7.0, 7.0, 7.0], [(("int_repeat",), 1)], pad=3.0)
    out += rows("repeat/float", [0.123456789012, 0.123456789012, 2.0], [(("float_repeat",), 1)], pad=3.0)
    return out


# ---------------------------------------------------------------------------------------------------------------
# the widest codes
# ---------------------------------------------------------------------------------------------------------------
def widest(lane, n=P):
    """series whose every datapoint after the first is the widest code of its mode and tier: float mode (both
    int_opt), zero delta-of-delta and the 78 / 66-bit XOR alternation (the hot tier); int mode, a 16-bit
    delta-of-delta bucket and 63-bit payloads.  Every lane starts at START0."""
    out = []
    for int_opt in (False, True):
        b = bits(100.0 + 0.123456789012345 * (lane + 1))
        vals = []
        for i in range(n):
            b ^= (2 ** 64 - 1) if i % 2 else _window(3 + i % 3, 5)
            vals.append(f64(b))
        ts = START0 + 10 * SEC * np.arange(1, n + 1, dtype=np.int64)
        out.append(Series("widest/float/%d" % int_opt, ts, np.array(vals), START0, 1, int_opt,
                          [(("widest_float", int_opt), i) for i in range(2, n)]))
    sg = -1.0 if lane % 2 else 1.0
    big = _below(63)
    vals = [sg * (0.0 if i % 2 == 0 else (big if i % 4 == 1 else -big)) for i in range(n)]
    d = [10 * SEC, 10 * SEC] + [(10 + (2047 if i % 2 == 0 else 0)) * SEC for i in range(2, n)]  # +-2047
    ts = np.array(START0 + np.cumsum(np.array(d, dtype=object)), dtype=np.int64)
    out.append(Series("widest/int", ts, np.array(vals), START0, 1, True,
                      [(("widest_int",), i) for i in range(3, n)]))
    return out


def corpus(lane=0):
    return _time(lane) + _xor(lane) + _int(lane) + widest(lane)


def cell_table():
    """every cell the corpus claims, from the edge lists above"""
    cells = set()
    for m in (False, True):
        for u in (1, 2, 3, 4):
            for d in dods(u):
                for rk in rems(u):
                    cells |= {("dod", m, u, d, rk), ("dod1", m, u, d, rk)}
            if u <= 2:
                cells |= {("overflow", m, u), ("overflow1", m, u)}
            cells |= {("delta0", m, u), ("delta_neg", m, u), ("start", m, u, "zero"), ("start", m, u, "negative")}
            if u != 4:
                cells.add(("start", m, u, "misaligned"))
        cells |= {("xor", m, k) for k in ("zero", "lz63", "tz63", "ones", "exact", "wider_lead", "wider_trail",
                                          "narrower", "alt78", "alt66")}
        cells |= {("special", m, k) for k in SPECIALS}
        cells.add(("widest_float", m))
    for k in range(0, 64):
        for n in ([k] if k else []) + ([k + 1] if k <= 62 else []):
            cells |= {("int_sig", n, "+"), ("int_sig", n, "-")}
    cells |= {("int_first_sig", 64), ("int_diff_overflow",), ("int_newsig0",), ("mult7",), ("float_changed", 0),
              ("float_changed", 2), ("int_repeat",), ("float_repeat",), ("widest_int",)}
    cells |= {("track", d, h) for d in (2, 3, 4) for h in (4, 5, 6)}
    cells |= {("mult", m, k) for m in range(1, 7) for k in ("step", "jump")}
    cells |= {("e13", m, w) for m in range(1, 7) for w in ("at", "below", "above", "int_below")}
    cells |= {("round", m, o) for m in range(0, 7) for o in (-2, -1, 1, 2)}
    return cells


# ---------------------------------------------------------------------------------------------------------------
# what a cell looks like in the stream
# ---------------------------------------------------------------------------------------------------------------
def check_cell(key, s, tr, i, oracle_status=0):
    """True when datapoint i of series s (its trace `tr`, from indep_m3tsz.decode of the oracle's stream) is the
    cell `key`; `oracle_status` is the oracle encoder's status on the series"""
    fam = key[0]
    if fam in ("overflow", "overflow1"):
        return oracle_status == 4 and len(tr) == i  # the stream holds the datapoints before the failing one
    if i >= len(tr):
        return False
    e = tr[i]
    if fam in ("dod", "dod1"):
        _, _, u, d, rk = key
        un = UNIT_NS[u]
        prev_t = s.start if i == 0 else int(s.ts[i - 1])
        prev_d = 0 if i == 0 else (prev_t - (s.start if i == 1 else int(s.ts[i - 2])))
        dd = int(s.ts[i]) - prev_t - prev_d
        if e["unit_changed"] or e["dod"] != d or _rem_kind(dd - d * un, un) != rk:
            return False
        want = 0 if d == 0 else (7 if -64 <= d <= 63 else (9 if -256 <= d <= 255 else (12 if -2048 <= d <= 2047
                                                                                        else (32 if u <= 2 else 64))))
        return e["bucket"] == want
    if fam == "delta0":
        return int(s.ts[i]) == int(s.ts[i - 1])
    if fam == "delta_neg":
        return int(s.ts[i]) < int(s.ts[i - 1])
    if fam == "start":
        kind = key[3]
        ok = {"zero": s.start == 0, "negative": s.start < 0,
              "misaligned": s.start % UNIT_NS[key[2]] != 0}[kind]
        return ok and e["unit_changed"] == (kind == "misaligned")
    if fam in ("xor", "widest_float"):
        if e["kind"] not in ("zero", "contained", "new") and not (key[:3] == ("xor", True, "zero")):
            return False
        if fam == "widest_float":
            return e["dod"] == 0 and e["kind"] in ("contained", "new") and e["nbits"] == 64
        kind = key[2]
        if kind == "zero":  # (int-optimised: a float repeat)
            return e["xor"] == 0 if not key[1] else (e["kind"] == "repeat" and e["is_float"])
        x, p = e["xor"], tr[i - 1]
        if kind == "lz63":
            return x == 1
        if kind == "tz63":
            return x == 1 << 63
        if kind == "ones":
            return x == 2 ** 64 - 1
        lz, tz = _lz_tz(x)
        plz, ptz = _lz_tz(p["xor"]) if p["kind"] in ("zero", "contained", "new", "full") else (None, None)
        if kind == "exact":
            return e["kind"] == "contained" and (lz, tz) == (plz, ptz)
        if kind == "wider_lead":
            return e["kind"] == "new" and (lz, tz) == (plz - 1, ptz)
        if kind == "wider_trail":
            return e["kind"] == "new" and (lz, tz) == (plz, ptz - 1)
        if kind == "narrower":
            return e["kind"] == "contained" and (lz, tz) == (plz + 1, ptz + 1)
        if kind == "alt78":
            return e["kind"] == "new" and (lz, tz) == (0, 0)
        if kind == "alt66":
            return e["kind"] == "contained" and (plz, ptz) == (0, 0)
    if fam == "special":
        b = e["bits"]
        kind = key[2]
        exp, man = (b >> 52) & 0x7FF, b & ((1 << 52) - 1)
        is_kind = {"nan_payload": exp == 0x7FF and man != 0, "zero": (b & ~(1 << 63)) == 0,
                   "inf": exp == 0x7FF and man == 0, "subnormal": exp == 0 and man != 0}[kind]
        if key[1] and kind in ("zero", "subnormal"):  # int-optimised: +-0 and the least subnormals are int-like (0)
            return is_kind or (e["kind"] in ("int_update", "int_diff", "repeat") and not e["is_float"])
        return is_kind
    if fam == "int_sig":
        n, sign = key[1], key[2]
        return e["kind"] in ("int_diff", "int_update") and e["sig"] == n and e["payload"].bit_length() == n and \
            e["neg"] == (sign == "+")
    if fam == "int_first_sig":
        return e["kind"] == "int_first" and e["sig"] == 64 and e["payload"] == 1 << 63
    if fam == "int_diff_overflow":
        return e["kind"] == "float_switch"
    if fam == "int_newsig0":
        return e["kind"] == "int_update" and e["sig_code"] == "zero" and e["sig"] == 0
    if fam == "track":
        _, drop, held = key
        S = tr[i - 1]["sig"]
        run = tr[i: i + held]
        if len(run) < held or any(r["kind"] not in ("int_diff", "int_update") for r in run):
            return False
        if drop >= 3 and held >= 5:  # the fifth drop sets the highest lower value
            hi = max(r["payload"].bit_length() for r in run[:5])
            return all(r["sig"] == S for r in run[:4]) and run[4]["sig_code"] == "set" and run[4]["sig"] == hi and \
                hi == S - drop + (1 if drop == 4 else 0)
        return all(r["sig"] == S and r["payload"].bit_length() <= S - drop + (drop == 4) for r in run)
    if fam == "mult":
        return e["kind"] == "int_update" and e["mult_code"] == "set" and e["mult"] == key[1]
    if fam == "mult7":
        return e["kind"] == "float_switch"
    if fam == "float_changed":
        return e["kind"] == "int_update" and e["mult_code"] == "set" and e["mult"] == key[1] and \
            tr[i - 1]["kind"] in ("float_switch", "contained", "new", "zero", "repeat")
    if fam == "e13":
        which = key[2]
        want_float = I.convert_to_int_float(abs(float(s.vals[i])), key[1])[2]
        if which == "at":
            assert want_float
        return e["kind"] == ("float_switch" if want_float else "int_diff") or \
            (not want_float and e["kind"] == "int_update")
    if fam == "round":
        return e["kind"] in ("int_diff", "int_update", "float_switch", "repeat")
    if fam == "int_repeat":
        return e["kind"] == "repeat" and not e["is_float"]
    if fam == "float_repeat":
        return e["kind"] == "repeat" and e["is_float"]
    if fam == "widest_int":
        return e["bucket"] == 12 and e["kind"] == "int_diff" and e["sig"] == 63
    raise KeyError(key)
