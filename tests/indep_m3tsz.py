"""A SECOND, independent restatement of the M3TSZ decoder in pure Python -- test infrastructure only.

The CPU oracle (oracle/m3tsz_oracle.c) and the CUDA kernels were written by the same hands; this decoder was
written separately, straight from the reference's iterator (m3tsz/iterator.go:81-219,
m3tsz/timestamp_iterator.go:80-361, m3tsz/float_encoder_iterator.go:105-165, scheme.go:40-242,
x/time/unit.go) without looking at the C code, and is used to cross-check the oracle's ENCODER and DECODER on
streams no golden vector of the reference covers (int-optimised encodes of arbitrary series).  Well-formed
streams only: a short read raises EOFError instead of reproducing the iterator's error swallowing."""
import struct

UNIT_NANOS = {1: 10 ** 9, 2: 10 ** 6, 3: 10 ** 3, 4: 1, 5: 60 * 10 ** 9, 6: 3600 * 10 ** 9, 7: 86400 * 10 ** 9,
              8: 365 * 86400 * 10 ** 9}  # x/time/unit.go:30-60 (second .. year)
# scheme.go:40-75: bucket value bits [7, 9, 12]; default bucket 32 bits for s / ms, 64 for us / ns
DEFAULT_BUCKET_BITS = {1: 32, 2: 32, 3: 64, 4: 64}
MARKER_OPCODE, MARKER_OPCODE_BITS, MARKER_VALUE_BITS = 0x100, 9, 2  # scheme.go:198-242
MARKER_EOS, MARKER_ANNOTATION, MARKER_TIME_UNIT = 0, 1, 2


class Bits:
    def __init__(self, data):
        self.v = int.from_bytes(data, "big")
        self.n = 8 * len(data)
        self.pos = 0

    def remaining(self):
        return self.n - self.pos

    def peek(self, k):
        if self.remaining() < k:
            return None
        return (self.v >> (self.n - self.pos - k)) & ((1 << k) - 1) if k else 0

    def read(self, k):
        r = self.peek(k)
        if r is None:
            raise EOFError("need %d bits, %d left" % (k, self.remaining()))
        self.pos += k
        return r


def _sign_extend(v, bits):
    return v - (1 << bits) if v >> (bits - 1) else v


def _initial_time_unit(start_ns, default_unit):  # timestamp_encoder.go:248-259
    if default_unit in UNIT_NANOS and start_ns % UNIT_NANOS[default_unit] == 0:
        return default_unit
    return 0


def _lz_tz(x):  # encoding.go:29-49: (64, 0) for zero
    if x == 0:
        return 64, 0
    return 64 - x.bit_length(), (x & -x).bit_length() - 1


def _read_varint(b):  # encoding/binary.ReadVarint over whole bytes read through the bit stream
    ux, shift = 0, 0
    while True:
        byte = b.read(8)
        ux |= (byte & 0x7F) << shift
        if byte < 0x80:
            break
        shift += 7
    x = ux >> 1
    return ~x if ux & 1 else x


def decode(data, int_optimized, default_unit=1, trace=None):
    """-> list of (timestamp_ns, value_bits_as_uint64, unit, annotation bytes or b"").

    `trace` (a list) receives one dict per datapoint, what the stream said about it: `dod` (in the unit; None after
    a unit change) and its `bucket` (0, 7, 9, 12, 32 or 64 value bits; "tu64" for the 64-bit nanoseconds after a
    unit change), `unit_changed`; the value code `kind` ("full", "zero", "contained", "new" for XOR codes; int mode
    also "float_first", "int_first", "repeat", "float_switch", "int_update", "int_diff"), with `xor` and `nbits`
    (payload bits) for XOR codes, `payload` and `neg` (the sign bit: 1 adds) for int codes, `sig_code` / `mult_code`
    (None, "same", "zero", "set") of a header, and `sig`, `mult`, `is_float`, `t` and `bits` after the datapoint."""
    b = Bits(bytes(data))
    out = []
    cur = {}
    prev_time = prev_delta = 0
    unit, unit_changed = 0, False
    prev_bits = prev_xor = 0
    int_val, mult, sig, is_float = 0.0, 0, 0, False
    if b.n == 0:
        return out

    def dod_or_marker():
        """timestamp_iterator.go:175-302 -> (dod_ns, done, annotation)"""
        nonlocal unit, unit_changed
        ann = b""
        while True:
            pk = b.peek(MARKER_OPCODE_BITS + MARKER_VALUE_BITS)
            if pk is not None and (pk >> MARKER_VALUE_BITS) == MARKER_OPCODE:
                mv = pk & 3
                if mv == MARKER_EOS:
                    b.read(11)
                    return 0, True, ann
                if mv == MARKER_ANNOTATION:
                    b.read(11)
                    n = _read_varint(b) + 1
                    assert n > 0
                    ann = bytes(b.read(8) for _ in range(n))
                    continue
                if mv == MARKER_TIME_UNIT:
                    b.read(11)
                    tu = b.read(8)
                    if 1 <= tu <= 8 and tu != unit:
                        unit_changed = True
                    unit = tu
                    continue
            break
        cur.update(unit_changed=unit_changed, dod=None, bucket="tu64")
        if unit_changed:  # readFullTimestamp: 64 bits of nanoseconds
            return _sign_extend(b.read(64), 64), False, ann
        assert unit in DEFAULT_BUCKET_BITS, "no time encoding scheme for unit %d" % unit
        if b.read(1) == 0:
            cur.update(dod=0, bucket=0)
            return 0, False, ann
        for ones, vbits in ((1, 7), (2, 9), (3, 12)):  # opcodes 10, 110, 1110
            if b.read(1) == 0:
                d = _sign_extend(b.read(vbits), vbits)
                cur.update(dod=d, bucket=vbits)
                return d * UNIT_NANOS[unit], False, ann
        vbits = DEFAULT_BUCKET_BITS[unit]
        d = _sign_extend(b.read(vbits), vbits)
        cur.update(dod=d, bucket=vbits)
        return d * UNIT_NANOS[unit], False, ann

    def read_full_float(kind="full"):
        nonlocal prev_bits, prev_xor
        prev_bits = prev_xor = b.read(64)
        cur.update(kind=kind, xor=prev_xor, nbits=64)

    def read_next_float():  # float_encoder_iterator.go:117-165
        nonlocal prev_bits, prev_xor
        if b.read(1) == 0:
            prev_xor = 0
            cur.update(kind="zero", xor=0, nbits=0)
            return
        if b.read(1) == 0:  # '10' contained
            pl, pt = _lz_tz(prev_xor)
            prev_xor = b.read(64 - pl - pt) << pt
            cur.update(kind="contained", nbits=64 - pl - pt)
        else:  # '11' uncontained
            hdr = b.read(12)
            lead, nbits = hdr >> 6, (hdr & 63) + 1
            prev_xor = b.read(nbits) << (64 - lead - nbits)
            cur.update(kind="new", nbits=nbits)
        cur["xor"] = prev_xor
        prev_bits ^= prev_xor

    def read_sig_mult():  # iterator.go:178-193
        nonlocal sig, mult
        cur.update(sig_code="same", mult_code="same")
        if b.read(1) == 1:
            sig = 0 if b.read(1) == 0 else b.read(6) + 1
            cur["sig_code"] = "set" if sig else "zero"
        if b.read(1) == 1:
            mult = b.read(3)
            cur["mult_code"] = "set"
            assert mult <= 6, "invalid multiplier"

    def read_int_diff():  # iterator.go:195-219 (sign bit 1 = add)
        nonlocal int_val
        neg = b.read(1)
        sign = 1.0 if neg == 1 else -1.0
        payload = b.read(sig)
        cur.update(neg=neg, payload=payload)
        int_val += sign * float(payload)

    first = True
    while True:
        cur = {"kind": None, "sig_code": None, "mult_code": None}
        if first:
            nt = _sign_extend(b.read(64), 64)
            if unit == 0:
                unit = _initial_time_unit(nt, default_unit)
            dod, done, ann = dod_or_marker()
            if done:
                break
            prev_delta += dod
            prev_time = nt + prev_delta
        else:
            dod, done, ann = dod_or_marker()
            if done:
                break
            prev_delta += dod
            prev_time += prev_delta
        if unit_changed:
            prev_delta, unit_changed = 0, False
        # ---- value ----
        if not int_optimized:
            read_full_float() if first else read_next_float()
        elif first:
            if b.read(1) == 1:
                read_full_float("float_first")
                is_float = True
            else:
                cur["kind"] = "int_first"
                read_sig_mult()
                read_int_diff()
        else:
            if b.read(1) == 0:  # update
                if b.read(1) == 1:
                    cur["kind"] = "repeat"
                elif b.read(1) == 1:
                    read_full_float("float_switch")
                    is_float = True
                else:
                    cur["kind"] = "int_update"
                    read_sig_mult()
                    read_int_diff()
                    is_float = False
            elif is_float:
                read_next_float()
            else:
                cur["kind"] = "int_diff"
                read_int_diff()
        if not int_optimized or is_float:
            vbits = prev_bits
        else:
            v = int_val if mult == 0 else int_val / (10.0 ** mult)
            vbits = struct.unpack("<Q", struct.pack("<d", v))[0]
        out.append((prev_time, vbits, unit, ann))
        if trace is not None:
            cur.update(t=prev_time, bits=vbits, sig=sig, mult=mult, is_float=is_float)
            trace.append(cur)
        first = False
        # the reference keys "first" on PrevTime == 0 (timestamp_iterator.go:89); same thing for real timestamps
        assert prev_time != 0
    return out


# =====================================================================================================
# Independent ENCODER (m3tsz/encoder.go:89-250, timestamp_encoder.go:72-259, float_encoder_iterator.go:69-103,
# int_sig_bits_tracker.go:35-91, m3tsz.go:78-127, ostream.go:133-221, scheme.go:198-211), also written
# separately from the C oracle.  Used to compare BYTES with the oracle's encoder.
# =====================================================================================================
import math

_MULT = [1.0]
for _i in range(6):
    _MULT.append(_MULT[-1] * 10.0)  # createMultipliers: repeated * 10.0
_MAX_INT, _MIN_INT, _MAX_OPT_INT = float(2 ** 63 - 1), float(-2 ** 63), 10.0 ** 13


def _f64_bits(v):
    return struct.unpack("<Q", struct.pack("<d", v))[0]


def _go_f2i(x):
    """int64(float64) as Go on amd64 does it (CVTTSD2SQ): out of range / NaN -> 0x8000000000000000"""
    if x != x or x >= 2.0 ** 63 or x < -2.0 ** 63:
        return -2 ** 63
    return int(x)


def _modf(v):  # math.Modf -> (int part, frac part)
    if math.isinf(v):
        return v, float("nan")
    f, i = math.modf(v)
    return i, f


def convert_to_int_float(v, cur_max_mult):
    """-> (val, mult, is_float)  m3tsz.go:78-119"""
    if cur_max_mult == 0 and v < _MAX_INT:
        i, r = _modf(v)
        if r == 0:
            return i, 0, False
    assert cur_max_mult <= 6
    sign = -1.0 if v < 0 else 1.0
    for mult in range(cur_max_mult, 7):
        val = v * _MULT[mult] * sign
        if val >= _MAX_OPT_INT:
            break
        i, r = _modf(val)
        if r == 0:
            return sign * i, mult, False
        elif r < 0.1:
            if math.nextafter(val, 0.0) <= i:
                return sign * i, mult, False
        elif r > 0.9:
            nxt = i + 1
            if math.nextafter(val, nxt) >= nxt:
                return sign * nxt, mult, False
    return v, 0, True


class _Out:
    def __init__(self):
        self.v, self.n = 0, 0

    def w(self, value, nbits):  # low nbits of value, MSB first; > 64 clamps (ostream.go:186-188)
        nbits = min(nbits, 64)
        if nbits <= 0:
            return
        self.v = (self.v << nbits) | (value & ((1 << nbits) - 1))
        self.n += nbits

    def finish(self):  # end-of-stream marker + zero padding (scheme.go:198-211)
        self.w(MARKER_OPCODE, MARKER_OPCODE_BITS)
        self.w(MARKER_EOS, MARKER_VALUE_BITS)
        pad = (-self.n) % 8
        return ((self.v << pad).to_bytes((self.n + pad) // 8, "big"))


def _num_sig(x):
    return x.bit_length()


def encode(start_ns, dps, int_optimized, default_unit=1):
    """dps: iterable of (timestamp_ns, value, unit, annotation bytes) -> stream bytes (b"" when empty)"""
    o = _Out()
    prev_time, prev_delta = start_ns, 0
    unit = _initial_time_unit(start_ns, default_unit)
    last_ann = None
    prev_bits = prev_xor = 0
    int_val, max_mult, is_float = 0.0, 0, False
    num_sig = cur_highest_lower = num_lower = 0
    n_enc = 0

    def write_xor(x):
        pl, pt = _lz_tz(prev_xor)
        cl, ct = _lz_tz(x)
        if x == 0:
            o.w(0, 1)
        elif cl >= pl and ct >= pt:
            o.w(2, 2)
            o.w(x >> pt, 64 - pl - pt)
        else:
            o.w(3, 2)
            o.w(cl, 6)
            o.w(64 - cl - ct - 1, 6)
            o.w(x >> ct, 64 - cl - ct)

    def write_full_float(bits):
        nonlocal prev_bits, prev_xor
        prev_bits = prev_xor = bits
        o.w(bits, 64)

    def write_next_float(bits):
        nonlocal prev_bits, prev_xor
        x = prev_bits ^ bits
        write_xor(x)
        prev_xor, prev_bits = x, bits

    def write_int_sig(sig):
        nonlocal num_sig
        if num_sig != sig:
            o.w(1, 1)
            if sig == 0:
                o.w(0, 1)
            else:
                o.w(1, 1)
                o.w(sig - 1, 6)
        else:
            o.w(0, 1)
        num_sig = sig

    def write_int_sig_mult(sig, mult, float_changed):
        nonlocal max_mult
        write_int_sig(sig)
        if mult > max_mult:
            o.w(1, 1)
            o.w(mult, 3)
            max_mult = mult
        elif num_sig == sig and max_mult == mult and float_changed:
            o.w(1, 1)
            o.w(max_mult, 3)
        else:
            o.w(0, 1)

    def write_int_val_diff(bits, neg):
        o.w(1 if neg else 0, 1)
        o.w(bits, num_sig)

    def track_new_sig(ns):
        nonlocal cur_highest_lower, num_lower
        new = num_sig
        if ns > num_sig:
            new = ns
        elif num_sig - ns >= 3:
            if num_lower == 0:
                cur_highest_lower = ns
            elif ns > cur_highest_lower:
                cur_highest_lower = ns
            num_lower += 1
            if num_lower >= 5:
                new = cur_highest_lower
                num_lower = 0
        else:
            num_lower = 0
        return new

    for t, v, u, ann in dps:
        # ---------------- timestamp (WriteTime) ----------------
        if n_enc == 0:
            o.w(prev_time & (2 ** 64 - 1), 64)
        if ann and ann != last_ann:
            o.w(MARKER_OPCODE, MARKER_OPCODE_BITS)
            o.w(MARKER_ANNOTATION, MARKER_VALUE_BITS)
            x = len(ann) - 1
            ux = (x << 1) ^ (x >> 63)  # zig-zag (x >= 0 here)
            while ux >= 0x80:
                o.w((ux & 0x7F) | 0x80, 8)
                ux >>= 7
            o.w(ux, 8)
            for byte in ann:
                o.w(byte, 8)
            last_ann = ann
        tu_changed = False
        if 1 <= u <= 8 and u != unit:
            o.w(MARKER_OPCODE, MARKER_OPCODE_BITS)
            o.w(MARKER_TIME_UNIT, MARKER_VALUE_BITS)
            o.w(u, 8)
            unit = u
            tu_changed = True
        delta = t - prev_time
        prev_time = t
        if tu_changed:
            o.w((delta - prev_delta) & (2 ** 64 - 1), 64)
            prev_delta = 0
        else:
            un = UNIT_NANOS[u]
            d = delta - prev_delta
            dod = abs(d) // un * (1 if d >= 0 else -1)  # Go's truncating division
            if u in (1, 2):
                assert -2 ** 31 <= dod < 2 ** 31, "deltaOfDelta overflows 32 bits"
            if dod == 0:
                o.w(0, 1)
            elif -64 <= dod <= 63:
                o.w(0b10, 2)
                o.w(dod, 7)
            elif -256 <= dod <= 255:
                o.w(0b110, 3)
                o.w(dod, 9)
            elif -2048 <= dod <= 2047:
                o.w(0b1110, 4)
                o.w(dod, 12)
            else:
                o.w(0b1111, 4)
                o.w(dod, DEFAULT_BUCKET_BITS[u])
            prev_delta = delta
        # ---------------- value ----------------
        if not int_optimized:
            write_full_float(_f64_bits(v)) if n_enc == 0 else write_next_float(_f64_bits(v))
        elif n_enc == 0:
            val, mult, isf = convert_to_int_float(v, 0)
            if isf:
                o.w(1, 1)
                write_full_float(_f64_bits(v))
                is_float, max_mult = True, mult
            else:
                o.w(0, 1)
                int_val = val
                neg_diff = True
                if val < 0:
                    neg_diff, val = False, -val
                bits = _go_f2i(val) & (2 ** 64 - 1)
                write_int_sig_mult(_num_sig(bits), mult, False)
                write_int_val_diff(bits, neg_diff)
        else:
            val, mult, isf = convert_to_int_float(v, max_mult)
            diff = 0.0 if isf else int_val - val
            if isf or diff >= _MAX_INT or diff <= _MIN_INT:
                fb = _f64_bits(val)
                if not is_float:
                    o.w(0, 1)
                    o.w(0, 1)
                    o.w(1, 1)
                    write_full_float(fb)
                    is_float, max_mult = True, mult
                elif fb == prev_bits:
                    o.w(0, 1)
                    o.w(1, 1)
                else:
                    o.w(1, 1)
                    write_next_float(fb)
            elif diff == 0 and not is_float and mult == max_mult:
                o.w(0, 1)
                o.w(1, 1)
            else:
                neg = diff < 0
                if neg:
                    diff = -diff
                bits = _go_f2i(diff) & (2 ** 64 - 1)
                new_sig = track_new_sig(_num_sig(bits))
                float_changed = is_float  # isFloat (false here) != enc.isFloat
                if mult > max_mult or num_sig != new_sig or float_changed:
                    o.w(0, 1)
                    o.w(0, 1)
                    o.w(0, 1)
                    write_int_sig_mult(new_sig, mult, float_changed)
                    write_int_val_diff(bits, neg)
                    is_float = False
                else:
                    o.w(1, 1)
                    write_int_val_diff(bits, neg)
                int_val = val
        n_enc += 1
    return o.finish() if n_enc else b""
