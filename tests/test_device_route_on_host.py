"""The bucket writes' ROUTE logic, compiled for the host from the .cu source text: `RouteEnc`, `route_enc_load`,
`route_at`, `route_last_value<INT_OPT>` and `route_series<INT_OPT>` (m3tsz_encode.cu) with `RouteParams` /
`RouteTouched` (m3tsz_kernels.h), on top of the encoder and state functions the append harness cuts out.  One
bucket is driven call by call the way the device drives it: the route decides every datapoint's target and
result, then each encoder the route sent datapoints to takes its share through the append harness's lane.  Between
calls only the states, slots, pool counter and table survive.

Every per-datapoint result and every encoder's snapshot and public prefix must equal the BufferBucket.write model
over the ORACLE encoder (bucket_model.py), over thousands of random write sequences and call splits in both modes:
out-of-order writes, duplicates, upserts, annotations, unit changes, delta-of-delta overflows, bad units, the
encoder limit and t == 0.  The append must take every datapoint the route sends it.  A CPU regression harness for
the device source; nothing of it ships."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O
from bucket_model import ERR_CAPACITY, SEC, Bucket, random_calls
from host_build import build_dev_append, constants, cut, fn, source_text

ROUTE_DRIVER = r"""
// one call of one bucket (series 0 of a one-series batch, series-major)
extern "C" int dev_route(int int_opt, m3tsz_encoder_state *state, uint64_t slot_words, m3tsz_encoder_state *pool,
                         uint64_t pool_capacity, uint64_t pool_slot_words, uint32_t *pool_count, int32_t *table, int K,
                         const int64_t *ts, const double *val, uint64_t n, const uint8_t *units, int unit,
                         const uint64_t *ann_off, const m3tsz_annotation_entry *ann_entries,
                         const uint8_t *ann_bytes, uint8_t *target, int8_t *result, RouteTouched *touched,
                         uint32_t *n_touched) {
  static uint32_t tile[7 * ENC_STRIDE];
  RouteParams p;
  memset(&p, 0, sizeof(p));
  p.state = state;
  p.n_series = 1;
  p.slot_words = slot_words;
  p.pool_state = pool;
  p.pool_capacity = pool_capacity;
  p.pool_slot_words = pool_slot_words;
  p.pool_count = pool_count;
  p.table = table;
  p.n_encoders = K;
  p.default_unit = 1;
  p.ts = ts;
  p.val = val;
  p.points_stride = n;
  p.unit = unit;
  p.units = units;
  p.ann_series_off = ann_off;
  p.ann_entries = ann_entries;
  p.ann_bytes = ann_bytes;
  p.target = target;
  p.result = result;
  int32_t status = -1;
  p.status = &status;
  p.touched = touched;
  p.n_touched = n_touched;
  if (int_opt)
    route_series<true>(p, 0, tile, 0);
  else
    route_series<false>(p, 0, tile, 0);
  return status;
}
"""


@pytest.fixture(scope="module")
def dev():
    enc, kh = source_text("m3tsz_encode.cu"), source_text("m3tsz_kernels.h")
    parts = [constants(enc, "ENC_GUARD"), cut(kh, r"struct RouteTouched(?= \{)"), cut(kh, r"struct RouteParams(?= \{)"),
             cut(enc, r"struct RouteEnc(?= \{)")]
    for name in ("route_enc_load", "route_at", "route_last_value", "route_series"):
        parts.append(cut(enc, fn(name)))
    lib = build_dev_append("dev_route_host", "\n".join(parts), ROUTE_DRIVER)
    vp = C.c_void_p
    lib.dev_route.restype = C.c_int
    lib.dev_route.argtypes = [C.c_int, vp, C.c_uint64, vp, C.c_uint64, C.c_uint64, vp, vp, C.c_int, vp, vp,
                              C.c_uint64, vp, C.c_int, vp, vp, vp, vp, vp, vp, vp]
    return lib


class HostBucket:
    """One bucket as the device keeps it: encoder 0's state and slot, a pool of records, the counter and the table."""

    def __init__(self, dev, start, int_opt, K, pool_records=16, slot_bytes=1 << 14):
        self.dev, self.int_opt, self.K = dev, int_opt, K
        self.state = np.zeros(16, dtype=np.uint64)
        self.slot = np.zeros(slot_bytes, dtype=np.uint8)
        self.pool = np.zeros((64, 16), dtype=np.uint64)
        self.pool_slots = np.zeros((64, slot_bytes), dtype=np.uint8)
        self.pool_records = pool_records
        self.count = np.zeros(1, dtype=np.uint32)
        self.table = np.full(max(1, K - 1), -1, dtype=np.int32)
        dev.dev_reset(self.state.ctypes.data, int(start), O.UNIT_S, int(int_opt))

    def _encoder(self, i):
        if i == 0:
            return self.state, self.slot
        r = int(self.table[i - 1])
        return self.pool[r], self.pool_slots[r]

    def write(self, call, units=False):
        n = len(call)
        if n == 0:
            return np.zeros(0, np.int8), 0
        ts = np.array([c[0] for c in call], dtype=np.int64)
        vals = np.array([c[1] for c in call], dtype=np.float64)
        un = np.array([c[2] for c in call], dtype=np.uint8)
        anns = [c[3] for c in call]
        ents = np.zeros((max(1, n), 2), dtype=np.uint64)  # m3tsz_annotation_entry: (dp_index | length << 32, off)
        blob, k = b"", 0
        for j, a in enumerate(anns):
            if a:
                ents[k, 0] = j | (len(a) << 32)
                ents[k, 1] = len(blob)
                blob += a
                k += 1
        ann_off = np.array([0, k], dtype=np.uint64)
        ab = np.frombuffer(blob + b"\0", dtype=np.uint8).copy()
        target = np.zeros(n, dtype=np.uint8)
        result = np.zeros(n, dtype=np.int8)
        touched = np.zeros((64, 4), dtype=np.uint32)
        n_touched = np.zeros(1, dtype=np.uint32)
        slot_words = self.slot.size // 4
        status = self.dev.dev_route(int(self.int_opt), self.state.ctypes.data, slot_words, self.pool.ctypes.data,
                                    self.pool_records, slot_words, self.count.ctypes.data, self.table.ctypes.data,
                                    self.K, ts.ctypes.data, vals.ctypes.data, n, un.ctypes.data if units else None,
                                    O.UNIT_S, ann_off.ctypes.data, ents.ctypes.data, ab.ctypes.data,
                                    target.ctypes.data, result.ctypes.data, touched.ctypes.data, n_touched.ctypes.data)
        listed = sorted(int(e) for e in touched[: n_touched[0], 2])
        assert listed == sorted(set(int(t) for t in target if 0 < t < 255)), "touched records"
        # each encoder's share, through the append lane
        for i in sorted(set(int(t) for t in target if t != 255)):
            sel = np.nonzero(target == i)[0]
            st, slot = self._encoder(i)
            a = [anns[j] for j in sel]
            off = np.zeros(len(sel), dtype=np.uint32)
            ln = np.zeros(len(sel), dtype=np.uint32)
            b = b""
            for q, x in enumerate(a):
                off[q], ln[q] = len(b), len(x)
                b += x
            bb = np.frombuffer(b + b"\0", dtype=np.uint8).copy()
            tsel, vsel, usel = ts[sel].copy(), vals[sel].copy(), un[sel].copy()
            err = C.c_int()
            got = self.dev.dev_append(st.ctypes.data, slot.ctypes.data, tsel.ctypes.data, vsel.ctypes.data,
                                      usel.ctypes.data if units else None, O.UNIT_S, len(sel), off.ctypes.data,
                                      ln.ctypes.data, bb.ctypes.data, int(self.int_opt), 1, C.byref(err))
            assert (got, err.value) == (len(sel), 0), "the append refused a routed datapoint"
        return result, status

    def open(self):
        return 1 + int((self.table[: self.K - 1] >= 0).sum()) if self.K > 1 else 1

    def snapshot(self, i):
        st, slot = self._encoder(i)
        slot = slot.copy()
        n = self.dev.dev_snapshot(st.ctypes.data, slot.ctypes.data)
        return slot[:n].tobytes()

    def public(self, i):
        st = self._encoder(i)[0]
        return int(st[1]), int(st[2].view(np.int64)), float(st[3:4].view(np.float64)[0]), int(st[4])


def _check(hb, model, what):
    assert hb.open() == len(model.encs), what
    for i, e in enumerate(model.encs):
        assert hb.snapshot(i) == (e.stream() or b""), (what, i)
        num, last_ts, last_val, cs = hb.public(i)
        assert num == e.num_encoded(), (what, i)
        if num:
            t, v, err = e.last_encoded()
            assert err == 0 and t == last_ts, (what, i)
            assert np.float64(v).view(np.uint64) == np.float64(last_val).view(np.uint64), (what, i)
            assert e.last_annotation_checksum()[0] == cs, (what, i)


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("K", [1, 2, 4, 12])
def test_route_matches_the_bucket_model(dev, int_opt, K):
    start = 1599955200 * SEC
    n_seq = 0
    for seed in range(150):
        units, anns = seed % 3 == 1, seed % 2 == 0
        calls = random_calls(1000 * K + seed + (7 if int_opt else 0), start, 14, 6, int_opt, units=units, anns=anns)
        hb = HostBucket(dev, start, int_opt, K, pool_records=64)
        model = Bucket(start, int_opt, K)
        for c, call in enumerate(calls):
            res, status = hb.write(call, units=units)
            assert status == 0, (seed, c)
            exp = [model.write(*dp) for dp in call]
            assert list(res) == exp, (seed, c, call)
            _check(hb, model, (seed, c))
        n_seq += 1
    assert n_seq == 150


@pytest.mark.parametrize("int_opt", [True, False])
def test_route_same_call_upserts_and_duplicates(dev, int_opt):
    """equality against a datapoint written earlier in the same call: LastEncoded from the encoder's own value step
    (the scaled int in int mode, 0 without it: (t, 1.5) twice is then an upsert)"""
    start = 1599955200 * SEC
    t = start + 10 * SEC
    cases = [
        [(t, 1.5, 1, b""), (t, 1.5, 1, b"")],
        [(t, 2.0, 1, b""), (t, 2.0, 1, b""), (t, 3.0, 1, b""), (t, 3.0, 1, b""), (t, 2.0, 1, b"")],
        [(t, 1.25, 1, b"a"), (t, 1.25, 1, b"a"), (t, 1.25, 1, b""), (t, 1.25, 1, b"a")],
        [(t, 7.0, 1, b""), (t + SEC, 8.0, 1, b""), (t, 7.0, 1, b""), (t, 9.0, 1, b""), (t + SEC, 8.0, 1, b"")],
        [(0, 1.0, 1, b""), (t, 1.0, 1, b""), (0, 1.0, 1, b"")],
        [(-5, 1.0, 1, b""), (t, 2.0, 1, b""), (-5, 1.0, 1, b"")],
        [(t, float("nan"), 1, b""), (t, float("nan"), 1, b"")],
        [(t, 0.1, 1, b""), (t, 0.1, 1, b""), (t, 1e300, 1, b""), (t, 1e300, 1, b"")],
    ]
    for K in (1, 2, 3, 12):
        for k, call in enumerate(cases):
            hb = HostBucket(dev, start, int_opt, K)
            model = Bucket(start, int_opt, K)
            for split in ([call], [call[:1], call[1:]], [[dp] for dp in call]):
                hb = HostBucket(dev, start, int_opt, K)
                model = Bucket(start, int_opt, K)
                for part in split:
                    res, status = hb.write(part)
                    assert status == 0
                    assert list(res) == [model.write(*dp) for dp in part], (K, k, split)
                    _check(hb, model, (K, k))


@pytest.mark.parametrize("int_opt", [True, False])
def test_route_capacity_stops_the_series_and_resending_gives_the_unstopped_result(dev, int_opt):
    """an exhausted pool stops the series at the datapoint that needs a record: it and every later datapoint of the
    call get CAPACITY and nothing of them is written; with more records, sending exactly those again gives what one
    unstopped call gives"""
    start = 1599955200 * SEC
    for seed in range(60):
        calls = random_calls(seed + 555, start, 10, 8, int_opt, anns=seed % 2 == 0, rare=False)
        hb = HostBucket(dev, start, int_opt, 6, pool_records=1)
        model = Bucket(start, int_opt, 6)
        stopped = 0
        for c, call in enumerate(calls):
            res, status = hb.write(call)
            if status == ERR_CAPACITY:
                j = int(np.argmax(res == ERR_CAPACITY))
                assert (res[j:] == ERR_CAPACITY).all()
                exp = [model.write(*dp) for dp in call[:j]]
                assert list(res[:j]) == exp
                _check(hb, model, (seed, c, "stopped"))
                hb.pool_records = 64  # grow the pool, send the rest again
                res2, status2 = hb.write(call[j:])
                assert status2 == 0
                assert list(res2) == [model.write(*dp) for dp in call[j:]]
                hb.pool_records = int(hb.count[0]) + 1
                stopped += 1
            else:
                assert status == 0
                assert list(res) == [model.write(*dp) for dp in call]
            _check(hb, model, (seed, c))
    assert stopped > 0
