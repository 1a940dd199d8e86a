"""The composed oracle of m3tsz_aggregate_tiles_rollup_annotated (rollup_ann_oracle_lib) on the CPU: against the plain
rollup's oracle when no source is annotated, against the annotated element for one-member groups without
discard_nan, and against a restatement of its annotation path written from the Go source (the source element's
flush with cState.annotation, generic_elem.go:933-936; AddUnique passing metric.Annotation, :278-281; Gauge / Counter
Update's MaybeReplaceAnnotation, aggregation/common.go:49-61) over tests/indep_m3tsz.py, across 1 / 2 / 5-call splits
(the element's values come from the same element oracle; see restated_call).  Also
the annotated forward stage's reference conversion and 2^27 check and the fold's annotation step, compiled for the
host from the .cu source text."""
import ctypes as C
import math

import numpy as np
import pytest

import agg_oracle_lib as A
import ann_oracle_lib as N
import elem_oracle_lib as E
import indep_m3tsz as I
import oracle_lib as O
import rollup_ann_oracle_lib as RA
import rollup_oracle_lib as R
import xf_oracle_lib as X
from host_build import compile, constants, cut, fn, source_text
from test_independent_rollup import fold_counter, fold_gauge

SEC = 10 ** 9
STEP = 60 * SEC
R0 = 1_700_000_040 * SEC
START = R0 - 10 * STEP
N_WIN = 12
POOL = [b"a", b"bb", bytes([0x08, 0x01, 0x10, 0x01]), bytes(range(70))]
# (metric, source type, pre-ops, rollup types, post-ops)
PIPES = [(A.METRIC_COUNTER, A.AGG_SUM, [3], [7], [4]), (A.METRIC_GAUGE, A.AGG_LAST, [], [2, 3, 7], []),
         (A.METRIC_GAUGE, A.AGG_MEAN, [1, 2], [1, 4, 6, 8, 9], [4, 5]),
         (A.METRIC_COUNTER, A.AGG_MAX, [5], [2, 3, 9], [3])]


def source(rng, annotated=True, nan=True):
    n = int(rng.integers(1, 60))
    t = R0 - STEP + np.cumsum(rng.integers(1, 40, n)) * SEC
    enc = O.Encoder(START, True)
    for i in range(n):
        v = math.nan if nan and rng.random() < 0.08 else float(rng.integers(-50, 500))
        a = POOL[int(rng.integers(0, len(POOL)))] if annotated and rng.random() < 0.25 else b""
        assert enc.encode(int(t[i]), v, O.UNIT_S, a) == 0
    return enc.stream() or b""


def groups(rng, S, G):
    lists = [list(rng.integers(0, S, int(rng.integers(0, 6)))) for _ in range(G)]
    off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
    return off, np.array([m for x in lists for m in x], dtype=np.int32)


def test_without_annotations_is_the_plain_rollup():
    rng = np.random.default_rng(1)
    streams = [source(rng, annotated=False) for _ in range(14)]
    off, mem = groups(rng, 14, 9)
    for metric, src, pre, types, post in PIPES:
        for discard in (True, False):
            a = RA.aggregate_tiles_rollup_annotated(RA.decode_sources(streams, True, False), True, R0, STEP, N_WIN,
                                                    metric, src, pre, off, mem, types, post, discard,
                                                    np.zeros(14, X.XF_STATE_DTYPE), np.zeros(9, E.ELEM_STATE_DTYPE))
            b = R.aggregate_tiles_rollup(R.decode_sources(streams, True, False), True, R0, STEP, N_WIN, metric, src,
                                         pre, off, mem, types, post, discard, np.zeros(14, X.XF_STATE_DTYPE),
                                         np.zeros(9, E.ELEM_STATE_DTYPE))
            assert a == b


def test_one_member_groups_are_the_annotated_element():
    """Last -> Rollup [Last], one member, no pre-ops, no discard: the local element with annotations"""
    rng = np.random.default_rng(2)
    streams = [source(rng) for _ in range(10)]
    off, mem = np.arange(11, dtype=np.int64), np.arange(10, dtype=np.int32)
    for post in ([], [4], [3, 5]):
        rows, _ = RA.aggregate_tiles_rollup_annotated(RA.decode_sources(streams, True, False), True, R0, STEP, N_WIN,
                                                      A.METRIC_GAUGE, A.AGG_LAST, [], off, mem, [A.AGG_LAST], post,
                                                      False, np.zeros(10, X.XF_STATE_DTYPE),
                                                      np.zeros(10, E.ELEM_STATE_DTYPE))
        for s in range(10):
            want, counts, err = N.aggregate_tiles_annotated_series(streams[s], True, R0, STEP, N_WIN, A.METRIC_GAUGE,
                                                                   [A.AGG_LAST], post, False, E.new_element_state())
            assert err == 0 and rows[0][s] == (0, want[0], counts[0]), (post, s)


def restated_call(streams, metric, src, pre, off, mem, types, post, discard, xs, gs, w0, n_win):
    """the whole call, with the annotation path restated and the value path partly shared.  Restated: the decoder
    and encoder (indep_m3tsz), each source window's last annotation, the discard of a NaN forward, the fold's
    arithmetic (test_independent_rollup's fold_gauge / fold_counter) and the group annotation (MaybeReplaceAnnotation
    in listed order), and which datapoints of a row carry it.  Shared with the composed oracle: the window values
    (agg_oracle_lib), the pre-op chain (xf_oracle_lib) and the rollup element with its post-ops (elem_oracle_lib),
    which tests of their own check against the reference's goldens."""
    r0 = R0 + w0 * STEP
    fwd, wann, new = [], [], []
    for s, data in enumerate(streams):
        dps = I.decode(data, True)
        ts = np.array([d[0] for d in dps], dtype=np.int64)
        vals = np.array([d[1] for d in dps], dtype=np.uint64).view(np.float64)
        ann = {}
        for t, _, _, a in dps:  # the source element's window keeps the last non-empty annotation it was given
            if a and r0 <= t < r0 + n_win * STEP:
                ann[(t - r0) // STEP] = a
        st = xs[s: s + 1].copy()
        wt, wv = A.aggregate_tiles_series_ex(ts, vals, r0, STEP, n_win, metric, src)
        f = {}
        for t, v in zip(wt.tolist(), wv.tolist()):
            to, vo = X.transform_series(pre, False, STEP, st, [t], [v])
            if not (discard and math.isnan(float(vo[0]))):
                f[(t - r0) // STEP - 1] = float(vo[0])
        fwd.append(f)
        wann.append(ann)
        new.append(st[0])
    rows = []
    for g in range(len(off) - 1):
        ms = [int(m) for m in mem[off[g]: off[g + 1]]]
        wt, wv, wa = [], [], []
        for w in range(n_win):
            got = [m for m in ms if w in fwd[m]]
            if not got:
                continue
            vs = [fwd[m][w] for m in got]
            a = b""
            for m in got:  # MaybeReplaceAnnotation: a non-empty annotation replaces, an empty one keeps
                if wann[m].get(w):
                    a = wann[m][w]
            wt.append(r0 + (w + 1) * STEP)
            wa.append(a)
            if metric == A.METRIC_COUNTER:
                s_, c, mn, mx, sq = fold_counter(vs)
                wv.append([A.counter_value_of(t_, s_, c, mn, mx, sq) for t_ in types])
            else:
                s_, c, mn, mx, last, sq = fold_gauge(vs)
                wv.append([A.gauge_value_of_ex(t_, s_, c, mn, mx, last, sq) for t_ in types])
        st = gs[g: g + 1].copy()
        res = E.element_series(post, discard, STEP, len(types), st, np.array(wt, dtype=np.int64),
                               np.array(wv, dtype=np.float64).reshape(len(wt), len(types)))
        gs[g] = st[0]
        half = max(STEP // 2, 1)
        row = []
        for to, vo in res:
            dps, i = [], 0
            for t, a in zip(wt, wa):  # every datapoint of the window (a Reset's second one too) carries it
                while i < len(to) and (int(to[i]) == t or (5 in post and int(to[i]) == t + half)):
                    dps.append((int(to[i]), float(vo[i]), 1, a))
                    i += 1
            assert i == len(to)
            row.append(I.encode(r0, dps, True) if dps else b"")
        rows.append(row)
    for s in range(len(streams)):
        xs[s] = new[s]
    return rows


def test_restatement_across_splits():
    rng = np.random.default_rng(3)
    for metric, src, pre, types, post in PIPES:
        streams = [source(rng) for _ in range(12)]
        decoded = RA.decode_sources(streams, True, False)
        off, mem = groups(rng, 12, 7)
        for discard in (True, False):
            for edges in ([0, 12], [0, 5, 12], [0, 2, 3, 7, 11, 12]):
                xs1, gs1 = np.zeros(12, X.XF_STATE_DTYPE), np.zeros(7, E.ELEM_STATE_DTYPE)
                xs2, gs2 = np.zeros(12, X.XF_STATE_DTYPE), np.zeros(7, E.ELEM_STATE_DTYPE)
                for a, b in zip(edges[:-1], edges[1:]):
                    want, src_st = RA.aggregate_tiles_rollup_annotated(decoded, True, R0 + a * STEP, STEP, b - a,
                                                                       metric, src, pre, off, mem, types, post,
                                                                       discard, xs1, gs1)
                    got = restated_call(streams, metric, src, pre, off, mem, types, post, discard, xs2, gs2, a, b - a)
                    assert src_st == [0] * 12
                    assert [[want[j][g][1] for j in range(len(types))] for g in range(7)] == got
                    assert xs1.tobytes() == xs2.tobytes() and gs1.tobytes() == gs2.tobytes()


def test_later_forward_without_annotation_keeps_the_earlier():
    """a window whose later members forward no annotation keeps the earlier member's"""
    streams = []
    for v, a in ((1.0, b"first"), (2.0, b""), (3.0, b"")):
        enc = O.Encoder(START, True)
        assert enc.encode(R0 + 5 * SEC, v, O.UNIT_S, a) == 0
        streams.append(enc.stream())
    rows, _ = RA.aggregate_tiles_rollup_annotated(RA.decode_sources(streams, True, False), True, R0, STEP, 1,
                                                  A.METRIC_GAUGE, A.AGG_LAST, [], np.array([0, 3]),
                                                  np.array([0, 1, 2], dtype=np.int32), [A.AGG_SUM], [], True,
                                                  np.zeros(3, X.XF_STATE_DTYPE), np.zeros(1, E.ELEM_STATE_DTYPE))
    dps = I.decode(rows[0][0][1], True)
    assert [(d[0], d[3]) for d in dps] == [(R0 + STEP, b"first")]


DRIVER = r"""
extern "C" int dev_ann_ref(uint64_t ref, const uint64_t *src_off, uint64_t s, uint64_t *out) {
  const bool ok = rollup_ann_ref(ref, src_off, s);
  *out = ref;
  return ok ? 1 : 0;
}
extern "C" uint64_t dev_ann_fold(const uint32_t *ann_bits, const uint64_t *refs, size_t n, uint32_t lane) {
  uint64_t g = 0;
  for (size_t i = 0; i < n; i++) rollup_ann_add(g, ann_bits[i], lane, refs + i);
  return g;
}
"""


@pytest.fixture(scope="module")
def dev():
    enc = source_text("m3tsz_encode.cu")
    body = "\n".join([constants(source_text("m3tsz_kernels.h"), "kBlockAnnLenBits"), cut(enc, fn("rollup_ann_ref")),
                      cut(enc, fn("rollup_ann_add"))])
    lib = compile("dev_rollup_ann_host", body, DRIVER)
    vp = C.c_void_p
    lib.dev_ann_ref.restype = C.c_int
    lib.dev_ann_ref.argtypes = [C.c_uint64, vp, C.c_uint64, vp]
    lib.dev_ann_fold.restype = C.c_uint64
    lib.dev_ann_fold.argtypes = [vp, vp, C.c_size_t, C.c_uint32]
    return lib


def _ref(lib, ref, offs, s):
    o = np.asarray(offs, dtype=np.uint64)
    out = np.zeros(1, dtype=np.uint64)
    ok = lib.dev_ann_ref(ref, o.ctypes.data_as(C.c_void_p) if len(o) else None, s, out.ctypes.data_as(C.c_void_p))
    return bool(ok), int(out[0])


def test_device_reference_conversion(dev):
    offs = [0, 48, (1 << 33) + 16]
    # (bit offset in the stream) << 32 | length -> (bit offset in the batch) << 27 | length
    assert _ref(dev, (77 << 32) | 4, offs, 1) == (True, ((48 * 8 + 77) << 27) | 4)
    assert _ref(dev, (5 << 32) | 1, offs, 2) == (True, ((((1 << 33) + 16) * 8 + 5) << 27) | 1)
    assert _ref(dev, 0, offs, 1) == (True, 0)  # no annotation
    assert _ref(dev, (9 << 32) | ((1 << 27) - 1), offs, 0) == (True, (9 << 27) | ((1 << 27) - 1))
    assert _ref(dev, (9 << 32) | (1 << 27), offs, 0)[0] is False  # 2^27 bytes: STREAM_TOO_LARGE
    assert _ref(dev, (9 << 32) | ((1 << 28) - 1), offs, 0)[0] is False
    # over source blocks the reference is batch-addressed already
    assert _ref(dev, (123 << 27) | 9, [], 0) == (True, (123 << 27) | 9)


def test_device_fold_step(dev):
    rng = np.random.default_rng(7)
    for _ in range(2000):
        n = int(rng.integers(0, 8))
        lane = int(rng.integers(0, 32))
        bits = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
        refs = rng.integers(1, 1 << 62, n, dtype=np.uint64)
        want = 0
        for b, r in zip(bits.tolist(), refs.tolist()):
            if (b >> lane) & 1:
                want = r
        got = dev.dev_ann_fold(bits.ctypes.data_as(C.c_void_p), refs.ctypes.data_as(C.c_void_p), n, lane)
        assert got == want
