"""The annotation a tile carries (m3tsz_aggregate_tiles_annotated), on the CPU: the window rule of the oracle
(tests/ann_oracle.c m3o_window_annotations, composed in ann_oracle_lib.aggregate_tiles_annotated_series) reproduces
tests/golden/m3tsz_tile_annotation_goldens.json, and a second statement in pure Python -- the rule written from
aggregation/common.go:47-61 and generic_elem.go:567 over tests/indep_m3tsz.py's decoder and encoder, the element of
test_independent_element.py -- writes the same bytes as the oracle on random annotated streams."""
import json
import os

import numpy as np
import pytest

import agg_oracle_lib as A
import ann_oracle_lib as N
import elem_oracle_lib as E
import indep_m3tsz as I
import oracle_lib as O
from test_independent_element import MultiElement, random_element_pipeline, random_types

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "m3tsz_tile_annotation_goldens.json")
SEC = 10 ** 9
# annotation.Payload{OpenMetricsFamilyType: COUNTER, OpenMetricsHandleValueResets: true} (fields 1 and 2, varints)
PROM_COUNTER_PAYLOAD = bytes([0x08, 0x01, 0x10, 0x01])


def _goldens():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


def _encode_source(start_ns, dps, int_optimized=True):
    """the reference encoder over (t, value, annotation) -> stream bytes"""
    enc = O.Encoder(int(start_ns), int_optimized)
    for t, v, a in dps:
        assert enc.encode(int(t), float(v), O.UNIT_S, a) == 0
    return enc.stream() or b""


def _first_annotations(tile, int_optimized=True):
    """(t, annotation Current() reports) of every datapoint of a tile stream"""
    out, err = O.decode_all(tile, int_optimized)
    assert err == 0
    return [(t, a) for t, _, _, a in out]


@pytest.mark.parametrize("case", _goldens(), ids=lambda c: c["name"])
def test_goldens_window_rule(case):
    ts = np.array([d[0] for d in case["datapoints"]], dtype=np.int64)
    anns = [bytes.fromhex(d[2]) for d in case["datapoints"]]
    ids = [i if a else -1 for i, a in enumerate(anns)]
    win = N.window_annotations(ts, ids, case["start_ns"], case["step_ns"], case["n_windows"])
    assert [anns[i] if i >= 0 else b"" for i in win] == [bytes.fromhex(a) for a in case["want_windows"]]
    assert _indep_window_annotations([(int(t), a) for t, a in zip(ts, anns)], case["start_ns"], case["step_ns"],
                                     case["n_windows"]) == [bytes.fromhex(a) for a in case["want_windows"]]


@pytest.mark.parametrize("case", _goldens(), ids=lambda c: c["name"])
def test_goldens_through_the_tile_path(case):
    """the goldens' datapoints encoded with their annotations, then the oracle's tile path: the first datapoint of
    each window's tile reports the window's annotation, later ones none"""
    dps = [(d[0], d[1], bytes.fromhex(d[2])) for d in case["datapoints"]]
    src = _encode_source(case["start_ns"] - 6 * SEC, dps)
    types = [7] if case["metric_type"] == A.METRIC_COUNTER else [1, 7]  # Sum; Last and Sum
    st = E.new_element_state()
    streams, counts, err = N.aggregate_tiles_annotated_series(src, True, case["start_ns"], case["step_ns"],
                                                              case["n_windows"], case["metric_type"], types, [], True,
                                                              st)
    assert err == 0
    want = [bytes.fromhex(a) for a in case["want_windows"]]
    for j in range(len(types)):
        got = _first_annotations(streams[j])
        assert len(got) == counts[j] == case["n_windows"]
        last = b""
        for w, (t, a) in enumerate(got):
            assert t == case["start_ns"] + (w + 1) * case["step_ns"]
            # the encoder writes a window's annotation only when it differs from the last one written
            assert a == (want[w] if want[w] and want[w] != last else b""), (w, a)
            last = want[w] or last


def _indep_window_annotations(dps, start_ns, step_ns, n_windows):
    """consumeState.annotation of each window: MaybeReplaceAnnotation(empty, agg.Annotation()), where every Update
    of the window's aggregation replaced it with a non-empty annotation"""
    win = [b""] * n_windows
    for t, a in dps:
        if t < start_ns or not a:
            continue
        w = (t - start_ns) // step_ns
        if w < n_windows:
            win[w] = a
    return win


def indep_tiles_annotated(src, int_optimized, start_ns, step_ns, n_windows, metric, types, ops, discard):
    """the second statement: decode (indep_m3tsz), the window rule, the element over the aggregation oracle's
    window values (test_independent_element.MultiElement), encode (indep_m3tsz) with each window's annotation"""
    dps = I.decode(src, int_optimized)
    ts = np.array([d[0] for d in dps], dtype=np.int64)
    vals = np.array([d[1] for d in dps], dtype=np.uint64).view(np.float64)
    win = _indep_window_annotations([(d[0], d[3]) for d in dps], start_ns, step_ns, n_windows)
    wt, wv = E.element_windows(ts, vals, start_ns, step_ns, n_windows, metric, types)
    e = MultiElement(len(ops), len(types))
    rows = [[] for _ in types]
    for i, t in enumerate(wt.tolist()):
        a = win[(t - start_ns) // step_ns - 1]
        for j, out in enumerate(e.flush(ops, step_ns, discard, t, wv[i].view(np.uint64).tolist())):
            rows[j] += [(tt, float(np.uint64(v).view(np.float64)), 1, a) for tt, v in out]
    return [I.encode(start_ns, r, int_optimized) for r in rows], e.state_record()


def random_annotated_source(rng, start_ns, step_ns, n_windows, n):
    """a sorted stream with a few out-of-order datapoints, some outside the range, and annotations of 1..300 bytes
    at random datapoints (some repeated)"""
    span = (n_windows + 2) * step_ns
    ts = np.sort(rng.integers(start_ns - step_ns, start_ns - step_ns + span, size=n)).astype(np.int64)
    ts = np.unique(ts)
    order = list(ts)
    for _ in range(int(rng.integers(0, 3))):  # move a datapoint later in the stream (out of order)
        if len(order) > 3:
            i = int(rng.integers(0, len(order) - 2))
            order.insert(len(order) - 1, order.pop(i))
    pool = [bytes(rng.integers(0, 256, size=int(rng.choice([1, 2, 5, 63, 64, 200, 300]))).astype(np.uint8))
            for _ in range(4)]
    dps = []
    for t in order:
        a = pool[int(rng.integers(0, len(pool)))] if rng.random() < 0.3 else b""
        dps.append((int(t), float(rng.integers(-50, 500)) / (1 if rng.random() < 0.7 else 8), a))
    return dps


def test_random_annotated_tiles_match_oracle():
    rng = np.random.default_rng(20261017)
    step = 60 * SEC
    start = 1_700_000_040 * SEC
    for it in range(120):
        int_opt = bool(it % 2)
        nw = int(rng.integers(1, 12))
        dps = random_annotated_source(rng, start, step, nw, int(rng.integers(1, 60)))
        src = _encode_source(start - 2 * step, dps, int_opt)
        metric = A.METRIC_GAUGE if rng.random() < 0.5 else A.METRIC_COUNTER
        types = random_types(rng, metric)
        ops = random_element_pipeline(rng) if rng.random() < 0.6 else []
        discard = bool(rng.random() < 0.5)
        st = E.new_element_state()
        got, _, err = N.aggregate_tiles_annotated_series(src, int_opt, start, step, nw, metric, types, ops, discard,
                                                         st)
        assert err == 0
        exp, rec = indep_tiles_annotated(src, int_opt, start, step, nw, metric, types, ops, discard)
        assert got == exp, (it, types, ops, discard)
        assert rec.tobytes() == st.tobytes(), it


def test_prometheus_counter_payload_on_the_first_tile():
    """a Prometheus counter's series: the Payload on datapoint 0 only; the first tile reports it, as the query's
    Prometheus conversion reads FirstAnnotation()"""
    start = 1_700_000_000 * SEC
    dps = [(start + (i + 1) * 10 * SEC, float(i), PROM_COUNTER_PAYLOAD if i == 0 else b"") for i in range(60)]
    src = _encode_source(start, dps)
    st = E.new_element_state()
    streams, counts, err = N.aggregate_tiles_annotated_series(src, True, start, 60 * SEC, 10, A.METRIC_COUNTER, [7],
                                                              [], True, st)
    assert err == 0 and counts == [10]
    got = _first_annotations(streams[0])
    assert got[0][1] == PROM_COUNTER_PAYLOAD and all(a == b"" for _, a in got[1:])
