"""The tile path of m3tsz_aggregate_tiles_blocks for one series, composed from the pinned oracles: the reference
iterator over each source block (ann_oracle_lib.decode_annotated), the blocks' datapoints concatenated in the listed
order, the window rule (ann_oracle_lib.window_annotations), the element (elem_oracle_lib) and the reference encoder
writing every datapoint of a window with the window's annotation.  Test infrastructure only."""
import numpy as np

import ann_oracle_lib as N
import elem_oracle_lib as E
import oracle_lib as O

TRANSFORM_RESET = 5


def decode_blocks(blocks, int_optimized, default_unit=O.UNIT_S):
    """each block decoded on its own, concatenated: (ts, values, annotation per datapoint, err).  An empty block adds
    nothing; the first block that fails gives the error."""
    ts, vals, anns = [], [], []
    for b in blocks:
        if len(b) == 0:
            continue
        t, v, a, err = N.decode_annotated(b, int_optimized, default_unit)
        if err:
            return np.zeros(0, np.int64), np.zeros(0, np.float64), [], err
        ts.append(t)
        vals.append(v)
        anns += a
    if not ts:
        return np.zeros(0, np.int64), np.zeros(0, np.float64), [], 0
    return np.concatenate(ts), np.concatenate(vals), anns, 0


def tiles_from_datapoints(ts, vals, anns, int_optimized, start_ns, step_ns, n_windows, metric_type, agg_types, ops,
                          discard_nan, state, out_unit=O.UNIT_S, default_unit=O.UNIT_S):
    """the element's tiles over one datapoint sequence; `state` is updated in place -> (bytes per type, datapoints
    per type).  anns[i] is datapoint i's annotation (b"" for none)."""
    k = len(agg_types)
    ids = np.array([i if a else -1 for i, a in enumerate(anns)], dtype=np.int64)
    win = N.window_annotations(ts, ids, start_ns, step_ns, n_windows)
    wt, wv = E.element_windows(ts, vals, start_ns, step_ns, n_windows, metric_type, agg_types)
    res = E.element_series(ops, discard_nan, step_ns, k, state, wt, wv)
    reset = TRANSFORM_RESET in [int(o) for o in ops]
    rw = int(max(float(int(step_ns) // 2), 1.0))
    streams, counts = [], []
    for j in range(k):
        to, vo = res[j]
        enc = O.Encoder(int(start_ns), int_optimized, default_unit)
        i = 0
        for t in wt.tolist():  # a type writes a window's datapoint, then its Reset datapoint, or neither
            if i < len(to) and int(to[i]) == t:
                w = (t - int(start_ns)) // int(step_ns) - 1
                a = anns[win[w]] if win[w] >= 0 else b""
                for _ in range(2 if (reset and t + rw != 0) else 1):
                    rc = enc.encode(int(to[i]), float(vo[i]), out_unit, a)
                    assert rc == 0, rc
                    i += 1
        assert i == len(to)
        streams.append(enc.stream() or b"")
        counts.append(len(to))
    return streams, counts


def aggregate_tiles_blocks_series(blocks, int_optimized, start_ns, step_ns, n_windows, metric_type, agg_types, ops,
                                  discard_nan, state, annotations, out_unit=O.UNIT_S, default_unit=O.UNIT_S):
    """m3tsz_aggregate_tiles_blocks for one series given as its blocks' streams; `state` is updated in place unless a
    block fails -> (bytes per type, datapoints per type, error)"""
    ts, vals, anns, err = decode_blocks(blocks, int_optimized, default_unit)
    k = len(agg_types)
    if err:
        return [b""] * k, [0] * k, err
    if not annotations:
        anns = [b""] * len(ts)
    streams, counts = tiles_from_datapoints(ts, vals, anns, int_optimized, start_ns, step_ns, n_windows, metric_type,
                                            agg_types, ops, discard_nan, state, out_unit, default_unit)
    return streams, counts, 0


def concat_stream(blocks, int_optimized, start_ns, default_unit=O.UNIT_S):
    """one stream that encodes the blocks' datapoints, concatenated, with their annotations (the reference encoder
    writes an annotation only when it differs from the last one written)"""
    ts, vals, anns, err = decode_blocks(blocks, int_optimized, default_unit)
    assert err == 0
    enc = O.Encoder(int(start_ns), int_optimized, default_unit)
    for t, v, a in zip(ts.tolist(), vals.tolist(), anns):
        assert enc.encode(int(t), float(v), O.UNIT_S, a) == 0
    return enc.stream() or b""
