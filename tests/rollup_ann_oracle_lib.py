"""m3tsz_aggregate_tiles_rollup_annotated composed from the pinned oracles: the reference iterator over every source
(one stream, or its blocks concatenated: ann_oracle_lib / blocks_oracle_lib), the window-annotation rule
(tests/ann_oracle.c), the forward and fold of rollup_oracle_lib, the element oracle for the rollup element and the
reference encoder writing every datapoint of a group window with the group window's annotation.  The annotation
selection is this module's own: the last non-empty annotation, in listed member order, among the members whose value
for the window was forwarded.  Test infrastructure only."""
import numpy as np

import ann_oracle_lib as N
import blocks_oracle_lib as B
import elem_oracle_lib as E
import oracle_lib as O
import rollup_oracle_lib as R

TRANSFORM_RESET = 5


def decode_sources(sources, int_optimized, blocks):
    """each source's (ts, values, annotation per datapoint (b"" for none), err): sources[s] is one stream, or with
    blocks=True the list of its block streams"""
    out = []
    for src in sources:
        if blocks:
            out.append(B.decode_blocks(src, int_optimized))
        else:
            ts, vals, anns, err = N.decode_annotated(src, int_optimized)
            out.append((ts, vals, anns, err) if not err else (ts[:0], vals[:0], [], err))
    return out


def source_window_annotations(ts, anns, start_ns, step_ns, n_windows):
    """{window: annotation} of one source: the last datapoint of each window that carries one"""
    ids = np.array([i if a else -1 for i, a in enumerate(anns)], dtype=np.int64)
    win = N.window_annotations(ts, ids, start_ns, step_ns, n_windows)
    return {w: anns[int(win[w])] for w in range(n_windows) if win[w] >= 0}


def group_annotation(fwd, src_ann, members, w):
    """MaybeReplaceAnnotation over the members that forwarded window w, in listed order"""
    a = b""
    for m in members:
        if w in fwd[m] and src_ann[m].get(w, b""):
            a = src_ann[m][w]
    return a


def encode_rows(res, wt, anns, start_ns, step_ns, reset, int_optimized):
    """the rollup element's rows: each window's datapoints (its Reset datapoint too) with the window's annotation"""
    rw = int(max(float(int(step_ns) // 2), 1.0))
    out = []
    for to, vo in res:
        enc = O.Encoder(int(start_ns), int_optimized, O.UNIT_S)
        i = 0
        for t, a in zip(wt, anns):
            if i < len(to) and int(to[i]) == t:
                for _ in range(2 if (reset and t + rw != 0) else 1):
                    assert enc.encode(int(to[i]), float(vo[i]), O.UNIT_S, a) == 0
                    i += 1
        assert i == len(to)
        out.append((enc.stream() or b"", len(to)))
    return out


def aggregate_tiles_rollup_annotated(decoded, int_optimized, start_ns, step_ns, n_windows, metric_type, src_type,
                                     pre_ops, group_off, members, rollup_types, post_ops, discard_nan, src_state,
                                     group_state, saved_rows=None):
    """m3tsz_aggregate_tiles_rollup_annotated on decoded sources (decode_sources); the records as in
    rollup_oracle_lib.aggregate_tiles_rollup.  -> (rows [k][G] of (status, bytes, n_tiles), source statuses [S])"""
    S, G, k = len(decoded), len(group_off) - 1, len(rollup_types)
    discard = bool(discard_nan)
    fwd, src_ann, src_status, new_src = [], [], [], []
    for s, (ts, vals, anns, err) in enumerate(decoded):
        src_status.append(int(err))
        st = src_state[s: s + 1].copy()
        if err:
            fwd.append({})
            src_ann.append({})
        else:
            fwd.append(R.forward_series(ts, vals, start_ns, step_ns, n_windows, metric_type, src_type, pre_ops,
                                        discard, st))
            src_ann.append(source_window_annotations(ts, anns, start_ns, step_ns, n_windows))
        new_src.append(st[0])
    reset = TRANSFORM_RESET in [int(o) for o in post_ops]
    rows = [[None] * G for _ in range(k)]
    group_saved = [True] * G
    n_mem = len(members)
    for g in range(G):
        lo, hi = int(group_off[g]), int(group_off[g + 1])
        err = 0
        if lo > hi or hi > n_mem:
            err = R.ERR_INVALID_ARG
        else:
            for i in range(lo, hi):
                m = int(members[i])
                e = R.ERR_INVALID_ARG if m >= S else src_status[m]
                if e:
                    err = e
                    break
        if err:
            group_saved[g] = False
            for j in range(k):
                rows[j][g] = (err, b"", 0)
            continue
        mem = [int(members[i]) for i in range(lo, hi)]
        wt, wv, wa = [], [], []
        for w in range(n_windows):
            vs = [fwd[m][w] for m in mem if w in fwd[m]]
            if not vs:
                continue
            wt.append(int(start_ns) + (w + 1) * int(step_ns))
            wv.append([R.rollup_value_of(metric_type, a, vs) for a in rollup_types])
            wa.append(group_annotation(fwd, src_ann, mem, w))
        st = group_state[g: g + 1].copy()
        res = E.element_series(post_ops, discard, step_ns, k, st,
                               np.asarray(wt, dtype=np.int64), np.asarray(wv, dtype=np.float64).reshape(len(wt), k))
        for j, (b, n) in enumerate(encode_rows(res, wt, wa, start_ns, step_ns, reset, int_optimized)):
            rows[j][g] = (0, b, n)
        if saved_rows is not None and not saved_rows(g):
            group_saved[g] = False
            continue
        group_state[g] = st[0]
    blocked = set()
    for g in range(G):
        if not group_saved[g]:
            lo, hi = int(group_off[g]), min(int(group_off[g + 1]), n_mem)
            blocked.update(int(members[i]) for i in range(lo, hi))
    for s in range(S):
        if src_status[s] == 0 and s not in blocked:
            src_state[s] = new_src[s]
    return rows, src_status
