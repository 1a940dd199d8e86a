"""m3tsz_aggregate_tiles_rollup composed from the pinned oracles: the aggregation oracle's windows of every source
(agg_oracle_lib), each source's chain through the transformation oracle with its record (xf_oracle_lib), the fold of
every group window in listed order (tests/rollup_oracle.c -> tests/libm3tsz_rollup_oracle.so), the element oracle
for the rollup element with the post-ops and its record (elem_oracle_lib) and the reference encoder.  Test
infrastructure only; __graft_entry__.build() compiles the library, and build_c_oracle() rebuilds it when the
source is newer."""
import ctypes as C

import numpy as np

import agg_oracle_lib as A
import blocks_oracle_lib as B
import elem_oracle_lib as E
import oracle_lib as O
import xf_oracle_lib as X
from host_build import build_c_oracle

ERR_INVALID_ARG = 101  # M3TSZ_ERR_INVALID_ARG


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


_lib = None


def _rollup_lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build_c_oracle("rollup"))
        vp = C.c_void_p
        L.m3o_rollup_gauge.restype = None
        L.m3o_rollup_gauge.argtypes = [vp, C.c_size_t, vp, vp]
        L.m3o_rollup_counter.restype = None
        L.m3o_rollup_counter.argtypes = [vp, C.c_size_t, vp]
        _lib = L
    return _lib


def fold_gauge(values):
    """-> (sum, count, min, max, last, sum_sq) of one rollup window given its values in listed order"""
    v = np.ascontiguousarray(values, dtype=np.float64)
    o = np.zeros(5, dtype=np.float64)
    c = np.zeros(1, dtype=np.int64)
    _rollup_lib().m3o_rollup_gauge(_ptr(v), len(v), _ptr(o), _ptr(c))
    return o[0], int(c[0]), o[1], o[2], o[3], o[4]


def fold_counter(values):
    """-> (sum, count, min, max, sum_sq) int64 of one rollup window given its values in listed order"""
    v = np.ascontiguousarray(values, dtype=np.float64)
    o = np.zeros(5, dtype=np.int64)
    _rollup_lib().m3o_rollup_counter(_ptr(v), len(v), _ptr(o))
    return tuple(int(x) for x in o)


def rollup_value_of(metric_type, agg_type, values):
    """ValueOf(agg_type) of the rollup window that received `values` (listed order)"""
    if metric_type == A.METRIC_COUNTER:
        s, c, mn, mx, sq = fold_counter(values)
        return A.counter_value_of(agg_type, s, c, mn, mx, sq)
    s, c, mn, mx, last, sq = fold_gauge(values)
    return A.gauge_value_of_ex(agg_type, s, c, mn, mx, last, sq)


def forward_series(ts, vals, start_ns, step_ns, n_windows, metric_type, src_type, pre_ops, discard_nan, state):
    """the source element's forwarded values: {window index: value} for every non-empty window whose value through
    pre_ops is not discarded (a Reset op forwards nothing extra); `state` (xf_oracle_lib.new_transform_state()) is
    updated in place"""
    wt, wv = A.aggregate_tiles_series_ex(ts, vals, start_ns, step_ns, n_windows, metric_type, src_type)
    out = {}
    for t, v in zip(wt.tolist(), wv.tolist()):
        to, vo = X.transform_series(pre_ops, discard_nan, step_ns, state, [t], [v])
        if len(to):  # the window's own datapoint comes first
            assert int(to[0]) == t
            out[(t - int(start_ns)) // int(step_ns) - 1] = float(vo[0])
    return out


def decode_sources(sources, int_optimized, blocks):
    """each source's (ts, values, err): sources[s] is one stream, or with blocks=True the list of its block streams"""
    out = []
    for src in sources:
        if blocks:
            ts, vals, _, err = B.decode_blocks(src, int_optimized)
        else:
            ts, vals, n, err = O.decode_series(src, int_optimized, cap=8192)
            ts, vals = ts[:n], vals[:n]
        out.append((ts, vals, err))
    return out


def aggregate_tiles_rollup(decoded, int_optimized, start_ns, step_ns, n_windows, metric_type, src_type, pre_ops,
                           group_off, members, rollup_types, post_ops, discard_nan, src_state, group_state,
                           saved_rows=None):
    """m3tsz_aggregate_tiles_rollup on decoded sources (decode_sources).  src_state (XF_STATE_DTYPE [S]) and
    group_state (ELEM_STATE_DTYPE [G]) are updated in place by the record rules.  saved_rows(g) -> False marks a group
    whose rows the device could not write (CAPACITY): its record and its members' are not saved.
    -> (rows [k][G] of (status, bytes, n_tiles), source statuses [S])"""
    S, G, k = len(decoded), len(group_off) - 1, len(rollup_types)
    # DiscardNaNAggregatedValues drops a NaN in processValue whether or not the element has transformations
    # (generic_elem.go:892-894): on the source elements and on the rollup element alike
    discard = bool(discard_nan)
    fwd, src_status, new_src = [], [], []
    for s, (ts, vals, err) in enumerate(decoded):
        src_status.append(int(err))
        st = src_state[s: s + 1].copy()
        fwd.append({} if err else forward_series(ts, vals, start_ns, step_ns, n_windows, metric_type, src_type,
                                                 pre_ops, discard, st))
        new_src.append(st[0])
    rows = [[None] * G for _ in range(k)]
    group_saved = [True] * G
    n_mem = len(members)
    for g in range(G):
        lo, hi = int(group_off[g]), int(group_off[g + 1])
        err = 0
        if lo > hi or hi > n_mem:
            err = ERR_INVALID_ARG
        else:
            for i in range(lo, hi):
                m = int(members[i])
                e = ERR_INVALID_ARG if m >= S else src_status[m]
                if e:
                    err = e
                    break
        if err:
            group_saved[g] = False
            for j in range(k):
                rows[j][g] = (err, b"", 0)
            continue
        mem = [int(members[i]) for i in range(lo, hi)]
        wt, wv = [], []
        for w in range(n_windows):
            vs = [fwd[m][w] for m in mem if w in fwd[m]]
            if not vs:
                continue
            wt.append(int(start_ns) + (w + 1) * int(step_ns))
            wv.append([rollup_value_of(metric_type, a, vs) for a in rollup_types])
        st = group_state[g: g + 1].copy()
        res = E.element_series(post_ops, discard, step_ns, k, st,
                               np.asarray(wt, dtype=np.int64), np.asarray(wv, dtype=np.float64).reshape(len(wt), k))
        for j, (to, vo) in enumerate(res):
            b = O.encode_series(to, vo, start_ns, O.UNIT_S, int_optimized) if len(to) else b""
            rows[j][g] = (0, b, len(to))
        if saved_rows is not None and not saved_rows(g):
            group_saved[g] = False
            continue
        group_state[g] = st[0]
    # a source's record: it decoded and every group that lists it was saved (as far as the group's range names it)
    blocked = set()
    for g in range(G):
        if not group_saved[g]:
            lo, hi = int(group_off[g]), min(int(group_off[g + 1]), n_mem)
            blocked.update(int(members[i]) for i in range(lo, hi))
    for s in range(S):
        if src_status[s] == 0 and s not in blocked:
            src_state[s] = new_src[s]
    return rows, src_status
