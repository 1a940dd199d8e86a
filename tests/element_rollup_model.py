"""A pure-Python model of element sets through a rollup (m3tsz_element_set_forward, DESIGN.md §4.12), composed from
the element-set model (element_set_model.ElementModel: the sources' and the groups' windows, records, watermarks and
consume) and the tile rollup's oracles (rollup_oracle_lib: the forward of a window's value through the pre-ops with
the source-side NaN discard, and the AddUnique fold of a window's values in listed order).  The closed rule and the
commit rule are stated here on their own.  Test infrastructure only."""
import numpy as np

import agg_oracle_lib as A
import rollup_oracle_lib as R
import xf_oracle_lib as X
from element_set_model import ERR_CAPACITY, ERR_CLOSED, ERR_INVALID_ARG, OK, ElementModel

__all__ = ["SourceModel", "GroupModel", "forward", "OK", "ERR_CAPACITY", "ERR_CLOSED", "ERR_INVALID_ARG"]


class SourceModel(ElementModel):
    """A source element: an element of one type (the rollup's source type) whose Consume forwards instead of writing.
    Its pre-ops run on the first 96 bytes of its record (the transform state xf_window runs on), and discard_nan
    drops a NaN value with or without ops, as rollup_oracle_lib.forward_series does."""

    def __init__(self, metric_type, src_type, resolution_ns, ops=(), discard_nan=False, open_windows=4):
        super().__init__(metric_type, [src_type], resolution_ns, ops, discard_nan, open_windows)
        self.src_type = src_type
        self.discard_src = bool(discard_nan)

    def pending(self, target):
        """Consume(target) without committing: ([(start, value, forwarded)] in start order, the new record)"""
        flush = sorted(ws for ws in self.windows if ws + self.res <= target)
        xs = np.frombuffer(self.state.tobytes()[:96], dtype=X.XF_STATE_DTYPE).copy()
        out = []
        for ws in flush:
            v = float(self.value_of(ws, self.src_type))
            to, vo = X.transform_series(self.ops, self.discard_src, self.res, xs, [ws + self.res], [v])
            fwd = len(to) > 0  # (a Reset's extra datapoint comes second and is not forwarded)
            out.append((ws, float(vo[0]) if fwd else None, fwd))
        rec = self.state.copy()
        rec.view(np.uint8)[:96] = np.frombuffer(xs.tobytes(), dtype=np.uint8)
        return out, rec

    def commit(self, target, rec):
        flush = sorted(ws for ws in self.windows if ws + self.res <= target)
        for ws in flush:
            del self.windows[ws]
        if flush:
            self.watermark = flush[-1] + self.res
            self.last_consumed = flush[-1]
            self.state = rec


class GroupModel(ElementModel):
    """A group element (the rollup element): its windows hold the values AddUnique gave them, in order, and their
    aggregates are rollup_oracle_lib's fold of those values; consume is the element set's (the group side keeps the
    element set's discard-with-ops rule)."""

    def fits(self, starts):
        """the new windows of `starts` (not open, not closed) fit the free slots"""
        new = {ws for ws in starts if ws not in self.windows and not self.closed(ws)}
        return self.R is None or len(self.windows) + len(new) <= self.R

    def add_unique(self, ws, v):
        """-> False: the window is closed and the value dropped"""
        if self.closed(ws):
            return False
        self.windows.setdefault(ws, []).append(v)
        return True

    def aggregates(self, ws):
        vs = self.windows[ws]
        if self.metric_type == A.METRIC_COUNTER:
            s, c, mn, mx, sq = R.fold_counter(vs)
            return {"sum": s, "count": c, "min": mn, "max": mx, "sum_sq": sq}
        s, c, mn, mx, last, sq = R.fold_gauge(vs)
        return {"sum": float(s), "count": int(c), "min": float(mn), "max": float(mx), "last": float(last),
                "last_at": ws + self.res, "sum_sq": float(sq)}

    def value_of(self, ws, agg):
        return R.rollup_value_of(self.metric_type, agg, self.windows[ws])


def forward(sources, groups, target, group_off, members):
    """m3tsz_element_set_forward over SourceModel / GroupModel lists, in place -> (source statuses, group statuses).
    Rules: the group's range and indices (INVALID_ARG), then its new windows against its free slots (CAPACITY) -- a
    failed group folds nothing and holds back the members its range names; the fold in listed order, each member's
    windows in start order, a closed window's values dropped (AGGREGATION_CLOSED); every source not held back
    commits, the others keep everything and take the failed group's status (INVALID_ARG over CAPACITY)."""
    S, G, n_mem = len(sources), len(groups), len(members)
    pend = [s.pending(target) for s in sources]
    gst = [OK] * G
    mark = [0] * S
    for g in range(G):
        lo, hi = int(group_off[g]), int(group_off[g + 1])
        if lo > hi or hi > n_mem or any(int(members[i]) >= S for i in range(lo, hi)):
            gst[g] = ERR_INVALID_ARG
        else:
            mem = [int(members[i]) for i in range(lo, hi)]
            vals = [(ws, v) for m in mem for ws, v, fwd in pend[m][0] if fwd]
            if not groups[g].fits([ws for ws, _ in vals]):
                gst[g] = ERR_CAPACITY
            else:
                for ws, v in vals:
                    if not groups[g].add_unique(ws, v):
                        gst[g] = ERR_CLOSED
        if gst[g] in (ERR_CAPACITY, ERR_INVALID_ARG) and lo <= hi:
            for i in range(lo, min(hi, n_mem)):
                m = int(members[i])
                if m < S:
                    mark[m] = max(mark[m], gst[g])
    for s in range(S):
        if not mark[s]:
            sources[s].commit(target, pend[s][1])
    return mark, gst
