"""A pure-Python model of the element sets (m3tsz_element_set_*, DESIGN.md §4.12): the aggregator's elements fed
datapoint by datapoint.  Built from the window oracle (agg_oracle_lib: Gauge / Counter Update and ValueOf over one
window's datapoints, in add order) and the element oracle (elem_oracle_lib: the transformations on the element record);
the closed-window and capacity rules are stated here on their own.  Test infrastructure only.

Two rules for a write to a window that has been consumed:
  - "watermark" (this library): every window ending at or before the end of the last window consumed is closed;
  - "reference" (GenericElem): only the last window consumed stays closed (expireValuesWithLock keeps it for the binary
    transformations, generic_elem.go:291-358); a write to an older one goes through findOrCreate, which opens a fresh
    window, and the next Consume flushes it after the later windows already flushed."""
import numpy as np

import agg_oracle_lib as A
import elem_oracle_lib as E

OK, ERR_INVALID_ARG, ERR_CLOSED, ERR_CAPACITY = 0, 101, 17, 100
INT64_MIN = -(1 << 63)
ZERO_TIME_NS = 62135596800 * 1_000_000_000  # the zero time (year 1) before the Unix epoch


def window_start(t, res):
    """time.Time.Truncate(res): truncation of the time since the zero time (Python's % floors)"""
    return t - (t + ZERO_TIME_NS) % res


class ElementModel:
    """One element: open windows {start: [(t, v bits)] in add order}, its record and its watermark."""

    def __init__(self, metric_type, agg_types, resolution_ns, ops=(), discard_nan=False, open_windows=4,
                 rule="watermark"):
        self.metric_type, self.agg_types, self.res = metric_type, list(agg_types), int(resolution_ns)
        self.ops, self.discard = list(ops), bool(discard_nan) and len(ops) > 0  # (as aggregate_tiles_types)
        self.R, self.rule = open_windows, rule
        self.windows = {}
        self.watermark = INT64_MIN
        self.last_consumed = None
        self.state = E.new_element_state()

    def closed(self, ws):
        if self.rule == "reference":
            return ws == self.last_consumed
        return ws + self.res <= self.watermark

    def add(self, points):
        """points [(t, value bits)] in order -> (results, status)"""
        res, status = [], OK
        for t, vb in points:
            if status != OK:
                res.append(ERR_CAPACITY)
                continue
            ws = window_start(t, self.res)
            if ws < INT64_MIN:
                res.append(ERR_INVALID_ARG)
            elif self.closed(ws):
                res.append(ERR_CLOSED)
            elif ws not in self.windows and self.R is not None and len(self.windows) >= self.R:
                status = ERR_CAPACITY
                res.append(ERR_CAPACITY)
            else:
                self.windows.setdefault(ws, []).append((t, vb))
                res.append(OK)
        return res, status

    def aggregates(self, ws):
        """the window's aggregates, as the device's slots hold them"""
        pts = self.windows[ws]
        ts = np.array([t for t, _ in pts], dtype=np.int64)
        vs = np.array([v for _, v in pts], dtype=np.uint64).view(np.float64)
        if self.metric_type == A.METRIC_COUNTER:
            s, c, mn, mx, sq = (int(x[0]) for x in A.downsample_counter(ts, vs, ws, self.res, 1))
            return {"sum": s, "count": c, "min": mn, "max": mx, "sum_sq": sq}
        s, c, mn, mx, last, la, sq = (x[0] for x in A.downsample_gauge_ex(ts, vs, ws, self.res, 1))
        return {"sum": float(s), "count": int(c), "min": float(mn), "max": float(mx), "last": float(last),
                "last_at": int(la), "sum_sq": float(sq)}

    def value_of(self, ws, agg):
        a = self.aggregates(ws)
        if self.metric_type == A.METRIC_COUNTER:
            return A.counter_value_of(agg, a["sum"], a["count"], a["min"], a["max"], a["sum_sq"])
        return A.gauge_value_of_ex(agg, a["sum"], a["count"], a["min"], a["max"], a["last"], a["sum_sq"])

    def consume(self, target):
        """Consume(target) -> [(ts, values)] per type, the datapoints flushed"""
        flush = sorted(ws for ws in self.windows if ws + self.res <= target)
        k = len(self.agg_types)
        ends = np.array([ws + self.res for ws in flush], dtype=np.int64)
        vals = np.array([[self.value_of(ws, a) for a in self.agg_types] for ws in flush],
                        dtype=np.float64).reshape(len(flush), k)
        out = E.element_series(self.ops, self.discard, self.res, k, self.state, ends, vals)
        for ws in flush:
            del self.windows[ws]
        if flush:
            self.watermark = flush[-1] + self.res
            self.last_consumed = flush[-1]
        return out
