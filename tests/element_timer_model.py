"""A pure-Python model of the Timer element sets (m3tsz_element_set_*_timer, DESIGN.md §4.12): the element-set model's
windows, closed-window rule and record (element_set_model, elem_oracle_lib) with each window an aggregation.Timer of
the independent restatement (indep_timer).  The capacity rule and the batch rule are stated here on their own.  Test
infrastructure only.

  - Batch rule: a row marked as a continuation joins the previous row's batch; one in row 0, or one whose timestamp
    differs from its batch's first, refuses the whole element (every row ERR_INVALID_ARG, nothing changes).
  - Capacity rule: a window holds at most `sample_capacity` values, list samples and pending values together.  A batch
    that would exceed it, or that needs a new window when all R are open, is ERR_CAPACITY, and so is every later row
    of the element in the call."""
import numpy as np

import elem_oracle_lib as E
from element_set_model import ERR_CAPACITY, ERR_CLOSED, ERR_INVALID_ARG, INT64_MIN, OK, window_start
from indep_timer import Timer

MAX_ELEMENT_TYPES = 8


def split_batches(rows, marks):
    """rows [(t, v)] and continuation marks -> [(first row, [rows])], or None when the marks break the batch rule"""
    out = []
    for i, ((t, v), m) in enumerate(zip(rows, marks)):
        if m:
            if not out or t != out[-1][1][0][0]:
                return None
            out[-1][1].append((t, v))
        else:
            out.append((i, [(t, v)]))
    return out


class TimerElementModel:
    def __init__(self, agg_types, resolution_ns, ops=(), discard_nan=False, open_windows=4, sample_capacity=64,
                 eps=1e-3, every=1024):
        self.types, self.res = list(agg_types), int(resolution_ns)
        self.ops, self.discard = list(ops), bool(discard_nan) and len(ops) > 0
        self.R, self.cap, self.eps, self.every = open_windows, int(sample_capacity), float(eps), int(every)
        self.windows = {}  # start -> Timer
        self.watermark = INT64_MIN
        self.state = E.new_element_state()

    def add(self, rows, marks=None):
        """rows [(t, value float)] in order, marks (continuations) -> (per-row results, status)"""
        marks = [0] * len(rows) if marks is None else list(marks)
        batches = split_batches(rows, marks)
        if batches is None:
            return [ERR_INVALID_ARG] * len(rows), ERR_INVALID_ARG
        res, status = [], OK
        for _, b in batches:
            r = ERR_CAPACITY
            if status == OK:
                ws = window_start(b[0][0], self.res)
                if ws < INT64_MIN:
                    r = ERR_INVALID_ARG
                elif ws + self.res <= self.watermark:
                    r = ERR_CLOSED
                else:
                    w = self.windows.get(ws)
                    size = w.stream.size() if w is not None else 0
                    if (w is None and len(self.windows) >= self.R) or size + len(b) > self.cap:
                        status = r = ERR_CAPACITY
                    else:
                        if w is None:
                            w = self.windows[ws] = Timer(self.types, self.eps, self.every)
                        w.add_batch([v for _, v in b])
                        r = OK
            res += [r] * len(b)
        return res, status

    def consume(self, target):
        """Consume(target) -> [(ts, values)] per type"""
        flush = sorted(ws for ws in self.windows if ws + self.res <= target)
        k = len(self.types)
        ends = np.array([ws + self.res for ws in flush], dtype=np.int64)
        vals = np.array([self.windows[ws].values() for ws in flush], dtype=np.float64).reshape(len(flush), k)
        if k <= MAX_ELEMENT_TYPES:
            out = E.element_series(self.ops, self.discard, self.res, k, self.state, ends, vals)
        else:  # (no ops: every window's value, the record untouched)
            out = [(ends.copy(), vals[:, j].copy()) for j in range(k)]
        for ws in flush:
            del self.windows[ws]
        if flush:
            self.watermark = flush[-1] + self.res
        return out
