"""A pure-Python model of Timer element sets through a rollup (m3tsz_element_set_forward_timer, DESIGN.md §4.12),
composed from the Timer element-set model (element_timer_model: the sources' and the groups' windows, watermarks,
records and consume) and the element-rollup model's group and commit rules (element_rollup_model.forward), with each
folded value one Timer.Add: the independent Timer's add_batch of that one value.  The capacity rule is stated here on
its own.  Test infrastructure only.

  - Forward: a source's due windows in start order, each window's ValueOf(the source type) after Flush, through the
    pre-ops on the record's transform state; discard_nan drops a NaN with or without ops.
  - Capacity: a group fails when its new windows outnumber its free slots, or when a window it touches would hold more
    than sample_capacity values: its list samples + pending values + the values folded into it in the call."""
from collections import Counter

import numpy as np

import xf_oracle_lib as X
from element_rollup_model import ERR_CAPACITY, ERR_CLOSED, ERR_INVALID_ARG, OK, forward
from element_timer_model import TimerElementModel
from indep_timer import Timer

__all__ = ["TimerSourceModel", "TimerGroupModel", "forward", "OK", "ERR_CAPACITY", "ERR_CLOSED", "ERR_INVALID_ARG"]


class TimerSourceModel(TimerElementModel):
    """A Timer source element of one type whose Consume forwards instead of writing"""

    def __init__(self, src_type, resolution_ns, ops=(), discard_nan=False, open_windows=4, sample_capacity=64,
                 eps=1e-3, every=1024):
        super().__init__([src_type], resolution_ns, ops, discard_nan, open_windows, sample_capacity, eps, every)
        self.discard_src = bool(discard_nan)

    def pending(self, target):
        """Consume(target) without committing: ([(start, value, forwarded)] in start order, the new record)"""
        flush = sorted(ws for ws in self.windows if ws + self.res <= target)
        xs = np.frombuffer(self.state.tobytes()[:96], dtype=X.XF_STATE_DTYPE).copy()
        out = []
        for ws in flush:
            v = float(self.windows[ws].values()[0])  # (Flush; a second one recomputes the same quantiles)
            to, vo = X.transform_series(self.ops, self.discard_src, self.res, xs, [ws + self.res], [v])
            fwd = len(to) > 0
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
            self.state = rec


class TimerGroupModel(TimerElementModel):
    """A group element (the rollup element, a Timer): each folded value is one Timer.Add into its window"""

    def closed(self, ws):
        return ws + self.res <= self.watermark

    def fits(self, starts):
        """the values going to `starts` (one entry per value) fit the free slots and the sample capacity"""
        n = Counter(ws for ws in starts if not self.closed(ws))
        new = [ws for ws in n if ws not in self.windows]
        if len(self.windows) + len(new) > self.R:
            return False
        return all((self.windows[ws].stream.size() if ws in self.windows else 0) + k <= self.cap
                   for ws, k in n.items())

    def add_unique(self, ws, v):
        """Timer.Add(v) into window ws -> False: the window is closed and the value dropped"""
        if self.closed(ws):
            return False
        if ws not in self.windows:
            self.windows[ws] = Timer(self.types, self.eps, self.every)
        self.windows[ws].add_batch([v])
        return True
