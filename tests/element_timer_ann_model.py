"""A pure-Python model of the Timer element sets that keep annotations (m3tsz_element_set_*_timer_annotated, DESIGN.md
§4.12), composed without changing them from the Timer element-set model (element_timer_model), the annotated
element-set model (element_set_ann_model: each open window's annotation, the consume's per-datapoint annotations and
the reference encoder oracle the output rows are checked against) and, for the rollup, the Timer rollup model
(element_timer_rollup_model) with the annotated rollup's group rule (element_rollup_ann_model.forward).

The rule stated here on its own: a batch has one annotation, its first row's (a BatchTimer carries one,
AppendTimerSample one per sample); an annotation on a continuation row breaks the batch rule (every row ERR_INVALID_ARG,
nothing changes).  After the closed and invalid-start checks, a batch whose annotation is longer than the slots'
capacity stops the element with ERR_CAPACITY; an accepted batch with a non-empty annotation replaces its window's
(MaybeReplaceAnnotation, aggregation/timer.go:57-76), NaN samples included.  Test infrastructure only."""
import oracle_lib as O
from element_rollup_ann_model import AnnotatedSource, forward
from element_set_ann_model import AnnotatedElementModel
from element_set_model import ERR_CAPACITY, ERR_INVALID_ARG, INT64_MIN, OK, window_start
from element_timer_model import TimerElementModel, split_batches
from element_timer_rollup_model import TimerGroupModel, TimerSourceModel

__all__ = ["AnnotatedTimerModel", "AnnotatedTimerSource", "AnnotatedTimerGroup", "forward"]


class AnnotatedTimerModel(AnnotatedElementModel):
    """One Timer element that keeps annotations, with (start_ns) one reference encoder per type for its output rows"""

    def __init__(self, agg_types, resolution_ns, ops=(), discard_nan=False, open_windows=4, sample_capacity=64,
                 eps=1e-3, every=1024, capacity=None, start_ns=None, int_optimized=True, default_unit=O.UNIT_S,
                 out_unit=O.UNIT_S):
        self.m = self._model(agg_types, resolution_ns, ops, discard_nan, open_windows, sample_capacity, eps, every)
        self.capacity = capacity
        self.ann = {}  # window start -> its annotation (b"" for none)
        self.out_unit = out_unit
        self.enc = None
        if start_ns is not None:
            self.enc = [O.Encoder(int(start_ns), int_optimized, default_unit) for _ in agg_types]

    @staticmethod
    def _model(*args):
        return TimerElementModel(*args)

    def add(self, rows, marks=None, anns=None):
        """rows [(t, value float)], marks (continuations), anns (per row bytes, b"" none) -> (results, status)"""
        marks = [0] * len(rows) if marks is None else list(marks)
        anns = [b""] * len(rows) if anns is None else [bytes(a) for a in anns]
        batches = split_batches(rows, marks)
        if batches is None or any(a and m for a, m in zip(anns, marks)):
            return [ERR_INVALID_ARG] * len(rows), ERR_INVALID_ARG
        res, status = [], OK
        for first, b in batches:
            a = anns[first]
            ws = window_start(b[0][0], self.m.res)
            if status != OK:
                r = ERR_CAPACITY
            elif ws < INT64_MIN or ws + self.m.res <= self.m.watermark:
                r = self.m.add(b, [0] + [1] * (len(b) - 1))[0][0]  # (refused: INVALID_ARG / CLOSED, nothing changes)
            elif self.capacity is not None and len(a) > self.capacity:
                status = r = ERR_CAPACITY
            else:
                rr, status = self.m.add(b, [0] + [1] * (len(b) - 1))
                r = rr[0]
                if r == OK:
                    self.ann.setdefault(ws, b"")
                    if a:
                        self.ann[ws] = a
            res += [r] * len(b)
        return res, status


class AnnotatedTimerSource(AnnotatedTimerModel, AnnotatedSource):
    """A Timer source that keeps annotations: the annotated Timer add over a TimerSourceModel, forwarded as
    AnnotatedSource forwards"""

    def __init__(self, src_type, resolution_ns, ops=(), discard_nan=False, open_windows=4, sample_capacity=64,
                 eps=1e-3, every=1024, capacity=None):
        AnnotatedTimerModel.__init__(self, [src_type], resolution_ns, ops, discard_nan, open_windows, sample_capacity,
                                     eps, every, capacity)
        self.m = TimerSourceModel(src_type, resolution_ns, ops, discard_nan, open_windows, sample_capacity, eps, every)


class _TimerGroup(TimerGroupModel):
    """the Timer group, with the flag element_rollup_ann_model.forward sets: an annotation too long for the slots"""
    too_long = False

    def fits(self, starts):
        return not self.too_long and super().fits(starts)


class AnnotatedTimerGroup(AnnotatedTimerModel):
    """A Timer group element that keeps annotations (its consume is the annotated Timer consume)"""

    @staticmethod
    def _model(*args):
        return _TimerGroup(*args)
