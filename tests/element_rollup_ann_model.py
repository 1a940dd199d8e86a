"""A pure-Python model of element sets through a rollup that keep annotations (m3tsz_element_set_forward_annotated,
DESIGN.md §4.12), composed without changing them from the element-rollup model (tests/element_rollup_model.py: the
sources, the groups, the forward and its commit rule) and the annotated element-set model
(tests/element_set_ann_model.py: each open window's annotation, the annotated add and consume).

The group annotation selection is stated here on its own, from the rule of rollup_ann_oracle_lib.group_annotation:
a group window takes the last non-empty annotation, in listed member order, among the members that forwarded a value
to it (MaybeReplaceAnnotation through AddUnique, generic_elem.go:278-281, aggregation/common.go:47-61).  Unlike the
tile call's windows, group windows persist across calls: a window already open keeps its annotation unless a forwarded
value brings one, and a window the call opens starts with none.  A value whose group window is closed brings nothing;
a NaN that discard_nan drops is not forwarded.  A group one of whose values that would fold carries an annotation
longer than the group slots' capacity gets CAPACITY under the element-rollup model's rule.  Test infrastructure
only."""
import element_rollup_model as ER
import rollup_ann_oracle_lib as RA
from element_rollup_model import ERR_CAPACITY, ERR_CLOSED, ERR_INVALID_ARG, OK, GroupModel, SourceModel
from element_set_ann_model import AnnotatedElementModel

__all__ = ["AnnotatedSource", "AnnotatedGroup", "forward", "OK", "ERR_CAPACITY", "ERR_CLOSED", "ERR_INVALID_ARG"]


class AnnotatedSource(AnnotatedElementModel):
    """A source element that keeps annotations: the annotated element-set model over an element_rollup_model
    SourceModel (add(points) takes [(t, value bits, annotation)])."""

    def __init__(self, metric_type, src_type, resolution_ns, ops=(), discard_nan=False, open_windows=4,
                 capacity=None):
        super().__init__(metric_type, [src_type], resolution_ns, ops, discard_nan, open_windows, capacity)
        self.m = SourceModel(metric_type, src_type, resolution_ns, ops, discard_nan, open_windows)

    def slot_annotation(self, ws):
        """what a forward reads of window ws's slot: its annotation, none for a length above the capacity"""
        a = self.ann.get(ws, b"")
        return b"" if self.capacity is not None and len(a) > self.capacity else a

    def set_length_above_capacity(self, ws):
        """open window ws's slot length reads as more than the capacity (none) until an annotation replaces it"""
        assert ws in self.m.windows and self.capacity is not None
        self.ann[ws] = b"\0" * (self.capacity + 8)

    def forwarded(self, target):
        """Consume(target) without committing: [(start, value, annotation)] of the windows it forwards, start order"""
        out, _ = self.m.pending(target)
        return [(ws, v, self.slot_annotation(ws)) for ws, v, fwd in out if fwd]

    def _committed(self):
        self.ann = {ws: a for ws, a in self.ann.items() if ws in self.m.windows}


class _Group(GroupModel):
    """element_rollup_model's group, with a flag the annotated forward sets: an annotation too long for the slots"""
    too_long = False

    def fits(self, starts):
        return not self.too_long and super().fits(starts)


class AnnotatedGroup(AnnotatedElementModel):
    """A group element that keeps annotations: the annotated element-set model (consume) over an element_rollup_model
    GroupModel"""

    def __init__(self, metric_type, agg_types, resolution_ns, ops=(), discard_nan=False, open_windows=4,
                 capacity=None, start_ns=None, int_optimized=True):
        super().__init__(metric_type, agg_types, resolution_ns, ops, discard_nan, open_windows, capacity, start_ns,
                         int_optimized)
        self.m = _Group(metric_type, agg_types, resolution_ns, ops, discard_nan, open_windows)


def forward(sources, groups, target, group_off, members):
    """m3tsz_element_set_forward_annotated over AnnotatedSource / AnnotatedGroup lists, in place -> (source
    statuses, group statuses): element_rollup_model.forward on the values, with the annotation capacity rule joining
    its capacity check, and each folded group window's annotation selected as the module docstring states"""
    S, n_mem = len(sources), len(members)
    fw = [s.forwarded(target) for s in sources]
    taken = []  # per group: {window start: the annotation its members bring (b"" for none)}
    for g, grp in enumerate(groups):
        lo, hi = int(group_off[g]), int(group_off[g + 1])
        grp.m.too_long = False
        taken.append({})
        if lo > hi or hi > n_mem or any(int(members[i]) >= S for i in range(lo, hi)):
            continue  # (INVALID_ARG: the element-rollup model's own rule)
        mem = [int(members[i]) for i in range(lo, hi)]
        fwd = [{ws: v for ws, v, _ in fw[m]} for m in mem]  # per listed position
        src_ann = [{ws: a for ws, _, a in fw[m]} for m in mem]
        starts = {ws for f in fwd for ws in f if not grp.m.closed(ws)}
        grp.m.too_long = grp.capacity is not None and any(
            len(a) > grp.capacity for sa in src_ann for ws, a in sa.items() if ws in starts)
        taken[g] = {ws: RA.group_annotation(fwd, src_ann, range(len(mem)), ws) for ws in starts}
    mark, gst = ER.forward([s.m for s in sources], [grp.m for grp in groups], target, group_off, members)
    for g, grp in enumerate(groups):
        grp.m.too_long = False
        if gst[g] in (OK, ERR_CLOSED):
            for ws, a in taken[g].items():
                if a:
                    grp.ann[ws] = a
                else:
                    grp.ann.setdefault(ws, b"")
    for s in sources:
        s._committed()
    return mark, gst
