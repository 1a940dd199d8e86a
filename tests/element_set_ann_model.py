"""A pure-Python model of the element sets that keep annotations (m3tsz_element_set_*_annotated, DESIGN.md §4.12),
composed over the element-set model (tests/element_set_model.py) without changing it.

The rule, stated from the reference: Gauge.Update / Counter.Update keep the last non-empty annotation of the
datapoints a window takes (MaybeReplaceAnnotation, aggregation/common.go:47-61), whatever the value; Consume copies it
into the flush state (generic_elem.go:567) and every datapoint flushed for the window carries it, the Reset datapoint
included (generic_elem.go:923-931).  Refused datapoints change nothing.  Each window slot holds at most `capacity`
bytes: a datapoint the element would accept with a longer annotation stops the element with CAPACITY, as a new
window with every slot open does.

The expected output streams come from the reference encoder oracle (oracle_lib.Encoder), each row fed every datapoint
flushed for it with its annotation, as tests/ann_oracle_lib.py composes the tile path.  Test infrastructure only."""
import numpy as np

import oracle_lib as O
from element_set_model import ERR_CAPACITY, INT64_MIN, OK, ElementModel, window_start

TRANSFORM_RESET = 5


class AnnotatedElementModel:
    """One element: the element-set model, each open window's annotation, and (with start_ns) one reference encoder
    per aggregation type that every flushed datapoint is written to."""

    def __init__(self, metric_type, agg_types, resolution_ns, ops=(), discard_nan=False, open_windows=4,
                 capacity=None, start_ns=None, int_optimized=True, default_unit=O.UNIT_S, out_unit=O.UNIT_S):
        self.m = ElementModel(metric_type, agg_types, resolution_ns, ops, discard_nan, open_windows)
        self.capacity = capacity
        self.ann = {}  # window start -> its annotation (b"" for none)
        self.out_unit = out_unit
        self.enc = None
        if start_ns is not None:
            self.enc = [O.Encoder(int(start_ns), int_optimized, default_unit) for _ in agg_types]

    @property
    def state(self):
        return self.m.state

    @property
    def watermark(self):
        return self.m.watermark

    def window_annotation(self, ws):
        return self.ann[ws]

    def add(self, points):
        """points [(t, value bits, annotation bytes)] in order -> (results, status)"""
        res, status = [], OK
        for t, vb, a in points:
            if status != OK:
                res.append(ERR_CAPACITY)
                continue
            ws = window_start(t, self.m.res)
            accepted = ws >= INT64_MIN and not self.m.closed(ws)
            if accepted and self.capacity is not None and len(a) > self.capacity:
                status = ERR_CAPACITY
                res.append(ERR_CAPACITY)
                continue
            r, status = self.m.add([(t, vb)])
            res.append(r[0])
            if r[0] == OK:
                self.ann.setdefault(ws, b"")
                if a:
                    self.ann[ws] = bytes(a)
        return res, status

    def consume(self, target):
        """Consume(target) -> [(ts, values, annotations)] per type, the datapoints flushed; with encoders, also
        writes them to the type's stream"""
        flush = sorted(ws for ws in self.m.windows if ws + self.m.res <= target)
        anns = [self.ann.pop(ws) for ws in flush]
        out = self.m.consume(target)
        reset = TRANSFORM_RESET in self.m.ops
        rw = int(max(float(self.m.res // 2), 1.0))  # the Reset datapoint's offset (as ann_oracle_lib)
        got = []
        for j, (to, vo) in enumerate(out):
            per = []
            i = 0
            for ws, a in zip(flush, anns):  # a type writes a window's datapoint, then its Reset datapoint, or neither
                t = ws + self.m.res
                if i < len(to) and int(to[i]) == t:
                    for _ in range(2 if (reset and t + rw != 0) else 1):
                        per.append(a)
                        i += 1
            assert i == len(to)
            if self.enc is not None:
                for t, v, a in zip(to.tolist(), vo.tolist(), per):
                    assert self.enc[j].encode(int(t), float(v), self.out_unit, a) == 0
            got.append((to, vo, per))
        return got

    def streams(self):
        """the output rows' bytes so far, one per type"""
        return [e.stream() or b"" for e in self.enc]


def annotation_words(length):
    """the words the encoder-set append's room check counts for an annotation (m3tsz_encode.cu encode_row)"""
    return (length + 3) // 4 + 4 if length else 0


def annotated_points(points, rng, payloads, p_annotated=0.5):
    """[(t, value bits)] -> [(t, value bits, annotation)], each datapoint carrying one of `payloads` with
    probability p_annotated, else none"""
    out = []
    for t, vb in points:
        a = payloads[int(rng.integers(0, len(payloads)))] if rng.random() < p_annotated else b""
        out.append((t, vb, a))
    return out


def sparse_annotations(cols):
    """per-element columns [(t, value bits, annotation)] -> (series_off int64 [N + 1], entries uint8 [E, 16], bytes
    uint8), the encoder-set append's sparse list with dp_index counting rows of each element's column"""
    off, ent, buf = [0], [], bytearray()
    for c in cols:
        for i, (_, _, a) in enumerate(c):
            if a:
                ent.append((i, len(a), len(buf)))
                buf += a
        off.append(len(ent))
    e = np.zeros(max(1, len(ent)), dtype=[("dp_index", "<u4"), ("length", "<u4"), ("byte_offset", "<u8")])
    for k, x in enumerate(ent):
        e[k] = x
    b = np.frombuffer(bytes(buf) or b"\0", dtype=np.uint8).copy()
    return np.array(off, dtype=np.int64), e.view(np.uint8).reshape(-1, 16), b
