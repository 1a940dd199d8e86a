"""A pure-Python model of Timer element-set rollups across shards (m3tsz_element_set_forward_write_timer /
_add_forwarded_timer, DESIGN.md §4.12), composed from existing models: the writer is element_forwarded_model's
forward_write over TimerSourceModel lists (element_timer_rollup_model: each due window's ValueOf through the pre-ops),
and the add is element_forwarded_model's AddUnique rules over TimerGroupModel windows with a per-window seen-set, each
value one Timer.Add (the independent Timer's add_batch of that one value).  Test infrastructure only.

  - Rule 6 (sample capacity), after the duplicate check: a record whose values would take its window past
    sample_capacity samples (the stream's size() -- list samples and pending values -- plus the record's values) is
    ERR_CAPACITY and stops the element for the rest of the call; its source is not marked seen and a window it would
    have opened stays closed."""
from element_forwarded_model import ERR_DUPLICATE_SOURCE, forward_write
from element_set_model import INT64_MIN, window_start
from element_timer_rollup_model import ERR_CAPACITY, ERR_CLOSED, ERR_INVALID_ARG, OK, TimerGroupModel, TimerSourceModel
from indep_timer import Timer

__all__ = ["TimerSourceModel", "TimerForwardedGroupModel", "forward_write", "add_forwarded_timer", "OK",
           "ERR_CAPACITY", "ERR_CLOSED", "ERR_INVALID_ARG", "ERR_DUPLICATE_SOURCE"]


class TimerForwardedGroupModel(TimerGroupModel):
    """A Timer group element fed by forwarded records: its windows' Timers and the source ids each open window has
    seen (a window the element no longer holds has seen none)."""

    def __init__(self, *a, source_capacity=64, **k):
        super().__init__(*a, **k)
        self.source_capacity = source_capacity
        self.seen = {}

    def seen_by(self, ws):
        return self.seen.get(ws, set()) if ws in self.windows else set()


def add_forwarded_timer(groups, records):
    """AddUnique of the records, in order, into TimerForwardedGroupModel lists, in place -> (results, element
    statuses)"""
    results, status = [], [OK] * len(groups)
    for key, t, vals, sid, version, reserved in records:
        if key >= len(groups):
            results.append(ERR_INVALID_ARG)
            continue
        g = groups[key]
        if status[key] != OK:  # (add's stop rule: every later record of the element)
            results.append(ERR_CAPACITY)
            continue
        if not vals or version or reserved:
            results.append(ERR_INVALID_ARG)
            continue
        ws = window_start(t, g.res) - g.res
        if ws < INT64_MIN:
            results.append(ERR_INVALID_ARG)
        elif g.closed(ws):
            results.append(ERR_CLOSED)
        elif sid >= g.source_capacity or (ws not in g.windows and len(g.windows) >= g.R):
            status[key] = ERR_CAPACITY
            results.append(ERR_CAPACITY)
        elif sid in g.seen_by(ws):
            results.append(ERR_DUPLICATE_SOURCE)
        elif (g.windows[ws].stream.size() if ws in g.windows else 0) + len(vals) > g.cap:
            status[key] = ERR_CAPACITY
            results.append(ERR_CAPACITY)
        else:
            if ws not in g.windows:
                g.windows[ws] = Timer(g.types, g.eps, g.every)
                g.seen[ws] = set()
            g.seen[ws].add(sid)
            for v in vals:
                g.windows[ws].add_batch([v])
            results.append(OK)
    return results, status
