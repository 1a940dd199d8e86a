"""A pure-Python model of element-set rollups across shards (m3tsz_element_set_forward_write / _add_forwarded,
DESIGN.md §4.12), composed from the element rollup model (element_rollup_model: the sources' forward and commit, the
group windows' fold) with the forwarded writer's buckets (forwarded_writer.go: one record per rollup key and window,
its values in write order) and AddUnique's per-window sourcesSeen (generic_elem.go:241-288).  Test infrastructure
only."""
from element_rollup_model import ERR_CAPACITY, ERR_CLOSED, ERR_INVALID_ARG, OK, GroupModel, SourceModel
from element_set_model import INT64_MIN, window_start

ERR_DUPLICATE_SOURCE = 18

__all__ = ["SourceModel", "ForwardedGroupModel", "write_buckets", "forward_write", "add_forwarded", "OK",
           "ERR_CAPACITY", "ERR_CLOSED", "ERR_INVALID_ARG", "ERR_DUPLICATE_SOURCE"]


class ForwardedGroupModel(GroupModel):
    """A group element fed by forwarded records: its windows' values (GroupModel) and the source ids each open window
    has seen (a window the element no longer holds has seen none)."""

    def __init__(self, *a, source_capacity=64, **k):
        super().__init__(*a, **k)
        self.source_capacity = source_capacity
        self.seen = {}

    def seen_by(self, ws):
        return self.seen.get(ws, set()) if ws in self.windows else set()


def write_buckets(writes):
    """The forwarded writer's buckets (forwardedAggregation.write / onDone): writes [(key, time_ns, value)] in write
    order -> records [(key, time_ns, [values])], keys in first-write order, each key's times ascending, each bucket's
    values in write order"""
    by_key = {}
    for key, t, v in writes:
        by_key.setdefault(key, {}).setdefault(t, []).append(v)
    return [(key, t, vals) for key, b in by_key.items() for t, vals in sorted(b.items())]


def forward_write(sources, target, group_off, members, source_id, keys=None, metric_capacity=None,
                  value_capacity=None):
    """The source shard's writer over SourceModel lists, in place -> (records [(key, time_ns, [values], source_id,
    version, reserved)], source statuses, group statuses, counts).  Each valid group's distinct forwarded starts in
    ascending order, its members' values in listed order; the groups whose records and values end within the
    capacities are written, every later one fails with CAPACITY; a failed group holds its members back."""
    S, G, n_mem = len(sources), len(group_off) - 1, len(members)
    pend = [s.pending(target) for s in sources]
    gst, mark, records = [OK] * G, [0] * S, []
    need_r = need_v = wrote_r = wrote_v = 0
    for g in range(G):
        lo, hi = int(group_off[g]), int(group_off[g + 1])
        if lo > hi or hi > n_mem or any(int(members[i]) >= S for i in range(lo, hi)):
            gst[g] = ERR_INVALID_ARG
        else:
            key = g if keys is None else int(keys[g])
            res = sources[0].res if sources else 0
            buckets = write_buckets([(key, ws + res, v) for i in range(lo, hi)
                                     for ws, v, fwd in pend[int(members[i])][0] if fwd])
            nr, nv = len(buckets), sum(len(b) for _, _, b in buckets)
            fits = (metric_capacity is None or need_r + nr <= metric_capacity) and \
                   (value_capacity is None or need_v + nv <= value_capacity)
            need_r, need_v = need_r + nr, need_v + nv
            if fits:
                records += [(k, t, vals, source_id, 0, 0) for k, t, vals in buckets]
                wrote_r, wrote_v = need_r, need_v
            else:
                gst[g] = ERR_CAPACITY
        if gst[g] in (ERR_CAPACITY, ERR_INVALID_ARG) and lo <= hi:
            for i in range(lo, min(hi, n_mem)):
                m = int(members[i])
                if m < S:
                    mark[m] = max(mark[m], gst[g])
    for s in range(S):
        if not mark[s]:
            sources[s].commit(target, pend[s][1])
    return records, mark, gst, (wrote_r, wrote_v, need_r, need_v)


def add_forwarded(groups, records):
    """AddUnique of the records, in order, into ForwardedGroupModel lists, in place -> (results, element statuses)"""
    results, status = [], [OK] * len(groups)
    for key, t, vals, sid, version, reserved in records:
        if key >= len(groups):
            results.append(ERR_INVALID_ARG)
            continue
        g = groups[key]
        if status[key] != OK:  # (add's stop rule: every later record of the element, whatever it holds)
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
        elif sid >= g.source_capacity or (ws not in g.windows and g.R is not None and len(g.windows) >= g.R):
            status[key] = ERR_CAPACITY
            results.append(ERR_CAPACITY)
        elif sid in g.seen_by(ws):
            results.append(ERR_DUPLICATE_SOURCE)
        else:
            if ws not in g.windows:
                g.seen[ws] = set()
            g.seen[ws].add(sid)
            for v in vals:
                g.windows.setdefault(ws, []).append(v)
            results.append(OK)
    return results, status
