"""An independent pure-Python restatement of the aggregator's Timer (aggregation/timer.go) over the CM stream
(aggregation/quantile/cm/stream.go, heap.go), written from the reference's semantics without looking at the C oracle
(tests/timer_oracle.c) or the device code; the tests require the three to agree bit for bit.  Test infrastructure only.

The sorted list is a Python list of [value, num_ranks, delta] entries with cursors as positions (the reference's
linked list and arena are not observable); the pending minHeaps are plain Python lists pushed and heapsorted exactly
as heap.go does, because where -0 / +0 and NaN samples land depends on their array order."""
import math
import struct

NAN_GO = struct.unpack("<d", struct.pack("<Q", 0x7FF8000000000001))[0]  # math.NaN()
NAN_INVALID = struct.unpack("<d", struct.pack("<Q", 0xFFF8000000000000))[0]  # amd64's invalid-operation NaN

TYPE_QUANTILE = {5: 0.5, 10: 0.1, 11: 0.2, 12: 0.3, 13: 0.4, 14: 0.5, 15: 0.6, 16: 0.7, 17: 0.8, 18: 0.9, 19: 0.95,
                 20: 0.99, 21: 0.999, 22: 0.9999, 23: 0.25, 24: 0.75}


def go_int64(f):
    """int64(f) on amd64: truncation; NaN and out of range give math.MinInt64"""
    if not (-9223372036854775808.0 <= f < 9223372036854775808.0):
        return -(1 << 63)
    return int(f)


def pooled_quantiles(types):
    """Types.PooledQuantiles: quantile types in listed order, Median and P50 deduplicated"""
    out, median = [], False
    for t in types:
        if t not in TYPE_QUANTILE:
            continue
        if t in (5, 14):
            if median:
                continue
            median = True
        out.append(TYPE_QUANTILE[t])
    return out


def _push(h, v):
    h.append(v)
    i = len(h) - 1
    while i > 0:
        p = (i - 1) // 2
        if h[p] <= h[i]:
            break
        h[p], h[i] = h[i], h[p]
        i = p


def _sort_desc(h):
    n = len(h) - 1
    while n > 0:
        h[0], h[n] = h[n], h[0]
        i = small = 0
        while True:
            left = 2 * small + 1
            right = left + 1
            if left < n and h[left] < h[small]:
                small = left
            if right < n and h[right] < h[small]:
                small = right
            if small == i:
                break
            h[i], h[small] = h[small], h[i]
            i = small
        n -= 1


class Stream:
    """cm.Stream of one window.  `size()` is its list samples plus pending values."""

    def __init__(self, quantiles, eps=1e-3, every=1024):
        self.q, self.eps, self.every = list(quantiles), float(eps), int(every)
        self.samples = []  # [value, num_ranks, delta]
        self.less, self.more = [], []
        self.ins = None  # insert cursor: an index into samples, None for nil
        self.comp = None  # compress cursor
        self.n_values = 0
        self.comp_min_rank = 0
        self.counter = 0
        self.computed = [0.0] * len(self.q)

    def size(self):
        return len(self.samples) + len(self.less) + len(self.more)

    def _reset_cursor(self):
        self.less, self.more = self.more, self.less
        self.ins = 0

    def _threshold(self, rank):
        out, eps = (1 << 63) - 1, 2.0 * self.eps
        n = self.n_values
        for q in self.q:
            if rank >= go_int64(q * float(n)):
                m = go_int64(eps * float(rank) / q)
            else:
                m = go_int64(eps * float(n - rank) / (1.0 - q))
            out = min(out, m)
        return out

    def _insert(self):
        comp_value = self.samples[self.comp][0] if self.comp is not None else float("nan")
        _sort_desc(self.more)
        vals = self.more
        idx = len(vals) - 1
        s = self.samples
        pos = self.ins
        while pos is not None and pos < len(s):
            cur = s[pos]
            while idx >= 0 and vals[idx] <= cur[0]:
                v = vals[idx]
                idx -= 1
                s.insert(pos, [v, 1, cur[1] + cur[2] - 1])
                pos += 1
                if self.comp is not None and self.comp >= pos - 1:
                    self.comp += 1
                if comp_value >= v:
                    self.comp_min_rank += 1
                self.n_values += 1
            pos += 1
        while idx >= 0 and vals[idx] >= s[-1][0]:
            s.append([vals[idx], 1, 0])
            idx -= 1
            self.n_values += 1
        self.more = []
        self._reset_cursor()

    def _compress(self):
        s = self.samples
        if len(s) < 3:
            return
        if self.comp is None:
            c = len(s) - 2
            self.comp_min_rank = self.n_values - 1 - s[c][1]
            self.comp = c - 1
        while self.comp != 0:
            c = self.comp
            cur, nxt = s[c], s[c + 1]
            max_rank = self.comp_min_rank + cur[1] + cur[2]
            thr = self._threshold(max_rank)
            self.comp_min_rank -= cur[1]
            if cur[1] + nxt[1] + nxt[2] <= thr:
                if self.ins == c:
                    self.ins = c  # the next sample moves into position c
                elif self.ins is not None and self.ins > c:
                    self.ins -= 1
                nxt[1] += cur[1]
                del s[c]
            self.comp = c - 1
        self.comp = None

    def add_batch(self, values):
        values = list(values)
        if not values:
            return
        if not self.samples:
            self.samples.append([values[0], 1, 0])
            self.ins = 0
            self.n_values += 1
            values = values[1:]
        ipv = self.samples[self.ins][0]
        counter = self.counter
        for v in values:
            _push(self.less if v < ipv else self.more, v)
            if counter == self.every:
                self._insert()
                self._compress()
                counter = 0
            counter += 1
        self.counter = counter

    def flush(self):
        while self.less or self.more:
            if not self.more:
                self._reset_cursor()
            self._insert()
            self._compress()
        self._calc()

    def _calc(self):
        if not self.q or self.n_values == 0:
            return
        s = self.samples
        if self.n_values <= 3:
            buf = [x[0] for x in s]
            for i, q in enumerate(self.q):
                idx = go_int64(q * float(len(buf)))
                self.computed[i] = buf[min(idx, len(buf) - 1)]
            return
        ranks = [go_int64(math.ceil(q * float(self.n_values))) for q in self.q]
        thrs = [go_int64(math.ceil(float(self._threshold(r)) / 2.0)) for r in ranks]
        min_rank = max_rank = 0
        idx, prev = 0, 0
        for pos in range(len(s)):
            if idx >= len(self.q):
                break
            max_rank = min_rank + s[pos][1] + s[pos][2]
            if max_rank > ranks[idx] + thrs[idx] or min_rank > ranks[idx]:
                self.computed[idx] = s[prev][0]
                idx += 1
            min_rank += s[pos][1]
            prev = pos
        for i in range(idx, len(self.q)):
            if max_rank >= ranks[i] + thrs[i] or min_rank > ranks[i]:
                self.computed[i] = s[prev][0]

    def quantile(self, q):
        if not self.samples:
            return 0.0
        if q == 0.0:
            return self.samples[0][0]
        if q == 1.0:
            return self.samples[-1][0]
        for i, qt in enumerate(self.q):
            if qt >= q:
                return self.computed[i]
        return NAN_GO


class Timer:
    """aggregation.Timer of one window with the element's types"""

    def __init__(self, types, eps=1e-3, every=1024):
        self.types = list(types)
        self.stream = Stream(pooled_quantiles(self.types), eps, every)
        self.count, self.sum, self.sum_sq = 0, 0.0, 0.0

    def add_batch(self, values):
        values = [float(v) for v in values]
        self.count += len(values)
        for v in values:
            self.sum += v
            self.sum_sq += v * v
        self.stream.add_batch(values)

    def values(self):
        """ValueOf of every type, after Flush"""
        self.stream.flush()
        out = []
        for t in self.types:
            if t in TYPE_QUANTILE:
                out.append(self.stream.quantile(TYPE_QUANTILE[t]))
            elif t == 2:
                out.append(self.stream.quantile(0.0))
            elif t == 3:
                out.append(self.stream.quantile(1.0))
            elif t == 4:
                out.append(0.0 if self.count == 0 else self.sum / float(self.count))
            elif t == 6:
                out.append(float(self.count))
            elif t == 7:
                out.append(self.sum)
            elif t == 8:
                out.append(self.sum_sq)
            elif t == 9:
                div = self.count * (self.count - 1)
                if div == 0:
                    out.append(0.0)
                else:
                    x = (float(self.count) * self.sum_sq - self.sum * self.sum) / float(div)
                    out.append(x if x != x else NAN_INVALID if x < 0 else math.sqrt(x))
            else:
                out.append(0.0)
        return out
