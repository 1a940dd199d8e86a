"""Independent pure-Python model of the reference's iterator layer above the codec -- encoding/iterators.go:56-262,
multi_reader_iterator.go:62-155, series_iterator.go:74-215 -- written as a direct object model (an Iterator per
decoded reader sequence, `iterators` with its `values` / `earliest` slices and swap-removal, MultiReaderIterator
over block slices, SeriesIterator over replicas with the [start, end) filter), cross-checked against the C merge
oracle (oracle/m3tsz_merge_oracle.c, itself pinned by the reference's table tests) on random fetch shapes:
replicas x block slices x readers per slice, duplicate timestamps with different values (the tie-break order
that swap-removal perturbs), empty readers, reader errors, out-of-order blocks, range filters, equal-timestamp
strategies -- also over NaN payloads, +-Inf and +-0, where the strategies' sort and frequency count follow Go's
comparison rules rather than Python's."""
import numpy as np
import pytest

import oracle_lib as O

TIME_MAX = (1 << 63) - 1
ERR_OUT_OF_ORDER = 13


class SeqIter:
    """a ReaderIterator over one decoded sequence; a decode error surfaces on the Next() after the last datapoint"""

    def __init__(self, ts, vals, err):
        self.ts, self.vals, self.fail = ts, vals, err
        self.i, self.err = -1, 0

    def next(self):
        if self.i + 1 < len(self.ts):
            self.i += 1
            return True
        self.i = len(self.ts)
        self.err = self.fail
        return False

    def current(self):
        return self.ts[self.i], self.vals[self.i]


def insertion_sort(items, less):
    """sort.Slice on <= 12 elements (the merge's limit) is Go's insertionSortLessFunc, in place: the order it leaves
    in `earliest` is where the next current() starts from.  With NaN values `less` is not a strict weak order, and
    this is the order Go produces, not Python's list.sort."""
    for i in range(1, len(items)):
        j = i
        while j > 0 and less(items[j], items[j - 1]):
            items[j], items[j - 1] = items[j - 1], items[j]
            j -= 1


class Iterators:  # iterators.go
    def __init__(self):
        self.values, self.earliest, self.earliest_at = [], [], TIME_MAX
        self.filtering, self.f_start, self.f_end = False, 0, 0
        self.strategy = 0

    def current(self):
        e = self.earliest
        val = lambda it: it.current()[1]
        if self.strategy == 1:    # IterateHighestValue: sort by <, take the last
            insertion_sort(e, lambda a, b: val(a) < val(b))
        elif self.strategy == 2:  # IterateLowestValue
            insertion_sort(e, lambda a, b: val(a) > val(b))
        elif self.strategy == 3:  # IterateHighestFrequencyValue
            # valueFrequencies is a map[float64]int: a key is found again only by ==, so +0 and -0 are one key and
            # a NaN key is never found again (every NaN increment adds a new entry; the lookup in `less` reads 0)
            freq = lambda it: sum(1 for o in e if val(o) == val(it))
            insertion_sort(e, lambda a, b: freq(a) < freq(b))
        return e[-1].current()

    def push(self, it):
        if self.filtering and not self.to_filter_next(it):
            return False
        self.values.append(it)
        self.try_add_earliest(it)
        return True

    def try_add_earliest(self, it):
        t = it.current()[0]
        if t == self.earliest_at:
            self.earliest.append(it)
        elif t < self.earliest_at:
            self.earliest = [it]
            self.earliest_at = t

    def to_filter_next(self, it):
        nxt = True
        while nxt:
            t = it.current()[0]
            if t < self.f_start:
                nxt = it.next()
                continue
            if t >= self.f_end:
                nxt = False
            break
        return nxt

    def move_to_valid_next(self):
        while True:
            prev_at = self.earliest_at
            n = len(self.values)
            for it in list(self.earliest):
                nxt = it.next()
                if nxt and self.filtering:
                    nxt = self.to_filter_next(it)
                if it.err:
                    self.reset()
                    return False, it.err
                if nxt:
                    continue
                idx = next(k for k, c in enumerate(self.values) if c is it)
                self.values[idx] = self.values[n - 1]
                self.values.pop()
                n -= 1
            self.earliest = []
            if n == 0:
                self.reset()
                return False, 0
            self.earliest_at = TIME_MAX
            for it in self.values:
                self.try_add_earliest(it)
            if self.filtering and not (self.f_start <= self.earliest_at < self.f_end):
                continue  # the reference recurses: moveToValidNext again
            if self.earliest_at < prev_at:
                self.reset()
                return False, ERR_OUT_OF_ORDER
            return True, 0

    def reset(self):
        self.values, self.earliest, self.earliest_at = [], [], TIME_MAX


class MultiReaderIter:  # multi_reader_iterator.go
    def __init__(self, slices):
        self.iters = Iterators()
        self.slices, self.k = slices, -1  # slicesIter: k = current slice
        self.err, self.first_next, self.has_slices = 0, True, True
        self.move_to_next()

    def has_next(self):
        return not self.err and (len(self.iters.values) > 0 or self.has_slices)

    def next(self):
        if not self.first_next:
            if not self.has_next():
                return False
            self.move_to_next()
        self.first_next = False
        return self.has_next()

    def current(self):
        return self.iters.current()

    def move_to_next(self):
        while True:
            if self.iters.values:
                self.move_iterators_to_next()
            if self.iters.values or self.err:
                return
            if self.k + 1 >= len(self.slices):
                self.has_slices = False
                return
            self.k += 1
            for it in self.slices[self.k]:
                if it.next():
                    self.iters.push(it)
                elif not self.err and it.err:
                    self.err = it.err
            if not self.iters.values and not self.err:
                continue
            return

    def move_iterators_to_next(self):
        while True:
            prev = self.iters.earliest_at
            nxt, err = self.iters.move_to_valid_next()
            if not self.err and err:
                self.err = err
                return
            if err or not nxt:
                return
            if self.iters.earliest_at != prev:
                return


def series_iterate(replicas, start, end, strategy):  # series_iterator.go
    iters = Iterators()
    err = 0
    if start != 0 and end != 0:
        iters.filtering, iters.f_start, iters.f_end = True, start, end
    iters.strategy = strategy
    for rep in replicas:
        if not rep.next() or not iters.push(rep):
            if rep.err:
                err = rep.err
    out = []
    first_next = True
    while True:
        if not first_next:
            if err or not iters.values:
                break
            while True:  # moveToNext
                prev = iters.earliest_at
                nxt, e = iters.move_to_valid_next()
                if e:
                    err = e
                    break
                if not nxt or iters.earliest_at != prev:
                    break
        first_next = False
        if err or not iters.values:
            break
        out.append(iters.current())
    return out, err


def _random_case(rng, n_series):
    seqs, n_points, status = [], [], []
    slice_off, replica_off, series_off = [0], [0], [0]
    base = 1_600_000_000 * 10 ** 9
    for _ in range(n_series):
        n_rep = int(rng.integers(0, 5))
        n_blocks = int(rng.integers(1, 4))
        block_len = 40 * 10 ** 9
        for _r in range(n_rep):
            order = list(range(n_blocks))
            if rng.random() < 0.08:
                order.reverse()  # out-of-order blocks: errOutOfOrderIterator
            for b in order:
                if rng.random() < 0.15:
                    slice_off.append(slice_off[-1])  # a slice with no readers
                    continue
                for _q in range(int(rng.integers(1, 4))):
                    n = int(rng.integers(0, 12))
                    t = np.sort(base + b * block_len + rng.integers(0, 40, size=n) * 10 ** 9)
                    t = np.unique(t)  # a reader's own timestamps are increasing
                    v = np.round(rng.normal(size=len(t)) * 3)  # few distinct values: ties for the strategies
                    seqs.append((t, v))
                    n_points.append(len(t))
                    status.append(int(rng.choice([0, 0, 0, 0, 0, 0, 1, 12])) if rng.random() < 0.2 else 0)
                slice_off.append(len(seqs))
            replica_off.append(len(slice_off) - 1)
        series_off.append(len(replica_off) - 1)
    cap = max([1] + n_points)
    ts = np.zeros((max(1, len(seqs)), cap), dtype=np.int64)
    vals = np.zeros((max(1, len(seqs)), cap), dtype=np.float64)
    for q, (t, v) in enumerate(seqs):
        ts[q, : len(t)], vals[q, : len(t)] = t, v
    return (seqs, ts, vals, np.array(n_points + ([] if seqs else [0]), dtype=np.uint32),
            np.array(status + ([] if seqs else [0]), dtype=np.int32), slice_off, replica_off, series_off, base)


# Values where the strategies' comparisons are subtle: NaN (three payloads, one of them negative) is neither < nor >
# anything and never equal to itself, the two zeros are ==, the infinities compare like numbers.
SPECIAL_BITS = np.array([0x7FF8000000000000, 0x7FF8000000000001, 0xFFF8000000000000, 0x7FF0000000000000,
                         0xFFF0000000000000, 0x0000000000000000, 0x8000000000000000], dtype=np.uint64)
SPECIAL_VALUES = SPECIAL_BITS.view(np.float64).tolist() + [1.0, -2.5, 3.0]
SPECIAL_START = 1_600_000_000 * 10 ** 9


def special_value_series(rng, n_series, replicas=(1, 12), readers=(1, 4), n_blocks=(1, 2)):
    """Series in the nested form of test_merge_oracle.build: replicas x block slices x readers x [(value, ts)].
    Timestamps come from a grid of 8 per block, so most of them are equal across replicas and across the readers of
    a slice; every value comes from SPECIAL_VALUES (bits kept: Python floats carry NaN payloads)."""
    series = []
    for _ in range(n_series):
        reps = []
        for _r in range(int(rng.integers(replicas[0], replicas[1] + 1))):
            slices = []
            for b in range(int(rng.integers(n_blocks[0], n_blocks[1] + 1))):
                rds = []
                for _q in range(int(rng.integers(readers[0], readers[1] + 1))):
                    slots = np.unique(rng.integers(0, 8, size=int(rng.integers(0, 9))))
                    rds.append([(SPECIAL_VALUES[int(rng.integers(0, len(SPECIAL_VALUES)))],
                                 SPECIAL_START + int(b * 8 + k) * 10 ** 9) for k in slots])
                slices.append(rds)
            reps.append(slices)
        series.append(reps)
    return series


SPECIAL_RANGE = (SPECIAL_START + 3 * 10 ** 9, SPECIAL_START + 12 * 10 ** 9)  # cuts into both blocks


def model_merge(series, start, end, strategy):
    """the object model over series in test_merge_oracle.build's nested form -> [(datapoints, err)] per series"""
    out = []
    for replicas in series:
        reps = []
        for slices in replicas:
            its = []
            for readers in slices:
                sl = []
                for rd in readers:
                    err = 0
                    if isinstance(rd, tuple):
                        rd, err = rd
                    sl.append(SeqIter([t for _, t in rd], [v for v, _ in rd], err))
                its.append(sl)
            reps.append(MultiReaderIter(its))
        out.append(series_iterate(reps, start, end, strategy))
    return out


def bits(values):
    return np.array(values, dtype=np.float64).view(np.uint64)


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("strategy", [0, 1, 2, 3])
def test_iterator_layer_model_matches_merge_oracle_on_special_values(seed, strategy):
    """NaN with payloads, +-Inf and +-0 at equal timestamps: the strategies' sort with < / > (false on NaN), the
    frequency count (0 for NaN, one key for +-0) and the insertion order they leave in `earliest`, 1 to 12 replicas,
    1 to 4 readers per slice, the range filter on and off; every value compared bit for bit."""
    from test_merge_oracle import build
    rng = np.random.default_rng(700 + seed * 11 + strategy)
    series = special_value_series(rng, 80)
    ts, vals, npts, st, slice_off, replica_off, series_off = build(series)
    ties = 0
    for start, end in ((0, 0), SPECIAL_RANGE):
        o_ts, o_val, o_n, o_st = O.series_merge_batch(ts, vals, npts, st, slice_off, replica_off, series_off,
                                                      start=start, end=end, strategy=strategy)
        for s, (out, err) in enumerate(model_merge(series, start, end, strategy)):
            assert int(o_st[s]) == err == 0, (s, int(o_st[s]), err)
            assert int(o_n[s]) == len(out), (s, int(o_n[s]), len(out))
            assert o_ts[s, : len(out)].tolist() == [p[0] for p in out], s
            assert (o_val[s, : len(out)].view(np.uint64) == bits([p[1] for p in out])).all(), s
            if not start:
                ties += len(out) < sum(len(rd) for r in series[s] for sl in r for rd in sl)
    assert ties > 40  # most series merge equal timestamps


@pytest.mark.parametrize("seed", range(8))
@pytest.mark.parametrize("strategy", [0, 1, 2, 3])
def test_iterator_layer_model_matches_merge_oracle(seed, strategy):
    rng = np.random.default_rng(500 + seed * 7 + strategy)
    n_series = 60
    seqs, ts, vals, n_points, status, slice_off, replica_off, series_off, base = _random_case(rng, n_series)
    for flt in (False, True):
        start, end = (base + 15 * 10 ** 9, base + 95 * 10 ** 9) if flt else (0, 0)
        o_ts, o_val, o_n, o_st = O.series_merge_batch(ts, vals, n_points, status, slice_off, replica_off, series_off,
                                                      start=start, end=end, strategy=strategy,
                                                      out_cap=max(1, int(n_points.sum())))
        errors = 0
        for s in range(n_series):
            reps = []
            for r in range(series_off[s], series_off[s + 1]):
                slices = []
                for k in range(replica_off[r], replica_off[r + 1]):
                    slices.append([SeqIter(seqs[q][0].tolist(), seqs[q][1].tolist(), int(status[q]))
                                   for q in range(slice_off[k], slice_off[k + 1])])
                reps.append(MultiReaderIter(slices))
            out, err = series_iterate(reps, start, end, strategy)
            assert int(o_st[s]) == err, (s, flt, int(o_st[s]), err)
            assert int(o_n[s]) == len(out), (s, flt, int(o_n[s]), len(out))
            assert o_ts[s, : len(out)].tolist() == [p[0] for p in out], (s, flt)
            assert o_val[s, : len(out)].tolist() == [p[1] for p in out], (s, flt)
            errors += err != 0
        assert errors > 0  # reader errors and out-of-order blocks are part of every case
