"""The multi-block tile oracle (blocks_oracle_lib: each source block decoded on its own, the datapoints concatenated,
then the pinned window, element and encoder oracles) checked against the single-stream oracles it must reduce to,
and fileset.read_block_range on volumes written with write_fileset."""
import math
import os

import numpy as np

import agg_oracle_lib as A
import ann_oracle_lib as N
import blocks_oracle_lib as B
import elem_oracle_lib as E
import oracle_lib as O
from m3_b200 import fileset

SEC = 10 ** 9
STEP = 60 * SEC
N_WIN = 24
R0 = 1_700_000_040 * SEC            # range start (window-aligned)
BS = 7 * STEP + 13 * SEC            # source block size: not a multiple of the step, so windows straddle blocks
B0 = R0 - BS // 2                   # first block's start: block 0 begins before the range
AB, PS, INC, ADD, RST = 1, 2, 3, 4, 5
GAUGE, COUNTER = A.METRIC_GAUGE, A.METRIC_COUNTER
# (metric, types, ops): as the annotated tile tests' elements
ELEMENTS = [
    (GAUGE, [1], []),
    (COUNTER, [7], [RST]),
    (GAUGE, [2, 3, 7], [ADD]),
    (GAUGE, [1, 2, 3], []),
    (GAUGE, [8, 9], [RST, AB]),
    (COUNTER, [2, 3, 7], [INC, ADD]),
]


def encode(dps, int_opt, start):
    """(t, v, unit, annotation) -> one stream (b"" for none)"""
    enc = O.Encoder(int(start), int_opt)
    for t, v, u, a in dps:
        assert enc.encode(int(t), float(v), u, a) == 0
    return enc.stream() or b""


def block_points(rng, b, ann_pool=(), unit=O.UNIT_S, floats=False, nan_run=False, ooo=False, stray=False):
    """datapoints of source block b: in order inside the block, optionally a NaN run, an out-of-order datapoint,
    and a datapoint that falls in another block's windows or outside the range"""
    lo = B0 + b * BS
    gap = int(rng.integers(7, 50)) * SEC
    t = lo + int(rng.integers(0, 20)) * SEC
    if unit == O.UNIT_MS:
        t += int(rng.integers(1, 1000)) * 10 ** 6
    out = []
    while t < lo + BS:
        v = float(rng.integers(-50, 500))
        if floats:
            v += float(rng.random())
        out.append([t, v, unit, b""])
        t += gap
    if nan_run and len(out) > 4:
        for i in range(1, 4):
            out[i][1] = math.nan
    if ooo and len(out) > 3:
        out[1], out[2] = out[2], out[1]
    if stray and out:
        where = int(rng.choice([-3, 2, 40]))  # an earlier block's window, a later block's, past the range
        out.insert(len(out) // 2, [lo + where * BS // 2 + 17 * SEC, 3.0, O.UNIT_S, b""])
    for d in out:
        if ann_pool and rng.random() < 0.15:
            d[3] = ann_pool[int(rng.integers(0, len(ann_pool)))]
    return out


def random_series(rng, n_blocks, int_opt, annotations):
    """a series' block streams: missing (empty) blocks, unit and int / float changes between blocks, equal timestamps
    across a boundary, NaN runs, out-of-order and stray datapoints"""
    pool = [b"a", b"bb", bytes(range(40))] if annotations else []
    blocks, prev_last = [], None
    for b in range(n_blocks):
        if n_blocks > 2 and 0 < b < n_blocks - 1 and rng.random() < 0.2:
            blocks.append(b"")  # missing from a middle block
            prev_last = None
            continue
        unit = O.UNIT_MS if rng.random() < 0.2 else O.UNIT_S
        dps = block_points(rng, b, pool, unit=unit, floats=rng.random() < 0.4, nan_run=rng.random() < 0.3,
                           ooo=rng.random() < 0.3, stray=rng.random() < 0.2)
        if prev_last is not None and rng.random() < 0.3:
            dps.insert(0, [prev_last, 1.5, O.UNIT_S, b""])  # equal timestamps in two blocks
        blocks.append(encode(dps, int_opt, B0 + b * BS))
        prev_last = dps[-1][0] if dps[-1][0] >= B0 + b * BS else None
    return blocks


def plain_series(rng, n_blocks, int_opt):
    """blocks in seconds without annotations, empty blocks or stray datapoints: what one re-encoded stream holds
    exactly"""
    return [encode(block_points(rng, b, floats=rng.random() < 0.4, nan_run=rng.random() < 0.3,
                                ooo=rng.random() < 0.3), int_opt, B0 + b * BS) for b in range(n_blocks)]


def test_one_block_reduces_to_the_single_stream_oracles():
    rng = np.random.default_rng(1)
    for int_opt in (True, False):
        for _ in range(6):
            blk = random_series(rng, 1, int_opt, True)
            for metric, types, ops in ELEMENTS:
                for discard in (True, False):
                    s1, s2 = E.new_element_state(), E.new_element_state()
                    got = B.aggregate_tiles_blocks_series(blk, int_opt, R0, STEP, N_WIN, metric, types, ops, discard,
                                                          s1, True)
                    want = N.aggregate_tiles_annotated_series(blk[0], int_opt, R0, STEP, N_WIN, metric, types, ops,
                                                              discard, s2)
                    assert got == want and s1.tobytes() == s2.tobytes()
                    # without annotations: the multi-type oracle's datapoints
                    s3, s4 = E.new_element_state(), E.new_element_state()
                    rows, counts, err = B.aggregate_tiles_blocks_series(blk, int_opt, R0, STEP, N_WIN, metric, types,
                                                                        ops, discard, s3, False)
                    ts, vals, _, _ = N.decode_annotated(blk[0], int_opt)
                    res = E.aggregate_tiles_types_series(ts, vals, R0, STEP, N_WIN, metric, types, ops, discard, s4)
                    assert err == 0 and s3.tobytes() == s4.tobytes()
                    for j, (to, vo) in enumerate(res):
                        dt, dv, _, e = N.decode_annotated(rows[j], int_opt) if rows[j] else ([], [], [], 0)
                        assert counts[j] == len(to) and list(dt) == list(to)
                        assert np.array_equal(np.asarray(dv, dtype=np.float64).view(np.int64),
                                              np.asarray(vo, dtype=np.float64).view(np.int64))


def test_without_annotations_equals_the_concatenated_stream():
    rng = np.random.default_rng(2)
    for int_opt in (True, False):
        for n_blocks in (2, 5, 12):
            blk = plain_series(rng, n_blocks, int_opt)
            one = B.concat_stream(blk, int_opt, B0)
            for metric, types, ops in ELEMENTS:
                s1, s2 = E.new_element_state(), E.new_element_state()
                got = B.aggregate_tiles_blocks_series(blk, int_opt, R0, STEP, N_WIN, metric, types, ops, True, s1,
                                                      False)
                want = N.aggregate_tiles_annotated_series(one, int_opt, R0, STEP, N_WIN, metric, types, ops, True, s2)
                assert got == want and s1.tobytes() == s2.tobytes(), (n_blocks, metric, types, ops)


def boundary_annotation_case(int_opt):
    """block 0's first datapoint (before the range) and block 1's first (inside it) both carry b"gauge": each block's
    stream writes it, so window w1 keeps it; one stream re-encoding the concatenation writes it once, on block 0's
    first datapoint, and no window of the range has it.  -> (blocks, w1)"""
    d0 = [[B0 + 5 * SEC, 1.0, O.UNIT_S, b"gauge"]] + [[B0 + (5 + 30 * i) * SEC, float(i), O.UNIT_S, b""]
                                                       for i in range(1, 15)]
    d1 = [[B0 + BS + (9 + 30 * i) * SEC, float(i), O.UNIT_S, b"gauge" if i == 0 else b""] for i in range(15)]
    assert d0[0][0] < R0 <= d1[0][0]
    return [encode(d0, int_opt, B0), encode(d1, int_opt, B0 + BS)], (d1[0][0] - R0) // STEP


def test_block_first_annotation_is_kept():
    for int_opt in (True, False):
        blocks, w1 = boundary_annotation_case(int_opt)
        ts, _, anns, _ = B.decode_blocks(blocks, int_opt)
        ids = np.array([i if a else -1 for i, a in enumerate(anns)], dtype=np.int64)
        win = N.window_annotations(ts, ids, R0, STEP, N_WIN)
        one = B.concat_stream(blocks, int_opt, B0)
        ts1, _, anns1, _ = N.decode_annotated(one, int_opt)
        ids1 = np.array([i if a else -1 for i, a in enumerate(anns1)], dtype=np.int64)
        win1 = N.window_annotations(ts1, ids1, R0, STEP, N_WIN)
        assert [w for w in range(N_WIN) if win[w] != win1[w]] == [w1]
        assert anns[win[w1]] == b"gauge" and win1[w1] == -1
        got, _, _ = B.aggregate_tiles_blocks_series(blocks, int_opt, R0, STEP, N_WIN, GAUGE, [1], [], True,
                                                    E.new_element_state(), True)
        want, _, _ = N.aggregate_tiles_annotated_series(one, int_opt, R0, STEP, N_WIN, GAUGE, [1], [], True,
                                                        E.new_element_state())
        t_got, _, a_got, _ = N.decode_annotated(got[0], int_opt)
        t_want, _, a_want, _ = N.decode_annotated(want[0], int_opt)
        assert list(t_got) == list(t_want) and not any(a_want)
        assert [a for a in a_got if a] == [b"gauge"] and a_got[list(t_got).index(R0 + (w1 + 1) * STEP)] == b"gauge"


def test_corrupt_middle_block_is_the_error():
    rng = np.random.default_rng(3)
    blk = plain_series(rng, 5, True)
    bad = blk[:2] + [blk[2][: len(blk[2]) // 2]] + blk[3:]
    err_mid = N.decode_annotated(bad[2], True)[3]
    assert err_mid != 0
    st = E.new_element_state()
    rows, counts, err = B.aggregate_tiles_blocks_series(bad, True, R0, STEP, N_WIN, GAUGE, [1, 2], [], True, st, False)
    assert err == err_mid and rows == [b"", b""] and counts == [0, 0]
    assert st.tobytes() == E.new_element_state().tobytes()
    # empty blocks and no blocks: no datapoints, no error
    assert B.decode_blocks([b"", b""], True)[3] == 0 and B.decode_blocks([], True)[3] == 0


def _write_block(prefix, b, series, volume=0, tag_suffix=b""):
    ids = sorted(series)
    blob = b"".join(series[i] for i in ids)
    off = np.cumsum([0] + [len(series[i]) for i in ids[:-1]])
    fileset.write_fileset(prefix, "src", 3, B0 + b * BS, BS, ids, blob, off, [len(series[i]) for i in ids],
                          tags=[i + b"-tags" + tag_suffix for i in ids], volume=volume)


def test_read_block_range(tmp_path):
    rng = np.random.default_rng(4)
    prefix = str(tmp_path)
    streams = {}  # (id, block) -> bytes
    ids = [b"s%02d" % i for i in range(9)]
    for b in range(4):
        present = [i for k, i in enumerate(ids) if not (k % 3 == 1 and b in (1, 2)) and not (k == 8 and b == 0)]
        series = {i: encode(block_points(rng, b), True, B0 + b * BS) for i in present}
        if b == 2:  # two volumes of one block: the later one is the default
            _write_block(prefix, b, {i: encode(block_points(rng, b), True, B0 + b * BS) for i in present[:3]})
            _write_block(prefix, b, series, volume=1, tag_suffix=b"-v1")
        else:
            _write_block(prefix, b, series)
        for i, s in series.items():
            streams[(i, b)] = s
    r = fileset.read_block_range(prefix, "src", 3, [B0 + b * BS for b in range(4)])
    assert r.volumes == [0, 0, 1, 0]
    assert r.ids == sorted(ids) and len(r.block_off) == len(ids) + 1 and r.block_off[0] == 0
    for s, i in enumerate(r.ids):
        got = [bytes(r.data[o: o + n]) for o, n in zip(r.offsets[r.block_off[s]: r.block_off[s + 1]],
                                                       r.sizes[r.block_off[s]: r.block_off[s + 1]])]
        want = [streams[(i, b)] for b in range(4) if (i, b) in streams]  # block order, missing blocks left out
        assert got == want, i
        last = max(b for b in range(4) if (i, b) in streams)
        assert r.tags[s] == i + b"-tags" + (b"-v1" if last == 2 else b"")
    for q in range(len(r.offsets)):
        assert r.data_checksums[q] == fileset.adler32(bytes(r.data[r.offsets[q]: r.offsets[q] + r.sizes[q]]))
    # every block's data file lies at a 16-byte-aligned offset: a segment sits at (that base) + its index offset
    for s, i in enumerate(r.ids):
        q = int(r.block_off[s])
        for b in range(4):
            if (i, b) not in streams:
                continue
            fs = fileset.read_fileset(prefix, "src", 3, B0 + b * BS, r.volumes[b])
            k = fs.ids.index(i)
            assert (int(r.offsets[q]) - int(fs.offsets[k])) % 16 == 0, (i, b)
            q += 1
    # an explicit volume list: block 2's first volume holds three series
    r2 = fileset.read_block_range(prefix, "src", 3, [B0 + 2 * BS], volumes=[0])
    assert r2.volumes == [0] and len(r2.ids) == 3 and list(r2.block_off) == [0, 1, 2, 3]
