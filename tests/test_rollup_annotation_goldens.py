"""The reference's AddUnique tests of a rollup element's annotation (tests/golden/m3tsz_rollup_annotation_goldens.json,
written by scripts/make_goldens.py) driven through the composed oracle of m3tsz_aggregate_tiles_rollup_annotated
(rollup_ann_oracle_lib).  Every forwarded value becomes one source series with one datapoint at the step's time,
carrying the step's annotation; after step k the group is the sources of steps 0..k in order, rolled up with
[Count, Sum].  What the test asserts after each step must hold for the rolled-up rows: the window's sum and count,
and the annotation in effect at the window's datapoint, as the reference iterator reads it back."""
import json
import os

import numpy as np
import pytest

import ann_oracle_lib as N
import elem_oracle_lib as E
import oracle_lib as O
import rollup_ann_oracle_lib as RA
import xf_oracle_lib as X

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "m3tsz_rollup_annotation_goldens.json")
SEC = 10 ** 9
COUNT, SUM, LAST = 6, 7, 1
COUNTER = 1


def _cases():
    return json.load(open(GOLDEN))["cases"]


def _stream(t, v, a):
    enc = O.Encoder(200 * SEC, True)
    assert enc.encode(int(t), float(v), O.UNIT_S, a) == 0
    return enc.stream()


def _ann(h):
    return b"" if h is None else bytes.fromhex(h)


@pytest.mark.parametrize("case", _cases(), ids=lambda c: c["name"])
def test_goldens_through_the_composed_oracle(case):
    step, starts = case["resolution_ns"], case["window_starts_ns"]
    r0, n_win = starts[0], len(starts)
    src_type = SUM if case["metric_type"] == COUNTER else LAST
    streams, upto = [], []
    for st in case["steps"]:
        for v in st["values"]:
            streams.append(_stream(st["at_ns"], v, _ann(st["annotation"])))
        upto.append(len(streams))
    decoded = RA.decode_sources(streams, True, blocks=False)
    for k, st in enumerate(case["steps"]):
        n = upto[k]
        off, mem = np.array([0, n], dtype=np.int64), np.arange(n, dtype=np.int32)
        rows, src = RA.aggregate_tiles_rollup_annotated(decoded[:n], True, r0, step, n_win, case["metric_type"],
                                                        src_type, [], off, mem, [COUNT, SUM], [], False,
                                                        np.zeros(n, X.XF_STATE_DTYPE), np.zeros(1, E.ELEM_STATE_DTYPE))
        assert src == [0] * n and rows[0][0][0] == 0 and rows[1][0][0] == 0
        out = {}
        for j, name in ((0, "count"), (1, "sum")):
            ts, vals, anns, err = N.decode_annotated(rows[j][0][1], True)
            assert err == 0
            out[name] = (ts.tolist(), vals.tolist(), anns)
        for want in st["want"]:
            w = want["window"]
            t = starts[w] + step  # the tile's timestamp: the window's end
            for name in ("count", "sum"):
                ts, vals, anns = out[name]
                i = ts.index(t)
                if name in want:
                    assert vals[i] == float(want[name]), (case["name"], k, want, name)
                if "annotation" in want:
                    # the encoder writes an annotation only when it differs from the last one written
                    in_effect = next((a for a in reversed(anns[: i + 1]) if a), b"")
                    assert in_effect == _ann(want["annotation"]), (case["name"], k, want, name)


@pytest.mark.parametrize("case", _cases(), ids=lambda c: c["name"])
def test_goldens_through_the_selection(case):
    """the composed oracle's selection alone: each step's source forwards its values to its window with its
    annotation, members in step order"""
    step, starts = case["resolution_ns"], case["window_starts_ns"]
    fwd, src_ann = [], []
    for k, st in enumerate(case["steps"]):
        w = (st["at_ns"] - starts[0]) // step
        fwd.append({w: st["values"][-1]})
        src_ann.append({w: _ann(st["annotation"])} if st["annotation"] else {})
        for want in st["want"]:
            if "annotation" in want:
                got = RA.group_annotation(fwd, src_ann, list(range(k + 1)), want["window"])
                assert got == _ann(want["annotation"]), (case["name"], k, want)


def test_a_later_forward_without_annotation_keeps_the_earlier():
    """the rule the goldens pin (a later forward with none keeps the annotation), inside one window"""
    fwd = [{0: 1.0}, {0: 2.0}, {0: 3.0}]
    src_ann = [{0: b"x"}, {}, {0: b""}]
    assert RA.group_annotation(fwd, src_ann, [0, 1, 2], 0) == b"x"
    assert RA.group_annotation(fwd, src_ann, [1, 2], 0) == b""
