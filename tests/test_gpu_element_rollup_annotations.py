"""Element sets through a rollup that keep annotations on the GPU (m3tsz_element_set_forward_annotated, DESIGN.md
§4.12), in both int_optimized modes and both pipelines of tests/test_gpu_element_rollup.py, with contiguous and random
memberships: the reference's AddUnique annotation goldens through the device calls; annotated adds over 1, 2, 5 and 17
calls with forwards and annotated group consumes between them, equal to the CPU model (tests/element_rollup_ann_model.py)
byte for byte; byte identity with aggregate_tiles_rollup(annotations=True) where the two rules agree; the plain
calls' bytes when no datapoint carries an annotation; both CAPACITY retries; the argument checks; 100 k sources sampled
against the model; and a run on a non-blocking stream behind a sleep."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from element_rollup_ann_model import (ERR_CAPACITY, ERR_CLOSED, OK, AnnotatedGroup, AnnotatedSource,
                                       forward)
from element_set_ann_model import sparse_annotations
from m3_b200 import capi
from test_element_set_model import _bits
from test_gpu_element_annotations import _add
from test_gpu_element_annotations import _point_major as _ann_point_major
from test_gpu_element_rollup import (COUNTER, DEV, LAST, PIPES, RES, START, SUM, _dev, finite_series,
                                     memberships)
from test_gpu_element_rollup import sets as plain_sets
from test_gpu_elements import _point_major, _rows

pytestmark = pytest.mark.gpu

SEC = 1_000_000_000
COUNT = 6
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "m3tsz_rollup_annotation_goldens.json")
PROM = bytes([0x08, 0x01, 0x10, 0x01])  # annotation.Payload{COUNTER, HandleValueResets: true}
PAYLOADS = [b"", b"", PROM, b"gauge", bytes(range(1, 40))]


@pytest.fixture(scope="module")
def codecs():
    from m3_b200.codec import BatchCodec
    return {True: BatchCodec(0, int_optimized=True), False: BatchCodec(0, int_optimized=False)}


def ann_sets(codec, S, G, pipe, discard, R=8, src_R=8, src_cap=64, g_cap=64):
    metric, src_type, pre, types, post = pipe
    starts = lambda n: torch.full((n,), START, dtype=torch.int64, device=DEV)
    src = codec.element_set(starts(S), metric, [src_type], RES, transforms=pre, discard_nan=discard,
                            open_windows=src_R, stride=0, annotation_capacity=src_cap)
    grp = codec.element_set(starts(G), metric, types, RES, transforms=post, discard_nan=discard, open_windows=R,
                            annotation_capacity=g_cap)
    return src, grp


def ann_models(pipe, S, G, discard, int_opt, R=8, src_R=8, src_cap=64, g_cap=64):
    metric, src_type, pre, types, post = pipe
    return ([AnnotatedSource(metric, src_type, RES, pre, discard, open_windows=src_R, capacity=src_cap)
             for _ in range(S)],
            [AnnotatedGroup(metric, types, RES, post, discard, open_windows=R, capacity=g_cap, start_ns=START,
                            int_optimized=int_opt) for _ in range(G)])


def open_annotations(es):
    """{(element, window start): annotation} of an annotated set's open slots"""
    cnt, start = es.win["count"].cpu().numpy(), es.win["start"].cpu().numpy()
    ln, by = es.ann_len.cpu().numpy(), es.ann_bytes.cpu().numpy()
    return {(s, int(start[r, s])): by[r, s, : ln[r, s]].tobytes()
            for r in range(cnt.shape[0]) for s in range(cnt.shape[1]) if cnt[r, s]}


def model_annotations(models):
    return {(s, ws): m.ann[ws] for s, m in enumerate(models) for ws in m.m.windows}


def check_against(src, grp, sms, gms):
    rows, G, k = _rows(grp), grp.n_elements, len(grp.agg_types)
    for g, m in enumerate(gms):
        want = m.streams()
        for j in range(k):
            assert rows[j * G + g] == want[j], (g, j)
    for es, ms in ((src, sms), (grp, gms)):
        elem, wm = es.elem.cpu().numpy(), es.watermark.cpu().numpy()
        for s, m in enumerate(ms):
            assert elem[s].tobytes() == m.state.tobytes(), s
            assert int(wm[s]) == m.watermark, s
        assert open_annotations(es) == model_annotations(ms)


def annotated_cols(rng, cols, p=0.6):
    return [[(t, v, PAYLOADS[int(rng.integers(0, len(PAYLOADS)))] if rng.random() < p else b"") for t, v in c]
            for c in cols]


@pytest.mark.parametrize("int_opt", [True, False])
def test_goldens_through_the_device_calls(codecs, int_opt):
    """each golden step's values as new sources added and forwarded in order into one group that stays open across
    the steps; after each step the group slot's count, sum and annotation are what the reference asserts"""
    codec = codecs[int_opt]
    for case in json.load(open(GOLDEN))["cases"]:
        step, starts, metric = case["resolution_ns"], case["window_starts_ns"], case["metric_type"]
        pipe = (metric, SUM if metric == COUNTER else LAST, [], [COUNT, SUM], [])
        n = sum(len(st["values"]) for st in case["steps"])
        t0 = lambda k: torch.full((k,), starts[0], dtype=torch.int64, device=DEV)
        src = codec.element_set(t0(n), metric, [pipe[1]], step, open_windows=4, stride=0, annotation_capacity=64)
        grp = codec.element_set(t0(1), metric, [COUNT, SUM], step, open_windows=4, annotation_capacity=64)
        k = 0
        for st in case["steps"]:
            mem = list(range(k, k + len(st["values"])))
            ann = b"" if st["annotation"] is None else bytes.fromhex(st["annotation"])
            cols = [[] for _ in range(n)]
            for s, v in zip(mem, st["values"]):
                cols[s] = [(st["at_ns"], _bits(v), ann)]
            assert _add(src, cols)[1] == [0] * n
            k += len(mem)
            sst, gst = src.forward(starts[-1] + step, _dev(np.array([0, len(mem)])),
                                   _dev(np.array(mem, dtype=np.int32)), grp)
            assert int(sst.abs().sum()) == 0 and gst.tolist() == [OK]
            got = open_annotations(grp)
            cnt, start, sm = grp.win["count"].cpu().numpy(), grp.win["start"].cpu().numpy(), grp.win["sum"].cpu().numpy()
            for want in st["want"]:
                ws = starts[want["window"]]
                r = [r for r in range(4) if cnt[r, 0] and start[r, 0] == ws][0]
                if "count" in want:
                    assert cnt[r, 0] == want["count"] and sm[r, 0] == want["sum"], (case["name"], want)
                if "annotation" in want:
                    wa = b"" if want["annotation"] is None else bytes.fromhex(want["annotation"])
                    assert got[(0, ws)] == wa, (case["name"], want)


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("pipe", range(len(PIPES)))
@pytest.mark.parametrize("kind", ["contiguous", "random"])
@pytest.mark.parametrize("n_calls", [1, 2, 5, 17])
def test_adds_over_calls_equal_the_model(codecs, int_opt, pipe, kind, n_calls):
    """annotated adds split over n_calls calls, each followed by an annotated forward and an annotated group consume
    at a tick that moves with the calls (late datapoints to closed windows included): results, statuses, rows,
    records, watermarks and both sets' open-slot annotations equal the model"""
    codec = codecs[int_opt]
    rng = np.random.default_rng(3000 + 100 * pipe + 10 * n_calls + int_opt + (kind == "random") * 7)
    S, G, W = 60, 9, 8
    metric = PIPES[pipe][0]
    cols = annotated_cols(rng, [finite_series(rng, W, metric) for _ in range(S)])
    for c in cols:
        if c and rng.random() < 0.2:
            c.append((c[-1][0], _bits(float("nan")), b"nan"))  # an annotated NaN (discard_nan drops it)
    off, mem = memberships(rng, S, G, kind)
    if kind == "random":
        mem[5] = mem[4]  # a member listed twice
    discard = bool(n_calls % 2)
    src, grp = ann_sets(codec, S, G, PIPES[pipe], discard)
    sms, gms = ann_models(PIPES[pipe], S, G, discard, int_opt)
    cuts = [np.sort(rng.integers(0, len(c) + 1, n_calls - 1)).tolist() for c in cols]
    d_off, d_mem = _dev(off), _dev(mem)
    for call in range(n_calls):
        parts = [c[([0] + cuts[s] + [len(c)])[call]: ([0] + cuts[s] + [len(c)])[call + 1]] for s, c in enumerate(cols)]
        got = _add(src, parts)
        for s, m in enumerate(sms):
            assert (got[0][s], got[1][s]) == m.add(parts[s]), (call, s)
        target = START + ((call + 1) * W // n_calls) * RES
        sst, gst = src.forward(target, d_off, d_mem, grp)
        wst, wgst = forward(sms, gms, target, off, mem)
        assert sst.cpu().tolist() == wst and gst.cpu().tolist() == wgst, call
        assert set(wgst) <= {OK, ERR_CLOSED}
        if call % 2 == 0 or call + 1 == n_calls:  # (otherwise group windows stay open into the next call)
            assert int(grp.consume(target).abs().sum()) == 0
            for m in gms:
                m.consume(target)
        check_against(src, grp, sms, gms)


def tile_rollup_annotated(codec, cols, pipe, discard, off, mem, n_windows):
    """aggregate_tiles_rollup(annotations=True) over annotated streams of the same datapoints -> (bytes per row,
    source records, group records)"""
    metric, src_type, pre, types, post = pipe
    S, G = len(cols), len(off) - 1
    P = max([len(c) for c in cols] + [1])
    ts = np.zeros((S, P), dtype=np.int64)
    vb = np.zeros((S, P), dtype=np.uint64)
    for s, c in enumerate(cols):
        for i, (t, v, _) in enumerate(c):
            ts[s, i], vb[s, i] = t, v
    n = torch.tensor([len(c) for c in cols], dtype=torch.int32, device=DEV)
    ann = tuple(_dev(a) for a in sparse_annotations(cols))
    enc = codec.encode(_dev(ts), _dev(vb.view(np.float64)), torch.full((S,), START, dtype=torch.int64, device=DEV),
                       n_points=n, annotations=ann)
    assert int(enc.status.abs().sum()) == 0
    offs = torch.arange(S, dtype=torch.int64, device=DEV) * enc.out.shape[1]
    xs, gs = codec.transform_state(S), codec.element_state(G)
    out, _, sst = codec.aggregate_tiles_rollup(enc.out.view(-1), offs, START, RES, n_windows, src_type, _dev(off),
                                               _dev(mem), types, metric_type=metric, pre_transforms=pre,
                                               post_transforms=post, discard_nan=discard, src_state=xs,
                                               group_state=gs, lengths=enc.out_len, annotations=True)
    assert int(out.status.abs().sum()) == 0 and int(sst.abs().sum()) == 0
    packed = out.packed.cpu().numpy()
    o, ln = out.offsets.reshape(-1).cpu().numpy(), out.out_len.reshape(-1).cpu().numpy()
    return [packed[o[r]: o[r] + ln[r]].tobytes() for r in range(len(ln))], xs, gs


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("pipe", range(len(PIPES)))
@pytest.mark.parametrize("kind", ["contiguous", "random"])
def test_equals_aggregate_tiles_rollup_annotated(codecs, int_opt, pipe, kind):
    """Byte identity with aggregate_tiles_rollup(annotations=True) when every datapoint carries an annotation that
    differs from its source's previous one.  Why that suffices: the stream then writes every datapoint's annotation
    (it skips only a repeat of the last one written), so the tile call reads each datapoint's annotation as given, and
    a tile source window's annotation -- the last its stream wrote in the window -- is the last annotation added to
    the element window, which is the element set's rule; every forwarded window then carries one, so both folds take
    the last forwarded member's in listed order.  The adds come in stream order, and every forward happens at a tick
    after which no datapoint reaches an earlier window, so each group window takes all its values in one call, as the
    tile call's windows do.  (With a repeated annotation, or none, the tile source window may carry none where the
    element window keeps its last one, and across members in listed order the group window's annotation can differ.)"""
    codec = codecs[int_opt]
    rng = np.random.default_rng(4000 + 10 * pipe + int_opt + (kind == "random") * 7)
    S, G, W = 60, 9, 8
    metric = PIPES[pipe][0]
    cols = [[(t, v, b"a%d" % (i % 2) + bytes([s % 251])) for i, (t, v) in enumerate(finite_series(rng, W, metric))]
            for s in range(S)]
    off, mem = memberships(rng, S, G, kind)
    discard = bool(pipe)
    src, grp = ann_sets(codec, S, G, PIPES[pipe], discard)
    cuts = [np.sort(rng.integers(0, len(c) + 1, 2)).tolist() for c in cols]
    d_off, d_mem = _dev(off), _dev(mem)
    for call in range(3):
        parts = [c[([0] + cuts[s] + [len(c)])[call]: ([0] + cuts[s] + [len(c)])[call + 1]] for s, c in enumerate(cols)]
        assert int(np.abs(_add(src, parts)[1]).sum()) == 0
        pending = [c[([0] + cuts[s] + [len(c)])[call + 1]:] for s, c in enumerate(cols)]
        firsts = [p[0][0] - (p[0][0] - START) % RES for p in pending if p]
        if call < 2 and firsts:
            sst, gst = src.forward(min(firsts), d_off, d_mem, grp)
            assert int(sst.abs().sum()) == 0 and int(gst.abs().sum()) == 0
            assert int(grp.consume(min(firsts)).abs().sum()) == 0
    sst, gst = src.forward(START + W * RES, d_off, d_mem, grp)
    assert int(sst.abs().sum()) == 0 and int(gst.abs().sum()) == 0
    assert int(grp.consume(START + W * RES).abs().sum()) == 0
    want, xs, gs = tile_rollup_annotated(codec, cols, PIPES[pipe], discard, off, mem, W)
    assert _rows(grp) == want
    assert torch.equal(grp.elem, gs) and torch.equal(src.elem[:, :96], xs)


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("pipe", range(len(PIPES)))
def test_no_annotation_writes_the_plain_bytes(codecs, int_opt, pipe):
    """annotated sets whose datapoints carry none: the annotated forward and consume write the plain calls' rows,
    records and slots"""
    codec = codecs[int_opt]
    rng = np.random.default_rng(50 + pipe + int_opt)
    S, G, W = 40, 6, 6
    cols = [finite_series(rng, W, PIPES[pipe][0]) for _ in range(S)]
    off, mem = memberships(rng, S, G, "random")
    a_src, a_grp = ann_sets(codec, S, G, PIPES[pipe], False)
    p_src, p_grp = plain_sets(codec, S, G, PIPES[pipe], False)
    for tick in range(3):
        part = [[p for p in c if START + 2 * tick * RES <= p[0] < START + 2 * (tick + 1) * RES] for c in cols]
        _add(a_src, [[(t, v, b"") for t, v in c] for c in part])
        p_src.add(*_point_major(part))
        target = START + 2 * (tick + 1) * RES
        for src, grp in ((a_src, a_grp), (p_src, p_grp)):
            sst, gst = src.forward(target, _dev(off), _dev(mem), grp)
            assert int(sst.abs().sum()) == 0 and int(gst.abs().sum()) == 0
            assert int(grp.consume(target - RES * (tick % 2)).abs().sum()) == 0
    assert _rows(a_grp) == _rows(p_grp)
    for a, p in ((a_src, p_src), (a_grp, p_grp)):
        assert torch.equal(a.elem, p.elem) and torch.equal(a.watermark, p.watermark)
        for f in p.win:
            assert torch.equal(a.win[f], p.win[f]), f
    assert int(a_grp.ann_len.abs().sum()) == 0


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("pipe", range(len(PIPES)))
@pytest.mark.parametrize("stop", ["open_windows", "annotation_capacity"])
def test_capacity_stop_and_retry_of_the_failed_groups(codecs, int_opt, pipe, stop):
    """groups with too few open windows, or a forwarded annotation longer than their slots, fold nothing and hold
    their members back; growing and forwarding again with only the failed groups listed gives the bytes, records and
    slot annotations of one unstopped run"""
    codec = codecs[int_opt]
    rng = np.random.default_rng(77 + pipe + int_opt + (stop == "annotation_capacity") * 10)
    S, G, W = 48, 8, 5
    metric = PIPES[pipe][0]
    cols = annotated_cols(rng, [finite_series(rng, W, metric) for _ in range(S)], p=0.3)
    if stop == "annotation_capacity":  # a few sources bring a 39-byte payload into slots of 16 bytes
        for s in rng.choice(S, 4, replace=False):
            cols[s] = [(t, v, PAYLOADS[-1]) for t, v, _ in cols[s]]
    off, mem = memberships(rng, S, G, "random")
    small = dict(R=2) if stop == "open_windows" else dict(g_cap=16)
    src, grp = ann_sets(codec, S, G, PIPES[pipe], False, **small)
    want_src, want_grp = ann_sets(codec, S, G, PIPES[pipe], False, R=W, g_cap=64)
    for s_, g_ in ((src, grp), (want_src, want_grp)):
        assert int(np.abs(_add(s_, cols)[1]).sum()) == 0
    sst, gst = src.forward(START + W * RES, _dev(off), _dev(mem), grp)
    gst, sst = gst.cpu().numpy(), sst.cpu().numpy()
    failed = [g for g in range(G) if gst[g] != OK]
    assert failed and set(gst.tolist()) <= {OK, ERR_CAPACITY}
    held = {int(m) for g in failed for m in mem[off[g]: off[g + 1]]}
    assert {s for s in range(S) if sst[s] != OK} == held and set(sst[list(held)].tolist()) == {ERR_CAPACITY}
    grp.grow(open_windows=W) if stop == "open_windows" else grp.grow(annotation_capacity=64)
    lens = np.array([off[g + 1] - off[g] if g in failed else 0 for g in range(G)])
    off2 = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    mem2 = np.concatenate([mem[off[g]: off[g + 1]] for g in failed]).astype(np.int32)
    sst, gst = src.forward(START + W * RES, _dev(off2), _dev(mem2), grp)
    assert int(sst.abs().sum()) == 0 and int(gst.abs().sum()) == 0
    sst, gst = want_src.forward(START + W * RES, _dev(off), _dev(mem), want_grp)
    assert int(sst.abs().sum()) == 0 and int(gst.abs().sum()) == 0
    for s_, g_ in ((src, grp), (want_src, want_grp)):
        assert int(g_.consume(START + W * RES).abs().sum()) == 0
    assert _rows(grp) == _rows(want_grp)
    assert torch.equal(grp.elem, want_grp.elem) and torch.equal(src.elem, want_src.elem)
    assert torch.equal(src.watermark, want_src.watermark) and torch.equal(grp.watermark, want_grp.watermark)


def _forward_annotated(codec, src, grp, off, mem, sa, ga, target=START):
    st = torch.zeros(max(src.n_elements, grp.n_elements), dtype=torch.int32, device=DEV)
    return capi.lib().m3tsz_element_set_forward_annotated(
        codec.ctx.handle, C.byref(codec.opts), C.byref(src._desc()), sa, target, off.data_ptr(), mem.data_ptr(),
        mem.numel(), off.numel() - 1, C.byref(grp._desc()), ga, st.data_ptr(), st.data_ptr(), None)


def test_argument_checks(codecs):
    codec = codecs[True]
    pipe = (COUNTER, SUM, [], [SUM], [])
    src, grp = ann_sets(codec, 4, 2, pipe, False)
    off, mem = _dev(np.array([0, 2, 4])), _dev(np.array([0, 1, 2, 3], dtype=np.int32))
    ok = lambda: _forward_annotated(codec, src, grp, off, mem, C.byref(src._ann()), C.byref(grp._ann()))
    assert ok() == capi.OK
    # a plain source set cannot feed a group set that keeps annotations
    plain_src, _ = plain_sets(codec, 4, 2, pipe, False)
    with pytest.raises(ValueError):
        plain_src.forward(START, off, mem, grp)
    # an annotated source set feeds a plain group set through the plain call
    _, plain_grp = plain_sets(codec, 4, 2, pipe, False)
    assert int(src.forward(START, off, mem, plain_grp)[0].abs().sum()) == 0
    cases = {"NULL src_ann": (None, C.byref(grp._ann())), "NULL group_ann": (C.byref(src._ann()), None)}
    for name, field, value in (("capacity 12", "capacity", 12), ("capacity 0", "capacity", 0),
                               ("capacity above the maximum", "capacity", capi.MAX_ELEMENT_ANNOTATION + 8),
                               ("reserved", "reserved", 1), ("misaligned lengths", "d_len", grp.ann_len.data_ptr() + 2),
                               ("misaligned bytes", "d_bytes", grp.ann_bytes.data_ptr() + 4)):
        a = grp._ann()
        setattr(a, field, value)
        cases[name] = (C.byref(src._ann()), C.byref(a))
    alias = grp._ann()
    alias.d_bytes = src.ann_bytes.data_ptr()
    cases["group bytes over the source bytes"] = (C.byref(src._ann()), C.byref(alias))
    alias2 = src._ann()
    alias2.d_len = grp.ann_len.data_ptr()
    cases["source lengths over the group lengths"] = (C.byref(alias2), C.byref(grp._ann()))
    for name, (sa, ga) in cases.items():
        assert _forward_annotated(codec, src, grp, off, mem, sa, ga) == capi.ERR_INVALID_ARG, name
    # and the plain forward's own checks
    bad = codec.element_set(torch.full((3,), START, dtype=torch.int64, device=DEV), COUNTER, [SUM], RES,
                            annotation_capacity=64)
    with pytest.raises(capi.M3tszError):
        src.forward(START, off, mem, bad)


def test_invalid_and_closed_groups_against_the_model(codecs):
    codec = codecs[True]
    pipe = PIPES[1]
    S, G = 3, 3
    src, grp = ann_sets(codec, S, G, pipe, False)
    sms, gms = ann_models(pipe, S, G, False, True)
    for tick in range(2):
        cols = [[(START + tick * RES, _bits(1.0 + s), b"s%d" % s)] for s in range(S)]
        if tick:
            cols[2].append((START, _bits(9.0), b"late"))  # (source 2 consumed that window: the add refuses it)
        got = _add(src, cols)
        for s, m in enumerate(sms):
            assert (got[0][s], got[1][s]) == m.add(cols[s])
        off, mem = np.array([0, 2, 1, 4], dtype=np.int64), np.array([7, 0, 2, 2], dtype=np.int32)
        if tick:  # source 0, held back at tick 0, forwards its first window into group 2, which consumed it
            off, mem = np.array([0, 1, 2, 3], dtype=np.int64), np.array([1, 2, 0], dtype=np.int32)
        target = START + (tick + 1) * RES
        sst, gst = src.forward(target, _dev(off), _dev(mem), grp)
        wst, wgst = forward(sms, gms, target, off, mem)
        assert gst.cpu().tolist() == wgst and sst.cpu().tolist() == wst
        assert int(grp.consume(target).abs().sum()) == 0
        for m in gms:
            m.consume(target)
        check_against(src, grp, sms, gms)
    assert wgst[2] == ERR_CLOSED


def test_large_set_sampled(codecs):
    """100 k sources, 10 k groups of 10 random members, the Prometheus payload or another on every datapoint;
    sampled groups' rows against the model"""
    codec = codecs[True]
    pipe = PIPES[0]
    rng = np.random.default_rng(21)
    S, G, W = 100_000, 10_000, 3
    off = np.arange(0, G * 10 + 1, 10, dtype=np.int64)
    mem = rng.integers(0, S, G * 10).astype(np.int32)
    src, grp = ann_sets(codec, S, G, pipe, True, R=4, src_R=4, src_cap=64, g_cap=64)
    n = rng.integers(0, 4, (W, S))
    P = int(n.sum(0).max())
    ts = np.zeros((P, S), dtype=np.int64)
    vals = np.zeros((P, S), dtype=np.float64)
    counts = np.zeros(S, dtype=np.int32)
    pay = [PROM, b"gauge", bytes(range(1, 40))]
    which = rng.integers(0, len(pay), (P, S))
    for w in range(W):
        for s in np.nonzero(n[w])[0]:
            for _ in range(n[w, s]):
                ts[counts[s], s] = START + w * RES + int(rng.integers(0, 60)) * SEC
                vals[counts[s], s] = float(rng.integers(0, 1000))
                counts[s] += 1
    # the sparse list: every datapoint annotated, dp_index counting the element's rows
    series_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    ent = np.zeros(int(counts.sum()), dtype=[("dp_index", "<u4"), ("length", "<u4"), ("byte_offset", "<u8")])
    lens = np.array([len(p) for p in pay])
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    for s in range(S):
        k = np.arange(counts[s])
        sl = slice(series_off[s], series_off[s + 1])
        ent["dp_index"][sl], ent["length"][sl], ent["byte_offset"][sl] = k, lens[which[k, s]], offs[which[k, s]]
    blob = np.frombuffer(b"".join(pay), dtype=np.uint8).copy()
    ann = (_dev(series_off), _dev(ent.view(np.uint8).reshape(-1, 16)), _dev(blob))
    res, st = src.add(_dev(ts), _dev(vals), _dev(counts), annotations=ann)
    assert int(st.abs().sum()) == 0
    sst, gst = src.forward(START + W * RES, _dev(off), _dev(mem), grp)
    assert int(sst.abs().sum()) == 0 and int(gst.abs().sum()) == 0
    assert int(grp.consume(START + W * RES).abs().sum()) == 0
    rows = _rows(grp)
    for g in sorted(rng.choice(G, 40, replace=False).tolist()):
        members = [int(m) for m in mem[off[g]: off[g + 1]]]
        uniq = sorted(set(members))
        sms, gms = ann_models(pipe, len(uniq), 1, True, True, R=4, src_R=4)
        for i, s in enumerate(uniq):
            k = int(counts[s])
            assert sms[i].add([(int(ts[j, s]), _bits(vals[j, s]), pay[which[j, s]]) for j in range(k)])[1] == OK
        forward(sms, gms, START + W * RES, [0, len(members)], [uniq.index(m) for m in members])
        gms[0].consume(START + W * RES)
        assert rows[g] == gms[0].streams()[0], g


def test_non_blocking_stream_behind_a_sleep(codecs):
    """annotated adds and an annotated forward on a non-blocking pool stream behind a sleep: the calls return before
    the stream runs them, and the results, with an annotated consume after them, equal the same run on the default
    stream byte for byte"""
    codec = codecs[True]
    pipe = PIPES[0]
    rng = np.random.default_rng(9)
    S, G, W = 200, 20, 4
    cols = annotated_cols(rng, [finite_series(rng, W, COUNTER) for _ in range(S)])
    off, mem = memberships(rng, S, G, "random")

    def inputs():  # (device copies made before the sleep: a pageable copy would wait for the stream)
        return ann_sets(codec, S, G, pipe, False) + (_ann_point_major(cols), _dev(off), _dev(mem))

    def run(src, grp, pm, d_off, d_mem):
        src.add(*pm[:3], annotations=pm[3])
        return src.forward(START + W * RES, d_off, d_mem, grp)

    ref_in = inputs()
    ref = run(*ref_in)
    assert int(ref_in[1].consume(START + W * RES).abs().sum()) == 0
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        got_in = inputs()
        side.synchronize()
        torch.cuda._sleep(1_000_000_000)
        got = run(*got_in)
        assert not side.query(), "the add or the forward waited for its stream"
        status = got_in[1].consume(START + W * RES)
    side.synchronize()
    assert int(status.abs().sum()) == 0
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
    assert _rows(got_in[1]) == _rows(ref_in[1])
    for a, b in ((got_in[0], ref_in[0]), (got_in[1], ref_in[1])):
        sa, sb = a.state(), b.state()
        assert torch.equal(sa["elem"], sb["elem"]) and torch.equal(sa["watermark"], sb["watermark"])
        assert torch.equal(sa["ann_len"], sb["ann_len"]) and torch.equal(sa["ann_bytes"], sb["ann_bytes"])
        for f in sa["win"]:
            assert torch.equal(sa["win"][f], sb["win"][f])
