"""Timer element sets through a rollup that keep annotations on the GPU (m3tsz_element_set_forward_timer_annotated,
DESIGN.md §4.12), in both int_optimized modes: annotated Timer sources forwarded into annotated Timer groups with
random memberships (members listed twice, sources in several groups), two due windows per source and forward, the
group rows equal byte for byte to the CPU model (tests/element_timer_ann_model.py) and its reference encoder; the
annotation-capacity, open-window and sample-room stops, each with grow and a re-run of exactly the failed groups; the
plain forward's bytes without annotations; the host checks of the new call and the refusals in both directions; a run
on a caller's non-blocking stream behind a sleep."""
import ctypes as C

import numpy as np
import pytest
import torch

from element_timer_ann_model import AnnotatedTimerGroup, AnnotatedTimerSource, forward
from m3_b200 import capi
from test_gpu_element_timer_annotations import DEV, RES, START, _add, _random_cols, _rows

pytestmark = pytest.mark.gpu

SEC = 1_000_000_000
GROUP_TYPES = [capi.AGG_MAX, capi.AGG_P50, capi.AGG_P99]


@pytest.fixture(scope="module")
def codecs():
    from m3_b200.codec import BatchCodec
    return {True: BatchCodec(0, int_optimized=True), False: BatchCodec(0, int_optimized=False)}


def _sets(codec, S, G, capacity=64, g_capacity=64, R=4, g_R=4, g_cap=256):
    full = lambda n: torch.full((n,), START, dtype=torch.int64, device=DEV)
    src = codec.element_set(full(S), capi.METRIC_TIMER, [capi.AGG_P99], RES, open_windows=R, sample_capacity=64,
                            annotation_capacity=capacity, stride=0)
    grp = codec.element_set(full(G), capi.METRIC_TIMER, GROUP_TYPES, RES, open_windows=g_R, sample_capacity=g_cap,
                            annotation_capacity=g_capacity)
    return src, grp


def _models(S, G, int_opt, capacity=64, g_capacity=64, R=4, g_R=4, g_cap=256):
    sms = [AnnotatedTimerSource(capi.AGG_P99, RES, open_windows=R, capacity=capacity) for _ in range(S)]
    gms = [AnnotatedTimerGroup(GROUP_TYPES, RES, open_windows=g_R, sample_capacity=g_cap, capacity=g_capacity,
                               start_ns=START, int_optimized=int_opt) for _ in range(G)]
    return sms, gms


def _forward_and_check(src, grp, sms, gms, target, off, mem):
    d_off = torch.from_numpy(np.asarray(off, dtype=np.int64)).to(DEV)
    d_mem = torch.from_numpy(np.asarray(mem, dtype=np.int32)).to(DEV)
    sst, gst = src.forward_timer(target, d_off, d_mem, grp)
    want = forward(sms, gms, target, off, mem)
    assert (sst.cpu().tolist(), gst.cpu().tolist()) == want
    return want


def _consume_and_check(grp, gms, target):
    assert grp.consume(target).cpu().tolist() == [0] * len(gms)
    for m in gms:
        m.consume(target)
    rows, G = _rows(grp), grp.n_elements
    for g, m in enumerate(gms):
        for j, want in enumerate(m.streams()):
            assert rows[j * G + g] == want, (g, j)


def _random_run(codec, int_opt, rng, S=96, G=24):
    src, grp = _sets(codec, S, G)
    sms, gms = _models(S, G, int_opt)
    lens = rng.integers(0, 8, G)
    mem = rng.integers(0, S, int(lens.sum())).tolist()
    mem[-1] = mem[0]  # a member listed twice
    off = np.concatenate([[0], np.cumsum(lens)]).tolist()
    cols = _random_cols(rng, S, 4, p_ann=0.5)
    multi = 0
    for w in (0, 2):  # two windows per add, so each forward takes two due windows of a source
        _add(src, sms, [[r for r in c if w <= (r[0] - START) // RES < w + 2] for c in cols])
        multi += sum(len(m.forwarded(START + (w + 2) * RES)) > 1 for m in sms)
        _forward_and_check(src, grp, sms, gms, START + (w + 2) * RES, off, mem)
        _consume_and_check(grp, gms, START + (w + 2) * RES)
    assert multi > 0


@pytest.mark.parametrize("int_opt", [True, False])
def test_random_groups_equal_the_model(codecs, int_opt):
    _random_run(codecs[int_opt], int_opt, np.random.default_rng(21 + int_opt))


@pytest.mark.parametrize("int_opt", [True, False])
@pytest.mark.parametrize("stop", ["annotation", "open_windows", "samples"])
def test_capacity_stops_then_grow(codecs, int_opt, stop):
    """each capacity stop fails the group whole and holds its members back; growing that limit and re-running the
    failed group gives the model's result"""
    limits = {"annotation": dict(g_capacity=8), "open_windows": dict(g_R=1), "samples": dict(g_cap=2)}[stop]
    src, grp = _sets(codecs[int_opt], 3, 1, **limits)
    sms, gms = _models(3, 1, int_opt, **limits)
    cols = [[(START + SEC, 1.0, 0, b"short")], [(START + 2 * SEC, 2.0, 0, b"x" * 24)],
            [(START + RES + SEC, 3.0, 0, b"later")] if stop == "open_windows" else [(START + 3 * SEC, 3.0, 0, b"")]]
    _add(src, sms, cols)
    target = START + 2 * RES
    assert _forward_and_check(src, grp, sms, gms, target, [0, 3], [0, 1, 2]) == ([capi.ERR_CAPACITY] * 3,
                                                                                [capi.ERR_CAPACITY])
    assert int(grp.win["count"].sum()) == 0
    grp.grow(**{"annotation": dict(annotation_capacity=32), "open_windows": dict(open_windows=2),
                "samples": dict(sample_capacity=8)}[stop])
    for m in gms:
        m.capacity, m.m.R, m.m.cap = grp.annotation_capacity, grp.open_windows, grp.sample_capacity
    assert _forward_and_check(src, grp, sms, gms, target, [0, 3], [0, 1, 2]) == ([0] * 3, [0])
    _consume_and_check(grp, gms, target)


def test_plain_bytes_without_annotations(codecs):
    codec = codecs[True]
    rng = np.random.default_rng(23)
    S, G = 32, 8
    a_src, a_grp = _sets(codec, S, G)
    full = lambda n: torch.full((n,), START, dtype=torch.int64, device=DEV)
    p_src = codec.element_set(full(S), capi.METRIC_TIMER, [capi.AGG_P99], RES, sample_capacity=64, stride=0)
    p_grp = codec.element_set(full(G), capi.METRIC_TIMER, GROUP_TYPES, RES, sample_capacity=256)
    cols = _random_cols(rng, S, 1, p_ann=0.0)
    from test_gpu_element_timer_annotations import _inputs
    ts, vs, n, bt, ann = _inputs(cols)
    a_src.add(ts, vs, n, annotations=ann, batch=bt)
    p_src.add(ts, vs, n, batch=bt)
    off = torch.tensor([0, 4, 8, 8, 12, 16, 20, 28, 32], dtype=torch.int64, device=DEV)
    mem = torch.arange(S, dtype=torch.int32, device=DEV)
    ra, rp = a_src.forward_timer(START + RES, off, mem, a_grp), p_src.forward_timer(START + RES, off, mem, p_grp)
    assert all(torch.equal(x, y) for x, y in zip(ra, rp))
    assert torch.equal(a_grp.consume(START + RES), p_grp.consume(START + RES))
    assert _rows(a_grp) == _rows(p_grp)
    with pytest.raises(ValueError):  # an annotated group set needs an annotated source set
        p_src.forward_timer(START + RES, off, mem, a_grp)


def test_argument_checks_and_cross_refusals(codecs):
    codec = codecs[True]
    L = capi.lib()
    src, grp = _sets(codec, 4, 2)
    full = lambda n: torch.full((n,), START, dtype=torch.int64, device=DEV)
    g_src = codec.element_set(full(4), capi.METRIC_GAUGE, [capi.AGG_LAST], RES, annotation_capacity=8, stride=0)
    g_grp = codec.element_set(full(2), capi.METRIC_GAUGE, [capi.AGG_LAST], RES, annotation_capacity=8)
    off = torch.tensor([0, 2, 4], dtype=torch.int64, device=DEV)
    mem = torch.arange(4, dtype=torch.int32, device=DEV)
    sst, gst = torch.zeros(4, dtype=torch.int32, device=DEV), torch.zeros(2, dtype=torch.int32, device=DEV)
    h, o = codec.ctx.handle, C.byref(codec.opts)
    p = lambda t: C.c_void_p(t.data_ptr())
    cs = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def fwd(s_set, g_set, sa, ga, s_streams=None, g_streams=None):
        return L.m3tsz_element_set_forward_timer_annotated(
            h, o, C.byref(s_set._desc()), C.byref(s_streams or src._streams()), sa, START, p(off), p(mem), 4, 2,
            C.byref(g_set._desc()), C.byref(g_streams or grp._streams()), ga, p(sst), p(gst), cs)

    good_s, good_g = C.byref(src._ann()), C.byref(grp._ann())
    assert fwd(src, grp, good_s, good_g) == 0
    assert fwd(src, grp, None, good_g) == capi.ERR_INVALID_ARG
    assert fwd(src, grp, good_s, None) == capi.ERR_INVALID_ARG
    for field, bad in (("capacity", 12), ("capacity", 0), ("capacity", capi.MAX_ELEMENT_ANNOTATION + 8),
                       ("reserved", 1)):
        for which in ("src", "grp"):
            a = (src if which == "src" else grp)._ann()
            setattr(a, field, bad)
            args = (C.byref(a), good_g) if which == "src" else (good_s, C.byref(a))
            assert fwd(src, grp, *args) == capi.ERR_INVALID_ARG, (field, bad, which)
    a = grp._ann()
    a.d_len = src.ann_len.data_ptr()  # the group lengths over the source lengths
    assert fwd(src, grp, good_s, C.byref(a)) == capi.ERR_INVALID_ARG
    a = grp._ann()
    a.d_bytes = src.ann_bytes.data_ptr() + 8  # the group bytes inside the source bytes
    assert fwd(src, grp, good_s, C.byref(a)) == capi.ERR_INVALID_ARG
    # the new call refuses Gauge sets as source or group
    assert fwd(g_src, grp, C.byref(g_src._ann()), good_g) == capi.ERR_INVALID_ARG
    assert fwd(src, g_grp, good_s, C.byref(g_grp._ann())) == capi.ERR_INVALID_ARG
    # m3tsz_element_set_forward_annotated keeps refusing Timer sets
    assert L.m3tsz_element_set_forward_annotated(h, o, C.byref(src._desc()), good_s, START, p(off), p(mem), 4, 2,
                                                 C.byref(grp._desc()), good_g, p(sst), p(gst),
                                                 cs) == capi.ERR_INVALID_ARG
    torch.cuda.synchronize()
    with pytest.raises(ValueError):  # forward keeps refusing Timer sets
        src.forward(START, off, mem, grp)


def test_on_a_non_blocking_stream(codecs):
    torch.cuda.synchronize()
    s = torch.cuda.Stream()  # (torch creates its streams non-blocking)
    with torch.cuda.stream(s):
        torch.cuda._sleep(1_000_000)
        _random_run(codecs[False], False, np.random.default_rng(31), S=64, G=16)
