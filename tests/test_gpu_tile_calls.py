"""The host checks and launch bookkeeping that the seven tile aggregation entry points share: the window range each
call rejects before it launches anything, what a call with no series does, and how many launches a successful call
adds to m3tsz_ctx_launch_count."""
import ctypes as C

import pytest
import torch

import oracle_lib as O
from m3_b200 import capi
from test_gpu_transforms import N_WIN, R0, WIN, _batch, _csr

pytestmark = pytest.mark.gpu

S = 8
INT64_MAX = 2 ** 63 - 1
LAST, MIN, MAX, SUM = 1, 2, 3, 7
ADD = 4
CALLS = ["batch", "ex", "transform", "types", "annotated", "blocks", "blocks_annotated", "rollup"]
# fused decode, start fill, encode, status pass; + the longest-source read with annotations; the rollup adds its
# forward, fold and two-launch commit passes
LAUNCHES = {"batch": 4, "ex": 4, "transform": 4, "types": 4, "annotated": 5, "blocks": 4, "blocks_annotated": 5,
            "rollup": 8}


@pytest.fixture(scope="module")
def codec():
    from m3_b200.codec import BatchCodec
    return BatchCodec(0, int_optimized=True)


@pytest.fixture(scope="module")
def sources():
    blob, off, _ = _csr(_batch(True, S=S, damage=False))
    return blob, off


def i32s(*xs):
    return (C.c_int32 * len(xs))(*xs)


class Outputs:
    """packed outputs for 2 rows per series (the largest element below), *d_total_bytes set to a marker"""

    def __init__(self, codec, n_series):
        n = 2 * max(1, n_series)
        self.cap = n * (codec.encode_bound(N_WIN) + 4096)
        self.packed = torch.empty(self.cap, dtype=torch.uint8, device="cuda")
        self.offsets = torch.empty(n, dtype=torch.int64, device="cuda")
        self.out_len = torch.empty(n, dtype=torch.int64, device="cuda")
        self.status = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        self.n_tiles = torch.empty(n, dtype=torch.int32, device="cuda")
        self.total = torch.full((1,), 12345, dtype=torch.int64, device="cuda")
        self.src_status = torch.empty(max(1, n_series), dtype=torch.int32, device="cuda")

    def args(self, align):
        return (align, self.packed.data_ptr(), self.cap, self.offsets.data_ptr(), self.out_len.data_ptr(),
                self.status.data_ptr(), self.n_tiles.data_ptr(), self.total.data_ptr())


def call(codec, sources, name, n_series, start, step, n_win, out, align=64):
    """one call of entry point `name` over the first n_series sources; returns its status"""
    L, h, o = capi.lib(), codec.ctx.handle, C.byref(codec.opts)
    blob, off = sources
    src = (blob.data_ptr(), blob.numel(), off.data_ptr(), None)
    blocks = torch.arange(n_series + 1, dtype=torch.int64, device="cuda")  # one source block per series
    outs = out.args(align)
    if name == "batch":
        return L.m3tsz_aggregate_tiles_batch(h, o, *src, n_series, start, step, n_win, LAST, O.UNIT_S, *outs, None)
    if name == "ex":
        return L.m3tsz_aggregate_tiles_ex(h, o, *src, n_series, start, step, n_win, capi.METRIC_COUNTER, SUM,
                                          O.UNIT_S, *outs, None)
    if name == "transform":
        return L.m3tsz_aggregate_tiles_transform(h, o, *src, n_series, start, step, n_win, capi.METRIC_GAUGE, LAST,
                                                 O.UNIT_S, *outs, i32s(ADD), 1, 1, None, None)
    if name in ("types", "annotated"):
        fn = L.m3tsz_aggregate_tiles_types if name == "types" else L.m3tsz_aggregate_tiles_annotated
        return fn(h, o, *src, n_series, start, step, n_win, capi.METRIC_GAUGE, i32s(MIN, MAX), 2, O.UNIT_S, *outs,
                  i32s(ADD), 1, 1, None, None)
    if name in ("blocks", "blocks_annotated"):
        return L.m3tsz_aggregate_tiles_blocks(h, o, *src, n_series, blocks.data_ptr(), n_series, start, step, n_win,
                                              capi.METRIC_GAUGE, i32s(MIN, MAX), 2, O.UNIT_S, *outs, i32s(ADD), 1, 1,
                                              None, 1 if name == "blocks_annotated" else 0, None)
    assert name == "rollup"
    # group g is source g alone
    group_off = torch.arange(n_series + 1, dtype=torch.int64, device="cuda")
    members = torch.arange(max(1, n_series), dtype=torch.int32, device="cuda")
    return L.m3tsz_aggregate_tiles_rollup(h, o, *src, n_series, None, n_series, start, step, n_win,
                                          capi.METRIC_COUNTER, SUM, i32s(ADD), 1, group_off.data_ptr(),
                                          members.data_ptr(), n_series, n_series, i32s(MIN, MAX), 2, i32s(ADD), 1, 1,
                                          None, None, O.UNIT_S, *outs, out.src_status.data_ptr(), None)


BAD_WINDOWS = [
    (R0, WIN, 0),                                  # no window
    (R0, 0, N_WIN),                                # step 0
    (R0, -WIN, N_WIN),                             # negative step
    (INT64_MAX - N_WIN * WIN + 1, WIN, N_WIN),     # the range ends past INT64_MAX
]


@pytest.mark.parametrize("name", CALLS)
def test_bad_window_range_launches_nothing(codec, sources, name):
    out = Outputs(codec, S)
    n0 = codec.launch_count()
    for start, step, n_win in BAD_WINDOWS:
        assert call(codec, sources, name, S, start, step, n_win, out) == capi.ERR_INVALID_ARG, (start, step, n_win)
    assert codec.launch_count() == n0
    # the last range that fits is accepted
    assert call(codec, sources, name, S, INT64_MAX - N_WIN * WIN, WIN, N_WIN, out) == capi.OK


@pytest.mark.parametrize("name", CALLS)
def test_successful_call_launches(codec, sources, name):
    out = Outputs(codec, S)
    n0 = codec.launch_count()
    assert call(codec, sources, name, S, R0, WIN, N_WIN, out) == capi.OK
    torch.cuda.synchronize()
    assert codec.launch_count() - n0 == LAUNCHES[name]
    rows = S if name in ("batch", "ex", "transform") else 2 * S
    assert (out.status[:rows] == 0).all()


@pytest.mark.parametrize("name", [c for c in CALLS if c != "rollup"])
def test_no_series(codec, sources, name):
    """a single-element call with no series zeroes *d_total_bytes and returns OK before it looks at the windows or
    the packed outputs"""
    out = Outputs(codec, 0)
    n0 = codec.launch_count()
    for start, step, n_win in BAD_WINDOWS + [(R0, WIN, N_WIN)]:
        out.total.fill_(12345)
        assert call(codec, sources, name, 0, start, step, n_win, out, align=3) == capi.OK
        assert int(out.total.item()) == 0
    assert codec.launch_count() == n0


def test_rollup_no_series(codec, sources):
    """the rollup checks its windows even without sources, and its packed outputs only when it has rows"""
    out = Outputs(codec, 0)
    n0 = codec.launch_count()
    for start, step, n_win in BAD_WINDOWS:
        assert call(codec, sources, "rollup", 0, start, step, n_win, out) == capi.ERR_INVALID_ARG
    assert codec.launch_count() == n0
    out.total.fill_(12345)
    assert call(codec, sources, "rollup", 0, R0, WIN, N_WIN, out, align=3) == capi.OK
    torch.cuda.synchronize()
    assert int(out.total.item()) == 0
    assert codec.launch_count() - n0 == 4  # the forward pass, the fold and the commit's two launches


@pytest.mark.parametrize("name", CALLS)
def test_bad_packed_outputs_launch_nothing(codec, sources, name):
    out = Outputs(codec, S)
    n0 = codec.launch_count()
    for align in (0, 3, 128):
        assert call(codec, sources, name, S, R0, WIN, N_WIN, out, align=align) == capi.ERR_INVALID_ARG
    assert codec.launch_count() == n0
