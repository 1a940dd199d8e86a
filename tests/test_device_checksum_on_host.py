"""The segment-checksum kernel (m3_b200/csrc/m3tsz_checksum.cu, one warp per stream) run on the host from its CUDA
source: the 32 lanes of a warp are executed one after the other, lane 0 last; the only warp-collective piece, the
shuffle reduction `warp_sum_u64` (contract: lane 0 receives the warp's total), is restated as an accumulator.  The
lane-strided chunking, the dp4a partial sums, the head / tail handling and the final modular arithmetic are the
device source.  Compared with zlib.adler32 (= ts.Segment.CalculateChecksum, src/dbnode/ts/segment.go:60-76) for
every alignment and a range of lengths, CSR and (offset, size) addressing, expected-checksum mismatches."""
import ctypes as C
import zlib

import numpy as np
import pytest

from host_build import compile, constants, cut, source_text

# warp_sum_u64's contract -- lane 0 ends up with the sum over the warp -- for lanes executed 31, 30, .. 0
WARP_SUM = r"""
namespace m3tsz {
static thread_local uint64_t g_acc[2];
static thread_local int g_call;
static inline uint64_t warp_sum_u64(uint64_t v) { g_acc[g_call] += v; return g_acc[g_call++]; }
}
"""

DRIVER = r"""
extern "C" void dev_checksum(const uint8_t *streams, uint64_t streams_bytes, const uint64_t *offsets,
                             const uint64_t *lengths, uint64_t n_series, const uint32_t *expected, uint32_t *out,
                             int32_t *status) {
  using namespace m3tsz;
  ChecksumParams p;
  memset(&p, 0, sizeof(p));
  p.streams = streams; p.streams_bytes = streams_bytes; p.offsets = offsets; p.lengths = lengths;
  p.n_series = n_series; p.expected = expected; p.out = out; p.status = status;
  blockDim.x = CK_WARPS * 32;
  for (uint64_t s = 0; s < n_series; s++) {
    g_acc[0] = g_acc[1] = 0;
    for (int lane = 31; lane >= 0; lane--) {
      const uint64_t t = s * 32 + (uint64_t)lane;
      blockIdx.x = (unsigned)(t / blockDim.x);
      threadIdx.x = (unsigned)(t % blockDim.x);
      g_call = 0;
      checksum_kernel(p);
    }
  }
}
"""


@pytest.fixture(scope="module")
def dev():
    src = source_text("m3tsz_checksum.cu")
    body = src[src.index("namespace m3tsz {"): src.index("cudaError_t launch_checksum")] + "\n}  // namespace m3tsz\n"
    body = body.replace(cut(body, r"__device__[^\n;{]*\bwarp_sum_u64\s*\("), "// (warp_sum_u64: see WARP_SUM)\n")
    body = body.replace("#pragma unroll", "")
    params = "namespace m3tsz {\n%s\n%s\n}\n" % (constants(source_text("m3tsz_common.cuh"), "FULL_MASK"),
                                                 cut(source_text("m3tsz_kernels.h"), r"struct ChecksumParams"))
    assert "__shfl" not in body and "<<<" not in body
    lib = compile("dev_ck_host", WARP_SUM + params + body, DRIVER)
    lib.dev_checksum.restype = None
    return lib


def _run(dev, buf, offsets, lengths=None, expected=None):
    S = len(offsets) - 1 if lengths is None else len(lengths)
    out = np.zeros(S, dtype=np.uint32)
    st = np.zeros(S, dtype=np.int32)
    p = lambda a: None if a is None else C.c_void_p(a.ctypes.data)
    dev.dev_checksum(p(buf), C.c_uint64(len(buf)), p(offsets), p(lengths), C.c_uint64(S), p(expected), p(out), p(st))
    return out, st


def test_checksum_kernel_on_host_every_alignment_and_length(dev):
    rng = np.random.default_rng(1)
    lens = list(range(0, 70)) + [127, 128, 129, 511, 512, 513, 1000, 4096, 10_000, 65_521, 70_000]
    base = np.zeros(16 * 1024 * 1024 // 64, dtype=np.uint8)  # (only sized by need below)
    streams, offs, pos = [], [0], 0
    for n in lens:
        for align in range(16):
            pad = (align - pos) % 16
            pos += pad
            streams.append((pos, rng.integers(0, 256, size=n, dtype=np.uint8)))
            pos += n
            offs.append(pos)
    raw = np.zeros(pos + 32, dtype=np.uint8)
    # 16-byte aligned backing store so that `align` is the real address alignment
    store = np.zeros(len(raw) + 16, dtype=np.uint8)
    shift = (-store.ctypes.data) % 16
    buf = store[shift: shift + len(raw)]
    starts = np.zeros(len(streams), dtype=np.uint64)
    lengths = np.zeros(len(streams), dtype=np.uint64)
    for i, (o, d) in enumerate(streams):
        buf[o: o + len(d)] = d
        starts[i], lengths[i] = o, len(d)
    out, st = _run(dev, buf, starts, lengths)
    for i, (o, d) in enumerate(streams):
        assert out[i] == zlib.adler32(d.tobytes()), (i, len(d), o % 16)
    assert (st == 0).all()
    # expected checksums: one wrong entry is reported, the rest pass
    exp = out.copy()
    exp[7] ^= 1
    out2, st2 = _run(dev, buf, starts, lengths, expected=exp)
    assert st2[7] != 0 and (np.delete(st2, 7) == 0).all() and (out2 == out).all()


def test_checksum_kernel_on_host_csr_and_invalid_entries(dev):
    rng = np.random.default_rng(2)
    sizes = rng.integers(0, 3000, size=300)
    offs = np.zeros(len(sizes) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(sizes)
    store = np.zeros(int(offs[-1]) + 48, dtype=np.uint8)
    shift = (-store.ctypes.data) % 16
    buf = store[shift: shift + int(offs[-1]) + 16]
    buf[: int(offs[-1])] = rng.integers(0, 256, size=int(offs[-1]), dtype=np.uint8)
    out, st = _run(dev, buf[: int(offs[-1])], offs)
    for i in range(len(sizes)):
        assert out[i] == zlib.adler32(buf[int(offs[i]): int(offs[i + 1])].tobytes()), i
    assert (st == 0).all()
    # an entry that runs past the buffer is rejected, not read
    starts = np.array([0, 10], dtype=np.uint64)
    lengths = np.array([5, int(offs[-1])], dtype=np.uint64)
    out, st = _run(dev, buf[: int(offs[-1])], starts, lengths)
    assert st[0] == 0 and st[1] != 0 and out[1] == 0
