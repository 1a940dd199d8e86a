"""Fileset data/index ingestion (SURVEY.md §8f row N2): maps the reference's on-disk
fileset -- /root/reference/src/dbnode/persist/fs/{write.go,read.go,files.go,fs.go},
msgpack schema persist/fs/msgpack/{schema.go,encoder.go}, persist/schema/types.go:40-78 --
onto the batch decoder's inputs with zero re-packing:

    data file   = the series' streams back to back            -> d_streams (as is)
    index entry = (Index, ID, Size, Offset, DataChecksum, EncodedTags, IndexChecksum)
                                                               -> d_offsets / d_lengths / expected Adler-32

so a fileset is uploaded once, its segment checksums are verified ON THE DEVICE
(m3tsz_checksum_batch, what persist/fs/read.go:395-397 does per entry on the CPU) and it is
decoded by ONE m3tsz_decode_batch_ex launch.  The msgpack framing of the small metadata files
(info / index / digest / checkpoint) is host control plane and is parsed here in Python; only the
framing is restated (positive/negative fixint, (u)int8..64, bin8..32, fixarray / array16), nothing
of the codec.  `write_fileset` produces the same files (used by the tests and by the benchmark tool
to persist GPU-encoded blocks; volume layout of persist/fs/files.go:1729-1737):

    <prefix>/data/<namespace>/<shard>/fileset-<blockStartNanos>-<volume>-{info,index,data,digest,checkpoint,...}.db
"""
import os
import struct
import zlib
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np

# msgpack/schema.go:44-72,96-112
_VERSION = 1
_ROOT, _INDEX_INFO, _SUMMARIES_INFO, _BLOOM_INFO, _INDEX_ENTRY = 1, 2, 3, 4, 5
_N_ROOT, _N_INDEX_INFO, _N_INDEX_ENTRY = 2, 11, 7
MAJOR_VERSION, MINOR_VERSION = 1, 1  # persist/schema/types.go:32-37
_SUFFIXES = ("info", "index", "summaries", "bloomfilter", "data", "digest", "checkpoint")


def adler32(b) -> int:
    """digest.Checksum (src/dbnode/digest/digest.go:36-38) = hash/adler32 (m3db/stackadler32)."""
    return zlib.adler32(b) & 0xFFFFFFFF


# ------------------------------------------------------------------ msgpack framing
def _enc_int(v: int) -> bytes:
    """vmihailenco/msgpack EncodeInt: the shortest representation."""
    if 0 <= v <= 0x7F:
        return struct.pack("B", v)
    if -32 <= v < 0:
        return struct.pack("b", v)
    if v >= 0:
        if v <= 0xFF:
            return b"\xcc" + struct.pack("B", v)
        if v <= 0xFFFF:
            return b"\xcd" + struct.pack(">H", v)
        if v <= 0xFFFFFFFF:
            return b"\xce" + struct.pack(">I", v)
        return b"\xcf" + struct.pack(">Q", v)
    if v >= -0x80:
        return b"\xd0" + struct.pack("b", v)
    if v >= -0x8000:
        return b"\xd1" + struct.pack(">h", v)
    if v >= -0x80000000:
        return b"\xd2" + struct.pack(">i", v)
    return b"\xd3" + struct.pack(">q", v)


def _enc_bytes(b: bytes) -> bytes:
    if b is None:
        return b"\xc0"
    n = len(b)
    if n <= 0xFF:
        return b"\xc4" + struct.pack("B", n) + b
    if n <= 0xFFFF:
        return b"\xc5" + struct.pack(">H", n) + b
    return b"\xc6" + struct.pack(">I", n) + b


def _enc_array(n: int) -> bytes:
    if n <= 15:
        return struct.pack("B", 0x90 | n)
    return b"\xdc" + struct.pack(">H", n)


def _root(obj_type: int) -> bytes:  # encodeRootObject, msgpack/encoder.go:380-384
    return _enc_int(_VERSION) + _enc_array(_N_ROOT) + _enc_int(obj_type)


class _Reader:
    def __init__(self, buf: bytes, pos: int = 0):
        self.b = buf
        self.p = pos

    def _take(self, n):
        if self.p + n > len(self.b):
            raise EOFError("fileset: truncated msgpack stream")
        v = self.b[self.p:self.p + n]
        self.p += n
        return v

    def value(self):
        c = self._take(1)[0]
        if c <= 0x7F:
            return c
        if c >= 0xE0:
            return c - 0x100
        if 0x90 <= c <= 0x9F:
            return ("array", c & 0x0F)
        if c == 0xC0:
            return None
        if c == 0xCC:
            return self._take(1)[0]
        if c == 0xCD:
            return struct.unpack(">H", self._take(2))[0]
        if c == 0xCE:
            return struct.unpack(">I", self._take(4))[0]
        if c == 0xCF:
            return struct.unpack(">Q", self._take(8))[0]
        if c == 0xD0:
            return struct.unpack("b", self._take(1))[0]
        if c == 0xD1:
            return struct.unpack(">h", self._take(2))[0]
        if c == 0xD2:
            return struct.unpack(">i", self._take(4))[0]
        if c == 0xD3:
            return struct.unpack(">q", self._take(8))[0]
        if c == 0xC4:
            return bytes(self._take(self._take(1)[0]))
        if c == 0xC5:
            return bytes(self._take(struct.unpack(">H", self._take(2))[0]))
        if c == 0xC6:
            return bytes(self._take(struct.unpack(">I", self._take(4))[0]))
        if c == 0xDC:
            return ("array", struct.unpack(">H", self._take(2))[0])
        if c == 0xCB:
            return struct.unpack(">d", self._take(8))[0]
        raise ValueError("fileset: unsupported msgpack code 0x%02x at %d" % (c, self.p - 1))

    def array(self) -> int:
        v = self.value()
        if not (isinstance(v, tuple) and v[0] == "array"):
            raise ValueError("fileset: expected an array")
        return v[1]

    def root(self, want_type: int):
        version = self.value()
        n = self.array()  # root = [objectType, object]; the object (an array of fields) follows
        typ = self.value()
        if n != _N_ROOT:
            raise ValueError("fileset: root object with %d fields" % n)
        if typ != want_type:
            raise ValueError("fileset: object type %r, expected %r" % (typ, want_type))
        return version

    def skip(self, n_fields):
        for _ in range(n_fields):
            v = self.value()
            if isinstance(v, tuple):
                self.skip(v[1])


# ------------------------------------------------------------------ model
@dataclass
class Info:  # schema.IndexInfo, persist/schema/types.go:40-52
    block_start: int
    block_size: int
    entries: int
    major_version: int = MAJOR_VERSION
    minor_version: int = MINOR_VERSION
    volume_index: int = 0
    snapshot_time: int = 0
    file_type: int = 0
    snapshot_id: bytes = b""
    summaries: int = 0
    bloom_m: int = 0
    bloom_k: int = 0


@dataclass
class FilesetData:
    info: Info
    ids: List[bytes]
    tags: List[bytes]
    offsets: np.ndarray         # int64 [n] Offset of every stream in the data file
    sizes: np.ndarray           # int64 [n] Size
    data_checksums: np.ndarray  # uint32 [n] DataChecksum (Adler-32 of the segment)
    data: np.ndarray            # uint8 [data file bytes] (memory map)


def fileset_path(prefix: str, namespace: str, shard: int, block_start_ns: int, volume: int, suffix: str) -> str:
    """ShardDataDirPath + filesetFileForTimeAndVolumeIndex (persist/fs/files.go:1503-1507,1729-1747)."""
    return os.path.join(prefix, "data", namespace, str(shard),
                        "fileset-%d-%d-%s.db" % (block_start_ns, volume, suffix))


# ------------------------------------------------------------------ writer
def write_fileset(prefix: str, namespace: str, shard: int, block_start_ns: int, block_size_ns: int,
                  ids: Sequence[bytes], streams_blob, offsets: Sequence[int], sizes: Sequence[int],
                  tags: Optional[Sequence[bytes]] = None, volume: int = 0,
                  data_checksums: Optional[Sequence[int]] = None) -> str:
    """Writes one fileset volume in the reference's format (persist/fs/write.go): the data file is
    `streams_blob` AS IS when its streams are already in write order (sorted by ID like
    writeAll's index entries, write.go:406-470), index entries carry (Offset, Size, DataChecksum).
    Empty summaries / bloom-filter files are written (this tool reads by full index scan)."""
    n = len(ids)
    blob = np.ascontiguousarray(np.frombuffer(streams_blob, dtype=np.uint8)
                                if not isinstance(streams_blob, np.ndarray) else streams_blob, dtype=np.uint8)
    d = os.path.dirname(fileset_path(prefix, namespace, shard, block_start_ns, volume, "info"))
    os.makedirs(d, exist_ok=True)
    order = sorted(range(n), key=lambda i: ids[i])  # index entries are written sorted by ID
    # data file: segments in index order, contiguous
    data_parts, new_off, pos = [], [0] * n, 0
    for i in order:
        seg = blob[int(offsets[i]): int(offsets[i]) + int(sizes[i])]
        data_parts.append(seg)
        new_off[i] = pos
        pos += len(seg)
    data = np.concatenate(data_parts) if data_parts else np.zeros(0, dtype=np.uint8)
    index = bytearray()
    for k, i in enumerate(order):
        seg = data[new_off[i]: new_off[i] + int(sizes[i])]
        cs = int(data_checksums[i]) if data_checksums is not None else adler32(seg.tobytes())
        start = len(index)
        index += _root(_INDEX_ENTRY) + _enc_array(_N_INDEX_ENTRY)
        index += _enc_int(k) + _enc_bytes(bytes(ids[i])) + _enc_int(int(sizes[i])) + _enc_int(new_off[i])
        index += _enc_int(cs) + _enc_bytes(bytes(tags[i]) if tags is not None else b"")
        index += _enc_int(adler32(bytes(index[start:])))  # IndexChecksum, encoder.go:337-338
    info = (_root(_INDEX_INFO) + _enc_array(_N_INDEX_INFO) + _enc_int(block_start_ns) + _enc_int(block_size_ns) +
            _enc_int(n) + _enc_int(MAJOR_VERSION) + _enc_array(1) + _enc_int(0) + _enc_array(2) + _enc_int(0) +
            _enc_int(0) + _enc_int(0) + _enc_int(0) + _enc_bytes(b"") + _enc_int(volume) + _enc_int(MINOR_VERSION))
    files = {"info": bytes(info), "index": bytes(index), "summaries": b"", "bloomfilter": b"",
             "data": data.tobytes()}
    for suffix, content in files.items():
        with open(fileset_path(prefix, namespace, shard, block_start_ns, volume, suffix), "wb") as f:
            f.write(content)
    # digests of (info, index, summaries, bloom filter, data), write.go:382-388; little endian, digest/buffer.go:33-36
    digests = b"".join(struct.pack("<I", adler32(files[s])) for s in ("info", "index", "summaries", "bloomfilter", "data"))
    with open(fileset_path(prefix, namespace, shard, block_start_ns, volume, "digest"), "wb") as f:
        f.write(digests)
    with open(fileset_path(prefix, namespace, shard, block_start_ns, volume, "checkpoint"), "wb") as f:
        f.write(struct.pack("<I", adler32(digests)))  # write.go:638-655
    return d


# ------------------------------------------------------------------ reader
def read_fileset(prefix: str, namespace: str, shard: int, block_start_ns: int, volume: int = 0,
                 verify_digests: bool = True) -> FilesetData:
    """persist/fs/read.go Open + readIndexAndSortByOffsetAsc (:264-330) without the per-entry data
    reads: the data file is mapped whole, its index entries become offset / size / checksum arrays."""
    def p(s):
        return fileset_path(prefix, namespace, shard, block_start_ns, volume, s)

    if not os.path.exists(p("checkpoint")):
        raise FileNotFoundError("fileset: no checkpoint file (incomplete volume): " + p("checkpoint"))
    digests = open(p("digest"), "rb").read()
    if struct.unpack("<I", open(p("checkpoint"), "rb").read(4))[0] != adler32(digests):
        raise ValueError("fileset: checkpoint does not match the digest file")
    want = dict(zip(("info", "index", "summaries", "bloomfilter", "data"), struct.unpack("<5I", digests[:20])))
    info_b = open(p("info"), "rb").read()
    index_b = open(p("index"), "rb").read()
    if verify_digests:
        if adler32(info_b) != want["info"] or adler32(index_b) != want["index"]:
            raise ValueError("fileset: info / index file digest mismatch")
    r = _Reader(info_b)
    r.root(_INDEX_INFO)
    nf = r.array()
    block_start, block_size, entries, major = r.value(), r.value(), r.value(), r.value()
    r.array()
    summaries = r.value()
    r.array()
    bm, bk = r.value(), r.value()
    rest = [r.value() for _ in range(max(0, min(nf, 11) - 6))]  # snapshotTime, fileType, snapshotID, volume, minor
    rest += [0, 0, b"", 0, 0][len(rest):]
    info = Info(block_start, block_size, entries, major, rest[4], rest[3], rest[0], rest[1], rest[2] or b"",
                summaries, bm, bk)
    ids, tags = [], []
    offsets = np.zeros(entries, dtype=np.int64)
    sizes = np.zeros(entries, dtype=np.int64)
    checks = np.zeros(entries, dtype=np.uint32)
    r = _Reader(index_b)
    for k in range(entries):
        start = r.p
        r.root(_INDEX_ENTRY)
        nf = r.array()
        idx, id_, size, off, dcs, tg = r.value(), r.value(), r.value(), r.value(), r.value(), r.value()
        if nf >= 7:  # V3: the entry's own checksum over everything before it (decoder.go)
            before = r.p
            ics = r.value()
            if (ics & 0xFFFFFFFF) != adler32(index_b[start:before]):
                raise ValueError("fileset: index entry %d checksum mismatch" % k)
        r.skip(max(0, nf - 7))
        ids.append(id_)
        tags.append(tg or b"")
        offsets[k], sizes[k], checks[k] = off, size, dcs & 0xFFFFFFFF
    data = np.memmap(p("data"), dtype=np.uint8, mode="r") if os.path.getsize(p("data")) else np.zeros(0, np.uint8)
    if entries and int((offsets + sizes).max()) > data.shape[0]:
        raise ValueError("fileset: an index entry points past the end of the data file")
    return FilesetData(info, ids, tags, offsets, sizes, checks, data)


# ------------------------------------------------------------------ device ingestion
def decode_fileset(codec, fs: FilesetData, max_points: int, verify_checksums: bool = True, want_events: int = 0):
    """Uploads the data file as is, verifies every segment's Adler-32 on the device against the
    index entries (persist/fs/read.go:395-397, seek.go:370-373) and decodes all series with one
    launch.  Returns (DecodeResult, checksum_status int32 [n] or None)."""
    import torch
    dev = codec.device
    n = len(fs.ids)
    nbytes = int(fs.data.shape[0])
    d_data = torch.empty(nbytes + 16, dtype=torch.uint8, device=dev)
    if nbytes:
        d_data[:nbytes].copy_(torch.from_numpy(np.array(fs.data, copy=True)), non_blocking=False)
    d_off = torch.from_numpy(fs.offsets).to(dev)
    d_len = torch.from_numpy(fs.sizes).to(dev)
    status = None
    if verify_checksums and n:
        _, status = codec.segment_checksums(d_data[:nbytes], d_off, lengths=d_len,
                                            expected=torch.from_numpy(fs.data_checksums.view(np.int32)).to(dev))
    res = codec.decode(d_data[:nbytes], d_off, max_points, lengths=d_len, want_events=want_events)
    return res, status


# ------------------------------------------------------------------ a block range (tile aggregation)
@dataclass
class BlockRange:
    """The inputs of m3tsz_aggregate_tiles_blocks for a range of source blocks: `data` holds the blocks' data files,
    each at a 16-byte-aligned offset; segment q is data[offsets[q]: offsets[q] + sizes[q]] with the expected Adler-32
    data_checksums[q]; series s (ids[s], in ID order) is segments block_off[s] .. block_off[s + 1] - 1, one per block
    that lists the series, in block order."""
    block_starts: List[int]
    volumes: List[int]
    ids: List[bytes]
    tags: List[bytes]           # from the last block that lists the series
    data: np.ndarray            # uint8
    offsets: np.ndarray         # int64 [n_segments]
    sizes: np.ndarray           # int64 [n_segments]
    data_checksums: np.ndarray  # uint32 [n_segments]
    block_off: np.ndarray       # int64 [n_series + 1]


def latest_volume(prefix: str, namespace: str, shard: int, block_start_ns: int) -> int:
    """The highest volume index of a block that has a checkpoint file (a complete volume)."""
    d = os.path.dirname(fileset_path(prefix, namespace, shard, block_start_ns, 0, "checkpoint"))
    head = "fileset-%d-" % block_start_ns
    vols = []
    for f in os.listdir(d) if os.path.isdir(d) else ():
        if f.startswith(head) and f.endswith("-checkpoint.db"):
            v = f[len(head):-len("-checkpoint.db")]
            if v.isdigit():
                vols.append(int(v))
    if not vols:
        raise FileNotFoundError("fileset: no complete volume of block %d in %s" % (block_start_ns, d))
    return max(vols)


def read_block_range(prefix: str, namespace: str, shard: int, block_starts: Sequence[int],
                     volumes: Optional[Sequence[int]] = None) -> BlockRange:
    """Reads one volume per source block (default: each block's latest complete volume) and lays the blocks out as
    m3tsz_aggregate_tiles_blocks reads them: the union of the series IDs in ID order, and for each series one
    segment per block that lists it, in the order of `block_starts`.  The data files are copied as they are; the
    caller uploads `data` and verifies the segments with BatchCodec.segment_checksums against data_checksums."""
    block_starts = [int(b) for b in block_starts]
    if volumes is None:
        volumes = [latest_volume(prefix, namespace, shard, b) for b in block_starts]
    volumes = [int(v) for v in volumes]
    if len(volumes) != len(block_starts):
        raise ValueError("fileset: one volume per block")
    sets = [read_fileset(prefix, namespace, shard, b, v) for b, v in zip(block_starts, volumes)]
    base, pos = [], 0
    for fs in sets:
        pos = (pos + 15) & ~15
        base.append(pos)
        pos += int(fs.data.shape[0])
    data = np.zeros((pos + 15) & ~15, dtype=np.uint8)
    for b, fs in zip(base, sets):
        data[b: b + fs.data.shape[0]] = fs.data
    where = [{id_: k for k, id_ in enumerate(fs.ids)} for fs in sets]
    ids = sorted(set().union(*where)) if where else []
    tags, offsets, sizes, checks, block_off = [], [], [], [], [0]
    for id_ in ids:
        tag = b""
        for j, fs in enumerate(sets):
            k = where[j].get(id_)
            if k is None:
                continue
            offsets.append(base[j] + int(fs.offsets[k]))
            sizes.append(int(fs.sizes[k]))
            checks.append(int(fs.data_checksums[k]))
            tag = fs.tags[k]
        tags.append(tag)
        block_off.append(len(offsets))
    return BlockRange(block_starts, volumes, ids, tags, data, np.array(offsets, dtype=np.int64),
                      np.array(sizes, dtype=np.int64), np.array(checks, dtype=np.uint32),
                      np.array(block_off, dtype=np.int64))
