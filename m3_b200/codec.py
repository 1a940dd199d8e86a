"""Batch codec over the C ABI, with torch tensors as device memory.

torch is plumbing here (device allocations, streams, torch.distributed); every
codec operation is one call into libm3tsz_b200.so (hand-written sm_90a
kernels).  Nothing in this module computes on the CPU.
"""
import ctypes as C
from dataclasses import dataclass
from typing import Optional

import torch

from . import capi


def _ptr(t: Optional[torch.Tensor]):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _cuda_stream_ptr(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _check_records(t: Optional[torch.Tensor], n: int, nbytes: int):
    """A tile call's optional record tensor: uint8 [n, nbytes], contiguous, on the device."""
    if t is not None:
        assert t.is_cuda and t.is_contiguous() and t.dtype == torch.uint8
        assert t.shape == (n, nbytes)


@dataclass
class DecodeResult:
    ts: torch.Tensor        # int64  [S, max_points]
    values: torch.Tensor    # float64 [S, max_points]
    n_points: torch.Tensor  # int32 (uint32 bits) [S]
    status: torch.Tensor    # int32 [S]
    unit: torch.Tensor      # uint8 [S]
    annotations: Optional[torch.Tensor]  # uint8 view of m3tsz_annotation_ref [S, 16] or None
    unit_first: Optional[torch.Tensor] = None   # uint8 [S]: unit in force at the first datapoint
    events: Optional[torch.Tensor] = None       # uint8 [E, 32] view of m3tsz_dp_event (want_events)
    event_count: Optional[torch.Tensor] = None  # int64 [1]: events produced (may exceed E)


@dataclass
class EncodeResult:
    out: torch.Tensor      # uint8 [S, out_stride] slots
    out_len: torch.Tensor  # int64 [S]
    status: torch.Tensor   # int32 [S]


@dataclass
class PackedResult:
    packed: torch.Tensor   # uint8 [capacity]
    offsets: torch.Tensor  # int64 [S] start of every stream (completion order, not monotonic)
    out_len: torch.Tensor  # int64 [S]
    status: torch.Tensor   # int32 [S]
    total: torch.Tensor    # int64 [1] bytes used


@dataclass
class DownsampleResult:
    sum: torch.Tensor    # float64 [W, S] (window-major)
    count: torch.Tensor  # int64 [W, S]
    min: torch.Tensor    # float64 [W, S]
    max: torch.Tensor    # float64 [W, S]
    n_points: torch.Tensor
    status: torch.Tensor
    last: Optional[torch.Tensor] = None     # float64 [W, S] Gauge.Last() (want_last)
    last_at: Optional[torch.Tensor] = None  # int64 [W, S] Gauge.LastAt() in ns
    # Gauge sumSq (want_sum_sq), float64 [W, S]; a Counter's (metric=METRIC_COUNTER) is int64 [W, S], like its
    # sum / min / max
    sum_sq: Optional[torch.Tensor] = None
    metric: int = capi.METRIC_GAUGE


class BatchCodec:
    """Device-resident batch encode / decode (the drop-in for the per-series
    loops at the reference's batch sites, SURVEY.md §3.2/§3.3)."""

    def __init__(self, device=0, int_optimized=True, default_unit=capi.UNIT_S):
        if not torch.cuda.is_available():
            raise capi.M3tszError(capi.ERR_NO_DEVICE, "torch sees no CUDA device")
        self.device = torch.device("cuda", device if isinstance(device, int) else device.index)
        self.ctx = capi.Context(self.device.index)
        self.opts = capi.Options(int(bool(int_optimized)), int(default_unit))
        self.int_optimized = bool(int_optimized)
        self.default_unit = int(default_unit)

    # ------------------------------------------------------------------ decode
    def decode(self, streams: torch.Tensor, offsets: torch.Tensor, max_points: int,
               want_annotations=False, out: Optional[DecodeResult] = None,
               lengths: Optional[torch.Tensor] = None, want_events=0, point_major=False) -> DecodeResult:
        """streams: uint8 [total] on device; offsets: int64 [S+1] on device (byte offsets), or
        int64 [S] starts + `lengths` int64 [S] (streams placed anywhere, index-entry style).
        want_events = capacity of the per-datapoint unit / annotation event table (0: none).
        point_major: outputs are [max_points, S] (step-major, coalesced stores) instead of [S, max_points]."""
        assert streams.dtype == torch.uint8 and streams.is_cuda and streams.is_contiguous()
        assert offsets.dtype == torch.int64 and offsets.is_cuda and offsets.is_contiguous()
        S = offsets.numel() - 1 if lengths is None else lengths.numel()
        dev = self.device
        if out is None:
            shape = (max_points, S) if point_major else (S, max_points)
            out = DecodeResult(
                ts=torch.empty(shape, dtype=torch.int64, device=dev),
                values=torch.empty(shape, dtype=torch.float64, device=dev),
                n_points=torch.empty(S, dtype=torch.int32, device=dev),
                status=torch.empty(S, dtype=torch.int32, device=dev),
                unit=torch.empty(S, dtype=torch.uint8, device=dev),
                annotations=(torch.empty((S, 16), dtype=torch.uint8, device=dev)
                             if want_annotations else None))
        ex = capi.DecodeExtras()
        ex.d_lengths = lengths.data_ptr() if lengths is not None else None
        ex.point_major = 1 if point_major else 0
        if want_events:
            if out.unit_first is None:
                out.unit_first = torch.empty(S, dtype=torch.uint8, device=dev)
            if out.events is None or out.events.shape[0] < want_events:
                out.events = torch.zeros((int(want_events), 32), dtype=torch.uint8, device=dev)
            if out.event_count is None:
                out.event_count = torch.zeros(1, dtype=torch.int64, device=dev)
            out.event_count.zero_()
            ex.d_unit_first = out.unit_first.data_ptr()
            ex.d_events = out.events.data_ptr()
            ex.events_capacity = int(out.events.shape[0])
            ex.d_event_count = out.event_count.data_ptr()
        rc = capi.lib().m3tsz_decode_batch_ex(
            self.ctx.handle, C.byref(self.opts), _ptr(streams), streams.numel(), _ptr(offsets), S,
            _ptr(out.ts), _ptr(out.values), max_points, _ptr(out.n_points), _ptr(out.status),
            _ptr(out.unit), _ptr(out.annotations), C.byref(ex), _cuda_stream_ptr(dev))
        self.ctx.check(rc, "m3tsz_decode_batch_ex")
        return out

    def decode_downsample(self, streams, offsets, range_start_ns, window_ns, n_windows,
                          out: Optional[DownsampleResult] = None, want_last=False, metric=capi.METRIC_GAUGE,
                          want_sum_sq=False, lengths: Optional[torch.Tensor] = None) -> DownsampleResult:
        """Window-major [W, S] aggregates of aggregation.Gauge (metric=METRIC_GAUGE; want_sum_sq adds sumSq, and
        with it last / last_at) or aggregation.Counter (metric=METRIC_COUNTER: int64 sum / min / max / sum_sq of
        int64(value)).  `lengths` (int64 [S]) gives stream s = offsets[s] .. + lengths[s]."""
        assert streams.dtype == torch.uint8 and streams.is_cuda
        assert offsets.dtype == torch.int64 and offsets.is_cuda
        if metric != capi.METRIC_GAUGE or want_sum_sq or lengths is not None:
            return self._decode_downsample_ex(streams, offsets, range_start_ns, window_ns, n_windows, out,
                                              want_last, metric, want_sum_sq, lengths)
        S = offsets.numel() - 1
        dev = self.device
        if out is None:
            mk = lambda dt: torch.empty((n_windows, S), dtype=dt, device=dev)
            out = DownsampleResult(
                sum=mk(torch.float64), count=mk(torch.int64), min=mk(torch.float64), max=mk(torch.float64),
                n_points=torch.empty(S, dtype=torch.int32, device=dev),
                status=torch.empty(S, dtype=torch.int32, device=dev),
                last=mk(torch.float64) if want_last else None, last_at=mk(torch.int64) if want_last else None)
        if want_last:  # a different kernel: it also keeps Gauge.Last() / LastAt()
            rc = capi.lib().m3tsz_decode_downsample_last_batch(
                self.ctx.handle, C.byref(self.opts), _ptr(streams), streams.numel(), _ptr(offsets), S,
                int(range_start_ns), int(window_ns), int(n_windows), _ptr(out.sum), _ptr(out.count),
                _ptr(out.min), _ptr(out.max), _ptr(out.last), _ptr(out.last_at), _ptr(out.n_points),
                _ptr(out.status), _cuda_stream_ptr(dev))
            self.ctx.check(rc, "m3tsz_decode_downsample_last_batch")
            return out
        rc = capi.lib().m3tsz_decode_downsample_batch(
            self.ctx.handle, C.byref(self.opts), _ptr(streams), streams.numel(), _ptr(offsets), S,
            int(range_start_ns), int(window_ns), int(n_windows), _ptr(out.sum), _ptr(out.count),
            _ptr(out.min), _ptr(out.max), _ptr(out.n_points), _ptr(out.status), _cuda_stream_ptr(dev))
        self.ctx.check(rc, "m3tsz_decode_downsample_batch")
        return out

    def _decode_downsample_ex(self, streams, offsets, range_start_ns, window_ns, n_windows, out, want_last, metric,
                              want_sum_sq, lengths) -> DownsampleResult:
        counter = metric == capi.METRIC_COUNTER
        if metric not in (capi.METRIC_GAUGE, capi.METRIC_COUNTER) or (counter and want_last):
            raise capi.M3tszError(capi.ERR_INVALID_ARG, "metric %r with want_last=%r" % (metric, want_last))
        S = offsets.numel() - 1 if lengths is None else lengths.numel()
        dev = self.device
        if out is None:
            mk = lambda dt: torch.empty((n_windows, S), dtype=dt, device=dev)
            agg = torch.int64 if counter else torch.float64
            last = want_last or (want_sum_sq and not counter)  # the Gauge's sumSq kernel keeps last / lastAt
            out = DownsampleResult(
                sum=mk(agg), count=mk(torch.int64), min=mk(agg), max=mk(agg),
                n_points=torch.empty(S, dtype=torch.int32, device=dev),
                status=torch.empty(S, dtype=torch.int32, device=dev),
                last=mk(torch.float64) if last and not counter else None,
                last_at=mk(torch.int64) if last and not counter else None,
                sum_sq=mk(agg) if (want_sum_sq or counter) else None, metric=metric)
        o = capi.DownsampleOutputs()
        o.metric_type = metric
        addr = lambda t: t.data_ptr() if t is not None else None
        if counter:
            o.d_counter_sum, o.d_counter_min, o.d_counter_max = addr(out.sum), addr(out.min), addr(out.max)
            o.d_counter_sum_sq = addr(out.sum_sq)
        else:
            o.d_sum, o.d_min, o.d_max = addr(out.sum), addr(out.min), addr(out.max)
            o.d_sum_sq, o.d_last, o.d_last_at = addr(out.sum_sq), addr(out.last), addr(out.last_at)
        o.d_count, o.d_n_points, o.d_status = addr(out.count), addr(out.n_points), addr(out.status)
        rc = capi.lib().m3tsz_decode_downsample_ex(
            self.ctx.handle, C.byref(self.opts), _ptr(streams), streams.numel(), _ptr(offsets), _ptr(lengths), S,
            int(range_start_ns), int(window_ns), int(n_windows), C.byref(o), _cuda_stream_ptr(dev))
        self.ctx.check(rc, "m3tsz_decode_downsample_ex")
        return out

    # ------------------------------------------------------------------ encode
    def encode_bound(self, n_points: int) -> int:
        return int(capi.lib().m3tsz_encode_bound(int(n_points)))

    def encode(self, ts: torch.Tensor, values: torch.Tensor, start: torch.Tensor,
               unit=capi.UNIT_S, n_points: Optional[torch.Tensor] = None,
               units: Optional[torch.Tensor] = None, annotations=None,
               out_stride: Optional[int] = None, out: Optional[EncodeResult] = None,
               point_major=False) -> EncodeResult:
        """ts int64 [S,P], values float64 [S,P], start int64 [S] (all on device).
        annotations: optional (series_off int64 [S+1], entries uint8 [E,16], bytes uint8 [B]).
        point_major: ts / values are [P,S] (step-major, what decode(point_major=True) writes)."""
        assert ts.dtype == torch.int64 and values.dtype == torch.float64
        assert ts.is_cuda and values.is_cuda and ts.is_contiguous() and values.is_contiguous()
        assert start.dtype == torch.int64 and start.is_cuda
        S, P = (ts.shape[1], ts.shape[0]) if point_major else ts.shape
        dev = self.device
        if out_stride is None:
            out_stride = self.encode_bound(P)
        if out is None:
            out = EncodeResult(
                out=torch.empty((S, out_stride), dtype=torch.uint8, device=dev),
                out_len=torch.empty(S, dtype=torch.int64, device=dev),
                status=torch.empty(S, dtype=torch.int32, device=dev))
        a_off = a_ent = a_bytes = None
        if annotations is not None:
            a_off, a_ent, a_bytes = annotations
        ex = capi.EncodeExtras()
        ex.point_major_input = 1 if point_major else 0
        rc = capi.lib().m3tsz_encode_batch_ex(
            self.ctx.handle, C.byref(self.opts), _ptr(ts), _ptr(values), S, P, _ptr(n_points),
            _ptr(start), int(unit), _ptr(units), _ptr(a_off), _ptr(a_ent), _ptr(a_bytes),
            _ptr(out.out), out.out.shape[1], _ptr(out.out_len), _ptr(out.status), C.byref(ex),
            _cuda_stream_ptr(dev))
        self.ctx.check(rc, "m3tsz_encode_batch_ex")
        return out

    def encode_packed(self, ts, values, start, unit=capi.UNIT_S, n_points=None, units=None,
                      annotations=None, align=64, capacity: Optional[int] = None, slot_bytes=0,
                      out: Optional["PackedResult"] = None, point_major=False) -> "PackedResult":
        """Encodes straight into one packed buffer (no slots, no compaction pass).  Streams are
        placed in completion order: stream s = packed[offsets[s] : offsets[s] + out_len[s]].
        point_major: ts / values are [P, S] (step-major)."""
        S, P = (ts.shape[1], ts.shape[0]) if point_major else ts.shape
        dev = self.device
        if out is None:
            if capacity is None:
                capacity = S * (self.encode_bound(P) if units is None else
                                int(capi.lib().m3tsz_encode_bound_units(P, 1)))
            out = PackedResult(
                packed=torch.empty(capacity, dtype=torch.uint8, device=dev),
                offsets=torch.empty(S, dtype=torch.int64, device=dev),
                out_len=torch.empty(S, dtype=torch.int64, device=dev),
                status=torch.empty(S, dtype=torch.int32, device=dev),
                total=torch.zeros(1, dtype=torch.int64, device=dev))
        a_off = a_ent = a_bytes = None
        if annotations is not None:
            a_off, a_ent, a_bytes = annotations
        ex = capi.EncodeExtras()
        ex.point_major_input = 1 if point_major else 0
        rc = capi.lib().m3tsz_encode_batch_packed_ex(
            self.ctx.handle, C.byref(self.opts), _ptr(ts), _ptr(values), S, P, _ptr(n_points),
            _ptr(start), int(unit), _ptr(units), _ptr(a_off), _ptr(a_ent), _ptr(a_bytes),
            int(slot_bytes), int(align), _ptr(out.packed), out.packed.numel(), _ptr(out.offsets),
            _ptr(out.out_len), _ptr(out.status), _ptr(out.total), C.byref(ex) if point_major else None,
            _cuda_stream_ptr(dev))
        self.ctx.check(rc, "m3tsz_encode_batch_packed_ex")
        return out

    def compact(self, enc: EncodeResult, align=64, capacity: Optional[int] = None):
        """Packs slots into (packed uint8 [total], offsets int64 [S+1])."""
        S, stride = enc.out.shape
        dev = self.device
        if capacity is None:
            capacity = int(enc.out_len.sum().item()) + S * align + 16
        packed = torch.empty(capacity, dtype=torch.uint8, device=dev)
        offsets = torch.empty(S + 1, dtype=torch.int64, device=dev)
        rc = capi.lib().m3tsz_compact_streams(
            self.ctx.handle, _ptr(enc.out), stride, _ptr(enc.out_len), S, int(align), _ptr(packed),
            capacity, _ptr(offsets), _cuda_stream_ptr(dev))
        self.ctx.check(rc, "m3tsz_compact_streams")
        return packed, offsets

    def encoder_set(self, start: torch.Tensor, stride: int) -> "EncoderSet":
        """S open encoders on the device (S = start.numel(), start int64 [S] ns), each with a slot of `stride`
        bytes (a multiple of 16): the write path's encoders, appended to over many calls."""
        return EncoderSet(self, start, stride)

    def element_set(self, start: torch.Tensor, metric_type, agg_types, resolution_ns, transforms=(),
                    discard_nan=False, open_windows=4, stride: Optional[int] = None,
                    out_unit=capi.UNIT_S, annotation_capacity=0, sample_capacity: Optional[int] = None, eps=1e-3,
                    insert_and_compress_every=1024, source_capacity=0) -> "ElementSet":
        """N aggregator elements fed datapoint by datapoint (m3tsz_element_set_*, N = start.numel(), start int64
        [N] ns): one metric type (capi.METRIC_GAUGE / METRIC_COUNTER), resolution, strictly ascending list of
        aggregation types and transformation list, checked and applied as in aggregate_tiles_types (discard_nan
        only with transformations).  Each element keeps up to `open_windows` open windows; its flushed windows go to
        an encoder set of k * N rows (row j * N + s: element s under agg_types[j]) with slots of `stride` bytes
        (default: room for 128 datapoints per row at their worst case), written with `out_unit`.
        annotation_capacity > 0 (a multiple of 8, at most capi.MAX_ELEMENT_ANNOTATION): the elements keep annotations
        (m3tsz_element_set_*_annotated), each open window up to that many bytes of its last non-empty one.
        stride=0: a set without output rows, a rollup's source set (ElementSet.forward); consume() and stream()
        refuse it.
        capi.METRIC_TIMER (m3tsz_element_set_*_timer): every type but Last (up to capi.MAX_TIMER_TYPES without
        transformations), each open window an aggregation.Timer over the CM stream with `eps` and
        `insert_and_compress_every` (the aggregator's StreamOptions), holding at most `sample_capacity` values (list
        samples and pending values together; required).  With annotation_capacity a Timer set keeps annotations too
        (m3tsz_element_set_*_timer_annotated: a batch's annotation is its first row's).  It forwards through a rollup
        with ElementSet.forward_timer, not forward.
        source_capacity > 0 (a multiple of 32, at most capi.MAX_FORWARD_SOURCES): the set is a rollup's group set fed
        across shards (ElementSet.add_forwarded), each open window keeping which of that many source ids it has
        seen."""
        return ElementSet(self, start, metric_type, agg_types, resolution_ns, transforms, discard_nan, open_windows,
                          stride, out_unit, annotation_capacity, sample_capacity, eps, insert_and_compress_every,
                          source_capacity)

    def bucket_set(self, start: torch.Tensor, stride: int, encoders=4, pool_records: Optional[int] = None,
                   pool_stride: Optional[int] = None) -> "BucketSet":
        """S buffer buckets (BufferBucket.write, m3tsz_encoder_set_write): encoder 0 of bucket s is an encoder set
        of slots of `stride` bytes; up to encoders - 1 more per bucket open on demand from a pool of `pool_records`
        (default S) records of `pool_stride` (default `stride`) bytes."""
        return BucketSet(self, start, stride, encoders, start.numel() if pool_records is None else pool_records,
                         stride if pool_stride is None else pool_stride)

    # ------------------------------------------------------------------ merge (row N1)
    def merge_series(self, ts, values, n_points, seq_status, slice_off, replica_off, series_off,
                     out_cap, start_ns=0, end_ns=0, strategy=0, point_major=False):
        """seriesIterator / multiReaderIterator semantics over decoded streams (device tensors;
        offsets int64).  Returns (ts_out [S,out_cap], val_out, n_out int32 [S], status int32 [S]);
        point_major: inputs are [cap, n_seq] and outputs [out_cap, S] (step-major)."""
        S = series_off.numel() - 1
        dev = self.device
        shape = (out_cap, S) if point_major else (S, out_cap)
        ts_out = torch.empty(shape, dtype=torch.int64, device=dev)
        val_out = torch.empty(shape, dtype=torch.float64, device=dev)
        n_out = torch.empty(S, dtype=torch.int32, device=dev)
        status = torch.empty(S, dtype=torch.int32, device=dev)
        cap, n_seq = (ts.shape[0], ts.shape[1]) if point_major else (ts.shape[1], ts.shape[0])
        rc = capi.lib().m3tsz_merge_series_batch_ex(
            self.ctx.handle, _ptr(ts), _ptr(values), cap, _ptr(n_points), _ptr(seq_status),
            _ptr(slice_off), _ptr(replica_off), _ptr(series_off), S, int(start_ns), int(end_ns),
            int(strategy), _ptr(ts_out), _ptr(val_out), out_cap, _ptr(n_out), _ptr(status), n_seq,
            1 if point_major else 0, 1 if point_major else 0, _cuda_stream_ptr(dev))
        self.ctx.check(rc, "m3tsz_merge_series_batch_ex")
        return ts_out, val_out, n_out, status

    # ------------------------------------------------------------ query-side consumers (rows N3, N4)
    def prom_convert(self, ts, values, n_points, resolution_ns=0, handle_resets=None, tolerance=0.0,
                     tolerance_until_ns=0, out_cap=None):
        """iteratorToPromResult over decoded / merged series in HBM.  Returns
        (ts_ms int64 [S,out_cap], values float64 [S,out_cap], n_out int32 [S], status int32 [S])."""
        S, cap = ts.shape
        dev = self.device
        if out_cap is None:
            out_cap = cap + 1 if handle_resets is not None else cap
        ts_out = torch.empty((S, out_cap), dtype=torch.int64, device=dev)
        val_out = torch.empty((S, out_cap), dtype=torch.float64, device=dev)
        n_out = torch.empty(S, dtype=torch.int32, device=dev)
        status = torch.empty(S, dtype=torch.int32, device=dev)
        rc = capi.lib().m3tsz_prom_convert_batch(
            self.ctx.handle, _ptr(ts), _ptr(values), cap, _ptr(n_points), S, int(resolution_ns),
            _ptr(handle_resets), float(tolerance), int(tolerance_until_ns), _ptr(ts_out), _ptr(val_out),
            out_cap, _ptr(n_out), _ptr(status), _cuda_stream_ptr(dev))
        self.ctx.check(rc, "m3tsz_prom_convert_batch")
        return ts_out, val_out, n_out, status

    def aggregate_tiles(self, streams, offsets, start_ns, step_ns, n_windows, agg_type=capi.AGG_LAST,
                        out_unit=capi.UNIT_S, lengths=None, align=64, capacity=None,
                        out: Optional["PackedResult"] = None, metric_type=capi.METRIC_GAUGE, transforms=(),
                        discard_nan=True, state: Optional[torch.Tensor] = None):
        """storage.TileAggregator compute: decode -> Gauge (or Counter: metric_type=METRIC_COUNTER) per Step
        window -> re-encode (packed).  Returns (PackedResult, n_tiles int32 [S]).
        transforms: the pipeline's transformation ids (capi.TRANSFORM_*), applied in order to every non-empty
        window's value (m3tsz_aggregate_tiles_transform); discard_nan drops a window whose result is NaN; state
        (transform_state(S)) carries each series' previous window and Add sums from one call to the next."""
        S = offsets.numel() - 1 if lengths is None else lengths.numel()
        dev = self.device
        transforms = [int(t) for t in transforms]
        if out is None and capacity is None:
            rows = 2 * n_windows if capi.TRANSFORM_RESET in transforms else n_windows
            capacity = S * self.encode_bound(rows)
        out, n_tiles = self._tile_outputs(S, capacity, out)
        if transforms:
            _check_records(state, S, capi.TRANSFORM_STATE_BYTES)
            ops = (C.c_int32 * len(transforms))(*transforms)
            rc = capi.lib().m3tsz_aggregate_tiles_transform(
                self.ctx.handle, C.byref(self.opts), _ptr(streams), streams.numel(), _ptr(offsets),
                _ptr(lengths), S, int(start_ns), int(step_ns), int(n_windows), int(metric_type), int(agg_type),
                int(out_unit), int(align), _ptr(out.packed), out.packed.numel(), _ptr(out.offsets),
                _ptr(out.out_len), _ptr(out.status), _ptr(n_tiles), _ptr(out.total), ops, len(transforms),
                1 if discard_nan else 0, _ptr(state), _cuda_stream_ptr(dev))
            self.ctx.check(rc, "m3tsz_aggregate_tiles_transform")
            return out, n_tiles
        if metric_type != capi.METRIC_GAUGE or agg_type in (capi.AGG_SUMSQ, capi.AGG_STDEV):
            rc = capi.lib().m3tsz_aggregate_tiles_ex(
                self.ctx.handle, C.byref(self.opts), _ptr(streams), streams.numel(), _ptr(offsets),
                _ptr(lengths), S, int(start_ns), int(step_ns), int(n_windows), int(metric_type), int(agg_type),
                int(out_unit), int(align), _ptr(out.packed), out.packed.numel(), _ptr(out.offsets),
                _ptr(out.out_len), _ptr(out.status), _ptr(n_tiles), _ptr(out.total), _cuda_stream_ptr(dev))
            self.ctx.check(rc, "m3tsz_aggregate_tiles_ex")
            return out, n_tiles
        rc = capi.lib().m3tsz_aggregate_tiles_batch(
            self.ctx.handle, C.byref(self.opts), _ptr(streams), streams.numel(), _ptr(offsets),
            _ptr(lengths), S, int(start_ns), int(step_ns), int(n_windows), int(agg_type), int(out_unit),
            int(align), _ptr(out.packed), out.packed.numel(), _ptr(out.offsets), _ptr(out.out_len),
            _ptr(out.status), _ptr(n_tiles), _ptr(out.total), _cuda_stream_ptr(dev))
        self.ctx.check(rc, "m3tsz_aggregate_tiles_batch")
        return out, n_tiles

    def transform_state(self, n_series: int) -> torch.Tensor:
        """A zeroed m3tsz_transform_state per series (uint8 [S, 96]): every series a new element, for
        aggregate_tiles(..., transforms=..., state=...)."""
        return torch.zeros((n_series, capi.TRANSFORM_STATE_BYTES), dtype=torch.uint8, device=self.device)

    def aggregate_tiles_types(self, streams, offsets, start_ns, step_ns, n_windows, agg_types,
                              metric_type=capi.METRIC_GAUGE, out_unit=capi.UNIT_S, lengths=None, align=64,
                              capacity=None, transforms=(), discard_nan=True, state: Optional[torch.Tensor] = None,
                              annotations=False, blocks: Optional[torch.Tensor] = None):
        """An element with several aggregation types (m3tsz_aggregate_tiles_types): one decode + windows, then one
        stream per (type, series).  agg_types: strictly ascending aggregation.Type ids (capi.AGG_*), 1..8 of them;
        transforms / discard_nan as in aggregate_tiles, except that the Add op's sums are shared by the types, as in
        the reference's element.  state (element_state(S)) carries each series' element from one call to the next.
        Returns (PackedResult, n_tiles int32 [k, S]); the result's offsets / out_len / status are [k, S] views, row j
        being agg_types[j].  annotations=True (m3tsz_aggregate_tiles_annotated): every window's datapoints also carry
        the window's annotation, that of the last datapoint in stream order inside the window that has one; the
        default capacity then adds each source stream's length to every row's bound.
        blocks (int64 [S + 1] device tensor; m3tsz_aggregate_tiles_blocks): offsets / lengths then describe segments,
        one per (series, source block), and series s is segments blocks[s] .. blocks[s + 1] - 1, decoded one after
        another as one datapoint sequence (fileset.read_block_range returns these inputs); with annotations the
        default capacity adds each series' summed segment lengths."""
        n_seg = offsets.numel() - 1 if lengths is None else lengths.numel()
        S = n_seg if blocks is None else blocks.numel() - 1
        dev = self.device
        types = [int(t) for t in agg_types]
        transforms = [int(t) for t in transforms]
        k = len(types)
        if capacity is None:
            rows = 2 * n_windows if capi.TRANSFORM_RESET in transforms else n_windows
            capacity = k * S * self.encode_bound(rows)
            if annotations and blocks is not None:  # ... of different ones of its series' segments
                seg = (offsets[1:] - offsets[:-1]) if lengths is None else lengths
                cs = torch.cat([torch.zeros(1, dtype=torch.int64, device=seg.device), torch.cumsum(seg, 0)])
                b = blocks.clamp(0, n_seg)
                src_bytes = int((cs[b[1:]] - cs[b[:-1]]).clamp(min=0).sum().item())
                capacity += k * (src_bytes + 16 * S)
            elif annotations:  # a row's annotations are copies of different ones of its source stream
                src_bytes = (int(offsets[-1].item() - offsets[0].item()) if lengths is None
                             else int(lengths.sum().item()))
                capacity += k * (src_bytes + 16 * S)
            capacity = max(1, capacity)
        out, n_tiles = self._tile_outputs(max(1, k) * S, capacity)
        _check_records(state, S, capi.ELEMENT_STATE_BYTES)
        types_a = (C.c_int32 * max(1, k))(*types)
        ops = (C.c_int32 * max(1, len(transforms)))(*transforms)
        if blocks is not None:
            assert blocks.is_cuda and blocks.dtype == torch.int64 and blocks.is_contiguous()
            rc = capi.lib().m3tsz_aggregate_tiles_blocks(
                self.ctx.handle, C.byref(self.opts), _ptr(streams), streams.numel(), _ptr(offsets), _ptr(lengths),
                n_seg, _ptr(blocks), S, int(start_ns), int(step_ns), int(n_windows), int(metric_type), types_a, k,
                int(out_unit), int(align), _ptr(out.packed), out.packed.numel(), _ptr(out.offsets), _ptr(out.out_len),
                _ptr(out.status), _ptr(n_tiles), _ptr(out.total), ops, len(transforms), 1 if discard_nan else 0,
                _ptr(state), 1 if annotations else 0, _cuda_stream_ptr(dev))
            self.ctx.check(rc, "m3tsz_aggregate_tiles_blocks")
            return self._types_views(out, n_tiles, k, S)
        fn = capi.lib().m3tsz_aggregate_tiles_annotated if annotations else capi.lib().m3tsz_aggregate_tiles_types
        rc = fn(
            self.ctx.handle, C.byref(self.opts), _ptr(streams), streams.numel(), _ptr(offsets), _ptr(lengths), S,
            int(start_ns), int(step_ns), int(n_windows), int(metric_type), types_a, k, int(out_unit), int(align),
            _ptr(out.packed), out.packed.numel(), _ptr(out.offsets), _ptr(out.out_len), _ptr(out.status),
            _ptr(n_tiles), _ptr(out.total), ops, len(transforms), 1 if discard_nan else 0, _ptr(state),
            _cuda_stream_ptr(dev))
        self.ctx.check(rc, "m3tsz_aggregate_tiles_annotated" if annotations else "m3tsz_aggregate_tiles_types")
        return self._types_views(out, n_tiles, k, S)

    def _tile_outputs(self, n, capacity, out: Optional["PackedResult"] = None):
        """The packed outputs of a tile call with n rows (unless the caller passes them) and its n_tiles."""
        dev = self.device
        if out is None:
            out = PackedResult(
                packed=torch.empty(capacity, dtype=torch.uint8, device=dev),
                offsets=torch.empty(n, dtype=torch.int64, device=dev),
                out_len=torch.empty(n, dtype=torch.int64, device=dev),
                status=torch.empty(n, dtype=torch.int32, device=dev),
                total=torch.zeros(1, dtype=torch.int64, device=dev))
        return out, torch.empty(n, dtype=torch.int32, device=dev)

    @staticmethod
    def _types_views(out, n_tiles, k, S):
        out.offsets = out.offsets.view(k, S)
        out.out_len = out.out_len.view(k, S)
        out.status = out.status.view(k, S)
        return out, n_tiles.view(k, S)

    def aggregate_tiles_rollup(self, streams, offsets, start_ns, step_ns, n_windows, src_type, group_off, members,
                               rollup_types, metric_type=capi.METRIC_GAUGE, pre_transforms=(), post_transforms=(),
                               discard_nan=True, src_state: Optional[torch.Tensor] = None,
                               group_state: Optional[torch.Tensor] = None, lengths=None,
                               blocks: Optional[torch.Tensor] = None, capacity=None, out_unit=capi.UNIT_S, align=64,
                               annotations=False):
        """Tile aggregation through a rollup (m3tsz_aggregate_tiles_rollup): every source series is an element of
        (metric_type, src_type) whose window values run through pre_transforms and are forwarded; group g is the
        sources members[group_off[g] .. group_off[g + 1]) (int64 [G + 1] and int32 [n] device tensors), whose
        forwarded values are folded in that order into one element per group with rollup_types (strictly ascending,
        1..8) and post_transforms.  src_state (transform_state(S)) and group_state (element_state(G)) carry the
        chains from call to call.  offsets / lengths / blocks address the sources as in aggregate_tiles_types.
        annotations=True (m3tsz_aggregate_tiles_rollup_annotated): each group window also carries the last non-empty
        annotation, in listed order, of the members that forwarded a value to it, and its rows write it; the default
        capacity then adds, per rollup type, the source bytes of every listed member.
        Returns (PackedResult with [k, G] views, n_tiles int32 [k, G], source statuses int32 [S])."""
        n_seg = offsets.numel() - 1 if lengths is None else lengths.numel()
        S = n_seg if blocks is None else blocks.numel() - 1
        assert group_off.numel() >= 1, "group_off has G + 1 entries"
        G = group_off.numel() - 1
        dev = self.device
        types = [int(t) for t in rollup_types]
        pre = [int(t) for t in pre_transforms]
        post = [int(t) for t in post_transforms]
        k = len(types)
        if capacity is None:
            rows = 2 * n_windows if capi.TRANSFORM_RESET in post else n_windows
            capacity = k * G * self.encode_bound(rows)
            if annotations and members.numel():  # a group row's annotations are copies of different ones of its members'
                seg = (offsets[1:] - offsets[:-1]) if lengths is None else lengths
                if blocks is None:
                    src_len = seg
                else:
                    cs = torch.cat([torch.zeros(1, dtype=torch.int64, device=seg.device), torch.cumsum(seg, 0)])
                    b = blocks.clamp(0, n_seg)
                    src_len = (cs[b[1:]] - cs[b[:-1]]).clamp(min=0)
                m = members.long()
                ok = (m >= 0) & (m < S)
                member_bytes = int(src_len[m.clamp(0, max(0, S - 1))][ok].clamp(min=0).sum().item()) if S else 0
                capacity += k * (member_bytes + 16 * G)
            capacity = max(1, capacity)
        out, n_tiles = self._tile_outputs(k * G, capacity)
        src_status = torch.empty(max(1, S), dtype=torch.int32, device=dev)
        assert group_off.is_cuda and group_off.dtype == torch.int64 and group_off.is_contiguous()
        assert members.is_cuda and members.dtype == torch.int32 and members.is_contiguous()
        if blocks is not None:
            assert blocks.is_cuda and blocks.dtype == torch.int64 and blocks.is_contiguous()
        _check_records(src_state, S, capi.TRANSFORM_STATE_BYTES)
        _check_records(group_state, G, capi.ELEMENT_STATE_BYTES)
        i32s = lambda xs: (C.c_int32 * max(1, len(xs)))(*xs)
        fn = "m3tsz_aggregate_tiles_rollup_annotated" if annotations else "m3tsz_aggregate_tiles_rollup"
        rc = getattr(capi.lib(), fn)(
            self.ctx.handle, C.byref(self.opts), _ptr(streams), streams.numel(), _ptr(offsets), _ptr(lengths),
            n_seg, _ptr(blocks), S, int(start_ns), int(step_ns), int(n_windows), int(metric_type), int(src_type),
            i32s(pre), len(pre), _ptr(group_off), _ptr(members), members.numel(), G, i32s(types), k, i32s(post),
            len(post), 1 if discard_nan else 0, _ptr(src_state), _ptr(group_state), int(out_unit), int(align),
            _ptr(out.packed), out.packed.numel(), _ptr(out.offsets), _ptr(out.out_len), _ptr(out.status),
            _ptr(n_tiles), _ptr(out.total), _ptr(src_status), _cuda_stream_ptr(dev))
        self.ctx.check(rc, fn)
        out, n_tiles = self._types_views(out, n_tiles, k, G)
        return out, n_tiles, src_status[:S]

    def element_state(self, n_series: int) -> torch.Tensor:
        """A zeroed m3tsz_element_state per series (uint8 [S, 160]): every series a new element, for
        aggregate_tiles_types(..., state=...)."""
        return torch.zeros((n_series, capi.ELEMENT_STATE_BYTES), dtype=torch.uint8, device=self.device)

    def segment_checksums(self, streams, offsets, lengths=None, expected=None):
        """Adler-32 of every stream (ts.Segment.CalculateChecksum, src/dbnode/ts/segment.go:60-76)
        over the decoder's CSR layout; with `lengths` (int64 [S]) stream s = offsets[s] .. +lengths[s]
        (any placement, `offsets` may then have S entries); `expected` (int32/uint32 [S], the index entries' DataChecksum) turns differences
        into status M3TSZ_ERR_CHECKSUM_MISMATCH.  Returns (checksums int32-viewed-as-uint32 [S],
        status int32 [S])."""
        S = offsets.numel() - 1 if lengths is None else lengths.numel()
        dev = self.device
        out = torch.empty(S, dtype=torch.int32, device=dev)
        status = torch.empty(S, dtype=torch.int32, device=dev)
        rc = capi.lib().m3tsz_checksum_batch(
            self.ctx.handle, _ptr(streams), streams.numel(), _ptr(offsets),
            None if lengths is None else _ptr(lengths), S, None if expected is None else _ptr(expected),
            _ptr(out), _ptr(status), _cuda_stream_ptr(dev))
        self.ctx.check(rc, "m3tsz_checksum_batch")
        return out, status

    # ------------------------------------------------------------ host-buffer calls
    def decode_host(self, h_streams, h_offsets, max_points, h_ts, h_values, h_n_points, h_status):
        """All arguments are host tensors (pinned or pageable); copies are inside the call."""
        S = h_offsets.numel() - 1
        rc = capi.lib().m3tsz_decode_batch_host(
            self.ctx.handle, C.byref(self.opts), _ptr(h_streams), h_streams.numel(), _ptr(h_offsets),
            S, _ptr(h_ts), _ptr(h_values), max_points, _ptr(h_n_points), _ptr(h_status), None, None)
        self.ctx.check(rc, "m3tsz_decode_batch_host")

    def encode_host(self, h_ts, h_values, h_start, unit, h_packed, h_offsets, h_out_len, h_status,
                    align=64):
        """Host tensors in, ONE packed stream buffer + CSR offsets (int64 [S+1]) out."""
        S, P = h_ts.shape
        rc = capi.lib().m3tsz_encode_batch_host(
            self.ctx.handle, C.byref(self.opts), _ptr(h_ts), _ptr(h_values), S, P, None,
            _ptr(h_start), int(unit), None, None, None, None, 0, int(align), _ptr(h_packed),
            h_packed.numel(), _ptr(h_offsets), _ptr(h_out_len), _ptr(h_status))
        self.ctx.check(rc, "m3tsz_encode_batch_host")

    def decode_downsample_host(self, h_streams, h_offsets, range_start_ns, window_ns, n_windows,
                               h_sum, h_count, h_min, h_max, h_n_points, h_status):
        S = h_offsets.numel() - 1
        rc = capi.lib().m3tsz_decode_downsample_batch_host(
            self.ctx.handle, C.byref(self.opts), _ptr(h_streams), h_streams.numel(), _ptr(h_offsets),
            S, int(range_start_ns), int(window_ns), int(n_windows), _ptr(h_sum), _ptr(h_count),
            _ptr(h_min), _ptr(h_max), _ptr(h_n_points), _ptr(h_status))
        self.ctx.check(rc, "m3tsz_decode_downsample_batch_host")

    def fetch_host(self, h_streams, h_offsets, h_slice_off, h_replica_off, h_series_off, max_points, out_cap,
                   h_ts_out, h_val_out, h_n_out, h_status, start_ns=0, end_ns=0, strategy=0):
        """Host tensors in and out: compressed replica streams up, merged series down."""
        n_seq = h_offsets.numel() - 1
        S = h_series_off.numel() - 1
        rc = capi.lib().m3tsz_fetch_batch_host(
            self.ctx.handle, C.byref(self.opts), _ptr(h_streams), h_streams.numel(), _ptr(h_offsets), n_seq,
            _ptr(h_slice_off), _ptr(h_replica_off), _ptr(h_series_off), S, int(max_points), int(start_ns),
            int(end_ns), int(strategy), _ptr(h_ts_out), _ptr(h_val_out), int(out_cap), _ptr(h_n_out),
            _ptr(h_status))
        self.ctx.check(rc, "m3tsz_fetch_batch_host")

    def launch_count(self):
        return self.ctx.launch_count()


class EncoderSet:
    """Open encoders that live on the device (m3tsz_encoder_set_*): a state tensor uint8 [S, 128]
    (m3tsz_encoder_state) and a slot buffer uint8 [S, stride].  append() continues every stream, stream()
    snapshots them without closing; the public prefix of the state answers NumEncoded / LastEncoded /
    LastAnnotationChecksum / Len without a launch."""

    def __init__(self, codec: BatchCodec, start: torch.Tensor, stride: int):
        assert stride > 0 and stride % 16 == 0
        self.codec = codec
        self.n_series = start.numel()
        dev = codec.device
        self.state = torch.empty((self.n_series, capi.ENCODER_STATE_BYTES), dtype=torch.uint8, device=dev)
        self.buf = torch.zeros((self.n_series, stride), dtype=torch.uint8, device=dev)
        self.reset(start)

    @property
    def stride(self) -> int:
        return self.buf.shape[1]

    def reset(self, start: torch.Tensor):
        """Reset(start) of every encoder: empty streams (the slots' bytes are then free)."""
        assert start.dtype == torch.int64 and start.is_cuda and start.numel() == self.n_series
        start = start.contiguous()
        rc = capi.lib().m3tsz_encoder_set_reset(self.codec.ctx.handle, C.byref(self.codec.opts), _ptr(self.state),
                                                self.n_series, _ptr(start), _cuda_stream_ptr(self.codec.device))
        self.codec.ctx.check(rc, "m3tsz_encoder_set_reset")

    def append(self, ts: torch.Tensor, values: torch.Tensor, n_points: Optional[torch.Tensor] = None,
               units: Optional[torch.Tensor] = None, annotations=None, point_major=False, unit=capi.UNIT_S):
        """Appends ts / values int64 / float64 [S, P] ([P, S] when point_major) to the encoders; n_points
        (int32 [S]) takes the first n_points[s] of series s, 0 leaves it untouched.  units / annotations as
        BatchCodec.encode (series-major only; annotation dp_index counts within this call).  Returns
        (n_appended int32 [S], status int32 [S]): a series stops at its first failing datapoint, and its state
        is as after the last datapoint taken."""
        assert ts.dtype == torch.int64 and values.dtype == torch.float64
        assert ts.is_cuda and values.is_cuda and ts.is_contiguous() and values.is_contiguous()
        S, P = (ts.shape[1], ts.shape[0]) if point_major else ts.shape
        assert S == self.n_series
        dev = self.codec.device
        if P == 0:  # nothing to append (an empty tensor may have no storage to point at)
            return (torch.zeros(S, dtype=torch.int32, device=dev), torch.zeros(S, dtype=torch.int32, device=dev))
        n_appended = torch.empty(S, dtype=torch.int32, device=dev)
        status = torch.empty(S, dtype=torch.int32, device=dev)
        a_off = a_ent = a_bytes = None
        if annotations is not None:
            a_off, a_ent, a_bytes = annotations
        rc = capi.lib().m3tsz_encoder_set_append(
            self.codec.ctx.handle, C.byref(self.codec.opts), _ptr(self.state), S, _ptr(ts), _ptr(values), P,
            _ptr(n_points), int(unit), _ptr(units), _ptr(a_off), _ptr(a_ent), _ptr(a_bytes),
            1 if point_major else 0, _ptr(self.buf), self.stride, _ptr(n_appended), _ptr(status),
            _cuda_stream_ptr(dev))
        self.codec.ctx.check(rc, "m3tsz_encoder_set_append")
        return n_appended, status

    def stream(self) -> EncodeResult:
        """Stream() of every encoder: out = the slot buffer [S, stride], out_len = the snapshot lengths (0 for an
        empty encoder), as BatchCodec.encode returns them.  compact() takes it as it is; decode takes
        out.view(-1) with offsets = self.offsets() and lengths = out_len."""
        dev = self.codec.device
        out_len = torch.empty(self.n_series, dtype=torch.int64, device=dev)
        rc = capi.lib().m3tsz_encoder_set_stream(self.codec.ctx.handle, _ptr(self.state), self.n_series,
                                                 _ptr(self.buf), self.stride, _ptr(out_len), _cuda_stream_ptr(dev))
        self.codec.ctx.check(rc, "m3tsz_encoder_set_stream")
        return EncodeResult(out=self.buf, out_len=out_len,
                            status=torch.zeros(self.n_series, dtype=torch.int32, device=dev))

    def offsets(self) -> torch.Tensor:
        """Start of every slot in buf.view(-1), for decode(..., lengths=...)."""
        return torch.arange(self.n_series, dtype=torch.int64, device=self.codec.device) * self.stride

    def grow(self, stride: int):
        """Moves the slots into a buffer of `stride` bytes each (the state holds positions, not pointers)."""
        assert stride % 16 == 0 and stride >= self.stride
        buf = torch.zeros((self.n_series, stride), dtype=torch.uint8, device=self.codec.device)
        buf[:, : self.stride] = self.buf
        self.buf = buf

    # public prefix of m3tsz_encoder_state: start_ns, num_encoded, last_ts, last_value, ann_checksum, bits
    def _field(self, i):
        return self.state.view(torch.int64)[:, i]

    @property
    def num_encoded(self) -> torch.Tensor:
        return self._field(1)

    @property
    def last_encoded(self):
        """(ts int64 [S], value float64 [S]): LastEncoded(), meaningful where num_encoded > 0."""
        return self._field(2), self.state.view(torch.float64)[:, 3]

    @property
    def ann_checksum(self) -> torch.Tensor:
        """LastAnnotationChecksum() as int64 [S] (the uint64's bits)."""
        return self._field(4)

    @property
    def len(self) -> torch.Tensor:
        """Len(): stream bytes with the tail, 0 for an empty encoder."""
        n, bits = self._field(1), self._field(5)
        return torch.where(n > 0, (bits + 11 + 7) // 8, torch.zeros_like(bits))


class BucketSet:
    """Buffer buckets on the device: per series up to `encoders` (K) in-order encoders, as BufferBucket keeps them
    (src/dbnode/storage/series/buffer.go:1261-1391).  Encoder 0 of every series is `primary` (an EncoderSet); the
    others come from an overflow pool: `pool` uint8 [M, 128] states, `pool_buf` uint8 [M, pool_stride] slots,
    `pool_count` int32 [1] records in use and `table` int32 [S, K-1] (the pool record of encoder i + 1, -1: not
    open).  write() routes every datapoint as BufferBucket.write does; read() merges a bucket's encoders as a
    reader of the open block sees them."""

    def __init__(self, codec: BatchCodec, start: torch.Tensor, stride: int, encoders: int, pool_records: int,
                 pool_stride: int):
        assert 1 <= encoders <= capi.MAX_BUCKET_ENCODERS
        assert pool_stride > 0 and pool_stride % 16 == 0 and pool_records > 0
        self.codec = codec
        self.encoders = int(encoders)
        self.primary = EncoderSet(codec, start, stride)
        self.n_series = self.primary.n_series
        dev = codec.device
        M = int(pool_records) if self.encoders > 1 else 0
        self.pool = torch.zeros((M, capi.ENCODER_STATE_BYTES), dtype=torch.uint8, device=dev)
        self.pool_buf = torch.zeros((M, pool_stride), dtype=torch.uint8, device=dev)
        self.pool_count = torch.zeros(1, dtype=torch.int32, device=dev)
        self.table = torch.full((self.n_series, self.encoders - 1), -1, dtype=torch.int32, device=dev)

    def reset(self, start: torch.Tensor):
        """Reset(start) of every bucket: encoder 0 empty, every overflow record free."""
        self.primary.reset(start)
        self.pool_count.zero_()
        self.table.fill_(-1)

    def write(self, ts: torch.Tensor, values: torch.Tensor, n_points: Optional[torch.Tensor] = None,
              units: Optional[torch.Tensor] = None, annotations=None, point_major=False, unit=capi.UNIT_S):
        """BufferBucket.write of every datapoint, in call order per series; inputs as EncoderSet.append.  Returns
        (result int8 in the inputs' shape: 0 written, -1 unchanged, else the failed write's status; status int32
        [S]: OK, ERR_CAPACITY -- that datapoint and the rest of the series were not written: grow() and send them
        again -- or ERR_INVALID_ARG)."""
        assert ts.dtype == torch.int64 and values.dtype == torch.float64
        assert ts.is_cuda and values.is_cuda and ts.is_contiguous() and values.is_contiguous()
        S, P = (ts.shape[1], ts.shape[0]) if point_major else ts.shape
        assert S == self.n_series
        dev = self.codec.device
        result = torch.zeros(ts.shape, dtype=torch.int8, device=dev)
        status = torch.zeros(S, dtype=torch.int32, device=dev)
        if P == 0:
            return result, status
        a_off = a_ent = a_bytes = None
        if annotations is not None:
            a_off, a_ent, a_bytes = annotations
        M = self.pool.shape[0]
        pr = self.primary
        rc = capi.lib().m3tsz_encoder_set_write(
            self.codec.ctx.handle, C.byref(self.codec.opts), _ptr(pr.state), _ptr(pr.buf), pr.stride, S,
            _ptr(self.pool) if M else None, _ptr(self.pool_buf) if M else None, self.pool_stride, M,
            _ptr(self.pool_count), _ptr(self.table) if self.encoders > 1 else None, self.encoders, _ptr(ts),
            _ptr(values), P, _ptr(n_points), int(unit), _ptr(units), _ptr(a_off), _ptr(a_ent), _ptr(a_bytes),
            1 if point_major else 0, _ptr(result), _ptr(status), _cuda_stream_ptr(dev))
        self.codec.ctx.check(rc, "m3tsz_encoder_set_write")
        return result, status

    @property
    def stride(self) -> int:
        return self.primary.stride

    @property
    def pool_stride(self) -> int:
        return self.pool_buf.shape[1]

    def grow(self, stride: Optional[int] = None, pool_stride: Optional[int] = None,
             pool_records: Optional[int] = None):
        """Larger primary slots, pool slots or pool (every record keeps its position)."""
        if stride is not None:
            self.primary.grow(stride)
        M, ps = self.pool.shape[0], self.pool_stride
        M2 = M if pool_records is None or self.encoders == 1 else int(pool_records)
        ps2 = ps if pool_stride is None else int(pool_stride)
        assert M2 >= M and ps2 >= ps and ps2 % 16 == 0
        if (M2, ps2) != (M, ps):
            pool = torch.zeros((M2, capi.ENCODER_STATE_BYTES), dtype=torch.uint8, device=self.codec.device)
            pool[:M] = self.pool
            buf = torch.zeros((M2, ps2), dtype=torch.uint8, device=self.codec.device)
            buf[:M, :ps] = self.pool_buf
            self.pool, self.pool_buf = pool, buf

    def open_encoders(self) -> torch.Tensor:
        """Encoders open per bucket, int64 [S] (encoder 0 always counts)."""
        return 1 + (self.table >= 0).sum(1)

    def encoder_state(self, i: int):
        """(state uint8 [S, 128] of encoder i of every bucket, open bool [S]); rows of buckets where encoder i is
        not open are zero.  The public prefix (m3tsz_encoder_state) answers NumEncoded / LastEncoded /
        LastAnnotationChecksum / Len, as EncoderSet's accessors read it."""
        if i == 0:
            return self.primary.state, torch.ones(self.n_series, dtype=torch.bool, device=self.codec.device)
        rec = self.table[:, i - 1].long()
        is_open = rec >= 0
        st = self.pool[rec.clamp(min=0)] * is_open[:, None].to(torch.uint8)
        return st, is_open

    def num_encoded(self, i: int) -> torch.Tensor:
        return self.encoder_state(i)[0].view(torch.int64)[:, 1]

    def last_encoded(self, i: int):
        st = self.encoder_state(i)[0]
        return st.view(torch.int64)[:, 2], st.view(torch.float64)[:, 3]

    def ann_checksum(self, i: int) -> torch.Tensor:
        return self.encoder_state(i)[0].view(torch.int64)[:, 4]

    def stream(self):
        """Stream() of every encoder: (primary EncodeResult [S], pool EncodeResult [records in use]); pool record r
        of bucket s is table[s, i - 1] for encoder i."""
        used = int(self.pool_count.item())
        dev = self.codec.device
        pool_len = torch.zeros(used, dtype=torch.int64, device=dev)
        if used:
            rc = capi.lib().m3tsz_encoder_set_stream(self.codec.ctx.handle, _ptr(self.pool), used,
                                                     _ptr(self.pool_buf), self.pool_stride, _ptr(pool_len),
                                                     _cuda_stream_ptr(dev))
            self.codec.ctx.check(rc, "m3tsz_encoder_set_stream")
        pool = EncodeResult(out=self.pool_buf[:used], out_len=pool_len,
                            status=torch.zeros(used, dtype=torch.int32, device=dev))
        return self.primary.stream(), pool

    def read(self, out_cap: int, start_ns=0, end_ns=0):
        """What a reader of the open block sees (BufferBucket.streams, buffer.go:1366-1391, merged by a
        MultiReaderIterator): every encoder's snapshot decoded, then merged per series -- encoder 0, then the open
        overflow encoders by index, as readers of one block slice, equal timestamps going to the last pushed.
        Returns merge_series' (ts [S, out_cap], values, n int32 [S], status int32 [S])."""
        prim, pool = self.stream()
        S, dev = self.n_series, self.codec.device
        decs = []
        for enc, n in ((prim, S), (pool, pool.out.shape[0])):
            if n == 0:
                continue
            stride = enc.out.shape[1]
            offs = torch.arange(n, dtype=torch.int64, device=dev) * stride
            d = self.codec.decode(enc.out.reshape(-1), offs, out_cap, lengths=enc.out_len)
            # an empty encoder is no stream at all (streams() skips it)
            empty = enc.out_len == 0
            d.n_points.masked_fill_(empty, 0)
            d.status.masked_fill_(empty, 0)
            decs.append(d)
        cat = lambda f: torch.cat([getattr(d, f) for d in decs])
        ts, vals, npts, st = cat("ts"), cat("values"), cat("n_points"), cat("status")
        # sequences in series order: encoder 0 of s, then its open overflow records in encoder order
        idx = torch.cat([torch.arange(S, dtype=torch.int64, device=dev)[:, None], S + self.table.long()], 1)
        is_open = torch.cat([torch.ones((S, 1), dtype=torch.bool, device=dev), self.table >= 0], 1)
        seq = idx[is_open]
        counts = is_open.sum(1)
        slice_off = torch.zeros(S + 1, dtype=torch.int64, device=dev)
        slice_off[1:] = torch.cumsum(counts, 0)
        ident = torch.arange(S + 1, dtype=torch.int64, device=dev)
        return self.codec.merge_series(ts[seq].contiguous(), vals[seq].contiguous(), npts[seq].contiguous(),
                                       st[seq].contiguous(), slice_off, ident, ident, out_cap, start_ns, end_ns,
                                       strategy=0)


class ForwardedBatch:
    """The records a shard's forwarded writer wrote (ElementSet.forward_write): `metrics` uint8 [M, 40] rows of
    capi.ForwardedMetric (key, time_ns, value_off, n_values, source_id, version, reserved), `values` float64 [V], and
    `counts` (metrics written, values written, metrics needed, values needed).  Pointer-free: a batch can be copied
    or sent as bytes."""

    def __init__(self, metrics: torch.Tensor, values: torch.Tensor, counts):
        self.metrics, self.values, self.counts = metrics, values, tuple(int(c) for c in counts)

    def fields(self):
        """The records as numpy arrays {"key", "time_ns", "value_off", "n_values", "source_id", "version",
        "reserved"}."""
        import numpy as np
        a = self.metrics.cpu().numpy().reshape(-1, capi.FORWARDED_METRIC_BYTES)
        u64 = lambda o: a[:, o:o + 8].copy().view(np.uint64)[:, 0]
        u32 = lambda o: a[:, o:o + 4].copy().view(np.uint32)[:, 0]
        return {"key": u64(0), "time_ns": u64(8).view(np.int64), "value_off": u64(16), "n_values": u32(24),
                "source_id": u32(28), "version": u32(32), "reserved": u32(36)}

    @staticmethod
    def concat(batches) -> "ForwardedBatch":
        """One batch of the given batches' records in order, each batch's value offsets moved past the values
        before it."""
        batches = list(batches)
        ms, vs, base = [], [], 0
        for b in batches:
            m = b.metrics.clone()
            if m.shape[0]:
                off = m[:, 16:24].contiguous().view(torch.int64).view(-1) + base
                m[:, 16:24] = off.view(torch.uint8).view(-1, 8)
            ms.append(m)
            vs.append(b.values)
            base += b.values.numel()
        dev = batches[0].metrics.device if batches else "cuda"
        metrics = torch.cat(ms) if ms else torch.zeros((0, capi.FORWARDED_METRIC_BYTES), dtype=torch.uint8, device=dev)
        values = torch.cat(vs) if vs else torch.zeros(0, dtype=torch.float64, device=dev)
        return ForwardedBatch(metrics, values, (metrics.shape[0], values.numel(), metrics.shape[0], values.numel()))


class ElementSet:
    """Aggregator elements on the device (m3tsz_element_set_*, DESIGN.md §4.12).  The caller-side arrays: `win`, the
    open-window slots window-slot-major [R, N] (start, count -- 0 for a free slot -- sum, min, max, sum_sq, and for
    the Gauge last / last_at; a Counter's aggregates are int64), `elem` uint8 [N, 160] (m3tsz_element_state),
    `watermark` int64 [N] (the end of the last window consumed, INT64_MIN for none) and `out`, the EncoderSet the
    flushed windows are appended to.  add() puts datapoints into open windows, consume() flushes the windows that
    ended by a target time.  With an annotation capacity the set keeps annotations: `ann_len` int32 [R, N] (bytes of
    each slot's annotation, 0 for none) and `ann_bytes` uint8 [R, N, capacity], and every call is the annotated one.
    A Timer set (metric_type capi.METRIC_TIMER) keeps start, count, sum and sum_sq (float64) per slot, and each slot's
    CM stream in `streams`: "header" uint8 [R, N, 64] and the sample arrays [R, sample_capacity, N] ("value",
    "num_ranks", "delta", "prev", "next", "heap_a", "heap_b"); every call is the Timer one."""

    def __init__(self, codec: BatchCodec, start: torch.Tensor, metric_type, agg_types, resolution_ns, transforms,
                 discard_nan, open_windows, stride, out_unit, annotation_capacity=0, sample_capacity=None, eps=1e-3,
                 insert_and_compress_every=1024, source_capacity=0):
        assert start.dtype == torch.int64 and start.is_cuda
        self.codec = codec
        self.metric_type = int(metric_type)
        self.agg_types = [int(t) for t in agg_types]
        self.transforms = [int(t) for t in transforms]
        self.discard_nan = bool(discard_nan)
        self.resolution_ns = int(resolution_ns)
        self.out_unit = int(out_unit)
        self.n_elements = start.numel()
        k, N, R = len(self.agg_types), self.n_elements, int(open_windows)
        assert k >= 1 and R >= 1
        self._types = (C.c_int32 * k)(*self.agg_types)
        self._ops = (C.c_int32 * max(1, len(self.transforms)))(*self.transforms)
        dev = codec.device
        counter = self.metric_type == capi.METRIC_COUNTER
        agg = torch.int64 if counter else torch.float64
        names = [("start", torch.int64), ("count", torch.int64), ("sum", agg), ("min", agg), ("max", agg),
                 ("sum_sq", agg)] + ([] if counter else [("last", torch.float64), ("last_at", torch.int64)])
        self.streams = None
        if self.timer:
            if sample_capacity is None or int(sample_capacity) < 1:
                raise ValueError("a Timer set needs sample_capacity >= 1")
            names = [("start", torch.int64), ("count", torch.int64), ("sum", torch.float64),
                     ("sum_sq", torch.float64)]
            self.eps, self.insert_and_compress_every = float(eps), int(insert_and_compress_every)
            self.streams = {"header": torch.zeros((R, N, capi.TIMER_STREAM_HEADER_BYTES), dtype=torch.uint8,
                                                  device=dev)}
            for f, t in self._STREAM_ARRAYS:
                self.streams[f] = torch.zeros((R, int(sample_capacity), N), dtype=t, device=dev)
        self.win = {f: torch.zeros((R, N), dtype=t, device=dev) for f, t in names}
        self.elem = torch.zeros((N, capi.ELEMENT_STATE_BYTES), dtype=torch.uint8, device=dev)
        self.watermark = torch.empty(N, dtype=torch.int64, device=dev)
        self.ann_len = self.ann_bytes = None
        if annotation_capacity:
            self.ann_len = torch.zeros((R, N), dtype=torch.int32, device=dev)
            self.ann_bytes = torch.zeros((R, N, int(annotation_capacity)), dtype=torch.uint8, device=dev)
        self.source_bits = None
        if source_capacity:
            self.source_bits = torch.zeros((R, int(source_capacity) // 32, N), dtype=torch.int32, device=dev)
        if stride is None:
            stride = int(capi.lib().m3tsz_encode_bound_units(128, 1))
        start = start.contiguous()
        self.out = EncoderSet(codec, start.repeat(k), stride) if stride else None
        self.reset(start)

    _STREAM_ARRAYS = (("value", torch.float64), ("num_ranks", torch.int64), ("delta", torch.int64),
                      ("prev", torch.int32), ("next", torch.int32), ("heap_a", torch.float64),
                      ("heap_b", torch.float64))

    @property
    def timer(self) -> bool:
        return self.metric_type == capi.METRIC_TIMER

    @property
    def open_windows(self) -> int:
        return self.win["start"].shape[0]

    @property
    def sample_capacity(self) -> int:
        return 0 if self.streams is None else self.streams["value"].shape[1]

    def _streams(self):
        st = capi.ElementTimerStreams()
        st.d_header = self.streams["header"].data_ptr()
        for f, _ in self._STREAM_ARRAYS:
            setattr(st, "d_" + f, self.streams[f].data_ptr())
        st.sample_capacity = self.sample_capacity
        st.insert_and_compress_every = self.insert_and_compress_every
        st.eps = self.eps
        return st

    def _desc(self):
        w = self.win
        d = capi.ElementSet()
        d.n_elements = self.n_elements
        d.n_windows = self.open_windows
        d.metric_type = self.metric_type
        d.resolution_ns = self.resolution_ns
        d.agg_types = C.cast(self._types, C.POINTER(C.c_int32))
        d.n_types = len(self.agg_types)
        d.n_ops = len(self.transforms)
        d.ops = C.cast(self._ops, C.POINTER(C.c_int32))
        d.discard_nan = 1 if self.discard_nan else 0
        for f in ("start", "count", "sum", "min", "max", "sum_sq", "last", "last_at"):
            setattr(d, "d_win_" + f, w[f].data_ptr() if f in w else None)
        d.d_elem = self.elem.data_ptr()
        d.d_watermark = self.watermark.data_ptr()
        if self.out is not None:
            d.d_out_state = self.out.state.data_ptr()
            d.d_out_buf = self.out.buf.data_ptr()
            d.out_stride = self.out.stride
        return d

    def _require_output(self):
        if self.out is None:
            raise ValueError("this element set has no output rows (stride=0): it is a rollup's source set")

    @property
    def annotation_capacity(self) -> int:
        return 0 if self.ann_bytes is None else self.ann_bytes.shape[2]

    def _ann(self):
        a = capi.ElementAnnotations()
        a.d_len = self.ann_len.data_ptr()
        a.d_bytes = self.ann_bytes.data_ptr()
        a.capacity = self.annotation_capacity
        return a

    def reset(self, start: torch.Tensor):
        """Every element new: windows free, records zero, nothing consumed, output rows Reset(start[s])."""
        assert start.dtype == torch.int64 and start.is_cuda and start.numel() == self.n_elements
        start = start.contiguous()
        d = self._desc()
        rc = capi.lib().m3tsz_element_set_reset(self.codec.ctx.handle, C.byref(self.codec.opts), C.byref(d),
                                                _ptr(start), _cuda_stream_ptr(self.codec.device))
        self.codec.ctx.check(rc, "m3tsz_element_set_reset")
        if self.ann_len is not None:
            self.ann_len.zero_()

    def add(self, ts: torch.Tensor, values: torch.Tensor, n_points: Optional[torch.Tensor] = None,
            annotations=None, batch: Optional[torch.Tensor] = None):
        """AddUnion of point-major ts / values int64 / float64 [P, N]: element s takes n_points[s] (int32 [N]; all P
        when None) of its column, in order.  Returns (result int8 [P, N]: 0 added, else ERR_AGGREGATION_CLOSED /
        ERR_CAPACITY / ERR_INVALID_ARG, rows past an element's count left 0; status int32 [N]: OK, ERR_CAPACITY --
        that datapoint and the element's later ones were not added: grow() and add them again -- or
        ERR_INVALID_ARG).  annotations (a set with an annotation capacity only): (series_off int64 [N + 1], entries
        capi.AnnotationEntry rows as uint8 [E, 16], bytes uint8) as EncoderSet.append takes them, dp_index counting
        rows of the element's column; an annotation longer than the capacity stops the element with ERR_CAPACITY
        (grow(annotation_capacity=...) and add again).
        A Timer set (m3tsz_element_set_add_timer): batch (int8 [P, N], optional) marks the rows that continue the
        previous row's batch (BatchTimer; None: every row is its own, AppendTimerSample).  A batch is taken or refused
        whole; ERR_CAPACITY (too few open windows, or more than sample_capacity values in its window's slot) stops the
        element: grow() and add exactly the refused rows again.  A continuation in row 0, or one with another
        timestamp than its batch's first row, refuses the element (ERR_INVALID_ARG, untouched).  With annotations
        (m3tsz_element_set_add_timer_annotated) a batch's annotation is its first row's entry; an annotation on a
        continuation row refuses the element the same way."""
        assert ts.dtype == torch.int64 and values.dtype == torch.float64 and ts.shape == values.shape
        assert ts.is_cuda and values.is_cuda and ts.is_contiguous() and values.is_contiguous()
        assert ts.dim() == 2 and ts.shape[1] == self.n_elements
        if n_points is not None:
            assert n_points.dtype == torch.int32 and n_points.is_cuda and n_points.is_contiguous()
            assert n_points.numel() == self.n_elements
        dev = self.codec.device
        P = ts.shape[0]
        result = torch.zeros(ts.shape, dtype=torch.int8, device=dev)
        status = torch.zeros(self.n_elements, dtype=torch.int32, device=dev)
        if P == 0:
            return result, status
        d = self._desc()
        if self.timer:
            if batch is not None:
                assert batch.dtype == torch.int8 and batch.is_cuda and batch.is_contiguous()
                assert batch.shape == ts.shape
            if self.ann_len is None:
                assert annotations is None, "a set without an annotation capacity takes no annotations"
                rc = capi.lib().m3tsz_element_set_add_timer(
                    self.codec.ctx.handle, C.byref(self.codec.opts), C.byref(d), C.byref(self._streams()), _ptr(ts),
                    _ptr(values), P, _ptr(n_points), _ptr(batch), _ptr(result), _ptr(status), _cuda_stream_ptr(dev))
                self.codec.ctx.check(rc, "m3tsz_element_set_add_timer")
                return result, status
            a_off, a_ent, a_bytes = annotations if annotations is not None else (None, None, None)
            rc = capi.lib().m3tsz_element_set_add_timer_annotated(
                self.codec.ctx.handle, C.byref(self.codec.opts), C.byref(d), C.byref(self._streams()),
                C.byref(self._ann()), _ptr(ts), _ptr(values), P, _ptr(n_points), _ptr(batch), _ptr(a_off),
                _ptr(a_ent), _ptr(a_bytes), _ptr(result), _ptr(status), _cuda_stream_ptr(dev))
            self.codec.ctx.check(rc, "m3tsz_element_set_add_timer_annotated")
            return result, status
        assert batch is None, "only a Timer set takes batches"
        if self.ann_len is None:
            assert annotations is None, "a set without an annotation capacity takes no annotations"
            rc = capi.lib().m3tsz_element_set_add(self.codec.ctx.handle, C.byref(self.codec.opts), C.byref(d),
                                                  _ptr(ts), _ptr(values), P, _ptr(n_points), _ptr(result),
                                                  _ptr(status), _cuda_stream_ptr(dev))
            self.codec.ctx.check(rc, "m3tsz_element_set_add")
            return result, status
        a_off = a_ent = a_bytes = None
        if annotations is not None:
            a_off, a_ent, a_bytes = annotations
        a = self._ann()
        rc = capi.lib().m3tsz_element_set_add_annotated(
            self.codec.ctx.handle, C.byref(self.codec.opts), C.byref(d), C.byref(a), _ptr(ts), _ptr(values), P,
            _ptr(n_points), _ptr(a_off), _ptr(a_ent), _ptr(a_bytes), _ptr(result), _ptr(status),
            _cuda_stream_ptr(dev))
        self.codec.ctx.check(rc, "m3tsz_element_set_add_annotated")
        return result, status

    def consume(self, target_ns) -> torch.Tensor:
        """Consume(target_ns): every open window that ended by target_ns, in order, through the element and onto
        the output rows.  Returns status int32 [N]: OK, ERR_CAPACITY (the element's output slots lack room: it is
        unchanged; grow(stride=...) and consume again), or a row's append status."""
        self._require_output()
        dev = self.codec.device
        status = torch.empty(self.n_elements, dtype=torch.int32, device=dev)
        d = self._desc()
        if self.timer and self.ann_len is None:
            rc = capi.lib().m3tsz_element_set_consume_timer(self.codec.ctx.handle, C.byref(self.codec.opts),
                                                            C.byref(d), C.byref(self._streams()), int(target_ns),
                                                            self.out_unit, _ptr(status), _cuda_stream_ptr(dev))
            self.codec.ctx.check(rc, "m3tsz_element_set_consume_timer")
            return status
        if self.timer:
            rc = capi.lib().m3tsz_element_set_consume_timer_annotated(
                self.codec.ctx.handle, C.byref(self.codec.opts), C.byref(d), C.byref(self._streams()),
                C.byref(self._ann()), int(target_ns), self.out_unit, _ptr(status), _cuda_stream_ptr(dev))
            self.codec.ctx.check(rc, "m3tsz_element_set_consume_timer_annotated")
            return status
        if self.ann_len is None:
            rc = capi.lib().m3tsz_element_set_consume(self.codec.ctx.handle, C.byref(self.codec.opts), C.byref(d),
                                                      int(target_ns), self.out_unit, _ptr(status),
                                                      _cuda_stream_ptr(dev))
            self.codec.ctx.check(rc, "m3tsz_element_set_consume")
            return status
        a = self._ann()
        rc = capi.lib().m3tsz_element_set_consume_annotated(self.codec.ctx.handle, C.byref(self.codec.opts),
                                                            C.byref(d), C.byref(a), int(target_ns), self.out_unit,
                                                            _ptr(status), _cuda_stream_ptr(dev))
        self.codec.ctx.check(rc, "m3tsz_element_set_consume_annotated")
        return status

    def grow(self, open_windows: Optional[int] = None, stride: Optional[int] = None,
             annotation_capacity: Optional[int] = None, sample_capacity: Optional[int] = None,
             source_capacity: Optional[int] = None):
        """More open-window slots per element (the slots are copied; the new ones are free), larger output slots
        (EncoderSet.grow) and / or, for a set that keeps annotations, more annotation bytes per slot (copied), or for a
        Timer set more stream samples per slot (copied), or for a set fed by add_forwarded more source ids per slot
        (copied)."""
        if source_capacity is not None and source_capacity != self.source_capacity:
            assert self.source_bits is not None and source_capacity > self.source_capacity
            b = torch.zeros((self.open_windows, int(source_capacity) // 32, self.n_elements), dtype=torch.int32,
                            device=self.source_bits.device)
            b[:, : self.source_bits.shape[1]] = self.source_bits
            self.source_bits = b
        if sample_capacity is not None and sample_capacity != self.sample_capacity:
            assert self.timer and sample_capacity > self.sample_capacity
            C0 = self.sample_capacity
            for f, a in self.streams.items():
                if f != "header":
                    b = torch.zeros((a.shape[0], int(sample_capacity), a.shape[2]), dtype=a.dtype, device=a.device)
                    b[:, :C0] = a
                    self.streams[f] = b
        if open_windows is not None and open_windows != self.open_windows:
            R = self.open_windows
            assert open_windows > R
            for f, a in self.win.items():
                b = torch.zeros((open_windows, self.n_elements), dtype=a.dtype, device=a.device)
                b[:R] = a
                self.win[f] = b
            if self.ann_len is not None:
                ln = torch.zeros((open_windows, self.n_elements), dtype=torch.int32, device=self.ann_len.device)
                ln[:R] = self.ann_len
                by = torch.zeros((open_windows,) + tuple(self.ann_bytes.shape[1:]), dtype=torch.uint8,
                                 device=self.ann_bytes.device)
                by[:R] = self.ann_bytes
                self.ann_len, self.ann_bytes = ln, by
            if self.source_bits is not None:
                b = torch.zeros((open_windows,) + tuple(self.source_bits.shape[1:]), dtype=torch.int32,
                                device=self.source_bits.device)
                b[:R] = self.source_bits
                self.source_bits = b
            if self.streams is not None:
                for f, a in self.streams.items():
                    b = torch.zeros((open_windows,) + tuple(a.shape[1:]), dtype=a.dtype, device=a.device)
                    b[:R] = a
                    self.streams[f] = b
        if annotation_capacity is not None and annotation_capacity != self.annotation_capacity:
            assert self.ann_bytes is not None and annotation_capacity > self.annotation_capacity
            by = torch.zeros(tuple(self.ann_bytes.shape[:2]) + (int(annotation_capacity),), dtype=torch.uint8,
                             device=self.ann_bytes.device)
            by[:, :, : self.annotation_capacity] = self.ann_bytes
            self.ann_bytes = by
        if stride is not None:
            self._require_output()
            if stride != self.out.stride:
                self.out.grow(stride)

    def stream(self) -> EncodeResult:
        """The output rows' snapshot (EncoderSet.stream): row j * N + s is element s under agg_types[j]."""
        self._require_output()
        return self.out.stream()

    def forward(self, target_ns, group_off: torch.Tensor, members: torch.Tensor, groups: "ElementSet"):
        """This set as a rollup's source set (m3tsz_element_set_forward, DESIGN.md §4.12): every element's open
        windows that ended by target_ns go, through ValueOf of the set's one type and its transformations, to the
        groups that list it; group g of `groups` (an ElementSet of the same metric type and resolution, one element
        per group) takes the values of the sources members[group_off[g] .. group_off[g + 1])
        (int64 [G + 1] and int32 [n] device tensors, as aggregate_tiles_rollup takes them), in that order, into its
        window with the source window's start.  Returns (source statuses int32 [N]: OK, or the status of a failed
        group that held the source back; group statuses int32 [G]: OK, ERR_AGGREGATION_CLOSED -- a window that ended
        by the group's watermark was dropped --, ERR_CAPACITY -- too few open windows: groups.grow(open_windows=...)
        and forward again with exactly the failed groups --, or ERR_INVALID_ARG).
        When `groups` keeps annotations (m3tsz_element_set_forward_annotated) this set must keep them too: each
        forwarded window carries its annotation, and each value with one replaces its group window's annotation, in
        the listed member order.  A group whose forwarded annotation is longer than its capacity gets ERR_CAPACITY
        too: groups.grow(annotation_capacity=...) and forward again with exactly the failed groups.  A group set
        without annotations takes the plain call, whatever this set keeps.  Timer sets forward with forward_timer."""
        assert isinstance(groups, ElementSet)
        if self.timer or groups.timer:
            raise ValueError("Timer sets take no forward")
        if groups.ann_len is not None and self.ann_len is None:
            raise ValueError("a group set that keeps annotations needs a source set that keeps them")
        assert group_off.is_cuda and group_off.dtype == torch.int64 and group_off.is_contiguous()
        assert members.is_cuda and members.dtype == torch.int32 and members.is_contiguous()
        G = group_off.numel() - 1
        assert G >= 0, "group_off has G + 1 entries"
        dev = self.codec.device
        src_status = torch.empty(max(1, self.n_elements), dtype=torch.int32, device=dev)
        group_status = torch.empty(max(1, G), dtype=torch.int32, device=dev)
        d, gd = self._desc(), groups._desc()
        if groups.ann_len is None:
            rc = capi.lib().m3tsz_element_set_forward(
                self.codec.ctx.handle, C.byref(self.codec.opts), C.byref(d), int(target_ns), _ptr(group_off),
                _ptr(members), members.numel(), G, C.byref(gd), _ptr(src_status), _ptr(group_status),
                _cuda_stream_ptr(dev))
            self.codec.ctx.check(rc, "m3tsz_element_set_forward")
            return src_status[: self.n_elements], group_status[:G]
        a, ga = self._ann(), groups._ann()
        rc = capi.lib().m3tsz_element_set_forward_annotated(
            self.codec.ctx.handle, C.byref(self.codec.opts), C.byref(d), C.byref(a), int(target_ns), _ptr(group_off),
            _ptr(members), members.numel(), G, C.byref(gd), C.byref(ga), _ptr(src_status), _ptr(group_status),
            _cuda_stream_ptr(dev))
        self.codec.ctx.check(rc, "m3tsz_element_set_forward_annotated")
        return src_status[: self.n_elements], group_status[:G]

    def forward_timer(self, target_ns, group_off: torch.Tensor, members: torch.Tensor, groups: "ElementSet"):
        """forward for Timer sets (m3tsz_element_set_forward_timer, DESIGN.md §4.12), with the same arguments and
        return values: this set (one type, any but Last; its transformations the pre-rollup ones) flushes each due
        window's stream and forwards ValueOf(its type); group g of `groups` (a Timer set of the same resolution)
        takes each value as one Timer.Add into its window with the source window's start, members in listed order.
        A group gets ERR_CAPACITY when it needs more windows than it has free slots, or when a window it touches
        would hold more than groups.sample_capacity values: its list samples and pending values plus every value
        this call folds into it.  Nothing is then folded into the group and its members are held back:
        groups.grow(open_windows=..., sample_capacity=...) and forward again with exactly the failed groups, which
        gives the result of one unstopped call.
        Annotations follow forward's rule: when `groups` keeps them (m3tsz_element_set_forward_timer_annotated) this
        set must keep them too, and a group whose forwarded annotation is longer than its capacity gets ERR_CAPACITY
        (groups.grow(annotation_capacity=...)); a group set without annotations takes the plain call."""
        assert isinstance(groups, ElementSet)
        if not (self.timer and groups.timer):
            raise ValueError("forward_timer takes Timer sets; other sets forward with forward")
        if groups.ann_len is not None and self.ann_len is None:
            raise ValueError("a group set that keeps annotations needs a source set that keeps them")
        assert group_off.is_cuda and group_off.dtype == torch.int64 and group_off.is_contiguous()
        assert members.is_cuda and members.dtype == torch.int32 and members.is_contiguous()
        G = group_off.numel() - 1
        assert G >= 0, "group_off has G + 1 entries"
        dev = self.codec.device
        src_status = torch.empty(max(1, self.n_elements), dtype=torch.int32, device=dev)
        group_status = torch.empty(max(1, G), dtype=torch.int32, device=dev)
        d, gd = self._desc(), groups._desc()
        if groups.ann_len is None:
            rc = capi.lib().m3tsz_element_set_forward_timer(
                self.codec.ctx.handle, C.byref(self.codec.opts), C.byref(d), C.byref(self._streams()), int(target_ns),
                _ptr(group_off), _ptr(members), members.numel(), G, C.byref(gd), C.byref(groups._streams()),
                _ptr(src_status), _ptr(group_status), _cuda_stream_ptr(dev))
            self.codec.ctx.check(rc, "m3tsz_element_set_forward_timer")
            return src_status[: self.n_elements], group_status[:G]
        rc = capi.lib().m3tsz_element_set_forward_timer_annotated(
            self.codec.ctx.handle, C.byref(self.codec.opts), C.byref(d), C.byref(self._streams()),
            C.byref(self._ann()), int(target_ns), _ptr(group_off), _ptr(members), members.numel(), G, C.byref(gd),
            C.byref(groups._streams()), C.byref(groups._ann()), _ptr(src_status), _ptr(group_status),
            _cuda_stream_ptr(dev))
        self.codec.ctx.check(rc, "m3tsz_element_set_forward_timer_annotated")
        return src_status[: self.n_elements], group_status[:G]

    @property
    def source_capacity(self) -> int:
        return 0 if self.source_bits is None else self.source_bits.shape[1] * 32

    def forward_write(self, target_ns, group_off: torch.Tensor, members: torch.Tensor, source_id: int,
                      keys: Optional[torch.Tensor] = None, metric_capacity: Optional[int] = None,
                      value_capacity: Optional[int] = None):
        """This set as a rollup's source set on shard `source_id` (m3tsz_element_set_forward_write, DESIGN.md
        §4.12): every element's open windows that ended by target_ns are forwarded as in forward(), but instead of a
        fold each group g (members[group_off[g] .. group_off[g + 1]), as forward() takes them) writes one record per
        distinct forwarded window start, in ascending order: key keys[g] (int64 [G]; None: g), time_ns the window's
        end, its members' values in listed order.  Groups are written in order while they fit metric_capacity /
        value_capacity (default: room for every record); every later group gets ERR_CAPACITY and holds its members
        back, so calling again with exactly the failed groups and more room gives the rest.  Returns (ForwardedBatch,
        source statuses int32 [N], group statuses int32 [G]: OK, ERR_CAPACITY or ERR_INVALID_ARG).  Timer sets write
        with forward_write_timer."""
        if self.timer:
            raise ValueError("Timer sets take no forward_write; they write with forward_write_timer")
        return self._forward_write(target_ns, group_off, members, source_id, keys, metric_capacity, value_capacity)

    def forward_write_timer(self, target_ns, group_off: torch.Tensor, members: torch.Tensor, source_id: int,
                            keys: Optional[torch.Tensor] = None, metric_capacity: Optional[int] = None,
                            value_capacity: Optional[int] = None):
        """forward_write for a Timer set (m3tsz_element_set_forward_write_timer, DESIGN.md §4.12), with the same
        arguments and return values: this set (one type, any but Last; its transformations the pre-rollup ones)
        flushes each due window's stream and forwards ValueOf(its type), as forward_timer does."""
        if not self.timer:
            raise ValueError("forward_write_timer takes a Timer set; other sets write with forward_write")
        return self._forward_write(target_ns, group_off, members, source_id, keys, metric_capacity, value_capacity)

    def _forward_write(self, target_ns, group_off, members, source_id, keys, metric_capacity, value_capacity):
        assert group_off.is_cuda and group_off.dtype == torch.int64 and group_off.is_contiguous()
        assert members.is_cuda and members.dtype == torch.int32 and members.is_contiguous()
        if keys is not None:
            assert keys.is_cuda and keys.dtype == torch.int64 and keys.is_contiguous()
            assert keys.numel() == group_off.numel() - 1
        G = group_off.numel() - 1
        assert G >= 0, "group_off has G + 1 entries"
        if metric_capacity is None:
            metric_capacity = members.numel() * self.open_windows
        if value_capacity is None:
            value_capacity = members.numel() * self.open_windows
        dev = self.codec.device
        metrics = torch.zeros((max(1, int(metric_capacity)), capi.FORWARDED_METRIC_BYTES), dtype=torch.uint8,
                              device=dev)
        values = torch.zeros(max(1, int(value_capacity)), dtype=torch.float64, device=dev)
        counts = torch.zeros(4, dtype=torch.int64, device=dev)
        src_status = torch.empty(max(1, self.n_elements), dtype=torch.int32, device=dev)
        group_status = torch.empty(max(1, G), dtype=torch.int32, device=dev)
        head = (self.codec.ctx.handle, C.byref(self.codec.opts), C.byref(self._desc()))
        tail = (int(target_ns), _ptr(group_off), _ptr(members), members.numel(), G, _ptr(keys), int(source_id),
                metrics.data_ptr(), int(metric_capacity), values.data_ptr(), int(value_capacity), counts.data_ptr(),
                _ptr(src_status), _ptr(group_status), _cuda_stream_ptr(dev))
        if self.timer:
            name = "m3tsz_element_set_forward_write_timer"
            rc = getattr(capi.lib(), name)(*head, C.byref(self._streams()), *tail)
        else:
            name = "m3tsz_element_set_forward_write"
            rc = getattr(capi.lib(), name)(*head, *tail)
        self.codec.ctx.check(rc, name)
        c = counts.tolist()
        batch = ForwardedBatch(metrics[: c[0]], values[: c[1]], c)
        return batch, src_status[: self.n_elements], group_status[:G]

    def add_forwarded(self, batches):
        """AddUnique of forwarded metrics (m3tsz_element_set_add_forwarded, DESIGN.md §4.12) into this set, which
        needs a source_capacity: one ForwardedBatch or a list, concatenated in the given order (value offsets
        rebased), each element taking its records in that order.  Returns (result int8 [M] in record order: OK,
        ERR_INVALID_ARG, ERR_AGGREGATION_CLOSED, ERR_CAPACITY -- the element stopped: grow() and send the refused
        records again --, or ERR_DUPLICATE_SOURCE -- the window has seen that source --; status int32 [N]: OK or
        ERR_CAPACITY).  Timer sets add with add_forwarded_timer."""
        if self.timer:
            raise ValueError("Timer sets take no add_forwarded; they add with add_forwarded_timer")
        return self._add_forwarded(batches)

    def add_forwarded_timer(self, batches):
        """add_forwarded for a Timer set (m3tsz_element_set_add_forwarded_timer, DESIGN.md §4.12), with the same
        arguments and return values: each accepted record's values are Timer.Adds into its window, in order.  A
        record that would take its window past sample_capacity samples also stops the element with ERR_CAPACITY:
        grow(open_windows=..., sample_capacity=...) and send the refused records (or the whole batch) again."""
        if not self.timer:
            raise ValueError("add_forwarded_timer takes a Timer set; other sets add with add_forwarded")
        return self._add_forwarded(batches)

    def _add_forwarded(self, batches):
        if self.source_bits is None:
            raise ValueError("add_forwarded needs an element set with a source_capacity")
        b = batches if isinstance(batches, ForwardedBatch) else ForwardedBatch.concat(batches)
        metrics, values = b.metrics.contiguous(), b.values.contiguous()
        M = metrics.shape[0]
        dev = self.codec.device
        result = torch.zeros(max(1, M), dtype=torch.int8, device=dev)
        status = torch.zeros(max(1, self.n_elements), dtype=torch.int32, device=dev)
        src = capi.ElementSources()
        src.d_bits = self.source_bits.data_ptr()
        src.capacity = self.source_capacity
        head = (self.codec.ctx.handle, C.byref(self.codec.opts), C.byref(self._desc()))
        tail = (C.byref(src), metrics.data_ptr() if M else None, M, values.data_ptr() if values.numel() else None,
                values.numel(), result.data_ptr(), status.data_ptr(), _cuda_stream_ptr(dev))
        if self.timer:
            name = "m3tsz_element_set_add_forwarded_timer"
            rc = getattr(capi.lib(), name)(*head, C.byref(self._streams()), *tail)
        else:
            name = "m3tsz_element_set_add_forwarded"
            rc = getattr(capi.lib(), name)(*head, *tail)
        self.codec.ctx.check(rc, name)
        return result[:M], status[: self.n_elements]

    def state(self):
        """Copies of the element-side state: {"win": {field: [R, N]}, "elem": uint8 [N, 160], "watermark": [N]},
        with annotations "ann_len" [R, N] and "ann_bytes" [R, N, capacity], for a Timer set "streams", and with a
        source capacity "source_bits" int32 [R, capacity / 32, N]."""
        st = {"win": {f: a.clone() for f, a in self.win.items()}, "elem": self.elem.clone(),
              "watermark": self.watermark.clone()}
        if self.ann_len is not None:
            st["ann_len"], st["ann_bytes"] = self.ann_len.clone(), self.ann_bytes.clone()
        if self.streams is not None:
            st["streams"] = {f: a.clone() for f, a in self.streams.items()}
        if self.source_bits is not None:
            st["source_bits"] = self.source_bits.clone()
        return st
