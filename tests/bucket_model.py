"""BufferBucket.write (src/dbnode/storage/series/buffer.go:1261-1364) over the ORACLE encoder: the model the bucket
writes on the device are checked against, and a generator of write traffic that exercises every branch of it."""
import random

import numpy as np

import oracle_lib as O
from m3_b200.encoding import xxh64

ERR_NO_DATAPOINTS, ERR_DOD_OVERFLOW, ERR_UNRECOGNIZED_UNIT = 3, 4, 6
ERR_TOO_MANY_ENCODERS, ERR_CAPACITY = 16, 100
SEC = 10 ** 9


class Bucket:
    """One bucket: in-order encoders with their lastWriteAt, at most K of them (EncodersPerBlockLimit)."""

    def __init__(self, start, int_opt, K, default_unit=O.UNIT_S):
        self.start, self.int_opt, self.K, self.default_unit = int(start), bool(int_opt), int(K), default_unit
        self.encs = [O.Encoder(self.start, self.int_opt, default_unit)]
        self.dps = [[]]
        self.lw = [0]  # resetTo: lastWriteAt of the first encoder is 0, not the block start (buffer.go:1246-1248)

    def write(self, t, v, u=O.UNIT_S, ann=b""):
        """0 written, -1 unchanged (no-op), else the error status"""
        t, v, ann = int(t), float(v), bytes(ann)
        for i, e in enumerate(self.encs):
            if t == self.lw[i]:
                _, lv, err = e.last_encoded()
                if err:
                    return err
                cs, err = e.last_annotation_checksum()
                if err:
                    return err
                if lv == v and cs == xxh64(ann):
                    return -1
                continue
            if t > self.lw[i]:
                return self._encode(i, t, v, u, ann)
        if len(self.encs) >= self.K:
            return ERR_TOO_MANY_ENCODERS
        # a new encoder at the block start (timestamp.Truncate(blockSize)); dropped again if its first write fails
        self.encs.append(O.Encoder(self.start, self.int_opt, self.default_unit))
        self.dps.append([])
        self.lw.append(None)
        err = self._encode(len(self.encs) - 1, t, v, u, ann)
        if err:
            self.encs.pop()
            self.dps.pop()
            self.lw.pop()
        return err

    def _encode(self, i, t, v, u, ann):
        err = self.encs[i].encode(t, v, u, ann)
        if err:
            # the codec drops a failing datapoint whole (DESIGN.md §6): the encoder is as after its last write
            e = O.Encoder(self.start, self.int_opt, self.default_unit)
            for dp in self.dps[i]:
                assert e.encode(*dp) == 0
            self.encs[i] = e
            return err
        self.dps[i].append((t, v, u, ann))
        self.lw[i] = t
        return 0

    def streams(self):
        """Stream() of every encoder, b"" for an empty one"""
        return [e.stream() or b"" for e in self.encs]

    def read(self):
        """what a reader of the bucket sees: the encoders' streams decoded (each with its iterator error) and merged,
        equal timestamps to the last pushed -> (ts, values, status)"""
        decs = [O.decode_all(s, self.int_opt, self.default_unit) if s else ([], 0) for s in self.streams()]
        seqs = [d[0] for d in decs]
        cap = max(1, max(len(q) for q in seqs))
        ts = np.zeros((len(seqs), cap), dtype=np.int64)
        vals = np.zeros((len(seqs), cap), dtype=np.float64)
        for k, q in enumerate(seqs):
            for j, dp in enumerate(q):
                ts[k, j], vals[k, j] = dp[0], dp[1]
        n = np.array([len(q) for q in seqs], dtype=np.uint32)
        seq_status = np.array([d[1] for d in decs], dtype=np.int32)
        to, vo, no, st = O.series_merge_batch(ts, vals, n, seq_status, [0, len(seqs)], [0, 1], [0, 1],
                                              out_cap=max(1, int(n.sum())))
        return to[0, : no[0]], vo[0, : no[0]], int(st[0])


def random_calls(seed, start, n_calls, max_pts, int_opt, units=False, anns=False, rare=True):
    """Write traffic for one bucket: each call a list of (t, v, unit, annotation).  Mostly in order; late
    datapoints, exact duplicates (no-ops), rewrites with a new value (upserts) and, with `rare`, t == 0, a
    second-unit delta-of-delta overflow and (with `units`) unit changes and unrecognised units."""
    r = random.Random(seed)
    t_next = start + 10 * SEC
    written = []  # (t, v, u, ann) sent so far
    vals_pool = [1.0, 1.5, 2.0, 7.25, -3.0, 1e9, 0.1, 123456.789]
    calls = []
    for _ in range(n_calls):
        call = []
        for _ in range(r.choice([0, 1, 1, 2, 3, max_pts])):
            kind = r.random()
            u = O.UNIT_S
            if units and r.random() < 0.15:
                u = r.choice([O.UNIT_MS, O.UNIT_US, O.UNIT_NS, O.UNIT_MS] + ([0, 9] if rare else []))
            ann = b""
            if anns and r.random() < 0.3:
                ann = r.choice([b"", b"a", b"proto-v1", bytes(range(40))])
            v = r.choice(vals_pool) if r.random() < 0.5 else round(r.gauss(0, 100), r.choice([0, 1, 2, 6]))
            if not int_opt and r.random() < 0.3:
                v = float(r.randint(-5, 5))
            if kind < 0.12 and written:  # exact duplicate of an earlier write
                t, v, u, ann = r.choice(written)
            elif kind < 0.25 and written:  # upsert: a written timestamp with another value or annotation
                t = r.choice(written)[0]
            elif kind < 0.40:  # late
                t = t_next - r.randint(1, 10) * 10 * SEC
            elif rare and kind < 0.42:
                t = 0
            elif rare and kind < 0.44:
                t = t_next + (1 << 32) * SEC  # a second-unit delta-of-delta overflows 32 bits
            else:
                t = t_next
                t_next += 10 * SEC
            call.append((t, v, u, ann))
            written.append((t, v, u, ann))
        calls.append(call)
    return calls
