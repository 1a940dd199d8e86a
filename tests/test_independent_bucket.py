"""BufferBucket.write (storage/series/buffer.go:1261-1364) restated a second time, in pure Python over the independent
encoder of tests/indep_m3tsz.py, with no use of the oracle or of the device source: an encoder is the list of the
datapoints it took; LastEncoded().Value is restated from encoder.go's value grammar (the scaled int in int mode, the
float's bits in float mode, 0 without the int optimisation); the annotation check compares the bytes of the last
annotation WRITTEN; the time checks follow timestamp_encoder.go.  Both this restatement and the model the device is
checked against (bucket_model.Bucket, over the oracle encoder) must reproduce the reference's write tables
(tests/golden/m3tsz_buffer_goldens.json: wasWritten, errors, encoder counts, the read), and they must agree with
each other -- results, stream bytes and read -- on random write sequences in both modes."""
import json
import os

import pytest

import indep_m3tsz as I
import oracle_lib as O
from bucket_model import ERR_TOO_MANY_ENCODERS, SEC, Bucket, random_calls

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "m3tsz_buffer_goldens.json")))
START = 1599955200 * SEC  # a block start (a multiple of 2 h)
UNIT_NANOS = {1: 10 ** 9, 2: 10 ** 6, 3: 10 ** 3, 4: 1, 5: 60 * 10 ** 9, 6: 3600 * 10 ** 9, 7: 86400 * 10 ** 9,
              8: 365 * 86400 * 10 ** 9}
MAX_BUCKET = 12


class IndepBucket:
    def __init__(self, start, int_opt, K, default_unit=1):
        self.start, self.int_opt, self.K, self.du = start, int_opt, K, default_unit
        self.encs = [[]]  # the datapoints each in-order encoder took
        self.lw = [0]

    def last_value(self, dps):  # LastEncoded().Value, encoder.go:305-319 over the value grammar :112-231
        if not self.int_opt:
            return 0.0
        is_float, int_val, max_mult, fv = False, 0.0, 0, 0.0
        for k, (_, v, _, _) in enumerate(dps):
            val, mult, isf = I.convert_to_int_float(v, 0 if k == 0 else max_mult)
            if k == 0:
                if isf:
                    is_float, max_mult, fv = True, mult, v
                else:
                    int_val, max_mult = val, max(max_mult, mult)
                continue
            diff = 0.0 if isf else int_val - val
            if isf or diff >= 2.0 ** 63 or diff <= -(2.0 ** 63):
                if not is_float:
                    is_float, max_mult = True, mult
                fv = val
            else:
                if not (diff == 0 and not is_float and mult == max_mult):
                    max_mult = max(max_mult, mult)
                    is_float = False
                int_val = val
        return fv if is_float else int_val

    def last_ann(self, dps):  # the last annotation written: an empty one writes nothing
        return next((a for _, _, _, a in reversed(dps) if a), b"")

    def time_error(self, dps, t, u):  # timestamp_encoder.go:104-164 against the encoder's time state
        if not 1 <= u <= 8:
            return 6
        unit, prev_t, prev_d = I._initial_time_unit(self.start, self.du), self.start, 0
        for tt, _, uu, _ in dps:
            if uu != unit:
                unit, prev_d = uu, 0
            else:
                prev_d = tt - prev_t
            prev_t = tt
        if u != unit or u > 2:
            return 0
        d = (t - prev_t) - prev_d
        dod = abs(d) // UNIT_NANOS[u] * (1 if d >= 0 else -1)
        return 0 if -2 ** 31 <= dod < 2 ** 31 else 4

    def write(self, t, v, u=1, ann=b""):
        for i, dps in enumerate(self.encs):
            if t == self.lw[i]:
                if not dps:
                    return 3  # LastEncoded of an empty encoder
                if self.last_value(dps) == v and self.last_ann(dps) == ann:
                    return -1
                continue
            if t > self.lw[i]:
                err = self.time_error(dps, t, u)
                if not err:
                    dps.append((t, v, u, ann))
                    self.lw[i] = t
                return err
        if len(self.encs) >= self.K:
            return ERR_TOO_MANY_ENCODERS
        err = self.time_error([], t, u)
        if not err:
            self.encs.append([(t, v, u, ann)])
            self.lw.append(t)
        return err

    def streams(self):
        return [I.encode(self.start, dps, self.int_opt, self.du) for dps in self.encs]

    def read(self):  # last pushed wins on equal timestamps: a later encoder overrides an earlier one
        merged = {}
        for dps in self.encs:
            for t, v, _, _ in dps:
                merged[t] = v
        return sorted(merged.items())


def _golden_cases():
    return [pytest.param(c, id=c["name"]) for c in GOLD["cases"]]


@pytest.mark.parametrize("impl", ["model", "indep"])
@pytest.mark.parametrize("case", _golden_cases())
def test_both_statements_reproduce_the_reference_tables(case, impl):
    K = case["limit"] or MAX_BUCKET
    b = Bucket(START, True, K) if impl == "model" else IndepBucket(START, True, K)
    for w in case["writes"]:
        r = b.write(START + w["offset_ns"], w["value"], w["unit"], b"")
        assert (r == 0) == w["written"], (w, r)
        assert (r == ERR_TOO_MANY_ENCODERS) == (w["error"] == "too many encoders per block"), (w, r)
        assert r in (0, -1, ERR_TOO_MANY_ENCODERS), (w, r)
    if "encoders" in case:
        assert len(b.encs) == case["encoders"]
    if "last_encoded_offsets_ns" in case:
        last = ([e.last_encoded()[0] for e in b.encs] if impl == "model" else [d[-1][0] for d in b.encs])
        assert [t - START for t in last] == case["last_encoded_offsets_ns"]
    exp = [(START + o, v) for o, v in case["read"]]
    if impl == "model":
        ts, vals, st = b.read()
        assert st == 0 and list(zip(ts.tolist(), vals.tolist())) == exp
    else:
        assert b.read() == exp


@pytest.mark.parametrize("int_opt", [True, False])
def test_the_restatement_agrees_with_the_model(int_opt):
    n = 0
    for seed in range(300):
        K = (1, 2, 4, 12)[seed % 4]
        calls = random_calls(seed * 13 + 5 + int_opt, START, 12, 6, int_opt, units=seed % 3 == 1,
                             anns=seed % 2 == 0)
        m, ind = Bucket(START, int_opt, K), IndepBucket(START, int_opt, K)
        for c, call in enumerate(calls):
            for dp in call:
                assert ind.write(*dp) == m.write(*dp), (seed, c, dp)
                n += 1
        assert ind.streams() == m.streams(), seed
        ts, vals, st = m.read()
        if st == 0:
            assert ind.read() == list(zip(ts.tolist(), vals.tolist())), seed
    assert n > 5000


def test_a_first_write_far_before_the_block_start_reads_as_the_reference_reads_it():
    """a t == 0 write that opens an encoder of a bucket whose block starts ~1.6e9 s later: the encoder's stream holds
    the datapoint, and the reference's iterator reports EOF after it (the oracle's, which the device's decode and
    merge reproduce: test_gpu_bucket_write checks the read's status against it)"""
    for int_opt in (True, False):
        b = Bucket(START, int_opt, 2)
        assert b.write(START + 10 * SEC, 1.0) == 0
        assert b.write(0, 2.5) == 0
        dps, err = O.decode_all(b.streams()[1], int_opt)
        assert [(d[0], d[1]) for d in dps] == [(0, 2.5)] and err == 1  # M3TSZ_ERR_EOF
        assert IndepBucket(START, int_opt, 2).time_error([], 0, 1) == 0
