#!/usr/bin/env python3
"""Transcribes the reference's own golden vectors for the M3TSZ path into
tests/golden/m3tsz_goldens.json, those of the aggregator's Gauge / Counter arithmetic into
tests/golden/m3tsz_agg_goldens.json, the buffer bucket's write tables into
tests/golden/m3tsz_buffer_goldens.json, the aggregator's transformations of a flushed window into
tests/golden/m3tsz_transform_goldens.json, and the flushes of an element with several aggregation types into
tests/golden/m3tsz_element_types_goldens.json, and the steps of a rollup (the values a source element forwards, what
the rollup element folds, when the forwarded list flushes) into tests/golden/m3tsz_rollup_goldens.json, and the
annotations a rollup element keeps from what it is forwarded into tests/golden/m3tsz_rollup_annotation_goldens.json.

Run in the build container only (it reads /root/reference, which does not exist
on the GPU box):   python scripts/make_goldens.py

Every vector records the reference test file:line it was taken from.  Byte
arrays and datapoint tables are transcribed by hand below (they are test DATA,
not implementation); the long base64 fixtures are pulled out of the Go test
files mechanically so they cannot be mistyped.
"""
import json
import os
import re

REF = "/root/reference/src/dbnode/encoding"
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden",
                   "m3tsz_goldens.json")
# the aggregator's Gauge with expensive aggregations and its Counter (tests/agg_oracle_lib.py)
OUT_AGG = os.path.join(os.path.dirname(OUT), "m3tsz_agg_goldens.json")
# BufferBucket.write (storage/series/buffer.go:1261-1364): the write tables of storage/series/buffer_test.go
OUT_BUFFER = os.path.join(os.path.dirname(OUT), "m3tsz_buffer_goldens.json")
# the transformations of a flushed window (metrics/transformation, GenericElem.processValue)
OUT_XF = os.path.join(os.path.dirname(OUT), "m3tsz_transform_goldens.json")
# an element's several aggregation types (GenericElem.processValue's loop over aggTypes)
OUT_ELEM = os.path.join(os.path.dirname(OUT), "m3tsz_element_types_goldens.json")
OUT_ANN = os.path.join(os.path.dirname(OUT), "m3tsz_tile_annotation_goldens.json")
# a rollup: the source element's forwarded values, the rollup element's folds and the forwarded list's flush times
OUT_ROLLUP = os.path.join(os.path.dirname(OUT), "m3tsz_rollup_goldens.json")
# the annotation a rollup element keeps: AddUnique passes metric.Annotation to Gauge / Counter Update
OUT_ROLLUP_ANN = os.path.join(os.path.dirname(OUT), "m3tsz_rollup_annotation_goldens.json")
OUT_ELEM_CONSUME = os.path.join(os.path.dirname(OUT), "m3tsz_element_consume_goldens.json")

SEC = 1_000_000_000
MS = 1_000_000
US = 1_000
S, MSU, USU, NSU = 1, 2, 3, 4  # xtime.Unit values (src/x/time/unit.go:30-42)

TEST_START = 1427162400 * SEC      # encoder_test.go:42
DP_START = 1427162462 * SEC        # encoder_test.go:216


def hx(bs):
    return bytes(bs).hex()


def go_strings(path, var):
    src = open(path).read()
    m = re.search(r"var %s = \[\]string\{(.*?)\n\}" % var, src, re.S)
    return re.findall(r'"([A-Za-z0-9+/=]+)"', m.group(1))


def main():
    g = {}

    # ---- bit I/O: ostream_test.go:44-71 ----
    g["ostream_write_bits"] = {
        "src": "encoding/ostream_test.go:44-71",
        "steps": [
            {"value": v, "nbits": n, "bytes": hx(b), "pos": p}
            for v, n, b, p in [
                (0x1, 1, [0x80], 1),
                (0x4, 3, [0xc0], 4),
                (0xa, 4, [0xca], 8),
                (0xfe, 8, [0xca, 0xfe], 8),
                (0xaafe, 7, [0xca, 0xfe, 0xfc], 7),
                (0x3, 2, [0xca, 0xfe, 0xfd, 0x80], 1),
                (0x1234567890abcdef, 64,
                 [0xca, 0xfe, 0xfd, 0x89, 0x1a, 0x2b, 0x3c, 0x48, 0x55, 0xe6, 0xf7, 0x80], 1),
                (0x1, 0,
                 [0xca, 0xfe, 0xfd, 0x89, 0x1a, 0x2b, 0x3c, 0x48, 0x55, 0xe6, 0xf7, 0x80], 1),
                (0x1, 65,
                 [0xca, 0xfe, 0xfd, 0x89, 0x1a, 0x2b, 0x3c, 0x48, 0x55, 0xe6, 0xf7, 0x80, 0x0, 0x0,
                  0x0, 0x0, 0x0, 0x0, 0x0, 0x80], 1),
            ]
        ],
    }
    # ---- istream_test.go:32-186 ----
    g["istream_read_bits"] = {
        "src": "encoding/istream_test.go:32-52",
        "bytes": hx([0xca, 0xfe, 0xfd, 0x89, 0x1a, 0x2b, 0x3c, 0x48, 0x55, 0xe6, 0xf7, 0x80, 0x0,
                     0x0, 0x0, 0x0, 0x0, 0x0, 0x0, 0x80]),
        "nbits": [1, 3, 4, 8, 7, 2, 64, 64],
        "expected": [0x1, 0x4, 0xa, 0xfe, 0x7e, 0x3, 0x1234567890abcdef, 0x1],
        "then_read_8_is_eof": True,
    }
    g["istream_peek_bits"] = {
        "src": "encoding/istream_test.go:76-100",
        "bytes": hx([0xa9, 0xfe, 0xfe, 0xdf, 0x9b, 0x57, 0x21, 0xf1]),
        "cases": [[0, 0], [1, 0x1], [8, 0xa9], [10, 0x2a7], [13, 0x153f], [16, 0xa9fe],
                  [32, 0xa9fefedf], [64, 0xa9fefedf9b5721f1]],
    }
    g["istream_peek_error"] = {"src": "encoding/istream_test.go:102-108", "bytes": "0102",
                               "peek": 20}
    g["istream_read_after_peek"] = {
        "src": "encoding/istream_test.go:110-133", "bytes": "abcd",
        "peek10": 0x2af, "peek20_eof": True, "reads": [[2, 0x2], [9, 0x15e]], "then_read_8_is_eof": True,
    }
    g["istream_peek_after_read"] = {
        "src": "encoding/istream_test.go:135-162",
        "bytes": hx([0x1, 0x2, 0x3, 0x4, 0x5, 0x6, 0x7, 0x8, 0x9, 0xA]),
        "ops": [["read", 16, 0x102], ["peek", 63, 0x30405060708090A >> 1],
                ["peek", 64, 0x30405060708090A], ["read", 1, 0], ["peek", 63, 0x30405060708090A],
                ["peek_eof", 64, 0]],
    }

    # ---- field level: encoder_test.go:54-123 ----
    g["write_dod_unit_unchanged"] = {
        "src": "encoding/m3tsz/encoder_test.go:54-81",
        "cases": [
            {"delta_ns": d, "unit": u, "bytes": hx(b), "pos": p}
            for d, u, b, p in [
                (0, S, [0x0], 1),
                (32 * SEC, S, [0x90, 0x0], 1),
                (-63 * SEC, S, [0xa0, 0x80], 1),
                (-128 * SEC, S, [0xd8, 0x0], 4),
                (255 * SEC, S, [0xcf, 0xf0], 4),
                (-2048 * SEC, S, [0xe8, 0x0], 8),
                (2047 * SEC, S, [0xe7, 0xff], 8),
                (4096 * SEC, S, [0xf0, 0x0, 0x1, 0x0, 0x0], 4),
                (-4096 * SEC, S, [0xff, 0xff, 0xff, 0x0, 0x0], 4),
                (4096 * SEC, NSU, [0xf0, 0x0, 0x0, 0x3b, 0x9a, 0xca, 0x0, 0x0, 0x0], 4),
                (-4096 * SEC, NSU, [0xff, 0xff, 0xff, 0xc4, 0x65, 0x36, 0x0, 0x0, 0x0], 4),
            ]
        ],
    }
    g["write_dod_unit_changed"] = {
        "src": "encoding/m3tsz/encoder_test.go:83-101",
        "cases": [
            {"delta_ns": d, "bytes": hx(b), "pos": p}
            for d, b, p in [
                (0, [0] * 8, 8),
                (32 * MS, [0x0, 0x0, 0x0, 0x0, 0x1, 0xe8, 0x48, 0x0], 8),
                (-63 * US, [0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0x9, 0xe8], 8),
            ]
        ],
    }
    g["write_xor"] = {
        "src": "encoding/m3tsz/encoder_test.go:103-123",
        "cases": [
            {"prev_xor": a, "cur_xor": b, "bytes": hx(c), "pos": p}
            for a, b, c, p in [
                (0x4028000000000000, 0, [0x0], 1),
                (0x4028000000000000, 0x0120000000000000, [0x80, 0x90], 6),
                (0x0120000000000000, 0x4028000000000000, [0xc1, 0x2e, 0x1, 0x40], 2),
            ]
        ],
    }
    # TestWriteAnnotation encoder_test.go:125-155 (NewTimestampEncoder(0, ns); writeAnnotation)
    g["write_annotation"] = {
        "src": "encoding/m3tsz/encoder_test.go:125-155",
        "cases": [
            {"annotation": "", "bytes": "", "pos": 0},
            {"annotation": "0102", "bytes": hx([0x80, 0x20, 0x40, 0x20, 0x40]), "pos": 3},
            {"annotation": "ff" * 8,
             "bytes": hx([0x80, 0x21, 0xdf, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xe0]), "pos": 3},
        ],
    }
    # TestWriteTimeUnit encoder_test.go:172-205 (TimeUnit forced to None before the call)
    g["write_time_unit"] = {
        "src": "encoding/m3tsz/encoder_test.go:172-205",
        "cases": [
            {"unit": 0, "result": False, "bytes": "", "pos": 0},
            {"unit": S, "result": True, "bytes": "804020", "pos": 3},
            {"unit": 255, "result": False, "bytes": "", "pos": 0},
        ],
    }
    # TestInitTimeUnit encoder_test.go:395-410
    g["init_time_unit"] = {
        "src": "encoding/m3tsz/encoder_test.go:395-410",
        "cases": [
            {"start_ns": 1, "unit": S, "expected": 0},
            {"start_ns": 1 * SEC, "unit": S, "expected": S},
            {"start_ns": 1 * SEC, "unit": 0, "expected": 0},
        ],
    }

    # ---- full streams (intOptimized=false): encoder_test.go:207-393 <-> iterator_test.go:181-385 ----
    def dps(rows):
        return [{"ts": DP_START + off, "value": v, "unit": u, "annotation": a} for off, v, u, a in rows]

    g["streams"] = [
        {
            "name": "no_annotation",
            "src": "encoding/m3tsz/encoder_test.go:207-245, iterator_test.go:181-222",
            "int_optimized": False, "encoder_start": TEST_START,
            "datapoints": dps([
                (0, 12, S, ""), (60 * SEC, 12, S, ""), (120 * SEC, 24, S, ""),
                (-76 * SEC, 24, S, ""), (-16 * SEC, 24, S, ""), (2092 * SEC, 15, S, ""),
                (4200 * SEC, 12, S, "")]),
            "decoded_annotations": ["", "", "", "", "", "", ""],
            "bytes": hx([
                0x13, 0xce, 0x4c, 0xa4, 0x30, 0xcb, 0x40, 0x0, 0x9f, 0x20, 0x14, 0x0, 0x0,
                0x0, 0x0, 0x0, 0x0, 0x5f, 0x8c, 0xb0, 0x3a, 0x0, 0xe1, 0x0, 0x78, 0x0, 0x0,
                0x40, 0x6, 0x58, 0x76, 0x8e, 0x0, 0x0]),
            "raw": hx([
                0x13, 0xce, 0x4c, 0xa4, 0x30, 0xcb, 0x40, 0x0, 0x9f, 0x20, 0x14, 0x0, 0x0,
                0x0, 0x0, 0x0, 0x0, 0x5f, 0x8c, 0xb0, 0x3a, 0x0, 0xe1, 0x0, 0x78, 0x0, 0x0,
                0x40, 0x6, 0x58, 0x76, 0x8c]),
            "raw_pos": 6,
        },
        {
            "name": "with_annotation",
            "src": "encoding/m3tsz/encoder_test.go:247-289, iterator_test.go:224-269",
            "int_optimized": False, "encoder_start": TEST_START,
            "datapoints": dps([
                (0, 12, S, "0a"), (60 * SEC, 12, S, "0a"), (120 * SEC, 24, S, ""),
                (-76 * SEC, 24, S, ""), (-16 * SEC, 24, S, "0102"), (2092 * SEC, 15, S, ""),
                (4200 * SEC, 12, S, "")]),
            "decoded_annotations": ["0a", "", "", "", "0102", "", ""],
            "bytes": hx([
                0x13, 0xce, 0x4c, 0xa4, 0x30, 0xcb, 0x40, 0x0, 0x80, 0x20, 0x1, 0x53, 0xe4,
                0x2, 0x80, 0x0, 0x0, 0x0, 0x0, 0x0, 0xb, 0xf1, 0x96, 0x7, 0x40, 0x10, 0x4,
                0x8, 0x4, 0xb, 0x84, 0x1, 0xe0, 0x0, 0x1, 0x0, 0x19, 0x61, 0xda, 0x38, 0x0]),
            "raw": hx([
                0x13, 0xce, 0x4c, 0xa4, 0x30, 0xcb, 0x40, 0x0, 0x80, 0x20, 0x1, 0x53, 0xe4,
                0x2, 0x80, 0x0, 0x0, 0x0, 0x0, 0x0, 0xb, 0xf1, 0x96, 0x7, 0x40, 0x10, 0x4,
                0x8, 0x4, 0xb, 0x84, 0x1, 0xe0, 0x0, 0x1, 0x0, 0x19, 0x61, 0xda, 0x30]),
            "raw_pos": 4,
        },
        {
            "name": "with_time_unit",
            "src": "encoding/m3tsz/encoder_test.go:291-327, iterator_test.go:271-313",
            "int_optimized": False, "encoder_start": TEST_START,
            "datapoints": dps([
                (0, 12, S, ""), (60 * SEC, 12, S, ""), (120 * SEC, 24, S, ""),
                (-76 * SEC, 24, S, ""), (-16 * SEC, 24, S, ""),
                (-15500000000, 15, NSU, ""), (-1400 * MS, 12, MSU, ""),
                (-10 * SEC, 12, S, ""), (10 * SEC, 12, S, "")]),
            "decoded_annotations": [""] * 9,
            "bytes": hx([
                0x13, 0xce, 0x4c, 0xa4, 0x30, 0xcb, 0x40, 0x0, 0x9f, 0x20, 0x14, 0x0, 0x0,
                0x0, 0x0, 0x0, 0x0, 0x5f, 0x8c, 0xb0, 0x3a, 0x0, 0xe1, 0x0, 0x40, 0x20,
                0x4f, 0xff, 0xff, 0xff, 0x22, 0x58, 0x60, 0xd0, 0xc, 0xb0, 0xee, 0x1, 0x1,
                0x0, 0x0, 0x0, 0x1, 0xa4, 0x36, 0x76, 0x80, 0x47, 0x0, 0x80, 0x7f, 0xff,
                0xff, 0xff, 0x7f, 0xd9, 0x9a, 0x80, 0x11, 0x44, 0x0]),
        },
        {
            "name": "with_annotation_and_time_unit",
            "src": "encoding/m3tsz/encoder_test.go:329-393, iterator_test.go:315-385",
            "int_optimized": False, "encoder_start": TEST_START,
            "datapoints": dps([
                (0, 12, S, "0a"), (60 * SEC, 12, S, ""), (120 * SEC, 24, S, ""),
                (-76 * SEC, 24, S, "0102"), (-16 * SEC, 24, MSU, ""),
                (-15500 * MS, 15, MSU, "030405"), (-14000 * MS, 12, S, "")]),
            "decoded_annotations": ["0a", "", "", "0102", "", "030405", ""],
            "bytes": hx([
                0x13, 0xce, 0x4c, 0xa4, 0x30, 0xcb, 0x40, 0x0, 0x80, 0x20, 0x1, 0x53, 0xe4,
                0x2, 0x80, 0x0, 0x0, 0x0, 0x0, 0x0, 0xb, 0xf1, 0x96, 0x6, 0x0, 0x81, 0x0,
                0x81, 0x68, 0x2, 0x1, 0x1, 0x0, 0x0, 0x0, 0x1d, 0xcd, 0x65, 0x0, 0x0, 0x20,
                0x8, 0x20, 0x18, 0x20, 0x2f, 0xf, 0xa6, 0x58, 0x77, 0x0, 0x80, 0x40, 0x0,
                0x0, 0x0, 0xe, 0xe6, 0xb2, 0x80, 0x23, 0x80, 0x0]),
        },
    ]

    # ---- iterator field level: iterator_test.go:44-179 ----
    g["read_next_timestamp"] = {
        "src": "encoding/m3tsz/iterator_test.go:44-88",
        "cases": [
            {"prev_delta_ns": pd, "unit": u, "bytes": hx(b), "expected_delta_ns": ed}
            for pd, u, b, ed in [
                (62 * SEC, S, [0x0], 62 * SEC),
                (65 * SEC, S, [0xa0, 0x0], 1 * SEC),
                (65 * SEC, S, [0x90, 0x0], 97 * SEC),
                (65 * SEC, S, [0xd0, 0x0], -191 * SEC),
                (65 * SEC, S, [0xcf, 0xf0], 320 * SEC),
                (65 * SEC, S, [0xe8, 0x0], -1983 * SEC),
                (65 * SEC, S, [0xe7, 0xff], 2112 * SEC),
                (65 * SEC, S, [0xf0, 0x0, 0x1, 0x0, 0x0], 4161 * SEC),
                (65 * SEC, S, [0xff, 0xff, 0xff, 0x0, 0x0], -4031 * SEC),
                (65 * SEC, NSU, [0xff, 0xff, 0xff, 0xc4, 0x65, 0x36, 0x0, 0x0, 0x0], -4031 * SEC),
                (65 * SEC, S, [0x80, 0x40, 0x40, 0x0, 0x0, 0x0, 0x0, 0x0, 0x0, 0x7d, 0x0],
                 65000001 * US),
            ]
        ],
        "error_stream": "01",  # readFirstTimestamp, then readNextTimestamp x2 all error
    }
    g["read_next_value"] = {
        "src": "encoding/m3tsz/iterator_test.go:90-115",
        "cases": [
            {"prev_value": pv, "prev_xor": px, "bytes": hx(b), "expected_xor": ex, "expected_value": ev}
            for pv, px, b, ex, ev in [
                (0x1234, 0x4028000000000000, [0x0], 0x0, 0x1234),
                (0xaaaaaa, 0x4028000000000000, [0x80, 0x90], 0x0120000000000000, 0x0120000000aaaaaa),
                (0xdeadbeef, 0x0120000000000000, [0xc1, 0x2e, 0x1, 0x40], 0x4028000000000000,
                 0x40280000deadbeef),
            ]
        ],
        "error_stream": "f0",
    }
    g["read_annotation"] = {
        "src": "encoding/m3tsz/iterator_test.go:117-149",
        "cases": [
            {"bytes": "00ff", "annotation": "ff"},
            {"bytes": "020203", "annotation": "0203"},
            {"bytes": "0e" + "ff" * 8, "annotation": "ff" * 8},
            {"bytes": "10" + "ff" * 9, "annotation": "ff" * 9},
        ],
    }
    g["read_time_unit"] = {
        "src": "encoding/m3tsz/iterator_test.go:151-179",
        "cases": [
            {"unit": MSU, "bytes": "01", "expected_unit": S, "expected_changed": True},
            {"unit": S, "bytes": "00", "expected_unit": 0, "expected_changed": False},
        ],
    }
    g["iterator_error_streams"] = {
        "src": "encoding/m3tsz/iterator_test.go:265-269,387-394",
        "cases": [
            {"bytes": hx([0x0, 0x0, 0x0, 0x0, 0x55, 0x10, 0xc5, 0x20, 0x80, 0x20, 0x1, 0x50, 0x8]),
             "int_optimized": False, "note": "annotation truncated: Next false, not done, has error"},
            {"bytes": hx([0x0, 0x0, 0x0, 0x0, 0x55, 0x10, 0xc5, 0x20, 0x80, 0x41, 0x20, 0x0, 0x0]),
             "int_optimized": False, "note": "unexpected time unit: Next false, Err != nil"},
        ],
    }

    # ---- DoD overflow error cases: encoder_test.go:581-730 (values checked below) ----
    g["fixtures_b64"] = {
        "src": "encoding/m3tsz/encoder_benchmark_test.go:36-47 (intOptimized=true)",
        "streams": go_strings(os.path.join(REF, "m3tsz", "encoder_benchmark_test.go"),
                              "sampleSeriesBase64"),
        "expected_points": [720, 720, 719, 720, 719, 720, 719, 720, 720, 720],
    }
    src = open(os.path.join(REF, "m3tsz", "iterator_test.go")).read()
    m = re.search(r'b64 := "([A-Za-z0-9+/=]+)"', src)
    g["regression_b64"] = {
        "src": "encoding/m3tsz/iterator_test.go:396-412 (intOptimized=true; first value -2^63, sig=64)",
        "stream": m.group(1),
    }

    # ---- roundtrip_test.go:270-285 overflow datapoints (property: round-trips in both modes) ----
    large = float(2 ** 63)  # float64(math.MaxInt64 - 1)
    g["overflow_values"] = {
        "src": "encoding/m3tsz/roundtrip_test.go:270-285",
        "values": [large, 10, -large, 10, -large, large, -12, large, 14.5, large, -large,
                   12.34858499392, large],
        "start_ns": DP_START, "step_ns": SEC,
    }
    g["precision_value"] = {"src": "encoding/m3tsz/roundtrip_test.go:94-106", "value": 187.80131100000006}

    # ---- aggregation.Gauge tables: src/aggregator/aggregation/gauge_test.go ----
    # time.Now() in the Go tests is strictly increasing between calls: times are given as offsets.
    g["gauge"] = {
        "src": "aggregator/aggregation/gauge_test.go:35-57 (default), :59-105 (UpdatePrevious prefix), "
               ":117-170 (custom types), :173-195 (last, out of order)",
        "cases": [
            {"name": "1..100", "src_line": "gauge_test.go:35-48,121-147",
             "times": list(range(100)), "values": [float(i) for i in range(1, 101)],
             "last": 100.0, "count": 100, "mean": 50.5, "max": 100.0, "min": 1.0, "sum": 5050.0},
            {"name": "empty", "src_line": "gauge_test.go:49-57,149-170",
             "times": [], "values": [],
             "last": 0.0, "count": 0, "mean": 0.0, "max": "NaN", "min": "NaN", "sum": 0.0},
            {"name": "1,2,3", "src_line": "gauge_test.go:64-75",
             "times": [0, 1, 2], "values": [1.0, 2.0, 3.0],
             "last": 3.0, "count": 3, "mean": 2.0, "max": 3.0, "min": 1.0, "sum": 6.0},
            {"name": "last out of order", "src_line": "gauge_test.go:173-195",
             # timeMid = now+60s; pre = mid-1s; prepre = mid-1s; after = mid+1s
             "times": [60, 59, 61, 59], "values": [42.0, 41.0, 43.0, 40.0],
             "last": 43.0, "out_of_order": 2},  # the test asserts only Last() and the counter
        ],
    }

    # ---- Prometheus conversion epilogue: src/query/storage/prom_converter_test.go ----
    HOUR, MIN = 3600 * SEC, 60 * SEC
    T0 = 1600000000 // 3600 * 3600 * SEC  # xtime.Now().Truncate(time.Hour): any hour-aligned instant

    def dps(*pairs):
        return [[T0 + off, v] for off, v in pairs]

    def samples(*pairs):
        return [[(T0 + off) // MS, v] for off, v in pairs]

    g["prom_counter_normalization"] = {
        "src": "query/storage/prom_converter_test.go:319-440 (resolutionThreshold = 5m default, options.go:30; "
               "handleResets = isCounter && maxResolution >= threshold, prom_converter.go:74-82)",
        "resolution_threshold_ns": 5 * MIN,
        "cases": [
            {"name": "low resolution gauge", "is_counter": False, "max_resolution_ns": HOUR,
             "given": dps((0, 1), (HOUR, 2)), "want": samples((0, 1), (HOUR, 2))},
            {"name": "high resolution gauge", "is_counter": False, "max_resolution_ns": MIN,
             "given": dps((0, 1), (MIN, 2)), "want": samples((0, 1), (MIN, 2))},
            {"name": "low resolution counter, no datapoints", "is_counter": True, "max_resolution_ns": HOUR,
             "given": [], "want": []},
            {"name": "low resolution counter, one datapoint", "is_counter": True, "max_resolution_ns": HOUR,
             "given": dps((0, 1)), "want": samples((0, 1))},
            {"name": "high resolution counter with no resets", "is_counter": True, "max_resolution_ns": MIN,
             "given": dps((0, 1), (MIN, 2), (2 * MIN, 2), (3 * MIN, 3)),
             "want": samples((0, 1), (MIN, 2), (2 * MIN, 2), (3 * MIN, 3))},
            {"name": "high resolution counter with resets", "is_counter": True, "max_resolution_ns": MIN,
             "given": dps((0, 10), (MIN, 3), (2 * MIN, 5), (3 * MIN, 8)),
             "want": samples((0, 10), (MIN, 3), (2 * MIN, 5), (3 * MIN, 8))},
            {"name": "low resolution counter with no resets", "is_counter": True, "max_resolution_ns": HOUR,
             "given": dps((0, 1), (MIN, 2), (HOUR, 2), (HOUR + MIN, 3)),
             "want": samples((MIN, 2), (HOUR + MIN, 3))},
            {"name": "low resolution counter with resets", "is_counter": True, "max_resolution_ns": HOUR,
             "given": dps((0, 10), (MIN, 3), (HOUR, 5), (HOUR + MIN, 8)),
             "want": samples((MIN, 13), (HOUR + MIN, 18))},
        ],
    }
    a, b = 187.80131100000006, 187.801311
    g["prom_value_decrease_tolerance"] = {
        "src": "query/storage/prom_converter_test.go:444-500 (datapoint i at now + i minutes)",
        "now_ns": T0, "step_ns": MIN,
        "cases": [
            {"name": "no tolerance", "given": [a, b, a, b, 200, 199.99], "tolerance": 0, "until_ns": 0,
             "want": [a, b, a, b, 200, 199.99]},
            {"name": "low tolerance", "given": [a, b, a, b, 200, 199.99], "tolerance": 0.00000001,
             "until_ns": T0 + HOUR, "want": [a, a, a, a, 200, 199.99]},
            {"name": "high tolerance", "given": [a, b, a, b, 200, 199.99], "tolerance": 0.0001,
             "until_ns": T0 + HOUR, "want": [a, a, a, a, 200, 200]},
            {"name": "tolerance expired", "given": [200, 199.99, 200, 199.99, 200, 199.99], "tolerance": 0.0001,
             "until_ns": T0, "want": [200, 199.99, 200, 199.99, 200, 199.99]},
            {"name": "tolerance expires in the middle", "given": [200, 199.99, 200, 199.99, 200, 199.99],
             "tolerance": 0.0001, "until_ns": T0 + 3 * MIN, "want": [200, 200, 200, 199.99, 200, 199.99]},
        ],
    }

    # ---- the expensive aggregations and the Counter: src/aggregator/aggregation/{gauge,counter,common}_test.go ----
    # (a file of their own, tests/golden/m3tsz_agg_goldens.json, bound by tests/agg_oracle_lib.py).  value_of maps
    # aggregation.Type ids to the expected ValueOf; "stdev" entries hold [expected, delta] (require.InDelta)
    hundred = [float(i) for i in range(1, 101)]
    agg = {
        "src": "aggregator/aggregation/gauge_test.go:59-75,108-170, counter_test.go:33-43,54-87, "
               "common_test.go:31-33",
        "gauge": [
            {"name": "1..100 expensive", "src_line": "gauge_test.go:108-147", "times": list(range(100)),
             "values": hundred,
             "value_of": {"1": 100.0, "2": 1.0, "3": 100.0, "4": 50.5, "6": 100.0, "7": 5050.0, "8": 338350.0},
             "stdev": [29.01149, 0.001]},
            {"name": "empty expensive", "src_line": "gauge_test.go:149-170", "times": [], "values": [],
             "value_of": {"1": 0.0, "2": "NaN", "3": "NaN", "4": 0.0, "6": 0.0, "7": 0.0, "8": 0.0},
             "stdev": [0.0, 0.0]},
            {"name": "1,2,3 expensive", "src_line": "gauge_test.go:59-75", "times": [0, 1, 2],
             "values": [1.0, 2.0, 3.0],
             "value_of": {"1": 3.0, "2": 1.0, "3": 3.0, "4": 2.0, "6": 3.0, "8": 14.0}},
        ],
        "counter": [
            {"name": "1..100 default", "src_line": "counter_test.go:33-43", "values": hundred,
             "sum": 5050, "value_of": {"7": 5050.0, "6": 100.0, "4": 50.5}},
            {"name": "1..100 expensive", "src_line": "counter_test.go:54-87", "values": hundred, "sum": 5050,
             "value_of": {"2": 1.0, "3": 100.0, "4": 50.5, "6": 100.0, "7": 5050.0, "8": 338350.0},
             "stdev": [29.01149, 0.001], "invalid_value_of": {"1": 0.0}},
        ],
        "stdev": [{"src_line": "common_test.go:31-33", "count": 100, "sum_sq": 338350.0, "sum": 5050.0,
                   "want": 29.01149, "delta": 0.001}],
    }

    # ---- buffer buckets: storage/series/buffer_test.go (the bucket writes, m3tsz_encoder_set_write) ----
    # Every case is one bucket at a block start; each write is (offset from the block start in ns, value, unit) with
    # the reference's wasWritten and error.  "read" is what the reference asserts a reader of the bucket sees,
    # (offset, value) in time order; "encoders" the number of in-order encoders it asserts, where it does.
    # TestEncoderLimit asserts no read: its "read" is its successful writes in time order (the offsets are
    # distinct).  Its limit 0 means no limit.
    def limit_case(desc, limit, writes):
        ws = [{"offset_ns": off * MS, "value": float(i), "unit": MSU, "written": not tm,
               "error": "too many encoders per block" if tm else None} for i, (off, tm) in enumerate(writes)]
        read = sorted((w["offset_ns"], w["value"]) for w in ws if w["written"])
        return {"name": "TestEncoderLimit/" + desc, "src_line": "buffer_test.go:2022-2255", "limit": limit,
                "writes": ws, "read": [list(r) for r in read]}

    def sec_writes(rows):
        return [{"offset_ns": off * SEC, "value": float(v), "unit": S, "written": w, "error": None}
                for off, v, w in rows]

    buffer = {
        "src": "dbnode/storage/series/buffer_test.go",
        "cases": [
            {"name": "TestBufferWriteOutOfOrder", "src_line": "buffer_test.go:337-381", "limit": 0,
             "writes": sec_writes([(0, 1, True), (10, 2, True), (5, 3, True)]), "encoders": 2,
             "last_encoded_offsets_ns": [10 * SEC, 5 * SEC],
             "read": [[0, 1.0], [5 * SEC, 3.0], [10 * SEC, 2.0]]},
            {"name": "TestBufferBucketWriteDuplicateUpserts", "src_line": "buffer_test.go:574-638", "limit": 0,
             "writes": sec_writes([(0, 1, True), (10, 2, True), (50, 3, True), (50, 4, True),
                                   (10, 5, True), (40, 6, True), (60, 7, True),
                                   (40, 8, True), (70, 9, True),
                                   (10, 10, True), (80, 11, True)]),
             "read": [[0, 1.0], [10 * SEC, 10.0], [40 * SEC, 8.0], [50 * SEC, 4.0], [60 * SEC, 7.0],
                      [70 * SEC, 9.0], [80 * SEC, 11.0]]},
            {"name": "TestBufferBucketDuplicatePointsNotWrittenButUpserted", "src_line": "buffer_test.go:640-709",
             "limit": 0,
             "writes": sec_writes([(0, 1, True), (0, 1, False), (0, 1, False), (0, 1, False), (10, 2, True),
                                   (0, 1, True), (10, 2, False), (10, 5, True),
                                   (0, 1, True), (20, 8, True),
                                   (0, 10, True), (20, 10, True)]),
             "read": [[0, 10.0], [10 * SEC, 5.0], [20 * SEC, 10.0]]},
            limit_case("one encoder, no limit", 0, [(1, False), (2, False), (3, False), (4, False)]),
            limit_case("many encoders, no limit", 0, [(o, False) for o in range(9, 1, -1)]),
            limit_case("within limit", 3, [(3, False), (2, False), (1, False)]),
            limit_case("within limit, many writes", 2,
                       [(10, False), (11, False), (12, False), (1, False), (2, False), (13, False), (3, False)]),
            limit_case("too many encoders", 3, [(5, False), (4, False), (3, False), (2, True)]),
            limit_case("too many encoders, more writes", 2,
                       [(10, False), (2, False), (3, False), (11, False), (1, True), (4, False)]),
        ],
    }

    # ---- transformations: metrics/transformation/{binary,unary,unary_multi}_test.go and the flush sequences of
    # aggregator/aggregator/elem_test.go up to their first resend / update.  A case is one element: `ops`
    # (transformation.Type ids: 1 Absolute, 2 PerSecond, 3 Increase, 4 Add, 5 Reset), the resolution `step_ns`,
    # DiscardNaNAggregatedValues, an optional starting state (the binary op's previous window) and its flushes
    # ("calls"), each the non-empty windows (end, value) it consumes and the datapoints it writes, in order.
    # Values are numbers, or "NaN:<64-bit hex>" for an exact NaN ("NaN:7ff8000000000001" is emptyDatapoint).
    EMPTY = "NaN:7ff8000000000001"
    NOW = 1_600_000_000_123_456_789  # the reset tests' time.Now()

    def per_second(i, prev, curr, want):
        return {"name": "TestPerSecond/%d" % i, "src_line": "metrics/transformation/binary_test.go:30-78",
                "ops": [2], "step_ns": 10 * SEC, "discard_nan": False,
                "state": {"has_prev": 1, "prev_t": prev[0] * SEC, "prev_v": prev[1]},
                "calls": [{"windows": [[curr[0] * SEC, curr[1]]], "want": [[curr[0] * SEC, want]]}]}

    def absolute(i, t, v, want):
        return {"name": "TestAbsolute/%d" % i, "src_line": "metrics/transformation/unary_test.go:29-51",
                "ops": [1], "step_ns": 10 * SEC, "discard_nan": False, "state": None,
                "calls": [{"windows": [[t, v]], "want": [[t, want]]}]}

    ps = [((1230, 25.0), (1240, 30.0), 0.5), ((1230, 25.0), (1240, 30.0), 0.5), ((1230, 25.0), (1230, 20.0), EMPTY),
          ((1230, "NaN:7ff8000000000001"), (1240, 20.0), EMPTY), ((1230, 20.0), (1240, "NaN:7ff8000000000001"), EMPTY),
          ((1230, 30.0), (1240, 20.0), EMPTY)]
    xf = {
        "src": "metrics/transformation/{binary,unary,unary_multi}_test.go, aggregator/aggregator/elem_test.go",
        "cases": [per_second(i, *c) for i, c in enumerate(ps)] +
                 [absolute(i, *c) for i, c in enumerate([(0, 1.2, 1.2), (0, -1.2, 1.2), (1234, -1.2, 1.2)])] + [
            {"name": "TestReset", "src_line": "metrics/transformation/unary_multi_test.go:29-38", "ops": [5],
             "step_ns": 30 * SEC, "discard_nan": False, "state": None,
             "calls": [{"windows": [[NOW, 1000.0]], "want": [[NOW, 1000.0], [NOW + 15 * SEC, 0.0]]}]},
            {"name": "TestResetAtLeast1Nanosecond", "src_line": "metrics/transformation/unary_multi_test.go:40-49",
             "ops": [5], "step_ns": 1, "discard_nan": False, "state": None,
             "calls": [{"windows": [[NOW, 1000.0]], "want": [[NOW, 1000.0], [NOW + 1, 0.0]]}]},
            # Sum of one value per window, resolution 10 s (testStoragePolicy), Consume(0) / (220 s) / (240 s)
            {"name": "TestGaugeElemReset", "src_line": "aggregator/aggregator/elem_test.go:2238-2305", "ops": [5],
             "step_ns": 10 * SEC, "discard_nan": False, "state": None,
             "calls": [{"windows": [], "want": []},
                       {"windows": [[220 * SEC, 123.0]], "want": [[220 * SEC, 123.0], [225 * SEC, 0.0]]},
                       {"windows": [[230 * SEC, 456.0], [240 * SEC, 589.0]],
                        "want": [[230 * SEC, 456.0], [235 * SEC, 0.0], [240 * SEC, 589.0], [245 * SEC, 0.0]]}]},
            # the default Gauge type (Last) of testGauge (123.456) in two windows, Increase
            {"name": "TestGaugeElemConsumeResendBuffer", "src_line": "aggregator/aggregator/elem_test.go:1709-1765",
             "ops": [3], "step_ns": 10 * SEC, "discard_nan": True, "state": None,
             "calls": [{"windows": [[220 * SEC, 123.456]], "want": [[220 * SEC, 123.456]]},
                       {"windows": [[230 * SEC, 123.456]], "want": [[230 * SEC, 0.0]]}]},
            # Last, Increase (then a rollup: the forwarded values are the transformation's)
            {"name": "TestGaugeElemResendBufferForwarding",
             "src_line": "aggregator/aggregator/elem_test.go:2095-2199", "ops": [3], "step_ns": 10 * SEC,
             "discard_nan": True, "state": None,
             "calls": [{"windows": [], "want": []},
                       {"windows": [[220 * SEC, 123.0]], "want": [[220 * SEC, 123.0]]},
                       {"windows": [[230 * SEC, 456.0], [240 * SEC, 589.0]],
                        "want": [[230 * SEC, 333.0], [240 * SEC, 133.0]]}],
             "consumed": [123.0, 456.0, 589.0]},
        ],
    }

    # ---- an element's several aggregation types: the flushes of elem_test.go's custom-aggregation tests with the
    # default pipeline (testAggregationTypes = {Mean, Sum}, elem_test.go:58; one value per window, resolution 10 s,
    # windows starting at 210 s and 220 s, Consume(0) / (220 s) / (230 s)).  A case is one element: its metric type
    # (1 Counter, 3 Gauge), its aggregation.Type ids in order, `ops` as above, and its flushes, each the non-empty
    # windows (end, [value of every type]) and what every type writes (want[j]: type j's datapoints).
    def types_case(name, src_line, metric_type, val):
        return {"name": name, "src_line": src_line, "metric_type": metric_type, "agg_types": [4, 7], "ops": [],
                "step_ns": 10 * SEC, "discard_nan": True,
                "calls": [{"windows": [], "want": [[], []]},
                          {"windows": [[220 * SEC, [val, val]]], "want": [[[220 * SEC, val]], [[220 * SEC, val]]]},
                          {"windows": [[230 * SEC, [val, val]]], "want": [[[230 * SEC, val]], [[230 * SEC, val]]]}]}

    elem = {
        "src": "aggregator/aggregator/elem_test.go",
        "cases": [
            # testCounter.CounterVal = 1234 (elem_test.go:79-83): Mean and Sum of one value
            types_case("TestCounterElemConsumeCustomAggregationDefaultPipeline", "aggregator/aggregator/elem_test.go:532",
                       1, 1234.0),
            # testGauge.GaugeVal = 123.456 (elem_test.go:89-93)
            types_case("TestGaugeElemConsumeCustomAggregationDefaultPipeline", "aggregator/aggregator/elem_test.go:1826",
                       3, 123.456),
        ],
    }

    # ---- the annotation a window is flushed with (aggregation/common.go:47-61 MaybeReplaceAnnotation, called by
    # Gauge.Update / Counter.Update; consumeState.annotation, aggregator/generic_elem.go:567): the datapoints as they
    # reach the element, in order, and each window's annotation ("" for none).  time.Now() in the aggregation tests
    # is a timestamp inside one window here.
    def ann_case(name, source, metric_type, start_ns, step_ns, n_windows, dps, want):
        return {"name": name, "source": source, "metric_type": metric_type, "start_ns": start_ns,
                "step_ns": step_ns, "n_windows": n_windows,
                "datapoints": [[t, v, a.hex()] for t, v, a in dps], "want_windows": [a.hex() for a in want]}

    # elem_test.go:56 (10 s resolution), :120-125 (testTimestamps, testAlignedStarts), :79-83 (CounterVal 1234)
    ts3 = [216 * SEC, 217 * SEC, 221 * SEC]
    ann = {
        "description": "The annotation each aggregation window keeps: the last non-empty one of its datapoints "
                       "(aggregation/common.go:47-61, gauge.go:54-57, counter.go:77), transcribed from the "
                       "reference's annotation tests by scripts/make_goldens.py.  datapoints: [t_ns, value, "
                       "annotation hex] in stream order; want_windows: each window's annotation hex, \"\" for none.",
        "cases": [
            ann_case("TestGaugeReturnsLastNonEmptyAnnotation", "aggregator/aggregation/gauge_test.go:99-106", 3,
                     210 * SEC, 10 * SEC, 1,
                     [(216 * SEC, 1.1, b"first"), (217 * SEC, 2.1, b"second"), (218 * SEC, 3.1, b"")],
                     [b"second"]),
            ann_case("TestCounterReturnsLastNonEmptyAnnotation", "aggregator/aggregation/counter_test.go:45-52", 1,
                     210 * SEC, 10 * SEC, 1,
                     [(216 * SEC, 1.0, b"first"), (217 * SEC, 2.0, b"second"), (218 * SEC, 3.0, b"")],
                     [b"second"]),
            ann_case("TestCounterElemAddUnion", "aggregator/aggregator/elem_test.go:215-252", 1, 210 * SEC,
                     10 * SEC, 2,
                     [(ts3[0], 1234.0, b"\x01"), (ts3[1], 1234.0, b""), (ts3[2], 1234.0, b"\x02")],
                     [b"\x01", b"\x02"]),
            ann_case("TestCounterElemAddUnionWithCustomAggregation", "aggregator/aggregator/elem_test.go:254-300", 1,
                     210 * SEC, 10 * SEC, 2,
                     [(ts3[0], 1234.0, b"\x01"), (ts3[1], 1234.0, b""), (ts3[2], 1234.0, b"")],
                     [b"\x01", b""]),
        ],
    }

    # ---- a rollup.  testPipeline (elem_test.go:94-117) is Absolute, PerSecond, then a rollup: the source element
    # forwards only each window's value through the two transformations (generic_elem.go:912-937), at the window's
    # end (10 s resolution, windows starting at 210, 220, 230 s with one value each, elem_test.go:597-607 and
    # :1891-1901, DiscardNaNAggregatedValues off).  "windows": (end, ValueOf(type)) of the non-empty windows; "want":
    # the forwarded (timestamp, value), "NaN" for a NaN; "consumed": the binary op's input after the last window.
    def fwd_case(name, src_line, metric_type, src_type):
        return {"name": name, "src_line": src_line, "metric_type": metric_type, "src_type": src_type,
                "ops": [1, 2], "step_ns": 10 * SEC, "discard_nan": False,
                "windows": [[220 * SEC, -123.0], [230 * SEC, -456.0], [240 * SEC, -589.0]],
                "want": [[220 * SEC, "NaN"], [230 * SEC, 33.3], [240 * SEC, 13.3]], "consumed": 589.0}

    # The rollup element's AddUnique (generic_elem.go:246-281): the values each window received, in order, and what
    # the test asserts after them ("eps": the test's relative tolerance; sum_sq only where the element's types are
    # expensive, testAggregationTypesExpensive = {SumSq}, elem_test.go:59).  The resends (Version > 0) and the
    # duplicate-source errors of these tests are not part of the fold.
    def fold(values, **want):
        return {"values": values, "want": want}

    rollup = {
        "description": "The steps of a rollup, transcribed from the reference's aggregator tests by "
                       "scripts/make_goldens.py: the values a source element forwards (forward), the rollup "
                       "element's fold of the values a window receives (folds), and the forwarded list's flush "
                       "timestamps (flush).",
        "forward": [
            fwd_case("TestCounterElemConsumeCustomAggregationCustomPipeline",
                     "aggregator/aggregator/elem_test.go:596-724", 1, 7),
            fwd_case("TestGaugeElemConsumeCustomAggregationCustomPipeline",
                     "aggregator/aggregator/elem_test.go:1890-2012", 3, 1),
        ],
        "folds": [
            {"name": "TestCounterElemAddUnique", "src_line": "aggregator/aggregator/elem_test.go:308-390",
             "metric_type": 1,
             "steps": [fold([345.0], sum=345, count=1), fold([345.0, 500.0], sum=845, count=2),
                       fold([278.0], sum=278, count=1)]},
            {"name": "TestCounterElemAddUniqueWithCustomAggregation",
             "src_line": "aggregator/aggregator/elem_test.go:392-466", "metric_type": 1,
             "steps": [fold([12.0], sum=12, max=12, sum_sq=144), fold([12.0, 14.0], sum=26, max=14),
                       fold([20.0], sum=20, max=20, sum_sq=400, count=1)]},
            {"name": "TestGaugeElemAddUnique", "src_line": "aggregator/aggregator/elem_test.go:1473-1570",
             "metric_type": 3,
             "steps": [fold([12.3, 34.5], sum=46.8, count=2), fold([12.3, 34.5, 50.0], sum=96.8, count=3),
                       fold([27.8], sum=27.8, count=1)]},
            {"name": "TestGaugeElemAddUniqueWithCustomAggregation",
             "src_line": "aggregator/aggregator/elem_test.go:1572-1643", "metric_type": 3,
             "steps": [fold([1.2], sum=1.2, max=1.2, sum_sq=1.44),
                       fold([1.2, 1.4], sum=2.6, max=1.4, eps=1e-10),
                       fold([2.0], sum=2.0, max=2.0, sum_sq=4.0)]},
        ],
        # list_test.go:815-1022: a counter (123) and a gauge (1.762) element with pipeline Rollup [Max] each take
        # AddUnique at the aligned 210 s and 220 s (10 s resolution); the list flushes each window's value with the
        # window's START as its timestamp (forwardedMetricTimestampNanos, list.go:621-623)
        "flush": {"name": "TestForwardedMetricListFlushConsumingAndCollectingForwardedMetrics",
                  "src_line": "aggregator/aggregator/list_test.go:815-1022", "resolution_ns": 10 * SEC,
                  "agg_type": 3,
                  "elements": [{"metric_type": 1, "value": 123.0}, {"metric_type": 3, "value": 1.762}],
                  "added_at_ns": [210 * SEC, 220 * SEC], "want_flush_ns": [210 * SEC, 220 * SEC]},
    }

    # ---- annotations through a rollup.  The rollup element's AddUnique (generic_elem.go:246-281) passes
    # metric.Annotation to Add, and Gauge / Counter Update keep the last non-empty one (MaybeReplaceAnnotation,
    # aggregation/common.go:49-61).  Each step is one AddUnique: the forwarding source, the time it is added at,
    # the forwarded values, their annotation (hex, null for none), and what the test asserts after it about the
    # windows (index into window_starts_ns; "annotation" null is the test's require.Nil).  testAnnot is
    # []byte("testAnnotation") (elem_test.go:55), testTimestamps 216 / 217 / 221 s (:120-122), testAlignedStarts
    # 210 / 220 s (:123-125), 10 s resolution.  The resend with versions (:1547-1559) is left out.
    test_annot = hx(b"testAnnotation")

    def add_unique(source, at_s, values, annotation, *want):
        return {"source": source, "at_ns": at_s * SEC, "values": values, "annotation": annotation,
                "want": list(want)}

    rollup_ann = {
        "description": "The annotation a rollup element keeps, transcribed from the reference's AddUnique tests "
                       "by scripts/make_goldens.py: each step's forwarded values and annotation, and what the "
                       "test asserts after it (sum, count, Annotation()) about each window.",
        "cases": [
            {"name": "TestCounterElemAddUnique", "src_line": "aggregator/aggregator/elem_test.go:312-364",
             "metric_type": 1, "resolution_ns": 10 * SEC, "window_starts_ns": [210 * SEC, 220 * SEC],
             "steps": [
                 add_unique(1234, 216, [345.0], None, {"window": 0, "sum": 345, "count": 1, "annotation": None}),
                 add_unique(5678, 217, [500.0], test_annot,
                            {"window": 0, "sum": 845, "count": 2, "annotation": test_annot}),
                 add_unique(1234, 221, [278.0], None, {"window": 1, "sum": 278, "count": 1},
                            {"window": 0, "annotation": test_annot}),
             ]},
            {"name": "TestGaugeElemAddUnique", "src_line": "aggregator/aggregator/elem_test.go:1478-1526",
             "metric_type": 3, "resolution_ns": 10 * SEC, "window_starts_ns": [210 * SEC, 220 * SEC],
             "steps": [
                 add_unique(1234, 216, [12.3, 34.5], None,
                            {"window": 0, "sum": 46.8, "count": 2, "annotation": None}),
                 add_unique(5678, 217, [50.0], test_annot,
                            {"window": 0, "sum": 96.8, "count": 3, "annotation": test_annot}),
                 add_unique(1234, 221, [27.8], None, {"window": 0, "annotation": test_annot},
                            {"window": 1, "sum": 27.8, "count": 1}),
             ]},
        ],
    }

    # ---- an element fed datapoint by datapoint (element sets): GenericElem.AddUnion's window contents and
    # Consume(target)'s flushed datapoints, from elem_test.go.  testTimestamps are 216 / 217 / 221 s,
    # testAlignedStarts 210 / 220 / 230 s (:120-125), resolution 10 s (:56), testGauge.GaugeVal 123.456 (:89-93),
    # testCounter.CounterVal 1234 (:79-83), testAggregationTypesExpensive {SumSq} (:59).  The default types are Last
    # (Gauge) and Sum (Counter).  An "adds" case adds its datapoints one per step and lists the windows the test
    # asserts on after each (only the fields it asserts; the reference tracks sumSq only with an expensive type, so the
    # default cases assert nothing of it here).  The Counter's datapoints are those of the case of the same name in
    # m3tsz_tile_annotation_goldens.json ("datapoints_from").  A "consumes" case starts from the windows the test
    # builds, one datapoint each ("windows": start, the value; testGaugeElemWithData stores its datapoint at the start
    # minus 1 ns, :3135-3136, which only sets lastAt), and lists each Consume's target and each type's datapoints.
    g_val, c_val = 123.456, 1234.0

    def win(start_s, **fields):
        return dict({"start_ns": start_s * SEC}, **fields)

    elem_consume = {
        "description": "An aggregator element fed datapoint by datapoint, transcribed from the reference's element "
                       "tests by scripts/make_goldens.py: the windows AddUnion leaves (adds) and the datapoints each "
                       "Consume(target) flushes at the window's end (consumes).",
        "adds": [
            {"name": "TestGaugeElemAddUnion", "src_line": "aggregator/aggregator/elem_test.go:1383-1424",
             "metric_type": 3, "agg_types": [1], "resolution_ns": 10 * SEC,
             "datapoints": [[216 * SEC, g_val], [217 * SEC, g_val], [221 * SEC, g_val]],
             "want_windows": [[win(210, last=g_val, sum=g_val)],
                              [win(210, last=g_val, sum=2 * g_val)],
                              [win(210), win(220, last=g_val, sum=g_val)]]},
            {"name": "TestGaugeElemAddUnionWithCustomAggregation",
             "src_line": "aggregator/aggregator/elem_test.go:1426-1471", "metric_type": 3, "agg_types": [8],
             "resolution_ns": 10 * SEC,
             "datapoints": [[216 * SEC, g_val], [217 * SEC, g_val], [221 * SEC, g_val]],
             "want_windows": [[win(210, last=g_val, sum=g_val, mean=g_val, sum_sq=g_val * g_val)],
                              [win(210, last=g_val, max=g_val, sum=2 * g_val, sum_sq=2 * g_val * g_val)],
                              [win(210), win(220, last=g_val, max=g_val)]]},
            {"name": "TestCounterElemAddUnion", "src_line": "aggregator/aggregator/elem_test.go:215-259",
             "metric_type": 1, "agg_types": [7], "resolution_ns": 10 * SEC,
             "datapoints_from": "m3tsz_tile_annotation_goldens.json",
             "want_windows": [[win(210, sum=1234, count=1)],
                              [win(210, sum=2468, count=2)],
                              [win(210, count=2), win(220, sum=1234)]]},
            {"name": "TestCounterElemAddUnionWithCustomAggregation",
             "src_line": "aggregator/aggregator/elem_test.go:261-306", "metric_type": 1, "agg_types": [8],
             "resolution_ns": 10 * SEC, "datapoints_from": "m3tsz_tile_annotation_goldens.json",
             "want_windows": [[win(210, sum=1234, max=1234, sum_sq=1234 * 1234)],
                              [win(210, sum=2468, max=1234, sum_sq=2 * 1234 * 1234)],
                              [win(210), win(220, sum=1234, max=1234, sum_sq=1234 * 1234)]]},
        ],
        "consumes": [
            {"name": "TestCounterElemConsumeDefaultAggregationDefaultPipeline",
             "src_line": "aggregator/aggregator/elem_test.go:468-530", "metric_type": 1, "agg_types": [7],
             "resolution_ns": 10 * SEC, "windows": [[210 * SEC, c_val], [220 * SEC, c_val]],
             "steps": [{"target_ns": 0, "want": [[]]},
                       {"target_ns": 220 * SEC, "want": [[[220 * SEC, c_val]]]},
                       {"target_ns": 230 * SEC, "want": [[[230 * SEC, c_val]]]}]},
            {"name": "TestGaugeElemConsumeDefaultAggregationDefaultPipeline",
             "src_line": "aggregator/aggregator/elem_test.go:1645-1707", "metric_type": 3, "agg_types": [1],
             "resolution_ns": 10 * SEC, "windows": [[210 * SEC, g_val], [220 * SEC, g_val]],
             "steps": [{"target_ns": 0, "want": [[]]},
                       {"target_ns": 220 * SEC, "want": [[[220 * SEC, g_val]]]},
                       {"target_ns": 230 * SEC, "want": [[[230 * SEC, g_val]]]}]},
        ],
    }

    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    with open(OUT, "w") as f:
        json.dump(g, f, indent=1)
    print("wrote", OUT, "fixtures:", len(g["fixtures_b64"]["streams"]))
    with open(OUT_AGG, "w") as f:
        json.dump(agg, f, indent=1)
    print("wrote", OUT_AGG)
    with open(OUT_BUFFER, "w") as f:
        json.dump(buffer, f, indent=1)
    print("wrote", OUT_BUFFER)
    with open(OUT_XF, "w") as f:
        json.dump(xf, f, indent=1)
    print("wrote", OUT_XF)
    with open(OUT_ELEM, "w") as f:
        json.dump(elem, f, indent=1)
    print("wrote", OUT_ELEM)
    with open(OUT_ANN, "w") as f:
        json.dump(ann, f, indent=1)
    print("wrote", OUT_ANN)
    with open(OUT_ROLLUP, "w") as f:
        json.dump(rollup, f, indent=1)
    print("wrote", OUT_ROLLUP)
    with open(OUT_ROLLUP_ANN, "w") as f:
        json.dump(rollup_ann, f, indent=1)
    print("wrote", OUT_ROLLUP_ANN)
    with open(OUT_ELEM_CONSUME, "w") as f:
        json.dump(elem_consume, f, indent=1)
    print("wrote", OUT_ELEM_CONSUME)
    timer_goldens()
    timer_rollup_goldens()
    timer_annotation_goldens()
    forwarded_goldens()
    timer_forwarded_goldens()


def timer_goldens():
    """tests/golden/m3tsz_timer_goldens.json: the reference's exact Timer and CM stream expectations, transcribed from
    its tests (values as written there; the "tolerance" cases state a property instead of values).  Types are
    aggregation.Type ids; "batches" lists [values, times]: AddBatch(values) `times` times, in order; eps / every are
    the stream options."""
    out = os.path.join(os.path.dirname(OUT), "m3tsz_timer_goldens.json")
    default = [2, 3, 4, 5, 6, 7, 8, 9, 14, 19, 20]  # the default Timer types, ascending
    batch_timer = [1.0, 3.5, 2.2, 6.5, 4.8]
    cases = [
        {"name": "TestTimerAggregations", "src_line": "aggregator/aggregation/timer_test.go:109-180",
         "eps": 1e-3, "every": 1024, "batches": [[[float(i)], 1] for i in range(1, 101)],
         "types": [2, 3, 4, 5, 6, 7, 8, 14, 19, 20],
         "want": {"2": 1.0, "3": 100.0, "4": 50.5, "5": 50.0, "6": 100.0, "7": 5050.0, "8": 338350.0, "14": 50.0,
                  "19": 95.0}},
        {"name": "TestTimerElemBatchTimer", "src_line": "aggregator/aggregator/elem_test.go:84-88,3196-3210",
         "eps": 1e-3, "every": 1024, "batches": [[batch_timer, 1]], "types": default,
         "want": {"7": 18.0, "8": 83.38, "4": 3.6, "2": 1.0, "3": 6.5, "6": 5.0, "9": 2.15522620622523, "5": 3.5,
                  "14": 3.5, "19": 6.5, "20": 6.5}},
        {"name": "TestStreamWithOnePositiveSample", "src_line": "aggregator/aggregation/quantile/cm/stream_test.go:56-68",
         "eps": 0.01, "every": 1024, "batches": [[[100.0], 1]], "types": [2, 3, 14, 18, 20],
         "want": {"2": 100.0, "3": 100.0, "14": 100.0, "18": 100.0, "20": 100.0}},
        {"name": "TestStreamWithOneNegativeSample", "src_line": "aggregator/aggregation/quantile/cm/stream_test.go:70-82",
         "eps": 0.01, "every": 1024, "batches": [[[-100.0], 1]], "types": [2, 3, 14, 18, 20],
         "want": {"2": -100.0, "3": -100.0, "14": -100.0, "18": -100.0, "20": -100.0}},
        {"name": "TestStreamWithThreeSamples", "src_line": "aggregator/aggregation/quantile/cm/stream_test.go:84-99",
         "eps": 0.01, "every": 1024, "batches": [[[100.0], 1], [[200.0], 1], [[300.0], 1]], "types": [2, 3, 14, 18, 20],
         "want": {"2": 100.0, "3": 300.0, "14": 200.0, "18": 300.0, "20": 300.0}},
    ]
    for every in (1024, 100):
        cases.append({"name": "TestStreamWithSkewedDistribution/every=%d" % every,
                      "src_line": "aggregator/aggregation/quantile/cm/stream_test.go:206-221", "eps": 0.01,
                      "every": every, "batches": [[[1.0], 10000], [[10000000.0], 1]], "types": [2, 3, 14, 18, 20],
                      "want": {"2": 1.0, "3": 10000000.0, "14": 1.0, "18": 1.0, "20": 1.0}})
    tolerance = []
    for order in ("increasing", "decreasing"):
        for every in (1024, 100):
            tolerance.append({"name": "TestStreamWith%sSamples/every=%d" % (order.capitalize(), every),
                              "src_line": "aggregator/aggregation/quantile/cm/stream_test.go:144-176",
                              "order": order, "n": 100000, "eps": 0.01, "every": every, "types": [2, 3, 14, 18, 20],
                              "quantiles": {"14": 0.5, "18": 0.9, "20": 0.99}})
    with open(out, "w") as f:
        json.dump({"cases": cases, "tolerance": tolerance}, f, indent=1)
    print("wrote", out)


def timer_rollup_goldens():
    """tests/golden/m3tsz_timer_rollup_goldens.json: the reference's Timer rollup expectations.  "add_unique" cases are
    TimerElem.AddUnique calls in order ([at_s, value] each, a Timer.Add into the window of at_s) with what the reference
    checks after a step ("count", "sum", "sum_sq", "q0.5": Quantile(0.5); sums as InEpsilon 1e-10, the rest exact).
    "pipeline" cases are a Timer source's windows ([start_s, samples]) consumed at each target through its type and
    pre-rollup transformations; "want" lists the forwarded [time_s, value] in order ("NaN" for a NaN), compared
    exactly as verifyForwardedMetrics does."""
    out = os.path.join(os.path.dirname(OUT), "m3tsz_timer_rollup_goldens.json")
    default = [2, 3, 4, 5, 6, 7, 8, 9, 14, 19, 20]  # the default Timer types, ascending
    add_unique = [
        {"name": "TestTimerElemAddUnique", "src_line": "aggregator/aggregator/elem_test.go:120-125,927-999",
         "resolution_s": 10, "types": default, "eps": 1e-3, "every": 1024,
         "steps": [{"add": [216, 11.1]}, {"add": [216, 12.2]},
                   {"add": [216, 13.3], "window_s": 210, "want": {"count": 3, "sum": 36.6, "q0.5": 12.2}},
                   {"add": [217, 14.4], "window_s": 210, "want": {"count": 4, "sum": 51.0}},
                   {"add": [221, 20.0], "window_s": 220, "want": {"count": 1, "sum": 20.0, "sum_sq": 400.0}}]},
    ]
    pipeline = [
        {"name": "TestTimerElemConsumeCustomAggregationCustomPipeline",
         "src_line": "aggregator/aggregator/elem_test.go:94-110,1138-1264", "resolution_s": 10, "src_type": 2,
         "pre_ops": [1, 2], "discard_nan": False, "rollup_types": [3],
         "windows": [[210, [123.0, 1245.0]], [220, [456.0]], [230, [589.0, 1120.0]]],
         "consumes": [{"target_s": 0, "want": []}, {"target_s": 220, "want": [[220, "NaN"]]},
                      {"target_s": 240, "want": [[230, 33.3], [240, 13.3]]}]},
    ]
    with open(out, "w") as f:
        json.dump({"add_unique": add_unique, "pipeline": pipeline}, f, indent=1)
    print("wrote", out)


def timer_annotation_goldens():
    """tests/golden/m3tsz_timer_annotation_goldens.json: the reference's Timer annotation expectation.  "adds" lists
    Timer.Add calls in order as [value, annotation] (null for a nil annotation); "want" is Annotation() after them."""
    out = os.path.join(os.path.dirname(OUT), "m3tsz_timer_annotation_goldens.json")
    cases = [
        {"name": "TestTimerReturnsLastNonEmptyAnnotation", "src_line": "aggregator/aggregation/timer_test.go:212-222",
         "adds": [[1.1, "first"], [2.1, "second"], [3.1, None]], "want": "second"},
    ]
    with open(out, "w") as f:
        json.dump({"cases": cases}, f, indent=1)
    print("wrote", out)


def forwarded_goldens():
    """tests/golden/m3tsz_forwarded_goldens.json: the reference's AddUnique and forwarded-writer expectations.
    "add_unique" cases are AddUnique calls in order, each step [at_s, values, source_id] with the result the reference
    returns ("ok" or "duplicate") and what it checks after the step: "windows_s" the open window starts, and in
    "window_s" the aggregation's "sum" / "count" / "max" / "sum_sq" (sums with "eps" as InEpsilon, the rest exact).
    The reference checks SumSq only where it computes it (an expensive type in the list, the custom forms).  Steps with
    a version above 0 (a resend) and the tombstoned element's errElemClosed are not transcribed.  "writer" cases are
    writeFn calls in order as [id, time_ns, value] and the ForwardedMetrics onDone sends as [id, time_ns, values]."""
    out = os.path.join(os.path.dirname(OUT), "m3tsz_forwarded_goldens.json")
    src = "aggregator/aggregator/elem_test.go:120-125,"
    add_unique = [
        {"name": "TestCounterElemAddUnique", "src_line": src + "308-390", "metric": "counter", "resolution_s": 10,
         "custom": False,
         "steps": [[216, [345.0], 1234, "ok", [210], 210, {"sum": 345, "count": 1}],
                   [217, [500.0], 5678, "ok", [210], 210, {"sum": 845, "count": 2}],
                   [221, [278.0], 1234, "ok", [210, 220], 220, {"sum": 278, "count": 1}],
                   [221, [278.0], 1234, "duplicate", [210, 220], 220, {"sum": 278, "count": 1}]]},
        {"name": "TestCounterElemAddUniqueWithCustomAggregation", "src_line": src + "392-466", "metric": "counter",
         "resolution_s": 10, "custom": True,
         "steps": [[216, [12.0], 1234, "ok", [210], 210, {"sum": 12, "max": 12, "sum_sq": 144}],
                   [217, [14.0], 5678, "ok", [210], 210, {"sum": 26, "max": 14}],
                   [221, [20.0], 1234, "ok", [210, 220], 220, {"sum": 20, "max": 20, "sum_sq": 400}],
                   [221, [30.0], 1234, "duplicate", [210, 220], 220, {"sum": 20, "count": 1, "sum_sq": 400}]]},
        {"name": "TestGaugeElemAddUnique", "src_line": src + "1473-1546", "metric": "gauge", "resolution_s": 10,
         "custom": False,
         "steps": [[216, [12.3, 34.5], 1234, "ok", [210], 210, {"sum": 46.8, "count": 2}],
                   [217, [50.0], 5678, "ok", [210], 210, {"sum": 96.8, "count": 3}],
                   [221, [27.8], 1234, "ok", [210, 220], 220, {"sum": 27.8, "count": 1}],
                   [221, [27.8], 1234, "duplicate", [210, 220], 220, {"sum": 27.8, "count": 1}]]},
        {"name": "TestGaugeElemAddUniqueWithCustomAggregation", "src_line": src + "1572-1643", "metric": "gauge",
         "resolution_s": 10, "custom": True,
         "steps": [[216, [1.2], 1234, "ok", [210], 210, {"sum": 1.2, "max": 1.2, "sum_sq": 1.44}],
                   [217, [1.4], 5678, "ok", [210], 210, {"sum": 2.6, "max": 1.4, "eps": 1e-10}],
                   [221, [2.0], 1234, "ok", [210, 220], 220, {"sum": 2.0, "max": 2.0, "sum_sq": 4.0}],
                   [221, [3.0], 1234, "duplicate", [210, 220], 220, {"sum": 2.0, "max": 2.0, "sum_sq": 4.0}]]},
    ]
    writer = [
        {"name": "TestForwardedWriterPrepare", "src_line": "aggregator/aggregator/forwarded_writer_test.go:351-435",
         "source_id": 0,
         "writes": [["foo", 1234, 3.4], ["foo", 1234, 3.5], ["foo", 1240, 98.2], ["bar", 1238, 3.4],
                    ["bar", 1239, 3.5]],
         "want": [["foo", 1234, [3.4, 3.5]], ["foo", 1240, [98.2]], ["bar", 1238, [3.4]], ["bar", 1239, [3.5]]]},
    ]
    with open(out, "w") as f:
        json.dump({"add_unique": add_unique, "writer": writer}, f, indent=1)
    print("wrote", out)


def timer_forwarded_goldens():
    """tests/golden/m3tsz_timer_forwarded_goldens.json: the reference's TimerElem.AddUnique expectations with their
    source ids.  Each step is [at_s, values, source_id] with the result the reference returns ("ok" or "duplicate") and
    what it checks after the step: "windows_s" the open window starts, and in "window_s" the Timer's "count", "sum",
    "sum_sq" (sums as InEpsilon 1e-10, the rest exact), "q0.5" (Quantile(0.5)) and "seen" (source ids whose
    sourcesSeen entry it asserts).  The tombstoned element's errElemClosed is not transcribed."""
    out = os.path.join(os.path.dirname(OUT), "m3tsz_timer_forwarded_goldens.json")
    default = [2, 3, 4, 5, 6, 7, 8, 9, 14, 19, 20]  # the default Timer types, ascending
    cases = [
        {"name": "TestTimerElemAddUnique", "src_line": "aggregator/aggregator/elem_test.go:120-125,927-999",
         "resolution_s": 10, "types": default, "eps": 1e-3, "every": 1024,
         "steps": [[216, [11.1], 1, "ok", [210], 210, {}],
                   [216, [12.2], 2, "ok", [210], 210, {}],
                   [216, [13.3], 3, "ok", [210], 210, {"count": 3, "sum": 36.6, "q0.5": 12.2}],
                   [217, [14.4], 4, "ok", [210], 210, {"count": 4, "sum": 51.0}],
                   [221, [20.0], 1, "ok", [210, 220], 220, {"count": 1, "sum": 20.0}],
                   [221, [30.0], 1, "duplicate", [210, 220], 220,
                    {"count": 1, "sum": 20.0, "sum_sq": 400.0, "seen": [1]}]]},
    ]
    with open(out, "w") as f:
        json.dump({"add_unique": cases}, f, indent=1)
    print("wrote", out)


if __name__ == "__main__":
    main()
