"""Calibration tables (pe_calibration_get / pe_calibration_set, csrc/calib_table.cpp) without a GPU: the reader under ASAN + UBSan,
with a named case and message for every refusal that needs no engine, and a mutation fuzzer over valid tables."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "caffe_rtpose_b200", "csrc")


@pytest.fixture(scope="module")
def fuzzer(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("calib") / "fuzz_calibration_table")
    r = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-I", SRC,
                        os.path.join(ROOT, "tests", "fuzz", "fuzz_calibration_table.cpp"), os.path.join(SRC, "calib_table.cpp"), "-o", exe],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


def test_every_refusal_names_its_line_or_layer(fuzzer):
    r = subprocess.run([fuzzer, "cases"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    got = {}
    for line in r.stdout.splitlines():
        name, rc, msg = line.split(" ", 2)
        got[name] = (int(rc), msg)
    want = {
        "valid": "ok",
        "valid_comments": "ok",
        "empty": "empty calibration table",
        "version": "line 1: calibration table version 2: this library reads version 1",
        "precision": "line 2: the table is for precision 5, the engine runs precision 6",
        "weights": "line 3: the table was calibrated with other weights",
        "weights_syntax": "line 3: weights hash '12345' is not 16 hex digits",
        "missing": "layer conv3_1 is missing",
        "missing_last": "layer conv6_1 is missing (the table ends before it)",
        "duplicated": "line 7: layer conv3_1 appears twice (first on line 6)",
        "out_of_order": "line 6: layer conv4_1 is out of order: the engine runs conv3_1 here",
        "unknown": "line 6: unknown layer conv9_9",
        "kind": "line 6: layer conv3_1 stores f16 in the table, s8 in the engine",
        "exponent": "line 6: layer conv3_1: log2 scale 101 is outside [-100, 100]",
        "exponent_syntax": "line 6: layer conv3_1: log2 scale '3.5' is not an integer",
        "trailing_text": "line 6: trailing text 'extra'",
        "trailing_line": "line 10: expected 'layer <name> <kind> <log2 scale>', found 'end'",
        "header_order": "line 2: expected 'precision ...', found 'weights'",
    }
    assert set(got) == set(want)
    for name, msg in want.items():
        rc, text = got[name]
        assert (rc == 0) == (msg == "ok"), (name, rc, text)
        assert msg in text, (name, text)


def test_reader_survives_mutated_tables(fuzzer):
    r = subprocess.run([fuzzer, "fuzz", "20000"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.stdout[-500:], r.stderr[-3000:])
    accepted, rejected = [int(v) for v in r.stdout.split()[1::2]]
    assert accepted > 50 and rejected > 5000   # comments, blank lines and equal digits pass; everything else is refused
