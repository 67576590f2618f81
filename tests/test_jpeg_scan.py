"""CPU tests of scan images (pe_jpeg_read_scan) and of the GPU entropy decoder's algorithm run on the host
(pe_jpeg_scan_to_coefs_host): the coefficient image it builds from a scan image must equal pe_jpeg_read_coefs's byte for byte, on
both host routes, at every subsequence length, on clean and on corrupt streams.  tests/golden/jpeg_scans.npz was written by OpenCV's
libjpeg with tools/gen_jpeg_scan_fixtures.py (restart intervals, optimised tables, 4:2:2, grey, DHT-less Motion-JPEG frames, SOS
component order other than SOF order)."""
import os
import subprocess

import numpy as np
import pytest

from caffe_rtpose_b200 import engine, synth
from test_jpeg_coefs import fixtures as coef_fixtures, read_coefs_rc, route

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCAN_FIXTURES = os.path.join(ROOT, "tests", "golden", "jpeg_scans.npz")
ONE_PER_SEGMENT = 1 << 30          # a subsequence longer than any segment
SUBSEQ = (32, 64, 1024, ONE_PER_SEGMENT)
HEADER = 2784


def scan_fixtures():
    z = np.load(SCAN_FIXTURES)
    return {k: z[k].tobytes() for k in z.files}


def all_fixtures():
    out = dict(coef_fixtures())
    out.update(scan_fixtures())
    return out


def is_progressive(data):
    return data[2:].find(b"\xff\xc2") >= 0


def read_scan_rc(data, cap=None):
    n = engine.lib().pe_jpeg_read_scan(data, len(data), None, 0)
    if n < 0:
        return n, None
    buf = np.zeros(max(n if cap is None else cap, 1), np.uint8)
    rc = engine.lib().pe_jpeg_read_scan(data, len(data), buf.ctypes.data, n if cap is None else cap)
    return rc, buf


def coefs_full_rc(data):
    """pe_jpeg_read_coefs's outcome after the whole file (its size query stops at the frame header)"""
    rc, buf = read_coefs_rc(data)
    return rc, buf


def scan_fields(buf):
    i32 = buf[512:576].view(np.int32)
    i64 = buf[576:608].view(np.int64)
    return {"magic": int(buf[512:516].view(np.uint32)[0]), "num_scan_comps": int(i32[1]), "scan_comp": list(i32[2:5]),
            "dc_table": list(i32[5:8]), "ac_table": list(i32[8:11]), "restart": int(i32[11]), "mcux": int(i32[12]),
            "mcuy": int(i32[13]), "num_segments": int(i32[14]), "seg_table_offset": int(i64[0]), "data_offset": int(i64[1]),
            "data_bytes": int(i64[2]), "total_bytes": int(i64[3])}


def segments(buf):
    f = scan_fields(buf)
    return buf[f["seg_table_offset"]:f["data_offset"]].view(np.int64).reshape(-1, 2)


def test_return_codes_on_the_fixtures():
    for name, data in all_fixtures().items():
        rc, buf = read_scan_rc(data)
        if is_progressive(data):
            assert rc == -3, name
            continue
        crc, coefs = coefs_full_rc(data)
        assert rc > 0 and crc > 0, (name, rc, crc)
        assert np.array_equal(buf[:512], coefs[:512]), name    # the coefficient header pe_jpeg_read_coefs writes


def test_layout_size_query_and_short_cap():
    data = scan_fixtures()["422_restart7_q98"]
    n = engine.lib().pe_jpeg_read_scan(data, len(data), None, 0)
    buf = engine.read_jpeg_scan(data)
    assert n == buf.size
    f = scan_fields(buf)
    assert f["magic"] == 0x4E43534A and f["num_scan_comps"] == 3 and f["scan_comp"] == [0, 1, 2]
    assert f["dc_table"] == [0, 1, 1] and f["ac_table"] == [0, 1, 1]
    assert (f["restart"], f["mcux"], f["mcuy"]) == (7, 9, 13)          # 131 x 97 at 4:2:2: MCUs of 16 x 8
    assert f["num_segments"] == (9 * 13 + 6) // 7
    assert f["seg_table_offset"] == HEADER and f["data_offset"] == HEADER + 16 * f["num_segments"]
    assert f["total_bytes"] == f["data_offset"] + f["data_bytes"] == n
    seg = segments(buf)
    ecs = buf[f["data_offset"]:]
    sos = data.find(b"\xff\xda")
    start = sos + 2 + int.from_bytes(data[sos + 2:sos + 4], "big")
    assert bytes(ecs) == data[start:start + f["data_bytes"]]          # the entropy-coded bytes, stuffing and RST markers kept
    assert seg[0, 0] == 0
    for k in range(1, len(seg)):                                       # segment k starts right behind RST((k - 1) % 8)
        assert bytes(ecs[seg[k, 0] - 2:seg[k, 0]]) == bytes([0xFF, 0xD0 + (k - 1) % 8]), k
        assert seg[k - 1, 0] + seg[k - 1, 1] == seg[k, 0] - 2
    assert read_scan_rc(data, n - 1)[0] == -1
    rc, big = read_scan_rc(data, n + 64)
    assert rc == n and np.array_equal(big[:n], buf)
    assert engine.lib().pe_jpeg_read_scan(None, 0, None, 0) == -1
    with pytest.raises(engine.PoseEngineError, match="host entropy stage"):
        engine.read_jpeg_scan(coef_fixtures()["444_83x61_progressive"])


@pytest.mark.parametrize("fast", [True, False], ids=["fast-route", "general-route"])
def test_host_run_of_the_gpu_algorithm_equals_read_coefs_on_the_fixtures(fast):
    with route(fast):
        for name, data in all_fixtures().items():
            if is_progressive(data):
                continue
            ref = engine.read_jpeg_coefs(data)
            scan = engine.read_jpeg_scan(data)
            for S in SUBSEQ:
                got, ok = engine.jpeg_scan_to_coefs_host(scan, S)
                assert ok and np.array_equal(got, ref), (name, S)


@pytest.mark.parametrize("size", [(1280, 720), (1920, 1080)], ids=["720p", "1080p"])
def test_host_run_of_the_gpu_algorithm_at_camera_sizes(size):
    w, h = size
    for q in (50, 85, 98):
        data = engine.encode_jpeg(synth.make_frame(q, h, w), q)
        ref = engine.read_jpeg_coefs(data)
        scan = engine.read_jpeg_scan(data)
        for S in SUBSEQ:
            got, ok = engine.jpeg_scan_to_coefs_host(scan, S)
            assert ok and np.array_equal(got, ref), (q, S)


def dc_category_error(data, category):
    """the first DC table's symbol for `category` becomes 16 + category: the first block that uses it has a DC category above 15"""
    d = bytearray(data)
    p = d.find(b"\xff\xc4")
    assert p > 0
    s = p + 4
    while s < p + 2 + int.from_bytes(d[p + 2:p + 4], "big"):
        tc, n = d[s] >> 4, sum(d[s + 1:s + 17])
        if tc == 0:
            vals = d[s + 17:s + 17 + n]
            i = vals.index(category)
            d[s + 17 + i] = 16 + category
            return bytes(d)
        s += 17 + n
    raise AssertionError("no DC table")


def corrupt_streams():
    """truncated data (the zero tail), a missing RST, extra / misplaced RSTs and other markers inside the data, DC errors"""
    files = scan_fixtures()
    rng = np.random.default_rng(7)
    out = []
    for name in ("420_restart7", "422_restart1_q98", "420_optimized", "grey_restart7", "sos_order_cr_cb_restart1"):
        data = files[name]
        sos = data.find(b"\xff\xda")
        body = sos + 2 + int.from_bytes(data[sos + 2:sos + 4], "big")
        out += [data[:k] for k in range(body, len(data), max(1, (len(data) - body) // 12))]          # truncations
        rst = [i for i in range(body, len(data) - 1) if data[i] == 0xFF and 0xD0 <= data[i + 1] <= 0xD7]
        if rst:
            k = rst[len(rst) // 2]
            out.append(data[:k] + data[k + 2:])                                                    # a missing RST
            out.append(data[:k] + b"\xff\xd3" + data[k:])                                          # an extra RST
            d = bytearray(data); d[k + 1] ^= 1; out.append(bytes(d))                               # the wrong RST number
        for m in (b"\xff\xd0", b"\xff\xd9", b"\xff\xc4", b"\xff\xfe", b"\xff\xff"):                 # markers inside the data
            k = int(rng.integers(body, len(data) - 2))
            out.append(data[:k] + m + data[k:])
        for _ in range(25):                                                                        # byte and bit flips in the data
            d = bytearray(data)
            for _ in range(int(rng.integers(1, 4))):
                d[int(rng.integers(body, len(d) - 2))] = int(rng.integers(0, 256))
            out.append(bytes(d))
        for cat in (0, 3, 6):
            try:
                out.append(dc_category_error(data, cat))
            except ValueError:
                pass
    return out


def test_host_run_of_the_gpu_algorithm_on_corrupt_streams():
    codes = {}
    for fast in (True, False):
        with route(fast):
            for d in corrupt_streams():
                crc, ref = coefs_full_rc(d)
                src, scan = read_scan_rc(d)
                if src == -3:
                    continue
                if src < 0:
                    assert src == crc, (src, crc)
                    codes["parser"] = codes.get("parser", 0) + 1
                    continue
                assert crc > 0 or crc == -1, crc
                for S in SUBSEQ:
                    got, ok = engine.jpeg_scan_to_coefs_host(scan, S)
                    assert ok == (crc > 0), (S, crc)      # the data error is flagged exactly where the host stage rejects the file
                    if ok:
                        assert np.array_equal(got, ref), S
                codes["decoded" if crc > 0 else "dc error"] = codes.get("decoded" if crc > 0 else "dc error", 0) + 1
    assert codes.get("parser") and codes.get("decoded") and codes.get("dc error"), codes


def test_missing_restart_marker_is_an_error():
    data = scan_fixtures()["420_restart7"]
    sos = data.find(b"\xff\xda")
    rst = [i for i in range(sos, len(data) - 1) if data[i] == 0xFF and 0xD0 <= data[i + 1] <= 0xD7]
    d = data[:rst[-1]] + data[rst[-1] + 2:]
    assert engine.lib().pe_jpeg_read_scan(d, len(d), None, 0) == -1 == read_coefs_rc(d)[0]


def test_scan_stage_survives_mutations_under_sanitizers(tmp_path):
    src = os.path.join(ROOT, "caffe_rtpose_b200", "csrc")
    exe = str(tmp_path / "fuzz_jpeg_scan")
    r = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined",
                        "-I", os.path.join(ROOT, "include"), "-I", src, os.path.join(ROOT, "tests", "fuzz", "fuzz_jpeg_scan.cpp"),
                        os.path.join(src, "jpeg_dec.cpp"), "-o", exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    files = scan_fixtures()
    paths = []
    for name in ("420_restart7", "422_restart1_q98", "grey_restart7", "mjpeg_no_dht", "sos_order_cr_cb"):
        p = tmp_path / (name + ".jpg")
        p.write_bytes(files[name])
        paths.append(str(p))
    for fast in ("1", "0"):
        r = subprocess.run([exe, "200"] + paths, capture_output=True, text=True, timeout=900, env=dict(os.environ, PE_JPEG_FAST=fast))
        assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
        assert "mismatches 0" in r.stdout and not r.stdout.startswith("decoded 0 "), r.stdout


BIN = os.path.join(ROOT, "caffe_rtpose_b200", "rtpose.bin")


def test_video_read_scan_matches_the_frames():
    from test_jpeg_coefs import strip_dht, write_mjpeg_avi
    import ctypes as C
    import tempfile
    jpegs = [strip_dht(engine.encode_jpeg(synth.make_frame(30 + i, 48, 64), 90)) for i in range(3)]
    jpegs.append(coef_fixtures()["420_64x48_progressive"])
    with tempfile.TemporaryDirectory() as d:
        avi = os.path.join(d, "clip.avi")
        write_mjpeg_avi(avi, jpegs, 64, 48)
        L = engine.lib()
        v = C.c_void_p()
        assert L.pe_video_open(avi.encode(), C.byref(v)) == 0
        try:
            for i, j in enumerate(jpegs):
                n = L.pe_video_read_scan(v, i, None, 0)
                if is_progressive(j):
                    assert n == -3
                    continue
                buf = np.zeros(n, np.uint8)
                assert L.pe_video_read_scan(v, i, buf.ctypes.data, n) == n
                assert np.array_equal(buf, engine.read_jpeg_scan(j)), i
            assert L.pe_video_read_scan(v, 99, None, 0) == -1   # -PE_ERR_INVALID: outside the video
        finally:
            L.pe_video_close(v)


def test_cli_gpu_entropy_refusals_and_help():
    for extra in (["--synthetic", "4"], []):   # no --video / --image_dir: the camera
        r = subprocess.run([BIN, "--gpu_entropy", "--model", "COCO", "--resolution", "64x48"] + extra, capture_output=True, text=True, timeout=60)
        assert r.returncode == 1 and "--gpu_entropy decodes JPEG files on the GPU: it needs --image_dir or a Motion-JPEG --video" in r.stderr, r.stderr
    r = subprocess.run([BIN, "--help"], capture_output=True, text=True, timeout=60)
    assert '--gpu_entropy (' in r.stdout and 'default: "false"' in r.stdout.split("--gpu_entropy (")[1].split("\n")[0]


def test_cli_gpu_entropy_producer_stage_without_gpu(tmp_path):
    """--decode_bench --gpu_entropy: sequential JPEGs become scan images, progressive ones coefficient images, other files and
    undecodable ones take the host decoder; the frame accounting is the same as without the flag"""
    from test_jpeg_coefs import strip_dht, write_mjpeg_avi
    d = tmp_path / "imgs"
    d.mkdir()
    for i in range(8):
        (d / ("f%02d.jpg" % i)).write_bytes(engine.encode_jpeg(synth.make_frame(i, 48, 64), 90))
    (d / "f08.jpg").write_bytes(coef_fixtures()["444_83x61_progressive"])
    (d / "f09.jpg").write_bytes(b"\xff\xd8 not a jpeg")
    (d / "f10.ppm").write_bytes(b"P6\n64 48\n255\n" + synth.make_frame(9, 48, 64).tobytes())
    avi = str(tmp_path / "clip.avi")
    write_mjpeg_avi(avi, [strip_dht(engine.encode_jpeg(synth.make_frame(20 + i, 48, 64), 90)) for i in range(6)], 64, 48)
    for src, n in ((["--image_dir", str(d)], 10), (["--video", avi, "--novideo_realtime"], 6)):
        outs = []
        for flag in ([], ["--gpu_decode"], ["--gpu_entropy"]):
            r = subprocess.run([BIN] + src + ["--decode_bench", "--num_producers", "3", "--model", "COCO", "--resolution", "64x48"] + flag,
                               capture_output=True, text=True, timeout=120)
            assert r.returncode == 0, r.stderr
            outs.append(r.stdout.strip().splitlines()[-1].split(" in ")[0])
        assert outs[0] == outs[1] == outs[2], outs
        assert outs[0].startswith("decoded %d frames" % n), outs


def test_dc_error_followed_by_a_header_error():
    """the coefficient stage stops at the scan's data error (-1); the scan stage does not decode, parses on and reports the later
    header's error instead (-2 for an SOF3 after the scan): both refuse the file"""
    data = dc_category_error(scan_fixtures()["420_optimized"], 0)
    eoi = data.rfind(b"\xff\xd9")
    d = data[:eoi] + b"\xff\xc3\x00\x0b\x08\x00\x10\x00\x10\x01\x01\x11\x00" + data[eoi:]
    assert coefs_full_rc(d)[0] == -1 and engine.lib().pe_jpeg_read_scan(d, len(d), None, 0) == -2
