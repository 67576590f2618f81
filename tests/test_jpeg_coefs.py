"""CPU tests of the JPEG coefficient stage (pe_jpeg_read_coefs): the host half of GPU JPEG decoding.  The coefficient image it
returns, transformed by pe_decode_jpeg's own IDCT / upsampling / colour code (pe_jpeg_coefs_to_bgr), must give pe_decode_jpeg's
bytes on every fixture and on both decoder routes; corrupt and unsupported streams get pe_decode_jpeg's return codes.  The
fixtures (tests/golden/jpeg_coefs.npz) were written by OpenCV's libjpeg with tools/gen_jpeg_fixtures.py."""
import os
import subprocess

import numpy as np
import pytest

from caffe_rtpose_b200 import engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = os.path.join(ROOT, "tests", "golden", "jpeg_coefs.npz")


def fixtures():
    z = np.load(FIXTURES)
    return {k: z[k].tobytes() for k in z.files}


def route(fast):
    """PE_JPEG_FAST is read per call: 1 = the fast route (one interleaved sequential scan), 0 = the general route."""
    class _Route:
        def __enter__(self):
            self.old = os.environ.get("PE_JPEG_FAST")
            os.environ["PE_JPEG_FAST"] = "1" if fast else "0"

        def __exit__(self, *a):
            if self.old is None:
                del os.environ["PE_JPEG_FAST"]
            else:
                os.environ["PE_JPEG_FAST"] = self.old
    return _Route()


def read_coefs_rc(data, cap=None):
    n = engine.lib().pe_jpeg_read_coefs(data, len(data), None, 0)
    if n < 0:
        return n, None
    buf = np.zeros(max(n, 1) if cap is None else max(cap, 1), np.uint8)
    rc = engine.lib().pe_jpeg_read_coefs(data, len(data), buf.ctypes.data, n if cap is None else cap)
    return rc, buf


def decode_rc(data):
    w, h = engine.C.c_int(), engine.C.c_int()
    rc = engine.lib().pe_decode_jpeg(data, len(data), engine.C.byref(w), engine.C.byref(h), None, 0)
    if rc != 0:
        return rc, None
    out = np.zeros((h.value, w.value, 3), np.uint8)
    rc = engine.lib().pe_decode_jpeg(data, len(data), engine.C.byref(w), engine.C.byref(h), out.ctypes.data, out.size)
    return rc, out if rc == 0 else None


def test_fixtures_cover_the_variants():
    seen = set()
    for name, data in fixtures().items():
        hd = engine.jpeg_coef_header(engine.read_jpeg_coefs(data))
        y = hd["comps"][0]
        seen.add("grey" if hd["num_comps"] == 1 else {(1, 1): "444", (2, 1): "422", (2, 2): "420"}[(y["h"], y["v"])])
        if data[2:].find(b"\xff\xc2") >= 0:
            seen.add("progressive")
        if data.find(b"\xff\xdd") >= 0:
            seen.add("restart")
        if hd["width"] % (8 * hd["hmax"]) and hd["height"] % (8 * hd["vmax"]):
            seen.add("partial MCU")
        if hd["num_comps"] == 3 and hd["hmax"] == 2 and hd["comps"][1]["dw"] <= 2:
            seen.add("narrow chroma")
        if max(int(c["quant"].max()) for c in hd["comps"]) > 255:
            seen.add("16-bit tables")
    assert seen >= {"grey", "444", "422", "420", "progressive", "restart", "partial MCU", "narrow chroma", "16-bit tables"}, seen


@pytest.mark.parametrize("fast", [True, False], ids=["fast-route", "general-route"])
def test_host_reconstruction_of_coefficients_equals_decode_jpeg(fast):
    with route(fast):
        for name, data in fixtures().items():
            ref = engine.decode_jpeg(data)
            buf = engine.read_jpeg_coefs(data)
            hd = engine.jpeg_coef_header(buf)
            assert hd["magic"] == 0x4345504A and (hd["width"], hd["height"]) == (ref.shape[1], ref.shape[0]), name
            assert hd["total_bytes"] == buf.size, name
            assert np.array_equal(engine.jpeg_coefs_to_bgr(buf), ref), name


def test_both_routes_store_the_same_coefficients():
    for name, data in fixtures().items():
        with route(True):
            a = engine.read_jpeg_coefs(data)
        with route(False):
            b = engine.read_jpeg_coefs(data)
        assert np.array_equal(a, b), name


def test_layout_of_the_coefficient_image():
    data = fixtures()["420_83x61"]
    buf = engine.read_jpeg_coefs(data)
    hd = engine.jpeg_coef_header(buf)
    assert (hd["num_comps"], hd["hmax"], hd["vmax"]) == (3, 2, 2)
    y, cb, cr = hd["comps"]
    assert (y["bw"], y["bh"], y["dw"], y["dh"]) == (12, 8, 83, 61)      # 6 x 4 MCUs of 16 x 16
    assert (cb["bw"], cb["bh"], cb["dw"], cb["dh"]) == (6, 4, 42, 31) == (cr["bw"], cr["bh"], cr["dw"], cr["dh"])
    assert y["offset"] == 512 and cb["offset"] == 512 + 12 * 8 * 128 and cr["offset"] == cb["offset"] + 6 * 4 * 128
    assert hd["total_bytes"] == cr["offset"] + 6 * 4 * 128
    coef = buf[512:].view(np.int16)
    assert coef[0] != 0 and np.abs(coef).max() < 2048   # DC of the first luma block first; 8-bit data stays in 11 bits


def test_size_query_short_cap_and_bad_arguments():
    data = fixtures()["422_83x61"]
    n = engine.lib().pe_jpeg_read_coefs(data, len(data), None, 0)
    assert n > 512
    assert read_coefs_rc(data, n - 1)[0] == -1
    rc, buf = read_coefs_rc(data, n + 100)
    assert rc == n and np.array_equal(buf[:n], engine.read_jpeg_coefs(data))
    assert engine.lib().pe_jpeg_read_coefs(None, 0, None, 0) == -1
    assert engine.lib().pe_jpeg_read_coefs(b"\xff\xd8", 2, None, 0) == -1
    with pytest.raises(engine.PoseEngineError):
        engine.read_jpeg_coefs(b"not a jpeg at all")
    bad = engine.read_jpeg_coefs(data)
    bad[4] ^= 1   # width no longer matches the block grid
    with pytest.raises(engine.PoseEngineError, match="malformed"):
        engine.jpeg_coefs_to_bgr(bad)
    with pytest.raises(engine.PoseEngineError, match="truncated"):
        engine.jpeg_coefs_to_bgr(engine.read_jpeg_coefs(data)[:-1])


def _unsupported_variants(data):
    """byte edits that make pe_decode_jpeg answer -2: lossless / arithmetic SOF, 12-bit samples, 4:1:1 sampling"""
    sof = data.find(b"\xff\xc0")
    assert sof > 0
    out = []
    for m in (0xC3, 0xC9):
        d = bytearray(data); d[sof + 1] = m; out.append(bytes(d))
    d = bytearray(data); d[sof + 4] = 12; out.append(bytes(d))
    d = bytearray(data); d[sof + 11] = 0x41; out.append(bytes(d))   # Y sampling 4x1
    return out


def test_corrupt_and_unsupported_files_get_decode_jpeg_codes():
    rng = np.random.default_rng(5)
    files = fixtures()
    streams = []
    for name in ("420_83x61", "422_restart3", "444_83x61_progressive", "grey_51x29", "420_progressive_restart2"):
        data = files[name]
        streams += [data[:k] for k in range(0, len(data), max(1, len(data) // 40))]   # truncations
        for _ in range(60):
            d = bytearray(data)
            for _ in range(int(rng.integers(1, 4))):
                d[int(rng.integers(2, len(d)))] = int(rng.integers(0, 256))
            streams.append(bytes(d))
    streams += [b"\xff\xd8" + rng.integers(0, 256, 3000, dtype=np.uint8).tobytes() for _ in range(20)]
    unsupported = _unsupported_variants(files["420_83x61"])
    streams += unsupported
    codes = {}
    for fast in (True, False):
        with route(fast):
            for d in streams:
                rc, ref = decode_rc(d)
                crc, buf = read_coefs_rc(d)
                assert (crc > 0) == (rc == 0) and (rc == 0 or crc == rc), (rc, crc)
                codes[rc] = codes.get(rc, 0) + 1
                if rc == 0:   # corrupt but decodable: the coefficient route must give the very same pixels
                    assert np.array_equal(engine.jpeg_coefs_to_bgr(buf), ref)
    assert codes.get(-1) and codes.get(0) and codes.get(-2, 0) >= 2 * len(unsupported), codes
    for d in unsupported:
        assert engine.lib().pe_jpeg_read_coefs(d, len(d), None, 0) == -2


def test_coefficient_stage_survives_mutations_under_sanitizers(tmp_path):
    src = os.path.join(ROOT, "caffe_rtpose_b200", "csrc")
    exe = str(tmp_path / "fuzz_jpeg_coefs")
    r = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined",
                        "-I", os.path.join(ROOT, "include"), "-I", src, os.path.join(ROOT, "tests", "fuzz", "fuzz_jpeg_coefs.cpp"),
                        os.path.join(src, "jpeg_dec.cpp"), "-o", exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    files = fixtures()
    paths = []
    for name in ("420_83x61", "422_restart3", "444_dqt16_progressive", "grey_progressive", "420_narrow_3x13"):
        p = tmp_path / (name + ".jpg")
        p.write_bytes(files[name])
        paths.append(str(p))
    for fast in ("1", "0"):
        r = subprocess.run([exe, "300"] + paths, capture_output=True, text=True, timeout=900, env=dict(os.environ, PE_JPEG_FAST=fast))
        assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
        assert "mismatches 0" in r.stdout


BIN = os.path.join(ROOT, "caffe_rtpose_b200", "rtpose.bin")


def write_mjpeg_avi(path, jpegs, w, h, fps=25):
    """Minimal AVI 1.0 (RIFF hdrl(avih, strl(strh, strf)) + movi of '00dc' chunks) holding the given JPEG frames."""
    import struct as st

    def chunk(tag, data):
        return tag + st.pack("<I", len(data)) + data + (b"\0" if len(data) % 2 else b"")
    avih = st.pack("<IIIIIIIIIIIIII", 1000000 // fps, 0, 0, 0x10, len(jpegs), 0, 1, 0, w, h, 0, 0, 0, 0)
    strh = b"vids" + b"MJPG" + st.pack("<IHHIIIIIIIIHHHH", 0, 0, 0, 0, 1, fps, 0, len(jpegs), 0, 0xFFFFFFFF, 0, 0, 0, w, h)
    strf = st.pack("<IiiHH4sIiiII", 40, w, h, 1, 24, b"MJPG", 0, 0, 0, 0, 0)
    hdrl = b"hdrl" + chunk(b"avih", avih) + chunk(b"LIST", b"strl" + chunk(b"strh", strh) + chunk(b"strf", strf))
    movi = b"movi" + b"".join(chunk(b"00dc", j) for j in jpegs)
    body = b"AVI " + chunk(b"LIST", hdrl) + chunk(b"LIST", movi)
    with open(path, "wb") as f:
        f.write(b"RIFF" + st.pack("<I", len(body)) + body)


def strip_dht(jpeg):
    """Motion-JPEG frames usually leave the (standard) Huffman tables out"""
    p = jpeg.find(b"\xff\xc4")
    n = int.from_bytes(jpeg[p + 2:p + 4], "big")
    return jpeg[:p] + jpeg[p + 2 + n:]


def test_cli_gpu_decode_refuses_sources_without_jpeg_files():
    for extra in (["--synthetic", "4"], []):   # no --video / --image_dir: the camera
        r = subprocess.run([BIN, "--gpu_decode", "--model", "COCO", "--resolution", "64x48"] + extra, capture_output=True, text=True, timeout=60)
        assert r.returncode == 1 and "--gpu_decode reconstructs JPEG files on the GPU: it needs --image_dir or a Motion-JPEG --video" in r.stderr, r.stderr
    r = subprocess.run([BIN, "--help"], capture_output=True, text=True, timeout=60)
    assert '--gpu_decode (' in r.stdout and 'default: "false"' in r.stdout.split("--gpu_decode (")[1].split("\n")[0]


def test_cli_gpu_decode_producer_stage_without_gpu(tmp_path):
    """--decode_bench --gpu_decode: the producers run only the entropy stage for .jpg files and Motion-JPEG frames; other files,
    and JPEGs the coefficient stage refuses, take the host decoder; the frame accounting is the same as without the flag"""
    from caffe_rtpose_b200 import synth
    d = tmp_path / "imgs"
    d.mkdir()
    for i in range(8):
        (d / ("f%02d.jpg" % i)).write_bytes(engine.encode_jpeg(synth.make_frame(i, 48, 64), 90))
    (d / "f08.jpg").write_bytes(b"\xff\xd8 not a jpeg")
    (d / "f09.ppm").write_bytes(b"P6\n64 48\n255\n" + synth.make_frame(9, 48, 64).tobytes())
    avi = str(tmp_path / "clip.avi")
    write_mjpeg_avi(avi, [strip_dht(engine.encode_jpeg(synth.make_frame(20 + i, 48, 64), 90)) for i in range(6)], 64, 48)
    for src in (["--image_dir", str(d)], ["--video", avi, "--novideo_realtime"]):
        outs = []
        for flag in ([], ["--gpu_decode"]):
            r = subprocess.run([BIN] + src + ["--decode_bench", "--num_producers", "3", "--model", "COCO", "--resolution", "64x48"] + flag,
                               capture_output=True, text=True, timeout=120)
            assert r.returncode == 0, r.stderr
            outs.append(r.stdout.strip().splitlines()[-1].split(" in ")[0])
        assert outs[0] == outs[1], outs
        assert outs[0].startswith("decoded %d frames" % (9 if src[0] == "--image_dir" else 6)), outs
