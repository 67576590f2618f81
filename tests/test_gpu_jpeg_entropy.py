"""GPU entropy decoding (pe_jpeg_decode_scans, pe_forward_jpeg_scans / PoseEngine.forward_jpeg(entropy="gpu")): the host only parses
the file into a scan image, the GPU decodes the Huffman data.  The device coefficient images must equal pe_jpeg_read_coefs's bit for
bit, the frames decode_jpeg's, and maps, peaks and joints those of the host entropy route and of host decoding plus upload.  Frames
are read back as in test_gpu_jpeg.py: pe_render's uint8 output with person assembly switched off."""
import ctypes as C

import numpy as np
import pytest

from caffe_rtpose_b200 import engine, synth
from test_gpu_jpeg import _results, _same, camera_jpeg, make_engine, no_people, shown_frame, with_route
from test_jpeg_scan import SUBSEQ, all_fixtures, coefs_full_rc, corrupt_streams, dc_category_error, is_progressive, read_scan_rc, scan_fixtures


def _decode(e, jpegs, S):
    scans = [engine.read_jpeg_scan(j) for j in jpegs]
    return e.decode_jpeg_scans(scans, S)


@pytest.mark.gpu
def test_device_coefficients_equal_read_coefs_on_every_fixture():
    e = make_engine(64, 48)
    checked = 0
    for name, data in all_fixtures().items():
        if is_progressive(data):
            continue
        ref = engine.read_jpeg_coefs(data)
        for S in SUBSEQ:
            outs, st = _decode(e, [data], S)
            assert st == [0] and np.array_equal(outs[0], ref), (name, S, int((outs[0] != ref).sum()))
            checked += 1
    assert checked >= 4 * 40
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(1280, 720), (1920, 1080)], ids=["720p", "1080p"])
def test_device_coefficients_at_camera_sizes_in_batches(size):
    """batches of 1 and 9 frames whose entropy-coded lengths differ widely (quality 10 .. 98)"""
    w, h = size
    e = make_engine(64, 48, max_batch=9)
    jpegs = [camera_jpeg(40 + i, h, w, q) for i, q in enumerate((98, 10, 85, 50, 95, 20, 90, 70, 98))]
    refs = [engine.read_jpeg_coefs(j) for j in jpegs]
    for S in SUBSEQ:
        for batch in ([0], list(range(9))):
            outs, st = _decode(e, [jpegs[i] for i in batch], S)
            assert st == [0] * len(batch)
            for o, i in zip(outs, batch):
                assert np.array_equal(o, refs[i]), (S, i)
    e.close()


@pytest.mark.gpu
def test_device_decoder_on_corrupt_streams():
    """the status is flagged exactly where pe_jpeg_read_coefs rejects the data; everything else is bit-identical"""
    e = make_engine(64, 48, max_batch=4)
    flagged = decoded = 0
    for d in corrupt_streams():
        crc, ref = coefs_full_rc(d)
        src, scan = read_scan_rc(d)
        if src < 0:
            continue
        for S in (32, 1024):
            outs, st = e.decode_jpeg_scans([scan], S)
            assert (st[0] == 0) == (crc > 0), (S, crc, st)
            if crc > 0:
                assert np.array_equal(outs[0], ref), S
        flagged += crc < 0
        decoded += crc > 0
    assert flagged and decoded
    e.close()


@pytest.mark.gpu
def test_forward_jpeg_gpu_entropy_shows_decode_jpeg_frames():
    files = scan_fixtures()
    by_size = {}
    for name, data in files.items():
        h, w, _ = engine.decode_jpeg(data).shape
        by_size.setdefault((w, h), []).append(name)
    for (w, h), names in sorted(by_size.items()):
        for disp in ((w, h), (320, 192)):   # display size, and through the warp
            e = make_engine(*disp)
            no_people(e)
            for name in names:
                ref = engine.decode_jpeg(files[name])
                scale = e.forward_jpeg([files[name]], entropy="gpu")
                got = shown_frame(e)
                assert scale == e.forward_jpeg([files[name]])
                if disp == (w, h):
                    assert scale == 1.0
                    assert np.array_equal(got, ref), name
                assert np.array_equal(got, shown_frame(e)), name
            e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", [engine.PREC_F16X2, engine.PREC_F16X1], ids=["parity", "fast"])
def test_forward_jpeg_gpu_entropy_equals_host_routes(precision):
    """maps, peaks and joints of entropy="gpu" against entropy="host" and host decode + upload, for 1 and 9 frames, three calls each
    (the third replays a CUDA graph)"""
    disp_w, disp_h = 320, 192
    a = make_engine(disp_w, disp_h, 160, 96, precision=precision, max_batch=9)
    b = make_engine(disp_w, disp_h, 160, 96, precision=precision, max_batch=9)
    c = make_engine(disp_w, disp_h, 160, 96, precision=precision, max_batch=9)
    seed = 500
    for (w, h) in ((disp_w, disp_h), (1280, 720)):
        for n in (1, 9):
            for call in range(3):
                jpegs = [camera_jpeg(seed + i, h, w, (98, 85, 60)[i % 3]) for i in range(n)]
                seed += n
                s_a = a.forward_jpeg(jpegs, entropy="gpu")
                s_b = b.forward_jpeg(jpegs, entropy="host")
                frames = [engine.decode_jpeg(j) for j in jpegs]
                if (w, h) == (disp_w, disp_h):
                    c.forward_frames(frames)
                    s_c = 1.0
                else:
                    s_c = c.forward_camera_frames(frames)
                assert s_a == s_b == s_c
                ra = _results(a, n)
                _same(ra, _results(b, n))
                _same(ra, _results(c, n))
                for i in range(n):
                    assert np.array_equal(a.render(i, 0), b.render(i, 0)), (w, h, n, call, i)
    for x in (a, b, c):
        x.close()


@pytest.mark.gpu
def test_forward_jpeg_scans_from_pinned_buffers():
    jpegs = [camera_jpeg(600 + i, 192, 320, q) for i, q in enumerate((95, 70, 98))]
    e = make_engine(320, 192, 160, 96, max_batch=3)
    L = engine.lib()
    scans = [engine.read_jpeg_scan(j) for j in jpegs]
    pinned = []
    for s in scans:
        p = L.pe_host_alloc(s.size)
        assert p
        C.memmove(p, s.ctypes.data, s.size)
        pinned.append(p)
    try:
        ptrs = (C.c_void_p * 3)(*pinned)
        sc = C.c_double()
        assert L.pe_forward_jpeg_scans(e._h, ptrs, 3, C.byref(sc)) == 0 and sc.value == 1.0
        got = _results(e, 3)
        e.forward_jpeg(scans, entropy="gpu")
        _same(got, _results(e, 3))
        e.forward_jpeg(jpegs)
        _same(got, _results(e, 3))
    finally:
        for p in pinned:
            L.pe_host_free(p)
    e.close()


@pytest.mark.gpu
def test_bad_frame_in_a_batch():
    """a frame with a DC category above 15: pe_fetch gives PE_ERR_IO for it alone, the other frames' results are unchanged"""
    jpegs = [camera_jpeg(700 + i, 192, 320, 90) for i in range(4)]
    bad = dc_category_error(jpegs[2], 2)
    assert coefs_full_rc(bad)[0] == -1 and read_scan_rc(bad)[0] > 0
    e = make_engine(320, 192, 160, 96, max_batch=4)
    e.forward_jpeg(jpegs, entropy="gpu")
    good = [e.fetch(i) for i in range(4)]
    e.forward_jpeg(jpegs[:2] + [bad] + jpegs[3:], entropy="gpu")
    for i in (0, 1, 3):
        _same(list(e.fetch(i)), list(good[i]))
    with pytest.raises(engine.PoseEngineError, match=r"error 4: frame 2: corrupt JPEG data \(DC category above 15\) in MCU \d+"):
        e.fetch(2)
    e.forward_jpeg(jpegs, entropy="gpu")   # the next forward has no error
    _same(list(e.fetch(2)), list(good[2]))
    e.close()


@pytest.mark.gpu
def test_forward_jpeg_scans_refuses_bad_batches():
    files = scan_fixtures()
    e = make_engine(160, 120, max_batch=2)
    with pytest.raises(engine.PoseEngineError, match="one size per call"):
        e.forward_jpeg([files["420_restart7"], files["422_q50"]], entropy="gpu")
    bad = engine.read_jpeg_scan(files["420_restart7"])
    bad[512] ^= 0xFF
    with pytest.raises(engine.PoseEngineError, match="not a pe_jpeg_read_scan image"):
        e.forward_jpeg([bad], entropy="gpu")
    bad = engine.read_jpeg_scan(files["420_restart7"])
    bad[2784 + 16 + 8] += 1   # segment 1 longer than the data
    bad[2784 + 16 + 12] = 0x40
    with pytest.raises(engine.PoseEngineError, match="not a pe_jpeg_read_scan image"):
        e.forward_jpeg([bad], entropy="gpu")
    e.forward_jpeg([files["420_restart7"]], entropy="gpu")   # the handle still works
    e.close()


@pytest.mark.gpu
def test_cli_gpu_entropy_writes_the_same_files(tmp_path):
    """rtpose.bin --gpu_entropy (2 handles on one GPU, 3 producers, 3 frames per forward) writes the JSON files and rendered frames
    of the host decoder: an --image_dir mixing sequential, progressive and other-size JPEGs with a .ppm, an unreadable file and a file
    whose data has a DC category above 15 (dropped by both), and a Motion-JPEG --video whose frame 5 has such data (dropped by both, as
    the producers are several)"""
    from test_gpu_jpeg import _run_cli
    from test_jpeg_coefs import fixtures as coef_fixtures, strip_dht, write_mjpeg_avi
    d = tmp_path / "imgs"
    d.mkdir()
    for i in range(9):
        h, w = (192, 320) if i % 3 else (237, 421)
        (d / ("f%02d.jpg" % i)).write_bytes(camera_jpeg(800 + i, h, w, 95))
    (d / "f09.jpg").write_bytes(coef_fixtures()["420_83x61_progressive"])
    (d / "f10.jpg").write_bytes(dc_category_error(camera_jpeg(810, 192, 320, 95), 3))
    (d / "f11.ppm").write_bytes(b"P6\n320 192\n255\n" + synth.make_frame(811, 192, 320)[:, :, ::-1].tobytes())
    (d / "f12.jpg").write_bytes(b"\xff\xd8 not a jpeg")
    frames = [strip_dht(camera_jpeg(900 + i, 270, 480, 90)) for i in range(8)]
    frames[5] = dc_category_error(camera_jpeg(905, 270, 480, 90), 3)   # (this frame keeps its DHT, which carries the error)
    avi = str(tmp_path / "clip.avi")
    write_mjpeg_avi(avi, frames, 480, 270)
    for src, n in ((["--image_dir", str(d)], 11), (["--video", avi, "--novideo_realtime"], 7)):
        runs = []
        for k, flag in enumerate(([], ["--gpu_entropy"])):
            out = tmp_path / ("%s_%d" % (src[0][2:], k))
            out.mkdir()
            runs.append(_run_cli(src, out, flag))
        assert len(runs[0][0]) == n and len(runs[0][1]) == n, (len(runs[0][0]), n)
        assert runs[0] == runs[1]
