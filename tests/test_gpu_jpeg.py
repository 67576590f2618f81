"""GPU JPEG reconstruction (pe_forward_jpeg_coefs / PoseEngine.forward_jpeg): the host decodes only the entropy stage, the GPU
dequantises, inverse-transforms, upsamples and converts colour.  The frame it builds must be bit-identical to pe_decode_jpeg's, and
everything downstream (maps, peaks, joints) identical to decoding on the host and uploading the pixels.

The reconstructed frame is read back through pe_render's uint8 output of the frame the last forward used: with person assembly
switched off (min_subset_cnt above any possible count) nothing is drawn on it, so the image is the device frame buffer itself."""
import ctypes as C
import os

import numpy as np
import pytest

from caffe_rtpose_b200 import engine, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = os.path.join(ROOT, "tests", "golden", "jpeg_coefs.npz")
_WEIGHTS = {}


def weights():
    if not _WEIGHTS:
        _WEIGHTS["w"] = synth.make_weights(engine.COCO_18, "he")
    return _WEIGHTS["w"]


def make_engine(disp_w, disp_h, net_w=64, net_h=48, precision=engine.PREC_F16X2, max_batch=1):
    e = engine.PoseEngine(engine.COCO_18, net_w, net_h, disp_w, disp_h, precision=precision, max_batch=max_batch)
    e.set_weights(weights())
    return e


def no_people(e):
    e.set_connect_params(1 << 30, 1e30, 0.05, 9)


def shown_frame(e, idx=0):
    return e.render(idx, 0)


def fixtures():
    z = np.load(FIXTURES)
    return {k: z[k].tobytes() for k in z.files}


def with_route(fast, fn):
    old = os.environ.get("PE_JPEG_FAST")
    os.environ["PE_JPEG_FAST"] = "1" if fast else "0"
    try:
        return fn()
    finally:
        if old is None:
            del os.environ["PE_JPEG_FAST"]
        else:
            os.environ["PE_JPEG_FAST"] = old


def camera_jpeg(seed, h, w, quality=98):
    """a camera-like frame (smooth content + noise) through the project's own baseline 4:2:0 encoder"""
    return engine.encode_jpeg(synth.make_frame(seed, h, w), quality)


@pytest.mark.gpu
def test_gpu_reconstruction_is_bit_identical_on_every_fixture():
    by_size = {}
    for name, data in fixtures().items():
        h, w, _ = engine.decode_jpeg(data).shape
        by_size.setdefault((w, h), []).append(name)
    files = fixtures()
    checked = 0
    for (w, h), names in sorted(by_size.items()):
        e = make_engine(w, h)
        no_people(e)
        ref0 = engine.decode_jpeg(files[names[0]])
        e.forward_frames([ref0])   # the read-back itself: a host-decoded frame comes back unchanged
        assert e.fetch(0)[0] == 0 and np.array_equal(shown_frame(e), ref0)
        for name in names:
            ref = engine.decode_jpeg(files[name])
            for fast in (True, False):
                scale = with_route(fast, lambda: e.forward_jpeg([files[name]]))
                assert scale == 1.0
                got = shown_frame(e)
                assert np.array_equal(got, ref), (name, fast, int((got != ref).any(2).sum()))
                checked += 1
        e.close()
    assert checked == 2 * len(files)


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(1280, 720), (1920, 1080)], ids=["720p", "1080p"])
def test_gpu_reconstruction_is_bit_identical_at_camera_sizes(size):
    w, h = size
    e = make_engine(w, h, 160, 96, max_batch=3)
    no_people(e)
    jpegs = [camera_jpeg(s, h, w, q) for s, q in ((11, 98), (12, 90), (13, 75))]
    refs = [engine.decode_jpeg(j) for j in jpegs]
    assert e.forward_jpeg(jpegs) == 1.0
    for i, ref in enumerate(refs):
        got = shown_frame(e, i)
        assert np.array_equal(got, ref), (i, int((got != ref).any(2).sum()))
    e.close()


def _results(e, n):
    out = [e.fetch_maps(n)]
    for i in range(n):
        cnt, joints, peaks = e.fetch(i)
        out += [cnt, joints, peaks]
    return out


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        if isinstance(x, np.ndarray):
            assert x.shape == y.shape and np.array_equal(x, y)
        else:
            assert x == y


@pytest.mark.gpu
@pytest.mark.parametrize("precision", [engine.PREC_F16X2, engine.PREC_F16X1], ids=["parity", "fast"])
def test_forward_jpeg_equals_host_decode_and_upload(precision):
    """maps, peaks and joints of forward_jpeg against pe_decode_jpeg + forward_frames (display size) and + forward_camera_frames
    (other sizes: the GPU warpAffine, frame.scale), for 1 and 9 frames; three calls each, the third replaying a CUDA graph"""
    disp_w, disp_h = 320, 192
    a = make_engine(disp_w, disp_h, 160, 96, precision=precision, max_batch=9)
    b = make_engine(disp_w, disp_h, 160, 96, precision=precision, max_batch=9)
    seed = 100
    for (w, h) in ((disp_w, disp_h), (421, 237), (1280, 720)):
        for n in (1, 9):
            for call in range(3):
                jpegs = [camera_jpeg(seed + i, h, w, 95) for i in range(n)]
                seed += n
                frames = [engine.decode_jpeg(j) for j in jpegs]
                s_a = a.forward_jpeg(jpegs)
                if (w, h) == (disp_w, disp_h):
                    b.forward_frames(frames)
                    s_b = 1.0
                else:
                    s_b = b.forward_camera_frames(frames)
                assert s_a == s_b, (w, h, n, call)
                _same(_results(a, n), _results(b, n))
                for i in range(n):   # the frame pe_render draws on is the reconstructed (and warped) one
                    assert np.array_equal(a.render(i, 0), b.render(i, 0)), (w, h, n, call, i)
    a.close()
    b.close()


@pytest.mark.gpu
def test_forward_jpeg_from_pinned_buffers_and_mixed_sampling():
    """coefficient images in pe_host_alloc memory (asynchronous DMA) give the same results as pageable ones; the frames of one
    call may differ in chroma sampling and quantisation tables as long as they share the size"""
    files = fixtures()
    names = ["444_83x61", "422_83x61", "420_83x61_progressive", "420_83x61"]
    e = make_engine(83, 61, max_batch=4)
    no_people(e)
    L = engine.lib()
    bufs = [engine.read_jpeg_coefs(files[k]) for k in names]
    pinned = []
    for b in bufs:
        p = L.pe_host_alloc(b.size)
        assert p
        C.memmove(p, b.ctypes.data, b.size)
        pinned.append(p)
    try:
        ptrs = (C.c_void_p * len(pinned))(*pinned)
        s = C.c_double()
        assert L.pe_forward_jpeg_coefs(e._h, ptrs, len(pinned), C.byref(s)) == 0 and s.value == 1.0
        for i, k in enumerate(names):
            assert np.array_equal(shown_frame(e, i), engine.decode_jpeg(files[k])), k
        maps = e.fetch_maps(4)
        e.forward_jpeg(bufs)
        assert np.array_equal(maps, e.fetch_maps(4))
    finally:
        for p in pinned:
            L.pe_host_free(p)
    e.close()


@pytest.mark.gpu
def test_forward_jpeg_refuses_bad_batches():
    files = fixtures()
    e = make_engine(83, 61, max_batch=2)
    with pytest.raises(engine.PoseEngineError, match="one size per call"):
        e.forward_jpeg([files["420_83x61"], files["420_64x48"]])
    bad = engine.read_jpeg_coefs(files["420_83x61"])
    bad[0] ^= 0xFF
    with pytest.raises(engine.PoseEngineError, match="not a pe_jpeg_read_coefs header"):
        e.forward_jpeg([bad])
    bad = engine.read_jpeg_coefs(files["420_83x61"])
    bad[32 + 8] += 1   # luma block grid wider than the frame header implies
    with pytest.raises(engine.PoseEngineError, match="not a pe_jpeg_read_coefs header"):
        e.forward_jpeg([bad])
    with pytest.raises(engine.PoseEngineError, match="outside"):
        e.forward_jpeg([files["420_83x61"]] * 3)
    e.forward_jpeg([files["420_83x61"]])   # the handle still works
    e.close()


BIN = os.path.join(ROOT, "caffe_rtpose_b200", "rtpose.bin")


def _run_cli(src, out, extra):
    import subprocess
    args = [BIN] + src + ["--model", "COCO", "--caffeproto", "/nonexistent.prototxt", "--random_init", "he", "--resolution", "320x192",
                          "--net_resolution", "160x96", "--write_json", str(out / "json"), "--write_frames", str(out / "frames"),
                          "--frame_format", "bmp", "--no_display", "--no_frame_drops", "--num_gpu", "1", "--engines_per_gpu", "2",
                          "--num_producers", "3", "--batch", "3"] + extra
    r = subprocess.run(args, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return {p: (out / "json" / p).read_bytes() for p in sorted(os.listdir(out / "json"))}, \
        {p: (out / "frames" / p).read_bytes() for p in sorted(os.listdir(out / "frames"))}


@pytest.mark.gpu
def test_cli_gpu_decode_writes_the_same_files(tmp_path):
    """rtpose.bin --gpu_decode (2 handles on one GPU, 3 producers, 3 frames per forward): the JSON files and the rendered frames equal
    those of the host decoder, for an --image_dir that mixes display-size and other-size JPEGs with a .ppm and an undecodable file,
    and for a Motion-JPEG --video (frames without their DHT segment, warped to the display size)"""
    from test_jpeg_coefs import strip_dht, write_mjpeg_avi
    d = tmp_path / "imgs"
    d.mkdir()
    for i in range(10):
        h, w = (192, 320) if i % 3 else (237, 421)
        (d / ("f%02d.jpg" % i)).write_bytes(camera_jpeg(200 + i, h, w, 95))
    (d / "f10.ppm").write_bytes(b"P6\n320 192\n255\n" + synth.make_frame(210, 192, 320)[:, :, ::-1].tobytes())
    (d / "f11.jpg").write_bytes(b"\xff\xd8 not a jpeg")
    avi = str(tmp_path / "clip.avi")
    write_mjpeg_avi(avi, [strip_dht(camera_jpeg(300 + i, 270, 480, 90)) for i in range(7)], 480, 270)
    for src, n in ((["--image_dir", str(d)], 11), (["--video", avi, "--novideo_realtime"], 7)):
        runs = []
        for k, flag in enumerate(([], ["--gpu_decode"])):
            out = tmp_path / ("%s_%d" % (src[0][2:], k))
            out.mkdir()
            runs.append(_run_cli(src, out, flag))
        assert len(runs[0][0]) == n and len(runs[0][1]) == n
        assert runs[0] == runs[1]
