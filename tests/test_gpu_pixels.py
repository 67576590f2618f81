"""pe_forward_pixels / PoseEngine.forward_pixels on the GPU: decoder-format frames (NV12, I420, YUYV, RGB, BGR) in pageable, page-locked
or device memory, converted on the GPU.  Everything the forward produces - maps, peaks, people, joints, frame.scale and pe_render's
canvas and image of the converted display frame - must equal pe_forward_camera_frames on cv2.cvtColor of the same frame, a route
pinned to cv2's warpAffine.  Also: an NVDEC-shaped surface (pitch 2048, chroma after 1088 rows, 0xEE padding), batches of separate
allocations across CUDA-graph replays, and ordering after unfinished work on torch's current stream."""
import ctypes as C

import cv2
import numpy as np
import pytest
import torch

from caffe_rtpose_b200 import engine, synth

pytestmark = pytest.mark.gpu

NET_W, NET_H, DISP_W, DISP_H = 160, 96, 1280, 720
SIZES = [(1280, 720), (1920, 1080), (640, 360), (480, 848)]   # display size, 1080p, smaller, portrait
FORMATS = [engine.PIX_NV12, engine.PIX_I420, engine.PIX_YUYV, engine.PIX_RGB, engine.PIX_BGR]
_CACHE = {}


def weights():
    if "w" not in _CACHE:
        _CACHE["w"] = synth.make_weights(engine.COCO_18, "he")
    return _CACHE["w"]


def make_engine(max_batch=1):
    e = engine.PoseEngine(engine.COCO_18, NET_W, NET_H, DISP_W, DISP_H, precision=engine.PREC_F16X2, max_batch=max_batch)
    e.set_weights(weights())
    return e


def to_format(bgr, fmt):
    """a decoder frame with camera-like content: the BGR frame in fmt (cv2's layouts)"""
    h, w, _ = bgr.shape
    if fmt == engine.PIX_BGR:
        return bgr.copy()
    if fmt == engine.PIX_RGB:
        return cv2.cvtColor(bgr, cv2.COLOR_BGR2RGB)
    i420 = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420)
    if fmt == engine.PIX_I420:
        return i420
    u = i420[h:h + h // 4].reshape(h // 2, w // 2)
    v = i420[h + h // 4:].reshape(h // 2, w // 2)
    if fmt == engine.PIX_NV12:
        return np.concatenate([i420[:h], np.stack([u, v], -1).reshape(h // 2, w)])
    out = np.empty((h, w, 2), np.uint8)   # YUYV: Y0 U Y1 V, chroma of the row pair
    out[..., 0] = i420[:h]
    out[:, 0::2, 1] = np.repeat(u, 2, 0)
    out[:, 1::2, 1] = np.repeat(v, 2, 0)
    return out


def frame_of(fmt, w, h, seed):
    return to_format(synth.make_frame(seed, h, w), fmt)


class Pinned:
    """a pe_host_alloc buffer seen as a numpy array"""
    def __init__(self, a):
        self.p = engine.lib().pe_host_alloc(a.nbytes)
        assert self.p
        self.arr = np.ctypeslib.as_array((C.c_uint8 * a.nbytes).from_address(self.p)).reshape(a.shape)
        self.arr[...] = a

    def free(self):
        engine.lib().pe_host_free(self.p)


def results(e, n=1, render=True):
    out = {"maps": e.fetch_maps(n)}
    for i in range(n):
        out["fetch%d" % i] = e.fetch(i)
        if render:
            img, canvas = e.render(i, 0, want_canvas=True)
            out["img%d" % i], out["canvas%d" % i] = img, canvas
    return out


def assert_same(a, b, tag):
    assert a.keys() == b.keys()
    for k in a:
        if k.startswith("fetch"):
            assert a[k][0] == b[k][0], (tag, k, "people")
            assert np.array_equal(a[k][1], b[k][1]) and np.array_equal(a[k][2], b[k][2]), (tag, k)
        else:
            assert np.array_equal(a[k], b[k]), (tag, k)


@pytest.mark.parametrize("w,h", SIZES)
def test_same_results_as_camera_route(w, h):
    e = make_engine()
    for fmt in FORMATS:
        frame = frame_of(fmt, w, h, seed=w + fmt)
        bgr = engine.pixels_to_bgr(frame, fmt)
        assert fmt == engine.PIX_BGR or np.array_equal(bgr, cv2.cvtColor(frame, {
            engine.PIX_NV12: cv2.COLOR_YUV2BGR_NV12, engine.PIX_I420: cv2.COLOR_YUV2BGR_I420,
            engine.PIX_YUYV: cv2.COLOR_YUV2BGR_YUYV, engine.PIX_RGB: cv2.COLOR_RGB2BGR}[fmt]))
        want_scale = e.forward_camera_frames([bgr])
        want = results(e)
        pinned = Pinned(frame)
        try:
            for kind, src in (("pageable", frame), ("pinned", pinned.arr), ("cuda", torch.from_numpy(frame).cuda())):
                scale = e.forward_pixels([src], fmt)
                assert scale == want_scale, (fmt, kind)
                assert_same(results(e), want, (fmt, kind, w, h))
        finally:
            e.sync()
            pinned.free()
    e.close()


def test_nvdec_shaped_surface():
    """NVDEC's 1080p NV12 surface: rows 2048 bytes apart, chroma after the 1088-row aligned height, padding all 0xEE"""
    w, h, pitch, aligned = 1920, 1080, 2048, 1088
    tight = frame_of(engine.PIX_NV12, w, h, seed=3)
    surf = torch.full((aligned + aligned // 2, pitch), 0xEE, dtype=torch.uint8, device="cuda")
    surf[:h, :w] = torch.from_numpy(tight[:h]).cuda()
    surf[aligned:aligned + h // 2, :w] = torch.from_numpy(tight[h:]).cuda()
    e = make_engine()
    want_scale = e.forward_pixels([tight], engine.PIX_NV12)
    want = results(e)
    scale = e.forward_pixels([surf[:h, :w]], engine.PIX_NV12, chroma_offset=pitch * aligned)
    assert scale == want_scale
    assert_same(results(e), want, "nvdec")
    # an I420 surface of FFmpeg's kind: chroma rows pitch/2 apart after the luma plane
    i420 = frame_of(engine.PIX_I420, w, h, seed=4)
    buf = torch.full((pitch * aligned * 3 // 2,), 0xEE, dtype=torch.uint8, device="cuda")
    buf[:pitch * aligned].view(aligned, pitch)[:h, :w] = torch.from_numpy(i420[:h]).cuda()
    chroma = torch.from_numpy(i420[h:].reshape(-1)).cuda().view(h, w // 2)   # U rows then V rows, w/2 bytes each
    cbase = pitch * aligned
    buf[cbase:cbase + (pitch // 2) * h].view(h, pitch // 2)[:, :w // 2] = chroma
    e.forward_pixels([i420], engine.PIX_I420)
    want = results(e)
    e.forward_pixels([buf[:pitch * h].view(h, pitch)[:, :w]], engine.PIX_I420, chroma_offset=cbase)
    assert_same(results(e), want, "i420 surface")
    e.close()


def test_batches_and_graph_replays():
    """max_batch frames from separate allocations, three calls (eager, capture, replay): identical to frame-by-frame calls; one
    batch mixes device, page-locked and pageable frames"""
    B = 4
    e = make_engine(max_batch=B)
    one = make_engine()
    frames = [frame_of(engine.PIX_NV12, 1920, 1080, seed=10 + i) for i in range(B)]
    singles = []
    for f in frames:
        one.forward_pixels([f], engine.PIX_NV12)
        singles.append(results(one, render=False))
    dev = [torch.from_numpy(f).cuda() for f in frames]
    for call in range(3):
        e.forward_pixels(dev, engine.PIX_NV12)
        maps = e.fetch_maps(B)
        for i in range(B):
            assert np.array_equal(maps[i:i + 1], singles[i]["maps"]), (call, i)
            got = e.fetch(i)
            assert got[0] == singles[i]["fetch0"][0] and np.array_equal(got[1], singles[i]["fetch0"][1]), (call, i)
            assert np.array_equal(got[2], singles[i]["fetch0"][2]), (call, i)
    pinned = Pinned(frames[1])
    try:
        e.forward_pixels([dev[0], pinned.arr, frames[2], dev[3]], engine.PIX_NV12)
        maps = e.fetch_maps(B)
    finally:
        pinned.free()
    for i in range(B):
        assert np.array_equal(maps[i:i + 1], singles[i]["maps"]), ("mixed", i)
    e.close()
    one.close()


def test_waits_for_torch_stream():
    """the frame is written on torch's current stream behind a long sleep; forward_pixels is called without synchronising"""
    frame = frame_of(engine.PIX_NV12, 1920, 1080, seed=21)
    e = make_engine()
    e.forward_pixels([frame], engine.PIX_NV12)
    want = results(e)
    src = torch.from_numpy(frame).cuda()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        dst = torch.zeros_like(src)
        torch.cuda._sleep(1 << 28)   # ~0.15 s of device time before the write
        dst.copy_(src)
        e.forward_pixels([dst], engine.PIX_NV12)
    assert_same(results(e), want, "stream order")
    e.close()


def test_refusals_launch_nothing():
    e = make_engine()
    L = engine.lib()
    frame = torch.zeros((1620, 1920), dtype=torch.uint8, device="cuda")
    ptrs = (C.c_void_p * 1)(frame.data_ptr())
    s = C.c_double()
    before = L.pe_launch_count(e._h)
    for pf, words in ((engine._PixelFormat(7, 1920, 1080, 0, 0), "pixel format"),
                      (engine._PixelFormat(engine.PIX_NV12, 1919, 1080, 0, 0), "odd width"),
                      (engine._PixelFormat(engine.PIX_NV12, 1920, 1080, 1918, 0), "pitch"),
                      (engine._PixelFormat(engine.PIX_NV12, 1920, 1080, 0, 1920 * 1079), "chroma_offset")):
        assert L.pe_forward_pixels(e._h, C.byref(pf), ptrs, 1, C.byref(s)) == 1
        assert words in L.pe_last_error(e._h).decode()
    pf = engine._PixelFormat(engine.PIX_NV12, 1920, 1080, 0, 0)
    assert L.pe_forward_pixels(e._h, C.byref(pf), (C.c_void_p * 1)(None), 1, C.byref(s)) == 1
    assert "null frame 0" in L.pe_last_error(e._h).decode()
    assert L.pe_forward_pixels(e._h, C.byref(pf), ptrs, 2, C.byref(s)) == 1   # n above max_batch
    assert L.pe_launch_count(e._h) == before
    if torch.cuda.device_count() > 1:
        other = torch.zeros((1620, 1920), dtype=torch.uint8, device="cuda:1")
        assert L.pe_forward_pixels(e._h, C.byref(pf), (C.c_void_p * 1)(other.data_ptr()), 1, C.byref(s)) == 1
        assert "GPU 1" in L.pe_last_error(e._h).decode()
    e.close()
