"""pe_forward_pixels on the GPU with the formats beyond NV12 / I420 / YUYV / RGB (NV21, YV12, UYVY, P016, planar RGB) and the colour
flags (BT.709, full range) on every YUV format, from device, page-locked and pageable memory, at the display size and another size.
Everything the forward produces - maps, peaks, people, joints, frame.scale and pe_render's canvas and image of the converted display
frame - must equal pe_forward_camera_frames on pe_pixels_to_bgr of the same frame (the host reference, pinned to cv2 and float64 in
test_pixel_formats.py).  Also: an NVDEC-shaped 1080p P016 surface, a planar RGB CUDA tensor sliced from a larger allocation and
read in place, mixed batches across CUDA-graph replays, and refusals that launch nothing."""
import ctypes as C

import cv2
import numpy as np
import pytest
import torch

from caffe_rtpose_b200 import engine, synth
from test_gpu_pixels import assert_same, make_engine, results

pytestmark = pytest.mark.gpu

SIZES = [(1280, 720), (1920, 1080)]   # the display size, and a size that is warped
YUV = [engine.PIX_NV12, engine.PIX_I420, engine.PIX_YUYV, engine.PIX_NV21, engine.PIX_YV12, engine.PIX_UYVY, engine.PIX_P016]
COLOURS = [("bt601", False), ("bt601", True), ("bt709", False), ("bt709", True)]
CASES = [(f, m, fr) for f in YUV for m, fr in COLOURS] + [(engine.PIX_RGBP, "bt601", False)]


def to_format(bgr, fmt, seed=0):
    """a decoder frame with camera-like content: the BGR frame in fmt (cv2's layouts; P016 with random low bytes)"""
    h, w, _ = bgr.shape
    if fmt == engine.PIX_RGBP:
        return np.ascontiguousarray(cv2.cvtColor(bgr, cv2.COLOR_BGR2RGB).transpose(2, 0, 1))
    i420 = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420)
    u = i420[h:h + h // 4].reshape(h // 2, w // 2)
    v = i420[h + h // 4:].reshape(h // 2, w // 2)
    if fmt == engine.PIX_I420:
        return i420
    if fmt == engine.PIX_YV12:
        return np.concatenate([i420[:h].reshape(-1), v.reshape(-1), u.reshape(-1)]).reshape(h * 3 // 2, w)
    if fmt in (engine.PIX_NV12, engine.PIX_NV21, engine.PIX_P016):
        uv = np.stack([v, u] if fmt == engine.PIX_NV21 else [u, v], -1).reshape(h // 2, w)
        f = np.concatenate([i420[:h], uv])
        if fmt == engine.PIX_P016:
            f = (f.astype(np.uint16) << 8) | np.random.default_rng(seed).integers(0, 256, f.shape, dtype=np.uint16)
        return f
    out = np.empty((h, w, 2), np.uint8)   # YUYV: Y0 U Y1 V, chroma of the row pair
    out[..., 0] = i420[:h]
    out[:, 0::2, 1] = np.repeat(u, 2, 0)
    out[:, 1::2, 1] = np.repeat(v, 2, 0)
    return out[..., ::-1].copy() if fmt == engine.PIX_UYVY else out


def frame_of(fmt, w, h, seed):
    return to_format(synth.make_frame(seed, h, w), fmt, seed)


class Pinned:
    """a pe_host_alloc buffer seen as a numpy array of a's dtype and shape"""
    def __init__(self, a):
        self.p = engine.lib().pe_host_alloc(a.nbytes)
        assert self.p
        self.arr = np.ctypeslib.as_array((C.c_uint8 * a.nbytes).from_address(self.p)).view(a.dtype).reshape(a.shape)
        self.arr[...] = a

    def free(self):
        engine.lib().pe_host_free(self.p)


@pytest.mark.parametrize("w,h", SIZES)
def test_same_results_as_camera_route(w, h):
    e = make_engine()
    for fmt, matrix, full in CASES:
        tag = (fmt, matrix, full, w, h)
        frame = frame_of(fmt, w, h, seed=w + fmt)
        bgr = engine.pixels_to_bgr(frame, fmt, matrix=matrix, full_range=full)
        want_scale = e.forward_camera_frames([bgr])
        want = results(e)
        pinned = Pinned(frame)
        try:
            for kind, src in (("pageable", frame), ("pinned", pinned.arr), ("cuda", torch.from_numpy(frame).cuda())):
                scale = e.forward_pixels([src], fmt, matrix=matrix, full_range=full)
                assert scale == want_scale, (tag, kind)
                assert_same(results(e), want, (tag, kind))
        finally:
            e.sync()
            pinned.free()
    e.close()


def test_nvdec_shaped_p016_surface():
    """NVDEC's 1080p P016 surface: rows 4096 bytes apart, chroma after the 1088-row aligned height, padding all 0xEEEE"""
    w, h, pitch_el, aligned = 1920, 1080, 2048, 1088
    tight = frame_of(engine.PIX_P016, w, h, seed=3)
    surf = torch.full((aligned + aligned // 2, pitch_el), 0xEEEE, dtype=torch.uint16, device="cuda")
    surf[:h, :w] = torch.from_numpy(tight[:h]).cuda()
    surf[aligned:aligned + h // 2, :w] = torch.from_numpy(tight[h:]).cuda()
    e = make_engine()
    for matrix, full in COLOURS:
        want_scale = e.forward_pixels([tight], engine.PIX_P016, matrix=matrix, full_range=full)
        want = results(e)
        scale = e.forward_pixels([surf[:h, :w]], engine.PIX_P016, chroma_offset=2 * pitch_el * aligned, matrix=matrix, full_range=full)
        assert scale == want_scale
        assert_same(results(e), want, ("p016 surface", matrix, full))
    e.close()


def test_rgbp_cuda_tensor_read_in_place():
    w, h = 1920, 1080
    tight = frame_of(engine.PIX_RGBP, w, h, seed=5)
    big = torch.full((3, h + 8, w + 64), 0xEE, dtype=torch.uint8, device="cuda")
    big[:, :h, :w] = torch.from_numpy(tight).cuda()
    view = big[:, :h, :w]
    ptr, pf, obj, _ = engine._pixel_view(view, engine.PIX_RGBP)
    assert obj is view and ptr == big.data_ptr() and pf.pitch == w + 64 and pf.chroma_offset == (h + 8) * (w + 64)
    e = make_engine()
    want_scale = e.forward_camera_frames([engine.pixels_to_bgr(tight, engine.PIX_RGBP)])
    want = results(e)
    assert e.forward_pixels([view], engine.PIX_RGBP) == want_scale
    assert_same(results(e), want, "rgbp view")
    e.close()


@pytest.mark.parametrize("fmt,matrix,full", [(engine.PIX_P016, "bt709", False), (engine.PIX_RGBP, "bt601", False),
                                             (engine.PIX_NV21, "bt709", True), (engine.PIX_UYVY, "bt601", True)])
def test_batches_and_graph_replays(fmt, matrix, full):
    """max_batch frames from separate allocations, three calls (eager, capture, replay): identical to frame-by-frame calls; one
    batch mixes device, page-locked and pageable frames"""
    B = 4
    e = make_engine(max_batch=B)
    one = make_engine()
    frames = [frame_of(fmt, 1920, 1080, seed=10 + i) for i in range(B)]
    singles = []
    for f in frames:
        one.forward_pixels([f], fmt, matrix=matrix, full_range=full)
        singles.append(results(one, render=False))
    dev = [torch.from_numpy(f).cuda() for f in frames]
    pinned = Pinned(frames[1])
    try:
        for call, batch in enumerate([dev, dev, dev, [dev[0], pinned.arr, frames[2], dev[3]]]):
            e.forward_pixels(batch, fmt, matrix=matrix, full_range=full)
            maps = e.fetch_maps(B)
            for i in range(B):
                assert np.array_equal(maps[i:i + 1], singles[i]["maps"]), (call, i)
                got = e.fetch(i)
                assert got[0] == singles[i]["fetch0"][0] and np.array_equal(got[1], singles[i]["fetch0"][1]), (call, i)
                assert np.array_equal(got[2], singles[i]["fetch0"][2]), (call, i)
    finally:
        e.sync()
        pinned.free()
    e.close()
    one.close()


def test_mixed_plane_strides_refused():
    """one call reads its frames with one layout: an RGBP view into a taller allocation (plane stride (h + 8) * w) and a tight
    tensor (h * w) in one batch are refused in either order, before anything is launched; each alone converts"""
    w, h = 640, 360
    e = make_engine(max_batch=2)
    L = engine.lib()
    tight = torch.from_numpy(frame_of(engine.PIX_RGBP, w, h, seed=7)).cuda()
    big = torch.zeros((3, h + 8, w), dtype=torch.uint8, device="cuda")
    big[:, :h] = tight
    view = big[:, :h, :]
    before = L.pe_launch_count(e._h)
    for batch in ([view, tight], [tight, view]):
        with pytest.raises(ValueError, match="plane stride"):
            e.forward_pixels(batch, engine.PIX_RGBP)
    assert L.pe_launch_count(e._h) == before
    e.forward_pixels([tight, tight], engine.PIX_RGBP)
    want = e.fetch_maps(2)
    e.forward_pixels([view, big[:, :h, :]], engine.PIX_RGBP)
    assert np.array_equal(e.fetch_maps(2), want)
    e.close()


def test_refusals_launch_nothing():
    e = make_engine()
    L = engine.lib()
    frame = torch.zeros((1620, 1920), dtype=torch.int16, device="cuda")
    ptrs = (C.c_void_p * 1)(frame.data_ptr())
    odd = (C.c_void_p * 1)(frame.data_ptr() + 1)
    s = C.c_double()
    before = L.pe_launch_count(e._h)
    P = engine._PixelFormat
    refused = [(P(f, 1920, 1080, 0, 0), ptrs, "pixel format") for f in range(5, 16)] + [
        (P(engine.PIX_RGB | engine.PIX_FLAG_BT709, 1920, 1080, 0, 0), ptrs, "colour flags"),
        (P(engine.PIX_RGBP | engine.PIX_FLAG_FULL_RANGE, 1920, 1080, 0, 0), ptrs, "colour flags"),
        (P(engine.PIX_NV12 | 0x400, 1920, 1080, 0, 0), ptrs, "unknown flag bits"),
        (P(engine.PIX_P016, 1920, 1080, 0, 0), odd, "odd P016 frame pointer"),
        (P(engine.PIX_P016, 1920, 1080, 3841, 0), ptrs, "odd P016 pitch"),
        (P(engine.PIX_P016, 1920, 1080, 0, 3840 * 1080 + 1), ptrs, "odd P016 chroma_offset"),
        (P(engine.PIX_RGBP, 1920, 1080, 0, 1920 * 1079), ptrs, "overlap"),
        (P(engine.PIX_UYVY, 1919, 1080, 0, 0), ptrs, "odd width"),
    ]
    for pf, p, words in refused:
        assert L.pe_forward_pixels(e._h, C.byref(pf), p, 1, C.byref(s)) == 1, words
        assert words in L.pe_last_error(e._h).decode()
    assert L.pe_launch_count(e._h) == before
    e.close()
