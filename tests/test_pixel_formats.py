"""The decoder formats beyond NV12 / I420 / YUYV / RGB (NV21, YV12, UYVY, P016, planar RGB) and the colour flags (BT.709, full
range) on the host (pe_pixels_to_bgr / engine.pixels_to_bgr), the reference of pe_forward_pixels's GPU conversion:

  - NV21, YV12 and UYVY equal cv2.cvtColor bit for bit, tight and pitched, with detached chroma;
  - full-range BT.601 equals cv2's COLOR_YCrCb2BGR, and studio-range BT.601 COLOR_YUV2BGR_NV12, for all 2^24 (Y, U, V);
  - BT.709 (studio, full) is within 1 of the float64 conversion, rounded half up and saturated, for all 2^24 (Y, U, V);
  - P016 is within 1 of float64 for every 10-bit code of each component in a seeded sample of 2^24 triples, in all four
    matrix / range cases, and a frame of samples v << 8 converts exactly as the 8-bit frame of v;
  - planar RGB is a transpose to BGR, also from views with padded plane and row strides;
  - malformed formats, flags and pointers are PE_ERR_INVALID with the reason, and nothing is written;
  - ptxas reports no spills for any pixels_to_bgr_kernel instance.
"""
import ctypes as C
import re

import cv2
import numpy as np
import pytest
import torch

from caffe_rtpose_b200 import engine
from test_conv_build import tu_build

SIZES = [(2, 2), (64, 48), (1922, 1082)]   # (w, h)
CV = {engine.PIX_NV21: cv2.COLOR_YUV2BGR_NV21, engine.PIX_YV12: cv2.COLOR_YUV2BGR_YV12, engine.PIX_UYVY: cv2.COLOR_YUV2BGR_UYVY}
SEMI = (engine.PIX_NV12, engine.PIX_NV21, engine.PIX_P016)
BT601, BT709 = (0.299, 0.114), (0.2126, 0.0722)
CASES = [("bt601", False), ("bt601", True), ("bt709", False), ("bt709", True)]


def shape_of(fmt, w, h):
    return (h, w, 2) if fmt == engine.PIX_UYVY else (3, h, w) if fmt == engine.PIX_RGBP else (h * 3 // 2, w)


def c_convert(fmt, buf, w, h, pitch=0, chroma_offset=0):
    out = np.zeros((h, w, 3), np.uint8)
    pf = engine._PixelFormat(fmt, w, h, pitch, chroma_offset)
    rc = engine.lib().pe_pixels_to_bgr(C.byref(pf), buf.ctypes.data, out.ctypes.data, out.size)
    return rc, out


def padded(fmt, frame, w, h, pitch, chroma_offset):
    """frame (cv2's layout) as bytes with `pitch` bytes per row and its chroma plane at chroma_offset, everything else 0xEE"""
    rows = frame.view(np.uint8).reshape(frame.shape[0], -1)
    row = rows.shape[1]
    if fmt == engine.PIX_UYVY:
        buf = np.full(pitch * h, 0xEE, np.uint8)
        for y in range(h):
            buf[y * pitch:y * pitch + row] = rows[y]
        return buf
    buf = np.full(chroma_offset + pitch * h, 0xEE, np.uint8)
    for y in range(h):
        buf[y * pitch:y * pitch + row] = rows[y]
    chroma = rows[h:].reshape(-1)
    cw, cp = (row, pitch) if fmt in SEMI else (w // 2, pitch // 2)
    for r in range(len(chroma) // cw):
        buf[chroma_offset + r * cp:chroma_offset + r * cp + cw] = chroma[r * cw:(r + 1) * cw]
    return buf


@pytest.mark.parametrize("w,h", SIZES)
@pytest.mark.parametrize("fmt", [engine.PIX_NV21, engine.PIX_YV12, engine.PIX_UYVY])
def test_equals_cv2_cvtcolor(fmt, w, h):
    rng = np.random.default_rng(w * 5 + h + fmt)
    frame = rng.integers(0, 256, shape_of(fmt, w, h), dtype=np.uint8)
    edges = rng.choice(np.array([0, 16, 128, 235, 255], np.uint8), frame.shape)   # every saturation edge of the formula
    for f in (frame, edges):
        assert np.array_equal(engine.pixels_to_bgr(f, fmt), cv2.cvtColor(f, CV[fmt]))
    want = cv2.cvtColor(frame, CV[fmt])
    row = frame.reshape(frame.shape[0], -1).shape[1]
    pitch = row + 2 * (11 + w % 5)   # even, so YV12 chroma rows are pitch/2 apart
    layouts = [(pitch, 0)] + ([(pitch, pitch * (h + 8) + 6)] if fmt != engine.PIX_UYVY else [])
    for p, co in layouts:
        rc, out = c_convert(fmt, padded(fmt, frame, w, h, p, co or p * h), w, h, p, co)
        assert rc == 0 and np.array_equal(out, want), (p, co)
    wide = np.full((frame.shape[0], row + 64), 0xEE, np.uint8)   # the wrapper takes the pitch from the row stride
    wide[:, :row] = frame.reshape(frame.shape[0], -1)
    assert np.array_equal(engine.pixels_to_bgr(wide[:, :row].reshape(frame.shape), fmt), want)


# ---- the per-pixel functions over every (Y, U, V)

@pytest.fixture(scope="module")
def triples():
    """a 4096 x 4096 NV12 frame holding each of the 2^24 (Y, U, V) once: quad q has U = (q >> 6) & 255, V = q >> 14 and its four
    luma samples ((q & 63) << 2) + 0..3.  Returns (frame, per-pixel Y, U, V), uint8, 64 MB in all, freed with the module."""
    n = 4096
    q = np.arange((n // 2) ** 2, dtype=np.int32).reshape(n // 2, n // 2)
    Y = np.empty((n, n), np.uint8)
    for dy in range(2):
        for dx in range(2):
            Y[dy::2, dx::2] = ((q & 63) << 2) + dy * 2 + dx
    U, V = ((q >> 6) & 255).astype(np.uint8), (q >> 14).astype(np.uint8)
    frame = np.empty((n * 3 // 2, n), np.uint8)
    frame[:n] = Y
    frame[n:, 0::2], frame[n:, 1::2] = U, V
    up = lambda c: np.repeat(np.repeat(c, 2, 0), 2, 1)
    return frame, Y, up(U), up(V)


def test_all_triples_are_covered(triples):
    _, Y, U, V = (t.astype(np.int32) for t in triples)
    assert (np.bincount((Y | U << 8 | V << 16).ravel(), minlength=1 << 24) == 1).all()


def test_bt601_studio_equals_cv2_nv12_for_every_triple(triples):
    frame = triples[0]
    assert np.array_equal(engine.pixels_to_bgr(frame, engine.PIX_NV12), cv2.cvtColor(frame, cv2.COLOR_YUV2BGR_NV12))


def test_bt601_full_range_equals_cv2_ycrcb_for_every_triple(triples):
    frame, Y, U, V = triples
    ycrcb = np.stack([Y, V, U], -1)
    want = cv2.cvtColor(ycrcb, cv2.COLOR_YCrCb2BGR)
    assert np.array_equal(engine.pixels_to_bgr(frame, engine.PIX_NV12, full_range=True), want)


def exact_bgr(Y, U, V, matrix, full, bits=8):
    """the real-valued conversion in float64, rounded half up and saturated; studio-range luma below black counts as black"""
    kr, kb = BT709 if matrix == "bt709" else BT601
    kg = 1 - kr - kb
    s = float(1 << (bits - 8))
    y, u, v = Y / s, U / s - 128, V / s - 128
    if not full:
        y, u, v = np.maximum(y - 16, 0) * (255 / 219), u * (255 / 224), v * (255 / 224)
    b, g, r = y + 2 * (1 - kb) * u, y - 2 * kb * (1 - kb) / kg * u - 2 * kr * (1 - kr) / kg * v, y + 2 * (1 - kr) * v
    return np.clip(np.floor(np.stack([b, g, r], -1) + 0.5), 0, 255).astype(np.int16)


def within_one(got, Y, U, V, matrix, full, bits, tag):
    """max |got - exact| over row chunks; returns the share of exact bytes"""
    exact = 0
    for r in range(0, Y.shape[0], 512):
        want = exact_bgr(Y[r:r + 512], U[r:r + 512], V[r:r + 512], matrix, full, bits)
        d = np.abs(got[r:r + 512].astype(np.int16) - want)
        assert d.max() <= 1, (tag, r, int(d.max()))
        exact += int((d == 0).sum())
    share = exact / got.size
    print("%s: %.4f %% of the bytes equal the float64 conversion, the rest within 1" % (tag, 100 * share))
    return share


@pytest.mark.parametrize("full", [False, True])
def test_bt709_within_one_of_float64_for_every_triple(triples, full):
    frame, Y, U, V = triples
    got = engine.pixels_to_bgr(frame, engine.PIX_NV12, matrix="bt709", full_range=full)
    assert within_one(got, Y, U, V, "bt709", full, 8, "BT.709 %s range" % ("full" if full else "studio")) > 0.9


# ---- 16-bit samples

@pytest.fixture(scope="module")
def p016_sample():
    """a 4096 x 4096 P016 frame and its per-pixel Y, U, V (uint16, 128 MB in all, freed with the module): each 10-bit code (v << 6,
    as P010 stores it) of each component swept against random partners, 10-bit codes throughout, and random 16-bit samples - 2^24
    triples from a fixed seed"""
    n, rng = 4096, np.random.default_rng(16)
    code = lambda k: ((np.arange(k) % 1024) << 6).astype(np.uint16)
    Y = rng.integers(0, 1 << 16, (n, n), dtype=np.uint16)
    Y[:n // 4] = code(n // 4 * n).reshape(n // 4, n)
    Y[n // 4:n // 2] = rng.integers(0, 1024, (n // 4, n)) << 6
    U = rng.integers(0, 1 << 16, (n // 2, n // 2), dtype=np.uint16)
    V = rng.integers(0, 1 << 16, (n // 2, n // 2), dtype=np.uint16)
    m = n // 8   # quad rows per band
    U[:m] = code(m * n // 2).reshape(m, n // 2)
    V[m:2 * m] = code(m * n // 2).reshape(m, n // 2)
    U[2 * m:3 * m] = rng.integers(0, 1024, (m, n // 2)) << 6
    V[2 * m:3 * m] = rng.integers(0, 1024, (m, n // 2)) << 6
    frame = np.empty((n * 3 // 2, n), np.uint16)
    frame[:n] = Y
    frame[n:, 0::2], frame[n:, 1::2] = U, V
    up = lambda c: np.repeat(np.repeat(c, 2, 0), 2, 1)
    return frame, Y, up(U), up(V)


@pytest.mark.parametrize("matrix,full", CASES)
def test_p016_within_one_of_float64(p016_sample, matrix, full):
    frame, Y, U, V = p016_sample
    for comp in (Y, U, V):   # every 10-bit code of each component is in the sample
        assert np.isin(np.arange(1024) << 6, comp).all()
    got = engine.pixels_to_bgr(frame, engine.PIX_P016, matrix=matrix, full_range=full)
    within_one(got, Y, U, V, matrix, full, 16, "P016 %s %s range" % (matrix, "full" if full else "studio"))


@pytest.mark.parametrize("matrix,full", CASES)
def test_p016_of_shifted_bytes_equals_8_bit(triples, matrix, full):
    """the 16-bit formula is the 8-bit one with 8 more fractional bits: v << 8 converts exactly as v"""
    frame = triples[0]
    wide = frame.astype(np.uint16) << 8
    assert np.array_equal(engine.pixels_to_bgr(wide, engine.PIX_P016, matrix=matrix, full_range=full),
                          engine.pixels_to_bgr(frame, engine.PIX_NV12, matrix=matrix, full_range=full))


def test_p016_pitched_and_detached_chroma():
    rng = np.random.default_rng(7)
    w, h = 1922, 1082
    frame = rng.integers(0, 1 << 16, (h * 3 // 2, w), dtype=np.uint16)
    want = engine.pixels_to_bgr(frame, engine.PIX_P016, matrix="bt709")
    pitch = 2 * w + 2 * 37
    for co in (0, pitch * (h + 6) + 10):
        buf = padded(engine.PIX_P016, frame, w, h, pitch, co or pitch * h)
        rc, out = c_convert(engine.PIX_P016 | engine.PIX_FLAG_BT709, buf, w, h, pitch, co)
        assert rc == 0 and np.array_equal(out, want), co
    wide = np.full((frame.shape[0], w + 40), 0xEEEE, np.uint16)
    wide[:, :w] = frame
    assert np.array_equal(engine.pixels_to_bgr(wide[:, :w], engine.PIX_P016, matrix="bt709"), want)
    assert np.array_equal(engine.pixels_to_bgr(torch.from_numpy(wide)[:, :w], engine.PIX_P016, matrix="bt709"), want)


def test_flags_leave_the_default_unchanged_and_apply_to_every_yuv_format():
    rng = np.random.default_rng(3)
    w, h = 64, 48
    nv12 = rng.integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)
    y, uv = nv12[:h], nv12[h:].reshape(h // 2, w // 2, 2)
    i420 = np.concatenate([y.reshape(-1), uv[..., 0].reshape(-1), uv[..., 1].reshape(-1)]).reshape(h * 3 // 2, w)
    yv12 = np.concatenate([y.reshape(-1), uv[..., 1].reshape(-1), uv[..., 0].reshape(-1)]).reshape(h * 3 // 2, w)
    nv21 = np.concatenate([y, uv[..., ::-1].reshape(h // 2, w)])
    yuyv = np.empty((h, w, 2), np.uint8)   # the chroma of the upper row of each pair, and a lower row that repeats it
    yuyv[..., 0] = y
    yuyv[:, 0::2, 1], yuyv[:, 1::2, 1] = np.repeat(uv[..., 0], 2, 0), np.repeat(uv[..., 1], 2, 0)
    uyvy = yuyv[..., ::-1].copy()
    same = [(engine.PIX_NV12, nv12), (engine.PIX_I420, i420), (engine.PIX_YV12, yv12), (engine.PIX_NV21, nv21),
            (engine.PIX_YUYV, yuyv), (engine.PIX_UYVY, uyvy), (engine.PIX_P016, nv12.astype(np.uint16) << 8)]
    for matrix, full in CASES:
        want = engine.pixels_to_bgr(nv12, engine.PIX_NV12, matrix=matrix, full_range=full)
        for fmt, f in same:
            assert np.array_equal(engine.pixels_to_bgr(f, fmt, matrix=matrix, full_range=full), want), (fmt, matrix, full)
    assert not np.array_equal(engine.pixels_to_bgr(nv12, engine.PIX_NV12, matrix="bt709"),
                              engine.pixels_to_bgr(nv12, engine.PIX_NV12))


# ---- planar RGB

@pytest.mark.parametrize("w,h", SIZES)
def test_rgbp_is_a_transpose(w, h):
    rng = np.random.default_rng(w + h)
    f = rng.integers(0, 256, (3, h, w), dtype=np.uint8)
    want = np.ascontiguousarray(f.transpose(1, 2, 0)[..., ::-1])
    assert np.array_equal(engine.pixels_to_bgr(f, engine.PIX_RGBP), want)
    big = np.full((3, h + 5, w + 7), 0xEE, np.uint8)   # padded plane and row strides, read in place
    big[:, :h, :w] = f
    view = big[:, :h, :w]
    ptr, pf, obj, _ = engine._pixel_view(view, engine.PIX_RGBP)
    assert obj is view and pf.pitch == w + 7 and pf.chroma_offset == (h + 5) * (w + 7)
    assert np.array_equal(engine.pixels_to_bgr(view, engine.PIX_RGBP), want)
    t = torch.from_numpy(big)[:, :h, :w]
    assert engine._pixel_view(t, engine.PIX_RGBP)[2] is t
    assert np.array_equal(engine.pixels_to_bgr(t, engine.PIX_RGBP), want)
    # the C layout: plane distance set explicitly, the gap between planes left as 0xEE
    pitch, co = w + 3, (w + 3) * h + 17
    buf = np.full(2 * co + pitch * h, 0xEE, np.uint8)
    for k in range(3):
        buf[k * co:k * co + pitch * h].reshape(h, pitch)[:, :w] = f[k]
    rc, out = c_convert(engine.PIX_RGBP, buf, w, h, pitch, co)
    assert rc == 0 and np.array_equal(out, want)
    # a (3, h, w) permute of an HWC array interleaves the planes row by row: copied first
    hwc = np.ascontiguousarray(f.transpose(1, 2, 0))
    assert np.array_equal(engine.pixels_to_bgr(hwc.transpose(2, 0, 1), engine.PIX_RGBP), want)


def test_a_batch_shares_one_layout():
    """pe_forward_pixels reads every frame of a call with one layout: RGBP frames with different plane strides (a view into a
    taller allocation and a tight tensor) are refused before anything reaches the engine, in either order"""
    h, w = 4, 6
    view = torch.zeros((3, h + 8, w), dtype=torch.uint8)[:, :h, :]
    tight = torch.zeros((3, h, w), dtype=torch.uint8)
    views = [engine._pixel_view(f, engine.PIX_RGBP) for f in (view, tight)]
    assert [v[1].chroma_offset for v in views] == [(h + 8) * w, h * w]
    for batch in (views, views[::-1]):
        with pytest.raises(ValueError, match="plane stride"):
            engine._batch_format(batch)
    assert engine._batch_format([views[1], engine._pixel_view(tight.clone(), engine.PIX_RGBP)]).chroma_offset == h * w
    nv12 = np.zeros((6, 4), np.uint8)
    with pytest.raises(ValueError, match="row stride"):   # and, as before, the row stride
        engine._batch_format([engine._pixel_view(nv12, engine.PIX_NV12),
                              engine._pixel_view(np.zeros((6, 8), np.uint8)[:, :4], engine.PIX_NV12)])


# ---- refusals

W8, H6 = 8, 6
BAD = [("format %d" % f, dict(fmt=f), "pixel format") for f in range(5, 16)] + [
    ("format 21", dict(fmt=21), "pixel format"),
    ("format 255", dict(fmt=255), "pixel format"),
    ("flag on format 7", dict(fmt=7 | 0x100), "pixel format"),
    ("unknown bit 0x400", dict(fmt=engine.PIX_NV12 | 0x400), "unknown flag bits"),
    ("unknown bit 0x10000", dict(fmt=engine.PIX_P016 | 0x10000), "unknown flag bits"),
    ("BT.709 on BGR", dict(fmt=engine.PIX_BGR | 0x100), "colour flags"),
    ("full range on RGB", dict(fmt=engine.PIX_RGB | 0x200), "colour flags"),
    ("both flags on RGBP", dict(fmt=engine.PIX_RGBP | 0x300), "colour flags"),
    ("odd NV21 width", dict(fmt=engine.PIX_NV21, w=5), "odd width"),
    ("odd NV21 height", dict(fmt=engine.PIX_NV21, h=5), "odd height"),
    ("odd YV12 width", dict(fmt=engine.PIX_YV12, w=5), "odd width"),
    ("odd YV12 height", dict(fmt=engine.PIX_YV12, h=5), "odd height"),
    ("odd UYVY width", dict(fmt=engine.PIX_UYVY, w=5), "odd width"),
    ("odd P016 width", dict(fmt=engine.PIX_P016, w=5), "odd width"),
    ("odd P016 height", dict(fmt=engine.PIX_P016, h=5), "odd height"),
    ("UYVY pitch below 2w", dict(fmt=engine.PIX_UYVY, pitch=2 * W8 - 2), "pitch"),
    ("NV21 pitch below w", dict(fmt=engine.PIX_NV21, pitch=W8 - 1), "pitch"),
    ("P016 pitch below 2w", dict(fmt=engine.PIX_P016, pitch=2 * W8 - 2), "pitch"),
    ("RGBP pitch below w", dict(fmt=engine.PIX_RGBP, pitch=W8 - 1), "pitch"),
    ("odd YV12 pitch", dict(fmt=engine.PIX_YV12, pitch=9), "odd YV12 pitch"),
    ("odd P016 pitch", dict(fmt=engine.PIX_P016, pitch=2 * W8 + 1), "odd P016 pitch"),
    ("odd P016 chroma offset", dict(fmt=engine.PIX_P016, co=2 * W8 * H6 + 1), "odd P016 chroma_offset"),
    ("odd P016 pointer", dict(fmt=engine.PIX_P016, odd_ptr=True), "odd P016 frame pointer"),
    ("NV21 chroma inside the luma plane", dict(fmt=engine.PIX_NV21, co=W8 * H6 - 1), "chroma_offset"),
    ("YV12 chroma inside the luma plane", dict(fmt=engine.PIX_YV12, pitch=8, co=8), "chroma_offset"),
    ("P016 chroma inside the luma plane", dict(fmt=engine.PIX_P016, co=2 * W8 * H6 - 2), "chroma_offset"),
    ("RGBP planes overlap", dict(fmt=engine.PIX_RGBP, co=W8 * H6 - 1), "overlap"),
    ("negative RGBP plane stride", dict(fmt=engine.PIX_RGBP, co=-W8 * H6), "overlap"),
    ("P016 pitch * height overflows", dict(fmt=engine.PIX_P016, pitch=1 << 62), "overflows"),
    ("RGBP plane stride overflows", dict(fmt=engine.PIX_RGBP, co=1 << 62), "overflows"),
    ("P016 chroma offset overflows", dict(fmt=engine.PIX_P016, co=(1 << 63) - 16), "overflows"),
    ("RGBP span beyond 2^56", dict(fmt=engine.PIX_RGBP, co=1 << 55), "2^56"),
]


@pytest.mark.parametrize("name,kw,words", BAD, ids=[b[0] for b in BAD])
def test_validation(name, kw, words):
    L = engine.lib()
    fmt, w, h = kw["fmt"], kw.get("w", W8), kw.get("h", H6)
    buf = np.zeros(1 << 12, np.uint8)
    out = np.zeros(3 * w * h, np.uint8)
    pf = engine._PixelFormat(fmt, w, h, kw.get("pitch", 0), kw.get("co", 0))
    rc = L.pe_pixels_to_bgr(C.byref(pf), buf.ctypes.data + (1 if kw.get("odd_ptr") else 0), out.ctypes.data, out.size)
    assert rc == 1, name   # PE_ERR_INVALID
    msg = L.pe_last_error(None).decode()
    assert words in msg, (name, msg)
    assert not out.any(), "nothing is written on a refusal"


def test_python_wrapper_shapes():
    z = lambda *s, dt=np.uint8: np.zeros(s, dt)
    for fmt in (engine.PIX_NV21, engine.PIX_YV12):
        assert engine.pixels_to_bgr(z(6, 4), fmt).shape == (4, 4, 3)
        with pytest.raises(ValueError):
            engine.pixels_to_bgr(z(5, 4), fmt)   # rows are h*3/2
    assert engine.pixels_to_bgr(z(4, 4, 2), engine.PIX_UYVY).shape == (4, 4, 3)
    assert engine.pixels_to_bgr(z(6, 4, dt=np.uint16), engine.PIX_P016).shape == (4, 4, 3)
    assert engine.pixels_to_bgr(z(3, 4, 6), engine.PIX_RGBP).shape == (4, 6, 3)
    for bad_shape, fmt in (((4, 4, 3), engine.PIX_UYVY), ((4, 6, 3), engine.PIX_RGBP), ((4, 4, 6), engine.PIX_RGBP),
                           ((6, 4, 1), engine.PIX_P016)):
        with pytest.raises(ValueError):
            engine.pixels_to_bgr(z(*bad_shape, dt=np.uint16 if fmt == engine.PIX_P016 else np.uint8), fmt)
    for fmt, shape in ((engine.PIX_NV12, (6, 4)), (engine.PIX_NV21, (6, 4)), (engine.PIX_YV12, (6, 4)), (engine.PIX_I420, (6, 4)),
                       (engine.PIX_UYVY, (4, 4, 2)), (engine.PIX_YUYV, (4, 4, 2)), (engine.PIX_RGB, (4, 4, 3)),
                       (engine.PIX_BGR, (4, 4, 3)), (engine.PIX_RGBP, (3, 4, 4))):
        with pytest.raises(TypeError):   # uint16 is P016's alone
            engine.pixels_to_bgr(z(*shape, dt=np.uint16), fmt)
        with pytest.raises(TypeError):
            engine.pixels_to_bgr(torch.zeros(shape, dtype=torch.uint16), fmt)
    with pytest.raises(TypeError):
        engine.pixels_to_bgr(z(6, 4), engine.PIX_P016)   # P016 is uint16
    with pytest.raises(ValueError, match="matrix"):
        engine.pixels_to_bgr(z(6, 4), engine.PIX_NV12, matrix="bt2020")
    with pytest.raises(engine.PoseEngineError, match="colour flags"):
        engine.pixels_to_bgr(z(4, 4, 3), engine.PIX_RGB, matrix="bt709")
    with pytest.raises(engine.PoseEngineError, match="colour flags"):
        engine.pixels_to_bgr(z(3, 4, 4), engine.PIX_RGBP, full_range=True)
    with pytest.raises(ValueError, match="chroma_offset"):
        engine._pixel_view(z(3, 4, 4), engine.PIX_RGBP, chroma_offset=48)
    # a P016 view keeps its byte pitch; a torch uint16 tensor's strides are in elements
    wide = z(6, 10, dt=np.uint16)
    assert engine._pixel_view(wide[:, :4], engine.PIX_P016)[1].pitch == 20
    assert engine._pixel_view(torch.from_numpy(wide)[:, :4], engine.PIX_P016)[1].pitch == 20
    assert engine._pixel_view(z(6, 4), engine.PIX_NV12, None, engine.PIX_FLAG_BT709 | engine.PIX_FLAG_FULL_RANGE)[1].format == 0x303


# ---- the kernel as ptxas builds it

build = tu_build("pixels.cu")


def test_no_spills(build):
    log = build[0]
    kernels, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"(?:Compiling entry function|Function properties for) '?(\w+)", line)
        if m:
            cur = m.group(1) if "pixels_to_bgr_kernel" in m.group(1) else None
            if cur:
                kernels.setdefault(cur, [])
            continue
        if cur:
            kernels[cur].append(line)
    assert len(kernels) == 6, sorted(kernels)   # one instance per memory layout
    for name, lines in kernels.items():
        spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", "\n".join(lines))
        assert spill and spill.groups() == ("0", "0"), (name, lines)
