"""Decoder-format frames on the host (pe_pixels_to_bgr / engine.pixels_to_bgr): the reference of pe_forward_pixels's GPU conversion.
It must equal cv2.cvtColor bit for bit for NV12, I420, YUYV and RGB (BGR is the identity), read pitched frames and detached chroma
planes without touching the padding, and refuse every malformed pe_pixel_format with PE_ERR_INVALID and a reason."""
import ctypes as C

import cv2
import numpy as np
import pytest

from caffe_rtpose_b200 import engine

SIZES = [(2, 2), (64, 48), (1922, 1082)]   # (w, h)
CV = {engine.PIX_NV12: cv2.COLOR_YUV2BGR_NV12, engine.PIX_I420: cv2.COLOR_YUV2BGR_I420, engine.PIX_YUYV: cv2.COLOR_YUV2BGR_YUYV,
      engine.PIX_RGB: cv2.COLOR_RGB2BGR}
SHAPE = {engine.PIX_NV12: lambda w, h: (h * 3 // 2, w), engine.PIX_I420: lambda w, h: (h * 3 // 2, w),
         engine.PIX_YUYV: lambda w, h: (h, w, 2), engine.PIX_RGB: lambda w, h: (h, w, 3), engine.PIX_BGR: lambda w, h: (h, w, 3)}


def cv_bgr(frame, fmt):
    return frame.copy() if fmt == engine.PIX_BGR else cv2.cvtColor(frame, CV[fmt])


def extreme_frame(fmt, w, h, rng):
    """luma bytes from {0, 16, 235, 255}, chroma bytes from {0, 128, 255}: every saturation edge of the fixed-point formula"""
    Y, UV = np.array([0, 16, 235, 255], np.uint8), np.array([0, 128, 255], np.uint8)
    f = np.empty(SHAPE[fmt](w, h), np.uint8)
    if fmt in (engine.PIX_NV12, engine.PIX_I420):
        f[:h] = rng.choice(Y, (h, w))
        f[h:] = rng.choice(UV, (h // 2, w))
    elif fmt == engine.PIX_YUYV:
        f[..., 0] = rng.choice(Y, (h, w))
        f[..., 1] = rng.choice(UV, (h, w))
    else:
        f[:] = rng.choice(np.array([0, 1, 127, 128, 254, 255], np.uint8), f.shape)
    return f


@pytest.mark.parametrize("w,h", SIZES)
@pytest.mark.parametrize("fmt", [engine.PIX_NV12, engine.PIX_I420, engine.PIX_YUYV, engine.PIX_RGB, engine.PIX_BGR])
def test_equals_cv2_cvtcolor(fmt, w, h):
    rng = np.random.default_rng(w * 7 + h + fmt)
    for frame in (rng.integers(0, 256, SHAPE[fmt](w, h), dtype=np.uint8), extreme_frame(fmt, w, h, rng)):
        assert np.array_equal(engine.pixels_to_bgr(frame, fmt), cv_bgr(frame, fmt))


def padded(fmt, frame, w, h, pitch, chroma_offset):
    """frame laid out with `pitch` bytes per row and (NV12 / I420) its chroma plane at chroma_offset, everything else 0xEE"""
    planar = fmt in (engine.PIX_NV12, engine.PIX_I420)
    rows = frame.reshape(frame.shape[0], -1)
    row = rows.shape[1]
    if not planar:
        buf = np.full(pitch * h, 0xEE, np.uint8)
        for y in range(h):
            buf[y * pitch:y * pitch + row] = rows[y]
        return buf
    buf = np.full(chroma_offset + pitch * h, 0xEE, np.uint8)
    for y in range(h):
        buf[y * pitch:y * pitch + w] = rows[y]
    chroma = rows[h:].reshape(-1)   # tight: NV12 h/2 rows of w, I420 U then V, h/2 rows of w/2 each
    cw, cp = (w, pitch) if fmt == engine.PIX_NV12 else (w // 2, pitch // 2)
    for r in range(len(chroma) // cw):
        buf[chroma_offset + r * cp:chroma_offset + r * cp + cw] = chroma[r * cw:(r + 1) * cw]
    return buf


def c_convert(fmt, buf, w, h, pitch=0, chroma_offset=0, cap=None):
    out = np.zeros((h, w, 3), np.uint8)
    pf = engine._PixelFormat(fmt, w, h, pitch, chroma_offset)
    rc = engine.lib().pe_pixels_to_bgr(C.byref(pf), buf.ctypes.data if buf is not None else None, out.ctypes.data,
                                        out.size if cap is None else cap)
    return rc, out


@pytest.mark.parametrize("w,h", SIZES)
@pytest.mark.parametrize("fmt", [engine.PIX_NV12, engine.PIX_I420, engine.PIX_YUYV, engine.PIX_RGB, engine.PIX_BGR])
def test_padded_pitch_and_detached_chroma(fmt, w, h):
    rng = np.random.default_rng(w + h * 3 + fmt)
    frame = rng.integers(0, 256, SHAPE[fmt](w, h), dtype=np.uint8)
    want = cv_bgr(frame, fmt)
    row = frame.reshape(frame.shape[0], -1).shape[1]
    pitch = row + 2 * (11 + w % 5)   # even, so I420 chroma rows are pitch/2 apart
    layouts = [(pitch, 0)]
    if fmt in (engine.PIX_NV12, engine.PIX_I420):
        layouts.append((pitch, pitch * (h + 8) + 6))   # an NVDEC-style surface: chroma after the aligned height
    for p, co in layouts:
        buf = padded(fmt, frame, w, h, p, co or p * h)
        rc, out = c_convert(fmt, buf, w, h, p, co)
        assert rc == 0 and np.array_equal(out, want), (p, co)
    # the Python wrapper takes the pitch from the row stride: a column slice of a wider allocation
    wide = rng.integers(0, 256, (frame.shape[0], row + 64), dtype=np.uint8)
    wide[:, :row] = frame.reshape(frame.shape[0], -1)
    view = wide[:, :row].reshape(frame.shape)
    assert not view.flags.c_contiguous or frame.shape[0] == 1
    assert np.array_equal(engine.pixels_to_bgr(view, fmt), want)


def test_yuyv_to_bgr_keeps_its_results():
    rng = np.random.default_rng(5)
    for w, h in SIZES:
        f = rng.integers(0, 256, (h, w, 2), dtype=np.uint8)
        assert np.array_equal(engine.yuyv_to_bgr(f), cv2.cvtColor(f, cv2.COLOR_YUV2BGR_YUYV))


BAD = [
    ("format -1", dict(fmt=-1), "pixel format"),
    ("format 5", dict(fmt=5), "pixel format"),
    ("width 0", dict(w=0), "frame size"),
    ("height 0", dict(h=0), "frame size"),
    ("negative width", dict(w=-4), "frame size"),
    ("width 16386", dict(w=16386), "frame size"),
    ("height 16386", dict(h=16386), "frame size"),
    ("odd YUYV width", dict(fmt=engine.PIX_YUYV, w=5), "odd width"),
    ("odd NV12 width", dict(fmt=engine.PIX_NV12, w=5), "odd width"),
    ("odd NV12 height", dict(fmt=engine.PIX_NV12, h=5), "odd height"),
    ("odd I420 width", dict(fmt=engine.PIX_I420, w=5), "odd width"),
    ("odd I420 height", dict(fmt=engine.PIX_I420, h=5), "odd height"),
    ("BGR pitch below 3w", dict(fmt=engine.PIX_BGR, pitch=3 * 8 - 1), "pitch"),
    ("RGB pitch below 3w", dict(fmt=engine.PIX_RGB, pitch=3 * 8 - 1), "pitch"),
    ("YUYV pitch below 2w", dict(fmt=engine.PIX_YUYV, pitch=2 * 8 - 2), "pitch"),
    ("NV12 pitch below w", dict(fmt=engine.PIX_NV12, pitch=7), "pitch"),
    ("negative pitch", dict(pitch=-64), "pitch"),
    ("odd I420 pitch", dict(fmt=engine.PIX_I420, pitch=9), "odd I420 pitch"),
    ("NV12 chroma inside the luma plane", dict(fmt=engine.PIX_NV12, pitch=8, co=8 * 6 - 1), "chroma_offset"),
    ("I420 chroma inside the luma plane", dict(fmt=engine.PIX_I420, pitch=8, co=8), "chroma_offset"),
    ("negative chroma offset", dict(fmt=engine.PIX_NV12, co=-1), "chroma_offset"),
    ("pitch * height overflows", dict(pitch=1 << 62), "overflows"),
    ("chroma offset overflows", dict(fmt=engine.PIX_NV12, co=(1 << 63) - 16), "overflows"),
    ("span beyond 2^56", dict(fmt=engine.PIX_NV12, co=1 << 56), "2^56"),
    ("null frame", dict(buf=None), "null"),
    ("small cap", dict(cap=8 * 6 * 3 - 1), "cap"),
]


@pytest.mark.parametrize("name,kw,words", BAD, ids=[b[0] for b in BAD])
def test_validation(name, kw, words):
    L = engine.lib()
    fmt, w, h = kw.get("fmt", engine.PIX_BGR), kw.get("w", 8), kw.get("h", 6)
    buf = kw.get("buf", np.zeros(1 << 12, np.uint8))
    out = np.zeros(max(1, 3 * max(w, 1) * max(h, 1)) if abs(w) < 100 and abs(h) < 100 else 16, np.uint8)
    pf = engine._PixelFormat(fmt, w, h, kw.get("pitch", 0), kw.get("co", 0))
    cap = kw.get("cap", out.size)
    rc = L.pe_pixels_to_bgr(C.byref(pf), buf.ctypes.data if buf is not None else None, out.ctypes.data, cap)
    assert rc == 1, name   # PE_ERR_INVALID
    msg = L.pe_last_error(None).decode()
    assert words in msg, (name, msg)
    assert not out.any(), "nothing is written on a refusal"


def test_null_format_and_output():
    L = engine.lib()
    buf = np.zeros(64, np.uint8)
    out = np.zeros(64, np.uint8)
    assert L.pe_pixels_to_bgr(None, buf.ctypes.data, out.ctypes.data, out.size) == 1
    assert "null" in L.pe_last_error(None).decode()
    pf = engine._PixelFormat(engine.PIX_BGR, 2, 2, 0, 0)
    assert L.pe_pixels_to_bgr(C.byref(pf), buf.ctypes.data, None, 12) == 1
    assert "null" in L.pe_last_error(None).decode()


def test_python_wrapper_checks():
    with pytest.raises(ValueError):
        engine.pixels_to_bgr(np.zeros((4, 4, 3), np.uint8), 9)
    with pytest.raises(ValueError):
        engine.pixels_to_bgr(np.zeros((4, 4, 3), np.uint8), engine.PIX_YUYV)   # YUYV is (h, w, 2)
    with pytest.raises(ValueError):
        engine.pixels_to_bgr(np.zeros((5, 4), np.uint8), engine.PIX_NV12)      # rows are h*3/2
    with pytest.raises(TypeError):
        engine.pixels_to_bgr(np.zeros((6, 4), np.uint16), engine.PIX_NV12)
    with pytest.raises(engine.PoseEngineError, match="odd width"):
        engine.pixels_to_bgr(np.zeros((6, 5), np.uint8), engine.PIX_NV12)
    # reversed rows (a negative stride) are copied, not read backwards
    f = np.random.default_rng(1).integers(0, 256, (6, 4, 3), dtype=np.uint8)
    assert np.array_equal(engine.pixels_to_bgr(f[::-1], engine.PIX_RGB), cv2.cvtColor(np.ascontiguousarray(f[::-1]), cv2.COLOR_RGB2BGR))
