// Decoder-format frames (pe_pixel_format, poseengine.h) -> uint8 BGR: the per-pixel arithmetic of cv::cvtColor shared by the CUDA
// kernel (pixels.cu), the host reference pe_pixels_to_bgr and the camera's pe_yuyv_to_bgr, and the layout checks of every entry
// point that reads such frames.
//
// OpenCV's YUV -> BGR conversions (imgproc color_yuv, COLOR_YUV2BGR_YUYV / _NV12 / _I420) share one ITU-R BT.601 studio-range
// fixed-point formula: 20-bit constants, max(Y - 16, 0) * CY plus the chroma terms of the pixel's (nearest-neighbour) chroma sample,
// >> 20, saturated to uint8.  4:2:2 pairs and 4:2:0 quads differ only in how many luma samples share one chroma sample.
#pragma once
#include <stdint.h>

#include <string>

#include "../../include/poseengine.h"

#ifndef PE_HD
#ifdef __CUDACC__
#define PE_HD __host__ __device__ __forceinline__
#else
#define PE_HD inline
#endif
#endif

namespace pe_pix {

constexpr int SHIFT = 20, CY = 1220542, CUB = 2116026, CUG = -409993, CVG = -852492, CVR = 1673527, HALF = 1 << (SHIFT - 1);
constexpr int MAX_SIDE = 16384;

PE_HD uint8_t sat8(int v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

// the chroma terms of one U, V sample, rounding half included
struct Chroma { int b, g, r; };
PE_HD Chroma chroma(int u, int v) {
    u -= 128; v -= 128;
    return {HALF + CUB * u, HALF + CVG * v + CUG * u, HALF + CVR * v};
}
PE_HD void yuv_px(int y, const Chroma& c, uint8_t* d) {
    const int yy = (y - 16 > 0 ? y - 16 : 0) * CY;
    d[0] = sat8((yy + c.b) >> SHIFT); d[1] = sat8((yy + c.g) >> SHIFT); d[2] = sat8((yy + c.r) >> SHIFT);
}
// a YUYV pair Y0 U Y1 V -> two BGR pixels
PE_HD void yuyv_pair(const uint8_t* s, uint8_t* d) {
    const Chroma c = chroma(s[1], s[3]);
    yuv_px(s[0], c, d); yuv_px(s[2], c, d + 3);
}
// a 4:2:0 quad: two luma samples of each of two rows and their shared U, V -> 2x2 BGR pixels (d0: upper row, d1: lower row)
PE_HD void quad420(const uint8_t* y0, const uint8_t* y1, int u, int v, uint8_t* d0, uint8_t* d1) {
    const Chroma c = chroma(u, v);
    yuv_px(y0[0], c, d0); yuv_px(y0[1], c, d0 + 3);
    yuv_px(y1[0], c, d1); yuv_px(y1[1], c, d1 + 3);
}
PE_HD void rgb_px(const uint8_t* s, uint8_t* d) { d[0] = s[2]; d[1] = s[1]; d[2] = s[0]; }

// A checked pe_pixel_format with its defaults resolved.  span: bytes from a frame's start to one past its last byte.
struct Layout {
    int format, w, h;
    long long pitch, chroma, span;
};

// Checks a format that arrived from outside the program; false and the reason in *err when it is unusable.  Every product is
// checked for overflow, so span is exact.
inline bool layout_of(const pe_pixel_format* f, Layout* L, std::string* err) {
    auto bad = [&](const std::string& m) { *err = m; return false; };
    if (!f) return bad("null pixel format");
    if (f->format < PE_PIX_BGR || f->format > PE_PIX_I420)
        return bad("pixel format " + std::to_string(f->format) + " is not one of PE_PIX_BGR .. PE_PIX_I420");
    const int w = f->width, h = f->height, fm = f->format;
    if (w <= 0 || h <= 0 || w > MAX_SIDE || h > MAX_SIDE)
        return bad("frame size " + std::to_string(w) + "x" + std::to_string(h) + " outside 1 .. " + std::to_string(MAX_SIDE));
    const bool planar = fm == PE_PIX_NV12 || fm == PE_PIX_I420;
    if ((fm == PE_PIX_YUYV || planar) && (w & 1)) return bad("odd width " + std::to_string(w) + ": chroma is shared by pixel pairs");
    if (planar && (h & 1)) return bad("odd height " + std::to_string(h) + ": 4:2:0 chroma is shared by row pairs");
    const long long row = (long long)w * (fm <= PE_PIX_RGB ? 3 : fm == PE_PIX_YUYV ? 2 : 1);
    const long long pitch = f->pitch ? f->pitch : row;
    if (pitch < row) return bad("pitch " + std::to_string(f->pitch) + " is below the row's " + std::to_string(row) + " bytes");
    if (fm == PE_PIX_I420 && (pitch & 1)) return bad("odd I420 pitch " + std::to_string(pitch) + ": chroma rows are pitch/2 apart");
    long long luma, span;
    if (__builtin_mul_overflow(pitch, (long long)h, &luma)) return bad("pitch " + std::to_string(pitch) + " overflows the frame size");
    long long chroma = 0;
    if (!planar) {
        span = luma - pitch + row;
    } else {
        chroma = f->chroma_offset ? f->chroma_offset : luma;
        if (chroma < luma)
            return bad("chroma_offset " + std::to_string(f->chroma_offset) + " lies inside the luma plane (pitch * height = " +
                       std::to_string(luma) + ")");
        // NV12: h/2 interleaved rows `pitch` apart; I420: U then V, h/2 rows each, pitch/2 apart
        const long long tail = fm == PE_PIX_NV12 ? pitch * (h / 2 - 1) + w : (pitch / 2) * (h - 1) + w / 2;
        if (__builtin_add_overflow(chroma, tail, &span)) return bad("chroma_offset " + std::to_string(chroma) + " overflows the frame size");
    }
    // staging a batch of host frames takes 64 spans: keep that product far from overflowing
    if (span >= (1LL << 56)) return bad("the frame spans " + std::to_string(span) + " bytes, more than 2^56");
    *L = {fm, w, h, pitch, chroma, span};
    return true;
}

}  // namespace pe_pix
