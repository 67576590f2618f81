// Decoder-format frames (pe_pixel_format, poseengine.h) -> uint8 BGR: the per-pixel arithmetic shared by the CUDA kernel
// (pixels.cu), the host reference pe_pixels_to_bgr and the camera's pe_yuyv_to_bgr, and the layout checks of every entry point
// that reads such frames.
//
// OpenCV's YUV -> BGR conversions (imgproc color_yuv, COLOR_YUV2BGR_YUYV / _UYVY / _NV12 / _NV21 / _I420 / _YV12) share one
// ITU-R BT.601 studio-range fixed-point formula: 20-bit constants, max(Y - 16, 0) * CY plus the chroma terms of the pixel's
// (nearest-neighbour) chroma sample, >> 20, saturated to uint8.  4:2:2 pairs and 4:2:0 quads differ only in how many luma samples
// share one chroma sample.  Every matrix and range here is that formula with other constants (Colour):
//   - full range has no luma offset and CY = 2^20, so the sum is Y + ((chroma terms + 2^19) >> 20).  OpenCV's COLOR_YCrCb2BGR
//     (full-range BT.601) is Y + ((chroma terms + 2^13) >> 14) with 14-bit constants; the same constants << 6 give the same bytes.
//   - BT.709 constants are rounded to 20 bits from Kr = 0.2126, Kb = 0.0722 (Kg = 1 - Kr - Kb = 0.7152):
//       R = Y' + 2 (1 - Kr) V'                            = Y' + 1.5748 V'
//       G = Y' - 2 Kb (1 - Kb) / Kg U' - 2 Kr (1 - Kr) / Kg V' = Y' - 0.187324 U' - 0.468124 V'
//       B = Y' + 2 (1 - Kb) U'                            = Y' + 1.8556 U'
//     full range:   Y' = Y, U' = U - 128, V' = V - 128;
//     studio range: Y' = max(Y - 16, 0) * 255/219, U' = (U - 128) * 255/224, V' likewise, so CY = round(2^20 * 255/219) and
//                   each chroma constant carries the factor 255/224.
//     Luma below 16 counts as black in studio range, as OpenCV's BT.601 formula has it.
//   - 16-bit samples (PE_PIX_P016, significant bits at the top) run the same formula with 8 more fractional bits: offsets 16*256
//     and 128*256, >> 28, in 64-bit sums.  A sample v << 8 therefore converts exactly as the 8-bit sample v.
#pragma once
#include <stdint.h>

#include <string>
#include <type_traits>

#include "../../include/poseengine.h"

#ifndef PE_HD
#ifdef __CUDACC__
#define PE_HD __host__ __device__ __forceinline__
#else
#define PE_HD inline
#endif
#endif

namespace pe_pix {

constexpr int SHIFT = 20, MAX_SIDE = 16384;

// one matrix and range: the luma offset (16 studio, 0 full) and the 20-bit constants
struct Colour { int yoff, cy, cub, cug, cvg, cvr; };
constexpr Colour BT601_STUDIO = {16, 1220542, 2116026, -409993, -852492, 1673527};       // OpenCV's (1.164, 2.018, ...) * 2^20
constexpr Colour BT601_FULL = {0, 1 << 20, 29049 * 64, -5636 * 64, -11698 * 64, 22987 * 64};   // OpenCV's YCrCb2BGR 14-bit << 6
constexpr Colour BT709_STUDIO = {16, 1220945, 2215014, -223607, -558796, 1879825};
constexpr Colour BT709_FULL = {0, 1 << 20, 1945738, -196424, -490864, 1651297};

inline Colour colour_of(int format) {
    const bool full = format & PE_PIX_FLAG_FULL_RANGE;
    return format & PE_PIX_FLAG_BT709 ? (full ? BT709_FULL : BT709_STUDIO) : (full ? BT601_FULL : BT601_STUDIO);
}

PE_HD uint8_t sat8(int v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

// S: the sample type, uint8_t or uint16_t.  16-bit samples have E = 8 more fractional bits and need 64-bit sums.
template <typename S> using Acc = typename std::conditional<sizeof(S) == 1, int, long long>::type;
template <typename S> struct Chroma { Acc<S> b, g, r; };

// the chroma terms of one U, V sample, rounding half included
template <typename S> PE_HD Chroma<S> chroma(const Colour& m, int u, int v) {
    constexpr int E = 8 * (sizeof(S) - 1);
    const Acc<S> half = (Acc<S>)1 << (SHIFT + E - 1);
    u -= 128 << E; v -= 128 << E;
    return {half + (Acc<S>)m.cub * u, half + (Acc<S>)m.cvg * v + (Acc<S>)m.cug * u, half + (Acc<S>)m.cvr * v};
}
template <typename S> PE_HD void yuv_px(const Colour& m, int y, const Chroma<S>& c, uint8_t* d) {
    constexpr int E = 8 * (sizeof(S) - 1);
    y -= m.yoff << E;
    const Acc<S> yy = (Acc<S>)(y > 0 ? y : 0) * m.cy;
    d[0] = sat8((int)((yy + c.b) >> (SHIFT + E)));
    d[1] = sat8((int)((yy + c.g) >> (SHIFT + E)));
    d[2] = sat8((int)((yy + c.r) >> (SHIFT + E)));
}
// a packed 4:2:2 pair -> two BGR pixels: Y0 U Y1 V (YUYV, yo = 0) or U Y0 V Y1 (UYVY, yo = 1)
PE_HD void pair422(const Colour& m, const uint8_t* s, int yo, uint8_t* d) {
    const Chroma<uint8_t> c = chroma<uint8_t>(m, s[1 - yo], s[3 - yo]);
    yuv_px(m, s[yo], c, d); yuv_px(m, s[yo + 2], c, d + 3);
}
// a 4:2:0 quad: two luma samples of each of two rows and their shared U, V -> 2x2 BGR pixels (d0: upper row, d1: lower row)
template <typename S> PE_HD void quad420(const Colour& m, const S* y0, const S* y1, int u, int v, uint8_t* d0, uint8_t* d1) {
    const Chroma<S> c = chroma<S>(m, u, v);
    yuv_px(m, y0[0], c, d0); yuv_px(m, y0[1], c, d0 + 3);
    yuv_px(m, y1[0], c, d1); yuv_px(m, y1[1], c, d1 + 3);
}
PE_HD void rgb_px(const uint8_t* s, uint8_t* d) { d[0] = s[2]; d[1] = s[1]; d[2] = s[0]; }
// one pixel of three planes R, G, B that start `plane` bytes apart
PE_HD void rgbp_px(const uint8_t* s, long long plane, uint8_t* d) { d[0] = s[2 * plane]; d[1] = s[plane]; d[2] = s[0]; }

// the format without its colour flags
PE_HD int base_of(int format) { return format & 0xff; }
// UYVY: luma second; NV21, YV12: V before U
PE_HD bool swapped(int base) { return base == PE_PIX_UYVY || base == PE_PIX_NV21 || base == PE_PIX_YV12; }
inline bool is_yuv(int base) { return base != PE_PIX_BGR && base != PE_PIX_RGB && base != PE_PIX_RGBP; }

// A checked pe_pixel_format with its defaults resolved.  format: PE_PIX_* without flags; chroma: the first chroma plane's offset
// (RGBP: the distance between planes); span: bytes from a frame's start to one past its last byte.
struct Layout {
    int format, w, h;
    Colour col;
    long long pitch, chroma, span;
};

// Checks a format that arrived from outside the program; false and the reason in *err when it is unusable.  Every product is
// checked for overflow, so span is exact.
inline bool layout_of(const pe_pixel_format* f, Layout* L, std::string* err) {
    auto bad = [&](const std::string& m) { *err = m; return false; };
    if (!f) return bad("null pixel format");
    const int fm = base_of(f->format), flags = f->format & ~0xff;
    if (f->format < 0 || fm > PE_PIX_RGBP || (fm > PE_PIX_I420 && fm < PE_PIX_NV21))
        return bad("pixel format " + std::to_string(f->format) + " is not one of PE_PIX_BGR .. PE_PIX_I420, PE_PIX_NV21 .. PE_PIX_RGBP");
    if (flags & ~(PE_PIX_FLAG_BT709 | PE_PIX_FLAG_FULL_RANGE))
        return bad("pixel format " + std::to_string(f->format) + " has unknown flag bits (only PE_PIX_FLAG_BT709 and "
                   "PE_PIX_FLAG_FULL_RANGE exist)");
    if (flags && !is_yuv(fm))
        return bad("pixel format " + std::to_string(f->format) + ": the colour flags apply to YUV formats, not to BGR, RGB or RGBP");
    const int w = f->width, h = f->height;
    if (w <= 0 || h <= 0 || w > MAX_SIDE || h > MAX_SIDE)
        return bad("frame size " + std::to_string(w) + "x" + std::to_string(h) + " outside 1 .. " + std::to_string(MAX_SIDE));
    const bool packed422 = fm == PE_PIX_YUYV || fm == PE_PIX_UYVY;
    const bool semi = fm == PE_PIX_NV12 || fm == PE_PIX_NV21 || fm == PE_PIX_P016, planar = fm == PE_PIX_I420 || fm == PE_PIX_YV12;
    const bool p016 = fm == PE_PIX_P016;
    if ((packed422 || semi || planar) && (w & 1)) return bad("odd width " + std::to_string(w) + ": chroma is shared by pixel pairs");
    if ((semi || planar) && (h & 1)) return bad("odd height " + std::to_string(h) + ": 4:2:0 chroma is shared by row pairs");
    const long long row = (long long)w * (fm <= PE_PIX_RGB ? 3 : packed422 || p016 ? 2 : 1);
    const long long pitch = f->pitch ? f->pitch : row;
    if (pitch < row) return bad("pitch " + std::to_string(f->pitch) + " is below the row's " + std::to_string(row) + " bytes");
    if (planar && (pitch & 1))
        return bad(std::string(fm == PE_PIX_I420 ? "odd I420" : "odd YV12") + " pitch " + std::to_string(pitch) + ": chroma rows are pitch/2 apart");
    if (p016 && (pitch & 1)) return bad("odd P016 pitch " + std::to_string(pitch) + ": samples are 2 bytes");
    long long luma, span;
    if (__builtin_mul_overflow(pitch, (long long)h, &luma)) return bad("pitch " + std::to_string(pitch) + " overflows the frame size");
    long long chroma = 0;
    if (!semi && !planar && fm != PE_PIX_RGBP) {
        span = luma - pitch + row;
    } else {
        chroma = f->chroma_offset ? f->chroma_offset : luma;
        if (chroma < luma)
            return bad("chroma_offset " + std::to_string(f->chroma_offset) + " lies inside the " +
                       (fm == PE_PIX_RGBP ? "R plane, so the RGBP planes overlap" : "luma plane") + " (pitch * height = " +
                       std::to_string(luma) + ")");
        if (p016 && (chroma & 1)) return bad("odd P016 chroma_offset " + std::to_string(chroma) + ": samples are 2 bytes");
        // NV12 / NV21 / P016: h/2 interleaved rows `pitch` apart; I420 / YV12: two planes of h/2 rows pitch/2 apart; RGBP: two more
        // planes like the first, `chroma` apart
        long long start = chroma, tail;
        if (fm == PE_PIX_RGBP) {
            if (__builtin_mul_overflow(chroma, 2LL, &start)) return bad("chroma_offset " + std::to_string(chroma) + " overflows the frame size");
            tail = luma - pitch + row;
        } else {
            tail = semi ? pitch * (h / 2 - 1) + row : (pitch / 2) * (h - 1) + w / 2;
        }
        if (__builtin_add_overflow(start, tail, &span)) return bad("chroma_offset " + std::to_string(chroma) + " overflows the frame size");
    }
    // staging a batch of host frames takes 64 spans: keep that product far from overflowing
    if (span >= (1LL << 56)) return bad("the frame spans " + std::to_string(span) + " bytes, more than 2^56");
    *L = {fm, w, h, colour_of(f->format), pitch, chroma, span};
    return true;
}

}  // namespace pe_pix
