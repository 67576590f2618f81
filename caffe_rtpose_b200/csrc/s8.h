// Host quantisation of one output channel's weights for PE_PREC_S8X1 (engine.cu packs every channel with it, after the range
// ratios of its input channels are folded in):
//   sigma = max|w| / 127 in fp32,   q = clamp(rint(w / sigma), -127, 127) in fp32 (rint: ties to even),
// and an all-zero channel has sigma = 0 and q = 0.  The epilogue multiplies the s32 sum by sigma (times the range scales).
// Plain C++ without CUDA, so that a CPU test compiles it on its own.
#pragma once
#include <math.h>
#include <stddef.h>
#include <stdint.h>

namespace pe {

inline float s8_quantize_channel(const float* w, size_t n, int8_t* q) {
    float m = 0.f;
    for (size_t i = 0; i < n; i++) m = fmaxf(m, fabsf(w[i]));
    const float sigma = m / 127.f;
    for (size_t i = 0; i < n; i++) {
        float r = sigma > 0.f ? rintf(w[i] / sigma) : 0.f;
        r = fminf(fmaxf(r, -127.f), 127.f);
        q[i] = (int8_t)r;
    }
    return sigma;
}

// PE_PREC_S8X2: a 16-bit integer v in [-32768, 32639] as two s8 planes, hi = (v + 128) >> 8 (arithmetic shift) and lo = v - 256 hi,
// both in [-128, 127], so that v = 256 hi + lo exactly.  The kernels' epilogue and max pool split and merge the same way.
inline void s8x2_split(int v, int8_t* hi, int8_t* lo) {
    const int h = (v + 128) >> 8;
    *hi = (int8_t)h;
    *lo = (int8_t)(v - 256 * h);
}

// Host quantisation of one output channel's weights for PE_PREC_S8X2, as s8_quantize_channel with 16-bit integers:
//   sigma = max|w| / 32639 in fp32,   q = clamp(rint(w / sigma), -32639, 32639) in fp32,
// split into the planes hi[i], lo[i] (s8x2_split); an all-zero channel has sigma = 0 and q = 0.
inline float s8x2_quantize_channel(const float* w, size_t n, int8_t* hi, int8_t* lo) {
    float m = 0.f;
    for (size_t i = 0; i < n; i++) m = fmaxf(m, fabsf(w[i]));
    const float sigma = m / 32639.f;
    for (size_t i = 0; i < n; i++) {
        float r = sigma > 0.f ? rintf(w[i] / sigma) : 0.f;
        r = fminf(fmaxf(r, -32639.f), 32639.f);
        s8x2_split((int)r, hi + i, lo + i);
    }
    return sigma;
}

}  // namespace pe
