// The reference's full-resolution "resized_map" (ImResizeLayer, imresize_layer.cu:98-193) as a pure function of the
// stride-8 maps: shared by the post-processing kernels (post.cu) and the renderers (render.cu).  Bit-identical to the
// reference kernel (explicit round-to-nearest intrinsics in nvcc's contraction pattern).
#pragma once
#include "common.h"
#include "kernels.h"

namespace pe {

// ------------------------------------------------------------------------------------------------
// cubic_interpolation (imresize_layer.cu:8-18) with nvcc's contraction pattern (see oracle.cpp)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float cubic_ref(float v0, float v1, float v2, float v3, float d) {
    const float h = __fmul_rn(0.5f, v0);
    const float a = __fmaf_rn(v3, 0.5f, __fmaf_rn(v2, -1.5f, __fmaf_rn(v1, 1.5f, -h)));
    const float t1 = __fmul_rn(__fmul_rn(__fmul_rn(a, d), d), d);
    const double b = __fma_rn((double)v3, -0.5, __fma_rn((double)v2, 2.0, (double)__fmaf_rn(v1, -2.5f, v0)));
    const double dd = (double)d;
    double acc = __fma_rn(dd, __dmul_rn(dd, b), (double)t1);
    const float t3 = __fmul_rn(d, __fmaf_rn(v2, 0.5f, -h));
    acc = __dadd_rn(acc, (double)t3);
    acc = __dadd_rn(acc, (double)v1);
    return __double2float_rn(acc);
}

// cubic_ref split into the part that depends only on the four taps and the part that depends on the fraction d: full-resolution
// neighbours along one axis share their taps (8 outputs per source interval at stride 8), so a thread that walks along the axis
// evaluates cubic_prep once per interval and cubic_eval per output - the same operations on the same operands in the same order
// as cubic_ref (bit-identical), with 3 instead of 8 float<->double conversions and ~12 instead of ~30 arithmetic instructions per output.
struct CubicTaps { float a, c; double b, v1; };
__device__ __forceinline__ CubicTaps cubic_prep(float v0, float v1, float v2, float v3) {
    CubicTaps t;
    const float h = __fmul_rn(0.5f, v0);
    t.a = __fmaf_rn(v3, 0.5f, __fmaf_rn(v2, -1.5f, __fmaf_rn(v1, 1.5f, -h)));
    t.b = __fma_rn((double)v3, -0.5, __fma_rn((double)v2, 2.0, (double)__fmaf_rn(v1, -2.5f, v0)));
    t.c = __fmaf_rn(v2, 0.5f, -h);
    t.v1 = (double)v1;
    return t;
}
__device__ __forceinline__ float cubic_eval(const CubicTaps& t, float d, double dd) {   // dd == (double)d
    const float t1 = __fmul_rn(__fmul_rn(__fmul_rn(t.a, d), d), d);
    double acc = __fma_rn(dd, __dmul_rn(dd, t.b), (double)t1);
    acc = __dadd_rn(acc, (double)__fmul_rn(d, t.c));
    acc = __dadd_rn(acc, t.v1);
    return __double2float_rn(acc);
}

struct FullRes {
    const float* maps;     // this frame: [copies][C][h8][w8]
    const AxisTap* xt;     // [S][net_w]
    const AxisTap* yt;     // [S][net_h]
    const FlipTap* flip;   // [C]
    int S, copies, C, h8, w8, net_w, net_h;
    float inv_div;         // (float)copies
};

// The average's copies: n < S is scale n, n >= S the mirror of scale n - S (the flip test).  A mirrored copy contributes
// sign[c] * R(M')[perm[c]][y][net_w-1-x]: its own channel and sign, and the scale's x taps read backwards.  Every reader of the
// full-resolution maps goes through these three, so the average is defined here only.
__device__ __forceinline__ const float* copy_plane(const FullRes& fr, int n, int c, float* sign) {
    *sign = 1.f;
    if (n >= fr.S) {
        const FlipTap f = fr.flip[c];
        c = f.ch;
        *sign = f.sign;
    }
    return fr.maps + ((size_t)n * fr.C + c) * fr.h8 * fr.w8;
}
__device__ __forceinline__ AxisTap copy_xtap(const FullRes& fr, int n, int x) {
    return n < fr.S ? fr.xt[n * fr.net_w + x] : fr.xt[(n - fr.S) * fr.net_w + fr.net_w - 1 - x];
}
__device__ __forceinline__ const AxisTap* copy_ytab(const FullRes& fr, int n) { return fr.yt + (n < fr.S ? n : n - fr.S) * fr.net_h; }

// resized_map[c][y][x] of the reference, evaluated from the stride-8 maps; with the flip test the average over 2S copies
__device__ __forceinline__ float fullres_at(const FullRes& fr, int c, int y, int x) {
    float sum = 0.f;
    for (int n = 0; n < fr.copies; n++) {
        float sign;
        const float* s = copy_plane(fr, n, c, &sign);
        const AxisTap ax = copy_xtap(fr, n, x);
        const AxisTap ay = copy_ytab(fr, n)[y];
        const float* r0 = s + (size_t)ay.i0 * fr.w8;
        const float* r1 = s + (size_t)ay.i1 * fr.w8;
        const float* r2 = s + (size_t)ay.i2 * fr.w8;
        const float* r3 = s + (size_t)ay.i3 * fr.w8;
        const float t0 = cubic_ref(__ldg(r0 + ax.i0), __ldg(r0 + ax.i1), __ldg(r0 + ax.i2), __ldg(r0 + ax.i3), ax.d);
        const float t1 = cubic_ref(__ldg(r1 + ax.i0), __ldg(r1 + ax.i1), __ldg(r1 + ax.i2), __ldg(r1 + ax.i3), ax.d);
        const float t2 = cubic_ref(__ldg(r2 + ax.i0), __ldg(r2 + ax.i1), __ldg(r2 + ax.i2), __ldg(r2 + ax.i3), ax.d);
        const float t3 = cubic_ref(__ldg(r3 + ax.i0), __ldg(r3 + ax.i1), __ldg(r3 + ax.i2), __ldg(r3 + ax.i3), ax.d);
        sum = __fadd_rn(sum, __fmul_rn(sign, cubic_ref(t0, t1, t2, t3, ay.d)));   // sign is +-1: exact
    }
    return __fdiv_rn(sum, fr.inv_div);
}

__device__ __forceinline__ FullRes make_fullres(const PostDev& pd, int frame) {
    FullRes fr;
    fr.S = pd.p.num_scales; fr.copies = pd.copies; fr.C = pd.p.num_maps; fr.h8 = pd.p.h8; fr.w8 = pd.p.w8;
    fr.net_w = pd.p.net_w; fr.net_h = pd.p.net_h;
    fr.maps = pd.maps + (size_t)frame * fr.copies * fr.C * fr.h8 * fr.w8;
    fr.xt = pd.xtab; fr.yt = pd.ytab; fr.flip = pd.flip;
    fr.inv_div = (float)fr.copies;
    return fr;
}

}  // namespace pe
