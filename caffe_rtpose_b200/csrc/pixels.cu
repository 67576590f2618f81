// Decoder-format frames -> tight uint8 BGR on the GPU (pe_forward_pixels), with the arithmetic of pixels.cuh.  One launch converts
// a batch: blockIdx.y is the frame, whose (pitched) source is read through the pointer table in the kernel parameters, so frames
// may sit in separate allocations - device memory the caller owns, or the engine's copies of host frames.  One kernel instance per
// memory layout, with the chroma order and the colour constants in the arguments: one thread per 2x2 quad (4:2:0), per pixel pair
// (4:2:2) or per pixel (RGB, RGBP).  BGR sources need no kernel: the engine copies them into place with cudaMemcpy2DAsync.
#include "kernels.h"
#include "pixels.cuh"

namespace pe {

enum PixLayout { PACKED422, SEMI420_8, SEMI420_16, PLANAR420, PACKED_RGB, PLANAR_RGB };

static int layout_kind(int format) {
    switch (format) {
        case PE_PIX_YUYV: case PE_PIX_UYVY: return PACKED422;
        case PE_PIX_NV12: case PE_PIX_NV21: return SEMI420_8;
        case PE_PIX_P016: return SEMI420_16;
        case PE_PIX_I420: case PE_PIX_YV12: return PLANAR420;
        case PE_PIX_RGB: return PACKED_RGB;
        case PE_PIX_RGBP: return PLANAR_RGB;
        default: return -1;
    }
}

// the U, V sample of 4:2:0 quad (qx, qy) of frame s: interleaved (NV12, NV21, P016) or in two planes (I420, YV12); sw: V first
template <typename S, bool SEMI>
PE_HD void chroma420(const uint8_t* s, const PixArgs& a, int qx, int qy, bool sw, int* u, int* v) {
    if (SEMI) {
        const S* c = (const S*)(s + a.chroma + qy * a.pitch) + 2 * qx;
        *u = c[sw]; *v = c[!sw];
    } else {
        const long long cp = a.pitch >> 1, plane = cp * (a.h >> 1);
        const uint8_t* c = s + a.chroma + qy * cp + qx;
        *u = c[sw ? plane : 0]; *v = c[sw ? 0 : plane];
    }
}

template <int K>
__global__ void __launch_bounds__(256) pixels_to_bgr_kernel(PixArgs a) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x, f = blockIdx.y;
    const uint8_t* s = a.src[f];
    uint8_t* d = a.dst + (size_t)f * a.w * a.h * 3;
    const bool sw = pe_pix::swapped(a.format);
    if (K == SEMI420_8 || K == SEMI420_16 || K == PLANAR420) {
        using S = typename std::conditional<K == SEMI420_16, uint16_t, uint8_t>::type;
        const int qw = a.w >> 1, hh = a.h >> 1;
        if (idx >= qw * hh) return;
        const int qx = idx % qw, qy = idx / qw;
        const S* y0 = (const S*)(s + 2LL * qy * a.pitch) + 2 * qx;
        int u, v;
        chroma420<S, K != PLANAR420>(s, a, qx, qy, sw, &u, &v);
        uint8_t* d0 = d + ((size_t)2 * qy * a.w + 2 * qx) * 3;
        pe_pix::quad420<S>(a.col, y0, (const S*)((const uint8_t*)y0 + a.pitch), u, v, d0, d0 + (size_t)a.w * 3);
    } else if (K == PACKED422) {
        const int pw = a.w >> 1;
        if (idx >= pw * a.h) return;
        const int px = idx % pw, y = idx / pw;
        pe_pix::pair422(a.col, s + (long long)y * a.pitch + 4 * px, sw, d + ((size_t)y * a.w + 2 * px) * 3);
    } else {
        if (idx >= a.w * a.h) return;
        const int x = idx % a.w, y = idx / a.w;
        if (K == PACKED_RGB) pe_pix::rgb_px(s + (long long)y * a.pitch + 3 * x, d + (size_t)idx * 3);
        else pe_pix::rgbp_px(s + (long long)y * a.pitch + x, a.chroma, d + (size_t)idx * 3);
    }
}

int launch_pixels_to_bgr(const PixArgs& a, int n, cudaStream_t st) {
    const int k = layout_kind(a.format);
    const int units = k == PACKED_RGB || k == PLANAR_RGB ? a.w * a.h : k == PACKED422 ? (a.w / 2) * a.h : (a.w / 2) * (a.h / 2);
    const dim3 grid((units + 255) / 256, n);
    switch (k) {
        case PACKED422: pixels_to_bgr_kernel<PACKED422><<<grid, 256, 0, st>>>(a); break;
        case SEMI420_8: pixels_to_bgr_kernel<SEMI420_8><<<grid, 256, 0, st>>>(a); break;
        case SEMI420_16: pixels_to_bgr_kernel<SEMI420_16><<<grid, 256, 0, st>>>(a); break;
        case PLANAR420: pixels_to_bgr_kernel<PLANAR420><<<grid, 256, 0, st>>>(a); break;
        case PACKED_RGB: pixels_to_bgr_kernel<PACKED_RGB><<<grid, 256, 0, st>>>(a); break;
        case PLANAR_RGB: pixels_to_bgr_kernel<PLANAR_RGB><<<grid, 256, 0, st>>>(a); break;
        default: return 0;
    }
    return 1;
}

// the same loops on the host for frame src[0]: the reference the kernel is tested against (pe_pixels_to_bgr)
void pixels_to_bgr_host(const PixArgs& a) {
    const uint8_t* s = a.src[0];
    const size_t row = (size_t)a.w * 3;
    const int k = layout_kind(a.format);
    const bool sw = pe_pix::swapped(a.format);
    for (int y = 0; y < a.h; y++) {
        const uint8_t* sr = s + (long long)y * a.pitch;
        uint8_t* d = a.dst + y * row;
        switch (k) {
            case PACKED_RGB: for (int x = 0; x < a.w; x++) pe_pix::rgb_px(sr + 3 * x, d + 3 * x); break;
            case PLANAR_RGB: for (int x = 0; x < a.w; x++) pe_pix::rgbp_px(sr + x, a.chroma, d + 3 * x); break;
            case PACKED422: for (int x = 0; x < a.w; x += 2) pe_pix::pair422(a.col, sr + 2 * x, sw, d + 3 * x); break;
            case SEMI420_8: case SEMI420_16: case PLANAR420:   // quads, two rows at a time
                if (y & 1) break;
                for (int x = 0; x < a.w; x += 2) {
                    int u, v;
                    if (k == SEMI420_16) {
                        chroma420<uint16_t, true>(s, a, x / 2, y / 2, sw, &u, &v);
                        const uint16_t* y0 = (const uint16_t*)sr + x;
                        pe_pix::quad420<uint16_t>(a.col, y0, (const uint16_t*)(sr + a.pitch) + x, u, v, d + 3 * x, d + row + 3 * x);
                        continue;
                    }
                    if (k == SEMI420_8) chroma420<uint8_t, true>(s, a, x / 2, y / 2, sw, &u, &v);
                    else chroma420<uint8_t, false>(s, a, x / 2, y / 2, sw, &u, &v);
                    pe_pix::quad420<uint8_t>(a.col, sr + x, sr + a.pitch + x, u, v, d + 3 * x, d + row + 3 * x);
                }
                break;
            default: memcpy(d, sr, row);   // BGR
        }
    }
}

}  // namespace pe
