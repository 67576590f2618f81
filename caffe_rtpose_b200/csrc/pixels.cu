// Decoder-format frames -> tight uint8 BGR on the GPU (pe_forward_pixels), with cv::cvtColor's arithmetic from pixels.cuh.  One
// launch converts a batch: blockIdx.y is the frame, whose (pitched) source is read through the pointer table in the kernel
// parameters, so frames may sit in separate allocations - device memory the caller owns, or the engine's copies of host frames.
// One thread per 2x2 quad (NV12, I420), per pixel pair (YUYV) or per pixel (RGB).  BGR sources need no kernel: the engine copies
// them into place with cudaMemcpy2DAsync.
#include "kernels.h"
#include "pixels.cuh"

namespace pe {

template <int F>
__global__ void __launch_bounds__(256) pixels_to_bgr_kernel(PixArgs a) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x, f = blockIdx.y;
    const uint8_t* s = a.src[f];
    uint8_t* d = a.dst + (size_t)f * a.w * a.h * 3;
    if (F == PE_PIX_NV12 || F == PE_PIX_I420) {
        const int qw = a.w >> 1, hh = a.h >> 1;
        if (idx >= qw * hh) return;
        const int qx = idx % qw, qy = idx / qw;
        const uint8_t* y0 = s + 2LL * qy * a.pitch + 2 * qx;
        int u, v;
        if (F == PE_PIX_NV12) {
            const uint8_t* c = s + a.chroma + (long long)qy * a.pitch + 2 * qx;
            u = c[0]; v = c[1];
        } else {
            const long long cp = a.pitch >> 1;
            const uint8_t* c = s + a.chroma + qy * cp + qx;
            u = c[0]; v = c[cp * hh];
        }
        uint8_t* d0 = d + ((size_t)2 * qy * a.w + 2 * qx) * 3;
        pe_pix::quad420(y0, y0 + a.pitch, u, v, d0, d0 + (size_t)a.w * 3);
    } else if (F == PE_PIX_YUYV) {
        const int pw = a.w >> 1;
        if (idx >= pw * a.h) return;
        const int px = idx % pw, y = idx / pw;
        pe_pix::yuyv_pair(s + (long long)y * a.pitch + 4 * px, d + ((size_t)y * a.w + 2 * px) * 3);
    } else {
        if (idx >= a.w * a.h) return;
        const int x = idx % a.w, y = idx / a.w;
        pe_pix::rgb_px(s + (long long)y * a.pitch + 3 * x, d + (size_t)idx * 3);
    }
}

int launch_pixels_to_bgr(const PixArgs& a, int n, cudaStream_t st) {
    const int units = a.format == PE_PIX_RGB ? a.w * a.h : a.format == PE_PIX_YUYV ? (a.w / 2) * a.h : (a.w / 2) * (a.h / 2);
    const dim3 grid((units + 255) / 256, n);
    switch (a.format) {
        case PE_PIX_RGB: pixels_to_bgr_kernel<PE_PIX_RGB><<<grid, 256, 0, st>>>(a); break;
        case PE_PIX_YUYV: pixels_to_bgr_kernel<PE_PIX_YUYV><<<grid, 256, 0, st>>>(a); break;
        case PE_PIX_NV12: pixels_to_bgr_kernel<PE_PIX_NV12><<<grid, 256, 0, st>>>(a); break;
        case PE_PIX_I420: pixels_to_bgr_kernel<PE_PIX_I420><<<grid, 256, 0, st>>>(a); break;
        default: return 0;
    }
    return 1;
}

// the same loops on the host for frame src[0]: the reference the kernel is tested against (pe_pixels_to_bgr)
void pixels_to_bgr_host(const PixArgs& a) {
    const uint8_t* s = a.src[0];
    const size_t row = (size_t)a.w * 3;
    for (int y = 0; y < a.h; y++) {
        const uint8_t* sr = s + (long long)y * a.pitch;
        uint8_t* d = a.dst + y * row;
        switch (a.format) {
            case PE_PIX_BGR: memcpy(d, sr, row); break;
            case PE_PIX_RGB: for (int x = 0; x < a.w; x++) pe_pix::rgb_px(sr + 3 * x, d + 3 * x); break;
            case PE_PIX_YUYV: for (int x = 0; x < a.w; x += 2) pe_pix::yuyv_pair(sr + 2 * x, d + 3 * x); break;
            default:   // NV12 / I420: quads, two rows at a time
                if (y & 1) break;
                for (int x = 0; x < a.w; x += 2) {
                    int u, v;
                    if (a.format == PE_PIX_NV12) {
                        const uint8_t* c = s + a.chroma + (long long)(y / 2) * a.pitch + x;
                        u = c[0]; v = c[1];
                    } else {
                        const long long cp = a.pitch / 2;
                        const uint8_t* c = s + a.chroma + (y / 2) * cp + x / 2;
                        u = c[0]; v = c[cp * (a.h / 2)];
                    }
                    pe_pix::quad420(sr + x, sr + a.pitch + x, u, v, d + 3 * x, d + row + 3 * x);
                }
        }
    }
}

}  // namespace pe
