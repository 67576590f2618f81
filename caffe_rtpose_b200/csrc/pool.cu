// 2x2 stride-2 MAX pooling (ceil dims), channel-slice copy and layout conversion on the flat padded layout.
//
// Pooling semantics: src/caffe/layers/pooling_layer.cpp:90-93 (ceil), :128-187 (max over the window clipped
// to the image).  Activations are either fp32 [M][C] or 16-bit "planes" whose SUM is the value (split
// precision for the wgmma conv, see conv_tc.cu); the max is taken on the reconstructed value and the
// winner's planes are copied, which keeps the split exact.
#include "common.h"
#include "kernels.h"

namespace pe {

__global__ void __launch_bounds__(256) pool_f32_kernel(PoolArgs a) {
    const int cv = a.C / 4;  // float4 groups
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long rows_out = (long long)a.N * a.Hso * a.Wpo;
    if (idx >= rows_out * cv) return;
    const int g = (int)(idx % cv);
    const long long mo = idx / cv;
    const int n = (int)(mo / ((long long)a.Hso * a.Wpo));
    const int rem = (int)(mo % ((long long)a.Hso * a.Wpo));
    const int yo = rem / a.Wpo, xo = rem % a.Wpo;
    if (xo >= a.Wo || yo >= a.Ho) return;
    float4 best = make_float4(-3.402823466e+38F, -3.402823466e+38F, -3.402823466e+38F, -3.402823466e+38F);
    for (int dy = 0; dy < 2; dy++)
        for (int dx = 0; dx < 2; dx++) {
            const int yi = 2 * yo + dy, xi = 2 * xo + dx;
            if (yi < a.Hi && xi < a.Wi) {
                const long long mi = ((long long)n * a.Hsi + yi) * a.Wpi + xi;
                const float4 v = *((const float4*)((const float*)a.in + mi * a.C) + g);
                best.x = v.x > best.x ? v.x : best.x; best.y = v.y > best.y ? v.y : best.y;
                best.z = v.z > best.z ? v.z : best.z; best.w = v.w > best.w ? v.w : best.w;
            }
        }
    *((float4*)((float*)a.out + mo * a.C) + g) = best;
}

template <int PLANES, bool F16>
__global__ void __launch_bounds__(256) pool_planes_kernel(PoolArgs a) {
    const unsigned cv = a.C / 8;  // 8 channels (16 bytes) per thread and plane
    const int n = blockIdx.y;     // grid.y = image; 32-bit index math inside an image
    const unsigned per_img = (unsigned)a.Hso * (unsigned)a.Wpo;
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= per_img * cv) return;
    const int g = (int)(idx % cv);
    const unsigned rem = idx / cv;
    const int yo = (int)(rem / (unsigned)a.Wpo), xo = (int)(rem % (unsigned)a.Wpo);
    if (xo >= a.Wo || yo >= a.Ho) return;
    const long long mo = (long long)n * per_img + rem;
    // issue all window loads first (4 positions x PLANES x 16 B in flight per thread), then reduce
    uint4 v[4][PLANES];
    bool ok[4];
#pragma unroll
    for (int w = 0; w < 4; w++) {
        const int yi = 2 * yo + (w >> 1), xi = 2 * xo + (w & 1);
        ok[w] = yi < a.Hi && xi < a.Wi;
        const long long mi = ((long long)n * a.Hsi + (ok[w] ? yi : 2 * yo)) * a.Wpi + (ok[w] ? xi : 2 * xo);
#pragma unroll
        for (int p = 0; p < PLANES; p++)
            v[w][p] = __ldg((const uint4*)((const __nv_bfloat16*)a.in + (size_t)p * a.in_plane + mi * a.C) + g);
    }
    uint4 o[PLANES];
#pragma unroll
    for (int j = 0; j < 8; j++) {
        float best = -3.402823466e+38F;
        int bw = 0;
#pragma unroll
        for (int w = 0; w < 4; w++) {
            float sum = 0.f;
#pragma unroll
            for (int p = 0; p < PLANES; p++) sum += plane_to_float<F16>(((const uint16_t*)&v[w][p])[j]);
            if (ok[w] && sum > best) { best = sum; bw = w; }
        }
#pragma unroll
        for (int p = 0; p < PLANES; p++) {
            uint16_t h = ((const uint16_t*)&v[0][p])[j];
            if (bw == 1) h = ((const uint16_t*)&v[1][p])[j];
            if (bw == 2) h = ((const uint16_t*)&v[2][p])[j];
            if (bw == 3) h = ((const uint16_t*)&v[3][p])[j];
            ((uint16_t*)&o[p])[j] = h;
        }
    }
#pragma unroll
    for (int p = 0; p < PLANES; p++)
        *((uint4*)((__nv_bfloat16*)a.out + (size_t)p * a.out_plane + mo * a.C) + g) = o[p];
}

int launch_pool(const PoolArgs& a, cudaStream_t st) {
    const long long rows_out = (long long)a.N * a.Hso * a.Wpo;
    const PlaneFmt f = a.fmt;
    if (f.planes == 0) {
        const long long total = rows_out * (a.C / 4);
        pool_f32_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(a);
    } else {
        const unsigned per = (unsigned)a.Hso * a.Wpo * (a.C / 8);
        const dim3 grid((per + 255) / 256, a.N);
        if (f.planes == 1 && f.f16) pool_planes_kernel<1, true><<<grid, 256, 0, st>>>(a);
        else if (f.planes == 1) pool_planes_kernel<1, false><<<grid, 256, 0, st>>>(a);
        else if (f.planes == 2) pool_planes_kernel<2, PARITY_F16><<<grid, 256, 0, st>>>(a);
        else pool_planes_kernel<3, false><<<grid, 256, 0, st>>>(a);
    }
    return 1;
}

// copy the first `channels` channels of every row (all planes); 16-byte chunks
__global__ void __launch_bounds__(256) copy_channels_kernel(CopyArgs a) {
    const int chunks = a.channels * a.elem_bytes / 16;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int np = a.fmt.planes == 0 ? 1 : a.fmt.planes;
    if (idx >= a.M * chunks * np) return;
    const int ch = (int)(idx % chunks);
    const long long r = idx / chunks;
    const long long row = r % a.M;
    const int p = (int)(r / a.M);
    const size_t off = ((size_t)p * a.plane + (size_t)row * a.pitch) * a.elem_bytes + (size_t)ch * 16;
    *(uint4*)((char*)a.dst + off) = *(const uint4*)((const char*)a.src + off);
}
int launch_copy_channels(const CopyArgs& a, cudaStream_t st) {
    const int chunks = a.channels * a.elem_bytes / 16;
    const long long total = a.M * chunks * (a.fmt.planes == 0 ? 1 : a.fmt.planes);
    copy_channels_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(a);
    return 1;
}

__global__ void __launch_bounds__(256) act_to_nchw_kernel(const void* act, int pitch, int coff, int c, long long plane,
                                                          PlaneFmt fmt, Geo g, float scale, float* out) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)g.N * c * g.H * g.W;
    if (idx >= total) return;
    const int x = (int)(idx % g.W);
    const int y = (int)((idx / g.W) % g.H);
    const int ch = (int)((idx / ((long long)g.W * g.H)) % c);
    const int n = (int)(idx / ((long long)g.W * g.H * c));
    const long long m = ((long long)n * g.Hs + y) * g.Wp + x;
    float v = 0.f;
    if (fmt.planes == 0) v = ((const float*)act)[m * pitch + coff + ch];
    else for (int p = 0; p < fmt.planes; p++) {
        const uint16_t h = ((const uint16_t*)act)[p * plane + m * pitch + coff + ch];
        v += fmt.f16 ? plane_to_float<true>(h) : plane_to_float<false>(h);
    }
    out[idx] = v * scale;   // a power of two: exact
}
int launch_act_to_nchw(const void* act, int pitch, int coff, int c, long long plane, PlaneFmt fmt, const Geo& g, float scale,
                       float* out, cudaStream_t st) {
    const long long total = (long long)g.N * c * g.H * g.W;
    act_to_nchw_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(act, pitch, coff, c, plane, fmt, g, scale, out);
    return 1;
}

}  // namespace pe
