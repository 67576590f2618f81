// Frame -> network input on the GPU.
//
// Replaces the single-threaded host loop of getFrameFromCam (examples/rtpose/rtpose.cpp:508-518):
//   per scale i: cv::resize(display_img, (tw,th), INTER_AREA)  ->  process_and_pad_image(..., normalize=1)
//   (rtpose.cpp:239-269: centre pad with zeros, v/256 - 0.5, planar BGR), followed by a 2.9 MB/scale H2D copy.
// Here the uint8 display image is uploaded once (2.76 MB) and two kernels produce the conv stack's input:
//   1. area_resize_kernel  - OpenCV's INTER_AREA arithmetic (resizeArea_<uchar,float,float> /
//      resizeAreaFast_), bit-exact: float accumulation in table order, no FMA, round-half-even saturate;
//   2. input_im2col_kernel - pad + normalise + gather the 3x3x3 patch of every pixel, so that conv1_1
//      becomes a K=27 GEMM on the same implicit-GEMM kernel as every other layer.
#include "common.h"
#include "kernels.h"

namespace pe {

__global__ void __launch_bounds__(256) area_resize_kernel(PreArgs a) {
    const int s = blockIdx.y, f = blockIdx.z;
    const AreaTab t = a.tab[s];
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= t.tw * t.th) return;
    const int dx = idx % t.tw, dy = idx / t.tw;
    const uint8_t* src = a.frames + (size_t)f * a.disp_h * a.disp_w * 3;
    uint8_t* dst = a.resized + ((size_t)(f * a.S + s) * a.net_h * a.net_w + (size_t)dy * t.tw + dx) * 3;
    if (t.tw == a.disp_w && t.th == a.disp_h) {  // cv::resize with equal sizes copies
        const uint8_t* p = src + ((size_t)dy * a.disp_w + dx) * 3;
        dst[0] = p[0]; dst[1] = p[1]; dst[2] = p[2];
        return;
    }
    if (t.linear) {   // one axis enlarges: OpenCV's fixed-point bilinear with area-mode positions (11-bit coefficients)
        const int* lx = t.lin_x + dx * 3;
        const int* ly = t.lin_y + dy * 3;
        const int x0 = lx[0], x1 = min(x0 + 1, a.disp_w - 1), y0 = ly[0], y1 = min(y0 + 1, a.disp_h - 1);
        const uint8_t* r0 = src + (size_t)y0 * a.disp_w * 3;
        const uint8_t* r1 = src + (size_t)y1 * a.disp_w * 3;
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const int h0 = r0[x0 * 3 + c] * lx[1] + r0[x1 * 3 + c] * lx[2];
            const int h1 = r1[x0 * 3 + c] * lx[1] + r1[x1 * 3 + c] * lx[2];
            const int v = ((ly[1] * (h0 >> 4)) >> 16) + ((ly[2] * (h1 >> 4)) >> 16);
            dst[c] = (uint8_t)min(max((v + 2) >> 2, 0), 255);
        }
        return;
    }
    if (t.fast) {  // integer ratios: resizeAreaFast_ (2x2 uses the (sum+2)>>2 SIMD specialisation)
        int s0 = 0, s1 = 0, s2 = 0;
        for (int yy = 0; yy < t.iscale_y; yy++)
            for (int xx = 0; xx < t.iscale_x; xx++) {
                const uint8_t* p = src + ((size_t)(dy * t.iscale_y + yy) * a.disp_w + dx * t.iscale_x + xx) * 3;
                s0 += p[0]; s1 += p[1]; s2 += p[2];
            }
        if (t.iscale_x == 2 && t.iscale_y == 2) {
            dst[0] = (uint8_t)((s0 + 2) >> 2); dst[1] = (uint8_t)((s1 + 2) >> 2); dst[2] = (uint8_t)((s2 + 2) >> 2);
        } else {
            const float sc = __fdiv_rn(1.f, (float)(t.iscale_x * t.iscale_y));
            dst[0] = (uint8_t)min(max(__float2int_rn(__fmul_rn((float)s0, sc)), 0), 255);
            dst[1] = (uint8_t)min(max(__float2int_rn(__fmul_rn((float)s1, sc)), 0), 255);
            dst[2] = (uint8_t)min(max(__float2int_rn(__fmul_rn((float)s2, sc)), 0), 255);
        }
        return;
    }
    float sum0 = 0.f, sum1 = 0.f, sum2 = 0.f;
    const int k0 = t.x_ofs[dx], k1 = t.x_ofs[dx + 1];
    const int j0 = t.y_ofs[dy], j1 = t.y_ofs[dy + 1];
    for (int j = j0; j < j1; j++) {
        const uint8_t* row = src + (size_t)t.y_si[j] * a.disp_w * 3;
        const float beta = t.y_alpha[j];
        float b0 = 0.f, b1 = 0.f, b2 = 0.f;
        for (int k = k0; k < k1; k++) {
            const uint8_t* p = row + (size_t)t.x_si[k] * 3;
            const float alpha = t.x_alpha[k];
            b0 = __fadd_rn(b0, __fmul_rn((float)p[0], alpha));
            b1 = __fadd_rn(b1, __fmul_rn((float)p[1], alpha));
            b2 = __fadd_rn(b2, __fmul_rn((float)p[2], alpha));
        }
        sum0 = __fadd_rn(sum0, __fmul_rn(beta, b0));
        sum1 = __fadd_rn(sum1, __fmul_rn(beta, b1));
        sum2 = __fadd_rn(sum2, __fmul_rn(beta, b2));
    }
    dst[0] = (uint8_t)min(max(__float2int_rn(sum0), 0), 255);
    dst[1] = (uint8_t)min(max(__float2int_rn(sum1), 0), 255);
    dst[2] = (uint8_t)min(max(__float2int_rn(sum2), 0), 255);
}

// cv::warpAffine(frame, diag(s,s), display size, INTER_CUBIC, BORDER_CONSTANT 0) of rtpose.cpp:474-487, OpenCV's
// fixed-point arithmetic (imgproc/imgwarp.cpp): source coordinates in 1/32 pixel from integer tables built on the host
// exactly as OpenCV builds adelta/bdelta/X0/Y0, 16 bicubic (a = -0.75) weights as shorts summing to 2^15,
// (sum + 2^14) >> 15, saturate.  Bit-exact against cv2 (tests/golden/warp_cv2.npz).
__global__ void __launch_bounds__(256) warp_affine_cubic_kernel(WarpArgs a) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= a.dw * a.dh) return;
    const int x = idx % a.dw, y = idx / a.dw, f = blockIdx.y;
    const int X = (a.x0[y] + a.adelta[x]) >> 5, Y = (a.y0[y] + a.bdelta[x]) >> 5;
    const int sx = (X >> 5) - 1, sy = (Y >> 5) - 1;
    const short* w = a.tab + ((Y & 31) * 32 + (X & 31)) * 16;
    const uint8_t* src = a.src + (size_t)f * a.sw * a.sh * 3;
    int acc0 = 0, acc1 = 0, acc2 = 0;
#pragma unroll
    for (int k1 = 0; k1 < 4; k1++) {
        const int yy = sy + k1;
        if (yy < 0 || yy >= a.sh) continue;
#pragma unroll
        for (int k2 = 0; k2 < 4; k2++) {
            const int xx = sx + k2;
            if (xx < 0 || xx >= a.sw) continue;
            const uint8_t* p = src + ((size_t)yy * a.sw + xx) * 3;
            const int ww = w[k1 * 4 + k2];
            acc0 += p[0] * ww; acc1 += p[1] * ww; acc2 += p[2] * ww;
        }
    }
    uint8_t* d = a.dst + ((size_t)f * a.dw * a.dh + idx) * 3;
    d[0] = (uint8_t)min(max((acc0 + (1 << 14)) >> 15, 0), 255);
    d[1] = (uint8_t)min(max((acc1 + (1 << 14)) >> 15, 0), 255);
    d[2] = (uint8_t)min(max((acc2 + (1 << 14)) >> 15, 0), 255);
}
int launch_warp_affine(const WarpArgs& a, int nframes, cudaStream_t st) {
    warp_affine_cubic_kernel<<<dim3((a.dw * a.dh + 255) / 256, nframes), 256, 0, st>>>(a);
    return 1;
}

// The flip test (PreArgs::flip): every im2col kernel also writes the copy of its image mirrored in x over the whole net width, in the
// same pass.  Mirrored pixel net_w-1-x holds the patch of pixel x with the taps of each row reversed: patch channel k = (r*3+s)*3+c
// of the mirror is channel mirror_k(k) = (r*3+2-s)*3+c of the original.  Frame f's copies are [S originals][S mirrored].
__device__ __forceinline__ int out_image(const PreArgs& a, int n) { return a.flip ? n + (n / a.S) * a.S : n; }   // source image n = S*f + s
__host__ __device__ constexpr int mirror_k(int k) { return k < 27 ? (k / 9 * 3 + 2 - k / 3 % 3) * 3 + k % 3 : k; }

// S8X1: one s8 plane of 128 channels per pixel, the 27 patch values at scale 2^8 - p - 128 from the uint8 path (exact), and
// sat(rint(x * 256)) from a planar fp32 input - in the first 32 bytes (channels 27..31 written as 0); the rest stays zero from
// init.  S8X2 runs the same kernel: these bytes are its hi plane, and its lo plane stays zero from init, so it stores the
// 16-bit integers (p - 128) x 2^8.  SRC as in input_im2col_kernel.  One thread = one pixel.
template <int SRC>
__global__ void __launch_bounds__(256) input_im2col_s8_kernel(PreArgs a, const float* planar, int nimages) {
    const int n = blockIdx.y;
    const unsigned per_img = (unsigned)a.net_h * (unsigned)a.net_w;
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= per_img) return;
    const int y = (int)(idx / (unsigned)a.net_w), x = (int)(idx % (unsigned)a.net_w);
    const AreaTab& t = a.tab[SRC == 0 ? n % a.S : 0];
    const uint8_t* img = a.resized + (size_t)n * a.net_h * a.net_w * 3;
    int8_t qs[27];
#pragma unroll
    for (int k = 0; k < 27; k++) {
        const int tap = k / 3, c = k % 3;
        const int yy = y + tap / 3 - 1, xx = x + tap % 3 - 1;
        int q = 0;
        if (yy >= 0 && yy < a.net_h && xx >= 0 && xx < a.net_w) {
            if (SRC == 0) {
                const int oy = yy - t.padh, ox = xx - t.padw;
                if (oy >= 0 && oy < t.th && ox >= 0 && ox < t.tw) q = (int)img[((size_t)oy * t.tw + ox) * 3 + c] - 128;
            } else {
                q = __float2int_rn(fminf(fmaxf(__fmul_rn(planar[((size_t)n * 3 + c) * a.net_h * a.net_w + (size_t)yy * a.net_w + xx], 256.f),
                                               -128.f), 127.f));
            }
        }
        qs[k] = (int8_t)q;
    }
    auto store = [&](int img_out, int px, bool mirrored) {
        uint32_t pk[8] = {};
#pragma unroll
        for (int k = 0; k < 27; k++) pk[k / 4] |= ((uint32_t)qs[mirrored ? mirror_k(k) : k] & 0xffu) << (8 * (k % 4));
        const long long m = ((long long)img_out * a.Hs + y) * a.Wp + px;
        uint4* o = (uint4*)((int8_t*)a.out + (size_t)m * a.kp);
        o[0] = make_uint4(pk[0], pk[1], pk[2], pk[3]);
        o[1] = make_uint4(pk[4], pk[5], pk[6], pk[7]);
    };
    const int no = out_image(a, n);
    store(no, x, false);
    if (a.flip) store(no + a.S, a.net_w - 1 - x, true);
}
static void launch_im2col_s8(const PreArgs& a, const float* planar, int nimages, cudaStream_t st) {
    const unsigned per = (unsigned)a.net_h * a.net_w;
    if (planar) input_im2col_s8_kernel<1><<<dim3((per + 255) / 256, nimages), 256, 0, st>>>(a, planar, nimages);
    else input_im2col_s8_kernel<0><<<dim3((per + 255) / 256, nimages), 256, 0, st>>>(a, nullptr, nimages);
}

template <bool F16> __device__ __forceinline__ void split3(float x, uint16_t& h, uint16_t& m, uint16_t& l) {
    h = float_to_plane<F16>(x);
    const float r = __fsub_rn(x, plane_to_float<F16>(h));
    m = float_to_plane<F16>(r);
    l = float_to_plane<F16>(__fsub_rn(r, plane_to_float<F16>(m)));
}

// Row m, channels 8*part .. 8*part+7 of the im2col'ed input from patch(k), or with `mirrored` from patch(mirror_k(k))
template <int SRC, class Patch>
__device__ __forceinline__ void input_im2col_store(const PreArgs& a, long long m, int part, const Patch& patch, int mirrored) {
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; j++) v[j] = patch(mirrored ? mirror_k(part * 8 + j) : part * 8 + j);
    if (a.fmt.planes == 0) {
        float4* o = (float4*)((float*)a.out + (size_t)m * a.kp + part * 8);
        o[0] = make_float4(v[0], v[1], v[2], v[3]);
        o[1] = make_float4(v[4], v[5], v[6], v[7]);
    } else {
        uint32_t pk[3][4];
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
            uint16_t h0, m0, l0, h1, m1, l1;
            if (a.fmt.f16()) { split3<true>(v[j], h0, m0, l0); split3<true>(v[j + 1], h1, m1, l1); }
            else { split3<false>(v[j], h0, m0, l0); split3<false>(v[j + 1], h1, m1, l1); }
            pk[0][j / 2] = (uint32_t)h0 | ((uint32_t)h1 << 16);
            pk[1][j / 2] = (uint32_t)m0 | ((uint32_t)m1 << 16);
            pk[2][j / 2] = (uint32_t)l0 | ((uint32_t)l1 << 16);
        }
        __nv_bfloat16* o0 = (__nv_bfloat16*)a.out + (size_t)m * a.kp + part * 8;
        const int np = SRC == 0 ? 1 : a.fmt.planes;
        for (int p = 0; p < np; p++)
            *(uint4*)(o0 + (size_t)p * a.out_plane) = make_uint4(pk[p][0], pk[p][1], pk[p][2], pk[p][3]);
    }
}

// SRC = 0: uint8 resized images (pad + normalise here);  SRC = 1: planar fp32 net input (already padded/normalised)
// One thread = 8 consecutive patch channels of one pixel (k = 8*part .. 8*part+7, k = (r*3+s)*3 + c), so a row of
// the im2col'ed input is written with coalesced 16/32-byte vector stores.
template <int SRC>
__global__ void __launch_bounds__(256) input_im2col_kernel(PreArgs a, const float* planar, int nimages) {
    // uint8 pixels normalised by /256-0.5 are exact in bf16 (8 significant bits) and in fp16, so the SRC=0 path fills only the
    // hi plane and only the 32 channels that can be non-zero (27 used); everything else stays zero from init
    // (the engine clears the other planes when it switches from the planar-input path, see engine.cu).
    const int parts = (SRC == 0 && a.fmt.planes > 0) ? 4 : a.kp / 8;
    // grid.y = image; 32-bit index math inside an image (64-bit divisions cost hundreds of cycles on the GPU)
    const int n = blockIdx.y;
    const unsigned per_img = (unsigned)a.Hs * (unsigned)a.Wp;
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= per_img * (unsigned)parts) return;
    const int part = (int)(idx % (unsigned)parts);
    const unsigned rem = idx / (unsigned)parts;
    const int y = (int)(rem / (unsigned)a.Wp), x = (int)(rem % (unsigned)a.Wp);
    if (x >= a.net_w || y >= a.net_h) return;  // gap rows stay zero
    const int s = n % a.S;
    const AreaTab& t = a.tab[SRC == 0 ? s : 0];
    const uint8_t* img = a.resized + (size_t)n * a.net_h * a.net_w * 3;
    auto patch = [&](int k) {
        float val = 0.f;
        if (k < 27) {
            const int tap = k / 3, c = k % 3;
            const int yy = y + tap / 3 - 1, xx = x + tap % 3 - 1;
            if (yy >= 0 && yy < a.net_h && xx >= 0 && xx < a.net_w) {
                if (SRC == 0) {
                    const int oy = yy - t.padh, ox = xx - t.padw;
                    if (oy >= 0 && oy < t.th && ox >= 0 && ox < t.tw)
                        val = __fsub_rn(__fmul_rn((float)img[((size_t)oy * t.tw + ox) * 3 + c], 0.00390625f), 0.5f);   // x/256 == x*2^-8 exactly
                } else {
                    val = planar[((size_t)n * 3 + c) * a.net_h * a.net_w + (size_t)yy * a.net_w + xx];
                }
            }
        }
        return val;
    };
    const int no = out_image(a, n);
    input_im2col_store<SRC>(a, ((long long)no * a.Hs + y) * a.Wp + x, part, patch, 0);
    if (a.flip) input_im2col_store<SRC>(a, ((long long)(no + a.S) * a.Hs + y) * a.Wp + (a.net_w - 1 - x), part, patch, 1);
}

// Fast path of input_im2col_kernel<0> for the 16-bit plane modes: one thread = one pixel, the 3x3x3 patch comes from a
// shared-memory tile of the resized uint8 image (pad + v/256 - 0.5 applied on the way in, exact in fp16 and bf16), and the 32
// patch channels (27 used) of a pixel leave as 64 contiguous bytes, i.e. a warp writes 2 KB in one piece.  The generic kernel
// spent 8.7 M threads with nested bound checks on what is a 140 MB write (r1n: 160 us per 9-frame step).
template <bool F16>
__global__ void __launch_bounds__(256) input_im2col_u8_kernel(PreArgs a) {
    constexpr int TX = 32, TY = 8;
    __shared__ uint16_t tile[3][TY + 2][TX + 2];
    const int n = blockIdx.z, s = n % a.S;
    const AreaTab& t = a.tab[s];
    const uint8_t* img = a.resized + (size_t)n * a.net_h * a.net_w * 3;
    const int x0 = blockIdx.x * TX, y0 = blockIdx.y * TY;
    const int tid = threadIdx.y * 32 + threadIdx.x;
    for (int i = tid; i < 3 * (TY + 2) * (TX + 2); i += 256) {
        const int c = i % 3, px = i / 3;                       // channel fastest: consecutive threads read consecutive bytes
        const int ty = px / (TX + 2), tx = px % (TX + 2);
        const int yy = y0 + ty - 1, xx = x0 + tx - 1;
        float v = 0.f;
        if (yy >= 0 && yy < a.net_h && xx >= 0 && xx < a.net_w) {
            const int oy = yy - t.padh, ox = xx - t.padw;
            if (oy >= 0 && oy < t.th && ox >= 0 && ox < t.tw)
                v = __fsub_rn(__fmul_rn((float)img[((size_t)oy * t.tw + ox) * 3 + c], 0.00390625f), 0.5f);
        }
        tile[c][ty][tx] = float_to_plane<F16>(v);
    }
    __syncthreads();
    const int x = x0 + threadIdx.x, y = y0 + threadIdx.y;
    if (x >= a.net_w || y >= a.net_h) return;
    auto store = [&](int img_out, int px, bool mirrored) {
        uint16_t k[32];
#pragma unroll
        for (int tap = 0; tap < 9; tap++)
#pragma unroll
            for (int c = 0; c < 3; c++) k[tap * 3 + c] = tile[c][threadIdx.y + tap / 3][threadIdx.x + (mirrored ? 2 - tap % 3 : tap % 3)];
#pragma unroll
        for (int j = 27; j < 32; j++) k[j] = 0;
        const long long m = ((long long)img_out * a.Hs + y) * a.Wp + px;
        uint4* o = (uint4*)((uint16_t*)a.out + (size_t)m * a.kp);
#pragma unroll
        for (int q = 0; q < 4; q++)
            o[q] = make_uint4((uint32_t)k[q * 8] | ((uint32_t)k[q * 8 + 1] << 16), (uint32_t)k[q * 8 + 2] | ((uint32_t)k[q * 8 + 3] << 16),
                              (uint32_t)k[q * 8 + 4] | ((uint32_t)k[q * 8 + 5] << 16), (uint32_t)k[q * 8 + 6] | ((uint32_t)k[q * 8 + 7] << 16));
    };
    const int no = out_image(a, n);
    store(no, x, false);
    if (a.flip) store(no + a.S, a.net_w - 1 - x, true);
}

static int launch_im2col_u8(const PreArgs& a, cudaStream_t st) {
    if (a.fmt.s8()) { launch_im2col_s8(a, nullptr, a.nframes * a.S, st); return 1; }
    if (a.fmt.planes > 0 && a.kp >= 32) {
        const dim3 g((a.net_w + 31) / 32, (a.net_h + 7) / 8, a.nframes * a.S), b(32, 8);
        if (a.fmt.f16()) input_im2col_u8_kernel<true><<<g, b, 0, st>>>(a);
        else input_im2col_u8_kernel<false><<<g, b, 0, st>>>(a);
        return 1;
    }
    const unsigned work = (unsigned)a.Hs * a.Wp * (a.fmt.planes > 0 ? 4 : a.kp / 8);
    input_im2col_kernel<0><<<dim3((work + 255) / 256, a.nframes * a.S), 256, 0, st>>>(a, nullptr, a.nframes * a.S);
    return 1;
}
int launch_preprocess(const PreArgs& a, cudaStream_t st) {
    dim3 g((a.net_w * a.net_h + 255) / 256, a.S, a.nframes);
    area_resize_kernel<<<g, 256, 0, st>>>(a);
    return 1 + launch_im2col_u8(a, st);
}

int launch_input_from_planar(const float* planar, const PreArgs& a, int nimages, cudaStream_t st) {
    if (a.fmt.s8()) { launch_im2col_s8(a, planar, nimages, st); return 1; }
    const unsigned work = (unsigned)a.Hs * a.Wp * (a.kp / 8);
    input_im2col_kernel<1><<<dim3((work + 255) / 256, nimages), 256, 0, st>>>(a, planar, nimages);
    return 1;
}

}  // namespace pe
