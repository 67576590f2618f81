// JPEG reconstruction on the GPU: the coefficient images of pe_jpeg_read_coefs (host entropy stage, jpeg_dec.cpp) -> uint8 BGR
// frames, byte-identical to pe_decode_jpeg.  Two kernels, both in integer arithmetic that follows the host code step by step:
//   jpeg_idct_kernel   dequantisation + libjpeg's islow IDCT (jpeg_dec.cpp idct_islow: 64-bit products where the host uses jlong,
//                      the same descale / range limit and the zero-AC shortcuts) of every 8x8 block into component planes;
//   jpeg_color_kernel  "fancy" h2v1 / h2v2 chroma upsampling (triangle filters, libjpeg's rounding biases, replication when the
//                      chroma plane is at most 2 samples wide, 4:4:4 passed through) + fixed-point YCbCr -> BGR.
// Each frame carries its own header (size, sampling, quantisation tables) in device memory; the host checked it
// (jpeg_coefs.h coef_header_valid) before the copy.
#include "kernels.h"

namespace pe {

namespace {

constexpr int CONST_BITS = 13, PASS1_BITS = 2;
constexpr int F_0_298631336 = 2446, F_0_390180644 = 3196, F_0_541196100 = 4433, F_0_765366865 = 6270, F_0_899976223 = 7373, F_1_175875602 = 9633,
              F_1_501321110 = 12299, F_1_847759065 = 15137, F_1_961570560 = 16069, F_2_053119869 = 16819, F_2_562915447 = 20995, F_3_072711026 = 25172;
typedef long long jlong;

__device__ __forceinline__ jlong descale(jlong x, int n) { return (x + ((jlong)1 << (n - 1))) >> n; }
__device__ __forceinline__ uint32_t range_limit(jlong x) { x += 128; return (uint32_t)(x < 0 ? 0 : (x > 255 ? 255 : x)); }

// jpeg_dec.cpp idct_1d: one column / row, inputs in[k * stride]
__device__ __forceinline__ void idct_1d(const int* in, int stride, jlong* o) {
    jlong z2 = in[2 * stride], z3 = in[6 * stride];
    jlong z1 = (z2 + z3) * F_0_541196100;
    jlong tmp2 = z1 + z3 * (-F_1_847759065);
    jlong tmp3 = z1 + z2 * F_0_765366865;
    z2 = in[0];
    z3 = in[4 * stride];
    jlong tmp0 = (z2 + z3) * (1 << CONST_BITS);
    jlong tmp1 = (z2 - z3) * (1 << CONST_BITS);
    const jlong tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    tmp0 = in[7 * stride]; tmp1 = in[5 * stride]; tmp2 = in[3 * stride]; tmp3 = in[1 * stride];
    z1 = tmp0 + tmp3; z2 = tmp1 + tmp2; z3 = tmp0 + tmp2;
    jlong z4 = tmp1 + tmp3;
    const jlong z5 = (z3 + z4) * F_1_175875602;
    tmp0 *= F_0_298631336; tmp1 *= F_2_053119869; tmp2 *= F_3_072711026; tmp3 *= F_1_501321110;
    z1 *= -F_0_899976223; z2 *= -F_2_562915447; z3 *= -F_1_961570560; z4 *= -F_0_390180644;
    z3 += z5; z4 += z5;
    tmp0 += z1 + z3; tmp1 += z2 + z4; tmp2 += z2 + z3; tmp3 += z1 + z4;
    o[0] = tmp10 + tmp3; o[7] = tmp10 - tmp3; o[1] = tmp11 + tmp2; o[6] = tmp11 - tmp2;
    o[2] = tmp12 + tmp1; o[5] = tmp12 - tmp1; o[3] = tmp13 + tmp0; o[4] = tmp13 - tmp0;
}

__device__ __forceinline__ const pe_jpeg_coef_header* frame_header(const JpegArgs& a, int f) {
    return reinterpret_cast<const pe_jpeg_coef_header*>(a.coefs + (size_t)f * a.coef_stride);
}

// 8 threads per 8x8 block, 32 blocks per CTA: thread t loads row t (one 16-byte load) and dequantises it, transforms column t
// (pass 1), then row t (pass 2) and stores its 8 output bytes.  The 8 threads of a block sit in one warp: __syncwarp suffices.
// Block gb of a frame is the gb-th block of the concatenated components (the coefficient layout), its plane bytes the gb-th 64.
constexpr int IDCT_BLOCKS = 32, PITCH = 9;   // shared rows padded to 9 words: column and row accesses avoid bank conflicts
__global__ void __launch_bounds__(IDCT_BLOCKS * 8) jpeg_idct_kernel(JpegArgs a) {
    __shared__ int s_deq[IDCT_BLOCKS][8 * PITCH], s_ws[IDCT_BLOCKS][8 * PITCH];
    const int f = blockIdx.y, g = threadIdx.x >> 3, t = threadIdx.x & 7;
    const pe_jpeg_coef_header* hd = frame_header(a, f);
    const long long gb = (long long)blockIdx.x * IDCT_BLOCKS + g;
    const int nc = hd->num_comps;
    int c = 0;
    long long start = 0, nb = (long long)hd->comp[0].bw * hd->comp[0].bh;
    while (c + 1 < nc && gb >= start + nb) { start += nb; c++; nb = (long long)hd->comp[c].bw * hd->comp[c].bh; }
    const bool valid = gb < start + nb;   // uniform over the block's 8 threads
    int* dq = s_deq[g];
    int* ws = s_ws[g];
    if (valid) {
        const uint8_t* base = a.coefs + (size_t)f * a.coef_stride;
        const int4 raw = *reinterpret_cast<const int4*>(base + sizeof(pe_jpeg_coef_header) + (size_t)gb * 128 + t * 16);
        const uint4 qr = *reinterpret_cast<const uint4*>(hd->comp[c].quant + t * 8);
        const short* cv = reinterpret_cast<const short*>(&raw);
        const uint16_t* qv = reinterpret_cast<const uint16_t*>(&qr);
#pragma unroll
        for (int j = 0; j < 8; j++) dq[t * PITCH + j] = (int)((jlong)cv[j] * (jlong)qv[j]);
    }
    __syncwarp();
    if (valid) {   // pass 1: column t
        int in[8];
#pragma unroll
        for (int r = 0; r < 8; r++) in[r] = dq[r * PITCH + t];
        if ((in[1] | in[2] | in[3] | in[4] | in[5] | in[6] | in[7]) == 0) {
            const int dcv = (int)((jlong)in[0] * (1 << PASS1_BITS));
#pragma unroll
            for (int r = 0; r < 8; r++) ws[r * PITCH + t] = dcv;
        } else {
            jlong o[8];
            idct_1d(in, 1, o);
#pragma unroll
            for (int r = 0; r < 8; r++) ws[r * PITCH + t] = (int)descale(o[r], CONST_BITS - PASS1_BITS);
        }
    }
    __syncwarp();
    if (!valid) return;
    // pass 2: row t
    int w[8];
#pragma unroll
    for (int j = 0; j < 8; j++) w[j] = ws[t * PITCH + j];
    uint32_t lo, hi;
    if ((w[1] | w[2] | w[3] | w[4] | w[5] | w[6] | w[7]) == 0) {
        const uint32_t v = range_limit(descale((jlong)w[0], PASS1_BITS + 3)) * 0x01010101u;
        lo = hi = v;
    } else {
        jlong o[8];
        idct_1d(w, 1, o);
        uint32_t b[8];
#pragma unroll
        for (int j = 0; j < 8; j++) b[j] = range_limit(descale(o[j], CONST_BITS + PASS1_BITS + 3));
        lo = b[0] | b[1] << 8 | b[2] << 16 | b[3] << 24;
        hi = b[4] | b[5] << 8 | b[6] << 16 | b[7] << 24;
    }
    const int bw = hd->comp[c].bw;
    const long long local = gb - start;
    const long long by = local / bw, bx = local - by * bw;
    uint8_t* plane = a.planes + (size_t)f * a.plane_stride + (size_t)start * 64;
    *reinterpret_cast<uint2*>(plane + (size_t)(by * 8 + t) * (bw * 8) + bx * 8) = make_uint2(lo, hi);
}

// one chroma sample at full resolution (jpeg_dec.cpp upsample_row_impl): plane P with pitch pw and dw x dh real samples
__device__ __forceinline__ int upsample(const uint8_t* P, int pw, int dw, int dh, int hs, int vs, int x, int y) {
    if (hs == 1 && vs == 1) return P[(size_t)y * pw + x];
    auto row = [&](int r) { r = r < 0 ? 0 : (r >= dh ? dh - 1 : r); return P + (size_t)r * pw; };
    const int i = x >> 1;
    const bool odd = x & 1, fancy = dw > 2;
    const int nb = odd ? (i < dw - 1 ? i + 1 : dw - 1) : (i > 0 ? i - 1 : 0);   // the edge samples take their own value as neighbour
    if (vs == 1) {   // h2v1: 3/4 nearer + 1/4 farther sample, biases 1 (even) / 2 (odd)
        const uint8_t* in = row(y);
        if (!fancy) return in[i];
        return (in[i] * 3 + in[nb] + (odd ? 2 : 1)) >> 2;
    }
    const int r = y >> 1;   // h2v2: vertical 3:1 with the nearer row, then horizontal 3:1, biases 8 (even) / 7 (odd)
    const uint8_t* in0 = row(r);
    if (!fancy) return in0[i];
    const uint8_t* in1 = (y & 1) ? row(r + 1) : row(r - 1);
    const int ci = in0[i] * 3 + in1[i], cn = in0[nb] * 3 + in1[nb];
    return (ci * 3 + cn + (odd ? 7 : 8)) >> 4;
}

__device__ __forceinline__ uint8_t clamp255(int v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

// one thread per output pixel: grid (x tiles, rows, frames)
__global__ void __launch_bounds__(128) jpeg_color_kernel(JpegArgs a) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, f = blockIdx.z;
    if (x >= a.W) return;
    const pe_jpeg_coef_header* hd = frame_header(a, f);
    const uint8_t* planes = a.planes + (size_t)f * a.plane_stride;
    const pe_jpeg_coef_comp& yc = hd->comp[0];
    const int Y = planes[(size_t)y * yc.bw * 8 + x];
    uint8_t* o = a.dst + (size_t)f * a.W * a.H * 3 + ((size_t)y * a.W + x) * 3;
    if (hd->num_comps == 1) { o[0] = o[1] = o[2] = (uint8_t)Y; return; }
    const pe_jpeg_coef_comp &cbc = hd->comp[1], &crc = hd->comp[2];
    const uint8_t* pcb = planes + (size_t)yc.bw * yc.bh * 64;
    const uint8_t* pcr = pcb + (size_t)cbc.bw * cbc.bh * 64;
    const int b = upsample(pcb, cbc.bw * 8, cbc.dw, cbc.dh, yc.h, yc.v, x, y) - 128;
    const int r = upsample(pcr, crc.bw * 8, crc.dw, crc.dh, yc.h, yc.v, x, y) - 128;
    // jdcolor.c build_ycc_rgb_table, SCALEBITS 16 (jpeg_dec.cpp ycc_row_impl)
    o[0] = clamp255(Y + ((116130 * b + 32768) >> 16));
    o[1] = clamp255(Y + ((-22554 * b + 32768 - 46802 * r) >> 16));
    o[2] = clamp255(Y + ((91881 * r + 32768) >> 16));
}

}  // namespace

int launch_jpeg_reconstruct(const JpegArgs& a, cudaStream_t st) {
    jpeg_idct_kernel<<<dim3((unsigned)((a.max_blocks + IDCT_BLOCKS - 1) / IDCT_BLOCKS), a.n), IDCT_BLOCKS * 8, 0, st>>>(a);
    jpeg_color_kernel<<<dim3((a.W + 127) / 128, a.H, a.n), 128, 0, st>>>(a);
    return 2;
}

}  // namespace pe
