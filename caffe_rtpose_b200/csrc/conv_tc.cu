// wgmma / TMA implicit-GEMM convolution for sm_90a (H100), hand-written PTX.
//
// Replaces cudnnConvolutionForward + cudnnAddTensor + ReLU (src/caffe/layers/cudnn_conv_layer.cu:11-46,
// cudnn_relu_layer.cu:19) and the Concat copies (concat_layer.cu:40-43) for every 3x3 / 7x7 / 1x1
// convolution of the deploy graph.  Arithmetic contract = Caffe's conv (base_conv_layer.cpp:257-279):
// out = W * im2col(in) + bias, zero padding, stride 1.
//
// Mapping to the hardware
//   * GEMM view: D[m][co] = sum_{tap} sum_{c} A[m + shift(tap)][c] * Wt[co][tap*C + c], M = flat padded
//     pixels (common.h), so the A tile of one (tap, 64-channel block) is 128 consecutive rows at a shifted row
//     coordinate, and the k taps of one filter row read 128 + k - 1 consecutive rows: ONE TMA box {64 ch x 136 rows x
//     P planes} per (filter row, 64-channel block), the "A window"; tap q reads rows [q, q + 128) of it.  Zero padding
//     = TMA out-of-bounds fill + never-written gap rows.
//   * A producer warpgroup (one thread) stages A windows and B tiles with TMA (cp.async.bulk.tensor.3d, SWIZZLE_128B)
//     into two rings of shared-memory slots; completion and release on mbarriers.  It gives its registers to the
//     consumers (setmaxnreg).  Row tiles start at every image (blockIdx.x = image, tile), and TC_CLUSTER consecutive
//     row tiles form a thread block cluster: each CTA loads 1/TC_CLUSTER of every weight tile and multicasts it to all,
//     and a slot of the weight ring is refilled once the consumers of every CTA in the cluster have released it.
//   * Two consumer warpgroups (64 rows each) issue wgmma.mma_async m64nBNk16 from shared-memory descriptors,
//     accumulators in registers, fp32, with one wgmma group of K steps in flight behind the one being issued.
//   * Split precision: activations and weights are stored as P 16-bit "planes" whose sum is the fp32 value
//     (hi / lo); the kernel issues the cross products with pa + pb < P on the tensor core.  Each mode's format and
//     accumulation are a row of the precision table (precision.h; DESIGN.md section 3).  In the chunked modes hi*hi goes
//     to its own accumulator, cut into chunks of a few hundred K that are added in registers with round-to-nearest (the
//     tensor core's fp32 accumulation truncates, so a long chain drifts); the cross terms are 2^-11 smaller and run over
//     the whole tile in a second accumulator.
//   * Epilogue: sum, bias, ReLU, re-split into planes and store NHWC planes (channel-slice stores implement
//     Concat), or - for the last stage - the planar fp32 concat_stage7 blob.
#include <cuda.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <string>

#include "common.h"
#include "conv_tc.h"
#include "kernels.h"
#include "conv_tc_kernel.cuh"

namespace pe {

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) == cudaSuccess && qr == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

// Never below cout: the packed weights, the biases and the grid's N tiles all span cout_pad channels.
int tc_cout_pad(int cout) {
    if (cout > 64) return (cout + 127) / 128 * 128;
    if (cout > 48) return 64;
    if (cout > 32) return 48;
    if (cout > 16) return 32;
    return 16;
}
// Tile width: 128 output channels.  With 2 or 3 planes the hi*hi chunk, its running sum and the cross-term accumulator
// live in registers side by side: 3 x 64 per consumer thread at BN = 128, which fits in the consumers' 232 registers.
// Three planes (bf16x3, kept for A/B comparisons) stay at 64.
static int tc_bn(int cout_pad, int planes) { return std::min(cout_pad, planes == 3 ? 64 : 128); }

// box {one channel block = 128 bytes, b1, b2}; TMA only moves the bytes, so the data type is any of the element's size
static int encode(EncodeTiledFn enc, CUtensorMap* map, PlaneElem elem, const void* base, cuuint64_t d0, cuuint64_t d1, cuuint64_t d2,
                  cuuint64_t s1, cuuint64_t s2, cuuint32_t b1, cuuint32_t b2, CUtensorMapL2promotion l2) {
    cuuint64_t dims[3] = {d0, d1, d2};
    cuuint64_t strides[2] = {s1, s2};
    cuuint32_t box[3] = {(cuuint32_t)tc_block_ch(elem), b1, b2};
    cuuint32_t es[3] = {1, 1, 1};
    return (int)enc(map, elem_size(elem) == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, (void*)base, dims,
                    strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

int tc_layer_create(const TcLayerDesc& d, TcLayer& out, std::string& err) {
    EncodeTiledFn enc = get_encode();
    if (!enc) { err = "cuTensorMapEncodeTiled unavailable"; return -1; }
    const int kb = tc_block_ch(d.fmt.elem), eb = d.fmt.elem_bytes();
    if (d.in_cused % kb) { err = "input channels not a multiple of " + std::to_string(kb); return -1; }
    if (d.fmt.planes < 1 || d.fmt.planes > 3 || ((d.fmt.e4m3() || d.fmt.u8()) && d.fmt.planes != 1) || (d.fmt.s8() && d.fmt.planes > 2)) {
        err = "1 to 3 planes (e4m3, u8: 1; s8: 1 or 2)";
        return -1;
    }
    if (d.ksize < 1 || d.ksize > TC_KMAX) { err = "filter size above " + std::to_string(TC_KMAX) + " (A window rows)"; return -1; }
    out.d = d;
    out.bn = tc_bn(d.cout_pad, d.fmt.planes);
    CUtensorMap* maps = nullptr;
    if (posix_memalign((void**)&maps, 64, 3 * sizeof(CUtensorMap))) { err = "alloc"; return -1; }
    memset(maps, 0, 3 * sizeof(CUtensorMap));
    const cuuint64_t K = (cuuint64_t)d.ksize * d.ksize * d.in_cused;
    const cuuint64_t P = (cuuint64_t)d.fmt.planes;
    if (d.sparse) {   // conv_s8_sparse.cu: windows {128 ch, N + 8 rows} at N = 128 and 64; compressed values {64 B, 128 rows}, SWIZZLE_64B
        if (!d.fmt.s8() || d.cout_pad % 128) { err = "sparse layers are s8 with 128-channel output blocks"; free(maps); return -1; }
        int r = 0;
        for (int m = 0; m < 2 && !r; m++)
            r = encode(enc, &maps[2 * m], d.fmt.elem, d.in, d.in_cused, d.geo.M, 1, (cuuint64_t)d.in_pitch, (cuuint64_t)d.in_plane,
                       d.ksize == 1 ? 128 >> m : (128 >> m) + TC_KMAX - 1, 1, CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
        cuuint64_t dims[3] = {K / 2, (cuuint64_t)d.cout_pad, 1}, strides[2] = {K / 2, K / 2 * d.cout_pad};
        cuuint32_t box[3] = {64, 128, 1}, es[3] = {1, 1, 1};
        if (!r) r = (int)enc(&maps[1], CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, (void*)d.w, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                             CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r) { err = "cuTensorMapEncodeTiled failed: " + std::to_string(r); free(maps); return -1; }
        out.maps = maps;
        return 0;
    }
    // A: [planes][M][pitch], box {channel block, window rows, planes}
    int r = encode(enc, &maps[0], d.fmt.elem, d.in, d.in_cused, d.geo.M, P, (cuuint64_t)d.in_pitch * eb, (cuuint64_t)d.in_plane * eb,
                   tc_window_rows(d.ksize), d.fmt.planes,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
    // B: [planes][cout_pad][K], box {channel block, part of a plane, 1} (a CTA's share of a {64, bn, planes} tile is one or more such
    // boxes, tc_wbox_rows); and for half-width tiles (more CTAs for small problems, see tc_layer_launch)
    if (!r) r = encode(enc, &maps[1], d.fmt.elem, d.w, K, d.cout_pad, P, K * eb, K * eb * d.cout_pad, tc_wbox_rows(out.bn, d.fmt.planes), 1,
                       CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
    if (!r && out.bn >= 64) r = encode(enc, &maps[2], d.fmt.elem, d.w, K, d.cout_pad, P, K * eb, K * eb * d.cout_pad,
                                       tc_wbox_rows(out.bn / 2, d.fmt.planes), 1, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
    if (r) { err = "cuTensorMapEncodeTiled failed: " + std::to_string(r); free(maps); return -1; }
    out.maps = maps;
    return 0;
}

void tc_layer_destroy(TcLayer& l) {
    if (l.maps) free(l.maps);
    l.maps = nullptr;
}

int tc_layer_launch(const TcLayer& l, int nimg, cudaStream_t st, int share) {
    const TcLayerDesc& d = l.d;
    if (d.sparse) return tc_sparse_launch(l, nimg, st, share);   // conv_s8_sparse.cu
    TcArgs a;
    a.bias = d.bias;
    a.out = d.out; a.out_pitch = d.out_pitch; a.out_coff = d.out_coff; a.out_plane = d.out_plane;
    a.planar = d.planar; a.planar_C = d.planar_C; a.planar_coff = d.planar_coff;
    a.cout = d.cout; a.relu = d.relu; a.out_scale = d.out_scale; a.range = d.range;
    a.ksize = d.ksize; a.pad = d.pad; a.kblocks_per_tap = d.in_cused / tc_block_ch(d.fmt.elem); a.cin_k = d.in_cused;
    a.W = d.geo.W; a.H = d.geo.H; a.Wp = d.geo.Wp; a.Hs = d.geo.Hs;
    a.M = (long long)nimg * d.geo.Hs * d.geo.Wp;
    // hi*hi accumulation chunk of the chunked modes: one 7-tap filter row (448 K in 16 bits), two 3-tap rows (384 K) or four 1x1
    // blocks (256 K); e4m3 the same K steps of 128 channels (896, 768, 512 K: DESIGN.md section 6).  The others run one chain
    // over the whole K.
    const int nk = d.ksize * d.ksize * a.kblocks_per_tap;
    a.chunk_iters = d.chunked ? (d.ksize >= 7 ? 7 : (d.ksize >= 3 ? 6 : 4)) : nk;
    static int nsm = 0;
    if (!nsm) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev); }
    // Tile width: the full width is the efficient shape (the A tile is re-read per N tile), but a single frame at the
    // 46x82 level has only 33 row tiles for 132 SMs: take half the width when (CTAs that can run at once) x (relative
    // efficiency of the shape) is larger.  share: layers running concurrently on other streams take their part of the SMs.
    const long long mt = (a.M + TC_BM - 1) / TC_BM;
    const long long sms = std::max(1, nsm / (share < 1 ? 1 : share));
    int bn = l.bn, bmap = 1;
    if (l.bn >= 64) {
        const double sfull = (double)std::min<long long>(mt * (d.cout_pad / l.bn), sms) * 1.00;
        const double shalf = (double)std::min<long long>(mt * (d.cout_pad / (l.bn / 2)), sms) * 0.80;
        if (shalf > sfull) { bn = l.bn / 2; bmap = 2; }
    }
    // row tiles per image: up to its last pixel (H - 1) * Wp + W - 1; the grid in whole clusters
    a.tiles_img = ((d.geo.H - 1) * d.geo.Wp + d.geo.W + TC_BM - 1) / TC_BM;
    const long long tiles = ((long long)nimg * a.tiles_img + TC_CLUSTER - 1) / TC_CLUSTER * TC_CLUSTER;
    const dim3 grid((unsigned)tiles, (unsigned)(d.cout_pad / bn), 1);
    const PlaneFmt f = d.fmt;
    if (f.s8() && f.planes == 2) return launch_s8x2(l, a, grid, st, bmap, bn);            // conv_s8x2.cu
    if (f.u8() || d.out_elem == ELEM_U8) return launch_u8(l, a, grid, st, bmap, bn);   // conv_u8.cu
    if (f.elem != d.out_elem && d.out_elem != ELEM_E4M3) return launch_mixed(l, a, grid, st, bmap, bn);   // conv_mixed.cu
    if (d.out_elem == ELEM_E4M3) return launch_e4m3(l, a, grid, st, bmap, bn);   // conv_fp8.cu
    if (d.out_elem == ELEM_S8) return launch_s8(l, a, grid, st, bmap, bn);       // conv_s8.cu
    if (f.planes == 3) return launch_widths<3, ELEM_BF16, ELEM_BF16>(l, a, grid, st, bmap, bn);
    if (f.planes == 2) return launch_widths<2, ELEM_F16, ELEM_F16>(l, a, grid, st, bmap, bn);
    return f.f16() ? launch_widths<1, ELEM_F16, ELEM_F16>(l, a, grid, st, bmap, bn)
                   : launch_widths<1, ELEM_BF16, ELEM_BF16>(l, a, grid, st, bmap, bn);
}

}  // namespace pe
