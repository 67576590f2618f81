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
//     (hi / lo); the kernel issues the cross products with pa + pb < P on the tensor core.  The format (kernels.h,
//     PlaneFmt): P=2 fp16 = parity mode, ~1e-5 over the whole net (DESIGN.md section 3); P=1 fp16 = fast mode, the
//     parity mode's hi plane alone (one MMA per MAC); P=1 bf16 and P=3 bf16 are kept for A/B comparisons.
//     hi*hi goes to its own accumulator, cut into chunks of a few hundred K that are added in registers with
//     round-to-nearest (the tensor core's fp32 accumulation truncates, so a long chain drifts); the cross terms
//     are 2^-11 smaller and run over the whole tile in a second accumulator.  bf16x1 keeps one unchunked chain.
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

namespace pe {

struct TcArgs {
    const float* bias;
    __nv_bfloat16* out; int out_pitch, out_coff; long long out_plane;
    float* planar; int planar_C, planar_coff;
    int cout, relu;
    const float* out_scale;                   // -> 2^-k in the packed buffer: the weights of this layer carry a factor 2^k (fp16 planes)
    int ksize, pad, kblocks_per_tap, cin_k;   // cin_k = channels per tap in the weight K ordering
    int W, H, Wp, Hs;
    long long M;
    int tiles_img;                            // row tiles per image: blockIdx.x = image * tiles_img + tile
    int chunk_iters;                          // K iterations (64 channels of one tap each) per hi*hi accumulation chunk
    unsigned* range;                          // [0]: running max |stored value| of this layer as float bits (atomicMax; values are >= 0), or null
};

// ------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t"
            "}" : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    } while (!done);
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// The same box written to the same shared-memory offset of every CTA in `mask`, each CTA's mbarrier at `bar`'s offset
// receiving the bytes.
__device__ __forceinline__ void tma_load_3d_mc(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, uint16_t mask) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4, %5}], [%2], %6;"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "h"(mask) : "memory");
}

// Thread block clusters: rank within the cluster, a cluster-wide barrier of all threads, and an arrive on the mbarrier at
// `bar`'s offset in the shared memory of cluster CTA `rank`.  The arrive keeps the default .release.cta: it only has to
// follow the reads of the arriving warp's wgmma, which wgmma.wait_group has completed.  A .release.cluster arrive on the
// consumers' path made the conv stack 16 % slower than the kernel without clusters (H100 80GB HBM3, 400 W limit).
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
    asm volatile(
        "{\n\t"
        ".reg .b32 ra;\n\t"
        "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
        "mbarrier.arrive.shared::cluster.b64 _, [ra];\n\t"
        "}" ::"r"(smem_u32(bar)), "r"(rank) : "memory");
}

// Programmatic dependent launch (PDL): a conv kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may
// start while its predecessor in the stream drains.  Everything before pdl_wait() - barrier init, tensor-map prefetch,
// bias staging - overlaps the predecessor's tail; pdl_wait() returns once the predecessor grid has completed and its
// writes are visible.  No-ops without the launch attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// wgmma shared-memory matrix descriptor, K-major, SWIZZLE_128B (PTX ISA "Matrix Descriptor Format"):
//   [0,14) start address >> 4 | [16,30) LBO >> 4 (unused for swizzled K-major, 1) | [32,46) SBO >> 4
//   (8 rows x 128 B = 1024 B -> 64) | [62,64) layout type = 1 (SWIZZLE_128B).  TMA boxes start on 1024-byte
//   boundaries; the K=16 steps inside a 128-byte swizzle row advance the start address by 32 bytes, and a tap's row
//   shift inside an A window by 128 bytes per row.  The wgmma unit takes the swizzle's row phase from the address bits
//   [7,10) of each row, as TMA does when it writes the box, so a start address q rows into a box needs no correction:
//   the matrix base offset [49,52) stays 0 (on the H100, setting it to (start >> 7) & 7 shifts the pattern a second
//   time and reads wrong data).
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)64 << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }

// D(64 x N, fp32 registers) (+)= A(64 x 16) * B(N x 16)^T, both K-major in shared memory; scale_d = 0 overwrites D.
// Register j of a thread holds row 16*(warp%4) + lane/4 + 8*((j/2)%2), column 8*(j/4) + 2*(lane%4) + j%2.
template <int N> struct Wgmma;
template <> struct Wgmma<16> {
    template <bool F16> __device__ __forceinline__ static void mma(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
        if (F16) asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "l"(da), "l"(db), "r"(scale_d));
        else asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "l"(da), "l"(db), "r"(scale_d));
    }
};
template <> struct Wgmma<32> {
    template <bool F16> __device__ __forceinline__ static void mma(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
        if (F16) asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(da), "l"(db), "r"(scale_d));
        else asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(da), "l"(db), "r"(scale_d));
    }
};
template <> struct Wgmma<48> {
    template <bool F16> __device__ __forceinline__ static void mma(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
        if (F16) asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %26, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, %24, %25, p, 1, 1, 0, 0;\n}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
            : "l"(da), "l"(db), "r"(scale_d));
        else asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %26, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, %24, %25, p, 1, 1, 0, 0;\n}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
            : "l"(da), "l"(db), "r"(scale_d));
    }
};
template <> struct Wgmma<64> {
    template <bool F16> __device__ __forceinline__ static void mma(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
        if (F16) asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(da), "l"(db), "r"(scale_d));
        else asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(da), "l"(db), "r"(scale_d));
    }
};
template <> struct Wgmma<128> {
    template <bool F16> __device__ __forceinline__ static void mma(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
        if (F16) asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "l"(da), "l"(db), "r"(scale_d));
        else asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "l"(da), "l"(db), "r"(scale_d));
    }
};

// Range tracking of the 16-bit planes: every epilogue warp folds the largest |value| it stores into one word per layer.  The
// host reads it to calibrate per-layer power-of-two activation scales (engine.cu, pe_calibrate) and to report values that
// left the fp16 range instead of letting inf / flushed zeros poison the following layers silently.
__device__ __forceinline__ void range_publish(unsigned* range, float m) {
    if (!range) return;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(range, __float_as_uint(m));
}

// ------------------------------------------------------------------------------------------------
// the kernel
// ------------------------------------------------------------------------------------------------
constexpr int TC_BM = 128;           // rows per CTA tile: two consumer warpgroups x 64
constexpr int TC_BK = 64;            // 16-bit elements per K block = one 128-byte swizzle row
constexpr int TC_WROWS = TC_BM + 8;  // rows of an A window: the tile plus the row shifts q = 1..8 of a filter row (k <= 9)
constexpr int TC_KMAX = TC_WROWS - TC_BM + 1;
constexpr int TC_THREADS = 384;      // warpgroup 0: TMA producer, warpgroups 1-2: consumers
constexpr int TC_PRODUCER_REGS = 40, TC_CONSUMER_REGS = 232;   // setmaxnreg: 128 x 40 + 256 x 232 <= 65536
constexpr int TC_SMEM_BUDGET = 220 * 1024;   // of the 227 KB a block may use on H100; the rest: alignment + static

// CTAs along M that share every weight tile: each loads 1/TC_CLUSTER of the tile from L2 and multicasts it to all of them,
// so the L2 -> shared-memory traffic of the weights, most of the kernel's, drops by this factor.  A windows stay per CTA.
constexpr int TC_CLUSTER = 2;

// A consumer warp has finished reading weight slot b (its wgmma groups have completed): tell the producer of every CTA in the
// cluster, since each weight tile is written into all of them; and release window slot w after its last tap (w >= 0).
__device__ __forceinline__ void tc_release(uint64_t* bempty, uint64_t* wempty, int b, int w, int lane) {
    __syncwarp();
    if (lane < TC_CLUSTER) mbar_arrive_cluster(&bempty[b], lane);
    if (w >= 0 && lane == 0) mbar_arrive(&wempty[w]);
}

// Rows of the A window box: a 1x1 filter row is a single tap and reads only the tile's 128 rows.
__host__ __device__ constexpr int tc_window_rows(int ksize) { return ksize == 1 ? TC_BM : TC_WROWS; }

// Rows of the weight box {64, rows, 1 plane}.  A CTA's share of a tile is P*BN/TC_CLUSTER of its P*BN rows (planes stacked),
// loaded in boxes that divide both that share and a plane, so none crosses a plane; a multiple of 8 rows keeps every box on
// a 1024-byte swizzle atom.
__host__ __device__ constexpr int tc_gcd(int a, int b) { return b ? tc_gcd(b, a % b) : a; }
__host__ __device__ constexpr int tc_wbox_rows(int bn, int planes) { return tc_gcd(planes * bn / TC_CLUSTER, bn); }

template <int BN, int PLANES> struct TcShape {
    static constexpr int A_BYTES = PLANES * TC_WROWS * 128;   // an A window slot: 17 KB per plane, a multiple of 1024 B
    static constexpr int B_PLANE = BN * 128;
    static constexpr int B_BYTES = PLANES * B_PLANE;
    // a window serves k consecutive weight tiles, so the weight ring is the deeper one
    static constexpr int W_STAGES = 3 * A_BYTES + 6 * B_BYTES <= TC_SMEM_BUDGET ? 3 : 2;
    static constexpr int B_FIT = (TC_SMEM_BUDGET - W_STAGES * A_BYTES) / B_BYTES;
    static constexpr int B_STAGES = B_FIT > 8 ? 8 : B_FIT;
    static constexpr int SMEM = W_STAGES * A_BYTES + B_STAGES * B_BYTES + 1024;
};

template <int BN, int PLANES, bool F16>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_wg_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const TcArgs a) {
    using S = TcShape<BN, PLANES>;
    constexpr int WS = S::W_STAGES, BS = S::B_STAGES;
    constexpr int NACC = BN / 2;   // fp32 registers per thread of one m64 x BN accumulator
    static_assert(S::B_STAGES >= 2, "shared memory holds fewer than two weight tiles");
    constexpr int WBOX = tc_wbox_rows(BN, PLANES), WSHARE = PLANES * BN / TC_CLUSTER;
    static_assert(WSHARE * TC_CLUSTER == PLANES * BN && WBOX % 8 == 0, "weight tile does not split into whole swizzle atoms");

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);   // SWIZZLE_128B needs 1024 B
    uint8_t* const wring = smem;                          // A windows
    uint8_t* const bring = smem + WS * S::A_BYTES;        // B tiles, written by the TMA multicasts of the whole cluster
    __shared__ __align__(8) uint64_t wfull[WS], wempty[WS], bfull[BS], bempty[BS];
    __shared__ float s_bias[BN];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // Row tiles start at every image, so none covers only the gap rows after an image's last pixel.  A CTA past the last
    // image (grid.x is rounded up to whole clusters) runs the load / consume protocol with its cluster and stores nothing.
    const int img = blockIdx.x / a.tiles_img;
    const long long m0 = (long long)img * a.Hs * a.Wp + (long long)(blockIdx.x % a.tiles_img) * TC_BM;
    const int n0 = blockIdx.y * BN;
    const int ks = a.ksize, taps = ks * ks;
    const int num_k = taps * a.kblocks_per_tap;

    if (threadIdx.x == 0) {
        // bempty: released by the 8 consumer warps of every CTA in the cluster, since each weight tile is written into all
        for (int s = 0; s < WS; s++) { mbar_init(&wfull[s], 1); mbar_init(&wempty[s], 8); }
        for (int s = 0; s < BS; s++) { mbar_init(&bfull[s], 1); mbar_init(&bempty[s], 8 * TC_CLUSTER); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    }
    for (int i = threadIdx.x; i < BN; i += TC_THREADS) s_bias[i] = (n0 + i < a.cout) ? a.bias[n0 + i] : 0.f;
    cluster_sync();   // every CTA's barriers are initialised before any multicast or remote arrive reaches them
    pdl_launch_dependents();
    pdl_wait();

    if (warp < 4) {
        // ===== TMA producer: per (64-channel block, filter row) one A window {64 ch, 136 rows, P planes}, then per tap
        // of the row this CTA's share of the B tile {64, BN, P}, multicast to the cluster; K order = channel block,
        // filter row, tap (the order of the weight K index) =====
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(TC_PRODUCER_REGS));
        if (threadIdx.x == 0) {
            const uint32_t a_tx = PLANES * tc_window_rows(ks) * 128;
            const int f0 = (int)cluster_ctarank() * WSHARE;   // first row of this CTA's share in the stacked planes
            int wc = 0, bc = 0;   // windows / weight tiles issued
            for (int kb = 0; kb < a.kblocks_per_tap; kb++)
                for (int r = 0; r < ks; r++, wc++) {
                    const int w = wc % WS;
                    mbar_wait(&wempty[w], ((uint32_t)(wc / WS) & 1u) ^ 1u);
                    mbar_expect_tx(&wfull[w], a_tx);
                    const int row0 = (int)(m0 + (long long)(r - a.pad) * a.Wp - a.pad);
                    tma_load_3d(wring + (size_t)w * S::A_BYTES, &tmA, &wfull[w], kb * TC_BK, row0, 0);
                    for (int q = 0; q < ks; q++, bc++) {
                        const int b = bc % BS;
                        mbar_wait(&bempty[b], ((uint32_t)(bc / BS) & 1u) ^ 1u);   // free in every CTA of the cluster
                        mbar_expect_tx(&bfull[b], S::B_BYTES);                    // the whole tile, from all the CTAs
#pragma unroll
                        for (int f = f0; f < f0 + WSHARE; f += WBOX)
                            tma_load_3d_mc(bring + (size_t)b * S::B_BYTES + (size_t)f * 128, &tmB, &bfull[b],
                                           (r * ks + q) * a.cin_k + kb * TC_BK, n0 + f % BN, f / BN, (uint16_t)((1u << TC_CLUSTER) - 1));
                    }
                }
            // The partners' consumers arrive on this CTA's bempty: stay until the last use of every slot is released.
            for (int i = 0; i < BS; i++, bc++) mbar_wait(&bempty[bc % BS], ((uint32_t)(bc / BS) & 1u) ^ 1u);
        }
        return;
    }
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(TC_CONSUMER_REGS));

    // ===== consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of the tile =====
    const int wg = (warp >> 2) - 1;
    float acc_h[NACC], sum_h[NACC], acc_c[NACC];
#pragma unroll
    for (int j = 0; j < NACC; j++) { acc_h[j] = 0.f; sum_h[j] = 0.f; acc_c[j] = 0.f; }
    const int cs = a.chunk_iters;
    const uint32_t a_plane = tc_window_rows(ks) * 128;   // plane stride of the window as the TMA box lays it out
    // K steps (it: one tap x 64 channels) in hi*hi chunks of cs steps, the last one possibly shorter.  One wgmma group stays
    // in flight: step s is issued before step s - 1 is waited for, and only then are step s - 1's weight slot (and its
    // window, after the window's last tap) released.  A chunk ends with wait_group 0 and the round-to-nearest chunk sum in
    // straight-line code, so no accumulator is read while a group writing it is in flight.
    int it = 0, wc = 0, q = 0;   // K step, window, tap within the window
    for (int c0 = 0; c0 < num_k; c0 += cs) {
        const int n = min(cs, num_k - c0);
        int prev_b = 0, prev_w = -1;   // the previous step's weight slot, and its window slot if that was the window's last tap
        for (int s = 0; s < n; s++, it++) {
            const int w = wc % WS;
            if (q == 0) mbar_wait(&wfull[w], (uint32_t)(wc / WS) & 1u);
            const int b = it % BS;
            mbar_wait(&bfull[b], (uint32_t)(it / BS) & 1u);
            // tap q: window rows [q + 64 wg, q + 64 wg + 64)
            const uint32_t sa = smem_u32(wring + (size_t)w * S::A_BYTES) + (uint32_t)(wg * 64 * 128) + (uint32_t)(q * 128);
            const uint32_t sb = smem_u32(bring + (size_t)b * S::B_BYTES);
            const uint32_t h_acc = s != 0;   // 0: hi*hi chunk starts from zero
            wg_fence();
#pragma unroll
            for (int k = 0; k < TC_BK / 16; k++) {
                Wgmma<BN>::template mma<F16>(acc_h, wg_desc(sa + k * 32), wg_desc(sb + k * 32), (k != 0) | h_acc);
                if constexpr (PLANES > 1) {
#pragma unroll
                    for (int pa = 0; pa < PLANES; pa++)
#pragma unroll
                        for (int pb = 0; pb < PLANES - pa; pb++) {
                            if (pa + pb == 0) continue;
                            const uint32_t first = it == 0 && k == 0 && pa + pb == 1 && pa == 0;
                            Wgmma<BN>::template mma<F16>(acc_c, wg_desc(sa + pa * a_plane + k * 32),
                                                         wg_desc(sb + pb * S::B_PLANE + k * 32), first ? 0u : 1u);
                        }
                }
            }
            wg_commit();
            wg_wait_1();
            if (s > 0) tc_release(bempty, wempty, prev_b, prev_w, lane);
            prev_b = b;
            prev_w = q == ks - 1 ? w : -1;
            if (++q == ks) { q = 0; wc++; }
        }
        wg_wait_all();
        tc_release(bempty, wempty, prev_b, prev_w, lane);
#pragma unroll
        for (int j = 0; j < NACC; j++) sum_h[j] = __fadd_rn(sum_h[j], acc_h[j]);
    }

    // ===== epilogue: sum, bias, ReLU, re-split into planes, store =====
    const int per_img = a.Hs * a.Wp;
    const int cout8 = (a.cout + 7) & ~7;
    const float out_scale = __ldg(a.out_scale);
    float range_max = 0.f;   // largest |value| this warp stores (range tracking of the fp16 planes, see TcArgs::range)
#pragma unroll
    for (int hr = 0; hr < 2; hr++) {
        const long long m = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + hr * 8;
        const int n = (int)(m / per_img), rem = (int)(m % per_img);
        const int y = rem / a.Wp, x = rem % a.Wp;
        // gap rows are never written and stay zero; the rows of the next image belong to its own tiles
        if (m >= a.M || n != img || x >= a.W || y >= a.H) continue;
#pragma unroll
        for (int g = 0; g < BN / 8; g++) {
            const int c = g * 8 + (lane & 3) * 2, j = g * 4 + hr * 2;
            const int co = n0 + c;
            float v[2];
#pragma unroll
            for (int e = 0; e < 2; e++) {
                float t = PLANES > 1 ? __fadd_rn(sum_h[j + e], acc_c[j + e]) : sum_h[j + e];
                t = __fmaf_rn(t, out_scale, s_bias[c + e]);   // out_scale is a power of two: exact
                if (a.relu) t = fmaxf(t, 0.f);
                v[e] = t;
                if (co + e < a.cout) range_max = fmaxf(range_max, fabsf(t));
            }
            if (a.planar) {
#pragma unroll
                for (int e = 0; e < 2; e++)
                    if (co + e < a.cout) a.planar[(((size_t)n * a.planar_C + a.planar_coff + co + e) * a.H + y) * a.W + x] = v[e];
            } else if (co < cout8) {
                __nv_bfloat16* orow = a.out + (size_t)m * a.out_pitch + a.out_coff + co;
#pragma unroll
                for (int p = 0; p < PLANES; p++) *(uint32_t*)(orow + (size_t)p * a.out_plane) = split_pair<F16>(v[0], v[1]);
            }
        }
    }
    range_publish(a.range, range_max);
}

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

static int env_int(const char* name, int dflt) {
    const char* v = getenv(name);
    return v ? atoi(v) : dflt;
}

template <int BN, int PLANES, bool F16>
static int launch_inst(const TcLayer& l, const TcArgs& a, dim3 grid, cudaStream_t st, int bmap) {
    auto kern = conv_wg_kernel<BN, PLANES, F16>;
    constexpr int smem = TcShape<BN, PLANES>::SMEM;
    int dev = 0;
    cudaGetDevice(&dev);
    static std::atomic<unsigned long long> attr_done{0};   // bit d: attribute set on device d (it is per device; several threads launch)
    if (!(attr_done.load(std::memory_order_acquire) >> (dev & 63) & 1ull)) {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return -1;
        attr_done.fetch_or(1ull << (dev & 63), std::memory_order_release);
    }
    // PDL (see pdl_wait): back-to-back conv kernels overlap the next one's prologue with the previous one's tail
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = dim3(TC_THREADS, 1, 1); cfg.dynamicSmemBytes = (size_t)smem; cfg.stream = st;
    cudaLaunchAttribute at[2];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    // clusters of TC_CLUSTER row tiles share the weight tiles (see conv_wg_kernel); grid.x is a multiple of TC_CLUSTER
    at[1].id = cudaLaunchAttributeClusterDimension;
    at[1].val.clusterDim.x = TC_CLUSTER; at[1].val.clusterDim.y = 1; at[1].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 2;
    const CUtensorMap* maps = (const CUtensorMap*)l.maps;
    return cudaLaunchKernelEx(&cfg, kern, maps[0], maps[bmap], a) == cudaSuccess ? 1 : -1;
}

template <int BN>
static int launch_bn(const TcLayer& l, const TcArgs& a, dim3 grid, cudaStream_t st, int bmap) {
    const PlaneFmt f = l.d.fmt;
    if (f.planes == 1) return f.f16 ? launch_inst<BN, 1, true>(l, a, grid, st, bmap) : launch_inst<BN, 1, false>(l, a, grid, st, bmap);
    if (f.planes == 2 && f.f16 == PARITY_F16) return launch_inst<BN, 2, PARITY_F16>(l, a, grid, st, bmap);
    if constexpr (BN <= 64) { if (f.planes == 3 && !f.f16) return launch_inst<BN, 3, false>(l, a, grid, st, bmap); }
    return -1;   // no kernel for this tile width and plane format (tc_bn never picks one)
}

static int encode(EncodeTiledFn enc, CUtensorMap* map, const void* base, cuuint64_t d0, cuuint64_t d1, cuuint64_t d2, cuuint64_t s1,
                  cuuint64_t s2, cuuint32_t b1, cuuint32_t b2, CUtensorMapL2promotion l2) {
    cuuint64_t dims[3] = {d0, d1, d2};
    cuuint64_t strides[2] = {s1, s2};
    cuuint32_t box[3] = {(cuuint32_t)TC_BK, b1, b2};
    cuuint32_t es[3] = {1, 1, 1};
    return (int)enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, (void*)base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

int tc_layer_create(const TcLayerDesc& d, TcLayer& out, std::string& err) {
    EncodeTiledFn enc = get_encode();
    if (!enc) { err = "cuTensorMapEncodeTiled unavailable"; return -1; }
    if (d.in_cused % TC_BK) { err = "input channels not a multiple of 64"; return -1; }
    if (d.fmt.planes < 1 || d.fmt.planes > 3) { err = "1 to 3 planes"; return -1; }
    if (d.ksize < 1 || d.ksize > TC_KMAX) { err = "filter size above " + std::to_string(TC_KMAX) + " (A window rows)"; return -1; }
    out.d = d;
    out.bn = tc_bn(d.cout_pad, d.fmt.planes);
    CUtensorMap* maps = nullptr;
    if (posix_memalign((void**)&maps, 64, 3 * sizeof(CUtensorMap))) { err = "alloc"; return -1; }
    memset(maps, 0, 3 * sizeof(CUtensorMap));
    const cuuint64_t K = (cuuint64_t)d.ksize * d.ksize * d.in_cused;
    const cuuint64_t P = (cuuint64_t)d.fmt.planes;
    // A: [planes][M][pitch], box {64, window rows, planes}
    int r = encode(enc, &maps[0], d.in, d.in_cused, d.geo.M, P, (cuuint64_t)d.in_pitch * 2, (cuuint64_t)d.in_plane * 2,
                   tc_window_rows(d.ksize), d.fmt.planes,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
    // B: [planes][cout_pad][K], box {64, part of a plane, 1} (a CTA's share of a {64, bn, planes} tile is one or more such
    // boxes, tc_wbox_rows); and for half-width tiles (more CTAs for small problems, see tc_layer_launch)
    if (!r) r = encode(enc, &maps[1], d.w, K, d.cout_pad, P, K * 2, K * 2 * d.cout_pad, tc_wbox_rows(out.bn, d.fmt.planes), 1,
                       CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
    if (!r && out.bn >= 64) r = encode(enc, &maps[2], d.w, K, d.cout_pad, P, K * 2, K * 2 * d.cout_pad, tc_wbox_rows(out.bn / 2, d.fmt.planes), 1,
                                       CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
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
    TcArgs a;
    a.bias = d.bias;
    a.out = (__nv_bfloat16*)d.out; a.out_pitch = d.out_pitch; a.out_coff = d.out_coff; a.out_plane = d.out_plane;
    a.planar = d.planar; a.planar_C = d.planar_C; a.planar_coff = d.planar_coff;
    a.cout = d.cout; a.relu = d.relu; a.out_scale = d.out_scale; a.range = d.range;
    a.ksize = d.ksize; a.pad = d.pad; a.kblocks_per_tap = d.in_cused / TC_BK; a.cin_k = d.in_cused;
    a.W = d.geo.W; a.H = d.geo.H; a.Wp = d.geo.Wp; a.Hs = d.geo.Hs;
    a.M = (long long)nimg * d.geo.Hs * d.geo.Wp;
    // hi*hi accumulation chunk with split planes and in the fp16 fast mode: one 7-tap filter row (448 K), two 3-tap rows (384 K)
    // or four 1x1 blocks (256 K); bf16x1 runs one chain over the whole K
    const int nk = d.ksize * d.ksize * a.kblocks_per_tap;
    a.chunk_iters = (d.fmt.planes >= 2 || d.fmt.f16) ? (d.ksize >= 7 ? 7 : (d.ksize >= 3 ? 6 : 4)) : nk;
    static int nsm = 0;
    if (!nsm) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev); }
    // Tile width: the full width is the efficient shape (the A tile is re-read per N tile), but a single frame at the
    // 46x82 level has only 33 row tiles for 132 SMs: take half the width when (CTAs that can run at once) x (relative
    // efficiency of the shape) is larger.  share: layers running concurrently on other streams take their part of the SMs.
    const long long mt = (a.M + TC_BM - 1) / TC_BM;
    const long long sms = std::max(1, nsm / (share < 1 ? 1 : share));
    static const int narrow_env = env_int("PE_TC_NARROW", 1);
    int bn = l.bn, bmap = 1;
    if (narrow_env && l.bn >= 64) {
        const double sfull = (double)std::min<long long>(mt * (d.cout_pad / l.bn), sms) * 1.00;
        const double shalf = (double)std::min<long long>(mt * (d.cout_pad / (l.bn / 2)), sms) * 0.80;
        if (shalf > sfull) { bn = l.bn / 2; bmap = 2; }
    }
    // row tiles per image: up to its last pixel (H - 1) * Wp + W - 1; the grid in whole clusters
    a.tiles_img = ((d.geo.H - 1) * d.geo.Wp + d.geo.W + TC_BM - 1) / TC_BM;
    const long long tiles = ((long long)nimg * a.tiles_img + TC_CLUSTER - 1) / TC_CLUSTER * TC_CLUSTER;
    const dim3 grid((unsigned)tiles, (unsigned)(d.cout_pad / bn), 1);
    switch (bn) {
        case 128: return launch_bn<128>(l, a, grid, st, bmap);
        case 64: return launch_bn<64>(l, a, grid, st, bmap);
        case 48: return launch_bn<48>(l, a, grid, st, bmap);
        case 32: return launch_bn<32>(l, a, grid, st, bmap);
        default: return launch_bn<16>(l, a, grid, st, bmap);
    }
}

}  // namespace pe
