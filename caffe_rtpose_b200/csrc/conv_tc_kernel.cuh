// Kernel side of the wgmma / TMA implicit-GEMM convolution (see conv_tc.cu for the design): argument block, PTX
// wrappers, conv_wg_kernel and its launcher.  Shared by conv_tc.cu (16-bit planes), conv_fp8.cu (e4m3), conv_s8.cu (s8) and
// conv_s8x2.cu (two s8 planes).
#pragma once
#include <cuda.h>
#include <cuda_fp8.h>

#include <atomic>
#include <type_traits>

#include "common.h"
#include "conv_tc.h"
#include "kernels.h"

namespace pe {

struct TcArgs {
    const float* bias;
    void* out; int out_pitch, out_coff; long long out_plane;   // output planes of the kernel's OUT element kind (pitch in elements)
    float* planar; int planar_C, planar_coff;
    int cout, relu;
    const float* out_scale;                   // -> 2^-k in the packed buffer: the weights of this layer carry a factor 2^k (fp16 planes);
                                              // s8: -> the per-channel epilogue factors f_c [cout_pad]
    int ksize, pad, kblocks_per_tap, cin_k;   // cin_k = channels per tap in the weight K ordering
    int W, H, Wp, Hs;
    long long M;
    int tiles_img;                            // row tiles per image: blockIdx.x = image * tiles_img + tile
    int chunk_iters;                          // K iterations (one channel block of one tap each) per hi*hi accumulation chunk
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

// D(64 x N) (+)= A(64 x K) * B(N x K)^T, both K-major in shared memory (the only layout the 8-bit kinds take, so no transpose
// operands); scale_d = 0 overwrites D.  One K step is 32 bytes of the 128-byte swizzle rows: k16 in fp16 / bf16, k32 in e4m3 / s8.
// Register j of a thread holds row 16*(warp%4) + lane/4 + 8*((j/2)%2), column 8*(j/4) + 2*(lane%4) + j%2.  s8 accumulates in
// s32: the products and their sums are exact integers, so nothing is chunked while |acc| stays inside s32 (the engine bounds K,
// Precision::max_k).
template <int N, int ELEM> struct Wgmma;
#define PE_WG_OUT8 "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
#define PE_WG_OUT16 PE_WG_OUT8, "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
#define PE_WG_OUT24 PE_WG_OUT16, "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
#define PE_WG_OUT32 PE_WG_OUT24, "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
#define PE_WG_OUT64 PE_WG_OUT32, "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), \
    "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]),  \
    "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]),  \
    "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
#define PE_WG_OUT8_S32 "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7])
#define PE_WG_OUT16_S32 PE_WG_OUT8_S32, "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
#define PE_WG_OUT24_S32 PE_WG_OUT16_S32, "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23])
#define PE_WG_OUT32_S32 PE_WG_OUT24_S32, "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
#define PE_WG_OUT64_S32 PE_WG_OUT32_S32, "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), \
    "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]),      \
    "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]),      \
    "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
#define PE_WG_REGS8 "%0,%1,%2,%3,%4,%5,%6,%7"
#define PE_WG_REGS16 PE_WG_REGS8 ",%8,%9,%10,%11,%12,%13,%14,%15"
#define PE_WG_REGS24 PE_WG_REGS16 ",%16,%17,%18,%19,%20,%21,%22,%23"
#define PE_WG_REGS32 PE_WG_REGS24 ",%24,%25,%26,%27,%28,%29,%30,%31"
#define PE_WG_REGS64 PE_WG_REGS32 ",%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54," \
    "%55,%56,%57,%58,%59,%60,%61,%62,%63"
// Wgmma<N, ELEM>: NR accumulator registers, then operands %NR (A), %NR+1 (B), %NR+2 (scale_d).  K: the K step; TYPES: the
// type suffix; ACC / OUT: the accumulator type and register list (PE_WG_OUTn##OUT); IMM: the immediates after the predicate.
#define PE_WGMMA(N, NR, DA, DB, SD, ELEM, K, TYPES, ACC, OUT, IMM)                                                             \
    template <> struct Wgmma<N, ELEM> {                                                                                         \
        __device__ __forceinline__ static void mma(ACC* d, uint64_t da, uint64_t db, uint32_t scale_d) {                        \
            asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %" #SD ", 0;\n"                                                     \
                         "wgmma.mma_async.sync.aligned.m64n" #N "k" #K "." TYPES " {" PE_WG_REGS##NR "}, %" #DA ", %" #DB ", p" \
                         IMM ";\n}"                                                                                             \
                         : PE_WG_OUT##NR##OUT : "l"(da), "l"(db), "r"(scale_d));                                                \
        }                                                                                                                       \
    };
#define PE_WGMMA_WIDTHS(ELEM, K, TYPES, ACC, OUT, IMM)          \
    PE_WGMMA(16, 8, 8, 9, 10, ELEM, K, TYPES, ACC, OUT, IMM)    \
    PE_WGMMA(32, 16, 16, 17, 18, ELEM, K, TYPES, ACC, OUT, IMM) \
    PE_WGMMA(48, 24, 24, 25, 26, ELEM, K, TYPES, ACC, OUT, IMM) \
    PE_WGMMA(64, 32, 32, 33, 34, ELEM, K, TYPES, ACC, OUT, IMM) \
    PE_WGMMA(128, 64, 64, 65, 66, ELEM, K, TYPES, ACC, OUT, IMM)
PE_WGMMA_WIDTHS(ELEM_F16, 16, "f32.f16.f16", float, , ", 1, 1, 0, 0")
PE_WGMMA_WIDTHS(ELEM_BF16, 16, "f32.bf16.bf16", float, , ", 1, 1, 0, 0")
PE_WGMMA_WIDTHS(ELEM_E4M3, 32, "f32.e4m3.e4m3", float, , ", 1, 1")
PE_WGMMA_WIDTHS(ELEM_S8, 32, "s32.s8.s8", int, _S32, "")
PE_WGMMA_WIDTHS(ELEM_U8, 32, "s32.u8.s8", int, _S32, "")   // u8 activations (A) x s8 weights (B), the s8 rate

// fp32 -> s8, round to nearest even, saturating to [-128, 127] (cvt.rni.sat.s8.f32; NaN gives 0)
__device__ __forceinline__ uint32_t f32_to_s8(float x) {
    int q;
    asm("cvt.rni.sat.s8.f32 %0, %1;" : "=r"(q) : "f"(x));
    return (uint32_t)q & 0xffu;
}

// fp32 -> u8, round to nearest even, saturating to [0, 255] (cvt.rni.sat.u8.f32; NaN gives 0)
__device__ __forceinline__ uint32_t f32_to_u8(float x) {
    uint32_t q;
    asm("cvt.rni.sat.u8.f32 %0, %1;" : "=r"(q) : "f"(x));
    return q & 0xffu;
}

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
// Channels per K block of an element kind (PlaneElem): always one 128-byte swizzle row, so e4m3 blocks hold 128 channels.
// The alternative, 64-channel e4m3 blocks in SWIZZLE_64B boxes, would pad a 185-channel Concat to 192 instead of 256 (the
// stage inputs: 28 % fewer MACs in Mconv1), but it keeps the fp16 kernel's number of K steps - each step's mbarrier waits,
// releases and descriptor arithmetic - while halving the tensor-core work per step, so the per-step overhead would eat the
// gain everywhere else.  128-channel blocks keep every byte of the fp16 geometry (boxes, slots, descriptors, the 32-byte K
// advance) and halve the steps.  The engine pads e4m3 and s8 activations to 128 channels (Precision::act_cpad).
__host__ __device__ constexpr int tc_block_ch(PlaneElem elem) { return 128 / elem_size(elem); }
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

// Rows of the weight box {channel block, rows, 1 plane}.  A CTA's share of a tile is P*BN/TC_CLUSTER of its P*BN rows (planes stacked),
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

// ELEM: element kind of the A windows and weight tiles; OUT: of the stored output planes (conv1_1 of the e4m3 mode reads
// its fp16 im2col input and writes e4m3).  ELEM = OUT = s8: s32 accumulators over the whole K (the host sets chunk_iters to
// it), and the per-channel epilogue t = acc * f_c + b'_c (no FMA) before cvt.rni.sat.s8.  ELEM = u8 (PE_PREC_FLAG_U8): the same
// with u8 x s8 MMAs; OUT = u8: ReLU, then cvt.rni.sat.u8.  PLANES = 2, ELEM = OUT = s8 (PE_PREC_S8X2): hi*hi into acc_h and
// hi*lo + lo*hi into acc_c, both s32 over the whole K; the epilogue takes S = 256 acc_h + acc_c in 64 bits (exact), t = float(S) *
// f_c + b'_c, and stores v = sat(rint(t)) in [-32768, 32639] as the planes hi = (v + 128) >> 8, lo = v - 256 hi (s8.h).
template <int BN, int PLANES, int ELEM, int OUT>
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
    constexpr bool S8 = ELEM == ELEM_S8 || ELEM == ELEM_U8;   // integer sums and the per-channel epilogue
    __shared__ float s_bias[S8 ? 2 * BN : BN];   // s8 / u8: the biases, then the per-channel factors

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // Row tiles start at every image, so none covers only the gap rows after an image's last pixel.  A CTA past the last
    // image (grid.x is rounded up to whole clusters) runs the load / consume protocol with its cluster and stores nothing.
    const int img = blockIdx.x / a.tiles_img;
    const long long m0 = (long long)img * a.Hs * a.Wp + (long long)(blockIdx.x % a.tiles_img) * TC_BM;
    const int n0 = blockIdx.y * BN;
    const int ks = a.ksize, taps = ks * ks;
    const int num_k = taps * a.kblocks_per_tap;
    constexpr int KB = tc_block_ch(PlaneElem(ELEM));

    if (threadIdx.x == 0) {
        // bempty: released by the 8 consumer warps of every CTA in the cluster, since each weight tile is written into all
        for (int s = 0; s < WS; s++) { mbar_init(&wfull[s], 1); mbar_init(&wempty[s], 8); }
        for (int s = 0; s < BS; s++) { mbar_init(&bfull[s], 1); mbar_init(&bempty[s], 8 * TC_CLUSTER); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    }
    for (int i = threadIdx.x; i < BN; i += TC_THREADS) s_bias[i] = (n0 + i < a.cout) ? a.bias[n0 + i] : 0.f;
    if constexpr (S8)
        for (int i = threadIdx.x; i < BN; i += TC_THREADS) s_bias[BN + i] = (n0 + i < a.cout) ? a.out_scale[n0 + i] : 0.f;
    cluster_sync();   // every CTA's barriers are initialised before any multicast or remote arrive reaches them
    pdl_launch_dependents();
    pdl_wait();

    if (warp < 4) {
        // ===== TMA producer: per (channel block, filter row) one A window {KB ch, 136 rows, P planes}, then per tap of the
        // row this CTA's share of the B tile {KB, BN, P}, multicast to the cluster (KB = 64 channels in 16 bits, 128 in e4m3:
        // 128 bytes either way); K order = channel block,
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
                    tma_load_3d(wring + (size_t)w * S::A_BYTES, &tmA, &wfull[w], kb * KB, row0, 0);
                    for (int q = 0; q < ks; q++, bc++) {
                        const int b = bc % BS;
                        mbar_wait(&bempty[b], ((uint32_t)(bc / BS) & 1u) ^ 1u);   // free in every CTA of the cluster
                        mbar_expect_tx(&bfull[b], S::B_BYTES);                    // the whole tile, from all the CTAs
#pragma unroll
                        for (int f = f0; f < f0 + WSHARE; f += WBOX)
                            tma_load_3d_mc(bring + (size_t)b * S::B_BYTES + (size_t)f * 128, &tmB, &bfull[b],
                                           (r * ks + q) * a.cin_k + kb * KB, n0 + f % BN, f / BN, (uint16_t)((1u << TC_CLUSTER) - 1));
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
    using Acc = std::conditional_t<S8, int, float>;
    Acc acc_h[NACC], acc_c[NACC];   // acc_c: the cross products of two planes
    float sum_h[NACC];
#pragma unroll
    for (int j = 0; j < NACC; j++) { acc_h[j] = 0.f; sum_h[j] = 0.f; acc_c[j] = 0.f; }
    const int cs = a.chunk_iters;
    const uint32_t a_plane = tc_window_rows(ks) * 128;   // plane stride of the window as the TMA box lays it out
    // K steps (it: one tap x one channel block) in hi*hi chunks of cs steps, the last one possibly shorter.  One wgmma group stays
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
            for (int k = 0; k < 4; k++) {   // 32-byte K steps of the 128-byte rows: k16 in 16 bits, k32 in e4m3
                Wgmma<BN, ELEM>::mma(acc_h, wg_desc(sa + k * 32), wg_desc(sb + k * 32), (k != 0) | h_acc);
                if constexpr (PLANES > 1) {
#pragma unroll
                    for (int pa = 0; pa < PLANES; pa++)
#pragma unroll
                        for (int pb = 0; pb < PLANES - pa; pb++) {
                            if (pa + pb == 0) continue;
                            const uint32_t first = it == 0 && k == 0 && pa + pb == 1 && pa == 0;
                            Wgmma<BN, ELEM>::mma(acc_c, wg_desc(sa + pa * a_plane + k * 32), wg_desc(sb + pb * S::B_PLANE + k * 32),
                                                 first ? 0u : 1u);
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
        if constexpr (!S8) {
#pragma unroll
            for (int j = 0; j < NACC; j++) sum_h[j] = __fadd_rn(sum_h[j], acc_h[j]);
        }
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
                float t;
                if constexpr (S8 && PLANES == 2) {
                    const long long sum = 256LL * acc_h[j + e] + acc_c[j + e];
                    t = __fadd_rn(__fmul_rn(__ll2float_rn(sum), s_bias[BN + c + e]), s_bias[c + e]);
                } else if constexpr (S8) {
                    t = __fadd_rn(__fmul_rn(__int2float_rn(acc_h[j + e]), s_bias[BN + c + e]), s_bias[c + e]);
                } else {
                    t = PLANES > 1 ? __fadd_rn(sum_h[j + e], acc_c[j + e]) : sum_h[j + e];
                    t = __fmaf_rn(t, out_scale, s_bias[c + e]);   // out_scale is a power of two: exact
                }
                if (a.relu) t = fmaxf(t, 0.f);
                v[e] = t;
                if (co + e < a.cout) range_max = fmaxf(range_max, fabsf(t));
            }
            if (a.planar) {
#pragma unroll
                for (int e = 0; e < 2; e++)
                    if (co + e < a.cout) a.planar[(((size_t)n * a.planar_C + a.planar_coff + co + e) * a.H + y) * a.W + x] = v[e];
            } else if constexpr (OUT == ELEM_S8 && PLANES == 2) {
                if (co < cout8) {
                    uint32_t hi = 0, lo = 0;
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        const int q = min(max(__float2int_rn(v[e]), -32768), 32639);   // rint, saturated (NaN gives 0)
                        const int h = (q + 128) >> 8;
                        hi |= ((uint32_t)h & 0xffu) << (8 * e);
                        lo |= ((uint32_t)(q - 256 * h) & 0xffu) << (8 * e);
                    }
                    int8_t* o = (int8_t*)a.out + (size_t)m * a.out_pitch + a.out_coff + co;
                    *(uint16_t*)o = (uint16_t)hi;
                    *(uint16_t*)(o + a.out_plane) = (uint16_t)lo;
                }
            } else if constexpr (OUT == ELEM_S8) {
                if (co < cout8)
                    *(uint16_t*)((int8_t*)a.out + (size_t)m * a.out_pitch + a.out_coff + co) = (uint16_t)(f32_to_s8(v[0]) | f32_to_s8(v[1]) << 8);
            } else if constexpr (OUT == ELEM_U8) {
                if (co < cout8)
                    *(uint16_t*)((uint8_t*)a.out + (size_t)m * a.out_pitch + a.out_coff + co) = (uint16_t)(f32_to_u8(v[0]) | f32_to_u8(v[1]) << 8);
            } else if (OUT == ELEM_E4M3) {
                // round to nearest, saturating to +-448 as the range check expects (a larger |t| is PE_ERR_RANGE)
                if (co < cout8)
                    *(__nv_fp8x2_storage_t*)((uint8_t*)a.out + (size_t)m * a.out_pitch + a.out_coff + co) =
                        __nv_cvt_float2_to_fp8x2(make_float2(v[0], v[1]), __NV_SATFINITE, __NV_E4M3);
            } else if (co < cout8) {
                __nv_bfloat16* orow = (__nv_bfloat16*)a.out + (size_t)m * a.out_pitch + a.out_coff + co;
#pragma unroll
                for (int p = 0; p < PLANES; p++) *(uint32_t*)(orow + (size_t)p * a.out_plane) = split_pair<OUT == ELEM_F16>(v[0], v[1]);
            }
        }
    }
    range_publish(a.range, range_max);
}

template <int BN, int PLANES, int ELEM, int OUT>
static int launch_inst(const TcLayer& l, const TcArgs& a, dim3 grid, cudaStream_t st, int bmap) {
    auto kern = conv_wg_kernel<BN, PLANES, ELEM, OUT>;
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

// The instance <bn, PLANES, ELEM, OUT> for the grid's tile width bn.  Three planes run at BN <= 64 only (tc_bn).
template <int PLANES, int ELEM, int OUT>
static int launch_widths(const TcLayer& l, const TcArgs& a, dim3 grid, cudaStream_t st, int bmap, int bn) {
    switch (bn) {
        case 128: if constexpr (PLANES < 3) return launch_inst<128, PLANES, ELEM, OUT>(l, a, grid, st, bmap); else return -1;
        case 64: return launch_inst<64, PLANES, ELEM, OUT>(l, a, grid, st, bmap);
        case 48: return launch_inst<48, PLANES, ELEM, OUT>(l, a, grid, st, bmap);
        case 32: return launch_inst<32, PLANES, ELEM, OUT>(l, a, grid, st, bmap);
        case 16: return launch_inst<16, PLANES, ELEM, OUT>(l, a, grid, st, bmap);
        default: return -1;
    }
}

// Layers with e4m3 output (conv_fp8.cu), s8 layers (conv_s8.cu), the format boundaries of mixed engines (conv_mixed.cu), the
// layers that read or store u8 (conv_u8.cu) and the two-plane s8 layers (conv_s8x2.cu):
// their instances live in translation units of their own.
int launch_e4m3(const TcLayer& l, const TcArgs& a, dim3 grid, cudaStream_t st, int bmap, int bn);
int launch_s8(const TcLayer& l, const TcArgs& a, dim3 grid, cudaStream_t st, int bmap, int bn);
int launch_mixed(const TcLayer& l, const TcArgs& a, dim3 grid, cudaStream_t st, int bmap, int bn);
int launch_u8(const TcLayer& l, const TcArgs& a, dim3 grid, cudaStream_t st, int bmap, int bn);
int launch_s8x2(const TcLayer& l, const TcArgs& a, dim3 grid, cudaStream_t st, int bmap, int bn);

}  // namespace pe
