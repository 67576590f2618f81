// The 2:4-sparse s8 convolution (PE_PREC_S8X1 layers whose packed weights are 2:4 in every aligned group of four, engine.cu
// picks them at pe_commit_weights).  wgmma.mma_async.sp m64nNk64 s8 x s8 -> s32 runs a logical K of 64 in the issue slot of a
// dense k32 MMA, but only its A operand can be sparse, so the roles of conv_wg_kernel (conv_tc_kernel.cuh) are swapped:
//   * A: the compressed weights, 64 output channels per consumer warpgroup, 128 per CTA: per K step (one tap x one 128-channel
//     block) a TMA box {64 B, 128 rows} (SWIZZLE_64B) of the values and a 2 KB bulk copy of the metadata words (s8_sparse.h),
//     into one slot of the weight ring, on one mbarrier.  Each thread reads its two metadata words from the slot.
//   * B: the activation window of conv_wg_kernel with N pixel rows instead of 128: per (128-channel block, filter row) one TMA
//     box {128 B, N + 8 rows}; tap q reads rows [q, q + N) through the descriptor start address.
//   * A K step is two sparse MMAs, k64 each: A advances 32 compressed bytes in its 64-byte swizzle row, B 64 bytes in its
//     128-byte one.
// The accumulator holds output channels in rows and pixels in columns.  The sums are the dense kernel's exact s32 sums (the
// pruned weights are zeros either way), and the epilogue is its per-channel t = acc * f_c + b'_c without FMA, ReLU,
// cvt.rni.sat.s8, so a sparse layer gives the dense layer's bits.  NHWC s8 outputs are staged in shared memory and leave in
// 16-byte vectors; the planar fp32 maps are pixel-contiguous per channel and store from the registers.  Kept from the dense
// kernel: producer / consumer warpgroups with setmaxnreg, the mbarrier rings, one wgmma group in flight, PDL, row tiles that
// start at every image (gap rows are never written), range_publish of the unrounded maximum.  No cluster multicast: the
// compressed tile is 5/8 of the dense one's bytes (metadata included).
#include "conv_tc_kernel.cuh"
#include "s8_sparse.h"

namespace pe {

struct SpArgs {
    const float* bias;      // b'_c [cout_pad], then the factors f_c [cout_pad]
    const uint8_t* meta;    // the layer's metadata (s8_sparse.h)
    int8_t* out; int out_pitch, out_coff;
    float* planar; int planar_C, planar_coff;
    int cout, relu;
    int ksize, pad, kblocks_per_tap;
    int W, H, Wp, Hs;
    long long M;
    int tiles_img;          // pixel tiles per image: blockIdx.x = image * tiles_img + tile
    unsigned* range;
};

__host__ __device__ constexpr int sp_window_rows(int ksize, int n) { return ksize == 1 ? n : n + TC_KMAX - 1; }

template <int N> struct SpShape {
    static constexpr int X_BYTES = (N + TC_KMAX - 1) * 128;   // a window slot: 9 or 17 KB, a multiple of 1024 B
    static constexpr int V_BYTES = SP_BM * 64;                // compressed values of one K step
    static constexpr int W_BYTES = V_BYTES + SP_META_STEP;    // + their metadata: 10 KB
    static constexpr int XS = 3, WS = 8;
    static constexpr int STAGE_BYTES = 2 * N * 64;            // NHWC staging: per warpgroup [N pixels][64 channels]
    static constexpr int SMEM = XS * X_BYTES + WS * W_BYTES + STAGE_BYTES + 1024;
    static_assert(SMEM <= TC_SMEM_BUDGET, "sparse tile does not fit in shared memory");
};

// K-major SWIZZLE_64B descriptor of the compressed weights: 64-byte rows, 8-row atoms of 512 B (SBO), layout type 2.
__device__ __forceinline__ uint64_t sp_desc(uint32_t saddr) {
    return (uint64_t)((saddr >> 4) & 0x3FFF) | (uint64_t)1 << 16 | (uint64_t)(512 >> 4) << 32 | (uint64_t)2 << 62;
}
// bytes from global memory to shared memory, completing on `bar` (non-tensor bulk copy; size a multiple of 16)
__device__ __forceinline__ void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// D(64 x N) (+)= A(64 x 64, 2:4 sparse, metadata e) * B(N x 64)^T; sparsity selector 0 (8-bit types: every thread holds metadata)
template <int N> struct WgmmaSp;
#define PE_WGSP(N, NR, DA, DB, E, SD)                                                                                        \
    template <> struct WgmmaSp<N> {                                                                                          \
        __device__ __forceinline__ static void mma(int* d, uint64_t da, uint64_t db, uint32_t e, uint32_t scale_d) {         \
            asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %" #SD ", 0;\n"                                                  \
                         "wgmma.mma_async.sp.sync.aligned.m64n" #N "k64.s32.s8.s8 {" PE_WG_REGS##NR "}, %" #DA ", %" #DB \
                         ", %" #E ", 0, p;\n}"                                                                               \
                         : PE_WG_OUT##NR##_S32 : "l"(da), "l"(db), "r"(e), "r"(scale_d));                                   \
        }                                                                                                                    \
    };
PE_WGSP(64, 32, 32, 33, 34, 35)
PE_WGSP(128, 64, 64, 65, 66, 67)

template <int N>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_wg_kernel_sparse(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, const SpArgs a) {
    using S = SpShape<N>;
    constexpr int XS = S::XS, WS = S::WS, NACC = N / 2;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint8_t* const xring = smem;                         // activation windows
    uint8_t* const wring = smem + XS * S::X_BYTES;       // compressed weights + metadata
    uint8_t* const stage = wring + WS * S::W_BYTES;
    __shared__ __align__(8) uint64_t xfull[XS], xempty[XS], wfull[WS], wempty[WS];
    __shared__ float s_epi[2 * SP_BM];   // b'_c, then f_c

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int img = blockIdx.x / a.tiles_img;
    const long long m0 = (long long)img * a.Hs * a.Wp + (long long)(blockIdx.x % a.tiles_img) * N;
    const int n0 = blockIdx.y * SP_BM;
    const int ks = a.ksize, num_k = ks * ks * a.kblocks_per_tap;

    if (threadIdx.x == 0) {
        for (int s = 0; s < XS; s++) { mbar_init(&xfull[s], 1); mbar_init(&xempty[s], 8); }
        for (int s = 0; s < WS; s++) { mbar_init(&wfull[s], 1); mbar_init(&wempty[s], 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmX) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmW) : "memory");
    }
    for (int i = threadIdx.x; i < SP_BM; i += TC_THREADS) {
        const bool in = n0 + i < a.cout;
        s_epi[i] = in ? a.bias[n0 + i] : 0.f;
        s_epi[SP_BM + i] = in ? a.bias[(size_t)gridDim.y * SP_BM + n0 + i] : 0.f;
    }
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();

    if (warp < 4) {
        // ===== TMA producer: per (channel block, filter row) one window, then per tap of the row one weight slot =====
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(TC_PRODUCER_REGS));
        if (threadIdx.x == 0) {
            const uint32_t x_tx = sp_window_rows(ks, N) * 128;
            const uint8_t* meta = a.meta + (size_t)blockIdx.y * num_k * SP_META_STEP;
            int xc = 0, wc = 0;
            for (int kb = 0; kb < a.kblocks_per_tap; kb++)
                for (int r = 0; r < ks; r++, xc++) {
                    const int x = xc % XS;
                    mbar_wait(&xempty[x], ((uint32_t)(xc / XS) & 1u) ^ 1u);
                    mbar_expect_tx(&xfull[x], x_tx);
                    tma_load_3d(xring + (size_t)x * S::X_BYTES, &tmX, &xfull[x], kb * 128, (int)(m0 + (long long)(r - a.pad) * a.Wp - a.pad), 0);
                    for (int q = 0; q < ks; q++, wc++) {
                        const int b = wc % WS, step = (r * ks + q) * a.kblocks_per_tap + kb;   // K order of the packed weights
                        mbar_wait(&wempty[b], ((uint32_t)(wc / WS) & 1u) ^ 1u);
                        mbar_expect_tx(&wfull[b], S::W_BYTES);
                        tma_load_3d(wring + (size_t)b * S::W_BYTES, &tmW, &wfull[b], step * 64, n0, 0);
                        bulk_load(wring + (size_t)b * S::W_BYTES + S::V_BYTES, meta + (size_t)step * SP_META_STEP, SP_META_STEP, &wfull[b]);
                    }
                }
        }
        return;
    }
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(TC_CONSUMER_REGS));

    // ===== consumers: warpgroup wg owns output channels [64 wg, 64 wg + 64) of the tile =====
    const int wg = (warp >> 2) - 1, t = threadIdx.x - 128;
    int acc[NACC];
#pragma unroll
    for (int j = 0; j < NACC; j++) acc[j] = 0;
    // one wgmma group in flight, as in conv_wg_kernel: step s is issued before step s - 1 is waited for and its slots released
    int xc = 0, q = 0, prev_b = 0, prev_x = -1;
    for (int it = 0; it < num_k; it++) {
        const int x = xc % XS, b = it % WS;
        if (q == 0) mbar_wait(&xfull[x], (uint32_t)(xc / XS) & 1u);
        mbar_wait(&wfull[b], (uint32_t)(it / WS) & 1u);
        const uint8_t* ws = wring + (size_t)b * S::W_BYTES;
        const uint32_t e0 = ((const uint32_t*)(ws + S::V_BYTES))[t], e1 = ((const uint32_t*)(ws + S::V_BYTES))[256 + t];
        const uint32_t sa = smem_u32(ws) + (uint32_t)(wg * 64 * 64);
        const uint32_t sb = smem_u32(xring + (size_t)x * S::X_BYTES) + (uint32_t)(q * 128);
        wg_fence();
        WgmmaSp<N>::mma(acc, sp_desc(sa), wg_desc(sb), e0, it != 0);
        WgmmaSp<N>::mma(acc, sp_desc(sa + 32), wg_desc(sb + 64), e1, 1u);
        wg_commit();
        wg_wait_1();
        if (it > 0) {
            __syncwarp();
            if (lane == 0) { mbar_arrive(&wempty[prev_b]); if (prev_x >= 0) mbar_arrive(&xempty[prev_x]); }
        }
        prev_b = b;
        prev_x = q == ks - 1 ? x : -1;
        if (++q == ks) { q = 0; xc++; }
    }
    wg_wait_all();
    __syncwarp();
    if (lane == 0) { mbar_arrive(&wempty[prev_b]); if (prev_x >= 0) mbar_arrive(&xempty[prev_x]); }

    // ===== epilogue: register j of a thread holds channel 16 (warp % 4) + lane / 4 + 8 ((j / 2) % 2) of the warpgroup's 64 and
    // pixel 8 (j / 4) + 2 (lane % 4) + j % 2 of the tile =====
    const int per_img = a.Hs * a.Wp, cout8 = (a.cout + 7) & ~7;
    uint8_t* const st = stage + (size_t)wg * N * 64;
    float range_max = 0.f;
#pragma unroll
    for (int cp = 0; cp < N / 8; cp++)
#pragma unroll
        for (int e = 0; e < 2; e++) {
            const int col = cp * 8 + (lane & 3) * 2 + e;
            const long long m = m0 + col;
            const int n = (int)(m / per_img), rem = (int)(m % per_img);
            const int y = rem / a.Wp, x = rem % a.Wp;
            const bool valid = m < a.M && n == img && x < a.W && y < a.H;
#pragma unroll
            for (int hr = 0; hr < 2; hr++) {
                const int cl = (warp & 3) * 16 + (lane >> 2) + hr * 8, c = wg * 64 + cl, co = n0 + c;
                float v = __fadd_rn(__fmul_rn(__int2float_rn(acc[cp * 4 + hr * 2 + e]), s_epi[SP_BM + c]), s_epi[c]);
                if (a.relu) v = fmaxf(v, 0.f);
                if (valid && co < a.cout) {
                    range_max = fmaxf(range_max, fabsf(v));
                    if (a.planar) a.planar[(((size_t)n * a.planar_C + a.planar_coff + co) * a.H + y) * a.W + x] = v;
                }
                if (!a.planar) st[col * 64 + cl] = (uint8_t)f32_to_s8(v);
            }
        }
    if (!a.planar) {
        asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");   // the warpgroup's staging is complete
        for (int i = t & 127; i < N * 4; i += 128) {
            const int col = i >> 2, c0 = n0 + wg * 64 + (i & 3) * 16;
            const long long m = m0 + col;
            const int n = (int)(m / per_img), rem = (int)(m % per_img);
            const int y = rem / a.Wp, x = rem % a.Wp;
            if (m >= a.M || n != img || x >= a.W || y >= a.H || c0 >= cout8) continue;
            int8_t* dst = a.out + (size_t)m * a.out_pitch + a.out_coff + c0;
            const uint8_t* src = st + col * 64 + (i & 3) * 16;
            if (c0 + 16 <= cout8) *(uint4*)dst = *(const uint4*)src;
            else *(uint2*)dst = *(const uint2*)src;   // the last 8 channels of cout8
        }
    }
    range_publish(a.range, range_max);
}

template <int N>
static int sp_launch(const TcLayer& l, const SpArgs& a, dim3 grid, cudaStream_t st, int xmap) {
    auto kern = conv_wg_kernel_sparse<N>;
    constexpr int smem = SpShape<N>::SMEM;
    int dev = 0;
    cudaGetDevice(&dev);
    static std::atomic<unsigned long long> attr_done{0};   // bit d: attribute set on device d
    if (!(attr_done.load(std::memory_order_acquire) >> (dev & 63) & 1ull)) {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return -1;
        attr_done.fetch_or(1ull << (dev & 63), std::memory_order_release);
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = dim3(TC_THREADS, 1, 1); cfg.dynamicSmemBytes = (size_t)smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    const CUtensorMap* maps = (const CUtensorMap*)l.maps;
    return cudaLaunchKernelEx(&cfg, kern, maps[xmap], maps[1], a) == cudaSuccess ? 1 : -1;
}

int tc_sparse_launch(const TcLayer& l, int nimg, cudaStream_t st, int share) {
    const TcLayerDesc& d = l.d;
    const long long K = (long long)d.ksize * d.ksize * d.in_cused;
    SpArgs a;
    a.bias = d.bias; a.meta = (const uint8_t*)d.w + (size_t)d.cout_pad * K / 2;
    a.out = (int8_t*)d.out; a.out_pitch = d.out_pitch; a.out_coff = d.out_coff;
    a.planar = d.planar; a.planar_C = d.planar_C; a.planar_coff = d.planar_coff;
    a.cout = d.cout; a.relu = d.relu; a.range = d.range;
    a.ksize = d.ksize; a.pad = d.pad; a.kblocks_per_tap = d.in_cused / 128;
    a.W = d.geo.W; a.H = d.geo.H; a.Wp = d.geo.Wp; a.Hs = d.geo.Hs;
    a.M = (long long)nimg * d.geo.Hs * d.geo.Wp;
    static int nsm = 0;
    if (!nsm) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev); }
    // Pixel tile width: 128, or 64 when that fills more SMs, by tc_layer_launch's rule for its channel tile width
    const long long mt = (a.M + 127) / 128, cb = d.cout_pad / SP_BM;
    const long long sms = std::max(1, nsm / (share < 1 ? 1 : share));
    const bool half = (double)std::min<long long>(2 * mt * cb, sms) * 0.80 > (double)std::min<long long>(mt * cb, sms) * 1.00;
    const int n = half ? 64 : 128;
    a.tiles_img = ((d.geo.H - 1) * d.geo.Wp + d.geo.W + n - 1) / n;
    const dim3 grid((unsigned)(nimg * a.tiles_img), (unsigned)cb, 1);
    return half ? sp_launch<64>(l, a, grid, st, 2) : sp_launch<128>(l, a, grid, st, 0);
}

}  // namespace pe
