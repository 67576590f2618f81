// Post-processing on the GPU: multi-scale ImResize/average fused with the NMS peak finder, PAF line
// integral, greedy bipartite limb assignment and person assembly.
//
// What it replaces (SURVEY.md section 8a rows a3-a5):
//   ImResizeLayer::Forward_gpu + imresize_cubic_kernel   src/caffe/cpm/layers/imresize_layer.cu:98-193
//   NmsLayer::Forward_gpu (register/scan/write)          src/caffe/cpm/layers/nms_layer.cu:14-184
//   connectLimbs / connectLimbsCOCO (host C++)           examples/rtpose/rtpose.cpp:549-751, 808-1076
//
// GPU-first design: the reference materialises a 55 MB full-resolution tensor (57x368x656 fp32), copies
// it to the host and walks it on one CPU thread.  Here the full-resolution value of any (channel,y,x) is a
// pure function of the 0.86 MB stride-8 maps (L2 resident), so it is evaluated ON THE FLY wherever the
// algorithm looks at it: the NMS tiles, the 7x7 centroid windows and the 10 PAF samples per candidate
// pair.  Nothing full-resolution is ever written; the only outputs are the 14 KB peaks blob and the joints.
//
// Arithmetic: every float/double operation below is written with explicit round-to-nearest intrinsics in
// the order (and with the FMA contractions) that nvcc emits for the reference kernels, and that the host
// compiler emits for connectLimbs*, so results are bit-identical to the oracle (tests/test_gpu_post.py).
#include "common.h"
#include "kernels.h"
#include "fullres.cuh"

namespace pe {

// s_pos[128] (nms_write_kernel), the 128-bit occupancy masks (limb_greedy_kernel), s_new[128] and s_conn_of_slot[130]
// (assemble_kernel: slots 0..max_peaks) hold every peak of one part
static_assert(PE_MAX_PEAKS <= 127, "post.cu's per-part shared tables hold at most 127 peaks");

// Per-scale, per-output-coordinate source taps of imresize_cubic_kernel (imresize_layer.cu:110-140).
// Built once per (net size, scales) by axis_table_kernel with the kernel's own arithmetic.
__global__ void axis_table_kernel(AxisTap* tab, int t, int ori, int num_scales, float start_scale, float scale_gap) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = blockIdx.y;
    if (x >= t || n >= num_scales) return;
    const float f = __fmaf_rn((float)n, scale_gap, __fsub_rn(1.0f, start_scale));
    const int pad = (int)floorf(__fmul_rn((float)(ori / 2), f));
    const int o = ori - 2 * pad;
    const float q = __fdiv_rn((float)t, (float)o);
    const float offset = __fmaf_rn(q, 0.5f, -0.5f);
    const float on_ori = __fmul_rn(__fsub_rn((float)x, offset), __fdiv_rn((float)o, (float)t));
    int n1 = __double2int_rz(__dadd_rn((double)on_ori, 1e-5));
    n1 = n1 < 0 ? 0 : n1;
    AxisTap a;
    a.i0 = ((n1 - 1 < 0) ? n1 : (n1 - 1)) + pad;
    const int n2 = (n1 + 1 >= o) ? (o - 1) : (n1 + 1);
    a.i3 = ((n2 + 1 >= o) ? (o - 1) : (n2 + 1)) + pad;
    a.d = __fsub_rn(on_ori, (float)n1);
    a.i1 = n1 + pad;
    a.i2 = n2 + pad;
    tab[(size_t)n * t + x] = a;
}

// ------------------------------------------------------------------------------------------------
// Kernel 1: resize + nms_register_kernel (nms_layer.cu:14-46) fused.
// One CTA pass = one 32 x NMS_TY full-resolution tile of one (frame, part); values incl. the 1-pixel halo are
// produced in shared memory, the strict 8-neighbour test runs from there, and each warp row becomes
// one 32-bit word of the peak bitmask (warp ballot) - raster order is preserved by construction.
// ------------------------------------------------------------------------------------------------
#define NMS_TX 32
#define NMS_TY 46        // rows per tile pass (368 = 8 x 46, 736 = 16 x 46)
#define NMS_HROWS 12     // source rows a 48-row window can touch at stride 8 (48 / 8 + 4 taps, rounded up), else the non-separable path runs
#define NMS_THREADS 128  // 128 threads, <= 88 registers, < 10 KB shared memory: a CTA fits next to a resident conv CTA of another handle
constexpr int NMS_COLS = NMS_TX + 2;                              // tile columns incl. the halo
constexpr int NMS_ROWS = NMS_TY + 2;
constexpr int NMS_NSEG = NMS_THREADS / NMS_COLS;                  // column threads per tile column (3)
constexpr int NMS_SEG = (NMS_ROWS + NMS_NSEG - 1) / NMS_NSEG;     // consecutive rows one thread walks down (17)
constexpr int NMS_XCH = 4;                                        // consecutive columns one thread of the horizontal pass produces
constexpr int NMS_NXCH = (NMS_COLS + NMS_XCH - 1) / NMS_XCH;
// ncu r2p: the previous version (one vertical cubic_ref per thread and pixel, flat-index divisions, five tap loads) issued 161 warp
// instructions per cubic at 80 % issue utilisation for ~30 of arithmetic.  Here a thread walks DOWN one tile column: the four taps
// of a vertical cubic change every 8 rows at stride 8, so cubic_prep runs once per source interval and cubic_eval (3 conversions,
// 4 fp64 + 4 fp32 operations) per pixel, row fractions come from a per-tile table, sums over the scales stay in registers.
__global__ void __launch_bounds__(NMS_THREADS) nms_flags_kernel(PostDev pd) {
    __shared__ float tile[NMS_ROWS][NMS_COLS];
    __shared__ float hrow[NMS_HROWS][NMS_COLS];
    __shared__ double s_ydd[NMS_ROWS];
    __shared__ float s_yd[NMS_ROWS];
    __shared__ uint32_t s_yi[NMS_ROWS];      // the four source rows of a tile row relative to the window's first, one byte each
    const int part = blockIdx.z % pd.p.num_parts, frame = blockIdx.z / pd.p.num_parts;
    const FullRes fr = make_fullres(pd, frame);
    const int W = pd.p.net_w, H = pd.p.net_h;
    const int x0 = blockIdx.x * NMS_TX - 1;
    const int tiles_y = (H + NMS_TY - 1) / NMS_TY;
    const int ctx = threadIdx.x % NMS_COLS, cseg = threadIdx.x / NMS_COLS;       // vertical pass: my column and row segment
    const bool cactive = cseg < NMS_NSEG && x0 + ctx >= 0 && x0 + ctx < W;
    // A CTA walks several row tiles (blockIdx.y, + gridDim.y, ...)
    for (int tile_y = blockIdx.y; tile_y < tiles_y; tile_y += gridDim.y) {
    const int y0 = tile_y * NMS_TY - 1;
    const int ylo = max(y0, 0), yhi = min(y0 + NMS_TY + 1, H - 1);
    // Separable evaluation: the horizontal cubic of a (source row, x) pair does not depend on the output row,
    // so it is computed once per tile (<= NMS_HROWS source rows) instead of 4x per output pixel.  Same
    // operations on the same operands as fullres_at -> bit-identical values.
    bool separable = true;
    for (int n = 0; n < fr.copies; n++) {
        const int rlo = copy_ytab(fr, n)[ylo].i0, rhi = copy_ytab(fr, n)[yhi].i3;
        if (rhi - rlo + 1 > NMS_HROWS) separable = false;
    }
    if (separable) {
        float acc[NMS_SEG];
#pragma unroll
        for (int j = 0; j < NMS_SEG; j++) acc[j] = 0.f;
        for (int n = 0; n < fr.copies; n++) {
            const AxisTap* yt = copy_ytab(fr, n);
            const int rlo = yt[ylo].i0, rhi = yt[yhi].i3;
            const int nrows = rhi - rlo + 1;
            float sign;
            const float* s = copy_plane(fr, n, part, &sign);
            __syncthreads();                                   // the previous scale's tables and rows have been consumed
            for (int i = threadIdx.x; i < NMS_ROWS; i += NMS_THREADS) {
                const int y = y0 + i;
                uint32_t pk = 0xffffffffu;                     // row outside the image
                if (y >= 0 && y < H) {
                    const AxisTap ay = yt[y];
                    pk = (uint32_t)(ay.i0 - rlo) | (uint32_t)(ay.i1 - rlo) << 8 | (uint32_t)(ay.i2 - rlo) << 16 | (uint32_t)(ay.i3 - rlo) << 24;
                    s_yd[i] = ay.d;
                    s_ydd[i] = (double)ay.d;
                }
                s_yi[i] = pk;
            }
            // horizontal pass: one thread per (source row, run of NMS_XCH columns); the taps change every 8 columns
            for (int it = threadIdx.x; it < nrows * NMS_NXCH; it += NMS_THREADS) {
                const int r = it / NMS_NXCH, c0 = (it % NMS_NXCH) * NMS_XCH;
                const float* row = s + (size_t)(rlo + r) * fr.w8;
                int p0 = -1, p1 = -1, p2 = -1, p3 = -1;
                CubicTaps ct = {0.f, 0.f, 0.0, 0.0};
#pragma unroll
                for (int k = 0; k < NMS_XCH; k++) {
                    const int tx = c0 + k, x = x0 + tx;
                    if (tx < NMS_COLS) {
                        float v = 0.f;
                        if (x >= 0 && x < W) {
                            const AxisTap ax = copy_xtap(fr, n, x);
                            if (ax.i0 != p0 || ax.i1 != p1 || ax.i2 != p2 || ax.i3 != p3) {
                                p0 = ax.i0; p1 = ax.i1; p2 = ax.i2; p3 = ax.i3;
                                ct = cubic_prep(__ldg(row + p0), __ldg(row + p1), __ldg(row + p2), __ldg(row + p3));
                            }
                            v = cubic_eval(ct, ax.d, (double)ax.d);
                        }
                        hrow[r][tx] = v;
                    }
                }
            }
            __syncthreads();
            // vertical pass: down my column, taps re-prepared when the source interval changes
            if (cactive) {
                uint32_t cur = 0xfffffffeu;
                CubicTaps ct = {0.f, 0.f, 0.0, 0.0};
#pragma unroll
                for (int j = 0; j < NMS_SEG; j++) {
                    const int ty = cseg * NMS_SEG + j;
                    if (ty < NMS_ROWS) {
                        const uint32_t pk = s_yi[ty];
                        if (pk != 0xffffffffu) {
                            if (pk != cur) {
                                cur = pk;
                                ct = cubic_prep(hrow[pk & 255u][ctx], hrow[(pk >> 8) & 255u][ctx], hrow[(pk >> 16) & 255u][ctx], hrow[pk >> 24][ctx]);
                            }
                            acc[j] = __fadd_rn(acc[j], __fmul_rn(sign, cubic_eval(ct, s_yd[ty], s_ydd[ty])));
                        }
                    }
                }
            }
        }
        if (cseg < NMS_NSEG) {
#pragma unroll
            for (int j = 0; j < NMS_SEG; j++) {
                const int ty = cseg * NMS_SEG + j;
                if (ty < NMS_ROWS) tile[ty][ctx] = fr.copies == 1 ? acc[j] : __fdiv_rn(acc[j], fr.inv_div);   // x / 1.0f == x; outside the image: 0
            }
        }
    } else {
        constexpr int NOUT = NMS_ROWS * NMS_COLS;
        for (int i = threadIdx.x; i < NOUT; i += NMS_THREADS) {
            const int ty = i / NMS_COLS, tx = i % NMS_COLS;
            const int x = x0 + tx, y = y0 + ty;
            float v = 0.f;
            if (x >= 0 && x < W && y >= 0 && y < H) v = fullres_at(fr, part, y, x);
            tile[ty][tx] = v;
        }
    }
    __syncthreads();
    // strict 8-neighbour test: a warp walks down its rows with the 3 x 3 window sliding through registers (3 shared-memory loads
    // per pixel instead of 9), lane = column, one ballot = one 32-bit word of the bitmask
    {
        constexpr int NW = NMS_THREADS / 32, RPW = (NMS_TY + NW - 1) / NW;
        const int lx = threadIdx.x & 31, r0 = (threadIdx.x >> 5) * RPW, r1 = min(r0 + RPW, NMS_TY);
        const int x = blockIdx.x * NMS_TX + lx;
        const bool x_in = x > 0 && x < W - 1;
        const int words_per_row = (W + 31) / 32;
        unsigned* frow = pd.flags + ((size_t)(frame * pd.p.num_parts + part) * H) * words_per_row + blockIdx.x;
        const float thr = pd.p.nms_threshold;
        float a0 = tile[r0][lx], a1 = tile[r0][lx + 1], a2 = tile[r0][lx + 2];
        float b0 = tile[r0 + 1][lx], b1 = tile[r0 + 1][lx + 1], b2 = tile[r0 + 1][lx + 2];
        for (int ly = r0; ly < r1; ly++) {
            const float c0 = tile[ly + 2][lx], c1 = tile[ly + 2][lx + 1], c2 = tile[ly + 2][lx + 2];
            const int y = tile_y * NMS_TY + ly;
            const bool peak = x_in && y > 0 && y < H - 1 && b1 > thr && b1 > a1 && b1 > c1 && b1 > b0 && b1 > b2 && b1 > a0 && b1 > c0 &&
                              b1 > c2 && b1 > a2;
            const unsigned word = __ballot_sync(0xffffffffu, peak);
            if (lx == 0 && y < H) frow[(size_t)y * words_per_row] = word;
            a0 = b0; a1 = b1; a2 = b2; b0 = c0; b1 = c1; b2 = c2;
        }
    }
    __syncthreads();   // tile[] is rewritten by the next row tile
    }
}

// ------------------------------------------------------------------------------------------------
// Kernel 2: thrust::exclusive_scan + writeResultKernel (nms_layer.cu:176, 49-113) fused.
// One CTA per (frame, part): block-wide popcount scan of the bitmask words gives every peak its raster
// rank; the first max_peaks get the 7x7 score-weighted centroid (window values re-evaluated on the fly,
// including the reference's width-for-height bound that aliases into the next channel's first rows).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256, 6) nms_write_kernel(PostDev pd) {
    __shared__ int s_scan[256];
    __shared__ int s_pos[128];       // flat y*W+x of the first max_peaks peaks
    __shared__ float s_win[4][49];
    __shared__ float s_own[4];
    __shared__ int s_total;
    const int part = blockIdx.x, frame = blockIdx.y;
    const int W = pd.p.net_w, H = pd.p.net_h, MP = pd.p.max_peaks;
    const int words_per_row = (W + 31) / 32;
    const int nwords = H * words_per_row;
    const unsigned* flags = pd.flags + (size_t)(frame * pd.p.num_parts + part) * nwords;
    const int per = (nwords + 255) / 256;
    const int w0 = threadIdx.x * per, w1 = min(w0 + per, nwords);
    int cnt = 0;
    for (int w = w0; w < w1; w++) cnt += __popc(flags[w]);
    s_scan[threadIdx.x] = cnt;
    __syncthreads();
    // Hillis-Steele inclusive scan over 256 counts
    for (int off = 1; off < 256; off <<= 1) {
        int v = 0;
        if ((int)threadIdx.x >= off) v = s_scan[threadIdx.x - off];
        __syncthreads();
        s_scan[threadIdx.x] += v;
        __syncthreads();
    }
    int rank = s_scan[threadIdx.x] - cnt;  // exclusive
    if (threadIdx.x == 255) s_total = s_scan[255];
    for (int w = w0; w < w1 && rank < MP; w++) {
        unsigned bits = flags[w];
        const int y = w / words_per_row, xb = (w % words_per_row) * 32;
        while (bits && rank < MP) {
            const int b = __ffs(bits) - 1;
            bits &= bits - 1;
            s_pos[rank++] = y * W + xb + b;
        }
    }
    __syncthreads();
    const int total = s_total;
    const int n = min(total, MP);
    float* out = pd.peaks + (size_t)(frame * pd.p.num_parts + part) * (MP + 1) * 3;
    if (threadIdx.x == 0) out[0] = (float)total;  // total, not clamped (nms_layer.cu:110)
    const FullRes fr = make_fullres(pd, frame);
    const int g = threadIdx.x >> 6, l = threadIdx.x & 63;
    for (int base = 0; base < n; base += 4) {
        const int k = base + g;
        if (k < n && l < 49) {
            const int px = s_pos[k] % W, py = s_pos[k] / W;
            const int dy = l / 7 - 3, dx = l % 7 - 3;
            const int yy = py + dy, xx = px + dx;
            const bool in_win = yy > 0 && yy < W && xx > 0 && xx < W;      // sic: W for both (nms_layer.cu:79,81)
            // l == 24 also evaluates the peak's own value (nms_layer.cu:99) when a portrait net's row >= W puts it outside the window
            float v = 0.f;
            if (in_win || l == 24) {
                // rows >= H alias the following channel's first rows: src_pointer[(y+dy)*width + x+dx]
                const int cc = part + yy / H, ry = yy % H;
                v = (cc < pd.p.num_maps) ? fullres_at(fr, cc, ry, xx) : 0.f;
            }
            s_win[g][l] = in_win ? v : 0.f;
            if (l == 24) s_own[g] = v;
        }
        __syncthreads();
        if (k < n && l == 0) {
            const int px = s_pos[k] % W, py = s_pos[k] / W;
            float x_acc = 0.f, y_acc = 0.f, score_acc = 0.f;
            for (int dy = -3; dy < 4; dy++) {
                if ((py + dy) > 0 && (py + dy) < W) {
                    for (int dx = -3; dx < 4; dx++) {
                        if ((px + dx) > 0 && (px + dx) < W) {
                            const float score = s_win[g][(dy + 3) * 7 + dx + 3];
                            if (score > 0) {
                                x_acc = __fmaf_rn((float)(px + dx), score, x_acc);
                                y_acc = __fmaf_rn((float)(py + dy), score, y_acc);
                                score_acc = __fadd_rn(score_acc, score);
                            }
                        }
                    }
                }
            }
            float* o = out + (k + 1) * 3;
            o[0] = __fdiv_rn(x_acc, score_acc);
            o[1] = __fdiv_rn(y_acc, score_acc);
            o[2] = s_own[g];
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------
// Kernel 3: PAF line integral (rtpose.cpp:900-949 / 611-647).  One thread per candidate pair (i,j);
// grid = (pair chunks, limb, frame).  Candidates that pass go to a per-limb list keyed by their
// position p = (i-1)*nB + (j-1) in the reference's nested loop (used as the tie-break of the sort).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) paf_score_kernel(PostDev pd) {
    const int limb = blockIdx.y, frame = blockIdx.z;
    const ModelDev& md = pd.md;
    const int MP = pd.p.max_peaks, poff = 3 * (MP + 1);
    const int pa = md.limb_seq[2 * limb], pb = md.limb_seq[2 * limb + 1];
    const float* peaks = pd.peaks + (size_t)frame * pd.p.num_parts * poff;
    const float* candA = peaks + pa * poff;
    const float* candB = peaks + pb * poff;
    const int nA = min((int)candA[0], MP), nB = min((int)candB[0], MP);
    const int npairs = nA * nB;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= npairs) return;
    const int i = p / nB + 1, j = p % nB + 1;
    const bool coco = pd.p.model != PE_MODEL_MPI_15;
    const float s_x = candA[i * 3], s_y = candA[i * 3 + 1];
    const float d_x = __fsub_rn(candB[j * 3], candA[i * 3]);
    const float d_y = __fsub_rn(candB[j * 3 + 1], candA[i * 3 + 1]);
    float norm_vec;
    if (coco) {
        norm_vec = __fsqrt_rn(__fadd_rn(__fmul_rn(d_x, d_x), __fmul_rn(d_y, d_y)));
    } else {  // pow(d_x,2) + pow(d_y,2) in double (rtpose.cpp:618)
        const double dx2 = __dmul_rn((double)d_x, (double)d_x), dy2 = __dmul_rn((double)d_y, (double)d_y);
        norm_vec = __double2float_rn(__dsqrt_rn(__dadd_rn(dx2, dy2)));
    }
    // !(>=) also rejects NaN endpoints: a portrait net's peaks below row W + 2 have an empty window, x = y = 0/0.  The reference
    // goes on to index the map with (int)roundf(NaN); the oracle rejects them as here (OrcConnectParams.clamp_counts)
    if (!((double)norm_vec >= 1e-6)) return;
    const float vec_x = __fdiv_rn(d_x, norm_vec), vec_y = __fdiv_rn(d_y, norm_vec);
    const FullRes fr = make_fullres(pd, frame);
    const int W = pd.p.net_w, H = pd.p.net_h;
    const int cx = md.map_idx[2 * limb], cy = md.map_idx[2 * limb + 1];
    float sum = 0.f;
    int count = 0;
    for (int lm = 0; lm < 10; lm++) {
        int my = (int)roundf(__fadd_rn(s_y, __fdiv_rn(__fmul_rn((float)lm, d_y), 10.0f)));
        int mx = (int)roundf(__fadd_rn(s_x, __fdiv_rn(__fmul_rn((float)lm, d_x), 10.0f)));
        // COCO clamps the upper bounds (rtpose.cpp:920-927); MPI does not (:629-633) and would read
        // past the channel - the engine clamps both (identical whenever the reference is in bounds).
        mx = min(max(mx, 0), W - 1);
        my = min(max(my, 0), H - 1);
        const float score = __fadd_rn(__fmul_rn(vec_x, fullres_at(fr, cx, my, mx)), __fmul_rn(vec_y, fullres_at(fr, cy, my, mx)));
        if (score > pd.p.inter_threshold) { sum = __fadd_rn(sum, score); count++; }
    }
    if (count > pd.p.inter_min_above) {
        const int lf = frame * pd.p.num_limbs + limb;
        const int slot = atomicAdd(&pd.cand_count[lf], 1);
        Cand c;
        c.conn = __fdiv_rn(sum, (float)count);
        c.p = p;
        pd.cands[(size_t)lf * MP * MP + slot] = c;
    }
}

// ------------------------------------------------------------------------------------------------
// Kernel 4: sort candidates by connection score (descending; ColumnCompare rtpose.cpp:144-152, ties
// broken by loop position - std::sort leaves them unspecified) + greedy one-to-one selection
// (rtpose.cpp:953-980).  One CTA per (limb, frame); bitonic sort on 64-bit keys in shared memory.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned order_key(float f) {  // monotone float -> uint
    const unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__global__ void __launch_bounds__(512) limb_greedy_kernel(PostDev pd) {
    extern __shared__ unsigned long long s_keys[];   // next_pow2(max_peaks^2) keys: 32 KB for COCO, 4 KB for MPI
    const int limb = blockIdx.x, frame = blockIdx.y;
    const int MP = pd.p.max_peaks, poff = 3 * (MP + 1);
    const int lf = frame * pd.p.num_limbs + limb;
    const int ncand = pd.cand_count[lf];
    const Cand* cands = pd.cands + (size_t)lf * MP * MP;
    int n2 = 1;
    while (n2 < ncand) n2 <<= 1;
    for (int i = threadIdx.x; i < n2; i += blockDim.x) {
        unsigned long long k = ~0ull;
        if (i < ncand) k = ((unsigned long long)(~order_key(cands[i].conn)) << 32) | (unsigned)cands[i].p;
        s_keys[i] = k;
    }
    __syncthreads();
    for (int k = 2; k <= n2; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < n2; i += blockDim.x) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long a = s_keys[i], b = s_keys[ixj];
                    const bool up = (i & k) == 0;
                    if ((a > b) == up) { s_keys[i] = b; s_keys[ixj] = a; }
                }
            }
            __syncthreads();
        }
    const ModelDev& md = pd.md;
    const int pa = md.limb_seq[2 * limb], pb = md.limb_seq[2 * limb + 1];
    const float* peaks = pd.peaks + (size_t)frame * pd.p.num_parts * poff;
    const int nA = min((int)peaks[pa * poff], MP), nB = min((int)peaks[pb * poff], MP);
    // decode the loop position p -> (i, j) for every candidate in parallel, so the inherently sequential greedy scan below
    // (up to max_peaks^2 candidates on noise maps) is a handful of instructions per candidate instead of a div/mod chain
    for (int r = threadIdx.x; r < ncand; r += blockDim.x) {
        const unsigned long long key = s_keys[r];
        const unsigned p = (unsigned)(key & 0xffffffffu);
        s_keys[r] = (key & 0xffffffff00000000ull) | ((unsigned long long)(p / nB + 1) << 16) | (unsigned long long)(p % nB + 1);
    }
    __syncthreads();
    // Greedy one-to-one selection in sorted order (rtpose.cpp:953-980) by ONE WARP, 32 candidates per step: within a
    // group the first candidate whose A and B are both still free is exactly the one the sequential scan would take
    // next; accept it, update the occupancy masks, re-test the later lanes, repeat.  Same picks in the same order, but
    // ~ncand/32 + #picks dependent steps instead of ncand.
    if (threadIdx.x < 32) {
        const int lane = threadIdx.x;
        const int num = min(nA, nB);
        Conn* out = pd.conns + (size_t)lf * MP;
        unsigned long long ua0 = 0, ua1 = 0, ub0 = 0, ub1 = 0;   // occupancy bitmasks (max_peaks <= 128)
        int cnt = 0;
        for (int base = 0; base < ncand && cnt < num; base += 32) {
            const int row = base + lane;
            bool valid = row < ncand;
            const unsigned long long key = valid ? s_keys[row] : 0ull;
            const int i = (int)((key >> 16) & 0xffffu) - 1, j = (int)(key & 0xffffu) - 1;
            while (cnt < num) {
                const bool a_used = valid && (((i < 64 ? ua0 : ua1) >> (i & 63)) & 1ull);
                const bool b_used = valid && (((j < 64 ? ub0 : ub1) >> (j & 63)) & 1ull);
                const unsigned m = __ballot_sync(0xffffffffu, valid && !a_used && !b_used);
                if (!m) break;
                const int f = __ffs(m) - 1;
                const int fi = __shfl_sync(0xffffffffu, i, f), fj = __shfl_sync(0xffffffffu, j, f);
                const unsigned fhi = __shfl_sync(0xffffffffu, (unsigned)(key >> 32), f);
                if (fi < 64) ua0 |= 1ull << fi; else ua1 |= 1ull << (fi - 64);
                if (fj < 64) ub0 |= 1ull << fj; else ub1 |= 1ull << (fj - 64);
                if (lane == 0) {
                    const unsigned ok = ~fhi;
                    const unsigned u = (ok & 0x80000000u) ? (ok & 0x7fffffffu) : ~ok;
                    Conn c;
                    c.a = pa * poff + (fi + 1) * 3 + 2;
                    c.b = pb * poff + (fj + 1) * 3 + 2;
                    c.score = __uint_as_float(u);
                    out[cnt] = c;
                }
                cnt++;
                if (lane == f) valid = false;
            }
        }
        if (lane == 0) pd.conn_count[lf] = cnt;
    }
}

// ------------------------------------------------------------------------------------------------
// Kernel 5: person assembly + joint output (rtpose.cpp:847-895, 984-1073).  Inherently sequential over
// limbs and connections; the scan over existing rows is parallel.  One CTA per frame.  Row layout as in
// the reference: num_parts index slots (flat index of the peak's score in the peaks blob, 0 = empty),
// then [num_parts+1] = score (double), [num_parts+2] = count.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256, 6) assemble_kernel(PostDev pd) {
    __shared__ int s_rows;
    __shared__ int s_conn_of_slot[130];   // peak slot of part A (1..max_peaks) -> connection index of this limb
    __shared__ int s_found[130];
    const int frame = blockIdx.x;
    const ModelDev& md = pd.md;
    const int P = pd.p.num_parts, MP = pd.p.max_peaks, poff = 3 * (MP + 1);
    const int S_CNT = P + 2, S_SCORE = P + 1, S_SIZE = P + 3;
    const bool coco = pd.p.model != PE_MODEL_MPI_15;
    const float* peaks = pd.peaks + (size_t)frame * P * poff;
    const int max_rows = pd.p.max_subset_rows;
    double* subset = pd.subset + (size_t)frame * max_rows * S_SIZE;
    if (threadIdx.x == 0) s_rows = 0;
    __syncthreads();

    // New rows of one limb are first described in shared memory by thread 0 (cheap, in reference order) and then
    // written to the subset table by the whole CTA (21 doubles per row).
    struct NewRow { int slot_a, slot_b; double va, vb, cnt, score; };
    __shared__ NewRow s_new[128];
    __shared__ int s_nnew;
    if (threadIdx.x == 0) s_nnew = 0;
    auto append = [&](int slot_a, double va, int slot_b, double vb, double cnt, double score) {
        // called by thread 0 only
        const int r = s_nnew;
        if (r < 128) { s_new[r] = NewRow{slot_a, slot_b, va, vb, cnt, score}; s_nnew = r + 1; }
    };
    auto flush = [&]() {   // called by all threads
        __syncthreads();
        const int n = s_nnew, base = s_rows;
        for (int t = threadIdx.x; t < n * S_SIZE; t += blockDim.x) {
            const int r = t / S_SIZE, q = t % S_SIZE;
            const NewRow nr = s_new[r];
            double v = 0.0;
            if (q == nr.slot_a) v = nr.va;
            else if (q == nr.slot_b) v = nr.vb;
            else if (q == S_CNT) v = nr.cnt;
            else if (q == S_SCORE) v = nr.score;
            if (base + r < max_rows) subset[(size_t)(base + r) * S_SIZE + q] = v;
        }
        __syncthreads();
        if (threadIdx.x == 0) { s_rows = min(base + n, max_rows); s_nnew = 0; }
        __syncthreads();
    };
    // The reference walks connections (and, in the nA==0/nB==0 branches, peaks) one at a time over all rows.
    // Within one limb every connection has a distinct part-A peak and rows created during the limb carry that
    // limb's own A peaks, so the per-connection row scans are independent: one parallel pass over the rows
    // (row -> its connection through s_conn_of_slot) followed by the in-order appends gives the same rows in the
    // same order.
    for (int k = 0; k < pd.p.num_limbs; k++) {
        const int pa = md.limb_seq[2 * k], pb = md.limb_seq[2 * k + 1];
        const int nA = min((int)peaks[pa * poff], MP), nB = min((int)peaks[pb * poff], MP);
        if (nA == 0 && nB == 0) continue;
        const int rows = s_rows;
        if (nA == 0 || nB == 0) {
            const int part = nA == 0 ? pb : pa, n = nA == 0 ? nB : nA;
            for (int i = threadIdx.x; i <= n; i += blockDim.x) s_found[i] = 0;
            __syncthreads();
            if (coco) {  // duplicate check exists only in connectLimbsCOCO (rtpose.cpp:852-860)
                for (int j = threadIdx.x; j < rows; j += blockDim.x) {
                    const double v = subset[(size_t)j * S_SIZE + part];
                    if (v != 0.0) {
                        const int slot = ((int)v - part * poff - 2) / 3;
                        if (slot >= 1 && slot <= n && (double)(part * poff + slot * 3 + 2) == v) s_found[slot] = 1;
                    }
                }
            }
            __syncthreads();
            if (threadIdx.x == 0)
                for (int i = 1; i <= n; i++)
                    if (!s_found[i]) {
                        const int off = part * poff + i * 3 + 2;
                        append(part, (double)off, -1, 0.0, 1.0, (double)peaks[off]);
                    }
            flush();
            continue;
        }
        const int lf = frame * pd.p.num_limbs + k;
        const int nc = pd.conn_count[lf];
        const Conn* conns = pd.conns + (size_t)lf * MP;
        if (k == 0) {
            if (threadIdx.x == 0)
                for (int i = 0; i < nc; i++) {
                    const Conn c = conns[i];
                    const double sc = __dadd_rn((double)__fadd_rn(peaks[c.a], peaks[c.b]), (double)c.score);
                    append(pa, (double)c.a, pb, (double)c.b, 2.0, sc);
                }
            flush();
            continue;
        }
        if (nc == 0) continue;
        for (int i = threadIdx.x; i <= MP; i += blockDim.x) { s_conn_of_slot[i] = -1; s_found[i] = 0; }
        __syncthreads();
        for (int i = threadIdx.x; i < nc; i += blockDim.x) s_conn_of_slot[(conns[i].a - pa * poff - 2) / 3] = i;
        __syncthreads();
        for (int j = threadIdx.x; j < rows; j += blockDim.x) {
            double* row = subset + (size_t)j * S_SIZE;
            const double v = row[pa];
            if (v != 0.0) {
                const int slot = ((int)v - pa * poff - 2) / 3;
                if (slot >= 1 && slot <= MP) {
                    const int ci = s_conn_of_slot[slot];
                    if (ci >= 0 && (double)conns[ci].a == v) {
                        const Conn c = conns[ci];
                        row[pb] = (double)c.b;
                        row[S_CNT] = row[S_CNT] + 1.0;
                        row[S_SCORE] = __dadd_rn(__dadd_rn(row[S_SCORE], (double)peaks[c.b]), (double)c.score);
                        s_found[ci] = 1;
                    }
                }
            }
        }
        __syncthreads();
        if (threadIdx.x == 0)
            for (int i = 0; i < nc; i++)
                if (!s_found[i]) {
                    const Conn c = conns[i];
                    const double sc = __dadd_rn((double)__fadd_rn(peaks[c.a], peaks[c.b]), (double)c.score);
                    append(pa, (double)c.a, pb, (double)c.b, 2.0, sc);
                }
        flush();
    }
    __syncthreads();
    // Output (rtpose.cpp:1051-1073): rows that pass the count / mean-score test, in creation order, at most 96.
    // Each thread owns a contiguous chunk of rows (order preserved), a block scan gives every kept row its slot.
    {
        __shared__ int s_scan[256];
        const int rows = s_rows;
        float* joints = pd.joints + (size_t)frame * PE_MAX_PEOPLE * P * 3;
        const int per = (rows + 255) / 256;
        const int r0 = threadIdx.x * per, r1 = min(r0 + per, rows);
        int kept = 0;
        for (int i = r0; i < r1; i++) {
            const double* row = subset + (size_t)i * S_SIZE;
            kept += (row[S_CNT] >= (double)pd.p.min_subset_cnt && __ddiv_rn(row[S_SCORE], row[S_CNT]) > (double)pd.p.min_subset_score) ? 1 : 0;
        }
        s_scan[threadIdx.x] = kept;
        __syncthreads();
        for (int off = 1; off < 256; off <<= 1) {
            int v = 0;
            if ((int)threadIdx.x >= off) v = s_scan[threadIdx.x - off];
            __syncthreads();
            s_scan[threadIdx.x] += v;
            __syncthreads();
        }
        int slot = s_scan[threadIdx.x] - kept;
        for (int i = r0; i < r1; i++) {
            const double* row = subset + (size_t)i * S_SIZE;
            if (!(row[S_CNT] >= (double)pd.p.min_subset_cnt && __ddiv_rn(row[S_SCORE], row[S_CNT]) > (double)pd.p.min_subset_score)) continue;
            if (slot < PE_MAX_PEOPLE) {
                for (int j = 0; j < P; j++) {
                    const int idx = (int)row[j];
                    float* o = joints + (size_t)slot * P * 3 + j * 3;
                    if (idx) {
                        o[2] = peaks[idx];
                        o[1] = __fdiv_rn(__fmul_rn(peaks[idx - 1], (float)pd.p.disp_h), (float)pd.p.net_h);
                        o[0] = __fdiv_rn(__fmul_rn(peaks[idx - 2], (float)pd.p.disp_w), (float)pd.p.net_w);
                    } else {
                        o[0] = o[1] = o[2] = 0.f;
                    }
                }
            }
            slot++;
        }
        if (threadIdx.x == 255) {
            pd.num_people[frame] = min(s_scan[255], PE_MAX_PEOPLE);
            pd.subset_rows[frame] = rows;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// host launchers
// ------------------------------------------------------------------------------------------------
void launch_axis_tables(AxisTap* xtab, AxisTap* ytab, const PostParams& p, cudaStream_t st) {
    axis_table_kernel<<<dim3((p.net_w + 127) / 128, p.num_scales), 128, 0, st>>>(xtab, p.net_w, p.w8, p.num_scales,
                                                                                   p.start_scale, p.scale_gap);
    axis_table_kernel<<<dim3((p.net_h + 127) / 128, p.num_scales), 128, 0, st>>>(ytab, p.net_h, p.h8, p.num_scales,
                                                                                   p.start_scale, p.scale_gap);
}

cudaError_t post_set_smem_limits() {
    // The sort keys of limb_greedy_kernel: next_pow2(max_peaks^2) x 8 bytes, 128 KB at max_peaks 91-127, above the 48 KB a launch
    // gets without opting in.  The attribute belongs to the kernel on this device, not to an engine, so every engine sets the
    // same ceiling, the one PE_MAX_PEAKS needs: an engine created later never lowers it under a live one.  Smaller launches
    // still get only what they ask for.
    int keys = 1;
    while (keys < PE_MAX_PEAKS * PE_MAX_PEAKS) keys <<= 1;
    return cudaFuncSetAttribute(limb_greedy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(unsigned long long) * keys));
}

int launch_post(const PostDev& pd, int nframes, cudaStream_t st) {
    const PostParams& p = pd.p;
    const int MP = p.max_peaks;
    cudaMemsetAsync(pd.peaks, 0, sizeof(float) * (size_t)nframes * p.num_parts * (MP + 1) * 3, st);
    cudaMemsetAsync(pd.cand_count, 0, sizeof(int) * (size_t)nframes * p.num_limbs, st);
    const int tiles_y = (p.net_h + NMS_TY - 1) / NMS_TY;
    dim3 g1((p.net_w + NMS_TX - 1) / NMS_TX, tiles_y < 8 ? tiles_y : 8, nframes * p.num_parts);
    nms_flags_kernel<<<g1, NMS_THREADS, 0, st>>>(pd);
    nms_write_kernel<<<dim3(p.num_parts, nframes), 256, 0, st>>>(pd);
    paf_score_kernel<<<dim3((MP * MP + 127) / 128, p.num_limbs, nframes), 128, 0, st>>>(pd);
    limb_greedy_kernel<<<dim3(p.num_limbs, nframes), 512, sizeof(unsigned long long) * pd.sort_stride, st>>>(pd);
    assemble_kernel<<<nframes, 256, 0, st>>>(pd);
    return 5;  // kernels launched
}

}  // namespace pe
