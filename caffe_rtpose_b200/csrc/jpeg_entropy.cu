// JPEG entropy decoding on the GPU: scan images (pe_jpeg_read_scan) -> the coefficient images pe_jpeg_read_coefs writes, bit for bit.
// The algorithm and the per-subsequence decode are in jpeg_entropy.cuh (shared with the host run pe_jpeg_scan_to_coefs_host).
// Three launches for all frames of a batch:
//   jpeg_scan_prep_kernel   per frame: coefficient header, decoder tables of the 8 Huffman slots, first subsequence of every segment,
//                           reset of the hand-over flags and the status;
//   jpeg_huffman_kernel     128 subsequences per CTA: speculative decode, synchronisation rounds in shared memory, then the hand-over
//                           from the previous CTA of the frame (decoupled look-back on a ticket order, so that a CTA only waits for one
//                           that is already running), block indices by a segmented prefix sum, and the write pass;
//   jpeg_dc_kernel          per frame and component: the DC differences -> values, a segmented prefix sum that restarts with every
//                           restart interval, in unsigned 32-bit arithmetic stored as short (the host's (unsigned)pred + diff).
#include <climits>

#include "jpeg_entropy.cuh"
#include "kernels.h"

namespace pe {

namespace {

using pe_jpeg::HuffDec;
using pe_jpeg::ScanCtx;
using pe_jpeg::State;

__constant__ uint8_t c_zigzag[64] = {0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
                                     35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

__device__ __forceinline__ const pe_jpeg_scan_header* scan_header(const JpegScanArgs& a, int f) {
    return reinterpret_cast<const pe_jpeg_scan_header*>(a.scans + (size_t)f * a.scan_stride);
}
__device__ __forceinline__ HuffDec* frame_tables(const JpegScanArgs& a, int f) { return reinterpret_cast<HuffDec*>(a.tabs) + (size_t)f * 8; }

constexpr int PREP_THREADS = 1024;
__global__ void __launch_bounds__(PREP_THREADS) jpeg_scan_prep_kernel(JpegScanArgs a) {
    const int f = blockIdx.x, t = threadIdx.x;
    const pe_jpeg_scan_header* h = scan_header(a, f);
    const uint8_t* base = a.scans + (size_t)f * a.scan_stride;
    uint8_t* coefs = a.coefs + (size_t)f * a.coef_stride;
    if (t < (int)sizeof(pe_jpeg_coef_header) / 8) reinterpret_cast<unsigned long long*>(coefs)[t] = reinterpret_cast<const unsigned long long*>(base)[t];
    HuffDec* tabs = frame_tables(a, f);
    if (t < 8) pe_jpeg::huff_canon(t < 4 ? h->dc_bits[t] : h->ac_bits[t - 4], tabs[t]);
    for (int i = t; i < 8 * 256; i += PREP_THREADS) tabs[i >> 8].vals[i & 255] = (i >> 8) < 4 ? h->dc_vals[i >> 8][i & 255] : h->ac_vals[(i >> 8) - 4][i & 255];
    if (t == 0) { a.status[f] = INT_MAX; a.tickets[f] = 0; }
    for (int i = t; i < a.ctas_max; i += PREP_THREADS) a.flags[(size_t)f * a.ctas_max + i] = 0;
    __syncthreads();
    for (int i = t; i < 8 << pe_jpeg::LOOK_BITS; i += PREP_THREADS) tabs[i >> pe_jpeg::LOOK_BITS].look[i & ((1 << pe_jpeg::LOOK_BITS) - 1)] =
        pe_jpeg::huff_look_entry(tabs[i >> pe_jpeg::LOOK_BITS], i & ((1 << pe_jpeg::LOOK_BITS) - 1));
    // first subsequence of every segment: exclusive prefix sum of max(1, ceil(8 * bytes / S)), a tile of 1024 segments at a time
    __shared__ int s_sum[PREP_THREADS];
    const int64_t* seg = reinterpret_cast<const int64_t*>(base + h->seg_table_offset);
    int* seg_sub = a.seg_sub + (size_t)f * a.seg_stride;
    const int nseg = h->num_segments;
    int carry = 0;
    for (int t0 = 0; t0 < nseg; t0 += PREP_THREADS) {
        const int s = t0 + t;
        const int v = s < nseg ? (int)pe_jpeg::subseq_count(seg[2 * s + 1], a.S) : 0;
        int x = v;
        s_sum[t] = x;
        __syncthreads();
        for (int off = 1; off < PREP_THREADS; off <<= 1) {
            const int y = t >= off ? s_sum[t - off] : 0;
            __syncthreads();
            x += y;
            s_sum[t] = x;
            __syncthreads();
        }
        if (s < nseg) seg_sub[s] = carry + x - v;
        if (s == nseg - 1) seg_sub[nseg] = carry + x;
        carry += s_sum[PREP_THREADS - 1];
        __syncthreads();
    }
}

constexpr int T = pe_jpeg::SYNC_THREADS;
__global__ void __launch_bounds__(T) jpeg_huffman_kernel(JpegScanArgs a) {
    __shared__ HuffDec s_tab[6];
    __shared__ uint8_t s_zz[64];
    __shared__ State s_ex[T];
    __shared__ long long s_v[T];
    __shared__ int s_h[T];
    __shared__ int s_cta;
    const int f = blockIdx.y, t = threadIdx.x;
    if (t == 0) s_cta = atomicAdd(a.tickets + f, 1);   // CTAs of a frame in the order they started: a predecessor is always running
    __syncthreads();
    const int cta = s_cta;
    const pe_jpeg_scan_header* h = scan_header(a, f);
    const uint8_t* base = a.scans + (size_t)f * a.scan_stride;
    const int* seg_sub = a.seg_sub + (size_t)f * a.seg_stride;
    const int nseg = h->num_segments;
    const int nsub = seg_sub[nseg];
    if ((long long)cta * T >= nsub) return;
    const int nsc = h->num_scan_comps;
    const HuffDec* tabs = frame_tables(a, f);
    for (int i = t; i < 2 * nsc * (int)(sizeof(HuffDec) / 4); i += T) {
        const int k = i / (int)(sizeof(HuffDec) / 4), w = i - k * (int)(sizeof(HuffDec) / 4);
        const HuffDec* src = tabs + ((k & 1) ? 4 + h->ac_table[k >> 1] : h->dc_table[k >> 1]);
        reinterpret_cast<int*>(s_tab + k)[w] = reinterpret_cast<const int*>(src)[w];
    }
    if (t < 64) s_zz[t] = c_zigzag[t];
    ScanCtx c;
    pe_jpeg::scan_slots(*h, c);
    c.data = base + h->data_offset;
    c.seg = reinterpret_cast<const int64_t*>(base + h->seg_table_offset);
    for (int k = 0; k < 3; k++) { c.dc[k] = s_tab + 2 * k; c.ac[k] = s_tab + 2 * k + 1; }
    c.zigzag = s_zz;
    __syncthreads();

    // this thread's subsequence: segment (binary search over the first subsequences), bounds, head / last of its segment
    const long long g = (long long)cta * T + t;
    const bool valid = g < nsub;
    int s = 0;
    bool head = true, last = true;
    long long stop = 0, n = 0;
    const uint8_t* d = c.data;
    State start = 0;
    if (valid) {
        int lo = 0, hi = nseg - 1;
        while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (seg_sub[mid] <= g) lo = mid; else hi = mid - 1; }
        s = lo;
        const long long j = g - seg_sub[s];
        d = c.data + c.seg[2 * s];
        n = c.seg[2 * s + 1];
        head = j == 0;
        last = g == seg_sub[s + 1] - 1;
        stop = last ? n * 8 : (j + 1) * a.S;
        start = head ? 0 : pe_jpeg::pack_state(pe_jpeg::canonical_pos(d, n, j * a.S), 0, 0);
    }
    auto nothing = [](long long, int, int) {};
    State ex = start;
    long long cnt = pe_jpeg::decode_run(c, d, n, &ex, stop, 1LL << 62, nothing);
    s_ex[t] = ex;
    // rounds: every thread takes its predecessor's exit state of the previous round until no start changes
    auto settle = [&]() {
        for (;;) {
            __syncthreads();
            const State ns = (!head && t > 0) ? s_ex[t - 1] : start;
            const bool changed = ns != start;
            __syncthreads();
            if (changed) {
                start = ex = ns;
                cnt = pe_jpeg::decode_run(c, d, n, &ex, stop, 1LL << 62, nothing);
                s_ex[t] = ex;
            }
            if (!__syncthreads_or(changed)) break;
        }
    };
    settle();
    // across CTAs: the previous CTA's final exit state and block index
    __shared__ long long s_carry_block;
    if (t == 0) {
        s_carry_block = 0;
        if (!head && cta > 0) {
            const size_t p = (size_t)f * a.ctas_max + cta - 1;
            volatile int* fl = a.flags + p;
            while (*fl == 0) __nanosleep(64);
            __threadfence();
            const volatile unsigned long long* pub = a.pub + 2 * p;
            const State cs = pub[0];
            s_carry_block = (long long)pub[1];
            if (cs != start) {
                start = ex = cs;
                cnt = pe_jpeg::decode_run(c, d, n, &ex, stop, 1LL << 62, nothing);
                s_ex[0] = ex;
            }
        }
    }
    settle();
    // first block (within the segment) of every subsequence: segmented inclusive prefix sum of the completed blocks
    long long v = cnt + (t == 0 && !head ? s_carry_block : 0);
    int hf = head || t == 0;
    s_v[t] = v; s_h[t] = hf;
    __syncthreads();
    for (int off = 1; off < T; off <<= 1) {
        long long pv = 0; int ph = 0;
        if (t >= off) { pv = s_v[t - off]; ph = s_h[t - off]; }
        __syncthreads();
        if (t >= off && !hf) { v += pv; hf = ph; }
        s_v[t] = v; s_h[t] = hf;
        __syncthreads();
    }
    if (t == T - 1) {   // hand-over to the next CTA of the frame
        const size_t p = (size_t)f * a.ctas_max + cta;
        a.pub[2 * p] = ex;
        a.pub[2 * p + 1] = (unsigned long long)v;
        __threadfence();
        atomicExch(a.flags + p, 1);
    }
    if (!valid) return;
    // write pass: from the synchronised state, into the zeroed coefficient image; the subsequence that holds the end of the data
    // continues into the zero bits until the segment's MCUs are complete
    const long long fb = v - cnt;
    const long long limit = pe_jpeg::segment_mcus(c, s) * c.nslots - fb;
    if (limit <= 0) return;
    uint8_t* coefs = a.coefs + (size_t)f * a.coef_stride;
    int* status = a.status + f;
    State st = start;
    pe_jpeg::decode_run(c, d, n, &st, last ? (1LL << 62) : stop, limit, [&](long long b, int zz, int val) {
        long long mcu = 0;
        const long long off = pe_jpeg::block_offset(*h, c, s, fb + b, &mcu);
        if (zz == -2) { atomicMin(status, (int)mcu); return; }
        reinterpret_cast<short*>(coefs + off)[zz < 0 ? 0 : s_zz[zz]] = (short)val;
    });
}

constexpr int DC_THREADS = 1024;
__global__ void __launch_bounds__(DC_THREADS) jpeg_dc_kernel(JpegScanArgs a) {
    __shared__ unsigned s_v[DC_THREADS];
    __shared__ int s_h[DC_THREADS];
    const int comp = blockIdx.x, f = blockIdx.y, t = threadIdx.x;
    const pe_jpeg_scan_header* h = scan_header(a, f);
    if (comp >= h->coef.num_comps) return;
    ScanCtx c;
    pe_jpeg::scan_slots(*h, c);
    int fs = -1, nbc = 0;
    for (int i = 0; i < c.nslots; i++)
        if (c.slot_comp[i] == comp) { if (fs < 0) fs = i; nbc++; }
    uint8_t* coefs = a.coefs + (size_t)f * a.coef_stride;
    const long long E = c.total_mcus * nbc, chunk = (E + DC_THREADS - 1) / DC_THREADS;
    const long long e0 = t * chunk, e1 = e0 + chunk < E ? e0 + chunk : E;
    auto element = [&](long long e, bool* reset) {   // the e-th block of the component in decode order
        const long long mcu = e / nbc;
        const int l = (int)(e - mcu * nbc);
        const int sg = c.restart ? (int)(mcu / c.restart) : 0;
        *reset = l == 0 && mcu == (long long)sg * c.restart;
        return reinterpret_cast<short*>(coefs + pe_jpeg::block_offset(*h, c, sg, (mcu - (long long)sg * c.restart) * c.nslots + fs + l, nullptr));
    };
    unsigned sum = 0;
    int hf = 0;
    for (long long e = e0; e < e1; e++) {
        bool r;
        const unsigned dv = (unsigned)(int)*element(e, &r);
        if (r) { sum = dv; hf = 1; } else { sum += dv; }
    }
    s_v[t] = sum; s_h[t] = hf;
    __syncthreads();
    for (int off = 1; off < DC_THREADS; off <<= 1) {
        unsigned pv = 0; int ph = 0;
        if (t >= off) { pv = s_v[t - off]; ph = s_h[t - off]; }
        __syncthreads();
        if (t >= off && !hf) { sum += pv; hf = ph; }
        s_v[t] = sum; s_h[t] = hf;
        __syncthreads();
    }
    unsigned run = t > 0 ? s_v[t - 1] : 0;
    for (long long e = e0; e < e1; e++) {
        bool r;
        short* dc = element(e, &r);
        const unsigned dv = (unsigned)(int)*dc;
        run = r ? dv : run + dv;
        *dc = (short)run;
    }
}

}  // namespace

size_t jpeg_huff_tables_bytes() { return sizeof(HuffDec) * 8; }

int launch_jpeg_entropy(const JpegScanArgs& a, cudaStream_t st) {
    jpeg_scan_prep_kernel<<<a.n, PREP_THREADS, 0, st>>>(a);
    jpeg_huffman_kernel<<<dim3((unsigned)a.ctas_max, a.n), T, 0, st>>>(a);
    jpeg_dc_kernel<<<dim3(3, a.n), DC_THREADS, 0, st>>>(a);
    return 3;
}

}  // namespace pe
