// Baseline JPEG decoder for --image_dir: the reference reads its input images with cv::imread
// (examples/rtpose/rtpose.cpp:302-391, getFrameFromDir), i.e. libjpeg with its defaults.  No libjpeg / OpenCV for C++ in
// this image, so the decoder is written out here and follows libjpeg's DEFAULT decompression arithmetic exactly, so that
// a frame decoded here equals cv::imread's bytes (tests/test_abi.py compares with cv2):
//   * Huffman sequential (SOF0 / SOF1) and progressive (SOF2: spectral selection + successive approximation) DCT, 8-bit,
//     interleaved and non-interleaved scans, restart intervals, 8- and 16-bit quantisation tables;
//   * the "islow" integer inverse DCT (13-bit constants, 2 extra bits after pass 1, Loeffler-Ligtenberg-Moschytz);
//   * "fancy" triangle-filter chroma upsampling for 2x1 and 2x2 subsampling (3/4-1/4 weights, libjpeg's rounding biases),
//     plain replication when the chroma plane is at most 2 samples wide;
//   * YCbCr -> RGB with libjpeg's 16-bit fixed-point tables.
// Not handled (return code -2): arithmetic-coded / lossless / hierarchical / 12-bit files, CMYK, chroma sampling other
// than 4:4:4 / 4:2:2 / 4:2:0.  EXIF orientation is ignored (as in the OpenCV 2.4 / 3.0 the reference was written for).
//
// Two routes to the same bytes.  The GENERAL route keeps every coefficient of the frame (needed by progressive and multi-scan
// files) and transforms afterwards.  The FAST route serves what a camera or cv::imwrite produces - one interleaved sequential
// scan - and is what feeds the GPUs in rtpose.bin (one H100 consumes 200-300 frames/s, a decoder thread of the general route
// delivers 45): a 64-bit bit reader that refills eight bytes at a time, a 10-bit lookahead that resolves an AC code AND its
// value bits in one table access, blocks transformed straight out of the entropy decoder (no coefficient image), the islow
// IDCT on eight columns at once in 32-bit AVX2 lanes (used only when the block's values are provably inside 32 bits; otherwise
// the 64-bit scalar form, so corrupt data decodes identically too), and row-wise fused upsampling + colour conversion.  Anything
// unusual (second scan, failure, no AVX2) re-runs the general route, whose result is the definition.  PE_JPEG_FAST=0 disables
// the fast route (tests compare the two).
// pe_jpeg_read_coefs stops after the entropy stage: both routes store the coefficient image (jpeg_coefs.h) instead of transforming
// it, and the GPU reconstructs the pixels (jpeg_gpu.cu); pe_jpeg_coefs_to_bgr is the same reconstruction on the host.
// Host code, no GPU.
#include "jpeg_tables.h"
#include "jpeg_coefs.h"
#include "jpeg_entropy.cuh"
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#if defined(__x86_64__) && defined(__GNUC__)
#include <immintrin.h>
#define PE_JPEG_X86 1
#else
#define PE_JPEG_X86 0
#endif

#include "../../include/poseengine.h"

namespace {

const uint8_t kZigzagNat[64] = {0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
                                35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

struct HuffTab {
    bool set = false;
    uint8_t bits[17] = {0};
    uint8_t vals[256] = {0};
    int mincode[17], maxcode[18], valptr[17];
    static constexpr int LOOK = 10;
    uint8_t look_len[1 << LOOK];   // 10-bit lookahead: code length (0 = longer than 10 bits)
    uint8_t look_sym[1 << LOOK];
    // AC tables: code + value bits resolved together when both fit into the lookahead.  value << 16 | run << 8 | total bits; 0 = not available
    int32_t fast_ac[1 << LOOK];
    bool build() {   // false: the code lengths over-subscribe the code space (corrupt DHT)
        int code = 0, k = 0;
        for (int l = 1; l <= 16; l++) {
            valptr[l] = k;
            mincode[l] = code;
            code += bits[l];
            if (code > (1 << l)) return false;
            k += bits[l];
            maxcode[l] = bits[l] ? code - 1 : -1;
            code <<= 1;
        }
        maxcode[17] = 0x7fffffff;
        memset(look_len, 0, sizeof look_len);
        k = 0;
        code = 0;
        for (int l = 1; l <= LOOK; l++) {
            for (int i = 0; i < bits[l]; i++, k++, code++) {
                const int first = code << (LOOK - l);
                for (int f = 0; f < (1 << (LOOK - l)); f++) { look_len[first + f] = (uint8_t)l; look_sym[first + f] = vals[k]; }
            }
            code <<= 1;
        }
        for (int i = 0; i < (1 << LOOK); i++) {
            fast_ac[i] = 0;
            const int l = look_len[i], r = look_sym[i] >> 4, sz = look_sym[i] & 15;
            if (l && sz && l + sz <= LOOK) {
                int v = (i >> (LOOK - l - sz)) & ((1 << sz) - 1);
                if (v < (1 << (sz - 1))) v = v - (1 << sz) + 1;   // extend()
                fast_ac[i] = (int32_t)((uint32_t)v << 16 | (uint32_t)r << 8 | (uint32_t)(l + sz));
            }
        }
        set = true;
        return true;
    }
};

struct BitReader {
    const uint8_t* p; const uint8_t* end;
    uint32_t acc = 0;
    int n = 0;
    bool hit_marker = false;
    void fill() {
        while (n <= 24) {
            uint32_t b = 0;
            if (!hit_marker && p < end) {
                b = *p;
                if (b == 0xFF) {
                    if (p + 1 < end && p[1] == 0) p += 2;
                    else { hit_marker = true; b = 0; }   // a marker: feed zeros (libjpeg does the same past the data)
                } else {
                    p++;
                }
            }
            acc |= b << (24 - n);
            n += 8;
        }
    }
    inline int peek(int k) { if (n < k) fill(); return (int)(acc >> (32 - k)); }
    inline void skip(int k) { acc <<= k; n -= k; }
    inline int get(int k) { if (k == 0) return 0; const int v = peek(k); skip(k); return v; }
    void reset() { acc = 0; n = 0; hit_marker = false; }
};

// Bit reader of the fast route: 64-bit window, refilled with up to eight bytes at once when none of them is 0xFF (no stuffing,
// no marker); otherwise byte by byte under the general reader's rules (FF00 = data byte FF, a marker stops the input and zeros follow).
struct FastBits {
    const uint8_t* p; const uint8_t* end;
    uint64_t acc = 0;
    int n = 0;
    bool hit_marker = false;
    void refill_slow() {
        while (n <= 56) {
            uint64_t b = 0;
            if (!hit_marker && p < end) {
                b = *p;
                if (b == 0xFF) {
                    if (p + 1 < end && p[1] == 0) p += 2;
                    else { hit_marker = true; b = 0; }
                } else {
                    p++;
                }
            }
            acc |= b << (56 - n);
            n += 8;
        }
    }
    inline void refill() {   // precondition n < 32; afterwards n > 56
        if (!hit_marker && end - p >= 8) {
            uint64_t v;
            memcpy(&v, p, 8);
            const uint64_t x = ~v;   // a zero byte of x = an FF byte of v
            if (!((x - 0x0101010101010101ull) & ~x & 0x8080808080808080ull)) {
                const int k = (64 - n) >> 3;   // whole bytes that fit: 5..8
                acc |= (__builtin_bswap64(v) & (~0ull << (64 - 8 * k))) >> n;
                p += k;
                n += 8 * k;
                return;
            }
        }
        refill_slow();
    }
    inline int peek(int k) { if (n < k) refill(); return (int)(acc >> (64 - k)); }
    inline void skip(int k) { acc <<= k; n -= k; }
    inline int get(int k) { if (k == 0) return 0; const int v = peek(k); skip(k); return v; }
    void reset() { acc = 0; n = 0; hit_marker = false; }
};

template <class Reader>
inline int huff_decode(Reader& br, const HuffTab& t) {
    const int look = br.peek(HuffTab::LOOK);
    const int l = t.look_len[look];
    if (l) { br.skip(l); return t.look_sym[look]; }
    int code = br.peek(16);
    for (int len = HuffTab::LOOK + 1; len <= 16; len++) {
        const int c = code >> (16 - len);
        if (t.maxcode[len] >= 0 && c <= t.maxcode[len] && c >= t.mincode[len]) {
            br.skip(len);
            return t.vals[t.valptr[len] + c - t.mincode[len]];
        }
    }
    br.skip(16);
    return 0;   // corrupt data: libjpeg warns and returns 0
}
inline int extend(int v, int s) { return v < (1 << (s - 1)) ? v - (1 << s) + 1 : v; }

// ---- jpeg_idct_islow: dequantise + inverse DCT of one block into 8 rows of the component plane
constexpr int CONST_BITS = 13, PASS1_BITS = 2;
constexpr int F_0_298631336 = 2446, F_0_390180644 = 3196, F_0_541196100 = 4433, F_0_765366865 = 6270, F_0_899976223 = 7373, F_1_175875602 = 9633,
              F_1_501321110 = 12299, F_1_847759065 = 15137, F_1_961570560 = 16069, F_2_053119869 = 16819, F_2_562915447 = 20995, F_3_072711026 = 25172;
typedef long long jlong;   // libjpeg's JLONG is `long` (64-bit on LP64): corrupt data must not overflow the intermediates
inline jlong descale(jlong x, int n) { return (x + ((jlong)1 << (n - 1))) >> n; }
inline uint8_t range_limit(jlong x) { x += 128; return (uint8_t)(x < 0 ? 0 : (x > 255 ? 255 : x)); }

inline void idct_1d(const int* in, int stride, jlong* o) {
    // even part
    jlong z2 = in[2 * stride], z3 = in[6 * stride];
    jlong z1 = (z2 + z3) * F_0_541196100;
    jlong tmp2 = z1 + z3 * (-F_1_847759065);
    jlong tmp3 = z1 + z2 * F_0_765366865;
    z2 = in[0];
    z3 = in[4 * stride];
    jlong tmp0 = (z2 + z3) * (1 << CONST_BITS);
    jlong tmp1 = (z2 - z3) * (1 << CONST_BITS);
    const jlong tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    // odd part
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

void idct_islow(const short* coef, const uint16_t* quant, uint8_t* out, int out_stride) {
    int deq[64], ws[64];
    jlong o[8];
    for (int i = 0; i < 64; i++) deq[i] = (int)((jlong)coef[i] * (jlong)quant[i]);
    for (int c = 0; c < 8; c++) {   // pass 1: columns
        if ((deq[8 + c] | deq[16 + c] | deq[24 + c] | deq[32 + c] | deq[40 + c] | deq[48 + c] | deq[56 + c]) == 0) {
            // libjpeg's shortcut for a column without AC terms; the general formula gives the same value (dc << PASS1_BITS)
            const int dcv = (int)((jlong)deq[c] * (1 << PASS1_BITS));   // 64-bit like the general path (corrupt 16-bit DQT x DC overflows int)
            for (int r = 0; r < 8; r++) ws[r * 8 + c] = dcv;
            continue;
        }
        idct_1d(deq + c, 8, o);
        for (int r = 0; r < 8; r++) ws[r * 8 + c] = (int)descale(o[r], CONST_BITS - PASS1_BITS);
    }
    for (int r = 0; r < 8; r++) {   // pass 2: rows
        const int* w = ws + r * 8;
        if ((w[1] | w[2] | w[3] | w[4] | w[5] | w[6] | w[7]) == 0) {   // same shortcut, again value-identical
            const uint8_t v = range_limit(descale((jlong)w[0], PASS1_BITS + 3));
            for (int c = 0; c < 8; c++) out[r * out_stride + c] = v;
            continue;
        }
        idct_1d(w, 1, o);
        for (int c = 0; c < 8; c++) out[r * out_stride + c] = range_limit(descale(o[c], CONST_BITS + PASS1_BITS + 3));
    }
}

#if PE_JPEG_X86
// ---- the same transform on eight columns at once: 32-bit AVX2 lanes -------------------------------------------------
// With every input of a pass bounded by B in magnitude, no intermediate of idct_1d exceeds 178219 * B (sum of the absolute
// constants along the longest path); B <= 8192 keeps that and the rounding constant below 2^31, so the 32-bit lanes hold
// exactly the values of the 64-bit scalar form.  Real image data stays far below the bound; blocks that do not (corrupt
// streams) take the scalar form.
#define PE_AVX2 __attribute__((target("avx2")))
#ifndef PE_IDCT32_BOUND
#define PE_IDCT32_BOUND 8192
#endif
constexpr int IDCT32_BOUND = PE_IDCT32_BOUND;   // tests build with a tiny bound to drive blocks through the scalar fallback

PE_AVX2 static inline void idct_1d_x8(const __m256i* in, __m256i* o) {
#define MULC(x, c) _mm256_mullo_epi32(x, _mm256_set1_epi32(c))
#define ADD(a, b) _mm256_add_epi32(a, b)
#define SUB(a, b) _mm256_sub_epi32(a, b)
    __m256i z2 = in[2], z3 = in[6];
    __m256i z1 = MULC(ADD(z2, z3), F_0_541196100);
    __m256i tmp2 = ADD(z1, MULC(z3, -F_1_847759065));
    __m256i tmp3 = ADD(z1, MULC(z2, F_0_765366865));
    z2 = in[0];
    z3 = in[4];
    __m256i tmp0 = _mm256_slli_epi32(ADD(z2, z3), CONST_BITS);
    __m256i tmp1 = _mm256_slli_epi32(SUB(z2, z3), CONST_BITS);
    const __m256i tmp10 = ADD(tmp0, tmp3), tmp13 = SUB(tmp0, tmp3), tmp11 = ADD(tmp1, tmp2), tmp12 = SUB(tmp1, tmp2);
    tmp0 = in[7]; tmp1 = in[5]; tmp2 = in[3]; tmp3 = in[1];
    z1 = ADD(tmp0, tmp3); z2 = ADD(tmp1, tmp2); z3 = ADD(tmp0, tmp2);
    __m256i z4 = ADD(tmp1, tmp3);
    const __m256i z5 = MULC(ADD(z3, z4), F_1_175875602);
    tmp0 = MULC(tmp0, F_0_298631336); tmp1 = MULC(tmp1, F_2_053119869); tmp2 = MULC(tmp2, F_3_072711026); tmp3 = MULC(tmp3, F_1_501321110);
    z1 = MULC(z1, -F_0_899976223); z2 = MULC(z2, -F_2_562915447); z3 = MULC(z3, -F_1_961570560); z4 = MULC(z4, -F_0_390180644);
    z3 = ADD(z3, z5); z4 = ADD(z4, z5);
    tmp0 = ADD(tmp0, ADD(z1, z3)); tmp1 = ADD(tmp1, ADD(z2, z4)); tmp2 = ADD(tmp2, ADD(z2, z3)); tmp3 = ADD(tmp3, ADD(z1, z4));
    o[0] = ADD(tmp10, tmp3); o[7] = SUB(tmp10, tmp3); o[1] = ADD(tmp11, tmp2); o[6] = SUB(tmp11, tmp2);
    o[2] = ADD(tmp12, tmp1); o[5] = SUB(tmp12, tmp1); o[3] = ADD(tmp13, tmp0); o[4] = SUB(tmp13, tmp0);
#undef MULC
#undef ADD
#undef SUB
}
PE_AVX2 static inline void transpose_8x8(__m256i* r) {
    const __m256i t0 = _mm256_unpacklo_epi32(r[0], r[1]), t1 = _mm256_unpackhi_epi32(r[0], r[1]);
    const __m256i t2 = _mm256_unpacklo_epi32(r[2], r[3]), t3 = _mm256_unpackhi_epi32(r[2], r[3]);
    const __m256i t4 = _mm256_unpacklo_epi32(r[4], r[5]), t5 = _mm256_unpackhi_epi32(r[4], r[5]);
    const __m256i t6 = _mm256_unpacklo_epi32(r[6], r[7]), t7 = _mm256_unpackhi_epi32(r[6], r[7]);
    const __m256i u0 = _mm256_unpacklo_epi64(t0, t2), u1 = _mm256_unpackhi_epi64(t0, t2);
    const __m256i u2 = _mm256_unpacklo_epi64(t1, t3), u3 = _mm256_unpackhi_epi64(t1, t3);
    const __m256i u4 = _mm256_unpacklo_epi64(t4, t6), u5 = _mm256_unpackhi_epi64(t4, t6);
    const __m256i u6 = _mm256_unpacklo_epi64(t5, t7), u7 = _mm256_unpackhi_epi64(t5, t7);
    r[0] = _mm256_permute2x128_si256(u0, u4, 0x20); r[1] = _mm256_permute2x128_si256(u1, u5, 0x20);
    r[2] = _mm256_permute2x128_si256(u2, u6, 0x20); r[3] = _mm256_permute2x128_si256(u3, u7, 0x20);
    r[4] = _mm256_permute2x128_si256(u0, u4, 0x31); r[5] = _mm256_permute2x128_si256(u1, u5, 0x31);
    r[6] = _mm256_permute2x128_si256(u2, u6, 0x31); r[7] = _mm256_permute2x128_si256(u3, u7, 0x31);
}
PE_AVX2 static inline bool all_within(const __m256i* v, int bound) {
    __m256i m = _mm256_abs_epi32(v[0]);
    for (int i = 1; i < 8; i++) m = _mm256_max_epu32(m, _mm256_abs_epi32(v[i]));   // abs(INT_MIN) stays 0x80000000: unsigned max keeps it largest
    return _mm256_testz_si256(_mm256_cmpgt_epi32(_mm256_xor_si256(m, _mm256_set1_epi32((int)0x80000000)),
                                                 _mm256_set1_epi32((int)(0x80000000u + (unsigned)bound))), _mm256_set1_epi32(-1));
}
// false: the block leaves the 32-bit-safe range -> the caller runs idct_islow
PE_AVX2 static bool idct_islow_avx2(const short* coef, const uint16_t* quant, uint8_t* out, int out_stride) {
    __m256i v[8], o[8];
    for (int r = 0; r < 8; r++)
        v[r] = _mm256_mullo_epi32(_mm256_cvtepi16_epi32(_mm_loadu_si128((const __m128i*)(coef + 8 * r))),
                                  _mm256_cvtepu16_epi32(_mm_loadu_si128((const __m128i*)(quant + 8 * r))));
    if (!all_within(v, IDCT32_BOUND)) return false;
    idct_1d_x8(v, o);                                   // pass 1: lane c = column c
    const __m256i r1 = _mm256_set1_epi32(1 << (CONST_BITS - PASS1_BITS - 1));
    for (int r = 0; r < 8; r++) v[r] = _mm256_srai_epi32(_mm256_add_epi32(o[r], r1), CONST_BITS - PASS1_BITS);   // workspace rows
    if (!all_within(v, IDCT32_BOUND)) return false;
    transpose_8x8(v);                                   // v[k] = workspace column k, lane r = row r
    idct_1d_x8(v, o);                                   // pass 2: o[c], lane r = output (r, c) before descaling
    const __m256i r2 = _mm256_set1_epi32(1 << (CONST_BITS + PASS1_BITS + 3 - 1)), c128 = _mm256_set1_epi32(128);
    for (int c = 0; c < 8; c++) o[c] = _mm256_add_epi32(_mm256_srai_epi32(_mm256_add_epi32(o[c], r2), CONST_BITS + PASS1_BITS + 3), c128);
    transpose_8x8(o);                                   // o[r] = output row r
    const __m256i order = _mm256_setr_epi32(0, 4, 1, 5, 2, 6, 3, 7);
    for (int h = 0; h < 2; h++) {                       // four rows at a time: saturate to bytes (= range_limit), 8 bytes per row
        const __m256i a = _mm256_packs_epi32(o[4 * h], o[4 * h + 1]), b = _mm256_packs_epi32(o[4 * h + 2], o[4 * h + 3]);
        const __m256i q = _mm256_permutevar8x32_epi32(_mm256_packus_epi16(a, b), order);
        alignas(32) uint64_t rows[4];
        _mm256_store_si256((__m256i*)rows, q);
        for (int r = 0; r < 4; r++) memcpy(out + (size_t)(4 * h + r) * out_stride, &rows[r], 8);
    }
    return true;
}
static const bool g_have_avx2 = __builtin_cpu_supports("avx2");
#else
static const bool g_have_avx2 = false;
#endif

// dequantise + inverse DCT of one block; dc_only: the entropy decoder wrote no AC coefficient (both passes take their zero-AC shortcut)
inline void idct_block(const short* coef, const uint16_t* quant, uint8_t* out, int out_stride, bool dc_only) {
    if (dc_only) {
        const int deq = (int)((jlong)coef[0] * (jlong)quant[0]);
        const int dcv = (int)((jlong)deq * (1 << PASS1_BITS));
        const uint8_t v = range_limit(descale((jlong)dcv, PASS1_BITS + 3));
        for (int r = 0; r < 8; r++) memset(out + (size_t)r * out_stride, v, 8);
        return;
    }
#if PE_JPEG_X86
    if (g_have_avx2 && idct_islow_avx2(coef, quant, out, out_stride)) return;
#endif
    idct_islow(coef, quant, out, out_stride);
}

struct Comp {
    int id = 0, h = 1, v = 1, tq = 0, td = 0, ta = 0;
    int pw = 0, ph = 0;     // plane size in samples, padded to whole MCUs
    int dw = 0, dh = 0;     // real (downsampled) samples
    int bw = 0, bh = 0;     // blocks per row / column of the padded plane
    int nbw = 0, nbh = 0;   // blocks that cover the real samples (extent of a non-interleaved scan)
    std::vector<uint8_t> plane;
    std::vector<short> coef;   // [bh][bw][64], natural order
    uint16_t q[64];
    bool q_latched = false;
    int pred = 0;
};

inline uint16_t rd16(const uint8_t* p) { return (uint16_t)((p[0] << 8) | p[1]); }

// One block of a scan (T.81 F.2.2 sequential, G.1.2 progressive; decode_mcu_* of libjpeg's jdhuff.c / jdphuff.c)
struct ScanParams { int Ss, Se, Ah, Al; bool progressive; };
inline bool decode_block(BitReader& br, Comp& c, const HuffTab* dc, const HuffTab* ac, short* blk, const ScanParams& sp, int& eobrun) {
    if (!sp.progressive) {
        int s = huff_decode(br, dc[c.td]);
        if (s > 15) return false;
        c.pred = (int)((unsigned)c.pred + (unsigned)(s ? extend(br.get(s), s) : 0));   // unsigned wrap: no UB on corrupt streams
        blk[0] = (short)c.pred;
        for (int k = 1; k < 64;) {
            const int rs = huff_decode(br, ac[c.ta]);
            const int r = rs >> 4;
            s = rs & 15;
            if (s == 0) { if (r != 15) break; k += 16; continue; }
            k += r;
            if (k > 63) break;
            blk[kZigzagNat[k]] = (short)extend(br.get(s), s);
            k++;
        }
        return true;
    }
    if (sp.Ss == 0) {
        if (sp.Ah == 0) {   // DC first
            const int s = huff_decode(br, dc[c.td]);
            if (s > 15) return false;
            c.pred = (int)((unsigned)c.pred + (unsigned)(s ? extend(br.get(s), s) : 0));
            blk[0] = (short)((unsigned)c.pred << sp.Al);
        } else if (br.get(1)) {   // DC refinement
            blk[0] = (short)(blk[0] | (1 << sp.Al));
        }
        return true;
    }
    if (sp.Ah == 0) {       // AC first
        if (eobrun > 0) { eobrun--; return true; }
        for (int k = sp.Ss; k <= sp.Se; k++) {
            const int rs = huff_decode(br, ac[c.ta]);
            const int r = rs >> 4, s = rs & 15;
            if (s) {
                k += r;
                if (k > 63) return false;
                blk[kZigzagNat[k]] = (short)(extend(br.get(s), s) * (1 << sp.Al));
            } else if (r == 15) {
                k += 15;
            } else {
                eobrun = 1 << r;
                if (r) eobrun += br.get(r);
                eobrun--;
                break;
            }
        }
        return true;
    }
    // AC refinement
    const int p1 = 1 << sp.Al, m1 = -(1 << sp.Al);
    int k = sp.Ss;
    if (eobrun == 0) {
        for (; k <= sp.Se; k++) {
            const int rs = huff_decode(br, ac[c.ta]);
            int r = rs >> 4, s = rs & 15;
            if (s) {
                s = br.get(1) ? p1 : m1;   // a newly non-zero coefficient is always +-1 at this bit
            } else if (r != 15) {
                eobrun = 1 << r;
                if (r) eobrun += br.get(r);
                break;
            }
            do {   // skip r still-zero coefficients, correcting the already non-zero ones on the way
                short* co = blk + kZigzagNat[k];
                if (*co != 0) {
                    if (br.get(1) && (*co & p1) == 0) *co = (short)(*co + (*co >= 0 ? p1 : m1));
                } else if (--r < 0) {
                    break;
                }
                k++;
            } while (k <= sp.Se);
            if (s) { if (k > 63) return false; blk[kZigzagNat[k]] = (short)s; }
        }
    }
    if (eobrun > 0) {
        for (; k <= sp.Se; k++) {
            short* co = blk + kZigzagNat[k];
            if (*co != 0 && br.get(1) && (*co & p1) == 0) *co = (short)(*co + (*co >= 0 ? p1 : m1));
        }
        eobrun--;
    }
    return true;
}

// Sequential block on the fast route: the symbols, bit positions and stop rules of decode_block's sequential branch
inline bool decode_block_seq(FastBits& br, int& pred, const HuffTab& dct, const HuffTab& act, short* blk, bool& dc_only) {
    if (br.n < 32) br.refill();
    int s = huff_decode(br, dct);
    if (s > 15) return false;
    pred = (int)((unsigned)pred + (unsigned)(s ? extend(br.get(s), s) : 0));
    blk[0] = (short)pred;
    dc_only = true;
    for (int k = 1; k < 64;) {
        if (br.n < 32) br.refill();   // a code (<= 16 bits) and its value (<= 15) are in the window
        const int look = (int)(br.acc >> (64 - HuffTab::LOOK));
        const int32_t fe = act.fast_ac[look];
        if (fe) {
            k += (fe >> 8) & 15;
            if (k > 63) { br.skip(act.look_len[look]); break; }   // the general route stops before the value bits
            br.skip(fe & 255);
            blk[kZigzagNat[k]] = (short)(fe >> 16);
            dc_only = false;
            k++;
            continue;
        }
        const int rs = huff_decode(br, act);
        const int r = rs >> 4;
        s = rs & 15;
        if (s == 0) { if (r != 15) break; k += 16; continue; }
        k += r;
        if (k > 63) break;
        blk[kZigzagNat[k]] = (short)extend(br.get(s), s);
        dc_only = false;
        k++;
    }
    return true;
}

// ---- output stage: chroma rows at full resolution + YCbCr -> BGR, one image row at a time ----
// libjpeg jdsample.c: h2v1_fancy_upsample / h2v2_fancy_upsample / replication fallbacks, one output row of a component with dw x dh
// real samples; out holds >= 2 * dw + 2 bytes, col >= dw uint16
template <bool DUMMY>
static inline __attribute__((always_inline)) void upsample_row_impl(const Comp& c, int hs, int vs, int y, int W, uint8_t* __restrict out,
                                                                    uint16_t* __restrict col) {
    const uint8_t* src = c.plane.data();
    const int pw = c.pw, dw = c.dw, dh = c.dh;
    auto row = [&](int r) { r = r < 0 ? 0 : (r >= dh ? dh - 1 : r); return src + (size_t)r * pw; };
    if (hs == 1 && vs == 1) { memcpy(out, row(y), W); return; }
    const bool fancy = dw > 2;
    if (vs == 1) {   // h2v1
        const uint8_t* __restrict in = row(y);
        if (!fancy) { for (int x = 0; x < dw; x++) out[2 * x] = out[2 * x + 1] = in[x]; return; }
        out[0] = in[0];
        out[1] = (uint8_t)((in[0] * 3 + in[1] + 2) >> 2);
        for (int x = 1; x < dw - 1; x++) {
            const int inv = in[x] * 3;
            out[2 * x] = (uint8_t)((inv + in[x - 1] + 1) >> 2);
            out[2 * x + 1] = (uint8_t)((inv + in[x + 1] + 2) >> 2);
        }
        out[2 * (dw - 1)] = (uint8_t)((in[dw - 1] * 3 + in[dw - 2] + 1) >> 2);
        out[2 * (dw - 1) + 1] = in[dw - 1];
        return;
    }
    const int r = y >> 1;   // h2v2
    const uint8_t* __restrict in0 = row(r);
    if (!fancy) { for (int x = 0; x < dw; x++) out[2 * x] = out[2 * x + 1] = in0[x]; return; }
    const uint8_t* __restrict in1 = (y & 1) ? row(r + 1) : row(r - 1);   // the nearer row weighs 3, the other 1
    for (int x = 0; x < dw; x++) col[x] = (uint16_t)(in0[x] * 3 + in1[x]);
    out[0] = (uint8_t)((col[0] * 4 + 8) >> 4);
    out[1] = (uint8_t)((col[0] * 3 + col[1] + 7) >> 4);
    for (int x = 1; x < dw - 1; x++) {
        const int t3 = col[x] * 3;
        out[2 * x] = (uint8_t)((t3 + col[x - 1] + 8) >> 4);
        out[2 * x + 1] = (uint8_t)((t3 + col[x + 1] + 7) >> 4);
    }
    out[2 * (dw - 1)] = (uint8_t)((col[dw - 1] * 3 + col[dw - 2] + 8) >> 4);
    out[2 * (dw - 1) + 1] = (uint8_t)((col[dw - 1] * 4 + 7) >> 4);
}
// jdcolor.c build_ycc_rgb_table, SCALEBITS 16: the table entries written out as the arithmetic that fills them
// (Cr_r = (FIX(1.40200) x + HALF) >> 16, Cb_b = (FIX(1.77200) x + HALF) >> 16, green = (-FIX(0.34414) cb - FIX(0.71414) cr + HALF) >> 16)
template <bool DUMMY>
static inline __attribute__((always_inline)) void ycc_row_impl(const uint8_t* __restrict yrow, const uint8_t* __restrict cb,
                                                               const uint8_t* __restrict cr, uint8_t* __restrict o, int W) {
    for (int x = 0; x < W; x++) {
        const int Y = yrow[x], b = cb[x] - 128, r = cr[x] - 128;
        int R = Y + ((91881 * r + 32768) >> 16);
        int G = Y + ((-22554 * b + 32768 - 46802 * r) >> 16);
        int B = Y + ((116130 * b + 32768) >> 16);
        R = R < 0 ? 0 : (R > 255 ? 255 : R);
        G = G < 0 ? 0 : (G > 255 ? 255 : G);
        B = B < 0 ? 0 : (B > 255 ? 255 : B);
        o[3 * x] = (uint8_t)B; o[3 * x + 1] = (uint8_t)G; o[3 * x + 2] = (uint8_t)R;
    }
}
template <bool DUMMY>
static inline __attribute__((always_inline)) void output_rows_impl(const std::vector<Comp>& comps, int hmax, int vmax, int W, int H, uint8_t* bgr) {
    const Comp& yc = comps[0];
    const int maxdw = comps[1].dw > comps[2].dw ? comps[1].dw : comps[2].dw;
    std::vector<uint8_t> cb((size_t)2 * maxdw + W + 64), cr((size_t)2 * maxdw + W + 64);
    std::vector<uint16_t> col((size_t)maxdw + 16);
    for (int y = 0; y < H; y++) {
        upsample_row_impl<DUMMY>(comps[1], hmax / comps[1].h, vmax / comps[1].v, y, W, cb.data(), col.data());
        upsample_row_impl<DUMMY>(comps[2], hmax / comps[2].h, vmax / comps[2].v, y, W, cr.data(), col.data());
        ycc_row_impl<DUMMY>(yc.plane.data() + (size_t)y * yc.pw, cb.data(), cr.data(), bgr + (size_t)y * W * 3, W);
    }
}
#if PE_JPEG_X86
PE_AVX2 static void output_rows_avx2(const std::vector<Comp>& comps, int hmax, int vmax, int W, int H, uint8_t* bgr) {
    output_rows_impl<true>(comps, hmax, vmax, W, H, bgr);
}
#endif
static void output_rows(const std::vector<Comp>& comps, int hmax, int vmax, int W, int H, uint8_t* bgr) {
#if PE_JPEG_X86
    if (g_have_avx2) return output_rows_avx2(comps, hmax, vmax, W, H, bgr);
#endif
    output_rows_impl<false>(comps, hmax, vmax, W, H, bgr);
}

// Coefficient output of pe_jpeg_read_coefs: the entropy stage alone, its result stored instead of transformed
struct CoefOut {
    uint8_t* buf;       // NULL: only the size is wanted
    long long cap;
    pe_jpeg_coef_header hdr;
    short* coef(int k) const { return (short*)(buf + hdr.comp[k].offset); }
};

// Scan output of pe_jpeg_read_scan: the fast route's scan recorded (tables, restart segments, entropy-coded bytes) instead of decoded
struct ScanOut {
    pe_jpeg_scan_header hdr;
    std::vector<int64_t> seg;   // offset, length per segment, offsets from `data`
    const uint8_t* data = nullptr;
};

static int decode_impl(const uint8_t* data, long long size, int* w, int* h, uint8_t* bgr, long long cap, bool allow_fast, CoefOut* co = nullptr,
                       ScanOut* so = nullptr);
static void reconstruct(std::vector<Comp>& comps, int hmax, int vmax, int W, int H, uint8_t* bgr);

}  // namespace

// JPEG bytes -> uint8 BGR HWC.  Returns 0 and the size in *w, *h (pixels are written when bgr != NULL and cap suffices),
// -1 = not a JPEG / truncated / corrupt, -2 = a JPEG this decoder does not handle (see the top of this file).
extern "C" int pe_decode_jpeg(const uint8_t* data, long long size, int* w, int* h, uint8_t* bgr, long long cap) {
    const char* env = getenv("PE_JPEG_FAST");
    return decode_impl(data, size, w, h, bgr, cap, !(env && env[0] == '0'));
}

namespace {
static int decode_impl(const uint8_t* data, long long size, int* w, int* h, uint8_t* bgr, long long cap, bool allow_fast, CoefOut* co, ScanOut* so) {
    if (!data || size < 4 || data[0] != 0xFF || data[1] != 0xD8) return -1;
    uint16_t quant[4][64];
    bool quant_set[4] = {false, false, false, false};
    HuffTab dc[4], ac[4];
    std::vector<Comp> comps;
    int W = 0, H = 0, restart = 0, hmax = 1, vmax = 1, mcux = 0, mcuy = 0;
    const uint8_t* p = data + 2;
    const uint8_t* end = data + size;
    bool have_sof = false, progressive = false, any_scan = false, eoi = false, fast_done = false;
    while (!eoi) {
        while (p < end && *p != 0xFF) p++;
        while (p < end && *p == 0xFF) p++;
        if (p >= end) break;                               // no EOI: libjpeg warns and uses what it has
        const int m = *p++;
        if (m == 0xD9) { eoi = true; break; }
        if (m == 0x00 || m == 0x01 || (m >= 0xD0 && m <= 0xD7)) continue;
        if (p + 2 > end) break;
        const int len = rd16(p);
        if (len < 2 || p + len > end) { if (any_scan) break; return -1; }
        const uint8_t* s = p + 2;
        const uint8_t* se = p + len;
        if (m == 0xDB) {                                   // DQT
            while (s < se) {
                const int pq = *s >> 4, tq = *s & 15;
                s++;
                if (tq > 3 || s + (pq ? 128 : 64) > se) return -1;
                for (int i = 0; i < 64; i++) quant[tq][kZigzagNat[i]] = pq ? rd16(s + 2 * i) : s[i];
                s += pq ? 128 : 64;
                quant_set[tq] = true;
            }
        } else if (m == 0xC4) {                            // DHT
            while (s < se) {
                const int tc = *s >> 4, th = *s & 15;
                s++;
                if (tc > 1 || th > 3 || s + 16 > se) return -1;
                HuffTab& t = tc ? ac[th] : dc[th];
                int n = 0;
                for (int l = 1; l <= 16; l++) { t.bits[l] = s[l - 1]; n += s[l - 1]; }
                s += 16;
                if (n > 256 || s + n > se) return -1;
                memcpy(t.vals, s, n);
                s += n;
                if (!t.build()) return -1;
            }
        } else if (m == 0xC0 || m == 0xC1 || m == 0xC2) {  // SOF0 / SOF1 sequential, SOF2 progressive (Huffman)
            if (have_sof) return -1;
            if (len < 8 || s[0] != 8) return -2;
            H = rd16(s + 1); W = rd16(s + 3);
            const int nc = s[5];
            if (W <= 0 || H <= 0) return -1;
            if ((nc != 1 && nc != 3) || len < 8 + 3 * nc) return -2;
            comps.resize(nc);
            for (int i = 0; i < nc; i++) {
                comps[i].id = s[6 + 3 * i]; comps[i].h = s[7 + 3 * i] >> 4; comps[i].v = s[7 + 3 * i] & 15; comps[i].tq = s[8 + 3 * i];
                if (comps[i].tq > 3 || comps[i].h < 1 || comps[i].v < 1) return -1;
            }
            if (nc == 1) { comps[0].h = comps[0].v = 1; }
            for (auto& c : comps) { hmax = c.h > hmax ? c.h : hmax; vmax = c.v > vmax ? c.v : vmax; }
            if (nc == 3) {
                const Comp& y = comps[0];
                if (comps[1].h != 1 || comps[1].v != 1 || comps[2].h != 1 || comps[2].v != 1) return -2;
                if (!((y.h == 1 && y.v == 1) || (y.h == 2 && y.v == 1) || (y.h == 2 && y.v == 2))) return -2;
            }
            progressive = m == 0xC2;
            have_sof = true;
            if (w) *w = W;
            if (h) *h = H;
            if (!bgr && !co) return 0;
            if (bgr && cap < (long long)W * H * 3) return -1;
            if (co) {   // the same geometry as below, written into the header
                pe_jpeg_coef_header& hd = co->hdr;
                memset(&hd, 0, sizeof hd);
                hd.magic = PE_JPEG_COEF_MAGIC; hd.width = W; hd.height = H; hd.num_comps = nc;
                for (int i = 0; i < nc; i++) { hd.comp[i].h = comps[i].h; hd.comp[i].v = comps[i].v; }
                if (!pe_jpeg::coef_layout(hd)) return -2;
                if (!so) {   // (a scan image's size is known only after the whole file)
                    if (!co->buf) return 0;
                    if (co->cap < hd.total_bytes) return -1;
                }
            }
            mcux = (W + 8 * hmax - 1) / (8 * hmax); mcuy = (H + 8 * vmax - 1) / (8 * vmax);
            for (auto& c : comps) {
                c.bw = mcux * c.h; c.bh = mcuy * c.v;
                c.pw = c.bw * 8; c.ph = c.bh * 8;
                c.dw = (W * c.h + hmax - 1) / hmax; c.dh = (H * c.v + vmax - 1) / vmax;
                c.nbw = (c.dw + 7) / 8; c.nbh = (c.dh + 7) / 8;
            }
        } else if ((m >= 0xC3 && m <= 0xCF) && m != 0xC4 && m != 0xC8 && m != 0xCC) {
            return -2;                                     // lossless, arithmetic, hierarchical
        } else if (m == 0xDD) {                            // DRI
            if (len < 4) return -1;
            restart = rd16(s);
        } else if (m == 0xDA) {                            // SOS: decode one scan into the coefficient arrays
            if (!have_sof || len < 3) return -1;          // a truncated segment (length field only) has no payload byte to read
            const int ns = s[0];
            if (ns < 1 || ns > (int)comps.size() || len < 6 + 2 * ns) return -1;
            std::vector<Comp*> sc;
            for (int i = 0; i < ns; i++) {
                const int cid = s[1 + 2 * i];
                Comp* c = nullptr;
                for (auto& cc : comps) if (cc.id == cid) c = &cc;
                if (!c) return -1;
                c->td = s[2 + 2 * i] >> 4; c->ta = s[2 + 2 * i] & 15;
                if (c->td > 3 || c->ta > 3) return -1;
                if (!c->q_latched) {   // libjpeg latches a component's table at its first scan
                    if (!quant_set[c->tq]) return -1;
                    memcpy(c->q, quant[c->tq], sizeof c->q);
                    c->q_latched = true;
                }
                sc.push_back(c);
            }
            if (!any_scan) {
                // Motion-JPEG frames (AVI 'MJPG', cameras) usually leave the DHT segment out when the tables are the Annex K ones:
                // like libjpeg(-turbo)'s jinit_huff_decoder -> std_huff_tables, slots 0 (luminance) and 1 (chrominance) that are
                // still undefined when decoding starts get the standard tables; a later DHT replaces them as usual.
                auto load_std = [](HuffTab& t, const uint8_t* bits, const uint8_t* vals, int nvals) {
                    if (t.set) return;
                    for (int l = 1; l <= 16; l++) t.bits[l] = bits[l - 1];
                    memcpy(t.vals, vals, (size_t)nvals);
                    t.build();
                };
                load_std(dc[0], pe_jpeg::kDcLumBits, pe_jpeg::kDcVal, 12);
                load_std(dc[1], pe_jpeg::kDcChrBits, pe_jpeg::kDcVal, 12);
                load_std(ac[0], pe_jpeg::kAcLumBits, pe_jpeg::kAcLumVal, 162);
                load_std(ac[1], pe_jpeg::kAcChrBits, pe_jpeg::kAcChrVal, 162);
            }
            ScanParams sp;
            sp.Ss = s[1 + 2 * ns]; sp.Se = s[2 + 2 * ns]; sp.Ah = s[3 + 2 * ns] >> 4; sp.Al = s[3 + 2 * ns] & 15;
            sp.progressive = progressive;
            if (progressive) {
                if (sp.Ss > sp.Se || sp.Se > 63 || sp.Al > 13 || (sp.Ss == 0 && sp.Se != 0) || (sp.Ss > 0 && ns != 1)) return -1;
            } else {
                sp.Ss = 0; sp.Se = 63; sp.Ah = sp.Al = 0;
            }
            for (Comp* c : sc) {
                const bool need_dc = !progressive || sp.Ss == 0, need_ac = !progressive || sp.Ss > 0;
                if ((need_dc && sp.Ah == 0 && !dc[c->td].set) || (need_ac && !ac[c->ta].set)) return -1;
                c->pred = 0;
            }
            if (fast_done) return so ? -3 : decode_impl(data, size, w, h, bgr, cap, false, co);   // more scans after a complete one: the general route decides
            // interleaved: MCUs of h x v blocks per component over the padded grid; single component: its real blocks
            const int units_x = ns > 1 ? mcux : sc[0]->nbw, units_y = ns > 1 ? mcuy : sc[0]->nbh;
            bool distinct = true;   // a (corrupt) scan that names a component twice accumulates coefficients: general route only
            for (int i = 0; i < ns; i++)
                for (int j = i + 1; j < ns; j++) distinct = distinct && sc[i] != sc[j];
            const bool fast_scan = !progressive && !any_scan && distinct && ns == (int)comps.size();
            if (so && !fast_scan) return -3;   // valid so far, but not one interleaved sequential scan: the host entropy stage
            if (so) {
                // ---- scan output: record the scan instead of decoding it.  Segment boundaries are a property of the bytes:
                //  * the sequential reader never consumes a marker (it stops at the first FF xx with xx != 00 and feeds zero bits), and
                //    the restart search starts where the reader stopped, which is at or after the segment's start but never past the
                //    first such FF.  So segment k begins right after the first FF D0..D7 pair at or after the start of segment k-1;
                //  * a segment's data ends at the first FF xx (xx != 00) at or after its start - an FF as the file's last byte too;
                //  * no RST pair where one is due: -1, as on both decoding routes.
                // The marker loop then continues from the last segment's start: the bytes from there to where the reader would have
                // stopped are data bytes and FF 00 pairs, which the loop skips, so it reaches the same next marker.
                pe_jpeg_scan_header& sh = so->hdr;
                const long long mcus = (long long)mcux * mcuy;
                const long long nseg = restart ? (mcus + restart - 1) / restart : 1;
                sh.magic = PE_JPEG_SCAN_MAGIC;
                sh.num_scan_comps = ns;
                for (int i = 0; i < ns; i++) {
                    sh.scan_comp[i] = (int32_t)(sc[i] - comps.data());
                    sh.dc_table[i] = sc[i]->td;
                    sh.ac_table[i] = sc[i]->ta;
                }
                sh.restart_interval = restart;
                sh.mcux = mcux; sh.mcuy = mcuy;
                sh.num_segments = (int32_t)nseg;
                for (int t = 0; t < 4; t++) {
                    if (dc[t].set) { memcpy(sh.dc_bits[t], dc[t].bits + 1, 16); memcpy(sh.dc_vals[t], dc[t].vals, 256); }
                    if (ac[t].set) { memcpy(sh.ac_bits[t], ac[t].bits + 1, 16); memcpy(sh.ac_vals[t], ac[t].vals, 256); }
                }
                const uint8_t* start = p + len;
                so->data = start;
                so->seg.assign((size_t)(2 * nseg), 0);
                const uint8_t* q = start;
                for (long long k = 0; k < nseg; k++) {
                    if (k > 0) {
                        while (q + 1 < end && !(q[0] == 0xFF && q[1] >= 0xD0 && q[1] <= 0xD7)) q++;
                        if (q + 1 >= end) return -1;
                        q += 2;
                    }
                    const uint8_t* e = q;
                    while (e < end && !(e[0] == 0xFF && (e + 1 >= end || e[1] != 0))) e += e[0] == 0xFF ? 2 : 1;
                    so->seg[2 * k] = q - start;
                    so->seg[2 * k + 1] = e - q;
                }
                sh.data_bytes = so->seg[2 * nseg - 2] + so->seg[2 * nseg - 1];
                fast_done = any_scan = true;
                p = q;
                continue;
            }
            if (allow_fast && fast_scan) {
                // ---- fast route: one interleaved sequential scan, every block transformed as it leaves the entropy decoder
                if (!co)
                    for (auto& c : comps) c.plane.resize((size_t)c.pw * c.ph);
                FastBits fb;
                fb.p = p + len; fb.end = end;
                int until = restart;
                alignas(32) short blk[64];
                bool ok = true;
                for (int uy = 0; uy < units_y && ok; uy++)
                    for (int ux = 0; ux < units_x && ok; ux++) {
                        if (restart && until == 0) {
                            const uint8_t* q = fb.p;
                            while (q + 1 < end && !(q[0] == 0xFF && q[1] >= 0xD0 && q[1] <= 0xD7)) q++;
                            if (q + 1 >= end) { ok = false; break; }
                            fb.p = q + 2;
                            fb.reset();
                            for (Comp* c : sc) c->pred = 0;
                            until = restart;
                        }
                        for (Comp* c : sc) {
                            const int nbx = ns > 1 ? c->h : 1, nby = ns > 1 ? c->v : 1;
                            for (int by = 0; by < nby && ok; by++)
                                for (int bx = 0; bx < nbx && ok; bx++) {
                                    const int col = ux * nbx + bx, rowb = uy * nby + by;
                                    // coefficient output: the block goes straight into the caller's buffer, untransformed
                                    short* dst = co ? co->coef((int)(c - comps.data())) + ((size_t)rowb * c->bw + col) * 64 : blk;
                                    memset(dst, 0, 64 * sizeof(short));
                                    bool dc_only = false;
                                    ok = decode_block_seq(fb, c->pred, dc[c->td], ac[c->ta], dst, dc_only);
                                    if (ok && !co) idct_block(blk, c->q, c->plane.data() + (size_t)rowb * 8 * c->pw + (size_t)col * 8, c->pw, dc_only);
                                }
                        }
                        if (restart) until--;
                    }
                if (!ok) return decode_impl(data, size, w, h, bgr, cap, false, co);   // the general route defines the outcome of broken streams
                fast_done = any_scan = true;
                p = fb.p;
                continue;
            }
            for (Comp* c : sc)
                if (c->coef.empty()) c->coef.assign((size_t)c->bw * c->bh * 64, 0);
            BitReader br;
            br.p = p + len; br.end = end;
            int eobrun = 0, until_restart = restart;
            bool ok = true;
            for (int uy = 0; uy < units_y && ok; uy++)
                for (int ux = 0; ux < units_x && ok; ux++) {
                    if (restart && until_restart == 0) {   // RSTn: resynchronise on the marker, reset predictions and EOB run
                        const uint8_t* q = br.p;
                        while (q + 1 < end && !(q[0] == 0xFF && q[1] >= 0xD0 && q[1] <= 0xD7)) q++;
                        if (q + 1 >= end) { ok = false; break; }
                        br.p = q + 2;
                        br.reset();
                        for (Comp* c : sc) c->pred = 0;
                        eobrun = 0;
                        until_restart = restart;
                    }
                    for (Comp* c : sc) {
                        const int nbx = ns > 1 ? c->h : 1, nby = ns > 1 ? c->v : 1;
                        for (int by = 0; by < nby && ok; by++)
                            for (int bx = 0; bx < nbx && ok; bx++) {
                                const int col = ux * nbx + bx, rowb = uy * nby + by;
                                ok = decode_block(br, *c, dc, ac, &c->coef[((size_t)rowb * c->bw + col) * 64], sp, eobrun);
                            }
                    }
                    if (restart) until_restart--;
                }
            if (!ok) return -1;
            any_scan = true;
            p = br.p;       // the reader stops at the next marker
            continue;
        }
        p += len;
    }
    if (!have_sof) return -1;
    if (!bgr && !co) return 0;
    if (!any_scan) return -1;
    if (co) {   // coefficient output: what the loop below would transform, and the tables it would use
        for (size_t k = 0; k < comps.size(); k++) {
            Comp& c = comps[k];
            if (!c.q_latched) { if (!quant_set[c.tq]) return -1; memcpy(c.q, quant[c.tq], sizeof c.q); }
            memcpy(co->hdr.comp[k].quant, c.q, sizeof c.q);
            if (fast_done) continue;   // already stored by the fast route
            const size_t n = (size_t)c.bw * c.bh * 64;
            if (c.coef.empty()) memset(co->coef((int)k), 0, n * sizeof(short));
            else memcpy(co->coef((int)k), c.coef.data(), n * sizeof(short));
        }
        if (so) {
            pe_jpeg_scan_header& sh = so->hdr;
            sh.coef = co->hdr;
            sh.seg_table_offset = (int64_t)sizeof sh;
            sh.data_offset = sh.seg_table_offset + (int64_t)(so->seg.size() * sizeof(int64_t));
            sh.total_bytes = sh.data_offset + sh.data_bytes;
            return 0;
        }
        memcpy(co->buf, &co->hdr, sizeof co->hdr);
        return 0;
    }
    for (auto& c : comps) {   // inverse DCT of every block (a component without any scan decodes as mid-grey, like libjpeg)
        if (fast_done) break;   // already transformed
        if (!c.q_latched) { if (!quant_set[c.tq]) return -1; memcpy(c.q, quant[c.tq], sizeof c.q); }
        if (c.coef.empty()) c.coef.assign((size_t)c.bw * c.bh * 64, 0);
        c.plane.assign((size_t)c.pw * c.ph, 0);
        for (int by = 0; by < c.bh; by++)
            for (int bx = 0; bx < c.bw; bx++)
                idct_block(&c.coef[((size_t)by * c.bw + bx) * 64], c.q, c.plane.data() + (size_t)by * 8 * c.pw + (size_t)bx * 8, c.pw, false);
    }
    reconstruct(comps, hmax, vmax, W, H, bgr);
    return 0;
}

// planes (every block transformed) -> BGR: grey replicated, or upsampled chroma + colour conversion
static void reconstruct(std::vector<Comp>& comps, int hmax, int vmax, int W, int H, uint8_t* bgr) {
    const int nc = (int)comps.size();
    if (nc == 1) {
        const Comp& c = comps[0];
        for (int y = 0; y < H; y++)
            for (int x = 0; x < W; x++) {
                const uint8_t g = c.plane[(size_t)y * c.pw + x];
                uint8_t* o = bgr + ((size_t)y * W + x) * 3;
                o[0] = o[1] = o[2] = g;
            }
        return;
    }
    output_rows(comps, hmax, vmax, W, H, bgr);
}
}  // namespace

extern "C" long long pe_jpeg_read_coefs(const uint8_t* data, long long size, void* buf, long long cap) {
    const char* env = getenv("PE_JPEG_FAST");
    CoefOut co;
    co.buf = (uint8_t*)buf;
    co.cap = cap;
    memset(&co.hdr, 0, sizeof co.hdr);
    const int rc = decode_impl(data, size, nullptr, nullptr, nullptr, 0, !(env && env[0] == '0'), &co);
    return rc ? rc : co.hdr.total_bytes;
}

extern "C" long long pe_jpeg_read_scan(const uint8_t* data, long long size, void* buf, long long cap) {
    CoefOut co;
    co.buf = nullptr;
    co.cap = 0;
    memset(&co.hdr, 0, sizeof co.hdr);
    ScanOut so;
    memset(&so.hdr, 0, sizeof so.hdr);
    const int rc = decode_impl(data, size, nullptr, nullptr, nullptr, 0, true, &co, &so);
    if (rc) return rc;
    const pe_jpeg_scan_header& sh = so.hdr;
    if (!buf) return sh.total_bytes;
    if (cap < sh.total_bytes) return -1;
    uint8_t* out = (uint8_t*)buf;
    memcpy(out, &sh, sizeof sh);
    memcpy(out + sh.seg_table_offset, so.seg.data(), so.seg.size() * sizeof(int64_t));
    memcpy(out + sh.data_offset, so.data, (size_t)sh.data_bytes);
    return sh.total_bytes;
}

// The GPU entropy decoder (jpeg_entropy.cu) on the host: the same decode (jpeg_entropy.cuh), with loops over the threads of a CTA
// in place of threads, the CTAs in order, and the rounds of the synchronisation exactly as the kernel runs them.
extern "C" long long pe_jpeg_scan_to_coefs_host(const void* scan, void* coefs, long long cap, int subseq_bits) {
    using namespace pe_jpeg;
    if (!scan || !coefs || subseq_bits < 8) return -1;
    const pe_jpeg_scan_header& h = *(const pe_jpeg_scan_header*)scan;
    const long long S = subseq_bits;
    long long nsub = 0;
    if (!scan_header_valid(h, S, &nsub) || cap < h.coef.total_bytes) return -1;
    std::vector<HuffDec> tabs(8);
    for (int t = 0; t < 8; t++) {
        HuffDec& d = tabs[t];
        huff_canon(t < 4 ? h.dc_bits[t] : h.ac_bits[t - 4], d);
        memcpy(d.vals, t < 4 ? h.dc_vals[t] : h.ac_vals[t - 4], 256);
        for (int i = 0; i < (1 << LOOK_BITS); i++) d.look[i] = huff_look_entry(d, i);
    }
    const uint8_t* base = (const uint8_t*)scan;
    ScanCtx c;
    scan_slots(h, c);
    c.data = base + h.data_offset;
    c.seg = (const int64_t*)(base + h.seg_table_offset);
    for (int k = 0; k < h.num_scan_comps; k++) { c.dc[k] = &tabs[h.dc_table[k]]; c.ac[k] = &tabs[4 + h.ac_table[k]]; }
    c.zigzag = kZigzagNat;
    uint8_t* out = (uint8_t*)coefs;
    memset(out, 0, (size_t)h.coef.total_bytes);
    memcpy(out, &h.coef, sizeof h.coef);
    std::vector<long long> first_sub((size_t)c.num_segments + 1, 0);
    for (int s = 0; s < c.num_segments; s++) first_sub[s + 1] = first_sub[s] + subseq_count(c.seg[2 * s + 1], S);
    const int T = SYNC_THREADS;
    long long err_mcu = -1;
    State carry_state = 0;
    long long carry_block = 0;
    std::vector<int> seg(T);
    std::vector<char> head(T), last(T);
    std::vector<long long> stop(T), cnt(T), fb(T);
    std::vector<State> start(T), ex(T), ns(T);
    int s = 0;
    for (long long g0 = 0; g0 < nsub; g0 += T) {
        auto run = [&](int t) {
            ex[t] = start[t];
            const int64_t* sg = c.seg + 2 * seg[t];
            cnt[t] = decode_run(c, c.data + sg[0], sg[1], &ex[t], stop[t], 1LL << 62, [](long long, int, int) {});
        };
        for (int t = 0; t < T; t++) {
            const long long g = g0 + t;
            head[t] = 1; last[t] = 1; seg[t] = 0; stop[t] = 0;
            if (g >= nsub) { start[t] = ex[t] = 0; cnt[t] = 0; continue; }
            while (first_sub[s + 1] <= g) s++;
            const long long j = g - first_sub[s], n = c.seg[2 * s + 1];
            seg[t] = s;
            head[t] = j == 0;
            last[t] = g == first_sub[s + 1] - 1;
            stop[t] = last[t] ? n * 8 : (j + 1) * S;
            start[t] = head[t] ? 0 : pack_state(canonical_pos(c.data + c.seg[2 * s], n, j * S), 0, 0);
            run(t);
        }
        auto settle = [&]() {   // rounds: every thread takes its predecessor's exit of the previous round
            for (;;) {
                bool any = false;
                for (int t = 0; t < T; t++) ns[t] = (!head[t] && t > 0) ? ex[t - 1] : start[t];
                for (int t = 0; t < T; t++)
                    if (ns[t] != start[t]) { start[t] = ns[t]; run(t); any = true; }
                if (!any) break;
            }
        };
        settle();
        if (!head[0] && g0 > 0 && carry_state != start[0]) {   // the previous CTA's final exit state
            start[0] = carry_state;
            run(0);
            settle();
        }
        for (int t = 0; t < T; t++) fb[t] = head[t] ? 0 : (t == 0 ? carry_block : fb[t - 1] + cnt[t - 1]);
        carry_state = ex[T - 1];
        carry_block = fb[T - 1] + cnt[T - 1];
        for (int t = 0; t < T && g0 + t < nsub; t++) {
            const long long limit = segment_mcus(c, seg[t]) * c.nslots - fb[t];
            if (limit <= 0) continue;
            const int64_t* sg = c.seg + 2 * seg[t];
            State st = start[t];
            const int sgi = seg[t];
            const long long f = fb[t];
            decode_run(c, c.data + sg[0], sg[1], &st, last[t] ? (1LL << 62) : stop[t], limit, [&](long long b, int zz, int v) {
                long long mcu = 0;
                const long long off = block_offset(h, c, sgi, f + b, &mcu);
                if (zz == -2) { if (err_mcu < 0 || mcu < err_mcu) err_mcu = mcu; return; }
                ((short*)(out + off))[zz < 0 ? 0 : c.zigzag[zz]] = (short)v;
            });
        }
    }
    // DC: per component a prefix sum of the differences that restarts with every segment, unsigned 32-bit as the host's pred
    for (int sg = 0; sg < c.num_segments; sg++) {
        unsigned pred[3] = {0, 0, 0};
        const long long nb = segment_mcus(c, sg) * c.nslots;
        for (long long b = 0; b < nb; b++) {
            short* blk = (short*)(out + block_offset(h, c, sg, b, nullptr));
            unsigned& pr = pred[c.slot_comp[b % c.nslots]];
            pr += (unsigned)(int)blk[0];
            blk[0] = (short)pr;
        }
    }
    return err_mcu >= 0 ? -4 : h.coef.total_bytes;
}

extern "C" int pe_jpeg_coefs_to_bgr(const void* coefs, uint8_t* bgr, long long cap) {
    if (!coefs || !bgr) return -1;
    pe_jpeg_coef_header hd;
    memcpy(&hd, coefs, sizeof hd);
    if (!pe_jpeg::coef_header_valid(hd) || cap < (long long)hd.width * hd.height * 3) return -1;
    std::vector<Comp> comps(hd.num_comps);
    for (int k = 0; k < hd.num_comps; k++) {
        Comp& c = comps[k];
        const pe_jpeg_coef_comp& h = hd.comp[k];
        c.h = h.h; c.v = h.v; c.bw = h.bw; c.bh = h.bh; c.dw = h.dw; c.dh = h.dh;
        c.pw = c.bw * 8; c.ph = c.bh * 8;
        memcpy(c.q, h.quant, sizeof c.q);
        c.plane.assign((size_t)c.pw * c.ph, 0);
        const short* coef = (const short*)((const uint8_t*)coefs + h.offset);
        for (int by = 0; by < c.bh; by++)
            for (int bx = 0; bx < c.bw; bx++)
                idct_block(coef + ((size_t)by * c.bw + bx) * 64, c.q, c.plane.data() + (size_t)by * 8 * c.pw + (size_t)bx * 8, c.pw, false);
    }
    reconstruct(comps, hd.hmax, hd.vmax, hd.width, hd.height, bgr);
    return 0;
}

