// Packed form of a 2:4-sparse PE_PREC_S8X1 layer (conv_s8_sparse.cu runs it).  Input: the dense s8 plane [cout_pad][K] of
// pack_conv_weights (K order: tap, then engine input channel), in which every aligned group of four weights holds at most two
// non-zeros; cout_pad a multiple of 128, K a multiple of 128.  Output, in this order:
//   values   [cout_pad][K / 2]: per group its two kept weights, the lower index first;
//   metadata [cout_pad / 128][K / 128][2][256] u32: per block of 128 output channels, per 128-channel K step, per k64 half h of
//            the step, one word per consumer thread t = 128 * wg + 32 * warp + lane (the register wgmma.sp reads): row
//            m = 64 * wg + 16 * warp + lane / 4 + 8 * (lane % 2) of the block, K columns 64 * h + 32 * ((lane / 2) % 2) + [0, 32)
//            of the step; group j of those 32 columns in bits [4j, 4j + 4) as i0 | i1 << 2, the indices of its two kept
//            weights, i0 < i1.  A group with fewer than two non-zeros keeps zeros at distinct indices (an empty group: 0, 1).
// Plain C++ without CUDA, so that a CPU test compiles it on its own.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>

namespace pe {

constexpr int SP_BM = 128;           // output channels per CTA tile, and the block of the metadata
constexpr int SP_META_STEP = 2048;   // metadata bytes per (channel block, K step): 2 halves x 256 threads x 4 bytes

inline size_t s8_sparse_bytes(int cout_pad, size_t K) { return (size_t)cout_pad * K / 2 + (size_t)cout_pad / SP_BM * (K / 128) * SP_META_STEP; }

// Indices (i0 < i1) of the weights group g keeps; false when it has more than two non-zeros.
inline bool s8_sparse_pair(const int8_t* g, int& i0, int& i1) {
    int n = 0, idx[4];
    for (int i = 0; i < 4; i++) if (g[i]) idx[n++] = i;
    if (n > 2) return false;
    if (n == 2) { i0 = idx[0]; i1 = idx[1]; }
    else if (n == 1) { i0 = idx[0] == 0 ? 0 : idx[0] == 3 ? 2 : idx[0]; i1 = idx[0] == 0 ? 1 : idx[0] == 3 ? 3 : idx[0] + 1; }
    else { i0 = 0; i1 = 1; }
    return true;
}

// Compresses q into dst (s8_sparse_bytes).  Returns false, dst partly written, when a group has more than two non-zeros.
inline bool s8_sparse_compress(const int8_t* q, int cout_pad, size_t K, uint8_t* dst) {
    int8_t* vals = (int8_t*)dst;
    uint32_t* meta = (uint32_t*)(dst + (size_t)cout_pad * K / 2);
    const size_t steps = K / 128;
    for (int co = 0; co < cout_pad; co++)
        for (size_t g = 0; g < K / 4; g++) {
            int i0 = 0, i1 = 1;
            if (!s8_sparse_pair(q + (size_t)co * K + 4 * g, i0, i1)) return false;
            vals[(size_t)co * (K / 2) + 2 * g] = q[(size_t)co * K + 4 * g + i0];
            vals[(size_t)co * (K / 2) + 2 * g + 1] = q[(size_t)co * K + 4 * g + i1];
        }
    for (int cb = 0; cb < cout_pad / SP_BM; cb++)
        for (size_t s = 0; s < steps; s++)
            for (int h = 0; h < 2; h++)
                for (int t = 0; t < 256; t++) {
                    const int wg = t / 128, warp = (t / 32) % 4, lane = t % 32;
                    const int co = cb * SP_BM + 64 * wg + 16 * warp + lane / 4 + 8 * (lane % 2);
                    const size_t k0 = s * 128 + 64 * h + 32 * ((lane / 2) % 2);
                    uint32_t word = 0;
                    for (int j = 0; j < 8; j++) {
                        int i0 = 0, i1 = 1;
                        s8_sparse_pair(q + (size_t)co * K + k0 + 4 * j, i0, i1);
                        word |= (uint32_t)(i0 | i1 << 2) << (4 * j);
                    }
                    meta[((cb * steps + s) * 2 + h) * 256 + t] = word;
                }
    return true;
}

}  // namespace pe
