// Entropy decoding of a scan image (pe_jpeg_read_scan, poseengine.h) into the coefficient image of pe_jpeg_read_coefs: the pieces
// shared by the CUDA kernels (jpeg_entropy.cu) and the host run of the same algorithm (pe_jpeg_scan_to_coefs_host, jpeg_dec.cpp),
// so that the algorithm can be checked and fuzzed without a GPU.
//
// Self-synchronising parallel Huffman decoding (Weissenberger & Schmidt, "Massively Parallel Huffman Decoding on GPUs", ICPP 2018):
// every restart segment is cut into subsequences of S bits; a thread decodes its subsequence from an assumed state and records the
// state where it crosses into the next one.  The decoder state is (bit position, block slot in the MCU, coefficient index in the
// block).  A segment's first subsequence starts from the true state; every other thread re-decodes from its predecessor's exit state
// until its own exit no longer changes - by induction the fixed point is the sequential decode, and a stream that never synchronises
// degenerates to sequential decoding.  Equal states decode identically from there on (the tables are fixed and DC values are
// differences), which is why comparing exit states suffices.
//
// Bit positions are raw: 8 * byte index in the segment's stuffed bytes + bit.  The reader skips the 00 after every FF, so a decoder
// position never lies inside a stuffing byte, and all threads compare positions in the same coordinates.  Past the segment's last
// byte the reader feeds zero bits, as the host reader does after a marker.
#pragma once
#include <stdint.h>

#include "jpeg_coefs.h"

#ifdef __CUDACC__
#define PE_HD __host__ __device__ __forceinline__
#else
#define PE_HD inline
#endif

namespace pe_jpeg {

static_assert(sizeof(pe_jpeg_scan_header) == 2784, "pe_jpeg_scan_header layout");

constexpr int LOOK_BITS = 10;          // lookahead of the Huffman decoder, as the host's HuffTab::LOOK
constexpr int SUBSEQ_BITS = 1024;      // default subsequence length S
constexpr int SYNC_THREADS = 128;      // subsequences per CTA (the host run groups them the same way)
constexpr int MAX_SLOTS = 6;           // blocks per MCU: 4 luma + 2 chroma at 4:2:0

// A Huffman table as the decoder uses it (the host HuffTab's derived tables)
struct HuffDec {
    uint16_t look[1 << LOOK_BITS];     // code length << 8 | symbol; 0 = no code of <= 10 bits
    int32_t mincode[17], maxcode[17], valptr[17];
    uint8_t vals[256];
};

// T.81 C.2 canonical codes from BITS (bits[l - 1] codes of length l); false when the lengths over-subscribe the code space
PE_HD bool huff_canon(const uint8_t* bits, HuffDec& t) {
    int code = 0, k = 0;
    for (int l = 1; l <= 16; l++) {
        t.valptr[l] = k;
        t.mincode[l] = code;
        code += bits[l - 1];
        if (code > (1 << l)) return false;
        k += bits[l - 1];
        t.maxcode[l] = bits[l - 1] ? code - 1 : -1;
        code <<= 1;
    }
    return true;
}
// lookahead entry i (the prefix code of <= 10 bits that i starts with); after huff_canon and with vals filled
PE_HD uint16_t huff_look_entry(const HuffDec& t, int i) {
    for (int l = 1; l <= LOOK_BITS; l++) {
        const int c = i >> (LOOK_BITS - l);
        if (t.maxcode[l] >= 0 && c >= t.mincode[l] && c <= t.maxcode[l]) return (uint16_t)(l << 8 | t.vals[t.valptr[l] + c - t.mincode[l]]);
    }
    return 0;
}
// jpeg_dec.cpp huff_decode on the 32 bits at the decoder position: symbol, and its code length in *len.  No match: 16 bits, symbol 0.
PE_HD int huff_decode(const HuffDec& t, uint32_t bits, int* len) {
    const uint16_t e = t.look[bits >> (32 - LOOK_BITS)];
    if (e) { *len = e >> 8; return e & 255; }
    const int code = (int)(bits >> 16);
    for (int l = LOOK_BITS + 1; l <= 16; l++) {
        const int c = code >> (16 - l);
        if (t.maxcode[l] >= 0 && c <= t.maxcode[l] && c >= t.mincode[l]) { *len = l; return t.vals[t.valptr[l] + c - t.mincode[l]]; }
    }
    *len = 16;
    return 0;
}
PE_HD int extend(int v, int s) { return v < (1 << (s - 1)) ? v - (1 << s) + 1 : v; }
PE_HD int popcount(unsigned x) {
#ifdef __CUDA_ARCH__
    return __popc(x);
#else
    return __builtin_popcount(x);
#endif
}

// Decoder state packed into one word, so that "no longer changes" is one comparison: raw bit position << 16 | slot << 8 | k
// (k = index of the next coefficient in zigzag order, 0 = the DC difference is next)
typedef unsigned long long State;
PE_HD State pack_state(long long pos, int slot, int k) { return (State)pos << 16 | (State)slot << 8 | (State)k; }
PE_HD long long state_pos(State s) { return (long long)(s >> 16); }

// A position that lands on a stuffing byte (the 00 after an FF) belongs to the next byte: an assumed start is put there
PE_HD long long canonical_pos(const uint8_t* d, long long n, long long pos) {
    const long long b = pos >> 3;
    if (b >= 1 && b < n && d[b] == 0 && d[b - 1] == 0xFF) return (b + 1) * 8;
    return pos;
}

// Everything the decoder needs about one frame's scan
struct ScanCtx {
    const uint8_t* data;               // entropy-coded bytes (data_offset)
    const int64_t* seg;                // segment table: offset, length
    int num_segments, restart, mcux, nslots;
    long long total_mcus;
    uint8_t slot_sc[MAX_SLOTS];        // scan component of each block slot
    uint8_t slot_comp[MAX_SLOTS];      // its SOF index
    uint8_t slot_bx[MAX_SLOTS], slot_by[MAX_SLOTS];   // block position inside the MCU
    const HuffDec* dc[3];              // tables of the scan's components
    const HuffDec* ac[3];
    const uint8_t* zigzag;             // zigzag index -> natural index
};

// MCU layout of the interleaved scan: the components in SOS order, h x v blocks each (1 x 1 for a grey image)
PE_HD void scan_slots(const pe_jpeg_scan_header& h, ScanCtx& c) {
    int n = 0;
    for (int k = 0; k < h.num_scan_comps; k++) {
        const int comp = h.scan_comp[k];
        const int hh = h.num_scan_comps > 1 ? h.coef.comp[comp].h : 1, vv = h.num_scan_comps > 1 ? h.coef.comp[comp].v : 1;
        for (int by = 0; by < vv; by++)
            for (int bx = 0; bx < hh; bx++) {
                c.slot_sc[n] = (uint8_t)k; c.slot_comp[n] = (uint8_t)comp; c.slot_bx[n] = (uint8_t)bx; c.slot_by[n] = (uint8_t)by;
                n++;
            }
    }
    c.nslots = n;
    c.restart = h.restart_interval;
    c.mcux = h.mcux;
    c.total_mcus = (long long)h.mcux * h.mcuy;
    c.num_segments = h.num_segments;
}

PE_HD long long segment_mcus(const ScanCtx& c, int s) {
    if (!c.restart) return c.total_mcus;
    const long long left = c.total_mcus - (long long)s * c.restart;
    return left < c.restart ? left : c.restart;
}
PE_HD long long subseq_count(long long bytes, long long S) { const long long n = (bytes * 8 + S - 1) / S; return n > 1 ? n : 1; }

// Byte offset in the coefficient image of block b (decode order) of segment s
PE_HD long long block_offset(const pe_jpeg_scan_header& h, const ScanCtx& c, int s, long long b, long long* mcu_out) {
    const long long mcu = (long long)s * c.restart + b / c.nslots;
    const int slot = (int)(b % c.nslots);
    const long long my = mcu / c.mcux, mx = mcu - my * c.mcux;
    const pe_jpeg_coef_comp& cc = h.coef.comp[c.slot_comp[slot]];
    const int hh = c.nslots > 1 ? cc.h : 1, vv = c.nslots > 1 ? cc.v : 1;
    const long long bx = mx * hh + c.slot_bx[slot], by = my * vv + c.slot_by[slot];
    if (mcu_out) *mcu_out = mcu;
    return cc.offset + (by * cc.bw + bx) * 128;
}

// The per-subsequence decode: decode_block's sequential branch (jpeg_dec.cpp) symbol by symbol from state *st over the segment's
// bytes d[0, n), while the position is below stop_pos and fewer than max_blocks blocks have been completed.  Returns the blocks
// completed; *st becomes the state reached.  emit(block, zigzag_or_-1, value) receives each coefficient (-1 = the DC difference) of
// block `block` (counted from the start state); a DC category above 15 - the host stage's error - is emitted as (block, -2, 0) and
// then decoded as category 0, so that the decode stays a function of the state (the frame is rejected anyway).
template <class Emit>
PE_HD long long decode_run(const ScanCtx& c, const uint8_t* d, long long n, State* st, long long stop_pos, long long max_blocks, Emit&& emit) {
    long long pos = state_pos(*st);
    int slot = (int)((*st >> 8) & 255), k = (int)(*st & 255);
    long long blocks = 0;
    while (pos < stop_pos && blocks < max_blocks) {
        // 5 bytes from the position's byte with the stuffing removed: 40 bits, enough for 7 bits of offset + a code and its value
        const long long b0 = pos >> 3;
        long long b = b0;
        uint64_t w = 0;
        unsigned ff = 0;                       // bit j: byte j was an FF, so a stuffing byte follows it
        for (int j = 0; j < 5; j++) {
            uint32_t v = 0;
            if (b < n) { v = d[b]; if (v == 0xFF) { ff |= 1u << j; b++; } }
            b++;
            w = w << 8 | v;
        }
        const int o = (int)(pos & 7);
        const uint32_t bits = (uint32_t)((w << (24 + o)) >> 32);
        int len = 0;
        bool end = false;
        const int sc = c.slot_sc[slot];
        if (k == 0) {
            int s = huff_decode(*c.dc[sc], bits, &len);
            if (s > 15) { emit(blocks, -2, 0); s = 0; }
            int v = 0;
            if (s) { v = extend((int)((bits << len) >> (32 - s)), s); len += s; }
            emit(blocks, -1, v);
            k = 1;
        } else {
            const int rs = huff_decode(*c.ac[sc], bits, &len);
            const int r = rs >> 4, s = rs & 15;
            if (s == 0) {
                if (r != 15) end = true;
                else if ((k += 16) > 63) end = true;
            } else if ((k += r) > 63) {
                end = true;                    // the block ends before the value bits are read
            } else {
                emit(blocks, k, extend((int)((bits << len) >> (32 - s)), s));
                len += s;
                if (++k > 63) end = true;
            }
        }
        const int t = o + len, j = t >> 3;     // the new position lies in byte j of the window
        pos = (b0 + j + popcount(ff & ((1u << j) - 1))) * 8 + (t & 7);
        if (end) {
            k = 0;
            blocks++;
            if (++slot == c.nslots) slot = 0;
        }
    }
    *st = pack_state(pos, slot, k);
    return blocks;
}

// Host-side check of a scan image before anything indexes with its numbers (the engine and the host run).  S: subsequence bits;
// *subseqs receives the frame's subsequence count.
inline bool scan_header_valid(const pe_jpeg_scan_header& h, long long S, long long* subseqs) {
    if (h.magic != PE_JPEG_SCAN_MAGIC || !coef_header_valid(h.coef) || h.num_scan_comps != h.coef.num_comps) return false;
    bool seen[3] = {false, false, false};
    for (int k = 0; k < h.num_scan_comps; k++) {
        const int c = h.scan_comp[k];
        if (c < 0 || c >= h.coef.num_comps || seen[c]) return false;
        seen[c] = true;
        if (h.dc_table[k] < 0 || h.dc_table[k] > 3 || h.ac_table[k] < 0 || h.ac_table[k] > 3) return false;
    }
    for (int t = 0; t < 8; t++) {
        HuffDec d;
        int sum = 0;
        const uint8_t* bits = t < 4 ? h.dc_bits[t] : h.ac_bits[t - 4];
        for (int l = 0; l < 16; l++) sum += bits[l];
        if (sum > 256 || !huff_canon(bits, d)) return false;
    }
    const int hmax = h.coef.hmax, vmax = h.coef.vmax;
    if (h.mcux != (h.coef.width + 8 * hmax - 1) / (8 * hmax) || h.mcuy != (h.coef.height + 8 * vmax - 1) / (8 * vmax)) return false;
    const long long mcus = (long long)h.mcux * h.mcuy;
    if (h.restart_interval < 0 || h.restart_interval > 65535) return false;
    const long long nseg = h.restart_interval ? (mcus + h.restart_interval - 1) / h.restart_interval : 1;
    if (h.num_segments != nseg || h.seg_table_offset != (long long)sizeof(pe_jpeg_scan_header)) return false;
    if (h.data_offset != h.seg_table_offset + 16 * nseg || h.data_bytes < 0 || h.data_bytes >= (1LL << 40)) return false;
    if (h.total_bytes != h.data_offset + h.data_bytes) return false;
    const int64_t* seg = (const int64_t*)((const uint8_t*)&h + h.seg_table_offset);
    long long subs = 0;
    for (long long s = 0; s < nseg; s++) {
        if (seg[2 * s] < 0 || seg[2 * s + 1] < 0 || seg[2 * s] > h.data_bytes || seg[2 * s + 1] > h.data_bytes - seg[2 * s]) return false;
        subs += subseq_count(seg[2 * s + 1], S);
    }
    if (subs >= (1LL << 31)) return false;
    *subseqs = subs;
    return true;
}

}  // namespace pe_jpeg
