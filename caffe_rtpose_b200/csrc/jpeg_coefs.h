// Layout of the coefficient image of pe_jpeg_read_coefs (poseengine.h): written by the host entropy stage (jpeg_dec.cpp), read by
// the host reference reconstruction and by the GPU kernels (jpeg_gpu.cu).  Everything that indexes with the header's numbers checks
// it here first, so that a malformed buffer is an error instead of an out-of-bounds access.
#pragma once
#include <stdint.h>

#include "../../include/poseengine.h"

namespace pe_jpeg {

static_assert(sizeof(pe_jpeg_coef_comp) == 160 && sizeof(pe_jpeg_coef_header) == 512, "pe_jpeg_coef_header layout");

// the geometry pe_decode_jpeg derives from the frame header (width, height, sampling factors): fills bw, bh, dw, dh, offset of
// every component and total_bytes.  false: sampling outside what the decoder accepts.
inline bool coef_layout(pe_jpeg_coef_header& h) {
    if (h.width <= 0 || h.height <= 0 || (h.num_comps != 1 && h.num_comps != 3)) return false;
    int hmax = 1, vmax = 1;
    for (int i = 0; i < h.num_comps; i++) {
        const pe_jpeg_coef_comp& c = h.comp[i];
        if (c.h < 1 || c.v < 1) return false;
        hmax = c.h > hmax ? c.h : hmax;
        vmax = c.v > vmax ? c.v : vmax;
    }
    if (h.num_comps == 1 && (h.comp[0].h != 1 || h.comp[0].v != 1)) return false;
    if (h.num_comps == 3) {
        const pe_jpeg_coef_comp& y = h.comp[0];
        if (h.comp[1].h != 1 || h.comp[1].v != 1 || h.comp[2].h != 1 || h.comp[2].v != 1) return false;
        if (!((y.h == 1 && y.v == 1) || (y.h == 2 && y.v == 1) || (y.h == 2 && y.v == 2))) return false;
    }
    h.hmax = hmax;
    h.vmax = vmax;
    const long long mcux = (h.width + 8LL * hmax - 1) / (8 * hmax), mcuy = (h.height + 8LL * vmax - 1) / (8 * vmax);
    long long off = (long long)sizeof(pe_jpeg_coef_header);
    for (int i = 0; i < h.num_comps; i++) {
        pe_jpeg_coef_comp& c = h.comp[i];
        c.bw = (int32_t)(mcux * c.h);
        c.bh = (int32_t)(mcuy * c.v);
        c.dw = (int32_t)(((long long)h.width * c.h + hmax - 1) / hmax);
        c.dh = (int32_t)(((long long)h.height * c.v + vmax - 1) / vmax);
        c.offset = off;
        off += (long long)c.bw * c.bh * 64 * (long long)sizeof(int16_t);
    }
    h.total_bytes = off;
    return true;
}

// a header as pe_jpeg_read_coefs writes it: every derived field equals what coef_layout computes from the primary ones
inline bool coef_header_valid(const pe_jpeg_coef_header& h) {
    if (h.magic != PE_JPEG_COEF_MAGIC) return false;
    pe_jpeg_coef_header g = h;
    if (!coef_layout(g) || g.hmax != h.hmax || g.vmax != h.vmax || g.total_bytes != h.total_bytes) return false;
    for (int i = 0; i < h.num_comps; i++) {
        const pe_jpeg_coef_comp &a = g.comp[i], &b = h.comp[i];
        if (a.bw != b.bw || a.bh != b.bh || a.dw != b.dw || a.dh != b.dh || a.offset != b.offset) return false;
    }
    return true;
}

}  // namespace pe_jpeg
