// The u8 instances of the wgmma / TMA convolution (PE_PREC_S8X1 | PE_PREC_FLAG_U8), in a translation unit of their own so that
// conv_tc.cu, conv_fp8.cu, conv_s8.cu and conv_mixed.cu keep exactly their instances.  The kernel is conv_wg_kernel
// (conv_tc_kernel.cuh).  A layer that reads a u8 activation runs wgmma m64nBNk32 u8 x s8 -> s32 (the s8 rate) into one accumulator
// over the whole K, with S8X1's per-channel epilogue t = __fadd_rn(__fmul_rn(__int2float_rn(acc), f_c), b'_c); a layer that stores
// u8 applies ReLU and cvt.rni.sat.u8.f32.  |acc| <= 255 * 127 * K, which the engine keeps inside s32 by refusing a K above
// U8_ACTIVATIONS.max_k (precision.h).  The instances:
//   <1, u8, u8>:  u8 in, u8 out, and the fp32 maps (the planar store of the same instance);
//   <1, u8, s8>:  u8 in, s8 out (a layer whose output shares a buffer with signed values: conv4_4_CPM);
//   <1, s8, u8>:  s8 in, u8 out (conv1_1, and the first layers of every stage, which read the s8 Concat buffers);
//   <1, u8, f16>: u8 in, fp16 out, and <1, f16, u8>: fp16 in (chunked fp32 sums, one factor per layer), u8 out - the format
//                 boundaries of mixed engines (pe_create_mixed).
#include "conv_tc_kernel.cuh"

namespace pe {

int launch_u8(const TcLayer& l, const TcArgs& a, dim3 grid, cudaStream_t st, int bmap, int bn) {
    const PlaneElem in = l.d.fmt.elem, out = l.d.out_elem;
    if (l.d.fmt.planes != 1) return -1;
    if (in == ELEM_U8 && out == ELEM_U8) return launch_widths<1, ELEM_U8, ELEM_U8>(l, a, grid, st, bmap, bn);
    if (in == ELEM_U8 && out == ELEM_S8) return launch_widths<1, ELEM_U8, ELEM_S8>(l, a, grid, st, bmap, bn);
    if (in == ELEM_S8 && out == ELEM_U8) return launch_widths<1, ELEM_S8, ELEM_U8>(l, a, grid, st, bmap, bn);
    if (in == ELEM_U8 && out == ELEM_F16) return launch_widths<1, ELEM_U8, ELEM_F16>(l, a, grid, st, bmap, bn);
    if (in == ELEM_F16 && out == ELEM_U8) return launch_widths<1, ELEM_F16, ELEM_U8>(l, a, grid, st, bmap, bn);
    return -1;   // u8 next to e4m3: no instance
}

}  // namespace pe
