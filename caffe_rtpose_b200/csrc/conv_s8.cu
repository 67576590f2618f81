// The s8 instances of the wgmma / TMA convolution (PE_PREC_S8X1), in a translation unit of their own so that conv_tc.cu and
// conv_fp8.cu keep exactly their instances.  The kernel is conv_wg_kernel (conv_tc_kernel.cuh) at ELEM = OUT = s8: 128-channel
// K blocks in the same 128-byte swizzle rows as e4m3, wgmma m64nBNk32 s8 x s8 -> s32 into one accumulator over the whole K (the
// sums are exact, so nothing is chunked), and the per-channel epilogue
//   t = __fadd_rn(__fmul_rn(__int2float_rn(acc), f_c), b'_c),  ReLU,  cvt.rni.sat.s8.f32
// (the fp32 maps store t).  Every layer, conv1_1 included, reads s8: the im2col'ed net input is p - 128 at scale 2^8.
// |acc| <= 128 * 127 * K, which the engine keeps inside s32 by refusing a K above Precision::max_k (precision.h).
#include "conv_tc_kernel.cuh"

namespace pe {

int launch_s8(const TcLayer& l, const TcArgs& a, dim3 grid, cudaStream_t st, int bmap, int bn) {
    return launch_widths<1, ELEM_S8, ELEM_S8>(l, a, grid, st, bmap, bn);
}

}  // namespace pe
