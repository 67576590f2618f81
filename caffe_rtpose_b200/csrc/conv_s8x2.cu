// The two-plane s8 instances of the wgmma / TMA convolution (PE_PREC_S8X2), in a translation unit of their own so that conv_tc.cu,
// conv_fp8.cu, conv_s8.cu, conv_u8.cu and conv_mixed.cu keep exactly their instances.  The kernel is conv_wg_kernel
// (conv_tc_kernel.cuh) at PLANES = 2, ELEM = OUT = s8: activations and weights are 16-bit integers v = 256 hi + lo in two s8
// planes; per K step wgmma m64nBNk32 s8 x s8 -> s32 runs hi*hi into acc_h and hi*lo + lo*hi into acc_c, both over the whole K
// (exact, so nothing is chunked), and the per-channel epilogue is
//   S = 256 * (int64) acc_h + acc_c,  t = __fadd_rn(__fmul_rn(__ll2float_rn(S), f_c), b'_c),  ReLU,  v = sat(rint(t)) in
//   [-32768, 32639], stored as hi = (v + 128) >> 8 and lo = v - 256 hi
// (the fp32 maps store t).  conv1_1 reads the im2col'ed net input of S8X1 (p - 128) in the hi plane and zeros in the lo plane,
// so it is an ordinary two-plane layer.  |acc_c| <= (128 * 128 + 128 * 127) * K, which the engine keeps inside s32 by refusing a
// K above Precision::max_k (precision.h).
#include "conv_tc_kernel.cuh"

namespace pe {

int launch_s8x2(const TcLayer& l, const TcArgs& a, dim3 grid, cudaStream_t st, int bmap, int bn) {
    if (l.d.fmt.planes != 2 || l.d.out_elem != ELEM_S8) return -1;
    return launch_widths<2, ELEM_S8, ELEM_S8>(l, a, grid, st, bmap, bn);
}

}  // namespace pe
