// The e4m3 instances of the wgmma / TMA convolution (PE_PREC_E4M3X1), in a translation unit of their own so that conv_tc.cu
// keeps exactly its 16-bit instances.  The kernel is conv_wg_kernel (conv_tc_kernel.cuh) at ELEM = e4m3: 128-channel K blocks
// in the same 128-byte swizzle rows, wgmma m64nBNk32 e4m3 x e4m3 -> fp32 with the fp16 fast mode's chunked round-to-nearest
// accumulation, and an epilogue that rounds to e4m3 with cvt.rn.satfinite.  conv1_1 keeps its fp16 im2col input: its instance
// reads fp16 and writes e4m3.
#include "conv_tc_kernel.cuh"

namespace pe {

int launch_e4m3(const TcLayer& l, const TcArgs& a, dim3 grid, cudaStream_t st, int bmap, int bn) {
    return l.d.fmt.f16() ? launch_widths<1, ELEM_F16, ELEM_E4M3>(l, a, grid, st, bmap, bn)
                         : launch_widths<1, ELEM_E4M3, ELEM_E4M3>(l, a, grid, st, bmap, bn);
}

}  // namespace pe
