// The format-boundary instances of the wgmma / TMA convolution for engines that run chosen layers in fp16 inside the e4m3 and s8
// modes (pe_create_mixed, DESIGN.md section 3), in a translation unit of their own so that conv_tc.cu, conv_fp8.cu and conv_s8.cu
// keep exactly their instances.  The kernel is conv_wg_kernel (conv_tc_kernel.cuh) unchanged; each instance's arithmetic is that
// of its input kind and only the store converts:
//   <1, e4m3, f16>: e4m3 MMAs, chunked fp32 sums, one factor per layer, stored as fp16 (split_pair);
//   <1, f16, s8>:   fp16 MMAs, chunked fp32 sums, one factor per layer, stored with cvt.rni.sat.s8.f32;
//   <1, s8, f16>:   s8 MMAs into one s32 accumulator, the per-channel epilogue t = acc * f_c + b'_c, stored as fp16.
// (fp16 -> e4m3 is conv1_1 of the e4m3 mode, in conv_fp8.cu.)
#include "conv_tc_kernel.cuh"

namespace pe {

int launch_mixed(const TcLayer& l, const TcArgs& a, dim3 grid, cudaStream_t st, int bmap, int bn) {
    const PlaneElem in = l.d.fmt.elem, out = l.d.out_elem;
    if (in == ELEM_E4M3 && out == ELEM_F16) return launch_widths<1, ELEM_E4M3, ELEM_F16>(l, a, grid, st, bmap, bn);
    if (in == ELEM_F16 && out == ELEM_S8) return launch_widths<1, ELEM_F16, ELEM_S8>(l, a, grid, st, bmap, bn);
    if (in == ELEM_S8 && out == ELEM_F16) return launch_widths<1, ELEM_S8, ELEM_F16>(l, a, grid, st, bmap, bn);
    return -1;   // e4m3 and s8 layers in one engine, or more than one plane: no instance
}

}  // namespace pe
