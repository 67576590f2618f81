// wgmma implicit-GEMM convolution (host interface).  See conv_tc.cu.
#pragma once
#include <string>

#include "common.h"
#include "kernels.h"

namespace pe {

struct TcLayerDesc {
    const void* in; int in_pitch, in_cused; long long in_plane;   // 16-bit planes [P][M][pitch]
    const void* w;                                                // 16-bit planes [P][cout_pad][K]
    const float* bias;
    int cout, cout_pad, ksize, pad, relu;
    PlaneFmt fmt;                                                 // plane count and fp16 / bf16 (kernels.h)
    const float* out_scale = nullptr;                             // device: epilogue factor 2^-k (weights packed with 2^k)
    unsigned* range = nullptr;                                    // device: running max |stored value| (float bits), or null
    Geo geo;                                                      // geo.N = max images
    void* out; int out_pitch, out_coff; long long out_plane;      // 16-bit planes, or
    float* planar; int planar_C, planar_coff;                     // final fp32 maps (N, planar_C, H, W)
};
struct TcLayer {
    void* maps = nullptr;   // host copy of the CUtensorMaps (A, B, B at half width), 64-byte aligned
    TcLayerDesc d;
    int bn = 0;
};

int tc_cout_pad(int cout);   // N-tile granularity used for a layer with `cout` outputs
int tc_layer_create(const TcLayerDesc& d, TcLayer& out, std::string& err);
void tc_layer_destroy(TcLayer& l);
// share: number of independent layers expected to run concurrently (2 when the L1 / L2 branches run on two streams): the tile
// width is then chosen for 1/share of the GPU.  Returns kernels launched, or -1 when the launch failed or no kernel fits.
int tc_layer_launch(const TcLayer& l, int nimg, cudaStream_t st, int share = 1);

}  // namespace pe
