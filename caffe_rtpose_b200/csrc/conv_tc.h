// wgmma implicit-GEMM convolution (host interface).  See conv_tc.cu.
#pragma once
#include <string>

#include "common.h"
#include "kernels.h"

namespace pe {

struct TcLayerDesc {
    const void* in; int in_pitch, in_cused; long long in_plane;   // planes [P][M][pitch] of fmt's element kind
    const void* w;                                                // planes [P][cout_pad][K] of fmt's element kind
    const float* bias;
    int cout, cout_pad, ksize, pad, relu;
    PlaneFmt fmt;                                                 // plane count and element kind of in and w (precision.h)
    PlaneElem out_elem;                                           // element kind of out (conv1_1 of E4M3X1: fp16 in, e4m3 out)
    bool chunked;                                                 // the mode's hi*hi accumulation (Precision::chunked)
    bool sparse = false;                                          // s8, w holds 2:4-compressed weights (s8_sparse.h): conv_s8_sparse.cu
    const float* out_scale = nullptr;                             // device: epilogue factor 2^-k (weights packed with 2^k)
    unsigned* range = nullptr;                                    // device: running max |stored value| (float bits), or null
    Geo geo;                                                      // geo.N = max images
    void* out; int out_pitch, out_coff; long long out_plane;      // fmt.planes planes of out_elem, or
    float* planar; int planar_C, planar_coff;                     // final fp32 maps (N, planar_C, H, W)
};
struct TcLayer {
    void* maps = nullptr;   // host copy of the CUtensorMaps (A, B, B at half width; sparse: windows of 128 pixels, compressed
                            // weights, windows of 64 pixels), 64-byte aligned
    TcLayerDesc d;
    int bn = 0;
};

int tc_cout_pad(int cout);   // N-tile granularity used for a layer with `cout` outputs
int tc_layer_create(const TcLayerDesc& d, TcLayer& out, std::string& err);
void tc_layer_destroy(TcLayer& l);
// share: number of independent layers expected to run concurrently (2 when the L1 / L2 branches run on two streams): the tile
// width is then chosen for 1/share of the GPU.  Returns kernels launched, or -1 when the launch failed or no kernel fits.
int tc_layer_launch(const TcLayer& l, int nimg, cudaStream_t st, int share = 1);
int tc_sparse_launch(const TcLayer& l, int nimg, cudaStream_t st, int share);   // conv_s8_sparse.cu, for d.sparse

}  // namespace pe
