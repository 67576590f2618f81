// Internal declarations shared by the engine's translation units (not part of the C ABI).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>

#include <string>
#include <vector>

#include "../../include/poseengine.h"

namespace pe {

// ---------------------------------------------------------------------------------------------
// Flat padded NHWC geometry.
// An activation of N images of HxW with C channels is stored as a 2-D matrix [M rows][C] where
//   row m = (n*Hs + y)*Wp + x,   Wp = W + gap,  Hs = H + gap,   gap >= largest conv pad at this level.
// Rows with x >= W or y >= H ("gap rows") are never written and stay zero, so a filter tap (r,s) of a
// stride-1 convolution with zero padding is a CONSTANT ROW SHIFT (r-pad)*Wp + (s-pad) of the whole
// matrix: the implicit-GEMM A operand of every tap is a plain 2-D tile (one TMA box), and Caffe's
// zero padding (im2col.cpp:35-46) falls out of the zero gap rows / TMA out-of-bounds fill.
// That holds only while pad <= gap: a larger pad reaches into the previous / next row or image.  So the
// plan sets each level's gap to max(1, largest pad of a convolution at that level) (NetPlan::gap; 1, 1, 1, 3
// for the built-in graphs, whose VGG levels run 3x3 and whose stride-8 stages run 7x7).
// Channel pitch: every activation's channel count is padded to the conv kernel's K block, the mode's act_cpad (precision.h;
// conv_tc_kernel.cuh explains the 128-byte block).  TMA needs global strides that are multiples of 16 bytes, which that
// padding covers.  The im2col'ed net input has a pitch of its own, the mode's kp_input.
// ---------------------------------------------------------------------------------------------
struct Geo {
    int W, H, gap, Wp, Hs, N;
    long long M;
};
inline Geo make_geo(int W, int H, int gap, int N) {
    Geo g;
    g.W = W; g.H = H; g.gap = gap; g.Wp = W + gap; g.Hs = H + gap; g.N = N;
    g.M = (long long)N * g.Hs * g.Wp;
    return g;
}

struct ModelTables {
    int num_parts, num_limbs, num_maps, max_peaks;
    const int* limb_seq;
    const int* map_idx;
};
const ModelTables& model_tables(int model);
const char* model_part_name(int model, int idx);
int model_flip_table(int model, std::vector<int>& perm, std::vector<float>& sign);   // plan.cpp: num_maps, or -1

// One convolution of the deploy graph in engine form.
struct ConvSpec {
    std::string name;          // prototxt layer name
    int cout, cin, k, pad, relu;
    int level;                 // 0: HxW, 1: /2, 2: /4, 3: /8
    int in_act, in_cused;      // input activation index and channels consumed (pitch may be larger)
    int out_act, out_coff;     // output activation (or -1: final planar maps) and channel offset
    int planar_coff;           // channel offset in concat_stage7 when out_act == -1
    std::vector<int> cin_map;  // engine input channel -> original cin index (-1: zero pad)
    std::vector<int> cin_prod; // engine input channel -> index of the conv that produced it (-1: zero pad / the net input)
    int im2col_input;          // conv1_1: the input activation already holds the 3x3x3 patch (K=27)
    double flops_per_image;
    int elem;                  // element kind (PlaneElem) of its arithmetic: of its input activation and packed weights
};
struct PoolSpec { std::string name; int in_act, out_act, level_in; };
struct CopySpec { int src_act, dst_act, channels; };  // duplicate F into the second concat buffer
struct ActSpec { int level, C; std::string blob; int blob_c; int elem; };  // blob: prototxt top living at channel 0; elem: PlaneElem
struct OpRef { int type, idx; };                      // 0 conv, 1 pool, 2 copy
// A fetchable blob: where it lives, which conv produced it (its stored values carry that conv's range scale; -1: the net
// input), and the first later op of the forward that overwrites its channels (empty: none; the ping-pong concat buffers).
struct BlobRef { std::string name; int act, coff, c; int prod = -1, pos = -1; std::string reused_by; };

struct NetPlan {
    int model = 0, c_l1 = 0, c_l2 = 0, kp_input = 0;
    // nms_param / imresize_param of the prototxt (caffe.proto:1471-1484); rtpose.cpp overrides threshold and scales at run time
    float nms_threshold = 0.5f; int nms_max_peaks = 20, nms_num_parts = 15;
    float resize_start_scale = 1.f, resize_scale_gap = 0.1f;
    std::vector<ActSpec> acts;
    std::vector<ConvSpec> convs;
    std::vector<PoolSpec> pools;
    std::vector<CopySpec> copies;
    std::vector<OpRef> order;
    std::vector<BlobRef> blobs;
    int input_act = 0;
    int gap[4] = {1, 1, 1, 1};   // per level: max(1, largest conv pad at that level), see Geo
};
struct NetDef;
// Element kinds of a plan (plan.cpp, DESIGN.md section 3): a conv layer listed in f16 computes in fp16, the others in
// base_elem (conv1_1: input_elem).  "narrow" in f16 stands for every conv layer that reads fewer than 128 channels.
// layout[k]: channel pad, net input pitch and Concat slot alignment of an activation of element kind k (PlaneElem).
struct ActLayout { int cpad, kp_input, slot_align; };
// u8 (PE_PREC_FLAG_U8, base_elem s8): an activation whose every writer stores values >= 0 (conv layers followed by ReLU, and
// max pools of them) and whose every reader computes in s8 is stored as u8, and its readers compute u8 x s8.
struct PlanFormats {
    int base_elem = 0, input_elem = 0;
    bool u8 = false;
    std::vector<std::string> f16;
    ActLayout layout[5] = {};   // one per PlaneElem (precision.h)
};
// plan from a parsed prototxt / built-in definition; -1 and a message when the graph is outside the supported family or the
// fp16 list breaks the format rules
int build_plan_from_net(const NetDef& net, const PlanFormats& f, NetPlan& out, std::string& err);
// One element kind throughout, Concat slots 8-aligned
int build_plan_from_net(const NetDef& net, int kp_input, int cpad, NetPlan& out, std::string& err);

// The packed K order of conv c's weights (engine.cu packs in it): K index kk = tap * c.in_cused + engine input channel, Concat
// slots at their aligned offsets (cin_map), conv1_1 the 27 values of its im2col'ed input.  Returns the index of weight (co, kk)
// in the Caffe blob [cout][cin][k][k], or -1 for a zero pad.
long long conv_weight_index(const ConvSpec& c, int co, int kk);
// 2:4 structured sparsity in that order: every aligned group of four packed weights of every output channel of w (Caffe
// layout) holds at most two non-zeros.  Padding is zero.
bool conv_weights_2to4(const ConvSpec& c, const float* w);
// Magnitude pruning to 2:4 in that grouping, in place: each group keeps its two largest |w|, the lower K index on a tie.
void conv_prune_2to4(const ConvSpec& c, float* w);

// ---------------------------------------------------------------------------------------------
// kernel argument blocks
// ---------------------------------------------------------------------------------------------
struct ConvArgs {
    const void* in; int in_pitch; long long in_plane;     // fp32 [M][pitch] or bf16 planes
    const void* w;                                        // SIMT: fp32 [K][cout_pad]
    const float* bias;
    void* out; int out_pitch, out_coff; long long out_plane;
    float* planar; int planar_C, planar_coff;             // final maps (N, planar_C, H, W)
    int cin_pad, cout, cout_pad, ksize, pad, relu;
    int W, H, Wp, Hs, N; long long M;
};

struct PostParams {
    int model, num_parts, num_limbs, num_maps, max_peaks;
    int net_w, net_h, w8, h8, disp_w, disp_h, num_scales;
    float start_scale, scale_gap, nms_threshold;
    int min_subset_cnt; float min_subset_score, inter_threshold; int inter_min_above;
    int max_subset_rows;   // num_limbs * max_peaks: a limb appends at most one row per peak of one part or per connection
};

#define PE_MAX_PEAKS 127   // largest nms_param.max_peaks a deploy file may set (plan.cpp); post.cu's shared tables hold that many
#define PE_MAX_SCALES 8

}  // namespace pe
