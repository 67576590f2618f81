// libposeengine.so - C ABI implementation (include/poseengine.h).  Host orchestration of one GPU worker:
// what warmup()/processFrame() do around caffe::Net in examples/rtpose/rtpose.cpp:173-237, 1079-1203,
// re-designed for the H100: a fixed execution plan (plan.cpp) over flat padded NHWC activations, one stream,
// asynchronous forwards, KB-sized results returned through pinned memory.  No CPU fallback anywhere.
#include <math.h>
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "common.h"
#include "kernels.h"
#include "conv_tc.h"
#include "jpeg_coefs.h"
#include "jpeg_entropy.cuh"
#include "pixels.cuh"
#include <climits>
#include "prototxt.h"

// NVTX ranges (header-only nvtx3: resolved at run time, no-ops without a profiler attached) around the phases of a forward, so that
// nsys / ncu timelines read like the reference's stage names (SURVEY.md section 5)
#include <nvtx3/nvToolsExt.h>
struct NvtxRange { explicit NvtxRange(const char* n) { nvtxRangePushA(n); } ~NvtxRange() { nvtxRangePop(); } };

using namespace pe;

static thread_local std::string g_create_error;

struct HostWeights { std::vector<float> w, b; bool set = false; };

struct pe_engine {
    pe_config cfg;
    NetPlan plan;
    const ModelTables* mt = nullptr;
    ModelTables mt_own;     // model tables with the prototxt's nms max_peaks
    Geo geo[4];
    PlaneFmt fmt = {0, false};   // storage of activations and packed weights (kernels.h): 0 planes = fp32 SIMT
    int elem = 4;
    std::vector<void*> acts;        // device
    std::vector<long long> act_plane;  // elements per plane
    std::vector<HostWeights> hw;    // per conv
    bool committed = false;
    // packed weights (one device buffer): per conv offsets (bytes)
    void* d_packed = nullptr; size_t packed_bytes = 0;
    std::shared_ptr<void> packed_owner;   // frees d_packed when the last handle using it goes (pe_share_weights)
    // fp16-plane range management (F16X2, F16X1): per-conv-output power-of-two scale s (stored value = true value * s), the true
    // biases / weight-scale inverses the packed epilogue fields derive from, and the kernels' running max |stored value| per conv
    std::vector<float> conv_scale, wsi;   // per conv: scale of its stored output; inverse of the power of two folded into its weights
    std::vector<std::vector<float>> bias_true;
    unsigned* d_range = nullptr;
    bool calibrated = false, check_range = false;
    std::vector<size_t> w_off, b_off;
    size_t w11_off = 0;             // fp32 [27][64] weights + 64 biases of conv1_1 for the direct kernel (0: not packed)
    float w11_scale = 1.f;          // activation scale currently folded into that copy
    bool conv11_direct = false;     // PE_CONV11_DIRECT=1: conv1_1 by conv1_1_direct_kernel (fp32 CUDA cores, no im2col'ed input) instead of
                                    // the im2col + implicit-GEMM path (the tensor path is the default)
    bool input_from_frames = false; // the last forward came from uint8 frames: d_resized holds conv1_1's input
    bool input_act_stale = false;   // ... and the im2col'ed input activation was not produced (conv1_1 direct)
    std::vector<int> cout_pad, cin_pad;
    std::vector<TcLayer> tc;        // wgmma per-conv launch state
    // io
    cudaStream_t stream = nullptr;
    // Second lane: the L2 branch of every stage runs on its own stream next to the L1 branch (they only meet at the stage
    // boundaries), so the tail of one layer overlaps the head of an independent one and a single frame fills more SMs.
    cudaStream_t stream2 = nullptr;
    bool two_lanes = false;
    std::vector<int> op_lane;                    // per plan.order entry
    std::vector<std::vector<int>> op_waits;      // convs on the OTHER lane whose completion this op needs
    std::vector<cudaEvent_t> conv_done;          // per conv: recorded after its launch when another lane waits for it
    int last_lane1_conv = -1;
    cudaEvent_t ev[16] = {};
    uint8_t* d_frames = nullptr; uint8_t* d_resized = nullptr;
    uint8_t* h_frames = nullptr;    // pinned staging
    float* d_planar = nullptr; float* h_planar = nullptr;
    std::vector<void*> d_tabs;
    PreArgs pre;
    float* d_maps = nullptr; float* h_maps = nullptr;
    PostDev post;
    float* h_joints = nullptr; int* h_num_people = nullptr; float* h_peaks = nullptr;
    AxisTap *d_xtab = nullptr, *d_ytab = nullptr;
    float start_scale_f, scale_gap_f;
    int last_n = 0;
    // raw camera frames (any size) -> display image: warpAffine tables for the last (orig_w, orig_h)
    uint8_t* d_raw = nullptr; size_t raw_cap = 0; uint8_t* h_raw = nullptr; size_t h_raw_cap = 0;
    int warp_w = 0, warp_h = 0; double warp_scale = 1.0;
    int *d_wa = nullptr, *d_wb = nullptr, *d_wx0 = nullptr, *d_wy0 = nullptr; short* d_wtab = nullptr;
    // decoder-format host frames (pe_forward_pixels) copied to the device before conversion; pe_stream_wait's event
    uint8_t* d_pix = nullptr; size_t pix_cap = 0;
    cudaEvent_t ev_wait = nullptr;
    bool input_lo_dirty = false;
    // JPEG coefficient images (pe_forward_jpeg_coefs): device copies, pinned staging for pageable callers, component planes
    uint8_t* d_jcoef = nullptr; size_t jcoef_cap = 0; uint8_t* h_jcoef = nullptr; size_t h_jcoef_cap = 0;
    uint8_t* d_jplanes = nullptr; size_t jplanes_cap = 0;
    // JPEG scan images (pe_forward_jpeg_scans): device copies, pinned staging, the decoder's work space, per-frame status
    uint8_t* d_jscan = nullptr; size_t jscan_cap = 0; uint8_t* h_jscan = nullptr; size_t h_jscan_cap = 0;
    uint8_t* d_jwork = nullptr; size_t jwork_cap = 0;
    uint8_t* h_jstatus = nullptr; size_t h_jstatus_cap = 0;
    int jstatus_n = 0;   // frames of the last forward whose status h_jstatus holds (0: the last forward was not from scan images)
    // renderers: canvas, uint8 image, heat-map scratch (allocated on first pe_render); display frames of the last forward
    float* d_canvas = nullptr; uint8_t* d_render_u8 = nullptr; uint8_t* d_render_src = nullptr; float* d_heat = nullptr; size_t heat_cap = 0;
    const uint8_t* last_frames = nullptr;
    // CUDA graphs of the steady-state forward (92 conv + pool/copy + 5 parse kernels + result copies), one per batch
    // size; the first forward of a size runs eagerly, the second is captured, later ones replay.  Invalidated by
    // any setter whose value is baked into kernel arguments.
    struct GraphEntry { cudaGraphExec_t exec = nullptr; long long launches = 0; int seen = 0; };
    std::map<int, GraphEntry> graphs;
    bool use_graphs = true;   // the planar-input path wrote non-zero lo planes / channels >= 32 of the input buffer
    long long launches = 0;
    std::string err;
    double flops_per_scale = 0;
};

static void drop_graphs(pe_engine* e);
static int setup_lanes(pe_engine* e);

static int fail(pe_engine* e, int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (e) e->err = buf; else g_create_error = buf;
    return code;
}
#define CK(e, call) do { cudaError_t err_ = (call); if (err_ != cudaSuccess) \
    return fail(e, PE_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(err_), __FILE__, __LINE__); } while (0)

extern "C" const char* pe_last_error(const pe_engine* e) { return e ? e->err.c_str() : g_create_error.c_str(); }

// ---------------------------------------------------------------------------------------------
// model descriptor tables
// ---------------------------------------------------------------------------------------------
extern "C" int pe_model_num_parts(int model) { return model_tables(model).num_parts; }
extern "C" int pe_model_num_limbs(int model) { return model_tables(model).num_limbs; }
extern "C" const int* pe_model_limb_sequence(int model) { return model_tables(model).limb_seq; }
extern "C" const int* pe_model_map_idx(int model) { return model_tables(model).map_idx; }
extern "C" const char* pe_model_part_name(int model, int idx) { return model_part_name(model, idx); }

// ---------------------------------------------------------------------------------------------
// INTER_AREA decimation tables (OpenCV imgproc/resize.cpp computeResizeAreaTab), built on the host
// in double precision exactly as cv::resize does, then used by area_resize_kernel.
// ---------------------------------------------------------------------------------------------
static void area_table(int ssize, int dsize, double scale, std::vector<int>& ofs, std::vector<int>& si,
                       std::vector<float>& alpha) {
    ofs.assign(1, 0); si.clear(); alpha.clear();
    for (int dx = 0; dx < dsize; dx++) {
        const double fsx1 = dx * scale, fsx2 = fsx1 + scale;
        const double cell = std::min(scale, ssize - fsx1);
        int sx1 = (int)ceil(fsx1), sx2 = (int)floor(fsx2);
        sx2 = std::min(sx2, ssize - 1);
        sx1 = std::min(sx1, sx2);
        if (sx1 - fsx1 > 1e-3) { si.push_back(sx1 - 1); alpha.push_back((float)((sx1 - fsx1) / cell)); }
        for (int sx = sx1; sx < sx2; sx++) { si.push_back(sx); alpha.push_back((float)(1.0 / cell)); }
        if (fsx2 - sx2 > 1e-3) { si.push_back(sx2); alpha.push_back((float)(std::min(std::min(fsx2 - sx2, 1.), cell) / cell)); }
        ofs.push_back((int)si.size());
    }
}

template <typename T>
static int upload(pe_engine* e, const std::vector<T>& v, const T** out) {
    void* d = nullptr;
    CK(e, cudaMalloc(&d, std::max<size_t>(v.size(), 1) * sizeof(T)));
    CK(e, cudaMemcpy(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    e->d_tabs.push_back(d);
    *out = (const T*)d;
    return PE_OK;
}

static int build_pre_tables(pe_engine* e) {
    const pe_config& c = e->cfg;
    PreArgs& a = e->pre;
    memset(&a, 0, sizeof a);
    a.S = c.num_scales; a.disp_w = c.disp_w; a.disp_h = c.disp_h; a.net_w = c.net_w; a.net_h = c.net_h;
    for (int i = 0; i < c.num_scales; i++) {
        // rtpose.cpp:509-511: float scale = START_SCALE - i*SCALE_GAP; target = 16*ceil(NET*scale/16)
        const float scale = (float)(c.start_scale - i * c.scale_gap);
        const int tw = (int)(16 * ceil(c.net_w * scale / 16)), th = (int)(16 * ceil(c.net_h * scale / 16));
        if (tw > c.net_w || th > c.net_h || tw <= 0 || th <= 0)
            return fail(e, PE_ERR_INVALID, "scale %d gives target %dx%d outside net %dx%d (CHECK_LE rtpose.cpp:513-514)", i, tw,
                        th, c.net_w, c.net_h);
        AreaTab& t = a.tab[i];
        t.tw = tw; t.th = th; t.padw = (c.net_w - tw) / 2; t.padh = (c.net_h - th) / 2;
        const double inv_x = (double)tw / c.disp_w, inv_y = (double)th / c.disp_h;
        const double sx = 1. / inv_x, sy = 1. / inv_y;
        t.linear = !(tw == c.disp_w && th == c.disp_h) && (sx < 1 || sy < 1);
        if (t.linear) {
            // cv::resize leaves the area path when one axis enlarges: fixed-point bilinear, "area mode" positions
            // (imgproc/resize.cpp: sx = floor(dx*scale), fx = (dx+1) - (sx+1)*inv_scale clipped to [0,1), 11-bit coefficients)
            auto lin = [](int ssize, int dsize, std::vector<int>& tab) {
                const double inv = (double)dsize / ssize, scale = 1. / inv;
                tab.resize((size_t)dsize * 3);
                for (int d = 0; d < dsize; d++) {
                    int s0 = (int)floor(d * scale);
                    float f = (float)((d + 1) - (s0 + 1) * inv);
                    f = f <= 0 ? 0.f : f - floorf(f);
                    if (s0 < 0) { f = 0; s0 = 0; }
                    if (s0 >= ssize - 1) { f = 0; s0 = ssize - 1; }
                    tab[d * 3] = s0;
                    tab[d * 3 + 1] = (int)std::min(32767L, std::max(-32768L, lrintf((1.f - f) * 2048)));
                    tab[d * 3 + 2] = (int)std::min(32767L, std::max(-32768L, lrintf(f * 2048)));
                }
            };
            std::vector<int> lx, ly;
            lin(c.disp_w, tw, lx);
            lin(c.disp_h, th, ly);
            if (upload(e, lx, &t.lin_x) || upload(e, ly, &t.lin_y)) return PE_ERR_CUDA;
        }
        const int ix = (int)lrint(sx), iy = (int)lrint(sy);
        t.fast = fabs(sx - ix) < 2.220446049250313e-16 && fabs(sy - iy) < 2.220446049250313e-16;
        t.iscale_x = ix; t.iscale_y = iy;
        std::vector<int> ofs, si; std::vector<float> al;
        area_table(c.disp_w, tw, sx, ofs, si, al);
        if (upload(e, ofs, &t.x_ofs) || upload(e, si, &t.x_si) || upload(e, al, &t.x_alpha)) return PE_ERR_CUDA;
        area_table(c.disp_h, th, sy, ofs, si, al);
        if (upload(e, ofs, &t.y_ofs) || upload(e, si, &t.y_si) || upload(e, al, &t.y_alpha)) return PE_ERR_CUDA;
    }
    return PE_OK;
}

// ---------------------------------------------------------------------------------------------
// create / destroy
// ---------------------------------------------------------------------------------------------
static int pooled(int v) { return (int)ceilf((float)(v - 2) / 2) + 1; }  // pooling_layer.cpp:90-93, k=2 s=2 pad=0

static void set_post_params(pe_engine* e) {
    PostParams& p = e->post.p;
    const pe_config& c = e->cfg;
    p.model = c.model; p.num_parts = e->mt->num_parts; p.num_limbs = e->mt->num_limbs; p.num_maps = e->mt->num_maps;
    p.max_peaks = e->mt->max_peaks;
    p.net_w = c.net_w; p.net_h = c.net_h; p.w8 = e->geo[3].W; p.h8 = e->geo[3].H; p.disp_w = c.disp_w; p.disp_h = c.disp_h;
    p.num_scales = c.num_scales;
}

// Host-only view of the execution plan a prototxt (or, with path == NULL, the built-in graph of `model`) produces: one
// line per op, "conv <name> cout cin k relu level in_act in_cused out_act out_coff planar_coff", "pool <name> in out",
// "copy src dst channels", then "gap level g" per resolution level (the flat layout's gap, common.h), "nms threshold
// max_peaks num_parts" and "resize start_scale scale_gap".  No GPU needed.
extern "C" int pe_plan_describe(int model, const char* prototxt_path, char* buf, int cap) {
    NetDef net;
    std::string err;
    if (prototxt_path) {
        if (parse_prototxt_file(prototxt_path, net, err)) return -fail(nullptr, PE_ERR_IO, "%s: %s", prototxt_path, err.c_str());
    } else {
        if (model != PE_MODEL_MPI_15 && model != PE_MODEL_COCO_18) return -fail(nullptr, PE_ERR_INVALID, "unknown model %d", model);
        net = builtin_netdef(model, 6);
    }
    NetPlan p;
    if (build_plan_from_net(net, 64, 64, p, err)) return -fail(nullptr, PE_ERR_INVALID, "%s", err.c_str());
    std::string s = "model " + std::to_string(p.model) + "\n";
    char t[512];
    for (const OpRef& op : p.order) {
        if (op.type == 0) {
            const ConvSpec& c = p.convs[op.idx];
            snprintf(t, sizeof t, "conv %s %d %d %d %d %d %d %d %d %d %d\n", c.name.c_str(), c.cout, c.cin, c.k, c.relu, c.level, c.in_act, c.in_cused,
                     c.out_act, c.out_coff, c.planar_coff);
        } else if (op.type == 1) {
            snprintf(t, sizeof t, "pool %s %d %d\n", p.pools[op.idx].name.c_str(), p.pools[op.idx].in_act, p.pools[op.idx].out_act);
        } else {
            snprintf(t, sizeof t, "copy %d %d %d\n", p.copies[op.idx].src_act, p.copies[op.idx].dst_act, p.copies[op.idx].channels);
        }
        s += t;
    }
    for (int l = 0; l < 4; l++) {
        snprintf(t, sizeof t, "gap %d %d\n", l, p.gap[l]);
        s += t;
    }
    snprintf(t, sizeof t, "nms %g %d %d\nresize %g %g\n", p.nms_threshold, p.nms_max_peaks, p.nms_num_parts, p.resize_start_scale, p.resize_scale_gap);
    s += t;
    if (buf && (int)s.size() < cap) memcpy(buf, s.c_str(), s.size() + 1);
    return (int)s.size();
}

static int create_impl(const pe_config* cfg, const char* prototxt_path, pe_engine** out);
extern "C" int pe_create(const pe_config* cfg, pe_engine** out) { return create_impl(cfg, nullptr, out); }
// new caffe::Net(proto, TEST): the graph comes from the deploy prototxt (rtpose.cpp:183, net.cpp:30-50); cfg->model may be
// -1, the model then follows the Nms layer's num_parts as in rtpose.cpp:212-229.
extern "C" int pe_create_from_prototxt(const pe_config* cfg, const char* prototxt_path, pe_engine** out) {
    if (!prototxt_path) return fail(nullptr, PE_ERR_INVALID, "null prototxt path");
    return create_impl(cfg, prototxt_path, out);
}

static int create_impl(const pe_config* cfg_in, const char* prototxt_path, pe_engine** out) {
    if (!cfg_in || !out) return fail(nullptr, PE_ERR_INVALID, "null argument");
    *out = nullptr;
    pe_config cfg_copy = *cfg_in;
    pe_config* cfg = &cfg_copy;
    NetDef netdef;
    NetPlan proto_plan;
    if (prototxt_path) {
        std::string perr;
        if (parse_prototxt_file(prototxt_path, netdef, perr)) return fail(nullptr, PE_ERR_IO, "%s: %s", prototxt_path, perr.c_str());
        if (build_plan_from_net(netdef, cfg->precision ? 64 : 32, cfg->precision ? 64 : 16, proto_plan, perr))
            return fail(nullptr, PE_ERR_INVALID, "%s: %s", prototxt_path, perr.c_str());
        if (cfg->model >= 0 && cfg->model != proto_plan.model)
            return fail(nullptr, PE_ERR_INVALID, "%s describes the %s model (nms num_parts %d), the configuration asks for model %d", prototxt_path,
                        proto_plan.model == PE_MODEL_MPI_15 ? "MPI" : "COCO", proto_plan.nms_num_parts, cfg->model);
        cfg->model = proto_plan.model;
    }
    if (cfg->model != PE_MODEL_MPI_15 && cfg->model != PE_MODEL_COCO_18) return fail(nullptr, PE_ERR_INVALID, "unknown model %d", cfg->model);
    if (cfg->net_w <= 0 || cfg->net_h <= 0 || cfg->net_w % 8 || cfg->net_h % 8)
        return fail(nullptr, PE_ERR_INVALID, "net resolution %dx%d must be positive multiples of 8", cfg->net_w, cfg->net_h);
    if (cfg->num_scales < 1 || cfg->num_scales > PE_MAX_SCALES) return fail(nullptr, PE_ERR_INVALID, "num_scales %d out of [1,%d]", cfg->num_scales, PE_MAX_SCALES);
    if (cfg->max_batch < 1 || cfg->max_batch > 64) return fail(nullptr, PE_ERR_INVALID, "max_batch %d out of [1,64]", cfg->max_batch);
    if (cfg->disp_w <= 0 || cfg->disp_h <= 0) return fail(nullptr, PE_ERR_INVALID, "bad display resolution");
    if (cfg->precision < 0 || cfg->precision > 4) return fail(nullptr, PE_ERR_INVALID, "unknown precision %d", cfg->precision);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail(nullptr, PE_ERR_CUDA, "no CUDA device visible: the pose engine has no CPU fallback");
    if (cfg->device < 0 || cfg->device >= ndev) return fail(nullptr, PE_ERR_INVALID, "device %d out of range (%d visible)", cfg->device, ndev);

    pe_engine* e = new pe_engine();
    memset(&e->post, 0, sizeof e->post);   // PODs: every pointer must be null for pe_destroy on an early failure
    memset(&e->pre, 0, sizeof e->pre);
    e->cfg = *cfg;
    e->mt_own = model_tables(cfg->model);
    if (prototxt_path) e->mt_own.max_peaks = proto_plan.nms_max_peaks;   // nms_param.max_peaks (NmsLayer::GetMaxPeaks, rtpose.cpp:195)
    e->mt = &e->mt_own;
    e->fmt = plane_fmt(cfg->precision);
    if (const char* g = getenv("PE_GRAPH")) e->use_graphs = atoi(g) != 0;
    if (const char* g = getenv("PE_CONV11_DIRECT")) e->conv11_direct = atoi(g) != 0;
    if (const char* g = getenv("PE_CHECK_RANGE")) e->check_range = atoi(g) != 0;
    e->elem = e->fmt.planes == 0 ? 4 : 2;
    e->start_scale_f = (float)cfg->start_scale;  // ImResizeLayer::SetStartScale(float)
    e->scale_gap_f = (float)cfg->scale_gap;
    auto bail = [&](int rc) { g_create_error = e->err; pe_destroy(e); return rc; };
#define CKC(call) do { cudaError_t err_ = (call); if (err_ != cudaSuccess) { \
    fail(e, PE_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(err_), __FILE__, __LINE__); return bail(PE_ERR_CUDA); } } while (0)
    CKC(cudaSetDevice(cfg->device));
    if (e->fmt.planes) {
        cudaDeviceProp prop;
        CKC(cudaGetDeviceProperties(&prop, cfg->device));
        if (prop.major != 9) { fail(e, PE_ERR_INVALID, "wgmma precision modes need sm_90 (found sm_%d%d)", prop.major, prop.minor); return bail(PE_ERR_INVALID); }
    }
    CKC(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
    for (int i = 0; i < 16; i++) CKC(cudaEventCreate(&e->ev[i]));

    // the plan first: each level's gap is the largest pad of its convolutions (common.h)
    e->plan = prototxt_path ? proto_plan : build_plan(cfg->model, e->fmt.planes ? 64 : 32, e->fmt.planes ? 64 : 16);
    const int N = cfg->max_batch * cfg->num_scales;
    int w = cfg->net_w, h = cfg->net_h;
    for (int l = 0; l < 4; l++) {
        e->geo[l] = make_geo(w, h, e->plan.gap[l], N);
        w = pooled(w); h = pooled(h);
    }
    if (e->geo[3].W * 8 != cfg->net_w || e->geo[3].H * 8 != cfg->net_h) { fail(e, PE_ERR_INVALID, "net size not divisible by 8 after pooling"); return bail(PE_ERR_INVALID); }
    e->hw.resize(e->plan.convs.size());
    if (e->fmt.planes && setup_lanes(e)) return bail(PE_ERR_CUDA);
    // FLOPs (SURVEY.md section 8d): 2*Cout*Cin*k^2*Hout*Wout per conv and image
    e->flops_per_scale = 0;
    for (auto& c : e->plan.convs) {
        const Geo& g = e->geo[c.level];
        c.flops_per_image = 2.0 * c.cout * c.cin * c.k * c.k * g.H * g.W;
        e->flops_per_scale += c.flops_per_image;
    }
    // activations
    e->acts.assign(e->plan.acts.size(), nullptr);
    e->act_plane.assign(e->plan.acts.size(), 0);
    for (size_t i = 0; i < e->plan.acts.size(); i++) {
        const ActSpec& a = e->plan.acts[i];
        const Geo& g = e->geo[a.level];
        e->act_plane[i] = g.M * a.C;
        const size_t bytes = (size_t)e->act_plane[i] * e->elem * (e->fmt.planes ? e->fmt.planes : 1);
        CKC(cudaMalloc(&e->acts[i], bytes));
        CKC(cudaMemsetAsync(e->acts[i], 0, bytes, e->stream));
    }
    // io buffers
    const size_t frame_bytes = (size_t)cfg->disp_w * cfg->disp_h * 3;
    CKC(cudaMalloc(&e->d_frames, frame_bytes * cfg->max_batch));
    CKC(cudaMallocHost(&e->h_frames, frame_bytes * cfg->max_batch));
    CKC(cudaMalloc(&e->d_resized, (size_t)N * cfg->net_w * cfg->net_h * 3));
    const size_t planar_n = (size_t)N * 3 * cfg->net_w * cfg->net_h;
    CKC(cudaMalloc(&e->d_planar, planar_n * sizeof(float)));
    CKC(cudaMallocHost(&e->h_planar, planar_n * sizeof(float)));
    const size_t maps_n = (size_t)N * e->mt->num_maps * e->geo[3].W * e->geo[3].H;
    CKC(cudaMalloc(&e->d_maps, maps_n * sizeof(float)));
    CKC(cudaMemsetAsync(e->d_maps, 0, maps_n * sizeof(float), e->stream));
    CKC(cudaMallocHost(&e->h_maps, maps_n * sizeof(float)));
    if (build_pre_tables(e)) return bail(PE_ERR_INVALID);
    e->pre.frames = e->d_frames; e->pre.resized = e->d_resized;
    e->pre.out = e->acts[e->plan.input_act]; e->pre.kp = e->plan.kp_input;
    e->pre.out_plane = e->act_plane[e->plan.input_act]; e->pre.fmt = e->fmt;
    e->pre.Wp = e->geo[0].Wp; e->pre.Hs = e->geo[0].Hs;

    // post-processing state
    set_post_params(e);
    PostDev& pd = e->post;
    {
        PostParams& p = pd.p;
        p.start_scale = e->start_scale_f; p.scale_gap = e->scale_gap_f;
        // rtpose.cpp:212-226
        p.min_subset_cnt = 3; p.min_subset_score = 0.4f;
        if (cfg->model == PE_MODEL_MPI_15) { p.nms_threshold = 0.2f; p.inter_threshold = 0.01f; p.inter_min_above = 8; }
        else { p.nms_threshold = 0.05f; p.inter_threshold = 0.050f; p.inter_min_above = 9; }
    }
    for (int i = 0; i < 2 * e->mt->num_limbs; i++) { pd.md.limb_seq[i] = e->mt->limb_seq[i]; pd.md.map_idx[i] = e->mt->map_idx[i]; }
    const int B = cfg->max_batch, P = e->mt->num_parts, MP = e->mt->max_peaks, NL = e->mt->num_limbs;
    pd.maps = e->d_maps;
    CKC(cudaMalloc(&e->d_xtab, sizeof(AxisTap) * cfg->num_scales * cfg->net_w));
    CKC(cudaMalloc(&e->d_ytab, sizeof(AxisTap) * cfg->num_scales * cfg->net_h));
    pd.xtab = e->d_xtab; pd.ytab = e->d_ytab;
    const int wpr = (cfg->net_w + 31) / 32;
    CKC(cudaMalloc(&pd.flags, sizeof(unsigned) * (size_t)B * P * cfg->net_h * wpr));
    CKC(cudaMalloc(&pd.peaks, sizeof(float) * (size_t)B * P * (MP + 1) * 3));
    CKC(cudaMalloc(&pd.cands, sizeof(Cand) * (size_t)B * NL * MP * MP));
    CKC(cudaMalloc(&pd.cand_count, sizeof(int) * (size_t)B * NL));
    pd.sort_stride = 1;
    while (pd.sort_stride < MP * MP) pd.sort_stride <<= 1;
    CKC(cudaMalloc(&pd.conns, sizeof(Conn) * (size_t)B * NL * MP));
    CKC(cudaMalloc(&pd.conn_count, sizeof(int) * (size_t)B * NL));
    CKC(cudaMemset(pd.conn_count, 0, sizeof(int) * (size_t)B * NL));
    CKC(cudaMalloc(&pd.subset, sizeof(double) * (size_t)B * PE_MAX_SUBSET_ROWS * (P + 3)));
    CKC(cudaMalloc(&pd.subset_rows, sizeof(int) * B));
    CKC(cudaMalloc(&pd.joints, sizeof(float) * (size_t)B * PE_MAX_PEOPLE * P * 3));
    CKC(cudaMalloc(&pd.num_people, sizeof(int) * B));
    CKC(cudaMallocHost(&e->h_joints, sizeof(float) * (size_t)B * PE_MAX_PEOPLE * P * 3));
    CKC(cudaMallocHost(&e->h_num_people, sizeof(int) * B));
    CKC(cudaMallocHost(&e->h_peaks, sizeof(float) * (size_t)B * P * (MP + 1) * 3));
    launch_axis_tables(e->d_xtab, e->d_ytab, pd.p, e->stream);
    e->launches += 2;
    CKC(cudaStreamSynchronize(e->stream));
    *out = e;
    return PE_OK;
}

extern "C" void pe_destroy(pe_engine* e) {
    if (!e) return;
    cudaSetDevice(e->cfg.device);
    if (e->stream) cudaStreamSynchronize(e->stream);
    drop_graphs(e);
    for (void* p : e->acts) if (p) cudaFree(p);
    for (void* p : e->d_tabs) cudaFree(p);
    for (auto& t : e->tc) tc_layer_destroy(t);
    cudaFree(e->d_jcoef); cudaFreeHost(e->h_jcoef); cudaFree(e->d_jplanes);
    cudaFree(e->d_jscan); cudaFreeHost(e->h_jscan); cudaFree(e->d_jwork); cudaFreeHost(e->h_jstatus);
    cudaFree(e->d_pix); if (e->ev_wait) cudaEventDestroy(e->ev_wait);
    cudaFree(e->d_raw); cudaFreeHost(e->h_raw); cudaFree(e->d_wa); cudaFree(e->d_wb); cudaFree(e->d_wx0); cudaFree(e->d_wy0); cudaFree(e->d_wtab);
    e->packed_owner.reset(); cudaFree(e->d_range); cudaFree(e->d_frames); cudaFree(e->d_resized); cudaFree(e->d_planar); cudaFree(e->d_maps);
    cudaFreeHost(e->h_frames); cudaFreeHost(e->h_planar); cudaFreeHost(e->h_maps);
    cudaFree(e->d_xtab); cudaFree(e->d_ytab);
    cudaFree(e->d_canvas); cudaFree(e->d_render_u8); cudaFree(e->d_render_src); cudaFree(e->d_heat);
    PostDev& pd = e->post;
    cudaFree(pd.flags); cudaFree(pd.peaks); cudaFree(pd.cands); cudaFree(pd.cand_count); cudaFree(pd.conns);
    cudaFree(pd.conn_count); cudaFree(pd.subset); cudaFree(pd.subset_rows); cudaFree(pd.joints); cudaFree(pd.num_people);
    cudaFreeHost(e->h_joints); cudaFreeHost(e->h_num_people); cudaFreeHost(e->h_peaks);
    for (cudaEvent_t ev : e->conv_done) if (ev) cudaEventDestroy(ev);
    if (e->stream2) { cudaStreamSynchronize(e->stream2); cudaStreamDestroy(e->stream2); }
    for (int i = 0; i < 16; i++) if (e->ev[i]) cudaEventDestroy(e->ev[i]);
    if (e->stream) cudaStreamDestroy(e->stream);
    delete e;
}

// ---------------------------------------------------------------------------------------------
// weights
// ---------------------------------------------------------------------------------------------
extern "C" int pe_num_conv_layers(const pe_engine* e) { return e ? (int)e->plan.convs.size() : 0; }
extern "C" int pe_conv_layer_info(const pe_engine* e, int idx, char* name64, int* cout, int* cin, int* ksize) {
    if (!e || idx < 0 || idx >= (int)e->plan.convs.size()) return PE_ERR_INVALID;
    const ConvSpec& c = e->plan.convs[idx];
    if (name64) snprintf(name64, 64, "%s", c.name.c_str());
    if (cout) *cout = c.cout;
    if (cin) *cin = c.cin;
    if (ksize) *ksize = c.k;
    return PE_OK;
}
extern "C" int pe_set_conv_weights(pe_engine* e, const char* layer_name, const float* w, size_t nw, const float* b, size_t nb) {
    if (!e || !layer_name || !w || !b) return fail(e, PE_ERR_INVALID, "null argument");
    for (size_t i = 0; i < e->plan.convs.size(); i++) {
        const ConvSpec& c = e->plan.convs[i];
        if (c.name != layer_name) continue;
        // shape mismatch is fatal in the reference (net.cpp:770-786)
        if (nw != (size_t)c.cout * c.cin * c.k * c.k || nb != (size_t)c.cout)
            return fail(e, PE_ERR_INVALID, "layer %s: expected %d x %d x %d x %d weights and %d biases", layer_name, c.cout, c.cin, c.k, c.k, c.cout);
        e->hw[i].w.assign(w, w + nw);
        e->hw[i].b.assign(b, b + nb);
        e->hw[i].set = true;
        e->committed = false;
        return PE_OK;
    }
    return PE_OK;  // unknown source layers are ignored (net.cpp:757-763)
}
extern "C" int pe_load_weights_file(pe_engine* e, const char* path) {
    if (!e || !path) return fail(e, PE_ERR_INVALID, "null argument");
    FILE* f = fopen(path, "rb");
    if (!f) return fail(e, PE_ERR_IO, "cannot open %s", path);
    char magic[4]; uint32_t hdr[2];
    if (fread(magic, 1, 4, f) != 4 || memcmp(magic, "RTPW", 4) || fread(hdr, 4, 2, f) != 2 || hdr[0] != 1) {
        fclose(f); return fail(e, PE_ERR_IO, "%s: not an RTPW v1 weight file", path);
    }
    fseek(f, 0, SEEK_END);
    const long long file_size = ftell(f);
    fseek(f, 12, SEEK_SET);
    for (uint32_t i = 0; i < hdr[1]; i++) {
        char name[64]; uint32_t dims[3];
        if (fread(name, 1, 64, f) != 64 || fread(dims, 4, 3, f) != 3) { fclose(f); return fail(e, PE_ERR_IO, "%s: truncated", path); }
        name[63] = 0;
        // the header is untrusted: the payload it announces must fit in the file before anything is allocated
        const unsigned long long nw64 = (unsigned long long)dims[0] * dims[1] * dims[2] * dims[2];
        if (dims[0] > (1u << 20) || dims[1] > (1u << 20) || dims[2] > 64 || (nw64 + dims[0]) * 4ull > (unsigned long long)(file_size - ftell(f))) {
            fclose(f);
            return fail(e, PE_ERR_IO, "%s: layer %s announces %u x %u x %u x %u weights, more than the file holds", path, name, dims[0], dims[1], dims[2], dims[2]);
        }
        const size_t nw = (size_t)nw64;
        std::vector<float> w(nw), b(dims[0]);
        if (fread(w.data(), 4, nw, f) != nw || fread(b.data(), 4, dims[0], f) != dims[0]) { fclose(f); return fail(e, PE_ERR_IO, "%s: truncated", path); }
        const int rc = pe_set_conv_weights(e, name, w.data(), nw, b.data(), b.size());
        if (rc) { fclose(f); return rc; }
    }
    fclose(f);
    return PE_OK;
}

static inline void split_bf16(float x, int planes, uint16_t* out) {
    float r = x;
    for (int p = 0; p < planes; p++) {
        uint32_t u; memcpy(&u, &r, 4);
        uint16_t h;
        if ((u & 0x7f800000u) == 0x7f800000u) h = (uint16_t)(u >> 16);
        else { const uint32_t lsb = (u >> 16) & 1u; h = (uint16_t)((u + 0x7fffu + lsb) >> 16); }  // RNE
        out[p] = h;
        const uint32_t hu = (uint32_t)h << 16; float hf; memcpy(&hf, &hu, 4);
        r = r - hf;
    }
}
static inline void split_fp16(float x, int planes, uint16_t* out) {   // IEEE fp16 planes (kernels.h)
    float r = x;
    for (int p = 0; p < planes; p++) {
        const __half h = __float2half_rn(r);
        out[p] = __half_as_ushort(h);
        r = r - __half2float(h);
    }
}

// byte layout of the packed weight buffer (a function of the plan and the precision only, so replicas agree on it)
static size_t packed_layout(pe_engine* e) {
    const size_t nc = e->plan.convs.size();
    e->w_off.assign(nc, 0); e->b_off.assign(nc, 0); e->cout_pad.assign(nc, 0); e->cin_pad.assign(nc, 0);
    size_t total = 0;
    auto align256 = [](size_t v) { return (v + 255) / 256 * 256; };
    for (size_t i = 0; i < nc; i++) {
        const ConvSpec& c = e->plan.convs[i];
        e->cin_pad[i] = c.in_cused;
        e->cout_pad[i] = e->fmt.planes ? tc_cout_pad(c.cout) : (c.cout + 63) / 64 * 64;
        const size_t K = (size_t)(c.im2col_input ? 1 : c.k * c.k) * e->cin_pad[i];
        e->w_off[i] = total;
        total = align256(total + K * e->cout_pad[i] * e->elem * (e->fmt.planes ? e->fmt.planes : 1));
        e->b_off[i] = total;
        total = align256(total + (size_t)(e->cout_pad[i] + 1) * 4);   // bias[cout_pad] + the layer's epilogue scale
    }
    e->w11_off = 0;
    if (nc && e->plan.convs[0].im2col_input && e->plan.convs[0].cout == 64 && e->plan.convs[0].k == 3) {
        e->w11_off = total;                                   // travels with the packed buffer (weight broadcast)
        total = align256(total + (27 * 64 + 64) * sizeof(float));
    }
    return total;
}

// Range scales.  Every conv output is stored as  true value * s  with s = conv_scale[producer] (a power of two; pools and copies
// pass values through unchanged).  A consumer whose input channels come from producers with DIFFERENT scales (a Concat: conv4_4_CPM
// next to the previous stage's L1 / L2 outputs) folds the ratios into its weights: packed w[ci] = w[ci] * s_ref / s(ci) * 2^k, so that
//   acc = 2^k * s_ref * sum_ci w[ci] * a[ci]     and     stored = acc * out_scale + bias,  out_scale = s_out / (2^k * s_ref),
// bias = true bias * s_out - all factors powers of two, hence exact, and ReLU commutes with them: range scaling is free at run time.
static float input_ref_scale(const pe_engine* e, const ConvSpec& c) {
    for (int pc : c.cin_prod) if (pc >= 0) return e->conv_scale[pc];
    return 1.f;   // the net input
}
static void fill_epilogue_fields(const pe_engine* e, int i, float* B) {
    const ConvSpec& c = e->plan.convs[i];
    const float s_ref = input_ref_scale(e, c);
    const float s_out = c.out_act >= 0 ? e->conv_scale[i] : 1.f;   // the planar stride-8 maps are true values
    for (int co = 0; co < c.cout; co++) B[co] = e->bias_true[i][co] * s_out;
    B[e->cout_pad[i]] = e->wsi[i] * s_out / s_ref;
}

// Weights of conv i into `dst` (the layer's region of the packed buffer, host copy): fp32 [K][cout_pad] for the SIMT mode, else
// P 16-bit planes [P][cout_pad][K] (K-major rows: the wgmma B operand) of w * 2^k, the per-channel range ratios folded in.
// Sets e->wsi[i] = 2^-k.
static void pack_conv_weights(pe_engine* e, int i, uint8_t* dst) {
    const ConvSpec& c = e->plan.convs[i];
    const HostWeights& hw = e->hw[i];
    const int taps = c.im2col_input ? 1 : c.k * c.k, cp = e->cin_pad[i], cop = e->cout_pad[i];
    const size_t K = (size_t)taps * cp;
    const float s_ref = input_ref_scale(e, c);
    std::vector<float> chan(cp, 1.f);   // s_ref / s(ci) per engine input channel
    for (int ec = 0; ec < cp && ec < (int)c.cin_prod.size(); ec++)
        if (c.cin_prod[ec] >= 0) chan[ec] = s_ref / e->conv_scale[c.cin_prod[ec]];
    auto src = [&](int co, int kk) -> float {  // engine K index -> Caffe weight (co, ci, r, s)
        if (c.im2col_input) {
            if (kk >= 27) return 0.f;
            const int tap = kk / 3, ci = kk % 3;
            return hw.w[((size_t)co * 3 + ci) * 9 + tap];
        }
        const int tap = kk / cp, ec = kk % cp;
        const int ci = ec < (int)c.cin_map.size() ? c.cin_map[ec] : -1;
        if (ci < 0) return 0.f;
        return hw.w[((size_t)co * c.cin + ci) * c.k * c.k + tap] * chan[ec];
    };
    memset(dst, 0, K * cop * e->elem * (e->fmt.planes ? e->fmt.planes : 1));
    float wscale_inv = 1.f;
    if (e->fmt.planes == 0) {  // fp32 [K][cout_pad]
        float* W = (float*)dst;
        for (size_t kk = 0; kk < K; kk++)
            for (int co = 0; co < c.cout; co++) W[kk * cop + co] = src(co, (int)kk);
    } else {
        uint16_t* W = (uint16_t*)dst;
        const size_t plane = (size_t)cop * K;
        // fp16 planes: scale the layer by 2^k so that max|w| lands in [2^13, 2^14) - small weights would otherwise
        // put their lo plane into fp16 subnormals.  Exact (power of two); the epilogue multiplies by 2^-k.
        float wscale = 1.f;
        if (e->fmt.f16) {
            float mx = 0.f;
            for (int co = 0; co < c.cout; co++)
                for (size_t kk = 0; kk < K; kk++) mx = fmaxf(mx, fabsf(src(co, (int)kk)));
            int ex = 0;
            if (mx > 0.f && mx < 3e38f) { frexpf(mx, &ex); wscale = ldexpf(1.f, std::max(-100, std::min(100, 14 - ex))); }
        }
        wscale_inv = 1.f / wscale;
        for (int co = 0; co < c.cout; co++)
            for (size_t kk = 0; kk < K; kk++) {
                uint16_t h[3];
                if (e->fmt.f16) split_fp16(src(co, (int)kk) * wscale, e->fmt.planes, h);
                else split_bf16(src(co, (int)kk), e->fmt.planes, h);
                for (int p = 0; p < e->fmt.planes; p++) W[p * plane + (size_t)co * K + kk] = h[p];
            }
    }
    e->wsi[i] = wscale_inv;
}

// per-layer launch state (TMA descriptors) over the packed buffer the handle currently points at
static int bind_packed(pe_engine* e) {
    const size_t nc = e->plan.convs.size();
    if (e->fmt.f16 && !e->d_range) {
        CK(e, cudaMalloc(&e->d_range, nc * sizeof(unsigned)));
        CK(e, cudaMemset(e->d_range, 0, nc * sizeof(unsigned)));
    }
    if (e->fmt.planes) {
        for (auto& t : e->tc) tc_layer_destroy(t);
        e->tc.assign(nc, TcLayer());
        for (size_t i = 0; i < nc; i++) {
            const ConvSpec& c = e->plan.convs[i];
            const Geo& g = e->geo[c.level];
            TcLayerDesc d;
            d.in = e->acts[c.in_act]; d.in_pitch = e->plan.acts[c.in_act].C; d.in_cused = c.in_cused; d.in_plane = e->act_plane[c.in_act];
            d.w = (char*)e->d_packed + e->w_off[i]; d.bias = (const float*)((char*)e->d_packed + e->b_off[i]);
            d.cout = c.cout; d.cout_pad = e->cout_pad[i]; d.ksize = c.im2col_input ? 1 : c.k; d.pad = c.im2col_input ? 0 : c.pad;
            d.relu = c.relu; d.fmt = e->fmt; d.geo = g; d.out_scale = d.bias + e->cout_pad[i];
            d.range = (e->fmt.f16 && e->d_range) ? e->d_range + i : nullptr;
            if (c.out_act >= 0) {
                d.out = e->acts[c.out_act]; d.out_pitch = e->plan.acts[c.out_act].C; d.out_coff = c.out_coff; d.out_plane = e->act_plane[c.out_act];
                d.planar = nullptr; d.planar_C = 0; d.planar_coff = 0;
            } else {
                d.out = nullptr; d.out_pitch = 0; d.out_coff = 0; d.out_plane = 0;
                d.planar = e->d_maps; d.planar_C = e->mt->num_maps; d.planar_coff = c.planar_coff;
            }
            std::string err;
            if (tc_layer_create(d, e->tc[i], err)) return fail(e, PE_ERR_CUDA, "layer %s: %s", c.name.c_str(), err.c_str());
        }
    }
    drop_graphs(e);
    e->committed = true;
    return PE_OK;
}

extern "C" int pe_commit_weights(pe_engine* e) {
    if (!e) return PE_ERR_INVALID;
    CK(e, cudaSetDevice(e->cfg.device));
    const size_t nc = e->plan.convs.size();
    for (size_t i = 0; i < nc; i++) {
        const ConvSpec& c = e->plan.convs[i];
        if (!e->hw[i].set || e->hw[i].w.size() != (size_t)c.cout * c.cin * c.k * c.k || e->hw[i].b.size() != (size_t)c.cout)
            return fail(e, PE_ERR_STATE, "weights of layer %s were never set%s", c.name.c_str(),
                        e->committed ? " on this handle (a broadcast replica keeps no fp32 copy: set every layer again)" : "");
    }
    const size_t total = packed_layout(e);
    e->bias_true.assign(nc, std::vector<float>());
    e->w11_scale = 1.f; e->calibrated = false;
    e->wsi.assign(nc, 1.f);
    e->conv_scale.assign(nc, 1.f);
    std::vector<uint8_t> host(total, 0);
    if (e->w11_off) {   // wT[k][co], k = c*9 + kh*3 + kw: Caffe's im2col row order (im2col.cpp:19-55)
        float* wT = (float*)(host.data() + e->w11_off);
        const HostWeights& h0 = e->hw[0];
        for (int co = 0; co < 64; co++) {
            for (int k = 0; k < 27; k++) wT[k * 64 + co] = h0.w[(size_t)co * 27 + k];
            wT[27 * 64 + co] = h0.b[co];
        }
    }
    for (size_t i = 0; i < nc; i++) {
        pack_conv_weights(e, (int)i, host.data() + e->w_off[i]);
        e->bias_true[i] = e->hw[i].b;
        fill_epilogue_fields(e, (int)i, (float*)(host.data() + e->b_off[i]));   // travels with the packed buffer (weight broadcast)
    }
    e->packed_owner.reset();
    e->d_packed = nullptr;
    void* dp = nullptr;
    CK(e, cudaMalloc(&dp, total));
    const int dev = e->cfg.device;
    e->packed_owner = std::shared_ptr<void>(dp, [dev](void* q) { int cur = 0; cudaGetDevice(&cur); cudaSetDevice(dev); cudaFree(q); cudaSetDevice(cur); });
    e->d_packed = dp;
    CK(e, cudaMemcpy(e->d_packed, host.data(), total, cudaMemcpyHostToDevice));
    e->packed_bytes = total;
    return bind_packed(e);
}

// Net::ShareTrainedLayersWith (src/caffe/net.cpp:682-706): a second net on the SAME GPU uses the first one's weights instead of
// loading them again - here the packed device buffer itself (no copy; it lives until the last handle that uses it is destroyed).
// For two worker handles per GPU (copies of one batch overlap the compute of the other, rtpose.bin --engines_per_gpu).
extern "C" int pe_share_weights(pe_engine* from, pe_engine* to) {
    if (!from || !to || from == to) return fail(from, PE_ERR_INVALID, "bad arguments");
    if (!from->committed) return fail(from, PE_ERR_STATE, "the source handle has no committed weights");
    if (to->cfg.device != from->cfg.device) return fail(from, PE_ERR_INVALID, "handles are on different GPUs (use pe_broadcast_weights)");
    if (to->cfg.model != from->cfg.model || to->cfg.precision != from->cfg.precision || to->plan.convs.size() != from->plan.convs.size())
        return fail(from, PE_ERR_INVALID, "the handles run different nets (model / precision / graph)");
    for (size_t i = 0; i < to->plan.convs.size(); i++) {
        const ConvSpec &a = from->plan.convs[i], &b = to->plan.convs[i];
        if (a.name != b.name || a.cout != b.cout || a.cin != b.cin || a.k != b.k) return fail(from, PE_ERR_INVALID, "layer %s differs between the handles", a.name.c_str());
    }
    CK(to, cudaSetDevice(to->cfg.device));
    CK(to, cudaStreamSynchronize(to->stream));
    if (packed_layout(to) != from->packed_bytes) return fail(from, PE_ERR_STATE, "packed layouts differ");
    to->packed_owner = from->packed_owner;
    to->d_packed = from->d_packed;
    to->packed_bytes = from->packed_bytes;
    for (auto& h : to->hw) { std::vector<float>().swap(h.w); std::vector<float>().swap(h.b); h.set = false; }
    to->conv_scale = from->conv_scale; to->calibrated = from->calibrated; to->bias_true.clear();
    return bind_packed(to);
}

// ---------------------------------------------------------------------------------------------
// One-time weight replica broadcast inside ONE process (rtpose.bin --num_gpu N).  The reference reads and parses the
// .caffemodel once per GPU (rtpose.cpp:183-184); here engines[0]'s packed device buffer goes to every other GPU with
// one grouped ncclBroadcast over NVLink.  This is the path's only collective.  NCCL is dlopen'ed (no link-time
// dependency, and a process that already carries torch's NCCL keeps using that one).
// ---------------------------------------------------------------------------------------------
#include <dlfcn.h>
typedef struct ncclComm* pe_ncclComm_t;
extern "C" int pe_broadcast_weights(pe_engine* const* engines, int n) {
    if (!engines || n < 1 || !engines[0]) return PE_ERR_INVALID;
    pe_engine* root = engines[0];
    if (!root->committed) return fail(root, PE_ERR_STATE, "engines[0] has no committed weights to broadcast");
    if (n == 1) return PE_OK;
    for (int i = 1; i < n; i++) {
        pe_engine* e = engines[i];
        if (!e || e->cfg.model != root->cfg.model || e->cfg.precision != root->cfg.precision || e->cfg.net_w != root->cfg.net_w ||
            e->cfg.net_h != root->cfg.net_h)
            return fail(root, PE_ERR_INVALID, "engine %d is not a replica of engine 0 (model / precision / net size differ)", i);
        if (!e->committed) {   // allocate the packed buffer + TMA maps with the same layout (values arrive by broadcast)
            for (size_t l = 0; l < e->plan.convs.size(); l++) {
                const ConvSpec& c = e->plan.convs[l];
                e->hw[l].w.assign((size_t)c.cout * c.cin * c.k * c.k, 0.f);
                e->hw[l].b.assign(c.cout, 0.f);
                e->hw[l].set = true;
            }
            const int rc = pe_commit_weights(e);
            if (rc) return rc;
            // the replica holds no fp32 copy: a later pe_set_conv_weights on a subset + pe_commit_weights must fail
            // ("weights of layer ... were never set") instead of packing from empty vectors
            for (auto& h : e->hw) { std::vector<float>().swap(h.w); std::vector<float>().swap(h.b); h.set = false; }
        }
        if (e->packed_bytes != root->packed_bytes) return fail(root, PE_ERR_STATE, "packed layouts differ");
    }
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return fail(root, PE_ERR_STATE, "NCCL is not available (%s)", dlerror());
    typedef int (*InitAllFn)(pe_ncclComm_t*, int, const int*);
    typedef int (*BcastFn)(const void*, void*, size_t, int, int, pe_ncclComm_t, cudaStream_t);
    typedef int (*VoidFn)(void);
    typedef int (*DestroyFn)(pe_ncclComm_t);
    typedef const char* (*ErrFn)(int);
    InitAllFn init_all = (InitAllFn)dlsym(h, "ncclCommInitAll");
    BcastFn bcast = (BcastFn)dlsym(h, "ncclBroadcast");
    VoidFn gstart = (VoidFn)dlsym(h, "ncclGroupStart"), gend = (VoidFn)dlsym(h, "ncclGroupEnd");
    DestroyFn destroy = (DestroyFn)dlsym(h, "ncclCommDestroy");
    ErrFn errstr = (ErrFn)dlsym(h, "ncclGetErrorString");
    if (!init_all || !bcast || !gstart || !gend || !destroy) return fail(root, PE_ERR_STATE, "NCCL symbols missing");
    std::vector<int> devs(n);
    for (int i = 0; i < n; i++) devs[i] = engines[i]->cfg.device;
    std::vector<pe_ncclComm_t> comms(n, nullptr);
    int rc = init_all(comms.data(), n, devs.data());
    if (rc) return fail(root, PE_ERR_CUDA, "ncclCommInitAll: %s", errstr ? errstr(rc) : "error");
    gstart();
    for (int i = 0; i < n && !rc; i++) {
        cudaSetDevice(devs[i]);
        rc = bcast(root->d_packed, engines[i]->d_packed, root->packed_bytes, 0 /*ncclChar*/, 0, comms[i], engines[i]->stream);
    }
    const int rc2 = gend();
    for (int i = 0; i < n; i++) { cudaSetDevice(devs[i]); cudaStreamSynchronize(engines[i]->stream); }
    for (int i = 0; i < n; i++) destroy(comms[i]);
    if (rc || rc2) return fail(root, PE_ERR_CUDA, "ncclBroadcast: %s", errstr ? errstr(rc ? rc : rc2) : "error");
    return PE_OK;
}

extern "C" size_t pe_packed_weights_bytes(const pe_engine* e) { return e ? e->packed_bytes : 0; }
extern "C" void* pe_packed_weights_device_ptr(pe_engine* e) { return e ? e->d_packed : nullptr; }

// ---------------------------------------------------------------------------------------------
// layer accessors
// ---------------------------------------------------------------------------------------------
static void drop_graphs(pe_engine* e) {
    for (auto& kv : e->graphs) if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
    e->graphs.clear();
}

extern "C" int pe_nms_get_max_peaks(const pe_engine* e) { return e ? e->mt->max_peaks : 0; }
extern "C" int pe_nms_get_num_parts(const pe_engine* e) { return e ? e->mt->num_parts : 0; }
extern "C" float pe_nms_get_threshold(const pe_engine* e) { return e ? e->post.p.nms_threshold : 0.f; }
extern "C" int pe_nms_set_threshold(pe_engine* e, float t) {
    if (!e) return PE_ERR_INVALID;
    if (e->post.p.nms_threshold != t) drop_graphs(e);
    e->post.p.nms_threshold = t;
    return PE_OK;
}
static int rebuild_axis(pe_engine* e) {
    CK(e, cudaSetDevice(e->cfg.device));
    e->post.p.start_scale = e->start_scale_f; e->post.p.scale_gap = e->scale_gap_f;
    drop_graphs(e);
    launch_axis_tables(e->d_xtab, e->d_ytab, e->post.p, e->stream);
    e->launches += 2;
    return PE_OK;
}
extern "C" int pe_resize_set_start_scale(pe_engine* e, float s) { if (!e) return PE_ERR_INVALID; e->start_scale_f = s; return rebuild_axis(e); }
extern "C" int pe_resize_set_scale_gap(pe_engine* e, float g) { if (!e) return PE_ERR_INVALID; e->scale_gap_f = g; return rebuild_axis(e); }
extern "C" float pe_resize_get_start_scale(const pe_engine* e) { return e ? e->start_scale_f : 0.f; }
extern "C" float pe_resize_get_scale_gap(const pe_engine* e) { return e ? e->scale_gap_f : 0.f; }
extern "C" int pe_set_connect_params(pe_engine* e, int min_cnt, float min_score, float inter_thr, int min_above) {
    if (!e) return PE_ERR_INVALID;
    PostParams& p = e->post.p;
    drop_graphs(e);
    p.min_subset_cnt = min_cnt; p.min_subset_score = min_score; p.inter_threshold = inter_thr; p.inter_min_above = min_above;
    return PE_OK;
}

// ---------------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------------
static int run_op(pe_engine* e, const OpRef& op, int nimg, cudaStream_t st = nullptr, int share = 1) {
    if (!st) st = e->stream;
    if (op.type == 0) {
        const ConvSpec& c = e->plan.convs[op.idx];
        const Geo& g = e->geo[c.level];
        const long long M = (long long)nimg * g.Hs * g.Wp;
        if (op.idx == 0 && c.im2col_input && e->conv11_direct && e->input_from_frames && e->w11_off && c.out_act >= 0) {
            PreArgs a = e->pre;
            a.nframes = nimg / e->cfg.num_scales;
            const float* wT = (const float*)((const char*)e->d_packed + e->w11_off);
            e->launches += launch_conv1_1_direct(a, wT, wT + 27 * 64, e->acts[c.out_act], e->plan.acts[c.out_act].C, e->act_plane[c.out_act],
                                                 c.relu, nimg, st);
            return PE_OK;
        }
        if (e->fmt.planes) {
            const int n = tc_layer_launch(e->tc[op.idx], nimg, st, share);
            if (n < 0) return fail(e, PE_ERR_CUDA, "conv %s: tensor-core launch failed or no kernel fits the tile (%s)", c.name.c_str(), cudaGetErrorString(cudaGetLastError()));
            e->launches += n;
            return PE_OK;
        }
        ConvArgs a;
        memset(&a, 0, sizeof a);
        a.in = e->acts[c.in_act]; a.in_pitch = e->plan.acts[c.in_act].C;
        a.w = (char*)e->d_packed + e->w_off[op.idx]; a.bias = (const float*)((char*)e->d_packed + e->b_off[op.idx]);
        if (c.out_act >= 0) { a.out = e->acts[c.out_act]; a.out_pitch = e->plan.acts[c.out_act].C; a.out_coff = c.out_coff; }
        else { a.planar = e->d_maps; a.planar_C = e->mt->num_maps; a.planar_coff = c.planar_coff; }
        a.cin_pad = e->cin_pad[op.idx]; a.cout = c.cout; a.cout_pad = e->cout_pad[op.idx];
        a.ksize = c.im2col_input ? 1 : c.k; a.pad = c.im2col_input ? 0 : c.pad; a.relu = c.relu;
        a.W = g.W; a.H = g.H; a.Wp = g.Wp; a.Hs = g.Hs; a.N = nimg; a.M = M;
        e->launches += launch_conv_simt(a, st);
    } else if (op.type == 1) {
        const PoolSpec& p = e->plan.pools[op.idx];
        const Geo& gi = e->geo[p.level_in]; const Geo& go = e->geo[p.level_in + 1];
        PoolArgs a;
        a.in = e->acts[p.in_act]; a.out = e->acts[p.out_act]; a.C = e->plan.acts[p.in_act].C;
        a.in_plane = e->act_plane[p.in_act]; a.out_plane = e->act_plane[p.out_act]; a.fmt = e->fmt;
        a.Wi = gi.W; a.Hi = gi.H; a.Wpi = gi.Wp; a.Hsi = gi.Hs; a.Wo = go.W; a.Ho = go.H; a.Wpo = go.Wp; a.Hso = go.Hs; a.N = nimg;
        e->launches += launch_pool(a, st);
    } else {
        const CopySpec& c = e->plan.copies[op.idx];
        const Geo& g = e->geo[3];
        CopyArgs a;
        a.src = e->acts[c.src_act]; a.dst = e->acts[c.dst_act]; a.pitch = e->plan.acts[c.src_act].C; a.channels = c.channels;
        a.elem_bytes = e->elem; a.M = (long long)nimg * g.Hs * g.Wp; a.plane = e->act_plane[c.src_act]; a.fmt = e->fmt;
        e->launches += launch_copy_channels(a, st);
    }
    return PE_OK;
}

static int run_post_and_return(pe_engine* e, int n) {
    e->post.maps = e->d_maps;
    e->launches += launch_post(e->post, n, e->stream);
    const int P = e->mt->num_parts, MP = e->mt->max_peaks;
    CK(e, cudaMemcpyAsync(e->h_joints, e->post.joints, sizeof(float) * (size_t)n * PE_MAX_PEOPLE * P * 3, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaMemcpyAsync(e->h_num_people, e->post.num_people, sizeof(int) * n, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaMemcpyAsync(e->h_peaks, e->post.peaks, sizeof(float) * (size_t)n * P * (MP + 1) * 3, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaGetLastError());
    e->last_n = n;
    e->jstatus_n = 0;
    return PE_OK;
}

static int run_net_eager(pe_engine* e, int n) {
    NvtxRange r("pe: conv stack + parse");
    const int nimg = n * e->cfg.num_scales;
    if (!e->two_lanes) {
        for (const OpRef& op : e->plan.order) { const int rc = run_op(e, op, nimg); if (rc) return rc; }
        return run_post_and_return(e, n);
    }
    // two lanes: an op waits for the convs of the other lane it reads from (events), everything else is stream order
    for (size_t k = 0; k < e->plan.order.size(); k++) {
        const OpRef& op = e->plan.order[k];
        cudaStream_t st = e->op_lane[k] ? e->stream2 : e->stream;
        for (int pc : e->op_waits[k]) CK(e, cudaStreamWaitEvent(st, e->conv_done[pc], 0));
        const int rc = run_op(e, op, nimg, st, 2);
        if (rc) return rc;
        if (op.type == 0 && e->conv_done[op.idx]) CK(e, cudaEventRecord(e->conv_done[op.idx], st));
    }
    if (e->last_lane1_conv >= 0) CK(e, cudaStreamWaitEvent(e->stream, e->conv_done[e->last_lane1_conv], 0));   // join before the parse stage
    return run_post_and_return(e, n);
}

// Lane assignment and cross-lane dependencies of the plan (branch *_L2 -> lane 1).  Enabled when every lane-1 op is a conv whose
// inputs come from convs (through pools / copies / concat slices) - true for the pose_deploy_linevec family.
static int setup_lanes(pe_engine* e) {
    const NetPlan& p = e->plan;
    const size_t nc = p.convs.size();
    e->op_lane.assign(p.order.size(), 0);
    e->op_waits.assign(p.order.size(), std::vector<int>());
    e->conv_done.assign(nc, nullptr);
    e->last_lane1_conv = -1;
    e->two_lanes = false;
    if (const char* g = getenv("PE_TWO_LANES")) { if (atoi(g) == 0) return PE_OK; }
    std::vector<int> conv_lane(nc, 0);
    int n1 = 0;
    for (size_t i = 0; i < nc; i++) {
        const std::string& nm = p.convs[i].name;
        if (nm.size() > 3 && nm.compare(nm.size() - 3, 3, "_L2") == 0) { conv_lane[i] = 1; n1++; }
    }
    if (!n1) return PE_OK;
    std::vector<char> need_event(nc, 0);
    for (size_t k = 0; k < p.order.size(); k++) {
        const OpRef& op = p.order[k];
        if (op.type != 0) continue;                         // pools and the F copy stay on lane 0 (the trunk)
        const int lane = conv_lane[op.idx];
        e->op_lane[k] = lane;
        if (lane) e->last_lane1_conv = op.idx;
        std::vector<int>& w = e->op_waits[k];
        for (int pc : p.convs[op.idx].cin_prod)
            if (pc >= 0 && conv_lane[pc] != lane && std::find(w.begin(), w.end(), pc) == w.end()) { w.push_back(pc); need_event[pc] = 1; }
    }
    // (The copy of the shared blob into the second concat buffer follows its producer on lane 0; the first lane-1 reader of that
    // buffer also waits for a lane-0 conv of the previous stage, which is behind the copy in stream order.)
    if (e->last_lane1_conv >= 0) need_event[e->last_lane1_conv] = 1;
    CK(e, cudaStreamCreateWithFlags(&e->stream2, cudaStreamNonBlocking));
    for (size_t i = 0; i < nc; i++)
        if (need_event[i]) CK(e, cudaEventCreateWithFlags(&e->conv_done[i], cudaEventDisableTiming));
    e->two_lanes = true;
    return PE_OK;
}

static int run_net(pe_engine* e, int n) {
    if (!e->committed) return fail(e, PE_ERR_STATE, "pe_commit_weights has not been called");
    if (!e->use_graphs) return run_net_eager(e, n);
    pe_engine::GraphEntry& g = e->graphs[n];
    if (g.exec) {
        CK(e, cudaGraphLaunch(g.exec, e->stream));
        e->launches += g.launches;
        e->last_n = n;
        e->jstatus_n = 0;
        return PE_OK;
    }
    if (g.seen++ == 0) return run_net_eager(e, n);   // first use of this batch size: eager (sets kernel attributes)
    // second use: capture the same sequence into a graph and launch it
    const long long before = e->launches;
    if (cudaStreamBeginCapture(e->stream, cudaStreamCaptureModeThreadLocal) != cudaSuccess) {
        cudaGetLastError();
        e->use_graphs = false;
        return run_net_eager(e, n);
    }
    const int rc = run_net_eager(e, n);
    cudaGraph_t graph = nullptr;
    const cudaError_t ce = cudaStreamEndCapture(e->stream, &graph);
    if (rc || ce != cudaSuccess || !graph) {
        cudaGetLastError();
        if (graph) cudaGraphDestroy(graph);
        e->launches = before;
        e->use_graphs = false;
        if (rc) return rc;
        return run_net_eager(e, n);
    }
    g.launches = e->launches - before;
    e->launches = before;
    const cudaError_t ie = cudaGraphInstantiate(&g.exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ie != cudaSuccess) { cudaGetLastError(); g.exec = nullptr; e->use_graphs = false; return run_net_eager(e, n); }
    CK(e, cudaGraphLaunch(g.exec, e->stream));
    e->launches += g.launches;
    e->last_n = n;
    e->jstatus_n = 0;
    return PE_OK;
}

static int check_n(pe_engine* e, int n) {
    if (!e) return PE_ERR_INVALID;
    if (n < 1 || n > e->cfg.max_batch) return fail(e, PE_ERR_INVALID, "n=%d outside [1, max_batch=%d]", n, e->cfg.max_batch);
    return PE_OK;
}

extern "C" int pe_forward_frames_device(pe_engine* e, const void* d_frames, int n) {
    NvtxRange r("pe_forward_frames_device");
    int rc = check_n(e, n); if (rc) return rc;
    CK(e, cudaSetDevice(e->cfg.device));
    PreArgs a = e->pre;
    a.frames = (const uint8_t*)d_frames; a.nframes = n;
    if (e->input_lo_dirty) {   // the uint8 path only writes the hi plane; drop what the planar path left behind
        const size_t bytes = (size_t)e->act_plane[e->plan.input_act] * e->elem * (e->fmt.planes ? e->fmt.planes : 1);
        CK(e, cudaMemsetAsync(e->acts[e->plan.input_act], 0, bytes, e->stream));
        e->input_lo_dirty = false;
    }
    const bool direct = e->conv11_direct && e->w11_off && e->plan.convs[0].out_act >= 0;
    e->launches += launch_preprocess(a, e->stream, !direct);
    if (!e->input_from_frames) drop_graphs(e);   // graphs captured on the planar-input path hold the other conv1_1 kernel
    e->input_from_frames = true;
    e->input_act_stale = direct;
    e->last_frames = (const uint8_t*)d_frames;
    return run_net(e, n);
}
extern "C" int pe_forward_frames(pe_engine* e, const uint8_t* const* frames, int n) {
    NvtxRange r("pe_forward_frames (H2D)");
    int rc = check_n(e, n); if (rc) return rc;
    if (!frames) return fail(e, PE_ERR_INVALID, "null frames");
    CK(e, cudaSetDevice(e->cfg.device));
    const size_t fb = (size_t)e->cfg.disp_w * e->cfg.disp_h * 3;
    // Page-locked caller buffers are DMA'd directly (fully asynchronous); pageable ones go through the
    // engine's pinned staging buffer, which forces a stream sync because that buffer is reused.
    bool pinned = true;
    for (int i = 0; i < n && pinned; i++) {
        cudaPointerAttributes at;
        if (!frames[i]) return fail(e, PE_ERR_INVALID, "null frame %d", i);
        if (cudaPointerGetAttributes(&at, frames[i]) != cudaSuccess || at.type != cudaMemoryTypeHost) { pinned = false; cudaGetLastError(); }
    }
    if (pinned) {
        for (int i = 0; i < n; i++)
            CK(e, cudaMemcpyAsync(e->d_frames + i * fb, frames[i], fb, cudaMemcpyHostToDevice, e->stream));
    } else {
        CK(e, cudaStreamSynchronize(e->stream));
        for (int i = 0; i < n; i++) memcpy(e->h_frames + i * fb, frames[i], fb);
        CK(e, cudaMemcpyAsync(e->d_frames, e->h_frames, fb * n, cudaMemcpyHostToDevice, e->stream));
    }
    return pe_forward_frames_device(e, e->d_frames, n);
}
// bicubic weight table of OpenCV's fixed-point remap (initInterTab2D(INTER_CUBIC, fixpt)): a = -0.75, 15-bit shorts,
// each 4x4 kernel normalised to sum 2^15 by nudging the largest/smallest central coefficient
static void build_warp_tab(std::vector<short>& tab) {
    tab.assign(32 * 32 * 16, 0);
    float t1[32][4];
    const float A = -0.75f, scale = 1.f / 32;
    for (int i = 0; i < 32; i++) {
        const float x = i * scale;
        t1[i][0] = ((A * (x + 1) - 5 * A) * (x + 1) + 8 * A) * (x + 1) - 4 * A;
        t1[i][1] = ((A + 2) * x - (A + 3)) * x * x + 1;
        t1[i][2] = ((A + 2) * (1 - x) - (A + 3)) * (1 - x) * (1 - x) + 1;
        t1[i][3] = 1.f - t1[i][0] - t1[i][1] - t1[i][2];
    }
    for (int i = 0; i < 32; i++)
        for (int j = 0; j < 32; j++) {
            short* w = tab.data() + (i * 32 + j) * 16;
            int isum = 0;
            for (int k = 0; k < 16; k++) {
                long r = lrintf(t1[i][k / 4] * t1[j][k % 4] * 32768.f);
                w[k] = (short)std::min(32767L, std::max(-32768L, r));
                isum += w[k];
            }
            if (isum != 32768) {
                int hi = 10, lo = 10;   // central 2x2 = indices 10, 11, 14, 15
                const int cen[4] = {10, 11, 14, 15};
                for (int c : cen) { if (w[c] < w[lo]) lo = c; else if (w[c] > w[hi]) hi = c; }
                if (isum < 32768) w[hi] = (short)(w[hi] - (isum - 32768));
                else w[lo] = (short)(w[lo] - (isum - 32768));
            }
        }
}

static int prepare_warp(pe_engine* e, int ow, int oh) {
    if (e->warp_w == ow && e->warp_h == oh && e->d_wa) return PE_OK;
    const int dw = e->cfg.disp_w, dh = e->cfg.disp_h;
    // rtpose.cpp:474-480
    const double s = (ow / (double)oh > dw / (double)dh) ? dw / (double)ow : dh / (double)oh;
    double M[6] = {s, 0, 0, 0, s, 0};
    double D = M[0] * M[4] - M[1] * M[3];
    D = D != 0 ? 1. / D : 0;
    const double A11 = M[4] * D, A22 = M[0] * D;
    M[0] = A11; M[1] *= -D; M[3] *= -D; M[4] = A22;
    const double b1 = -M[0] * M[2] - M[1] * M[5], b2 = -M[3] * M[2] - M[4] * M[5];
    M[2] = b1; M[5] = b2;
    std::vector<int> ad(dw), bd(dw), x0(dh), y0(dh);
    for (int x = 0; x < dw; x++) { ad[x] = (int)lrint(M[0] * x * 1024); bd[x] = (int)lrint(M[3] * x * 1024); }
    for (int y = 0; y < dh; y++) { x0[y] = (int)lrint((M[1] * y + M[2]) * 1024) + 16; y0[y] = (int)lrint((M[4] * y + M[5]) * 1024) + 16; }
    if (!e->d_wa) {
        std::vector<short> tab;
        build_warp_tab(tab);
        CK(e, cudaMalloc(&e->d_wa, dw * sizeof(int))); CK(e, cudaMalloc(&e->d_wb, dw * sizeof(int)));
        CK(e, cudaMalloc(&e->d_wx0, dh * sizeof(int))); CK(e, cudaMalloc(&e->d_wy0, dh * sizeof(int)));
        CK(e, cudaMalloc(&e->d_wtab, tab.size() * sizeof(short)));
        CK(e, cudaMemcpy(e->d_wtab, tab.data(), tab.size() * sizeof(short), cudaMemcpyHostToDevice));
    }
    CK(e, cudaStreamSynchronize(e->stream));
    CK(e, cudaMemcpy(e->d_wa, ad.data(), dw * sizeof(int), cudaMemcpyHostToDevice));
    CK(e, cudaMemcpy(e->d_wb, bd.data(), dw * sizeof(int), cudaMemcpyHostToDevice));
    CK(e, cudaMemcpy(e->d_wx0, x0.data(), dh * sizeof(int), cudaMemcpyHostToDevice));
    CK(e, cudaMemcpy(e->d_wy0, y0.data(), dh * sizeof(int), cudaMemcpyHostToDevice));
    e->warp_w = ow; e->warp_h = oh; e->warp_scale = s;
    return PE_OK;
}

// (re)allocates *p to hold at least `need` bytes; the stream is drained first because queued work may still use the old buffer
static int grow_buffer(pe_engine* e, uint8_t** p, size_t* cap, size_t need, bool host) {
    if (*cap >= need) return PE_OK;
    CK(e, cudaStreamSynchronize(e->stream));
    if (host) { cudaFreeHost(*p); *p = nullptr; CK(e, cudaMallocHost((void**)p, need)); }
    else { cudaFree(*p); *p = nullptr; CK(e, cudaMalloc((void**)p, need)); }
    *cap = need;
    return PE_OK;
}

// Where the routes that read frames of any size (pixels, camera, JPEG) build their W x H BGR frames: the display frames themselves
// at the display size (*scale = 1), else the warpAffine source d_raw (*scale = frame.scale).  finish_frames warps d_raw into the
// display frames when needed and runs the net.
static int frame_target(pe_engine* e, int W, int H, uint8_t** dst, double* scale) {
    if (W == e->cfg.disp_w && H == e->cfg.disp_h) {
        *dst = e->d_frames;
        if (scale) *scale = 1.0;
        return PE_OK;
    }
    int rc = prepare_warp(e, W, H); if (rc) return rc;
    rc = grow_buffer(e, &e->d_raw, &e->raw_cap, (size_t)W * H * 3 * e->cfg.max_batch, false); if (rc) return rc;
    *dst = e->d_raw;
    if (scale) *scale = e->warp_scale;
    return PE_OK;
}
static int finish_frames(pe_engine* e, int n, int W, int H) {
    if (W != e->cfg.disp_w || H != e->cfg.disp_h) {
        WarpArgs w;
        w.src = e->d_raw; w.dst = e->d_frames; w.sw = W; w.sh = H; w.dw = e->cfg.disp_w; w.dh = e->cfg.disp_h;
        w.adelta = e->d_wa; w.bdelta = e->d_wb; w.x0 = e->d_wx0; w.y0 = e->d_wy0; w.tab = e->d_wtab;
        e->launches += launch_warp_affine(w, n, e->stream);
    }
    return pe_forward_frames_device(e, e->d_frames, n);
}

extern "C" int pe_forward_pixels(pe_engine* e, const pe_pixel_format* fmt, const void* const* frames, int n, double* scale) {
    NvtxRange r("pe_forward_pixels");
    int rc = check_n(e, n); if (rc) return rc;
    pe_pix::Layout L;
    std::string why;
    if (!pe_pix::layout_of(fmt, &L, &why)) return fail(e, PE_ERR_INVALID, "%s", why.c_str());
    if (!frames) return fail(e, PE_ERR_INVALID, "null frames");
    CK(e, cudaSetDevice(e->cfg.device));
    enum { DEVICE, PINNED, PAGEABLE };
    int kind[PIX_MAX_FRAMES];
    bool any_host = false, any_pageable = false;
    for (int i = 0; i < n; i++) {
        if (!frames[i]) return fail(e, PE_ERR_INVALID, "null frame %d", i);
        cudaPointerAttributes at;
        if (cudaPointerGetAttributes(&at, frames[i]) != cudaSuccess) { cudaGetLastError(); at.type = cudaMemoryTypeUnregistered; }
        if (at.type == cudaMemoryTypeDevice && at.device != e->cfg.device)
            return fail(e, PE_ERR_INVALID, "frame %d is device memory of GPU %d, the engine runs on GPU %d", i, at.device, e->cfg.device);
        kind[i] = at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged ? DEVICE : at.type == cudaMemoryTypeHost ? PINNED : PAGEABLE;
        any_host |= kind[i] != DEVICE;
        any_pageable |= kind[i] == PAGEABLE;
    }
    uint8_t* dst;
    rc = frame_target(e, L.w, L.h, &dst, scale); if (rc) return rc;
    const bool bgr = L.format == PE_PIX_BGR;
    const size_t fb = (size_t)L.w * L.h * 3, span = (size_t)L.span, stride = (span + 255) & ~(size_t)255;
    // Pageable frames are staged in h_raw, which the queued work may still be reading: the stream is drained first.  Host frames
    // other than BGR are copied whole to d_pix, and the kernel converts them there.
    if (any_pageable) {
        rc = grow_buffer(e, &e->h_raw, &e->h_raw_cap, stride * e->cfg.max_batch, true); if (rc) return rc;
        CK(e, cudaStreamSynchronize(e->stream));
    }
    if (any_host && !bgr) { rc = grow_buffer(e, &e->d_pix, &e->pix_cap, stride * e->cfg.max_batch, false); if (rc) return rc; }
    PixArgs a;
    a.dst = dst; a.pitch = L.pitch; a.chroma = L.chroma; a.format = L.format; a.w = L.w; a.h = L.h;
    for (int i = 0; i < n; i++) {
        const uint8_t* src = (const uint8_t*)frames[i];
        if (kind[i] == PAGEABLE) { memcpy(e->h_raw + i * stride, src, span); src = e->h_raw + i * stride; }
        if (bgr) {   // BGR needs no conversion: the copy into place drops the pitch
            CK(e, cudaMemcpy2DAsync(dst + i * fb, (size_t)L.w * 3, src, (size_t)L.pitch, (size_t)L.w * 3, L.h, cudaMemcpyDefault, e->stream));
        } else if (kind[i] == DEVICE) {
            a.src[i] = src;
        } else {
            CK(e, cudaMemcpyAsync(e->d_pix + i * stride, src, span, cudaMemcpyHostToDevice, e->stream));
            a.src[i] = e->d_pix + i * stride;
        }
    }
    if (!bgr) e->launches += launch_pixels_to_bgr(a, n, e->stream);
    return finish_frames(e, n, L.w, L.h);
}

extern "C" int pe_forward_camera_frames(pe_engine* e, const uint8_t* const* frames, int n, int orig_w, int orig_h, double* scale) {
    const pe_pixel_format f = {PE_PIX_BGR, orig_w, orig_h, 0, 0};
    return pe_forward_pixels(e, &f, (const void* const*)frames, n, scale);
}

extern "C" int pe_stream_wait(pe_engine* e, void* cuda_stream) {
    if (!e) return PE_ERR_INVALID;
    CK(e, cudaSetDevice(e->cfg.device));
    if (!e->ev_wait) CK(e, cudaEventCreateWithFlags(&e->ev_wait, cudaEventDisableTiming));
    CK(e, cudaEventRecord(e->ev_wait, cuda_stream ? (cudaStream_t)cuda_stream : cudaStreamLegacy));
    CK(e, cudaStreamWaitEvent(e->stream, e->ev_wait, 0));
    return PE_OK;
}

extern "C" int pe_pixels_to_bgr(const pe_pixel_format* fmt, const void* frame, uint8_t* bgr, long long cap) {
    pe_pix::Layout L;
    std::string why;
    if (!pe_pix::layout_of(fmt, &L, &why)) return fail(nullptr, PE_ERR_INVALID, "%s", why.c_str());
    if (!frame || !bgr) return fail(nullptr, PE_ERR_INVALID, "null frame or output");
    if (cap < 3LL * L.w * L.h) return fail(nullptr, PE_ERR_INVALID, "cap %lld is below the %lld bytes of the BGR frame", cap, 3LL * L.w * L.h);
    PixArgs a;
    a.src[0] = (const uint8_t*)frame; a.dst = bgr; a.pitch = L.pitch; a.chroma = L.chroma; a.format = L.format; a.w = L.w; a.h = L.h;
    pixels_to_bgr_host(a);
    return PE_OK;
}

static int reconstruct_and_forward(pe_engine* e, int n, int W, int H, size_t stride, long long max_blocks, double* scale);

extern "C" int pe_forward_jpeg_coefs(pe_engine* e, const void* const* coefs, int n, double* scale) {
    NvtxRange r("pe_forward_jpeg_coefs (H2D + reconstruction)");
    int rc = check_n(e, n); if (rc) return rc;
    if (!coefs) return fail(e, PE_ERR_INVALID, "null coefficient images");
    CK(e, cudaSetDevice(e->cfg.device));
    // the kernels index with the headers' numbers: every header must be one pe_jpeg_read_coefs writes, all frames one size
    int W = 0, H = 0;
    long long max_bytes = 0, max_blocks = 0;
    std::vector<long long> bytes(n);
    for (int i = 0; i < n; i++) {
        if (!coefs[i]) return fail(e, PE_ERR_INVALID, "null coefficient image %d", i);
        pe_jpeg_coef_header hd;
        memcpy(&hd, coefs[i], sizeof hd);
        if (!pe_jpeg::coef_header_valid(hd)) return fail(e, PE_ERR_INVALID, "coefficient image %d: not a pe_jpeg_read_coefs header", i);
        if (i == 0) { W = hd.width; H = hd.height; }
        else if (hd.width != W || hd.height != H)
            return fail(e, PE_ERR_INVALID, "coefficient image %d is %dx%d, frame 0 %dx%d: one size per call", i, hd.width, hd.height, W, H);
        bytes[i] = hd.total_bytes;
        max_bytes = std::max(max_bytes, (long long)hd.total_bytes);
        max_blocks = std::max(max_blocks, (long long)(hd.total_bytes - (long long)sizeof hd) / 128);
    }
    const size_t stride = ((size_t)max_bytes + 255) & ~(size_t)255;
    rc = grow_buffer(e, &e->d_jcoef, &e->jcoef_cap, stride * n, false); if (rc) return rc;
    // page-locked caller buffers (pe_host_alloc) are DMA'd directly; pageable ones are staged, which drains the stream
    bool pinned = true;
    for (int i = 0; i < n && pinned; i++) {
        cudaPointerAttributes at;
        if (cudaPointerGetAttributes(&at, coefs[i]) != cudaSuccess || at.type != cudaMemoryTypeHost) { pinned = false; cudaGetLastError(); }
    }
    if (pinned) {
        for (int i = 0; i < n; i++) CK(e, cudaMemcpyAsync(e->d_jcoef + i * stride, coefs[i], bytes[i], cudaMemcpyHostToDevice, e->stream));
    } else {
        CK(e, cudaStreamSynchronize(e->stream));
        rc = grow_buffer(e, &e->h_jcoef, &e->h_jcoef_cap, stride * n, true); if (rc) return rc;
        for (int i = 0; i < n; i++) memcpy(e->h_jcoef + i * stride, coefs[i], bytes[i]);
        CK(e, cudaMemcpyAsync(e->d_jcoef, e->h_jcoef, stride * n, cudaMemcpyHostToDevice, e->stream));
    }
    return reconstruct_and_forward(e, n, W, H, stride, max_blocks, scale);
}

// coefficient images in e->d_jcoef (n frames of W x H, `stride` bytes apart) -> display frames -> the net
static int reconstruct_and_forward(pe_engine* e, int n, int W, int H, size_t stride, long long max_blocks, double* scale) {
    uint8_t* dst;
    int rc = frame_target(e, W, H, &dst, scale); if (rc) return rc;
    const size_t pstride = ((size_t)max_blocks * 64 + 255) & ~(size_t)255;
    rc = grow_buffer(e, &e->d_jplanes, &e->jplanes_cap, pstride * n, false); if (rc) return rc;
    JpegArgs ja;
    ja.coefs = e->d_jcoef; ja.coef_stride = (long long)stride; ja.planes = e->d_jplanes; ja.plane_stride = (long long)pstride;
    ja.dst = dst; ja.W = W; ja.H = H; ja.n = n; ja.max_blocks = max_blocks;
    e->launches += launch_jpeg_reconstruct(ja, e->stream);
    return finish_frames(e, n, W, H);
}

// Scan images -> coefficient images in e->d_jcoef (the entropy kernels), the per-frame status queued into e->h_jstatus.  Everything the
// kernels index with is checked here first; the launch shapes come from these sizes, so nothing waits for the device.
static int decode_scans(pe_engine* e, const void* const* scans, int n, int S, int* W, int* H, size_t* cstride, long long* max_blocks) {
    if (!scans) return fail(e, PE_ERR_INVALID, "null scan images");
    if (S < 8 || S > (1 << 30)) return fail(e, PE_ERR_INVALID, "subsequence length %d bits outside [8, 2^30]", S);
    long long max_scan = 0, max_coef = 0, max_seg = 0, max_sub = 0;
    std::vector<long long> bytes(n);
    for (int i = 0; i < n; i++) {
        if (!scans[i]) return fail(e, PE_ERR_INVALID, "null scan image %d", i);
        const pe_jpeg_scan_header& hd = *(const pe_jpeg_scan_header*)scans[i];
        long long subs = 0;
        if (!pe_jpeg::scan_header_valid(hd, S, &subs)) return fail(e, PE_ERR_INVALID, "scan image %d: not a pe_jpeg_read_scan image", i);
        if (i == 0) { *W = hd.coef.width; *H = hd.coef.height; }
        else if (hd.coef.width != *W || hd.coef.height != *H)
            return fail(e, PE_ERR_INVALID, "scan image %d is %dx%d, frame 0 %dx%d: one size per call", i, hd.coef.width, hd.coef.height, *W, *H);
        bytes[i] = hd.total_bytes;
        max_scan = std::max(max_scan, (long long)hd.total_bytes);
        max_coef = std::max(max_coef, (long long)hd.coef.total_bytes);
        max_blocks[0] = std::max(max_blocks[0], (long long)(hd.coef.total_bytes - (long long)sizeof hd.coef) / 128);
        max_seg = std::max(max_seg, (long long)hd.num_segments);
        max_sub = std::max(max_sub, subs);
    }
    auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
    const size_t sstride = al((size_t)max_scan);
    *cstride = al((size_t)max_coef);
    const int ctas = (int)((max_sub + pe_jpeg::SYNC_THREADS - 1) / pe_jpeg::SYNC_THREADS);
    const size_t tab_b = al(jpeg_huff_tables_bytes() * n), seg_b = al((size_t)(max_seg + 1) * 4 * n), pub_b = al((size_t)ctas * 16 * n),
                 flag_b = al((size_t)ctas * 4 * n), small_b = al((size_t)4 * n);
    int rc = grow_buffer(e, &e->d_jcoef, &e->jcoef_cap, *cstride * n, false); if (rc) return rc;
    rc = grow_buffer(e, &e->d_jscan, &e->jscan_cap, sstride * n, false); if (rc) return rc;
    rc = grow_buffer(e, &e->d_jwork, &e->jwork_cap, tab_b + seg_b + pub_b + flag_b + 2 * small_b, false); if (rc) return rc;
    rc = grow_buffer(e, &e->h_jstatus, &e->h_jstatus_cap, (size_t)4 * e->cfg.max_batch, true); if (rc) return rc;
    bool pinned = true;   // page-locked caller buffers (pe_host_alloc) are DMA'd directly; pageable ones are staged, which drains the stream
    for (int i = 0; i < n && pinned; i++) {
        cudaPointerAttributes at;
        if (cudaPointerGetAttributes(&at, scans[i]) != cudaSuccess || at.type != cudaMemoryTypeHost) { pinned = false; cudaGetLastError(); }
    }
    if (pinned) {
        for (int i = 0; i < n; i++) CK(e, cudaMemcpyAsync(e->d_jscan + i * sstride, scans[i], bytes[i], cudaMemcpyHostToDevice, e->stream));
    } else {
        CK(e, cudaStreamSynchronize(e->stream));
        rc = grow_buffer(e, &e->h_jscan, &e->h_jscan_cap, sstride * n, true); if (rc) return rc;
        for (int i = 0; i < n; i++) memcpy(e->h_jscan + i * sstride, scans[i], bytes[i]);
        CK(e, cudaMemcpyAsync(e->d_jscan, e->h_jscan, sstride * n, cudaMemcpyHostToDevice, e->stream));
    }
    CK(e, cudaMemsetAsync(e->d_jcoef, 0, *cstride * n, e->stream));
    JpegScanArgs a;
    a.scans = e->d_jscan; a.scan_stride = (long long)sstride;
    a.coefs = e->d_jcoef; a.coef_stride = (long long)*cstride;
    uint8_t* w = e->d_jwork;
    a.tabs = w; w += tab_b;
    a.seg_sub = (int*)w; a.seg_stride = max_seg + 1; w += seg_b;
    a.pub = (unsigned long long*)w; w += pub_b;
    a.flags = (int*)w; w += flag_b;
    a.tickets = (int*)w; w += small_b;
    a.status = (int*)w;
    a.ctas_max = ctas; a.n = n; a.S = S;
    e->launches += launch_jpeg_entropy(a, e->stream);
    CK(e, cudaMemcpyAsync(e->h_jstatus, a.status, (size_t)4 * n, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaGetLastError());
    return PE_OK;
}

extern "C" int pe_forward_jpeg_scans(pe_engine* e, const void* const* scans, int n, double* scale) {
    NvtxRange r("pe_forward_jpeg_scans (H2D + entropy decoding + reconstruction)");
    int rc = check_n(e, n); if (rc) return rc;
    CK(e, cudaSetDevice(e->cfg.device));
    int W = 0, H = 0;
    size_t stride = 0;
    long long max_blocks = 0;
    rc = decode_scans(e, scans, n, pe_jpeg::SUBSEQ_BITS, &W, &H, &stride, &max_blocks); if (rc) return rc;
    rc = reconstruct_and_forward(e, n, W, H, stride, max_blocks, scale); if (rc) return rc;
    e->jstatus_n = n;
    return PE_OK;
}

extern "C" int pe_jpeg_decode_scans(pe_engine* e, const void* const* scans, int n, int subseq_bits, void* const* coefs_out, int* status_out) {
    int rc = check_n(e, n); if (rc) return rc;
    if (!coefs_out) return fail(e, PE_ERR_INVALID, "null output buffers");
    CK(e, cudaSetDevice(e->cfg.device));
    int W = 0, H = 0;
    size_t stride = 0;
    long long max_blocks = 0;
    e->jstatus_n = 0;   // h_jstatus now holds this call's statuses, not those of the last forward
    rc = decode_scans(e, scans, n, subseq_bits ? subseq_bits : pe_jpeg::SUBSEQ_BITS, &W, &H, &stride, &max_blocks); if (rc) return rc;
    CK(e, cudaStreamSynchronize(e->stream));
    for (int i = 0; i < n; i++) {
        const pe_jpeg_scan_header& hd = *(const pe_jpeg_scan_header*)scans[i];
        if (!coefs_out[i]) return fail(e, PE_ERR_INVALID, "null output buffer %d", i);
        CK(e, cudaMemcpy(coefs_out[i], e->d_jcoef + i * stride, (size_t)hd.coef.total_bytes, cudaMemcpyDeviceToHost));
        if (status_out) { int st; memcpy(&st, e->h_jstatus + 4 * i, 4); status_out[i] = st == INT_MAX ? 0 : 1 + st; }
    }
    return PE_OK;
}

// ---------------------------------------------------------------------------------------------
// Range calibration of the fp16-plane modes (parity F16X2 and fast F16X1).  The planes hold value * s with a per-activation power-of-two s; without
// calibration s = 1, which suits nets whose activations are O(1e-2 .. 1e3) (the trained pose models).  A net outside that range -
// the prototxt's own gaussian(0.01) filler shrinks every layer until the maps are ~3e-11 - would flush to zero (or overflow to inf)
// silently.  pe_calibrate runs ONE forward layer by layer: each conv first runs with s_out = 1 while the epilogue records the
// largest |output| (fp32, before the fp16 split), s_out is set to bring that maximum into [32, 64) (1000x headroom to 65504), the
// epilogue fields are rewritten (fill_epilogue_fields) and the layer runs again.  Pools and copies pass stored values through; a layer
// whose input channels carry different scales (the Concat of conv4_4_CPM with the previous stage's outputs) gets the ratios folded
// into its re-packed weights (pack_conv_weights).  Afterwards the kernels keep recording the maxima: pe_range_status reports a
// layer that left the range (PE_ERR_RANGE), and with PE_CHECK_RANGE=1 every pe_fetch does.
// ---------------------------------------------------------------------------------------------
static int upload_fields(pe_engine* e, int i) {
    std::vector<float> B((size_t)e->cout_pad[i] + 1, 0.f);
    fill_epilogue_fields(e, i, B.data());
    CK(e, cudaMemcpyAsync((char*)e->d_packed + e->b_off[i], B.data(), B.size() * sizeof(float), cudaMemcpyHostToDevice, e->stream));
    return PE_OK;
}

static int upload_weights(pe_engine* e, int i) {   // re-pack layer i with the current input scales (host fp32 copy needed)
    const ConvSpec& c = e->plan.convs[i];
    const size_t K = (size_t)(c.im2col_input ? 1 : c.k * c.k) * e->cin_pad[i];
    std::vector<uint8_t> buf(K * e->cout_pad[i] * e->elem * (e->fmt.planes ? e->fmt.planes : 1));
    pack_conv_weights(e, i, buf.data());
    CK(e, cudaMemcpyAsync((char*)e->d_packed + e->w_off[i], buf.data(), buf.size(), cudaMemcpyHostToDevice, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    return PE_OK;
}

extern "C" int pe_calibrate(pe_engine* e, const uint8_t* const* frames, int n) {
    int rc = check_n(e, n); if (rc) return rc;
    if (!frames) return fail(e, PE_ERR_INVALID, "null frames");
    if (!e->committed) return fail(e, PE_ERR_STATE, "pe_commit_weights has not been called");
    if (!e->fmt.f16) return PE_OK;   // fp32 / bf16 modes have fp32's exponent range
    const size_t nc = e->plan.convs.size();
    if (e->bias_true.size() != nc || e->bias_true[0].empty() || e->hw[0].w.empty())
        return fail(e, PE_ERR_STATE, "this handle received its weights by broadcast / sharing: calibrate the source handle before replicating");
    CK(e, cudaSetDevice(e->cfg.device));
    drop_graphs(e);
    // frames -> device -> net input (the im2col path: conv1_1 is calibrated like every other layer)
    const size_t fb = (size_t)e->cfg.disp_w * e->cfg.disp_h * 3;
    CK(e, cudaStreamSynchronize(e->stream));
    for (int i = 0; i < n; i++) { if (!frames[i]) return fail(e, PE_ERR_INVALID, "null frame %d", i); memcpy(e->h_frames + i * fb, frames[i], fb); }
    CK(e, cudaMemcpyAsync(e->d_frames, e->h_frames, fb * n, cudaMemcpyHostToDevice, e->stream));
    PreArgs a = e->pre;
    a.frames = e->d_frames; a.nframes = n;
    const bool direct_was = e->conv11_direct;
    e->conv11_direct = false;
    e->launches += launch_preprocess(a, e->stream, true);
    e->input_from_frames = true; e->input_act_stale = false; e->last_frames = e->d_frames;
    const int nimg = n * e->cfg.num_scales;
    auto restore = [&](int code) { e->conv11_direct = direct_was; return code; };
    for (const OpRef& op : e->plan.order) {
        if (op.type != 0) { if ((rc = run_op(e, op, nimg))) return restore(rc); continue; }
        const int i = op.idx;
        const ConvSpec& c = e->plan.convs[i];
        // the producers of this layer's input are final: fold their scales into the weights if they are not all equal to what is packed
        bool mixed = false;
        const float s_ref = input_ref_scale(e, c);
        for (int pc : c.cin_prod) if (pc >= 0 && e->conv_scale[pc] != s_ref) mixed = true;
        if (mixed || e->calibrated) { if ((rc = upload_weights(e, i))) return restore(rc); }
        if (c.out_act >= 0) {
            e->conv_scale[i] = 1.f;               // measure the true output range: fp32 epilogue values, before the fp16 split
            if ((rc = upload_fields(e, i))) return restore(rc);
            CK(e, cudaMemsetAsync(e->d_range + i, 0, sizeof(unsigned), e->stream));
            if ((rc = run_op(e, op, nimg))) return restore(rc);
            unsigned bits = 0;
            CK(e, cudaMemcpyAsync(&bits, e->d_range + i, sizeof bits, cudaMemcpyDeviceToHost, e->stream));
            CK(e, cudaStreamSynchronize(e->stream));
            float m; memcpy(&m, &bits, 4);
            if (m > 0.f && m < 3e38f) { int ex = 0; frexpf(m, &ex); e->conv_scale[i] = ldexpf(1.f, std::max(-100, std::min(100, 6 - ex))); }   // m * s in [32, 64)
        }
        if ((rc = upload_fields(e, i))) return restore(rc);
        if ((rc = run_op(e, op, nimg))) return restore(rc);
    }
    e->conv11_direct = direct_was;
    if (e->w11_off) {   // the direct conv1_1 kernel has its own fp32 copy of the layer: fold the output scale into it
        const float s_out = e->conv_scale[0];
        std::vector<float> w(27 * 64 + 64);
        CK(e, cudaMemcpy(w.data(), (char*)e->d_packed + e->w11_off, w.size() * sizeof(float), cudaMemcpyDeviceToHost));
        const float rel = s_out / e->w11_scale;
        for (float& v : w) v *= rel;
        CK(e, cudaMemcpy((char*)e->d_packed + e->w11_off, w.data(), w.size() * sizeof(float), cudaMemcpyHostToDevice));
        e->w11_scale = s_out;
    }
    CK(e, cudaMemsetAsync(e->d_range, 0, nc * sizeof(unsigned), e->stream));
    e->calibrated = true;
    return run_post_and_return(e, n);
}

// Largest |stored value| / 65504 over the conv layers since the last call (PE_ERR_RANGE when a layer reached the fp16 limit, or when
// a layer's maximum fell below 2^-10 - its lo plane then lives in fp16 subnormals and parity is lost); *layer64 names the worst one.
extern "C" int pe_range_status(pe_engine* e, float* worst_ratio, char* layer64) {
    if (!e) return PE_ERR_INVALID;
    if (worst_ratio) *worst_ratio = 0.f;
    if (layer64) layer64[0] = 0;
    if (!e->d_range) return PE_OK;
    CK(e, cudaSetDevice(e->cfg.device));
    CK(e, cudaStreamSynchronize(e->stream));
    const size_t nc = e->plan.convs.size();
    std::vector<unsigned> bits(nc);
    CK(e, cudaMemcpy(bits.data(), e->d_range, nc * sizeof(unsigned), cudaMemcpyDeviceToHost));
    CK(e, cudaMemset(e->d_range, 0, nc * sizeof(unsigned)));
    float worst = 0.f, smallest = 3e38f;
    int iw = -1, is = -1;
    for (size_t i = 0; i < nc; i++) {
        if (e->plan.convs[i].out_act < 0) continue;   // fp32 maps
        float m; memcpy(&m, &bits[i], 4);
        if (bits[i] == 0) continue;                   // layer did not run since the last call
        if (!(m <= 3e38f) || m / 65504.f > worst) { worst = (m <= 3e38f) ? m / 65504.f : 2.f; iw = (int)i; }
        if (m < smallest) { smallest = m; is = (int)i; }
    }
    if (worst_ratio) *worst_ratio = worst;
    if (worst >= 1.f) {
        if (layer64) snprintf(layer64, 64, "%s", e->plan.convs[iw].name.c_str());
        return fail(e, PE_ERR_RANGE, "layer %s produced values outside the range of the fp16 planes (max |v| = %.3g x scale): run pe_calibrate",
                    e->plan.convs[iw].name.c_str(), worst * 65504.f);
    }
    if (is >= 0 && smallest < 9.765625e-4f) {
        if (layer64) snprintf(layer64, 64, "%s", e->plan.convs[is].name.c_str());
        return fail(e, PE_ERR_RANGE, "layer %s: largest stored value %.3g is below 2^-10, the fp16 planes lose precision: run pe_calibrate",
                    e->plan.convs[is].name.c_str(), smallest);
    }
    if (layer64 && iw >= 0) snprintf(layer64, 64, "%s", e->plan.convs[iw].name.c_str());
    return PE_OK;
}

extern "C" int pe_forward_net_input(pe_engine* e, const float* net_input, int n) {
    int rc = check_n(e, n); if (rc) return rc;
    if (!net_input) return fail(e, PE_ERR_INVALID, "null input");
    CK(e, cudaSetDevice(e->cfg.device));
    const size_t cnt = (size_t)n * e->cfg.num_scales * 3 * e->cfg.net_w * e->cfg.net_h;
    CK(e, cudaStreamSynchronize(e->stream));
    memcpy(e->h_planar, net_input, cnt * sizeof(float));
    CK(e, cudaMemcpyAsync(e->d_planar, e->h_planar, cnt * sizeof(float), cudaMemcpyHostToDevice, e->stream));
    PreArgs a = e->pre;
    a.nframes = n;
    e->launches += launch_input_from_planar(e->d_planar, a, n * e->cfg.num_scales, e->stream);
    e->input_lo_dirty = e->fmt.planes > 0;
    e->last_frames = nullptr;
    if (e->input_from_frames) drop_graphs(e);   // the captured graphs hold the other conv1_1 kernel
    e->input_from_frames = false;
    e->input_act_stale = false;
    return run_net(e, n);
}
extern "C" int pe_forward_maps(pe_engine* e, const float* maps8, int n) {
    int rc = check_n(e, n); if (rc) return rc;
    if (!maps8) return fail(e, PE_ERR_INVALID, "null maps");
    CK(e, cudaSetDevice(e->cfg.device));
    const size_t cnt = (size_t)n * e->cfg.num_scales * e->mt->num_maps * e->geo[3].W * e->geo[3].H;
    CK(e, cudaStreamSynchronize(e->stream));
    memcpy(e->h_maps, maps8, cnt * sizeof(float));
    CK(e, cudaMemcpyAsync(e->d_maps, e->h_maps, cnt * sizeof(float), cudaMemcpyHostToDevice, e->stream));
    e->last_frames = nullptr;
    return run_post_and_return(e, n);
}


// ---------------------------------------------------------------------------------------------
// renderers: render() of rtpose.cpp:271-300 on the canvas of frame `idx`
// ---------------------------------------------------------------------------------------------
extern "C" int pe_render(pe_engine* e, int idx, int part_to_show, int googly_eyes, const uint8_t* display_bgr, float* canvas,
                         uint8_t* bgr) {
    if (!e) return PE_ERR_INVALID;
    if (idx < 0 || idx >= e->last_n) return fail(e, PE_ERR_INVALID, "frame index %d outside the last forward (n=%d)", idx, e->last_n);
    const int P = e->mt->num_parts, W = e->cfg.disp_w, H = e->cfg.disp_h, nw = e->cfg.net_w, nh = e->cfg.net_h;
    const int max_show = e->cfg.model == PE_MODEL_MPI_15 ? e->mt->num_maps : P + 2 + e->mt->num_limbs;   // COCO: 0..39
    if (part_to_show < 0 || part_to_show > max_show)
        return fail(e, PE_ERR_INVALID, "part_to_show=%d outside [0, %d]", part_to_show, max_show);
    if (!display_bgr && !e->last_frames)
        return fail(e, PE_ERR_STATE, "the last forward had no display frame (net-input / map path): pass display_bgr");
    CK(e, cudaSetDevice(e->cfg.device));
    const size_t px = (size_t)W * H;
    if (!e->d_canvas) {
        CK(e, cudaMalloc(&e->d_canvas, px * 3 * sizeof(float)));
        CK(e, cudaMalloc(&e->d_render_u8, px * 3));
        CK(e, cudaMalloc(&e->d_render_src, px * 3));
    }
    const uint8_t* src = e->last_frames ? e->last_frames + (size_t)idx * px * 3 : nullptr;
    if (display_bgr) {
        CK(e, cudaMemcpyAsync(e->d_render_src, display_bgr, px * 3, cudaMemcpyHostToDevice, e->stream));
        src = e->d_render_src;
    }
    e->launches += launch_canvas_fill(src, e->d_canvas, W, H, e->stream);   // process_and_pad_image(normalize = 0), rtpose.cpp:349,1127
    const PostDev& pd = e->post;
    const float* poses = pd.joints + (size_t)idx * PE_MAX_PEOPLE * P * 3;
    auto heat = [&](int ch0, int nch) -> int {   // the channels a heat-map view reads, from the stride-8 maps
        const size_t need = (size_t)nch * nw * nh * sizeof(float);
        if (need > e->heat_cap) {
            cudaFree(e->d_heat); e->d_heat = nullptr; e->heat_cap = 0;
            CK(e, cudaMalloc(&e->d_heat, need));
            e->heat_cap = need;
        }
        e->launches += launch_fullres_fill(pd, idx, ch0, nch, e->d_heat, e->stream);
        return PE_OK;
    };
    int rc = PE_OK;
    if (part_to_show == 0) {
        e->launches += launch_skeleton(e->cfg.model, e->d_canvas, W, H, poses, pd.num_people + idx, googly_eyes, e->stream);
    } else if (e->cfg.model == PE_MODEL_MPI_15) {                 // render_mpi_parts: channel part_to_show-1
        if ((rc = heat(part_to_show - 1, 1))) return rc;
        e->launches += launch_heat_view(e->d_canvas, W, H, e->d_heat, nw, nh, 0, part_to_show - 1, 1, e->stream);
    } else if (part_to_show - 1 < P) {                            // render_coco_parts: one part map
        if ((rc = heat(part_to_show - 1, 1))) return rc;
        e->launches += launch_heat_view(e->d_canvas, W, H, e->d_heat, nw, nh, 1, part_to_show - 1, 1, e->stream);
    } else if (part_to_show - 1 == P) {                           // all part maps, nearest neighbour (heatmap2)
        if ((rc = heat(0, P))) return rc;
        e->launches += launch_heat_view(e->d_canvas, W, H, e->d_heat, nw, nh, 2, 0, P, e->stream);
    } else {                                                      // render_coco_aff (rtpose.cpp:286-296)
        int aff_part = ((part_to_show - 1) - P - 1) * 2, accum = 1;
        if (aff_part == 0) accum = e->mt->num_limbs; else aff_part -= 2;
        aff_part += 1 + P;
        if ((rc = heat(aff_part, 2 * accum))) return rc;
        e->launches += launch_heat_view(e->d_canvas, W, H, e->d_heat, nw, nh, 3, aff_part, 2 * accum, e->stream);
    }
    if (bgr) e->launches += launch_canvas_to_u8(e->d_canvas, e->d_render_u8, W, H, e->stream);   // postProcessFrame, rtpose.cpp:1286-1296
    if (canvas) CK(e, cudaMemcpyAsync(canvas, e->d_canvas, px * 3 * sizeof(float), cudaMemcpyDeviceToHost, e->stream));
    if (bgr) CK(e, cudaMemcpyAsync(bgr, e->d_render_u8, px * 3, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    CK(e, cudaGetLastError());
    return PE_OK;
}

// ---------------------------------------------------------------------------------------------
// render_mpi_parts / render_coco_parts / render_coco_aff of include/rtpose/renderFunctions.h with the reference's DEVICE-pointer
// arguments (src/rtpose/renderFunctions.cu:330-392, 977-1075): canvas = planar float BGR (3 x h_canvas x w_canvas), heatmaps =
// the full-resolution resized_map (C x h_net x w_net), poses = joints.  No engine handle: this is the drop-in for host code that
// keeps the reference's own buffers.  kind 0 / 1 / 2 = mpi_parts / coco_parts / coco_aff; `extra` = googly_eyes (kind 1) or
// num_parts_accum (kind 2).  Like the reference it renders frame 0 of the batch and synchronises the device.
// ---------------------------------------------------------------------------------------------
extern "C" int pe_render_device(int kind, float* canvas, int w_canvas, int h_canvas, int w_net, int h_net, const float* heatmaps,
                                const float* poses, const int* num_people, int n_frames, int part, int extra) {
    if (!canvas || w_canvas <= 0 || h_canvas <= 0 || kind < 0 || kind > 2) return PE_ERR_INVALID;
    const int np0 = (num_people && n_frames > 0) ? num_people[0] : 0;
    float* heat = const_cast<float*>(heatmaps);
    const size_t plane = (size_t)w_net * h_net;
    if (kind == 0) {          // render_mpi_parts: skeleton (only when somebody is there) or one channel as a heat map
        if (part == 0) { if (np0 != 0) launch_skeleton(PE_MODEL_MPI_15, canvas, w_canvas, h_canvas, poses, nullptr, 0, nullptr, np0); }
        else if (part > 0) { if (!heat) return PE_ERR_INVALID; launch_heat_view(canvas, w_canvas, h_canvas, heat + (size_t)(part - 1) * plane, w_net, h_net, 0, part - 1, 1, nullptr); }
    } else if (kind == 1) {   // render_coco_parts
        if (part == 0) { if (np0 != 0) launch_skeleton(PE_MODEL_COCO_18, canvas, w_canvas, h_canvas, poses, nullptr, extra, nullptr, np0); }
        else if (part > 0 && part < 58) {
            if (!heat) return PE_ERR_INVALID;
            if (part - 1 == 18) launch_heat_view(canvas, w_canvas, h_canvas, heat, w_net, h_net, 2, 0, 18, nullptr);
            else launch_heat_view(canvas, w_canvas, h_canvas, heat + (size_t)(part - 1) * plane, w_net, h_net, 1, part - 1, 1, nullptr);
        }
    } else {                  // render_coco_aff: `extra` consecutive (x, y) PAF channel pairs from channel `part`
        if (!heat || extra < 1) return PE_ERR_INVALID;
        launch_heat_view(canvas, w_canvas, h_canvas, heat + (size_t)part * plane, w_net, h_net, 3, part, 2 * extra, nullptr);
    }
    const cudaError_t err = cudaDeviceSynchronize();   // as the reference does after every render call
    return err == cudaSuccess ? PE_OK : fail(nullptr, PE_ERR_CUDA, "render: %s", cudaGetErrorString(err));
}

extern "C" int pe_sync(pe_engine* e) {
    if (!e) return PE_ERR_INVALID;
    CK(e, cudaSetDevice(e->cfg.device));
    CK(e, cudaStreamSynchronize(e->stream));
    return PE_OK;
}
extern "C" int pe_fetch(pe_engine* e, int idx, float* joints, int* num_people, float* peaks) {
    NvtxRange r("pe_fetch (sync + D2H results)");
    if (!e) return PE_ERR_INVALID;
    if (idx < 0 || idx >= e->last_n) return fail(e, PE_ERR_INVALID, "frame index %d outside the last forward (n=%d)", idx, e->last_n);
    int rc = pe_sync(e); if (rc) return rc;
    if (e->check_range && idx == 0) { rc = pe_range_status(e, nullptr, nullptr); if (rc) return rc; }   // PE_CHECK_RANGE=1: range problems are errors
    if (idx < e->jstatus_n) {   // a frame from a scan image whose entropy-coded data the host entropy stage rejects
        int mcu;
        memcpy(&mcu, e->h_jstatus + 4 * idx, 4);
        if (mcu != INT_MAX) return fail(e, PE_ERR_IO, "frame %d: corrupt JPEG data (DC category above 15) in MCU %d", idx, mcu);
    }
    const int P = e->mt->num_parts, MP = e->mt->max_peaks;
    if (num_people) *num_people = e->h_num_people[idx];
    if (joints) memcpy(joints, e->h_joints + (size_t)idx * PE_MAX_PEOPLE * P * 3, sizeof(float) * PE_MAX_PEOPLE * P * 3);
    if (peaks) memcpy(peaks, e->h_peaks + (size_t)idx * P * (MP + 1) * 3, sizeof(float) * P * (MP + 1) * 3);
    return PE_OK;
}
extern "C" int pe_fetch_maps(pe_engine* e, float* maps8, int n) {
    int rc = check_n(e, n); if (rc) return rc;
    CK(e, cudaSetDevice(e->cfg.device));
    const size_t cnt = (size_t)n * e->cfg.num_scales * e->mt->num_maps * e->geo[3].W * e->geo[3].H;
    CK(e, cudaMemcpyAsync(e->h_maps, e->d_maps, cnt * sizeof(float), cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    memcpy(maps8, e->h_maps, cnt * sizeof(float));
    return PE_OK;
}
extern "C" int pe_fetch_blob(pe_engine* e, const char* blob_name, float* out, size_t cap, int* c, int* h, int* w) {
    if (!e || !blob_name) return PE_ERR_INVALID;
    CK(e, cudaSetDevice(e->cfg.device));
    const int nimg = std::max(e->last_n, 1) * e->cfg.num_scales;
    for (const BlobRef& b : e->plan.blobs) {
        if (b.name != blob_name) continue;
        if (!b.reused_by.empty())
            return fail(e, PE_ERR_STATE, "blob %s is not kept: %s, later in every forward, reuses its buffer", blob_name, b.reused_by.c_str());
        Geo g = e->geo[e->plan.acts[b.act].level];
        g.N = nimg;
        const size_t cnt = (size_t)nimg * b.c * g.H * g.W;
        if (c) *c = b.c;
        if (h) *h = g.H;
        if (w) *w = g.W;
        if (!out) return PE_OK;
        if (cnt > cap) return fail(e, PE_ERR_INVALID, "blob %s needs %zu floats", blob_name, cnt);
        if (b.act == e->plan.input_act && e->input_act_stale) {   // conv1_1 ran from the uint8 images: materialise the net input on demand
            PreArgs a = e->pre;
            a.nframes = std::max(e->last_n, 1);
            e->launches += launch_im2col_u8(a, e->stream);
            e->input_act_stale = false;
        }
        float* d = nullptr;
        CK(e, cudaMalloc(&d, cnt * sizeof(float)));
        // stored value = true value * conv_scale[producer] (pools pass their producer's scale through; the net input has none)
        const float inv = (b.prod >= 0 && b.prod < (int)e->conv_scale.size()) ? 1.f / e->conv_scale[b.prod] : 1.f;
        e->launches += launch_act_to_nchw(e->acts[b.act], e->plan.acts[b.act].C, b.coff, b.c, e->act_plane[b.act], e->fmt, g, inv, d,
                                          e->stream);
        CK(e, cudaMemcpyAsync(out, d, cnt * sizeof(float), cudaMemcpyDeviceToHost, e->stream));
        CK(e, cudaStreamSynchronize(e->stream));
        cudaFree(d);
        return PE_OK;
    }
    return fail(e, PE_ERR_INVALID, "unknown blob %s", blob_name);
}

extern "C" void* pe_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaMallocHost(&p, bytes ? bytes : 1) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
extern "C" void pe_host_free(void* p) { if (p) cudaFreeHost(p); }

// ---------------------------------------------------------------------------------------------
// JSON (rtpose.cpp:1383-1416): ostream default formatting == %g
// ---------------------------------------------------------------------------------------------
extern "C" int pe_write_json(const float* joints, int num_people, int num_parts, double frame_scale, char* buf, int cap) {
    std::string s;
    char t[64];
    const double scale = 1.0 / frame_scale;
    s += "{\n\"version\":0.1,\n\"bodies\":[\n";
    for (int ip = 0; ip < num_people; ip++) {
        s += "{\n\"joints\":[";
        for (int ij = 0; ij < num_parts; ij++) {
            const float* j = joints + ((size_t)ip * num_parts + ij) * 3;
            snprintf(t, sizeof t, "%g,%g,%g", scale * j[0], scale * j[1], (double)j[2]);
            s += t;
            if (ij < num_parts - 1) s += ",";
        }
        s += "]\n}";
        if (ip < num_people - 1) s += ",\n";
    }
    s += "]\n}\n";
    if (buf && (int)s.size() < cap) memcpy(buf, s.c_str(), s.size() + 1);
    return (int)s.size();
}

// ---------------------------------------------------------------------------------------------
// Result comparison (DESIGN.md section 6 (3)): peaks, person count and joints of two fetched results of one frame
// ---------------------------------------------------------------------------------------------
extern "C" int pe_compare_results(const float* joints_a, int people_a, const float* peaks_a, const float* joints_b, int people_b,
                                  const float* peaks_b, int num_parts, int max_peaks, float tol_px, pe_result_diff* out) {
    if (!out || !peaks_a || !peaks_b || num_parts <= 0 || max_peaks < 0 || people_a < 0 || people_b < 0 || !(tol_px >= 0.f) ||
        (people_a > 0 && !joints_a) || (people_b > 0 && !joints_b))
        return PE_ERR_INVALID;
    memset(out, 0, sizeof *out);
    auto dist = [](const float* p, const float* q) { return hypot((double)p[0] - q[0], (double)p[1] - q[1]); };
    const size_t part_stride = (size_t)(max_peaks + 1) * 3;
    for (int p = 0; p < num_parts; p++) {
        const float* pa = peaks_a + p * part_stride;
        const float* pb = peaks_b + p * part_stride;
        const int ca = std::min((int)pa[0], max_peaks), cb = std::min((int)pb[0], max_peaks);
        if (ca != cb) { out->parts_count_differ++; continue; }
        for (int k = 1; k <= ca; k++)
            if (!(dist(pa + 3 * k, pb + 3 * k) <= tol_px)) out->peaks_moved++;
    }
    bool joints_ok = true;
    double worst = 0.0;
    for (int i = 0; i < std::min(people_a, people_b); i++) {
        const float* ja = joints_a + (size_t)i * num_parts * 3;
        const float* jb = joints_b + (size_t)i * num_parts * 3;
        bool same = true;
        for (int p = 0; p < num_parts && same; p++) same = (ja[3 * p + 2] > 0.f) == (jb[3 * p + 2] > 0.f);
        if (!same) continue;
        out->persons_matched++;
        for (int p = 0; p < num_parts; p++)
            if (ja[3 * p + 2] > 0.f) {
                const double d = dist(ja + 3 * p, jb + 3 * p);
                if (!(d <= tol_px)) joints_ok = false;
                worst = std::max(worst, d);
            }
    }
    out->max_joint_dist = (float)worst;
    out->identical = out->parts_count_differ == 0 && out->peaks_moved == 0 && people_a == people_b &&
                     out->persons_matched == people_a && joints_ok;
    return PE_OK;
}

// ---------------------------------------------------------------------------------------------
// measurement support
// ---------------------------------------------------------------------------------------------
extern "C" int pe_event_record(pe_engine* e, int slot) {
    if (!e || slot < 0 || slot >= 16) return PE_ERR_INVALID;
    CK(e, cudaSetDevice(e->cfg.device));
    CK(e, cudaEventRecord(e->ev[slot], e->stream));
    return PE_OK;
}
extern "C" int pe_event_elapsed_ms(pe_engine* e, int a, int b, float* ms) {
    if (!e || a < 0 || a >= 16 || b < 0 || b >= 16 || !ms) return PE_ERR_INVALID;
    CK(e, cudaSetDevice(e->cfg.device));
    CK(e, cudaEventSynchronize(e->ev[b]));
    CK(e, cudaEventElapsedTime(ms, e->ev[a], e->ev[b]));
    return PE_OK;
}
extern "C" int pe_profile_layers(pe_engine* e, int n, float* ms, char* names, double* flops, int cap) {
    int rc = check_n(e, n); if (rc) return rc;
    if (!e->committed) return fail(e, PE_ERR_STATE, "pe_commit_weights has not been called");
    CK(e, cudaSetDevice(e->cfg.device));
    const int nimg = n * e->cfg.num_scales;
    const int nops = (int)e->plan.order.size();
    std::vector<cudaEvent_t> evs(nops + 1);
    for (auto& v : evs) CK(e, cudaEventCreate(&v));
    CK(e, cudaEventRecord(evs[0], e->stream));
    for (int i = 0; i < nops; i++) {
        rc = run_op(e, e->plan.order[i], nimg);
        if (rc) return rc;
        CK(e, cudaEventRecord(evs[i + 1], e->stream));
    }
    CK(e, cudaStreamSynchronize(e->stream));
    int written = 0;
    for (int i = 0; i < nops && written < cap; i++) {
        const OpRef& op = e->plan.order[i];
        float t = 0.f;
        CK(e, cudaEventElapsedTime(&t, evs[i], evs[i + 1]));
        ms[written] = t;
        const char* nm = op.type == 0 ? e->plan.convs[op.idx].name.c_str() : op.type == 1 ? e->plan.pools[op.idx].name.c_str() : "copy_F";
        if (names) snprintf(names + 64 * written, 64, "%s", nm);
        if (flops) flops[written] = op.type == 0 ? e->plan.convs[op.idx].flops_per_image * nimg : 0.0;
        written++;
    }
    for (auto& v : evs) cudaEventDestroy(v);
    return written;
}
extern "C" long long pe_launch_count(const pe_engine* e) { return e ? e->launches : 0; }
extern "C" double pe_conv_flops_per_scale(const pe_engine* e) { return e ? e->flops_per_scale : 0.0; }
