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
#include "buffers.h"
#include "kernels.h"
#include "conv_tc.h"
#include "precision.h"
#include "e4m3.h"
#include "s8.h"
#include "s8_sparse.h"
#include "jpeg_coefs.h"
#include "jpeg_entropy.cuh"
#include "pixels.cuh"
#include <climits>
#include "prototxt.h"
#include "calib_table.h"

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
    const Precision* prec = nullptr;   // the precision mode's row (precision.h)
    bool u8 = false;                   // PE_PREC_FLAG_U8 (cfg.precision holds the mode without it): the plan's u8 activations
    bool flip = false;                 // the flip test (pe_set_flip_test): each frame's S images plus their S mirrors in x
    // What a captured forward graph references (activations, maps, post and result buffers, packed weights, d_range, axis tables) is
    // allocated once, in pe_create or commit, and never regrown: a replayed graph keeps its pointers.  Only input-route buffers grow,
    // and the per-image buffers (activations, maps: geo[*].N images) when pe_set_flip_test doubles them, which drops the graphs.
    std::vector<DeviceBuffer> acts;
    std::vector<long long> act_plane;  // elements per plane
    std::vector<HostWeights> hw;    // per conv
    bool committed = false;
    // packed weights at per-conv offsets (bytes); shared by the handles of pe_share_weights, freed when the last one goes
    std::shared_ptr<DeviceBuffer> packed;
    // range management of the fp16 and e4m3 modes (F16X2, F16X1, E4M3X1): per-conv-output power-of-two scale s (stored value = true value * s), the
    // weight-scale inverses the packed epilogue fields derive from (with the true biases hw[i].b), and the kernels' running max |stored value| per conv
    std::vector<float> conv_scale, wsi;   // per conv: scale of its stored output; inverse of the power of two folded into its weights
    std::vector<std::vector<float>> wsig;   // S8X1, S8X2: per conv, the per-output-channel weight step sigma_c of pack_conv_weights (s8.h)
    DeviceBuffer d_range;
    bool calibrated = false, check_range = false;
    // pe_calibrate_begin .. _end: per conv, the largest true |output| (recorded / conv_scale) over the forwards since begin
    bool collecting = false;
    int collect_forwards = 0;
    std::vector<float> collect_max;
    uint64_t weights_hash = 0; bool weights_hash_valid = false;   // of hw (calibration tables); reset by pe_commit_weights
    std::vector<size_t> w_off, b_off;
    std::vector<int> cout_pad, cin_pad;
    std::vector<char> sparse;       // per conv: runs the 2:4-sparse s8 kernel (chosen at pe_commit_weights, see sparse_eligible)
    bool force_sparse = false;      // pe_test_force_sparse: lift rule 4 of sparse_eligible at the next pe_commit_weights
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
    DeviceBuffer d_frames, d_resized, d_planar, d_maps;
    std::vector<DeviceBuffer> d_tabs;
    PreArgs pre{};
    DeviceBuffer d_post;   // the post-processing arrays of post and the axis tables d_xtab, d_ytab
    PostDev post{};
    AxisTap *d_xtab = nullptr, *d_ytab = nullptr;
    PinnedBuffer h_results;   // h_joints, h_num_people, h_peaks
    float* h_joints = nullptr; int* h_num_people = nullptr; float* h_peaks = nullptr;
    PinnedBuffer h_stage;   // staging of host input and of pe_fetch_maps: a forward uses it at most once, the host writes it after a drain
    float start_scale_f, scale_gap_f;
    int last_n = 0;
    // raw camera frames (any size) -> display image: warpAffine source, and tables (d_warp) for the last (orig_w, orig_h)
    DeviceBuffer d_raw, d_warp;
    int warp_w = 0, warp_h = 0; double warp_scale = 1.0;
    int *d_wa = nullptr, *d_wb = nullptr, *d_wx0 = nullptr, *d_wy0 = nullptr; short* d_wtab = nullptr;
    // decoder-format host frames (pe_forward_pixels) copied to the device before conversion; pe_stream_wait's event
    DeviceBuffer d_pix;
    cudaEvent_t ev_wait = nullptr;
    bool input_lo_dirty = false;   // the planar-input path wrote non-zero lo planes / channels >= 32 of the input buffer
    DeviceBuffer d_jcoef, d_jplanes;   // JPEG coefficient images (pe_forward_jpeg_coefs): device copies, component planes
    DeviceBuffer d_jscan, d_jwork;     // JPEG scan images (pe_forward_jpeg_scans): device copies, the decoder's work space
    PinnedBuffer h_jstatus;            // and its per-frame status
    int jstatus_n = 0;   // frames of the last forward whose status h_jstatus holds (0: the last forward was not from scan images)
    // renderers: canvas, uint8 image and display frame (d_render, on first pe_render), heat-map scratch; display frames of the last forward
    DeviceBuffer d_render, d_heat;
    const uint8_t* last_frames = nullptr;
    // CUDA graphs of the steady-state forward (92 conv + pool/copy + 5 parse kernels + result copies), one per batch
    // size; the first forward of a size runs eagerly, the second is captured, later ones replay.  Invalidated by
    // any setter whose value is baked into kernel arguments.
    struct GraphEntry { cudaGraphExec_t exec = nullptr; long long launches = 0; int seen = 0; };
    std::map<int, GraphEntry> graphs;
    bool use_graphs = true;   // cleared when capture or instantiation fails: every later forward runs eagerly
    long long launches = 0;
    std::string err;
    double flops_per_scale = 0;
};

static void drop_graphs(pe_engine* e);
static int setup_lanes(pe_engine* e);
static int bind_packed(pe_engine* e);

// Images the conv stack runs per frame: the S scales, and with the flip test their S mirrors
static int copies(const pe_engine* e) { return e->cfg.num_scales * (e->flip ? 2 : 1); }

// Storage of activation i: the mode's plane count in the element kind the plan gave it (plan.cpp: the kind of the conv layers
// that read it).  conv i's packed weights have the kind of its arithmetic, which is that of its input.
static PlaneFmt act_fmt(const pe_engine* e, int i) { return PlaneFmt{e->prec->fmt.planes, (PlaneElem)e->plan.acts[i].elem}; }
static PlaneFmt conv_wfmt(const pe_engine* e, int i) { return PlaneFmt{e->prec->fmt.planes, (PlaneElem)e->plan.convs[i].elem}; }
// Element kind conv i stores: its output activation's, or for the planar fp32 maps its own, which picks the kernel instance
static PlaneElem conv_out_elem(const pe_engine* e, int i) {
    const ConvSpec& c = e->plan.convs[i];
    return (PlaneElem)(c.out_act >= 0 ? e->plan.acts[c.out_act].elem : c.elem);
}
// Per-layer facts (precision.h, elem_row): those of the arithmetic from the row of conv i's kind, the range facts from the row
// of the kind it stores
static const Precision& conv_row(const pe_engine* e, int i) { return elem_row(*e->prec, (PlaneElem)e->plan.convs[i].elem); }
static const Precision& out_row(const pe_engine* e, int i) { return elem_row(*e->prec, conv_out_elem(e, i)); }
// floats of conv i's epilogue fields in the packed buffer: bias[cout_pad], then the layer's factor or one factor per channel
static size_t epi_floats(const pe_engine* e, int i) { return (size_t)e->cout_pad[i] + (conv_row(e, i).per_channel_epilogue ? e->cout_pad[i] : 1); }
static size_t fmt_bytes(PlaneFmt f) { return (size_t)f.elem_bytes() * (f.planes ? f.planes : 1); }   // bytes per element, all planes

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
    DeviceBuffer& d = e->d_tabs.emplace_back();
    CK(e, d.reserve(std::max<size_t>(v.size(), 1) * sizeof(T)));
    CK(e, cudaMemcpy(d.get(), v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    *out = d.get<const T>();
    return PE_OK;
}

// ImResize crops scale n of the stride-8 maps by floor(ori/2 * f_n) per side, f_n = n * gap + (1 - start) in float as
// axis_table_kernel computes it.  f_n in [0, 1) keeps the crop inside the maps and at least one source pixel wide.
static int check_resize_scales(pe_engine* e, float start_scale, float scale_gap, int num_scales) {
    for (int n = 0; n < num_scales; n++) {
        const float f = fmaf((float)n, scale_gap, 1.0f - start_scale);
        if (!(f >= 0.f && f < 1.f))
            return fail(e, PE_ERR_INVALID, "scale %d: start_scale %g and scale_gap %g give the ImResize crop factor %g, outside [0, 1)", n,
                        start_scale, scale_gap, f);
    }
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

// The four resolution levels' geometry for N images
static void image_geo(const pe_engine* e, int N, Geo* geo) {
    int w = e->cfg.net_w, h = e->cfg.net_h;
    for (int l = 0; l < 4; l++) {
        geo[l] = make_geo(w, h, e->plan.gap[l], N);
        w = pooled(w); h = pooled(h);
    }
}

// The per-image buffers - activations and stride-8 maps - for N images, zeroed (gap rows must be).  They are allocated next to the
// old ones first: when an allocation fails the engine is left as it was.  Existing layers are re-bound to the new buffers.
static int alloc_images(pe_engine* e, int N) {
    Geo geo[4];
    image_geo(e, N, geo);
    const size_t na = e->plan.acts.size();
    std::vector<DeviceBuffer> acts(na);
    std::vector<long long> plane(na);
    for (size_t i = 0; i < na; i++) {
        const ActSpec& a = e->plan.acts[i];
        plane[i] = geo[a.level].M * a.C;
        const size_t bytes = (size_t)plane[i] * fmt_bytes(act_fmt(e, (int)i));
        CK(e, acts[i].reserve(bytes));
        CK(e, cudaMemsetAsync(acts[i].get(), 0, bytes, e->stream));
    }
    DeviceBuffer maps;
    const size_t maps_bytes = (size_t)N * e->mt->num_maps * geo[3].W * geo[3].H * sizeof(float);
    CK(e, maps.reserve(maps_bytes));
    CK(e, cudaMemsetAsync(maps.get(), 0, maps_bytes, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));   // the old buffers go below: no queued work may still use them
    if (e->stream2) CK(e, cudaStreamSynchronize(e->stream2));
    for (int l = 0; l < 4; l++) e->geo[l] = geo[l];
    e->acts = std::move(acts);
    e->act_plane = std::move(plane);
    e->d_maps = std::move(maps);
    e->post.maps = e->d_maps.get<float>();
    e->pre.out = e->acts[e->plan.input_act].get();
    e->pre.out_plane = e->act_plane[e->plan.input_act];
    e->input_lo_dirty = false;
    if (!e->committed) return PE_OK;
    e->committed = false;   // until the layers point at the new buffers
    return bind_packed(e);
}

static void set_post_params(pe_engine* e) {
    PostParams& p = e->post.p;
    const pe_config& c = e->cfg;
    p.model = c.model; p.num_parts = e->mt->num_parts; p.num_limbs = e->mt->num_limbs; p.num_maps = e->mt->num_maps;
    p.max_peaks = e->mt->max_peaks;
    p.net_w = c.net_w; p.net_h = c.net_h; p.w8 = e->geo[3].W; p.h8 = e->geo[3].H; p.disp_w = c.disp_w; p.disp_h = c.disp_h;
    p.num_scales = c.num_scales;
}

// The net of a host-only query: the prototxt at `prototxt_path`, or with NULL the built-in graph of `model`.  0 or -PE_ERR_*.
static int query_net(int model, const char* prototxt_path, NetDef& net) {
    std::string err;
    if (prototxt_path) {
        if (parse_prototxt_file(prototxt_path, net, err)) return -fail(nullptr, PE_ERR_IO, "%s: %s", prototxt_path, err.c_str());
    } else {
        if (model != PE_MODEL_MPI_15 && model != PE_MODEL_COCO_18) return -fail(nullptr, PE_ERR_INVALID, "unknown model %d", model);
        net = builtin_netdef(model, 6);
    }
    return 0;
}

// Host-only view of the execution plan a prototxt (or, with path == NULL, the built-in graph of `model`) produces: one
// line per op, "conv <name> cout cin k relu level in_act in_cused out_act out_coff planar_coff", "pool <name> in out",
// "copy src dst channels", then "gap level g" per resolution level (the flat layout's gap, common.h), "nms threshold
// max_peaks num_parts" and "resize start_scale scale_gap".  No GPU needed.
extern "C" int pe_plan_describe(int model, const char* prototxt_path, char* buf, int cap) {
    NetDef net;
    std::string err;
    if (const int rc = query_net(model, prototxt_path, net)) return rc;
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

static const char* elem_name(PlaneFmt f) {
    static const char* names[] = {"bf16", "f16", "e4m3", "s8", "u8"};
    if (f.s8() && f.planes == 2) return "s8x2";   // PE_PREC_S8X2's 16-bit integers
    return f.planes == 0 ? "f32" : names[f.elem];
}

// A precision argument: the mode, and PE_PREC_FLAG_U8, which applies to PE_PREC_S8X1 only.  The mode alone selects every per-mode
// fact; the flag only changes the plan's element kinds (plan.cpp).
static int split_precision(int p, int* mode, bool* u8) {
    *mode = p & ~PE_PREC_FLAG_U8;
    *u8 = (p & PE_PREC_FLAG_U8) != 0;
    if (!known_mode(*mode)) return fail(nullptr, PE_ERR_INVALID, "unknown precision %d", p);
    if (*u8 && *mode != PE_PREC_S8X1)
        return fail(nullptr, PE_ERR_INVALID, "PE_PREC_FLAG_U8 (u8 activations) applies to PE_PREC_S8X1 (6) only, not to precision %d: u8 "
                    "activations are read by the integer MMA (u8 x s8)", *mode);
    return PE_OK;
}

// The plan of `net` in mode `prec` with the conv layers of `f16_layers` (comma-separated names and "narrow"; NULL or empty: none)
// in fp16.  Each element kind lays out its activations by its own row (elem_row); plan.cpp applies the format rules.  Mixing is
// for the one-byte modes E4M3X1 and S8X1 only: the other modes' plane counts or element kinds differ from F16X1's.
static int plan_for(const NetDef& net, int prec, bool u8, const char* f16_layers, NetPlan& p, std::string& err) {
    const Precision& base = precision(prec);
    PlanFormats f;
    f.base_elem = base.fmt.elem; f.input_elem = base.input_elem; f.u8 = u8;
    for (int k = 0; k < NUM_ELEMS; k++) {
        const Precision& r = elem_row(base, (PlaneElem)k);
        f.layout[k] = {r.act_cpad, r.kp_input, r.slot_align};
    }
    for (const char* s = f16_layers; s && *s;) {
        const char* end = strchr(s, ',');
        std::string name(s, end ? end - s : strlen(s));
        name.erase(0, name.find_first_not_of(" \t"));
        name.erase(name.find_last_not_of(" \t") + 1);
        if (!name.empty()) f.f16.push_back(name);
        s = end ? end + 1 : s + strlen(s);
    }
    if (!f.f16.empty() && prec != PE_PREC_E4M3X1 && prec != PE_PREC_S8X1) {
        err = "fp16 layers mix only with PE_PREC_E4M3X1 (5) and PE_PREC_S8X1 (6), not with precision " + std::to_string(prec);
        return -1;
    }
    return build_plan_from_net(net, f, p, err);
}

// Host-only view of the element kinds of a plan (DESIGN.md section 3): "act <index> <kind> <channel pitch> <blob or ->" per
// activation, then "conv <name> <compute kind> <stored kind> <in_act> <out_act>" per conv layer; f32: the planar maps or the
// FP32_SIMT mode.
extern "C" int pe_plan_formats(int model, const char* prototxt_path, int prec_arg, const char* f16_layers, char* buf, int cap) {
    NetDef net;
    std::string err;
    int prec = 0;
    bool u8 = false;
    if (const int rc = split_precision(prec_arg, &prec, &u8)) return -rc;
    if (const int rc = query_net(model, prototxt_path, net)) return rc;
    NetPlan p;
    if (plan_for(net, prec, u8, f16_layers, p, err)) return -fail(nullptr, PE_ERR_INVALID, "%s", err.c_str());
    const int planes = precision(prec).fmt.planes;
    std::string s;
    char t[512];
    for (size_t i = 0; i < p.acts.size(); i++) {
        const ActSpec& a = p.acts[i];
        snprintf(t, sizeof t, "act %zu %s %d %s\n", i, elem_name({planes, (PlaneElem)a.elem}), a.C, a.blob.empty() ? "-" : a.blob.c_str());
        s += t;
    }
    for (const ConvSpec& c : p.convs) {
        const PlaneFmt out = c.out_act >= 0 ? PlaneFmt{planes, (PlaneElem)p.acts[c.out_act].elem} : PlaneFmt{0, ELEM_BF16};
        snprintf(t, sizeof t, "conv %s %s %s %d %d\n", c.name.c_str(), elem_name({planes, (PlaneElem)c.elem}), elem_name(out), c.in_act, c.out_act);
        s += t;
    }
    if (buf && (int)s.size() < cap) memcpy(buf, s.c_str(), s.size() + 1);
    return (int)s.size();
}

// Magnitude pruning to 2:4 in the packed K order of the PE_PREC_S8X1 plan (plan.cpp, conv_prune_2to4): the grouping the engine
// tests at pe_commit_weights to pick the sparse kernel.
extern "C" int pe_prune_2to4(int model, const char* prototxt_path, const char* layer, float* w, int cout, int cin, int k) {
    if (!layer || !w) return -fail(nullptr, PE_ERR_INVALID, "pe_prune_2to4: null layer name or weights");
    NetDef net;
    std::string err;
    if (const int rc = query_net(model, prototxt_path, net)) return rc;
    NetPlan p;
    if (plan_for(net, PE_PREC_S8X1, false, nullptr, p, err)) return -fail(nullptr, PE_ERR_INVALID, "%s", err.c_str());
    for (const ConvSpec& c : p.convs) {
        if (c.name != layer) continue;
        if (c.im2col_input) return -fail(nullptr, PE_ERR_INVALID, "pe_prune_2to4: layer %s reads the im2col'ed net input and always runs dense", layer);
        if (c.cout != cout || c.cin != cin || c.k != k)
            return -fail(nullptr, PE_ERR_INVALID, "pe_prune_2to4: layer %s is %d x %d x %dx%d, not %d x %d x %dx%d", layer, c.cout, c.cin, c.k, c.k,
                         cout, cin, k, k);
        conv_prune_2to4(c, w);
        return PE_OK;
    }
    return -fail(nullptr, PE_ERR_INVALID, "pe_prune_2to4: unknown conv layer %s", layer);
}

static int create_impl(const pe_config* cfg, const char* prototxt_path, const char* f16_layers, pe_engine** out);
extern "C" int pe_create(const pe_config* cfg, pe_engine** out) { return create_impl(cfg, nullptr, nullptr, out); }
// new caffe::Net(proto, TEST): the graph comes from the deploy prototxt (rtpose.cpp:183, net.cpp:30-50); cfg->model may be
// -1, the model then follows the Nms layer's num_parts as in rtpose.cpp:212-229.
extern "C" int pe_create_from_prototxt(const pe_config* cfg, const char* prototxt_path, pe_engine** out) {
    if (!prototxt_path) return fail(nullptr, PE_ERR_INVALID, "null prototxt path");
    return create_impl(cfg, prototxt_path, nullptr, out);
}
extern "C" int pe_create_mixed(const pe_config* cfg, const char* prototxt_path, const char* f16_layers, pe_engine** out) {
    const int mode = cfg ? cfg->precision & ~PE_PREC_FLAG_U8 : 0;
    if (cfg && mode != PE_PREC_E4M3X1 && mode != PE_PREC_S8X1)
        return fail(nullptr, PE_ERR_INVALID, "pe_create_mixed: the base precision must be PE_PREC_E4M3X1 (5) or PE_PREC_S8X1 (6), not %d", mode);
    return create_impl(cfg, prototxt_path, f16_layers, out);
}

static int create_impl(const pe_config* cfg_in, const char* prototxt_path, const char* f16_layers, pe_engine** out) {
    if (!cfg_in || !out) return fail(nullptr, PE_ERR_INVALID, "null argument");
    *out = nullptr;
    pe_config cfg_copy = *cfg_in;
    pe_config* cfg = &cfg_copy;
    bool u8 = false;
    if (const int rc = split_precision(cfg_in->precision, &cfg->precision, &u8)) return rc;
    const Precision& prec = precision(cfg->precision);
    NetDef netdef;
    NetPlan plan;
    if (prototxt_path) {
        std::string perr;
        if (parse_prototxt_file(prototxt_path, netdef, perr)) return fail(nullptr, PE_ERR_IO, "%s: %s", prototxt_path, perr.c_str());
        if (plan_for(netdef, cfg->precision, u8, f16_layers, plan, perr))
            return fail(nullptr, PE_ERR_INVALID, "%s: %s", prototxt_path, perr.c_str());
        if (cfg->model >= 0 && cfg->model != plan.model)
            return fail(nullptr, PE_ERR_INVALID, "%s describes the %s model (nms num_parts %d), the configuration asks for model %d", prototxt_path,
                        plan.model == PE_MODEL_MPI_15 ? "MPI" : "COCO", plan.nms_num_parts, cfg->model);
        cfg->model = plan.model;
    }
    if (cfg->model != PE_MODEL_MPI_15 && cfg->model != PE_MODEL_COCO_18) return fail(nullptr, PE_ERR_INVALID, "unknown model %d", cfg->model);
    if (!prototxt_path) {
        std::string perr;
        if (plan_for(builtin_netdef(cfg->model, 6), cfg->precision, u8, f16_layers, plan, perr)) return fail(nullptr, PE_ERR_INVALID, "%s", perr.c_str());
    }
    if (cfg->net_w <= 0 || cfg->net_h <= 0 || cfg->net_w % 8 || cfg->net_h % 8)
        return fail(nullptr, PE_ERR_INVALID, "net resolution %dx%d must be positive multiples of 8", cfg->net_w, cfg->net_h);
    if (cfg->num_scales < 1 || cfg->num_scales > PE_MAX_SCALES) return fail(nullptr, PE_ERR_INVALID, "num_scales %d out of [1,%d]", cfg->num_scales, PE_MAX_SCALES);
    if (cfg->max_batch < 1 || cfg->max_batch > 64) return fail(nullptr, PE_ERR_INVALID, "max_batch %d out of [1,64]", cfg->max_batch);
    if (check_resize_scales(nullptr, (float)cfg->start_scale, (float)cfg->scale_gap, cfg->num_scales)) return PE_ERR_INVALID;
    if (cfg->disp_w <= 0 || cfg->disp_h <= 0) return fail(nullptr, PE_ERR_INVALID, "bad display resolution");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail(nullptr, PE_ERR_CUDA, "no CUDA device visible: the pose engine has no CPU fallback");
    if (cfg->device < 0 || cfg->device >= ndev) return fail(nullptr, PE_ERR_INVALID, "device %d out of range (%d visible)", cfg->device, ndev);

    pe_engine* e = new pe_engine();
    e->cfg = *cfg;
    e->mt_own = model_tables(cfg->model);
    if (prototxt_path) e->mt_own.max_peaks = plan.nms_max_peaks;   // nms_param.max_peaks (NmsLayer::GetMaxPeaks, rtpose.cpp:195)
    e->mt = &e->mt_own;
    e->prec = &prec;
    e->u8 = u8;
    if (const char* g = getenv("PE_CHECK_RANGE")) e->check_range = atoi(g) != 0;
    e->start_scale_f = (float)cfg->start_scale;  // ImResizeLayer::SetStartScale(float)
    e->scale_gap_f = (float)cfg->scale_gap;
    auto bail = [&](int rc) { g_create_error = e->err; pe_destroy(e); return rc; };
#define CKC(call) do { cudaError_t err_ = (call); if (err_ != cudaSuccess) { \
    fail(e, PE_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(err_), __FILE__, __LINE__); return bail(PE_ERR_CUDA); } } while (0)
    CKC(cudaSetDevice(cfg->device));
    if (prec.fmt.planes) {
        cudaDeviceProp prop;
        CKC(cudaGetDeviceProperties(&prop, cfg->device));
        if (prop.major != 9) { fail(e, PE_ERR_INVALID, "wgmma precision modes need sm_90 (found sm_%d%d)", prop.major, prop.minor); return bail(PE_ERR_INVALID); }
    }
    CKC(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
    for (int i = 0; i < 16; i++) CKC(cudaEventCreate(&e->ev[i]));

    // the plan first: each level's gap is the largest pad of its convolutions (common.h)
    e->plan = plan;
    for (const ConvSpec& c : e->plan.convs)   // the s32 bound of the layers that compute in s8, u8 or two s8 planes
        if (const long long max_k = elem_row(prec, (PlaneElem)c.elem).max_k) {
            const long long K = (long long)(c.im2col_input ? 1 : c.k * c.k) * c.in_cused;
            const bool cu8 = c.elem == ELEM_U8, x2 = prec.fmt.planes == 2;
            if (K > max_k) {
                fail(e, PE_ERR_INVALID, "layer %s: K = %lld (%dx%d taps x %d padded input channels) exceeds %lld, the largest K whose %s sums "
                     "stay inside s32 (|acc| <= %s x K): %s cannot run it", c.name.c_str(), K, c.k, c.k, c.in_cused, max_k,
                     cu8 ? "u8 x s8" : x2 ? "hi x lo + lo x hi" : "s8", cu8 ? "255 x 127" : x2 ? "(128 x 128 + 128 x 127)" : "128 x 127",
                     cu8 ? "PE_PREC_S8X1 with u8 activations" : x2 ? "PE_PREC_S8X2" : "PE_PREC_S8X1");
                return bail(PE_ERR_INVALID);
            }
        }
    const int N = cfg->max_batch * cfg->num_scales;
    image_geo(e, N, e->geo);
    if (e->geo[3].W * 8 != cfg->net_w || e->geo[3].H * 8 != cfg->net_h) { fail(e, PE_ERR_INVALID, "net size not divisible by 8 after pooling"); return bail(PE_ERR_INVALID); }
    e->hw.resize(e->plan.convs.size());
    if (prec.fmt.planes && setup_lanes(e)) return bail(PE_ERR_CUDA);
    // FLOPs (SURVEY.md section 8d): 2*Cout*Cin*k^2*Hout*Wout per conv and image
    e->flops_per_scale = 0;
    for (auto& c : e->plan.convs) {
        const Geo& g = e->geo[c.level];
        c.flops_per_image = 2.0 * c.cout * c.cin * c.k * c.k * g.H * g.W;
        e->flops_per_scale += c.flops_per_image;
    }
    // io buffers
    CKC(e->d_frames.reserve((size_t)cfg->disp_w * cfg->disp_h * 3 * cfg->max_batch));
    CKC(e->d_resized.reserve((size_t)N * cfg->net_w * cfg->net_h * 3));
    CKC(e->d_planar.reserve((size_t)N * 3 * cfg->net_w * cfg->net_h * sizeof(float)));
    if (build_pre_tables(e)) return bail(PE_ERR_INVALID);
    e->pre.frames = e->d_frames.get(); e->pre.resized = e->d_resized.get();
    e->pre.kp = e->plan.kp_input; e->pre.fmt = act_fmt(e, e->plan.input_act);
    e->pre.Wp = e->geo[0].Wp; e->pre.Hs = e->geo[0].Hs;
    // activations and maps
    if (alloc_images(e, N)) return bail(PE_ERR_CUDA);

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
    const size_t B = cfg->max_batch, P = e->mt->num_parts, MP = e->mt->max_peaks, NL = e->mt->num_limbs;
    pd.copies = cfg->num_scales;
    std::vector<int> perm;
    std::vector<float> sign;
    if (model_flip_table(cfg->model, perm, sign) != e->mt->num_maps) { fail(e, PE_ERR_INVALID, "model %d: a part or limb has no mirror", cfg->model); return bail(PE_ERR_INVALID); }
    std::vector<FlipTap> flip(perm.size());
    for (size_t c = 0; c < perm.size(); c++) flip[c] = {perm[c], sign[c]};
    pd.sort_stride = 1;
    while (pd.sort_stride < (int)(MP * MP)) pd.sort_stride <<= 1;
    CKC(post_set_smem_limits());
    pd.p.max_subset_rows = (int)(NL * MP);
    CKC(reserve_carved(e->d_post, [&](Carver& d) {   // the post-processing arrays and the axis tables
        pd.xtab = e->d_xtab = d.take<AxisTap>((size_t)cfg->num_scales * cfg->net_w); pd.ytab = e->d_ytab = d.take<AxisTap>((size_t)cfg->num_scales * cfg->net_h);
        pd.flip = d.take<FlipTap>(flip.size());
        pd.flags = d.take<unsigned>(B * P * cfg->net_h * ((cfg->net_w + 31) / 32)); pd.peaks = d.take<float>(B * P * (MP + 1) * 3);
        pd.cands = d.take<Cand>(B * NL * MP * MP); pd.cand_count = d.take<int>(B * NL);
        pd.conns = d.take<Conn>(B * NL * MP); pd.conn_count = d.take<int>(B * NL);
        pd.subset = d.take<double>(B * pd.p.max_subset_rows * (P + 3)); pd.subset_rows = d.take<int>(B);
        pd.joints = d.take<float>(B * PE_MAX_PEOPLE * P * 3); pd.num_people = d.take<int>(B);
    }));
    CKC(reserve_carved(e->h_results, [&](Carver& r) { e->h_joints = r.take<float>(B * PE_MAX_PEOPLE * P * 3); e->h_num_people = r.take<int>(B);
                                                       e->h_peaks = r.take<float>(B * P * (MP + 1) * 3); }));
    CKC(cudaMemset(pd.conn_count, 0, sizeof(int) * B * NL));
    CKC(cudaMemcpy((void*)pd.flip, flip.data(), flip.size() * sizeof(FlipTap), cudaMemcpyHostToDevice));
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
    for (auto& t : e->tc) tc_layer_destroy(t);
    if (e->ev_wait) cudaEventDestroy(e->ev_wait);
    for (cudaEvent_t ev : e->conv_done) if (ev) cudaEventDestroy(ev);
    if (e->stream2) { cudaStreamSynchronize(e->stream2); cudaStreamDestroy(e->stream2); }
    for (int i = 0; i < 16; i++) if (e->ev[i]) cudaEventDestroy(e->ev[i]);
    if (e->stream) cudaStreamDestroy(e->stream);
    delete e;   // the buffers free themselves, on the device set above (packed weights: on their own device)
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

static size_t conv_k(const pe_engine* e, int i) { return (size_t)(e->plan.convs[i].im2col_input ? 1 : e->plan.convs[i].k * e->plan.convs[i].k) * e->cin_pad[i]; }
// bytes of conv i's packed weights: the planes [P][cout_pad][K], or the compressed values and metadata of a sparse layer
static size_t weight_bytes(const pe_engine* e, int i) {
    return e->sparse[i] ? s8_sparse_bytes(e->cout_pad[i], conv_k(e, i)) : conv_k(e, i) * e->cout_pad[i] * fmt_bytes(conv_wfmt(e, i));
}

// byte layout of the packed weight buffer (a function of the plan, the precision and the sparse layers only, so replicas that
// take the sender's sparse layers agree on it)
static size_t packed_layout(pe_engine* e) {
    const size_t nc = e->plan.convs.size();
    e->w_off.assign(nc, 0); e->b_off.assign(nc, 0); e->cout_pad.assign(nc, 0); e->cin_pad.assign(nc, 0);
    size_t total = 0;
    auto align256 = [](size_t v) { return (v + 255) / 256 * 256; };
    for (size_t i = 0; i < nc; i++) {
        const ConvSpec& c = e->plan.convs[i];
        e->cin_pad[i] = c.in_cused;
        e->cout_pad[i] = e->sparse[i] ? (c.cout + SP_BM - 1) / SP_BM * SP_BM : e->prec->fmt.planes ? tc_cout_pad(c.cout) : (c.cout + 63) / 64 * 64;
        e->w_off[i] = total;
        total = align256(total + weight_bytes(e, (int)i));
        e->b_off[i] = total;
        total = align256(total + epi_floats(e, (int)i) * 4);
    }
    return total;
}

// Range scales.  Every conv output is stored as  true value * s  with s = conv_scale[producer] (a power of two; pools and copies
// pass values through unchanged).  A consumer whose input channels come from producers with DIFFERENT scales (a Concat: conv4_4_CPM
// next to the previous stage's L1 / L2 outputs) folds the ratios into its weights: packed w[ci] = w[ci] * s_ref / s(ci) * 2^k, so that
//   acc = 2^k * s_ref * sum_ci w[ci] * a[ci]     and     stored = acc * out_scale + bias,  out_scale = s_out / (2^k * s_ref),
// bias = true bias * s_out - all factors powers of two, hence exact, and ReLU commutes with them: range scaling is free at run time.
// S8X1 and S8X2 replace 2^k by a step per output channel (sigma_c, s8.h): acc * sigma_c ~ s_ref * sum w a, and the factor of channel c
// is f_c = sigma_c * s_out / s_ref.  The net input carries the mode's net_input_scale.
//
// The one rule that picks those powers of two (range scales and the weights' 2^k): the s that puts a maximum m into
// [2^(top-1), 2^top), exponent clamped to [-100, 100]; `otherwise` when m says nothing (0, infinite or NaN).
static float pow2_for(float m, int top, float otherwise = 1.f) {
    if (!(m > 0.f && m < 3e38f)) return otherwise;
    int ex = 0;
    frexpf(m, &ex);
    return ldexpf(1.f, std::max(-100, std::min(100, top - ex)));
}
static int log2_of_scale(float s) { int ex = 0; frexpf(s, &ex); return ex - 1; }
static float input_ref_scale(const pe_engine* e, const ConvSpec& c) {
    for (int pc : c.cin_prod) if (pc >= 0) return e->conv_scale[pc];
    return elem_row(*e->prec, (PlaneElem)e->plan.acts[c.in_act].elem).net_input_scale;   // the net input
}
static void fill_epilogue_fields(const pe_engine* e, int i, float* B) {
    const ConvSpec& c = e->plan.convs[i];
    const float s_ref = input_ref_scale(e, c);
    const float s_out = c.out_act >= 0 ? e->conv_scale[i] : 1.f;   // the planar stride-8 maps are true values
    for (int co = 0; co < c.cout; co++) B[co] = e->hw[i].b[co] * s_out;
    if (conv_row(e, i).per_channel_epilogue) {
        // S8X2's sum S = 256 acc_h + acc_c counts in units of 2^8 (the place of the dropped lo*lo): f_c carries that 2^8 too
        const float unit = conv_row(e, i).fmt.planes == 2 ? 256.f : 1.f;
        for (int co = 0; co < c.cout; co++) B[e->cout_pad[i] + co] = e->wsig[i][co] * (s_out / s_ref) * unit;
        return;
    }
    B[e->cout_pad[i]] = e->wsi[i] * s_out / s_ref;
}

// Weights of conv i into `dst` (the layer's region of the packed buffer, host copy): fp32 [K][cout_pad] for the SIMT mode, else
// P 16-bit planes [P][cout_pad][K] (K-major rows: the wgmma B operand) of w * 2^k, the per-channel range ratios folded in.
// Sets e->wsi[i] = 2^-k.  S8X1: one s8 plane [cout_pad][K], each output channel quantised on its own (s8.h); sets e->wsig[i].
// S8X2: the same with 16-bit integers in two s8 planes.
static int pack_conv_weights(pe_engine* e, int i, uint8_t* dst) {
    const ConvSpec& c = e->plan.convs[i];
    const HostWeights& hw = e->hw[i];
    const int taps = c.im2col_input ? 1 : c.k * c.k, cp = e->cin_pad[i], cop = e->cout_pad[i];
    const size_t K = (size_t)taps * cp;
    const float s_ref = input_ref_scale(e, c);
    std::vector<float> chan(cp, 1.f);   // s_ref / s(ci) per engine input channel
    for (int ec = 0; ec < cp && ec < (int)c.cin_prod.size(); ec++)
        if (c.cin_prod[ec] >= 0) chan[ec] = s_ref / e->conv_scale[c.cin_prod[ec]];
    auto src = [&](int co, int kk) -> float {  // engine K index -> Caffe weight (co, ci, r, s) (plan.cpp)
        const long long wi = conv_weight_index(c, co, kk);
        return wi < 0 ? 0.f : c.im2col_input ? hw.w[wi] : hw.w[wi] * chan[kk % cp];
    };
    const PlaneFmt wf = conv_wfmt(e, i);
    memset(dst, 0, weight_bytes(e, i));
    float wscale_inv = 1.f;
    if (wf.s8() && wf.planes == 2) {   // PE_PREC_S8X2: planes [hi, lo][cout_pad][K] of each channel's 16-bit integers (s8.h)
        int8_t* hi = (int8_t*)dst;
        int8_t* lo = hi + (size_t)cop * K;
        std::vector<float> wc(K);
        e->wsig[i].assign(cop, 0.f);
        for (int co = 0; co < c.cout; co++) {
            for (size_t kk = 0; kk < K; kk++) wc[kk] = src(co, (int)kk);
            e->wsig[i][co] = s8x2_quantize_channel(wc.data(), K, hi + (size_t)co * K, lo + (size_t)co * K);
        }
    } else if (wf.s8() || wf.u8()) {   // a u8 layer's weights are s8 too: its MMA is u8 x s8
        // a sparse layer quantises into a dense plane first and stores it compressed (s8_sparse.h); quantisation only adds zeros
        std::vector<int8_t> dense(e->sparse[i] ? K * cop : 0);
        int8_t* q = e->sparse[i] ? dense.data() : (int8_t*)dst;
        std::vector<float> wc(K);
        e->wsig[i].assign(cop, 0.f);
        for (int co = 0; co < c.cout; co++) {
            for (size_t kk = 0; kk < K; kk++) wc[kk] = src(co, (int)kk);
            e->wsig[i][co] = s8_quantize_channel(wc.data(), K, q + (size_t)co * K);
        }
        // the sparse choice was made from these fp32 weights, and quantisation only adds zeros: a group with three non-zeros here
        // means the choice and the weights disagree, and the compressed bytes would be wrong
        if (e->sparse[i] && !s8_sparse_compress(q, cop, K, dst))
            return fail(e, PE_ERR_STATE, "layer %s: its weights are not 2:4 but the layer was chosen to run sparse", c.name.c_str());
    } else if (wf.planes == 0) {  // fp32 [K][cout_pad]
        float* W = (float*)dst;
        for (size_t kk = 0; kk < K; kk++)
            for (int co = 0; co < c.cout; co++) W[kk * cop + co] = src(co, (int)kk);
    } else {
        uint16_t* W = (uint16_t*)dst;
        const size_t plane = (size_t)cop * K;
        // scale the layer by 2^k so that max|w| lands below 2^weight_top (precision.h).  Exact (power of two); the epilogue
        // multiplies by 2^-k.
        float wscale = 1.f;
        if (const int top = weight_top(wf.elem)) {
            float mx = 0.f;
            for (int co = 0; co < c.cout; co++)
                for (size_t kk = 0; kk < K; kk++) mx = fmaxf(mx, fabsf(src(co, (int)kk)));
            wscale = pow2_for(mx, top);
        }
        wscale_inv = 1.f / wscale;
        if (wf.e4m3()) {   // one byte per weight, [cout_pad][K]
            for (int co = 0; co < c.cout; co++)
                for (size_t kk = 0; kk < K; kk++) dst[(size_t)co * K + kk] = float_to_e4m3(src(co, (int)kk) * wscale);
        } else {
            for (int co = 0; co < c.cout; co++)
                for (size_t kk = 0; kk < K; kk++) {
                    uint16_t h[3];
                    if (wf.f16()) split_fp16(src(co, (int)kk) * wscale, wf.planes, h);
                    else split_bf16(src(co, (int)kk), wf.planes, h);
                    for (int p = 0; p < wf.planes; p++) W[p * plane + (size_t)co * K + kk] = h[p];
                }
        }
    }
    e->wsi[i] = wscale_inv;
    return PE_OK;
}

// per-layer launch state (TMA descriptors) over the packed buffer the handle currently points at
static int bind_packed(pe_engine* e) {
    const size_t nc = e->plan.convs.size();
    if (e->prec->ranged() && !e->d_range.size()) { CK(e, e->d_range.reserve(nc * sizeof(unsigned))); CK(e, cudaMemset(e->d_range.get(), 0, nc * sizeof(unsigned))); }
    if (e->prec->fmt.planes) {
        for (auto& t : e->tc) tc_layer_destroy(t);
        e->tc.assign(nc, TcLayer());
        for (size_t i = 0; i < nc; i++) {
            const ConvSpec& c = e->plan.convs[i];
            const Geo& g = e->geo[c.level];
            TcLayerDesc d;
            d.in = e->acts[c.in_act].get(); d.in_pitch = e->plan.acts[c.in_act].C; d.in_cused = c.in_cused; d.in_plane = e->act_plane[c.in_act];
            d.w = e->packed->get() + e->w_off[i]; d.bias = (const float*)(e->packed->get() + e->b_off[i]);
            d.cout = c.cout; d.cout_pad = e->cout_pad[i]; d.ksize = c.im2col_input ? 1 : c.k; d.pad = c.im2col_input ? 0 : c.pad;
            d.relu = c.relu; d.fmt = conv_wfmt(e, (int)i); d.geo = g; d.out_scale = d.bias + e->cout_pad[i];
            d.out_elem = conv_out_elem(e, (int)i); d.chunked = conv_row(e, (int)i).chunked; d.sparse = e->sparse[i];
            d.range = e->prec->ranged() ? e->d_range.get<unsigned>() + i : nullptr;
            if (c.out_act >= 0) {
                d.out = e->acts[c.out_act].get(); d.out_pitch = e->plan.acts[c.out_act].C; d.out_coff = c.out_coff; d.out_plane = e->act_plane[c.out_act];
                d.planar = nullptr; d.planar_C = 0; d.planar_coff = 0;
            } else {
                d.out = nullptr; d.out_pitch = 0; d.out_coff = 0; d.out_plane = 0;
                d.planar = e->d_maps.get<float>(); d.planar_C = e->mt->num_maps; d.planar_coff = c.planar_coff;
            }
            std::string err;
            if (tc_layer_create(d, e->tc[i], err)) return fail(e, PE_ERR_CUDA, "layer %s: %s", c.name.c_str(), err.c_str());
        }
    }
    drop_graphs(e);
    e->committed = true;
    return PE_OK;
}

// Layers that may run the 2:4-sparse kernel (conv_s8_sparse.cu) when their weights are 2:4 in the packed K order:
//   1. s8 arithmetic with an s8 or fp32-map output (not the fp16 layers of a mixed engine, nor their s8 -> fp16 boundary layers);
//   2. not conv1_1, whose im2col'ed input is no conv window;
//   4. the shape rule: only a layer class where the sparse kernel measures faster than the dense one.  As built it is slower in
//      every class of the shipped nets (DESIGN.md section 5: 7x7, first 7x7 of a stage, VGG 3x3, stage-1 3x3, conv1_x and 1x1,
//      1.2-2.2x the dense kernel's time), and no other shape has been measured, so no class qualifies and every layer runs dense.
//      pe_test_force_sparse lifts this rule, so that tests and tools/sparse_s8.py can run and measure the kernel.
// (Rule 3, the 2:4 weights, is checked by commit.)  An engine with u8 activations (PE_PREC_FLAG_U8) runs every layer dense: the
// sparse kernel is s8 x s8 only.  So does PE_PREC_S8X2: the sparse kernel reads one plane.
static bool sparse_eligible(const pe_engine* e, int i) {
    const ConvSpec& c = e->plan.convs[i];
    const PlaneFmt wf = conv_wfmt(e, i);
    return e->force_sparse && !e->u8 && wf.s8() && wf.planes == 1 && conv_out_elem(e, i) == ELEM_S8 && !c.im2col_input;
}

// Test hook, not part of the public header: with on != 0 the next pe_commit_weights of e picks the sparse kernel for every layer
// that rules 1-3 of sparse_eligible admit, ignoring the shape rule.  Returns 0, or PE_ERR_INVALID for a null handle or an engine
// with u8 activations.
extern "C" int pe_test_force_sparse(pe_engine* e, int on) {
    if (!e) return PE_ERR_INVALID;
    if (e->u8 && on) return fail(e, PE_ERR_INVALID, "pe_test_force_sparse: an engine with u8 activations runs no layer sparse (the sparse kernel is s8 x s8)");
    e->force_sparse = on != 0;
    return PE_OK;
}

// pe_commit_weights; `sparse_from`: the sparse layers to take (a broadcast replica, which has no weights to decide from), or null
// to choose them from the fp32 weights.  The choice is made before quantisation, so re-packing keeps it.
static int commit(pe_engine* e, const std::vector<char>* sparse_from) {
    if (!e) return PE_ERR_INVALID;
    if (e->collecting) return fail(e, PE_ERR_STATE, "a calibration collection is running: call pe_calibrate_end first");
    CK(e, cudaSetDevice(e->cfg.device));
    const size_t nc = e->plan.convs.size();
    e->weights_hash_valid = false;
    for (size_t i = 0; i < nc; i++) {
        const ConvSpec& c = e->plan.convs[i];
        if (!e->hw[i].set || e->hw[i].w.size() != (size_t)c.cout * c.cin * c.k * c.k || e->hw[i].b.size() != (size_t)c.cout)
            return fail(e, PE_ERR_STATE, "weights of layer %s were never set%s", c.name.c_str(),
                        e->committed ? " on this handle (a broadcast replica keeps no fp32 copy: set every layer again)" : "");
    }
    e->committed = false;   // the layout changes under the bound buffer: no forward until this commit succeeds
    e->sparse.assign(nc, 0);
    for (size_t i = 0; i < nc; i++)
        e->sparse[i] = sparse_from ? (*sparse_from)[i] : sparse_eligible(e, (int)i) && conv_weights_2to4(e->plan.convs[i], e->hw[i].w.data());
    const size_t total = packed_layout(e);
    e->calibrated = false;
    e->wsi.assign(nc, 1.f);
    e->wsig.assign(nc, std::vector<float>());
    e->conv_scale.assign(nc, 1.f);
    std::vector<uint8_t> host(total, 0);
    for (size_t i = 0; i < nc; i++) {
        if (pack_conv_weights(e, (int)i, host.data() + e->w_off[i])) return PE_ERR_STATE;
        fill_epilogue_fields(e, (int)i, (float*)(host.data() + e->b_off[i]));   // travels with the packed buffer (weight broadcast)
    }
    e->packed.reset();   // the old buffer goes first (unless another handle still uses it)
    e->packed = std::shared_ptr<DeviceBuffer>(new DeviceBuffer(), [dev = e->cfg.device](DeviceBuffer* b) { int cur = 0; cudaGetDevice(&cur); cudaSetDevice(dev); delete b; cudaSetDevice(cur); });
    CK(e, e->packed->reserve(total));
    CK(e, cudaMemcpy(e->packed->get(), host.data(), total, cudaMemcpyHostToDevice));
    return bind_packed(e);
}
extern "C" int pe_commit_weights(pe_engine* e) { return commit(e, nullptr); }

// Net::ShareTrainedLayersWith (src/caffe/net.cpp:682-706): a second net on the SAME GPU uses the first one's weights instead of
// loading them again - here the packed device buffer itself (no copy; it lives until the last handle that uses it is destroyed).
// For two worker handles per GPU (copies of one batch overlap the compute of the other, rtpose.bin --engines_per_gpu).
extern "C" int pe_share_weights(pe_engine* from, pe_engine* to) {
    if (!from || !to || from == to) return fail(from, PE_ERR_INVALID, "bad arguments");
    if (!from->committed) return fail(from, PE_ERR_STATE, "the source handle has no committed weights");
    if (to->cfg.device != from->cfg.device) return fail(from, PE_ERR_INVALID, "handles are on different GPUs (use pe_broadcast_weights)");
    if (to->cfg.model != from->cfg.model || to->cfg.precision != from->cfg.precision || to->plan.convs.size() != from->plan.convs.size())
        return fail(from, PE_ERR_INVALID, "the handles run different nets (model / precision / graph)");
    if (to->u8 != from->u8) return fail(from, PE_ERR_INVALID, "one handle has u8 activations (PE_PREC_FLAG_U8), the other not");
    for (size_t i = 0; i < to->plan.convs.size(); i++) {
        const ConvSpec &a = from->plan.convs[i], &b = to->plan.convs[i];
        if (a.name != b.name || a.cout != b.cout || a.cin != b.cin || a.k != b.k) return fail(from, PE_ERR_INVALID, "layer %s differs between the handles", a.name.c_str());
        if (a.elem != b.elem) return fail(from, PE_ERR_INVALID, "layer %s runs in fp16 in one handle only: the fp16 layers differ", a.name.c_str());
    }
    CK(to, cudaSetDevice(to->cfg.device));
    CK(to, cudaStreamSynchronize(to->stream));
    // the receiver runs the sender's packed buffer, sparse layers included; on a layout mismatch it keeps its own layout
    const std::vector<char> own_sparse = to->sparse;
    const std::vector<size_t> own_w = to->w_off, own_b = to->b_off;
    const std::vector<int> own_cout = to->cout_pad, own_cin = to->cin_pad;
    to->sparse = from->sparse;
    if (packed_layout(to) != from->packed->size()) {
        to->sparse = own_sparse; to->w_off = own_w; to->b_off = own_b; to->cout_pad = own_cout; to->cin_pad = own_cin;
        return fail(from, PE_ERR_STATE, "packed layouts differ");
    }
    to->packed = from->packed;
    for (auto& h : to->hw) { std::vector<float>().swap(h.w); std::vector<float>().swap(h.b); h.set = false; }
    to->conv_scale = from->conv_scale; to->calibrated = from->calibrated;
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
        if (e->u8 != root->u8) return fail(root, PE_ERR_INVALID, "engine %d is not a replica of engine 0 (u8 activations in one only)", i);
        bool same = e->plan.convs.size() == root->plan.convs.size();
        for (size_t l = 0; same && l < e->plan.convs.size(); l++) same = e->plan.convs[l].elem == root->plan.convs[l].elem;
        if (!same) return fail(root, PE_ERR_INVALID, "engine %d is not a replica of engine 0 (the fp16 layers differ)", i);
        // allocate the packed buffer + TMA maps with the same layout and sparse layers (values arrive by broadcast)
        if (!e->committed || e->sparse != root->sparse) {
            for (size_t l = 0; l < e->plan.convs.size(); l++) {
                const ConvSpec& c = e->plan.convs[l];
                e->hw[l].w.assign((size_t)c.cout * c.cin * c.k * c.k, 0.f);
                e->hw[l].b.assign(c.cout, 0.f);
                e->hw[l].set = true;
            }
            const int rc = commit(e, &root->sparse);
            if (rc) return rc;
            // the replica holds no fp32 copy: a later pe_set_conv_weights on a subset + pe_commit_weights must fail
            // ("weights of layer ... were never set") instead of packing from empty vectors
            for (auto& h : e->hw) { std::vector<float>().swap(h.w); std::vector<float>().swap(h.b); h.set = false; }
        }
        if (e->packed->size() != root->packed->size()) return fail(root, PE_ERR_STATE, "packed layouts differ");
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
        rc = bcast(root->packed->get(), engines[i]->packed->get(), root->packed->size(), 0 /*ncclChar*/, 0, comms[i], engines[i]->stream);
    }
    const int rc2 = gend();
    for (int i = 0; i < n; i++) { cudaSetDevice(devs[i]); cudaStreamSynchronize(engines[i]->stream); }
    for (int i = 0; i < n; i++) destroy(comms[i]);
    if (rc || rc2) return fail(root, PE_ERR_CUDA, "ncclBroadcast: %s", errstr ? errstr(rc ? rc : rc2) : "error");
    // the range scales travel inside the packed buffer; the replicas also take the host copy that pe_fetch_blob divides out and
    // the calibration state that an S8X1 forward requires
    for (int i = 1; i < n; i++) { engines[i]->conv_scale = root->conv_scale; engines[i]->calibrated = root->calibrated; }
    return PE_OK;
}

extern "C" size_t pe_packed_weights_bytes(const pe_engine* e) { return e && e->packed ? e->packed->size() : 0; }

extern "C" int pe_conv_layer_sparse(const pe_engine* e, int idx) {
    if (!e) return -PE_ERR_INVALID;
    if (idx < 0 || idx >= (int)e->plan.convs.size()) return -fail((pe_engine*)e, PE_ERR_INVALID, "conv layer index %d out of range", idx);
    if (!e->committed) return -fail((pe_engine*)e, PE_ERR_STATE, "pe_conv_layer_sparse: pe_commit_weights has not been called");
    return e->sparse[idx] ? 1 : 0;
}
extern "C" void* pe_packed_weights_device_ptr(pe_engine* e) { return e && e->packed ? e->packed->get() : nullptr; }

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
// A value that would crop outside the maps is refused: the old one stays, nothing is launched and the graphs are kept.
extern "C" int pe_resize_set_start_scale(pe_engine* e, float s) {
    if (!e) return PE_ERR_INVALID;
    if (int rc = check_resize_scales(e, s, e->scale_gap_f, e->cfg.num_scales)) return rc;
    e->start_scale_f = s;
    return rebuild_axis(e);
}
extern "C" int pe_resize_set_scale_gap(pe_engine* e, float g) {
    if (!e) return PE_ERR_INVALID;
    if (int rc = check_resize_scales(e, e->start_scale_f, g, e->cfg.num_scales)) return rc;
    e->scale_gap_f = g;
    return rebuild_axis(e);
}
extern "C" float pe_resize_get_start_scale(const pe_engine* e) { return e ? e->start_scale_f : 0.f; }
extern "C" float pe_resize_get_scale_gap(const pe_engine* e) { return e ? e->scale_gap_f : 0.f; }
extern "C" int pe_set_connect_params(pe_engine* e, int min_cnt, float min_score, float inter_thr, int min_above) {
    if (!e) return PE_ERR_INVALID;
    PostParams& p = e->post.p;
    drop_graphs(e);
    p.min_subset_cnt = min_cnt; p.min_subset_score = min_score; p.inter_threshold = inter_thr; p.inter_min_above = min_above;
    return PE_OK;
}

// The flip test.  Turning it on the first time doubles the per-image buffers; they stay that size when it is turned off again (a
// forward reads only its own images).  The results of earlier forwards are dropped: their maps have the other layout.
extern "C" int pe_set_flip_test(pe_engine* e, int on) {
    if (!e) return PE_ERR_INVALID;
    if (e->collecting)
        return fail(e, PE_ERR_STATE, "pe_set_flip_test: a calibration collection is running: call pe_calibrate_end first");
    if ((on != 0) == e->flip) return PE_OK;
    CK(e, cudaSetDevice(e->cfg.device));
    const int need = 2 * e->cfg.max_batch * e->cfg.num_scales;
    if (on && e->geo[0].N < need) { const int rc = alloc_images(e, need); if (rc) return rc; }
    CK(e, cudaStreamSynchronize(e->stream));
    drop_graphs(e);
    e->flip = on != 0;
    e->pre.flip = e->flip;
    e->post.copies = copies(e);
    e->last_n = 0;
    e->jstatus_n = 0;
    return PE_OK;
}
extern "C" int pe_get_flip_test(const pe_engine* e) { return e && e->flip ? 1 : 0; }

extern "C" int pe_model_flip_table(int model, int* perm, float* sign, int cap) {
    if (model != PE_MODEL_MPI_15 && model != PE_MODEL_COCO_18) return -fail(nullptr, PE_ERR_INVALID, "unknown model %d", model);
    std::vector<int> p;
    std::vector<float> s;
    const int n = model_flip_table(model, p, s);
    if (n < 0) return -fail(nullptr, PE_ERR_STATE, "model %d: a part or limb has no mirror", model);
    if (cap >= n) {
        if (perm) memcpy(perm, p.data(), n * sizeof(int));
        if (sign) memcpy(sign, s.data(), n * sizeof(float));
    }
    return n;
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
        if (e->prec->fmt.planes) {
            const int n = tc_layer_launch(e->tc[op.idx], nimg, st, share);
            if (n < 0) return fail(e, PE_ERR_CUDA, "conv %s: tensor-core launch failed or no kernel fits the tile (%s)", c.name.c_str(), cudaGetErrorString(cudaGetLastError()));
            e->launches += n;
            return PE_OK;
        }
        ConvArgs a;
        memset(&a, 0, sizeof a);
        a.in = e->acts[c.in_act].get(); a.in_pitch = e->plan.acts[c.in_act].C;
        a.w = e->packed->get() + e->w_off[op.idx]; a.bias = (const float*)(e->packed->get() + e->b_off[op.idx]);
        if (c.out_act >= 0) { a.out = e->acts[c.out_act].get(); a.out_pitch = e->plan.acts[c.out_act].C; a.out_coff = c.out_coff; }
        else { a.planar = e->d_maps.get<float>(); a.planar_C = e->mt->num_maps; a.planar_coff = c.planar_coff; }
        a.cin_pad = e->cin_pad[op.idx]; a.cout = c.cout; a.cout_pad = e->cout_pad[op.idx];
        a.ksize = c.im2col_input ? 1 : c.k; a.pad = c.im2col_input ? 0 : c.pad; a.relu = c.relu;
        a.W = g.W; a.H = g.H; a.Wp = g.Wp; a.Hs = g.Hs; a.N = nimg; a.M = M;
        e->launches += launch_conv_simt(a, st);
    } else if (op.type == 1) {
        const PoolSpec& p = e->plan.pools[op.idx];
        const Geo& gi = e->geo[p.level_in]; const Geo& go = e->geo[p.level_in + 1];
        PoolArgs a;
        a.in = e->acts[p.in_act].get(); a.out = e->acts[p.out_act].get(); a.C = e->plan.acts[p.in_act].C;
        a.in_plane = e->act_plane[p.in_act]; a.out_plane = e->act_plane[p.out_act]; a.fmt = act_fmt(e, p.in_act);
        a.Wi = gi.W; a.Hi = gi.H; a.Wpi = gi.Wp; a.Hsi = gi.Hs; a.Wo = go.W; a.Ho = go.H; a.Wpo = go.Wp; a.Hso = go.Hs; a.N = nimg;
        e->launches += launch_pool(a, st);
    } else {
        const CopySpec& c = e->plan.copies[op.idx];
        const Geo& g = e->geo[3];
        CopyArgs a;
        a.src = e->acts[c.src_act].get(); a.dst = e->acts[c.dst_act].get(); a.pitch = e->plan.acts[c.src_act].C; a.channels = c.channels;
        a.fmt = act_fmt(e, c.src_act); a.elem_bytes = a.fmt.elem_bytes(); a.M = (long long)nimg * g.Hs * g.Wp; a.plane = e->act_plane[c.src_act];
        e->launches += launch_copy_channels(a, st);
    }
    return PE_OK;
}

static int run_post_and_return(pe_engine* e, int n) {
    e->post.maps = e->d_maps.get<float>();
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
    const int nimg = n * copies(e);
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
    // at scale 1 almost every activation of a typical net quantises to 0
    if (e->prec->needs_calibration && !e->calibrated)
        return fail(e, PE_ERR_STATE, "PE_PREC_%s runs on calibrated range scales: call pe_calibrate (on the handle that owns the weights) before the first forward",
                    e->cfg.precision == PE_PREC_S8X2 ? "S8X2" : "S8X1");
    if (e->collecting) e->collect_forwards++;   // its maxima accumulate in d_range (folded by pe_range_status and pe_calibrate_end)
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

// (re)allocates b to hold at least `need` bytes; the stream is drained first because queued work may still use the old buffer
template <class B>
static int grow_buffer(pe_engine* e, B& b, size_t need) {
    if (b.size() >= need) return PE_OK;
    CK(e, cudaStreamSynchronize(e->stream));
    CK(e, b.reserve(need));
    return PE_OK;
}
// The pinned staging buffer with at least `need` bytes.  The stream is drained first, grown or not: queued copies may still read it.
static int stage(pe_engine* e, size_t need) { CK(e, cudaStreamSynchronize(e->stream)); return grow_buffer(e, e->h_stage, need); }

// n host buffers (bytes[i] bytes from src[i]) to dst + i * stride.  Every pointer is checked before anything is copied.  When all are
// page-locked (pe_host_alloc) they are DMA'd directly, fully asynchronously; otherwise they go through staging in one copy.
static int upload_host(pe_engine* e, const void* const* src, const std::vector<size_t>& bytes, int n, size_t stride, uint8_t* dst, const char* what) {
    bool pinned = true;
    for (int i = 0; i < n; i++) {
        if (!src[i]) return fail(e, PE_ERR_INVALID, "null %s %d", what, i);
        cudaPointerAttributes at;
        if (pinned && (cudaPointerGetAttributes(&at, src[i]) != cudaSuccess || at.type != cudaMemoryTypeHost)) { pinned = false; cudaGetLastError(); }
    }
    if (pinned) {
        for (int i = 0; i < n; i++) CK(e, cudaMemcpyAsync(dst + i * stride, src[i], bytes[i], cudaMemcpyHostToDevice, e->stream));
        return PE_OK;
    }
    if (const int rc = stage(e, stride * n)) return rc;
    for (int i = 0; i < n; i++) memcpy(e->h_stage.get() + i * stride, src[i], bytes[i]);
    CK(e, cudaMemcpyAsync(dst, e->h_stage.get(), stride * n, cudaMemcpyHostToDevice, e->stream));
    return PE_OK;
}

// n display frames in device memory -> the net input
static int preprocess_frames(pe_engine* e, const uint8_t* d_frames, int n) {
    PreArgs a = e->pre;
    a.frames = d_frames; a.nframes = n;
    if (e->input_lo_dirty) {   // the uint8 path only writes the hi plane; drop what the planar path left behind
        const size_t bytes = (size_t)e->act_plane[e->plan.input_act] * fmt_bytes(act_fmt(e, e->plan.input_act));
        CK(e, cudaMemsetAsync(e->acts[e->plan.input_act].get(), 0, bytes, e->stream));
        e->input_lo_dirty = false;
    }
    e->launches += launch_preprocess(a, e->stream);
    e->last_frames = d_frames;
    return PE_OK;
}
extern "C" int pe_forward_frames_device(pe_engine* e, const void* d_frames, int n) {
    NvtxRange r("pe_forward_frames_device");
    int rc = check_n(e, n); if (rc) return rc;
    CK(e, cudaSetDevice(e->cfg.device));
    if ((rc = preprocess_frames(e, (const uint8_t*)d_frames, n))) return rc;
    return run_net(e, n);
}
// n display frames in host memory -> e->d_frames
static int upload_frames(pe_engine* e, const uint8_t* const* frames, int n) {
    if (!frames) return fail(e, PE_ERR_INVALID, "null frames");
    const size_t fb = (size_t)e->cfg.disp_w * e->cfg.disp_h * 3;
    return upload_host(e, (const void* const*)frames, std::vector<size_t>(n, fb), n, fb, e->d_frames.get(), "frame");
}
extern "C" int pe_forward_frames(pe_engine* e, const uint8_t* const* frames, int n) {
    NvtxRange r("pe_forward_frames (H2D)");
    int rc = check_n(e, n); if (rc) return rc;
    CK(e, cudaSetDevice(e->cfg.device));
    if ((rc = upload_frames(e, frames, n))) return rc;
    return pe_forward_frames_device(e, e->d_frames.get(), n);
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
    if (e->warp_w == ow && e->warp_h == oh) return PE_OK;
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
    std::vector<short> tab; build_warp_tab(tab);
    e->warp_w = e->warp_h = 0;   // until every table below holds this size
    CK(e, reserve_carved(e->d_warp, [&](Carver& k) {   // one size per engine: allocated once, never while queued work reads it
        e->d_wa = k.take<int>(dw); e->d_wb = k.take<int>(dw); e->d_wx0 = k.take<int>(dh); e->d_wy0 = k.take<int>(dh); e->d_wtab = k.take<short>(tab.size());
    }));
    CK(e, cudaStreamSynchronize(e->stream));
    CK(e, cudaMemcpy(e->d_wtab, tab.data(), tab.size() * sizeof(short), cudaMemcpyHostToDevice));
    CK(e, cudaMemcpy(e->d_wa, ad.data(), dw * sizeof(int), cudaMemcpyHostToDevice));
    CK(e, cudaMemcpy(e->d_wb, bd.data(), dw * sizeof(int), cudaMemcpyHostToDevice));
    CK(e, cudaMemcpy(e->d_wx0, x0.data(), dh * sizeof(int), cudaMemcpyHostToDevice));
    CK(e, cudaMemcpy(e->d_wy0, y0.data(), dh * sizeof(int), cudaMemcpyHostToDevice));
    e->warp_w = ow; e->warp_h = oh; e->warp_scale = s;
    return PE_OK;
}

// Where the routes that read frames of any size (pixels, camera, JPEG) build their W x H BGR frames: the display frames themselves
// at the display size (*scale = 1), else the warpAffine source d_raw (*scale = frame.scale).  finish_frames warps d_raw into the
// display frames when needed and runs the net.
static int frame_target(pe_engine* e, int W, int H, uint8_t** dst, double* scale) {
    if (W == e->cfg.disp_w && H == e->cfg.disp_h) {
        *dst = e->d_frames.get();
        if (scale) *scale = 1.0;
        return PE_OK;
    }
    int rc = prepare_warp(e, W, H); if (rc) return rc;
    rc = grow_buffer(e, e->d_raw, (size_t)W * H * 3 * e->cfg.max_batch); if (rc) return rc;
    *dst = e->d_raw.get();
    if (scale) *scale = e->warp_scale;
    return PE_OK;
}
static int finish_frames(pe_engine* e, int n, int W, int H) {
    if (W != e->cfg.disp_w || H != e->cfg.disp_h) {
        WarpArgs w;
        w.src = e->d_raw.get(); w.dst = e->d_frames.get(); w.sw = W; w.sh = H; w.dw = e->cfg.disp_w; w.dh = e->cfg.disp_h;
        w.adelta = e->d_wa; w.bdelta = e->d_wb; w.x0 = e->d_wx0; w.y0 = e->d_wy0; w.tab = e->d_wtab;
        e->launches += launch_warp_affine(w, n, e->stream);
    }
    return pe_forward_frames_device(e, e->d_frames.get(), n);
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
        if (L.format == PE_PIX_P016 && ((uintptr_t)frames[i] & 1))
            return fail(e, PE_ERR_INVALID, "odd P016 frame pointer %d: samples are 2 bytes", i);
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
    // Pageable frames go through the staging buffer.  Host frames other than BGR are copied whole to d_pix and converted there.
    if (any_pageable && (rc = stage(e, stride * e->cfg.max_batch))) return rc;
    if (any_host && !bgr && (rc = grow_buffer(e, e->d_pix, stride * e->cfg.max_batch))) return rc;
    PixArgs a;
    a.dst = dst; a.pitch = L.pitch; a.chroma = L.chroma; a.format = L.format; a.w = L.w; a.h = L.h; a.col = L.col;
    for (int i = 0; i < n; i++) {
        const uint8_t* src = (const uint8_t*)frames[i];
        if (kind[i] == PAGEABLE) { memcpy(e->h_stage.get() + i * stride, src, span); src = e->h_stage.get() + i * stride; }
        if (bgr) {   // BGR needs no conversion: the copy into place drops the pitch
            CK(e, cudaMemcpy2DAsync(dst + i * fb, (size_t)L.w * 3, src, (size_t)L.pitch, (size_t)L.w * 3, L.h, cudaMemcpyDefault, e->stream));
        } else if (kind[i] == DEVICE) {
            a.src[i] = src;
        } else {
            CK(e, cudaMemcpyAsync(e->d_pix.get() + i * stride, src, span, cudaMemcpyHostToDevice, e->stream));
            a.src[i] = e->d_pix.get() + i * stride;
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
    if (L.format == PE_PIX_P016 && ((uintptr_t)frame & 1)) return fail(nullptr, PE_ERR_INVALID, "odd P016 frame pointer: samples are 2 bytes");
    if (cap < 3LL * L.w * L.h) return fail(nullptr, PE_ERR_INVALID, "cap %lld is below the %lld bytes of the BGR frame", cap, 3LL * L.w * L.h);
    PixArgs a;
    a.src[0] = (const uint8_t*)frame; a.dst = bgr; a.pitch = L.pitch; a.chroma = L.chroma; a.format = L.format; a.w = L.w; a.h = L.h;
    a.col = L.col;
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
    std::vector<size_t> bytes(n);
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
    rc = grow_buffer(e, e->d_jcoef, stride * n); if (rc) return rc;
    rc = upload_host(e, coefs, bytes, n, stride, e->d_jcoef.get(), "coefficient image"); if (rc) return rc;
    return reconstruct_and_forward(e, n, W, H, stride, max_blocks, scale);
}

// coefficient images in e->d_jcoef (n frames of W x H, `stride` bytes apart) -> display frames -> the net
static int reconstruct_and_forward(pe_engine* e, int n, int W, int H, size_t stride, long long max_blocks, double* scale) {
    uint8_t* dst;
    int rc = frame_target(e, W, H, &dst, scale); if (rc) return rc;
    const size_t pstride = ((size_t)max_blocks * 64 + 255) & ~(size_t)255;
    rc = grow_buffer(e, e->d_jplanes, pstride * n); if (rc) return rc;
    JpegArgs ja;
    ja.coefs = e->d_jcoef.get(); ja.coef_stride = (long long)stride; ja.planes = e->d_jplanes.get(); ja.plane_stride = (long long)pstride;
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
    std::vector<size_t> bytes(n);
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
    const size_t sstride = ((size_t)max_scan + 255) & ~(size_t)255;
    *cstride = ((size_t)max_coef + 255) & ~(size_t)255;
    const int ctas = (int)((max_sub + pe_jpeg::SYNC_THREADS - 1) / pe_jpeg::SYNC_THREADS);
    JpegScanArgs a;
    auto work = [&](Carver& k) {   // the decoder's work space
        a.tabs = k.take<uint8_t>(jpeg_huff_tables_bytes() * n); a.seg_sub = k.take<int>((size_t)(max_seg + 1) * n);
        a.pub = k.take<unsigned long long>((size_t)ctas * 2 * n); a.flags = k.take<int>((size_t)ctas * n); a.tickets = k.take<int>(n); a.status = k.take<int>(n);
    };
    Carver work_size(nullptr);
    work(work_size);
    int rc = grow_buffer(e, e->d_jcoef, *cstride * n); if (rc) return rc;
    rc = grow_buffer(e, e->d_jscan, sstride * n); if (rc) return rc;
    rc = grow_buffer(e, e->d_jwork, work_size.used()); if (rc) return rc;
    rc = grow_buffer(e, e->h_jstatus, (size_t)4 * e->cfg.max_batch); if (rc) return rc;
    rc = upload_host(e, scans, bytes, n, sstride, e->d_jscan.get(), "scan image"); if (rc) return rc;
    CK(e, cudaMemsetAsync(e->d_jcoef.get(), 0, *cstride * n, e->stream));
    a.scans = e->d_jscan.get(); a.scan_stride = (long long)sstride;
    a.coefs = e->d_jcoef.get(); a.coef_stride = (long long)*cstride;
    CK(e, reserve_carved(e->d_jwork, work));   // grown above: only lays the work space out
    a.seg_stride = max_seg + 1; a.ctas_max = ctas; a.n = n; a.S = S;
    e->launches += launch_jpeg_entropy(a, e->stream);
    CK(e, cudaMemcpyAsync(e->h_jstatus.get(), a.status, (size_t)4 * n, cudaMemcpyDeviceToHost, e->stream));
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
        CK(e, cudaMemcpy(coefs_out[i], e->d_jcoef.get() + i * stride, (size_t)hd.coef.total_bytes, cudaMemcpyDeviceToHost));
        if (status_out) { int st; memcpy(&st, e->h_jstatus.get() + 4 * i, 4); status_out[i] = st == INT_MAX ? 0 : 1 + st; }
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
    std::vector<float> B(epi_floats(e, i), 0.f);
    fill_epilogue_fields(e, i, B.data());
    CK(e, cudaMemcpyAsync(e->packed->get() + e->b_off[i], B.data(), B.size() * sizeof(float), cudaMemcpyHostToDevice, e->stream));
    return PE_OK;
}

static int upload_weights(pe_engine* e, int i) {   // re-pack layer i with the current input scales (host fp32 copy needed)
    std::vector<uint8_t> buf(weight_bytes(e, i));
    if (const int rc = pack_conv_weights(e, i, buf.data())) return rc;
    CK(e, cudaMemcpyAsync(e->packed->get() + e->w_off[i], buf.data(), buf.size(), cudaMemcpyHostToDevice, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    return PE_OK;
}

// Brings conv i's region of the packed buffer up to conv_scale: re-packs its weights when a producer's scale differs from
// `packed_with`, the scales they were packed with (the bytes depend only on the ratios of those scales), then rewrites its
// epilogue fields.
static int refresh_layer(pe_engine* e, int i, const std::vector<float>& packed_with) {
    for (int pc : e->plan.convs[i].cin_prod)
        if (pc >= 0 && e->conv_scale[pc] != packed_with[pc]) {
            const int rc = upload_weights(e, i); if (rc) return rc;
            break;
        }
    return upload_fields(e, i);
}

// The handle holds the fp32 weights of every layer (pe_set_conv_weights); a share receiver and a broadcast replica do not.
static bool owns_weights(const pe_engine* e) {
    return std::all_of(e->hw.begin(), e->hw.end(), [](const HostWeights& h) { return h.set; });
}

// The calls that change the scales re-pack and rewrite the packed buffer from the fp32 weights, so they need those weights and a
// buffer no other handle uses (a sharer would keep the old scales).
static int calib_owner_check(pe_engine* e, const char* what) {
    if (!e->committed) return fail(e, PE_ERR_STATE, "%s: pe_commit_weights has not been called", what);
    if (!e->prec->ranged()) return fail(e, PE_ERR_INVALID, "%s: precision %d has no range scales (only 2, 4, 5, 6 and 8 have)", what, e->cfg.precision);
    if (!owns_weights(e))
        return fail(e, PE_ERR_STATE, "%s: this handle received its weights by broadcast / sharing: calibrate the source handle, which owns them", what);
    if (e->packed.use_count() > 1)
        return fail(e, PE_ERR_STATE, "%s: this handle already shares its weights with another handle, which would keep the old scales: "
                    "calibrate before pe_share_weights", what);
    return PE_OK;
}

extern "C" int pe_calibrate(pe_engine* e, const uint8_t* const* frames, int n) {
    int rc = check_n(e, n); if (rc) return rc;
    if (!frames) return fail(e, PE_ERR_INVALID, "null frames");
    if (e->committed && !e->prec->ranged()) return PE_OK;   // fp32 / bf16 modes have fp32's exponent range
    if ((rc = calib_owner_check(e, "pe_calibrate"))) return rc;
    if (e->collecting) return fail(e, PE_ERR_STATE, "a calibration collection is running: call pe_calibrate_end first");
    CK(e, cudaSetDevice(e->cfg.device));
    drop_graphs(e);
    if ((rc = upload_frames(e, frames, n)) || (rc = preprocess_frames(e, e->d_frames.get(), n))) return rc;
    const std::vector<float> packed_with = e->conv_scale;
    const int nimg = n * copies(e);
    for (const OpRef& op : e->plan.order) {
        if (op.type != 0) { if ((rc = run_op(e, op, nimg))) return rc; continue; }
        const int i = op.idx;
        const bool stores = e->plan.convs[i].out_act >= 0;
        if (stores) e->conv_scale[i] = 1.f;   // measure the true output range: fp32 epilogue values, before the fp16 split
        if ((rc = refresh_layer(e, i, packed_with))) return rc;   // its producers are final (plan order)
        if (stores) {
            CK(e, cudaMemsetAsync(e->d_range.get<unsigned>() + i, 0, sizeof(unsigned), e->stream));
            if ((rc = run_op(e, op, nimg))) return rc;
            unsigned bits = 0;
            CK(e, cudaMemcpyAsync(&bits, e->d_range.get<unsigned>() + i, sizeof bits, cudaMemcpyDeviceToHost, e->stream));
            CK(e, cudaStreamSynchronize(e->stream));
            float m; memcpy(&m, &bits, 4);
            e->conv_scale[i] = pow2_for(m, out_row(e, i).range_top);
            if ((rc = upload_fields(e, i))) return rc;
        }
        if ((rc = run_op(e, op, nimg))) return rc;
    }
    CK(e, cudaMemsetAsync(e->d_range.get(), 0, e->plan.convs.size() * sizeof(unsigned), e->stream));
    e->calibrated = true;
    return run_post_and_return(e, n);
}

// During a collection (pe_calibrate_begin): the maxima the kernels recorded since d_range was last cleared, in true units, into the
// running maxima.  Scales are powers of two, so recorded / conv_scale is exact; NaN (a layer that produced one) is ignored.
static void fold_range(pe_engine* e, const std::vector<unsigned>& bits) {
    if (!e->collecting) return;
    for (size_t i = 0; i < bits.size(); i++) {
        if (e->plan.convs[i].out_act < 0 || bits[i] == 0) continue;
        float m; memcpy(&m, &bits[i], 4);
        if (m == m) e->collect_max[i] = fmaxf(e->collect_max[i], m / e->conv_scale[i]);
    }
}

// Largest |stored value| / range_limit (precision.h) over the conv layers since the last call.  PE_ERR_RANGE when a layer
// reached that limit, or when a layer's maximum fell below range_floor; both from the row of the kind the layer stores (out_row).
// s8, u8: the largest stored value is rint(max |t|).  *layer64 names the worst layer.
extern "C" int pe_range_status(pe_engine* e, float* worst_ratio, char* layer64) {
    if (!e) return PE_ERR_INVALID;
    if (worst_ratio) *worst_ratio = 0.f;
    if (layer64) layer64[0] = 0;
    if (!e->d_range.size()) return PE_OK;
    CK(e, cudaSetDevice(e->cfg.device));
    CK(e, cudaStreamSynchronize(e->stream));
    const size_t nc = e->plan.convs.size();
    std::vector<unsigned> bits(nc);
    CK(e, cudaMemcpy(bits.data(), e->d_range.get(), nc * sizeof(unsigned), cudaMemcpyDeviceToHost));
    CK(e, cudaMemset(e->d_range.get(), 0, nc * sizeof(unsigned)));
    fold_range(e, bits);
    float worst = 0.f, smallest = 3e38f, lowest = 3e38f;   // lowest: the smallest maximum relative to its layer's floor
    int iw = -1, is = -1;
    for (size_t i = 0; i < nc; i++) {
        if (e->plan.convs[i].out_act < 0) continue;   // fp32 maps
        const Precision& p = out_row(e, (int)i);
        float m; memcpy(&m, &bits[i], 4);
        if (bits[i] == 0) continue;                   // layer did not run since the last call
        if ((p.fmt.s8() || p.fmt.u8()) && m <= 3e38f) m = rintf(m);   // the kernels track |t| before the rounding: the stored value
        if (!(m <= 3e38f) || m / p.range_limit > worst) { worst = (m <= 3e38f) ? m / p.range_limit : 2.f; iw = (int)i; }
        if (m / p.range_floor < lowest) { lowest = m / p.range_floor; smallest = m; is = (int)i; }
    }
    if (worst_ratio) *worst_ratio = worst;
    if (worst >= 1.f) {
        const Precision& p = out_row(e, iw);
        if (layer64) snprintf(layer64, 64, "%s", e->plan.convs[iw].name.c_str());
        return fail(e, PE_ERR_RANGE, "layer %s produced values outside the range of %s (max |v| = %.3g x scale): run pe_calibrate",
                    e->plan.convs[iw].name.c_str(), p.range_what, worst * p.range_limit);
    }
    if (is >= 0 && lowest < 1.f) {
        const Precision& p = out_row(e, is);
        if (layer64) snprintf(layer64, 64, "%s", e->plan.convs[is].name.c_str());
        return fail(e, PE_ERR_RANGE, "layer %s: largest stored value %.3g is below %s, %s lose precision: run pe_calibrate",
                    e->plan.convs[is].name.c_str(), smallest, p.range_floor_text, p.range_what);
    }
    if (layer64 && iw >= 0) snprintf(layer64, 64, "%s", e->plan.convs[iw].name.c_str());
    return PE_OK;
}

// ---------------------------------------------------------------------------------------------
// Calibration over a set of frames (pe_calibrate_begin / _end) and calibration tables (pe_calibration_get / _set), DESIGN.md
// section 3.  The kernels record every layer's largest |stored value| on every forward, on every input route; a collection folds
// those maxima, divided by the layer's scale, into per-layer running maxima, and pe_calibrate_end sets the scales from them with
// pe_calibrate's rule.  A table carries the scales to another engine with the same weights.
// ---------------------------------------------------------------------------------------------
// The engine's table: every conv layer that stores an activation, with its stored kind and log2 scale
static CalibTable engine_table(pe_engine* e) {
    CalibTable t;
    t.precision = e->cfg.precision | (e->u8 ? PE_PREC_FLAG_U8 : 0);   // an S8X1 table and a u8 table refuse each other
    if (!e->weights_hash_valid) {   // name, fp32 weights, fp32 biases of every conv layer in plan order
        Fnv1a64 h;
        for (size_t i = 0; i < e->plan.convs.size(); i++) {
            const std::string& n = e->plan.convs[i].name;
            h.add(n.c_str(), n.size() + 1);
            h.add(e->hw[i].w.data(), e->hw[i].w.size() * sizeof(float));
            h.add(e->hw[i].b.data(), e->hw[i].b.size() * sizeof(float));
        }
        e->weights_hash = h.h;
        e->weights_hash_valid = true;
    }
    t.weights = e->weights_hash;
    for (size_t i = 0; i < e->plan.convs.size(); i++) {
        if (e->plan.convs[i].out_act < 0) continue;
        t.layers.push_back({e->plan.convs[i].name, elem_name({e->prec->fmt.planes, conv_out_elem(e, (int)i)}), log2_of_scale(e->conv_scale[i])});
    }
    return t;
}

// Sets the scales to `s`, re-packs the layers whose producers' scales changed (the Concat ratios and S8X1's per-channel quantisation
// are folded into the weights) and every layer's epilogue fields, drops the graphs and the range state.  *changed: layers whose scale moved.
static int apply_scales(pe_engine* e, const std::vector<float>& s, int* changed) {
    CK(e, cudaSetDevice(e->cfg.device));
    CK(e, cudaStreamSynchronize(e->stream));
    drop_graphs(e);
    const std::vector<float> old = e->conv_scale;
    e->conv_scale = s;
    int moved = 0;
    for (size_t i = 0; i < s.size(); i++) moved += s[i] != old[i];
    for (size_t i = 0; i < s.size(); i++) { const int rc = refresh_layer(e, (int)i, old); if (rc) return rc; }
    CK(e, cudaMemsetAsync(e->d_range.get(), 0, s.size() * sizeof(unsigned), e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    e->calibrated = true;
    if (changed) *changed = moved;
    return PE_OK;
}

extern "C" int pe_calibrate_begin(pe_engine* e) {
    if (!e) return PE_ERR_INVALID;
    int rc = calib_owner_check(e, "pe_calibrate_begin"); if (rc) return rc;
    if (e->collecting) return fail(e, PE_ERR_STATE, "pe_calibrate_begin: a collection is already running");
    if (e->prec->needs_calibration && !e->calibrated)
        return fail(e, PE_ERR_STATE, "pe_calibrate_begin: PE_PREC_%s forwards only on calibrated scales: start with pe_calibrate or pe_calibration_set",
                    e->cfg.precision == PE_PREC_S8X2 ? "S8X2" : "S8X1");
    CK(e, cudaSetDevice(e->cfg.device));
    CK(e, cudaStreamSynchronize(e->stream));
    CK(e, cudaMemset(e->d_range.get(), 0, e->plan.convs.size() * sizeof(unsigned)));   // maxima of earlier forwards do not count
    e->collect_max.assign(e->plan.convs.size(), 0.f);
    e->collect_forwards = 0;
    e->collecting = true;
    return PE_OK;
}

extern "C" int pe_calibrate_end(pe_engine* e, int* changed) {
    if (!e) return PE_ERR_INVALID;
    if (changed) *changed = 0;
    int rc = calib_owner_check(e, "pe_calibrate_end"); if (rc) return rc;
    if (!e->collecting) return fail(e, PE_ERR_STATE, "pe_calibrate_end: pe_calibrate_begin has not been called");
    if (!e->collect_forwards) return fail(e, PE_ERR_STATE, "pe_calibrate_end: no forward since pe_calibrate_begin");
    CK(e, cudaSetDevice(e->cfg.device));
    CK(e, cudaStreamSynchronize(e->stream));
    const size_t nc = e->plan.convs.size();
    std::vector<unsigned> bits(nc);
    CK(e, cudaMemcpy(bits.data(), e->d_range.get(), nc * sizeof(unsigned), cudaMemcpyDeviceToHost));
    fold_range(e, bits);
    e->collecting = false;
    std::vector<float> s = e->conv_scale;
    for (size_t i = 0; i < nc; i++)   // pe_calibrate's rule; a layer that recorded nothing keeps its scale
        if (e->plan.convs[i].out_act >= 0) s[i] = pow2_for(e->collect_max[i], out_row(e, (int)i).range_top, s[i]);
    return apply_scales(e, s, changed);
}

extern "C" int pe_calibration_get(const pe_engine* ce, char* buf, int cap) {
    if (!ce) return -PE_ERR_INVALID;
    pe_engine* e = const_cast<pe_engine*>(ce);   // the error text and the cached weights hash
    if (!e->committed) return -fail(e, PE_ERR_STATE, "pe_calibration_get: pe_commit_weights has not been called");
    if (!e->prec->ranged()) return -fail(e, PE_ERR_INVALID, "pe_calibration_get: precision %d has no range scales", e->cfg.precision);
    if (!owns_weights(e))
        return -fail(e, PE_ERR_STATE, "pe_calibration_get: this handle received its weights by broadcast / sharing: ask the handle that owns them");
    for (const ConvSpec& c : e->plan.convs)
        if (c.name.find_first_of(" \t\r\n#") != std::string::npos)
            return -fail(e, PE_ERR_INVALID, "pe_calibration_get: layer name '%s' cannot be written into a table (white space or '#')", c.name.c_str());
    const std::string s = write_calibration_table(engine_table(e));
    if (buf && (int)s.size() < cap) memcpy(buf, s.c_str(), s.size() + 1);
    return (int)s.size();
}

extern "C" int pe_calibration_set(pe_engine* e, const char* text) {
    if (!e) return PE_ERR_INVALID;
    int rc = calib_owner_check(e, "pe_calibration_set"); if (rc) return rc;
    if (e->collecting) return fail(e, PE_ERR_STATE, "pe_calibration_set: a calibration collection is running: call pe_calibrate_end first");
    if (!text) return fail(e, PE_ERR_INVALID, "pe_calibration_set: null table");
    const CalibTable want = engine_table(e);
    std::vector<int> k;
    std::string err;
    if (read_calibration_table(text, want, k, err)) return fail(e, PE_ERR_INVALID, "%s", err.c_str());
    std::vector<float> s = e->conv_scale;
    size_t j = 0;
    for (size_t i = 0; i < s.size(); i++)
        if (e->plan.convs[i].out_act >= 0) s[i] = ldexpf(1.f, k[j++]);
    return apply_scales(e, s, nullptr);
}

extern "C" int pe_forward_net_input(pe_engine* e, const float* net_input, int n) {
    int rc = check_n(e, n); if (rc) return rc;
    if (!net_input) return fail(e, PE_ERR_INVALID, "null input");
    CK(e, cudaSetDevice(e->cfg.device));
    const size_t cnt = (size_t)n * e->cfg.num_scales * 3 * e->cfg.net_w * e->cfg.net_h;
    if ((rc = stage(e, cnt * sizeof(float)))) return rc;   // a copy, so the caller may reuse its input when the call returns
    memcpy(e->h_stage.get(), net_input, cnt * sizeof(float));
    CK(e, cudaMemcpyAsync(e->d_planar.get(), e->h_stage.get(), cnt * sizeof(float), cudaMemcpyHostToDevice, e->stream));
    PreArgs a = e->pre;
    a.nframes = n;
    e->launches += launch_input_from_planar(e->d_planar.get<float>(), a, n * e->cfg.num_scales, e->stream);
    e->input_lo_dirty = e->prec->fmt.planes > 0;
    e->last_frames = nullptr;
    return run_net(e, n);
}
extern "C" int pe_forward_maps(pe_engine* e, const float* maps8, int n) {
    int rc = check_n(e, n); if (rc) return rc;
    if (!maps8) return fail(e, PE_ERR_INVALID, "null maps");
    CK(e, cudaSetDevice(e->cfg.device));
    const size_t cnt = (size_t)n * copies(e) * e->mt->num_maps * e->geo[3].W * e->geo[3].H;
    if ((rc = stage(e, cnt * sizeof(float)))) return rc;   // a copy, so the caller may reuse its input when the call returns
    memcpy(e->h_stage.get(), maps8, cnt * sizeof(float));
    CK(e, cudaMemcpyAsync(e->d_maps.get(), e->h_stage.get(), cnt * sizeof(float), cudaMemcpyHostToDevice, e->stream));
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
    float* d_canvas; uint8_t *d_u8, *d_src;   // one size per engine: allocated by the first call
    CK(e, reserve_carved(e->d_render, [&](Carver& k) { d_canvas = k.take<float>(px * 3); d_u8 = k.take<uint8_t>(px * 3); d_src = k.take<uint8_t>(px * 3); }));
    const uint8_t* src = e->last_frames ? e->last_frames + (size_t)idx * px * 3 : nullptr;
    if (display_bgr) {
        CK(e, cudaMemcpyAsync(d_src, display_bgr, px * 3, cudaMemcpyHostToDevice, e->stream));
        src = d_src;
    }
    e->launches += launch_canvas_fill(src, d_canvas, W, H, e->stream);   // process_and_pad_image(normalize = 0), rtpose.cpp:349,1127
    const PostDev& pd = e->post;
    const float* poses = pd.joints + (size_t)idx * PE_MAX_PEOPLE * P * 3;
    auto heat = [&](int ch0, int nch) -> int {   // the channels a heat-map view reads, from the stride-8 maps
        CK(e, e->d_heat.reserve((size_t)nch * nw * nh * sizeof(float)));
        e->launches += launch_fullres_fill(pd, idx, ch0, nch, e->d_heat.get<float>(), e->stream);
        return PE_OK;
    };
    int rc = PE_OK;
    if (part_to_show == 0) {
        e->launches += launch_skeleton(e->cfg.model, d_canvas, W, H, poses, pd.num_people + idx, googly_eyes, e->stream);
    } else if (e->cfg.model == PE_MODEL_MPI_15) {                 // render_mpi_parts: channel part_to_show-1
        if ((rc = heat(part_to_show - 1, 1))) return rc;
        e->launches += launch_heat_view(d_canvas, W, H, e->d_heat.get<float>(), nw, nh, 0, part_to_show - 1, 1, e->stream);
    } else if (part_to_show - 1 < P) {                            // render_coco_parts: one part map
        if ((rc = heat(part_to_show - 1, 1))) return rc;
        e->launches += launch_heat_view(d_canvas, W, H, e->d_heat.get<float>(), nw, nh, 1, part_to_show - 1, 1, e->stream);
    } else if (part_to_show - 1 == P) {                           // all part maps, nearest neighbour (heatmap2)
        if ((rc = heat(0, P))) return rc;
        e->launches += launch_heat_view(d_canvas, W, H, e->d_heat.get<float>(), nw, nh, 2, 0, P, e->stream);
    } else {                                                      // render_coco_aff (rtpose.cpp:286-296)
        int aff_part = ((part_to_show - 1) - P - 1) * 2, accum = 1;
        if (aff_part == 0) accum = e->mt->num_limbs; else aff_part -= 2;
        aff_part += 1 + P;
        if ((rc = heat(aff_part, 2 * accum))) return rc;
        e->launches += launch_heat_view(d_canvas, W, H, e->d_heat.get<float>(), nw, nh, 3, aff_part, 2 * accum, e->stream);
    }
    if (bgr) e->launches += launch_canvas_to_u8(d_canvas, d_u8, W, H, e->stream);   // postProcessFrame, rtpose.cpp:1286-1296
    if (canvas) CK(e, cudaMemcpyAsync(canvas, d_canvas, px * 3 * sizeof(float), cudaMemcpyDeviceToHost, e->stream));
    if (bgr) CK(e, cudaMemcpyAsync(bgr, d_u8, px * 3, cudaMemcpyDeviceToHost, e->stream));
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
        memcpy(&mcu, e->h_jstatus.get() + 4 * idx, 4);
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
    const size_t cnt = (size_t)n * copies(e) * e->mt->num_maps * e->geo[3].W * e->geo[3].H;
    if ((rc = grow_buffer(e, e->h_stage, cnt * sizeof(float)))) return rc;   // the copy queues behind the staging's readers
    CK(e, cudaMemcpyAsync(e->h_stage.get(), e->d_maps.get(), cnt * sizeof(float), cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    memcpy(maps8, e->h_stage.get(), cnt * sizeof(float));
    return PE_OK;
}
static float blob_scale(const pe_engine* e, const BlobRef& b) {
    if (b.prod >= 0 && b.prod < (int)e->conv_scale.size()) return e->conv_scale[b.prod];
    return b.act == e->plan.input_act ? elem_row(*e->prec, act_fmt(e, b.act).elem).net_input_scale : 1.f;
}
extern "C" int pe_blob_log2_scale(pe_engine* e, const char* blob_name, int* k) {
    if (!e || !blob_name || !k) return PE_ERR_INVALID;
    if (!e->prec->ranged()) return fail(e, PE_ERR_INVALID, "this precision has no range scales");
    for (const BlobRef& b : e->plan.blobs) {
        if (b.name != blob_name) continue;
        const float s = blob_scale(e, b);
        const int ex = log2_of_scale(s);
        if (ldexpf(1.f, ex) != s) return fail(e, PE_ERR_STATE, "blob %s: scale is not a power of two", blob_name);
        *k = ex;
        return PE_OK;
    }
    return fail(e, PE_ERR_INVALID, "unknown blob %s", blob_name);
}
extern "C" int pe_fetch_blob(pe_engine* e, const char* blob_name, float* out, size_t cap, int* c, int* h, int* w) {
    if (!e || !blob_name) return PE_ERR_INVALID;
    CK(e, cudaSetDevice(e->cfg.device));
    const int nimg = std::max(e->last_n, 1) * copies(e);
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
        DeviceBuffer d;
        CK(e, d.reserve(cnt * sizeof(float)));
        // stored value = true value * conv_scale[producer] (pools pass their producer's scale through; the net input has
        // the mode's net_input_scale); s8: q * 2^-k, exact in fp32
        const float inv = 1.f / blob_scale(e, b);
        e->launches += launch_act_to_nchw(e->acts[b.act].get(), e->plan.acts[b.act].C, b.coff, b.c, e->act_plane[b.act], act_fmt(e, b.act), g, inv,
                                          d.get<float>(), e->stream);
        CK(e, cudaMemcpyAsync(out, d.get(), cnt * sizeof(float), cudaMemcpyDeviceToHost, e->stream));
        CK(e, cudaStreamSynchronize(e->stream));
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
    const int nimg = n * copies(e);
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
