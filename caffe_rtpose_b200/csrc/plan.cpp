// Model descriptors and the engine's execution plan for the deploy graph.
//
// Reference: src/rtpose/modelDescriptorFactory.cpp:6-28 (MPI_15), 30-55 (COCO_18);
//            model/{coco,mpi}/pose_deploy_linevec.prototxt (92 conv, 80 ReLU, 3 pool, 6 concat).
// The plan is not a translation of Caffe's layer list: ReLU is fused into the conv epilogue, Concat is
// removed (producers write channel slices of a shared buffer), Split disappears, and conv1_1 consumes an
// im2col'ed input so that it is a K=27 1x1 GEMM.
#include <ctype.h>
#include <math.h>
#include <stdio.h>

#include <algorithm>
#include <map>

#include "common.h"
#include "precision.h"
#include "prototxt.h"

namespace pe {

static const int kLimbMPI[] = {0, 1, 1, 2, 2, 3, 3, 4, 1, 5, 5, 6, 6, 7, 1, 14, 14, 11, 11, 12, 12, 13, 14, 8, 8, 9, 9, 10};
static const int kMapMPI[] = {16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 38, 39, 40, 41, 42, 43, 32, 33, 34, 35, 36, 37};
static const int kLimbCOCO[] = {1, 2, 1, 5, 2, 3, 3, 4, 5, 6, 6, 7, 1, 8, 8, 9, 9, 10, 1, 11, 11, 12, 12, 13, 1, 0, 0, 14, 14, 16, 0, 15, 15, 17, 2, 16, 5, 17};
static const int kMapCOCO[] = {31, 32, 39, 40, 33, 34, 35, 36, 41, 42, 43, 44, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 47, 48, 49, 50, 53, 54, 51, 52, 55, 56, 37, 38, 45, 46};
static const char* kNamesMPI[] = {"Head", "Neck", "RShoulder", "RElbow", "RWrist", "LShoulder", "LElbow", "LWrist", "RHip",
                                  "RKnee", "RAnkle", "LHip", "LKnee", "LAnkle", "Chest", "Bkg"};
static const char* kNamesCOCO[] = {"Nose", "Neck", "RShoulder", "RElbow", "RWrist", "LShoulder", "LElbow", "LWrist", "RHip", "RKnee",
                                   "RAnkle", "LHip", "LKnee", "LAnkle", "REye", "LEye", "REar", "LEar", "Bkg"};

const ModelTables& model_tables(int model) {
    // max_peaks / num_parts: nms_param of the deploy prototxts (coco :2989-3000, mpi :2976-2999)
    static const ModelTables mpi = {15, 14, 44, 20, kLimbMPI, kMapMPI};
    static const ModelTables coco = {18, 19, 57, 64, kLimbCOCO, kMapCOCO};
    return model == PE_MODEL_MPI_15 ? mpi : coco;
}

// modelDescriptor.cpp:4-20 createPartToName: PAF channels are named "<A>-><B>(X|Y)"
const char* model_part_name(int model, int idx) {
    static std::vector<std::string> names[2];
    const int mi = model == PE_MODEL_MPI_15 ? 0 : 1;
    const ModelTables& t = model_tables(model);
    if (names[mi].empty()) {
        names[mi].assign(t.num_maps, "");
        for (int i = 0; i <= t.num_parts; i++) names[mi][i] = mi == 0 ? kNamesMPI[i] : kNamesCOCO[i];
        for (int l = 0; l < t.num_limbs; l++) {
            const std::string base = names[mi][t.limb_seq[2 * l]] + "->" + names[mi][t.limb_seq[2 * l + 1]];
            names[mi][t.map_idx[2 * l]] = base + "(X)";
            names[mi][t.map_idx[2 * l + 1]] = base + "(Y)";
        }
    }
    if (idx < 0 || idx >= t.num_maps) return "";
    return names[mi][idx].c_str();
}

// The flip test's channel map (DESIGN.md section 8): a part maps to its left/right twin by name ("RKnee" <-> "LKnee"; the centre
// parts and the background to themselves), limb (a, b) to the limb (perm a, perm b), and a limb's PAF channels to its mirror's,
// the x channel negated.  The result is an involution.  Returns num_maps, or -1 when a part or limb has no mirror.
int model_flip_table(int model, std::vector<int>& perm, std::vector<float>& sign) {
    const ModelTables& t = model_tables(model);
    perm.assign(t.num_maps, -1);
    sign.assign(t.num_maps, 1.f);
    for (int i = 0; i <= t.num_parts; i++) {
        const std::string n = model_part_name(model, i);
        perm[i] = i;
        if (n.size() < 2 || (n[0] != 'R' && n[0] != 'L') || !isupper((unsigned char)n[1])) continue;
        const std::string twin = (n[0] == 'R' ? "L" : "R") + n.substr(1);
        perm[i] = -1;
        for (int j = 0; j <= t.num_parts; j++)
            if (twin == model_part_name(model, j)) perm[i] = j;
        if (perm[i] < 0) return -1;
    }
    for (int k = 0; k < t.num_limbs; k++) {
        int m = -1;
        for (int j = 0; j < t.num_limbs; j++)
            if (t.limb_seq[2 * j] == perm[t.limb_seq[2 * k]] && t.limb_seq[2 * j + 1] == perm[t.limb_seq[2 * k + 1]]) m = j;
        if (m < 0) return -1;
        perm[t.map_idx[2 * k]] = t.map_idx[2 * m];
        perm[t.map_idx[2 * k + 1]] = t.map_idx[2 * m + 1];
        sign[t.map_idx[2 * k]] = -1.f;   // x points the other way in the mirror (rtpose.cpp:575-576 reads mapIdx[2k] as x)
    }
    for (int c = 0; c < t.num_maps; c++)
        if (perm[c] < 0 || perm[perm[c]] != c) return -1;
    return t.num_maps;
}

static int round_up(int v, int m) { return (v + m - 1) / m * m; }
static const int kMaxChannels = 16384;   // a user's prototxt is untrusted input: channel counts stay far inside int arithmetic (the pose nets use <= 512)

// ---------------------------------------------------------------------------------------------
// Execution plan from a network definition (prototxt or built-in).  What Net::Init does for the reference
// (net.cpp:30-280: blob wiring, shape inference, in-place ReLU) plus the engine's own layout decisions:
//   * ReLU is fused into the producing conv, Concat is removed: producers write channel slices of a shared buffer
//     (layout [blobs shared by several concats | the others], slots 8-aligned), consumers get a channel map;
//   * the concat buffers of successive stages ping-pong between two physical buffers; a blob that feeds several
//     concats (conv4_4_CPM) is written once and copied once;
//   * the last Concat (the bottom of ImResize) is never materialised in NHWC: its producers store the planar fp32
//     stride-8 maps directly.
// Supported: the deploy-graph family of model/{coco,mpi}/pose_deploy_linevec*.prototxt - stride-1 odd-kernel (<= 7)
// "same"-padded convolutions, in-place ReLU, 2x2/2 MAX pooling, channel Concat, ImResize(factor 8), Nms, any number
// of stages.  Anything else is reported as an error (the reference would run it through generic Caffe layers).
// ---------------------------------------------------------------------------------------------
int build_plan_from_net(const NetDef& net, const PlanFormats& fm, NetPlan& p, std::string& err) {
    p = NetPlan();
    const int NL = (int)net.layers.size();
    auto fail = [&](const std::string& m) { err = m; return -1; };
    if (net.inputs.size() != 1) return fail("expected exactly one net input, found " + std::to_string(net.inputs.size()));
    if (net.input_dims.size() >= 2 && net.input_dims[1] != 3) return fail("the net input must have 3 channels");
    const std::string input_blob = net.inputs[0];

    // ---- special layers and the model (rtpose.cpp:212-229 infers it from the Nms layer's num_parts)
    int resize_idx = -1, nms_idx = -1;
    for (int i = 0; i < NL; i++) {
        if (net.layers[i].type == "ImResize") resize_idx = i;
        if (net.layers[i].type == "Nms") nms_idx = i;
    }
    if (resize_idx < 0 || nms_idx < 0) return fail("the deploy net needs an ImResize and an Nms layer (layer_by_name(\"resize\"/\"nms\"), rtpose.cpp:194-199)");
    const ProtoLayer& nms = net.layers[nms_idx];
    const ProtoLayer& rsz = net.layers[resize_idx];
    if (nms.nms_num_parts == 15) p.model = PE_MODEL_MPI_15;
    else if (nms.nms_num_parts == 18) p.model = PE_MODEL_COCO_18;
    else return fail("Unknown number of parts! Couldn't set model (nms num_parts = " + std::to_string(nms.nms_num_parts) + ", rtpose.cpp:228)");
    if (rsz.resize_factor != 8.f) return fail("ImResize factor " + std::to_string(rsz.resize_factor) + " is not supported (the stride of the net is 8)");
    if (nms.nms_max_peaks < 1 || nms.nms_max_peaks > PE_MAX_PEAKS) return fail("nms max_peaks out of range");
    if (nms.bottoms.size() != 1 || rsz.tops.size() != 1 || nms.bottoms[0] != rsz.tops[0]) return fail("Nms must consume the ImResize output");
    const ModelTables& mt = model_tables(p.model);
    p.c_l1 = 2 * mt.num_limbs; p.c_l2 = mt.num_parts + 1;
    p.nms_threshold = nms.nms_threshold; p.nms_max_peaks = nms.nms_max_peaks; p.nms_num_parts = nms.nms_num_parts;
    p.resize_start_scale = rsz.resize_start_scale; p.resize_scale_gap = rsz.resize_scale_gap;

    // ---- producers / consumers / channels / levels
    std::map<std::string, int> producer, channels, level;
    std::map<std::string, std::vector<int>> consumers;
    channels[input_blob] = 3; level[input_blob] = 0;
    for (int i = 0; i < NL; i++) {
        const ProtoLayer& l = net.layers[i];
        if (l.tops.size() != 1) return fail("layer " + l.name + ": exactly one top expected");
        if (l.bottoms.empty()) return fail("layer " + l.name + ": no bottom");
        for (const std::string& b : l.bottoms) {
            if (!channels.count(b)) return fail("layer " + l.name + ": unknown bottom blob " + b);
            consumers[b].push_back(i);
        }
        const std::string& top = l.tops[0];
        const int lv = level[l.bottoms[0]];
        if (l.type == "Convolution") {
            if (l.bottoms.size() != 1) return fail("layer " + l.name + ": one bottom expected");
            if (l.num_output < 1 || l.kernel < 1 || l.kernel > 7 || l.kernel % 2 == 0 || l.pad != l.kernel / 2 || l.stride != 1)
                return fail("layer " + l.name + ": only stride-1 'same' convolutions with odd kernel <= 7 are supported (kernel " +
                            std::to_string(l.kernel) + ", pad " + std::to_string(l.pad) + ", stride " + std::to_string(l.stride) + ")");
            if (l.num_output > kMaxChannels) return fail("layer " + l.name + ": num_output " + std::to_string(l.num_output) + " is larger than this engine plans for (" + std::to_string(kMaxChannels) + ")");
            if (producer.count(top)) return fail("layer " + l.name + ": top " + top + " is produced twice");
            producer[top] = i; channels[top] = l.num_output; level[top] = lv;
        } else if (l.type == "ReLU") {
            if (l.bottoms[0] != top || !producer.count(top) || net.layers[producer[top]].type != "Convolution")
                return fail("layer " + l.name + ": ReLU must run in place on a convolution output");
        } else if (l.type == "Pooling") {
            if (l.pool_method != 0 || l.kernel != 2 || l.stride != 2 || l.pad != 0) return fail("layer " + l.name + ": only 2x2 stride-2 MAX pooling is supported");
            if (lv >= 3) return fail("layer " + l.name + ": more than three pooling levels");
            if (producer.count(top)) return fail("layer " + l.name + ": top " + top + " is produced twice");
            producer[top] = i; channels[top] = channels[l.bottoms[0]]; level[top] = lv + 1;
        } else if (l.type == "Concat") {
            if (l.concat_axis != 1) return fail("layer " + l.name + ": only channel concatenation (axis 1) is supported");
            int c = 0;
            for (const std::string& b : l.bottoms) {
                c += channels[b];
                if (level[b] != lv) return fail("layer " + l.name + ": bottoms of different resolution");
                if (c > kMaxChannels) return fail("layer " + l.name + ": more than " + std::to_string(kMaxChannels) + " channels");
            }
            producer[top] = i; channels[top] = c; level[top] = lv;
        } else if (l.type == "ImResize" || l.type == "Nms") {
            producer[top] = i; channels[top] = channels[l.bottoms[0]]; level[top] = lv;
        } else {
            return fail("layer " + l.name + ": layer type " + l.type + " is not on the pose path and not supported");
        }
    }
    const std::string final_blob = rsz.bottoms[0];
    if (!producer.count(final_blob) || net.layers[producer[final_blob]].type != "Concat")
        return fail("the bottom of ImResize must be a Concat (concat_stage7)");
    const int final_concat = producer[final_blob];
    if (level[final_blob] != 3) return fail("the net output must be at stride 8 (three pooling levels)");
    if (channels[final_blob] != mt.num_maps)
        return fail("the net output has " + std::to_string(channels[final_blob]) + " channels, the " + std::string(p.model == PE_MODEL_MPI_15 ? "MPI" : "COCO") +
                    " model needs " + std::to_string(mt.num_maps));
    std::map<std::string, int> final_off;   // blob -> channel offset inside concat_stage7
    {
        int off = 0;
        for (const std::string& b : net.layers[final_concat].bottoms) {
            if (!producer.count(b) || net.layers[producer[b]].type != "Convolution" || consumers[b].size() != 1)
                return fail("bottoms of the final Concat must be convolution outputs used nowhere else");
            final_off[b] = off; off += channels[b];
        }
    }

    // ---- concat buffers: slice layout shared by all non-final concats, two physical buffers
    std::vector<int> concats;
    for (int i = 0; i < NL; i++) if (net.layers[i].type == "Concat" && i != final_concat) concats.push_back(i);

    // ---- element kinds (DESIGN.md section 3).  A conv layer computes in fp16 when it is listed, else in the mode's kind (conv1_1
    // in the net input's).  Blobs that live in one buffer form a group: a pool's input and output (the pool passes the format
    // through), and every non-final Concat with its bottoms - the two ping-pong buffers and the shared conv4_4_CPM, which the copy
    // moves without converting.  A group takes the kind of the conv layers that read it, so those must agree.
    std::map<std::string, std::string> up;   // union-find over blob names
    auto root = [&](std::string b) { while (up.count(b) && up[b] != b) b = up[b]; return b; };
    auto unite = [&](const std::string& a, const std::string& b) { const std::string ra = root(a), rb = root(b); if (ra != rb) up[ra] = rb; };
    for (int i = 0; i < NL; i++) {
        const ProtoLayer& l = net.layers[i];
        if (l.type == "Pooling") unite(l.bottoms[0], l.tops[0]);
        if (l.type == "Concat" && i != final_concat) {
            for (const std::string& b : l.bottoms) unite(b, l.tops[0]);
            unite(l.tops[0], net.layers[concats[0]].tops[0]);
        }
    }
    std::map<std::string, int> conv_layer;                // conv name -> layer index
    std::map<std::string, std::vector<int>> readers;      // group -> conv layers reading it, in net order
    for (int i = 0; i < NL; i++)
        if (net.layers[i].type == "Convolution") { conv_layer[net.layers[i].name] = i; readers[root(net.layers[i].bottoms[0])].push_back(i); }
    std::map<std::string, bool> listed;
    bool narrow = false;
    for (const std::string& n : fm.f16) {
        if (n == "narrow") narrow = true;
        else if (!conv_layer.count(n)) return fail("unknown conv layer " + n + " in the fp16 layer list");
        else listed[n] = true;
    }
    if (narrow)   // every reader of the group reads fewer than 128 channels: its e4m3 / s8 K block is partly padding
        for (const auto& g : readers) {
            bool all = true;
            for (int i : g.second) all = all && channels[net.layers[i].bottoms[0]] < 128;
            if (all) for (int i : g.second) listed[net.layers[i].name] = true;
        }
    auto conv_elem = [&](int i) {
        const ProtoLayer& l = net.layers[i];
        return listed.count(l.name) ? (int)ELEM_F16 : l.bottoms[0] == input_blob ? fm.input_elem : fm.base_elem;
    };
    std::map<std::string, int> group_elem;
    for (const auto& g : readers) {
        for (int i : g.second)
            if (conv_elem(i) != conv_elem(g.second[0])) {
                std::string names;
                for (int j : g.second) names += (names.empty() ? "" : ", ") + net.layers[j].name;
                return fail("layers " + names + " read one buffer and must run in one format: list all of them as fp16 layers or none");
            }
        group_elem[g.first] = conv_elem(g.second[0]);
    }
    auto elem_of = [&](const std::string& blob) {
        auto it = group_elem.find(root(blob));
        return it == group_elem.end() ? fm.base_elem : it->second;
    };
    // u8 (PlanFormats::u8): a group of kind s8 - every conv layer that reads it computes in s8 - whose every writer is a conv layer
    // followed by ReLU (a pool writes into its input's group) holds values >= 0 only: it is stored as u8.  The net input (p - 128)
    // and a group that a layer without ReLU writes (the Concat buffers with the stage outputs, and so conv4_4_CPM's output) stay s8.
    if (fm.u8) {
        std::map<std::string, bool> nonneg;   // group -> every writer so far is a conv layer followed by ReLU
        nonneg[root(input_blob)] = false;
        for (int i = 0; i < NL; i++) {
            const ProtoLayer& l = net.layers[i];
            if (l.type != "Convolution") continue;
            bool relu = false;
            for (int u : consumers[l.tops[0]]) relu = relu || net.layers[u].type == "ReLU";
            const std::string g = root(l.tops[0]);
            nonneg[g] = (nonneg.count(g) ? nonneg[g] : true) && relu;
        }
        for (const auto& g : nonneg)
            if (g.second && elem_of(g.first) == ELEM_S8) group_elem[g.first] = ELEM_U8;
    }
    const int cc_elem = concats.empty() ? fm.base_elem : elem_of(net.layers[concats[0]].tops[0]);
    const int cpad = fm.layout[cc_elem].cpad, slot_align = fm.layout[cc_elem].slot_align;   // of the concat buffers

    std::map<std::string, int> n_in_concats;
    for (int ci : concats) for (const std::string& b : net.layers[ci].bottoms) n_in_concats[b]++;
    struct Slot { int caffe_off, eng_off, c; bool shared; };
    std::vector<std::vector<Slot>> slots(concats.size());   // per concat, per bottom (concat order)
    int cc_c = 0;
    for (size_t j = 0; j < concats.size(); j++) {
        const ProtoLayer& l = net.layers[concats[j]];
        if (level[l.tops[0]] != 3) return fail("layer " + l.name + ": Concat is only supported at stride 8");
        std::vector<Slot>& sl = slots[j];
        int coff = 0;
        for (const std::string& b : l.bottoms) {
            sl.push_back({coff, 0, channels[b], consumers[b].size() > 1});   // read by more than this Concat (conv4_4_CPM: every stage)
            coff += channels[b];
        }
        int eoff = 0;
        for (int pass = 0; pass < 2; pass++)        // shared blobs first
            for (Slot& sdef : sl)
                if (sdef.shared == (pass == 0)) { sdef.eng_off = eoff; eoff += round_up(sdef.c, slot_align); }
        const int total = round_up(eoff, cpad);
        if (j == 0) cc_c = total;
        else {   // the physical buffers are reused: every concat must have the layout of the first
            if (sl.size() != slots[0].size() || total != cc_c) return fail("layer " + l.name + ": Concat layouts differ between stages");
            for (size_t k = 0; k < sl.size(); k++) {
                if (sl[k].c != slots[0][k].c || sl[k].shared != slots[0][k].shared || sl[k].eng_off != slots[0][k].eng_off)
                    return fail("layer " + l.name + ": Concat layouts differ between stages");
                if (sl[k].shared && l.bottoms[k] != net.layers[concats[0]].bottoms[k]) return fail("layer " + l.name + ": shared Concat bottoms differ between stages");
            }
        }
        for (const Slot& sdef : sl) {
            const std::string& b = l.bottoms[&sdef - &sl[0]];
            if (!producer.count(b) || net.layers[producer[b]].type != "Convolution") return fail("layer " + l.name + ": Concat bottoms must be convolution outputs");
        }
    }
    const int nbuf = (int)std::min<size_t>(2, concats.size());
    // reuse is safe when every consumer of concat j is issued before the first producer of concat j+2
    for (size_t j = 0; j + 2 < concats.size(); j++) {
        int last_use = 0;
        for (int c : consumers[net.layers[concats[j]].tops[0]]) last_use = std::max(last_use, c);
        for (size_t k = 0; k < slots[j + 2].size(); k++)
            if (!slots[j + 2][k].shared && producer[net.layers[concats[j + 2]].bottoms[k]] < last_use)
                return fail("the stages overlap in a way the two-buffer concat scheme cannot hold");
    }

    auto new_act = [&](int lv, int c, const std::string& blob, int blob_c, int elem) {
        ActSpec a; a.level = lv; a.C = round_up(c, fm.layout[elem].cpad); a.blob = blob; a.blob_c = blob_c; a.elem = elem;
        p.acts.push_back(a);
        if (!blob.empty()) p.blobs.push_back({blob, (int)p.acts.size() - 1, 0, blob_c});
        return (int)p.acts.size() - 1;
    };
    auto ident = [](int n, int padded) {
        std::vector<int> m(padded, -1);
        for (int i = 0; i < n; i++) m[i] = i;
        return m;
    };
    struct Loc { int act = -1, coff = 0, cused = 0; std::vector<int> cmap, prod; };   // prod: producing conv per engine channel
    std::map<std::string, Loc> loc;
    std::map<std::string, int> conv_index;   // blob -> index in p.convs of its producer

    // network input, im2col'ed 3x3x3 patches: engine channel (r*3+s)*3+c  <-  original weight index (c, r, s)
    const int input_elem = elem_of(input_blob), kp_input = fm.layout[input_elem].kp_input;
    p.kp_input = kp_input;
    p.input_act = new_act(0, kp_input, "", 0, input_elem);
    p.acts[p.input_act].C = kp_input;
    p.blobs.push_back({input_blob, p.input_act, 12, 3});  // centre tap (r=1,s=1) of the patch = the net input itself
    int cc[2] = {-1, -1};
    std::map<std::string, std::pair<int, int>> concat_slot;   // blob -> (first concat index j, bottom position k)
    for (size_t j = 0; j < concats.size(); j++)
        for (size_t k = 0; k < slots[j].size(); k++)
            if (!concat_slot.count(net.layers[concats[j]].bottoms[k])) concat_slot[net.layers[concats[j]].bottoms[k]] = {(int)j, (int)k};

    for (int i = 0; i < NL; i++) {
        const ProtoLayer& l = net.layers[i];
        const std::string& top = l.tops[0];
        if (l.type == "Convolution") {
            ConvSpec c;
            c.name = l.name; c.cout = l.num_output; c.k = l.kernel; c.pad = l.pad; c.level = level[top];
            c.relu = 0;
            for (int u : consumers[top]) if (net.layers[u].type == "ReLU") c.relu = 1;
            c.planar_coff = 0; c.out_coff = 0; c.flops_per_image = 0; c.im2col_input = 0;
            c.elem = elem_of(l.bottoms[0]) == ELEM_U8 ? (int)ELEM_U8 : conv_elem(i);   // a reader of u8 computes u8 x s8
            // input
            if (l.bottoms[0] == input_blob) {
                if (l.kernel != 3) return fail("layer " + l.name + ": the first convolution must be 3x3 (it consumes the im2col'ed input)");
                c.cin = 3; c.in_act = p.input_act; c.in_cused = kp_input; c.im2col_input = 1;
            } else {
                const Loc& in = loc[l.bottoms[0]];
                if (in.act < 0) return fail("layer " + l.name + ": bottom " + l.bottoms[0] + " is not available as a convolution input");
                if (in.coff != 0) return fail("layer " + l.name + ": bottom " + l.bottoms[0] + " does not start at channel 0 of its buffer");
                c.cin = channels[l.bottoms[0]]; c.in_act = in.act; c.in_cused = in.cused; c.cin_map = in.cmap; c.cin_prod = in.prod;
            }
            // output
            if (final_off.count(top)) {
                if (c.relu) return fail("layer " + l.name + ": a ReLU on the net output is not supported");
                c.out_act = -1; c.planar_coff = final_off[top];
            } else if (concat_slot.count(top)) {
                if (cc[0] < 0) {   // the two ping-pong concat buffers [shared | stage outputs]
                    for (int b = 0; b < nbuf; b++) { cc[b] = new_act(3, cc_c, "", 0, cc_elem); p.acts[cc[b]].C = cc_c; }
                }
                const int j = concat_slot[top].first, k = concat_slot[top].second;
                const Slot& sdef = slots[j][k];
                c.out_act = cc[j % nbuf]; c.out_coff = sdef.eng_off;
                p.blobs.push_back({top, c.out_act, sdef.eng_off, sdef.c, (int)p.convs.size(), (int)p.order.size()});
                if (sdef.shared || consumers[top].size() > 1) {   // also read directly by convolutions (conv4_4_CPM feeds stage 1)
                    if (sdef.eng_off != 0) return fail("blob " + top + ": a directly consumed Concat bottom must be first in the buffer");
                    Loc o; o.act = c.out_act; o.coff = 0; o.cused = round_up(sdef.c, std::max(64, cpad)); o.cmap = ident(sdef.c, o.cused);
                    o.prod.assign(o.cused, -1);
                    for (int q = 0; q < sdef.c; q++) o.prod[q] = (int)p.convs.size();
                    if (o.cused > cc_c) return fail("blob " + top + ": too narrow concat buffer");
                    loc[top] = o;
                }
            } else {
                c.out_act = new_act(c.level, c.cout, top, c.cout, elem_of(top));
                p.blobs.back().prod = (int)p.convs.size(); p.blobs.back().pos = (int)p.order.size();
                Loc o; o.act = c.out_act; o.coff = 0; o.cused = p.acts[c.out_act].C; o.cmap = ident(c.cout, o.cused);
                o.prod.assign(o.cused, -1);
                for (int q = 0; q < c.cout; q++) o.prod[q] = (int)p.convs.size();
                loc[top] = o;
            }
            conv_index[top] = (int)p.convs.size();
            p.convs.push_back(c);
            p.order.push_back({0, (int)p.convs.size() - 1});
            if (concat_slot.count(top) && slots[concat_slot[top].first][concat_slot[top].second].shared && nbuf == 2) {
                p.copies.push_back({cc[0], cc[1], round_up(channels[top], slot_align)});   // whole 16-byte chunks, inside the slot
                p.order.push_back({2, (int)p.copies.size() - 1});
            }
        } else if (l.type == "Pooling") {
            const Loc& in = loc[l.bottoms[0]];
            if (in.act < 0 || in.coff != 0 || p.acts[in.act].level != level[l.bottoms[0]]) return fail("layer " + l.name + ": unsupported pooling input");
            const int out = new_act(level[top], channels[top], top, channels[top], elem_of(top));
            p.blobs.back().prod = in.prod.empty() ? -1 : in.prod[0]; p.blobs.back().pos = (int)p.order.size();
            if (p.acts[out].C != p.acts[in.act].C) return fail("layer " + l.name + ": channel pitch mismatch");
            p.pools.push_back({l.name, in.act, out, level[l.bottoms[0]]});
            p.order.push_back({1, (int)p.pools.size() - 1});
            Loc o; o.act = out; o.coff = 0; o.cused = p.acts[out].C; o.cmap = ident(channels[top], o.cused);
            o.prod = in.prod;   // max pooling passes the producer (and its scale) through
            loc[top] = o;
        } else if (l.type == "Concat" && i != final_concat) {
            size_t j = 0;
            while (concats[j] != i) j++;
            Loc o; o.act = cc[j % nbuf]; o.coff = 0; o.cused = cc_c; o.cmap.assign(cc_c, -1);
            if (o.act < 0) return fail("layer " + l.name + ": Concat before any of its producers");
            o.prod.assign(cc_c, -1);
            for (size_t k = 0; k < slots[j].size(); k++) {
                const Slot& sdef = slots[j][k];
                const int pc = conv_index[l.bottoms[k]];
                for (int q = 0; q < sdef.c; q++) { o.cmap[sdef.eng_off + q] = sdef.caffe_off + q; o.prod[sdef.eng_off + q] = pc; }
            }
            loc[top] = o;
        }
    }
    if (p.convs.empty() || !p.convs[0].im2col_input) return fail("the first layer must be a convolution on the net input");
    // A tap is a constant row shift of the flat padded layout only while pad <= gap (common.h, Geo)
    for (const ConvSpec& c : p.convs) p.gap[c.level] = std::max(p.gap[c.level], c.pad);
    // Every forward runs the whole order, so a blob whose channels a later op writes (a stage output in a ping-pong concat
    // buffer that a later stage reuses) holds that op's data after the forward: record the first such op.
    for (BlobRef& b : p.blobs)
        for (int k = b.pos + 1; k < (int)p.order.size() && b.reused_by.empty(); k++) {
            const OpRef& op = p.order[k];
            int act = -1, c0 = 0, c1 = 0;
            std::string who;
            if (op.type == 0) {
                const ConvSpec& c = p.convs[op.idx];
                act = c.out_act; c0 = c.out_coff; c1 = c.out_coff + round_up(c.cout, 8); who = c.name;   // epilogues store 8-channel groups
            } else if (op.type == 1) {
                act = p.pools[op.idx].out_act; c1 = p.acts[act].C; who = p.pools[op.idx].name;
            } else {
                act = p.copies[op.idx].dst_act; c1 = p.copies[op.idx].channels; who = "the copy of the shared concat input";
            }
            if (act == b.act && c0 < b.coff + b.c && b.coff < c1) b.reused_by = who;
        }
    return 0;
}

long long conv_weight_index(const ConvSpec& c, int co, int kk) {
    if (c.im2col_input) return kk < 27 ? ((long long)co * 3 + kk % 3) * 9 + kk / 3 : -1;   // tap = kk / 3, channel kk % 3
    const int tap = kk / c.in_cused, ec = kk % c.in_cused;
    const int ci = ec < (int)c.cin_map.size() ? c.cin_map[ec] : -1;
    return ci < 0 ? -1 : ((long long)co * c.cin + ci) * c.k * c.k + tap;
}

// Calls f(co, idx[4]) for every aligned group of four packed weights (idx: Caffe indices, -1 for padding)
template <class F> static void for_each_group(const ConvSpec& c, F f) {
    const int K = (c.im2col_input ? 1 : c.k * c.k) * c.in_cused;
    for (int co = 0; co < c.cout; co++)
        for (int g = 0; g + 4 <= K; g += 4) {
            long long idx[4];
            for (int i = 0; i < 4; i++) idx[i] = conv_weight_index(c, co, g + i);
            f(idx);
        }
}

bool conv_weights_2to4(const ConvSpec& c, const float* w) {
    bool ok = true;
    for_each_group(c, [&](const long long* idx) {
        int n = 0;
        for (int i = 0; i < 4; i++) n += idx[i] >= 0 && w[idx[i]] != 0.f;
        ok = ok && n <= 2;
    });
    return ok;
}

void conv_prune_2to4(const ConvSpec& c, float* w) {
    for_each_group(c, [&](const long long* idx) {
        auto mag = [&](int i) { return idx[i] >= 0 ? fabsf(w[idx[i]]) : -1.f; };
        int a = 0;   // the largest |w|, the lowest index first among equals; then the largest of the others
        for (int i = 1; i < 4; i++) if (mag(i) > mag(a)) a = i;
        int b = a == 0 ? 1 : 0;
        for (int i = 0; i < 4; i++) if (i != a && mag(i) > mag(b)) b = i;
        for (int i = 0; i < 4; i++) if (i != a && i != b && idx[i] >= 0) w[idx[i]] = 0.f;
    });
}

int build_plan_from_net(const NetDef& net, int kp_input, int cpad, NetPlan& p, std::string& err) {
    PlanFormats f;
    for (ActLayout& l : f.layout) l = {cpad, kp_input, 8};
    return build_plan_from_net(net, f, p, err);
}

}  // namespace pe
