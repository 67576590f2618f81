"""Generated pose graphs: every convolution shape the plan accepts, checked layer by layer against float64.

A deploy file may hold more than the two shipped nets use: any stride-1 "same" convolution with an odd kernel <= 7 at any of
the four resolution levels, any num_output up to 16384, Concat slots of any width (plan.cpp).  `pose_spec` writes such graphs in
the tests/golden/netspec_*.json format (conv1_1 3x3 on the input, three 2x2 pools, a shared F blob, 1-3 stages of L1 / L2
branches ending in the model's map counts, the final Concat, ImResize and Nms); CASES is a fixed list of them that together
covers k in {1, 3, 5, 7} at every level, output counts from 1 to 257 on both sides of every N-tile boundary, inputs that are
not a multiple of 64 on plain and concat bottoms, odd concat slots, three stages, a 7x7 on 1024 channels, the smallest nets
the engine creates (16x16 and 32x16: 2x2 and 4x2 pixels at stride 8) and images whose last pixel ends exactly on, and one
past, a 128-row tile boundary.  The input is the planar net input (pe_forward_net_input), random up to every border.

The flat padded layout (common.h) turns a filter tap into a constant row shift (r - pad) * Wp + (s - pad), which is zero
padding only while pad <= gap.  CPU part: every case plans, its gaps follow max(1, largest pad at the level), and a numpy
emulation of the row-shift addressing at those gaps equals torch.conv2d (at gap 1 a 7x7 does not).

GPU part: every conv of every case in every precision at 1 and 3 frames (both tile widths), one F16X2 case after
pe_calibrate, each against conv_ref of tests/test_gpu_conv_layers.py with |got - ref| <= B(layer) * mag + floor.  B(layer)
(`layer_bound`) restates the error models of the docstrings of test_gpu_conv_layers.py and test_gpu_fast_mode.py as a function
of the precision, k, the padded input channels and conv_tc.cu's hi*hi chunk length: a 7x7 on 1024 channels has 112 chunks,
not the <= 21 of the shipped nets, so the fixed B = 2^-17 does not hold for it.  For the shipped nets the function stays under
B_P2 / B_F1 (test_layer_bound_covers_the_shipped_nets).  Each (precision, layer class) is also held to MEASURED_MAX, about
2-2.5x the largest (|got - ref| - floor) / mag measured (the floor is the fp16-subnormal term, which dominates the small outputs
of a conv on a 1-channel input), and every pool top must equal the 2x2 max of its fetched bottom exactly.

Before the gap followed the plan (1 at levels 0-2 whatever the kernel), the 5x5 and 7x7 layers at levels 0-2 failed here with
errors of the order of the values themselves, e.g. the 7x7 conv1_2 of k5_k7_vgg in SIMT: 6809 of 87720 elements out, worst
err / mag 0.12.  And tc_cout_pad used to pad 65-127 outputs to 64: the grid then covered 64 channels only, and the biases
of such a layer were written past its slot of the packed buffer.

Measured on one H100 80GB HBM3 (400 W power limit), largest (|got - ref| - floor) / mag over all cases and both frame counts:
            im2col   1x1      3x3      5x5      7x7
  SIMT      2.26e-7  3.13e-7  3.01e-7  2.69e-7  3.37e-7
  F16X2     1.94e-7  3.09e-7  4.23e-7  2.62e-7  1.74e-7    (calibrated three_stages included)
  BF16X3    1.31e-7  2.20e-7  2.29e-7  1.19e-7  1.05e-7
  F16X1     5.93e-4  7.70e-4  8.03e-4  6.13e-4  3.51e-4    (held to about 2x; below 7x7 B is the tighter)
  BF16X1    4.23e-3  5.49e-3  6.55e-3  4.79e-3  2.62e-3    (held to B only)
The GPU part takes about 25 s on that card.
"""
import math

import numpy as np
import pytest
import torch

from caffe_rtpose_b200 import engine, synth
from test_gpu_conv_layers import B_P1, B_P2, U, Blobs, conv_layers, conv_ref, frames_for, plan_gaps, sample_pixels, tc_instance
from test_gpu_fast_mode import B_F1

F2, F1, P1, P3, SIMT = engine.PREC_F16X2, engine.PREC_F16X1, engine.PREC_BF16X1, engine.PREC_BF16X3, engine.PREC_FP32_SIMT
PRECS = {"simt": SIMT, "f16x2": F2, "f16x1": F1, "bf16x1": P1, "bf16x3": P3}
MAPS = {engine.COCO_18: (38, 19), engine.MPI_15: (28, 16)}   # L1 (PAF) and L2 (heat-map) channels


# ------------------------------------------------------------------------------------------ graph generator
def pose_spec(model, net_w, net_h, conv1_1, levels, branch, k_out=1, stages=1):
    """Layer table (tests/golden/netspec_*.json format) of a pose graph.

    conv1_1: its num_output (3x3 on the input).  levels: four lists of (k, num_output), the convolutions of resolution level
    0..3 (level 0 after conv1_1, a 2x2 pool before each next level); the last one of level 3 is F, shared by every stage.
    branch: (k, num_output) of the inner convolutions of each L1 / L2 branch; every branch ends in a k_out x k_out
    convolution to the model's map counts without ReLU.  Stage s >= 2 reads Concat [L1, L2, F] of stage s - 1."""
    c_l1, c_l2 = MAPS[model]
    layers = []

    def conv(name, bottom, k, co, relu=True):
        layers.append({"type": "Convolution", "name": name, "bottom": [bottom], "top": [name], "num_output": co,
                       "kernel_size": k, "pad": k // 2, "stride": 1})
        if relu:
            layers.append({"type": "ReLU", "name": "relu_" + name, "bottom": [name], "top": [name]})
        return name

    x = conv("conv1_1", "image", 3, conv1_1)
    for lv, convs in enumerate(levels):
        if lv:
            layers.append({"type": "Pooling", "name": "pool%d_stage1" % lv, "bottom": [x], "top": ["pool%d_stage1" % lv],
                           "kernel_size": 2, "stride": 2, "pad": 0, "pool": "MAX"})
            x = "pool%d_stage1" % lv
        for i, (k, co) in enumerate(convs):
            x = conv("conv%d_%d" % (lv + 1, i + 2 if lv == 0 else i + 1), x, k, co)
    F = x
    inp = F
    for s in range(1, stages + 1):
        outs = []
        for br, c_map in ((1, c_l1), (2, c_l2)):
            y = inp
            for i, (k, co) in enumerate(branch):
                y = conv("Mconv%d_stage%d_L%d" % (i + 1, s, br), y, k, co)
            outs.append(conv("Mconv%d_stage%d_L%d" % (len(branch) + 1, s, br), y, k_out, c_map, relu=False))
        if s < stages:
            inp = "concat_stage%d" % (s + 1)
            layers.append({"type": "Concat", "name": inp, "bottom": outs + [F], "top": [inp], "axis": 1})
    layers.append({"type": "Concat", "name": "concat_stage7", "bottom": outs[::-1], "top": ["concat_stage7"], "axis": 1})
    layers.append({"type": "ImResize", "name": "resize", "bottom": ["concat_stage7"], "top": ["resized_map"], "factor": 8.0,
                   "scale_gap": 0.3, "start_scale": 1.0})
    layers.append({"type": "Nms", "name": "nms", "bottom": ["resized_map"], "top": ["joints"], "threshold": 0.05,
                   "max_peaks": 20, "num_parts": 18 if model == engine.COCO_18 else 15})
    return {"input": "image", "input_dim": [1, 3, net_h, net_w], "layers": layers}


# name -> pose_spec arguments.  Output counts around the tile widths of tc_cout_pad (16 / 32 / 48 / 64 / 128 and its multiples);
# the large levels at 3 frames give full-width (BN 128) tiles, at 1 frame half-width ones.
CASES = {
    "k5_k7_vgg": dict(model=engine.COCO_18, net_w=64, net_h=48, conv1_1=129,
                      levels=[[(5, 129), (7, 9), (1, 33)], [(7, 257), (3, 17), (5, 49)], [(1, 7), (3, 65)], [(5, 100)]],
                      branch=[(3, 127)], k_out=5),
    # 336x24: the stride-8 level is 42x3 with gap 1, (H - 1) * Wp + W = 128 rows, exactly one row tile per image
    "k1_k3_wide": dict(model=engine.MPI_15, net_w=336, net_h=24, conv1_1=49,
                       levels=[[(3, 129), (1, 257)], [(1, 49), (3, 33)], [(3, 1), (1, 17)], [(3, 65), (1, 72)]],
                       branch=[(3, 33)], k_out=1),
    # 240x32: the stride-8 level is 30x4 with gap 3, (H - 1) * Wp + W = 129 rows, one past a row tile
    "three_stages": dict(model=engine.COCO_18, net_w=240, net_h=32, conv1_1=33,
                         levels=[[(7, 49), (5, 17)], [(5, 9), (7, 1)], [(5, 65)], [(3, 72)]],
                         branch=[(5, 7), (7, 129)], k_out=7, stages=3),
    # the smallest nets the engine creates (16 pixels a side, rtpose.cpp:513-514): 2x2 and 4x2 at stride 8, where a 7x7 reads
    # little but padding (gap rows and TMA out-of-bounds fill)
    "tiny_16x16": dict(model=engine.MPI_15, net_w=16, net_h=16, conv1_1=9,
                       levels=[[(7, 7)], [(5, 17)], [(7, 33)], [(1, 1024), (7, 100)]],
                       branch=[(3, 9)], k_out=3, stages=2),
    "tiny_32x16": dict(model=engine.COCO_18, net_w=32, net_h=16, conv1_1=1,
                       levels=[[(3, 65), (5, 33)], [(1, 9)], [(3, 49)], [(3, 257), (1, 72)]],
                       branch=[(1, 129), (7, 17)], k_out=1, stages=2),
}
FRAMES = (1, 3)


def case_spec(name):
    return pose_spec(**CASES[name])


def write_prototxt(name, tmp_path):
    spec = case_spec(name)
    p = tmp_path / ("%s.prototxt" % name)
    p.write_text(synth.netspec_to_prototxt(spec))
    return spec, str(p)


def parse_convs(text):
    """{name: dict(cout, cin, k, level, in_cused)} from the conv lines of pe_plan_describe."""
    out = {}
    for l in text.splitlines():
        f = l.split()
        if f[0] == "conv":
            out[f[1]] = dict(cout=int(f[2]), cin=int(f[3]), k=int(f[4]), level=int(f[6]), in_cused=int(f[8]))
    return out


def level_dims(net_w, net_h, level):
    w, h = net_w, net_h
    for _ in range(level):
        w, h = (w + 1) // 2, (h + 1) // 2
    return w, h


def spec_weights(spec, seed=1234):
    """W-he weights (N(0, 2 / fan_in)) and N(0, (0.1 x typical pre-activation)^2) biases per conv, from one seeded generator;
    the pre-activation scale follows the second moment through the graph (input 1/12, ReLU halves it)."""
    rng = np.random.default_rng(seed)
    layers = spec["layers"]
    relu = {l["bottom"][0] for l in layers if l["type"] == "ReLU"}
    m2, ch = {spec["input"]: 1.0 / 12}, {spec["input"]: 3}
    W = {}
    for l in layers:
        top, bot = l["top"][0], l["bottom"]
        if l["type"] == "Convolution":
            ci, co, k = ch[bot[0]], l["num_output"], l["kernel_size"]
            w = (rng.standard_normal((co, ci, k, k), dtype=np.float32) * np.float32(math.sqrt(2.0 / (ci * k * k)))).astype(np.float32)
            v = 2.0 * m2[bot[0]]
            b = (rng.standard_normal(co, dtype=np.float32) * np.float32(0.1 * math.sqrt(v))).astype(np.float32)
            W[l["name"]] = (w, b)
            m2[top], ch[top] = (v / 2 if top in relu else v), co
        elif l["type"] == "Pooling":
            m2[top], ch[top] = m2[bot[0]], ch[bot[0]]
        elif l["type"] == "Concat":
            ch[top] = sum(ch[b] for b in bot)
            m2[top] = sum(ch[b] * m2[b] for b in bot) / ch[top]
    return W


# ------------------------------------------------------------------------------------------ error model per layer
def chunk_iters(prec, k, nk):
    """conv_tc.cu tc_layer_launch: K steps (one tap x 64 channels) per hi*hi chunk; bf16x1 runs one chain over all nk."""
    if prec in (F2, P3, F1):
        return 7 if k >= 7 else 6 if k >= 3 else 4
    return nk


def layer_bound(prec, k, cin_pad, cin):
    """Rigorous |got - ref| / mag of one layer (u = 2^-24), the docstring models of test_gpu_conv_layers.py and
    test_gpu_fast_mode.py with their counts made functions of the layer: k the filter size the kernel runs (1 for the im2col'ed
    conv1_1), cin_pad its input channels per tap (a multiple of 64), cin the true ones (SIMT)."""
    if prec == SIMT:
        K = k * k * cin + 1
        return K * U / (1 - K * U)
    nk = k * k * cin_pad // 64                    # K steps of 64
    cs = chunk_iters(prec, k, nk)
    chunk_steps = 4 * min(cs, nk)                 # truncating K16 wgmma steps per hi*hi chunk, each <= 2^-23 of the partial
    chunks = -(-nk // cs)                         # round-to-nearest chunk sums
    steps = 4 * nk                                # K16 steps of the whole (cross-term / bf16x1) chain
    if prec == F2:   # weights re-split 4u, lo*lo dropped 4u, chunks, their sum, cross terms 2^-10 smaller, epilogue 6u
        return (8 + 2 * chunk_steps + chunks + 2 * steps / 1024 + 6) * U
    if prec == P3:   # weight planes 1u, dropped terms 3u, chunks, their sum, cross terms 2^-7 smaller, epilogue 3u
        return (4 + 2 * chunk_steps + chunks + 2 * steps / 128 + 3) * U
    if prec == F1:   # weights and output rounded to one fp16 plane, chunks, their sum, epilogue 1u
        return 2.0 ** -10 + (2 * chunk_steps + chunks + 1) * U
    return 2.0 ** -7 + 2 * steps * U              # P1: weights and output rounded to bf16, one truncating chain


def test_layer_bound_covers_the_shipped_nets():
    """The per-layer bound restates the fixed ones: every layer of the shipped graphs stays under B_P2 (P=2, P=3), B_F1 and
    B_P1; the 7x7 on 1024 channels of CASES does not."""
    for model in (engine.COCO_18, engine.MPI_15):
        for name, co, ci, k in synth.conv_table(model):
            ks, cp = (1, 64) if name == "conv1_1" else (k, -(-ci // 64) * 64)
            assert layer_bound(F2, ks, cp, ci) <= B_P2 and layer_bound(P3, ks, cp, ci) <= B_P2, name
            assert layer_bound(F1, ks, cp, ci) <= B_F1 and layer_bound(P1, ks, cp, ci) <= B_P1, name
    # Mconv1 (7x7, 185 -> 192 channels): 21 chunks of 28 steps, 93u as the docstring counts it
    assert layer_bound(F2, 7, 192, 185) == pytest.approx((8 + 56 + 21 + 588 / 512 + 6) * U)
    assert layer_bound(F2, 7, 1024, 1024) > B_P2


# ------------------------------------------------------------------------------------------ CPU: plans, gaps, the layout
def flat_conv(x, w, gap):
    """Emulation of the engine's addressing: x (N, C, H, W) in the flat padded layout [M][C] with the given gap, every tap a
    constant row shift of the whole matrix, rows outside [0, M) read as zero.  Returns (N, Cout, H, W)."""
    N, C, H, Wd = x.shape
    k = w.shape[2]
    pad = k // 2
    Wp, Hs = Wd + gap, H + gap
    M = N * Hs * Wp
    A = np.zeros((M, C))
    A.reshape(N, Hs, Wp, C)[:, :H, :Wd] = x.transpose(0, 2, 3, 1)
    out = np.zeros((M, w.shape[0]))
    for r in range(k):
        for s in range(k):
            sh = (r - pad) * Wp + (s - pad)
            src = np.zeros((M, C))
            lo, hi = max(0, -sh), min(M, M - sh)
            src[lo:hi] = A[lo + sh:hi + sh]
            out += src @ w[:, :, r, s].T
    return out.reshape(N, Hs, Wp, -1)[:, :H, :Wd].transpose(0, 3, 1, 2)


@pytest.mark.parametrize("name", list(CASES))
def test_case_plans_with_the_gap_rule(name, tmp_path):
    spec, path = write_prototxt(name, tmp_path)
    convs = parse_convs(engine.plan_describe(prototxt=path))
    want = [l for l in spec["layers"] if l["type"] == "Convolution"]
    assert list(convs) == [l["name"] for l in want]
    for l in want:
        assert (convs[l["name"]]["cout"], convs[l["name"]]["k"]) == (l["num_output"], l["kernel_size"])
    gaps = plan_gaps(prototxt=path)
    assert gaps == [max([1] + [c["k"] // 2 for c in convs.values() if c["level"] == lv]) for lv in range(4)]
    # the addressing at the plan's gap is Caffe's zero-padded convolution for every filter size of the case
    rng = np.random.default_rng(3)
    for k, lv in sorted({(c["k"], c["level"]) for c in convs.values()}):
        w_, h_ = level_dims(CASES[name]["net_w"], CASES[name]["net_h"], lv)
        x = rng.standard_normal((2, 3, h_, w_))
        w = rng.standard_normal((4, 3, k, k))
        want_y = torch.nn.functional.conv2d(torch.from_numpy(x), torch.from_numpy(w), padding=k // 2).numpy()
        np.testing.assert_allclose(flat_conv(x, w, gaps[lv]), want_y, rtol=1e-12, atol=1e-12)


def test_layout_needs_gap_at_least_pad():
    """The invariant: with gap 1 a 7x7's taps reach into the neighbouring row and image instead of the zero padding."""
    rng = np.random.default_rng(4)
    x = rng.standard_normal((2, 4, 10, 12))
    w = rng.standard_normal((3, 4, 7, 7))
    want = torch.nn.functional.conv2d(torch.from_numpy(x), torch.from_numpy(w), padding=3).numpy()
    np.testing.assert_allclose(flat_conv(x, w, 3), want, rtol=1e-12, atol=1e-12)
    bad = np.abs(flat_conv(x, w, 1) - want) > 1e-9
    assert bad[:, 0].sum() > 100 and not bad[:, :, 3:-3, 3:-3].any()   # every border pixel wrong, the interior right


def test_cases_cover_the_shape_space(tmp_path):
    seen_kl, couts, slots, flat_ends = set(), set(), set(), set()
    big7 = stages3 = False
    sizes = set()
    for name, c in CASES.items():
        spec, path = write_prototxt(name, tmp_path)
        convs = parse_convs(engine.plan_describe(prototxt=path))
        gaps = plan_gaps(prototxt=path)
        seen_kl |= {(v["k"], v["level"]) for v in convs.values()}
        couts |= {v["cout"] for v in convs.values()}
        big7 |= any(v["k"] == 7 and v["cin"] >= 1024 for v in convs.values())
        stages3 |= c.get("stages", 1) == 3
        slots.add(c["levels"][3][-1][1])
        sizes.add((c["net_w"], c["net_h"]))
        concat_in = {n for n in convs if n.startswith("Mconv1_stage") and not n.startswith("Mconv1_stage1_")}
        plain = [v for n, v in convs.items() if v["cin"] % 64 and n not in concat_in and n != "conv1_1"]
        concat = [v for n, v in convs.items() if v["cin"] % 64 and n in concat_in]
        assert plain, name
        for lv in range(4):
            w_, h_ = level_dims(c["net_w"], c["net_h"], lv)
            flat_ends.add(((h_ - 1) * (w_ + gaps[lv]) + w_) % 128)
        if c.get("stages", 1) > 1:
            assert concat, name
    assert {(k, lv) for k in (1, 3, 5, 7) for lv in range(4)} <= seen_kl
    assert {1, 7, 9, 17, 33, 49, 65, 100, 127, 129, 257} <= couts
    assert slots & {72, 100} and big7 and stages3 and {(16, 16), (32, 16)} <= sizes
    assert {0, 1} <= flat_ends, flat_ends


# ------------------------------------------------------------------------------------------ GPU
# largest (|got - ref| - floor) / mag per (precision, layer class), 2-2.5x the values of the module docstring; bf16x1 measures
# close to its B and is held to B only, as in test_gpu_conv_layers.py
MEASURED_MAX = {
    SIMT: {"im2col": 5.5e-7, "1x1": 7.5e-7, "3x3": 7.5e-7, "5x5": 6.5e-7, "7x7": 8.5e-7},
    F2: {"im2col": 4.5e-7, "1x1": 7.5e-7, "3x3": 1e-6, "5x5": 6.5e-7, "7x7": 4e-7},
    P3: {"im2col": 3.2e-7, "1x1": 5.5e-7, "3x3": 5.7e-7, "5x5": 3e-7, "7x7": 2.6e-7},
    F1: {"im2col": 1.2e-3, "1x1": 1.6e-3, "3x3": 1.6e-3, "5x5": 1.3e-3, "7x7": 7.5e-4},
    P1: {c: 1.0 for c in ("im2col", "1x1", "3x3", "5x5", "7x7")},
}


def layer_class(layer):
    return "im2col" if layer["name"] == "conv1_1" else "%dx%d" % (layer["k"], layer["k"])


def run_case(name, prec, calibrate, tmp_path):
    spec, path = write_prototxt(name, tmp_path)
    c = CASES[name]
    net_w, net_h = c["net_w"], c["net_h"]
    gaps = plan_gaps(prototxt=path)
    plan = parse_convs(engine.plan_describe(prototxt=path))
    W = spec_weights(spec)
    # start scale 0.5: the scale geometry (16-pixel multiples, rtpose.cpp:508-514) then admits a net height of 24
    eng = engine.PoseEngine(None, net_w, net_h, 2 * net_w, 2 * net_h, start_scale=0.5, precision=prec, prototxt=path,
                            max_batch=max(FRAMES))
    eng.set_weights(W)
    layers = conv_layers(None, spec)[0]
    pools = [l for l in spec["layers"] if l["type"] == "Pooling"]
    rng = np.random.default_rng(11)
    worst = {}
    for n in FRAMES:
        if calibrate:
            eng.calibrate(frames_for(n, 2 * net_w, 2 * net_h))
        # the planar net input, every pixel up to the borders, in the frame path's steps of 1/256 (exact in every plane format)
        eng.forward_net_input((rng.integers(0, 256, (n, 3, net_h, net_w)) / 256.0 - 0.5).astype(np.float32))
        blobs = Blobs(eng, n, None, W, spec)
        for layer in layers:
            w_, h_ = level_dims(net_w, net_h, layer["level"])
            pts = sample_pixels(n, h_, w_, gaps[layer["level"]], rng, 300)
            w, b = W[layer["name"]]
            x, y = blobs.get(layer["bottom"]), blobs.get(layer["top"])
            ref, mag = conv_ref(x, w, b, pts, layer["relu"])
            got = y[pts[:, 0], :, pts[:, 1], pts[:, 2]].astype(np.float64)
            err = np.abs(got - ref)
            ks, cp = (1, 64) if layer["name"] == "conv1_1" else (layer["k"], plan[layer["name"]]["in_cused"])
            B = layer_bound(prec, ks, cp, w.shape[1])
            floor = U * (float(np.abs(y).max()) / 32 if calibrate else 1.0) if prec in (F2, F1) else 0.0
            bad = err > B * mag + floor
            if bad.any():
                i, co = np.argwhere(bad)[0]
                raise AssertionError("%s, %d frame(s): %d of %d elements outside B=%.2e x mag + %.1e; first at (n, y, x) = %s channel "
                                     "%d: got %.9g, ref %.9g, mag %.3g; worst err/mag %.3e" % (
                                         layer["name"], n, int(bad.sum()), bad.size, B, floor, tuple(pts[i]), co, got[i, co], ref[i, co],
                                         mag[i, co], float((err / mag).max())))
            key = layer_class(layer)   # the accumulation error beyond the subnormal floor (small outputs of 1-channel inputs)
            worst[key] = max(worst.get(key, 0.0), float((np.maximum(err - floor, 0.0) / mag).max()))
        for p in pools:   # max pooling copies the winner: exact in every precision
            bot = blobs.get(p["bottom"][0])
            top = eng.fetch_blob(p["top"][0])[:n]
            N, C, H, Wd = bot.shape
            want = bot.reshape(N, C, H // 2, 2, Wd // 2, 2).max(axis=(3, 5))
            assert np.array_equal(top, want), "%s, %d frame(s): %d elements differ" % (p["name"], n, int((top != want).sum()))
    eng.close()
    print("\n%s %s%s: largest |got - ref| / mag per layer class: %s" % (
        name, [k for k, v in PRECS.items() if v == prec][0], " calibrated" if calibrate else "",
        " ".join("%s %.3e" % (k, worst[k]) for k in sorted(worst))))
    over = {k: v for k, v in worst.items() if v > MEASURED_MAX[prec][k]}
    assert not over, "accumulation error above what this kernel measured: %s" % over
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("name", list(CASES))
def test_generated_convs_vs_float64(name, prec, tmp_path):
    run_case(name, PRECS[prec], False, tmp_path)


@pytest.mark.gpu
def test_generated_convs_vs_float64_calibrated(tmp_path):
    """pe_calibrate gives every producer its own range scale: the concat inputs of stages 2 and 3 fold the ratios of three
    producers into their weights (pack_conv_weights) over the generated slot layout."""
    run_case("three_stages", F2, True, tmp_path)


@pytest.mark.gpu
def test_cases_launch_every_instance_at_every_filter_size(tmp_path):
    """Restating the width rule of tc_layer_launch (tc_instance): the cases launch every conv_wg_kernel<BN, P, F16> instance of
    every plane format with 5x5 filters, as with 1x1 (the im2col'ed conv1_1 included), 3x3 and 7x7."""
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    seen = set()
    for name, c in CASES.items():
        spec, path = write_prototxt(name, tmp_path)
        gaps = plan_gaps(prototxt=path)
        for layer in conv_layers(None, spec)[0]:
            w_, h_ = level_dims(c["net_w"], c["net_h"], layer["level"])
            ks = 1 if layer["name"] == "conv1_1" else layer["k"]
            co = [l for l in spec["layers"] if l["name"] == layer["name"]][0]["num_output"]
            for prec in (F2, F1, P1, P3):
                for n in FRAMES:
                    bn = tc_instance(co, ks, n * (h_ + gaps[layer["level"]]) * (w_ + gaps[layer["level"]]), prec, nsm)[0]
                    seen.add((bn, prec, ks))
    want = {(bn, prec, k) for k in (1, 3, 5, 7) for prec in (F2, F1, P1) for bn in (128, 64, 48, 32, 16)}
    want |= {(bn, P3, k) for k in (1, 3, 5, 7) for bn in (64, 48, 32, 16)}
    assert want <= seen, sorted(want - seen)
