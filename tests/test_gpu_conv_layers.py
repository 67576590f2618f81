"""Every convolution the engine runs, checked on its own against a float64 reference of the same layer.

The net-level tests compare the stride-8 maps with the oracle at 3e-5 of the map maximum.  An error confined to one N tile,
to the last row tile, to image borders or to one 64-channel block of the 185-channel concat input is averaged over 92 layers
there, and those tests ran with zero biases.  Here each layer L is checked alone:

  * input: `pe_fetch_blob` of L's bottom, i.e. exactly what the kernel read (the planes' sum; for `Mconv1_stageN` the Caffe
    concat order [L1, L2, conv4_4_CPM] assembled from the stage outputs, which only stages 5 and 6 still hold after a forward);
  * output: `pe_fetch_blob` of L's top, or the planar maps for the last stage;
  * reference at sampled output pixels, all output channels, in float64 from the fp32 weights and biases given to the engine:
    ref = sum a*w + b (ReLU if L has one) and mag = sum |a|*|w| + |b|;
  * per element  |got - ref| <= B * mag + floor.

The pixels: every pixel of the first and the last 128-row M tile (the last one partial), of every tile that straddles two
images of a batch, the image borders (x, y in {0, 1, W-2, W-1} / {0, 1, H-2, H-1}, where the zero padding comes from gap rows
and TMA out-of-bounds fill) and 1000 random ones.  Tiles are located in the flat padded layout of common.h: row
m = (n*Hs + y)*Wp + x, Wp = W + gap, Hs = H + gap, with the plan's gap (plan_gaps: 1 on the VGG levels and 3 at stride 8).

Error model (u = 2^-24; derived from the code, per product a*w and relative to mag):
  P=2 (fp16 hi + lo planes, conv_tc.cu)
      weights re-split into two fp16 planes (lo = the residual <= 2^-11 |w|, rounded)   4u
      lo*lo dropped: |a_lo| <= 2^-11 |a|, |w_lo| <= 2^-11 |w|                              4u
      hi*hi chunk: <= 28 truncating K16 steps (7x7: 7 iterations x 4, 3x3: 6 x 4,
        1x1: 4 x 4), each <= 2^-23 of the partial magnitude                              56u
      round-to-nearest sum of the chunks: <= 21 chunks (Mconv1: 3 blocks x 49 taps / 7) 21u
      cross accumulator, not chunked: <= 588 steps x 2^-23 x 2^-10 (cross terms' size)    2u
      epilogue: hi*hi + cross, *out_scale (exact) + bias (2u), fp16 hi + lo of the output (4u) 6u
      total 93u; B = 2^-17 = 128u.
  P=3 (bf16 planes): three 8-bit planes carry the weight's 24 bits (1u), the dropped terms pa + pb >= 3 are <= 2^-24 each
      (3u), the chunks and their sum as P=2 (77u), the cross accumulator <= 588 x 2^-23 x 2^-7 (10u), epilogue (3u): 94u;
      the same B.
  P=1 (bf16, unit roundoff 2^-8): weights and output rounded to bf16 (2^-8 each), one truncating chain of <= 588 steps
      (2^-13.8): B = 2^-7 + 2^-11.
  SIMT fp32: fmaf over K = k*k*Cin products, then the bias: gamma_{K+1} = (K+1)u / (1 - (K+1)u).
  conv1_1 direct (fp32 FMA over 27 taps + bias, stored as fp16 hi + lo at P=2): gamma_28 + 4u.
The fetched input is the exact sum of the planes, so the rounding of the activations does not enter.  floor: at P=2 the
output's lo plane can be an fp16 subnormal (spacing 2^-24 of the stored value = true value x the layer's range scale s):
2^-24 / s.  Uncalibrated s = 1; after pe_calibrate s >= 32 / max|output|, so the floor is 2^-24 max|output| / 32.  (Weights
are pre-scaled so that max|w| lies in [2^13, 2^14); a subnormal weight lo plane is below 2^-38 max|w| and neglected.)

The rigorous bound is far above what the hardware does on random-sign data: a truncating chain's error follows the partial
sums, which grow like sqrt(K) while mag grows like K.  The test therefore also holds the largest |got - ref| / mag of each
(precision, layer class) to MEASURED_MAX, 2-2.5x the values measured below (the kernels are deterministic and the data
seeded, so these maxima repeat exactly).  Without it, a kernel that stops chunking hi*hi passes: at P=2 its 7x7 layers reach
1.2e-6 of mag, 10x the value below but still 6x under B.

Measured on one H100 80GB HBM3 (700 W power limit), largest |got - ref| / mag over all configurations, full / half width:
            7x7              3x3              1x1 (BN 128 / 64 / 48, 32, 16)      conv1_1 im2col
  P=2       1.08e-7/1.04e-7  3.07e-7/2.80e-7  3.42e-7 / 3.31e-7 / 2.6e-7-2.8e-7   2.64e-7 (BN 64)
  P=3       6.96e-8 (BN 64)  2.17e-7 (64)     2.14e-7 (64), 1.80e-7 (32)         8.33e-8
  SIMT      4.11e-7          3.25e-7          2.99e-7                            2.20e-7
  conv1_1 direct (fp32 CUDA cores, P=2 output): 2.92e-7.  Calibrated range nets at 160x96 (P=2, half width): within the P=2 row.
  P=1       7.18e-4 (BN 128) 1.87e-3/1.39e-3  3.02e-3 (BN 128)                   4.67e-3 (B = 7.9e-3; held to B only)
"""
import functools
import json
import os

import numpy as np
import pytest
import torch

from caffe_rtpose_b200 import engine, synth

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
U = 2.0 ** -24
B_P2 = 2.0 ** -17
B_P1 = 2.0 ** -7 + 2.0 ** -11


# ------------------------------------------------------------------------------------------ float64 reference (CPU)
def conv_ref(x, w, b, pts, relu):
    """Zero-padded stride-1 'same' convolution at sampled output pixels, in float64.
    x (N, Cin, H, W), w (Cout, Cin, k, k), b (Cout), pts int (P, 3) rows (n, y, x).  Returns ref, mag (P, Cout):
    ref = sum a*w + b (then ReLU if relu), mag = sum |a|*|w| + |b|."""
    w = np.asarray(w, np.float64)
    co, ci, k, _ = w.shape
    p = k // 2
    xp = np.pad(np.asarray(x, np.float64), ((0, 0), (0, 0), (p, p), (p, p)))
    n, yy, xx = pts[:, 0], pts[:, 1], pts[:, 2]
    ref = np.zeros((len(pts), co))
    mag = np.zeros((len(pts), co))
    for r in range(k):
        for s in range(k):
            a = xp[n, :, yy + r, xx + s]            # (P, Cin)
            wt = w[:, :, r, s].T
            ref += a @ wt
            mag += np.abs(a) @ np.abs(wt)
    b = np.asarray(b, np.float64)
    ref += b
    mag += np.abs(b)
    return (np.maximum(ref, 0.0) if relu else ref), mag


def sample_pixels(N, H, W, gap, rng, n_random=1000):
    """(P, 3) unique (n, y, x): the first and last 128-row tiles, tiles straddling two images, image borders, random pixels."""
    Wp, Hs = W + gap, H + gap
    per = Hs * Wp
    M = N * per
    mt = (M + 127) // 128
    rows = [np.arange(0, min(128, M)), np.arange((mt - 1) * 128, M)]
    for t in range(mt):
        lo, hi = 128 * t, min(M, 128 * t + 128) - 1
        if lo // per != hi // per:
            rows.append(np.arange(lo, hi + 1))
    m = np.concatenate(rows)
    n, rem = m // per, m % per
    y, x = rem // Wp, rem % Wp
    keep = (x < W) & (y < H)
    pts = [np.stack([n, y, x], 1)[keep]]
    ey = np.array(sorted({0, 1, H - 2, H - 1} & set(range(H))))
    ex = np.array(sorted({0, 1, W - 2, W - 1} & set(range(W))))
    for i in range(N):
        gy, gx = np.meshgrid(ey, np.arange(W), indexing="ij")
        pts.append(np.stack([np.full(gy.size, i), gy.ravel(), gx.ravel()], 1))
        gy, gx = np.meshgrid(np.arange(H), ex, indexing="ij")
        pts.append(np.stack([np.full(gy.size, i), gy.ravel(), gx.ravel()], 1))
    pts.append(np.stack([rng.integers(0, N, n_random), rng.integers(0, H, n_random), rng.integers(0, W, n_random)], 1))
    return np.unique(np.concatenate(pts).astype(np.int64), axis=0)


def test_reference_matches_torch_conv2d():
    rng = np.random.default_rng(5)
    for k, N, ci, co, H, W in [(1, 1, 5, 3, 4, 6), (3, 2, 19, 70, 9, 7), (7, 2, 40, 17, 11, 10), (3, 3, 3, 64, 5, 13), (7, 1, 65, 48, 8, 8)]:
        x = rng.standard_normal((N, ci, H, W))
        w = rng.standard_normal((co, ci, k, k))
        b = rng.standard_normal(co)
        pts = sample_pixels(N, H, W, 1 if k < 7 else 3, rng, 50)
        full = torch.nn.functional.conv2d(torch.from_numpy(x), torch.from_numpy(w), torch.from_numpy(b), padding=k // 2).numpy()
        want = full[pts[:, 0], :, pts[:, 1], pts[:, 2]]
        for relu in (False, True):
            ref, _ = conv_ref(x, w, b, pts, relu)
            np.testing.assert_allclose(ref, np.maximum(want, 0) if relu else want, rtol=1e-12, atol=1e-12)


def test_reference_mag_by_hand():
    """3x3 kernel over a 2x2 image, one channel in, two out: mag adds |a||w| of the taps inside the image, plus |b|."""
    x = np.array([[[[1.0, -2.0], [3.0, -4.0]]]])
    w = np.zeros((2, 1, 3, 3))
    w[0, 0] = [[0, 0, 0], [0, 1, -1], [0, 1, 1]]      # out(0,0) = 1*1 - 1*(-2) + 1*3 + 1*(-4) = 2
    w[1, 0] = -w[0, 0]
    b = np.array([-0.5, 0.25])
    ref, mag = conv_ref(x, w, b, np.array([[0, 0, 0], [0, 1, 1]]), relu=False)
    np.testing.assert_array_equal(ref[0], [2.0 - 0.5, -2.0 + 0.25])
    np.testing.assert_array_equal(mag[0], [1 + 2 + 3 + 4 + 0.5, 1 + 2 + 3 + 4 + 0.25])
    # pixel (1, 1): only the centre tap (weight 1 on x = -4) lies inside the image; the padded taps add nothing
    np.testing.assert_array_equal(ref[1], [-4.0 - 0.5, 4.0 + 0.25])
    np.testing.assert_array_equal(mag[1], [4.5, 4.25])
    ref, _ = conv_ref(x, w, b, np.array([[0, 0, 0]]), relu=True)
    np.testing.assert_array_equal(ref[0], [1.5, 0.0])


def test_sample_covers_tiles_borders_and_straddles():
    rng = np.random.default_rng(0)
    N, H, W, gap = 2, 46, 82, 3
    pts = {tuple(p) for p in sample_pixels(N, H, W, gap, rng)}
    Wp, per = W + gap, (H + gap) * (W + gap)
    M = N * per
    last = (M - 1) // 128 * 128
    assert M % 128 and all((m // per, m % per // Wp, m % Wp) in pts for m in range(last, M) if m % Wp < W and m % per // Wp < H)
    straddle = [t for t in range(M // 128) if (128 * t) // per != (128 * t + 127) // per]
    assert straddle and all((m // per, m % per // Wp, m % Wp) in pts for m in range(128 * straddle[0], 128 * straddle[0] + 128)
                            if m % Wp < W and m % per // Wp < H)
    assert all((n, y, x) in pts for n in range(N) for y in (0, 1, H - 2, H - 1) for x in range(W))
    assert all((n, y, x) in pts for n in range(N) for y in range(H) for x in (0, 1, W - 2, W - 1))


# ------------------------------------------------------------------------------------------ the net and the width rule
def netspec(model):
    with open(os.path.join(GOLD, "netspec_%s.json" % ("coco" if model == engine.COCO_18 else "mpi"))) as f:
        return json.load(f)


def conv_layers(model, spec=None):
    """[dict(name, bottom, top, k, relu, level)] in prototxt order, plus the Concat layers by top and the final concat.
    spec: a layer table in the netspec format (default: the shipped graph of `model`)."""
    spec = spec or netspec(model)
    layers = spec["layers"]
    relu = {l["bottom"][0] for l in layers if l["type"] == "ReLU"}
    concat = {l["top"][0]: l["bottom"] for l in layers if l["type"] == "Concat"}
    level = {spec["input"]: 0}
    out = []
    for l in layers:
        if l["type"] in ("Convolution", "Concat", "ImResize", "Nms"):
            level[l["top"][0]] = level[l["bottom"][0]]
        elif l["type"] == "Pooling":
            level[l["top"][0]] = level[l["bottom"][0]] + 1
        if l["type"] == "Convolution":
            out.append(dict(name=l["name"], bottom=l["bottom"][0], top=l["top"][0], k=l["kernel_size"], relu=l["top"][0] in relu,
                            level=level[l["top"][0]]))
    final = [l for l in layers if l["type"] == "ImResize"][0]["bottom"][0]
    return out, concat, final


# Stage outputs in the ping-pong concat buffers that a later stage of the 6-stage nets overwrites (plan.cpp, nbuf = 2)
REUSED = {"conv5_5_CPM_L1", "conv5_5_CPM_L2", "Mconv7_stage2_L1", "Mconv7_stage2_L2", "Mconv7_stage3_L1", "Mconv7_stage3_L2"}


def checked_layers(model):
    """Conv layers whose input and output the engine still holds after a forward."""
    convs, concat, _ = conv_layers(model)
    out = []
    for c in convs:
        parts = concat.get(c["bottom"], [c["bottom"]])
        if c["top"] in REUSED or any(p in REUSED for p in parts):
            continue
        out.append(c)
    return out


# Restated from conv_tc.cu (tc_cout_pad, tc_bn, tc_layer_launch): the tile width a layer runs at.
def tc_cout_pad(cout):
    if cout > 64:
        return (cout + 127) // 128 * 128
    return 64 if cout > 48 else 48 if cout > 32 else 32 if cout > 16 else 16


def tc_instance(cout, ksize, M, planes, nsm, share=2):
    """(BN, planes, A-window rows) of conv_wg_kernel for one launch: full width, or half when (CTAs that can run at once) x
    0.80 is larger.  share = 2: the two lanes of a forward split the SMs."""
    cp = tc_cout_pad(cout)
    bn = min(cp, 64 if planes == 3 else 128)
    mt = (M + 127) // 128
    sms = max(1, nsm // share)
    if bn >= 64 and min(mt * (cp // (bn // 2)), sms) * 0.80 > min(mt * (cp // bn), sms) * 1.00:
        bn //= 2
    return bn, planes, 128 if ksize == 1 else 136


@functools.lru_cache(maxsize=None)
def plan_gaps(model=engine.COCO_18, prototxt=None):
    """[gap of level 0..3] of the flat padded layout, as the plan prints it (`gap <level> <g>` lines of pe_plan_describe)."""
    text = engine.plan_describe(model=None if prototxt else model, prototxt=prototxt)
    gaps = {int(l.split()[1]): int(l.split()[2]) for l in text.splitlines() if l.startswith("gap ")}
    return [gaps[l] for l in range(4)]


def level_geo(net_w, net_h, level, gaps=None):
    """(W, H, gap) of a resolution level; gaps: plan_gaps() of the net (default: the built-in graphs, both the same)."""
    w, h = net_w, net_h
    for _ in range(level):
        w, h = (w + 1) // 2, (h + 1) // 2
    return w, h, (gaps or plan_gaps())[level]


# ------------------------------------------------------------------------------------------ GPU configurations
def preact_std(W, model):
    """Typical pre-activation std of every layer of the net W under a variance-propagation model (input E[x^2] = 1/12, ReLU
    halves the second moment, pooling and concat keep it): the scale of the biases, so that they move the ReLU active set
    without swamping the sums."""
    spec = netspec(model)
    relu = {l["bottom"][0] for l in spec["layers"] if l["type"] == "ReLU"}
    m2 = {spec["input"]: 1.0 / 12}
    out = {}
    for l in spec["layers"]:
        top, bot = l["top"][0], l["bottom"]
        if l["type"] == "Convolution":
            w = W[l["name"]][0].astype(np.float64)
            v = w[0].size * float(np.mean(w * w)) * m2[bot[0]]
            out[l["name"]] = float(np.sqrt(v))
            m2[top] = v / 2 if top in relu else v
        elif l["type"] == "Pooling":
            m2[top] = m2[bot[0]]
        elif l["type"] == "Concat":
            ch = [W[b][0].shape[0] for b in bot]
            m2[top] = sum(c * m2[b] for c, b in zip(ch, bot)) / sum(ch)
    return out


def weights_with_biases(model, kind="he", grow=1.0):
    """W-he (or the caffe filler), weights times grow^1 per layer, with N(0, (0.1 x typical pre-activation)^2) biases."""
    W0 = {k: (w * np.float32(grow), b) for k, (w, b) in synth.make_weights(model, kind).items()}
    std = preact_std(W0, model)
    Wb = synth.make_weights(model, kind, bias_std={k: 0.1 * v for k, v in std.items()})
    return {k: (W0[k][0], Wb[k][1]) for k in W0}


# name -> (model, net_w, net_h, precision, frame counts to run, env, calibrate with weights kind/grow)
CONFIGS = {
    "coco_p2": (engine.COCO_18, 656, 368, engine.PREC_F16X2, (1, 2), {}, None),
    "mpi_p2": (engine.MPI_15, 496, 368, engine.PREC_F16X2, (1, 3), {}, None),
    "coco_p3": (engine.COCO_18, 656, 368, engine.PREC_BF16X3, (2,), {}, None),
    "coco_p1": (engine.COCO_18, 656, 368, engine.PREC_BF16X1, (2,), {}, None),
    "coco_simt": (engine.COCO_18, 656, 368, engine.PREC_FP32_SIMT, (2,), {}, None),
    "coco_conv11_direct": (engine.COCO_18, 656, 368, engine.PREC_F16X2, (1,), {"PE_CONV11_DIRECT": "1"}, None),
    "range_caffe_filler": (engine.COCO_18, 160, 96, engine.PREC_F16X2, (1,), {}, ("caffe", 1.0)),
    "range_growing": (engine.COCO_18, 160, 96, engine.PREC_F16X2, (1,), {}, ("he", 1.6)),
}
# largest |got - ref| / mag per layer class, 2-2.5x the H100's measured values (module docstring); P=1 is held to B only
MEASURED_MAX = {
    engine.PREC_F16X2: {"7x7": 2.5e-7, "3x3": 7e-7, "1x1": 8e-7, "im2col": 6e-7, "direct": 7e-7},
    engine.PREC_BF16X3: {"7x7": 1.6e-7, "3x3": 5e-7, "1x1": 5e-7, "im2col": 2e-7},
    engine.PREC_FP32_SIMT: {"7x7": 1e-6, "3x3": 8e-7, "1x1": 7e-7, "im2col": 5e-7},
}


def layers_for(cfg):
    model = CONFIGS[cfg][0]
    layers = checked_layers(model)
    return [l for l in layers if l["name"] == "conv1_1"] if CONFIGS[cfg][5].get("PE_CONV11_DIRECT") else layers


def frames_for(n, disp_w, disp_h):
    return [synth.make_frame(50 + i, disp_h, disp_w) for i in range(n)]


class Blobs:
    """Blobs of the engine's last forward (first nimg images), fetched once each.  spec: as conv_layers."""

    def __init__(self, eng, nimg, model, W, spec=None):
        self.eng, self.nimg, self.cache = eng, nimg, {}
        _, self.concat, final = conv_layers(model, spec)
        self.final_off, off = {}, 0
        for b in self.concat[final]:      # the last stage's outputs: channel slices of the planar maps (concat_stage7)
            c = W[b][0].shape[0]
            self.final_off[b] = (off, c)
            off += c
        self.maps = None

    def get(self, name):
        if name not in self.cache:
            if name in self.final_off:
                if self.maps is None:
                    self.maps = self.eng.fetch_maps(self.nimg)
                off, c = self.final_off[name]
                self.cache[name] = self.maps[:, off:off + c]
            elif name in self.concat:
                self.cache[name] = np.concatenate([self.get(b) for b in self.concat[name]], axis=1)
            else:
                self.cache[name] = self.eng.fetch_blob(name)[:self.nimg]
        return self.cache[name]


def bound(prec, layer, cin, direct):
    K = layer["k"] ** 2 * cin
    if direct:
        return 28 * U / (1 - 28 * U) + 4 * U
    if prec == engine.PREC_FP32_SIMT:
        return (K + 1) * U / (1 - (K + 1) * U)
    return B_P1 if prec == engine.PREC_BF16X1 else B_P2


def check_layer(layer, blobs, W, prec, pts, calibrated, direct):
    w, b = W[layer["name"]]
    x = blobs.get(layer["bottom"])
    y = blobs.get(layer["top"])
    ref, mag = conv_ref(x, w, b, pts, layer["relu"])
    got = y[pts[:, 0], :, pts[:, 1], pts[:, 2]].astype(np.float64)
    err = np.abs(got - ref)
    B = bound(prec, layer, w.shape[1], direct)
    floor = 0.0
    if prec == engine.PREC_F16X2:
        floor = U * (float(np.abs(y).max()) / 32 if calibrated else 1.0)
    bad = err > B * mag + floor
    if bad.any():
        i, c = np.argwhere(bad)[0]
        raise AssertionError("%s: %d of %d elements outside B=%.2e x mag + %.1e; first at (n, y, x) = %s channel %d: got %.9g, ref %.9g, "
                             "mag %.3g; worst err/mag %.3e" % (layer["name"], int(bad.sum()), bad.size, B, floor, tuple(pts[i]), c,
                                                               got[i, c], ref[i, c], mag[i, c], float((err / mag).max())))
    return float((err / mag).max())


def layer_class(layer):
    return "im2col" if layer["name"] == "conv1_1" else "%dx%d" % (layer["k"], layer["k"])


def run_config(cfg, monkeypatch):
    model, net_w, net_h, prec, counts, env, cal = CONFIGS[cfg]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    W = weights_with_biases(model, *(cal or ("he", 1.0)))
    disp_w, disp_h = 2 * net_w, 2 * net_h
    eng = engine.PoseEngine(model, net_w, net_h, disp_w, disp_h, precision=prec, max_batch=max(counts))
    eng.set_weights(W)
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    worst = {}
    rng = np.random.default_rng(11)
    for n in counts:
        frames = frames_for(n, disp_w, disp_h)
        if cal:
            eng.calibrate(frames)
        eng.forward_frames(frames)
        blobs = Blobs(eng, n, model, W)
        for layer in layers_for(cfg):
            w_, h_, gap = level_geo(net_w, net_h, layer["level"])
            pts = sample_pixels(n, h_, w_, gap, rng)
            r = check_layer(layer, blobs, W, prec, pts, cal is not None, bool(env.get("PE_CONV11_DIRECT")))
            if env.get("PE_CONV11_DIRECT"):
                width = "direct"
            elif prec == engine.PREC_FP32_SIMT:
                width = "simt"
            else:
                ks = 1 if layer["name"] == "conv1_1" else layer["k"]
                width = "BN=%d" % tc_instance(W[layer["name"]][0].shape[0], ks, n * (h_ + gap) * (w_ + gap), prec, nsm)[0]
            key = (layer_class(layer), width)
            worst[key] = max(worst.get(key, 0.0), r)
    eng.close()
    print("\n%s: largest |got - ref| / mag per (layer class, tile width):" % cfg)
    for key in sorted(worst, key=str):
        print("  %-7s %-7s %.3e" % (key[0], key[1], worst[key]))
    if prec in MEASURED_MAX:
        lim = MEASURED_MAX[prec]
        over = {k: v for k, v in worst.items() if v > lim["direct" if k[1] == "direct" else k[0]]}
        assert not over, "accumulation error above what this kernel measured: %s" % over
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_conv_layers_vs_float64(cfg, monkeypatch):
    run_config(cfg, monkeypatch)


@pytest.mark.gpu
def test_width_rule_covers_every_instance():
    """Restating the width rule of tc_layer_launch: the configurations above run every conv_wg_kernel instance the engine
    has, each filter size at full and half width, and a partial last row tile at every level."""
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    seen, partial = set(), set()
    for cfg, (model, net_w, net_h, prec, counts, env, _) in CONFIGS.items():
        if prec == engine.PREC_FP32_SIMT or env.get("PE_CONV11_DIRECT"):
            continue
        W = synth.make_weights(model)
        for n in counts:
            for layer in layers_for(cfg):
                w_, h_, gap = level_geo(net_w, net_h, layer["level"])
                M = n * (h_ + gap) * (w_ + gap)
                ks = 1 if layer["name"] == "conv1_1" else layer["k"]
                bn, p, rows = tc_instance(W[layer["name"]][0].shape[0], ks, M, prec, nsm)
                seen.add((bn, p, layer_class(layer)))
                seen.add((bn, p, rows))
                if M % 128:
                    partial.add(layer["level"])
    want = {(128, 2, c) for c in ("7x7", "3x3", "1x1")} | {(64, 2, c) for c in ("7x7", "3x3", "1x1", "im2col")}
    want |= {(48, 2, "1x1"), (32, 2, "1x1"), (16, 2, "1x1"), (64, 3, 136), (32, 3, 128), (128, 1, 136), (64, 1, 128)}
    assert want <= seen, sorted(want - seen, key=str)
    assert partial == {0, 1, 2, 3}, partial


@pytest.mark.gpu
def test_tile_widths_are_bit_identical():
    """Frame 0 alone (stage layers at half width) and frame 0 in a two-frame batch (full width): the kernel's K order per
    output element does not depend on BN, so every conv blob and the maps must be bit-identical."""
    model, net_w, net_h = engine.COCO_18, 656, 368
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    W = weights_with_biases(model)
    eng = engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=engine.PREC_F16X2, max_batch=2)
    eng.set_weights(W)
    frames = frames_for(2, 2 * net_w, 2 * net_h)
    out, widths = [], []
    for n in (1, 2):
        eng.forward_frames(frames[:n])
        out.append({l["top"]: eng.fetch_blob(l["top"])[:1].copy() for l in checked_layers(model) if l["top"] not in CONFIGS_FINAL})
        out[-1]["maps"] = eng.fetch_maps(n)[:1]
        w_, h_, gap = level_geo(net_w, net_h, 3)
        widths.append(tc_instance(128, 7, n * (h_ + gap) * (w_ + gap), engine.PREC_F16X2, nsm)[0])
    eng.close()
    assert widths == [64, 128], widths
    diff = [k for k in out[0] if not np.array_equal(out[0][k], out[1][k])]
    assert not diff, diff


CONFIGS_FINAL = {"Mconv7_stage6_L1", "Mconv7_stage6_L2"}


@pytest.mark.gpu
def test_fetch_blob_returns_true_values_after_calibration():
    model, net_w, net_h = engine.COCO_18, 160, 96
    W = weights_with_biases(model)
    frame = synth.make_frame(4, 2 * net_h, 2 * net_w)
    got = []
    for cal in (False, True):
        eng = engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=engine.PREC_F16X2)
        eng.set_weights(W)
        if cal:
            eng.calibrate([frame])
        eng.forward_frames([frame])
        got.append([eng.fetch_blob(b) for b in ("conv1_1", "pool1_stage1")])
        eng.close()
    for a, b in zip(*got):
        assert float(np.abs(a - b).max()) <= 1e-6 * float(np.abs(a).max())


@pytest.mark.gpu
def test_fetch_blob_refuses_overwritten_stage_outputs():
    """After a 6-stage forward the ping-pong concat buffers hold stages 4 and 5: the earlier stage outputs are refused with the
    reusing layer named, and a kept one still passes its float64 check."""
    model, net_w, net_h = engine.COCO_18, 160, 96
    W = weights_with_biases(model)
    eng = engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=engine.PREC_F16X2)
    eng.set_weights(W)
    eng.forward_frames([synth.make_frame(4, 2 * net_h, 2 * net_w)])
    refused = set()
    for l in conv_layers(model)[0]:
        if l["top"] in CONFIGS_FINAL:
            continue
        try:
            eng.fetch_blob(l["top"])
        except engine.PoseEngineError as ex:
            assert "reuses its buffer" in str(ex) and "Mconv7_stage" in str(ex), str(ex)
            refused.add(l["top"])
    assert refused == REUSED, refused
    with pytest.raises(engine.PoseEngineError, match="conv5_5_CPM_L1 is not kept: Mconv7_stage3_L1"):
        eng.fetch_blob("conv5_5_CPM_L1")
    layer = [l for l in checked_layers(model) if l["name"] == "Mconv7_stage5_L1"][0]
    blobs = Blobs(eng, 1, model, W)
    w_, h_, gap = level_geo(net_w, net_h, 3)
    check_layer(layer, blobs, W, engine.PREC_F16X2, sample_pixels(1, h_, w_, gap, np.random.default_rng(3)), False, False)
    eng.close()
