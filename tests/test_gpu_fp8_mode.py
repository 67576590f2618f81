"""The FP8 mode (PE_PREC_E4M3X1: one e4m3 plane of activations and weights, one FP8 MMA per MAC) on the GPU.

Per layer, every conv layer of COCO and MPI at one and three frames is checked against float64 with the sampling of
tests/test_gpu_conv_layers.py.  The reference is exact: the layer's stored e4m3 input (pe_fetch_blob) convolved in float64
with the weights the engine packed, w * 2^k rounded to e4m3 (torch's cast; max|w| * 2^k in [128, 256), 2^k exact) and
divided by 2^k again; conv1_1 reads the fp16 input with weights rounded to fp16 as in PE_PREC_F16X1.  The engines run
uncalibrated (scale 1: W-he activations stay far below 448), so no range ratio enters the weights.

The stored output is the e4m3 rounding of the kernel's fp32 value t, so t lies in the cell of reals that round to it (half
the e4m3 spacing on either side of the stored value: 2^-4 of it in relative terms for normal values, 2^-10 absolute below
2^-6; half as much below an exact power of two, where the spacing halves).  The checked quantity is the distance d from the
float64 reference to that cell, which is at most |t - ref|:
    d <= B * mag,    mag = sum |a||w| + |b|
It is the accumulation error that the output rounding does not hide.  The last stage's 1x1 layers write the planar fp32 maps,
unrounded: there d = |got - ref|, the raw accumulation error.
  B                 the accumulation.  Products of two e4m3 values are exact in fp32.  Hopper's FP8 wgmma adds them into an
                    accumulator that keeps fewer bits than fp32: assume 13 fraction bits, truncated, i.e. at most 2^-12 of
                    the partial magnitude per k32 MMA.  A hi*hi chunk is <= 7 K steps of 4 MMAs: 28 * 2^-12 of mag; the
                    round-to-nearest sum of the chunks and the epilogue add <= 24 * 2^-24.  B = 28 * 2^-12 + 2^-19.
Each layer class is also held to about 2x its measured maximum (MEASURED_MAX), so that a kernel without chunking or with a
wrong tap cannot hide under the loose rigorous bound.

Whole net, max pool, range, determinism and the audit: see the tests below.
"""
import numpy as np
import pytest
import torch

from caffe_rtpose_b200 import engine, synth
from oracle import orc
from test_gpu_conv_layers import (Blobs, checked_layers, conv_ref, frames_for, layer_class, level_geo, sample_pixels,
                                  tc_cout_pad, weights_with_biases)

pytestmark = pytest.mark.gpu
E8 = engine.PREC_E4M3X1
B_E8 = 28 * 2.0 ** -12 + 2.0 ** -19
CONFIGS = {"coco_e8": (engine.COCO_18, 656, 368, (1, 3)), "mpi_e8": (engine.MPI_15, 496, 368, (1, 3))}
# largest d / mag per layer class (module docstring), about 2x the values measured on an H100 80GB HBM3 (700 W power limit) over
# both configurations and tile widths: 7x7 7.3e-5, 3x3 2.1e-4, 1x1 1.1e-4, the fp32 1x1 map layers 2.1e-4, conv1_1 0 (held to
# 1e-5)
MEASURED_MAX = {"7x7": 1.5e-4, "3x3": 4.5e-4, "1x1": 2.5e-4, "1x1 fp32": 4.5e-4, "im2col": 1e-5}
# max |maps - oracle| / max |oracle| at 160x96, calibrated, about 2x the largest value measured on an H100 80GB HBM3 (700 W
# power limit): COCO 0.214 / 0.182 and MPI 0.166-0.178 / 0.189 (frames 0 / 1, one and two scales), the calibrated filler net
# 0.122, the calibrated 1.6x-per-layer net 0.238
TOL_NET = 0.5


def rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


def packed_weights(w, fp16):
    """The weights as the engine packs them: w * 2^k rounded to e4m3 (max|w| * 2^k in [128, 256)), or to fp16 for conv1_1
    (max|w| * 2^k in [2^13, 2^14)), divided by 2^k again (exact)."""
    mx = float(np.abs(w).max())
    if mx == 0:
        return w.astype(np.float64)
    _, ex = np.frexp(np.float32(mx))
    k = (14 if fp16 else 8) - int(ex)
    s = np.ldexp(np.float32(1), k)
    t = torch.from_numpy((w * s).astype(np.float32))
    r = t.half().float() if fp16 else t.to(torch.float8_e4m3fn).float()
    return r.double().numpy() / float(s)


def e4m3_cell(g):
    """[lo, hi]: the reals that round to nearest e4m3 value g (float64 array of stored values, scale 1)."""
    a = np.abs(g)
    e = np.floor(np.log2(np.where(a > 0, a, 1.0)))
    normal = a >= 2.0 ** -6
    up = np.where(normal, 2.0 ** (e - 4), 2.0 ** -10)                             # half the spacing above |g|
    down = np.where(normal & (a == 2.0 ** e) & (e > -6), 2.0 ** (e - 5), up)     # below a power of two the spacing halves
    return np.where(g >= 0, g - down, g - up), np.where(g >= 0, g + up, g + down)


def check_layer(layer, blobs, W, pts):
    """(layer class, d / mag) of one layer: d the distance of the float64 reference from the rounding cell of the stored
    e4m3 output, or from the fp32 output itself for the planar maps."""
    w, b = W[layer["name"]]
    x, y = blobs.get(layer["bottom"]), blobs.get(layer["top"])
    wq = packed_weights(w, layer["name"] == "conv1_1")
    ref, mag = conv_ref(x, wq, b, pts, layer["relu"])
    got = y[pts[:, 0], :, pts[:, 1], pts[:, 2]].astype(np.float64)
    fp32 = layer["top"] in blobs.final_off
    if fp32:
        d = np.abs(got - ref)
    else:
        lo, hi = e4m3_cell(got)
        d = np.maximum(0.0, np.maximum(ref - hi, lo - ref))
    bad = d > B_E8 * mag
    if bad.any():
        i, c = np.argwhere(bad)[0]
        raise AssertionError("%s: %d of %d elements outside the bound; first at %s channel %d: got %.9g, ref %.9g, mag %.3g"
                             % (layer["name"], int(bad.sum()), bad.size, tuple(pts[i]), c, got[i, c], ref[i, c], mag[i, c]))
    return layer_class(layer) + (" fp32" if fp32 else ""), float((d / mag).max())


def tc_instance_e8(cout, M, nsm, share=2):
    """The tile width of tc_layer_launch, restated (e4m3 runs one plane: full width up to 128)."""
    cp = tc_cout_pad(cout)
    bn = min(cp, 128)
    mt = (M + 127) // 128
    sms = max(1, nsm // share)
    if bn >= 64 and min(mt * (cp // (bn // 2)), sms) * 0.80 > min(mt * (cp // bn), sms) * 1.00:
        bn //= 2
    return bn


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_conv_layers_vs_float64(cfg):
    model, net_w, net_h, counts = CONFIGS[cfg]
    W = weights_with_biases(model)
    eng = engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=E8, max_batch=max(counts))
    eng.set_weights(W)
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(11)
    worst = {}
    for n in counts:
        eng.forward_frames(frames_for(n, 2 * net_w, 2 * net_h))
        rc, ratio, layer_name = eng.range_status()
        assert rc == 0, (rc, ratio, layer_name)
        blobs = Blobs(eng, n, model, W)
        for layer in checked_layers(model):
            w_, h_, gap = level_geo(net_w, net_h, layer["level"])
            cls, r = check_layer(layer, blobs, W, sample_pixels(n, h_, w_, gap, rng))
            bn = tc_instance_e8(W[layer["name"]][0].shape[0], n * (h_ + gap) * (w_ + gap), nsm)
            key = (cls, bn)
            worst[key] = max(worst.get(key, 0.0), r)
    eng.close()
    print("\n%s: largest distance of the reference from the output's rounding cell / mag per (layer class, BN):" % cfg)
    for key in sorted(worst, key=str):
        print("  %-7s BN=%-4d %.3e" % (key[0], key[1], worst[key]))
    if MEASURED_MAX is not None:
        over = {k: v for k, v in worst.items() if v > MEASURED_MAX[k[0]]}
        assert not over, "accumulation error above what this kernel measured: %s" % over


def test_configs_launch_every_e4m3_instance():
    """Restating the tile-width rule: the configurations above launch every e4m3 instance, BN 16-128 (the 1x1 map layers:
    MPI's 15 and 28 channels, COCO's 19 and 38), 3x3 and 7x7 at full and half width, and conv1_1's fp16-input instance."""
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    seen = set()
    for model, net_w, net_h, counts in CONFIGS.values():
        W = synth.make_weights(model)
        for n in counts:
            for layer in checked_layers(model):
                w_, h_, gap = level_geo(net_w, net_h, layer["level"])
                seen.add((tc_instance_e8(W[layer["name"]][0].shape[0], n * (h_ + gap) * (w_ + gap), nsm), layer_class(layer)))
    want = {(128, "7x7"), (64, "7x7"), (128, "3x3"), (64, "3x3"), (128, "1x1"), (48, "1x1"), (32, "1x1"), (16, "1x1")}
    assert want <= seen, sorted(want - seen, key=str)
    assert {bn for bn, c in seen if c == "im2col"} <= {64, 32}


def test_tile_widths_are_bit_identical():
    """Frame 0 alone (stage layers at half width) and frame 0 in a batch of two (full width) give bit-identical blobs."""
    model, net_w, net_h = engine.COCO_18, 656, 368
    W = weights_with_biases(model)
    eng = engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=E8, max_batch=2)
    eng.set_weights(W)
    frames = frames_for(2, 2 * net_w, 2 * net_h)
    final = {"Mconv7_stage6_L1", "Mconv7_stage6_L2"}
    out = []
    for n in (1, 2):
        eng.forward_frames(frames[:n])
        out.append({l["top"]: eng.fetch_blob(l["top"])[:1].copy() for l in checked_layers(model) if l["top"] not in final})
        out[-1]["maps"] = eng.fetch_maps(n)[:1]
    eng.close()
    diff = [k for k in out[0] if not np.array_equal(out[0][k], out[1][k])]
    assert not diff, diff


def test_max_pool_exact():
    """Every pool top equals the 2x2 max (ceil mode) of its e4m3 input exactly."""
    model, net_w, net_h = engine.COCO_18, 320, 176
    W = weights_with_biases(model)
    eng = engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=E8, max_batch=2)
    eng.set_weights(W)
    eng.forward_frames(frames_for(2, 2 * net_w, 2 * net_h))
    for bottom, top in (("conv1_2", "pool1_stage1"), ("conv2_2", "pool2_stage1"), ("conv3_4", "pool3_stage1")):
        x, y = eng.fetch_blob(bottom)[:2], eng.fetch_blob(top)[:2]
        H, Wd = x.shape[2], x.shape[3]
        xp = np.full((2, x.shape[1], (H + 1) // 2 * 2, (Wd + 1) // 2 * 2), -np.inf, np.float32)
        xp[:, :, :H, :Wd] = x
        want = xp.reshape(2, x.shape[1], xp.shape[2] // 2, 2, xp.shape[3] // 2, 2).max(axis=(3, 5))
        assert np.array_equal(y, want), top
    eng.close()


def whole_net(model, S, W, calibrate=True):
    net_w, net_h = 160, 96
    frames = [synth.make_frame(20 + i, 192, 320) for i in range(2)]
    onet = orc.Net(model)
    onet.set_weights(W)
    x = [orc.preprocess(f, net_h, net_w, S, 1.0, 0.25) for f in frames]
    eng = engine.PoseEngine(model, net_w, net_h, 320, 192, num_scales=S, start_scale=1.0, scale_gap=0.25, precision=E8, max_batch=2)
    eng.set_weights(W)
    if calibrate:
        eng.calibrate(frames)
    return eng, frames, [onet.forward(xi) for xi in x]


@pytest.mark.parametrize("S", [1, 2])
@pytest.mark.parametrize("model", [engine.COCO_18, engine.MPI_15])
def test_whole_net_vs_oracle(model, S):
    """Calibrated, 160x96: stride-8 maps against the oracle; the same batch twice (the second a CUDA-graph replay) gives
    bit-identical maps, peaks and joints."""
    eng, frames, omaps = whole_net(model, S, synth.make_weights(model, "he", seed=7))
    calls = []
    for _ in range(3):
        eng.forward_frames(frames)
        calls.append((eng.fetch_maps(2).copy(), [eng.fetch(k) for k in range(2)]))
    maps = calls[0][0]
    errs = [rel(maps[i * S:(i + 1) * S], omaps[i]) for i in range(2)]
    print("\nE4M3X1 %s 160x96 S=%d: maps vs oracle %s" % ("COCO" if model == engine.COCO_18 else "MPI", S, ["%.3e" % e for e in errs]))
    assert max(errs) < TOL_NET
    for c in calls[1:]:
        assert np.array_equal(c[0], maps)
        for (na, ja, pa), (nb, jb, pb) in zip(c[1], calls[0][1]):
            assert na == nb and np.array_equal(ja, jb) and np.array_equal(pa, pb)
    eng.close()


@pytest.mark.parametrize("kind", ["caffe_filler", "growing"])
def test_range_reported_and_calibrated(kind):
    """Uncalibrated, the prototxt's gaussian(0.01) filler and the 1.6x-per-layer net leave e4m3's range: PE_ERR_RANGE with a
    layer named.  Calibrated, both meet the whole-net bound, and a replayed CUDA graph reproduces the calibration forward."""
    model, net_w, net_h = engine.COCO_18, 160, 96
    if kind == "caffe_filler":
        W = synth.make_weights(model, "caffe")
    else:
        W = {k: (w * np.float32(1.6), b) for k, (w, b) in synth.make_weights(model, "he").items()}
    frame = synth.make_frame(3, 2 * net_h, 2 * net_w)
    onet = orc.Net(model)
    onet.set_weights(W)
    omaps = onet.forward(orc.preprocess(frame, net_h, net_w, 1, 1.0, 0.3))
    eng = engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=E8)
    eng.set_weights(W)
    eng.forward_frames([frame])
    eng.sync()
    rc, worst, layer = eng.range_status()
    assert rc == 5 and layer, (rc, worst, layer)              # PE_ERR_RANGE, the layer named
    eng.calibrate([frame])
    cal = eng.fetch_maps(1).copy()
    err = rel(cal, omaps)
    print("\nE4M3X1 calibrated %s: maps vs oracle %.3e" % (kind, err))
    assert err < TOL_NET
    for _ in range(3):
        eng.forward_frames([frame])
        assert np.array_equal(eng.fetch_maps(1), cal)
    rc, worst, layer = eng.range_status()
    assert rc == 0 and worst < 0.5, (rc, worst, layer)
    eng.close()


def test_audit_against_parity_on_bench_step():
    """pe_compare_results of E4M3X1 (calibrated) against F16X2 on one bench step (C2: 656x368, 9 frames, W-he).  Only
    checked to be well formed: He-init noise maps are the worst case for pose agreement, so the numbers are reported."""
    model, B = engine.COCO_18, 9
    W = synth.make_weights(model, "he")
    frames = [synth.make_frame(i, 720, 1280) for i in range(B)]
    res = {}
    for prec in (engine.PREC_F16X2, E8):
        e = engine.PoseEngine(model, 656, 368, 1280, 720, max_batch=B, precision=prec)
        e.set_weights(W)
        if prec == E8:
            e.calibrate(frames[:1])
        e.forward_frames(frames)
        res[prec] = ([e.fetch(k) for k in range(B)], e.fetch_maps(B).copy())
        e.close()
    d = [engine.compare_results(a, b, 1e-3 * 1280 / 656) for a, b in zip(res[E8][0], res[engine.PREC_F16X2][0])]
    print("\nE4M3X1 vs F16X2, bench step: map error %.3e of the parity maximum; frames identical %d/%d, persons matched %d/%d, "
          "max joint distance %.1f px" % (rel(res[E8][1], res[engine.PREC_F16X2][1]), sum(x["identical"] for x in d), B,
                                          sum(x["persons_matched"] for x in d), sum(r[0] for r in res[engine.PREC_F16X2][0]),
                                          max(x["max_joint_dist"] for x in d)))
    for x in d:
        assert set(x) >= {"identical", "parts_count_differ", "peaks_moved", "persons_matched", "max_joint_dist"}
        assert x["persons_matched"] >= 0 and x["max_joint_dist"] >= 0
