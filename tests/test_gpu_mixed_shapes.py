"""Mixed precision (pe_create_mixed) on the generated pose graphs of tests/test_conv_shapes.py.

For each case and each base (E4M3X1 uncalibrated, S8X1 calibrated on the first forward's frames), an engine with the case's
fp16 list (LISTS), at one and three frames.  Every conv is checked with the per-layer checks of
tests/test_gpu_mixed_precision.py: s8 layers bit for bit, including those that store fp16; e4m3 layers with B_E8; fp16 layers
with the accumulation bound of test_conv_shapes.layer_bound for F16X1 at the layer's own K, without its 2^-10 term for the
weights' rounding, since the reference convolves the packed weights.  (The fixed B_F16 = 2^-17 holds for the shipped nets
only.)  Every pool top equals the 2x2 max of its bottom, and each (compute kind, fp32 output, layer class) is held to about 2x
its measured maximum.

The lists make the cases run all 15 boundary instances of conv_mixed.cu, <1, e4m3, f16>, <1, f16, s8> and <1, s8, f16> at
BN 16, 32, 48, 64 and 128: asserted with the device's SM count and, without a GPU, at 132 SMs.
"""
import numpy as np
import pytest
import torch

from caffe_rtpose_b200 import engine
from test_conv_shapes import CASES, F1, FRAMES, layer_bound, layer_class, level_dims, spec_weights, write_prototxt
from test_gpu_conv_layers import conv_layers, frames_for, plan_gaps, sample_pixels
from test_gpu_mixed_precision import float_layer, s8_layer
from test_gpu_s8_mode import IntBlobs, tc_bn
from test_gpu_s8_shapes import NSM_H100, check_pools

E8, S8 = engine.PREC_E4M3X1, engine.PREC_S8X1
# the fp16 layers per case: with them the cases reach every boundary instance at 1 and 3 frames
LISTS = {"k5_k7_vgg": "conv1_3,conv2_1,conv3_1", "k1_k3_wide": "conv1_2", "three_stages": "conv1_3", "tiny_16x16": "narrow",
         "tiny_32x16": "narrow"}
WANT_BOUNDARY = {(c, o, bn) for c, o in (("e4m3", "f16"), ("f16", "s8"), ("s8", "f16")) for bn in (16, 32, 48, 64, 128)}
# largest d / mag per (compute kind, "f32" for the planar maps, layer class) over the cases, both bases and both frame counts,
# about 2x the values measured on an H100 80GB HBM3 (700 W power limit): e4m3 1x1 3.4e-5, 3x3 6.7e-5, 5x5 6.9e-5, 7x7 5.0e-5,
# fp32 maps 1x1 1.2e-4, 5x5 7.6e-5, 7x7 7.0e-5; fp16 1x1 2.8e-9, 3x3 5.2e-9, 5x5 4.7e-8, 7x7 8.8e-9, conv1_1 0 (held to
# 5e-8 as in tests/test_gpu_mixed_precision.py), fp32 maps 1x1 1.2e-7, 3x3 1.1e-7.  The s8 layers are bit-exact.
MEASURED_MAX = {("e4m3", "", "1x1"): 7e-5, ("e4m3", "", "3x3"): 1.4e-4, ("e4m3", "", "5x5"): 1.4e-4, ("e4m3", "", "7x7"): 1e-4,
                ("e4m3", "f32", "1x1"): 2.4e-4, ("e4m3", "f32", "5x5"): 1.6e-4, ("e4m3", "f32", "7x7"): 1.4e-4,
                ("f16", "", "1x1"): 6e-9, ("f16", "", "3x3"): 1.1e-8, ("f16", "", "5x5"): 1e-7, ("f16", "", "7x7"): 2e-8,
                ("f16", "", "im2col"): 5e-8, ("f16", "f32", "1x1"): 2.5e-7, ("f16", "f32", "3x3"): 2.5e-7}


def boundary_instances(tmp_path, nsm):
    """{(compute kind, stored kind, BN)} of the layers whose stored kind differs from their compute kind, over the cases at
    FRAMES in both bases."""
    seen = set()
    for base in (E8, S8):
        for name, c in CASES.items():
            spec, path = write_prototxt(name, tmp_path)
            gaps = plan_gaps(prototxt=path)
            kinds = engine.plan_formats(None, base, LISTS[name], prototxt=path)["convs"]
            cout = {l["name"]: l["num_output"] for l in spec["layers"] if l["type"] == "Convolution"}
            for layer in conv_layers(None, spec)[0]:
                compute, out = kinds[layer["name"]][:2]
                w_, h_ = level_dims(c["net_w"], c["net_h"], layer["level"])
                g = gaps[layer["level"]]
                for n in FRAMES:
                    if out not in (compute, "f32"):
                        seen.add((compute, out, tc_bn(cout[layer["name"]], n * (h_ + g) * (w_ + g), nsm)))
    return seen


def test_lists_reach_every_boundary_instance_at_132_sms(tmp_path):
    seen = boundary_instances(tmp_path, NSM_H100)
    assert WANT_BOUNDARY <= seen, sorted(WANT_BOUNDARY - seen)


@pytest.mark.gpu
def test_lists_reach_every_boundary_instance(tmp_path):
    seen = boundary_instances(tmp_path, torch.cuda.get_device_properties(0).multi_processor_count)
    print("\n(compute, stored, BN) of the boundary layers: %s" % sorted(seen))
    assert WANT_BOUNDARY <= seen, sorted(WANT_BOUNDARY - seen)


@pytest.mark.gpu
@pytest.mark.parametrize("base", [E8, S8])
@pytest.mark.parametrize("name", list(CASES))
def test_generated_convs_mixed(name, base, tmp_path):
    spec, path = write_prototxt(name, tmp_path)
    c = CASES[name]
    net_w, net_h = c["net_w"], c["net_h"]
    gaps = plan_gaps(prototxt=path)
    fmt = engine.plan_formats(None, base, LISTS[name], prototxt=path)
    W = spec_weights(spec)
    eng = engine.PoseEngine(None, net_w, net_h, 2 * net_w, 2 * net_h, start_scale=0.5, precision=base, prototxt=path,
                            max_batch=max(FRAMES), f16_layers=LISTS[name])
    eng.set_weights(W)
    if base == S8:
        eng.calibrate(frames_for(FRAMES[0], 2 * net_w, 2 * net_h))
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(11)
    worst, run = {}, set()
    for n in FRAMES:
        eng.forward_frames(frames_for(n, 2 * net_w, 2 * net_h))
        ib = IntBlobs(eng, n, None, W, spec)
        kscale = ib.k if base == S8 else (lambda blob: np.zeros(ib.blobs.get(blob).shape[1], int))
        for layer in conv_layers(None, spec)[0]:
            compute, out, in_act = fmt["convs"][layer["name"]][:3]
            w_, h_ = level_dims(net_w, net_h, layer["level"])
            g = gaps[layer["level"]]
            pts = sample_pixels(n, h_, w_, g, rng, 300)
            if compute == "s8":
                r = s8_layer(layer, ib, W, out, pts)
            else:
                B = None
                if compute == "f16":   # F16X1's bound at this K, the weight rounding taken out (the reference uses them packed)
                    ks, cp = (1, 64) if layer["name"] == "conv1_1" else (layer["k"], fmt["acts"][in_act][1])
                    B = layer_bound(F1, ks, cp, W[layer["name"]][0].shape[1]) - 2.0 ** -10
                r = float_layer(layer, eng, ib.blobs, kscale, W, compute, out, pts, B)
            key = (compute, "f32" if out == "f32" else "", layer_class(layer))
            worst[key] = max(worst.get(key, 0.0), r)
            if out not in (compute, "f32"):
                run.add((compute, out, tc_bn(W[layer["name"]][0].shape[0], n * (h_ + g) * (w_ + g), nsm)))
        check_pools(eng, spec, ib.blobs, n, "%d frame(s)" % n)
    eng.close()
    print("\n%s base %d + %s: largest d / mag per (compute kind, fp32 output, layer class): %s" % (
        name, base, LISTS[name], {"/".join(filter(None, k)): "%.3e" % v for k, v in sorted(worst.items())}))
    print("  (compute, stored, BN) run: %s" % sorted(run))
    over = {k: v for k, v in worst.items() if k[0] != "s8" and v > MEASURED_MAX[k]}   # s8_layer has checked s8 bit for bit
    assert not over, "accumulation error above what this kernel measured: %s" % over
