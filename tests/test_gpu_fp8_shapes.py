"""The FP8 mode (PE_PREC_E4M3X1) on the generated pose graphs of tests/test_conv_shapes.py.

Every conv of every case, at one and three frames, against float64 with the bound of tests/test_gpu_fp8_mode.py: the distance
d of the reference (the engine's stored input, the e4m3-rounded weights) from the rounding cell of the stored e4m3 output is at
most B * mag.  The cases exercise what the shipped nets do not: Concat slots of 7, 72 and 129 channels (e4m3 slots are 16-byte,
i.e. 16-channel, aligned, and the shared F of 72 channels is copied into the second concat buffer in whole 16-byte chunks),
a shared F of 72 or 100 channels read directly by stage 1 (one 128-channel K block), 5x5 filters and three stages.  The
reference reads each Concat part where its producer wrote it, while stage 3 of "three_stages" reads F from the copy in the
second buffer: a copy that dropped channels fails there.

The last stage's convolutions write the planar fp32 maps unrounded, so there d = |got - ref| is the raw accumulation error of
the chunked FP8 accumulation.  In "three_stages" that layer is a 7x7 on 129 channels (padded to 256): 49 K steps of 128
channels in chunks of 7 steps, 896 K each - the longest chunk the mode runs - so its error measures the chunk length.
Max pooling is checked exact.

Calibrated, three_stages: pe_calibrate gives every producer its own range scale, so the Concat readers of stages 2 and 3 fold
power-of-two range ratios of three producers into their e4m3 weights; the reference rounds the weights with those ratios
folded in (float_layer of tests/test_gpu_mixed_precision.py).  The width rule restated: the cases run every one-byte instance
at every filter size (tests/test_gpu_s8_shapes.py states it without a GPU).
"""
import numpy as np
import pytest
import torch

from caffe_rtpose_b200 import engine
from test_conv_shapes import CASES, FRAMES, layer_class, level_dims, spec_weights, write_prototxt
from test_gpu_conv_layers import Blobs, conv_layers, conv_ref, frames_for, plan_gaps, sample_pixels
from test_gpu_fp8_mode import B_E8, e4m3_cell, packed_weights
from test_gpu_mixed_precision import float_layer
from test_gpu_s8_mode import IntBlobs
from test_gpu_s8_shapes import WANT_ONE_BYTE, one_byte_widths

pytestmark = pytest.mark.gpu
E8 = engine.PREC_E4M3X1
# largest d / mag per layer class over the cases, about 2x the values measured on an H100 80GB HBM3 (700 W power limit):
# 1x1 1.6e-4, 3x3 8.2e-5, 5x5 6.7e-5, 7x7 6.6e-5; fp32 maps 1x1 1.1e-4, 3x3 7.1e-5, 5x5 1.5e-4, 7x7 7.3e-5; conv1_1 0 (held to 1e-5)
MEASURED_MAX = {"1x1": 3.5e-4, "3x3": 1.8e-4, "5x5": 1.5e-4, "7x7": 1.5e-4, "1x1 fp32": 2.5e-4, "3x3 fp32": 1.5e-4,
                "5x5 fp32": 3.2e-4, "7x7 fp32": 1.5e-4, "im2col": 1e-5}


@pytest.mark.parametrize("name", list(CASES))
def test_generated_convs_vs_float64_e4m3(name, tmp_path):
    spec, path = write_prototxt(name, tmp_path)
    c = CASES[name]
    net_w, net_h = c["net_w"], c["net_h"]
    gaps = plan_gaps(prototxt=path)
    W = spec_weights(spec)
    eng = engine.PoseEngine(None, net_w, net_h, 2 * net_w, 2 * net_h, start_scale=0.5, precision=E8, prototxt=path,
                            max_batch=max(FRAMES))
    eng.set_weights(W)
    layers = conv_layers(None, spec)[0]
    pools = [l for l in spec["layers"] if l["type"] == "Pooling"]
    rng = np.random.default_rng(11)
    worst = {}
    for n in FRAMES:
        # the planar net input in the frame path's steps of 1/256 (exact in the fp16 input plane)
        eng.forward_net_input((rng.integers(0, 256, (n, 3, net_h, net_w)) / 256.0 - 0.5).astype(np.float32))
        blobs = Blobs(eng, n, None, W, spec)
        for layer in layers:
            w_, h_ = level_dims(net_w, net_h, layer["level"])
            pts = sample_pixels(n, h_, w_, gaps[layer["level"]], rng, 300)
            w, b = W[layer["name"]]
            x, y = blobs.get(layer["bottom"]), blobs.get(layer["top"])
            ref, mag = conv_ref(x, packed_weights(w, layer["name"] == "conv1_1"), b, pts, layer["relu"])
            got = y[pts[:, 0], :, pts[:, 1], pts[:, 2]].astype(np.float64)
            fp32 = layer["top"] in blobs.final_off
            if fp32:
                d = np.abs(got - ref)
            else:
                lo, hi = e4m3_cell(got)
                d = np.maximum(0.0, np.maximum(ref - hi, lo - ref))
            bad = d > B_E8 * mag
            if bad.any():
                i, co = np.argwhere(bad)[0]
                raise AssertionError("%s, %d frame(s): %d of %d elements outside B x mag; first at (n, y, x) = %s channel %d: got "
                                     "%.9g, ref %.9g, mag %.3g" % (layer["name"], n, int(bad.sum()), bad.size, tuple(pts[i]), co,
                                                                  got[i, co], ref[i, co], mag[i, co]))
            key = layer_class(layer) + (" fp32" if fp32 else "")
            worst[key] = max(worst.get(key, 0.0), float((d / mag).max()))
        for p in pools:   # max pooling copies the winner: exact
            bot = blobs.get(p["bottom"][0])
            top = eng.fetch_blob(p["top"][0])[:n]
            N, C, H, Wd = bot.shape
            want = bot.reshape(N, C, H // 2, 2, Wd // 2, 2).max(axis=(3, 5))
            assert np.array_equal(top, want), "%s, %d frame(s): %d elements differ" % (p["name"], n, int((top != want).sum()))
    eng.close()
    print("\n%s e4m3x1: largest d / mag per layer class: %s" % (name, " ".join("%s %.3e" % (k, worst[k]) for k in sorted(worst))))
    if MEASURED_MAX is not None:
        over = {k: v for k, v in worst.items() if v > MEASURED_MAX[k]}
        assert not over, "accumulation error above what this kernel measured: %s" % over


def test_generated_convs_vs_float64_e4m3_calibrated(tmp_path):
    name = "three_stages"
    spec, path = write_prototxt(name, tmp_path)
    c = CASES[name]
    net_w, net_h = c["net_w"], c["net_h"]
    gaps = plan_gaps(prototxt=path)
    kinds = engine.plan_formats(None, E8, None, prototxt=path)["convs"]
    W = spec_weights(spec)
    eng = engine.PoseEngine(None, net_w, net_h, 2 * net_w, 2 * net_h, start_scale=0.5, precision=E8, prototxt=path,
                            max_batch=max(FRAMES))
    eng.set_weights(W)
    rng = np.random.default_rng(11)
    worst, mixed = {}, set()
    for n in FRAMES:
        eng.calibrate(frames_for(n, 2 * net_w, 2 * net_h))
        eng.forward_net_input((rng.integers(0, 256, (n, 3, net_h, net_w)) / 256.0 - 0.5).astype(np.float32))
        ib = IntBlobs(eng, n, None, W, spec)
        for layer in conv_layers(None, spec)[0]:
            w_, h_ = level_dims(net_w, net_h, layer["level"])
            pts = sample_pixels(n, h_, w_, gaps[layer["level"]], rng, 300)
            compute, out = kinds[layer["name"]][:2]
            r = float_layer(layer, eng, ib.blobs, ib.k, W, compute, out, pts)
            key = layer_class(layer) + (" fp32" if out == "f32" else "")
            worst[key] = max(worst.get(key, 0.0), r)
            if len(set(ib.k(layer["bottom"]))) > 1:
                mixed.add(layer["name"])
    eng.close()
    print("\n%s e4m3x1 calibrated: largest d / mag per layer class: %s; readers of mixed range scales: %s" % (
        name, " ".join("%s %.3e" % (k, worst[k]) for k in sorted(worst)), sorted(mixed)))
    assert {"Mconv1_stage%d_L%d" % (s, b) for s in (2, 3) for b in (1, 2)} <= mixed, mixed
    over = {k: v for k, v in worst.items() if v > MEASURED_MAX[k]}
    assert not over, "accumulation error above what this kernel measured: %s" % over


def test_cases_run_every_one_byte_instance(tmp_path):
    seen = one_byte_widths(tmp_path, torch.cuda.get_device_properties(0).multi_processor_count)
    assert WANT_ONE_BYTE <= seen, sorted(WANT_ONE_BYTE - seen, key=str)
