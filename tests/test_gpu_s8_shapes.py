"""The INT8 mode (PE_PREC_S8X1) on the generated pose graphs of tests/test_conv_shapes.py, and its s32 sums near their bound.

Per layer: every conv of every case, at one and three frames, calibrated on the first forward's frames, bit for bit against
the integer reference of tests/test_gpu_s8_mode.py (check_layer) at the pixels of sample_pixels.  The cases run what the
shipped nets do not: 5x5 filters, output counts from 1 to 257 around every tile width, s8 Concat slots of 7, 72 and 129
channels (16-channel aligned), the copy of a 72-channel shared F into the second concat buffer in whole 16-byte chunks, K up
to 49 x 1024, and the smallest nets.  Two cases also zero every third output channel of several layers (a 5x5 layer, the
shared F and a stage output among them) and keep their biases of both signs: such a channel has sigma_c = 0, so q = 0,
f_c = 0 and t = b'_c (s8.h), as in trained checkpoints with dead channels.  Every pool top equals the 2x2 max of its bottom.

Whole stack: on three_stages and tiny_16x16 (two frames, calibrated) the integer chain of every layer, pool and Concat from
the stored net input equals pe_fetch_maps bit for bit, across the ping-pong concat buffers and the copy of F.

The accumulator bound: a 7x7 on 2688 s8 channels, K = 49 x 2688 = 131712 (99.7% of precision.h's 132104), with inputs and
weights near the s8 limits drives |acc| above 2^30.  Its fp32 maps (t unrounded) must equal the reference bit for bit, with
many sums above 2^24 that are not multiples of their fp32 spacing, so that __int2float_rn actually rounds there (measured on
an H100 80GB HBM3, 700 W power limit: F from -128 to -48, 45% saturated; largest |acc| 0.746 x 2^31; all 3648 compared sums
above 2^24, 3604 of them not representable in fp32).  With __int2float_rz in the epilogue, 1050 of its 2432 L1 map values
differ, while the per-case and whole-stack tests of this module still pass.  He-init
weights keep the sums of the cases far below 2^24, where every conversion is exact: the largest |acc| per case is printed,
2^15.5 - 2^16.9 on an H100 80GB HBM3 (700 W power limit).

Instance coverage: restating the width rule, the cases run every one-byte instance (BN 16 - 128) at every filter size.
"""
import numpy as np
import pytest
import torch

from caffe_rtpose_b200 import engine, synth
from test_conv_shapes import CASES, FRAMES, layer_class, level_dims, pose_spec, spec_weights, write_prototxt
from test_gpu_conv_layers import conv_layers, frames_for, plan_gaps, sample_pixels
from test_gpu_s8_mode import IntBlobs, check_layer, fold, int_acc_at, quantize, tc_bn, whole_stack

S8 = engine.PREC_S8X1
NSM_H100 = 132   # SMs of an H100 SXM5, the width rule's input for the CPU coverage tests
# every third output channel of these layers is dead (all weights zero): 5x5 layers, the shared F (a Concat producer), the
# stage outputs written into the concat buffer, and 5x5 / 7x7 map layers
DEAD = {"k5_k7_vgg": ["conv1_2", "conv2_3", "conv3_2", "Mconv1_stage1_L1", "Mconv2_stage1_L1", "Mconv2_stage1_L2"],
        "three_stages": ["conv1_3", "conv3_1", "conv4_1", "Mconv3_stage1_L1", "Mconv3_stage1_L2", "Mconv2_stage2_L2",
                         "Mconv3_stage3_L1"]}
# (BN, layer class) of every one-byte conv instance: each tile width at every filter size, and the im2col'ed conv1_1 at the
# widths the cases give it
WANT_ONE_BYTE = {(bn, c) for bn in (16, 32, 48, 64, 128) for c in ("1x1", "3x3", "5x5", "7x7")}
WANT_ONE_BYTE |= {(bn, "im2col") for bn in (16, 48, 64, 128)}


def case_weights(name, spec):
    """spec_weights, with the dead channels of DEAD: weights zero, biases of alternating sign and 1-3x the layer's largest."""
    W = spec_weights(spec)
    rng = np.random.default_rng(17)
    for layer in DEAD.get(name, []):
        w, b = W[layer][0].copy(), W[layer][1].copy()
        dead = np.arange(0, w.shape[0], 3)
        w[dead] = 0
        sign = np.where(np.arange(len(dead)) % 2 == 0, 1.0, -1.0)
        b[dead] = (sign * np.abs(b).max() * rng.uniform(1, 3, len(dead))).astype(np.float32)
        W[layer] = (w, b)
    return W


def s8_engine(path, net_w, net_h, n, start_scale=0.5):
    # start scale 0.5: the scale geometry (16-pixel multiples, rtpose.cpp) then admits a net height of 24
    return engine.PoseEngine(None, net_w, net_h, 2 * net_w, 2 * net_h, start_scale=start_scale, precision=S8, prototxt=path,
                             max_batch=n)


def check_pools(eng, spec, blobs, n, what):
    for p in [l for l in spec["layers"] if l["type"] == "Pooling"]:   # max pooling copies the winner: exact
        bot = blobs.get(p["bottom"][0])
        top = eng.fetch_blob(p["top"][0])[:n]
        N, C, H, Wd = bot.shape
        want = bot.reshape(N, C, H // 2, 2, Wd // 2, 2).max(axis=(3, 5))
        assert np.array_equal(top, want), "%s, %s: %d elements differ" % (p["name"], what, int((top != want).sum()))


def one_byte_widths(tmp_path, nsm):
    """{(BN, layer class)} the cases launch at FRAMES in a one-plane one-byte mode (S8X1, E4M3X1: the same width rule)."""
    seen = set()
    for name, c in CASES.items():
        spec, path = write_prototxt(name, tmp_path)
        gaps = plan_gaps(prototxt=path)
        cout = {l["name"]: l["num_output"] for l in spec["layers"] if l["type"] == "Convolution"}
        for layer in conv_layers(None, spec)[0]:
            w_, h_ = level_dims(c["net_w"], c["net_h"], layer["level"])
            g = gaps[layer["level"]]
            for n in FRAMES:
                seen.add((tc_bn(cout[layer["name"]], n * (h_ + g) * (w_ + g), nsm), layer_class(layer)))
    return seen


# ------------------------------------------------------------------------------------------ CPU
def test_cases_run_every_one_byte_instance_at_132_sms(tmp_path):
    """The cases keep covering every one-byte instance at every filter size on an H100 SXM5 (132 SMs)."""
    seen = one_byte_widths(tmp_path, NSM_H100)
    assert WANT_ONE_BYTE <= seen, sorted(WANT_ONE_BYTE - seen, key=str)


def bound_spec(c_f=2688):
    """COCO maps from a 7x7 on c_f channels of F (conv4_1, no ReLU) at 64x64: K = 49 x c_f."""
    spec = pose_spec(engine.COCO_18, 64, 64, conv1_1=8, levels=[[(1, 8)], [], [(1, 8)], [(1, c_f)]], branch=[], k_out=7)
    spec["layers"] = [l for l in spec["layers"] if l["name"] != "relu_conv4_1"]
    return spec


def test_bound_net_plans_at_the_bound(tmp_path):
    """F's s8 pitch is 2688 (K = 131712 <= 132104); 2689 channels pad to 2816 in s8."""
    for c_f, pitch in ((2688, 2688), (2689, 2816)):
        path = tmp_path / ("bound_%d.prototxt" % c_f)
        path.write_text(synth.netspec_to_prototxt(bound_spec(c_f)))
        acts = engine.plan_formats(None, S8, None, prototxt=str(path))["acts"]
        assert [a[:2] for a in acts if a[2] == "conv4_1"] == [("s8", pitch)], acts


# ------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_cases_run_every_one_byte_instance(tmp_path):
    seen = one_byte_widths(tmp_path, torch.cuda.get_device_properties(0).multi_processor_count)
    print("\n(BN, layer class) run: %s" % sorted(seen, key=str))
    assert WANT_ONE_BYTE <= seen, sorted(WANT_ONE_BYTE - seen, key=str)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_generated_convs_bit_exact(name, tmp_path):
    spec, path = write_prototxt(name, tmp_path)
    c = CASES[name]
    net_w, net_h = c["net_w"], c["net_h"]
    gaps = plan_gaps(prototxt=path)
    W = case_weights(name, spec)
    eng = s8_engine(path, net_w, net_h, max(FRAMES))
    eng.set_weights(W)
    eng.calibrate(frames_for(FRAMES[0], 2 * net_w, 2 * net_h))
    layers = conv_layers(None, spec)[0]
    rng = np.random.default_rng(11)
    count, acc_max, dead = 0, 0.0, 0
    for n in FRAMES:
        eng.forward_frames(frames_for(n, 2 * net_w, 2 * net_h))
        ib = IntBlobs(eng, n, None, W, spec)
        for layer in layers:
            w_, h_ = level_dims(net_w, net_h, layer["level"])
            cnt, a = check_layer(layer, ib, W, sample_pixels(n, h_, w_, gaps[layer["level"]], rng, 300))
            count, acc_max = count + cnt, max(acc_max, a)
            if layer["name"] in DEAD.get(name, []):
                dead += len(range(0, W[layer["name"]][0].shape[0], 3))
        check_pools(eng, spec, ib.blobs, n, "%d frame(s)" % n)
    eng.close()
    print("\n%s s8x1: %d values bit-exact (%d dead output channels per frame count); largest |acc| %d = 2^%.1f"
          % (name, count, dead // len(FRAMES), acc_max, np.log2(acc_max)))
    assert acc_max < 2 ** 24   # He-init sums: every float(acc) is exact here, which is why the bound test below exists


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["three_stages", "tiny_16x16"])
def test_generated_whole_stack_bit_exact(name, tmp_path):
    """Two frames, calibrated on the first: the integer chain from the stored net input equals pe_fetch_maps bit for bit."""
    spec, path = write_prototxt(name, tmp_path)
    c = CASES[name]
    net_w, net_h = c["net_w"], c["net_h"]
    W = case_weights(name, spec)
    frames = [synth.make_frame(30 + i, 2 * net_h, 2 * net_w) for i in range(2)]
    eng = s8_engine(path, net_w, net_h, 2)
    eng.set_weights(W)
    eng.calibrate(frames[:1])
    eng.forward_frames(frames)
    maps = eng.fetch_maps(2).astype(np.float64)
    want = whole_stack(spec, W, eng, 2)
    eng.close()
    bad = maps != want
    assert not bad.any(), "%d of %d map values differ, max |diff| %.3g" % (int(bad.sum()), bad.size, float(np.abs(maps - want).max()))


def bound_weights(spec):
    """conv1_1 splits the input into a bright channel 0 (weights > 0, ReLU) and a dim channel 1 (weights < 0); conv1_2 and
    conv3_1 pass the channels through; F_c = -(beta_c x0 + beta_c / 6 x1).  Calibrated on a dim frame (x0 = 0), F's scale
    is set by beta / 6; on the mirrored bright frame (x1 = 0) F is 6x larger, from -48 to far past -128 (saturated) across
    channels.  The map layers' weights are negative, 0.8-1 of each channel's largest: q from about -101 to -127."""
    rng = np.random.default_rng(5)
    W = {}
    w1 = np.zeros((8, 3, 3, 3), np.float32)
    w1[0], w1[1] = 1.0 / 27, -1.0 / 27
    w1[2:] = rng.uniform(-1, 1, (6, 3, 3, 3)).astype(np.float32) / 27
    W["conv1_1"] = (w1, np.zeros(8, np.float32))
    for name in ("conv1_2", "conv3_1"):
        W[name] = (np.eye(8, dtype=np.float32)[:, :, None, None], np.zeros(8, np.float32))
    c_f = [l["num_output"] for l in spec["layers"] if l["name"] == "conv4_1"][0]
    beta = rng.uniform(0.25, 1.0, c_f).astype(np.float32)
    wf = np.zeros((c_f, 8, 1, 1), np.float32)
    wf[:, 0, 0, 0], wf[:, 1, 0, 0] = -beta, -beta / 6
    W["conv4_1"] = (wf, np.zeros(c_f, np.float32))
    for name, co in (("Mconv1_stage1_L1", 38), ("Mconv1_stage1_L2", 19)):
        top = rng.uniform(0.5, 2.0, (co, 1, 1, 1))
        W[name] = ((-top * rng.uniform(0.8, 1.0, (co, c_f, 7, 7))).astype(np.float32),
                   rng.standard_normal(co).astype(np.float32) * np.float32(100))
    return W


@pytest.mark.gpu
def test_accumulator_at_its_bound(tmp_path):
    spec = bound_spec()
    path = tmp_path / "bound.prototxt"
    path.write_text(synth.netspec_to_prototxt(spec))
    over = tmp_path / "bound_2689.prototxt"
    over.write_text(synth.netspec_to_prototxt(bound_spec(2689)))
    with pytest.raises(engine.PoseEngineError, match="Mconv1_stage1_L1") as ex:
        s8_engine(str(over), 64, 64, 1, 1.0)
    assert "132104" in str(ex.value)

    W = bound_weights(spec)
    rng = np.random.default_rng(2)
    dim = rng.integers(16, 48, (128, 128, 3)).astype(np.uint8)   # net input from -0.44 to -0.31
    bright = (255 - rng.integers(16, 48, (128, 128, 3))).astype(np.uint8)   # from 0.31 to 0.44
    eng = s8_engine(str(path), 64, 64, 1, 1.0)   # the frame fills the net input: no padding of value 0
    eng.set_weights(W)
    eng.calibrate([dim])
    eng.forward_frames([bright])
    eng.sync()
    rc, worst, layer = eng.range_status()
    assert rc == 5 and layer in {l["name"] for l in conv_layers(None, spec)[0]}, (rc, worst, layer)   # F saturates
    ib = IntBlobs(eng, 1, None, W, spec)
    f = ib.ints("conv4_1")
    every = np.stack(np.meshgrid([0], np.arange(8), np.arange(8), indexing="ij"), -1).reshape(-1, 3)
    for l in conv_layers(None, spec)[0]:
        w_, h_ = level_dims(64, 64, l["level"])
        pts = every if l["level"] == 3 else sample_pixels(1, h_, w_, plan_gaps(prototxt=str(path))[l["level"]], rng, 300)
        check_layer(l, ib, W, pts)   # every map value, t unrounded, bit for bit
    acc = np.concatenate([int_acc_at(ib.ints("conv4_1"), quantize(fold(W[m][0], ib.k("conv4_1")))[1], every)
                          for m in ("Mconv1_stage1_L1", "Mconv1_stage1_L2")], axis=1)
    eng.close()
    big = np.abs(acc) > 2 ** 24
    ulp = np.ldexp(1.0, np.floor(np.log2(np.where(big, np.abs(acc), 1))).astype(int) - 23)
    rounded = big & (np.mod(acc, ulp) != 0)
    print("\nK = 131712: F from %d to %d (%.0f%% at -128); largest |acc| %d = %.4f x 2^31; %d of %d sums above 2^24, %d of them not "
          "representable in fp32" % (f.min(), f.max(), 100 * np.mean(f == -128), np.abs(acc).max(), np.abs(acc).max() / 2 ** 31,
                                     int(big.sum()), acc.size, int(rounded.sum())))
    assert np.abs(acc).max() > 2 ** 30
    assert rounded.sum() >= acc.size // 2
