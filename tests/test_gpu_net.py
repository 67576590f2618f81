"""GPU parity of preprocess + the convolution stack (SIMT fp32 and wgmma split-precision) + the end-to-end
frame path, through the C ABI, against the oracle (Caffe CPU arithmetic)."""
import numpy as np
import pytest

from caffe_rtpose_b200 import engine, synth
from oracle import orc

pytestmark = pytest.mark.gpu

# max |engine - oracle| / max |oracle| on the stride-8 maps.  fp32 reorders sums (BLAS vs GPU): ~5e-6.
# bf16x2: operands carry 16 significand bits and the tensor core accumulates in truncated fp32: ~2e-4.
# bf16x3 (three bf16 planes, hi*hi chunked as in the parity mode) and bf16x1 (the non-parity "fast" mode) are only
# sanity-checked here; tests/test_gpu_conv_layers.py holds every layer of every mode to its float64 error bound.
# measured on H100 (smoke(), 160x96): SIMT 4.1e-6, parity mode 8.7e-6
# (the parity-mode bound is about 3x the measured value)
TOL = {engine.PREC_FP32_SIMT: 5e-5, engine.PREC_BF16X2: 3e-5, engine.PREC_BF16X3: 1e-3, engine.PREC_BF16X1: 6e-2}


def rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


@pytest.fixture(scope="module")
def small():
    model, net_w, net_h = engine.COCO_18, 160, 96
    W = synth.make_weights(model, "he")
    onet = orc.Net(model)
    onet.set_weights(W)
    frames = [synth.make_frame(i, 192, 320) for i in range(2)]
    x = [orc.preprocess(f, net_h, net_w, 1, 1.0, 0.3) for f in frames]
    omaps = [onet.forward(xi) for xi in x]
    return dict(model=model, net_w=net_w, net_h=net_h, W=W, onet=onet, frames=frames, x=x, omaps=omaps)


def test_preprocess_net_taller_than_display():
    """C5-style geometry (992x736 net from 1280x720 frames): the y axis enlarges, so cv::resize(INTER_AREA) is OpenCV's
    fixed-point bilinear area mode for scale 1.0 and the area decimation for the smaller scales."""
    net_w, net_h, disp_w, disp_h, S = 496, 368, 640, 360, 2
    eng = engine.PoseEngine(engine.COCO_18, net_w, net_h, disp_w, disp_h, num_scales=S, start_scale=1.0, scale_gap=0.15,
                            precision=engine.PREC_FP32_SIMT)
    eng.set_weights(synth.make_weights(engine.COCO_18, "caffe"))
    f = synth.make_frame(9, disp_h, disp_w)
    eng.forward_frames([f])
    assert np.array_equal(eng.fetch_blob("image")[:S], orc.preprocess(f, net_h, net_w, S, 1.0, 0.15))
    eng.close()


@pytest.mark.parametrize("S,start,gap", [(1, 1.0, 0.3), (3, 1.0, 0.15)])
def test_preprocess_bit_exact(S, start, gap):
    net_w, net_h, disp_w, disp_h = 320, 176, 640, 360
    eng = engine.PoseEngine(engine.COCO_18, net_w, net_h, disp_w, disp_h, num_scales=S, start_scale=start, scale_gap=gap,
                            precision=engine.PREC_FP32_SIMT, max_batch=2)
    eng.set_weights(synth.make_weights(engine.COCO_18, "caffe"))
    frames = [synth.make_frame(7, disp_h, disp_w), synth.make_frame(8, disp_h, disp_w)]
    eng.forward_frames(frames)
    img = eng.fetch_blob("image")
    for i, f in enumerate(frames):
        assert np.array_equal(img[i * S:(i + 1) * S], orc.preprocess(f, net_h, net_w, S, start, gap))
    eng.close()


@pytest.mark.parametrize("prec", [engine.PREC_FP32_SIMT, engine.PREC_BF16X2, engine.PREC_BF16X3, engine.PREC_BF16X1])
def test_conv_stack_vs_oracle(small, prec):
    s = small
    eng = engine.PoseEngine(s["model"], s["net_w"], s["net_h"], 320, 192, precision=prec, max_batch=2)
    eng.set_weights(s["W"])
    eng.forward_frames(s["frames"])
    maps = eng.fetch_maps(2)
    for i in range(2):
        assert rel(maps[i:i + 1], s["omaps"][i]) < TOL[prec]
    # same result through the reference's own upload path (planar fp32 net input, rtpose.cpp:1131-1133)
    eng.forward_net_input(np.concatenate(s["x"]))
    maps2 = eng.fetch_maps(2)
    assert rel(maps2, maps) < (1e-6 if prec == engine.PREC_FP32_SIMT else TOL[prec])
    eng.close()


@pytest.mark.parametrize("prec", [engine.PREC_FP32_SIMT, engine.PREC_BF16X2])
def test_layerwise_blobs(small, prec):
    s = small
    eng = engine.PoseEngine(s["model"], s["net_w"], s["net_h"], 320, 192, precision=prec)
    eng.set_weights(s["W"])
    eng.forward_frames(s["frames"][:1])
    for blob in ["conv1_1", "conv1_2", "pool1_stage1", "conv2_2", "pool2_stage1", "conv3_4", "pool3_stage1", "conv4_2",
                 "conv4_4_CPM", "conv5_3_CPM_L1", "conv5_4_CPM_L2", "Mconv1_stage2_L1", "Mconv5_stage4_L2", "Mconv6_stage6_L1"]:
        got = eng.fetch_blob(blob)[:1]
        ref = s["onet"].forward_blob(s["x"][0], blob, got.shape[1:])
        assert rel(got, ref) < TOL[prec], blob
    eng.close()


def test_mpi_model_and_multiscale():
    model, net_w, net_h, S = engine.MPI_15, 160, 96, 2
    W = synth.make_weights(model, "he", seed=7)
    onet = orc.Net(model)
    onet.set_weights(W)
    frame = synth.make_frame(3, 192, 320)
    x = orc.preprocess(frame, net_h, net_w, S, 1.0, 0.25)
    omaps = onet.forward(x)
    for prec in (engine.PREC_FP32_SIMT, engine.PREC_BF16X2):
        eng = engine.PoseEngine(model, net_w, net_h, 320, 192, num_scales=S, start_scale=1.0, scale_gap=0.25, precision=prec)
        eng.set_weights(W)
        eng.forward_frames([frame])
        assert rel(eng.fetch_maps(1), omaps) < TOL[prec]
        eng.close()


def match_peaks(pk, opk, full, thr, eps):
    """Peak lists must agree except where the oracle's decision margin is below eps (fp reorder noise):
    every oracle peak with margin > eps is found (<= 2e-3 px, |score| <= eps) and vice versa."""
    P = pk.shape[0]
    bad = 0
    for p in range(P):
        a = pk[p, 1:1 + int(min(pk[p, 0, 0], pk.shape[1] - 1))]
        b = opk[p, 1:1 + int(min(opk[p, 0, 0], opk.shape[1] - 1))]
        for src, dst in ((a, b), (b, a)):
            for (x, y, s) in src:
                if len(dst) and np.min(np.hypot(dst[:, 0] - x, dst[:, 1] - y)) < 2e-3:
                    continue
                xi, yi = int(round(x)), int(round(y))
                win = full[p, max(yi - 4, 0):yi + 5, max(xi - 4, 0):xi + 5]
                top2 = np.sort(win.ravel())[-2:]
                margin = min(abs(s - thr), top2[1] - top2[0])
                if margin > eps:
                    bad += 1
    return bad


@pytest.mark.parametrize("prec", [engine.PREC_FP32_SIMT, engine.PREC_BF16X2])
def test_end_to_end_frame(small, prec):
    """uint8 frame -> joints through the public call, He-init weights (noise maps: many peaks, rarely a person)."""
    s = small
    eng = engine.PoseEngine(s["model"], s["net_w"], s["net_h"], 320, 192, precision=prec)
    eng.set_weights(s["W"])
    eng.nms_layer.SetThreshold(0.6)
    eng.forward_frames(s["frames"][:1])
    cnt, joints, peaks = eng.fetch(0)
    thr, p = orc.default_params(s["model"])
    ocnt, oj, opk, omaps = s["onet"].process_frame(s["frames"][0], s["net_h"], s["net_w"], nms_threshold=0.6)
    full = orc.imresize(omaps, s["net_h"], s["net_w"], 1.0, 0.3)
    eps = 20 * TOL[prec] * float(np.abs(omaps).max())
    assert match_peaks(peaks, opk, full, 0.6, eps) == 0
    assert abs(int(peaks[:, 0, 0].sum()) - int(opk[:, 0, 0].sum())) <= 0.02 * opk[:, 0, 0].sum() + 2
    assert cnt == ocnt
    eng.close()


def test_errors_are_reported_not_fatal():
    with pytest.raises(engine.PoseEngineError, match="multiples of 8"):
        engine.PoseEngine(engine.COCO_18, 100, 50, 320, 192)
    with pytest.raises(engine.PoseEngineError, match="CHECK_LE"):
        engine.PoseEngine(engine.COCO_18, 328, 184, 656, 368)
    eng = engine.PoseEngine(engine.COCO_18, 160, 96, 320, 192, precision=engine.PREC_FP32_SIMT)
    with pytest.raises(engine.PoseEngineError, match="never set|commit"):
        eng.forward_frames([synth.make_frame(0, 192, 320)])
    with pytest.raises(engine.PoseEngineError, match="expected"):
        eng.set_weights({"conv1_1": (np.zeros((64, 3, 5, 5), np.float32), np.zeros(64, np.float32))}, commit=False)
    eng.close()


def test_load_caffemodel_equals_set_weights(small, tmp_path):
    """Net::CopyTrainedLayersFrom path: a .caffemodel written in the reference's wire format loads to the same net."""
    s = small
    p = str(tmp_path / "he.caffemodel")
    engine.write_caffemodel(p, s["W"], synth.conv_table(s["model"]))
    eng = engine.PoseEngine(s["model"], s["net_w"], s["net_h"], 320, 192, precision=engine.PREC_BF16X2)
    eng.load_caffemodel(p)
    eng.forward_frames(s["frames"][:1])
    maps = eng.fetch_maps(1)
    eng.set_weights(s["W"])
    eng.forward_frames(s["frames"][:1])
    assert np.array_equal(maps, eng.fetch_maps(1))
    # shape mismatch is fatal in the reference (net.cpp:770-786) and an error here
    bad = dict(s["W"])
    bad["conv1_2"] = (np.zeros((64, 64, 1, 1), np.float32), np.zeros(64, np.float32))
    tbl = [(n, co, ci, (1 if n == "conv1_2" else k)) for n, co, ci, k in synth.conv_table(s["model"])]
    engine.write_caffemodel(p, bad, tbl)
    with pytest.raises(engine.PoseEngineError):
        eng.load_caffemodel(p)
    eng.close()


@pytest.mark.parametrize("prec", [engine.PREC_FP32_SIMT, engine.PREC_BF16X2])
def test_joint_coordinates_within_1e3_px(small, prec):
    """north_star bar: joint coordinates within 1e-3 px and identical person/limb assignment.  He-init noise at the
    default thresholds yields a dozen spurious "people"; wherever the assignment pattern agrees (it does unless a peak
    sits on a decision boundary) the coordinates must agree to 1e-3 net px."""
    s = small
    eng = engine.PoseEngine(s["model"], s["net_w"], s["net_h"], 320, 192, precision=prec)
    eng.set_weights(s["W"])
    eng.forward_frames(s["frames"][:1])
    cnt, joints, peaks = eng.fetch(0)
    ocnt, oj, opk, _ = s["onet"].process_frame(s["frames"][0], s["net_h"], s["net_w"])
    eng.close()
    assert ocnt >= 5
    assert cnt == ocnt
    assert np.array_equal(joints[:, :, 2] > 0, oj[:, :, 2] > 0)          # identical part -> person assignment
    scale = 320.0 / s["net_w"]                                            # joints are reported in display pixels
    assert np.abs(joints[:, :, :2] - oj[:, :, :2]).max() / scale < 1e-3
    assert np.abs(joints[:, :, 2] - oj[:, :, 2]).max() < 20 * TOL[prec]


@pytest.mark.parametrize("sh,sw", [(270, 480), (150, 200), (192, 320), (400, 360)])
def test_camera_frames_warp_affine_bit_exact(sh, sw):
    """Frames of any size: the display image (warpAffine INTER_CUBIC, rtpose.cpp:474-487) and then the net input must equal
    the oracle's (OpenCV fixed-point arithmetic restated, pinned to cv2) bit for bit; frame.scale feeds the JSON."""
    net_w, net_h, disp_w, disp_h = 160, 96, 320, 192
    eng = engine.PoseEngine(engine.COCO_18, net_w, net_h, disp_w, disp_h, precision=engine.PREC_FP32_SIMT, max_batch=2)
    eng.set_weights(synth.make_weights(engine.COCO_18, "caffe"))
    frames = [synth.make_frame(31, sh, sw), synth.make_frame(32, sh, sw)]
    s = eng.forward_camera_frames(frames)
    img = eng.fetch_blob("image")
    for i, f in enumerate(frames):
        disp, os_ = orc.display_image(f, disp_w, disp_h)
        assert s == os_
        assert np.array_equal(img[i:i + 1], orc.preprocess(disp, net_h, net_w, 1, 1.0, 0.3))
    eng.close()


def test_load_caffemodel_serialised_by_google_protobuf(small, tmp_path):
    """Net::CopyTrainedLayersFrom on a complete .caffemodel that this repo's writer never touched: Google's protobuf runtime
    serialises all 92 layers (descriptors of tools/gen_caffemodel_fixture.py, V2 `layer` blocks with the fields a Caffe snapshot
    carries); the loaded net must equal the one fed through pe_set_conv_weights bit for bit."""
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location("gen_cm", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                                         "tools", "gen_caffemodel_fixture.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    s = small
    Net = gen.build("caffe_full", True)
    net = Net()
    net.name = "COCO_pose_deploy"
    for name, co, ci, k in synth.conv_table(s["model"]):
        l = net.layer.add()
        l.name, l.type, l.phase = name, "Convolution", 1
        l.bottom.append("b"); l.top.append(name)
        l.convolution_param.num_output = co
        w, b = s["W"][name]
        for arr in (w, b):
            blob = l.blobs.add()
            blob.shape.dim.extend(arr.shape)
            blob.data.extend(arr.ravel().tolist())
        r = net.layer.add()
        r.name, r.type = "relu_" + name, "ReLU"
    p = str(tmp_path / "pb.caffemodel")
    open(p, "wb").write(net.SerializeToString())
    eng = engine.PoseEngine(s["model"], s["net_w"], s["net_h"], 320, 192, precision=engine.PREC_BF16X2)
    eng.load_caffemodel(p)
    eng.forward_frames(s["frames"][:1])
    maps = eng.fetch_maps(1)
    eng.set_weights(s["W"])
    eng.forward_frames(s["frames"][:1])
    assert np.array_equal(maps, eng.fetch_maps(1))
    eng.close()
