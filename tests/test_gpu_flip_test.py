"""The flip test on the H100 (pe_set_flip_test): the mirrored net inputs every im2col kernel writes, the parse and the renderers on
the average of 2S copies, every input route, calibration and the CLI.  The CPU restatement of the average is flip_average
(tests/test_flip_test.py).  Everything here is bit-exact unless a comparison says otherwise."""
import os
import subprocess

import numpy as np
import pytest
import torch

from caffe_rtpose_b200 import engine, synth
from oracle import orc
from test_flip_test import _mirror_people, flip_average
from test_gpu_fast_mode import BIN, write_bmp
from test_gpu_render import compare_cpu

pytestmark = pytest.mark.gpu

START, GAP = 1.0, 0.25   # crop factors 0, 0.25, 0.5: flip_average needs scales whose start scale is exact (test_flip_test.py)
RANGED = (engine.PREC_F16X2, engine.PREC_F16X1, engine.PREC_E4M3X1, engine.PREC_S8X1)
# (precision, u8 activations, fp16 layers): every mode, S8X1 with u8 activations and a mixed engine
MODES = [(p, False, None) for p in range(7)] + [(engine.PREC_S8X1, True, None), (engine.PREC_S8X1, False, "narrow")]


def mode_id(m):
    return "p%d%s%s" % (m[0], "-u8" if m[1] else "", "-" + m[2] if m[2] else "")


def he_engine(model, net_w, net_h, S, prec=engine.PREC_F16X2, max_batch=2, u8=False, f16=None, disp=None, weights=True, **kw):
    disp_w, disp_h = disp or (2 * net_w, 2 * net_h)
    eng = engine.PoseEngine(model, net_w, net_h, disp_w, disp_h, num_scales=S, start_scale=START, scale_gap=GAP, precision=prec,
                            max_batch=max_batch, u8_activations=u8, f16_layers=f16, **kw)
    if weights:
        eng.set_weights(synth.make_weights(model, "he"))
    return eng


def frames_of(n, h, w, seed=0):
    return [synth.make_frame(seed + i, h, w) for i in range(n)]


def by_frame(maps, n, k):
    return maps.reshape((n, k) + maps.shape[1:])


def oracle_flip_parse(model, maps8_frame, net_w, net_h, disp_w, disp_h, eng):
    full = flip_average(model, maps8_frame, net_h, net_w, START, GAP)
    thr, params = orc.default_params(model)
    peaks = orc.nms(full, orc.num_parts(model), eng.max_peaks, thr)
    cnt, joints = orc.connect(model, full, peaks, disp_w, disp_h, params)
    return full, peaks, cnt, joints


def assert_parse(eng, idx, peaks, cnt, joints, tag=""):
    got_cnt, got_joints, got_peaks = eng.fetch(idx)
    assert np.array_equal(got_peaks, peaks, equal_nan=True), (tag, idx)   # portrait nets: NaN peaks, as in test_gpu_post.py
    assert got_cnt == cnt and np.array_equal(got_joints, joints), (tag, idx, got_cnt, cnt)


def test_off_means_off():
    """A handle that ran with the flip test and turned it off gives a fresh handle's maps, peaks and joints, eager and from graphs."""
    model, frames = engine.COCO_18, frames_of(2, 192, 320)
    used, fresh = he_engine(model, 160, 96, 2), he_engine(model, 160, 96, 2)
    used.set_flip_test(True)
    assert used.flip_test
    used.forward_frames(frames)
    used.fetch(0)
    used.set_flip_test(False)
    assert not used.flip_test
    for step in range(3):   # eager, captured, replayed
        out = []
        for eng in (used, fresh):
            eng.forward_frames(frames)
            out.append((eng.fetch_maps(2), [eng.fetch(i) for i in range(2)]))
        assert np.array_equal(out[0][0], out[1][0]), step
        for a, b in zip(out[0][1], out[1][1]):
            assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]), step
    used.close()
    fresh.close()


def check_mirrored_copies(eng, frames, S, net_w, net_h, ns):
    """With the flip test, frame f's maps are [the flip-off maps of f][the flip-off maps of f's planar net input reversed in x]."""
    for n in ns:
        eng.set_flip_test(False)
        eng.forward_frames(frames[:n])
        base = eng.fetch_maps(n)
        planar = np.concatenate([orc.preprocess(f, net_h, net_w, S, START, GAP) for f in frames[:n]])
        eng.forward_net_input(np.ascontiguousarray(planar[..., ::-1]))
        mirrored = eng.fetch_maps(n)
        eng.set_flip_test(True)
        for rep in range(2):   # eager, then captured
            eng.forward_frames(frames[:n])
            got = by_frame(eng.fetch_maps(n), n, 2 * S)
            assert np.array_equal(got[:, :S], by_frame(base, n, S)), (n, rep)
            assert np.array_equal(got[:, S:], by_frame(mirrored, n, S)), (n, rep)
        assert np.abs(got[:, S:]).max() > 0


@pytest.mark.parametrize("model", [engine.COCO_18, engine.MPI_15])
@pytest.mark.parametrize("mode", MODES, ids=mode_id)
def test_mirrored_copies(mode, model):
    prec, u8, f16 = mode
    frames = frames_of(2, 192, 320, seed=5)
    for S in (1, 3):
        eng = he_engine(model, 160, 96, S, prec, max_batch=2, u8=u8, f16=f16)
        if prec in RANGED:
            eng.calibrate(frames[:1])
        check_mirrored_copies(eng, frames, S, 160, 96, (1, 2))
        eng.close()


@pytest.mark.parametrize("prec", [engine.PREC_F16X2, engine.PREC_S8X1])
def test_mirrored_copies_c2(prec):
    """The benchmark's workload: COCO 656x368, one scale, nine 1280x720 frames per forward."""
    frames = frames_of(9, 720, 1280, seed=40)
    eng = he_engine(engine.COCO_18, 656, 368, 1, prec, max_batch=9, disp=(1280, 720))
    if prec in RANGED:
        eng.calibrate(frames[:1])
    check_mirrored_copies(eng, frames, 1, 656, 368, (9,))
    eng.close()


# (model, net_w, net_h, S, people per frame): the parse tests' shapes that admit START / GAP, including a net narrower than a
# tile, a portrait net and a batch of frames with different person counts
PARSE_CASES = [
    (engine.COCO_18, 320, 176, 1, (8,)), (engine.MPI_15, 240, 176, 2, (5,)), (engine.COCO_18, 320, 176, 3, (6, 3)),
    (engine.COCO_18, 656, 368, 1, (24,)), (engine.MPI_15, 496, 368, 3, (12,)), (engine.COCO_18, 48, 48, 2, (2,)),
    (engine.COCO_18, 368, 656, 3, (12,)),
]


def flip_scene(model, net_w, net_h, S, n_people, seed):
    """2S stride-8 copies of one frame: a scene at S scales, then the mirrored scene at S scales, as a net would see them."""
    people = synth.make_people(model, n_people, net_w, net_h, seed=seed, drop_prob=0.15)
    maps = synth.make_maps(model, people, net_w, net_h, num_scales=S, start_scale=START, scale_gap=GAP, seed=seed)
    mirrored = synth.make_maps(model, _mirror_people(model, people, net_w - 1), net_w, net_h, num_scales=S, start_scale=START,
                               scale_gap=GAP, seed=seed + 100)
    return np.concatenate([maps, mirrored])


@pytest.mark.parametrize("model,net_w,net_h,S,counts", PARSE_CASES, ids=["-".join(map(str, c[:4])) for c in PARSE_CASES])
def test_parse_bit_exact(model, net_w, net_h, S, counts):
    """Map injection of n x 2S maps: peaks and joints equal orc.nms / orc.connect on the CPU flip average, at the default and at a
    lowered NMS threshold."""
    disp_w, disp_h = 2 * net_w, 2 * net_h
    eng = he_engine(model, net_w, net_h, S, engine.PREC_FP32_SIMT, max_batch=len(counts), weights=False, flip_test=True)
    scenes = [flip_scene(model, net_w, net_h, S, c, seed) for seed, c in enumerate(counts, 1)]
    thr0, params = orc.default_params(model)
    for thr in (thr0, thr0 / 4):
        eng.nms_layer.SetThreshold(thr)
        eng.forward_maps(np.concatenate(scenes))
        for i, sc in enumerate(scenes):
            full = flip_average(model, sc, net_h, net_w, START, GAP)
            peaks = orc.nms(full, orc.num_parts(model), eng.max_peaks, thr)
            cnt, joints = orc.connect(model, full, peaks, disp_w, disp_h, params)
            if thr == thr0 and net_w >= 240:
                assert cnt >= 1
            assert_parse(eng, i, peaks, cnt, joints, thr)
    with pytest.raises(ValueError):
        eng.forward_maps(np.concatenate(scenes)[:-1])   # not a whole number of frames of 2S copies
    eng.close()


def test_every_route_parses_its_own_maps():
    """For every input route, the peaks and joints of a flip-test forward are the CPU flip parse of the maps the engine fetched."""
    model, net_w, net_h, S, n = engine.COCO_18, 160, 96, 2, 2
    disp_w, disp_h = 2 * net_w, 2 * net_h
    eng = he_engine(model, net_w, net_h, S, engine.PREC_F16X2, max_batch=n, flip_test=True)
    frames = frames_of(n, disp_h, disp_w, seed=60)
    odd = frames_of(n, 250, 410, seed=70)
    dev = torch.from_numpy(np.stack(frames)).cuda()
    torch.cuda.synchronize()
    routes = {
        "frames": lambda: eng.forward_frames(frames),
        "frames_device": lambda: eng.forward_frames_device(dev.data_ptr(), n),
        "camera_frames": lambda: eng.forward_camera_frames(odd),
        "pixels_rgb": lambda: eng.forward_pixels([np.ascontiguousarray(f[..., ::-1]) for f in odd], engine.PIX_RGB),
        "jpeg_coefs": lambda: eng.forward_jpeg([engine.encode_jpeg(f) for f in frames], entropy="host"),
        "jpeg_scans": lambda: eng.forward_jpeg([engine.encode_jpeg(f) for f in odd], entropy="gpu"),
        "net_input": lambda: eng.forward_net_input(np.concatenate([orc.preprocess(f, net_h, net_w, S, START, GAP) for f in frames])),
    }
    for name, fwd in routes.items():
        fwd()
        maps = by_frame(eng.fetch_maps(n), n, 2 * S)
        assert np.abs(maps[:, S:]).max() > 0, name
        for i in range(n):
            _, peaks, cnt, joints = oracle_flip_parse(model, maps[i], net_w, net_h, disp_w, disp_h, eng)
            assert_parse(eng, i, peaks, cnt, joints, name)
    eng.close()


@pytest.mark.parametrize("S", [1, 2])
def test_render_views(S):
    """The skeleton, one part, all parts, all PAFs and one PAF with the flip test: orc.render on the CPU flip average, within the
    render tests' tolerance (compare_cpu)."""
    model, net_w, net_h = engine.COCO_18, 320, 176
    disp_w, disp_h = 2 * net_w, 2 * net_h
    eng = he_engine(model, net_w, net_h, S, engine.PREC_FP32_SIMT, max_batch=1, weights=False, flip_test=True)
    sc = flip_scene(model, net_w, net_h, S, 7, seed=21)
    eng.forward_maps(sc)
    full, _, cnt, joints = oracle_flip_parse(model, sc, net_w, net_h, disp_w, disp_h, eng)
    assert cnt >= 3
    frame = synth.make_frame(21, disp_h, disp_w)
    canvas0 = orc.canvas_from_u8(frame)
    for part in (0, 1, 19, 20, 21, 39):
        img, canvas = eng.render(0, part, False, display_bgr=frame, want_canvas=True)
        compare_cpu("flip S%d p%d" % (S, part), canvas, img, orc.render(model, canvas0, net_w, net_h, full, joints, cnt, part, False))
    eng.close()


def test_calibration_tables_and_sharing():
    """A collection pass with the flip test on works, and counts the mirrored copies; a calibration table applies whether the flip
    test is on or off; a handle with the flip test runs on weights shared by one without it."""
    model, frames = engine.COCO_18, frames_of(2, 192, 320, seed=80)
    src = he_engine(model, 160, 96, 1, engine.PREC_S8X1)
    src.calibrate(frames[:1])
    table = src.calibration_table()
    src.set_flip_test(True)
    src.calibrate_begin()
    with pytest.raises(engine.PoseEngineError, match="collection"):
        src.set_flip_test(False)
    src.forward_frames(frames)
    src.sync()
    src.calibrate_end()
    assert src.flip_test
    src.calibrate(frames[:1])   # pe_calibrate with the flip test on: the ranges of both copies
    flipped_table = src.calibration_table()
    src.set_flip_test(False)
    src.set_calibration_table(table)
    src.forward_frames(frames)
    want = src.fetch_maps(2)
    other = he_engine(model, 160, 96, 1, engine.PREC_S8X1, flip_test=True)
    other.set_calibration_table(table)   # a table of a flip-off handle on a flip-on handle, and back
    other.forward_frames(frames)
    assert np.array_equal(by_frame(other.fetch_maps(2), 2, 2)[:, 0], by_frame(want, 2, 1)[:, 0])
    src.set_calibration_table(flipped_table)
    src.set_flip_test(True)
    other.set_calibration_table(flipped_table)
    for e in (src, other):
        e.forward_frames(frames)
    assert np.array_equal(src.fetch_maps(2), other.fetch_maps(2))
    # sharing: a flip-test handle on the packed weights of a handle without it, and the other way round
    src.set_flip_test(False)
    src.set_calibration_table(table)
    for flip in (True, False):
        dst = he_engine(model, 160, 96, 1, engine.PREC_S8X1, weights=False, flip_test=flip)
        engine.share_weights(src, dst)
        dst.forward_frames(frames)
        src.forward_frames(frames)
        got, ref = dst.fetch_maps(2), src.fetch_maps(2)
        assert np.array_equal(by_frame(got, 2, 2 if flip else 1)[:, 0], by_frame(ref, 2, 1)[:, 0]), flip
        dst.close()
    for e in (src, other):
        e.close()


def test_fetch_blob_and_state():
    """pe_fetch_blob returns 2 x n x S images with the flip test, each frame's mirrored net inputs its inputs reversed in x; turning
    the flip test on drops the last forward's results."""
    model, frames, S = engine.COCO_18, frames_of(2, 192, 320, seed=90), 2
    eng = he_engine(model, 160, 96, S, engine.PREC_F16X2)
    eng.forward_frames(frames)
    base = eng.fetch_blob("image")
    eng.set_flip_test(True)
    with pytest.raises(engine.PoseEngineError):
        eng.fetch(0)   # the results of the forward before the switch are gone
    eng.forward_frames(frames)
    blob = by_frame(eng.fetch_blob("image"), 2, 2 * S)
    assert np.array_equal(blob[:, :S], by_frame(base, 2, S))
    assert np.array_equal(blob[:, S:], blob[:, :S][..., ::-1])
    assert np.array_equal(by_frame(base, 2, S)[0], orc.preprocess(frames[0], 96, 160, S, START, GAP))
    eng.close()


def test_cli_flip_test_json(tmp_path):
    """rtpose.bin --flip_test writes the JSON of PoseEngine(..., flip_test=True) on the same frames and weights, and says so."""
    model, n = engine.COCO_18, 6
    W = synth.make_weights(model, "he", seed=3)
    cm = tmp_path / "w.caffemodel"
    engine.write_caffemodel(str(cm), W, synth.conv_table(model))
    imgs = tmp_path / "imgs"
    imgs.mkdir()
    frames = [synth.make_frame(200 + i, 192, 320) for i in range(n)]
    for i, f in enumerate(frames):
        write_bmp(str(imgs / ("f%03d.bmp" % i)), f)
    out = tmp_path / "json"
    r = subprocess.run([BIN, "--image_dir", str(imgs), "--caffemodel", str(cm), "--model", "COCO", "--resolution", "320x192",
                        "--net_resolution", "160x96", "--no_frame_drops", "--no_display", "--precision", "4", "--calibrate_range=false",
                        "--flip_test", "--write_json", str(out)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "flip test on" in r.stderr, r.stderr[-2000:]
    eng = engine.PoseEngine(model, 160, 96, 320, 192, precision=engine.PREC_F16X1, flip_test=True)
    eng.set_weights(W)
    for i, f in enumerate(frames):
        eng.forward_frames([f])
        cnt, joints, _ = eng.fetch(0)
        assert (out / ("f%03d.json" % i)).read_text() == eng.json(joints), i
    eng.close()
