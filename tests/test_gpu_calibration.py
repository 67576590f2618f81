"""Calibration over a set of frames (pe_calibrate_begin / pe_calibrate_end, PoseEngine.calibrate_on) and calibration tables
(pe_calibration_get / pe_calibration_set) on the GPU, in every mode with range scales and one mixed engine, at the small net
sizes of the mode tests with He weights (zero biases).  The display size has the net's aspect ratio, so the resized frame needs
no pad: with zero biases and ReLU the net is then close to homogeneous, and a frame whose contrast is 8x lower has activations
about 8x smaller at every layer - beyond the 2-4x headroom of the INT8 target window."""
import os
import subprocess

import numpy as np
import pytest
import torch

from caffe_rtpose_b200 import engine, synth
from test_prototxt import spec_prototxt

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "caffe_rtpose_b200", "rtpose.bin")
NET_W, NET_H, DISP_W, DISP_H = 160, 96, 320, 192
# (precision, f16_layers)
MODES = {"f16x2": (engine.PREC_F16X2, None), "f16x1": (engine.PREC_F16X1, None), "e4m3x1": (engine.PREC_E4M3X1, None),
         "s8x1": (engine.PREC_S8X1, None), "s8x1_narrow": (engine.PREC_S8X1, "narrow")}


def make(mode, weights=None, model=engine.COCO_18, max_batch=1, **kw):
    prec, f16 = MODES[mode]
    eng = engine.PoseEngine(model, NET_W, NET_H, DISP_W, DISP_H, precision=prec, f16_layers=f16, max_batch=max_batch, **kw)
    eng.set_weights(weights if weights is not None else synth.make_weights(model, "he"))
    return eng


def low_contrast(h):
    return (128 + np.round((h.astype(np.float64) - 128) / 8)).astype(np.uint8)


def outputs(eng, frames):
    eng.forward_frames(frames)
    res = [eng.fetch(i) for i in range(len(frames))]
    return eng.fetch_maps(len(frames)), [r[0] for r in res], [r[1] for r in res], [r[2] for r in res]


def same_outputs(a, b):
    assert np.array_equal(a[0], b[0])
    assert a[1] == b[1]
    for x, y in zip(a[2], b[2]):
        assert np.array_equal(x, y)
    for x, y in zip(a[3], b[3]):
        assert np.array_equal(x, y)


def log2_scale(eng, blob):
    try:
        return eng.blob_log2_scale(blob)
    except engine.PoseEngineError as err:   # a layer whose top is not a blob of its own name
        return str(err)


def layers(table):
    return {l.split()[1]: (l.split()[2], int(l.split()[3])) for l in table.splitlines() if l.startswith("layer ")}


@pytest.mark.parametrize("mode", list(MODES))
def test_one_pass_after_pe_calibrate_changes_nothing(mode):
    F = synth.make_frame(3, DISP_H, DISP_W)
    eng = make(mode)
    eng.calibrate([F])
    t0 = eng.calibration_table()
    before = outputs(eng, [F])
    eng.calibrate_begin()
    eng.forward_frames([F])
    assert eng.calibrate_end() == 0
    assert eng.calibration_table() == t0
    same_outputs(outputs(eng, [F]), before)
    eng.close()


@pytest.mark.parametrize("mode", list(MODES))
def test_pe_calibrate_after_a_net_input_forward_sees_only_its_frames(mode):
    # the planar route writes the input's lo planes; the calibration forward must clear them as pe_forward_frames does
    F = synth.make_frame(6, DISP_H, DISP_W)
    ref = make(mode)
    ref.calibrate([F])
    want = ref.fetch_maps(1), ref.calibration_table()
    ref.close()
    eng = make(mode)
    eng.set_calibration_table(eng.calibration_table())   # scale 1 everywhere, as created; lets S8X1 forward
    x = np.random.default_rng(6).standard_normal((eng.cfg.num_scales, 3, NET_H, NET_W)).astype(np.float32) * 100
    eng.forward_net_input(x)
    eng.calibrate([F])
    assert np.array_equal(eng.fetch_maps(1), want[0])
    assert eng.calibration_table() == want[1]
    eng.close()


@pytest.mark.parametrize("mode", list(MODES))
def test_low_contrast_calibration_is_repaired_by_passes_over_the_set(mode):
    H = synth.make_frame(0, DISP_H, DISP_W)
    L = low_contrast(H)
    ref = make(mode)
    ref.calibrate([H])
    want = ref.calibration_table()
    ref.close()
    for order in ((L, H), (H, L)):
        eng = make(mode)
        eng.calibrate([L])
        eng.range_status()
        eng.forward_frames([H])
        eng.sync()
        rc, worst, name = eng.range_status()
        if mode in ("s8x1", "e4m3x1"):   # the busy frame saturates a layer calibrated on the quiet one
            assert rc == 5 and worst >= 1.0, (rc, worst, name)
        passes = eng.calibrate_on([[f] for f in order])
        print("%s order %s: %d passes" % (mode, "LH" if order[0] is L else "HL", passes))
        got = eng.calibration_table()
        assert got == want   # L's maxima stay below H's at every layer: the set's table is H's
        eng.forward_frames([L])
        eng.forward_frames([H])
        eng.sync()
        assert eng.range_status()[0] == 0
        # one more pass changes nothing: every layer's largest stored value over {L, H} lies in its kind's target window
        eng.calibrate_begin()
        eng.forward_frames([L])
        eng.forward_frames([H])
        assert eng.calibrate_end() == 0
        eng.close()


def test_every_input_route_collects_the_same():
    frames = [synth.make_frame(10 + i, DISP_H, DISP_W) for i in range(3)]
    tables = []
    for route in ("frames", "pixels_rgb", "pixels_bgr_device"):
        eng = make("s8x1")
        eng.calibrate([frames[0]])
        for _ in range(len(layers(eng.calibration_table()))):
            eng.calibrate_begin()
            for f in frames:
                if route == "frames":
                    eng.forward_frames([f])
                elif route == "pixels_rgb":
                    eng.forward_pixels([np.ascontiguousarray(f[:, :, ::-1])], engine.PIX_RGB)
                else:
                    eng.forward_pixels([torch.from_numpy(f).cuda()], engine.PIX_BGR)
                eng.sync()
            if eng.calibrate_end() == 0:
                break
        tables.append(eng.calibration_table())
        eng.close()
    assert tables[0] == tables[1] == tables[2]


@pytest.mark.parametrize("mode", list(MODES))
def test_a_table_reproduces_the_engine(mode):
    W = synth.make_weights(engine.COCO_18, "he")
    cal = [synth.make_frame(20 + i, DISP_H, DISP_W) for i in range(2)]
    held = [synth.make_frame(40 + i, DISP_H, DISP_W) for i in range(2)]
    a = make(mode, W, max_batch=2)
    a.calibrate([cal[0]])
    a.calibrate_on([[low_contrast(cal[1])], cal])
    text = a.calibration_table()
    b = make(mode, W, max_batch=2)
    b.set_calibration_table(text)
    assert b.calibration_table() == text
    want = outputs(a, held)
    same_outputs(outputs(b, held), want)
    for name, *_ in a.conv_layers():
        assert log2_scale(b, name) == log2_scale(a, name), name
    c = engine.PoseEngine(engine.COCO_18, NET_W, NET_H, DISP_W, DISP_H, precision=MODES[mode][0], f16_layers=MODES[mode][1], max_batch=2)
    engine.share_weights(b, c)
    same_outputs(outputs(c, held), want)
    if torch.cuda.device_count() > 1:   # and across pe_broadcast_weights
        d = engine.PoseEngine(engine.COCO_18, NET_W, NET_H, DISP_W, DISP_H, precision=MODES[mode][0], f16_layers=MODES[mode][1], max_batch=2,
                              device=1)
        engine.broadcast_weights([b, d])
        same_outputs(outputs(d, held), want)
        d.close()
    for e in (a, b, c):
        e.close()


def test_refusals(tmp_path):
    F = synth.make_frame(5, DISP_H, DISP_W)
    a = make("s8x1")
    a.calibrate([F])
    text = a.calibration_table()

    def refused(eng, t, msg, code=1):
        with pytest.raises(engine.PoseEngineError, match=msg) as ei:
            eng.set_calibration_table(t)
        assert "error %d:" % code in str(ei.value)
    other = make("s8x1", synth.make_weights(engine.COCO_18, "he", seed=7))
    refused(other, text, "calibrated with other weights")
    narrow = make("s8x1_narrow")
    refused(narrow, text, "stores s8 in the table, f16 in the engine")
    mpi = make("s8x1", model=engine.MPI_15)
    refused(mpi, text, "unknown layer|out of order|missing|other weights")
    _, path = spec_prototxt("mpi_2", tmp_path)
    two = engine.PoseEngine(None, NET_W, NET_H, DISP_W, DISP_H, precision=engine.PREC_S8X1, prototxt=path)
    two.set_weights(synth.make_weights(engine.MPI_15, "he", stages=2))
    mpi.calibrate([F])
    refused(two, mpi.calibration_table(), "other weights|unknown layer|missing")
    refused(a, text.replace("precision 6", "precision 5"), "precision 5")
    # a receiving handle, and an owner whose weights are already shared
    recv = engine.PoseEngine(engine.COCO_18, NET_W, NET_H, DISP_W, DISP_H, precision=engine.PREC_S8X1)
    engine.share_weights(a, recv)
    for eng in (recv, a):
        refused(eng, text, "broadcast / sharing|shares its weights", code=3)
        for call in (eng.calibrate_begin, eng.calibrate_end):
            with pytest.raises(engine.PoseEngineError, match="error 3:"):
                call()
    # pe_calibrate on the owner would re-pack the buffer recv runs on while recv keeps the old scales
    with pytest.raises(engine.PoseEngineError, match="error 3:.*shares its weights"):
        a.calibrate([F])
    # modes without range scales
    for prec in (engine.PREC_FP32_SIMT, engine.PREC_BF16X1, engine.PREC_BF16X3):
        e = engine.PoseEngine(engine.COCO_18, NET_W, NET_H, DISP_W, DISP_H, precision=prec)
        e.set_weights(synth.make_weights(engine.COCO_18, "he"))
        for call in (e.calibrate_begin, lambda: e.calibrate_end(), e.calibration_table, lambda: e.set_calibration_table(text)):
            with pytest.raises(engine.PoseEngineError, match="error 1:.*no range scales"):
                call()
        e.close()
    # end without a forward; pe_calibrate, a table and pe_commit_weights during a collection
    e = make("e4m3x1")
    with pytest.raises(engine.PoseEngineError, match="error 3:.*pe_calibrate_begin has not been called"):
        e.calibrate_end()
    e.calibrate_begin()
    with pytest.raises(engine.PoseEngineError, match="error 3:.*no forward since pe_calibrate_begin"):
        e.calibrate_end()
    for call in (lambda: e.calibrate([F]), lambda: e.set_calibration_table(e.calibration_table()), e.commit_weights):
        with pytest.raises(engine.PoseEngineError, match="error 3:.*collection"):
            call()
    e.forward_frames([F])
    e.range_status()   # reading the range state during a collection loses nothing
    assert e.calibrate_end() > 0
    e.close()
    # INT8 begin before any calibration
    s = make("s8x1")
    with pytest.raises(engine.PoseEngineError, match="error 3:.*pe_calibrate or pe_calibration_set"):
        s.calibrate_begin()
    s.set_calibration_table(text)   # replaces the pe_calibrate the first forward requires
    s.forward_frames([F])
    s.fetch(0)
    for e in (s, a, other, narrow, mpi, two, recv):
        e.close()


def test_cli_calibration_dir_and_table(tmp_path):
    W = synth.make_weights(engine.COCO_18, "he", seed=3)
    cm = tmp_path / "w.caffemodel"
    engine.write_caffemodel(str(cm), W, synth.conv_table(engine.COCO_18))
    imgs, cal = tmp_path / "imgs", tmp_path / "cal"
    imgs.mkdir()
    cal.mkdir()
    for i in range(4):
        (imgs / ("f%03d.jpg" % i)).write_bytes(engine.encode_jpeg(synth.make_frame(100 + i, DISP_H, DISP_W)))
    sizes = [(DISP_W, DISP_H), (DISP_W, DISP_H), (400, 240), (256, 256), (256, 256), (DISP_W, DISP_H)]
    for i, (w, h) in enumerate(sizes):
        f = synth.make_frame(200 + i, h, w)
        (cal / ("c%03d.jpg" % i)).write_bytes(engine.encode_jpeg(low_contrast(f) if i % 2 else f))
    common = [BIN, "--image_dir", str(imgs), "--caffemodel", str(cm), "--model", "COCO", "--resolution", "%dx%d" % (DISP_W, DISP_H),
              "--net_resolution", "%dx%d" % (NET_W, NET_H), "--no_frame_drops", "--no_display", "--precision", "6", "--batch", "2"]
    t0, t, j1, j2 = tmp_path / "t0.txt", tmp_path / "t.txt", tmp_path / "j1", tmp_path / "j2"
    r = subprocess.run(common + ["--save_calibration", str(t0), "--write_json", str(tmp_path / "j0")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    r = subprocess.run(common + ["--calibration_dir", str(cal), "--save_calibration", str(t), "--write_json", str(j1)], capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    print("\n" + "\n".join(l for l in r.stderr.splitlines() if "calibration pass" in l))
    r = subprocess.run(common + ["--calibration_table", str(t), "--write_json", str(j2)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "calibration table" in r.stderr
    for i in range(4):
        a, b = [(o / ("f%03d.json" % i)).read_text() for o in (j1, j2)]
        assert a == b and a.startswith("{")
    # the same passes in Python, from the same synthetic-frame calibration, on the same decoded frames, in the same batches
    eng = make("s8x1", W, max_batch=2)
    eng.set_calibration_table(t0.read_text())
    dec = [engine.decode_jpeg((cal / ("c%03d.jpg" % i)).read_bytes()) for i in range(len(sizes))]
    batches = []
    for f in dec:
        if batches and batches[-1][0].shape == f.shape and len(batches[-1]) < 2:
            batches[-1].append(f)
        else:
            batches.append([f])
    passes = eng.calibrate_on(batches)
    assert eng.calibration_table() == t.read_text()
    print("calibrate_on: %d passes" % passes)
    eng.close()
