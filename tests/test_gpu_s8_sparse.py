"""2:4-sparse s8 layers (PE_PREC_S8X1, csrc/conv_s8_sparse.cu) on the GPU, bit for bit against the integer reference of
tests/test_gpu_s8_mode.py.

The shape rule of pe_conv_layer_sparse keeps every layer dense as built (the kernel measures slower in every class of the
shipped nets, DESIGN.md section 5), so the tests that run the kernel turn that rule off with the test hook pe_test_force_sparse
(sparse_engine); test_shape_rule_keeps_pruned_weights_dense checks the rule itself.

A sparse layer's s32 sums are the dense kernel's exact sums (the pruned weights are zeros in both), and its epilogue is the
same fp32 sequence, so every check here is the dense mode's bit-exact check with no new tolerance: check_layer per conv layer
at sampled pixels, and whole_stack (the integer chain of the whole net) against pe_fetch_maps.  The weights are He-init with
non-zero biases, magnitude-pruned to 2:4 by engine.prune_2to4.

Pixel tiles: one frame at 656x368 (COCO) or 496x368 (MPI) runs the stride-8 layers at 64 pixels per tile and the VGG layers at
128; nine frames at 320x176 run the stride-8 layers at 128.
"""
import subprocess

import numpy as np
import pytest

from caffe_rtpose_b200 import engine, synth
from test_conv_shapes import CASES, FRAMES, level_dims, write_prototxt
from test_gpu_conv_layers import checked_layers, conv_layers, frames_for, level_geo, netspec, plan_gaps, sample_pixels, weights_with_biases
from test_gpu_s8_mode import BIN, IntBlobs, check_layer, whole_stack, write_bmp
from test_gpu_s8_shapes import case_weights, s8_engine

pytestmark = pytest.mark.gpu
S8 = engine.PREC_S8X1
CONFIGS = {"coco_1": (engine.COCO_18, 656, 368, 1), "coco_9": (engine.COCO_18, 320, 176, 9),
           "mpi_1": (engine.MPI_15, 496, 368, 1), "mpi_9": (engine.MPI_15, 320, 176, 9)}


def eligible(model=None, prototxt=None):
    """The layers rules 1-3 of pe_conv_layer_sparse admit in a plain S8X1 engine: s8 arithmetic, s8 or fp32-map output, not
    reading the im2col'ed net input."""
    convs = engine.plan_formats(model, S8, None, prototxt=prototxt)["convs"]
    first_in = min(v[2] for v in convs.values())
    return sorted(n for n, (comp, out, ia, _) in convs.items() if comp == "s8" and out in ("s8", "f32") and ia != first_in)


def force_sparse(eng):
    assert engine.lib().pe_test_force_sparse(eng._h, 1) == 0
    return eng


def sparse_engine(*args, **kw):
    """A PoseEngine whose commits pick the sparse kernel for every layer rules 1-3 admit (pe_test_force_sparse)."""
    return force_sparse(engine.PoseEngine(*args, **kw))


def check_all_layers(eng, layers, W, n, net_w, net_h, gaps=None, model=None, spec=None, seed=11):
    ib = IntBlobs(eng, n, model, W, spec)
    rng = np.random.default_rng(seed)
    count = 0
    for layer in layers:
        w_, h_, gap = level_geo(net_w, net_h, layer["level"], gaps)
        count += check_layer(layer, ib, W, sample_pixels(n, h_, w_, gap, rng, 300))[0]
    return count


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_pruned_net_bit_exact(cfg):
    """Every admitted layer runs sparse, every conv layer is bit-exact, and the whole stack equals pe_fetch_maps."""
    model, net_w, net_h, n = CONFIGS[cfg]
    W = engine.prune_2to4(weights_with_biases(model), model)
    eng = sparse_engine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=S8, max_batch=n)
    eng.set_weights(W)
    assert sorted(eng.sparse_layers()) == eligible(model)
    frames = frames_for(n, 2 * net_w, 2 * net_h)
    eng.calibrate(frames[:1])
    eng.forward_frames(frames)
    count = check_all_layers(eng, checked_layers(model), W, n, net_w, net_h, model=model)
    maps = eng.fetch_maps(n).astype(np.float64)
    want = whole_stack(netspec(model), W, eng, n)
    eng.close()
    bad = maps != want
    assert not bad.any(), "%d of %d map values differ" % (int(bad.sum()), bad.size)
    print("\n%s: %d sparse layers, %d values bit-exact, whole stack exact" % (cfg, len(eligible(model)), count))


def test_unpruned_weights_run_dense():
    """He-init weights are not 2:4: no layer runs sparse, even with the shape rule lifted."""
    for model in (engine.COCO_18, engine.MPI_15):
        eng = sparse_engine(model, 160, 96, 320, 192, precision=S8)
        eng.set_weights(synth.make_weights(model, "he"))
        assert eng.sparse_layers() == []
        eng.close()


def test_shape_rule_keeps_pruned_weights_dense(tmp_path):
    """The shape rule as built: pruned weights run dense on the shipped nets and on every generated case (5x5 filters and output
    counts 1-257 included, which are not measured)."""
    for model in (engine.COCO_18, engine.MPI_15):
        eng = engine.PoseEngine(model, 160, 96, 320, 192, precision=S8)
        eng.set_weights(engine.prune_2to4(synth.make_weights(model, "he"), model))
        assert eng.sparse_layers() == []
        eng.close()
    for name in CASES:
        spec, path = write_prototxt(name, tmp_path)
        eng = s8_engine(path, CASES[name]["net_w"], CASES[name]["net_h"], 1)
        eng.set_weights(engine.prune_2to4(case_weights(name, spec), prototxt=path))
        assert eng.sparse_layers() == [], name
        eng.close()


@pytest.mark.parametrize("name", list(CASES))
def test_generated_convs_pruned_bit_exact(name, tmp_path):
    """Every generated case of test_conv_shapes.py, pruned (dead channels included), bit-exact per layer at 1 and 3 frames."""
    spec, path = write_prototxt(name, tmp_path)
    c = CASES[name]
    net_w, net_h = c["net_w"], c["net_h"]
    gaps = plan_gaps(prototxt=path)
    W = engine.prune_2to4(case_weights(name, spec), prototxt=path)
    eng = force_sparse(s8_engine(path, net_w, net_h, max(FRAMES)))
    eng.set_weights(W)
    assert sorted(eng.sparse_layers()) == eligible(prototxt=path)
    eng.calibrate(frames_for(FRAMES[0], 2 * net_w, 2 * net_h))
    layers = conv_layers(None, spec)[0]
    count = 0
    for n in FRAMES:
        eng.forward_frames(frames_for(n, 2 * net_w, 2 * net_h))
        ib = IntBlobs(eng, n, None, W, spec)
        rng = np.random.default_rng(11)
        for layer in layers:
            w_, h_ = level_dims(net_w, net_h, layer["level"])
            count += check_layer(layer, ib, W, sample_pixels(n, h_, w_, gaps[layer["level"]], rng, 300))[0]
    eng.close()
    print("\n%s pruned: %d sparse layers, %d values bit-exact" % (name, len(eligible(prototxt=path)), count))


PATTERNS = [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3), (0,), (1,), (2,), (3,), ()]


def pattern_weights(w):
    """w (co, ci, k, k), unpruned and without zeros, with ci a multiple of 4 and no Concat in front: the groups of four input
    channels cycle through every non-zero pattern (six pairs, four singles, empty) over output channels, groups and taps, so
    every group has exactly its pattern's non-zeros."""
    co, ci, k, _ = w.shape
    out = np.zeros_like(w)
    for o in range(co):
        for g in range(ci // 4):
            for t in range(k * k):
                for i in PATTERNS[(o + 3 * g + 5 * t) % len(PATTERNS)]:
                    out[o, 4 * g + i, t // k, t % k] = w[o, 4 * g + i, t // k, t % k]
    return out


def test_every_nonzero_pattern_bit_exact():
    model, net_w, net_h = engine.COCO_18, 320, 176
    full = weights_with_biases(model)
    W = engine.prune_2to4(full, model)
    name = "conv5_1_CPM_L1"   # 3x3 on conv4_4_CPM's 128 channels, no Concat in front: groups are input channels 4g..4g+3
    assert (full[name][0] != 0).all()
    W[name] = (pattern_weights(full[name][0]), full[name][1])
    eng = sparse_engine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=S8)
    eng.set_weights(W)
    assert name in eng.sparse_layers()
    frames = frames_for(1, 2 * net_w, 2 * net_h)
    eng.calibrate(frames)
    eng.forward_frames(frames)
    check_all_layers(eng, [l for l in checked_layers(model) if l["name"] == name], W, 1, net_w, net_h, model=model)
    eng.close()


def test_three_nonzeros_keep_one_layer_dense():
    """One group of one layer with three non-zeros makes that layer dense; every layer stays bit-exact."""
    model, net_w, net_h = engine.MPI_15, 320, 176
    W = engine.prune_2to4(weights_with_biases(model), model)
    name = "Mconv3_stage2_L2"
    w = W[name][0].copy()
    w[5, 0:3, 2, 4] = [0.01, -0.02, 0.03]
    W[name] = (w, W[name][1])
    eng = sparse_engine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=S8)
    eng.set_weights(W)
    assert sorted(eng.sparse_layers()) == [n for n in eligible(model) if n != name]
    frames = frames_for(1, 2 * net_w, 2 * net_h)
    eng.calibrate(frames)
    eng.forward_frames(frames)
    check_all_layers(eng, checked_layers(model), W, 1, net_w, net_h, model=model)
    eng.close()


def test_calibration_keeps_sparse_layers_and_tables_reproduce():
    """calibrate_on passes and set_calibration_table re-pack the weights and keep the same sparse layers, exact; a table saved
    from a sparse engine, applied to a fresh engine with the same weights, gives bit-identical maps."""
    model, net_w, net_h = engine.COCO_18, 320, 176
    W = engine.prune_2to4(weights_with_biases(model), model)
    frames = [synth.make_frame(40 + i, 2 * net_h, 2 * net_w) for i in range(3)]
    eng = sparse_engine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=S8, max_batch=2)
    eng.set_weights(W)
    want = eligible(model)
    eng.calibrate(frames[:1])
    eng.calibrate_on([frames[:2], frames[2:]])
    assert sorted(eng.sparse_layers()) == want
    eng.forward_frames(frames[:2])
    check_all_layers(eng, checked_layers(model), W, 2, net_w, net_h, model=model)
    maps = eng.fetch_maps(2).copy()
    table = eng.calibration_table()
    fresh = sparse_engine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=S8, max_batch=2)
    fresh.set_weights(W)
    fresh.set_calibration_table(table)
    assert sorted(fresh.sparse_layers()) == want
    fresh.forward_frames(frames[:2])
    assert np.array_equal(fresh.fetch_maps(2), maps)
    eng.set_calibration_table(table)
    assert sorted(eng.sparse_layers()) == want
    eng.forward_frames(frames[:2])
    assert np.array_equal(eng.fetch_maps(2), maps)
    eng.close()
    fresh.close()


def sparse_source(device=0):
    model, net_w, net_h = engine.COCO_18, 160, 96
    frame = synth.make_frame(5, 2 * net_h, 2 * net_w)
    e0 = sparse_engine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=S8, device=device)
    e0.set_weights(engine.prune_2to4(synth.make_weights(model, "he"), model))
    e0.calibrate([frame])
    return e0, frame, lambda dev: engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=S8, device=dev)


def same_results(engs, frame):
    res = []
    for e in engs:
        e.forward_frames([frame])
        cnt, joints, peaks = e.fetch(0)
        res.append((cnt, joints.copy(), peaks.copy(), e.fetch_maps(1).copy(), e.fetch_blob("conv4_4_CPM")[:1].copy()))
    for r in res[1:]:
        assert r[0] == res[0][0]
        for a, b in zip(r[1:], res[0][1:]):
            assert np.array_equal(a, b)


def test_share_weights_takes_sparse_layers():
    e0, frame, make = sparse_source()
    e1 = make(0)
    engine.share_weights(e0, e1)
    assert e1.sparse_layers() == e0.sparse_layers() and e0.sparse_layers()
    same_results([e0, e1], frame)
    e0.close()
    e1.close()


def test_broadcast_weights_takes_sparse_layers():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    e0, frame, make = sparse_source()
    e2 = make(1)
    engine.broadcast_weights([e0, e2])
    assert e2.sparse_layers() == e0.sparse_layers() and e0.sparse_layers()
    same_results([e0, e2], frame)
    e0.close()
    e2.close()


def test_cli_pruned_caffemodel(tmp_path):
    """rtpose.bin --precision 6 on a pruned .caffemodel logs the sparse layer count (0: the shape rule keeps every layer dense
    as built) and writes the JSON the Python path gives."""
    model, n = engine.COCO_18, 3
    W = engine.prune_2to4(synth.make_weights(model, "he", seed=3), model)
    cm = tmp_path / "w.caffemodel"
    engine.write_caffemodel(str(cm), W, synth.conv_table(model))
    imgs = tmp_path / "imgs"
    imgs.mkdir()
    frames = [synth.make_frame(100 + i, 192, 320) for i in range(n)]
    for i, f in enumerate(frames):
        write_bmp(str(imgs / ("f%03d.bmp" % i)), f)
    out, table = tmp_path / "json", tmp_path / "calib.txt"
    r = subprocess.run([BIN, "--image_dir", str(imgs), "--caffemodel", str(cm), "--model", "COCO", "--resolution", "320x192",
                        "--net_resolution", "160x96", "--no_frame_drops", "--no_display", "--precision", "6", "--write_json",
                        str(out), "--save_calibration", str(table)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    want = 0
    assert "%d of 92 conv layers run 2:4 sparse" % want in r.stderr, r.stderr[-2000:]
    eng = engine.PoseEngine(model, 160, 96, 320, 192, precision=S8)
    eng.set_weights(W)
    eng.set_calibration_table(table.read_text())   # the scales of the CLI's start-up calibration
    for i, f in enumerate(frames):
        eng.forward_frames([f])
        cnt, joints, _ = eng.fetch(0)
        assert (out / ("f%03d.json" % i)).read_text() == engine.write_json(joints[:cnt], eng.num_parts), i
    eng.close()
