"""The 16-bit integer mode (PE_PREC_S8X2: two s8 planes of activations and weights, three s8 MMAs per MAC, exact s32 sums) on
the GPU.

Every layer is a deterministic function of integers followed by fixed fp32 operations (poseengine.h), so it is checked bit for
bit, as tests/test_gpu_s8_mode.py does for S8X1.  A layer's input integers v are pe_fetch_blob of its bottom times 2^k
(pe_blob_log2_scale), split into hi = (v + 128) >> 8 and lo = v - 256 hi.  The reference folds 2^-k of every input channel into
the fp32 weights (exact), quantises each output channel as the packer does (sigma_c = max|w| / 32639, q = clamp(rint(w /
sigma_c), -32639, 32639) in float32, split the same way), sums hi*hi and hi*lo + lo*hi in float64 (exact integers far below
2^53), and applies the epilogue in float32 without FMA:
    S = 256 A + C,  t = fl(fl(float32(S) * f_c) + b'_c),  f_c = 2^8 sigma_c 2^k_out,  b'_c = b_c 2^k_out,  ReLU,
    v = clip(rint(t), -32768, 32639).
The stored output must equal v * 2^-k_out; the layers that write the fp32 maps (k_out = 0) must equal t.
"""
import os
import subprocess

import numpy as np
import pytest
import torch

from caffe_rtpose_b200 import engine, synth
from oracle import orc
from test_conv_shapes import CASES, FRAMES, level_dims, pose_spec, spec_weights, write_prototxt
from test_prototxt import spec_prototxt
from test_gpu_conv_layers import (checked_layers, conv_layers, frames_for, level_geo, netspec, plan_gaps, sample_pixels,
                                  weights_with_biases)
from test_gpu_flip_test import check_mirrored_copies, frames_of, he_engine
from test_gpu_s8_mode import CONFIGS, IntBlobs, fold, int_acc_at, int_conv_full, rel, write_bmp
from test_gpu_s8_shapes import DEAD, case_weights, check_pools

pytestmark = pytest.mark.gpu
X2 = engine.PREC_S8X2
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "caffe_rtpose_b200", "rtpose.bin")
# max |maps - oracle| / max |oracle| at 160x96, calibrated, about 2x the largest value measured on an H100 80GB HBM3 (700 W power
# limit): COCO 1.28e-3 - 2.12e-3 and MPI 1.19e-3 - 1.49e-3 (frames 0 / 1, one and two scales); see test_whole_net_vs_oracle
TOL_NET = 4.5e-3


def split(v):
    hi = np.floor((v + 128) / 256)
    return hi, v - 256 * hi


def quantize(w):
    """Per output channel (axis 0) of float32 weights: (sigma float32 (co,), hi, lo float64 of w's shape)."""
    w = np.asarray(w, np.float32)
    flat = w.reshape(w.shape[0], -1)
    sigma = (np.abs(flat).max(axis=1) / np.float32(32639)).astype(np.float32)
    safe = np.where(sigma > 0, sigma, np.float32(1))
    q = np.where(sigma[:, None] > 0, np.clip(np.rint(flat / safe[:, None]), -32639, 32639), 0.0).reshape(w.shape)
    hi, lo = split(q.astype(np.float64))
    return sigma, hi, lo


def epilogue(A, C, sigma, b, k_out, relu, planar):
    """The kernel's epilogue on the float64 integer sums A = sum hi*hi, C = sum hi*lo + lo*hi (..., co)."""
    S = (256 * A + C).astype(np.int64)
    f = (sigma * np.float32(2.0 ** k_out * 256)).astype(np.float32)
    bb = (np.asarray(b, np.float32) * np.float32(2.0 ** k_out)).astype(np.float32)
    t = (S.astype(np.float32) * f).astype(np.float32)
    t = (t + bb).astype(np.float32)
    if relu:
        t = np.maximum(t, np.float32(0))
    return t.astype(np.float64) if planar else np.clip(np.rint(t), -32768, 32639).astype(np.float64)


class Int16Blobs(IntBlobs):
    def ints(self, name):
        x = self.blobs.get(name).astype(np.float64)
        v = x * np.ldexp(1.0, self.k(name))[None, :, None, None]
        assert np.array_equal(v, np.rint(v)) and v.min() >= -32768 and v.max() <= 32639, name
        return v


def check_layer(layer, ib, W, pts):
    """Bit-exact check of one conv layer at sampled pixels; returns the number of compared values."""
    w, b = W[layer["name"]]
    sigma, hw, lw = quantize(fold(w, ib.k(layer["bottom"])))
    ha, la = split(ib.ints(layer["bottom"]))
    A = int_acc_at(ha, hw, pts)
    C = int_acc_at(ha, lw, pts) + int_acc_at(la, hw, pts)
    planar = layer["top"] in ib.blobs.final_off
    k_out = 0 if planar else ib.eng.blob_log2_scale(layer["top"])
    want = epilogue(A, C, sigma, b, k_out, layer["relu"], planar)
    y = ib.blobs.get(layer["top"])
    got = y[pts[:, 0], :, pts[:, 1], pts[:, 2]].astype(np.float64)
    got = got if planar else got * 2.0 ** k_out
    bad = got != want
    if bad.any():
        i, c = np.argwhere(bad)[0]
        raise AssertionError("%s: %d of %d values differ; first at (n, y, x) = %s channel %d: got %.9g, want %.9g (k_out %d)"
                             % (layer["name"], int(bad.sum()), bad.size, tuple(pts[i]), c, got[i, c], want[i, c], k_out))
    return bad.size


def whole_stack(spec, W, eng, nimg):
    """The net of `spec` in integers up to its final Concat from the engine's stored input, as check_layer over whole images."""
    convs, concat, final = conv_layers(None, spec)
    pools = {l["top"][0]: l["bottom"][0] for l in spec["layers"] if l["type"] == "Pooling"}
    inp = spec["input"]
    k = {inp: eng.blob_log2_scale(inp)}
    val = {inp: eng.fetch_blob(inp)[:nimg].astype(np.float64) * 2.0 ** k[inp]}
    by_top = {l["top"]: l for l in convs}

    def get(name):
        if name in val:
            return val[name], k[name]
        if name in pools:
            x, kk = get(pools[name])
            N, C, H, Wd = x.shape
            xp = np.full((N, C, (H + 1) // 2 * 2, (Wd + 1) // 2 * 2), -np.inf)
            xp[:, :, :H, :Wd] = x
            val[name] = xp.reshape(N, C, xp.shape[2] // 2, 2, xp.shape[3] // 2, 2).max(axis=(3, 5))
            k[name] = kk
        elif name in concat:
            parts = [get(b) for b in concat[name]]
            val[name] = np.concatenate([p[0] for p in parts], axis=1)
            k[name] = np.concatenate([np.full(p[0].shape[1], p[1]) if np.ndim(p[1]) == 0 else p[1] for p in parts])
        else:
            layer = by_top[name]
            x, kin = get(layer["bottom"])
            kin = np.full(x.shape[1], kin) if np.ndim(kin) == 0 else kin
            w, b = W[layer["name"]]
            sigma, hw, lw = quantize(fold(w, kin))
            ha, la = split(x)
            A = int_conv_full(ha, hw).transpose(0, 2, 3, 1)
            C = (int_conv_full(ha, lw) + int_conv_full(la, hw)).transpose(0, 2, 3, 1)
            planar = name in concat[final]
            kk = 0 if planar else eng.blob_log2_scale(name)
            val[name] = epilogue(A, C, sigma, b, kk, layer["relu"], planar).transpose(0, 3, 1, 2)
            k[name] = kk
        return val[name], k[name]

    return np.concatenate([get(b)[0] for b in concat[final]], axis=1)


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_conv_layers_bit_exact(cfg, tmp_path):
    """Every conv layer of both models and of a prototxt net, at one frame (the stride-8 layers at BN 64) and nine (BN 128)."""
    model, net_w, net_h, n = CONFIGS[cfg]
    spec, path = spec_prototxt(model, tmp_path) if isinstance(model, str) else (None, None)
    m = engine.MPI_15 if path else model
    W = spec_weights(spec) if spec else weights_with_biases(m)
    eng = engine.PoseEngine(None if path else m, net_w, net_h, 2 * net_w, 2 * net_h, precision=X2, max_batch=n, prototxt=path)
    eng.set_weights(W)
    frames = frames_for(n, 2 * net_w, 2 * net_h)
    eng.calibrate(frames[:1])
    eng.forward_frames(frames)
    gaps = plan_gaps(prototxt=path) if path else None
    ib = Int16Blobs(eng, n, None if path else m, W, spec)
    rng = np.random.default_rng(11)
    layers = conv_layers(None, spec)[0] if spec else checked_layers(m)
    count = 0
    for layer in layers:
        w_, h_, gap = level_geo(net_w, net_h, layer["level"], gaps)
        count += check_layer(layer, ib, W, sample_pixels(n, h_, w_, gap, rng, 300))
    eng.close()
    print("\n%s s8x2: %d layers, %d values bit-exact" % (cfg, len(layers), count))


@pytest.mark.parametrize("name", list(CASES))
def test_generated_convs_bit_exact(name, tmp_path):
    """The generated graphs of test_conv_shapes.py (5x5 filters, every tile width, odd Concat slots, dead channels), at one and
    three frames, every conv layer and max pool."""
    spec, path = write_prototxt(name, tmp_path)
    c = CASES[name]
    net_w, net_h = c["net_w"], c["net_h"]
    gaps = plan_gaps(prototxt=path)
    W = case_weights(name, spec)
    eng = engine.PoseEngine(None, net_w, net_h, 2 * net_w, 2 * net_h, start_scale=0.5, precision=X2, prototxt=path,
                            max_batch=max(FRAMES))
    eng.set_weights(W)
    eng.calibrate(frames_for(FRAMES[0], 2 * net_w, 2 * net_h))
    layers = conv_layers(None, spec)[0]
    rng = np.random.default_rng(11)
    count = 0
    for n in FRAMES:
        eng.forward_frames(frames_for(n, 2 * net_w, 2 * net_h))
        ib = Int16Blobs(eng, n, None, W, spec)
        for layer in layers:
            w_, h_ = level_dims(net_w, net_h, layer["level"])
            count += check_layer(layer, ib, W, sample_pixels(n, h_, w_, gaps[layer["level"]], rng, 300))
        check_pools(eng, spec, ib.blobs, n, "%d frame(s)" % n)
    eng.close()
    print("\n%s s8x2: %d values bit-exact (%d layers with dead channels)" % (name, count, len(DEAD.get(name, []))))


@pytest.mark.parametrize("model", [engine.COCO_18, engine.MPI_15])
def test_whole_stack_bit_exact(model):
    """160x96, calibrated, two frames: the integer chain of every layer, max pool and Concat from the stored net input equals
    pe_fetch_maps bit for bit."""
    net_w, net_h = 160, 96
    W = weights_with_biases(model)
    frames = [synth.make_frame(30 + i, 2 * net_h, 2 * net_w) for i in range(2)]
    eng = engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=X2, max_batch=2)
    eng.set_weights(W)
    eng.calibrate(frames[:1])
    eng.forward_frames(frames)
    maps = eng.fetch_maps(2).astype(np.float64)
    want = whole_stack(netspec(model), W, eng, 2)
    eng.close()
    bad = maps != want
    assert not bad.any(), "%d of %d map values differ, max |diff| %.3g" % (int(bad.sum()), bad.size, float(np.abs(maps - want).max()))


def test_max_pool_exact():
    """Every pool top equals the 2x2 max (ceil mode) of its two-plane input exactly, at the pool's own scale."""
    model, net_w, net_h = engine.COCO_18, 656, 368
    eng = engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=X2)
    eng.set_weights(weights_with_biases(model))
    frames = frames_for(1, 2 * net_w, 2 * net_h)
    eng.calibrate(frames)
    eng.forward_frames(frames)
    for bottom, top in (("conv1_2", "pool1_stage1"), ("conv2_2", "pool2_stage1"), ("conv3_4", "pool3_stage1")):
        x, y = eng.fetch_blob(bottom)[:1], eng.fetch_blob(top)[:1]
        k = eng.blob_log2_scale(bottom)
        assert eng.blob_log2_scale(top) == k
        v = x.astype(np.float64) * 2.0 ** k
        assert np.abs(v).max() > 256   # the hi plane carries the values
        H, Wd = x.shape[2], x.shape[3]
        xp = np.full((1, x.shape[1], (H + 1) // 2 * 2, (Wd + 1) // 2 * 2), -np.inf, np.float32)
        xp[:, :, :H, :Wd] = x
        want = xp.reshape(1, x.shape[1], xp.shape[2] // 2, 2, xp.shape[3] // 2, 2).max(axis=(3, 5))
        assert np.array_equal(y, want), top
    eng.close()


@pytest.mark.parametrize("S", [1, 2])
@pytest.mark.parametrize("model", [engine.COCO_18, engine.MPI_15])
def test_whole_net_vs_oracle(model, S):
    """Calibrated, 160x96: stride-8 maps against the oracle (fp32), and the same batch three times (eager, captured, replayed)
    gives bit-identical maps, peaks and joints.

    Tolerance: every layer rounds its output to a step 2^-k with the stored maximum in [2^13, 2^14), an absolute error of up
    to 2^-14 of the layer's maximum, and its weights to half of sigma_c, 2^-16 of the channel's largest weight.  The step is
    absolute: a value far below its layer's maximum keeps correspondingly fewer significant bits, so for the bulk of the
    activations the rounding is of the order of fp16's relative 2^-11, and it compounds over the 20 (MPI) to 52 (COCO) layers
    of the deepest path as the fast mode's does.
    Measured 1.19e-3 - 2.12e-3 of the map maximum (TOL_NET); held to about twice that."""
    net_w, net_h = 160, 96
    W = synth.make_weights(model, "he", seed=7)
    frames = [synth.make_frame(20 + i, 192, 320) for i in range(2)]
    onet = orc.Net(model)
    onet.set_weights(W)
    omaps = [onet.forward(orc.preprocess(f, net_h, net_w, S, 1.0, 0.25)) for f in frames]
    eng = engine.PoseEngine(model, net_w, net_h, 320, 192, num_scales=S, start_scale=1.0, scale_gap=0.25, precision=X2, max_batch=2)
    eng.set_weights(W)
    eng.calibrate(frames)
    calls = []
    for _ in range(3):
        eng.forward_frames(frames)
        calls.append((eng.fetch_maps(2).copy(), [eng.fetch(k) for k in range(2)]))
    maps = calls[0][0]
    errs = [rel(maps[i * S:(i + 1) * S], omaps[i]) for i in range(2)]
    print("\nS8X2 %s 160x96 S=%d: maps vs oracle %s" % ("COCO" if model == engine.COCO_18 else "MPI", S, ["%.3e" % e for e in errs]))
    assert max(errs) < TOL_NET
    for c in calls[1:]:
        assert np.array_equal(c[0], maps)
        for (na, ja, pa), (nb, jb, pb) in zip(c[1], calls[0][1]):
            assert na == nb and np.array_equal(ja, jb) and np.array_equal(pa, pb)
    rc, worst, layer = eng.range_status()
    assert rc == 0 and 0 < worst < 1, (rc, worst, layer)
    eng.close()


def test_calibration_required_range_and_tables():
    """A forward before pe_calibrate is PE_ERR_STATE.  After it the calibration frame's stored maxima lie in [2^13, 2^14) (ratio
    to 32639 in [0.25, 0.502)), and the net input is at k = 16.  A calibration table round-trips onto a second engine (bit-identical
    maps); an S8X1 table and an S8X2 table refuse each other.  A handle calibrated on a flat grey frame and then given a busy
    frame leaves the range: PE_ERR_RANGE with a layer named."""
    model, net_w, net_h = engine.COCO_18, 160, 96
    W = synth.make_weights(model, "he")
    busy = synth.make_frame(3, 2 * net_h, 2 * net_w)
    eng = engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=X2)
    eng.set_weights(W)
    with pytest.raises(engine.PoseEngineError, match="pe_calibrate"):
        eng.forward_frames([busy])
    eng.calibrate([busy])
    eng.forward_frames([busy])
    want = eng.fetch_maps(1).copy()
    rc, worst, layer = eng.range_status()
    assert rc == 0 and 0.25 <= worst < 16384.5 / 32639, (rc, worst, layer)
    assert eng.blob_log2_scale("image") == 16
    table = eng.calibration_table()
    assert "precision 8\n" in table and " s8x2 " in table
    other = engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=X2)
    other.set_weights(W)
    other.set_calibration_table(table)
    other.forward_frames([busy])
    assert np.array_equal(other.fetch_maps(1), want)
    s8 = engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=engine.PREC_S8X1)
    s8.set_weights(W)
    with pytest.raises(engine.PoseEngineError, match="precision"):
        s8.set_calibration_table(table)
    s8.calibrate([busy])
    with pytest.raises(engine.PoseEngineError, match="precision"):
        other.set_calibration_table(s8.calibration_table())
    for e in (eng, other, s8):
        e.close()
    grey = np.full((2 * net_h, 2 * net_w, 3), 100, np.uint8)
    eng = engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=X2)
    eng.set_weights(W)
    eng.calibrate([grey])
    eng.range_status()
    eng.forward_frames([busy])
    eng.sync()
    rc, worst, layer = eng.range_status()
    print("\nS8X2 calibrated on grey, busy frame: rc %d, worst %.3g, layer %s" % (rc, worst, layer))
    assert rc == 5 and layer in {l[0] for l in eng.conv_layers()}, (rc, worst, layer)
    eng.close()


def calibrated_source(device=0):
    model, net_w, net_h = engine.COCO_18, 160, 96
    frame = synth.make_frame(5, 2 * net_h, 2 * net_w)
    e0 = engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=X2, device=device)
    e0.set_weights(synth.make_weights(model, "he"))
    e0.calibrate([frame])
    return e0, frame, lambda dev: engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=X2, device=dev)


def forward_results(engs, frame):
    res = []
    for e in engs:
        e.forward_frames([frame])
        cnt, joints, peaks = e.fetch(0)
        res.append((cnt, joints.copy(), peaks.copy(), e.fetch_maps(1).copy(), e.fetch_blob("conv4_4_CPM")[:1].copy()))
    for e in engs:
        e.close()
    for r in res[1:]:
        assert r[0] == res[0][0]
        for a, b in zip(r[1:], res[0][1:]):
            assert np.array_equal(a, b)


def test_share_weights_bit_identical():
    e0, frame, make = calibrated_source()
    e1 = make(0)
    engine.share_weights(e0, e1)
    forward_results([e0, e1], frame)


def test_broadcast_weights_bit_identical():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    e0, frame, make = calibrated_source()
    e2 = make(1)
    engine.broadcast_weights([e0, e2])
    forward_results([e0, e2], frame)


def test_no_sparse_layers():
    """pe_conv_layer_sparse is 0 for every layer, even with every layer's weights 2:4 and the sparse shape rule lifted
    (pe_test_force_sparse), while an S8X1 engine given the same weights runs layers sparse."""
    model = engine.COCO_18
    W = engine.prune_2to4(synth.make_weights(model, "he"), model=model)
    got = {}
    for prec in (engine.PREC_S8X1, X2):
        eng = engine.PoseEngine(model, 160, 96, 320, 192, precision=prec)
        assert engine.lib().pe_test_force_sparse(eng._h, 1) == 0
        eng.set_weights(W)
        got[prec] = eng.sparse_layers()
        eng.close()
    assert got[engine.PREC_S8X1] and got[X2] == []


@pytest.mark.parametrize("model", [engine.COCO_18, engine.MPI_15])
def test_flip_test_mirrored_copies(model):
    """With the flip test on, each frame's maps are its flip-off maps and those of its planar net input reversed in x, bit for
    bit, at one and three scales (as test_gpu_flip_test.py checks for the other modes)."""
    frames = frames_of(2, 192, 320, seed=5)
    for S in (1, 3):
        eng = he_engine(model, 160, 96, S, X2, max_batch=2)
        eng.calibrate(frames[:1])
        check_mirrored_copies(eng, frames, S, 160, 96, (1, 2))
        eng.close()


def test_accumulator_bound_refused(tmp_path):
    """A generated prototxt whose 7x7 layer reads 1400 channels (K = 49 x 1408 padded > 65793) fails at precision 8 with
    PE_ERR_INVALID naming the layer and the bound; the same file builds at precision 6 (its bound is 132104)."""
    spec = pose_spec(engine.MPI_15, 16, 16, conv1_1=8, levels=[[(3, 8)], [(3, 8)], [(3, 8)], [(1, 1400), (7, 16)]], branch=[(1, 8)])
    path = tmp_path / "big_k.prototxt"
    path.write_text(synth.netspec_to_prototxt(spec))
    with pytest.raises(engine.PoseEngineError, match="conv4_2") as ex:
        engine.PoseEngine(None, 16, 16, 32, 32, precision=X2, prototxt=str(path))
    assert "65793" in str(ex.value) and "PE_PREC_S8X2" in str(ex.value)
    eng = engine.PoseEngine(None, 16, 16, 32, 32, precision=engine.PREC_S8X1, prototxt=str(path))
    assert "conv4_2" in {l[0] for l in eng.conv_layers()}
    eng.close()


def test_cli_precision_7_json(tmp_path):
    """rtpose.bin --precision 8 on the Python engine's calibration table writes, for every frame of an --image_dir, the JSON of
    PoseEngine(precision=PREC_S8X2) with that table; --audit_every 1 prints its comparison with the parity mode and leaves the
    JSON unchanged."""
    model, n = engine.COCO_18, 6
    W = synth.make_weights(model, "he", seed=3)
    cm = tmp_path / "w.caffemodel"
    engine.write_caffemodel(str(cm), W, synth.conv_table(model))
    imgs = tmp_path / "imgs"
    imgs.mkdir()
    frames = [synth.make_frame(100 + i, 192, 320) for i in range(n)]
    for i, f in enumerate(frames):
        write_bmp(str(imgs / ("f%03d.bmp" % i)), f)
    eng = engine.PoseEngine(model, 160, 96, 320, 192, precision=X2)
    eng.set_weights(W)
    eng.calibrate(frames[:1])
    table = tmp_path / "table.txt"
    table.write_text(eng.calibration_table())
    want = []
    for f in frames:
        eng.forward_frames([f])
        want.append(eng.json(eng.fetch(0)[1]))
    eng.close()
    common = [BIN, "--image_dir", str(imgs), "--caffemodel", str(cm), "--model", "COCO", "--resolution", "320x192",
              "--net_resolution", "160x96", "--no_frame_drops", "--no_display", "--precision", "8", "--calibration_table", str(table)]
    for audit in (False, True):
        out = tmp_path / ("json_audit%d" % audit)
        r = subprocess.run(common + ["--write_json", str(out)] + (["--audit_every", "1"] if audit else []), capture_output=True,
                           text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        assert ("Audit summary: " in r.stderr) is audit, r.stderr[-2000:]
        if audit:
            print("\n" + "\n".join(l for l in r.stderr.splitlines() if "Audit" in l))
        for i in range(n):
            assert (out / ("f%03d.json" % i)).read_text() == want[i], (audit, i)
