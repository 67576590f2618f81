"""Mixed precision (pe_create_mixed: chosen conv layers in fp16 inside PE_PREC_E4M3X1 and PE_PREC_S8X1) on the GPU.

Equivalence: with every conv layer listed, either base computes exactly what PE_PREC_F16X1 computes (same plan, same packed
weights, same calibration), and with an empty list exactly what its base mode computes.

Per layer against float64, with the sampling of tests/test_gpu_conv_layers.py at both tile widths (one frame at 656x368, three
at 320x176).  The list is `narrow` + the 7x7 layers of stage 2 + the stage-input group (both branches' first layers of every
stage), so that every boundary occurs: fp16 -> e4m3 / s8 (conv2_1, Mconv5_stage2_*), e4m3 / s8 -> fp16 (conv4_4_CPM and every
stage's Mconv7, whose outputs fill the fp16 stage-input buffer), and a Concat whose producers computed in another format.
  * fp16 layers: the float64 reference of the stored input with the weights rounded as the engine packs them (fp16 at max|w| in
    [2^13, 2^14), after the power-of-two range ratios of a mixed-scale Concat input are folded in); the distance d of that
    reference from the rounding cell of the stored output (fp16, e4m3 or s8) is at most the accumulation error, bounded by
    B_F16 * mag, mag = sum |a||w| + |b| (tests/test_gpu_conv_layers.py: 93u of chunked truncating fp16 sums < 2^-17).
  * e4m3 layers: the same with weights rounded to e4m3 (max|w| in [128, 256)) and B_E8 of tests/test_gpu_fp8_mode.py.
  * s8 layers, including those that store fp16: bit for bit against the integer reference of tests/test_gpu_s8_mode.py (the
    fp16 ones store t rounded to nearest fp16).
The E4M3X1 engine runs uncalibrated (scale 1: He-init activations stay far inside e4m3), the S8X1 engine calibrated.  Each class
is also held to about 2x its measured maximum (MEASURED_MAX).

Whole net against the oracle, range reporting, calibration, CUDA-graph replay, weight sharing and the CLI: see the tests below.
"""
import os
import subprocess

import numpy as np
import pytest
import torch

from caffe_rtpose_b200 import engine, synth
from oracle import orc
from test_gpu_conv_layers import Blobs, checked_layers, conv_ref, frames_for, layer_class, level_geo, sample_pixels
from test_gpu_fp8_mode import B_E8, e4m3_cell
from test_gpu_fp8_mode import TOL_NET as TOL_E8
from test_gpu_s8_mode import IntBlobs, epilogue, fold, int_acc_at, quantize, tc_bn, write_bmp
from test_gpu_s8_mode import TOL_NET as TOL_S8
from test_gpu_conv_layers import weights_with_biases

pytestmark = pytest.mark.gpu
E8, S8, F1 = engine.PREC_E4M3X1, engine.PREC_S8X1, engine.PREC_F16X1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "caffe_rtpose_b200", "rtpose.bin")
B_F16 = 2.0 ** -17
STAGE_INPUTS = ["conv5_1_CPM_L1", "conv5_1_CPM_L2"] + ["Mconv1_stage%d_L%d" % (s, b) for s in range(2, 7) for b in (1, 2)]
LIST = ["narrow"] + ["Mconv%d_stage2_L%d" % (i, b) for i in range(2, 6) for b in (1, 2)] + STAGE_INPUTS
# largest d / mag per (compute kind, "f32" for the planar maps, layer class), about 2x the values measured on an H100 80GB HBM3
# (700 W power limit) over COCO and MPI and both tile widths: e4m3 1x1 2.5e-4, 3x3 1.9e-4, 7x7 8.7e-5, the fp32 map layers
# 2.1e-4; fp16 3x3 1.2e-7, 7x7 5.3e-8, conv1_1 2.3e-8.  The s8 layers are bit-exact.
MEASURED_MAX = {("e4m3", "", "1x1"): 5e-4, ("e4m3", "", "3x3"): 4e-4, ("e4m3", "", "7x7"): 1.8e-4, ("e4m3", "f32", "1x1"): 4.5e-4,
                ("f16", "", "3x3"): 2.5e-7, ("f16", "", "7x7"): 1.1e-7, ("f16", "", "im2col"): 5e-8,
                ("s8", "", "1x1"): 0.0, ("s8", "", "3x3"): 0.0, ("s8", "", "7x7"): 0.0, ("s8", "f32", "1x1"): 0.0}


def rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


def last_error(eng):
    return engine.lib().pe_last_error(eng._h).decode()


def kinds(model, base, layers):
    return engine.plan_formats(model, base, layers)["convs"]


def mixed(model, net_w, net_h, base, layers, n=1, **kw):
    return engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=base, max_batch=n, f16_layers=layers, **kw)


# ------------------------------------------------------------------------------------------ equivalence
def results(eng, frames, blobs):
    eng.forward_frames(frames)
    n = len(frames)
    fetched = [eng.fetch(i) for i in range(n)]
    rc, worst, layer = eng.range_status()
    return (eng.fetch_maps(n).copy(), [(c, j.copy(), p.copy()) for c, j, p in fetched], (rc, worst, layer),
            {b: eng.blob_log2_scale(b) for b in blobs})


def same(a, b):
    assert np.array_equal(a[0], b[0])
    for (ca, ja, pa), (cb, jb, pb) in zip(a[1], b[1]):
        assert ca == cb and np.array_equal(ja, jb) and np.array_equal(pa, pb)
    assert a[2] == b[2] and a[3] == b[3], (a[2], b[2])


@pytest.mark.parametrize("model", [engine.COCO_18, engine.MPI_15])
def test_every_layer_listed_is_f16x1_and_an_empty_list_is_the_base(model):
    """Calibrated on the same frame: maps, peaks, joints, pe_range_status and every conv blob's scale exponent bit for bit."""
    net_w, net_h = 320, 176
    W = synth.make_weights(model, "he", seed=5)
    frames = [synth.make_frame(40 + i, 2 * net_h, 2 * net_w) for i in range(2)]
    names = list(kinds(model, F1, None))
    blobs = [n for n in names if not n.startswith("Mconv7_stage6")] + ["image"]

    def run(prec, layers):
        e = mixed(model, net_w, net_h, prec, layers, 2) if layers is not None else \
            engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=prec, max_batch=2)
        e.set_weights(W)
        e.calibrate(frames[:1])
        r = results(e, frames, blobs)
        e.close()
        return r

    ref16 = run(F1, None)
    for base in (E8, S8):
        same(run(base, names), ref16)
        same(run(base, ""), run(base, None))


# ------------------------------------------------------------------------------------------ per layer
def packed(w, kind):
    """The weights as the engine packs them: w * 2^k rounded to fp16 (max in [2^13, 2^14)) or e4m3 ([128, 256)), over 2^k."""
    mx = float(np.abs(w).max())
    if mx == 0:
        return w.astype(np.float64)
    _, ex = np.frexp(np.float32(mx))
    s = np.ldexp(np.float32(1), (14 if kind == "f16" else 8) - int(ex))
    t = torch.from_numpy((w * s).astype(np.float32))
    r = t.half().float() if kind == "f16" else t.to(torch.float8_e4m3fn).float()
    return r.double().numpy() / float(s)


def cell(got, kind, k):
    """[lo, hi]: the true values (stored value at scale 2^k, fetched / 2^k) that round to the stored `got`."""
    v = got * 2.0 ** k
    if kind == "e4m3":
        lo, hi = e4m3_cell(v)
    elif kind == "s8":
        sat_hi, sat_lo = v >= 127, v <= -128
        lo, hi = np.where(sat_hi, 126.5, v - 0.5), np.where(sat_lo, -127.5, v + 0.5)
        lo, hi = np.where(sat_lo, -np.inf, lo), np.where(sat_hi, np.inf, hi)
    else:
        a = np.abs(v)
        e = np.floor(np.log2(np.where(a > 0, a, 1.0)))
        normal = a >= 2.0 ** -14
        up = np.where(normal, 2.0 ** (e - 11), 2.0 ** -25)
        down = np.where(normal & (a == 2.0 ** e) & (e > -14), 2.0 ** (e - 12), up)
        lo, hi = np.where(v >= 0, v - down, v - up), np.where(v >= 0, v + up, v + down)
    return lo * 2.0 ** -k, hi * 2.0 ** -k


def float_layer(layer, eng, blobs, kscale, W, compute, out, pts, bound=None):
    """d / mag of an fp16 or e4m3 layer (module docstring); bound: the layer's B instead of B_F16 / B_E8."""
    w, b = W[layer["name"]]
    kin = kscale(layer["bottom"])
    r = np.ldexp(1.0, kin.max() - kin).astype(np.float32)   # the power-of-two range ratios the packer folds in
    wq = packed((w * r[None, :, None, None]).astype(np.float32), compute) / r[None, :, None, None]
    x, y = blobs.get(layer["bottom"]), blobs.get(layer["top"])
    ref, mag = conv_ref(x, wq, b, pts, layer["relu"])
    got = y[pts[:, 0], :, pts[:, 1], pts[:, 2]].astype(np.float64)
    if out == "f32":
        d = np.abs(got - ref)
    else:
        lo, hi = cell(got, out, int(kscale(layer["top"])[0]))
        d = np.maximum(0.0, np.maximum(ref - hi, lo - ref))
    B = bound or (B_F16 if compute == "f16" else B_E8)
    bad = d > B * mag
    if bad.any():
        i, c = np.argwhere(bad)[0]
        raise AssertionError("%s (%s -> %s): %d of %d elements outside the bound; first at %s channel %d: got %.9g, ref %.9g, mag %.3g"
                             % (layer["name"], compute, out, int(bad.sum()), bad.size, tuple(pts[i]), c, got[i, c], ref[i, c], mag[i, c]))
    return float((d / mag).max())


def s8_layer(layer, ib, W, out, pts):
    """Bit-exact check of an s8 layer; `out` f16: the stored value is t rounded to nearest fp16."""
    w, b = W[layer["name"]]
    sigma, q = quantize(fold(w, ib.k(layer["bottom"])))
    acc = int_acc_at(ib.ints(layer["bottom"]), q, pts)
    planar = out == "f32"
    k_out = 0 if planar else ib.eng.blob_log2_scale(layer["top"])
    t = epilogue(acc, sigma, b, k_out, layer["relu"], True)
    want = t if planar else np.clip(np.rint(t), -128, 127) if out == "s8" else t.astype(np.float16).astype(np.float64)
    got = ib.blobs.get(layer["top"])[pts[:, 0], :, pts[:, 1], pts[:, 2]].astype(np.float64) * (1 if planar else 2.0 ** k_out)
    bad = got != want
    if bad.any():
        i, c = np.argwhere(bad)[0]
        raise AssertionError("%s (s8 -> %s): %d of %d values differ; first at %s channel %d: got %.9g, want %.9g"
                             % (layer["name"], out, int(bad.sum()), bad.size, tuple(pts[i]), c, got[i, c], want[i, c]))
    return 0.0


@pytest.mark.parametrize("base", [E8, S8])
@pytest.mark.parametrize("model", [engine.COCO_18, engine.MPI_15])
def test_conv_layers_vs_float64(model, base):
    W = weights_with_biases(model)
    conv_kinds = kinds(model, base, LIST)
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(11)
    worst, boundaries = {}, set()
    for net_w, net_h, n in ((656 if model == engine.COCO_18 else 496, 368, 1), (320, 176, 3)):
        eng = mixed(model, net_w, net_h, base, LIST, n)
        eng.set_weights(W)
        frames = frames_for(n, 2 * net_w, 2 * net_h)
        if base == S8:
            eng.calibrate(frames[:1])
        eng.forward_frames(frames)
        rc, ratio, name = eng.range_status()
        assert rc == 0, (rc, ratio, name)
        ib = IntBlobs(eng, n, model, W)
        kscale = ib.k if base == S8 else (lambda blob: np.zeros(ib.blobs.get(blob).shape[1], int))
        for layer in checked_layers(model):
            compute, out = conv_kinds[layer["name"]][:2]
            w_, h_, gap = level_geo(net_w, net_h, layer["level"])
            pts = sample_pixels(n, h_, w_, gap, rng, 300)
            if compute == "s8":
                r = s8_layer(layer, ib, W, out, pts)
            else:
                r = float_layer(layer, eng, ib.blobs, kscale, W, compute, out, pts)
            bn = tc_bn(W[layer["name"]][0].shape[0], n * (h_ + gap) * (w_ + gap), nsm)
            key = (compute, out if out == "f32" else "", layer_class(layer))
            worst[key] = max(worst.get(key, 0.0), r)
            boundaries.add((compute, out, bn))
        eng.close()
    print("\n%s base %d: largest d / mag per (compute kind, fp32 output, layer class): %s" % (
        "COCO" if model == engine.COCO_18 else "MPI", base, {"/".join(filter(None, k)): "%.3e" % v for k, v in sorted(worst.items())}))
    print("  (compute, stored, BN) run: %s" % sorted(boundaries))
    kind = "e4m3" if base == E8 else "s8"
    assert {(c, o) for c, o, _ in boundaries} >= {("f16", kind), (kind, "f16"), ("f16", "f16"), (kind, kind)}
    over = {k: v for k, v in worst.items() if v > MEASURED_MAX[k]}
    assert not over, "accumulation error above what this kernel measured: %s" % over


# ------------------------------------------------------------------------------------------ whole net, replay
@pytest.mark.parametrize("base,tol", [(E8, TOL_E8), (S8, TOL_S8)])
@pytest.mark.parametrize("model", [engine.COCO_18, engine.MPI_15])
def test_whole_net_vs_oracle_and_replay(model, base, tol):
    """Calibrated, 160x96, two frames, `narrow` + the stage-input group: maps against the oracle within the base mode's bound,
    and the second (captured) and third (replayed) forwards reproduce the calibration forward bit for bit."""
    net_w, net_h = 160, 96
    W = synth.make_weights(model, "he", seed=7)
    frames = [synth.make_frame(20 + i, 192, 320) for i in range(2)]
    onet = orc.Net(model)
    onet.set_weights(W)
    omaps = [onet.forward(orc.preprocess(f, net_h, net_w, 1, 1.0, 0.25)) for f in frames]
    eng = mixed(model, net_w, net_h, base, ["narrow"] + STAGE_INPUTS, 2)
    eng.set_weights(W)
    eng.calibrate(frames)
    calls = [(eng.fetch_maps(2).copy(), [eng.fetch(k) for k in range(2)])]
    for _ in range(3):
        eng.forward_frames(frames)
        calls.append((eng.fetch_maps(2).copy(), [eng.fetch(k) for k in range(2)]))
    errs = [rel(calls[1][0][i:i + 1], omaps[i]) for i in range(2)]
    print("\nbase %d + narrow + stage inputs, %s 160x96: maps vs oracle %s" % (base, "COCO" if model == engine.COCO_18 else "MPI",
                                                                              ["%.3e" % e for e in errs]))
    assert max(errs) < tol
    for c in calls[1:]:
        assert np.array_equal(c[0], calls[0][0])
        for (na, ja, pa), (nb, jb, pb) in zip(c[1], calls[0][1]):
            assert na == nb and np.array_equal(ja, jb) and np.array_equal(pa, pb)
    eng.close()


# ------------------------------------------------------------------------------------------ range and calibration
def test_range_reports_fp16_layers_against_fp16_limits():
    """Uncalibrated, fp16 layers whose values shrink below 2^-10 (the prototxt's gaussian(0.01) filler) or grow past 65504
    (He weights x 1.6 per layer) are PE_ERR_RANGE with fp16's texts; an S8X1 base refuses an uncalibrated forward, and after
    pe_calibrate its fp16 net input has scale 1."""
    model, net_w, net_h = engine.COCO_18, 160, 96
    frame = synth.make_frame(3, 2 * net_h, 2 * net_w)
    conv_kinds = kinds(model, E8, None)
    he = synth.make_weights(model, "he")
    for W, what in ((synth.make_weights(model, "caffe"), "is below 2^-10, the fp16 planes lose precision"),
                    ({k: (w * np.float32(1.6), b) for k, (w, b) in he.items()}, "outside the range of the fp16 planes")):
        eng = mixed(model, net_w, net_h, E8, list(conv_kinds))   # every layer in fp16
        eng.set_weights(W)
        eng.forward_frames([frame])
        eng.sync()
        rc, worst, layer = eng.range_status()
        assert rc == 5 and layer in conv_kinds and what in last_error(eng), (rc, worst, layer, last_error(eng))
        eng.close()
    eng = mixed(model, net_w, net_h, S8, "narrow")
    eng.set_weights(synth.make_weights(model, "he"))
    with pytest.raises(engine.PoseEngineError, match="pe_calibrate"):
        eng.forward_frames([frame])
    eng.calibrate([frame])
    eng.forward_frames([frame])
    rc, worst, layer = eng.range_status()
    assert rc == 0 and 0 < worst < 1, (rc, worst, layer)
    assert eng.blob_log2_scale("image") == 0   # an fp16 net input at scale 1, as in F16X1
    eng.close()


def test_range_names_an_fp16_layer_in_a_mixed_engine():
    """E4M3X1 + narrow, uncalibrated: conv1_2's weights x 2^-14 (conv2_1's x 2^14 undo it, biases are 0) leave conv1_2's fp16
    output below 2^-10 while the e4m3 layers keep their usual range, so pe_range_status names conv1_2 with fp16's floor, not
    e4m3's 2^-2.  pe_calibrate clears it."""
    model, net_w, net_h = engine.COCO_18, 160, 96
    frame = synth.make_frame(3, 2 * net_h, 2 * net_w)
    W = synth.make_weights(model, "he")
    W["conv1_2"] = (W["conv1_2"][0] * np.float32(2.0 ** -14), W["conv1_2"][1])
    W["conv2_1"] = (W["conv2_1"][0] * np.float32(2.0 ** 14), W["conv2_1"][1])   # conv2_1 undoes it: the rest is unchanged
    eng = mixed(model, net_w, net_h, E8, "narrow")
    eng.set_weights(W)
    eng.forward_frames([frame])
    eng.sync()
    rc, worst, layer = eng.range_status()
    assert rc == 5 and layer == "conv1_2" and "below 2^-10, the fp16 planes" in last_error(eng), (rc, layer, last_error(eng))
    eng.calibrate([frame])
    eng.forward_frames([frame])
    rc, worst, layer = eng.range_status()
    assert rc == 0, (rc, worst, layer)
    eng.close()


# ------------------------------------------------------------------------------------------ sharing
def test_share_and_broadcast_need_the_same_fp16_layers():
    model, net_w, net_h = engine.COCO_18, 160, 96
    frame = synth.make_frame(5, 2 * net_h, 2 * net_w)
    for base in (E8, S8):
        e0 = mixed(model, net_w, net_h, base, "narrow")
        e0.set_weights(synth.make_weights(model, "he"))
        e0.calibrate([frame])
        e1, e2 = mixed(model, net_w, net_h, base, "narrow"), mixed(model, net_w, net_h, base, "conv1_1")
        with pytest.raises(engine.PoseEngineError, match="fp16 layers differ"):
            engine.share_weights(e0, e2)
        with pytest.raises(engine.PoseEngineError, match="fp16 layers differ"):
            engine.broadcast_weights([e0, e2])
        engine.share_weights(e0, e1)
        res = []
        for e in (e0, e1):
            e.forward_frames([frame])
            cnt, joints, peaks = e.fetch(0)
            res.append((cnt, joints.copy(), peaks.copy(), e.fetch_maps(1).copy(), e.fetch_blob("conv2_1")[:1].copy()))
        assert res[0][0] == res[1][0] and all(np.array_equal(a, b) for a, b in zip(res[0][1:], res[1][1:]))
        for e in (e0, e1, e2):
            e.close()
    if torch.cuda.device_count() >= 2:
        e0 = mixed(model, net_w, net_h, S8, "narrow")
        e0.set_weights(synth.make_weights(model, "he"))
        e0.calibrate([frame])
        r = mixed(model, net_w, net_h, S8, "narrow", device=1)
        engine.broadcast_weights([e0, r])
        res = []
        for e in (e0, r):
            e.forward_frames([frame])
            res.append(e.fetch_maps(1).copy())
            e.close()
        assert np.array_equal(res[0], res[1])


# ------------------------------------------------------------------------------------------ CLI
def test_cli_matches_the_python_path(tmp_path):
    """rtpose.bin --precision 5 --f16_layers narrow --audit_every 1 writes the JSON of the Python path on the same frames and
    weights, and prints the audit summary."""
    model, n = engine.COCO_18, 12
    W = synth.make_weights(model, "he", seed=3)
    cm = tmp_path / "w.caffemodel"
    engine.write_caffemodel(str(cm), W, synth.conv_table(model))
    imgs = tmp_path / "imgs"
    imgs.mkdir()
    frames = [synth.make_frame(100 + i, 192, 320) for i in range(n)]
    for i, f in enumerate(frames):
        write_bmp(str(imgs / ("f%03d.bmp" % i)), f)
    out = tmp_path / "json"
    r = subprocess.run([BIN, "--image_dir", str(imgs), "--caffemodel", str(cm), "--model", "COCO", "--resolution", "320x192",
                        "--net_resolution", "160x96", "--no_frame_drops", "--no_display", "--precision", "5", "--calibrate_range=false",
                        "--f16_layers", "narrow", "--audit_every", "1", "--write_json", str(out)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "Audit summary: " in r.stderr, r.stderr[-2000:]
    print("\n" + "\n".join(l for l in r.stderr.splitlines() if "Audit summary" in l))
    eng = mixed(model, 160, 96, E8, "narrow")
    eng.set_weights(W)
    for i, f in enumerate(frames):
        eng.forward_frames([f])
        cnt, joints, _ = eng.fetch(0)
        assert (out / ("f%03d.json" % i)).read_text() == eng.json(joints), i
    eng.close()
