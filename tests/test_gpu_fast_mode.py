"""The fast mode (PE_PREC_F16X1: one fp16 plane of activations and weights, one MMA per MAC) on the GPU.

Per layer, every conv layer of COCO and MPI at one and several frames is checked against float64 with the sampling and the
reference of tests/test_gpu_conv_layers.py: |got - ref| <= B * mag + floor, mag = sum |a||w| + |b|.  Error model of one fp16
plane (u = 2^-24, derived from conv_tc.cu; the fetched input is the stored plane itself, so the activations' rounding does
not enter):
    weights w * 2^k rounded to one fp16 plane (max|w| in [2^13, 2^14), 2^k exact): 2^-11 per product     2^-11
    hi*hi chunks of <= 28 truncating K16 steps, each <= 2^-23 of the partial magnitude                       56u
    round-to-nearest sum of <= 21 chunks                                                                     21u
    epilogue: *out_scale (exact) + bias (one rounding)                                                        1u
    the output rounded to one fp16 plane                                                                  2^-11
  total 2^-10 + 78u;  B = 2^-10 + 2^-17.  floor: an fp16 subnormal output has spacing 2^-24 of the stored value, i.e.
  2^-24 / s in true values (s the layer's range scale; s = 1 uncalibrated).
Each layer class is also held to 2-2.5x its measured maximum (MEASURED_MAX), so that a kernel without chunking or with a
dropped term cannot hide under the loose rigorous bound.

Whole net, range and audit: see the tests below.  Tolerances against the oracle are about 3x the measured map error."""
import os
import subprocess

import numpy as np
import pytest
import torch

from caffe_rtpose_b200 import engine, synth
from oracle import orc
from test_gpu_conv_layers import (Blobs, checked_layers, conv_ref, frames_for, layer_class, level_geo, sample_pixels,
                                  tc_instance, weights_with_biases)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "caffe_rtpose_b200", "rtpose.bin")
U = 2.0 ** -24
B_F1 = 2.0 ** -10 + 2.0 ** -17
F1 = engine.PREC_F16X1

# name -> (model, net_w, net_h, frame counts)
CONFIGS = {"coco_f1": (engine.COCO_18, 656, 368, (1, 2)), "mpi_f1": (engine.MPI_15, 496, 368, (1, 3))}
# largest |got - ref| / mag per layer class, about 2x the values measured on an H100 80GB HBM3 (700 W power limit) over both
# configurations and tile widths: 7x7 9.1e-5, 3x3 2.0e-4, 1x1 4.5e-4, conv1_1 (im2col) 5.3e-4; for conv1_1 B is the tighter
MEASURED_MAX = {"7x7": 2e-4, "3x3": 4.5e-4, "1x1": 9e-4, "im2col": 1.1e-3}
# max |maps - oracle| / max |oracle| at 160x96, about 3x the largest measured value (same card): COCO 1.7e-3 / 1.9e-3, MPI
# 1.8e-3 / 1.5e-3 (two scales), calibrated filler net 1.0e-3, calibrated 1.6x-per-layer net 2.1e-3
TOL_NET = 6e-3


def rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


def check_layer(layer, blobs, W, pts, scale_floor):
    w, b = W[layer["name"]]
    x, y = blobs.get(layer["bottom"]), blobs.get(layer["top"])
    ref, mag = conv_ref(x, w, b, pts, layer["relu"])
    got = y[pts[:, 0], :, pts[:, 1], pts[:, 2]].astype(np.float64)
    err = np.abs(got - ref)
    bad = err > B_F1 * mag + U * scale_floor
    assert not bad.any(), "%s: %d of %d elements outside B x mag; worst err/mag %.3e" % (layer["name"], int(bad.sum()), bad.size,
                                                                                       float((err / mag).max()))
    return float((err / mag).max())


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_conv_layers_vs_float64(cfg):
    model, net_w, net_h, counts = CONFIGS[cfg]
    W = weights_with_biases(model)
    eng = engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=F1, max_batch=max(counts))
    eng.set_weights(W)
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(11)
    worst = {}
    for n in counts:
        eng.forward_frames(frames_for(n, 2 * net_w, 2 * net_h))
        blobs = Blobs(eng, n, model, W)
        for layer in checked_layers(model):
            w_, h_, gap = level_geo(net_w, net_h, layer["level"])
            r = check_layer(layer, blobs, W, sample_pixels(n, h_, w_, gap, rng), 1.0)
            ks = 1 if layer["name"] == "conv1_1" else layer["k"]
            bn = tc_instance(W[layer["name"]][0].shape[0], ks, n * (h_ + gap) * (w_ + gap), 1, nsm)[0]
            key = (layer_class(layer), bn)
            worst[key] = max(worst.get(key, 0.0), r)
    eng.close()
    print("\n%s: largest |got - ref| / mag per (layer class, BN):" % cfg)
    for key in sorted(worst, key=str):
        print("  %-7s BN=%-4d %.3e" % (key[0], key[1], worst[key]))
    if MEASURED_MAX is not None:
        over = {k: v for k, v in worst.items() if v > MEASURED_MAX[k[0]]}
        assert not over, "accumulation error above what this kernel measured: %s" % over


def test_configs_launch_every_f16x1_instance():
    """Restating the tile-width rule of tc_layer_launch: the configurations above launch conv_wg_kernel<BN, 1, fp16> at every
    width the rule can pick, each filter size at full and half width."""
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    seen = set()
    for model, net_w, net_h, counts in CONFIGS.values():
        W = synth.make_weights(model)
        for n in counts:
            for layer in checked_layers(model):
                w_, h_, gap = level_geo(net_w, net_h, layer["level"])
                ks = 1 if layer["name"] == "conv1_1" else layer["k"]
                bn, _, rows = tc_instance(W[layer["name"]][0].shape[0], ks, n * (h_ + gap) * (w_ + gap), 1, nsm)
                seen |= {(bn, layer_class(layer)), (bn, rows)}
    want = {(128, c) for c in ("7x7", "3x3", "1x1")} | {(64, c) for c in ("7x7", "3x3", "1x1", "im2col")}
    want |= {(48, "1x1"), (32, "1x1"), (16, "1x1"), (128, 136), (64, 136), (128, 128), (64, 128)}
    assert want <= seen, sorted(want - seen, key=str)


@pytest.mark.parametrize("model", [engine.COCO_18, engine.MPI_15])
def test_whole_net_vs_oracle(model):
    """160x96, two scales: stride-8 maps against the oracle; frame k of a batch equals frame k alone; the third call (CUDA-graph
    replay) equals the eager forward; the planar net-input path equals the frame path."""
    net_w, net_h, S = 160, 96, 2
    W = synth.make_weights(model, "he", seed=7)
    frames = [synth.make_frame(20 + i, 192, 320) for i in range(2)]
    onet = orc.Net(model)
    onet.set_weights(W)
    x = [orc.preprocess(f, net_h, net_w, S, 1.0, 0.25) for f in frames]
    eng = engine.PoseEngine(model, net_w, net_h, 320, 192, num_scales=S, start_scale=1.0, scale_gap=0.25, precision=F1, max_batch=2)
    eng.set_weights(W)
    calls = []
    for _ in range(3):
        eng.forward_frames(frames)
        calls.append((eng.fetch_maps(2).copy(), [eng.fetch(k) for k in range(2)]))
    maps = calls[0][0]
    errs = [rel(maps[i * S:(i + 1) * S], onet.forward(x[i])) for i in range(2)]
    print("\nF16X1 %s 160x96 S=2: maps vs oracle %s" % ("COCO" if model == engine.COCO_18 else "MPI", ["%.3e" % e for e in errs]))
    assert max(errs) < TOL_NET
    assert np.array_equal(calls[2][0], maps)
    for (na, ja, pa), (nb, jb, pb) in zip(calls[2][1], calls[0][1]):
        assert na == nb and np.array_equal(ja, jb) and np.array_equal(pa, pb)
    for k in range(2):
        eng.forward_frames([frames[k]])
        assert np.array_equal(eng.fetch_maps(1), maps[k * S:(k + 1) * S]), k
    eng.forward_net_input(np.concatenate(x))
    assert np.array_equal(eng.fetch_maps(2), maps)
    eng.close()


@pytest.mark.parametrize("kind", ["caffe_filler", "growing"])
def test_range_reported_and_calibrated(kind):
    model, net_w, net_h = engine.COCO_18, 160, 96
    if kind == "caffe_filler":
        W = synth.make_weights(model, "caffe")
    else:
        W = {k: (w * np.float32(1.6), b) for k, (w, b) in synth.make_weights(model, "he").items()}
    frame = synth.make_frame(3, 2 * net_h, 2 * net_w)
    onet = orc.Net(model)
    onet.set_weights(W)
    omaps = onet.forward(orc.preprocess(frame, net_h, net_w, 1, 1.0, 0.3))
    eng = engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=F1)
    eng.set_weights(W)
    eng.forward_frames([frame])
    eng.sync()
    rc, worst, layer = eng.range_status()
    assert rc == 5 and layer, (rc, worst, layer)              # PE_ERR_RANGE, the layer named
    eng.calibrate([frame])
    err = rel(eng.fetch_maps(1), omaps)
    print("\nF16X1 calibrated %s: maps vs oracle %.3e" % (kind, err))
    assert err < TOL_NET
    for _ in range(3):
        eng.forward_frames([frame])
    rc, worst, layer = eng.range_status()
    assert rc == 0 and worst < 0.05, (rc, worst, layer)
    eng.close()


def test_compare_results_parity_self_and_simt_on_injected_maps():
    model = engine.COCO_18
    frame = synth.make_frame(5, 192, 320)
    e = engine.PoseEngine(model, 160, 96, 320, 192, precision=engine.PREC_F16X2)
    e.set_weights(synth.make_weights(model, "he"))
    e.forward_frames([frame])
    a = e.fetch(0)
    e.forward_frames([frame])
    d = engine.compare_results(a, e.fetch(0), 1e-3)
    assert d["identical"] and d["persons_matched"] == a[0], d
    e.close()
    people = synth.make_people(model, 6, 320, 176, seed=4)
    maps8 = synth.make_maps(model, people, 320, 176, seed=4)
    res = []
    for prec in (engine.PREC_FP32_SIMT, engine.PREC_F16X2):
        e = engine.PoseEngine(model, 320, 176, 640, 352, precision=prec)
        e.forward_maps(maps8)
        res.append(e.fetch(0))
        e.close()
    d = engine.compare_results(res[0], res[1], 1e-3)
    assert d["identical"] and res[0][0] >= 3 and d["persons_matched"] == res[0][0], d


def test_share_weights_f16x1_bit_identical():
    model = engine.COCO_18
    e0 = engine.PoseEngine(model, 160, 96, 320, 192, precision=F1)
    e1 = engine.PoseEngine(model, 160, 96, 320, 192, precision=F1)
    e0.set_weights(synth.make_weights(model, "he"))
    engine.share_weights(e0, e1)
    frame = synth.make_frame(6, 192, 320)
    out = []
    for e in (e0, e1):
        e.forward_frames([frame])
        n, j, p = e.fetch(0)
        out.append((n, j, p, e.fetch_maps(1)))
    assert out[0][0] == out[1][0] and all(np.array_equal(a, b) for a, b in zip(out[0][1:], out[1][1:]))
    e2 = engine.PoseEngine(model, 160, 96, 320, 192, precision=engine.PREC_F16X2)
    with pytest.raises(engine.PoseEngineError):
        engine.share_weights(e0, e2)
    for e in (e0, e1, e2):
        e.close()


def write_bmp(path, bgr):
    h, w, _ = bgr.shape
    row = (w * 3 + 3) // 4 * 4
    data = np.zeros((h, row), np.uint8)
    data[:, :w * 3] = bgr[::-1].reshape(h, w * 3)
    hdr = b"BM" + (54 + data.size).to_bytes(4, "little") + b"\0\0\0\0" + (54).to_bytes(4, "little")
    hdr += (40).to_bytes(4, "little") + w.to_bytes(4, "little") + h.to_bytes(4, "little") + (1).to_bytes(2, "little")
    hdr += (24).to_bytes(2, "little") + b"\0" * 24
    with open(path, "wb") as f:
        f.write(hdr + data.tobytes())


def test_cli_audit(tmp_path):
    """rtpose.bin --precision 4: the JSON of the Python F16X1 path on the same frames and weights; --audit_every 1 prints the
    audit status and summary lines and leaves the JSON unchanged."""
    model, n = engine.COCO_18, 30
    W = synth.make_weights(model, "he", seed=3)
    cm = tmp_path / "w.caffemodel"
    engine.write_caffemodel(str(cm), W, synth.conv_table(model))
    imgs = tmp_path / "imgs"
    imgs.mkdir()
    frames = [synth.make_frame(100 + i, 192, 320) for i in range(n)]
    for i, f in enumerate(frames):
        write_bmp(str(imgs / ("f%03d.bmp" % i)), f)
    common = [BIN, "--image_dir", str(imgs), "--caffemodel", str(cm), "--model", "COCO", "--resolution", "320x192",
              "--net_resolution", "160x96", "--no_frame_drops", "--no_display", "--precision", "4", "--calibrate_range=false"]
    outs = []
    for audit in (False, True):
        out = tmp_path / ("json_audit%d" % audit)
        r = subprocess.run(common + ["--write_json", str(out)] + (["--audit_every", "1"] if audit else []), capture_output=True,
                           text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        assert ("Audit:" in r.stderr and "Audit summary: " in r.stderr) is audit, r.stderr[-2000:]
        if audit:
            print("\n" + "\n".join(l for l in r.stderr.splitlines() if "Audit" in l))
        outs.append(out)
    eng = engine.PoseEngine(model, 160, 96, 320, 192, precision=F1)
    eng.set_weights(W)
    for i, f in enumerate(frames):
        eng.forward_frames([f])
        cnt, joints, _ = eng.fetch(0)
        want = eng.json(joints)
        for out in outs:
            assert (out / ("f%03d.json" % i)).read_text() == want, (out, i)
    eng.close()
