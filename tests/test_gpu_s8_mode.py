"""The INT8 mode (PE_PREC_S8X1: one s8 plane of activations and weights, one s8 MMA per MAC, exact s32 sums) on the GPU.

Every s8 layer is a deterministic function of integers followed by fixed fp32 operations (poseengine.h), so it is checked bit
for bit.  A layer's input integers are pe_fetch_blob of its bottom times 2^k (pe_blob_log2_scale; a Concat input takes each
part's own k).  The reference folds 2^-k of every input channel into the fp32 weights (exact), quantises each output channel
as the packer does (sigma_c = max|w| / 127, q = clamp(rint(w / sigma_c), -127, 127), in float32), sums the integer products
in float64 (exact: |acc| <= 128 x 127 x K < 2^53), and applies the epilogue in float32 without FMA:
    t = fl(fl(float32(acc) * f_c) + b'_c),  f_c = sigma_c * 2^k_out,  b'_c = b_c * 2^k_out,  ReLU,  q = clip(rint(t), -128, 127).
The stored output must equal q * 2^-k_out; the layers that write the fp32 maps (k_out = 0) must equal t.  Folding 2^-k of the
input into the weights instead of the engine's ratio to one reference channel scales every weight of an output channel by the
same power of two, which changes neither q nor f_c.

Whole net, max pool, range, calibration, replay, weight sharing, the accumulator bound and the CLI: see the tests below.
"""
import os
import subprocess

import numpy as np
import pytest
import torch

from caffe_rtpose_b200 import engine, synth
from oracle import orc
from test_conv_shapes import spec_weights
from test_gpu_conv_layers import (Blobs, checked_layers, conv_layers, frames_for, layer_class, level_geo, netspec, plan_gaps,
                                  sample_pixels, tc_cout_pad, weights_with_biases)
from test_prototxt import spec_prototxt

pytestmark = pytest.mark.gpu
S8 = engine.PREC_S8X1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "caffe_rtpose_b200", "rtpose.bin")
# name -> (model or prototxt netspec, net_w, net_h, frames per forward).  One frame at 656x368 runs the stride-8 layers at half
# width (BN 64), nine frames at 320x176 at full width (BN 128).
CONFIGS = {"coco_1": (engine.COCO_18, 656, 368, 1), "coco_9": (engine.COCO_18, 320, 176, 9), "mpi_1": (engine.MPI_15, 496, 368, 1),
           "mpi2_proto_1": ("mpi_2", 240, 176, 1)}
# max |maps - oracle| / max |oracle| at 160x96, calibrated, about 2x the largest value measured on an H100 80GB HBM3 (700 W power
# limit): COCO 0.141-0.152 and MPI 0.130-0.181 (frames 0 / 1, one and two scales); see test_whole_net_vs_oracle
TOL_NET = 0.35


def rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


def quantize(w):
    """Per output channel (axis 0) of float32 weights: (sigma float32 (co,), q float64 of w's shape)."""
    w = np.asarray(w, np.float32)
    flat = w.reshape(w.shape[0], -1)
    sigma = (np.abs(flat).max(axis=1) / np.float32(127)).astype(np.float32)
    safe = np.where(sigma > 0, sigma, np.float32(1))
    q = np.where(sigma[:, None] > 0, np.clip(np.rint(flat / safe[:, None]), -127, 127), 0.0)
    return sigma, q.reshape(w.shape).astype(np.float64)


def fold(w, k_in):
    """w (co, ci, k, k) float32 with 2^-k_in of every input channel folded in (exact)."""
    return (np.asarray(w, np.float32) * np.ldexp(np.float32(1), -np.asarray(k_in))[None, :, None, None].astype(np.float32)).astype(np.float32)


def epilogue(acc, sigma, b, k_out, relu, planar):
    """The kernel's epilogue on float64 integer sums acc (..., co): the stored integers (or t for the planar maps)."""
    f = (sigma * np.float32(2.0 ** k_out)).astype(np.float32)
    bb = (np.asarray(b, np.float32) * np.float32(2.0 ** k_out)).astype(np.float32)
    t = (acc.astype(np.float32) * f).astype(np.float32)
    t = (t + bb).astype(np.float32)
    if relu:
        t = np.maximum(t, np.float32(0))
    return t.astype(np.float64) if planar else np.clip(np.rint(t), -128, 127).astype(np.float64)


def int_acc_at(xint, q, pts):
    """sum of integer products of a 'same' convolution at sampled output pixels pts (n, y, x): float64 (P, co), exact."""
    co, ci, k, _ = q.shape
    p = k // 2
    xp = np.pad(xint, ((0, 0), (0, 0), (p, p), (p, p)))
    n, yy, xx = pts[:, 0], pts[:, 1], pts[:, 2]
    acc = np.zeros((len(pts), co))
    for r in range(k):
        for s in range(k):
            acc += xp[n, :, yy + r, xx + s] @ q[:, :, r, s].T
    return acc


def int_conv_full(xint, q):
    """The whole 'same' convolution of integer float64 tensors on the CPU in float64 (im2col + GEMM: exact)."""
    k = q.shape[2]
    return torch.nn.functional.conv2d(torch.from_numpy(xint), torch.from_numpy(q), padding=k // 2).numpy()


class IntBlobs:
    """The stored integers and their k of the blobs of an engine's last forward (first nimg images)."""

    def __init__(self, eng, nimg, model, W, spec=None):
        self.eng, self.blobs = eng, Blobs(eng, nimg, model, W, spec)
        self.concat = self.blobs.concat

    def k(self, name):
        if name in self.concat:
            return np.concatenate([np.full(self.blobs.get(b).shape[1], self.eng.blob_log2_scale(b)) for b in self.concat[name]])
        return np.full(self.blobs.get(name).shape[1], self.eng.blob_log2_scale(name))

    def ints(self, name):
        x = self.blobs.get(name).astype(np.float64)
        v = x * np.ldexp(1.0, self.k(name))[None, :, None, None]
        assert np.array_equal(v, np.rint(v)) and np.abs(v).max() <= 128, name
        return v


def check_layer(layer, ib, W, pts):
    """Bit-exact check of one conv layer at sampled pixels; returns (the number of compared values, the largest |acc|)."""
    w, b = W[layer["name"]]
    sigma, q = quantize(fold(w, ib.k(layer["bottom"])))
    acc = int_acc_at(ib.ints(layer["bottom"]), q, pts)
    planar = layer["top"] in ib.blobs.final_off
    k_out = 0 if planar else ib.eng.blob_log2_scale(layer["top"])
    want = epilogue(acc, sigma, b, k_out, layer["relu"], planar)
    y = ib.blobs.get(layer["top"])
    got = y[pts[:, 0], :, pts[:, 1], pts[:, 2]].astype(np.float64)
    got = got if planar else got * 2.0 ** k_out
    bad = got != want
    if bad.any():
        i, c = np.argwhere(bad)[0]
        raise AssertionError("%s: %d of %d values differ; first at (n, y, x) = %s channel %d: got %.9g, want %.9g (k_out %d)"
                             % (layer["name"], int(bad.sum()), bad.size, tuple(pts[i]), c, got[i, c], want[i, c], k_out))
    return bad.size, float(np.abs(acc).max())


def make_engine(cfg, tmp_path, W=None):
    model, net_w, net_h, n = CONFIGS[cfg]
    spec, path = spec_prototxt(model, tmp_path) if isinstance(model, str) else (None, None)
    m = engine.MPI_15 if path else model
    W = W or (spec_weights(spec) if spec else weights_with_biases(m))
    eng = engine.PoseEngine(None if path else m, net_w, net_h, 2 * net_w, 2 * net_h, precision=S8, max_batch=n, prototxt=path)
    eng.set_weights(W)
    return eng, m, spec, W, path


def tc_bn(cout, M, nsm, share=2):
    """The tile width of tc_layer_launch for one plane (full width up to 128, half when it fills more SMs)."""
    cp = tc_cout_pad(cout)
    bn = min(cp, 128)
    mt = (M + 127) // 128
    sms = max(1, nsm // share)
    if bn >= 64 and min(mt * (cp // (bn // 2)), sms) * 0.80 > min(mt * (cp // bn), sms) * 1.00:
        bn //= 2
    return bn


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_conv_layers_bit_exact(cfg, tmp_path):
    eng, model, spec, W, path = make_engine(cfg, tmp_path)
    _, net_w, net_h, n = CONFIGS[cfg]
    frames = frames_for(n, 2 * net_w, 2 * net_h)
    eng.calibrate(frames[:1])
    eng.forward_frames(frames)
    gaps = plan_gaps(prototxt=path) if path else None
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    ib = IntBlobs(eng, n, None if path else model, W, spec)
    rng = np.random.default_rng(11)
    layers = conv_layers(None, spec)[0] if spec else checked_layers(model)
    seen, count = set(), 0
    for layer in layers:
        w_, h_, gap = level_geo(net_w, net_h, layer["level"], gaps)
        count += check_layer(layer, ib, W, sample_pixels(n, h_, w_, gap, rng, 300))[0]
        seen.add((layer_class(layer), tc_bn(W[layer["name"]][0].shape[0], n * (h_ + gap) * (w_ + gap), nsm)))
    eng.close()
    print("\n%s: %d layers, %d values bit-exact; (layer class, BN) run: %s" % (cfg, len(layers), count, sorted(seen, key=str)))


def test_configs_run_both_tile_widths():
    """Restating the width rule: the configurations above run the 7x7 and 3x3 layers at full and half width, and the 1x1 map
    layers at BN 16 - 48."""
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    seen = set()
    for cfg, (model, net_w, net_h, n) in CONFIGS.items():
        if isinstance(model, str):
            continue
        W = synth.make_weights(model)
        for layer in checked_layers(model):
            w_, h_, gap = level_geo(net_w, net_h, layer["level"])
            seen.add((tc_bn(W[layer["name"]][0].shape[0], n * (h_ + gap) * (w_ + gap), nsm), layer_class(layer)))
    want = {(128, "7x7"), (64, "7x7"), (128, "3x3"), (64, "3x3"), (128, "1x1"), (48, "1x1"), (32, "1x1"), (16, "1x1")}
    assert want <= seen, sorted(want - seen, key=str)


def whole_stack(spec, W, eng, nimg):
    """The net of the layer table `spec` (netspec format) in integers up to its final Concat from the engine's stored input
    (pe_fetch_blob of the input x 2^8): every conv as in check_layer over the whole image (each at the k the engine
    calibrated), 2x2 max pooling (ceil mode) and Concat."""
    convs, concat, final = conv_layers(None, spec)
    spec_layers = [l for l in spec["layers"] if l["type"] == "Pooling"]
    inp = spec["input"]
    k = {inp: eng.blob_log2_scale(inp)}
    val = {inp: eng.fetch_blob(inp)[:nimg].astype(np.float64) * 2.0 ** k[inp]}
    pools = {l["top"][0]: l["bottom"][0] for l in spec_layers}

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
            sigma, q = quantize(fold(w, kin))
            acc = int_conv_full(x, q).transpose(0, 2, 3, 1)
            planar = name in concat[final]
            kk = 0 if planar else eng.blob_log2_scale(name)
            val[name] = epilogue(acc, sigma, b, kk, layer["relu"], planar).transpose(0, 3, 1, 2)
            k[name] = kk
        return val[name], k[name]

    by_top = {l["top"]: l for l in convs}
    return np.concatenate([get(b)[0] for b in concat[final]], axis=1)


@pytest.mark.parametrize("model", [engine.COCO_18, engine.MPI_15])
def test_whole_stack_bit_exact(model):
    """160x96, calibrated, two frames: the integer chain of every layer, max pool and Concat from the stored net input equals
    pe_fetch_maps bit for bit."""
    net_w, net_h = 160, 96
    W = weights_with_biases(model)
    frames = [synth.make_frame(30 + i, 2 * net_h, 2 * net_w) for i in range(2)]
    eng = engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=S8, max_batch=2)
    eng.set_weights(W)
    eng.calibrate(frames[:1])
    eng.forward_frames(frames)
    maps = eng.fetch_maps(2).astype(np.float64)
    want = whole_stack(netspec(model), W, eng, 2)
    eng.close()
    bad = maps != want
    assert not bad.any(), "%d of %d map values differ, max |diff| %.3g" % (int(bad.sum()), bad.size, float(np.abs(maps - want).max()))


def test_max_pool_exact(tmp_path):
    """Every pool top equals the 2x2 max (ceil mode) of its s8 input exactly."""
    eng, model, _, W, _ = make_engine("coco_1", tmp_path)
    frames = frames_for(1, 2 * 656, 2 * 368)
    eng.calibrate(frames)
    eng.forward_frames(frames)
    for bottom, top in (("conv1_2", "pool1_stage1"), ("conv2_2", "pool2_stage1"), ("conv3_4", "pool3_stage1")):
        x, y = eng.fetch_blob(bottom)[:1], eng.fetch_blob(top)[:1]
        assert eng.blob_log2_scale(bottom) == eng.blob_log2_scale(top)
        H, Wd = x.shape[2], x.shape[3]
        xp = np.full((1, x.shape[1], (H + 1) // 2 * 2, (Wd + 1) // 2 * 2), -np.inf, np.float32)
        xp[:, :, :H, :Wd] = x
        want = xp.reshape(1, x.shape[1], xp.shape[2] // 2, 2, xp.shape[3] // 2, 2).max(axis=(3, 5))
        assert np.array_equal(y, want), top
    eng.close()


@pytest.mark.parametrize("S", [1, 2])
@pytest.mark.parametrize("model", [engine.COCO_18, engine.MPI_15])
def test_whole_net_vs_oracle(model, S):
    """Calibrated, 160x96: stride-8 maps against the oracle (fp32), and the same batch three times (the second is captured
    into a CUDA graph, the third replays it) gives bit-identical maps, peaks and joints.

    Tolerance: every layer rounds its output to a step 2^-k with the stored maximum in [32, 64), an absolute error of up to
    2^-7 of the layer's maximum (half a step against a maximum of at least 64 half-steps), and its weights to half of sigma_c,
    2^-8 of the channel's largest weight.  Most activations are a small fraction of their layer's maximum, so relative to
    the values themselves these roundings are far coarser than the e4m3 mode's 2^-4, and they compound over the 20 (MPI) to
    52 (COCO) layers of the deepest path.  Measured 0.130-0.181 of the map maximum (TOL_NET); held to about twice that, which
    stays below the e4m3 mode's bound (0.5)."""
    net_w, net_h = 160, 96
    W = synth.make_weights(model, "he", seed=7)
    frames = [synth.make_frame(20 + i, 192, 320) for i in range(2)]
    onet = orc.Net(model)
    onet.set_weights(W)
    omaps = [onet.forward(orc.preprocess(f, net_h, net_w, S, 1.0, 0.25)) for f in frames]
    eng = engine.PoseEngine(model, net_w, net_h, 320, 192, num_scales=S, start_scale=1.0, scale_gap=0.25, precision=S8, max_batch=2)
    eng.set_weights(W)
    eng.calibrate(frames)
    calls = []
    for _ in range(3):
        eng.forward_frames(frames)
        calls.append((eng.fetch_maps(2).copy(), [eng.fetch(k) for k in range(2)]))
    maps = calls[0][0]
    errs = [rel(maps[i * S:(i + 1) * S], omaps[i]) for i in range(2)]
    print("\nS8X1 %s 160x96 S=%d: maps vs oracle %s" % ("COCO" if model == engine.COCO_18 else "MPI", S, ["%.3e" % e for e in errs]))
    assert max(errs) < TOL_NET
    for c in calls[1:]:
        assert np.array_equal(c[0], maps)
        for (na, ja, pa), (nb, jb, pb) in zip(c[1], calls[0][1]):
            assert na == nb and np.array_equal(ja, jb) and np.array_equal(pa, pb)
    rc, worst, layer = eng.range_status()
    assert rc == 0 and 0 < worst < 1, (rc, worst, layer)
    eng.close()


def test_calibration_required_and_range():
    """A forward before pe_calibrate is PE_ERR_STATE naming pe_calibrate.  After it the range is within bounds: the calibration
    frame's stored maxima lie in [32, 64) (ratio to 127 in [0.25, 0.5]).  A handle calibrated on a flat grey frame and then
    given a busy frame leaves the s8 range: PE_ERR_RANGE with a layer named."""
    model, net_w, net_h = engine.COCO_18, 160, 96
    W = synth.make_weights(model, "he")
    busy = synth.make_frame(3, 2 * net_h, 2 * net_w)
    eng = engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=S8)
    eng.set_weights(W)
    with pytest.raises(engine.PoseEngineError, match="pe_calibrate"):
        eng.forward_frames([busy])
    eng.calibrate([busy])
    eng.forward_frames([busy])
    rc, worst, layer = eng.range_status()
    assert rc == 0 and 0.25 <= worst < 64.5 / 127, (rc, worst, layer)
    assert eng.blob_log2_scale("image") == 8
    eng.close()
    grey = np.full((2 * net_h, 2 * net_w, 3), 100, np.uint8)   # a flat net input of -28 / 256
    eng = engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=S8)
    eng.set_weights(W)
    eng.calibrate([grey])
    eng.range_status()
    eng.forward_frames([busy])
    eng.sync()
    rc, worst, layer = eng.range_status()
    print("\nS8X1 calibrated on grey, busy frame: rc %d, worst %.3g, layer %s" % (rc, worst, layer))
    assert rc == 5 and layer, (rc, worst, layer)
    assert layer in {l[0] for l in eng.conv_layers()}
    eng.close()


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


def calibrated_source(device=0):
    model, net_w, net_h = engine.COCO_18, 160, 96
    frame = synth.make_frame(5, 2 * net_h, 2 * net_w)
    e0 = engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=S8, device=device)
    e0.set_weights(synth.make_weights(model, "he"))
    e0.calibrate([frame])
    return e0, frame, lambda dev: engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=S8, device=dev)


def test_share_weights_bit_identical():
    """A pe_share_weights handle runs on the calibrated source's packed buffer and gives its maps, peaks, joints and blobs
    bit for bit."""
    e0, frame, make = calibrated_source()
    e1 = make(0)
    engine.share_weights(e0, e1)
    forward_results([e0, e1], frame)


def test_broadcast_weights_bit_identical():
    """A pe_broadcast_weights replica on a second GPU gives the calibrated source's results bit for bit."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    e0, frame, make = calibrated_source()
    e2 = make(1)
    engine.broadcast_weights([e0, e2])
    forward_results([e0, e2], frame)


def test_accumulator_bound_refused(tmp_path):
    """A generated prototxt whose 7x7 layer reads 2700 channels (K = 49 x 2816 padded > 132104) fails pe_create_from_prototxt at
    precision 6 with PE_ERR_INVALID naming the layer; the same file builds at precision 2."""
    from test_conv_shapes import pose_spec
    spec = pose_spec(engine.MPI_15, 16, 16, conv1_1=8, levels=[[(3, 8)], [(3, 8)], [(3, 8)], [(1, 2700), (7, 16)]], branch=[(1, 8)])
    path = tmp_path / "big_k.prototxt"
    path.write_text(synth.netspec_to_prototxt(spec))
    with pytest.raises(engine.PoseEngineError, match="conv4_2") as ex:
        engine.PoseEngine(None, 16, 16, 32, 32, precision=S8, prototxt=str(path))
    assert "132104" in str(ex.value)
    eng = engine.PoseEngine(None, 16, 16, 32, 32, precision=engine.PREC_F16X2, prototxt=str(path))
    assert "conv4_2" in {l[0] for l in eng.conv_layers()}
    eng.close()


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


def test_cli_precision_6(tmp_path):
    """rtpose.bin --precision 6 (calibrated at start-up) writes one JSON per frame of an --image_dir; --audit_every 1 prints
    its comparison with the parity mode (the summary line) and leaves the JSON unchanged."""
    model, n = engine.COCO_18, 6
    W = synth.make_weights(model, "he", seed=3)
    cm = tmp_path / "w.caffemodel"
    engine.write_caffemodel(str(cm), W, synth.conv_table(model))
    imgs = tmp_path / "imgs"
    imgs.mkdir()
    for i in range(n):
        write_bmp(str(imgs / ("f%03d.bmp" % i)), synth.make_frame(100 + i, 192, 320))
    common = [BIN, "--image_dir", str(imgs), "--caffemodel", str(cm), "--model", "COCO", "--resolution", "320x192",
              "--net_resolution", "160x96", "--no_frame_drops", "--no_display", "--precision", "6"]
    outs = []
    for audit in (False, True):
        out = tmp_path / ("json_audit%d" % audit)
        r = subprocess.run(common + ["--write_json", str(out)] + (["--audit_every", "1"] if audit else []), capture_output=True,
                           text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        assert ("Audit summary: " in r.stderr) is audit, r.stderr[-2000:]
        if audit:
            print("\n" + "\n".join(l for l in r.stderr.splitlines() if "Audit" in l))
        outs.append(out)
    for i in range(n):
        a, b = [(o / ("f%03d.json" % i)).read_text() for o in outs]
        assert a == b and a.startswith("{"), (i, a[:200])
