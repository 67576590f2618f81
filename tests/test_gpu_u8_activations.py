"""u8 activations in the INT8 mode (PE_PREC_S8X1 | PE_PREC_FLAG_U8) on the GPU.

Every integer layer is checked bit for bit with the integer reference of tests/test_gpu_s8_mode.py: the input integers are
pe_fetch_blob x 2^k (u8 inputs in [0, 255], s8 in [-128, 127]), the weights are quantised per channel, the products summed in
float64 (exact: |acc| <= 255 x 127 x K < 2^53), and the epilogue t = fl(fl(float32(acc) * f_c) + b'_c), ReLU, runs in float32
without FMA.  The stored value is rint(t) clipped to [0, 255] for a u8 output and to [-128, 127] for an s8 output, t itself for
the fp32 maps and t rounded to fp16 for the fp16 outputs of a mixed engine.  The fp16 layers of mixed engines are held to the
fp16 accumulation bound of tests/test_gpu_mixed_precision.py.

Whole stack, pools, generated graphs, calibration and tables, CUDA-graph replay, weight sharing, the accumulator bound, the
whole net against the oracle (beside S8X1 in the same run) and the CLI: see the tests below.
"""
import os
import subprocess

import numpy as np
import pytest
import torch

from caffe_rtpose_b200 import engine, synth
from oracle import orc
from test_conv_shapes import CASES, FRAMES, pose_spec, write_prototxt
from test_gpu_conv_layers import Blobs, checked_layers, conv_layers, conv_ref, frames_for, level_geo, netspec, plan_gaps, sample_pixels
from test_gpu_conv_layers import weights_with_biases
from test_gpu_mixed_precision import B_F16, float_layer, packed
from test_gpu_s8_mode import CONFIGS, TOL_NET, epilogue, fold, int_acc_at, int_conv_full, quantize, rel, write_bmp
from test_gpu_s8_shapes import case_weights
from test_conv_shapes import spec_weights
from test_prototxt import spec_prototxt

pytestmark = pytest.mark.gpu
S8 = engine.PREC_S8X1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "caffe_rtpose_b200", "rtpose.bin")
SEVEN = ["Mconv%d_stage%d_L%d" % (i, s, b) for s in range(2, 7) for i in range(1, 6) for b in (1, 2)] + ["conv5_1_CPM_L1", "conv5_1_CPM_L2"]
LIMITS = {"u8": (0, 255), "s8": (-128, 127)}


def u8_engine(model, net_w, net_h, n=1, **kw):
    return engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=S8, max_batch=n, u8_activations=True, **kw)


def formats(model, path=None, f16=None):
    return engine.plan_formats(model if path is None else None, S8, f16, prototxt=path, u8_activations=True)


class KindBlobs:
    """The stored integers and their k of the blobs of an engine's last forward (first nimg images), each checked against the
    range of its stored kind."""

    def __init__(self, eng, nimg, model, W, fm, spec=None):
        self.eng, self.blobs = eng, Blobs(eng, nimg, model, W, spec)
        self.concat = self.blobs.concat
        self.kind = {a[2]: a[0] for a in fm["acts"] if a[2]}

    def k(self, name):
        if name in self.concat:
            return np.concatenate([np.full(self.blobs.get(b).shape[1], self.eng.blob_log2_scale(b)) for b in self.concat[name]])
        return np.full(self.blobs.get(name).shape[1], self.eng.blob_log2_scale(name))

    def ints(self, name):
        v = self.blobs.get(name).astype(np.float64) * np.ldexp(1.0, self.k(name))[None, :, None, None]
        lo, hi = LIMITS[self.kind.get(name, "s8")]
        assert np.array_equal(v, np.rint(v)) and v.min() >= lo and v.max() <= hi, (name, v.min(), v.max())
        return v


def store(t, kind):
    """The stored value of epilogue output t (float64 of float32) in `kind`."""
    if kind == "f32":
        return t
    if kind == "f16":
        return t.astype(np.float16).astype(np.float64)
    lo, hi = LIMITS[kind]
    return np.clip(np.rint(t), lo, hi)


def check_layer(layer, ib, W, out, pts):
    """Bit-exact check of an integer layer (s8 or u8 input) storing `out`; returns the number of compared values."""
    w, b = W[layer["name"]]
    sigma, q = quantize(fold(w, ib.k(layer["bottom"])))
    acc = int_acc_at(ib.ints(layer["bottom"]), q, pts)
    planar = out == "f32"
    k_out = 0 if planar else ib.eng.blob_log2_scale(layer["top"])
    want = store(epilogue(acc, sigma, b, k_out, layer["relu"], True), out)
    got = ib.blobs.get(layer["top"])[pts[:, 0], :, pts[:, 1], pts[:, 2]].astype(np.float64) * (1 if planar else 2.0 ** k_out)
    bad = got != want
    if bad.any():
        i, c = np.argwhere(bad)[0]
        raise AssertionError("%s (-> %s): %d of %d values differ; first at (n, y, x) = %s channel %d: got %.9g, want %.9g (k_out %d)"
                             % (layer["name"], out, int(bad.sum()), bad.size, tuple(pts[i]), c, got[i, c], want[i, c], k_out))
    return bad.size


def f16_to_u8_layer(layer, ib, W, pts):
    """An fp16 layer that stores u8: the float64 reference (fp16-packed weights) within B_F16 * mag of the rounding cell of the
    stored integer v (stored / 2^k): [v - 1/2, v + 1/2], open below at 0 and above at 255."""
    w, b = W[layer["name"]]
    kin = ib.k(layer["bottom"])
    r = np.ldexp(1.0, kin.max() - kin).astype(np.float32)
    wq = packed((w * r[None, :, None, None]).astype(np.float32), "f16") / r[None, :, None, None]
    ref, mag = conv_ref(ib.blobs.get(layer["bottom"]), wq, b, pts, layer["relu"])
    k = ib.eng.blob_log2_scale(layer["top"])
    v = ib.blobs.get(layer["top"])[pts[:, 0], :, pts[:, 1], pts[:, 2]].astype(np.float64) * 2.0 ** k
    lo = np.where(v <= 0, -np.inf, v - 0.5) * 2.0 ** -k
    hi = np.where(v >= 255, np.inf, v + 0.5) * 2.0 ** -k
    d = np.maximum(0.0, np.maximum(ref - hi, lo - ref))
    assert (d <= B_F16 * mag).all(), (layer["name"], float((d / mag).max()))
    return float((d / mag).max())


# ------------------------------------------------------------------------------------------ per layer
def make_engine(cfg, tmp_path):
    model, net_w, net_h, n = CONFIGS[cfg]
    spec, path = spec_prototxt(model, tmp_path) if isinstance(model, str) else (None, None)
    m = engine.MPI_15 if path else model
    W = spec_weights(spec) if spec else weights_with_biases(m)
    eng = u8_engine(None if path else m, net_w, net_h, n, prototxt=path)
    eng.set_weights(W)
    return eng, m, spec, W, path


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_conv_layers_bit_exact(cfg, tmp_path):
    eng, model, spec, W, path = make_engine(cfg, tmp_path)
    _, net_w, net_h, n = CONFIGS[cfg]
    fm = formats(model, path)
    frames = frames_for(n, 2 * net_w, 2 * net_h)
    eng.calibrate(frames[:1])
    eng.forward_frames(frames)
    gaps = plan_gaps(prototxt=path) if path else None
    ib = KindBlobs(eng, n, None if path else model, W, fm, spec)
    rng = np.random.default_rng(11)
    layers = conv_layers(None, spec)[0] if spec else checked_layers(model)
    count, pairs = 0, set()
    for layer in layers:
        comp, out = fm["convs"][layer["name"]][:2]
        w_, h_, gap = level_geo(net_w, net_h, layer["level"], gaps)
        count += check_layer(layer, ib, W, out, sample_pixels(n, h_, w_, gap, rng, 300))
        pairs.add((comp, out))
    eng.close()
    print("\n%s: %d layers, %d values bit-exact; (compute, stored): %s" % (cfg, len(layers), count, sorted(pairs)))
    assert {("u8", "u8"), ("s8", "u8"), ("u8", "f32")} <= pairs, pairs


def whole_stack(spec, W, eng, nimg, fm):
    """The integer chain of the net of `spec` from the stored net input to its final Concat (test_gpu_s8_mode.whole_stack) with
    each conv's output stored in the kind of the plan."""
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
            sigma, q = quantize(fold(w, kin))
            acc = int_conv_full(x, q).transpose(0, 2, 3, 1)
            out = fm["convs"][layer["name"]][1]
            kk = 0 if out == "f32" else eng.blob_log2_scale(name)
            val[name] = store(epilogue(acc, sigma, b, kk, layer["relu"], True), out).transpose(0, 3, 1, 2)
            k[name] = kk
        return val[name], k[name]

    return np.concatenate([get(b)[0] for b in concat[final]], axis=1)


@pytest.mark.parametrize("model", [engine.COCO_18, engine.MPI_15])
def test_whole_stack_bit_exact(model):
    """160x96, calibrated, two frames: the integer chain of every layer, max pool and Concat equals pe_fetch_maps bit for bit."""
    net_w, net_h = 160, 96
    W = weights_with_biases(model)
    frames = [synth.make_frame(30 + i, 2 * net_h, 2 * net_w) for i in range(2)]
    eng = u8_engine(model, net_w, net_h, 2)
    eng.set_weights(W)
    eng.calibrate(frames[:1])
    eng.forward_frames(frames)
    maps = eng.fetch_maps(2).astype(np.float64)
    want = whole_stack(netspec(model), W, eng, 2, formats(model))
    eng.close()
    bad = maps != want
    assert not bad.any(), "%d of %d map values differ, max |diff| %.3g" % (int(bad.sum()), bad.size, float(np.abs(maps - want).max()))


def test_max_pool_exact():
    """Every pool top (u8) equals the 2x2 max (ceil mode) of its u8 input exactly."""
    model, net_w, net_h = engine.COCO_18, 656, 368
    fm = formats(model)
    eng = u8_engine(model, net_w, net_h)
    eng.set_weights(weights_with_biases(model))
    frames = frames_for(1, 2 * net_w, 2 * net_h)
    eng.calibrate(frames)
    eng.forward_frames(frames)
    kinds = {a[2]: a[0] for a in fm["acts"] if a[2]}
    for bottom, top in (("conv1_2", "pool1_stage1"), ("conv2_2", "pool2_stage1"), ("conv3_4", "pool3_stage1")):
        assert kinds[bottom] == kinds[top] == "u8"
        x, y = eng.fetch_blob(bottom)[:1], eng.fetch_blob(top)[:1]
        assert eng.blob_log2_scale(bottom) == eng.blob_log2_scale(top)
        H, Wd = x.shape[2], x.shape[3]
        xp = np.full((1, x.shape[1], (H + 1) // 2 * 2, (Wd + 1) // 2 * 2), -np.inf, np.float32)
        xp[:, :, :H, :Wd] = x
        want = xp.reshape(1, x.shape[1], xp.shape[2] // 2, 2, xp.shape[3] // 2, 2).max(axis=(3, 5))
        assert np.array_equal(y, want) and y.min() >= 0, top
        assert (x * 2.0 ** eng.blob_log2_scale(bottom)).max() >= 64   # calibrated into [64, 128)
    eng.close()


@pytest.mark.parametrize("name", list(CASES))
def test_generated_convs_bit_exact(name, tmp_path):
    """Every conv of every generated case at one and three frames, and every pool top."""
    spec, path = write_prototxt(name, tmp_path)
    c = CASES[name]
    net_w, net_h = c["net_w"], c["net_h"]
    gaps = plan_gaps(prototxt=path)
    W = case_weights(name, spec)
    fm = formats(None, path)
    eng = engine.PoseEngine(None, net_w, net_h, 2 * net_w, 2 * net_h, start_scale=0.5, precision=S8, prototxt=path,
                            max_batch=max(FRAMES), u8_activations=True)
    eng.set_weights(W)
    eng.calibrate(frames_for(FRAMES[0], 2 * net_w, 2 * net_h))
    layers = conv_layers(None, spec)[0]
    rng = np.random.default_rng(11)
    for n in FRAMES:
        eng.forward_frames(frames_for(n, 2 * net_w, 2 * net_h))
        ib = KindBlobs(eng, n, None, W, fm, spec)
        for layer in layers:
            w_, h_, gap = level_geo(net_w, net_h, layer["level"], gaps)
            check_layer(layer, ib, W, fm["convs"][layer["name"]][1], sample_pixels(n, h_, w_, gap, rng, 200))
        for p in [l for l in spec["layers"] if l["type"] == "Pooling"]:
            bot = ib.blobs.get(p["bottom"][0])
            top = eng.fetch_blob(p["top"][0])[:n]
            N, C, H, Wd = bot.shape
            assert np.array_equal(top, bot.reshape(N, C, H // 2, 2, Wd // 2, 2).max(axis=(3, 5))), p["name"]
    eng.close()
    assert any(v[0] == "u8" for v in fm["convs"].values()), name


@pytest.mark.parametrize("f16", ["narrow", "seven"])
@pytest.mark.parametrize("model", [engine.COCO_18, engine.MPI_15])
def test_mixed_engines(model, f16):
    """S8X1 + u8 with `narrow` or the 7x7 group in fp16, calibrated, three frames at 320x176: the s8 and u8 layers bit for bit,
    the fp16 layers within the fp16 accumulation bound."""
    net_w, net_h, n = 320, 176, 3
    lst = "narrow" if f16 == "narrow" else SEVEN
    W = weights_with_biases(model)
    fm = formats(model, None, lst)
    eng = u8_engine(model, net_w, net_h, n, f16_layers=lst)
    eng.set_weights(W)
    frames = frames_for(n, 2 * net_w, 2 * net_h)
    eng.calibrate(frames[:1])
    eng.forward_frames(frames)
    rc, ratio, name = eng.range_status()
    assert rc == 0, (rc, ratio, name)
    ib = KindBlobs(eng, n, model, W, fm)
    rng = np.random.default_rng(11)
    pairs, worst = set(), 0.0
    for layer in checked_layers(model):
        comp, out = fm["convs"][layer["name"]][:2]
        w_, h_, gap = level_geo(net_w, net_h, layer["level"])
        pts = sample_pixels(n, h_, w_, gap, rng, 200)
        if comp in ("s8", "u8"):
            check_layer(layer, ib, W, out, pts)
        elif out == "u8":
            worst = max(worst, f16_to_u8_layer(layer, ib, W, pts))
        else:
            worst = max(worst, float_layer(layer, eng, ib.blobs, ib.k, W, comp, out, pts))
        pairs.add((comp, out))
    eng.close()
    print("\n%s + %s: (compute, stored) run: %s; fp16 layers: largest d / mag %.3e" % (
        "COCO" if model == engine.COCO_18 else "MPI", f16, sorted(pairs), worst))
    assert ("f16", "u8") in pairs and ("u8", "u8") in pairs
    if f16 == "seven":
        assert ("u8", "f16") in pairs


# ------------------------------------------------------------------------------------------ calibration
def outputs(eng, frames):
    eng.forward_frames(frames)
    res = [eng.fetch(i) for i in range(len(frames))]
    return eng.fetch_maps(len(frames)).copy(), [(c, j.copy(), p.copy()) for c, j, p in res]


def same_outputs(a, b):
    assert np.array_equal(a[0], b[0])
    for (ca, ja, pa), (cb, jb, pb) in zip(a[1], b[1]):
        assert ca == cb and np.array_equal(ja, jb) and np.array_equal(pa, pb)


def table_layers(t):
    return {l.split()[1]: (l.split()[2], int(l.split()[3])) for l in t.splitlines() if l.startswith("layer ")}


NET_W, NET_H = 160, 96


def he_engine(n=1, u8=True, model=engine.COCO_18, **kw):
    eng = engine.PoseEngine(model, NET_W, NET_H, 2 * NET_W, 2 * NET_H, precision=S8, max_batch=n, u8_activations=u8, **kw)
    eng.set_weights(synth.make_weights(model, "he"))
    return eng


def test_calibration_required_and_targets():
    """A forward before pe_calibrate is PE_ERR_STATE.  pe_calibrate puts the stored maximum of every u8 blob into [64, 128) and of
    every s8 blob into [32, 64) (the largest stored integer after rounding: [64, 128] and [32, 64]), and the following forward of
    the same frame reports a worst ratio in range."""
    busy = synth.make_frame(3, 2 * NET_H, 2 * NET_W)
    eng = he_engine()
    with pytest.raises(engine.PoseEngineError, match="pe_calibrate"):
        eng.forward_frames([busy])
    eng.calibrate([busy])
    fm = formats(engine.COCO_18)
    seen = {"u8": 0, "s8": 0}
    for name, (comp, out, _, oa) in fm["convs"].items():
        if out not in seen:
            continue
        try:
            x = eng.fetch_blob(name)[:1]
        except engine.PoseEngineError:
            continue   # a stage output that a later stage overwrites
        m = float(np.abs(x).max()) * 2.0 ** eng.blob_log2_scale(name)
        lo, hi = (64, 128) if out == "u8" else (32, 64)
        assert lo <= m <= hi, (name, out, m)
        seen[out] += 1
    assert seen["u8"] >= 50 and seen["s8"] >= 1, seen
    eng.forward_frames([busy])
    rc, worst, layer = eng.range_status()
    assert rc == 0 and 0.25 <= worst < 64.5 / 127, (rc, worst, layer)
    eng.close()


def test_passes_over_a_set_converge_to_one_batch():
    """calibrate_begin / _end passes over two frames, one of them 8x lower in contrast, give the table of pe_calibrate on both
    frames as one batch."""
    f = synth.make_frame(4, 2 * NET_H, 2 * NET_W)
    low = (128 + np.round((f.astype(np.float64) - 128) / 8)).astype(np.uint8)
    one = he_engine(2)
    one.calibrate([f, low])
    passes = he_engine(1)
    passes.calibrate([low])
    n = passes.calibrate_on([[low], [f]])
    print("\npasses: %d" % n)
    assert passes.calibration_table() == one.calibration_table()
    one.close()
    passes.close()


def test_table_round_trip_and_refusals():
    """A table gives bit-identical maps, peaks and joints; it records the flag (precision 262) and u8 kinds; an S8X1 table is
    refused by a u8 engine and the reverse."""
    frames = [synth.make_frame(6 + i, 2 * NET_H, 2 * NET_W) for i in range(2)]
    a = he_engine(2)
    a.calibrate(frames[:1])
    t = a.calibration_table()
    assert "\nprecision 262\n" in t and any(k == "u8" for k, _ in table_layers(t).values())
    b = he_engine(2)
    b.set_calibration_table(t)
    same_outputs(outputs(a, frames), outputs(b, frames))
    plain = he_engine(2, u8=False)
    plain.calibrate(frames[:1])
    with pytest.raises(engine.PoseEngineError, match="precision 262, the engine runs precision 6"):
        plain.set_calibration_table(t)
    with pytest.raises(engine.PoseEngineError, match="precision 6, the engine runs precision 262"):
        b.set_calibration_table(plain.calibration_table())
    for e in (a, b, plain):
        e.close()


def test_raised_u8_exponent_is_reported():
    """A table with one u8 layer's log2 scale raised by 3 (stored values 8x larger, past 255): pe_range_status is PE_ERR_RANGE
    naming that layer."""
    frame = synth.make_frame(7, 2 * NET_H, 2 * NET_W)
    a = he_engine()
    a.calibrate([frame])
    t = a.calibration_table()
    kind, k = table_layers(t)["conv3_2"]
    assert kind == "u8"
    bad = t.replace("layer conv3_2 u8 %d\n" % k, "layer conv3_2 u8 %d\n" % (k + 3))
    assert bad != t
    a.set_calibration_table(bad)
    a.range_status()
    a.forward_frames([frame])
    a.sync()
    rc, worst, layer = a.range_status()
    assert rc == 5 and layer == "conv3_2" and worst >= 1, (rc, worst, layer)
    a.close()


def test_graph_replays_reproduce_the_calibration_forward():
    """The results of pe_calibrate's forward equal those of the next three forwards of the same frames (eager, captured into a
    CUDA graph, replayed) bit for bit."""
    frames = [synth.make_frame(8 + i, 2 * NET_H, 2 * NET_W) for i in range(2)]
    eng = he_engine(2)
    eng.calibrate(frames)
    res = [eng.fetch(i) for i in range(2)]
    cal = (eng.fetch_maps(2).copy(), [(c, j.copy(), p.copy()) for c, j, p in res])
    for _ in range(3):
        same_outputs(outputs(eng, frames), cal)
    eng.close()


# ------------------------------------------------------------------------------------------ sharing, bound
def check_same(engs, frame):
    res = [outputs(e, [frame]) + (e.fetch_blob("conv4_3_CPM")[:1].copy(),) for e in engs]
    for r in res[1:]:
        same_outputs(r, res[0])
        assert np.array_equal(r[2], res[0][2])


def test_share_weights_bit_identical_and_refusals():
    """A pe_share_weights receiver gives the calibrated source's results bit for bit; sharing between a u8 and a plain S8X1
    handle, and the sparse test hook on a u8 engine, are refused."""
    frame = synth.make_frame(5, 2 * NET_H, 2 * NET_W)
    e0 = he_engine()
    e0.calibrate([frame])
    e1 = engine.PoseEngine(engine.COCO_18, NET_W, NET_H, 2 * NET_W, 2 * NET_H, precision=S8, u8_activations=True)
    engine.share_weights(e0, e1)
    check_same([e0, e1], frame)
    plain = engine.PoseEngine(engine.COCO_18, NET_W, NET_H, 2 * NET_W, 2 * NET_H, precision=S8)
    with pytest.raises(engine.PoseEngineError, match="u8 activations"):
        engine.share_weights(e0, plain)
    assert engine.lib().pe_test_force_sparse(e0._h, 1) == 1   # PE_ERR_INVALID
    assert e0.sparse_layers() == []
    for e in (e0, e1, plain):
        e.close()


def test_broadcast_weights_bit_identical():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    frame = synth.make_frame(5, 2 * NET_H, 2 * NET_W)
    e0 = he_engine()
    e0.calibrate([frame])
    e2 = engine.PoseEngine(engine.COCO_18, NET_W, NET_H, 2 * NET_W, 2 * NET_H, precision=S8, u8_activations=True, device=1)
    engine.broadcast_weights([e0, e2])
    check_same([e0, e2], frame)
    e0.close()
    e2.close()


def test_accumulator_bound_refused(tmp_path):
    """A 7x7 layer reading 1400 u8 channels (K = 49 x 1408 = 68992 > 66311) is refused with the layer named; plain S8X1, whose
    bound is 132104, builds the same file."""
    spec = pose_spec(engine.MPI_15, 16, 16, conv1_1=8, levels=[[(3, 8)], [(3, 8)], [(3, 8)], [(1, 1400), (7, 16)]], branch=[(1, 8)])
    path = tmp_path / "big_k.prototxt"
    path.write_text(synth.netspec_to_prototxt(spec))
    fm = formats(None, str(path))
    assert fm["convs"]["conv4_2"][0] == "u8"
    with pytest.raises(engine.PoseEngineError, match="conv4_2") as ex:
        engine.PoseEngine(None, 16, 16, 32, 32, precision=S8, prototxt=str(path), u8_activations=True)
    assert "66311" in str(ex.value) and "u8" in str(ex.value)
    eng = engine.PoseEngine(None, 16, 16, 32, 32, precision=S8, prototxt=str(path))
    eng.close()


# ------------------------------------------------------------------------------------------ whole net, CLI
@pytest.mark.parametrize("S", [1, 2])
@pytest.mark.parametrize("model", [engine.COCO_18, engine.MPI_15])
def test_whole_net_vs_oracle(model, S):
    """Calibrated, 160x96: stride-8 maps against the oracle held to S8X1's TOL_NET, printed beside S8X1's from the same run."""
    net_w, net_h = 160, 96
    W = synth.make_weights(model, "he", seed=7)
    frames = [synth.make_frame(20 + i, 192, 320) for i in range(2)]
    onet = orc.Net(model)
    onet.set_weights(W)
    omaps = [onet.forward(orc.preprocess(f, net_h, net_w, S, 1.0, 0.25)) for f in frames]
    errs = {}
    for u8 in (False, True):
        eng = engine.PoseEngine(model, net_w, net_h, 320, 192, num_scales=S, start_scale=1.0, scale_gap=0.25, precision=S8,
                                max_batch=2, u8_activations=u8)
        eng.set_weights(W)
        eng.calibrate(frames)
        eng.forward_frames(frames)
        maps = eng.fetch_maps(2)
        errs["u8" if u8 else "s8"] = [rel(maps[i * S:(i + 1) * S], omaps[i]) for i in range(2)]
        rc, worst, layer = eng.range_status()
        assert rc == 0 and 0 < worst < 1, (rc, worst, layer)
        eng.close()
    print("\n%s 160x96 S=%d: maps vs oracle, S8X1 %s, S8X1 + u8 %s" % ("COCO" if model == engine.COCO_18 else "MPI", S,
          ["%.3e" % e for e in errs["s8"]], ["%.3e" % e for e in errs["u8"]]))
    assert max(errs["u8"]) < TOL_NET


def test_cli_u8_activations(tmp_path):
    """rtpose.bin --precision 6 --u8_activations logs how many conv layers read u8, saves a flagged table, and writes the JSON the
    Python path gives with that table; with --f16_layers narrow and --audit_every 1 it runs and prints the audit summary."""
    model, n = engine.COCO_18, 3
    W = synth.make_weights(model, "he", seed=3)
    cm = tmp_path / "w.caffemodel"
    engine.write_caffemodel(str(cm), W, synth.conv_table(model))
    imgs = tmp_path / "imgs"
    imgs.mkdir()
    frames = [synth.make_frame(100 + i, 192, 320) for i in range(n)]
    for i, f in enumerate(frames):
        write_bmp(str(imgs / ("f%03d.bmp" % i)), f)
    common = [BIN, "--image_dir", str(imgs), "--caffemodel", str(cm), "--model", "COCO", "--resolution", "320x192",
              "--net_resolution", "160x96", "--no_frame_drops", "--no_display", "--precision", "6", "--u8_activations"]
    out, table = tmp_path / "json", tmp_path / "calib.txt"
    r = subprocess.run(common + ["--write_json", str(out), "--save_calibration", str(table)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    reads = sum(1 for c in formats(model)["convs"].values() if c[0] == "u8")
    assert "%d of 92 conv layers read u8 activations" % reads in r.stderr, r.stderr[-2000:]
    assert "\nprecision 262\n" in table.read_text()
    eng = engine.PoseEngine(model, 160, 96, 320, 192, precision=S8, u8_activations=True)
    eng.set_weights(W)
    eng.set_calibration_table(table.read_text())
    for i, f in enumerate(frames):
        eng.forward_frames([f])
        cnt, joints, _ = eng.fetch(0)
        assert (out / ("f%03d.json" % i)).read_text() == engine.write_json(joints[:cnt], eng.num_parts), i
    eng.close()
    r = subprocess.run(common + ["--f16_layers", "narrow", "--audit_every", "1", "--write_json", str(tmp_path / "j2")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "Audit summary: " in r.stderr, r.stderr[-2000:]
