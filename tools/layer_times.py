#!/usr/bin/env python3
"""Per-layer-class device time of one bench step (C2 geometry, LT_BATCH frames): events between the launches of
pe_profile_layers, median of 5 passes, summed per class, with algorithmic TFLOP/s per class, and the bytes the conv
kernel's TMA boxes bring from L2 into shared memory per class with the rate that implies."""
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from caffe_rtpose_b200 import engine, synth  # noqa: E402


def klass(name, fl):
    if fl == 0:
        return "pool/copy"
    if name in ("conv1_1", "conv1_2"):
        return "conv1_x"
    if name.startswith("conv5_") and name[6] in "123":
        return "stage1 3x3"
    if name.startswith("conv") and not name.startswith("conv5_"):
        return "vgg 3x3"
    if name.startswith("Mconv1_"):
        return "7x7 first"
    if name.startswith("Mconv") and name[5] in "2345":
        return "7x7"
    return "1x1"


NET_W, NET_H = 656, 368
CLUSTER = 2   # conv_tc.cu TC_CLUSTER: CTAs along M that share each weight tile through a TMA multicast


def tc_cout_pad(cout):
    if cout > 64:
        return (cout + 127) // 128 * 128
    return 64 if cout > 48 else 48 if cout > 32 else 32 if cout > 16 else 16


def l2_smem_bytes(cout, cin, k, H, W, gap, nimg, planes=2, cluster=CLUSTER):
    """Bytes the TMA boxes of one conv_wg_kernel launch bring from L2 into shared memory, at full tile width: per CTA and
    64-channel block, k A windows of {64, 136 rows (128 for 1x1), P} and k*k weight tiles of {64, BN, P}, of which the
    cluster loads each once.  CTAs: ceil(((H-1)*Wp + W) / 128) row tiles per image (grid rounded to whole clusters) times
    the N tiles.  The empty CTAs that round the grid up load their windows too."""
    cp = tc_cout_pad(cout)
    bn = min(cp, 64 if planes == 3 else 128)
    Wp = W + gap
    tiles = -(-nimg * -(-((H - 1) * Wp + W) // 128) // cluster) * cluster
    ctas = tiles * (cp // bn)
    kb = -(-cin // 64)
    window = planes * (128 if k == 1 else 136) * 128
    wtile = planes * bn * 128
    return ctas * kb * (k * window + k * k * wtile / cluster)


def layer_bytes(model, nimg):
    """{conv name: L2 -> shared-memory bytes} of one forward of nimg frames at the benchmark's net size."""
    out = {}
    gaps = {int(l.split()[1]): int(l.split()[2]) for l in engine.plan_describe(model=model).splitlines() if l.startswith("gap ")}
    for name, co, ci, k in synth.conv_table(model):
        level = 0 if name.startswith("conv1") else 1 if name.startswith("conv2") else 2 if name.startswith("conv3") else 3
        w, h = NET_W, NET_H
        for _ in range(level):
            w, h = (w + 1) // 2, (h + 1) // 2
        if name == "conv1_1":   # runs on the im2col'ed input: a 1x1 conv over 27 channels, padded to 64
            ci, k = 27, 1
        out[name] = l2_smem_bytes(co, ci, k, h, w, gaps[level], nimg)
    return out


def main():
    B = int(os.environ.get("LT_BATCH", "9"))
    model = engine.COCO_18
    eng = engine.PoseEngine(model, NET_W, NET_H, 1280, 720, max_batch=B, precision=engine.PREC_BF16X2)
    eng.set_weights(synth.make_weights(model, "he"))
    frames = [synth.make_frame(i) for i in range(B)]
    for _ in range(2):
        eng.forward_frames(frames)
        eng.sync()
    runs = [eng.profile_layers(B) for _ in range(5)]
    names = [n for n, _, _ in runs[0]]
    fl = [f for _, _, f in runs[0]]
    med = [statistics.median(r[i][1] for r in runs) for i in range(len(names))]
    lb = layer_bytes(model, B)
    agg, flops, l2 = {}, {}, {}
    for n, ms, f in zip(names, med, fl):
        k = klass(n, f)
        agg[k] = agg.get(k, 0.0) + ms
        flops[k] = flops.get(k, 0.0) + f
        l2[k] = l2.get(k, 0.0) + lb.get(n, 0.0)
    tot = sum(agg.values())
    out = {"total_ms": round(tot, 3), "conv_ms": round(tot - agg.get("pool/copy", 0), 3), "cluster": CLUSTER,
           "classes": {k: {"ms": round(v, 3), "tflops": round(flops[k] / v / 1e9, 1) if flops[k] else None,
                           "l2_gb": round(l2[k] / 1e9, 2) if l2[k] else None, "l2_tbps": round(l2[k] / v / 1e9, 2) if l2[k] else None}
                       for k, v in sorted(agg.items())}}
    if os.environ.get("LT_VERBOSE"):
        out["layers"] = [(n, round(m, 4)) for n, m in zip(names, med)]
    print(json.dumps(out), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
