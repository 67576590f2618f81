#!/usr/bin/env python3
"""Sensitivity sweep of mixed precision (pe_create_mixed): which conv layers are worth running in fp16 inside the FP8 and INT8 modes.

For each base (E4M3X1, S8X1) and each layer group, an engine runs with only that group in fp16 and is compared with the parity
mode (F16X2) on workload C2 of bench.py (COCO 656x368, 9 frames, the bench's seeded frames):
  * map_rel_err: max |maps - parity maps| / max |parity maps| on the He-init bench step and on the prototxt-filler net
    (gaussian(0.01) weights), both calibrated with pe_calibrate on frame 0 (tools/fast_mode.py);
  * pose agreement on the bench step: frames whose peaks, person count and joints equal the parity mode's (pe_compare_results at
    1e-3 net px), persons matched;
  * conv ms of one 9-frame step (pe_profile_layers, median of 5), the sum over the conv layers.
The groups are the layer classes of tools/layer_times.py:klass, each closed under the shared-buffer rule (layers that read one
buffer run in one format: both branches' first layers, and every stage's first layers with conv4_4_CPM's readers), plus
"none" (the base mode), "narrow" and "all".  Prints the card, its power limit and SM clocks, then one JSON line."""
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from caffe_rtpose_b200 import engine, synth  # noqa: E402
from fast_mode import B, DISP_H, DISP_W, MODEL, card, compare, make_engines, results  # noqa: E402
from layer_times import klass  # noqa: E402

BASES = {"e4m3x1": engine.PREC_E4M3X1, "s8x1": engine.PREC_S8X1}


def groups():
    """{group name: conv layers}: klass's classes closed under the shared-buffer rule, then narrow and all."""
    f = engine.plan_formats(MODEL, engine.PREC_F16X1)
    convs, acts = f["convs"], f["acts"]
    shared = {i for i, a in enumerate(acts) if a[2] is None and i != convs["conv1_1"][2]}   # the stage-input buffers

    def buffer(name):
        a = convs[name][2]
        return "stage inputs" if a in shared else a

    out = {}
    for name in convs:
        out.setdefault(klass(name, 1.0), set()).add(name)
    for g, names in out.items():
        bufs = {buffer(n) for n in names}
        names |= {n for n in convs if buffer(n) in bufs}
    return {**{g: sorted(n) for g, n in sorted(out.items())}, "narrow": ["narrow"], "all": list(convs)}


def conv_ms(eng, host):
    eng.forward_frames(host[:B])
    eng.sync()
    runs = [eng.profile_layers(B) for _ in range(5)]
    return round(sum(statistics.median(r[i][1] for r in runs) for i, (_, _, fl) in enumerate(runs[0]) if fl > 0), 3)


def run(spec, W, host, batch):
    e = make_engines(spec, W, n=1, calibrate=[host[0]])[0]   # the filler net leaves the fp16 range uncalibrated
    e.forward_frames(batch)
    res = results(e)
    ms = conv_ms(e, host)
    e.close()
    return res, ms


def main():
    info = card()
    print("card: %s" % json.dumps(info), flush=True)
    host = np.stack([synth.make_frame(i, DISP_H, DISP_W) for i in range(B)])
    batch = list(host)
    nets = {"bench_step": synth.make_weights(MODEL, "he"), "filler_net": synth.make_weights(MODEL, "caffe")}
    ref = {k: run((engine.PREC_F16X2, None), W, host, batch)[0] for k, W in nets.items()}
    gs = groups()
    out = {"groups": {g: (n if g not in ("narrow", "all") else g) for g, n in gs.items()}}
    for bname, base in BASES.items():
        out[bname] = {}
        for g, names in [("none", [])] + list(gs.items()):
            row = {}
            for k, W in nets.items():
                res, ms = run((base, ",".join(names)), W, host, batch)
                c = compare(res, ref[k])
                row[k] = {"map_rel_err": round(c["map_rel_err"], 4)}
                if k == "bench_step":
                    row[k].update(frames_identical=c["frames_identical"], persons_matched=c["persons_matched"],
                                  persons_ref=c["persons_ref"])
                    row["conv_ms"] = ms
            out[bname][g] = row
            print("%-7s %-12s %s" % (bname, g, json.dumps(row)), flush=True)
    print(json.dumps({"card": info, "workload": "C2 COCO 656x368, 9 frames per forward", "sweep": out}), flush=True)


if __name__ == "__main__":
    torch.cuda.init()
    main()
