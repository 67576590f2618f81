#!/usr/bin/env python3
"""Speed and accuracy of the fast mode (PE_PREC_F16X1) against the parity mode (F16X2) and bf16x1, in one run on one GPU.

Workload C2 of bench.py: COCO 656x368, one scale, 9 frames per forward, the bench's seeded 720p frames (synth.make_frame(i)),
W-he weights.  Per mode, alternating the modes over FM_ROUNDS rounds:
  * resident: frames/s of FM_STEPS forwards from device memory over two handles (CUDA events, as bench.py);
  * e2e: frames/s through forward_frames + fetch of every frame (host clock, as bench.py);
  * conv ms per layer class of one 9-frame step (pe_profile_layers, classes of tools/layer_times.py, median of 5).
On the resident loop's last step: the max error of the stride-8 maps relative to the parity mode's map maximum, and per frame
pe_compare_results against the parity mode at the north-star tolerance (1e-3 net px, in display px).  The same statistics on
the prototxt-filler net (gaussian(0.01) weights, maps ~3e-11), calibrated with pe_calibrate on the first frame.  The He-init
maps are noise with thousands of near-tie NMS decisions, so these pose statistics are a worst case, not what a trained
model shows.  Prints the card, its power limit and SM clocks, then one JSON line."""
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from caffe_rtpose_b200 import engine, synth  # noqa: E402
from layer_times import klass  # noqa: E402

MODEL, NET_W, NET_H, DISP_W, DISP_H, B = engine.COCO_18, 656, 368, 1280, 720, 9
MODES = {"f16x2": engine.PREC_F16X2, "f16x1": engine.PREC_F16X1, "bf16x1": engine.PREC_BF16X1}
TOL_PX = 1e-3 * max(DISP_W / NET_W, DISP_H / NET_H)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                           timeout=30)
        return dict(zip(q.split(","), [v.strip() for v in r.stdout.strip().split(",")]))
    except Exception as ex:   # the numbers below are then without their card: say so in the line
        return {"error": repr(ex)}


def make_engines(prec, W, n=2, calibrate=None):
    engs = [engine.PoseEngine(MODEL, NET_W, NET_H, DISP_W, DISP_H, max_batch=B, precision=prec) for _ in range(n)]
    engs[0].set_weights(W)
    if calibrate is not None:
        engs[0].calibrate(calibrate)
    for e in engs[1:]:
        engine.share_weights(engs[0], e)
    return engs


def results(eng):
    return [eng.fetch(k) for k in range(B)], eng.fetch_maps(B)


def compare(res, ref):
    """(max |maps - ref maps| / max |ref maps|, pose statistics over the frames) of one batch against the parity mode's."""
    (rs, maps), (rr, rmaps) = res, ref
    d = [engine.compare_results(a, b, TOL_PX) for a, b in zip(rs, rr)]
    return {"map_rel_err": float(np.abs(maps - rmaps).max() / np.abs(rmaps).max()),
            "frames_identical": sum(x["identical"] for x in d), "frames": len(d),
            "parts_count_differ": sum(x["parts_count_differ"] for x in d), "peaks_moved": sum(x["peaks_moved"] for x in d),
            "persons_matched": sum(x["persons_matched"] for x in d), "persons_ref": sum(r[0] for r in rr),
            "max_joint_dist_px": max(x["max_joint_dist"] for x in d)}


def timed(engs, dev, host, nb, steps, warmup):
    frame_bytes = DISP_H * DISP_W * 3
    nh = len(engs)
    for i in range(max(warmup, 2 * nh)):
        engs[i % nh].forward_frames_device(dev.data_ptr() + (i % nb) * B * frame_bytes, B)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for i in range(steps):
        engs[i % nh].forward_frames_device(dev.data_ptr() + ((warmup + i) % nb) * B * frame_bytes, B)
    for e in engs:
        e.sync()
    ev1.record()
    torch.cuda.synchronize()
    resident = B * steps / (ev0.elapsed_time(ev1) * 1e-3)
    last = results(engs[(steps - 1) % nh])
    last_batch = (warmup + steps - 1) % nb
    t0 = time.perf_counter()
    for i in range(steps):
        e = engs[i % nh]
        if i >= nh:
            for k in range(B):
                e.fetch(k)
        e.forward_frames([host[(i % nb) * B + k] for k in range(B)])
    for j in range(min(nh, steps)):
        for k in range(B):
            engs[(steps - 1 - j) % nh].fetch(k)
    e2e = B * steps / (time.perf_counter() - t0)
    return resident, e2e, last, last_batch


def conv_classes(eng, host):
    eng.forward_frames(host[:B])
    eng.sync()
    runs = [eng.profile_layers(B) for _ in range(5)]
    agg = {}
    for i, (name, _, fl) in enumerate(runs[0]):
        k = klass(name, fl)
        agg[k] = agg.get(k, 0.0) + statistics.median(r[i][1] for r in runs)
    out = {k: round(v, 3) for k, v in sorted(agg.items())}
    out["conv total"] = round(sum(v for k, v in agg.items() if k != "pool/copy"), 3)
    return out


def main():
    steps, warmup, rounds = (int(os.environ.get(k, d)) for k, d in (("FM_STEPS", "40"), ("FM_WARMUP", "4"), ("FM_ROUNDS", "3")))
    info = card()
    print("card: %s" % json.dumps(info), flush=True)
    n_frames = 72
    host_t = torch.empty((n_frames, DISP_H, DISP_W, 3), dtype=torch.uint8, pin_memory=True)
    host = host_t.numpy()
    for i in range(n_frames):
        host[i] = synth.make_frame(i, DISP_H, DISP_W)
    dev = host_t.cuda()
    nb = n_frames // B
    W = synth.make_weights(MODEL, "he")
    engs = {m: make_engines(p, W) for m, p in MODES.items()}
    out = {m: {"resident_fps": [], "e2e_fps": []} for m in MODES}
    last = {}
    for _ in range(rounds):
        for m in MODES:
            r, e, res, lb = timed(engs[m], dev, host, nb, steps, warmup)
            out[m]["resident_fps"].append(round(r, 1))
            out[m]["e2e_fps"].append(round(e, 1))
            last[m] = res
    for m in MODES:
        out[m]["conv_ms"] = conv_classes(engs[m][0], host)
        out[m]["vs_parity_bench_step"] = compare(last[m], last["f16x2"])
    for es in engs.values():
        for e in es:
            e.close()
    # the prototxt's own filler, calibrated on frame 0 (uncalibrated it leaves the fp16 range)
    Wc = synth.make_weights(MODEL, "caffe")
    batch = [host[lb * B + k] for k in range(B)]
    filler = {}
    for m in ("f16x2", "f16x1"):
        e = make_engines(MODES[m], Wc, n=1, calibrate=[host[0]])[0]
        e.forward_frames(batch)
        filler[m] = results(e)
        e.close()
    out["f16x1"]["vs_parity_filler_net"] = compare(filler["f16x1"], filler["f16x2"])
    print(json.dumps({"card": info, "workload": "C2 COCO 656x368, 9 frames per forward, W-he", "steps": steps, "rounds": rounds,
                      "tol_px": TOL_PX, "modes": out}), flush=True)


if __name__ == "__main__":
    main()
