#!/usr/bin/env python3
"""What the flip test (pe_set_flip_test) costs, per precision mode, in one run on one GPU.

Workload C2 of bench.py: COCO 656x368, one scale, 9 frames per forward, the bench's seeded 720p frames, W-he weights (E4M3X1 and
S8X1 calibrated with pe_calibrate on frame 0, with the flip test off).  For each mode of FT_MODES (default f16x2, f16x1, e4m3x1,
s8x1) two handles sharing one packed buffer run with the flip test off and two with it on; over FT_ROUNDS rounds the eight
configurations alternate:
  * resident: frames/s of FT_STEPS forwards from device memory (CUDA events, as bench.py and tools/fast_mode.py);
  * e2e: frames/s through forward_frames + fetch of every frame (host clock).
Afterwards, in a run of its own, torch.profiler records FT_PROFILE forwards of each configuration: the post stage's device time per
forward is the sum of its kernels (NMS, PAF scores, limb greedy, assembly), and the conv stack's is the sum of the conv kernels.
He-init maps are noise, so nothing here says what the flip test does to accuracy.  Prints the card, its power limit and SM clocks,
then one JSON line."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from caffe_rtpose_b200 import engine, synth  # noqa: E402
from fast_mode import B, DISP_H, DISP_W, MODEL, card, make_engines, timed  # noqa: E402

MODES = {"f16x2": engine.PREC_F16X2, "f16x1": engine.PREC_F16X1, "e4m3x1": engine.PREC_E4M3X1, "s8x1": engine.PREC_S8X1}
CALIBRATED = ("e4m3x1", "s8x1")
POST_KERNELS = ("nms_flags_kernel", "nms_write_kernel", "paf_score_kernel", "limb_greedy_kernel", "assemble_kernel")


def kernel_ms(engs, dev, n):
    """Device ms per forward of the post-stage kernels and of the conv kernels, from torch.profiler over n forwards."""
    frame_bytes = DISP_H * DISP_W * 3
    for i in range(4):   # eager, captured, replayed: the profiled forwards replay graphs like the timed ones
        engs[0].forward_frames_device(dev.data_ptr() + (i % 2) * B * frame_bytes, B)
    engs[0].sync()
    acts = [torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        for i in range(n):
            engs[0].forward_frames_device(dev.data_ptr() + (i % 2) * B * frame_bytes, B)
        engs[0].sync()
    post = conv = 0.0
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name, us = ev.name, ev.time_range.elapsed_us()
        if any(k in name for k in POST_KERNELS):
            post += us
        elif "conv" in name:
            conv += us
    return round(post / n / 1e3, 4), round(conv / n / 1e3, 3)


def main():
    steps, warmup, rounds, nprof = (int(os.environ.get(k, d)) for k, d in
                                    (("FT_STEPS", "40"), ("FT_WARMUP", "4"), ("FT_ROUNDS", "3"), ("FT_PROFILE", "10")))
    modes = [m for m in os.environ.get("FT_MODES", ",".join(MODES)).split(",")]
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
    engs = {}
    for m in modes:
        for flip in (False, True):
            es = make_engines((MODES[m], None), W, calibrate=[host[0]] if m in CALIBRATED else None)
            for e in es:
                e.set_flip_test(flip)
            engs[(m, flip)] = es
    out = {"%s%s" % (m, "+flip" if f else ""): {"resident_fps": [], "e2e_fps": []} for m, f in engs}
    for _ in range(rounds):
        for (m, f), es in engs.items():
            r, e, _, _ = timed(es, dev, host, nb, steps, warmup)
            key = "%s%s" % (m, "+flip" if f else "")
            out[key]["resident_fps"].append(round(r, 1))
            out[key]["e2e_fps"].append(round(e, 1))
    for (m, f), es in engs.items():
        post, conv = kernel_ms(es, dev, nprof)
        out["%s%s" % (m, "+flip" if f else "")].update({"post_ms": post, "conv_ms": conv})
    for es in engs.values():
        for e in es:
            e.close()
    print(json.dumps({"card": info, "workload": "C2 COCO 656x368, 9 frames per forward, W-he", "steps": steps, "rounds": rounds,
                      "profiled_forwards": nprof, "configs": out}), flush=True)


if __name__ == "__main__":
    main()
