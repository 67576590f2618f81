#!/usr/bin/env python3
"""How much the calibration frames change the error of the INT8 and FP8 modes (PE_PREC_S8X1, PE_PREC_E4M3X1).

Workload C2 of bench.py: COCO 656x368, one scale, 9 frames per forward, W-he weights.  Held out: the bench's frames
synth.make_frame(0..8).  Reference: the parity mode (F16X2) calibrated on the same synthetic frame rtpose.bin uses.  Per mode, three
calibrations:
  * synthetic: pe_calibrate on rtpose.bin's synthetic_frame(0) (what the CLI does without --calibration_dir);
  * set64: from there, calibrate_on over 64 other frames (synth.make_frame(100..163)) until a pass changes nothing;
  * low_contrast: the same passes over those frames at 1/8 of their contrast.
For each: max |maps - parity maps| / max |parity maps| on the held-out frames, the passes, the wall time of the calibration.
Prints the card and its power limit, then one JSON line.  He-init nets, not trained models: the numbers say how the calibration
set moves the error, not what a trained model shows."""
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from caffe_rtpose_b200 import engine, synth  # noqa: E402

MODEL, NET_W, NET_H, DISP_W, DISP_H, B = engine.COCO_18, 656, 368, 1280, 720, 9


def synthetic_frame(idx, w, h):
    """host/rtpose.cpp synthetic_frame: 128 + 100 sin((x + 31 c) / 41) cos((y + 17 idx) / 57), averaged with LCG noise"""
    sx = np.array([100.0 * math.sin((x + 31 * c) / 41.0) for x in range(w) for c in range(3)])
    cy = np.array([math.cos((y + 17 * idx) / 57.0) for y in range(h)])
    low = 128 + (sx[None, :] * cy[:, None]).astype(np.int64)   # (int) truncates toward zero like the C cast
    n = w * h * 3
    noise = np.empty(n, np.int64)
    s = (0x9E3779B9 * (idx + 1)) & 0xFFFFFFFF
    for i in range(n):
        s = (s * 1664525 + 1013904223) & 0xFFFFFFFF
        noise[i] = s >> 24
    v = (low.reshape(-1) + noise) // 2
    return np.clip(v, 0, 255).astype(np.uint8).reshape(h, w, 3)


def low_contrast(f):
    return (128 + np.round((f.astype(np.float64) - 128) / 8)).astype(np.uint8)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
    return r.stdout.strip()


def maps_of(eng, frames):
    eng.forward_frames(frames)
    return eng.fetch_maps(len(frames))


def main():
    print("card:", card())
    W = synth.make_weights(MODEL, "he")
    syn = synthetic_frame(0, DISP_W, DISP_H)
    held = [synth.make_frame(i) for i in range(B)]
    cal = [synth.make_frame(100 + i) for i in range(64)]
    low = [low_contrast(f) for f in cal]
    ref = engine.PoseEngine(MODEL, NET_W, NET_H, DISP_W, DISP_H, max_batch=B, precision=engine.PREC_F16X2)
    ref.set_weights(W)
    ref.calibrate([syn])
    rmaps = maps_of(ref, held)
    ref.close()
    out = {"workload": "C2 COCO 656x368 W-he, held-out bench frames 0-8", "card": card()}
    for name, prec in (("s8x1", engine.PREC_S8X1), ("e4m3x1", engine.PREC_E4M3X1)):
        for case, frames in (("synthetic", None), ("set64", cal), ("low_contrast", low)):
            eng = engine.PoseEngine(MODEL, NET_W, NET_H, DISP_W, DISP_H, max_batch=B, precision=prec)
            eng.set_weights(W)
            t0 = time.perf_counter()
            eng.calibrate([syn])
            passes = 0
            if frames is not None:
                passes = eng.calibrate_on([frames[i:i + B] for i in range(0, len(frames), B)])
            eng.sync()
            dt = time.perf_counter() - t0
            maps = maps_of(eng, held)
            err = float(np.abs(maps - rmaps).max() / np.abs(rmaps).max())
            rc, worst, layer = eng.range_status()
            out["%s_%s" % (name, case)] = {"map_rel_err": round(err, 4), "passes": passes, "calibration_s": round(dt, 2),
                                           "range_status": rc, "worst_ratio": round(worst, 3)}
            print(name, case, out["%s_%s" % (name, case)], flush=True)
            eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
