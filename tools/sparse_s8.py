#!/usr/bin/env python3
"""Speed of the 2:4-sparse s8 kernel (csrc/conv_s8_sparse.cu) against the dense one on workload C2 of bench.py (COCO 656x368,
9 frames per forward, two handles sharing one packed buffer, PE_PREC_S8X1 calibrated on frame 0).

Two weight sets, alternated for SP_ROUNDS rounds (default 3) of SP_STEPS timed steps (default 40) after SP_WARMUP (default 4):
  * dense:  He-init weights (not 2:4, so every layer runs the dense kernel);
  * sparse: the same weights through engine.prune_2to4, on handles whose commit runs every layer but conv1_1 on the sparse
    kernel (the test hook pe_test_force_sparse lifts the shape rule, which as built keeps every layer dense).
The MMA time does not depend on the values, so the two differ only in the kernels.  Per round: resident frames/s (frames
already on the GPU, CUDA events) and end-to-end frames/s (host frames in, results out); then conv ms per layer class of one
9-frame step (pe_profile_layers, median of 5).  Prints the card (name, power limit, SM clocks, read in this run), then one JSON
line."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402

from caffe_rtpose_b200 import engine, synth  # noqa: E402
from fast_mode import B, DISP_H, DISP_W, MODEL, NET_H, NET_W, card, conv_classes, timed  # noqa: E402


def make_engines(W, sparse, calibrate):
    """Two S8X1 handles sharing one packed buffer, calibrated on `calibrate`; `sparse`: the sparse kernel past the shape rule."""
    engs = [engine.PoseEngine(MODEL, NET_W, NET_H, DISP_W, DISP_H, max_batch=B, precision=engine.PREC_S8X1) for _ in range(2)]
    if sparse and engine.lib().pe_test_force_sparse(engs[0]._h, 1):
        raise engine.PoseEngineError("pe_test_force_sparse failed")
    engs[0].set_weights(W)
    engs[0].calibrate(calibrate)
    engine.share_weights(engs[0], engs[1])
    return engs


def main():
    steps, warmup, rounds = (int(os.environ.get(k, d)) for k, d in (("SP_STEPS", "40"), ("SP_WARMUP", "4"), ("SP_ROUNDS", "3")))
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
    sets = {"dense": W, "sparse": engine.prune_2to4(W, MODEL)}
    engs = {k: make_engines(w, k == "sparse", [host[0]]) for k, w in sets.items()}
    out = {k: {"sparse_layers": len(engs[k][0].sparse_layers()), "resident_fps": [], "e2e_fps": []} for k in sets}
    for _ in range(rounds):
        for k in sets:
            r, e, _, _ = timed(engs[k], dev, host, nb, steps, warmup)
            out[k]["resident_fps"].append(round(r, 1))
            out[k]["e2e_fps"].append(round(e, 1))
    for k in sets:
        out[k]["conv_ms"] = conv_classes(engs[k][0], host)
    for es in engs.values():
        for e in es:
            e.close()
    print(json.dumps({"card": card(), "workload": "C2 COCO 656x368, 9 frames per forward, S8X1, W-he", "steps": steps,
                      "rounds": rounds, "weights": out}), flush=True)


if __name__ == "__main__":
    torch.cuda.init()
    main()
