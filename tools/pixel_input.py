"""Cost of reading decoder frames through pe_forward_pixels, on bench.py's C2 workload (COCO, net 656x368, display 1280x720, parity
mode, nine frames per forward) with nine 1920x1080 NV12 frames resident on the device, as an NVDEC decoder leaves them:

  (a) conversion and warp kernels, device microseconds per frame (torch.profiler, CUDA activities, a run of their own);
  (b) resident frames/s through forward_pixels, in windows alternated with forward_frames_device on display-size BGR frames - the
      difference is what the new front costs;
  (c) frames/s of the route without it: download the NV12 frames, cv2.cvtColor on one host thread, then forward_camera_frames from
      page-locked memory, one batch after the other.

It prints one JSON line (and writes it to --out when given), with the card's name and power limit read in the same run.  Needs a GPU.
    python tools/pixel_input.py --steps 30 --rounds 3
"""
import argparse
import json
import os
import subprocess
import sys
import time

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from caffe_rtpose_b200 import engine, synth  # noqa: E402

NET_W, NET_H, DISP_W, DISP_H, B = 656, 368, 1280, 720, 9
SRC_W, SRC_H = 1920, 1080


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:   # the numbers stay valid, only their label is missing
        q = "nvidia-smi unavailable: %r" % (ex,)
    return {"nvidia_smi": q, "torch_name": torch.cuda.get_device_name()}


def nv12_of(bgr):
    h, w, _ = bgr.shape
    i420 = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420)
    u = i420[h:h + h // 4].reshape(h // 2, w // 2)
    v = i420[h + h // 4:].reshape(h // 2, w // 2)
    return np.concatenate([i420[:h], np.stack([u, v], -1).reshape(h // 2, w)])


def timed(engs, step, steps):
    """frames/s of `steps` forwards alternating over the handles, device-wide synchronised on both sides"""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        step(engs[i % len(engs)], i)
    for e in engs:
        e.sync()
    torch.cuda.synchronize()
    return B * steps / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3, help="alternated windows per route")
    ap.add_argument("--profile_steps", type=int, default=20)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("pixel_input.py measures on the GPU; none is visible")
    cv2.setNumThreads(1)   # route (c) converts on one host thread, as a decode loop without a thread pool does

    W = synth.make_weights(engine.COCO_18, "he")
    engs = [engine.PoseEngine(engine.COCO_18, NET_W, NET_H, DISP_W, DISP_H, max_batch=B, precision=engine.PREC_F16X2) for _ in range(2)]
    for e in engs:
        e.set_weights(W)
    src_bgr = [synth.make_frame(100 + i, SRC_H, SRC_W) for i in range(B)]
    nv12 = [torch.from_numpy(nv12_of(f)).cuda() for f in src_bgr]                 # nine separate device allocations
    disp = torch.from_numpy(np.stack([synth.make_frame(200 + i, DISP_H, DISP_W) for i in range(B)])).cuda()

    def pixels(e, i):
        e.forward_pixels(nv12, engine.PIX_NV12)

    def resident(e, i):
        e.forward_frames_device(disp.data_ptr(), B)

    nv_host = [torch.empty(f.shape, dtype=torch.uint8, pin_memory=True) for f in nv12]
    bgr_host = [torch.empty((SRC_H, SRC_W, 3), dtype=torch.uint8, pin_memory=True) for _ in range(B)]

    def today(e, i):   # download, convert on one host thread, upload from page-locked memory
        for d, h in zip(nv12, nv_host):
            h.copy_(d)
        for h, o in zip(nv_host, bgr_host):
            cv2.cvtColor(h.numpy(), cv2.COLOR_YUV2BGR_NV12, dst=o.numpy())
        e.forward_camera_frames([o.numpy() for o in bgr_host])
        e.fetch(0)

    # the three routes compute the same display frames: check once before timing
    engs[0].forward_pixels(nv12, engine.PIX_NV12)
    maps_gpu = engs[0].fetch_maps(B)
    today(engs[0], 0)
    same = bool(np.array_equal(maps_gpu, engs[0].fetch_maps(B)))

    for fn in (pixels, resident, today):   # warm-up: graph capture of both handles, allocations
        for i in range(4):
            fn(engs[i % 2], i)
    torch.cuda.synchronize()
    fps = {"pixels": [], "resident": [], "today": []}
    for _ in range(args.rounds):
        fps["pixels"].append(timed(engs, pixels, args.steps))
        fps["resident"].append(timed(engs, resident, args.steps))
        fps["today"].append(timed(engs, today, max(3, args.steps // 3)))

    # (a) kernel time per frame, profiler on, a run of its own
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.profile_steps):
            pixels(engs[i % 2], i)
        for e in engs:
            e.sync()
        torch.cuda.synchronize()
    us = {"pixels_to_bgr_kernel": 0.0, "warp_affine_cubic_kernel": 0.0}
    calls = dict.fromkeys(us, 0)
    for ka in prof.key_averages():
        for k in us:
            if k in ka.key:
                us[k] += ka.device_time_total
                calls[k] += ka.count
    n = args.profile_steps * B
    kernel_us = {k: (us[k] / n if calls[k] else None) for k in us}
    per_frame_bytes = SRC_W * SRC_H * 3 // 2 + 2 * SRC_W * SRC_H * 3 + DISP_W * DISP_H * 3   # NV12 in, BGR out and back in, display out

    med = {k: float(np.median(v)) for k, v in fps.items()}
    out = {
        "card": card(),
        "workload": "C2: COCO 656x368, display 1280x720, parity mode, %d x %dx%d NV12 frames per forward, two handles" % (B, SRC_W, SRC_H),
        "a_kernel_us_per_frame": kernel_us, "a_kernel_launches": calls, "a_bytes_per_frame": per_frame_bytes,
        "b_forward_pixels_fps": fps["pixels"], "b_forward_frames_device_fps": fps["resident"],
        "b_cost_pct": 100.0 * (med["resident"] / med["pixels"] - 1.0),
        "c_download_cvtcolor_camera_frames_fps": fps["today"],
        "routes_give_identical_maps": same,
    }
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    for e in engs:
        e.close()


if __name__ == "__main__":
    main()
