"""Cost of reading decoder frames through pe_forward_pixels, on bench.py's C2 workload (COCO, net 656x368, display 1280x720, parity
mode, nine frames per forward) with nine 1920x1080 frames resident on the device, as an NVDEC decoder leaves them.  --format picks
them: nv12 (the default), nv12_bt709_full (NV12 with PE_PIX_FLAG_BT709 | PE_PIX_FLAG_FULL_RANGE), p016 (NVDEC's 10/12-bit output)
or rgbp (a (3, h, w) planar RGB tensor):

  (a) conversion and warp kernels, device microseconds per frame (torch.profiler, CUDA activities, a run of their own);
  (b) resident frames/s through forward_pixels, in windows alternated with forward_frames_device on display-size BGR frames - the
      difference is what the new front costs;
  (c) nv12 only: frames/s of the route without it: download the NV12 frames, cv2.cvtColor on one host thread, then
      forward_camera_frames from page-locked memory, one batch after the other.

It prints one JSON line (and writes it to --out when given), with the card's name and power limit read in the same run.  Needs a GPU.
    python tools/pixel_input.py --steps 30 --rounds 3 [--format p016]
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


# --format: (PIX_* format, forward_pixels keywords, the frame in that format, bytes read per frame)
FORMATS = {
    "nv12": (engine.PIX_NV12, {}, nv12_of, SRC_W * SRC_H * 3 // 2),
    "nv12_bt709_full": (engine.PIX_NV12, {"matrix": "bt709", "full_range": True}, nv12_of, SRC_W * SRC_H * 3 // 2),
    "p016": (engine.PIX_P016, {}, lambda bgr: (nv12_of(bgr).astype(np.uint16) << 8) | 0x80, SRC_W * SRC_H * 3),
    "rgbp": (engine.PIX_RGBP, {}, lambda bgr: np.ascontiguousarray(bgr[..., ::-1].transpose(2, 0, 1)), SRC_W * SRC_H * 3),
}


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
    ap.add_argument("--format", default="nv12", choices=sorted(FORMATS))
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
    fmt, kw, convert, in_bytes = FORMATS[args.format]
    src = [torch.from_numpy(convert(f)).cuda() for f in src_bgr]                   # nine separate device allocations
    nv12 = src if args.format == "nv12" else None
    disp = torch.from_numpy(np.stack([synth.make_frame(200 + i, DISP_H, DISP_W) for i in range(B)])).cuda()

    def pixels(e, i):
        e.forward_pixels(src, fmt, **kw)

    def resident(e, i):
        e.forward_frames_device(disp.data_ptr(), B)

    nv_host = [torch.empty(f.shape, dtype=torch.uint8, pin_memory=True) for f in src] if nv12 else None
    bgr_host = [torch.empty((SRC_H, SRC_W, 3), dtype=torch.uint8, pin_memory=True) for _ in range(B)]

    def today(e, i):   # download, convert on one host thread, upload from page-locked memory
        for d, h in zip(nv12, nv_host):
            h.copy_(d)
        for h, o in zip(nv_host, bgr_host):
            cv2.cvtColor(h.numpy(), cv2.COLOR_YUV2BGR_NV12, dst=o.numpy())
        e.forward_camera_frames([o.numpy() for o in bgr_host])
        e.fetch(0)

    # the routes compute the same display frames: check once before timing (without (c): the host reference's frames)
    engs[0].forward_pixels(src, fmt, **kw)
    maps_gpu = engs[0].fetch_maps(B)
    if nv12:
        today(engs[0], 0)
    else:
        engs[0].forward_camera_frames([engine.pixels_to_bgr(t.cpu().numpy(), fmt, **kw) for t in src])
    same = bool(np.array_equal(maps_gpu, engs[0].fetch_maps(B)))

    routes = (pixels, resident, today) if nv12 else (pixels, resident)
    for fn in routes:   # warm-up: graph capture of both handles, allocations
        for i in range(4):
            fn(engs[i % 2], i)
    torch.cuda.synchronize()
    fps = {"pixels": [], "resident": [], "today": []}
    for _ in range(args.rounds):
        fps["pixels"].append(timed(engs, pixels, args.steps))
        fps["resident"].append(timed(engs, resident, args.steps))
        if nv12:
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
    per_frame_bytes = in_bytes + 2 * SRC_W * SRC_H * 3 + DISP_W * DISP_H * 3   # frame in, BGR out and back in, display out

    med = {k: float(np.median(v)) for k, v in fps.items() if v}   # (c) runs for nv12 only
    out = {
        "card": card(),
        "workload": "C2: COCO 656x368, display 1280x720, parity mode, %d x %dx%d %s frames per forward, two handles" % (
            B, SRC_W, SRC_H, args.format),
        "a_kernel_us_per_frame": kernel_us, "a_kernel_launches": calls, "a_bytes_per_frame": per_frame_bytes,
        "b_forward_pixels_fps": fps["pixels"], "b_forward_frames_device_fps": fps["resident"],
        "b_cost_pct": 100.0 * (med["resident"] / med["pixels"] - 1.0),
        "c_download_cvtcolor_camera_frames_fps": fps["today"] or None,
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
