"""Measurements of GPU JPEG decoding (rtpose.bin --gpu_decode, pe_forward_jpeg_coefs) on 720p quality-98 frames.

  host   frames/s of ONE producer thread: entropy stage only (--decode_bench --gpu_decode) against the full host decoder
         (--decode_bench); needs no GPU.
  gpu    per-frame device time of the two reconstruction kernels (torch.profiler CUDA activity over many forwards) and the
         bytes they move, against 3.35 TB/s of HBM3.
  e2e    rtpose.bin --image_dir frames/s at --precision 2 and 4 with few producer threads (the host is the bottleneck), runs with and
         without --gpu_decode alternating.

The result is printed as JSON; --out also writes it to a file.

usage: python tools/gpu_decode.py [--parts host,gpu,e2e] [--frames 400] [--out result.json]"""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
BIN = os.path.join(ROOT, "caffe_rtpose_b200", "rtpose.bin")
W, H = 1280, 720


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "no GPU"
    except OSError:
        return "no GPU"


def make_dir(n, distinct=40):
    from caffe_rtpose_b200 import engine, synth
    d = tempfile.mkdtemp(prefix="gpu_decode_")
    jpegs = [engine.encode_jpeg(synth.make_frame(i, H, W), 98) for i in range(distinct)]
    for i in range(n):
        with open(os.path.join(d, "f%05d.jpg" % i), "wb") as f:
            f.write(jpegs[i % distinct])
    return d, jpegs


def host_rates(d, reps=3):
    out = {}
    for rep in range(reps):
        for mode, flag in (("host_decode", []), ("entropy_only", ["--gpu_decode"])):
            r = subprocess.run([BIN, "--image_dir", d, "--decode_bench", "--num_producers", "1", "--model", "COCO", "--resolution", "%dx%d" % (W, H)]
                               + flag, capture_output=True, text=True, timeout=1200)
            assert r.returncode == 0, r.stderr[-2000:]
            fps = float(re.search(r"([0-9.]+) frames/s", r.stdout).group(1))
            out.setdefault(mode, []).append(fps)
    return {k: {"frames_per_s": sorted(v), "median": sorted(v)[len(v) // 2]} for k, v in out.items()}


def gpu_kernels(jpegs, batch=9, iters=40):
    import torch
    from caffe_rtpose_b200 import engine, synth
    e = engine.PoseEngine(engine.COCO_18, 656, 368, W, H, precision=engine.PREC_F16X2, max_batch=batch)
    e.set_weights(synth.make_weights(engine.COCO_18, "he"))
    bufs = [engine.read_jpeg_coefs(j) for j in jpegs[:batch]]
    for _ in range(3):
        e.forward_jpeg(bufs)
    e.sync()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            e.forward_jpeg(bufs)
        e.sync()
    times = {}
    for ev in prof.events():
        for k in ("jpeg_idct_kernel", "jpeg_color_kernel"):
            if k in ev.name:
                times.setdefault(k, []).append(ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total)
    e.close()
    hd = engine.jpeg_coef_header(bufs[0])
    blocks = (hd["total_bytes"] - 512) // 128
    # bytes each kernel must move per frame: coefficients in + planes out; planes in (each sample once) + BGR out
    need = {"jpeg_idct_kernel": (hd["total_bytes"] - 512) + 64 * blocks, "jpeg_color_kernel": 64 * blocks + W * H * 3}
    out = {}
    for k, v in times.items():
        us = sum(v) / len(v) / batch   # one launch covers the batch
        out[k] = {"launches": len(v), "us_per_frame": us, "bytes_per_frame": need[k],
                  "share_of_3.35TBps": need[k] / (us * 1e-6) / 3.35e12}
    out["coef_bytes_per_frame"] = int(hd["total_bytes"])
    return out


def e2e(d, producers=(2, 4, 8), precisions=(2, 4), reps=2):
    res = []
    for prec in precisions:
        for n in producers:
            for rep in range(reps):
                for flag in ([], ["--gpu_decode"]):
                    r = subprocess.run([BIN, "--image_dir", d, "--model", "COCO", "--caffeproto", "/nonexistent.prototxt", "--random_init", "he",
                                        "--resolution", "%dx%d" % (W, H), "--no_display", "--no_frame_drops", "--num_gpu", "1",
                                        "--precision", str(prec), "--num_producers", str(n)] + flag, capture_output=True, text=True, timeout=1800)
                    assert r.returncode == 0, r.stderr[-2000:]
                    m = re.search(r"# frames: (\d+)\s+\(([0-9.]+) frames/s overall", r.stderr)
                    res.append({"precision": prec, "producers": n, "gpu_decode": bool(flag), "frames": int(m.group(1)), "fps": float(m.group(2))})
                    print(json.dumps(res[-1]), flush=True)
    summary = {}
    for x in res:
        summary.setdefault("prec%d_prod%d_%s" % (x["precision"], x["producers"], "gpu" if x["gpu_decode"] else "host"), []).append(x["fps"])
    return {"runs": res, "fps": summary}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="host,gpu,e2e")
    ap.add_argument("--frames", type=int, default=400)
    ap.add_argument("--out", default="", help="also write the JSON result to this file")
    a = ap.parse_args()
    parts = a.parts.split(",")
    d, jpegs = make_dir(a.frames)
    try:
        result = {"card": card(), "cpu_cores": os.cpu_count(), "frame": "%dx%d quality 98 4:2:0" % (W, H), "jpeg_bytes": len(jpegs[0])}
        if "host" in parts:
            result["host"] = host_rates(d)
            print(json.dumps(result["host"]), flush=True)
        if "gpu" in parts:
            result["gpu"] = gpu_kernels(jpegs)
            print(json.dumps(result["gpu"]), flush=True)
        if "e2e" in parts:
            result["e2e"] = e2e(d)
        result["card_after"] = card()
    finally:
        shutil.rmtree(d, ignore_errors=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
