"""Measurements of GPU JPEG decoding on 720p frames, three routes: the host decoder, --gpu_decode (pe_forward_jpeg_coefs: entropy
stage on the host, reconstruction on the GPU) and --gpu_entropy (pe_forward_jpeg_scans: the host only parses, Huffman decoding on the
GPU too).  Workloads: quality 98 (the generator's detailed frames), quality 85 (camera-typical) and quality 85 with a restart marker
every 4 MCUs (cv2; "not measured" without it), since the synchronisation cost of the GPU Huffman decoder depends on the data.

  host   frames/s of ONE producer thread for each route (--decode_bench, --decode_bench --gpu_decode / --gpu_entropy); no GPU needed.
  gpu    per-frame device time of every JPEG kernel (torch.profiler CUDA activity over many forwards, a run of its own), the bytes the
         reconstruction kernels move against 3.35 TB/s, the entropy-coded GB/s of the Huffman kernels, and the JPEG kernels' share of
         the whole forward's device time (net at 656x368, parity mode).
  e2e    rtpose.bin --image_dir frames/s at --precision 2 and 4 with 2, 4 and 8 producer threads, the three routes alternating.

The result is printed as JSON; --out also writes it to a file.

usage: python tools/gpu_decode.py [--parts host,gpu,e2e] [--workloads q98,q85,q85_rst4] [--frames 400] [--reps 2] [--out result.json]"""
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


ROUTES = (("host_decode", []), ("gpu_decode", ["--gpu_decode"]), ("gpu_entropy", ["--gpu_entropy"]))
ENTROPY_KERNELS = ("jpeg_scan_prep_kernel", "jpeg_huffman_kernel", "jpeg_dc_kernel")
RECON_KERNELS = ("jpeg_idct_kernel", "jpeg_color_kernel")


def encode(workload, img):
    from caffe_rtpose_b200 import engine
    if workload == "q98":
        return engine.encode_jpeg(img, 98)
    if workload == "q85":
        return engine.encode_jpeg(img, 85)
    import cv2   # restart intervals: the project's encoder writes none
    ok, buf = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 85, cv2.IMWRITE_JPEG_RST_INTERVAL, int(workload.split("rst")[1])])
    assert ok
    return buf.tobytes()


def make_dir(n, workload, distinct=40):
    from caffe_rtpose_b200 import synth
    d = tempfile.mkdtemp(prefix="gpu_decode_")
    jpegs = [encode(workload, synth.make_frame(i, H, W)) for i in range(distinct)]
    for i in range(n):
        with open(os.path.join(d, "f%05d.jpg" % i), "wb") as f:
            f.write(jpegs[i % distinct])
    return d, jpegs


def host_rates(d, reps=3):
    out = {}
    for rep in range(reps):
        for mode, flag in ROUTES:
            r = subprocess.run([BIN, "--image_dir", d, "--decode_bench", "--num_producers", "1", "--model", "COCO", "--resolution", "%dx%d" % (W, H)]
                               + flag, capture_output=True, text=True, timeout=1200)
            assert r.returncode == 0, r.stderr[-2000:]
            fps = float(re.search(r"([0-9.]+) frames/s", r.stdout).group(1))
            out.setdefault(mode, []).append(fps)
    return {k: {"frames_per_s": sorted(v), "median": sorted(v)[len(v) // 2]} for k, v in out.items()}


def _profile(e, bufs, entropy, iters):
    import torch
    for _ in range(3):
        e.forward_jpeg(bufs, entropy=entropy)
    e.sync()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            e.forward_jpeg(bufs, entropy=entropy)
        e.sync()
    times, total = {}, 0.0
    for ev in prof.events():
        t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            total += t
        for k in RECON_KERNELS + ENTROPY_KERNELS:
            if k in ev.name:
                times.setdefault(k, []).append(t)
    return times, total


def gpu_kernels(jpegs, batch=9, iters=40):
    from caffe_rtpose_b200 import engine, synth
    e = engine.PoseEngine(engine.COCO_18, 656, 368, W, H, precision=engine.PREC_F16X2, max_batch=batch)
    e.set_weights(synth.make_weights(engine.COCO_18, "he"))
    bufs = [engine.read_jpeg_coefs(j) for j in jpegs[:batch]]
    scans = [engine.read_jpeg_scan(j) for j in jpegs[:batch]]
    times, total_host = _profile(e, bufs, "host", iters)
    etimes, total_gpu = _profile(e, scans, "gpu", iters)
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
    ecs = sum(int(s[576 + 16:576 + 24].view("int64")[0]) for s in scans) / len(scans)   # data_bytes of the scan header
    ent_us = 0.0
    for k in ENTROPY_KERNELS:
        v = etimes.get(k, [])
        us = sum(v) / max(len(v), 1) / batch
        ent_us += us
        out[k] = {"launches": len(v), "us_per_frame": us}
    out["entropy_coded_bytes_per_frame"] = int(ecs)
    out["huffman_GBps_entropy_coded"] = ecs / (out["jpeg_huffman_kernel"]["us_per_frame"] * 1e-6) / 1e9 if out["jpeg_huffman_kernel"]["us_per_frame"] else None
    out["entropy_kernels_us_per_frame"] = ent_us
    out["forward_device_us_per_frame"] = {"gpu_decode": total_host / iters / batch, "gpu_entropy": total_gpu / iters / batch}
    net_us = total_host / iters / batch - sum(out[k]["us_per_frame"] for k in RECON_KERNELS if k in out)
    out["entropy_kernels_share_of_net"] = ent_us / net_us if net_us > 0 else None
    return out


def e2e(d, producers=(2, 4, 8), precisions=(2, 4), reps=1):
    res = []
    for prec in precisions:
        for n in producers:
            for rep in range(reps):
                for route, flag in ROUTES:
                    r = subprocess.run([BIN, "--image_dir", d, "--model", "COCO", "--caffeproto", "/nonexistent.prototxt", "--random_init", "he",
                                        "--resolution", "%dx%d" % (W, H), "--no_display", "--no_frame_drops", "--num_gpu", "1",
                                        "--precision", str(prec), "--num_producers", str(n)] + flag, capture_output=True, text=True, timeout=1800)
                    assert r.returncode == 0, r.stderr[-2000:]
                    m = re.search(r"# frames: (\d+)\s+\(([0-9.]+) frames/s overall", r.stderr)
                    res.append({"precision": prec, "producers": n, "route": route, "frames": int(m.group(1)), "fps": float(m.group(2))})
                    print(json.dumps(res[-1]), flush=True)
    summary = {}
    for x in res:
        summary.setdefault("prec%d_prod%d_%s" % (x["precision"], x["producers"], x["route"]), []).append(x["fps"])
    return {"runs": res, "fps": summary}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="host,gpu,e2e")
    ap.add_argument("--frames", type=int, default=400)
    ap.add_argument("--workloads", default="q98,q85,q85_rst4")
    ap.add_argument("--e2e_workloads", default="q98,q85,q85_rst4")
    ap.add_argument("--reps", type=int, default=1, help="end-to-end runs per configuration")
    ap.add_argument("--out", default="", help="also write the JSON result to this file")
    a = ap.parse_args()
    parts = a.parts.split(",")
    result = {"card": card(), "cpu_cores": os.cpu_count(), "frame": "%dx%d 4:2:0" % (W, H)}
    for wl in a.workloads.split(","):
        try:
            d, jpegs = make_dir(a.frames, wl)
        except ImportError:
            result[wl] = "not measured (no cv2)"
            continue
        try:
            r = result[wl] = {"jpeg_bytes": len(jpegs[0])}
            if "host" in parts:
                r["host"] = host_rates(d)
                print(json.dumps({wl: r["host"]}), flush=True)
            if "gpu" in parts:
                r["gpu"] = gpu_kernels(jpegs)
                print(json.dumps({wl: r["gpu"]}), flush=True)
            if "e2e" in parts and wl in a.e2e_workloads.split(","):
                r["e2e"] = e2e(d, reps=a.reps)
        finally:
            shutil.rmtree(d, ignore_errors=True)
    result["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
