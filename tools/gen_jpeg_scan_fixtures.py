"""Writes tests/golden/jpeg_scans.npz: sequential JPEG streams for the GPU entropy decoder's tests, written by OpenCV's libjpeg
(restart intervals 1, 7 and 64, optimised Huffman tables, 4:2:2 / 4:2:0 / 4:4:4, grey) plus byte edits of them: Motion-JPEG frames
without their DHT segment, and a scan whose SOS lists the chroma components in the other order than the SOF.
usage: python tools/gen_jpeg_scan_fixtures.py"""
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from caffe_rtpose_b200 import synth  # noqa: E402

S420, S422, S444 = cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444


def enc(img, quality, restart=0, optimize=False, sampling=S420):
    params = [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_RST_INTERVAL, restart, cv2.IMWRITE_JPEG_OPTIMIZE, int(optimize)]
    if img.ndim == 3:
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, sampling]
    ok, buf = cv2.imencode(".jpg", img, params)
    assert ok
    return buf.tobytes()


def strip_dht(jpeg):
    while True:
        p = jpeg.find(b"\xff\xc4")
        if p < 0:
            return jpeg
        n = int.from_bytes(jpeg[p + 2:p + 4], "big")
        jpeg = jpeg[:p] + jpeg[p + 2 + n:]


def swap_sos_chroma(jpeg):
    """the SOS names Cr before Cb (each with its own tables): the blocks of an MCU then follow SOS order"""
    p = jpeg.find(b"\xff\xda")
    d = bytearray(jpeg)
    assert d[p + 4] == 3
    d[p + 7:p + 9], d[p + 9:p + 11] = jpeg[p + 9:p + 11], jpeg[p + 7:p + 9]
    return bytes(d)


def main():
    out = {}
    a = synth.make_frame(1, 120, 160)
    b = synth.make_frame(2, 97, 131)   # partial MCUs
    for r in (1, 7, 64):
        out["420_restart%d" % r] = enc(a, 85, r)
        out["422_restart%d_q98" % r] = enc(b, 98, r, sampling=S422)
    out["420_optimized"] = enc(a, 85, optimize=True)
    out["444_optimized_restart7"] = enc(b, 90, 7, optimize=True, sampling=S444)
    out["422_q50"] = enc(b, 50, sampling=S422)
    out["grey_restart7"] = enc(cv2.cvtColor(a, cv2.COLOR_BGR2GRAY), 85, 7)
    out["grey_q98"] = enc(cv2.cvtColor(b, cv2.COLOR_BGR2GRAY), 98)
    out["mjpeg_no_dht"] = strip_dht(enc(a, 85))
    out["mjpeg_no_dht_restart7"] = strip_dht(enc(b, 90, 7, sampling=S422))
    out["sos_order_cr_cb"] = swap_sos_chroma(enc(a, 85))
    out["sos_order_cr_cb_restart1"] = swap_sos_chroma(enc(b, 90, 1, sampling=S444))
    path = os.path.join(ROOT, "tests", "golden", "jpeg_scans.npz")
    np.savez_compressed(path, **{k: np.frombuffer(v, np.uint8) for k, v in out.items()})
    print("wrote %s: %d streams, %d bytes" % (path, len(out), os.path.getsize(path)))


if __name__ == "__main__":
    main()
