"""Writes tests/golden/jpeg_coefs.npz: small JPEG files (written by OpenCV's libjpeg) that cover what the coefficient stage
(pe_jpeg_read_coefs) and the GPU reconstruction must handle - 4:4:4 / 4:2:2 / 4:2:0, grey, progressive, restart intervals,
optimised Huffman tables, sizes that are not multiples of the MCU, chroma planes 1-2 samples wide, 16-bit quantisation tables.
The tests read the stored bytes, so the machines that run them need no OpenCV.  usage: python tools/gen_jpeg_fixtures.py"""
import os
import struct
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def dqt_to_16bit(data, factor):
    """Rewrites every DQT table as a 16-bit (Pq = 1) table with its entries multiplied by factor (clamped to 65535): a valid
    stream whose coefficients keep their values and whose dequantisation needs 16-bit entries."""
    out = bytearray(data[:2])
    p = 2
    while p < len(data):
        assert data[p] == 0xFF
        m = data[p + 1]
        if m == 0xDA:   # scan data to the end: copied as is
            out += data[p:]
            break
        ln = struct.unpack(">H", data[p + 2:p + 4])[0]
        seg = data[p + 4:p + 2 + ln]
        if m == 0xDB:
            body = bytearray()
            s = 0
            while s < len(seg):
                pq, tq = seg[s] >> 4, seg[s] & 15
                s += 1
                vals = (struct.unpack(">64H", seg[s:s + 128]) if pq else tuple(seg[s:s + 64]))
                s += 128 if pq else 64
                body.append(0x10 | tq)
                body += struct.pack(">64H", *[min(65535, v * factor) for v in vals])
            out += b"\xff\xdb" + struct.pack(">H", len(body) + 2) + body
        else:
            out += data[p:p + 2 + ln]
        p += 2 + ln
    return bytes(out)


def main():
    import cv2
    from caffe_rtpose_b200 import synth
    files = {}

    def pic(seed, h, w):
        img = synth.make_frame(seed, h, w)
        return cv2.GaussianBlur(img, (0, 0), 1.2) if min(h, w) > 8 else img

    Q = cv2.IMWRITE_JPEG_QUALITY
    S = cv2.IMWRITE_JPEG_SAMPLING_FACTOR
    samp = {"444": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, "422": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
            "420": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420}
    for name, sf in samp.items():
        for (h, w) in ((48, 64), (61, 83)):
            img = pic(1, h, w)
            files["%s_%dx%d" % (name, w, h)] = cv2.imencode(".jpg", img, [Q, 90, S, sf])[1].tobytes()
            files["%s_%dx%d_progressive" % (name, w, h)] = cv2.imencode(".jpg", img, [Q, 85, S, sf, cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()
        files["%s_restart3" % name] = cv2.imencode(".jpg", pic(2, 37, 59), [Q, 80, S, sf, cv2.IMWRITE_JPEG_RST_INTERVAL, 3])[1].tobytes()
        for w in (1, 2, 3, 4):   # chroma planes 1-2 samples wide (replication instead of the triangle filter)
            files["%s_narrow_%dx13" % (name, w)] = cv2.imencode(".jpg", pic(3, 13, w), [Q, 95, S, sf])[1].tobytes()
    files["420_progressive_restart2"] = cv2.imencode(".jpg", pic(4, 40, 70), [Q, 80, cv2.IMWRITE_JPEG_PROGRESSIVE, 1,
                                                                             cv2.IMWRITE_JPEG_RST_INTERVAL, 2])[1].tobytes()
    files["420_optimised_huffman"] = cv2.imencode(".jpg", pic(5, 45, 66), [Q, 92, cv2.IMWRITE_JPEG_OPTIMIZE, 1])[1].tobytes()
    files["420_q100"] = cv2.imencode(".jpg", pic(6, 33, 47), [Q, 100])[1].tobytes()
    files["420_q5"] = cv2.imencode(".jpg", pic(6, 33, 47), [Q, 5])[1].tobytes()
    files["grey_51x29"] = cv2.imencode(".jpg", pic(7, 29, 51)[:, :, 1], [Q, 90])[1].tobytes()
    files["grey_progressive"] = cv2.imencode(".jpg", pic(7, 29, 51)[:, :, 1], [Q, 90, cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()
    files["420_dqt16"] = dqt_to_16bit(cv2.imencode(".jpg", pic(8, 40, 56), [Q, 90])[1].tobytes(), 300)
    files["444_dqt16_progressive"] = dqt_to_16bit(cv2.imencode(".jpg", pic(8, 40, 56), [Q, 90, S, samp["444"],
                                                                                       cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes(), 7)
    noise = np.random.default_rng(9).integers(0, 256, (24, 40, 3), dtype=np.uint8)   # saturating colours: range limits
    files["420_noise_q100"] = cv2.imencode(".jpg", noise, [Q, 100])[1].tobytes()
    files["444_noise_q100"] = cv2.imencode(".jpg", noise, [Q, 100, S, samp["444"]])[1].tobytes()
    out = os.path.join(ROOT, "tests", "golden", "jpeg_coefs.npz")
    np.savez_compressed(out, **{k: np.frombuffer(v, np.uint8) for k, v in sorted(files.items())})
    print("%s: %d files, %d bytes" % (out, len(files), os.path.getsize(out)))


if __name__ == "__main__":
    main()
