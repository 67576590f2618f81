"""The INT8 mode (PE_PREC_S8X1) without a GPU.

* The host weight quantisation of the packer (csrc/s8.h), compiled on its own with g++, equals a numpy float32 restatement of
  the rule of poseengine.h - sigma = max|w| / 127, q = clamp(rint(w / sigma), -127, 127) - bit for bit: sigma's bits and every
  q, on random channels of several magnitudes, on channels whose values are exact .5 multiples of sigma (ties go to even), on
  all-zero channels (sigma = 0, q = 0) and on a channel with a single non-zero weight.
* The accumulator bound: the engine's largest K (precision.h) is the largest for which 128 x 127 x K fits in s32.
* conv_s8.cu, the s8 instances of conv_wg_kernel, built with -Xptxas -v: the checks of test_conv_build.py (no spills, no
  serialised wgmma, one wgmma group in flight) for every instance, the s8 MMA and the saturating s8 conversion in the SASS.
* rtpose.bin: --help lists --precision 6, and --precision 6 without range calibration is refused at start-up.
"""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from test_conv_build import check_no_spills_and_no_serialised_wgmma, check_one_wgmma_group_in_flight, tu_build
from test_precision_table import read_table

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "caffe_rtpose_b200", "csrc")
BIN = os.path.join(ROOT, "caffe_rtpose_b200", "rtpose.bin")
INSTANCES = 5   # <BN, 1, s8, s8> at BN = 16, 32, 48, 64, 128

HARNESS = r"""
#include <stdio.h>
#include <string.h>
#include <vector>
#include "s8.h"
int main() {   // per channel on stdin: n, then n float bits (hex) -> sigma bits (hex) and the n q values on one line
    size_t n;
    while (scanf("%zu", &n) == 1) {
        std::vector<float> w(n);
        std::vector<int8_t> q(n);
        for (size_t i = 0; i < n; i++) { unsigned u; if (scanf("%x", &u) != 1) return 1; memcpy(&w[i], &u, 4); }
        const float s = pe::s8_quantize_channel(w.data(), n, q.data());
        unsigned su; memcpy(&su, &s, 4);
        printf("%08x", su);
        for (size_t i = 0; i < n; i++) printf(" %d", q[i]);
        printf("\n");
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def quantize(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not found")
    d = tmp_path_factory.mktemp("s8")
    src, exe = d / "h.cpp", d / "h"
    src.write_text(HARNESS)
    subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-I", CSRC, str(src), "-o", str(exe)], check=True)

    def run(channels):
        text = "\n".join("%d %s" % (len(c), " ".join("%08x" % v for v in np.ascontiguousarray(c, np.float32).view(np.uint32)))
                         for c in channels)
        lines = subprocess.run([str(exe)], input=text, capture_output=True, text=True, check=True).stdout.splitlines()
        out = []
        for line in lines:
            f = line.split()
            out.append((np.array([int(f[0], 16)], np.uint32).view(np.float32)[0], np.array(f[1:], np.int64)))
        return out
    return run


def numpy_quantize(w):
    """The rule of poseengine.h in numpy float32: (sigma, q)."""
    w = np.asarray(w, np.float32)
    sigma = np.float32(np.abs(w).max()) / np.float32(127)
    if sigma == 0:
        return np.float32(0), np.zeros(w.size, np.int64)
    return np.float32(sigma), np.clip(np.rint(w / sigma), -127, 127).astype(np.int64)


def channels():
    rng = np.random.default_rng(8)
    out = [(rng.standard_normal(n) * s).astype(np.float32) for n in (27, 128, 1152, 6272) for s in (1e-4, 0.03, 1.0, 300.0)]
    out += [(rng.uniform(-1, 1, 500) * 2.0 ** e).astype(np.float32) for e in (-30, -3, 12)]
    # ties: sigma = 2^e exactly (max|w| = 127 * 2^e), every (j + 1/2) * sigma for j in -127..126, and the integers
    for e in (-7, 0, 3):
        t = np.concatenate([np.arange(-127, 127) + 0.5, np.arange(-127, 128), [127.0]]) * 2.0 ** e
        out.append(rng.permutation(t).astype(np.float32))
    out += [np.zeros(27, np.float32), np.zeros(1152, np.float32), np.array([0.0, -0.0, 0.0], np.float32)]
    one = np.zeros(64, np.float32)
    one[17] = -2.5e-3
    out.append(one)
    return out


def test_host_quantisation_equals_numpy(quantize):
    chans = channels()
    got = quantize(chans)
    assert len(got) == len(chans)
    ties = 0
    for w, (sigma, q) in zip(chans, got):
        ws, wq = numpy_quantize(w)
        assert np.float32(sigma).view(np.uint32) == np.float32(ws).view(np.uint32), (sigma, ws)
        assert np.array_equal(q, wq), np.flatnonzero(q != wq)[:10]
        assert np.abs(q).max(initial=0) <= 127
        if sigma > 0:
            r = w / np.float32(sigma)
            ties += int((r - np.floor(r) == 0.5).sum())
    assert ties >= 3 * 254   # the tie channels really hit exact halves: even q
    # the ties went to even integers, and the channel's maximum to exactly +-127
    sigma, q = got[-5]   # the tie channel at sigma = 2^3
    half = chans[-5] / np.float32(8) % 1 == 0.5
    assert sigma == 8.0 and half.sum() == 254 and np.all(q[half] % 2 == 0)
    assert got[-1][1][17] == -127 and np.count_nonzero(got[-1][1]) == 1


def test_accumulator_bound(tmp_path):
    """|acc| <= 128 x 127 x K: the engine's bound K = 132104 stays inside s32, K = 132105 does not."""
    max_k = read_table(tmp_path)["S8X1"]["max_k"]
    assert max_k == 132104
    assert 128 * 127 * max_k <= 2 ** 31 - 1 < 128 * 127 * (max_k + 1)
    assert 49 * 2816 > max_k   # a 7x7 on 2700 channels (padded to 2816) is over it; the shipped nets' largest K is 49 x 256


build = tu_build("conv_s8.cu")


def test_s8_instances_no_spills_and_no_serialised_wgmma(build):
    check_no_spills_and_no_serialised_wgmma(build[0], INSTANCES)


def test_s8_instances_keep_one_wgmma_group_in_flight(build):
    kernels = check_one_wgmma_group_in_flight(build[1], INSTANCES)
    widths = set()
    for name, text in kernels.items():
        m = re.findall(r"IGMMA\.64x(\d+)x32\.S8\.S8", text)
        assert m, name                                   # wgmma m64nNk32.s32.s8.s8
        widths |= {int(x) for x in m}
        assert "F2I.S8" in text, name                    # the epilogue's cvt.rni.sat.s8.f32
        assert not re.search(r"[HQ]GMMA", text), name    # no fp16 / fp8 MMA in an s8 instance
    assert widths == {16, 32, 48, 64, 128}, widths


def run_bin(args):
    return subprocess.run([BIN] + args, capture_output=True, text=True, timeout=60)


@pytest.fixture(scope="module")
def rtpose_bin():
    if not os.path.exists(BIN):
        pytest.skip("rtpose.bin not built")
    return BIN


def test_help_lists_precision_6(rtpose_bin):
    r = run_bin(["--help"])
    assert r.returncode == 0
    line = [l for l in r.stdout.splitlines() if l.strip().startswith("--precision ")][0]
    assert "6 INT8 mode" in line


@pytest.mark.parametrize("flag", ["--nocalibrate_range", "--calibrate_range=false"])
def test_precision_6_without_calibration_refused(rtpose_bin, flag):
    r = run_bin(["--synthetic", "2", "--model", "COCO", "--precision", "6", flag])
    assert r.returncode == 1 and "--precision 6" in r.stderr and "calibrate" in r.stderr, r.stderr
