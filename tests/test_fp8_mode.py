"""The FP8 mode (PE_PREC_E4M3X1) without a GPU.

* The host float -> e4m3 conversion of the packed weights (csrc/e4m3.h), compiled on its own with g++, equals torch's
  float8_e4m3fn cast wherever the result stays within +-448: on every e4m3 value, the midpoints between neighbours (ties to
  even) and the floats just either side of them, the subnormals, signed zero and random values over the whole range.  Larger
  magnitudes, infinities included, saturate to +-448 (0x7E / 0xFE), as cvt.rn.satfinite does on the device.
* conv_fp8.cu, the e4m3 instances of conv_wg_kernel, built with -Xptxas -v: the checks of test_conv_build.py (no spills, no
  serialised wgmma, one wgmma group in flight) for every instance, and the FP8 MMA in the SASS.
"""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from test_conv_build import check_no_spills_and_no_serialised_wgmma, check_one_wgmma_group_in_flight, tu_build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "caffe_rtpose_b200", "csrc")
# <BN, 1, e4m3, e4m3> and <BN, 1, fp16, e4m3> (conv1_1) at BN = 16, 32, 48, 64, 128
INSTANCES = 10

HARNESS = r"""
#include <stdio.h>
#include <string.h>
#include "e4m3.h"
int main() {   // float bits (hex) on stdin -> e4m3 byte per line
    unsigned u;
    while (scanf("%x", &u) == 1) { float f; memcpy(&f, &u, 4); printf("%d\n", pe::float_to_e4m3(f)); }
    return 0;
}
"""


@pytest.fixture(scope="module")
def to_e4m3(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not found")
    d = tmp_path_factory.mktemp("e4m3")
    src, exe = d / "h.cpp", d / "h"
    src.write_text(HARNESS)
    subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-I", CSRC, str(src), "-o", str(exe)], check=True)

    def run(x):
        x = np.ascontiguousarray(x, dtype=np.float32)
        out = subprocess.run([str(exe)], input="\n".join("%08x" % v for v in x.view(np.uint32)), capture_output=True, text=True,
                             check=True).stdout.split()
        return np.array(out, dtype=np.int64).astype(np.uint8)
    return run


def torch_e4m3(x):
    t = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(torch.float8_e4m3fn)
    return t.view(torch.uint8).numpy(), t.float().numpy()


def sweep():
    allv = torch.arange(256, dtype=torch.uint8).view(torch.float8_e4m3fn).float().numpy()
    fin = np.unique(allv[np.isfinite(allv)]).astype(np.float32)        # every finite value, -448 .. 448, one zero
    mids = ((fin[1:].astype(np.float64) + fin[:-1]) / 2).astype(np.float32)   # exact in fp32: the ties
    up, down = np.nextafter(mids, np.float32(np.inf)), np.nextafter(mids, np.float32(-np.inf))
    rng = np.random.default_rng(3)
    rand = np.concatenate([rng.standard_normal(4000) * s for s in (1e-3, 0.02, 1.0, 30.0, 200.0)]).astype(np.float32)
    sub = (np.arange(-40, 41) * 2.0 ** -12).astype(np.float32)            # around and inside the subnormals (spacing 2^-9)
    edge = np.array([0.0, -0.0, 2.0 ** -6, -2.0 ** -6, 2.0 ** -10, 3 * 2.0 ** -10, 2.0 ** -9, 2.0 ** -7 * 1.5, 448.0, -448.0,
                     447.99, 455.99, 456.0, 456.01, 463.99, -463.99], np.float32)   # 456: the tie of 416 / 448
    return np.concatenate([fin, mids, up, down, rand, sub, edge])


def test_host_e4m3_equals_torch(to_e4m3):
    x = sweep()
    got = to_e4m3(x)
    want, val = torch_e4m3(x)
    inside = np.isfinite(val) & (np.abs(val) <= 448)
    assert inside.sum() > 20000
    bad = np.flatnonzero(inside & (got != want))
    assert bad.size == 0, [(float(x[i]), int(got[i]), int(want[i])) for i in bad[:10]]
    # signed zero keeps its sign; the ties went to even mantissas
    assert to_e4m3(np.array([0.0, -0.0], np.float32)).tolist() == [0x00, 0x80]


def test_host_e4m3_saturates_beyond_448(to_e4m3):
    x = np.array([464.0, 464.01, 479.9, 480.0, 500.0, 1e6, 3e38, np.inf, -464.0, -480.0, -1e6, -np.inf], np.float32)
    got = to_e4m3(x)
    assert got.tolist() == [0x7E] * 8 + [0xFE] * 4, got
    _, val = torch_e4m3(x[[1, 3, 5]])
    assert np.isnan(val).all()   # torch's cast: NaN where the device saturates
    # 464 is the tie between 448 (even mantissa) and the first value past the format, so it rounds down like the device's
    assert to_e4m3(np.array([np.nan], np.float32))[0] & 0x7F == 0x7F


build = tu_build("conv_fp8.cu")


def test_fp8_instances_no_spills_and_no_serialised_wgmma(build):
    check_no_spills_and_no_serialised_wgmma(build[0], INSTANCES)


def test_fp8_instances_keep_one_wgmma_group_in_flight(build):
    kernels = check_one_wgmma_group_in_flight(build[1], INSTANCES)
    n_e4m3 = 0
    for name, text in kernels.items():
        assert "F2FP.SATFINITE.E4M3" in text, name     # the epilogue's cvt.rn.satfinite.e4m3x2.f32
        n_e4m3 += bool(re.search(r"QGMMA\.64x\d+x32\.F32\.E4M3\.E4M3", text))
    assert n_e4m3 == INSTANCES // 2, n_e4m3            # the fp16-input conv1_1 instances run fp16 MMAs
