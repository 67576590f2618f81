"""What ptxas makes of conv_wg_kernel (conv_tc.cu), checked without a GPU.

The consumer loop keeps one wgmma group in flight: it issues K step s, waits with wgmma.wait_group 1 for step s - 1 and
only then frees step s - 1's shared-memory slots; a hi*hi chunk ends with wait_group 0 and the round-to-nearest chunk sum.
ptxas can undo that silently: when it cannot prove that no accumulator register is touched while a group writing it is in
flight, it serialises the wgmma instructions (a performance warning) and waits for every group.  So for every instance:
no spills, no such warning, and in the SASS a WARPGROUP.DEPBAR.LE gsb0, 0x1 (the wait for all but the last group).
test_fp8_mode.py and test_s8_mode.py run the same build and checks on conv_fp8.cu and conv_s8.cu (tu_build and the check_
helpers).
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "caffe_rtpose_b200", "csrc")
NVCC = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
INSTANCES = 19   # <BN, P, F16>: BN 16-128 at P = 1 (fp16, bf16) and P = 2 (fp16); BN <= 64 at P = 3 (bf16)


def tu_build(tu):
    """A module fixture: (ptxas -v log, cuobjdump -sass listing) of csrc/<tu> compiled for sm_90a."""
    @pytest.fixture(scope="module")
    def build(tmp_path_factory):
        if NVCC is None:
            pytest.skip("nvcc not found")
        obj = str(tmp_path_factory.mktemp("conv_build") / (tu + ".o"))
        r = subprocess.run([NVCC, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC",
                            "--expt-relaxed-constexpr", "-Xptxas", "-v", "-x", "cu", "-c", os.path.join(CSRC, tu), "-o", obj],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-4000:]
        cuobjdump = os.path.join(os.path.dirname(os.path.realpath(NVCC)), "cuobjdump")
        sass = subprocess.run([cuobjdump if os.path.exists(cuobjdump) else "cuobjdump", "-sass", obj],
                              capture_output=True, text=True, check=True).stdout
        return r.stderr, sass
    return build


build = tu_build("conv_tc.cu")


def per_kernel(text, start):
    """{mangled conv_wg_kernel name: its lines} of ptxas's log or cuobjdump's listing."""
    out, cur = {}, None
    for line in text.splitlines():
        m = re.search(start, line)
        if m:
            cur = m.group(1) if "conv_wg_kernel" in m.group(1) else None
            if cur:
                out[cur] = []
            continue
        if cur:
            out[cur].append(line)
    return out


def check_no_spills_and_no_serialised_wgmma(log, instances):
    kernels = per_kernel(log, r"(?:Compiling entry function|Function properties for) '?(\w+)")
    assert len(kernels) == instances, sorted(kernels)
    for name, lines in kernels.items():
        text = "\n".join(lines)
        spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", text)
        assert spill and spill.groups() == ("0", "0"), (name, text)
    assert not re.search(r"wgmma.*serializ", log, re.I), [l for l in log.splitlines() if re.search("serializ", l, re.I)]


def check_one_wgmma_group_in_flight(sass, instances):
    """{kernel: its SASS text}, after checking every instance's waits."""
    kernels = per_kernel(sass, r"Function : (\w+)")
    assert len(kernels) == instances, sorted(kernels)
    for name, lines in kernels.items():
        waits = [l for l in lines if "WARPGROUP.DEPBAR.LE" in l]
        assert any("gsb0, 0x1" in l for l in waits), (name, waits)   # steady state: wait for all but the newest group
        assert any("gsb0, 0x0" in l for l in waits), (name, waits)   # chunk end: wait for every group
    return {name: "\n".join(lines) for name, lines in kernels.items()}


def test_no_spills_and_no_serialised_wgmma(build):
    check_no_spills_and_no_serialised_wgmma(build[0], INSTANCES)


def test_one_wgmma_group_stays_in_flight(build):
    check_one_wgmma_group_in_flight(build[1], INSTANCES)
