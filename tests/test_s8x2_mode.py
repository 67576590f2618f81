"""The 16-bit integer mode (PE_PREC_S8X2) without a GPU.

* The host weight quantisation of the packer (csrc/s8.h, s8x2_quantize_channel), compiled on its own with g++, equals a numpy
  float32 restatement of the rule of poseengine.h - sigma = max|w| / 32639, q = clamp(rint(w / sigma), -32639, 32639), split
  into hi = (q + 128) >> 8 and lo = q - 256 hi - bit for bit, on random channels of several magnitudes, on channels of exact
  .5 multiples of sigma (ties go to even), on all-zero channels and on a channel with a single non-zero weight (+-max).
* The split (s8x2_split) followed by 256 hi + lo is the identity on every v in [-32768, 32639], with both planes in [-128, 127].
* The precision row and the accumulator bound: K = 65793 is the largest for which (128 x 128 + 128 x 127) x K fits in s32.
* conv_s8x2.cu, the two-plane s8 instances of conv_wg_kernel, built with -Xptxas -v: no spills, no serialised wgmma, one wgmma
  group in flight, three s8 MMAs per K step and no fp16 / fp8 MMA.
* The SASS of every conv_wg_kernel instance of the other conv translation units is the one the mode's parent commit built
  (golden/conv_sass_sha256.json: SHA-256 of each kernel's cuobjdump -sass listing).
* The mode's number is 8, and 7 stays an unknown precision.
* rtpose.bin: --help lists --precision 8; --precision 8 without range calibration, the u8 flag with precision 8 and
  pe_create_mixed with base precision 8 are refused.
"""
import ctypes
import hashlib
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from test_conv_build import NVCC, check_no_spills_and_no_serialised_wgmma, check_one_wgmma_group_in_flight, tu_build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "caffe_rtpose_b200", "csrc")
BIN = os.path.join(ROOT, "caffe_rtpose_b200", "rtpose.bin")
GOLDEN = os.path.join(ROOT, "tests", "golden", "conv_sass_sha256.json")
INSTANCES = 5   # <BN, 2, s8, s8> at BN = 16, 32, 48, 64, 128
MAX_K = 65793
PE_ERR_INVALID = 1   # poseengine.h

HARNESS = r"""
#include <stdio.h>
#include <string.h>
#include <vector>
#include "s8.h"
int main(int argc, char** argv) {
    if (argc > 1) {   // split: every v in [-32768, 32639] -> a "v hi lo" line where 256 hi + lo != v, then the counts
        long bad = 0;
        for (int v = -32768; v <= 32639; v++) {
            int8_t hi, lo;
            pe::s8x2_split(v, &hi, &lo);
            if (256 * hi + lo != v) { printf("%d %d %d\n", v, hi, lo); bad++; }
        }
        printf("checked %d bad %ld\n", 32639 + 32768 + 1, bad);
        return 0;
    }
    size_t n;   // per channel on stdin: n, then n float bits (hex) -> sigma bits (hex), the n hi values, the n lo values
    while (scanf("%zu", &n) == 1) {
        std::vector<float> w(n);
        std::vector<int8_t> hi(n), lo(n);
        for (size_t i = 0; i < n; i++) { unsigned u; if (scanf("%x", &u) != 1) return 1; memcpy(&w[i], &u, 4); }
        const float s = pe::s8x2_quantize_channel(w.data(), n, hi.data(), lo.data());
        unsigned su; memcpy(&su, &s, 4);
        printf("%08x", su);
        for (size_t i = 0; i < n; i++) printf(" %d", hi[i]);
        for (size_t i = 0; i < n; i++) printf(" %d", lo[i]);
        printf("\n");
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not found")
    d = tmp_path_factory.mktemp("s8x2")
    src, exe = d / "h.cpp", d / "h"
    src.write_text(HARNESS)
    subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-I", CSRC, str(src), "-o", str(exe)], check=True)
    return str(exe)


def quantize_host(exe, channels):
    text = "\n".join("%d %s" % (len(c), " ".join("%08x" % v for v in np.ascontiguousarray(c, np.float32).view(np.uint32)))
                     for c in channels)
    lines = subprocess.run([exe], input=text, capture_output=True, text=True, check=True).stdout.splitlines()
    out = []
    for line, c in zip(lines, channels):
        f = line.split()
        vals = np.array(f[1:], np.int64)
        out.append((np.array([int(f[0], 16)], np.uint32).view(np.float32)[0], vals[:len(c)], vals[len(c):]))
    assert len(out) == len(channels)
    return out


def numpy_quantize(w):
    """The rule of poseengine.h in numpy float32: (sigma, q, hi, lo)."""
    w = np.asarray(w, np.float32)
    sigma = np.float32(np.abs(w).max()) / np.float32(32639)
    q = np.zeros(w.size, np.int64) if sigma == 0 else np.clip(np.rint(w / sigma), -32639, 32639).astype(np.int64)
    hi = (q + 128) >> 8
    return np.float32(sigma), q, hi, q - 256 * hi


def channels():
    rng = np.random.default_rng(16)
    out = [(rng.standard_normal(n) * s).astype(np.float32) for n in (27, 128, 1152, 6272) for s in (1e-4, 0.03, 1.0, 300.0)]
    out += [(rng.uniform(-1, 1, 500) * 2.0 ** e).astype(np.float32) for e in (-30, -3, 12)]
    # ties: sigma = 2^e exactly (max|w| = 32639 * 2^e), (j + 1/2) * sigma for j in -300..299 and around +-32639, and integers
    for e in (-7, 0, 3):
        j = np.concatenate([np.arange(-300, 300), np.arange(-32639, -32600), np.arange(32600, 32639)])
        t = np.concatenate([j + 0.5, j, [32639.0, -32639.0]]) * 2.0 ** e
        out.append(rng.permutation(t).astype(np.float32))
    out += [np.zeros(27, np.float32), np.zeros(1152, np.float32), np.array([0.0, -0.0, 0.0], np.float32)]
    for v in (-2.5e-3, 7.0):   # one non-zero weight: q = +-32639 there, 0 elsewhere
        one = np.zeros(64, np.float32)
        one[17] = v
        out.append(one)
    return out


def test_host_quantisation_equals_numpy(harness):
    chans = channels()
    got = quantize_host(harness, chans)
    ties = 0
    for w, (sigma, hi, lo) in zip(chans, got):
        ws, wq, whi, wlo = numpy_quantize(w)
        assert np.float32(sigma).view(np.uint32) == np.float32(ws).view(np.uint32), (sigma, ws)
        assert np.array_equal(hi, whi) and np.array_equal(lo, wlo), np.flatnonzero((hi != whi) | (lo != wlo))[:10]
        assert hi.min(initial=0) >= -128 and hi.max(initial=0) <= 127 and lo.min(initial=0) >= -128 and lo.max(initial=0) <= 127
        q = 256 * hi + lo
        assert np.abs(q).max(initial=0) <= 32639
        if sigma > 0:
            assert np.abs(q).max() == 32639   # the channel's maximum lands on the limit
            r = w / np.float32(sigma)
            ties += int((r - np.floor(r) == 0.5).sum())
    assert ties >= 3 * 600   # the tie channels really hit exact halves
    for k in (-8, -7, -6):   # the tie channels: every exact half went to an even q
        w, (sigma, hi, lo) = chans[k], got[k]
        r = w / np.float32(sigma)
        half = r - np.floor(r) == 0.5
        assert half.sum() >= 600 and np.all((256 * hi + lo)[half] % 2 == 0)
    for k, v in ((-2, -32639), (-1, 32639)):
        q = 256 * got[k][1] + got[k][2]
        assert q[17] == v and np.count_nonzero(q) == 1
    assert all(s == 0 and not h.any() and not lo.any() for s, h, lo in got[-5:-2])   # all-zero channels: sigma 0, q 0


def test_split_merge_identity(harness):
    out = subprocess.run([harness, "split"], capture_output=True, text=True, check=True).stdout.splitlines()
    assert out == ["checked 65408 bad 0"], out[:5]
    v = np.arange(-32768, 32640)
    hi = (v + 128) >> 8
    lo = v - 256 * hi
    assert hi.min() == -128 and hi.max() == 127 and lo.min() == -128 and lo.max() == 127
    assert np.array_equal(256 * hi + lo, v)


ROW_HARNESS = r"""
#include <stdio.h>
#include "precision.h"
int main() {
    const pe::Precision& p = pe::precision(PE_PREC_S8X2);
    printf("{\"planes\": %d, \"elem\": %d, \"input_elem\": %d, \"act_cpad\": %d, \"kp_input\": %d, \"slot_align\": %d, "
           "\"chunked\": %d, \"range_top\": %d, \"range_limit\": %.9g, \"range_floor\": %.9g, \"range_floor_text\": \"%s\", "
           "\"range_what\": \"%s\", \"net_input_scale\": %.9g, \"needs_calibration\": %d, \"max_k\": %lld, "
           "\"per_channel_epilogue\": %d, \"own_row\": %d, \"known_7\": %d, \"s8x1_max_k\": %lld}\n",
           p.fmt.planes, (int)p.fmt.elem, (int)p.input_elem, p.act_cpad, p.kp_input, p.slot_align, p.chunked, p.range_top,
           p.range_limit, p.range_floor, p.range_floor_text, p.range_what, p.net_input_scale, p.needs_calibration, p.max_k,
           p.per_channel_epilogue, &pe::elem_row(p, pe::ELEM_S8) == &p, (int)pe::known_mode(7), pe::precision(PE_PREC_S8X1).max_k);
    return 0;
}
"""


@pytest.fixture(scope="module")
def row(tmp_path_factory):
    if shutil.which("g++") is None or NVCC is None:
        pytest.skip("g++ or the CUDA headers not found")
    cuda_include = os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(NVCC))), "include")
    d = tmp_path_factory.mktemp("s8x2_row")
    src, exe = d / "row.cpp", d / "row"
    src.write_text(ROW_HARNESS)
    subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-Werror", "-I", CSRC, "-I", cuda_include, str(src), "-o", str(exe)],
                   check=True)
    return json.loads(subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout)


def test_precision_row(row):
    """Two s8 planes with S8X1's pads, exact unchunked sums with per-channel factors, calibration into [2^13, 2^14) against
    32639 with a floor of 2^8, the net input at 2^16 (S8X1's p - 128 in the hi plane), and its own row for every kind."""
    assert (row["planes"], row["elem"], row["input_elem"]) == (2, 3, 3)
    assert (row["act_cpad"], row["kp_input"], row["slot_align"]) == (128, 128, 16)
    assert not row["chunked"] and row["per_channel_epilogue"] and row["needs_calibration"]
    assert (row["range_top"], row["range_limit"], row["range_floor"], row["range_floor_text"], row["range_what"]) == (
        14, 32639.0, 256.0, "2^8", "the s8 plane pairs")
    assert row["net_input_scale"] == 65536.0
    assert row["own_row"] == 1 and row["known_7"] == 0
    assert row["s8x1_max_k"] == 132104


def test_accumulator_bound(row):
    """|acc_c| <= (128 x 128 + 128 x 127) x K: K = 65793 stays inside s32, 65794 does not; acc_h's bound is looser."""
    assert row["max_k"] == MAX_K
    assert (128 * 128 + 128 * 127) * MAX_K <= 2 ** 31 - 1 < (128 * 128 + 128 * 127) * (MAX_K + 1)
    assert 128 * 128 * MAX_K <= 2 ** 31 - 1
    assert 49 * 256 <= MAX_K < 49 * 1408   # the shipped nets' largest K fits; a 7x7 on 1408 padded channels does not


build = tu_build("conv_s8x2.cu")


def test_s8x2_instances_no_spills_and_no_serialised_wgmma(build):
    check_no_spills_and_no_serialised_wgmma(build[0], INSTANCES)


def test_s8x2_instances_keep_one_wgmma_group_in_flight(build):
    kernels = check_one_wgmma_group_in_flight(build[1], INSTANCES)
    widths = set()
    for name, text in kernels.items():
        assert re.search(r"conv_wg_kernelILi\d+ELi2ELi3ELi3E", name), name   # <BN, 2, s8, s8>
        m = re.findall(r"IGMMA\.64x(\d+)x32\.S8\.S8", text)
        assert m and len(m) % 3 == 0, name   # three s8 MMAs per 32-byte K step: hi*hi, hi*lo, lo*hi
        widths |= {int(x) for x in m}
        assert not re.search(r"[HQ]GMMA", text), name    # no fp16 / fp8 MMA
        assert "F2I.S64" in text or "I2F.S64" in text, name   # the 64-bit sum S = 256 acc_h + acc_c converted to fp32
    assert widths == {16, 32, 48, 64, 128}, widths


def kernel_hashes(sass):
    out, cur, buf = {}, None, []
    for line in sass.splitlines():
        m = re.search(r"Function : (\w+)", line)
        if m:
            if cur:
                out[cur] = hashlib.sha256("\n".join(buf).encode()).hexdigest()
            cur, buf = m.group(1), []
            continue
        if cur:
            buf.append(line)
    if cur:
        out[cur] = hashlib.sha256("\n".join(buf).encode()).hexdigest()
    return out


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        g = json.load(f)
    ver = subprocess.run([NVCC or "nvcc", "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if ver != g["nvcc"]:
        pytest.skip("the SASS hashes are of %s, this compiler is %s" % (g["nvcc"], ver))
    return g["units"]


@pytest.mark.parametrize("tu", ["conv_tc.cu", "conv_fp8.cu", "conv_s8.cu", "conv_u8.cu", "conv_mixed.cu", "conv_s8_sparse.cu"])
def test_existing_instances_keep_their_sass(tu, golden, tmp_path):
    """The two-plane s8 code paths of conv_tc_kernel.cuh are compile-time branches: every other instance is unchanged."""
    if NVCC is None:
        pytest.skip("nvcc not found")
    obj = str(tmp_path / (tu + ".o"))
    subprocess.run([NVCC, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC",
                    "--expt-relaxed-constexpr", "-x", "cu", "-c", os.path.join(CSRC, tu), "-o", obj], check=True)
    cuobjdump = os.path.join(os.path.dirname(os.path.realpath(NVCC)), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    got = kernel_hashes(sass)
    assert got == golden[tu], sorted(k for k in set(got) | set(golden[tu]) if got.get(k) != golden[tu].get(k))


def run_bin(args):
    return subprocess.run([BIN] + args, capture_output=True, text=True, timeout=60)


@pytest.fixture(scope="module")
def rtpose_bin():
    if not os.path.exists(BIN):
        pytest.skip("rtpose.bin not built")
    return BIN


def test_help_lists_precision_8(rtpose_bin):
    r = run_bin(["--help"])
    assert r.returncode == 0
    line = [l for l in r.stdout.splitlines() if l.strip().startswith("--precision ")][0]
    assert "8 16-bit integer mode" in line and "6 INT8 mode" in line


@pytest.mark.parametrize("flag", ["--nocalibrate_range", "--calibrate_range=false"])
def test_precision_8_without_calibration_refused(rtpose_bin, flag):
    r = run_bin(["--synthetic", "2", "--model", "COCO", "--precision", "8", flag])
    assert r.returncode == 1 and "--precision 8" in r.stderr and "calibrate" in r.stderr, r.stderr


def test_precision_8_cli_refusals(rtpose_bin):
    r = run_bin(["--synthetic", "2", "--model", "COCO", "--precision", "8", "--u8_activations"])
    assert r.returncode == 1 and "--u8_activations" in r.stderr, r.stderr
    r = run_bin(["--synthetic", "2", "--model", "COCO", "--precision", "8", "--f16_layers", "narrow"])
    assert r.returncode == 1 and "--f16_layers" in r.stderr, r.stderr


@pytest.fixture(scope="module")
def lib():
    path = os.path.join(ROOT, "caffe_rtpose_b200", "libposeengine.so")
    if not os.path.exists(path):
        pytest.skip("libposeengine.so not built")
    from caffe_rtpose_b200 import engine
    return engine.lib()


def test_abi_refusals_and_plan(lib):
    """Host-only ABI: the u8 flag and pe_create_mixed refuse precision 8 before any device is touched (PE_ERR_INVALID, the reason in
    pe_last_error(NULL)); pe_plan_formats describes every activation and layer of the plan as s8x2, f32 for the maps."""
    from caffe_rtpose_b200 import engine
    L = lib
    buf = ctypes.create_string_buffer(1 << 16)
    n = L.pe_plan_formats(engine.COCO_18, None, engine.PREC_S8X2 | engine.PREC_FLAG_U8, None, buf, len(buf))
    assert n == -PE_ERR_INVALID and b"PE_PREC_S8X1 (6) only" in L.pe_last_error(None)
    n = L.pe_plan_formats(engine.COCO_18, None, engine.PREC_S8X2, b"narrow", buf, len(buf))
    assert n == -PE_ERR_INVALID and b"not with precision 8" in L.pe_last_error(None)
    cfg = engine._Config(0, engine.COCO_18, 160, 96, 320, 192, 1, 1.0, 0.3, 1, engine.PREC_S8X2)
    h = ctypes.c_void_p()
    assert L.pe_create_mixed(ctypes.byref(cfg), None, b"conv1_1", ctypes.byref(h)) == PE_ERR_INVALID
    assert b"not 8" in L.pe_last_error(None)
    n = L.pe_plan_formats(engine.COCO_18, None, engine.PREC_S8X2, None, buf, n if n > 0 else len(buf))
    text = buf.value.decode()
    assert n == len(text) and text
    kinds = {line.split()[2] for line in text.splitlines() if line.startswith("act ")}
    assert kinds == {"s8x2"}, kinds
    convs = [line.split() for line in text.splitlines() if line.startswith("conv ")]
    assert {c[2] for c in convs} == {"s8x2"} and {c[3] for c in convs} == {"s8x2", "f32"}



def test_mixed_bases_refuse_s8x2_and_precision_7_stays_unknown(lib):
    """pe_plan_formats refuses S8X2 as a mixed-precision base while it describes its plain plan; precision 7, which no mode
    has, and 9, the first value past S8X2, are unknown precisions."""
    from caffe_rtpose_b200 import engine
    with pytest.raises(engine.PoseEngineError, match="PE_PREC_E4M3X1"):
        engine.plan_formats(engine.COCO_18, engine.PREC_S8X2, "conv1_1")
    engine.plan_formats(engine.COCO_18, engine.PREC_S8X2, "")
    for prec in (7, 9, 7 | engine.PREC_FLAG_U8):
        with pytest.raises(engine.PoseEngineError, match="unknown precision"):
            engine.plan_formats(engine.COCO_18, prec)
