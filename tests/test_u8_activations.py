"""u8 activations in the INT8 mode (PE_PREC_S8X1 | PE_PREC_FLAG_U8) without a GPU.

* The plan (pe_plan_formats) against a Python restatement of the rule of poseengine.h, on COCO, MPI, the 2-stage MPI prototxt and
  every generated graph of tests/test_conv_shapes.py, plain, with `narrow` and with the 7x7 layers in fp16: an activation is u8
  exactly when every conv layer that writes its buffer (a pool writes its input's buffer) is followed by ReLU, it is not the net
  input, and every conv layer that reads the buffer computes in s8 in the plan without the flag; a conv layer computes u8 exactly
  when it reads u8.  Apart from the u8 kinds the flagged plan is the plain one (same pitches, buffers and layers), and the plain
  plan holds no u8.
* The flag on any other mode is refused with the reason.
* The u8 facts of precision.h, compiled on their own: calibration into [64, 128), range limit 255, floor 8, and the K bound 66311,
  the largest K with 255 x 127 x K inside s32.
* conv_u8.cu, built with -Xptxas -v: the checks of test_conv_build.py (no spills, no serialised wgmma, one wgmma group in flight)
  for every instance, and the u8 x s8 integer MMA and the saturating u8 conversion in the SASS.
* rtpose.bin: --help lists --u8_activations; it is refused with another precision and without range calibration.
"""
import os
import re
import shutil
import subprocess

import pytest

from caffe_rtpose_b200 import engine
from test_conv_build import check_no_spills_and_no_serialised_wgmma, check_one_wgmma_group_in_flight, tu_build
from test_conv_shapes import CASES, write_prototxt
from test_gpu_conv_layers import netspec
from test_prototxt import spec_prototxt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "caffe_rtpose_b200", "csrc")
BIN = os.path.join(ROOT, "caffe_rtpose_b200", "rtpose.bin")
S8 = engine.PREC_S8X1
# the 7x7 group of the shipped nets: the 7x7 layers, closed under the shared-buffer rule (the stage-input buffers' readers)
SEVEN = ["Mconv%d_stage%d_L%d" % (i, s, b) for s in range(2, 7) for i in range(1, 6) for b in (1, 2)] + ["conv5_1_CPM_L1", "conv5_1_CPM_L2"]
# instances of conv_u8.cu: <BN, 1, in, out> at BN = 16, 32, 48, 64, 128 for (u8, u8), (u8, s8), (s8, u8), (u8, f16), (f16, u8)
INSTANCES = 25


def nets(tmp_path):
    """(label, model, prototxt path or None, netspec) of every graph the rule is checked on."""
    out = [("coco", engine.COCO_18, None, netspec(engine.COCO_18)), ("mpi", engine.MPI_15, None, netspec(engine.MPI_15))]
    spec, path = spec_prototxt("mpi_2", tmp_path)
    out.append(("mpi_2", None, path, spec))
    for name in CASES:
        spec, path = write_prototxt(name, tmp_path)
        out.append((name, None, path, spec))
    return out


def expected(spec, plain):
    """The rule over a netspec: ({blob: stored kind} of the u8 buffers' blobs, {conv: compute kind}) given the plain plan."""
    layers = spec["layers"]
    up = {}

    def root(b):
        while up.get(b, b) != b:
            b = up[b]
        return b

    def unite(a, b):
        ra, rb = root(a), root(b)
        if ra != rb:
            up[ra] = rb

    final = [l for l in layers if l["type"] == "ImResize"][0]["bottom"][0]
    concats = [l for l in layers if l["type"] == "Concat" and l["top"][0] != final]
    for l in layers:
        if l["type"] == "Pooling":
            unite(l["bottom"][0], l["top"][0])
    for l in concats:
        for b in l["bottom"]:
            unite(b, l["top"][0])
        unite(l["top"][0], concats[0]["top"][0])
    relu = {l["bottom"][0] for l in layers if l["type"] == "ReLU"}
    convs = [l for l in layers if l["type"] == "Convolution"]
    nonneg = {root(spec["input"]): False}
    for c in convs:
        g = root(c["top"][0])
        nonneg[g] = nonneg.get(g, True) and c["top"][0] in relu
    readers_s8 = {}
    for c in convs:
        g = root(c["bottom"][0])
        readers_s8[g] = readers_s8.get(g, True) and plain["convs"][c["name"]][0] == "s8"
    u8 = {g for g, ok in nonneg.items() if ok and readers_s8.get(g, True)}
    blobs = [l["top"][0] for l in layers if l["type"] in ("Convolution", "Pooling")] + [spec["input"]]
    kinds = {b: "u8" for b in blobs if root(b) in u8}
    compute = {c["name"]: "u8" if root(c["bottom"][0]) in u8 else plain["convs"][c["name"]][0] for c in convs}
    return kinds, compute


@pytest.mark.parametrize("f16", [None, "narrow", "seven"])
def test_plan_follows_the_rule(f16, tmp_path):
    checked = 0
    for label, model, path, spec in nets(tmp_path):
        conv_names = {l["name"] for l in spec["layers"] if l["type"] == "Convolution"}
        if f16 == "seven" and label not in ("coco", "mpi", "mpi_2"):
            continue   # the generated graphs do not have the shipped layer names
        layers = None if f16 is None else "narrow" if f16 == "narrow" else [n for n in SEVEN if n in conv_names]
        plain = engine.plan_formats(model, S8, layers, prototxt=path)
        flagged = engine.plan_formats(model, S8, layers, prototxt=path, u8_activations=True)
        kinds, compute = expected(spec, plain)
        for i, (kind, pitch, blob) in enumerate(flagged["acts"]):
            want = kinds.get(blob, plain["acts"][i][0]) if blob else plain["acts"][i][0]
            assert kind == want, (label, f16, i, blob, kind, want)
            assert (kind if kind != "u8" else "s8", pitch, blob) == plain["acts"][i], (label, i)
        assert len(flagged["acts"]) == len(plain["acts"])
        assert flagged["convs"].keys() == plain["convs"].keys()
        for name, (comp, store, ia, oa) in flagged["convs"].items():
            assert comp == compute[name], (label, f16, name, comp, compute[name])
            assert store == (flagged["acts"][oa][0] if oa >= 0 else "f32"), (label, name)
            p = plain["convs"][name]
            assert (comp.replace("u8", "s8"), store.replace("u8", "s8"), ia, oa) == p, (label, name)
        assert not any(a[0] == "u8" for a in plain["acts"])
        checked += 1
        if label in ("coco", "mpi") and f16 is None:
            # the shipped nets: the net input, the Concat buffers and conv4_4_CPM's output stay s8; the rest is u8
            s8_acts = [a for a in flagged["acts"] if a[0] == "s8"]
            assert len(s8_acts) == 3 and s8_acts[0][2] is None, s8_acts
            stores_s8 = {n for n, c in flagged["convs"].items() if c[1] == "s8"}
            assert "conv4_4_CPM" in stores_s8 and all(n.startswith(("conv4_4", "conv5_5", "Mconv7")) for n in stores_s8), stores_s8
            reads_s8 = {n for n, c in flagged["convs"].items() if c[0] == "s8"}
            assert "conv1_1" in reads_s8 and all(n == "conv1_1" or n.startswith(("conv5_1", "Mconv1")) for n in reads_s8), reads_s8
    assert checked >= 3


def test_flag_on_other_modes_refused():
    for prec in (engine.PREC_FP32_SIMT, engine.PREC_BF16X1, engine.PREC_F16X2, engine.PREC_F16X1, engine.PREC_E4M3X1):
        with pytest.raises(engine.PoseEngineError, match="PE_PREC_FLAG_U8.*PE_PREC_S8X1 .6. only, not to precision %d" % prec):
            engine.plan_formats(engine.COCO_18, prec, u8_activations=True)
    with pytest.raises(engine.PoseEngineError, match="PE_PREC_FLAG_U8.*not to precision 5"):
        engine.plan_formats(engine.COCO_18, engine.PREC_E4M3X1, "narrow", u8_activations=True)
    with pytest.raises(engine.PoseEngineError, match="unknown precision"):
        engine.plan_formats(engine.COCO_18, S8 | 0x200)


HARNESS = r"""
#include <stdio.h>
#include "precision.h"
int main() {
    const pe::Precision& s8 = pe::precision(PE_PREC_S8X1);
    const pe::Precision& u8 = pe::elem_row(s8, pe::ELEM_U8);
    printf("%d %d %g %g %lld %d %d %d %d %d\n", u8.fmt.elem, u8.range_top, u8.range_limit, u8.range_floor, u8.max_k,
           u8.per_channel_epilogue, u8.act_cpad, u8.slot_align, pe::elem_size(pe::ELEM_U8), &pe::elem_row(s8, pe::ELEM_S8) == &s8);
    return 0;
}
"""


def test_u8_facts(tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("g++ not found")
    src, exe = tmp_path / "h.cpp", tmp_path / "h"
    src.write_text(HARNESS)
    inc = ["-I", CSRC, "-I", "/usr/local/cuda/include"]
    subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-Werror"] + inc + [str(src), "-o", str(exe)], check=True)
    f = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    elem, top, limit, floor, max_k, per_channel, cpad, slot, size, s8_row = f
    assert int(elem) == 4 and int(size) == 1 and int(per_channel) == 1 and int(s8_row) == 1
    assert 2 ** (int(top) - 1) == 64 and 2 ** int(top) == 128            # stored maxima in [64, 128)
    assert float(limit) == 255 and float(floor) == 8
    assert (int(cpad), int(slot)) == (128, 16)                            # S8X1's layout
    k = int(max_k)
    assert k == 66311 and 255 * 127 * k <= 2 ** 31 - 1 < 255 * 127 * (k + 1)
    assert 12544 <= k                                                      # the shipped nets' largest K: 49 x 256


build = tu_build("conv_u8.cu")


def test_u8_instances_no_spills_and_no_serialised_wgmma(build):
    check_no_spills_and_no_serialised_wgmma(build[0], INSTANCES)


def test_u8_instances_keep_one_wgmma_group_in_flight(build):
    kernels = check_one_wgmma_group_in_flight(build[1], INSTANCES)
    widths, forms = set(), set()
    for name, text in kernels.items():
        i8 = re.findall(r"IGMMA\.64x(\d+)x32\.([SU]8)\.S8", text)
        h = re.findall(r"HGMMA\.64x(\d+)x16\.F32", text)
        assert i8 or h, name
        assert not re.search(r"QGMMA", text), name        # no fp8 MMA
        for n, a in i8:
            widths.add(int(n))
            forms.add(a)
        if "U8" in {a for _, a in i8}:
            assert "IGMMA" in text and not h, name        # a u8 reader runs the u8 x s8 integer MMA alone
        if "F2IP.U8.F32" in text:
            forms.add("store_u8")                          # the epilogue's cvt.rni.sat.u8.f32 (a pair per instruction)
    assert widths == {16, 32, 48, 64, 128}, widths
    assert forms == {"U8", "S8", "store_u8"}, forms


def run_bin(args):
    return subprocess.run([BIN] + args, capture_output=True, text=True, timeout=60)


@pytest.fixture(scope="module")
def rtpose_bin():
    if not os.path.exists(BIN):
        pytest.skip("rtpose.bin not built")
    return BIN


def test_help_lists_u8_activations(rtpose_bin):
    r = run_bin(["--help"])
    assert r.returncode == 0
    line = [l for l in r.stdout.splitlines() if l.strip().startswith("--u8_activations ")][0]
    assert "--precision 6" in line and 'default: "false"' in line


@pytest.mark.parametrize("args", [["--precision", "5"], ["--precision", "4"], ["--precision", "6", "--nocalibrate_range"],
                                  ["--precision", "6", "--calibrate_range=false"]])
def test_u8_activations_refused(rtpose_bin, args):
    r = run_bin(["--synthetic", "2", "--model", "COCO", "--u8_activations"] + args)
    assert r.returncode == 1 and "--u8_activations" in r.stderr and "--precision 6 with --calibrate_range" in r.stderr, r.stderr
