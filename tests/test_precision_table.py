"""The precision table (csrc/precision.h), compiled on its own with g++, against what poseengine.h and DESIGN.md promise for
every PE_PREC_* mode: storage format, channel pads, net input pitch, Concat slot alignment, which modes chunk their hi*hi
accumulation, the weight and calibration scales, the range limits and floors pe_range_status applies, the net input's scale,
which modes need pe_calibrate, and the s8 accumulator bound.
"""
import json
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "caffe_rtpose_b200", "csrc")
NVCC = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)

HARNESS = r"""
#include <stdio.h>
#include "precision.h"
int main() {   // one JSON object per row, keyed by the PE_PREC_* name
    static const struct { int id; const char* name; } modes[] = {
        {PE_PREC_FP32_SIMT, "FP32_SIMT"}, {PE_PREC_BF16X1, "BF16X1"}, {PE_PREC_F16X2, "F16X2"}, {PE_PREC_BF16X3, "BF16X3"},
        {PE_PREC_F16X1, "F16X1"}, {PE_PREC_E4M3X1, "E4M3X1"}, {PE_PREC_S8X1, "S8X1"}};
    static const char* elems[] = {"bf16", "f16", "e4m3", "s8"};
    static_assert(sizeof modes / sizeof modes[0] == pe::NUM_PRECISIONS, "one row per mode");
    for (const auto& m : modes) {
        const pe::Precision& p = pe::precision(m.id);
        printf("{\"name\": \"%s\", \"planes\": %d, \"elem\": \"%s\", \"elem_bytes\": %d, \"input_elem\": \"%s\", \"act_cpad\": %d, "
               "\"kp_input\": %d, \"slot_align\": %d, \"chunked\": %d, \"weight_top\": %d, \"input_weight_top\": %d, "
               "\"range_top\": %d, \"ranged\": %d, \"range_limit\": %.9g, \"range_floor\": %.9g, \"range_floor_text\": \"%s\", "
               "\"range_what\": \"%s\", \"net_input_scale\": %.9g, \"needs_calibration\": %d, \"max_k\": %lld, "
               "\"per_channel_epilogue\": %d}\n",
               m.name, p.fmt.planes, elems[p.fmt.elem], p.fmt.elem_bytes(), elems[p.input_elem], p.act_cpad, p.kp_input,
               p.slot_align, p.chunked, pe::weight_top(p.fmt.elem), pe::weight_top(p.input_elem), p.range_top, p.ranged(),
               p.range_limit, p.range_floor, p.range_floor_text ? p.range_floor_text : "", p.range_what ? p.range_what : "",
               p.net_input_scale, p.needs_calibration, p.max_k, p.per_channel_epilogue);
    }
    return 0;
}
"""


def read_table(workdir):
    """{mode name: {field: value}} of every row of precision.h."""
    if shutil.which("g++") is None or NVCC is None:
        pytest.skip("g++ or the CUDA headers not found")
    cuda_include = os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(NVCC))), "include")
    src, exe = os.path.join(workdir, "table.cpp"), os.path.join(workdir, "table")
    with open(src, "w") as f:
        f.write(HARNESS)
    subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-Werror", "-I", CSRC, "-I", cuda_include, src, "-o", exe], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout
    return {r["name"]: r for r in map(json.loads, out.splitlines())}


@pytest.fixture(scope="module")
def table(tmp_path_factory):
    return read_table(str(tmp_path_factory.mktemp("precision")))


SIXTEEN_BIT = ["BF16X1", "F16X2", "BF16X3", "F16X1"]
ONE_BYTE = ["E4M3X1", "S8X1"]


def test_storage_formats(table):
    fmt = {name: (r["planes"], r["elem"], r["elem_bytes"], r["input_elem"]) for name, r in table.items()}
    assert fmt == {"FP32_SIMT": (0, "bf16", 4, "bf16"), "BF16X1": (1, "bf16", 2, "bf16"), "F16X2": (2, "f16", 2, "f16"),
                   "BF16X3": (3, "bf16", 2, "bf16"), "F16X1": (1, "f16", 2, "f16"),
                   "E4M3X1": (1, "e4m3", 1, "f16"),   # the net input stays fp16: p/256 - 0.5 is exact there, not in e4m3
                   "S8X1": (1, "s8", 1, "s8")}


def test_channel_pads_and_slots(table):
    """Activations pad to one 128-byte K block (16 fp32 channels for the SIMT kernel); Concat slots to 16 bytes."""
    assert (table["FP32_SIMT"]["act_cpad"], table["FP32_SIMT"]["kp_input"], table["FP32_SIMT"]["slot_align"]) == (16, 32, 8)
    for name in SIXTEEN_BIT:
        assert (table[name]["act_cpad"], table[name]["kp_input"], table[name]["slot_align"]) == (64, 64, 8), name
    assert (table["E4M3X1"]["act_cpad"], table["E4M3X1"]["kp_input"], table["E4M3X1"]["slot_align"]) == (128, 64, 16)
    assert (table["S8X1"]["act_cpad"], table["S8X1"]["kp_input"], table["S8X1"]["slot_align"]) == (128, 128, 16)
    for name in SIXTEEN_BIT + ONE_BYTE:
        assert table[name]["act_cpad"] * table[name]["elem_bytes"] == 128, name


def test_accumulation(table):
    """hi*hi chunks in F16X2, BF16X3, F16X1 and E4M3X1; BF16X1 and S8X1 (exact integer sums) run one chain over K."""
    assert {name for name, r in table.items() if r["chunked"]} == {"F16X2", "BF16X3", "F16X1", "E4M3X1"}
    assert {name for name, r in table.items() if r["per_channel_epilogue"]} == {"S8X1"}
    assert {name: r["max_k"] for name, r in table.items() if r["max_k"]} == {"S8X1": 132104}


def test_weight_scales(table):
    """fp16 weights are scaled to max|w| in [2^13, 2^14), e4m3 to [128, 256); E4M3X1 packs conv1_1's fp16 weights as fp16."""
    assert {name: (r["weight_top"], r["input_weight_top"]) for name, r in table.items()} == {
        "FP32_SIMT": (0, 0), "BF16X1": (0, 0), "F16X2": (14, 14), "BF16X3": (0, 0), "F16X1": (14, 14), "E4M3X1": (8, 14),
        "S8X1": (0, 0)}


def test_range_scales(table):
    """pe_calibrate targets [32, 64) (fp16, s8) and [64, 128) (e4m3); pe_range_status's limits, floors and their texts."""
    ranged = {name: (r["range_top"], r["range_limit"], r["range_floor"], r["range_floor_text"], r["range_what"])
              for name, r in table.items() if r["ranged"]}
    fp16 = (6, 65504.0, 2.0 ** -10, "2^-10", "the fp16 planes")
    assert ranged == {"F16X2": fp16, "F16X1": fp16, "E4M3X1": (7, 448.0, 2.0 ** -2, "2^-2", "the e4m3 planes"),
                      "S8X1": (6, 127.0, 4.0, "4", "the s8 planes")}
    for name in set(table) - set(ranged):
        assert table[name]["range_top"] == 0, name


def test_net_input_and_calibration(table):
    """S8X1 stores the net input as p - 128 = (p/256 - 0.5) x 2^8 and refuses to forward before pe_calibrate."""
    assert {name: r["net_input_scale"] for name, r in table.items() if r["net_input_scale"] != 1} == {"S8X1": 256.0}
    assert {name for name, r in table.items() if r["needs_calibration"]} == {"S8X1"}
