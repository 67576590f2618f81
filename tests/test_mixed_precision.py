"""Mixed precision (pe_create_mixed, DESIGN.md section 3) without a GPU: the format-boundary instances of conv_mixed.cu, the
element kinds and channel pitches pe_plan_formats reports for the built-in nets, a 2-stage prototxt and generated graphs, and the
rtpose.bin flag.
"""
import os
import re
import subprocess

import pytest

from caffe_rtpose_b200 import engine
from test_conv_build import tu_build, check_no_spills_and_no_serialised_wgmma, check_one_wgmma_group_in_flight
from test_conv_shapes import write_prototxt
from test_prototxt import spec_prototxt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "caffe_rtpose_b200", "rtpose.bin")
INSTANCES = 15   # <BN, 1, ELEM, OUT> at BN 16-128 for (e4m3, f16), (f16, s8), (s8, f16)
ELEM = {1: "f16", 2: "e4m3", 3: "s8"}
MMA = {"f16": r"HGMMA\.64x(\d+)x16\.F32\b", "e4m3": r"QGMMA\.64x(\d+)x32\.F32\.E4M3\.E4M3", "s8": r"IGMMA\.64x(\d+)x32\.S8\.S8"}
NARROW = {"conv1_1", "conv1_2", "conv2_1"}

build = tu_build("conv_mixed.cu")


def test_mixed_instances_no_spills_and_no_serialised_wgmma(build):
    check_no_spills_and_no_serialised_wgmma(build[0], INSTANCES)


def test_mixed_instances_keep_one_wgmma_group_in_flight(build):
    """Each pair runs the MMA of its input kind, and an s8 output is stored with cvt.rni.sat.s8.f32."""
    kernels = check_one_wgmma_group_in_flight(build[1], INSTANCES)
    pairs = {}
    for name, text in kernels.items():
        bn, planes, elem, out = map(int, re.search(r"conv_wg_kernelILi(\d+)ELi(\d+)ELi(\d+)ELi(\d+)E", name).groups())
        assert planes == 1, name
        pairs.setdefault((ELEM[elem], ELEM[out]), set()).add(bn)
        for kind, pattern in MMA.items():
            widths = {int(w) for w in re.findall(pattern, text)}
            assert widths == ({bn} if kind == ELEM[elem] else set()), (name, kind, widths)
        assert ("F2I.S8" in text) == (ELEM[out] == "s8"), name
    assert pairs == {p: {16, 32, 48, 64, 128} for p in [("e4m3", "f16"), ("f16", "s8"), ("s8", "f16")]}, pairs


def formats(precision, f16_layers=None, model=None, prototxt=None):
    return engine.plan_formats(model, precision, f16_layers, prototxt)


def nets(tmp_path):
    _, path = spec_prototxt("mpi_2", tmp_path)
    return [dict(model=engine.COCO_18), dict(model=engine.MPI_15), dict(prototxt=path)]


def fp16_convs(f):
    return {name for name, c in f["convs"].items() if c[0] == "f16"}


def in_pitch(f, name):
    return f["acts"][f["convs"][name][2]][:2]


@pytest.mark.parametrize("base,kind", [(engine.PREC_E4M3X1, "e4m3"), (engine.PREC_S8X1, "s8")])
def test_narrow_runs_the_first_three_layers_in_fp16(base, kind, tmp_path):
    for net in nets(tmp_path):
        f = formats(base, "narrow", **net)
        assert fp16_convs(f) == NARROW, net
        assert in_pitch(f, "conv1_1") == ("f16", 64) and in_pitch(f, "conv1_2") == ("f16", 64) and in_pitch(f, "conv2_1") == ("f16", 64)
        assert f["convs"]["conv2_1"][1] == kind   # the boundary: conv2_1 computes in fp16 and stores the base kind
        for name, (compute, out, in_act, out_act) in f["convs"].items():
            if name not in NARROW:
                assert compute == kind and f["acts"][in_act][0] == kind and f["acts"][in_act][1] % 128 == 0, (net, name)
        assert in_pitch(f, "conv2_2") == (kind, 128)


def test_every_layer_listed_is_the_f16_plan(tmp_path):
    """Pitches, slots and kinds equal F16X1's plain plan; an empty list equals the base mode's plain plan."""
    for net in nets(tmp_path):
        plain16 = formats(engine.PREC_F16X1, **net)
        for base in (engine.PREC_E4M3X1, engine.PREC_S8X1):
            assert formats(base, list(plain16["convs"]), **net) == plain16, (net, base)
            assert formats(base, "", **net) == formats(base, **net) == formats(base, [], **net)
        # and the describe call's plain plans: f16 kinds at 64, e4m3 at 128 with an fp16 input, s8 at 128 with an s8 input
        assert {a[:2] for a in plain16["acts"]} <= {("f16", c) for c in range(64, 4096, 64)}
        e4m3 = formats(engine.PREC_E4M3X1, **net)
        assert e4m3["acts"][e4m3["convs"]["conv1_1"][2]][:2] == ("f16", 64) and e4m3["convs"]["conv1_1"][:2] == ("f16", "e4m3")
        s8 = formats(engine.PREC_S8X1, **net)
        assert s8["acts"][s8["convs"]["conv1_1"][2]][:2] == ("s8", 128)


@pytest.mark.parametrize("base", [engine.PREC_E4M3X1, engine.PREC_S8X1])
def test_a_split_shared_buffer_is_refused(base, tmp_path):
    """Mconv1_stage2_L1 reads the stage-input buffer with every stage's first layers and the readers of conv4_4_CPM."""
    for net in nets(tmp_path):
        with pytest.raises(engine.PoseEngineError) as ex:
            formats(base, "Mconv1_stage2_L1", **net)
        msg = str(ex.value)
        assert "Mconv1_stage2_L2" in msg and "conv5_1_CPM_L1" in msg and "conv5_1_CPM_L2" in msg, msg
        with pytest.raises(engine.PoseEngineError, match="conv5_1_CPM_L2"):
            formats(base, "conv5_1_CPM_L1", **net)   # the two branches' first layers read one buffer
    group = ["conv5_1_CPM_L1", "conv5_1_CPM_L2"] + ["Mconv1_stage%d_L%d" % (s, b) for s in range(2, 7) for b in (1, 2)]
    f = formats(base, group, model=engine.COCO_18)
    assert fp16_convs(f) == set(group) | ({"conv1_1"} if base == engine.PREC_E4M3X1 else set())   # E4M3X1: an fp16 conv1_1
    assert f["acts"].count(("f16", 192, None)) == 2   # the two stage-input buffers: 128 + 40 + 24 channels in fp16's slots


def test_unknown_names_and_other_bases_are_refused():
    with pytest.raises(engine.PoseEngineError, match="unknown conv layer conv9_9"):
        formats(engine.PREC_E4M3X1, "conv1_1,conv9_9", model=engine.COCO_18)
    for prec in (engine.PREC_FP32_SIMT, engine.PREC_BF16X1, engine.PREC_F16X2, engine.PREC_BF16X3, engine.PREC_F16X1):
        with pytest.raises(engine.PoseEngineError, match="PE_PREC_E4M3X1"):
            formats(prec, "conv1_1", model=engine.COCO_18)
        formats(prec, "", model=engine.COCO_18)
    with pytest.raises(engine.PoseEngineError, match="unknown precision"):
        formats(7, model=engine.COCO_18)
    # the list's syntax: spaces and empty entries are ignored
    assert fp16_convs(formats(engine.PREC_S8X1, " conv1_1 ,, conv1_2,", model=engine.MPI_15)) == {"conv1_1", "conv1_2"}


@pytest.mark.parametrize("name,narrow_f", [("three_stages", False), ("tiny_32x16", False), ("k1_k3_wide", True), ("k5_k7_vgg", True)])
def test_narrow_leaves_a_partly_narrow_group_alone(name, narrow_f, tmp_path):
    """F has 72 (100) channels.  With more than one stage the stage inputs are 129 channels wide and share F's buffer, so the
    group F's readers belong to is only partly narrow and stays in the base format; a one-stage net's F readers go to fp16."""
    spec, path = write_prototxt(name, tmp_path)
    f = formats(engine.PREC_S8X1, "narrow", prototxt=path)
    text = engine.plan_describe(prototxt=path)
    cin = {fl[1]: int(fl[3]) for fl in (l.split() for l in text.splitlines()) if fl[0] == "conv"}
    first = {n for n in f["convs"] if re.match(r"Mconv1_stage\d+_L\d", n)}
    stage1 = {n for n in first if "_stage1_" in n}
    assert all(cin[n] < 128 for n in stage1)
    assert (stage1 <= fp16_convs(f)) == narrow_f
    assert not (first - stage1) & fp16_convs(f)
    trunk = {n for n in f["convs"] if n.startswith("conv")}
    assert {n for n in trunk if cin[n] < 128} <= fp16_convs(f)
    assert not {n for n in trunk if cin[n] >= 128} & fp16_convs(f)
    for n, (compute, out, in_act, out_act) in f["convs"].items():   # every activation's pitch follows its kind
        kind, pitch = f["acts"][in_act][:2]
        assert kind == compute and pitch % (64 if kind == "f16" else 128) == 0, (n, kind, pitch)


def run_bin(args):
    return subprocess.run([BIN] + args, capture_output=True, text=True, timeout=60)


@pytest.fixture(scope="module")
def rtpose_bin():
    if not os.path.exists(BIN):
        pytest.skip("rtpose.bin not built")
    return BIN


def test_cli_flag(rtpose_bin):
    r = run_bin(["--help"])
    assert r.returncode == 0 and any(l.strip().startswith("--f16_layers ") for l in r.stdout.splitlines())
    r = run_bin(["--synthetic", "2", "--model", "COCO", "--precision", "4", "--f16_layers", "narrow"])
    assert r.returncode == 1 and "--precision 5 or 6" in r.stdout + r.stderr
    r = run_bin(["--synthetic", "2", "--model", "COCO", "--precision", "5", "--f16_layers", "conv1_1,convX"])
    assert r.returncode == 1 and "unknown conv layer convX" in r.stdout + r.stderr
    r = run_bin(["--synthetic", "2", "--model", "MPI", "--precision", "6", "--f16_layers", "Mconv1_stage3_L2"])
    assert r.returncode == 1 and "Mconv1_stage3_L1" in r.stdout + r.stderr
