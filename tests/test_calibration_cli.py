"""rtpose.bin's calibration flags (--calibration_dir, --calibration_table, --save_calibration) and the weight-broadcast fallback's
calibration hand-over, on a machine without a GPU: the ThreadSanitizer build of host/rtpose.cpp against tests/stub/stub_engine.cpp
(see test_host_pipeline.py) with the calibration calls of tests/stub/stub_calibration.cpp, which log one line each and report
scripted change counts."""
import os
import subprocess

import pytest

from test_host_pipeline import run, write_bmp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "caffe_rtpose_b200")
STUB_TABLE_FIRST = "pe_calibration 1"


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    if not os.path.exists(os.path.join(PKG, "libposeengine.so")):
        subprocess.check_call(["make", "-C", PKG, "-j8"])
    out = str(tmp_path_factory.mktemp("calibcli") / "rtpose_tsan")
    r = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=thread", "-Wall", "-I", os.path.join(ROOT, "include"),
                        os.path.join(PKG, "host", "rtpose.cpp"), os.path.join(ROOT, "tests", "stub", "stub_calibration.cpp"), "-o", out,
                        "-L", PKG, "-lposeengine", "-Wl,-rpath," + PKG, "-pthread"], capture_output=True, text=True, timeout=300)
    if r.returncode != 0 and "tsan" in r.stderr.lower():
        pytest.skip("this g++ has no ThreadSanitizer runtime")
    assert r.returncode == 0, r.stderr[-3000:]
    return out


@pytest.fixture()
def dirs(tmp_path):
    """a 3-frame --image_dir at the display size and a calibration directory of 5 images, two of them of other sizes"""
    imgs, cal = tmp_path / "images", tmp_path / "cal"
    imgs.mkdir()
    cal.mkdir()
    for i in range(3):
        write_bmp(str(imgs / ("im%02d.bmp" % i)), 40, 24, 100 + i)
    for i, (w, h) in enumerate([(40, 24), (40, 24), (64, 48), (64, 48), (40, 24)]):
        write_bmp(str(cal / ("c%02d.bmp" % i)), w, h, 200 + i)
    return imgs, cal


def base_args(imgs, tmp_path, precision=5):
    return ["--image_dir", str(imgs), "--resolution", "40x24", "--net_resolution", "48x32", "--write_json", str(tmp_path / "json"),
            "--no_frame_drops", "--batch", "2", "--engines_per_gpu", "1", "--precision", str(precision)]


def log_lines(path):
    return open(path).read().splitlines() if os.path.exists(path) else []


def test_calibration_dir_runs_passes_until_nothing_changes(exe, tmp_path, dirs):
    imgs, cal = dirs
    log, table = tmp_path / "stub.log", tmp_path / "t.txt"
    r = run(exe, base_args(imgs, tmp_path) + ["--calibration_dir", str(cal), "--save_calibration", str(table)],
            env={"STUB_LOG": str(log), "STUB_CALIB_CHANGED": "4,2,0,7"})
    assert r.returncode == 0, r.stderr[-3000:]
    lines = log_lines(log)
    # the synthetic-frame pe_calibrate comes first, then three passes: the third reports 0 changes and ends the calibration
    first_begin = next(i for i, l in enumerate(lines) if l.startswith("calibrate_begin"))
    assert any(l.startswith("calibrate engine=0") for l in lines[:first_begin])
    passes, cur = [], None
    for l in lines[first_begin:]:
        if l.startswith("calibrate_begin"):
            cur = []
        elif l.startswith("calibrate_end"):
            passes.append((cur, l))
            cur = None
        elif cur is not None and l.startswith("forward"):
            cur.append(l)
    assert [p[1] for p in passes] == ["calibrate_end engine=0 changed=4", "calibrate_end engine=0 changed=2",
                                                   "calibrate_end engine=0 changed=0"]
    for fwd, _ in passes:   # consecutive images of one size in batches of --batch; other sizes through the camera route
        assert [(f.split()[3], f.split()[4], f.split()[5]) for f in fwd] == [("n=2", "display", "size=40x24"), ("n=2", "camera", "size=64x48"),
                                                                             ("n=1", "display", "size=40x24")]
    for k, n in ((1, 4), (2, 2), (3, 0)):
        assert "calibration pass %d over 5 images: %d layers changed" % (k, n) in r.stderr
    # --save_calibration writes the library's text, after the passes; the run then serves its frames
    assert open(table).read().startswith(STUB_TABLE_FIRST + "\nprecision 5\n")
    assert len(os.listdir(tmp_path / "json")) == 3


def test_calibration_dir_gives_up_after_one_pass_per_layer(exe, tmp_path, dirs):
    imgs, cal = dirs
    log = tmp_path / "stub.log"
    r = run(exe, base_args(imgs, tmp_path) + ["--calibration_dir", str(cal)], env={"STUB_LOG": str(log), "STUB_CALIB_CHANGED": "1,1,1,1,1,1,1,1"})
    assert r.returncode == 1
    assert "the scales still moved after 6 passes" in r.stderr   # the stub's table has 6 ranged layers
    assert sum(l.startswith("calibrate_end") for l in log_lines(log)) == 6


def test_calibration_table_replaces_pe_calibrate(exe, tmp_path, dirs):
    imgs, _ = dirs
    log, table = tmp_path / "stub.log", tmp_path / "t.txt"
    table.write_text("pe_calibration 1\nprecision 6\nweights 0123456789abcdef\nlayer conv0 s8 -3\n")
    r = run(exe, base_args(imgs, tmp_path, precision=6) + ["--calibration_table", str(table)], env={"STUB_LOG": str(log)})
    assert r.returncode == 0, r.stderr[-3000:]
    lines = log_lines(log)
    sets = [l for l in lines if l.startswith("calibration_set")]
    assert sets == ["calibration_set engine=0 bytes=%d first=pe_calibration 1" % len(table.read_text())]
    assert not any(l.startswith("calibrate") for l in lines)
    assert lines.index(sets[0]) < next(i for i, l in enumerate(lines) if l.startswith("forward"))
    # a table the library refuses ends start-up with its message, before any frame
    bad = tmp_path / "bad.txt"
    bad.write_text("garbage\n")
    log2 = tmp_path / "stub2.log"
    r = run(exe, base_args(imgs, tmp_path, precision=6) + ["--calibration_table", str(bad)], env={"STUB_LOG": str(log2)})
    assert r.returncode == 1 and "not a calibration table" in r.stderr
    assert not any(l.startswith("forward") for l in log_lines(log2))
    r = run(exe, base_args(imgs, tmp_path, precision=6) + ["--calibration_table", str(tmp_path / "missing.txt")], env={"STUB_LOG": str(log2)})
    assert r.returncode == 1 and "cannot read the file" in r.stderr


def test_no_broadcast_fallback_gives_every_gpu_engine0_scales(exe, tmp_path, dirs):
    """Without NCCL every GPU loads the model itself.  The synthetic-frame calibration now runs on every GPU in every mode with
    range scales (it did only in INT8: an FP8 engine on GPU 1 ran at scale 1), and scales from --calibration_dir or
    --calibration_table reach GPU 1 as engine 0's table."""
    imgs, cal = dirs
    table = tmp_path / "t.txt"
    table.write_text("pe_calibration 1\nprecision 5\n")
    for extra, want_cal, want_set in (([], ["calibrate engine=0", "calibrate engine=1"], []),
                                      (["--calibration_dir", str(cal)], ["calibrate engine=0"], ["calibration_set engine=1"]),
                                      (["--calibration_table", str(table)], [], ["calibration_set engine=1"]),
                                      (["--nocalibrate_range"], [], [])):
        log = tmp_path / "stub.log"
        if log.exists():
            log.unlink()
        r = run(exe, base_args(imgs, tmp_path, precision=5) + ["--num_gpu", "2"] + extra, env={"STUB_LOG": str(log), "STUB_NO_NCCL": "1"})
        assert r.returncode == 0, r.stderr[-3000:]
        lines = log_lines(log)
        creates = {l.split()[1]: l.split()[2] for l in lines if l.startswith("create")}
        assert creates == {"engine=0": "device=0", "engine=1": "device=1"}
        assert [l for l in lines if l.startswith("calibrate ")] == want_cal, extra
        sets = [l for l in lines if l.startswith("calibration_set")]
        assert [l.split(" bytes=")[0] for l in sets if "engine=1" in l] == want_set, extra
        assert all("first=" + STUB_TABLE_FIRST in l for l in sets)


@pytest.mark.parametrize("args,msg", [
    (["--calibration_table", "T", "--calibration_dir", "D"], "does not combine with --calibration_dir"),
    (["--calibration_table", "T", "--nocalibrate_range", "--precision", "5"], "does not combine with --nocalibrate_range"),
    (["--calibration_dir", "D", "--precision", "3"], "--precision 2, 4, 5 or 6"),
    (["--save_calibration", "S", "--precision", "0"], "--precision 2, 4, 5 or 6"),
    (["--calibration_dir", "EMPTY"], "holds no .jpg"),
    (["--calibration_dir", "BAD"], "cannot decode"),
    (["--calibration_dir", "NOPE"], "does not exist"),
    (["--calibration_dir", "D", "--calibration_frames", "0"], "--calibration_frames must be at least 1"),
])
def test_refused_flag_combinations_exit_before_any_forward(exe, tmp_path, dirs, args, msg):
    imgs, cal = dirs
    (tmp_path / "empty").mkdir()
    (tmp_path / "bad").mkdir()
    (tmp_path / "bad" / "x.bmp").write_bytes(b"BM" + b"\0" * 20)
    table = tmp_path / "t.txt"
    table.write_text("pe_calibration 1\n")
    subst = {"T": str(table), "D": str(cal), "S": str(tmp_path / "s.txt"), "EMPTY": str(tmp_path / "empty"), "BAD": str(tmp_path / "bad"),
             "NOPE": str(tmp_path / "nope")}
    log = tmp_path / "stub.log"
    r = run(exe, base_args(imgs, tmp_path, precision=6) + [subst.get(a, a) for a in args], env={"STUB_LOG": str(log)})
    assert r.returncode == 1, r.stderr[-2000:]
    assert msg in r.stderr, r.stderr[-2000:]
    assert not any(l.startswith(("forward", "create")) for l in log_lines(log))
