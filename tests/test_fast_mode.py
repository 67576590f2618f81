"""CPU tests of the fast mode's host side: pe_compare_results (the comparison the audit and tools/fast_mode.py use) on
constructed results, and the rtpose.bin flags --precision 4 and --audit_every."""
import os
import subprocess

import numpy as np
import pytest

from caffe_rtpose_b200 import engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "caffe_rtpose_b200", "rtpose.bin")
P, MP = 18, 4


def result(people, seed=0):
    """(num_people, joints, peaks) as PoseEngine.fetch returns them: peak counts 1 + part % 3, persons with parts 0..9."""
    rng = np.random.default_rng(seed)
    peaks = np.zeros((P, MP + 1, 3), np.float32)
    for p in range(P):
        c = 1 + p % 3
        peaks[p, 0, 0] = c
        peaks[p, 1:1 + c, :2] = rng.uniform(0, 160, (c, 2))
        peaks[p, 1:1 + c, 2] = rng.uniform(0.1, 1, c)
    joints = np.zeros((people, P, 3), np.float32)
    joints[:, :10, :2] = rng.uniform(0, 320, (people, 10, 2))
    joints[:, :10, 2] = 1.0
    return people, joints, peaks


def test_identical_results():
    a = result(3)
    d = engine.compare_results(a, a, 1e-3)
    assert d == {"identical": True, "parts_count_differ": 0, "peaks_moved": 0, "persons_matched": 3, "max_joint_dist": 0.0}


@pytest.mark.parametrize("shift,moved", [(2e-3, True), (5e-4, False)])
def test_peak_moved_by_more_or_less_than_the_tolerance(shift, moved):
    a = result(2)
    pb = a[2].copy()
    pb[4, 1, 0] += shift
    d = engine.compare_results(a, (a[0], a[1], pb), 1e-3)
    assert d["identical"] is (not moved) and d["peaks_moved"] == int(moved) and d["parts_count_differ"] == 0


def test_joint_moved_beyond_tolerance_is_reported_with_its_distance():
    a = result(2)
    jb = a[1].copy()
    jb[1, 3, 0] += 3.0
    jb[1, 3, 1] += 4.0
    d = engine.compare_results(a, (a[0], jb, a[2]), 1e-3)
    assert not d["identical"] and d["persons_matched"] == 2 and d["max_joint_dist"] == pytest.approx(5.0, rel=1e-5)


def test_part_count_differs():
    a = result(1)
    pb = a[2].copy()
    pb[7, 0, 0] += 1
    d = engine.compare_results(a, (a[0], a[1], pb), 1e-3)
    assert not d["identical"] and d["parts_count_differ"] == 1 and d["peaks_moved"] == 0


def test_person_missing():
    a = result(3)
    d = engine.compare_results(a, (2, a[1][:2], a[2]), 1e-3)
    assert not d["identical"] and d["persons_matched"] == 2


def test_persons_in_swapped_order():
    """Person i of a is compared with person i of b: the same persons in another order are not identical.  With the same
    present parts they still match, and the joint distance shows how far apart they are."""
    a = result(2)
    jb = a[1][::-1].copy()
    d = engine.compare_results(a, (a[0], jb, a[2]), 1e-3)
    assert not d["identical"] and d["persons_matched"] == 2 and d["max_joint_dist"] > 1.0
    jb[0, 12, 2] = 0.7                      # person 0 of b gains a part: no longer the same person
    d = engine.compare_results(a, (a[0], jb, a[2]), 1e-3)
    assert not d["identical"] and d["persons_matched"] == 1


def test_no_people():
    a = result(0)
    assert engine.compare_results(a, a, 1e-3)["identical"]
    d = engine.compare_results(a, result(1), 1e-3)
    assert not d["identical"] and d["persons_matched"] == 0


def test_bad_arguments_are_refused():
    a = result(1)
    with pytest.raises(ValueError):
        engine.compare_results(a, (a[0], a[1], a[2][:, :2]), 1e-3)
    with pytest.raises(engine.PoseEngineError):
        engine.compare_results(a, a, -1.0)


def run(args):
    return subprocess.run([BIN] + args, capture_output=True, text=True, timeout=60)


def test_help_lists_precision_4_and_audit_every():
    r = run(["--help"])
    assert r.returncode == 0
    line = [l for l in r.stdout.splitlines() if l.strip().startswith("--precision ")][0]
    assert "4 fast mode" in line
    assert any(l.strip().startswith("--audit_every ") for l in r.stdout.splitlines())


@pytest.mark.parametrize("args,msg", [(["--precision", "2", "--audit_every", "5"], "with --precision 2 there is nothing to compare"),
                                      (["--precision", "4", "--audit_every", "-1"], "--audit_every must be 0")])
def test_audit_every_refused(args, msg):
    r = run(["--synthetic", "2", "--model", "COCO"] + args)
    assert r.returncode == 1 and msg in r.stderr, r.stderr
