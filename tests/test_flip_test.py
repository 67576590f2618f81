"""The flip test's definition on the CPU: the channel map of each model (pe_model_flip_table), what it does to real maps, and the
CPU restatement of the flip average that the GPU parse is checked against (tests/test_gpu_flip_test.py).  No GPU needed."""
import numpy as np
import pytest

from caffe_rtpose_b200 import engine, synth
from oracle import orc

MODELS = [engine.COCO_18, engine.MPI_15]


def _resize_one(maps8_n, net_h, net_w, start_scale, scale_gap, n):
    """The oracle's ImResize of ONE stride-8 copy at scale n, as the term it contributes to the S-scale sum: orc.imresize of that copy
    alone with the start scale that gives scale 0 the crop factor f_n of scale n (x / 1.0f is exact).  Needs 1 - (1 - f_n) == f_n
    in float32, which the scales these tests use satisfy."""
    one, gap32, start32 = np.float32(1), np.float32(scale_gap), np.float32(start_scale)
    f = np.float32(np.float64(n) * np.float64(gap32) + np.float64(one - start32))   # fmaf(n, gap, 1 - start): exact for these scales
    start_n = one - f
    assert one - start_n == f, "scale %d: crop factor %r has no exact start scale" % (n, f)
    return orc.imresize(maps8_n[None], net_h, net_w, float(start_n), float(scale_gap))


def flip_average(model, maps8, net_h, net_w, start_scale, scale_gap):
    """The full-resolution maps of one frame under the flip test, from its 2S stride-8 copies [S scales][S mirrored]: the
    oracle's per-copy ImResize, the mirrored ones read at net_w-1-x with channel perm[c] and sign[c], summed in copy order in
    float32 and divided by 2S, as fullres_at does."""
    perm, sign = engine.flip_table(model)
    two_s = maps8.shape[0]
    S = two_s // 2
    total = np.zeros((maps8.shape[1], net_h, net_w), np.float32)
    for n in range(two_s):
        r = _resize_one(maps8[n], net_h, net_w, start_scale, scale_gap, n % S)
        if n >= S:
            r = (r[perm][:, :, ::-1] * sign[:, None, None]).astype(np.float32)
        total = (total + r).astype(np.float32)
    return (total / np.float32(two_s)).astype(np.float32)


def _numpy_table(model):
    """pe_model_flip_table restated from the descriptor: L/R twins by name, limbs by their parts, PAF x channels negated."""
    L = engine.lib()
    P, NL = L.pe_model_num_parts(model), L.pe_model_num_limbs(model)
    names = [L.pe_model_part_name(model, i).decode() for i in range(P + 1 + 2 * NL)]
    ls, mi = L.pe_model_limb_sequence(model), L.pe_model_map_idx(model)
    limbs = [(ls[2 * k], ls[2 * k + 1]) for k in range(NL)]
    midx = [(mi[2 * k], mi[2 * k + 1]) for k in range(NL)]
    perm = list(range(len(names)))
    sign = [1.0] * len(names)
    for i in range(P + 1):
        n = names[i]
        if n[:1] in ("R", "L") and n[1:2].isupper():
            perm[i] = names.index({"R": "L", "L": "R"}[n[0]] + n[1:])
    for k, (a, b) in enumerate(limbs):
        j = limbs.index((perm[a], perm[b]))
        perm[midx[k][0]], perm[midx[k][1]] = midx[j]
        sign[midx[k][0]] = -1.0
    return np.array(perm, np.int32), np.array(sign, np.float32), names, limbs, midx


@pytest.mark.parametrize("model", MODELS)
def test_flip_table(model):
    perm, sign = engine.flip_table(model)
    want_perm, want_sign, names, limbs, midx = _numpy_table(model)
    P = engine.lib().pe_model_num_parts(model)
    assert len(perm) == len(names) == P + 1 + 2 * len(limbs)
    assert np.array_equal(perm[perm], np.arange(len(perm))), "not an involution"
    for i in range(P + 1):
        a, b = names[i], names[perm[i]]
        if perm[i] == i:
            assert a in ("Nose", "Neck", "Head", "Chest", "Bkg"), a
        else:
            assert {a[0], b[0]} == {"L", "R"} and a[1:] == b[1:], (a, b)
    for k, (a, b) in enumerate(limbs):   # every limb's image is a limb, and its PAF pair is that limb's
        j = limbs.index((perm[a], perm[b]))
        assert (perm[midx[k][0]], perm[midx[k][1]]) == midx[j]
    x_channels = {x for x, _ in midx}
    assert {c for c in range(len(sign)) if sign[c] == -1} == x_channels
    assert set(np.unique(sign)) == {-1.0, 1.0}
    assert np.array_equal(perm, want_perm) and np.array_equal(sign, want_sign)


def test_flip_table_errors():
    L = engine.lib()
    assert L.pe_model_flip_table(7, None, None, 0) == -1   # PE_ERR_INVALID
    n = L.pe_model_flip_table(engine.COCO_18, None, None, 0)
    assert n == 57 and L.pe_model_flip_table(engine.MPI_15, None, None, 0) == 44
    perm = np.full(n, -5, np.int32)
    assert L.pe_model_flip_table(engine.COCO_18, perm.ctypes.data, None, n - 1) == n
    assert (perm == -5).all(), "a short cap must write nothing"


def _mirror_people(model, people, axis):
    """The scene mirrored by x -> axis - x, every part relabelled with its twin."""
    perm, _ = engine.flip_table(model)
    return [{int(perm[p]): (axis - x, y) for p, (x, y) in person.items()} for person in people]


def _peak_set(peaks):
    return sorted((p, round(float(x), 1), round(float(y), 1)) for p in range(peaks.shape[0]) for x, y, _ in peaks[p, 1:1 + int(peaks[p, 0, 0])])


@pytest.mark.parametrize("model", MODELS)
def test_unflipped_mirror_matches_original(model):
    """Maps of the mirrored scene, un-flipped with the table, are the maps of the scene, and the oracle finds the scene's peaks (and,
    for MPI, whose synthetic scenes assemble stably, its persons) in the mirrored scene, mirrored and relabelled by the table.  A wrong
    pair or PAF sign in the table breaks this whatever the implementation."""
    net_w, net_h = 320, 176
    people = synth.make_people(model, 5, net_w, net_h, seed=11, drop_prob=0.0)
    maps = synth.make_maps(model, people, net_w, net_h, noise=0.0, seed=11)
    perm, sign = engine.flip_table(model)
    P = orc.num_parts(model)
    # synth rasterises heat maps at the stride-8 cell centres (symmetric under x -> net_w-1-x) and PAFs at the cell corners
    # (symmetric under x -> net_w-8-x): each is checked on the grid it is symmetric on
    for axis, chans in ((net_w - 1, slice(0, P + 1)), (net_w - 8, slice(P + 1, None))):
        mirrored = synth.make_maps(model, _mirror_people(model, people, axis), net_w, net_h, noise=0.0, seed=11)
        unflipped8 = mirrored[:, perm][..., ::-1] * sign[None, :, None, None]
        np.testing.assert_allclose(unflipped8[:, chans], maps[:, chans], atol=1e-5)
    mirrored = synth.make_maps(model, _mirror_people(model, people, net_w - 1), net_w, net_h, noise=0.0, seed=11)
    full = orc.imresize(maps, net_h, net_w, 1.0, 0.3)
    full_m = orc.imresize(mirrored, net_h, net_w, 1.0, 0.3)
    thr, params = orc.default_params(model)
    peaks, peaks_m = orc.nms(full, P, orc.max_peaks(model), thr), orc.nms(full_m, P, orc.max_peaks(model), thr)
    back = peaks_m[perm[:P]].copy()
    back[:, 1:, 0] = net_w - 1 - back[:, 1:, 0]
    got, want = _peak_set(back), _peak_set(peaks)
    assert len(got) == len(want) >= 5 * 5
    assert all(a[0] == b[0] and abs(a[1] - b[1]) < 0.5 and abs(a[2] - b[2]) < 0.5 for a, b in zip(got, want))
    if model == engine.MPI_15:
        cnt, joints = orc.connect(model, full, peaks, net_w, net_h, params)
        cnt_m, joints_m = orc.connect(model, full_m, peaks_m, net_w, net_h, params)
        assert cnt == cnt_m == 5
        jb = joints_m[:, perm[:P]].copy()
        jb[..., 0] = np.where(jb[..., 2] > 0, net_w - 1 - jb[..., 0], 0)
        key = lambda j: sorted(range(len(j)), key=lambda i: (round(float(j[i][1][0])), round(float(j[i][1][1]))))
        a, b = joints[key(joints)], jb[key(jb)]
        assert np.array_equal(a[..., 2] > 0, b[..., 2] > 0)
        assert np.abs(a[..., :2] - b[..., :2])[a[..., 2] > 0].max() < 0.5


@pytest.mark.parametrize("S", [1, 3])
def test_flip_average_restatement(S):
    """The per-copy decomposition reproduces the oracle's own S-scale average bit for bit, and the flip average of S scales and
    S all-zero mirrors is that average halved, bit for bit (x / 2S == (x / S) / 2 for normal floats)."""
    model, net_w, net_h, start, gap = engine.COCO_18, 160, 96, 1.0, 0.25
    rng = np.random.default_rng(S)
    maps = rng.normal(0, 1, (2 * S, orc.num_maps(model), net_h // 8, net_w // 8)).astype(np.float32)
    want = orc.imresize(maps[:S], net_h, net_w, start, gap)
    total = np.zeros_like(want)
    for n in range(S):
        total = (total + _resize_one(maps[n], net_h, net_w, start, gap, n)).astype(np.float32)
    assert np.array_equal((total / np.float32(S)).astype(np.float32), want)
    zero_mirrors = maps.copy()
    zero_mirrors[S:] = 0
    assert np.array_equal(flip_average(model, zero_mirrors, net_h, net_w, start, gap), (want / np.float32(2)).astype(np.float32))
