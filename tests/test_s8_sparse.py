"""2:4-sparse s8 layers without a GPU: the pruning of pe_prune_2to4, the compressed layout of csrc/s8_sparse.h, and what ptxas
makes of csrc/conv_s8_sparse.cu.

* Pruning (engine.prune_2to4) on the built-in COCO and MPI graphs and the generated graphs of test_conv_shapes.py (Concat slots
  of 7, 72 and 129 channels among them) leaves at most two non-zeros in every aligned group of four of the packed K order, and
  keeps exactly the numpy top-2 by magnitude, the lower index on a tie.  The order is restated here from plan.cpp's layout: a
  Concat input puts the blobs that other layers also read first, then the others, each slot 16-channel aligned; every input is
  padded to 128 channels; K = tap, then engine channel.
* Compression: s8_sparse.h, compiled on its own with g++, compresses random 2:4 planes in which the groups cycle through every
  non-zero pattern (six pairs, four singles, empty); a numpy restatement of the metadata expands values and metadata back to
  the dense plane exactly, and every index pair is ordered and distinct.
* The sparse instances build for sm_90a with no spills and no serialised wgmma, contain IGMMA.SP and keep one wgmma group in
  flight.
"""
import shutil
import subprocess

import numpy as np
import pytest

from caffe_rtpose_b200 import engine, synth
from test_conv_build import CSRC, check_no_spills_and_no_serialised_wgmma, check_one_wgmma_group_in_flight, tu_build
from test_conv_shapes import CASES, spec_weights, write_prototxt
from test_gpu_conv_layers import netspec

def round_up(v, m):
    return (v + m - 1) // m * m


def k_groups(spec):
    """{conv name: [(tap, [Caffe input channel or -1] * 4)]}: the aligned groups of four of the S8X1 packed K order."""
    layers = spec["layers"]
    channels, consumers = {spec["input"]: 3}, {}
    for l in layers:
        for b in l["bottom"]:
            consumers[b] = consumers.get(b, 0) + 1
        if l["type"] == "Convolution":
            channels[l["top"][0]] = l["num_output"]
        elif l["type"] == "Concat":
            channels[l["top"][0]] = sum(channels[b] for b in l["bottom"])
        elif l["type"] != "ReLU":
            channels[l["top"][0]] = channels[l["bottom"][0]]
    concat = {l["top"][0]: l["bottom"] for l in layers if l["type"] == "Concat"}
    final = [l for l in layers if l["type"] == "ImResize"][0]["bottom"][0]
    pools = {l["top"][0]: l["bottom"][0] for l in layers if l["type"] == "Pooling"}
    out = {}
    for l in layers:
        if l["type"] != "Convolution" or l["bottom"][0] == spec["input"]:
            continue
        b = l["bottom"][0]
        if b in concat and b != final:
            emap, coff, off = [], 0, {}
            for bb in concat[b]:
                off[bb] = coff
                coff += channels[bb]
            for shared in (True, False):
                for bb in concat[b]:
                    if (consumers[bb] > 1) == shared:
                        emap += list(range(off[bb], off[bb] + channels[bb])) + [-1] * (round_up(channels[bb], 16) - channels[bb])
        else:
            while b in pools:
                b = pools[b]
            emap = list(range(channels[b]))
        emap += [-1] * (round_up(len(emap), 128) - len(emap))
        k = l["kernel_size"]
        out[l["name"]] = [(t, emap[g:g + 4]) for t in range(k * k) for g in range(0, len(emap), 4)]
    return out


def check_pruned(spec, W, P):
    for name, groups in k_groups(spec).items():
        w, p = W[name][0], P[name][0]
        co, _, k, _ = w.shape
        wf, pf = w.reshape(co, -1, k * k), p.reshape(co, -1, k * k)
        kept = np.zeros(pf.shape, bool)
        for t, idx in groups:
            real = [i for i in idx if i >= 0]
            if not real:
                continue
            vals = np.abs(wf[:, real, t])                                     # (co, n)
            order = np.argsort(-vals, axis=1, kind="stable")[:, :2]           # top-2 by |w|, lower index first on a tie
            for o in range(co):
                for j in order[o]:
                    kept[o, real[j], t] = True
            assert ((pf[:, real, t] != 0).sum(axis=1) <= 2).all(), (name, t, idx)
        assert np.array_equal(pf, np.where(kept, wf, 0)), name
    assert np.array_equal(P[spec["layers"][0]["name"]][0], W[spec["layers"][0]["name"]][0])   # conv1_1 stays dense


@pytest.mark.parametrize("model", [engine.COCO_18, engine.MPI_15])
def test_prune_builtin_nets(model):
    W = synth.make_weights(model, "he", seed=5)
    W["conv3_2"] = (np.round(W["conv3_2"][0] * 4) / 4, W["conv3_2"][1])   # ties in magnitude
    check_pruned(netspec(model), W, engine.prune_2to4(W, model))


@pytest.mark.parametrize("name", list(CASES))
def test_prune_generated_graphs(name, tmp_path):
    spec, path = write_prototxt(name, tmp_path)
    W = spec_weights(spec)
    check_pruned(spec, W, engine.prune_2to4(W, prototxt=path))


def test_prune_refuses_bad_calls():
    L = engine.lib()
    for layer, shape in ((b"conv1_1", (64, 3, 3)), (b"nope", (64, 3, 3)), (b"conv1_2", (64, 64, 1))):
        buf = np.ones(int(np.prod(shape)) * shape[2], np.float32)
        assert L.pe_prune_2to4(engine.COCO_18, None, layer, buf, *shape) == -1, layer   # -PE_ERR_INVALID
        assert (buf == 1).all()


# ------------------------------------------------------------------------------------------ compression
COMPRESS = r"""
#include <stdio.h>
#include <vector>
#include "s8_sparse.h"
int main() {
    int cop; size_t K;
    if (scanf("%d %zu", &cop, &K) != 2) return 1;
    std::vector<int8_t> q((size_t)cop * K);
    for (auto& v : q) { int x; if (scanf("%d", &x) != 1) return 1; v = (int8_t)x; }
    std::vector<uint8_t> out(pe::s8_sparse_bytes(cop, K));
    if (!pe::s8_sparse_compress(q.data(), cop, K, out.data())) return 2;
    fwrite(out.data(), 1, out.size(), stdout);
    return 0;
}
"""


@pytest.fixture(scope="module")
def compress(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not found")
    d = tmp_path_factory.mktemp("s8_sparse")
    (d / "c.cpp").write_text(COMPRESS)
    subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-I", CSRC, str(d / "c.cpp"), "-o", str(d / "c")], check=True)

    def run(q):
        text = "%d %d\n" % q.shape + " ".join(map(str, q.reshape(-1).tolist()))
        r = subprocess.run([str(d / "c")], input=text.encode(), capture_output=True)
        return r.returncode, r.stdout
    return run


def expand(buf, cop, K):
    """The dense plane [cop][K] from values and metadata, by the layout of s8_sparse.h's comment."""
    vals = np.frombuffer(buf[:cop * K // 2], np.int8).reshape(cop, K // 2)
    meta = np.frombuffer(buf[cop * K // 2:], np.uint32).reshape(cop // 128, K // 128, 2, 256)
    dense = np.zeros((cop, K), np.int64)
    for cb in range(cop // 128):
        for s in range(K // 128):
            for h in range(2):
                for t in range(256):
                    wg, warp, lane = t // 128, (t // 32) % 4, t % 32
                    co = cb * 128 + 64 * wg + 16 * warp + lane // 4 + 8 * (lane % 2)
                    k0 = s * 128 + 64 * h + 32 * ((lane // 2) % 2)
                    word = int(meta[cb, s, h, t])
                    for j in range(8):
                        i0, i1 = (word >> (4 * j)) & 3, (word >> (4 * j + 2)) & 3
                        assert i0 < i1, (co, k0, j, i0, i1)
                        g = (k0 + 4 * j) // 4
                        dense[co, 4 * g + i0] = vals[co, 2 * g]
                        dense[co, 4 * g + i1] = vals[co, 2 * g + 1]
    return dense


PATTERNS = [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3), (0,), (1,), (2,), (3,), ()]


@pytest.mark.parametrize("cop,K", [(128, 128), (256, 384)])
def test_compress_expands_back_exactly(compress, cop, K):
    rng = np.random.default_rng(cop + K)
    q = np.zeros((cop, K), np.int64)
    for co in range(cop):
        for g in range(K // 4):
            for i in PATTERNS[(co * 7 + g) % len(PATTERNS)]:
                q[co, 4 * g + i] = rng.choice([-127, -1, 1, 127, *rng.integers(-127, 128, 4)]) or 5
    rc, out = compress(q)
    assert rc == 0 and len(out) == cop * K // 2 + cop // 128 * K // 128 * 2048
    assert np.array_equal(expand(out, cop, K), q)


def test_compress_refuses_three_nonzeros(compress):
    q = np.zeros((128, 128), np.int64)
    q[3, 4:7] = [1, 2, 3]
    assert compress(q)[0] == 2


# ------------------------------------------------------------------------------------------ build
build = tu_build("conv_s8_sparse.cu")
INSTANCES = 2   # pixel tiles of 128 and 64


def test_sparse_instances_no_spills_and_no_serialised_wgmma(build):
    check_no_spills_and_no_serialised_wgmma(build[0], INSTANCES)


def test_sparse_instances_keep_one_wgmma_group_in_flight(build):
    kernels = check_one_wgmma_group_in_flight(build[1], INSTANCES)
    for name, sass in kernels.items():
        assert "IGMMA.SP." in sass, name
