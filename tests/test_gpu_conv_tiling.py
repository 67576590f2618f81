"""Row tiles and weight-tile clusters of conv_wg_kernel on small nets (conv_tc.cu).

The kernel's row tiles start at every image: tile t of image i covers the flat padded rows [i*Hs*Wp + 128 t, + 128), with
ceil(((H-1)*Wp + W) / 128) tiles per image, and the grid is rounded up to whole clusters of CTAs that share each weight
tile through a TMA multicast.  At 160x96 the stride-8 level is 20x12 with a gap of 3: an image spans 15 x 23 = 345 rows, its
last pixel is row 272, so the last of its 3 tiles reaches 39 rows into the next image.  The 3 tiles per image at stride 8
and the 121 at full resolution make the grid odd for an odd frame count, so a cluster holds a CTA with no rows.  One frame
runs the stride-8 layers at half width and four frames run the stride-2 layers at full width.

Two properties are checked at 1-4 frames: every conv blob of frame k in a batch is bit-identical to frame k run alone (the
tiling changes which CTA computes a row, never its arithmetic), and every layer passes the float64 check of
test_gpu_conv_layers.py, on its sampled pixels plus the first and last row tile of every image.
"""
import numpy as np
import pytest
import torch

from caffe_rtpose_b200 import engine, synth
from test_gpu_conv_layers import (MEASURED_MAX, Blobs, CONFIGS_FINAL, check_layer, checked_layers, frames_for, layer_class,
                                  level_geo, sample_pixels, tc_instance, weights_with_biases)

NET_W, NET_H = 160, 96
COUNTS = (1, 2, 3, 4)


def tiles_per_image(H, W, gap):
    return -(-((H - 1) * (W + gap) + W) // 128)


def image_tile_pixels(N, H, W, gap):
    """(P, 3) (n, y, x) of every pixel in the first and the last row tile of each image, including the rows of the next
    image that the last tile spans."""
    Wp, per = W + gap, (H + gap) * (W + gap)
    T = tiles_per_image(H, W, gap)
    m = np.concatenate([i * per + np.r_[0:128, 128 * (T - 1):128 * T] for i in range(N)])
    m = m[m < N * per]
    n, rem = m // per, m % per
    y, x = rem // Wp, rem % Wp
    keep = (x < W) & (y < H)
    return np.stack([n, y, x], 1)[keep]


def test_tiles_cover_each_image_and_the_gap_is_shorter_than_a_tile():
    # 20x12 at stride 8: 3 tiles, the last one reaching into the next image
    W, H, gap = level_geo(NET_W, NET_H, 3)
    Wp, per = W + gap, (H + gap) * (W + gap)
    T = tiles_per_image(H, W, gap)
    assert (H, W, T, per) == (12, 20, 3, 345) and 128 * T > per
    last = (H - 1) * Wp + W - 1
    assert 128 * (T - 1) <= last < 128 * T
    assert tiles_per_image(96, 160, 1) == 121 and tiles_per_image(46, 82, 3) == 31
    pts = image_tile_pixels(2, H, W, gap)
    assert {tuple(p) for p in pts} == {(n, y, x) for n in range(2) for y in range(H) for x in range(W) if not 128 <= y * Wp + x < 256}


@pytest.mark.gpu
@pytest.mark.parametrize("model", [engine.COCO_18, engine.MPI_15], ids=["coco", "mpi"])
def test_batched_frames_match_frames_alone_and_float64(model):
    prec = engine.PREC_F16X2
    W = weights_with_biases(model)
    eng = engine.PoseEngine(model, NET_W, NET_H, 2 * NET_W, 2 * NET_H, precision=prec, max_batch=max(COUNTS))
    eng.set_weights(W)
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    frames = frames_for(max(COUNTS), 2 * NET_W, 2 * NET_H)
    layers = checked_layers(model)
    tops = [l["top"] for l in layers if l["top"] not in CONFIGS_FINAL]

    alone = []
    for f in frames:
        eng.forward_frames([f])
        alone.append({t: eng.fetch_blob(t)[:1].copy() for t in tops})
        alone[-1]["maps"] = eng.fetch_maps(1)[:1]

    rng = np.random.default_rng(7)
    worst, widths, odd = {}, set(), set()
    for n in COUNTS:
        eng.forward_frames(frames[:n])
        blobs = Blobs(eng, n, model, W)
        for k in range(n):
            diff = [t for t in tops if not np.array_equal(blobs.get(t)[k:k + 1], alone[k][t])]
            if not np.array_equal(eng.fetch_maps(n)[k:k + 1], alone[k]["maps"]):
                diff.append("maps")
            assert not diff, "frame %d of %d differs from the frame alone in %s" % (k, n, diff)
        for layer in layers:
            w_, h_, gap = level_geo(NET_W, NET_H, layer["level"])
            pts = np.unique(np.concatenate([sample_pixels(n, h_, w_, gap, rng, 200), image_tile_pixels(n, h_, w_, gap)]), axis=0)
            r = check_layer(layer, blobs, W, prec, pts, False, False)
            key = layer_class(layer)
            worst[key] = max(worst.get(key, 0.0), r)
            ks = 1 if layer["name"] == "conv1_1" else layer["k"]
            widths.add(tc_instance(W[layer["name"]][0].shape[0], ks, n * (h_ + gap) * (w_ + gap), prec, nsm)[0])
            if n * tiles_per_image(h_, w_, gap) % 2:
                odd.add(layer["level"])
    eng.close()
    print("\n%s at %dx%d: largest |got - ref| / mag per layer class: %s" % ("coco" if model == engine.COCO_18 else "mpi", NET_W, NET_H,
                                                                          {k: "%.3e" % v for k, v in sorted(worst.items())}))
    over = {k: v for k, v in worst.items() if v > MEASURED_MAX[prec][k]}
    assert not over, "accumulation error above what this kernel measured: %s" % over
    assert {128, 64} <= widths, widths   # both tile widths ran
    assert {0, 1, 3} <= odd, odd         # grids with an empty CTA in the last cluster
