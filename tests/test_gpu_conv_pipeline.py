"""The pipeline of conv_wg_kernel (conv_tc.cu) does not depend on timing.

The consumers keep one wgmma group in flight and free each shared-memory slot one K step late; the producer refills a weight
slot once the consumers of both CTAs of a cluster have freed it.  How far the producer runs ahead, and when the partner
CTA gets there, depends on what else runs on the GPU, never the arithmetic: every conv blob must be bit-identical with one
handle alone, with two handles forwarding at the same time on their own streams (their launches compete for the SMs), and
over CUDA-graph capture and replays.
"""
import hashlib

import numpy as np
import pytest

from caffe_rtpose_b200 import engine
from test_gpu_conv_layers import CONFIGS_FINAL, checked_layers, frames_for, weights_with_biases


def digests(eng, n, tops):
    """sha1 of every checked conv blob and the stride-8 maps of the last forward's n images (one blob on the host at a time)."""
    out = {t: hashlib.sha1(np.ascontiguousarray(eng.fetch_blob(t)[:n]).tobytes()).hexdigest() for t in tops}
    out["maps"] = hashlib.sha1(eng.fetch_maps(n).tobytes()).hexdigest()
    return out


def check_runs(model, prec, net_w, net_h, counts):
    W = weights_with_biases(model)
    tops = [l["top"] for l in checked_layers(model) if l["top"] not in CONFIGS_FINAL]
    engs = [engine.PoseEngine(model, net_w, net_h, 2 * net_w, 2 * net_h, precision=prec, max_batch=max(counts)) for _ in range(2)]
    for e in engs:
        e.set_weights(W)
    frames = frames_for(max(counts), 2 * net_w, 2 * net_h)
    for n in counts:
        engs[0].forward_frames(frames[:n])   # first forward of a batch size: eager launches
        ref = digests(engs[0], n, tops)
        runs = []
        for rep in range(2):                  # the second forward captures a CUDA graph, the third replays it
            engs[0].forward_frames(frames[:n])
            runs.append(("graph %d" % rep, digests(engs[0], n, tops)))
        for rep in range(2):                  # both handles in flight: their conv launches share the SMs
            engs[0].forward_frames(frames[:n])
            engs[1].forward_frames(frames[:n])
            runs.append(("concurrent %d, handle 0" % rep, digests(engs[0], n, tops)))
            runs.append(("concurrent %d, handle 1" % rep, digests(engs[1], n, tops)))
        for what, d in runs:
            diff = [k for k in ref if d[k] != ref[k]]
            assert not diff, "%d frames, %s: differs from the handle alone in %s" % (n, what, diff)
    for e in engs:
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [engine.PREC_F16X2, engine.PREC_F16X1], ids=["parity", "f16x1"])
def test_small_batches_identical_alone_concurrent_and_replayed(prec):
    # 160x96: one frame runs the stride-8 layers at half width, odd frame counts leave a row tile without rows
    check_runs(engine.COCO_18, prec, 160, 96, (1, 2, 3, 4))


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [engine.PREC_F16X2, engine.PREC_F16X1], ids=["parity", "f16x1"])
def test_bench_batch_identical_alone_concurrent_and_replayed(prec):
    # the benchmark's geometry: 9 frames at 656x368
    check_runs(engine.COCO_18, prec, 656, 368, (9,))
