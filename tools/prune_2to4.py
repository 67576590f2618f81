#!/usr/bin/env python3
"""Magnitude-prune a .caffemodel's conv weights to 2:4 in the engine's packed K order (engine.prune_2to4, pe_prune_2to4): the
grouping in which a --precision 6 engine can run a layer on the 2:4-sparse s8 kernel (pe_conv_layer_sparse; its shape rule
decides which layer classes do).

Pruning a trained model without fine-tuning changes its outputs: each group of four keeps only its two largest weights.
Prune and fine-tune with a 2:4 sparsity workflow (e.g. NVIDIA's ASP) for a model that keeps its accuracy, then check it with
this grouping.  The output holds the conv layers only (the layers the engine reads)."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from caffe_rtpose_b200 import engine  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("input", help="a .caffemodel of the COCO or MPI pose net (or of --prototxt)")
    ap.add_argument("output", help="the pruned .caffemodel")
    ap.add_argument("--prototxt", default=None, help="deploy prototxt of the net (default: the built-in graph of --model)")
    ap.add_argument("--model", default="COCO", choices=["COCO", "MPI"], help="built-in graph without --prototxt (default COCO)")
    args = ap.parse_args()
    model = None if args.prototxt else {"COCO": engine.COCO_18, "MPI": engine.MPI_15}[args.model]
    weights, table = {}, []
    for name, _, blobs in engine.read_caffemodel(args.input):
        if len(blobs) != 2 or len(blobs[0][1]) != 4:
            continue
        (w, shape), (b, _) = blobs
        weights[name] = (w.reshape(shape), b)
        table.append((name, shape[0], shape[1], shape[2]))
    pruned = engine.prune_2to4(weights, model=model, prototxt=args.prototxt)
    engine.write_caffemodel(args.output, pruned, table)
    kept = sum(int((pruned[n][0] != 0).sum()) for n in pruned)
    total = sum(pruned[n][0].size for n in pruned)
    print("%d conv layers, %.1f%% of the weights non-zero, written to %s" % (len(table), 100.0 * kept / max(total, 1), args.output))


if __name__ == "__main__":
    main()
