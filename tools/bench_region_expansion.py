"""K-label segmentation of a label image's regions by alpha-expansion (graphcut.expansion_from_labels, DESIGN.md §11
"Region graphs") on supervoxel images.

Workload: the jittered supervoxel image of tools/bench_labels.py (cell 4) over synthetic.two_blob_volume at 128^3 and
256^3, K = 3 and 4.  Label k costs ((image - mu_k) / 20)^2 per voxel with the means mu spread over the blob contrast
(0 .. 100), as CUDA tensors; the markers mark the blobs (last label) and the shell (label 0); the pair term is
boundary_stawiaski on the gradient magnitude.  Per run it reports the regions and pairs, the moves and cycles, the host
ms of the cost reduction (one region sum per label plane), the device ms of the move builds, solves and label updates
(summed and per move), the device ms of the whole loop and the host wall time from the call to the device labels.
Beside them: graph_from_labels + maxflow + mask (boundary_stawiaski, the same markers) on the same image, and
expansion_from_voxels on the same costs (boundary_difference_exponential).  The card's name, power limit and SM clock
are read in the same run.

    python tools/bench_region_expansion.py [--sizes 128,256] [--labels 3,4] [--reps 2] [--out results.json]
"""
import argparse
import json
import os
import sys
import time

import numpy

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_labels import volume  # noqa: E402
from bench_multilabel import _card, _costs  # noqa: E402


def _timed(fn, reps):
    """fn() run reps + 1 times (the first warms up); the median wall ms of the rest and the last result."""
    import torch
    times, out = [], None
    for r in range(reps + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        if r:
            times.append((time.perf_counter() - t0) * 1e3)
    return float(numpy.median(times)), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="128,256")
    ap.add_argument("--labels", default="3,4")
    ap.add_argument("--cell", type=int, default=4)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_region_expansion: no CUDA device (this measurement runs on the GPU only)")
    from medpy_b200 import graphcut, synthetic
    from medpy_b200.graphcut.energy_label import LabelContext
    rows = []
    print("card:", _card(), flush=True)
    for size in [int(s) for s in a.sizes.split(",")]:
        lab, grad, fg, bg = volume(size, a.cell, 1)
        vol = synthetic.two_blob_volume((size,) * 3, 1, with_prob=False)
        image_h = vol["image"]
        image = torch.from_numpy(image_h).cuda()
        term = graphcut.energy_label.boundary_stawiaski

        def binary():
            g = graphcut.graph_from_labels(lab, fg, bg, boundary_term=term, boundary_term_args=grad)
            g.maxflow()
            return graphcut.label_cut_mask(g)

        ms_binary, _ = _timed(binary, a.reps)
        for K in [int(k) for k in a.labels.split(",")]:
            costs = _costs(image, K)
            markers = numpy.where(fg, K, numpy.where(bg, 1, 0)).astype(numpy.uint8)
            ctx = LabelContext(lab)

            def reduce():
                return [ctx.native.region_sums(costs[k], ctx._mgc.SUM_BINCOUNT)[0] for k in range(K)]

            ms_reduce, _ = _timed(reduce, a.reps)
            del ctx
            ms_wall, (labels, region_labels, energy, st) = _timed(
                lambda: graphcut.expansion_from_labels(lab, costs, term, grad, markers=markers, stats=True), a.reps)
            markers_d = torch.from_numpy(markers).cuda()
            ms_voxels, (_, _, vst) = _timed(lambda: graphcut.expansion_from_voxels(
                costs, graphcut.energy_voxel.boundary_difference_exponential, (image_h, vol["sigma"], False),
                markers=markers_d, stats=True), a.reps)
            m = st["moves"]
            row = dict(size=size, cell=a.cell, K=K, regions=int(lab.max()), moves=m, cycles=st["cycles"],
                       converged=st["converged"], energy=energy, switched=st["switched"], ms_cost_reduction=ms_reduce,
                       ms_build=st["ms_build"], ms_solve=st["ms_solve"], ms_apply=st["ms_apply"],
                       ms_build_per_move=st["ms_build"] / m, ms_solve_per_move=st["ms_solve"] / m,
                       ms_apply_per_move=st["ms_apply"] / m, ms_loop_device=st["ms_total"], ms_wall=ms_wall,
                       ms_graph_from_labels_maxflow_mask=ms_binary, ms_expansion_from_voxels_wall=ms_voxels,
                       voxels_moves=vst["moves"], voxels_ms_loop_device=vst["ms_total"], card=_card())
            rows.append(row)
            print(json.dumps(row), flush=True)
            del costs, labels, markers_d
        del image
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
