"""Alpha-beta swap moves against alpha-expansion moves (DESIGN.md §11, "Swap moves") on the voxel, batch and region
units.

Workloads (K = 4):
  vol256, vol512  tools/bench_multilabel_metric.py's: synthetic.two_blob_volume at 256^3 / 512^3, label k costs
                  ((image - mu_k) / 20)^2 with the means over 0 .. 100, the blobs marked with the last label and the shell
                  with label 0, boundary_difference_exponential (expansion_from_voxels)
  slices          tools/bench_multilabel_batch.py's 512 z-slices of the 512^3 volume as 512 images of 512^2
                  (expansion_from_voxels_batch)
  regions         tools/bench_region_expansion.py's supervoxel image (cell 4) over the 256^3 volume, boundary_stawiaski
                  (expansion_from_labels)
Arms: expansion and swap under Potts, expansion and swap under truncated linear min(|i - j|, 2), and swap under
truncated quadratic min((i - j)^2, 4), run alternately after one warm-up round.  Per run: moves and cycles, the device ms
of the move builds, solves and label updates per move, the device ms of the whole loop, the host wall ms and the final
energy (the sum over the images for the batch).  The card's name, power limit and SM clock are read in the same run.

    python tools/bench_multilabel_swap.py [--workloads vol256,vol512,slices,regions] [--reps 2] [--out results.json]
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

from bench_multilabel import _card, _costs  # noqa: E402

K = 4


def _arms():
    i = numpy.arange(K)
    d = numpy.abs(i[:, None] - i[None, :])
    tl = numpy.minimum(d, 2).astype(numpy.float64)
    tq = numpy.minimum(d ** 2, 4).astype(numpy.float64)
    return [("expansion_potts", "expansion", None), ("swap_potts", "swap", None),
            ("expansion_truncated_linear", "expansion", tl), ("swap_truncated_linear", "swap", tl),
            ("swap_truncated_quadratic", "swap", tq)]


def _workload(name):
    """A function run(moves, V) -> (stats dict of the loop, energy) for the workload, on device-resident inputs."""
    import torch
    from medpy_b200 import graphcut, synthetic
    if name in ("vol256", "vol512"):
        vol = synthetic.two_blob_volume((int(name[3:]),) * 3, seed=0)
        image = torch.from_numpy(vol["image"]).cuda()
        costs = _costs(image, K)
        markers = torch.from_numpy(numpy.where(vol["fg"], K, numpy.where(vol["bg"], 1, 0)).astype(numpy.uint8)).cuda()
        args = (vol["image"], vol["sigma"], False)

        def run(moves, V):
            _, e, st = graphcut.expansion_from_voxels(costs, graphcut.energy_voxel.boundary_difference_exponential, args,
                                                      markers=markers, stats=True, label_distance=V, moves=moves)
            return st, e
        return run
    if name == "slices":
        vol = synthetic.two_blob_volume((512,) * 3, seed=0)
        images = torch.from_numpy(vol["image"]).cuda()
        means = torch.linspace(0.0, 100.0, K, device=images.device, dtype=torch.float32)
        costs = (((images[:, None] - means.reshape(1, K, 1, 1)) / 20.0) ** 2).contiguous()
        markers = torch.from_numpy(numpy.where(vol["fg"], K, numpy.where(vol["bg"], 1, 0)).astype(numpy.uint8)).cuda()
        images_h, sigma = vol["image"], vol["sigma"]

        def run(moves, V):
            _, e, st = graphcut.expansion_from_voxels_batch(costs, images_h, "difference_exponential", sigma=sigma,
                                                            markers=markers, stats=True, label_distance=V, moves=moves)
            return dict(moves=st["batch_moves"], cycles=st["batch_cycles"], converged=st["batch_converged"],
                        ms_build=st["ms_build"], ms_solve=st["ms_solve"], ms_apply=st["ms_apply"],
                        ms_total=st["ms_total"]), float(numpy.sum(e))
        return run
    from bench_labels import volume
    lab, grad, fg, bg = volume(256, 4, 1)
    vol = synthetic.two_blob_volume((256,) * 3, 1, with_prob=False)
    costs = _costs(torch.from_numpy(vol["image"]).cuda(), K)
    markers = numpy.where(fg, K, numpy.where(bg, 1, 0)).astype(numpy.uint8)

    def run(moves, V):
        _, _, e, st = graphcut.expansion_from_labels(lab, costs, graphcut.energy_label.boundary_stawiaski, grad,
                                                     markers=markers, stats=True, label_distance=V, moves=moves)
        return st, e
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="vol256,vol512,slices,regions")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_multilabel_swap: no CUDA device (this measurement runs on the GPU only)")
    rows = []
    print("card:", _card(), flush=True)
    for name in a.workloads.split(","):
        run = _workload(name)
        for r in range(a.reps + 1):                     # round 0 warms every arm up
            for arm, moves, V in _arms():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                st, energy = run(moves, V)
                torch.cuda.synchronize()
                wall = (time.perf_counter() - t0) * 1e3
                if not r:
                    continue
                m = st["moves"]
                row = dict(workload=name, K=K, arm=arm, rep=r, moves=m, cycles=st["cycles"], converged=st["converged"],
                           energy=energy, ms_build_per_move=st["ms_build"] / m, ms_solve_per_move=st["ms_solve"] / m,
                           ms_apply_per_move=st["ms_apply"] / m, ms_loop_device=st["ms_total"], ms_wall=wall,
                           card=_card())
                rows.append(row)
                print(json.dumps(row), flush=True)
        del run
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
