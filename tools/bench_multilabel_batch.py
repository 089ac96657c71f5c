"""Batched K-label segmentation (graphcut.expansion_from_voxels_batch, DESIGN.md §11 "Batches") against a loop of
graphcut.expansion_from_voxels, one call per image, on the same costs.

Workloads, with the cost model of tools/bench_multilabel.py (label k costs ((image - mu_k) / 20)^2, the means spread over
0 .. 100; the blobs marked with the last label and the shell with label 0; boundary_difference_exponential with the
volume's sigma):
  slices  the 512 z-slices of the 512^3 two-blob volume as 512 images of 512^2, K = 3 and 4
  vols    32 two-blob volumes of 128^3 (seeds 0..31), K = 4
The costs are CUDA tensors, the images host arrays (as the boundary terms take them).  Per workload and K it reports the
batch loop's moves and cycles, its build / solve / apply device ms per move, its whole-loop device ms and host wall ms;
for the per-image loop the sum of the calls' device ms and the host wall ms of the whole loop; and whether every image's
labels and switch counts are equal in the two arms (and which images differ).  The card's name, power limit and SM clock are read in the same run.

    python tools/bench_multilabel_batch.py [--workloads slices,vols] [--reps 2] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _workload(name):
    """(images (B, *image) float32, markers uint8 (B, *image) as 0 / 1 = shell / 2 = blob, sigma)."""
    from medpy_b200 import synthetic
    if name == "slices":
        vol = synthetic.two_blob_volume((512,) * 3, seed=0)
        return vol["image"], numpy.where(vol["fg"], 2, numpy.where(vol["bg"], 1, 0)).astype(numpy.uint8), vol["sigma"]
    vols = [synthetic.two_blob_volume((128,) * 3, seed=s) for s in range(32)]
    images = numpy.stack([v["image"] for v in vols])
    marks = numpy.stack([numpy.where(v["fg"], 2, numpy.where(v["bg"], 1, 0)) for v in vols]).astype(numpy.uint8)
    return images, marks, vols[0]["sigma"]


def _costs(image, K):
    import torch
    means = torch.linspace(0.0, 100.0, K, device=image.device, dtype=torch.float32)
    shape = (1, K) + (1,) * (image.dim() - 1)
    return (((image[:, None] - means.reshape(shape)) / 20.0) ** 2).contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="slices,vols")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_multilabel_batch: no CUDA device (this measurement runs on the GPU only)")
    from medpy_b200 import graphcut
    term = graphcut.energy_voxel.boundary_difference_exponential
    rows = []
    print("card:", _card(), flush=True)
    for name in a.workloads.split(","):
        images_h, marks, sigma = _workload(name)
        B = images_h.shape[0]
        images = torch.from_numpy(images_h).cuda()
        for K in ([3, 4] if name == "slices" else [4]):
            costs = _costs(images, K)
            markers_h = numpy.where(marks == 2, K, marks).astype(numpy.uint8)
            markers = torch.from_numpy(markers_h).cuda()
            for r in range(a.reps + 1):     # the first run of both arms warms up
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                labels, energies, st = graphcut.expansion_from_voxels_batch(costs, images_h, "difference_exponential",
                                                                            sigma=sigma, markers=markers, stats=True)
                torch.cuda.synchronize()
                wall = (time.perf_counter() - t0) * 1e3
                m = st["batch_moves"]
                row = dict(workload=name, images=B, image_shape=list(images_h.shape[1:]), K=K, moves=m,
                           cycles=st["batch_cycles"], converged=st["batch_converged"],
                           image_cycles=[min(st["cycles"]), max(st["cycles"])],
                           ms_build_per_move=st["ms_build"] / m, ms_solve_per_move=st["ms_solve"] / m,
                           ms_apply_per_move=st["ms_apply"] / m, ms_batch_device=st["ms_total"], ms_batch_wall=wall,
                           card=_card())
                # the per-image loop, on the same device costs
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                loop_dev, loop_moves, differ = 0.0, 0, []
                for b in range(B):
                    lab, e, s = graphcut.expansion_from_voxels(costs[b], term, (images_h[b], sigma, False),
                                                               markers=markers[b], stats=True)
                    loop_dev += s["ms_total"]
                    loop_moves += s["moves"]
                    if not (bool(torch.equal(lab, labels[b])) and s["switched"] == st["switched"][b]):
                        differ.append(b)
                torch.cuda.synchronize()
                row.update(loop_moves=loop_moves, ms_loop_device=loop_dev, ms_loop_wall=(time.perf_counter() - t0) * 1e3,
                           labels_equal=not differ, images_differing=differ)
                if not r:       # the first pass of both arms warms up
                    continue
                rows.append(row)
                print(json.dumps(row), flush=True)
            del costs, markers, labels
        del images
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
