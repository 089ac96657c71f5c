"""K-label segmentation by alpha-expansion (graphcut.expansion_from_voxels, DESIGN.md §11) on synthetic volumes.

Workload: synthetic.two_blob_volume at 256^3 and 512^3 with K = 3 and K = 4 labels.  Label k costs
((image - mu_k) / 20)^2 with the means mu spread over the blob contrast (0 .. 100); the markers of the volume mark the
blobs (last label) and the shell (label 0); the pair term is boundary_difference_exponential with the volume's sigma.
The costs are CUDA tensors (resident inputs); the labels come back as a CUDA tensor.  Per run it reports the moves and
cycles, the device ms of the move builds, solves and label updates (summed over the moves and per move), the device ms
of the whole loop, the host wall time from the call to the device labels, and the same volume's K = 2 cut
(graph_from_device_arrays with the regional term, maxflow, mask) as a yardstick.  The card's name, power limit and SM
clock are read in the same run.

    python tools/bench_multilabel.py [--sizes 256,512] [--labels 3,4] [--reps 2] [--out results.json]
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


def _costs(image, K):
    import torch
    means = torch.linspace(0.0, 100.0, K, device=image.device, dtype=torch.float32)
    return (((image[None] - means[:, None, None, None]) / 20.0) ** 2).contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="256,512")
    ap.add_argument("--labels", default="3,4")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_multilabel: no CUDA device (this measurement runs on the GPU only)")
    from medpy_b200 import graphcut, synthetic
    from medpy_b200.graphcut.device import graph_from_device_arrays
    rows = []
    print("card:", _card(), flush=True)
    for size in [int(s) for s in a.sizes.split(",")]:
        vol = synthetic.two_blob_volume((size,) * 3, seed=0)
        image_h = vol["image"]
        image = torch.from_numpy(image_h).cuda()
        prob = torch.from_numpy(vol["prob"]).cuda()
        fg = torch.from_numpy(vol["fg"]).cuda()
        bg = torch.from_numpy(vol["bg"]).cuda()
        # K = 2 yardstick: the binary cut of the same volume from resident inputs
        g = None
        k2 = []
        for r in range(a.reps + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            g = graph_from_device_arrays(fg, bg, image=image, boundary="difference_exponential", sigma=vol["sigma"],
                                         prob=prob, alpha=vol["alpha"], graph=g)
            g.maxflow()
            g.get_mask()
            torch.cuda.synchronize()
            if r:
                k2.append((time.perf_counter() - t0) * 1e3)
        del g
        for K in [int(k) for k in a.labels.split(",")]:
            costs = _costs(image, K)
            markers = torch.where(fg.bool(), K, torch.where(bg.bool(), 1, 0)).to(torch.uint8)
            args = (image_h, vol["sigma"], False)
            for r in range(a.reps + 1):     # the first run warms up
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                labels, energy, st = graphcut.expansion_from_voxels(
                    costs, graphcut.energy_voxel.boundary_difference_exponential, args, markers=markers, stats=True)
                torch.cuda.synchronize()
                wall = (time.perf_counter() - t0) * 1e3
                if not r:
                    continue
                m = st["moves"]
                row = dict(size=size, K=K, moves=m, cycles=st["cycles"], converged=st["converged"], energy=energy,
                           switched=st["switched"], ms_build=st["ms_build"], ms_solve=st["ms_solve"],
                           ms_apply=st["ms_apply"], ms_build_per_move=st["ms_build"] / m,
                           ms_solve_per_move=st["ms_solve"] / m, ms_apply_per_move=st["ms_apply"] / m,
                           ms_loop_device=st["ms_total"], ms_wall=wall, ms_k2_median=float(numpy.median(k2)),
                           card=_card())
                rows.append(row)
                print(json.dumps(row), flush=True)
            del costs, markers, labels
        del image, prob, fg, bg
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
