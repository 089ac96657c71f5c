"""K-label alpha-expansion with and without a label distance (graphcut.expansion_from_voxels, DESIGN.md §11, "Label
distances") on synthetic volumes: what the metric move and energy kernels cost against the Potts ones.

Workload: synthetic.two_blob_volume at 256^3 and 512^3 with K = 4 labels, the costs, markers and pair term of
tools/bench_multilabel.py.  Three arms run alternately after one warm-up run of each: no matrix (the Potts kernels),
V = 1 - I (the metric kernels on the Potts energy: the same labels and energy bits), and truncated linear
V = min(|i - j|, 2).  Per run it reports the moves and cycles, the device ms of the move builds, solves and label updates
per move, the device ms of the whole loop and the host wall time.  The card's name, power limit and SM clock are read in
the same run.

    python tools/bench_multilabel_metric.py [--sizes 256,512] [--reps 3] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

K = 4


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _arms():
    i = numpy.arange(K)
    return [("potts", None), ("potts_matrix", 1.0 - numpy.eye(K)),
            ("truncated_linear", numpy.minimum(numpy.abs(i[:, None] - i[None, :]), 2).astype(numpy.float64))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="256,512")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_multilabel_metric: no CUDA device (this measurement runs on the GPU only)")
    from medpy_b200 import graphcut, synthetic
    rows = []
    print("card:", _card(), flush=True)
    for size in [int(s) for s in a.sizes.split(",")]:
        vol = synthetic.two_blob_volume((size,) * 3, seed=0)
        image_h = vol["image"]
        image = torch.from_numpy(image_h).cuda()
        means = torch.linspace(0.0, 100.0, K, device=image.device, dtype=torch.float32)
        costs = (((image[None] - means[:, None, None, None]) / 20.0) ** 2).contiguous()
        fg = torch.from_numpy(vol["fg"]).cuda()
        bg = torch.from_numpy(vol["bg"]).cuda()
        markers = torch.where(fg.bool(), K, torch.where(bg.bool(), 1, 0)).to(torch.uint8)
        args = (image_h, vol["sigma"], False)
        results = {}
        for r in range(a.reps + 1):                     # round 0 warms every arm up
            for name, V in _arms():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                labels, energy, st = graphcut.expansion_from_voxels(
                    costs, graphcut.energy_voxel.boundary_difference_exponential, args, markers=markers, stats=True,
                    label_distance=V)
                torch.cuda.synchronize()
                wall = (time.perf_counter() - t0) * 1e3
                results[name] = (labels, energy, st["switched"])
                if not r:
                    continue
                m = st["moves"]
                row = dict(size=size, K=K, arm=name, rep=r, moves=m, cycles=st["cycles"], converged=st["converged"],
                           energy=energy, ms_build_per_move=st["ms_build"] / m, ms_solve_per_move=st["ms_solve"] / m,
                           ms_apply_per_move=st["ms_apply"] / m, ms_loop_device=st["ms_total"], ms_wall=wall,
                           card=_card())
                rows.append(row)
                print(json.dumps(row), flush=True)
        p, pm = results["potts"], results["potts_matrix"]
        same = bool(torch.equal(p[0], pm[0])) and numpy.float64(p[1]).tobytes() == numpy.float64(pm[1]).tobytes() \
            and p[2] == pm[2]
        print(json.dumps(dict(size=size, potts_matrix_bitwise_equal_potts=same)), flush=True)
        rows.append(dict(size=size, potts_matrix_bitwise_equal_potts=same))
        del image, costs, fg, bg, markers, results, labels
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
