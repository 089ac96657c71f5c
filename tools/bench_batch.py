"""Batched cuts against one cut per image, on device-resident inputs (DESIGN.md §3.1).

Workloads:
  (a) slices : the 512 z-slices of synthetic.two_blob_volume(512^3) as 512 independent 2-D images, each with its own
               sigma (the RMS neighbour difference of the slice) -- a stack segmented slice by slice;
  (b) cohort : 32 two-blob volumes of 128^3 with seeds 0..31 -- a cohort of small volumes.
Each arm (graph_from_voxels_batch once; graph_from_device_arrays + maxflow + get_mask per image) is warmed up, then
timed with CUDA events over --reps repetitions.  Every mask is compared image by image between the two arms.  The card's
name and power limit are printed with the numbers: a time means nothing without them.

    python tools/bench_batch.py [--reps 3] [--workloads slices,cohort]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _rms_sigma(t):
    """RMS of the neighbour differences of every image of a (B, ...) tensor, per image."""
    import torch
    acc = torch.zeros(t.shape[0], dtype=torch.float64, device=t.device)
    cnt = 0
    for ax in range(1, t.dim()):
        d = torch.diff(t.double(), dim=ax)
        acc += (d * d).flatten(1).sum(1)
        cnt += d[0].numel()
    return torch.sqrt(acc / cnt).tolist()


def _slices():
    import torch
    from medpy_b200 import synthetic
    v = synthetic.two_blob_volume((512, 512, 512), seed=0)
    d = {k: torch.from_numpy(numpy.ascontiguousarray(v[k])).cuda() for k in ("image", "prob", "fg", "bg")}
    return d, _rms_sigma(d["image"]), v["alpha"]


def _cohort():
    import torch
    from medpy_b200 import synthetic
    vs = [synthetic.two_blob_volume((128, 128, 128), seed=s) for s in range(32)]
    d = {k: torch.from_numpy(numpy.stack([v[k] for v in vs])).cuda() for k in ("image", "prob", "fg", "bg")}
    return d, [float(v["sigma"]) for v in vs], vs[0]["alpha"]


def _batched(d, sigmas, alpha):
    import medpy_b200.graphcut as gc
    g = gc.graph_from_voxels_batch(d["fg"], d["bg"], d["image"], "difference_exponential", sigma=sigmas, prob=d["prob"],
                                   alpha=alpha)
    e = g.maxflow()
    return e, g.get_mask()


def _loop(d, sigmas, alpha):
    from medpy_b200.graphcut.device import graph_from_device_arrays
    es, ms = [], []
    for b in range(d["image"].shape[0]):
        g = graph_from_device_arrays(d["fg"][b], d["bg"][b], d["image"][b], "difference_exponential", sigma=sigmas[b],
                                     prob=d["prob"][b], alpha=alpha)
        es.append(g.maxflow())
        ms.append(numpy.asarray(g.get_mask()).reshape(tuple(d["image"].shape[1:])))
    return numpy.array(es), numpy.stack(ms)


def _time(fn, reps):
    import torch
    fn()                                   # warm-up: module loads, pools, instantiations
    torch.cuda.synchronize()
    times, out = [], None
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return sorted(times)[len(times) // 2], out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workloads", default="slices,cohort")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_batch: no CUDA device")
    card = _card()
    for name in args.workloads.split(","):
        d, sigmas, alpha = {"slices": _slices, "cohort": _cohort}[name]()
        t_batch, (e_b, m_b) = _time(lambda: _batched(d, sigmas, alpha), args.reps)
        t_loop, (e_l, m_l) = _time(lambda: _loop(d, sigmas, alpha), args.reps)
        mism = [b for b in range(len(e_l)) if not (m_b[b] == m_l[b]).all()]
        rel = float(numpy.max(numpy.abs(e_b - e_l) / numpy.maximum(numpy.abs(e_l), 1e-300)))
        print(json.dumps({"workload": name, "images": int(d["image"].shape[0]), "image_shape": list(d["image"].shape[1:]),
                          "batched_ms": round(t_batch, 3), "loop_ms": round(t_loop, 3),
                          "speedup": round(t_loop / t_batch, 2), "mask_mismatch_images": mism,
                          "max_energy_rel_diff": rel, "card": card}), flush=True)
        del d


if __name__ == "__main__":
    main()
