"""Correcting a few images of a solved batch: a warm fold into the batch against a cold rebuild of the batch and against
one warm single-image handle per corrected image (DESIGN.md §3.1, "Warm edits").

Workload: the 512 z-slices of synthetic.two_blob_volume(512^3) as 512 independent 2-D images, each with its own sigma
(the RMS neighbour difference of the slice), as in tools/bench_batch.py.  A stroke is a foreground line across the
background between the two blobs (row 256, columns 200..311 of a slice); it goes on 1, 8 or 64 slices spread evenly
over the stack.  Inputs and stroke ids are device-resident.  Arms, each timed with CUDA events from the edit to the
masks on the host:
  warm   : add_seeds(stroke ids) + maxflow + get_mask on a solved graph_from_voxels_batch(..., warm=True);
  cold   : graph_from_voxels_batch with the stroke merged into the foreground markers + maxflow + get_mask;
  single : for each stroked slice, add_seeds + maxflow + get_mask on its own solved graph_from_device_arrays handle.
The build and first solve the warm arms start from are not timed.  Every arm is warmed up once, then run --reps times
(median reported).  The masks of the stroked slices must be equal across the three arms, and the whole batch mask
equal between warm and cold.  A fold ends in a full relabel reset over the whole batch lattice: its share of the warm
span is reported from the library's stats (ms_relabel_first: the first relabel of the re-solve; ms_relabel: all of
them).  The card's name and power limit are read in the same run.

Dense folds (--dense): add_tweights_warm(None, src, snk) with a nonzero weight on every voxel -- a GrabCut-style
regional update -- so every voxel is one entry of the fold and each image's run of entries is as long as it gets.  On
a cohort of 32 two-blob volumes of 128^3 and on one 256^3 volume as a batch of one, against the same call on one
single-image handle of the first volume.  Reported: the fold's device time (the library's ms_seeds), whose end is the
per-image sum of the constant changes, and the whole call + maxflow + masks span.

    python tools/bench_refine_batch.py [--reps 3] [--strokes 1,8,64] [--dense cohort,one256]
"""
import argparse
import json
import os
import sys

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_batch import _card, _slices  # noqa: E402


def _stroke(d, k):
    """The stroked slices and the stroke's voxels: local ids of one slice, batch ids over all stroked slices."""
    import torch
    B, Y, X = (int(s) for s in d["image"].shape)
    slices = numpy.unique(numpy.linspace(0, B - 1, k).round().astype(numpy.int64))
    local = numpy.arange(200, 312, dtype=numpy.int64) + 256 * X
    ids = (slices[:, None] * (Y * X) + local[None, :]).ravel()
    return slices, torch.as_tensor(local, device="cuda"), torch.as_tensor(ids, device="cuda")


def _events():
    import torch
    return torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


def _span(fn):
    """CUDA-event span of fn() (which ends with its results on the host), and fn's result."""
    a, b = _events()
    a.record()
    out = fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b), out


def _warm_batch(d, sigmas, alpha, ids):
    import medpy_b200.graphcut as gc
    g = gc.graph_from_voxels_batch(d["fg"], d["bg"], d["image"], "difference_exponential", sigma=sigmas, prob=d["prob"],
                                   alpha=alpha, warm=True)
    g.maxflow()
    s0 = g.stats()

    def edit():
        g.add_seeds(ids, None)
        g.maxflow()
        return g.get_mask()
    ms, mask = _span(edit)
    s1 = g.stats()
    return ms, mask, {k: s1[k] - s0[k] for k in ("ms_relabel_first", "ms_relabel", "ms_seeds", "ms_solve")}


def _cold_batch(d, sigmas, alpha, ids):
    import medpy_b200.graphcut as gc

    def run():
        fg = d["fg"].clone()
        fg.view(-1)[ids] = True
        g = gc.graph_from_voxels_batch(fg, d["bg"], d["image"], "difference_exponential", sigma=sigmas, prob=d["prob"],
                                       alpha=alpha)
        g.maxflow()
        return g.get_mask()
    ms, mask = _span(run)
    return ms, mask


def _singles(d, sigmas, alpha, slices, local):
    from medpy_b200.graphcut.device import graph_from_device_arrays
    shape = tuple(int(s) for s in d["image"].shape[1:])
    gs = []
    for b in (int(x) for x in slices):
        g = graph_from_device_arrays(d["fg"][b], d["bg"][b], d["image"][b], "difference_exponential", sigma=sigmas[b],
                                     prob=d["prob"][b], alpha=alpha)
        g.maxflow()
        gs.append(g)

    def edit():
        out = []
        for g in gs:
            g.add_seeds(local, None)
            g.maxflow()
            out.append(numpy.asarray(g.get_mask()).reshape(shape))
        return numpy.stack(out)
    return _span(edit)


def _dense_volumes(name):
    import torch
    from medpy_b200 import synthetic
    if name == "cohort":
        from bench_batch import _cohort
        return _cohort()
    v = synthetic.two_blob_volume((256, 256, 256), seed=0)
    d = {k: torch.from_numpy(numpy.ascontiguousarray(v[k][None])).cuda() for k in ("image", "prob", "fg", "bg")}
    return d, [float(v["sigma"])], v["alpha"]


def _dense_fold(g):
    """add_tweights_warm on every voxel of a solved graph: fold ms (ms_seeds), and the span of the call + solve + masks."""
    import torch
    shape = tuple(int(s) for s in g.shape)
    src = torch.full(shape, 0.05, dtype=torch.float64, device="cuda")
    snk = torch.zeros(shape, dtype=torch.float64, device="cuda")
    s0 = g.stats()

    def edit():
        g.add_tweights_warm(None, src, snk)
        g.maxflow()
        return g.get_mask()
    ms, _ = _span(edit)
    return g.stats()["ms_seeds"] - s0["ms_seeds"], ms


def _dense(name, reps, card):
    import medpy_b200.graphcut as gc
    from medpy_b200.graphcut.device import graph_from_device_arrays
    d, sigmas, alpha = _dense_volumes(name)
    rows = {"batch": [], "single": []}
    for rep in range(reps + 1):
        g = gc.graph_from_voxels_batch(d["fg"], d["bg"], d["image"], "difference_exponential", sigma=sigmas,
                                       prob=d["prob"], alpha=alpha, warm=True)
        g.maxflow()
        fold_b, span_b = _dense_fold(g)
        del g
        s = graph_from_device_arrays(d["fg"][0], d["bg"][0], d["image"][0], "difference_exponential", sigma=sigmas[0],
                                     prob=d["prob"][0], alpha=alpha)
        s.maxflow()
        fold_s, span_s = _dense_fold(s)
        del s
        if rep:
            rows["batch"].append((fold_b, span_b))
            rows["single"].append((fold_s, span_s))
    med = {a: sorted(r)[len(r) // 2] for a, r in rows.items()}
    print(json.dumps({
        "workload": "dense_" + name, "images": int(d["image"].shape[0]), "image_shape": list(d["image"].shape[1:]),
        "entries": int(d["image"].numel()), "batch_fold_ms": round(med["batch"][0], 3),
        "batch_span_ms": round(med["batch"][1], 3), "single_image_fold_ms": round(med["single"][0], 3),
        "single_image_span_ms": round(med["single"][1], 3),
        "batch_runs": [[round(a, 3), round(b, 3)] for a, b in rows["batch"]],
        "single_runs": [[round(a, 3), round(b, 3)] for a, b in rows["single"]], "card": card}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--strokes", default="1,8,64")
    ap.add_argument("--dense", default="", help="dense-fold workloads: cohort, one256 (comma separated)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_refine_batch: no CUDA device")
    card = _card()
    for name in (x for x in args.dense.split(",") if x):
        _dense(name, args.reps, card)
    if not args.strokes:
        return
    d, sigmas, alpha = _slices()
    for k in (int(x) for x in args.strokes.split(",")):
        slices, local, ids = _stroke(d, k)
        rows = {"warm": [], "cold": [], "single": []}
        stats = []
        masks = {}
        for rep in range(args.reps + 1):           # rep 0 warms every arm up and is not reported
            ms, masks["warm"], st = _warm_batch(d, sigmas, alpha, ids)
            if rep:
                rows["warm"].append(ms)
                stats.append(st)
            ms, masks["cold"] = _cold_batch(d, sigmas, alpha, ids)
            if rep:
                rows["cold"].append(ms)
            ms, masks["single"] = _singles(d, sigmas, alpha, slices, local)
            if rep:
                rows["single"].append(ms)
        med = {a: sorted(t)[len(t) // 2] for a, t in rows.items()}
        warm = sorted(range(len(stats)), key=lambda i: rows["warm"][i])[len(stats) // 2]
        st = stats[warm]
        equal_batch = bool((masks["warm"] == masks["cold"]).all())
        equal_slices = bool((masks["warm"][slices] == masks["single"]).all() and
                            (masks["cold"][slices] == masks["single"]).all())
        print(json.dumps({
            "workload": "slices", "images": int(d["image"].shape[0]), "stroked_slices": int(len(slices)),
            "stroke_voxels": int(ids.numel()), "warm_ms": round(med["warm"], 3), "cold_ms": round(med["cold"], 3),
            "single_ms": round(med["single"], 3), "warm_runs_ms": [round(x, 3) for x in rows["warm"]],
            "cold_runs_ms": [round(x, 3) for x in rows["cold"]], "single_runs_ms": [round(x, 3) for x in rows["single"]],
            "warm_fold_ms": round(st["ms_seeds"], 3), "warm_solve_ms": round(st["ms_solve"], 3),
            "first_relabel_ms": round(st["ms_relabel_first"], 3), "relabel_ms": round(st["ms_relabel"], 3),
            "first_relabel_share_of_warm": round(st["ms_relabel_first"] / rows["warm"][warm], 3),
            "relabel_share_of_warm": round(st["ms_relabel"] / rows["warm"][warm], 3),
            "masks_equal_warm_cold": equal_batch, "masks_equal_stroked_slices_all_arms": equal_slices,
            "card": card}), flush=True)


if __name__ == "__main__":
    main()
