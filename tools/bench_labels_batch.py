"""A batch of label images cut as one region graph against the same cuts one after the other (DESIGN.md §8, "A batch of
label images").

Cases:
  (a) slices : 512 2-D slices of 512^2 supervoxel maps (8x8 blocks, shifted per slice: about 4200 regions per slice),
               a float32 gradient, a foreground disk and a background frame per slice.  Arms: graph_from_labels_batch +
               maxflow + label_cut_masks, against a loop of graph_from_labels + maxflow + label_cut_mask per slice.
  (b) split  : graphcut_split(graphcut_stawiaski, ...) of a 256^3 supervoxel volume (8^3 blocks, about 32 800 regions)
               with minimal_edge_length=64, overlap 10 (64 sub-volumes), batch=True against batch=False.
Every arm is warmed up once, then the arms alternate for --reps rounds; medians of the host-clock spans (each span
ends with the masks on the host, so the device work is inside it).  Masks must be equal between the arms.  The card's
name, power limit and SM clock are read in the same run.

    python tools/bench_labels_batch.py [--reps 5] [--cases slices,split] [--out results/bench_labels_batch.json]
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
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def shifted_blocks(shape, cell, shift):
    """Labels 1..K of cell-sized blocks whose grid is shifted by `shift` voxels per axis (every id present)."""
    idx = numpy.indices(shape)
    lab = numpy.zeros(shape, numpy.int64)
    for d, s in enumerate(shape):
        n = (s - 1 + shift[d]) // cell + 1
        lab = lab * n + (idx[d] + shift[d]) // cell
    return (lab + 1).astype(numpy.int32)


def _median_times(arms, reps):
    out = {k: [] for k in arms}
    results = {}
    for k, fn in arms.items():              # warm-up
        results[k] = fn()
    for _ in range(reps):
        for k, fn in arms.items():
            t0 = time.perf_counter()
            results[k] = fn()
            out[k].append(1e3 * (time.perf_counter() - t0))
    return {k: float(numpy.median(v)) for k, v in out.items()}, results


def case_slices(reps):
    import medpy_b200.graphcut as gc
    el = gc.energy_label
    rng = numpy.random.default_rng(0)
    B, S = 512, 512
    labs = [shifted_blocks((S, S), 8, (int(z % 8), int((3 * z) % 8))) for z in range(B)]
    grads = [rng.random((S, S), dtype=numpy.float32) for _ in range(B)]
    yy, xx = numpy.indices((S, S))
    fg = (yy - S // 2) ** 2 + (xx - S // 2) ** 2 <= 30 ** 2
    bg = numpy.zeros((S, S), bool)
    bg[:4], bg[-4:], bg[:, :4], bg[:, -4:] = True, True, True, True

    def batch():
        g = gc.graph_from_labels_batch(labs, [fg] * B, [bg] * B, boundary_term=el.boundary_stawiaski, boundary_term_args=grads)
        g.maxflow()
        return g.label_cut_masks()

    def loop():
        masks = []
        for lab, grad in zip(labs, grads):
            g = gc.graph_from_labels(lab, fg, bg, boundary_term=el.boundary_stawiaski, boundary_term_args=grad)
            g.maxflow()
            masks.append(gc.label_cut_mask(g))
        return masks

    ms, res = _median_times({"batch": batch, "loop": loop}, reps)
    equal = all(numpy.array_equal(a, b) for a, b in zip(res["batch"], res["loop"]))
    regions = sum(int(l.max()) for l in labs)
    return dict(case="512 slices of 512^2, stawiaski", images=B, regions=regions, ms_batch=ms["batch"], ms_loop=ms["loop"],
                speedup=ms["loop"] / ms["batch"], masks_equal=equal)


def case_split(reps):
    import medpy_b200.graphcut as gc
    rng = numpy.random.default_rng(1)
    shape = (256, 256, 256)
    lab = shifted_blocks(shape, 8, (3, 5, 1))
    grad = rng.random(shape, dtype=numpy.float32)
    idx = numpy.indices(shape)
    fg = (idx[0] % 32 == 8) & (idx[1] % 32 == 8) & (idx[2] % 32 == 8)     # seeds in every 74^3 sub-volume
    bg = (idx[0] % 32 == 24) & (idx[1] % 32 == 24) & (idx[2] % 32 == 24)
    del idx
    arms = {k: (lambda b=b: gc.graphcut_split(gc.graphcut_stawiaski, lab, grad, fg, bg, 64, 10, batch=b))
            for k, b in (("batch", True), ("back_to_back", False))}
    ms, res = _median_times(arms, reps)
    return dict(case="graphcut_split of 256^3, minimal_edge_length=64", subvolumes=64, regions=int(lab.max()),
                ms_batch=ms["batch"], ms_back_to_back=ms["back_to_back"], speedup=ms["back_to_back"] / ms["batch"],
                masks_equal=bool(numpy.array_equal(res["batch"], res["back_to_back"])))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cases", default="slices,split")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_labels_batch: no CUDA device (nothing is measured without one)")
    rows = {"card": _card()}
    for c in a.cases.split(","):
        rows[c] = {"slices": case_slices, "split": case_split}[c](a.reps)
        print(json.dumps(rows[c]), flush=True)
    rows["card_after"] = _card()
    print(json.dumps({"card": rows["card"], "card_after": rows["card_after"]}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
