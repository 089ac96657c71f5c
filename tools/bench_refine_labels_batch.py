"""A stroke on a solved batch of label images, re-solved warm, against a cold rebuild of the batch (DESIGN.md §8, "A batch
of label images", "Warm edits").

The batch is case (a) of tools/bench_labels_batch.py: 512 2-D slices of 512^2 supervoxel maps (8x8 blocks, about 4200
regions per slice, 2.15 M regions in all), a float32 gradient, a foreground disk and a background frame per slice.  Each
round draws a new foreground stroke (a disk of radius 6) on 1 or on 8 of the slices.  Arms:
  warm : region_flags(strokes) + add_seeds on the warm batch, maxflow, label_cut_masks;
  cold : graph_from_labels_batch with every stroke drawn so far added to the foreground markers, maxflow,
         label_cut_masks.
The warm batch is built and solved once before the rounds; both arms are warmed up with one round, then they alternate
for --reps rounds, and the medians of the host-clock spans are reported (each span ends with the masks on the host).
After every round the masks of the two arms must be equal and the energies within 1e-9 relative.  The warm arm is also
split into its parts: flags + fold (the add_seeds calls fold at once), re-solve (with the solver's relabel and push
counts) and masks.  The card's name, power limit and SM clock are read in the same run.

    python tools/bench_refine_labels_batch.py [--reps 5] [--slices 1,8] [--out results/bench_refine_labels_batch.json]
"""
import argparse
import json
import os
import sys
import time

import numpy

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from bench_labels_batch import _card, shifted_blocks  # noqa: E402

B, S = 512, 512


def _inputs():
    rng = numpy.random.default_rng(0)
    labs = [shifted_blocks((S, S), 8, (int(z % 8), int((3 * z) % 8))) for z in range(B)]
    grads = [rng.random((S, S), dtype=numpy.float32) for _ in range(B)]
    yy, xx = numpy.indices((S, S))
    fg = (yy - S // 2) ** 2 + (xx - S // 2) ** 2 <= 30 ** 2
    bg = numpy.zeros((S, S), bool)
    bg[:4], bg[-4:], bg[:, :4], bg[:, -4:] = True, True, True, True
    return labs, grads, fg, bg


def _stroke(r):
    """Round r's stroke: a disk of radius 6 on a ring around the slice's centre, inside the background frame."""
    yy, xx = numpy.indices((S, S))
    a = 0.7 * r
    cy, cx = S // 2 + int(150 * numpy.sin(a)), S // 2 + int(150 * numpy.cos(a))
    return (yy - cy) ** 2 + (xx - cx) ** 2 <= 36


def case(slices, reps):
    import medpy_b200.graphcut as gc
    el = gc.energy_label
    labs, grads, fg, bg = _inputs()
    kw = dict(boundary_term=el.boundary_stawiaski, boundary_term_args=grads)
    edited = [300] if slices == 1 else list(range(30, B, 60))[:slices]
    warm = gc.graph_from_labels_batch(labs, [fg] * B, [bg] * B, warm=True, **kw)
    warm.maxflow()
    fgs = [fg.copy() for _ in range(B)]           # the cold arm's foreground markers: fg and every stroke so far
    parts = {"flags_fold": [], "solve": [], "masks": []}
    counts = {"global_relabels": [], "push_sweeps": []}
    spans = {"warm": [], "cold": []}

    def warm_round(r):
        st0 = warm.stats()
        t0 = time.perf_counter()
        stroke = _stroke(r)
        warm.add_seeds(fg=warm.region_flags([stroke if z in edited else None for z in range(B)]))
        t1 = time.perf_counter()
        e = warm.maxflow()
        t2 = time.perf_counter()
        masks = warm.label_cut_masks()
        t3 = time.perf_counter()
        st1 = warm.stats()
        parts["flags_fold"].append(1e3 * (t1 - t0))
        parts["solve"].append(1e3 * (t2 - t1))
        parts["masks"].append(1e3 * (t3 - t2))
        for k in counts:
            counts[k].append(st1[k] - st0[k])
        return e, masks, 1e3 * (t3 - t0)

    def cold_round(r):
        stroke = _stroke(r)
        for z in edited:
            fgs[z] |= stroke
        t0 = time.perf_counter()
        g = gc.graph_from_labels_batch(labs, fgs, [bg] * B, **kw)
        e = g.maxflow()
        masks = g.label_cut_masks()
        return e, masks, 1e3 * (time.perf_counter() - t0)

    equal, worst = True, 0.0
    for r in range(reps + 1):                       # round 0 warms both arms up
        ew, mw, tw = warm_round(r)
        ec, mc, tc = cold_round(r)
        equal &= all(numpy.array_equal(a, b) for a, b in zip(mw, mc))
        worst = max(worst, float(numpy.max(numpy.abs(ew - ec) / numpy.maximum(numpy.abs(ec), 1e-300))))
        if r:
            spans["warm"].append(tw)
            spans["cold"].append(tc)
    med = {k: float(numpy.median(v)) for k, v in spans.items()}
    return dict(case="stroke on {} of 512 slices of 512^2, stawiaski".format(slices), regions=int(warm.node_offsets[-1]),
                ms_warm=med["warm"], ms_cold=med["cold"], speedup=med["cold"] / med["warm"],
                warm_parts_ms={k: float(numpy.median(v[1:])) for k, v in parts.items()},
                warm_counts={k: float(numpy.median(v[1:])) for k, v in counts.items()},
                masks_equal=bool(equal), max_rel_energy_diff=worst, energies_within_1e9=bool(worst <= 1e-9))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--slices", default="1,8")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_refine_labels_batch: no CUDA device (nothing is measured without one)")
    rows = {"card": _card()}
    for s in a.slices.split(","):
        rows[s] = case(int(s), a.reps)
        print(json.dumps(rows[s]), flush=True)
    rows["card_after"] = _card()
    print(json.dumps({"card": rows["card"], "card_after": rows["card_after"]}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
