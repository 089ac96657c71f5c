"""Warm n-link decrements (GraphDouble.remove_nweights_warm / remove_nweights_dense_warm) on a solved graph against a
cold build of the same final graph.

Graphs: those of tools/bench_refine_nweights.py (config3_512, config3_256, config4, config3_eager).
Strokes, each applied to a freshly solved graph:
  unbrush    : the brush of bench_refine_nweights.py (+1 on both arcs of every pair in a ball) added and solved first,
               untimed, then removed with remove_nweights_warm (list form, host arrays);
  lambda_down: dense -kappa * w on every axis, kappa = 0.25, w = exp(-d^2 / sigma^2) computed with torch on the device
               (the lambda stroke of bench_refine_nweights.py with the opposite sign);
  cut_relax  : -50 % of w on both arcs of every pair that crosses the first solve's cut, list form, CUDA tensors.
Per stroke and run: the warm call + maxflow + mask into device memory (wall time, ending in a device synchronise), the call
alone, the fold / relabel / push device times; a cold build of the final graph term by term (regional term, markers and
the final n-link weights w - decrement through add_nweights_dense, w from torch as above, so its weights can differ from
the lazy build's in the last bits); the warm - cold energy and both mask hashes.  Runs alternate warm / cold.  The card
name and power limit are read in the same run.

    python tools/bench_refine_nweights_remove.py [--runs 3] [--graphs ...] [--strokes unbrush,lambda_down,cut_relax]
"""
import argparse
import json
import os
import sys
import time

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_refine import _card, _sha  # noqa: E402
from tools.bench_refine_nweights import _GRAPHS, _make, _setup  # noqa: E402

_STROKES = ("unbrush", "lambda_down", "cut_relax")


def _weights(shape, kind, vol):
    """w[d][p] of the pair p -> p + e_d, float64 on the device (0 on the last plane of d)."""
    import torch
    img = torch.as_tensor(vol["image"]).cuda().to(torch.float64)
    sigma = float(vol["sigma"])
    out = []
    for d in range(len(shape)):
        a, b = img.narrow(d, 0, shape[d] - 1), img.narrow(d, 1, shape[d] - 1)
        x = torch.maximum(a.abs(), b.abs()) if kind.startswith("maximum") else (a - b).abs()
        w = torch.zeros(shape, dtype=torch.float64, device="cuda")
        w.narrow(d, 0, shape[d] - 1).copy_(torch.exp(-(x * x) / (sigma * sigma)))
        out.append(w)
    return out


def _brush(shape):
    from medpy_b200 import synthetic
    nd = len(shape)
    st = [int(numpy.prod(shape[d + 1:])) for d in range(nd)]
    ball = synthetic._ball_mask(shape, (0.3,), 0.05, min_radius=1.0).ravel()
    c = numpy.unravel_index(numpy.arange(ball.size), shape)
    lo = [numpy.flatnonzero(ball & (c[d] + 1 < shape[d]) & numpy.roll(ball, -st[d])) for d in range(nd)]
    return numpy.concatenate(lo), numpy.concatenate([p + st[d] for d, p in enumerate(lo)])


def _cut(shape, mask, w):
    """(lo, hi, w of the pair) for every pair across the cut of `mask` (a device uint8 tensor), on the device."""
    import torch
    nd = len(shape)
    st = [int(numpy.prod(shape[d + 1:])) for d in range(nd)]
    m = mask.reshape(-1)
    lo, hi, ww = [], [], []
    for d in range(nd):
        keep = torch.zeros(shape, dtype=torch.bool, device="cuda")
        keep.narrow(d, 0, shape[d] - 1).fill_(True)
        p = torch.nonzero(keep.reshape(-1)).reshape(-1)
        p = p[m[p] != m[p + st[d]]]
        lo.append(p)
        hi.append(p + st[d])
        ww.append(w[d].reshape(-1)[p])
    return torch.cat(lo), torch.cat(hi), torch.cat(ww)


def _cold(shape, regional, vol, final):
    """The final graph built term by term: regional term, markers, then the final n-link weights."""
    from medpy_b200.graphcut.maxflow import GraphDouble
    g = GraphDouble(int(numpy.prod(shape)), 0, shape=shape)
    if regional:
        g.add_regional_probability(vol["prob"], vol["alpha"], True)
    g.add_markers(vol["fg"], vol["bg"])
    for d, w in enumerate(final):
        g.add_nweights_dense(d, w, w)
    return g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--graphs", default=",".join(_GRAPHS))
    ap.add_argument("--strokes", default=",".join(_STROKES))
    ap.add_argument("--out", default=None, help="also write the rows to this JSON file")
    args = ap.parse_args()
    graphs = [x for x in args.graphs.split(",") if x]
    names = [x for x in args.strokes.split(",") if x]
    if not set(graphs) <= set(_GRAPHS) or not set(names) <= set(_STROKES):
        ap.error("unknown graph or stroke")
    import torch
    card = _card()
    print(json.dumps(card), flush=True)
    out = []
    for gname in graphs:
        shape, kind, regional, env, vol = _setup(gname)
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            nd = len(shape)
            w = _weights(shape, kind, vol)
            lo, hi = _brush(shape)
            d_mask = torch.empty(shape, dtype=torch.uint8, device="cuda")
            d_mask_w = torch.empty(shape, dtype=torch.uint8, device="cuda")
            for sname in names:
                for run in range(args.runs):
                    g = _make(gname, kind, regional, vol)
                    g.maxflow()
                    if sname == "unbrush":
                        g.add_nweights_warm(lo, hi, 1.0, 1.0)
                        g.maxflow()
                    g._nat().get_mask_into(d_mask.data_ptr())
                    torch.cuda.synchronize()
                    if sname == "lambda_down":
                        def call(g):
                            for d in range(nd):
                                g.remove_nweights_dense_warm(d, 0.25 * w[d], 0.25 * w[d])
                        final = [0.75 * x for x in w]
                    elif sname == "cut_relax":
                        ci, cj, cw = _cut(shape, d_mask, w)
                        half = (0.5 * cw).contiguous()

                        def call(g):
                            g.remove_nweights_warm(ci, cj, half, half)
                        final = [x.clone() for x in w]
                        st = [int(numpy.prod(shape[d + 1:])) for d in range(nd)]
                        for d in range(nd):
                            sel = (cj - ci) == st[d]
                            final[d].view(-1)[ci[sel]] -= half[sel]
                    else:
                        def call(g):
                            g.remove_nweights_warm(lo, hi, 1.0, 1.0)
                        final = w
                    torch.cuda.synchronize()
                    s0 = dict(g.stats())
                    t0 = time.perf_counter()
                    call(g)
                    t1 = time.perf_counter()
                    if g.stats()["seed_folds"] <= s0["seed_folds"]:
                        raise SystemExit("stroke {} on {} folded nothing".format(sname, gname))
                    e_warm = g.maxflow()
                    g._nat().get_mask_into(d_mask_w.data_ptr())
                    torch.cuda.synchronize()
                    t2 = time.perf_counter()
                    s1 = g.stats()
                    warm_hash = _sha(d_mask_w.cpu().numpy())
                    del g
                    torch.cuda.synchronize()
                    c0 = time.perf_counter()
                    gc_ = _cold(shape, regional, vol, final)
                    e_cold = gc_.maxflow()
                    gc_._nat().get_mask_into(d_mask.data_ptr())
                    torch.cuda.synchronize()
                    c1 = time.perf_counter()
                    cold_hash = _sha(d_mask.cpu().numpy())
                    differing = int((d_mask_w != d_mask).sum())
                    del gc_
                    d = {k: s1[k] - s0.get(k, 0.0) for k in ("ms_seeds", "ms_seeds_host", "ms_solve", "ms_relabel", "ms_push",
                                                              "ms_caps", "push_sweeps", "global_relabels")}
                    row = dict(graph=gname, shape=list(shape), stroke=sname, run=run,
                               warm_wall_ms_call_to_device_mask=(t2 - t0) * 1e3, call_wall_ms=(t1 - t0) * 1e3,
                               cold_wall_ms_build_to_device_mask=(c1 - c0) * 1e3, masks_equal=warm_hash == cold_hash,
                               differing_voxels=differing, warm_mask_sha=warm_hash, cold_mask_sha=cold_hash,
                               energy_diff=e_warm - e_cold, energy=e_cold, **d, **card)
                    print(json.dumps(row), flush=True)
                    out.append(row)
            del d_mask, d_mask_w, w
            torch.cuda.empty_cache()
        finally:
            for k, v in old.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
