"""Warm n-link edits (GraphDouble.add_nweights_warm / add_nweights_dense_warm) on a solved graph against a cold rebuild.

Graphs (host inputs):
  config3_512  : config 3 at 512^3 (regional + difference_exponential), lazy fused build,
  config3_256  : the same energy at 256^3, lazy fused build,
  config4      : BASELINE config 4, 256x256x128x4, boundary_maximum_exponential, enable_warm(),
  config3_eager: config 3 at 512^3 from the eager fused build (MEDPY_GC_LAZY_CAPS=0), enable_warm().
Strokes, each applied to a freshly solved graph:
  brush  : list form, +w (w = 1) on both arcs of every lattice-neighbour pair inside a ball of radius 0.05 n around blob 1,
  box    : dense form along axis 0, 1.0 inside a box around blob 1, zero outside, as host (numpy) arrays,
  box_device: the same box as CUDA tensors, so that box - box_device is what the host arrays cost,
  lambda : dense kappa * w on every axis, kappa = 0.25, w = exp(-d^2 / sigma^2) (d = the image difference, or the larger
           magnitude for the maximum term) computed from the image with torch on the device.
Per stroke and run: the warm call + maxflow + mask into device memory (wall time, ending in a device synchronise), the call
alone (wall time up to its return), the relabel and push device times of the solve; a cold rebuild with the same
increments staged; a plain rebuild without them; the warm - cold energy and both mask hashes.  Every stroke must fold something.  Runs alternate warm / cold.  The card name
and power limit are read in the same run.

    python tools/bench_refine_nweights.py [--runs 3] [--graphs ...] [--strokes brush,box,box_device,lambda] [--out rows.json]
"""
import argparse
import json
import os
import sys
import time

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_refine import _card, _sha  # noqa: E402

_GRAPHS = ("config3_512", "config3_256", "config4", "config3_eager")
_STROKES = ("brush", "box", "box_device", "lambda")


def _setup(name):
    from medpy_b200 import synthetic
    if name == "config4":
        shape, kind, regional, env = (256, 256, 128, 4), "maximum_exponential", False, {}
    elif name == "config3_256":
        shape, kind, regional, env = (256, 256, 256), "difference_exponential", True, {}
    else:
        shape, kind, regional = (512, 512, 512), "difference_exponential", True
        env = {"MEDPY_GC_LAZY_CAPS": "0"} if name == "config3_eager" else {}
    vol = synthetic.two_blob_volume(shape, seed=0, with_prob=regional)
    return shape, kind, regional, env, vol


def _make(name, kind, regional, vol):
    import medpy_b200.graphcut as gc
    kw = dict(boundary_term=getattr(gc.energy_voxel, "boundary_" + kind), boundary_term_args=(vol["image"], vol["sigma"], False))
    if regional:
        kw.update(regional_term=gc.energy_voxel.regional_probability_map, regional_term_args=(vol["prob"], vol["alpha"]))
    g = gc.graph_from_voxels(vol["fg"], vol["bg"], **kw)
    if name in ("config4", "config3_eager"):
        g.enable_warm()
    return g


def _strokes(shape, kind, vol):
    import torch
    from medpy_b200 import synthetic
    nd = len(shape)
    st = [int(numpy.prod(shape[d + 1:])) for d in range(nd)]
    ball = synthetic._ball_mask(shape, (0.3,), 0.05, min_radius=1.0).ravel()
    c = numpy.unravel_index(numpy.arange(ball.size), shape)
    lo = numpy.concatenate([numpy.flatnonzero(ball & (c[d] + 1 < shape[d]) & numpy.roll(ball, -st[d])) for d in range(nd)])
    hi = numpy.concatenate([numpy.flatnonzero(ball & (c[d] + 1 < shape[d]) & numpy.roll(ball, -st[d])) + st[d]
                            for d in range(nd)])
    del c
    box = numpy.zeros(shape)
    box[tuple(slice(int(0.15 * s), max(int(0.45 * s), int(0.15 * s) + 1)) for s in shape)] = 1.0
    d_box = torch.from_numpy(box).cuda()
    img = torch.as_tensor(vol["image"]).cuda().to(torch.float64)
    sigma = float(vol["sigma"])
    lam = []
    for d in range(nd):
        a = img.narrow(d, 0, shape[d] - 1)
        b = img.narrow(d, 1, shape[d] - 1)
        x = torch.maximum(a.abs(), b.abs()) if kind.startswith("maximum") else (a - b).abs()
        w = torch.zeros(shape, dtype=torch.float64, device="cuda")
        w.narrow(d, 0, shape[d] - 1).copy_(0.25 * torch.exp(-(x * x) / (sigma * sigma)))
        lam.append(w)
    del img
    if lo.size == 0:
        raise SystemExit("the brush of shape {} is empty: the stroke would fold nothing".format(shape))
    return {"brush": lambda g: g.add_nweights_warm(lo, hi, 1.0, 1.0),
            "box": lambda g: g.add_nweights_dense_warm(0, box, box),
            "box_device": lambda g: g.add_nweights_dense_warm(0, d_box, d_box),
            "lambda": lambda g: [g.add_nweights_dense_warm(d, lam[d], lam[d]) for d in range(nd)]}


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
            d_mask = torch.empty(shape, dtype=torch.uint8, device="cuda")
            d_mask_w = torch.empty(shape, dtype=torch.uint8, device="cuda")
            strokes = _strokes(shape, kind, vol)
            for sname in names:
                for run in range(args.runs):
                    g = _make(gname, kind, regional, vol)
                    g.maxflow()
                    torch.cuda.synchronize()
                    s0 = dict(g.stats())
                    t0 = time.perf_counter()
                    strokes[sname](g)
                    t1 = time.perf_counter()
                    s_mid = g.stats()
                    if s_mid["seed_folds"] <= s0["seed_folds"]:
                        raise SystemExit("stroke {} on {} folded nothing".format(sname, gname))
                    e_warm = g.maxflow()
                    g._nat().get_mask_into(d_mask_w.data_ptr())
                    torch.cuda.synchronize()
                    t2 = time.perf_counter()
                    s1 = g.stats()
                    warm_hash = _sha(d_mask_w.cpu().numpy())
                    del g
                    # cold: the same increments staged before the first solve
                    torch.cuda.synchronize()
                    c0 = time.perf_counter()
                    gc_ = _make(gname, kind, regional, vol)
                    strokes[sname](gc_)
                    e_cold = gc_.maxflow()
                    gc_._nat().get_mask_into(d_mask.data_ptr())
                    torch.cuda.synchronize()
                    c1 = time.perf_counter()
                    cold_hash = _sha(d_mask.cpu().numpy())
                    differing = int((d_mask_w != d_mask).sum())
                    del gc_
                    # plain rebuild, nothing staged
                    torch.cuda.synchronize()
                    p0 = time.perf_counter()
                    gp = _make(gname, kind, regional, vol)
                    gp.maxflow()
                    gp._nat().get_mask_into(d_mask.data_ptr())
                    torch.cuda.synchronize()
                    p1 = time.perf_counter()
                    del gp
                    d = {k: s1[k] - s0.get(k, 0.0) for k in ("ms_seeds", "ms_seeds_host", "ms_solve", "ms_relabel", "ms_push",
                                                              "ms_caps", "push_sweeps", "global_relabels")}
                    row = dict(graph=gname, shape=list(shape), stroke=sname, run=run,
                               warm_wall_ms_call_to_device_mask=(t2 - t0) * 1e3, call_wall_ms=(t1 - t0) * 1e3,
                               cold_wall_ms_build_to_device_mask=(c1 - c0) * 1e3,
                               plain_rebuild_wall_ms=(p1 - p0) * 1e3, masks_equal=warm_hash == cold_hash,
                               differing_voxels=differing, warm_mask_sha=warm_hash, cold_mask_sha=cold_hash,
                               energy_diff=e_warm - e_cold, energy=e_cold, **d, **card)
                    print(json.dumps(row), flush=True)
                    out.append(row)
            del d_mask, d_mask_w, strokes
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
