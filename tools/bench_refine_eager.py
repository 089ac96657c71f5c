"""Warm re-solves on graphs the lazy fused build does not make, opted in with GraphDouble.enable_warm() before the first
solve (MGC_OPT_WARM), against a cold rebuild of the same graph.

Graphs (host inputs):
  config4      : BASELINE config 4, 256x256x128x4, boundary_maximum_exponential, no regional term (the per-term 4-D path),
  config3_eager: config 3 at 512^3 (regional + difference_exponential) from the eager fused build (MEDPY_GC_LAZY_CAPS=0),
  per_term     : the config 3 energy at 256^3 built term by term (add_regional_probability, add_boundary, add_markers).
Strokes, each applied to a freshly solved graph:
  fg_line       : add_seeds(fg = a line through the background between the two blobs),
  bg_ball       : add_seeds(bg = a ball of semi-axes 0.05 n + 1 inside blob 1; the + 1 keeps it non-empty on the 4-D
                  channel axis of extent 4),
  erase_markers : remove_seeds(fg = the foreground markers of blob 2),
  soft_line     : add_tweights_warm(line ids, 50, 0),
  regional_box  : add_tweights_warm(None, (p' - p) alpha, ((1 - p') - (1 - p)) alpha) inside a box around blob 1, zero
                  outside, p = sigmoid((image - 50) / 15), p' = sigmoid((image - 55) / 15), alpha = 0.1.
Per graph and run: (a) the first solve (maxflow, CUDA events around it) with and without enable_warm(), alternating -- the
cost of the opt-in -- and the wall time of a plain cold rebuild (build + maxflow + mask into device memory, no calls
staged).  Per stroke and run: (b) the warm call + maxflow + mask into device memory (wall time, ending in a device
synchronise), against a cold rebuild (build + the same calls staged + maxflow + mask into device memory); the mask hashes,
which must be equal up to exact ties of the cut (config 4's maximum term has structural ties, tests/test_gpu_fullsize.py),
the number of voxels where they differ, and the warm - cold energy.  Every stroke is checked to make at least one call (an empty call would
fold nothing and measure the cached result).  Ids and weights are computed before the timed call.  Runs alternate warm / cold.  The card name and power limit are read in the
same run.

    python tools/bench_refine_eager.py [--runs 3] [--graphs config4,config3_eager,per_term] [--strokes ...] [--out rows.json]
"""
import argparse
import json
import os
import sys
import time

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_refine import _card, _sha  # noqa: E402

_GRAPHS = ("config4", "config3_eager", "per_term")
_STROKES = ("fg_line", "bg_ball", "erase_markers", "soft_line", "regional_box")


def _setup(name):
    from medpy_b200 import synthetic
    if name == "config4":
        shape, kind, regional, env = (256, 256, 128, 4), "maximum_exponential", False, {}
    elif name == "config3_eager":
        shape, kind, regional, env = (512, 512, 512), "difference_exponential", True, {"MEDPY_GC_LAZY_CAPS": "0"}
    else:
        shape, kind, regional, env = (256, 256, 256), "difference_exponential", True, {}
    vol = synthetic.two_blob_volume(shape, seed=0, with_prob=regional)
    return shape, kind, regional, env, vol


def _make(name, shape, kind, regional, vol):
    import medpy_b200.graphcut as gc
    from medpy_b200.graphcut.maxflow import GraphDouble
    if name == "per_term":
        g = GraphDouble(int(numpy.prod(shape)), 0, shape=shape)
        g.add_regional_probability(vol["prob"], vol["alpha"], True)
        g.add_boundary(1, vol["image"], vol["sigma"], None, float("nan"))
        g.add_markers(vol["fg"], vol["bg"])
        g._flush()
        return g
    kw = dict(boundary_term=getattr(gc.energy_voxel, "boundary_" + kind), boundary_term_args=(vol["image"], vol["sigma"], False))
    if regional:
        kw.update(regional_term=gc.energy_voxel.regional_probability_map, regional_term_args=(vol["prob"], vol["alpha"]))
    return gc.graph_from_voxels(vol["fg"], vol["bg"], **kw)


def _strokes(shape, vol):
    from medpy_b200 import synthetic
    line = numpy.zeros(shape, bool)
    line[tuple(s // 2 for s in shape[:-1]) + (slice(int(0.4 * shape[-1]), int(0.6 * shape[-1])),)] = True
    ball = synthetic._ball_mask(shape, (0.3,), 0.05, min_radius=1.0)
    blob2 = vol["fg"] & synthetic._ball_mask(shape, (0.7,), 0.09, min_radius=0.5)
    img = vol["image"].astype(numpy.float64)
    p = 1.0 / (1.0 + numpy.exp(-(img - 50.0) / 15.0))
    p2 = 1.0 / (1.0 + numpy.exp(-(img - 55.0) / 15.0))
    keep = numpy.zeros(shape, bool)
    keep[tuple(slice(int(0.15 * s), max(int(0.45 * s), int(0.15 * s) + 1)) for s in shape)] = True
    src, snk = numpy.where(keep, (p2 - p) * 0.1, 0.0), numpy.where(keep, ((1.0 - p2) - (1.0 - p)) * 0.1, 0.0)
    line_ids, ball_ids, blob2_ids = numpy.flatnonzero(line), numpy.flatnonzero(ball), numpy.flatnonzero(blob2)
    for what, ids in (("line", line_ids), ("ball", ball_ids), ("blob 2 markers", blob2_ids)):
        if ids.size == 0:
            raise SystemExit("the {} of shape {} is empty: the stroke would fold nothing".format(what, shape))
    if not (src.any() or snk.any()):
        raise SystemExit("the regional box delta of shape {} is zero: the stroke would fold nothing".format(shape))
    return {"fg_line": lambda g: g.add_seeds(fg=line_ids),
            "bg_ball": lambda g: g.add_seeds(bg=ball_ids),
            "erase_markers": lambda g: g.remove_seeds(fg=blob2_ids),
            "soft_line": lambda g: g.add_tweights_warm(line_ids, 50.0, 0.0),
            "regional_box": lambda g: g.add_tweights_warm(None, src, snk)}


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
    stream = torch.cuda.current_stream()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for gname in graphs:
        shape, kind, regional, env, vol = _setup(gname)
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            d_mask = torch.empty(shape, dtype=torch.uint8, device="cuda")
            d_mask_w = torch.empty(shape, dtype=torch.uint8, device="cuda")
            # (a) the first solve with and without the opt-in, alternating
            for run in range(args.runs):
                for warm in (False, True):
                    g = _make(gname, shape, kind, regional, vol)
                    if warm:
                        g.enable_warm()
                    g._flush()
                    torch.cuda.synchronize()
                    ev0.record(stream)
                    e = g.maxflow()
                    ev1.record(stream)
                    torch.cuda.synchronize()
                    row = dict(graph=gname, shape=list(shape), part="first_solve", warm=warm, run=run,
                               solve_ms=ev0.elapsed_time(ev1), energy_hex=float(e).hex(), mask_sha=_sha(g.get_mask()),
                               ms_init=g.stats()["ms_init"], **card)
                    print(json.dumps(row), flush=True)
                    out.append(row)
                    del g
                # the plain cold rebuild: build + solve + mask into device memory, nothing staged
                torch.cuda.synchronize()
                c0 = time.perf_counter()
                g = _make(gname, shape, kind, regional, vol)
                e = g.maxflow()
                g._nat().get_mask_into(d_mask.data_ptr())
                torch.cuda.synchronize()
                row = dict(graph=gname, shape=list(shape), part="cold_plain", run=run,
                           cold_wall_ms_build_to_device_mask=(time.perf_counter() - c0) * 1e3, **card)
                print(json.dumps(row), flush=True)
                out.append(row)
                del g
            # (b) warm stroke against a cold rebuild with the same calls staged
            strokes = _strokes(shape, vol)
            for sname in names:
                for run in range(args.runs):
                    g = _make(gname, shape, kind, regional, vol)
                    g.enable_warm()
                    g.maxflow()
                    torch.cuda.synchronize()
                    s0 = dict(g.stats())
                    t0 = time.perf_counter()
                    strokes[sname](g)
                    t1 = time.perf_counter()
                    s_mid = g.stats()
                    if s_mid["seed_folds"] != s0["seed_folds"] + 1:
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
                    gc_ = _make(gname, shape, kind, regional, vol)
                    strokes[sname](gc_)
                    e_cold = gc_.maxflow()
                    gc_._nat().get_mask_into(d_mask.data_ptr())
                    torch.cuda.synchronize()
                    c1 = time.perf_counter()
                    cold_hash = _sha(d_mask.cpu().numpy())
                    differing = int((d_mask_w != d_mask).sum())
                    del gc_
                    d = {k: s1[k] - s0.get(k, 0.0) for k in ("ms_seeds", "ms_seeds_host", "ms_solve", "ms_relabel", "ms_push",
                                                              "ms_readout", "push_sweeps", "global_relabels")}
                    row = dict(graph=gname, shape=list(shape), part="stroke", stroke=sname, run=run,
                               call_wall_ms=(t1 - t0) * 1e3, warm_wall_ms_call_to_device_mask=(t2 - t0) * 1e3,
                               cold_wall_ms_build_to_device_mask=(c1 - c0) * 1e3, masks_equal=warm_hash == cold_hash, differing_voxels=differing,
                               warm_mask_sha=warm_hash, energy_diff=e_warm - e_cold, energy=e_cold, **d, **card)
                    print(json.dumps(row), flush=True)
                    out.append(row)
            del d_mask, d_mask_w
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
