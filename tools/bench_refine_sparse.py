"""Warm re-solves of general sparse graphs against today's cold re-solve.

Two graphs: the region graph of a 256^3 label volume with about 10^5 regions and a Stawiaski boundary term
(graph_from_labels), and a random general graph with 10^6 nodes (GraphDouble(sparse=True)).  Each round applies the same
calls to (a) a graph made without warm=True, whose next maxflow() solves from nothing, and (b) a graph made with
warm=True, whose next maxflow() continues from its residual state: a seed stroke, t-link updates and an edge brush.  The
two arms alternate; every time is the wall time of the calls plus maxflow() plus get_mask() (the native calls return
after their device work).  Masks must be equal and energies agree to 1e-9 relative.

    python tools/bench_refine_sparse.py [--rounds 4] [--graphs region,random] [--nodes 1000000]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def label_volume(side=256, cell=5.5, seed=1):
    """Jittered cubic cells: about (side / cell)^3 regions numbered 1..K."""
    rng = numpy.random.default_rng(seed)
    idx = numpy.indices((side,) * 3, dtype=numpy.int32)
    ncell = int(numpy.ceil(side / cell)) + 1
    key = numpy.zeros((side,) * 3, numpy.int64)
    for g in idx:
        key = key * ncell + ((g + rng.integers(-1, 2, size=g.shape)).clip(0, side - 1) / cell).astype(numpy.int64)
    _, inv = numpy.unique(key.ravel(), return_inverse=True)
    return (inv + 1).reshape(key.shape).astype(numpy.int32)


def region_graphs(args):
    import medpy_b200.graphcut as gc
    from medpy_b200.graphcut import energy_label
    lab = label_volume()
    rng = numpy.random.default_rng(2)
    grad = numpy.abs(rng.normal(0, 10, size=lab.shape))
    fg = numpy.zeros(lab.shape, bool)
    bg = numpy.zeros(lab.shape, bool)
    fg[100:140, 100:140, 100:140] = True
    bg[:, :, -1] = True
    kw = dict(boundary_term=energy_label.boundary_stawiaski, boundary_term_args=grad)
    cold = gc.graph_from_labels(lab, fg, bg, **kw)
    warm = gc.graph_from_labels(lab, fg, bg, warm=True, **kw)
    return cold, warm, int(lab.max())


def random_graphs(args):
    from medpy_b200.graphcut.maxflow import GraphDouble
    rng = numpy.random.default_rng(3)
    n = args.nodes
    i = rng.integers(0, n, size=3 * n)
    j = (i + rng.integers(1, 1000, size=i.size)) % n
    cap, rev = rng.uniform(0.1, 2.0, size=i.size), rng.uniform(0.1, 2.0, size=i.size)
    src, snk = rng.uniform(0, 3, size=n), rng.uniform(0, 3, size=n)
    out = []
    for warm in (False, True):
        g = GraphDouble(n, i.size, sparse=True, warm=warm)
        g.add_tweights_bulk(None, src, snk)
        g.sum_edges_bulk(i, j, cap, rev)
        out.append(g)
    return out[0], out[1], n


def rounds(cold, warm, n, args, name):
    rng = numpy.random.default_rng(4)
    t0 = time.perf_counter()
    ec, ew = cold.maxflow(), warm.maxflow()
    print(json.dumps(dict(graph=name, step="first solve", nodes=n, s=round(time.perf_counter() - t0, 3),
                          energy_diff=ew - ec)), flush=True)
    for r in range(args.rounds):
        fg = rng.choice(n, size=50, replace=False)
        bg = rng.choice(n, size=50, replace=False)
        tv = rng.choice(n, size=max(1, n // 100), replace=False)
        ts, tt = rng.uniform(0, 2, size=tv.size), rng.uniform(0, 2, size=tv.size)
        lo = rng.integers(0, n, size=200)
        hi = (lo + 1 + rng.integers(0, 50, size=lo.size)) % n
        keep = lo != hi
        lo, hi = lo[keep], hi[keep]
        w = rng.uniform(0.5, 2.0, size=lo.size)
        res = {}
        for arm, g in (("cold", cold), ("warm", warm)):
            t = time.perf_counter()
            for ids, s, k in ((fg, 65535.0, 0.0), (bg, 0.0, 65535.0)):
                g.add_tweights_bulk(ids, numpy.full(ids.size, s), numpy.full(ids.size, k))
            g.add_tweights_bulk(tv, ts, tt)
            g.sum_edges_bulk(lo, hi, w, w)
            e = g.maxflow()
            m = g.get_mask()
            res[arm] = (time.perf_counter() - t, e, m)
        (tc, e_c, m_c), (tw, e_w, m_w) = res["cold"], res["warm"]
        ok = bool(numpy.array_equal(m_c, m_w)) and abs(e_w - e_c) <= 1e-9 * max(abs(e_c), 1.0)
        print(json.dumps(dict(graph=name, round=r, cold_ms=round(1e3 * tc, 2), warm_ms=round(1e3 * tw, 2),
                              energy=e_c, energy_diff=e_w - e_c, same=ok,
                              warm_solve_ms=round(warm.stats()["ms_solve"], 2))), flush=True)
        if not ok:
            raise SystemExit("warm and cold disagree")


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--graphs", default="region,random")
    ap.add_argument("--nodes", type=int, default=1_000_000)
    args = ap.parse_args()
    print(json.dumps(dict(card=card())), flush=True)
    for name in args.graphs.split(","):
        cold, warm, n = (region_graphs if name == "region" else random_graphs)(args)
        rounds(cold, warm, n, args, name)


if __name__ == "__main__":
    main()
