"""A correction stroke on z-slab handles, re-solved warm (MGC_OPT_WARM, mgc_add_seeds into the solved slabs), against a
cold slab rebuild + solve of the graph with the stroke.

Two transports:
  one process (default): N slab handles of one lattice on cuda:0, stepped with the sequence of mgc_slab_solve and border
      messages moved by device copies (the driver of tests/test_gpu_slabs.py).  This is NOT representative of the NCCL
      transport: every exchange here is a host-synchronised device copy, and the N slabs share one GPU, so the times
      show the warm / cold ratio of the slab path, not multi-GPU times;
  under torchrun with >= 2 GPUs: one slab per GPU, medpy_b200.distributed.SlabSolver(warm=True), mgc_slab_solve over NCCL.
Graph: the two-blob volume of bench.py (regional + difference_exponential, fused slab build from device tensors).
Strokes: fg_line (add_seeds: a line through the background between the blobs, across every slab border) and bg_ball
(add_seeds: bg = a ball inside blob 1).  Per run: the graph is rebuilt and solved (untimed), then the stroke warm (fold +
solve + masks, wall time ending in a device synchronise; the one-GPU driver also reads the masks back to the host, in both
arms); then a cold run (reset + build with the stroke in the markers + solve + masks).  Warm and cold masks and energies
are compared.  The card name and power limit are read in the same run; anything not run is reported as not measured.

    python tools/bench_refine_slab.py [--shape 512,512,512] [--slabs 2,4] [--runs 3] [--out rows.json]
    torchrun --nproc-per-node N tools/bench_refine_slab.py --shape 512,512,512 [--runs 3]
"""
import argparse
import json
import os
import sys
import time

import numpy

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _volume(shape):
    from medpy_b200 import synthetic
    return synthetic.two_blob_volume(shape, seed=0, with_prob=True)


def _strokes(shape, vol):
    Z, Y, X = shape
    line = numpy.zeros(shape, bool)
    line[Z // 8: Z - Z // 8, Y // 2, X // 2] = True
    line &= ~vol["fg"] & ~vol["bg"]
    z, y, x = numpy.ogrid[:Z, :Y, :X]
    r = max(2, (3 * Z) // 100)
    # blob 1 of synthetic.two_blob_volume: centre 0.3 of every extent, radius 0.18, fg markers within 0.09 of the centre;
    # the ball lies between the two, 0.13 off the centre along the last axis
    ball = (z - int(0.3 * Z)) ** 2 + (y - int(0.3 * Y)) ** 2 + (x - int(0.43 * X)) ** 2 <= r * r
    ball &= ~vol["fg"] & ~vol["bg"]
    return {"fg_line": (line, None), "bg_ball": (None, ball)}


def _sync():
    import torch
    torch.cuda.synchronize()


def one_gpu(shape, n, runs, card):
    import torch
    from medpy_b200 import _lib
    from medpy_b200.distributed import KINDS, slab_bounds
    from test_gpu_slabs import Slabs
    vol = _volume(shape)
    bounds = [slab_bounds(shape[0], n, r) for r in range(n)]
    s = Slabs(shape, bounds)
    for h in s.hs:
        h.set_option(_lib._mgc.OPT_WARM, 1)
    dev = lambda a: None if a is None else torch.from_numpy(numpy.ascontiguousarray(a)).cuda()  # noqa: E731
    loc = [[dev(s.local(a, r)) for a in (vol["prob"], vol["image"])] for r in range(n)]
    d_mask = torch.empty(shape, dtype=torch.uint8, device="cuda")
    P = int(numpy.prod(shape[1:]))

    def build(fg, bg):
        for r, h in enumerate(s.hs):
            h.reset()
            p, img = loc[r]
            h.build_voxel_graph(p, float(vol["alpha"]), True, KINDS["difference_exponential"], img, float(vol["sigma"]),
                                None, float("nan"), dev(s.local(fg, r).view(numpy.uint8)), dev(s.local(bg, r).view(numpy.uint8)))

    def solve():
        s.solve("native")
        for (a, b), h in zip(bounds, s.hs):
            h.get_mask_into(d_mask[a:b].data_ptr())
        _sync()
        return s.energy, d_mask.cpu().numpy()

    rows = []
    for name, (fg_add, bg_add) in _strokes(shape, vol).items():
        ids = [None if m is None else numpy.flatnonzero(m) for m in (fg_add, bg_add)]
        local = []
        for r in range(n):
            a = bounds[r][0] - (1 if bounds[r][0] > 0 else 0)
            b = bounds[r][1] + (1 if bounds[r][1] < shape[0] else 0)
            local.append([None if x is None else numpy.ascontiguousarray(x[(x >= a * P) & (x < b * P)] - a * P) for x in ids])
        fg2 = vol["fg"] | (fg_add if fg_add is not None else False)
        bg2 = vol["bg"] | (bg_add if bg_add is not None else False)
        warm_ms, cold_ms, same = [], [], []
        for _ in range(runs):
            build(vol["fg"], vol["bg"])
            solve()
            t0 = time.perf_counter()
            for h, (f, g) in zip(s.hs, local):
                h.add_seeds(f, g)
            ew, mw = solve()
            warm_ms.append(1e3 * (time.perf_counter() - t0))
            t0 = time.perf_counter()
            build(fg2, bg2)
            ec, mc = solve()
            cold_ms.append(1e3 * (time.perf_counter() - t0))
            same.append(bool(numpy.array_equal(mw, mc)) and abs(ew - ec) <= 1e-9 * abs(ec))
        rows.append(dict(transport="one GPU, %d slab handles, device-copy exchanges (not the NCCL transport)" % n,
                         shape=list(shape), slabs=n, stroke=name, voxels=int(sum(0 if x is None else x.size for x in ids)),
                         warm_ms=[round(x, 2) for x in warm_ms], cold_ms=[round(x, 2) for x in cold_ms],
                         warm_equals_cold=all(same), **card))
    return rows


def nccl(shape, runs, card):
    import torch
    import torch.distributed as dist
    from medpy_b200 import distributed as md
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local_rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    vol = _volume(shape)
    s = md.SlabSolver(shape, warm=True)
    L = lambda a: torch.from_numpy(numpy.ascontiguousarray(s.local_slice(a))).cuda()  # noqa: E731

    def build(fg, bg):
        s.reset()
        s.build(L(fg.view(numpy.uint8)), L(bg.view(numpy.uint8)), image_local=L(vol["image"]), kind="difference_exponential",
                sigma=vol["sigma"], prob_local=L(vol["prob"]), alpha=vol["alpha"])

    def solve():
        s.solve()
        torch.cuda.synchronize()
        return s.energy(), s.mask()

    rows = []
    for name, (fg_add, bg_add) in _strokes(shape, vol).items():
        fg2 = vol["fg"] | (fg_add if fg_add is not None else False)
        bg2 = vol["bg"] | (bg_add if bg_add is not None else False)
        warm_ms, cold_ms, same = [], [], []
        for _ in range(runs):
            build(vol["fg"], vol["bg"])
            solve()
            dist.barrier()
            t0 = time.perf_counter()
            s.add_seeds(fg_add, bg_add)
            ew, mw = solve()
            dist.barrier()
            warm_ms.append(1e3 * (time.perf_counter() - t0))
            t0 = time.perf_counter()
            build(fg2, bg2)
            ec, mc = solve()
            dist.barrier()
            cold_ms.append(1e3 * (time.perf_counter() - t0))
            same.append(bool(numpy.array_equal(mw, mc)) and abs(ew - ec) <= 1e-9 * abs(ec))
        ok = torch.tensor([int(all(same))], device="cuda")
        dist.all_reduce(ok, op=dist.ReduceOp.MIN)
        rows.append(dict(transport="NCCL, %d GPUs, mgc_slab_solve" % s.world, shape=list(shape), slabs=s.world, stroke=name,
                         warm_ms=[round(x, 2) for x in warm_ms], cold_ms=[round(x, 2) for x in cold_ms],
                         warm_equals_cold=bool(ok.item()), **card))
    rank = dist.get_rank()
    dist.destroy_process_group()
    return rows if rank == 0 else []


def main():
    from tools.bench_refine import _card
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="512,512,512")
    ap.add_argument("--slabs", default="2,4")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    shape = tuple(int(x) for x in args.shape.split(","))
    card = _card()
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        rows = nccl(shape, args.runs, card)
    else:
        rows = [r for n in (int(x) for x in args.slabs.split(",")) for r in one_gpu(shape, n, args.runs, card)]
        rows.append(dict(transport="NCCL", measured=False, note="not measured: run under torchrun with >= 2 GPUs"))
    for r in rows:
        print(json.dumps(r))
    if args.out and rows:
        with open(args.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
