#!/usr/bin/env python
"""BASELINE config 5: 1024^3 fp32 volume, boundary_difference_exponential (sigma = RMS), z-slab partitioned across the
visible GPUs (torchrun) -- or, at a size that fits, on ONE GPU (plain python) as the oracle of the slab runs at the same
size (the reference's int32 ids cannot hold these instances, SURVEY.md §6).  Prints / writes one JSON object: energy
(repr + hex) and the sha256 of every one of the 8 canonical z-slabs of the mask, so an N-GPU run and the 1-GPU run can
be compared without moving the mask.  A single-GPU run needs ~88 B of device memory per voxel: 1024^3 (~94 GB) does
not fit one 80 GB H100, so the single-GPU oracle is run at a smaller --size (768^3 needs ~38 GB), and the slab runs
are compared at that size.

    python tools/run_1024.py --size 768 --out /tmp/c5_768_1gpu.json
    python -m torch.distributed.run --nproc-per-node 8 ... tools/run_1024.py [--size 768] --out /tmp/c5_8gpu.json
"""
import argparse
import hashlib
import json
import os
import sys
import time

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
NSLAB = 8
# solver state 78 (DESIGN.md §3) + lazy build's image copy 4 and marker bit planes 0.25 + resident image 4 + fg 1 + bg 1.
# Config 5 has no probability map; a run with a regional term would add the lazy build's 4 B copy of it.
BYTES_PER_VOXEL = 88.25


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    import torch
    from medpy_b200 import distributed as md, synthetic
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local_rank)
    shape = (args.size,) * 3
    n = args.size ** 3
    res = {"config": "config5 %d^3 difference_exponential" % args.size, "world": world, "shape": list(shape)}
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
        t0 = time.time()
        vol = md.slab_volume(shape, rank, world)
        gen = time.time() - t0
        s = md.SlabSolver(shape, rank=rank, world=world, device=local_rank)
        dev = torch.device("cuda", local_rank)
        d_img = torch.from_numpy(vol["image"]).to(dev)
        d_fg = torch.from_numpy(vol["fg"].view(numpy.uint8)).to(dev)
        d_bg = torch.from_numpy(vol["bg"].view(numpy.uint8)).to(dev)
        times = []
        for rep in range(args.reps):
            torch.cuda.synchronize(); dist.barrier()
            t0 = time.perf_counter()
            s.reset()
            s.add_boundary("difference_exponential", d_img, vol["sigma"], False)
            s.add_markers(d_fg, d_bg)
            s.solve()
            energy = s.energy()
            torch.cuda.synchronize(); dist.barrier()
            times.append(time.perf_counter() - t0)
        mask = s.mask()
        # canonical 8 slabs: with world == 8 each rank owns exactly one
        assert world == NSLAB and mask.shape[0] == args.size // NSLAB
        h = hashlib.sha256(numpy.ascontiguousarray(mask).tobytes()).hexdigest()
        hs = [None] * world
        dist.all_gather_object(hs, h)
        fg = torch.tensor([int(mask.sum())], dtype=torch.int64, device=dev)
        dist.all_reduce(fg)
        res.update(energy=repr(energy), energy_hex=float(energy).hex(), slab_sha256=hs, fg_voxels=int(fg.item()),
                   resident_s=times, mvox_s=n / min(times) / 1e6, gen_s=gen, sigma=vol["sigma"], stats=s.stats,
                   device_bytes=s.handle.stats()["device_bytes"])
        if rank == 0:
            print(json.dumps(res), flush=True)
            if args.out:
                json.dump(res, open(args.out, "w"))
        dist.destroy_process_group()
        return
    # ---- single GPU ----
    free, _ = torch.cuda.mem_get_info()
    if n * BYTES_PER_VOXEL > free:
        raise SystemExit("run_1024.py: %d^3 needs ~%.0f GB of device memory on one GPU, %.0f GB are free; use a smaller --size "
                         "or run it z-slab partitioned over several GPUs" % (args.size, n * BYTES_PER_VOXEL / 1e9, free / 1e9))
    import medpy_b200.graphcut as gc
    from medpy_b200.graphcut.device import graph_from_device_arrays
    t0 = time.time()
    vol = synthetic.two_blob_volume(shape, seed=0, with_prob=False)
    gen = time.time() - t0
    d_img = torch.from_numpy(vol["image"]).cuda()
    d_fg = torch.from_numpy(vol["fg"].view(numpy.uint8)).cuda()
    d_bg = torch.from_numpy(vol["bg"].view(numpy.uint8)).cuda()
    g = None
    times = []
    for rep in range(args.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        g = graph_from_device_arrays(d_fg, d_bg, image=d_img, boundary="difference_exponential", sigma=vol["sigma"], graph=g)
        energy = g.maxflow()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    mask = g.get_mask()
    per = args.size // NSLAB
    hs = [hashlib.sha256(numpy.ascontiguousarray(mask[i * per:(i + 1) * per]).tobytes()).hexdigest() for i in range(NSLAB)]
    st = g.stats()
    res.update(energy=repr(energy), energy_hex=float(energy).hex(), slab_sha256=hs, fg_voxels=int(mask.sum()),
               resident_s=times, mvox_s=n / min(times) / 1e6, gen_s=gen, sigma=vol["sigma"],
               stats={k: st[k] for k in ("push_sweeps", "global_relabels", "relabel_sweeps", "kernel_launches", "ms_terms", "ms_solve",
                                         "ms_push", "ms_relabel", "device_bytes")})
    print(json.dumps(res), flush=True)
    if args.out:
        json.dump(res, open(args.out, "w"))


if __name__ == "__main__":
    main()
