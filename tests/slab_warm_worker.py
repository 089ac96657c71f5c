"""torchrun worker for the multi-GPU warm slab test: every rank builds its slab of the same volume with
SlabSolver(warm=True), the ranks solve it over NCCL (mgc_slab_solve), fold one fg stroke given in global ids and solve it
again; rank 0 writes both energies and both gathered masks."""
import os
import sys

import numpy

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)


def volume(shape):
    from test_gpu_slabs import voxel_case
    return voxel_case(shape, seed=61)


def stroke(shape):
    """A fg stroke through the middle planes, across the slab borders of every partition into up to four slabs."""
    m = numpy.zeros(shape, bool)
    m[shape[0] // 4 - 2: shape[0] * 3 // 4 + 2, 2:5, 2: shape[2] - 2] = True
    return numpy.flatnonzero(m)


def main():
    import torch
    import torch.distributed as dist
    from medpy_b200 import distributed as md
    shape = tuple(int(s) for s in sys.argv[1].split("x"))
    out = sys.argv[2]
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local_rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    c = volume(shape)
    s = md.SlabSolver(shape, warm=True)
    L = s.local_slice
    s.build(L(c["fg"]).view(numpy.uint8), L(c["bg"]).view(numpy.uint8), image_local=L(c["image"]), kind=c["kind"],
            sigma=c["sigma"], prob_local=L(c["prob"]), alpha=c["alpha"])
    res = {}
    for k in range(2):
        if k:
            s.add_seeds(stroke(shape), None)
        s.solve()
        own = torch.from_numpy(numpy.ascontiguousarray(s.mask())).cuda()
        res["energy%d" % k] = s.energy()
        res["mask%d" % k] = md.gather_mask(s, own, shape)
    if dist.get_rank() == 0:
        numpy.savez(out, **res)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
