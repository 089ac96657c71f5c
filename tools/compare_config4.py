#!/usr/bin/env python
"""One-off: BASELINE config 4 at FULL size (256x256x128x4, maximum_exponential) -- GPU mask/energy against the BK oracle
port (bit-identical to the reference solver) run on the host.  maximum_* terms give every arc of a locally dominant voxel
the SAME weight, so exact capacity ties are structural; this measures how many voxels' cut membership is decided below
float64 rounding."""
import json, os, sys, time
import numpy
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from medpy_b200 import synthetic
import medpy_b200.graphcut as gc
from oracle import energy_terms as et, solvers

shape = tuple(int(x) for x in (sys.argv[1].split("x") if len(sys.argv) > 1 else "256x256x128x4".split("x")))
vol = synthetic.multispectral_volume(shape, seed=0)
g = gc.graph_from_voxels(vol["fg"], vol["bg"], boundary_term=gc.energy_voxel.boundary_maximum_exponential,
                         boundary_term_args=(vol["image"], vol["sigma"], False))
e = g.maxflow(); m = g.get_mask().copy(); st = g.stats()
del g
t0 = time.time()
prob = et.build_problem(vol["fg"], vol["bg"], boundary=("maximum_exponential", vol["image"], vol["sigma"], False))
t1 = time.time()
oflow, omask, tm = solvers.solve_port(prob)
t2 = time.time()
diff = (m != omask)
out = dict(shape=list(shape), gpu_energy=e, bk_energy=oflow, rel_err=abs(e - oflow) / abs(oflow), mask_hamming=int(diff.sum()),
           gpu_fg=int(m.sum()), bk_fg=int(omask.sum()), bk_terms_s=t1 - t0, bk_setup_s=tm["setup_s"], bk_maxflow_s=tm["maxflow_s"],
           gpu_solve_ms=st["ms_solve"])
if diff.any():
    idx = numpy.argwhere(diff)[:20]
    out["first_diffs"] = idx.tolist()
    # are the differing voxels tie voxels?  cut-energy of both masks with the oracle's weights
    out["cut_energy_gpu_mask"] = et.cut_energy(prob["shape"], prob["wf"], prob["wb"], prob["tr"], prob["flow_const"], m)
    out["cut_energy_bk_mask"] = et.cut_energy(prob["shape"], prob["wf"], prob["wb"], prob["tr"], prob["flow_const"], omask)
print(json.dumps(out), flush=True)
