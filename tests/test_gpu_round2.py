"""GPU tests of the round-2 kernels against each other and the oracle: the fused single-pass build (gc_build.cuh) must
leave exactly the graph the per-term kernels leave; the chunked upload, the TMA / plain image staging, the bit-packed
markers and the directional-sweep global relabel (gc_sweep.cuh) must not change any result; a solved graph refuses new
terms (ADVICE r1: re-solving on residual capacities gave silently wrong energies)."""
import os

import numpy
import pytest

pytestmark = pytest.mark.gpu


def _gc():
    import medpy_b200.graphcut as gc
    return gc


class _env:
    def __init__(self, **kw):
        self.kw = kw

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in self.kw}
        for k, v in self.kw.items():
            os.environ[k] = str(v)

    def __exit__(self, *a):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _build(vol, kind="difference_exponential", regional=True, spacing=False, image=None):
    gc = _gc()
    img = vol["image"] if image is None else image
    kw = dict(boundary_term=getattr(gc.energy_voxel, "boundary_" + kind))
    kw["boundary_term_args"] = (img, spacing) if kind.endswith("linear") else (img, vol["sigma"], spacing)
    if regional:
        kw.update(regional_term=gc.energy_voxel.regional_probability_map, regional_term_args=(vol["prob"], vol["alpha"]))
    return gc.graph_from_voxels(vol["fg"], vol["bg"], **kw)


def _snapshot(g, shape, count=4000, seed=0):
    """t-links and n-links of a random sample of voxels (all of them for small lattices)."""
    n = int(numpy.prod(shape))
    rng = numpy.random.default_rng(seed)
    ids = numpy.arange(n) if n <= count else rng.choice(n, size=count, replace=False)
    strides = [int(numpy.prod(shape[d + 1:])) for d in range(len(shape))]
    tr = numpy.asarray([g.get_trcap(int(p)) for p in ids])
    w = []
    for p in ids:
        p = int(p)
        for d, st in enumerate(strides):
            if (p // st) % shape[d] < shape[d] - 1:
                w.append(g.get_edge(p, p + st))
                w.append(g.get_edge(p + st, p))
    return tr, numpy.asarray(w)


@pytest.mark.parametrize("shape,kind,regional,spacing,dtype", [
    ((24, 28, 32), "difference_exponential", True, False, numpy.float32),      # TMA path (X % 4 == 0)
    ((17, 9, 45), "difference_exponential", True, False, numpy.float32),       # plain staging (odd X), ragged blocks
    ((9, 33, 64), "maximum_exponential", False, False, numpy.float32),
    ((12, 20, 40), "difference_division", True, (1.5, 0.5, 2.0), numpy.float64),
    ((16, 16, 48), "difference_linear", False, False, numpy.float32),
    ((10, 12, 16), "maximum_power", True, False, numpy.int16),
    ((6, 10, 80), "maximum_power", False, False, numpy.int16),                 # several x blocks, 2-byte elements (TMA box pad 8)
    ((8, 9, 96), "difference_division", False, False, numpy.uint8),            # 1-byte elements (TMA box pad 16)
    ((5, 18, 72), "difference_exponential", True, False, numpy.float64),
    ((8, 8, 104), "difference_linear", False, False, numpy.int32),
    ((7, 40), "difference_exponential", True, False, numpy.float32),           # 2-D input on the 3-D kernels
    ((1, 50), "difference_exponential", False, False, numpy.float32),
])
def test_fused_build_equals_per_term_kernels(shape, kind, regional, spacing, dtype):
    from medpy_b200 import synthetic
    vol = synthetic.two_blob_volume(shape, seed=3)
    img = vol["image"]
    if dtype == numpy.uint8:
        img = numpy.clip(numpy.round(img + 60.0), 0, 255).astype(dtype)
    elif numpy.issubdtype(dtype, numpy.integer):
        img = numpy.round(img).astype(dtype)
    else:
        img = img.astype(dtype)
    results = []
    for env in (dict(MEDPY_GC_FUSE=1), dict(MEDPY_GC_FUSE=0), dict(MEDPY_GC_FUSE=1, MEDPY_GC_CHUNKS=1),
                dict(MEDPY_GC_FUSE=1, MEDPY_GC_BUILD_TMA=0)):
        with _env(**env):
            g = _build(vol, kind, regional, spacing, image=img)
            tr, w = _snapshot(g, shape)
            flow = g.maxflow()
            results.append((tr, w, flow, g.get_mask(), g.stats()))
    tr0, w0, flow0, mask0, st0 = results[0]
    for tr, w, flow, mask, st in results[1:]:
        assert numpy.array_equal(tr, tr0)
        assert numpy.array_equal(w, w0, equal_nan=True)
        assert numpy.array_equal(mask, mask0)
        assert abs(flow - flow0) <= 1e-12 * max(1.0, abs(flow0))
    # the fused path really ran as one pass (no k_init_tile), the MEDPY_GC_FUSE=0 path as separate passes
    assert st0["ms_init"] == 0.0 and results[1][4]["ms_init"] > 0.0


def test_fused_build_vs_oracle_weights_and_tlinks():
    """The fused kernel against the numpy restatement of the reference's terms: t-links bit-exact, exp weights within 2e-13."""
    from medpy_b200 import synthetic
    from oracle import energy_terms as et
    shape = (12, 16, 36)
    vol = synthetic.two_blob_volume(shape, seed=7)
    g = _build(vol)
    prob = et.build_problem(vol["fg"], vol["bg"], regional=(vol["prob"], vol["alpha"]),
                            boundary=("difference_exponential", vol["image"], vol["sigma"], False))
    n = int(numpy.prod(shape))
    tr = numpy.asarray([g.get_trcap(p) for p in range(n)])
    assert numpy.array_equal(tr, prob["tr"])
    strides = [shape[1] * shape[2], shape[2], 1]
    for d, st in enumerate(strides):
        ids = [p for p in range(n) if (p // st) % shape[d] < shape[d] - 1][::7]
        w = numpy.asarray([g.get_edge(p, p + st) for p in ids])
        numpy.testing.assert_allclose(w, prob["wf"][d][ids], rtol=2e-13, atol=0)   # exp argument rounding: <= |arg| * 1.1e-16
        assert numpy.array_equal(w, numpy.asarray([g.get_edge(p + st, p) for p in ids]))
    oflow, omask, _ = __import__("oracle.solvers", fromlist=["x"]).solve_port(prob)
    assert numpy.array_equal(g.get_mask(), omask)
    assert abs(g.maxflow() - oflow) <= 1e-9 * abs(oflow)


def test_fused_build_reports_non_positive_weights():
    gc = _gc()
    img = numpy.zeros((4, 4, 8)); img[1, 1, 1] = 2.0
    fg = numpy.zeros((4, 4, 8)); fg[1, 1, 1] = 1
    bg = numpy.zeros((4, 4, 8)); bg[0, 0, 0] = 1
    with pytest.raises(ValueError):
        gc.graph_from_voxels(fg, bg, boundary_term=gc.energy_voxel.boundary_difference_division,
                             boundary_term_args=(img, 0.5, (-1.0, 1.0, 1.0)))


@pytest.mark.parametrize("shape,regional", [((64, 64, 64), False), ((40, 72, 56), False), ((48, 48, 48), True),
                                            ((48, 40, 20), False),      # rows of <= 32 voxels: one thread per row
                                            ((40, 40, 33), False),      # one warp per row from 33 voxels
                                            ((16, 16, 1024), False),    # the longest one-segment row
                                            ((12, 8, 1100), False)])    # two segments with a carry
def test_sweep_relabel_equals_worklist_relabel_and_oracle(shape, regional):
    """Directional sweeps in front of the worklist BFS (forced on for every relabel) vs the worklist BFS alone vs BK."""
    from medpy_b200 import synthetic
    from oracle import energy_terms as et, solvers
    vol = synthetic.two_blob_volume(shape, seed=11)
    out = []
    for env in (dict(MEDPY_GC_SWEEP=1, MEDPY_GC_SWEEP_FRAC=1000000), dict(MEDPY_GC_SWEEP=0), dict(),
                dict(MEDPY_GC_SWEEP_FRAC=1000000, MEDPY_GC_SWEEP_MIN_ROUNDS=1, MEDPY_GC_SWEEP_ROUNDS=4)):
        with _env(**env):
            g = _build(vol, regional=regional)
            out.append((g.maxflow(), g.get_mask(), g.stats()))
    prob = et.build_problem(vol["fg"], vol["bg"], regional=(vol["prob"], vol["alpha"]) if regional else None,
                            boundary=("difference_exponential", vol["image"], vol["sigma"], False))
    oflow, omask, _ = solvers.solve_port(prob)
    for flow, mask, st in out:
        assert numpy.array_equal(mask, omask)
        assert abs(flow - oflow) <= 1e-9 * abs(oflow)
        assert st["active_last"] == 0


def test_solved_graph_refuses_new_terms_until_reset():
    """maxflow() leaves residual capacities in place; adding a term then used to re-initialise the solver state on top of
    them (silently wrong energy, ADVICE r1).  Now: RuntimeError until reset()."""
    from medpy_b200 import synthetic
    from medpy_b200.graphcut.maxflow import GraphDouble
    from oracle import energy_terms as et, solvers
    shape = (16, 16, 16)
    vol = synthetic.two_blob_volume(shape, seed=2)
    g = _build(vol)
    e1 = g.maxflow()
    g.add_tweights(5, 3.0, 0.0)
    with pytest.raises(RuntimeError, match="reset"):
        g.maxflow()
    g.reset()
    g2 = GraphDouble(int(numpy.prod(shape)), 0, shape=shape)
    g2.add_regional_probability(vol["prob"], vol["alpha"], True)
    g2.add_boundary(1, vol["image"], vol["sigma"], None, float("nan"))
    g2.add_markers(vol["fg"], vol["bg"])
    assert g2.maxflow() == e1
    # the sequence the reference allows -- solve, add a t-weight, solve again -- through reset + rebuild equals the oracle
    prob = et.build_problem(vol["fg"], vol["bg"], regional=(vol["prob"], vol["alpha"]),
                            boundary=("difference_exponential", vol["image"], vol["sigma"], False))
    prob["flow_const"] = et.add_tweights_pass(prob["tr"], prob["flow_const"], 3.0, 0.0, where=numpy.arange(prob["tr"].size) == 5)
    oflow, omask, _ = solvers.solve_port(prob)
    g3 = GraphDouble(int(numpy.prod(shape)), 0, shape=shape)
    g3.add_regional_probability(vol["prob"], vol["alpha"], True)
    g3.add_boundary(1, vol["image"], vol["sigma"], None, float("nan"))
    g3.add_markers(vol["fg"], vol["bg"])
    g3.add_tweights(5, 3.0, 0.0)
    assert abs(g3.maxflow() - oflow) <= 1e-9 * abs(oflow)
    assert numpy.array_equal(g3.get_mask(), omask)


def test_non_native_byte_order_inputs():
    """'>f4' / '>i2' arrays (FITS / NIfTI readers) are converted, not read as native (ADVICE r1)."""
    from medpy_b200 import synthetic
    shape = (8, 12, 16)
    vol = synthetic.two_blob_volume(shape, seed=5)
    g_native = _build(vol)
    swapped = vol["image"].astype(">f4")
    g_swapped = _build(vol, image=swapped)
    assert g_native.maxflow() == g_swapped.maxflow()
    assert numpy.array_equal(g_native.get_mask(), g_swapped.get_mask())


def test_stream_switch_between_host_staged_terms_and_pool_trim():
    """mgc_set_stream between term calls whose inputs were staged from HOST memory (upload stream), then a pool trim and a
    second graph: results equal the single-stream run (VERDICT r1 robustness items)."""
    import torch
    from medpy_b200 import synthetic, _lib
    from medpy_b200.graphcut.maxflow import GraphDouble
    shape = (16, 24, 32)
    vol = synthetic.two_blob_volume(shape, seed=9)
    n = int(numpy.prod(shape))

    def build(switch):
        g = GraphDouble(n, 0, shape=shape)
        nat = g._nat()
        g._fresh = False
        s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
        if switch:
            nat.set_stream(s1.cuda_stream)
        nat.add_regional_probability(vol["prob"], vol["alpha"], True)
        if switch:
            nat.set_stream(s2.cuda_stream)
        nat.add_boundary(1, vol["image"], vol["sigma"], None, float("nan"))
        if switch:
            nat.set_stream(s1.cuda_stream)
        nat.add_markers(vol["fg"].view(numpy.uint8), vol["bg"].view(numpy.uint8))
        e = g.maxflow()
        m = g.get_mask()
        torch.cuda.synchronize()
        return e, m

    e0, m0 = build(False)
    e1, m1 = build(True)
    assert e0 == e1 and numpy.array_equal(m0, m1)
    _lib._mgc.trim_pools()
    e2, m2 = build(True)
    assert e0 == e2 and numpy.array_equal(m0, m2)
