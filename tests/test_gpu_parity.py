"""GPU parity tests (run on an H100 with ``-m gpu``): the CUDA path behind the reference API / C ABI
against (1) golden vectors produced by the unmodified reference, (2) the CPU oracle on seeded inputs at sizes
the oracle finishes in seconds, and (3) size-independent certificates at BASELINE sizes (max-flow == min-cut
duality evaluated independently with the oracle's weights).

Tolerances: integer / byte / index results bit-exact (masks, integer-capacity energies, t-links, the linear
and division weights); float64 energies within 1e-9 relative (north star allows 1e-5); exp / pow weights
within 2e-13 relative of numpy's (the exponential's argument is formed with the reciprocal of sigma^2, which moves it by
a few ulp; test_gpu_boundary_domain.py bounds every weight from the arithmetic instead, over the whole domain).
"""
import ctypes
import os

import numpy
import pytest

from conftest import golden

pytestmark = pytest.mark.gpu

NAMES = golden().names()


def _gc():
    import medpy_b200.graphcut as gc
    return gc


def _build_graph(c):
    gc = _gc()
    ev = gc.energy_voxel
    kw = {}
    if c["boundary"]:
        fn = getattr(ev, "boundary_" + c["boundary"])
        sp = tuple(c["spacing"]) if c["spacing"] else False
        if c["boundary"].endswith("linear"):
            kw.update(boundary_term=fn, boundary_term_args=(c["image"], sp))
        else:
            kw.update(boundary_term=fn, boundary_term_args=(c["image"], c["sigma"], sp))
    if c["prob"] is not None:
        kw.update(regional_term=ev.regional_probability_map, regional_term_args=(c["prob"], c["alpha"]))
    return gc.graph_from_voxels(c["fg"], c["bg"], **kw)


def _all_edges(g, shape):
    n = int(numpy.prod(shape))
    nd = len(shape)
    w = numpy.zeros((nd, n))
    wr = numpy.zeros((nd, n))
    stride = n
    for d in range(nd):
        stride //= shape[d]
        for p in range(n):
            if (p % (stride * shape[d])) // stride < shape[d] - 1:
                w[d, p] = g.get_edge(p, p + stride)
                wr[d, p] = g.get_edge(p + stride, p)
    return w, wr


@pytest.mark.parametrize("name", NAMES)
def test_golden_case(name):
    """Every golden case of the reference: n-link weights, t-links, flow and mask."""
    c = golden().case(name)
    g = _build_graph(c)
    shape = numpy.asarray(c["fg"]).shape
    n = int(numpy.prod(shape))
    small = n <= 600
    if small:
        w, wr = _all_edges(g, shape)
        exact = c["boundary"] is None or c["boundary"].split("_")[1] in ("linear", "division")
        ref = c["w"]
        if exact:
            assert numpy.array_equal(w, ref, equal_nan=True)
        else:
            numpy.testing.assert_allclose(w, ref, rtol=2e-13, atol=0)
        assert numpy.array_equal(w, wr, equal_nan=True)  # symmetric arcs (energy_voxel.py:664)
    tr = numpy.asarray([g.get_trcap(p) for p in range(min(n, 600))])
    assert numpy.array_equal(tr, c["tr"][: tr.size])
    flow = g.maxflow()
    mask = numpy.asarray([0 if g.termtype.SINK == g.what_segment(i) else 1 for i in range(n)]).reshape(shape)
    if numpy.isnan(c["flow"]):
        return  # zero-image linear terms: the reference only requires "does not raise"
    assert numpy.array_equal(mask, c["mask"].reshape(shape)), "mask differs from the reference's"
    assert numpy.array_equal(g.get_mask().reshape(shape), mask)
    assert abs(flow - c["flow"]) <= 1e-9 * max(1.0, abs(c["flow"])), (flow, c["flow"])
    if float(c["flow"]).is_integer() and name.startswith("ref_fixture_cut3d"):
        assert flow == 3.0  # tests/graphcut_/cut.py:50,96-102


def _oracle_solve(prob):
    from oracle import solvers
    return solvers.solve_port(prob)


def test_recorded_fuzz_cases_vs_reference():
    """The 120 cases tests/golden/fuzz_voxels_v1.json recorded from the unmodified reference (1-D..4-D, the eight
    boundary terms, five image dtypes, spacing, regional term, overlapping markers), regenerated from the recorded seed
    and solved through graph_from_voxels: the same cases raise ValueError; t-links equal the restatement's bit for bit
    (which test_oracle pins to the reference), n-link weights within the golden tolerances; flow and mask equal the
    reference's, a mask only up to an exact tie.  (The recorded set has no refused and no NaN-weight case; the branches
    for them keep the test right if it is re-recorded with another seed or size.)"""
    import json
    import sys
    import warnings
    from oracle import energy_terms as et
    from test_gpu_fullsize import _cut_difference_exact
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    import fuzz_voxels_against_reference as fuzz
    with open(fuzz.GOLDEN) as fh:
        z = json.load(fh)
    rng = numpy.random.default_rng(z["seed"])
    solved = refused = nan_weights = 0
    for i, rec in enumerate(z["records"]):
        c = fuzz.random_case(rng)
        c.setdefault("prob", None)
        shape = c["fg"].shape
        with warnings.catch_warnings(), numpy.errstate(all="ignore"):
            warnings.simplefilter("ignore")
            if rec.get("error"):
                with pytest.raises(ValueError):
                    _build_graph(c).maxflow()
                refused += 1
                continue
            prob = et.build_problem(c["fg"], c["bg"], regional=(c["prob"], c["alpha"]) if c["prob"] is not None else None,
                                    boundary=(c["boundary"], c["image"], c["sigma"], c["spacing"]))
            g = _build_graph(c)
        n = int(numpy.prod(shape))
        tr = numpy.asarray([g.get_trcap(p) for p in range(n)])
        assert numpy.array_equal(tr, prob["tr"]), (i, c["boundary"])
        w, wr = _all_edges(g, shape)
        want = numpy.stack([numpy.asarray(x, dtype=numpy.float64) for x in prob["wf"]])
        if c["boundary"].split("_")[1] in ("linear", "division"):
            assert numpy.array_equal(w, want, equal_nan=True), (i, c["boundary"])
        else:
            numpy.testing.assert_allclose(w, want, rtol=2e-13, atol=0, err_msg="case %d %s" % (i, c["boundary"]))
        assert numpy.array_equal(w, wr, equal_nan=True), i
        if numpy.isnan(want).any():
            nan_weights += 1    # as check() does: the reference only has to not raise
            continue
        flow = g.maxflow()
        mask = g.get_mask().ravel()
        rflow = float.fromhex(rec["flow"])
        rmask = numpy.frombuffer(rec["mask"].encode(), numpy.uint8) - ord("0")
        assert abs(flow - rflow) <= 1e-9 * max(1.0, abs(rflow)), (i, c["boundary"], flow, rflow)
        if not numpy.array_equal(mask, rmask):
            diff = _cut_difference_exact(prob, mask, rmask)
            assert abs(diff) <= 0.5 * numpy.spacing(abs(rflow)), (i, c["boundary"], "mask differs by more than a tie", diff)
        solved += 1
    assert solved + refused + nan_weights == len(z["records"]) and solved > 100, (solved, refused, nan_weights)


@pytest.mark.parametrize("shape,seed", [((32, 32, 32), 0), ((40, 24, 56), 1), ((20, 48, 33), 2)])
def test_config3_regional_plus_exponential_vs_oracle(shape, seed):
    """BASELINE config 3 at oracle-sized volumes: regional_probability_map + boundary_difference_exponential."""
    from medpy_b200 import synthetic
    from oracle import energy_terms as et
    gc = _gc()
    vol = synthetic.two_blob_volume(shape, seed=seed)
    g = gc.graph_from_voxels(vol["fg"], vol["bg"],
                             regional_term=gc.energy_voxel.regional_probability_map,
                             regional_term_args=(vol["prob"], vol["alpha"]),
                             boundary_term=gc.energy_voxel.boundary_difference_exponential,
                             boundary_term_args=(vol["image"], vol["sigma"], False))
    flow = g.maxflow()
    prob = et.build_problem(vol["fg"], vol["bg"], regional=(vol["prob"], vol["alpha"]),
                            boundary=("difference_exponential", vol["image"], vol["sigma"], False))
    oflow, omask, _ = _oracle_solve(prob)
    assert numpy.array_equal(g.get_mask(), omask)
    assert abs(flow - oflow) <= 1e-9 * abs(oflow)
    assert 0 < omask.sum() < omask.size


@pytest.mark.parametrize("shape,seed", [((32, 32, 32), 3), ((48, 40, 36), 4)])
def test_config2_boundary_only_vs_oracle(shape, seed):
    """BASELINE config 2 at oracle-sized volumes: boundary_difference_exponential, sigma = RMS difference."""
    from medpy_b200 import synthetic
    from oracle import energy_terms as et
    gc = _gc()
    vol = synthetic.two_blob_volume(shape, seed=seed, with_prob=False)
    g = gc.graph_from_voxels(vol["fg"], vol["bg"], boundary_term=gc.energy_voxel.boundary_difference_exponential,
                             boundary_term_args=(vol["image"], vol["sigma"], False))
    flow = g.maxflow()
    prob = et.build_problem(vol["fg"], vol["bg"],
                            boundary=("difference_exponential", vol["image"], vol["sigma"], False))
    oflow, omask, _ = _oracle_solve(prob)
    assert numpy.array_equal(g.get_mask(), omask)
    assert abs(flow - oflow) <= 1e-9 * abs(oflow)


def test_config1_difference_linear_64cubed_vs_oracle():
    """BASELINE config 1: 64^3 two-blob fp32, boundary_difference_linear (img, False)."""
    from medpy_b200 import synthetic
    from oracle import energy_terms as et
    gc = _gc()
    vol = synthetic.two_blob_volume((64, 64, 64), seed=0, with_prob=False)
    g = gc.graph_from_voxels(vol["fg"], vol["bg"], boundary_term=gc.energy_voxel.boundary_difference_linear,
                             boundary_term_args=(vol["image"], False))
    flow = g.maxflow()
    prob = et.build_problem(vol["fg"], vol["bg"], boundary=("difference_linear", vol["image"], None, False))
    oflow, omask, _ = _oracle_solve(prob)
    assert numpy.array_equal(g.get_mask(), omask)
    assert abs(flow - oflow) <= 1e-9 * abs(oflow)


def test_config4_multispectral_4d_vs_oracle():
    """BASELINE config 4 at oracle size: 4-D lattice (8-connected, channel axis linked), boundary_maximum_exponential."""
    from medpy_b200 import synthetic
    from oracle import energy_terms as et
    gc = _gc()
    vol = synthetic.multispectral_volume((24, 20, 16, 4), seed=5)
    g = gc.graph_from_voxels(vol["fg"], vol["bg"], boundary_term=gc.energy_voxel.boundary_maximum_exponential,
                             boundary_term_args=(vol["image"], vol["sigma"], False))
    flow = g.maxflow()
    prob = et.build_problem(vol["fg"], vol["bg"], boundary=("maximum_exponential", vol["image"], vol["sigma"], False))
    oflow, omask, _ = _oracle_solve(prob)
    assert numpy.array_equal(g.get_mask(), omask)
    assert abs(flow - oflow) <= 1e-9 * abs(oflow)


@pytest.mark.parametrize("shape", [(24, 24, 24), (16, 40, 28)])
def test_integer_capacities_bit_exact(shape):
    """Integer parity set (SURVEY.md §8d): integer weights through a user-written 2-argument boundary term;
    energy must equal the oracle's EXACTLY and the masks must be identical."""
    from medpy_b200 import synthetic
    from oracle import energy_terms as et
    gc = _gc()
    vol = synthetic.two_blob_volume(shape, seed=11, integer=True, with_prob=False)
    term = synthetic.integer_weight_boundary_term(vol["image"])
    g = gc.graph_from_voxels(vol["fg"], vol["bg"], boundary_term=term, boundary_term_args=(vol["image"],))
    flow = g.maxflow()
    # oracle problem with the same integer weights
    prob = et.build_problem(vol["fg"], vol["bg"])
    img = vol["image"].astype(numpy.float64)
    ws = []
    for d in range(3):
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[d] = slice(0, -1)
        hi[d] = slice(1, None)
        ws.append(1.0 + (255.0 - numpy.minimum(numpy.abs(img[tuple(lo)] - img[tuple(hi)]), 255.0)))
    prob["wf"] = prob["wb"] = et.dense_axis_arrays(shape, ws)
    oflow, omask, _ = _oracle_solve(prob)
    assert flow == oflow, (flow, oflow)
    assert float(flow).is_integer()
    assert numpy.array_equal(g.get_mask(), omask)


def test_element_wise_api_matches_bulk():
    """GCGraph.set_nweight / set_tweight / set_source_nodes (the reference's per-element API) give the same
    graph as the bulk terms."""
    gc = _gc()
    from oracle import energy_terms as et
    rng = numpy.random.default_rng(5)
    shape = (5, 6, 7)
    n = int(numpy.prod(shape))
    img = rng.normal(size=shape) * 10
    w = et.boundary_weights("difference_division", img, 3.0, False)
    graph = gc.GCGraph(n, 3 * n, shape=shape)
    stride = n
    for d in range(3):
        stride //= shape[d]
        full = numpy.zeros(shape)
        sl = [slice(None)] * 3
        sl[d] = slice(0, shape[d] - 1)
        full[tuple(sl)] = w[d]
        flat = full.ravel()
        for p in numpy.flatnonzero(flat > 0):
            graph.set_nweight(int(p), int(p + stride), float(flat[p]), float(flat[p]))
    fg = numpy.zeros(shape, bool); fg[1, 1, 1] = True
    bg = numpy.zeros(shape, bool); bg[4, 5, 6] = bg[0, 0, 0] = True
    src = rng.random(n) * 0.3
    snk = rng.random(n) * 0.3
    graph.set_tweights_all(numpy.stack([src, snk], axis=1))
    graph.set_source_nodes(numpy.flatnonzero(fg.ravel()))
    graph.set_sink_nodes(numpy.flatnonzero(bg.ravel()))
    g = graph.get_graph()
    flow = g.maxflow()
    prob = et.build_problem(fg, bg, boundary=("difference_division", img, 3.0, False))
    tr = numpy.zeros(n)
    fl = et.add_tweights_pass(tr, 0.0, src, snk)
    fl = et.add_tweights_pass(tr, fl, 65535.0, 0.0, where=fg.ravel())
    fl = et.add_tweights_pass(tr, fl, 0.0, 65535.0, where=bg.ravel())
    prob["tr"], prob["flow_const"] = tr, fl
    oflow, omask, _ = _oracle_solve(prob)
    assert numpy.array_equal(g.get_mask(), omask)
    assert abs(flow - oflow) <= 1e-9 * abs(oflow)


def test_weights_not_positive_raise_value_error():
    """GCGraph.set_nweight raises ValueError for weights <= 0 (graph.py:436-437).  The g-functions clamp
    non-positive values to DBL_MIN, so the only way there is a non-positive spacing (energy_voxel.py:657-658);
    an exact zero from the linear term becomes DBL_MIN and must NOT raise."""
    gc = _gc()
    img = numpy.zeros((4, 4), dtype=numpy.float64)
    img[0, 0] = 1.0
    img[0, 1] = -1.0
    fg = numpy.zeros((4, 4)); fg[3, 3] = 1
    bg = numpy.zeros((4, 4)); bg[0, 0] = 1
    # x = 2, M = 2 -> weight exactly 0 -> DBL_MIN, fine
    g = gc.graph_from_voxels(fg, bg, boundary_term=gc.energy_voxel.boundary_difference_linear, boundary_term_args=(img, False))
    assert g.get_edge(0, 1) == 2.2250738585072014e-308
    g.maxflow()
    with pytest.raises(ValueError):
        gc.graph_from_voxels(fg, bg, boundary_term=gc.energy_voxel.boundary_difference_division,
                             boundary_term_args=(img, 0.5, (-1.0, 1.0)))


def test_duality_certificate_256cubed():
    """BASELINE config 2 at full size (256^3 fp32, difference_exponential, sigma = RMS): the oracle solver is too
    slow here, so check optimality through max-flow/min-cut duality: the energy returned (constant + flow into
    the sink) must equal the capacity of the returned cut, evaluated independently with the ORACLE's float64
    weights.  Any feasible flow <= any cut, so equality proves both optimal."""
    from medpy_b200 import synthetic
    from oracle import energy_terms as et
    gc = _gc()
    shape = (256, 256, 256)
    vol = synthetic.two_blob_volume(shape, seed=0, with_prob=False)
    g = gc.graph_from_voxels(vol["fg"], vol["bg"], boundary_term=gc.energy_voxel.boundary_difference_exponential,
                             boundary_term_args=(vol["image"], vol["sigma"], False))
    flow = g.maxflow()
    mask = g.get_mask().astype(bool)
    assert mask[vol["fg"]].all() and not mask[vol["bg"]].any()
    # cut capacity with oracle weights, axis by axis to bound memory
    tr = numpy.zeros(mask.size)
    fl = et.add_tweights_pass(tr, 0.0, 65535.0, 0.0, where=vol["fg"].ravel())
    fl = et.add_tweights_pass(tr, fl, 0.0, 65535.0, where=vol["bg"].ravel())
    trr = tr.reshape(shape)
    e = fl + trr[(~mask) & (trr > 0)].sum() + (-trr[mask & (trr < 0)]).sum()
    img = vol["image"].astype(numpy.float64)
    for d in range(3):
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[d] = slice(0, -1)
        hi[d] = slice(1, None)
        cut = mask[tuple(lo)] != mask[tuple(hi)]
        x = numpy.abs(img[tuple(lo)][cut] - img[tuple(hi)][cut])
        e += et._g_exponential(x, vol["sigma"]).sum()
    assert abs(e - flow) <= 1e-9 * abs(flow), (e, flow)
    st = g.stats()
    assert st["active_last"] == 0


def test_c_abi_direct_ctypes():
    """Drive the path through the raw C ABI (include/medpy_b200_graphcut.h) the way a foreign binding would."""
    from medpy_b200 import build, synthetic
    from oracle import energy_terms as et
    lib = ctypes.CDLL(build.LIB)

    class Arr(ctypes.Structure):
        _fields_ = [("data", ctypes.c_void_p), ("dtype", ctypes.c_int32), ("mem", ctypes.c_int32),
                    ("strides", ctypes.c_int64 * 4)]

    def arr(a, dt):
        s = (ctypes.c_int64 * 4)(*(list(a.strides) + [0] * (4 - a.ndim)))
        return Arr(a.ctypes.data, dt, 0, s)

    lib.mgc_last_error.restype = ctypes.c_char_p
    shape = (20, 24, 28)
    vol = synthetic.two_blob_volume(shape, seed=9)
    h = ctypes.c_void_p()
    shp = (ctypes.c_int64 * 3)(*shape)
    assert lib.mgc_create(3, shp, -1, ctypes.byref(h)) == 0
    img = numpy.ascontiguousarray(vol["image"])
    prob = numpy.ascontiguousarray(vol["prob"])
    fg = numpy.ascontiguousarray(vol["fg"].astype(numpy.uint8))
    bg = numpy.ascontiguousarray(vol["bg"].astype(numpy.uint8))
    a_prob, a_img, a_fg, a_bg = arr(prob, 0), arr(img, 0), arr(fg, 2), arr(bg, 2)
    assert lib.mgc_add_regional_probability(h, ctypes.byref(a_prob), ctypes.c_double(0.1), 0) == 0
    assert lib.mgc_add_boundary(h, 1, ctypes.byref(a_img), ctypes.c_double(vol["sigma"]), None, ctypes.c_double(float("nan"))) == 0
    assert lib.mgc_add_markers(h, ctypes.byref(a_fg), ctypes.byref(a_bg)) == 0
    energy = ctypes.c_double()
    assert lib.mgc_maxflow(h, ctypes.byref(energy)) == 0, lib.mgc_last_error(h)
    mask = numpy.empty(shape, dtype=numpy.uint8)
    assert lib.mgc_get_mask(h, mask.ctypes.data_as(ctypes.c_void_p), 0) == 0
    seg = ctypes.c_int32()
    assert lib.mgc_what_segment(h, 0, ctypes.byref(seg)) == 0 and seg.value == 1  # corner voxel is a bg seed -> SINK
    # errors: bad kind -> MGC_E_ARG with a message, not a crash
    assert lib.mgc_add_boundary(h, 99, ctypes.byref(a_img), ctypes.c_double(1.0), None, ctypes.c_double(0.0)) == -1
    assert b"boundary" in lib.mgc_last_error(h)
    lib.mgc_destroy(h)
    p = et.build_problem(vol["fg"], vol["bg"], regional=(vol["prob"], 0.1),
                         boundary=("difference_exponential", vol["image"], vol["sigma"], False))
    oflow, omask, _ = _oracle_solve(p)
    assert numpy.array_equal(mask, omask)
    assert abs(energy.value - oflow) <= 1e-9 * abs(oflow)


def test_device_resident_inputs_via_cuda_array_interface():
    """torch CUDA tensors (``__cuda_array_interface__``) are consumed in place: no host round trip."""
    import torch
    from medpy_b200 import synthetic
    gc = _gc()
    shape = (24, 24, 24)
    vol = synthetic.two_blob_volume(shape, seed=2)
    args = dict(regional_term=gc.energy_voxel.regional_probability_map,
                boundary_term=gc.energy_voxel.boundary_difference_exponential)
    g1 = gc.graph_from_voxels(vol["fg"], vol["bg"], regional_term_args=(vol["prob"], 0.1),
                              boundary_term_args=(vol["image"], vol["sigma"], False), **args)
    from medpy_b200.graphcut.device import graph_from_device_arrays
    g2 = graph_from_device_arrays(torch.from_numpy(vol["fg"]).cuda(), torch.from_numpy(vol["bg"]).cuda(),
                                  image=torch.from_numpy(vol["image"]).cuda(), sigma=vol["sigma"],
                                  boundary="difference_exponential",
                                  prob=torch.from_numpy(vol["prob"]).cuda(), alpha=0.1)
    assert g1.maxflow() == g2.maxflow()
    assert numpy.array_equal(g1.get_mask(), g2.get_mask())


# ------------------------------------------------------------------------------------------------------
# z-slab path over NCCL (the N-slab runs on one GPU are in test_gpu_slabs.py)
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["regional", "boundary"])
def test_multi_gpu_nccl_slabs_vs_oracle(tmp_path, case):
    """All visible GPUs (>= 2) solve one 48x40x40 volume together over NCCL; result must equal the oracle's."""
    import subprocess
    import sys
    import torch
    ngpu = torch.cuda.device_count()
    if ngpu < 2:
        pytest.skip("needs at least 2 GPUs")
    from medpy_b200 import synthetic
    from oracle import energy_terms as et
    shape = (48, 40, 40)
    out = str(tmp_path / "r0.npz")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(min(ngpu, 4)),
           "--master-addr", "127.0.0.1", "--master-port", "29617", os.path.join(root, "tests", "slab_worker.py"),
           "x".join(map(str, shape)), case, out]
    subprocess.run(cmd, check=True, timeout=600)
    got = numpy.load(out)
    vol = synthetic.two_blob_volume(shape, seed=1, with_prob=(case == "regional"))
    prob = et.build_problem(vol["fg"], vol["bg"], regional=(vol["prob"], vol["alpha"]) if case == "regional" else None,
                            boundary=("difference_exponential", vol["image"], vol["sigma"], False))
    oflow, omask, _ = _oracle_solve(prob)
    assert numpy.array_equal(got["mask"], omask)
    assert abs(float(got["energy"]) - oflow) <= 1e-9 * abs(oflow)


# ------------------------------------------------------------------------------------------------------
# edge cases (SURVEY.md §4 "gaps the new repo must fill itself")
# ------------------------------------------------------------------------------------------------------
def _solve_both(fg, bg, regional=None, boundary=None):
    """(our flow, our mask, oracle flow, oracle mask) for one problem given in oracle.build_problem's terms."""
    from oracle import energy_terms as et
    gc = _gc()
    kw = {}
    if boundary is not None:
        kind, img, sigma, spacing = boundary
        fn = getattr(gc.energy_voxel, "boundary_" + kind)
        kw.update(boundary_term=fn, boundary_term_args=(img, spacing) if kind.endswith("linear") else (img, sigma, spacing))
    if regional is not None:
        kw.update(regional_term=gc.energy_voxel.regional_probability_map, regional_term_args=regional)
    g = gc.graph_from_voxels(fg, bg, **kw)
    flow = g.maxflow()
    assert g.maxflow() == flow          # Graph::maxflow may be called repeatedly (graph.h:129)
    with numpy.errstate(all="ignore"):
        prob = et.build_problem(fg, bg, regional=regional, boundary=boundary)
    oflow, omask, _ = _oracle_solve(prob)
    return flow, g.get_mask(), oflow, omask


@pytest.mark.parametrize("shape", [(9, 7, 13), (1, 1, 37), (3, 17, 1), (8, 8, 8), (16, 9, 24), (5, 5, 5, 3)])
def test_ragged_shapes_and_odd_extents(shape):
    """Partial tiles, odd x extents (no TMA path), degenerate axes, 4-D."""
    rng = numpy.random.default_rng(sum(shape))
    img = (rng.normal(size=shape) * 20).astype(numpy.float32)
    fg = rng.random(shape) < 0.06
    bg = (rng.random(shape) < 0.06) & ~fg
    f, m, of, om = _solve_both(fg, bg, regional=(rng.random(shape).astype(numpy.float32), 0.4),
                               boundary=("difference_exponential", img, 12.0, False))
    assert numpy.array_equal(m, om) and abs(f - of) <= 1e-9 * max(1.0, abs(of))


def test_missing_marker_sets_and_empty_graph():
    shape = (6, 7, 8)
    rng = numpy.random.default_rng(1)
    img = (rng.normal(size=shape) * 20).astype(numpy.float64)
    z = numpy.zeros(shape, bool)
    fg = z.copy(); fg[2, 3, 4] = True
    bg = z.copy(); bg[0, 0, 0] = True
    for f_, b_ in ((fg, z), (z, bg), (z, z)):
        f, m, of, om = _solve_both(f_, b_, boundary=("difference_division", img, 3.0, False))
        assert numpy.array_equal(m, om) and f == of
    # nothing at all: no terms, no markers -> flow 0, every node free -> mask 1 (graph.h:560-571 default SOURCE)
    g = _gc().graph_from_voxels(z, z)
    assert g.maxflow() == 0.0 and g.get_mask().all()


def test_strided_inputs_fortran_negative_and_broadcast():
    """Fortran order (as medpy.io.load returns), reversed views and broadcast markers all describe the same logical
    arrays as their contiguous copies (node ids are C-order over the LOGICAL shape, generate.py:170-172)."""
    from medpy_b200 import synthetic
    shape = (18, 20, 22)
    vol = synthetic.two_blob_volume(shape, seed=6)
    ref = _solve_both(vol["fg"], vol["bg"], regional=(vol["prob"], 0.1), boundary=("difference_exponential", vol["image"], vol["sigma"], False))
    gc = _gc()
    variants = [
        dict(img=numpy.asfortranarray(vol["image"]), prob=numpy.asfortranarray(vol["prob"]), fg=numpy.asfortranarray(vol["fg"]), bg=numpy.asfortranarray(vol["bg"])),
        dict(img=vol["image"][::-1][::-1], prob=numpy.ascontiguousarray(vol["prob"][:, ::-1])[:, ::-1], fg=vol["fg"], bg=vol["bg"]),
        dict(img=vol["image"].astype(numpy.float64)[:, :, ::1], prob=vol["prob"], fg=vol["fg"].astype(numpy.uint8), bg=vol["bg"].astype(numpy.int64)),
    ]
    for v in variants:
        g = gc.graph_from_voxels(v["fg"], v["bg"], regional_term=gc.energy_voxel.regional_probability_map,
                                 regional_term_args=(v["prob"], 0.1), boundary_term=gc.energy_voxel.boundary_difference_exponential,
                                 boundary_term_args=(v["img"], vol["sigma"], False))
        assert g.maxflow() == ref[0]
        assert numpy.array_equal(g.get_mask(), ref[1])
    assert numpy.array_equal(ref[1], ref[3])


def test_int16_maximum_terms_and_wraparound():
    """maximum_* terms take numpy.abs in the INPUT dtype (energy_voxel.py:558): abs(-32768) wraps for int16."""
    shape = (6, 6, 6)
    rng = numpy.random.default_rng(3)
    img = rng.integers(-300, 300, size=shape).astype(numpy.int16)
    img[1, 1, 1] = -32768
    fg = numpy.zeros(shape, bool); fg[2, 2, 2] = True
    bg = numpy.zeros(shape, bool); bg[0] = True
    for kind, sigma in (("maximum_exponential", 200.0), ("maximum_power", 0.5), ("difference_division", 50.0)):
        f, m, of, om = _solve_both(fg, bg, boundary=(kind, img, sigma, (1.0, 2.0, 0.5)))
        assert numpy.array_equal(m, om) and abs(f - of) <= 1e-9 * max(1.0, abs(of)), kind


def test_reset_reuses_the_handle():
    from medpy_b200 import synthetic
    from medpy_b200.graphcut.device import graph_from_device_arrays
    import torch
    vol = synthetic.two_blob_volume((20, 20, 20), seed=8)
    t = {k: torch.from_numpy(numpy.ascontiguousarray(vol[k])).cuda() for k in ("image", "prob")}
    fg, bg = torch.from_numpy(vol["fg"]).cuda(), torch.from_numpy(vol["bg"]).cuda()
    g = None
    outs = []
    for rep in range(3):
        g = graph_from_device_arrays(fg, bg, image=t["image"], boundary="difference_exponential", sigma=vol["sigma"],
                                     prob=t["prob"], alpha=0.1, graph=g)
        outs.append((g.maxflow(), g.get_mask().copy()))
    assert outs[0][0] == outs[1][0] == outs[2][0]
    assert numpy.array_equal(outs[0][1], outs[2][1])


def test_source_clamp_leaves_no_one_ulp_residuals():
    """Regression (found by the full-size 512^3 comparison with BK, tools/compare_fullsize.py): a strongly source-linked
    voxel whose out-capacities are all tiny must end up cut off from its sink-side neighbours with EVERY arc saturated.
    The solver clamps the source link to the sum of the out-capacities; without head-room the sequence of rounded
    subtractions could leave a one-ulp residual on the last arc and the voxel stayed "connected to the sink".
    4096 such voxels with random capacities, all other voxels sink-linked."""
    from oracle import energy_terms as et
    gc = _gc()
    rng = numpy.random.default_rng(123)
    shape = (33, 33, 33)
    n = int(numpy.prod(shape))
    centre = numpy.zeros(shape, bool)
    centre[1::2, 1::2, 1::2] = True
    src = numpy.where(centre, 1.0, 0.0).ravel()
    snk = numpy.where(centre, 0.0, 5.0).ravel()
    ws = []
    for d in range(3):
        short = list(shape); short[d] -= 1
        ws.append(10.0 ** rng.uniform(-9, -2, size=short))
    graph = gc.GCGraph(n, 3 * n, shape=shape)
    graph.set_tweights_dense(src, snk)
    for d in range(3):
        graph.set_nweights_dense(d, ws[d], ws[d])
    g = graph.get_graph()
    flow = g.maxflow()
    mask = g.get_mask()
    assert numpy.array_equal(mask.astype(bool), centre), "a saturated centre voxel is still connected to the sink"
    prob = et.build_problem(numpy.zeros(shape, bool), numpy.zeros(shape, bool))
    tr = numpy.zeros(n)
    prob["flow_const"] = et.add_tweights_pass(tr, 0.0, src, snk)
    prob["tr"] = tr
    prob["wf"] = prob["wb"] = et.dense_axis_arrays(shape, ws)
    oflow, omask, _ = _oracle_solve(prob)
    assert numpy.array_equal(mask, omask)
    assert abs(flow - oflow) <= 1e-9 * abs(oflow)


@pytest.mark.parametrize("shape,dtype", [((9, 8, 7), numpy.float32), ((33, 20, 17), numpy.float32), ((6, 5), numpy.float64),
                                         ((12,), numpy.float32), ((5, 4, 6, 3), numpy.float32), ((16, 9, 11), numpy.int16),
                                         ((1, 7, 1), numpy.float32)])
def test_gradient_magnitude_prewitt_equals_scipy(shape, dtype):
    """SURVEY.md §8 row f1: bin/medpy_gradient.py:79-85 = scipy.ndimage.generic_gradient_magnitude(img, prewitt,
    output=float32).  The arithmetic lives in SciPy (third-party dependency of the reference, present in this image);
    the GPU kernel must reproduce it bit for bit."""
    import scipy.ndimage as ndi
    from medpy_b200.gradient import gradient_magnitude_prewitt
    rng = numpy.random.default_rng(sum(shape))
    img = (rng.normal(size=shape) * 50).astype(dtype)
    want = numpy.zeros(shape, dtype=numpy.float32)
    ndi.generic_gradient_magnitude(img, ndi.prewitt, output=want)
    got = gradient_magnitude_prewitt(img)
    assert got.dtype == numpy.float32 and got.shape == tuple(shape)
    assert numpy.array_equal(got, want), float(numpy.abs(got - want).max())
    # Fortran-ordered input (as medpy.io.load returns) gives the same logical result
    assert numpy.array_equal(gradient_magnitude_prewitt(numpy.asfortranarray(img)), want)


def _prewitt_cases():
    """(name, image): uint8, int32 and float64 in 3-D and 4-D; extents 1, 2 and 3 on every axis; NaN, +-inf, -0 and
    subnormal cells; bool, uint16 and int64 (widened by the binding)."""
    rng = numpy.random.default_rng(77)
    cases = []
    for dtype in (numpy.uint8, numpy.int32, numpy.float64):
        for shape in ((7, 9, 11), (5, 4, 6, 3)):
            if dtype == numpy.uint8:
                img = rng.integers(0, 256, shape).astype(dtype)
            elif dtype == numpy.int32:
                img = rng.integers(-2 ** 31, 2 ** 31 - 1, shape, endpoint=True).astype(dtype)
            else:
                img = rng.normal(0.0, 1e3, shape)
            cases.append(("%s_%dd" % (numpy.dtype(dtype).name, len(shape)), img))
    for ext in (1, 2, 3):
        for nd in (1, 2, 3, 4):
            for ax in range(nd):
                shape = [4] * nd
                shape[ax] = ext
                cases.append(("ext%d_axis%d_of_%dd" % (ext, ax, nd), (rng.normal(size=shape) * 50).astype(numpy.float32)))
        cases.append(("ext%d_all_3d" % ext, (rng.normal(size=(ext, ext, ext)) * 50).astype(numpy.float32)))
    for dtype in (numpy.float32, numpy.float64):
        img = (rng.normal(size=(6, 7, 8)) * 50).astype(dtype)
        tiny = numpy.finfo(dtype).smallest_subnormal
        flat = img.reshape(-1)
        flat[[3, 60, 61, 200, 250]] = numpy.array([numpy.nan, numpy.inf, -numpy.inf, -0.0, tiny], dtype=dtype)
        flat[300:310] = numpy.array([tiny, -tiny, 3 * tiny, numpy.finfo(dtype).tiny, -0.0] * 2, dtype=dtype)
        cases.append(("specials_" + numpy.dtype(dtype).name, img))
        sub = (rng.normal(size=(5, 6, 7)) * 100 * tiny).astype(dtype)       # every cell subnormal
        cases.append(("all_subnormal_" + numpy.dtype(dtype).name, sub))
    cases.append(("bool", rng.random((6, 7, 9)) < 0.4))
    cases.append(("uint16", rng.integers(0, 65536, (6, 7, 9)).astype(numpy.uint16)))
    cases.append(("int64", rng.integers(-2 ** 40, 2 ** 40, (6, 7, 9)).astype(numpy.int64)))
    cases.append(("int64_4d", rng.integers(-1000, 1000, (3, 4, 5, 2)).astype(numpy.int64)))
    return cases


_PREWITT = _prewitt_cases()


@pytest.mark.parametrize("case", range(len(_PREWITT)), ids=[c[0] for c in _PREWITT])
def test_gradient_magnitude_prewitt_domain(case):
    """The Prewitt gradient magnitude against scipy bit for bit (NaN where scipy has NaN) over dtypes, dimensions,
    extents 1 to 3 (where mode 'reflect' folds both neighbours onto the cell or onto each other) and special cells."""
    import scipy.ndimage as ndi
    from medpy_b200.gradient import gradient_magnitude_prewitt
    _, img = _PREWITT[case]
    want = numpy.zeros(img.shape, dtype=numpy.float32)
    with numpy.errstate(all="ignore"):
        ndi.generic_gradient_magnitude(img, ndi.prewitt, output=want)
    got = gradient_magnitude_prewitt(img)
    assert got.dtype == numpy.float32 and got.shape == img.shape
    assert numpy.array_equal(got, want, equal_nan=True), numpy.flatnonzero(~((got == want) | (numpy.isnan(got) & numpy.isnan(want))))[:8]
