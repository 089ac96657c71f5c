"""Lazy push state: the fused 3-D build writes neither capacities nor tr nor excess, k_caps_tiles recomputes all three
per tile from copies of the image and the probability map and from the marker bit planes.  Every input form of the
t-links must give the eager build's (MEDPY_GC_LAZY_CAPS=0) values bit for bit, and every reader of tr / excess outside
the push path must see materialised values."""
import math

import numpy
import pytest

from test_gpu_lazy_caps import EAGER, LAZY, _build, _env, _ntiles, _same, _snapshot

pytestmark = pytest.mark.gpu


def _native_build(vol, prob, compute_f32, fg, bg, image=None):
    """The fused build through the native entry point, with the products' dtype chosen explicitly."""
    from medpy_b200.graphcut.maxflow import GraphDouble
    img = vol["image"] if image is None else image
    shape = tuple(img.shape)
    g = GraphDouble(int(numpy.prod(shape)), 0, shape=shape)
    g._fresh = False
    g._nat().build_voxel_graph(prob, float(vol["alpha"]), compute_f32, 3, img, float(vol["sigma"]), None, math.nan,
                               fg.view(numpy.uint8), bg.view(numpy.uint8))
    return g


@pytest.mark.parametrize("shape,case", [
    ((12, 20, 40), "prob_f64"),               # float64 map, float64 products
    ((14, 18, 64), "prob_f32_products_f64"),  # float32 map, float64 products
    ((20, 24, 72), "ragged_x"),               # X % 32 != 0 on the TMA path: the last warp row of a marker word is partial
    ((9, 13, 50), "ragged_x"),                # X % 4 != 0: plain staging
])
def test_lazy_push_state_t_link_inputs(shape, case):
    from medpy_b200 import synthetic
    vol = synthetic.two_blob_volume(shape, seed=7)
    if case == "prob_f64":
        vol = dict(vol, prob=vol["prob"].astype(numpy.float64))

        def make():
            return _build(vol)
    elif case == "prob_f32_products_f64":
        def make():
            return _native_build(vol, vol["prob"].astype(numpy.float32), False, vol["fg"], vol["bg"])
    else:
        def make():
            return _build(vol)

    res = []
    for env in (LAZY, EAGER):
        with _env(**env):
            links = _snapshot(make(), shape)
            g = make()
            res.append((links, (g.maxflow(), g.get_mask())))
    (tr0, w0), (tr1, w1) = res[0][0], res[1][0]
    assert numpy.array_equal(tr0, tr1)
    assert numpy.array_equal(w0, w1, equal_nan=True)
    _same(res[0][1], res[1][1])


def test_lazy_push_state_device_byte_markers():
    """float32 image and map with byte markers, all device-resident: the compile-time variant of the build (TIN = 1)."""
    import torch
    from medpy_b200 import synthetic
    from medpy_b200.graphcut.device import graph_from_device_arrays
    shape = (24, 32, 64)
    vol = synthetic.two_blob_volume(shape, seed=2)
    d = {k: torch.from_numpy(numpy.ascontiguousarray(vol[k].view(numpy.uint8) if k in ("fg", "bg") else vol[k])).cuda()
         for k in ("image", "prob", "fg", "bg")}

    def make():
        return graph_from_device_arrays(d["fg"], d["bg"], image=d["image"], boundary="difference_exponential",
                                        sigma=vol["sigma"], prob=d["prob"], alpha=vol["alpha"])

    res = []
    for env in (LAZY, EAGER):
        with _env(**env):
            links = _snapshot(make(), shape)
            g = make()
            res.append((links, (g.maxflow(), g.get_mask())))
    (tr0, w0), (tr1, w1) = res[0][0], res[1][0]
    assert numpy.array_equal(tr0, tr1)
    assert numpy.array_equal(w0, w1, equal_nan=True)
    _same(res[0][1], res[1][1])


def test_lazy_push_state_host_bit_markers():
    """Host marker volumes of >= 2^22 voxels cross PCIe bit-packed: the build reads the markers from bit words."""
    from medpy_b200 import synthetic
    shape = (64, 256, 256)
    vol = synthetic.two_blob_volume(shape, seed=4)
    res = []
    for env in (LAZY, EAGER):
        with _env(**env):
            links = _snapshot(_build(vol), shape, count=1500)
            g = _build(vol)
            res.append((links, (g.maxflow(), g.get_mask())))
    (tr0, w0), (tr1, w1) = res[0][0], res[1][0]
    assert numpy.array_equal(tr0, tr1)
    assert numpy.array_equal(w0, w1, equal_nan=True)
    _same(res[0][1], res[1][1])


def test_lazy_push_state_first_stop_test():
    """MEDPY_GC_FIRST_TEST=1: the stop test of the first round reads the excess of the build's own lists."""
    from medpy_b200 import synthetic
    shape = (32, 48, 64)
    vol = synthetic.two_blob_volume(shape, seed=6)
    res = []
    for env in (LAZY, EAGER):
        with _env(MEDPY_GC_FIRST_TEST="1", **env):
            g = _build(vol)
            res.append((g.maxflow(), g.get_mask(), g.stats()))
    _same(res[0][:2], res[1][:2])
    assert res[0][2]["push_sweeps"] == res[1][2]["push_sweeps"]
    assert res[0][2]["global_relabels"] == res[1][2]["global_relabels"]


def test_lazy_push_state_trcap_after_maxflow():
    """get_trcap after the flow on tiles the push passes never reached (their excess was never written by the build)."""
    from medpy_b200 import synthetic
    shape = (64, 64, 96)
    vol = synthetic.two_blob_volume(shape, seed=0)
    res = []
    for env in (LAZY, EAGER):
        with _env(**env):
            g = _build(vol)
            flow = g.maxflow()
            mat = g.stats()["tiles_materialised"]
            rng = numpy.random.default_rng(3)
            ids = rng.choice(int(numpy.prod(shape)), size=3000, replace=False)
            res.append((flow, g.get_mask(), numpy.asarray([g.get_trcap(int(p)) for p in ids]), mat))
    assert 0 < res[0][3] < _ntiles(shape)
    _same(res[0][:2], res[1][:2])
    # uninitialised excess would be far off; the flows themselves may differ in the last bits (cross-face atomics)
    assert numpy.allclose(res[0][2], res[1][2], rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("regional", [True, False])
def test_readout_clean_tiles_equal_full_readout(regional):
    """The read-out that reads the labels of dirty tiles only (MEDPY_GC_PARTIAL_RESET=1) gives the mask and the energy of
    the full read-out (=0); without a regional term the instance is a hard one, where sweeps run."""
    from medpy_b200 import synthetic
    shape = (48, 64, 96)
    vol = synthetic.two_blob_volume(shape, seed=8)
    res = []
    for flag in ("1", "0"):
        with _env(MEDPY_GC_PARTIAL_RESET=flag):
            g = _build(vol, regional=regional)
            flow = g.maxflow()
            res.append((flow, g.get_mask()))
    _same(*res)
