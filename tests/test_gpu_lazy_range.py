"""The lazy build's range test per staged block (gc_exprange.cuh): a block whose cells span a range that keeps every
argument of the exponential term ordinary runs the lean z-loop, any other block the per-warp vote.  Images that mix both
kinds of block in one volume must give exactly the eager build's graph (MEDPY_GC_LAZY_CAPS=0): t-links and n-links bit
for bit, masks identical, energies within 1e-12 relative -- through the host path (bit-packed markers), the device path
(the staged float32 configuration), the chunked upload and the debug invariants."""
import os

import numpy
import pytest

pytestmark = pytest.mark.gpu

EAGER, LAZY = dict(MEDPY_GC_LAZY_CAPS="0"), dict(MEDPY_GC_LAZY_CAPS="1")


class _env:
    def __init__(self, **kw):
        self.kw = kw

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in self.kw}
        os.environ.update({k: str(v) for k, v in self.kw.items()})

    def __exit__(self, *a):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _build(vol, image, sigma, kind="difference_exponential", regional=True):
    import medpy_b200.graphcut as gc
    kw = dict(boundary_term=getattr(gc.energy_voxel, "boundary_" + kind), boundary_term_args=(image, sigma, False))
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


def _same(a, b):
    flow_a, mask_a = a
    flow_b, mask_b = b
    assert numpy.array_equal(mask_a, mask_b)
    assert abs(flow_a - flow_b) <= 1e-12 * max(1.0, abs(flow_b))


def _outliers(img, n, value, seed):
    out = img.copy()
    rng = numpy.random.default_rng(seed)
    flat = out.reshape(-1)
    flat[rng.choice(flat.size, size=n, replace=False)] = value
    return out


def _case(name, shape):
    from medpy_b200 import synthetic
    vol = synthetic.two_blob_volume(shape, seed=4)
    img, sigma, kind, solve = vol["image"], vol["sigma"], "difference_exponential", True
    if name == "outliers":
        img = _outliers(img, 5, numpy.float32(1e4), 1)
    elif name == "nan_inf":
        img = img.copy()
        img[shape[0] // 2, 3, 5] = numpy.nan
        img[shape[0] - 2, shape[1] - 4, shape[2] - 3] = numpy.inf
        solve = False                      # NaN capacities: compare the graphs only
    elif name == "inf":
        img = img.copy()
        img[1, shape[1] // 2, shape[2] // 2] = numpy.inf
    elif name == "small_sigma":
        sigma = 0.5                        # nearly every block refused, some warps still ordinary
    elif name == "max_negative":
        img, kind = img - numpy.float32(60.0), "maximum_exponential"
    elif name == "float64":
        img = _outliers(img.astype(numpy.float64), 3, 5e3, 2)
    return vol, img, sigma, kind, solve


@pytest.mark.parametrize("name,shape", [
    ("outliers", (24, 28, 32)),
    ("outliers", (17, 9, 45)),             # plain staging (odd X), ragged blocks
    ("nan_inf", (24, 28, 32)),
    ("inf", (16, 24, 64)),
    ("small_sigma", (24, 28, 32)),
    ("small_sigma", (17, 9, 45)),
    ("max_negative", (9, 33, 64)),
    ("float64", (16, 20, 40)),
])
def test_lazy_range_mixed_blocks_equal_eager(name, shape):
    vol, img, sigma, kind, solve = _case(name, shape)
    links, solved = [], []
    for env in (LAZY, EAGER):
        with _env(**env):
            g = _build(vol, img, sigma, kind)
            links.append(_snapshot(g, shape))
            if solve:
                g = _build(vol, img, sigma, kind)
                solved.append((g.maxflow(), g.get_mask()))
    (tr0, w0), (tr1, w1) = links
    assert numpy.array_equal(tr0, tr1)
    assert numpy.array_equal(w0, w1, equal_nan=True)
    if solve:
        _same(*solved)


def test_lazy_range_chunked_upload_refused_blocks_in_late_chunk():
    """z-chunked host upload (builds launched with z_tile0 > 0): the refused blocks sit in the last chunk only."""
    from medpy_b200 import synthetic
    shape = (48, 24, 64)
    vol = synthetic.two_blob_volume(shape, seed=6)
    img = vol["image"].copy()
    img[40:, :, :] = _outliers(img[40:, :, :], 6, numpy.float32(1e4), 3)
    res = []
    for env in (dict(LAZY, MEDPY_GC_CHUNKS=4), dict(LAZY, MEDPY_GC_CHUNKS=1), dict(EAGER, MEDPY_GC_CHUNKS=4)):
        with _env(**env):
            g = _build(vol, img, vol["sigma"])
            res.append((g.maxflow(), g.get_mask()))
    _same(res[0], res[2])
    _same(res[1], res[2])


def test_lazy_range_device_arrays_staged_configuration():
    """Device arrays with float32 map and byte markers: the compile-time t-link configuration (TIN = 1)."""
    import torch
    from medpy_b200 import synthetic
    from medpy_b200.graphcut.device import graph_from_device_arrays
    shape = (32, 40, 64)
    vol = synthetic.two_blob_volume(shape, seed=8)
    for img, sigma in ((_outliers(vol["image"], 4, numpy.float32(1e4), 5), vol["sigma"]), (vol["image"], 0.5)):
        d = {k: torch.from_numpy(numpy.ascontiguousarray(vol[k].view(numpy.uint8) if k in ("fg", "bg") else vol[k])).cuda()
             for k in ("prob", "fg", "bg")}
        d_img = torch.from_numpy(numpy.ascontiguousarray(img)).cuda()
        res = []
        for env in (LAZY, EAGER):
            with _env(**env):
                g = graph_from_device_arrays(d["fg"], d["bg"], image=d_img, boundary="difference_exponential",
                                             sigma=sigma, prob=d["prob"], alpha=vol["alpha"])
                res.append((g.maxflow(), g.get_mask()))
        _same(*res)


def test_lazy_range_debug_checks_with_refused_blocks():
    """MEDPY_GC_DEBUG=1: residual-mask invariants and flow conservation around the solve of a lazy build whose volume
    mixes lean and refused blocks."""
    from medpy_b200 import synthetic
    shape = (24, 40, 48)
    vol = synthetic.two_blob_volume(shape, seed=5)
    img = _outliers(vol["image"], 6, numpy.float32(1e4), 7)
    res = []
    for env in (dict(LAZY, MEDPY_GC_DEBUG="1"), EAGER):
        with _env(**env):
            g = _build(vol, img, vol["sigma"])
            res.append((g.maxflow(), g.get_mask()))
    _same(*res)
