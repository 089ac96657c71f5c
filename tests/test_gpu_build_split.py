"""The lazy exponential build as two launches (gc_build.cuh): k_build_lean streams the blocks that pass their range test,
k_build_refused builds the others with the per-warp fallback.  MEDPY_GC_BUILD_REFUSE_ALL=1 sends every block to the
second launch, so one volume can be built both ways: energies bit for bit, masks, and sampled t-links and n-links must
be the same -- host inputs (bit-packed markers) with and without a regional term, device float32 inputs (the staged
configuration), ragged lattices whose x extent still allows TMA staging, and the z-chunked host upload.  The stats count
the refused blocks: none on a clean volume, all of them at a tiny sigma, some with planted outliers."""
import os

import numpy
import pytest

pytestmark = pytest.mark.gpu

LEAN, REFUSED = dict(MEDPY_GC_BUILD_REFUSE_ALL="0"), dict(MEDPY_GC_BUILD_REFUSE_ALL="1")


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


def _host_graph(vol, image, sigma, regional=True):
    import medpy_b200.graphcut as gc
    kw = dict(boundary_term=gc.energy_voxel.boundary_difference_exponential, boundary_term_args=(image, sigma, False))
    if regional:
        kw.update(regional_term=gc.energy_voxel.regional_probability_map, regional_term_args=(vol["prob"], vol["alpha"]))
    return gc.graph_from_voxels(vol["fg"], vol["bg"], **kw)


def _device_graph(vol, image, sigma):
    import torch
    from medpy_b200.graphcut.device import graph_from_device_arrays
    d = {k: torch.from_numpy(numpy.ascontiguousarray(vol[k].view(numpy.uint8) if k in ("fg", "bg") else vol[k])).cuda()
         for k in ("prob", "fg", "bg")}
    d_img = torch.from_numpy(numpy.ascontiguousarray(image)).cuda()
    return graph_from_device_arrays(d["fg"], d["bg"], image=d_img, boundary="difference_exponential", sigma=sigma,
                                    prob=d["prob"], alpha=vol["alpha"])


def _sample(g, shape, count=3000, seed=0):
    n = int(numpy.prod(shape))
    ids = numpy.random.default_rng(seed).choice(n, size=min(n, count), replace=False)
    strides = [int(numpy.prod(shape[d + 1:])) for d in range(3)]
    tr = numpy.asarray([g.get_trcap(int(p)) for p in ids])
    w = []
    for p in ids:
        p = int(p)
        for d, st in enumerate(strides):
            if (p // st) % shape[d] < shape[d] - 1:
                w.append(g.get_edge(p, p + st))
                w.append(g.get_edge(p + st, p))
    return tr, numpy.asarray(w)


def _both(make, shape, extra=None):
    """(energy, mask, refused blocks, t-links, n-links) of the lean and the forced-refused build."""
    out = []
    for env in (LEAN, REFUSED):
        with _env(**dict(env, **(extra or {}))):
            g = make()
            energy, mask = g.maxflow(), g.get_mask()
            refused = g.stats()["build_blocks_refused"]
            links = _sample(make(), shape)
            out.append((energy, mask, refused, links))
    return out


def _blocks(shape):
    return -(-shape[0] // 8) * -(-shape[1] // 8) * -(-shape[2] // 32)


def _assert_same(a, b):
    assert a[0] == b[0], (a[0], b[0])                # bit for bit
    assert numpy.array_equal(a[1], b[1])
    assert numpy.array_equal(a[3][0], b[3][0])
    assert numpy.array_equal(a[3][1], b[3][1])


@pytest.mark.parametrize("shape,regional", [
    ((24, 28, 32), True),
    ((24, 28, 32), False),
    ((21, 13, 36), True),         # ragged: x allows TMA staging, y and z not multiples of 8
    ((19, 30, 44), False),
    ((40, 48, 96), True),
])
def test_lean_equals_refused_host_inputs(shape, regional):
    from medpy_b200 import synthetic
    vol = synthetic.two_blob_volume(shape, seed=12)
    lean, ref = _both(lambda: _host_graph(vol, vol["image"], vol["sigma"], regional), shape)
    _assert_same(lean, ref)
    assert lean[2] == 0 and ref[2] == _blocks(shape)


def test_lean_equals_refused_device_float32_inputs():
    from medpy_b200 import synthetic
    shape = (32, 40, 64)
    vol = synthetic.two_blob_volume(shape, seed=8)
    lean, ref = _both(lambda: _device_graph(vol, vol["image"], vol["sigma"]), shape)
    _assert_same(lean, ref)
    assert lean[2] == 0 and ref[2] == _blocks(shape)


def test_lean_equals_refused_chunked_upload():
    from medpy_b200 import synthetic
    shape = (48, 24, 64)
    vol = synthetic.two_blob_volume(shape, seed=6)
    lean, ref = _both(lambda: _host_graph(vol, vol["image"], vol["sigma"]), shape, dict(MEDPY_GC_CHUNKS=4))
    _assert_same(lean, ref)
    assert lean[2] == 0 and ref[2] == _blocks(shape)


def test_refused_block_count():
    from medpy_b200 import synthetic
    shape = (32, 40, 64)
    vol = synthetic.two_blob_volume(shape, seed=3)
    img = vol["image"].copy()
    flat = img.reshape(-1)
    flat[numpy.random.default_rng(1).choice(flat.size, size=5, replace=False)] = numpy.float32(1e4)
    counts = {}
    for name, image, sigma in (("clean", vol["image"], vol["sigma"]), ("tiny_sigma", vol["image"], 1e-3),
                               ("outliers", img, vol["sigma"])):
        with _env(**LEAN):
            g = _host_graph(vol, image, sigma)
            g.maxflow()
            counts[name] = g.stats()["build_blocks_refused"]
    assert counts["clean"] == 0, counts
    assert counts["tiny_sigma"] == _blocks(shape), counts
    assert 0 < counts["outliers"] < _blocks(shape), counts
    # mixed lean and refused blocks still build what the forced-refused path builds
    lean, ref = _both(lambda: _host_graph(vol, img, vol["sigma"]), shape)
    _assert_same(lean, ref)
