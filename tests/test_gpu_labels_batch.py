"""GPU tests (``-m gpu``) of a batch of label images cut as one region graph (``graph_from_labels_batch``,
``mgc_labels_create_batch``, ``mgc_sparse_get_segment_energies``).

Every image of a batch must come out as its own ``graph_from_labels`` call: the fetched edges equal that image's own
``mgc_labels_boundary`` shifted by its node offset, bit for bit (the directed term's duplicated first pair included); the
region sums and atlas t-links are bit-identical; the mask equals the single call's and BK's (oracle.solvers); the energy
is within 1e-9 relative of both, and equal for integer capacities.  Fixtures come from tests/golden/ only.
"""
import os
import sys

import numpy
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import solvers  # noqa: E402

pytestmark = pytest.mark.gpu
os.environ.setdefault("MEDPY_GC_SPARSE_TIMEOUT", "30")

G = numpy.load(os.path.join(HERE, "golden", "golden_labels_v1.npz"))
NAMES = [str(n) for n in G["names"]]
FULL = [n for n in NAMES if n + "/directed" in G.files]
DTYPES = (numpy.float32, numpy.float64, numpy.uint8, numpy.int16, numpy.int32)


def _gc():
    import medpy_b200.graphcut as gc
    return gc


def _mgc():
    from medpy_b200 import _lib
    return _lib._mgc


def supervoxels(shape, cell, rng):
    """Jittered block labels 1..K over `shape` (every id present)."""
    grids = numpy.meshgrid(*[numpy.arange(s) for s in shape], indexing="ij")
    blocks = [numpy.clip(g + rng.integers(-1, 2, size=shape), 0, s - 1) // cell for g, s in zip(grids, shape)]
    lab = numpy.zeros(shape, numpy.int64)
    for b, s in zip(blocks, shape):
        lab = lab * (-(-s // cell)) + b
    _, inv = numpy.unique(lab, return_inverse=True)
    return (inv + 1).reshape(shape).astype(numpy.int32)


def gradient(shape, dtype, rng):
    if dtype == numpy.uint8:
        return rng.integers(0, 256, size=shape).astype(dtype)
    if dtype in (numpy.int16, numpy.int32):
        g = rng.integers(-300, 300, size=shape).astype(dtype)
        g.flat[0] = numpy.iinfo(dtype).min                # abs() wraps in the native arithmetic, not in the directed one
        return g
    return (rng.random(shape) * 4 - 1).astype(dtype)


def ragged_shapes(ndim, count, rng):
    return [tuple(int(rng.integers(2, 9 if ndim < 4 else 5)) for _ in range(ndim)) for _ in range(count)]


def markers(lab, rng):
    fg = numpy.zeros(lab.shape, bool)
    bg = numpy.zeros(lab.shape, bool)
    fg.flat[0] = True
    bg.flat[lab.size - 1] = True
    fg.flat[rng.integers(0, lab.size)] = True
    return fg, bg


def _native_batch(labs):
    return _mgc().LabelImage.batch([list(l.shape) for l in labs], numpy.concatenate([l.ravel() for l in labs]))


def _bits(a):
    return numpy.ascontiguousarray(a, dtype=numpy.float64).view(numpy.uint64)


@pytest.mark.parametrize("ndim", [1, 2, 3, 4])
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: numpy.dtype(d).name)
def test_edges_and_sums_equal_each_images_own_bit_for_bit(ndim, dtype):
    mgc = _mgc()
    rng = numpy.random.default_rng(10 * ndim + DTYPES.index(dtype))
    shapes = ragged_shapes(ndim, 7, rng)
    labs = [supervoxels(s, 2, rng) for s in shapes]
    labs[3] = numpy.ones(shapes[3], numpy.int32)                # one region: no edge
    grads = [gradient(s, dtype, rng) for s in shapes]
    nat = _native_batch(labs)
    off = nat.batch_offsets()
    assert off.tolist() == numpy.concatenate([[0], numpy.cumsum([l.max() for l in labs])]).tolist()
    assert nat.region_count() == off[-1]
    vals = numpy.concatenate([g.ravel() for g in grads])
    singles = [mgc.LabelImage(l) for l in labs]
    for kind, d in ((mgc.LABELS_ADJACENCY, 0.0), (mgc.LABELS_STAWIASKI, 0.0), (mgc.LABELS_STAWIASKI_DIRECTED, -0.3),
                    (mgc.LABELS_STAWIASKI_DIRECTED, 0.2)):
        got = nat.boundary(kind, None if kind == mgc.LABELS_ADJACENCY else vals, d)
        want = [s.boundary(kind, None if kind == mgc.LABELS_ADJACENCY else g, d) for s, g in zip(singles, grads)]
        assert numpy.array_equal(got[0], numpy.concatenate([w[0] + o for w, o in zip(want, off)]))
        assert numpy.array_equal(got[1], numpy.concatenate([w[1] + o for w, o in zip(want, off)]))
        for k in (2, 3):
            assert numpy.array_equal(_bits(got[k]), _bits(numpy.concatenate([w[k] for w in want]))), kind
    for mode in (mgc.SUM_BINCOUNT, mgc.SUM_PAIRWISE):
        s, c = nat.region_sums(vals, mode)
        want = [x.region_sums(g, mode) for x, g in zip(singles, grads)]
        assert numpy.array_equal(_bits(s), _bits(numpy.concatenate([w[0] for w in want])))
        assert numpy.array_equal(c, numpy.concatenate([w[1] for w in want]))


def test_directed_duplicated_first_pair_per_image():
    """Two regions split at the first voxel of every image: the directed term counts that pair twice, per image."""
    mgc = _mgc()
    labs = [numpy.asarray([1, 2, 2, 2], numpy.int32), numpy.asarray([1, 2, 2], numpy.int32), numpy.asarray([1, 1, 2], numpy.int32)]
    grads = [numpy.asarray([0.5, 1.5, 0.1, 0.2]), numpy.asarray([2.0, 0.0, 1.0]), numpy.asarray([3.0, 1.0, 0.5])]
    nat = _native_batch(labs)
    i, j, w, wr = nat.boundary(mgc.LABELS_STAWIASKI_DIRECTED, numpy.concatenate(grads), -0.25)
    assert i.tolist() == [0, 2, 4] and j.tolist() == [1, 3, 5]
    for b, (l, g) in enumerate(zip(labs, grads)):
        one = mgc.LabelImage(l).boundary(mgc.LABELS_STAWIASKI_DIRECTED, g, -0.25)
        assert _bits(w[b:b + 1]).tolist() == _bits(one[2]).tolist() and _bits(wr[b:b + 1]).tolist() == _bits(one[3]).tolist()


def _single(gc, lab, fg, bg, kw):
    g = gc.graph_from_labels(lab, fg, bg, **kw)
    return g.maxflow(), g.get_mask(), gc.label_cut_mask(g)


def _kw(term, grads, probs):
    """Term keywords: per-image lists for a batch, one image's arrays for a single call."""
    el = _gc().energy_label
    if term == "stawiaski":
        return dict(boundary_term=el.boundary_stawiaski, boundary_term_args=grads)
    if term == "means":
        return dict(boundary_term=el.boundary_difference_of_means, boundary_term_args=grads)
    if term == "directed":
        return dict(boundary_term=el.boundary_stawiaski_directed, boundary_term_args=(grads, -0.2))
    return dict(regional_term=el.regional_atlas, regional_term_args=(probs, 0.05),
                boundary_term=el.boundary_stawiaski, boundary_term_args=grads)


def _check_batch_vs_singles(labs, fgs, bgs, term, grads, probs, integer=False):
    gc = _gc()
    g = gc.graph_from_labels_batch(labs, fgs, bgs, **_kw(term, grads, probs))
    energies = g.maxflow()
    masks, vox = g.get_mask(), g.label_cut_masks()
    assert energies.shape == (len(labs),)
    total = g._graph.maxflow()
    assert energies.sum() == pytest.approx(total, rel=1e-9, abs=1e-12)
    assert numpy.array_equal(_bits(g.maxflow()), _bits(energies))             # the same bits every time
    for b in range(len(labs)):
        flow, mask, v = _single(gc, labs[b], fgs[b], bgs[b], _kw(term, grads[b], None if probs is None else probs[b]))
        assert numpy.array_equal(masks[b], mask), b
        assert numpy.array_equal(vox[b], v), b
        if integer:
            assert energies[b] == flow, b
        else:
            assert energies[b] == pytest.approx(flow, rel=1e-9, abs=1e-12), b
    return g


@pytest.mark.parametrize("term", ["stawiaski", "means", "directed", "atlas"])
@pytest.mark.parametrize("ndim", [1, 2, 3, 4])
def test_whole_cut_equals_single_calls(term, ndim):
    rng = numpy.random.default_rng(100 + ndim)
    shapes = ragged_shapes(ndim, 6, rng)
    labs = [supervoxels(s, 2, rng) for s in shapes]
    fgs, bgs = zip(*[markers(l, rng) for l in labs])
    fgs, bgs = list(fgs), list(bgs)
    bgs[2] = bgs[2] | fgs[2]                                    # a region under both markers
    labs[4] = numpy.ones(shapes[4], numpy.int32)                # one region, under both markers
    grads = [gradient(s, (numpy.float32, numpy.float64, numpy.int16)[ndim % 3], rng) for s in shapes]
    probs = [rng.random(s).astype(numpy.float32) for s in shapes]
    _check_batch_vs_singles(labs, fgs, bgs, term, grads, probs)


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: numpy.dtype(d).name)
def test_dtypes_stacked_and_bk(dtype):
    gc = _gc()
    rng = numpy.random.default_rng(7)
    labs = numpy.stack([supervoxels((12, 10), 3, rng) for _ in range(5)])
    fgs = numpy.zeros(labs.shape, bool)
    bgs = numpy.zeros(labs.shape, bool)
    fgs[:, 5, 5] = True
    bgs[:, 0, :] = True
    grads = numpy.stack([gradient((12, 10), dtype, rng) for _ in range(5)])
    g = _check_batch_vs_singles(list(labs), list(fgs), list(bgs), "stawiaski", list(grads), None)
    g2 = gc.graph_from_labels_batch(labs, fgs, bgs, boundary_term=gc.energy_label.boundary_stawiaski, boundary_term_args=grads)
    assert g2.label_cut_masks().shape == labs.shape
    assert numpy.array_equal(_bits(g2.maxflow()), _bits(g.maxflow()))
    mgc = _mgc()
    for b in range(5):                                          # BK on the image's own graph
        i, j, w, wr = mgc.LabelImage(labs[b]).boundary(mgc.LABELS_STAWIASKI, grads[b], 0.0)
        k = int(labs[b].max())
        fr = numpy.unique(labs[b][fgs[b]] - 1)
        br = numpy.unique(labs[b][bgs[b]] - 1)
        tw = [(fr, numpy.full(fr.size, 65535.0), numpy.zeros(fr.size)), (br, numpy.zeros(br.size), numpy.full(br.size, 65535.0))]
        rflow, rmask, _ = solvers.solve_sparse(k, i, j, w, wr, tw)
        assert numpy.array_equal(g.get_mask()[b], rmask)
        assert g.maxflow()[b] == pytest.approx(rflow, rel=1e-9)


def test_integer_capacities_are_exact():
    """Atlas t-links of an integer atlas with alpha 1 and no boundary term: every capacity is an integer."""
    gc = _gc()
    rng = numpy.random.default_rng(11)
    labs = [supervoxels(s, 2, rng) for s in ((9, 7), (5, 11), (8, 8))]
    fgs, bgs = zip(*[markers(l, rng) for l in labs])
    probs = [rng.integers(-3, 4, size=l.shape).astype(numpy.int32) for l in labs]
    el = gc.energy_label
    g = gc.graph_from_labels_batch(labs, list(fgs), list(bgs), regional_term=el.regional_atlas, regional_term_args=(probs, 1.0))
    again = gc.graph_from_labels_batch(labs, list(fgs), list(bgs), regional_term=el.regional_atlas, regional_term_args=(probs, 1.0))
    assert numpy.array_equal(_bits(g.maxflow()), _bits(again.maxflow()))      # two runs, the same bits
    for b in range(3):
        one = gc.graph_from_labels(labs[b], fgs[b], bgs[b], regional_term=el.regional_atlas, regional_term_args=(probs[b], 1.0))
        assert g.maxflow()[b] == one.maxflow() and numpy.array_equal(g.get_mask()[b], one.get_mask())


def test_batch_of_one_and_512_slices():
    gc = _gc()
    rng = numpy.random.default_rng(5)
    vol = supervoxels((512, 24, 24), 4, rng)
    slices = []
    for z in range(vol.shape[0]):                               # relabel every slice to 1..K
        _, inv = numpy.unique(vol[z], return_inverse=True)
        slices.append((inv + 1).reshape(vol[z].shape).astype(numpy.int32))
    grads = [gradient((24, 24), numpy.float32, rng) for _ in slices]
    fgs, bgs = zip(*[markers(s, rng) for s in slices])
    _check_batch_vs_singles(slices[:1], list(fgs[:1]), list(bgs[:1]), "stawiaski", grads[:1], None)
    g = _check_batch_vs_singles(slices, list(fgs), list(bgs), "stawiaski", grads, None)
    assert len(g.node_offsets) == 513 and g.stats()["images"] == 512


@pytest.mark.parametrize("tag", ["cut_stawiaski", "cut_means", "cut_directed_atlas"])
def test_golden_whole_cuts_as_batches(tag):
    gc = _gc()
    el = gc.energy_label
    # one ragged batch per number of dimensions and gradient dtype (a batch of mixed dtypes is computed in their common
    # one), and for the directed term per directedness and alpha (one of each per batch)
    groups = {}
    for nm in FULL:
        key = (G[nm + "/label"].ndim, G[nm + "/image"].dtype.str)
        if tag == "cut_directed_atlas":
            key += (float(G[nm + "/directedness"]), float(G[nm + "/alpha"]))
        groups.setdefault(key, []).append(nm)
    for names in groups.values():
        labs = [numpy.asfortranarray(G[nm + "/label"]) if bool(G[nm + "/label_forder"]) else G[nm + "/label"] for nm in names]
        imgs = [G[nm + "/image"] for nm in names]
        if tag == "cut_stawiaski":
            kw = dict(boundary_term=el.boundary_stawiaski, boundary_term_args=imgs)
        elif tag == "cut_means":
            kw = dict(boundary_term=el.boundary_difference_of_means, boundary_term_args=imgs)
        else:
            kw = dict(boundary_term=el.boundary_stawiaski_directed,
                      boundary_term_args=(imgs, float(G[names[0] + "/directedness"])),
                      regional_term=el.regional_atlas,
                      regional_term_args=([G[nm + "/prob"] for nm in names], float(G[names[0] + "/alpha"])))
        _golden_check(gc, labs, names, tag, kw)


def _golden_check(gc, labs, names, tag, kw):
    g = gc.graph_from_labels_batch(labs, [G[nm + "/fg"] for nm in names], [G[nm + "/bg"] for nm in names], **kw)
    energies, masks, vox = g.maxflow(), g.get_mask(), g.label_cut_masks()
    for b, nm in enumerate(names):
        want = G[nm + "/" + tag + "_mask"]
        assert numpy.array_equal(masks[b], want), nm
        assert numpy.array_equal(vox[b], want[numpy.asarray(labs[b]) - 1]), nm
        assert energies[b] == pytest.approx(float(G[nm + "/" + tag + "_flow"]), rel=1e-9, abs=1e-300), nm


def test_graphcut_split_batch_matches_pinned_result():
    gc = _gc()
    lab, grad, fg, bg = G["split/label"], G["split/gradient"], G["split/fg"], G["split/bg"]
    split = gc.graphcut_split(gc.graphcut_stawiaski, lab, grad, fg, bg, 10, 3, 2, batch=True)
    assert numpy.array_equal(split, G["split/split_mask"].astype(bool))
    jobs = [(lab[:7, :9], grad[:7, :9], fg[:7, :9], bg[:7, :9]), (lab[3:, 2:], grad[3:, 2:], fg[3:, 2:], bg[3:, 2:])]
    jobs = [j for j in jobs if j[2].any() and j[3].any()]
    got = gc.graphcut_stawiaski_batch(jobs)
    for a, j in zip(got, jobs):
        assert numpy.array_equal(a, gc.graphcut_stawiaski(j))


def test_split_clipped_subvolume_shapes():
    """graphcut_split's sub-volumes of a volume that does not divide evenly: the last ones along an axis are clipped."""
    gc = _gc()
    rng = numpy.random.default_rng(3)
    shape = (47, 35, 29)
    lab = supervoxels(shape, 3, rng)
    grad = gradient(shape, numpy.float32, rng)
    fg = numpy.zeros(shape, bool)
    bg = numpy.zeros(shape, bool)
    for c in (0, 12, 24, 36):                                   # seeds in every sub-volume
        fg[c + 4, ::7, ::7] = True
        bg[min(c + 9, 46), 3::7, 3::7] = True
    one = gc.graphcut_split(gc.graphcut_stawiaski, lab, grad, fg, bg, 12, 4)
    two = gc.graphcut_split(gc.graphcut_stawiaski, lab, grad, fg, bg, 12, 4, batch=True)
    assert numpy.array_equal(one, two)


def test_errors_and_no_markers():
    gc = _gc()
    el = gc.energy_label
    rng = numpy.random.default_rng(2)
    labs = [supervoxels((6, 6), 2, rng) for _ in range(3)]
    fgs, bgs = zip(*[markers(l, rng) for l in labs])
    fgs = list(fgs)
    fgs[1] = numpy.zeros((6, 6), bool)
    with pytest.raises(ValueError, match="label image 1: max"):
        gc.graph_from_labels_batch(labs, fgs, list(bgs), boundary_term=el.boundary_stawiaski,
                                   boundary_term_args=[numpy.ones((6, 6))] * 3)
    bad = list(labs)
    bad[2] = numpy.asarray([[1, 3], [3, 1]], numpy.int32)       # 2 missing: found on the device
    with pytest.raises(AttributeError, match="label image 2"):
        gc.graph_from_labels_batch(bad, list(fgs[:2]) + [numpy.ones((2, 2), bool)], list(bgs[:2]) + [numpy.ones((2, 2), bool)])
    mgc = _mgc()
    s = mgc.SparseGraph(4)
    s.add_tweights(None, numpy.ones(4), numpy.zeros(4))
    with pytest.raises(RuntimeError):
        s.set_option(mgc.OPT_SEGMENT_ENERGIES, 1)               # after add_tweights: MGC_E_STATE
    with pytest.raises(RuntimeError):
        s.segment_energies(numpy.asarray([0, 2, 4]))            # the option is not set


def test_mixed_dtypes_are_computed_in_their_common_dtype():
    """A float32 and a uint8 gradient meet in float32: each image is cut as its own call on the converted gradient."""
    gc = _gc()
    rng = numpy.random.default_rng(8)
    labs = [supervoxels((10, 12), 3, rng), supervoxels((9, 7), 3, rng)]
    grads = [gradient((10, 12), numpy.float32, rng), gradient((9, 7), numpy.uint8, rng)]
    fgs, bgs = zip(*[markers(l, rng) for l in labs])
    g = gc.graph_from_labels_batch(labs, list(fgs), list(bgs), boundary_term=gc.energy_label.boundary_stawiaski,
                                   boundary_term_args=grads)
    for b in range(2):
        flow, mask, _ = _single(gc, labs[b], fgs[b], bgs[b], _kw("stawiaski", grads[b].astype(numpy.float32), None))
        assert numpy.array_equal(g.get_mask()[b], mask)
        assert g.maxflow()[b] == pytest.approx(flow, rel=1e-9, abs=1e-12)
