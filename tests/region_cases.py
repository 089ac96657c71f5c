"""Seeded instances for the region-graph path: label images at scale for graph_from_labels and the four energy_label
terms, and general graphs for GCGraph and the sparse push-relabel.  No tests live here (test_region_cases.py checks the
generators on the CPU, test_gpu_region_scale.py runs them on the GPU).

Label volumes (``label_volume``), one per dimensionality, laid out along axis 0 in three zones:

* small regions: jittered blocks (``cell`` voxels per axis, each split into ``split`` random parts), with voxel 0 a
  region of its own -- so the first voxel pair of every axis is a border pair -- and C-order runs of exactly 7, 8, 127,
  128 and 129 voxels: the pairwise summation's short loop, its 8-way leaf and its halving tree;
* stripes: region A on the even, the background on the odd coordinates of the last axis, so that the (A, background)
  pair collects more than 10^5 border voxel pairs -- one key run across hundreds of 256-thread blocks;
* background only.

General graphs (``graph_case``) are dicts with ``n``, the sum_edge calls ``i, j, cap, rev`` and the add_tweights calls
``tw`` (a list of (nodes, src, snk) triples, replayed in order), plus ``exact`` (integer capacities whose sums stay
exact in float64) and geometry for the CPU checks.
"""
import math

import numpy

EXACT_SIZES = (1, 7, 8, 127, 128, 129)
RUN_STARTS = (1000, 3000, 5000, 7000, 9000)       # flat index of the first voxel of the 7 .. 129 voxel regions
BIG_REGION = 10 ** 4
BACKGROUND = 10 ** 5
LONG_RUN = 10 ** 5
MARKER = 65535.0

# rows along axis 0 of the small-region zone and of the stripe zone (the rest is background)
VOLUMES = {
    1: dict(shape=(1 << 18,), small=92144, stripe=110000, cell=3, split=1),
    2: dict(shape=(1024, 1024), small=844, stripe=120, cell=3, split=1),
    3: dict(shape=(128, 128, 128), small=116, stripe=8, cell=3, split=1),
    4: dict(shape=(32, 32, 32, 8), small=10, stripe=16, cell=2, split=4),
}

DTYPES = ("float32", "float64", "uint8", "int16", "int32")
EXTREMES = {
    "float32": (0.0, -0.0, 3.0e38, -1.0e-30, 1.0e-45),
    "float64": (0.0, -0.0, 1.0e200, -1.0e300, 5.0e-324),      # (1 / (1 + 1e200))^2 underflows: the DBL_MIN floor
    "uint8": (255, 0),
    "int16": (-32768, 32767, -1),
    "int32": (-2 ** 31, 2 ** 31 - 1, -1),
}
LABEL_LAYOUTS = ("c_int32", "c_int64", "c_uint16", "f_int32", "view")
VALUE_LAYOUTS = ("c", "f", "view", "swapped")
UINT16_DIMS = (1, 4)            # the volumes with at most 65535 regions


def label_volume(ndim):
    """dict(label int32 C-ordered 1..K, regions K, special {size: region id}, stripe (A, background) region ids)."""
    cfg = VOLUMES[ndim]
    shape = cfg["shape"]
    rng = numpy.random.default_rng(700 + ndim)
    idx = numpy.indices(shape, dtype=numpy.int64)
    row, last = idx[0], idx[-1]
    small = row < cfg["small"]
    stripe = (row >= cfg["small"]) & (row < cfg["small"] + cfg["stripe"])
    c = cfg["cell"]
    key = numpy.zeros(shape, numpy.int64)
    for g, s in zip(idx, shape):
        key = key * (-(-s // c) + 1) + numpy.clip(g + rng.integers(-1, 2, size=shape), 0, s - 1) // c
    del idx
    if cfg["split"] > 1:
        key = key * cfg["split"] + rng.integers(0, cfg["split"], size=shape)
    BG, A = 1, 2
    lab = numpy.where(small, key + 3, BG)
    lab[stripe & (last % 2 == 0)] = A
    flat = lab.reshape(-1)
    top = int(flat.max()) + 1
    flat[0] = top
    for k, (start, size) in enumerate(zip(RUN_STARTS, EXACT_SIZES[1:])):
        flat[start:start + size] = top + 1 + k
    _, inv = numpy.unique(flat, return_inverse=True)
    lab = (inv + 1).reshape(shape).astype(numpy.int32)
    flat = lab.reshape(-1)
    special = {1: int(flat[0])}
    special.update({size: int(flat[start]) for start, size in zip(RUN_STARTS, EXACT_SIZES[1:])})
    s0 = cfg["small"] * int(numpy.prod(shape[1:]))          # first voxel of the stripe zone (even last coordinate)
    return dict(label=lab, regions=int(flat.max()), special=special, stripe=(int(flat[s0]), int(flat[-1])),
                shape=shape)


def gradient(shape, dtype, seed, nonfinite=False):
    """A gradient image in `dtype`: moderate values, 1 % of the voxels set to the dtype's extremes (voxel 0 too, so the
    directed term's probing call sees one), and with `nonfinite` also NaN, +inf and -inf at 1 % each."""
    rng = numpy.random.default_rng(seed)
    n = int(numpy.prod(shape))
    dt = numpy.dtype(dtype)
    if dt.kind == "f":
        g = (rng.normal(0.0, 40.0, size=n) * (rng.random(n) > 0.05)).astype(dt)
    else:
        info = numpy.iinfo(dt)
        g = rng.integers(max(int(info.min), -300), min(int(info.max), 300) + 1, size=n).astype(dt)
    ext = numpy.asarray(EXTREMES[dt.name], dtype=dt)
    sel = rng.random(n) < 0.01
    g[sel] = rng.choice(ext, size=int(sel.sum()))
    g[0] = ext[0]
    if nonfinite:
        for v in (numpy.nan, numpy.inf, -numpy.inf):
            g[rng.random(n) < 0.01] = v
        g[1] = numpy.nan         # the successor of voxel 0 along the last axis
    return g.reshape(shape)


def atlas(shape, dtype, seed):
    return numpy.random.default_rng(seed).uniform(0.0, 1.0, size=shape).astype(dtype)


def markers(label, seed):
    """Foreground: the 129-voxel run and 0.1 % of the voxels; background: the last plane along axis 0 and 0.1 %."""
    rng = numpy.random.default_rng(seed)
    fg = rng.random(label.shape) < 0.001
    fg.reshape(-1)[RUN_STARTS[-1]:RUN_STARTS[-1] + 129] = True
    bg = rng.random(label.shape) < 0.001
    bg[-1] = True
    bg &= ~fg
    return fg, bg


def label_layout(lab, kind):
    """The same label image as C int32 / int64 / uint16, Fortran int32, or a strided, offset view into a larger array."""
    if kind == "c_int32":
        return numpy.ascontiguousarray(lab, dtype=numpy.int32)
    if kind == "c_int64":
        return lab.astype(numpy.int64)
    if kind == "c_uint16":
        assert int(lab.max()) <= 65535
        return lab.astype(numpy.uint16)
    if kind == "f_int32":
        return numpy.asfortranarray(lab, dtype=numpy.int32)
    assert kind == "view"
    big = numpy.zeros(lab.shape[:-1] + (2 * lab.shape[-1] + 1,), numpy.int32)
    view = big[..., 1::2]
    view[...] = lab
    return view


def value_layout(a, kind):
    """The same values Fortran-ordered, as a strided view (every other plane of a larger array) or byte-swapped."""
    if kind == "c":
        return numpy.ascontiguousarray(a)
    if kind == "f":
        return numpy.asfortranarray(a)
    if kind == "view":
        big = numpy.zeros((2 * a.shape[0] + 1,) + a.shape[1:], a.dtype)
        view = big[1::2]
        view[...] = a
        return view
    assert kind == "swapped"
    return a.astype(a.dtype.newbyteorder())


def volume_cases():
    """(ndim, gradient dtype) -> the layouts, atlas dtype and directedness sign that case uses; over the table every
    label layout, value layout, atlas dtype and sign occurs."""
    cases = {}
    for ndim in sorted(VOLUMES):
        lay = [k for k in LABEL_LAYOUTS if (k != "f_int32" or ndim > 1) and (k != "c_uint16" or ndim in UINT16_DIMS)]
        for d, dtype in enumerate(DTYPES):
            t = d + ndim
            cases[(ndim, dtype)] = dict(label_layout=lay[t % len(lay)], grad_layout=VALUE_LAYOUTS[t % 4],
                                        atlas_layout=VALUE_LAYOUTS[(t + 1) % 4],
                                        atlas_dtype="float32" if t % 2 else "float64",
                                        directedness=(-1.0 if t % 2 else 1.0) * 10.0 ** -(1 + t % 4),
                                        alpha=0.5 + 0.25 * (t % 3))
    return cases


# ---------------------------------------------------------------------------------------------------------------------
# general graphs
# ---------------------------------------------------------------------------------------------------------------------
def _graph(n, i, j, cap, rev, tw, exact, **extra):
    return dict(dict(kind="general", depth=None, sink_end=None), n=int(n), i=numpy.asarray(i, numpy.int64),
                j=numpy.asarray(j, numpy.int64), cap=numpy.asarray(cap, numpy.float64),
                rev=numpy.asarray(rev, numpy.float64), tw=tw, exact=exact, **extra)


def random_graph(seed, n, m, integer):
    """Uniform random pairs; random t-links plus 5 % marker links to each terminal."""
    rng = numpy.random.default_rng(seed)
    i = rng.integers(0, n, size=m)
    j = rng.integers(0, n, size=m)
    keep = i != j
    i, j = i[keep], j[keep]
    if integer:
        cap = rng.integers(1, 20, size=i.size).astype(float)
        rev = rng.integers(1, 20, size=i.size).astype(float)
        src = rng.integers(0, 30, size=n).astype(float)
        snk = rng.integers(0, 30, size=n).astype(float)
    else:
        cap = rng.uniform(1e-3, 2.0, size=i.size)
        rev = rng.uniform(1e-3, 2.0, size=i.size)
        src = rng.uniform(0.0, 3.0, size=n)
        snk = rng.uniform(0.0, 3.0, size=n)
    fg = rng.choice(n, size=n // 20, replace=False)
    bg = rng.choice(n, size=n // 20, replace=False)
    tw = [(numpy.arange(n), src, snk), (fg, numpy.full(fg.size, MARKER), numpy.zeros(fg.size)),
          (bg, numpy.zeros(bg.size), numpy.full(bg.size, MARKER))]
    return _graph(n, i, j, cap, rev, tw, integer)


def wide_graph(seed, n=1_300_000):
    """More nodes than the sparse kernels' grid holds threads (32 blocks x 256 threads per SM): every kernel runs its
    grid-stride loop.  Each node joins about one partner within 64 ids; integer capacities."""
    rng = numpy.random.default_rng(seed)
    i = rng.integers(0, n - 64, size=n)
    j = i + rng.integers(1, 64, size=n)
    cap = rng.integers(1, 9, size=n).astype(float)
    rev = rng.integers(1, 9, size=n).astype(float)
    t = rng.integers(-6, 7, size=n).astype(float)
    tw = [(numpy.arange(n), numpy.maximum(t, 0.0), numpy.maximum(-t, 0.0))]
    return _graph(n, i, j, cap, rev, tw, True)


def grid_graph(seed, shape):
    """A lattice with Stawiaski-like weights (1 / (1 + g))^2 -- DBL_MIN where g is huge -- marker t-links of 65535 on
    two blobs and on the faces, and node ids randomly permuted so that lattice neighbours sit in different blocks.
    Each weight is scaled by its own factor in [0.5, 1.5): a voxel whose gradient dominates all its pairs would
    otherwise give all its arcs one weight, and the resulting exact ties of the cut are decided by float64 rounding,
    differently by BK and by push-relabel."""
    rng = numpy.random.default_rng(seed)
    n = int(numpy.prod(shape))
    grad = numpy.abs(rng.normal(0.0, 2.0, size=shape))
    grad[rng.random(shape) < 0.02] = 1e200
    perm = rng.permutation(n).reshape(shape)
    ii, jj, ww = [], [], []
    for d in range(len(shape)):
        a = [slice(None)] * len(shape)
        b = [slice(None)] * len(shape)
        a[d], b[d] = slice(None, -1), slice(1, None)
        g = numpy.maximum(grad[tuple(a)], grad[tuple(b)]).ravel()
        w = numpy.maximum((1.0 / (1.0 + g)) ** 2 * rng.uniform(0.5, 1.5, size=g.size), numpy.finfo(numpy.float64).tiny)
        ii.append(perm[tuple(a)].ravel())
        jj.append(perm[tuple(b)].ravel())
        ww.append(w)
    w = numpy.concatenate(ww)
    coords = numpy.indices(shape)
    centre = numpy.asarray(shape) // 3
    fg = sum((c - m) ** 2 for c, m in zip(coords, centre)) <= (min(shape) // 6) ** 2
    bg = numpy.zeros(shape, bool)
    for d in range(len(shape)):
        sl = [slice(None)] * len(shape)
        sl[d] = -1
        bg[tuple(sl)] = True
    fgn, bgn = perm[fg], perm[bg & ~fg]
    tw = [(fgn, numpy.full(fgn.size, MARKER), numpy.zeros(fgn.size)), (bgn, numpy.zeros(bgn.size), numpy.full(bgn.size, MARKER))]
    return _graph(n, numpy.concatenate(ii), numpy.concatenate(jj), w, w.copy(), tw, False, kind="grid")


def star_graph(seed, leaves=100_000):
    """One hub joined to every leaf; the leaves carry random t-links of either sign, the hub a sink link wider than all
    its in-arcs together, so every source-linked leaf pushes into the hub at once (10^5 atomic updates of one excess)."""
    rng = numpy.random.default_rng(seed)
    n = leaves + 1
    i = numpy.zeros(leaves, numpy.int64)
    j = numpy.arange(1, n)
    cap = rng.integers(1, 5, size=leaves).astype(float)
    rev = rng.integers(1, 5, size=leaves).astype(float)
    t = rng.integers(-3, 4, size=leaves).astype(float)
    tw = [(numpy.asarray([0]), numpy.asarray([0.0]), numpy.asarray([5.0 * leaves])),
          (j, numpy.maximum(t, 0.0), numpy.maximum(-t, 0.0))]
    return _graph(n, i, j, cap, rev, tw, True, kind="star")


def star_cut(case):
    """(energy, mask) of a star in closed form: once the hub's side is fixed every leaf picks its cheaper side on its
    own.  BK's mask ("not SINK") is the largest source side among the minimum cuts, so ties go to the source and, when
    both hub sides are optimal, the two optimal source sides are united (BK's scans of the hub's 10^5 arcs make it too
    slow to be the checker at this size)."""
    from oracle import energy_label_terms as elt
    n = case["n"]
    tr, const = elt.add_tweights_replay(n, case["tw"])
    leaf = case["j"]
    assert (case["i"] == 0).all() and numpy.array_equal(numpy.sort(leaf), numpy.arange(1, n))
    a, b, t = case["cap"], case["rev"], tr[leaf]
    keep_src, keep_snk = numpy.maximum(-t, 0.0), numpy.maximum(t, 0.0)        # what a leaf loses on either side
    hub_s = (keep_src, a + keep_snk)          # hub on the source side: leaf S / leaf T
    hub_t = (b + keep_src, keep_snk)          # hub on the sink side
    e_s = max(-tr[0], 0.0) + float(numpy.minimum(*hub_s).sum())
    e_t = max(tr[0], 0.0) + float(numpy.minimum(*hub_t).sum())
    side_s, side_t = hub_s[0] <= hub_s[1], hub_t[0] <= hub_t[1]
    mask = numpy.zeros(n, numpy.uint8)
    if e_s <= e_t:
        mask[0] = 1
        mask[leaf] = side_s | (side_t if e_s == e_t else False)
    else:
        mask[leaf] = side_t
    return min(e_s, e_t) + const, mask


def bipartite_graph(seed, side=300):
    """Every left node joined to every right node; left nodes source-linked, right nodes sink-linked."""
    rng = numpy.random.default_rng(seed)
    n = 2 * side
    left, right = numpy.meshgrid(numpy.arange(side), numpy.arange(side, n), indexing="ij")
    i, j = left.ravel(), right.ravel()
    cap = rng.integers(0, 3, size=i.size).astype(float) + (rng.random(i.size) < 0.5)
    rev = rng.integers(1, 3, size=i.size).astype(float)
    src = rng.integers(100, 600, size=side).astype(float)
    snk = rng.integers(100, 600, size=side).astype(float)
    tw = [(numpy.arange(side), src, numpy.zeros(side)), (numpy.arange(side, n), numpy.zeros(side), snk)]
    return _graph(n, i, j, numpy.maximum(cap, 1.0), rev, tw, True, kind="bipartite")


def chain_graph(seed, length, increasing, rails=1):
    """A chain (rails=1) or a ladder (rails=2: two chains joined by a rung at every step) of `length` steps, sink-linked
    at one end and source-linked at the other, with a bottleneck in the middle.  Node ids grow away from the sink end
    (`increasing`) or towards it, so the BFS from the sink and the flow towards it travel along or against thread
    order."""
    rng = numpy.random.default_rng(seed)
    n = rails * length
    steps = numpy.arange(length)
    ids = steps if increasing else length - 1 - steps          # step 0 is the sink end
    node = numpy.stack([ids + r * length for r in range(rails)])
    ii, jj, cc, rr = [], [], [], []
    for r in range(rails):
        ii.append(node[r, 1:])                                   # away from the sink -> towards it
        jj.append(node[r, :-1])
        c = rng.integers(5, 9, size=length - 1).astype(float)
        c[length // 2] = 2.0 + r                                 # the bottleneck
        cc.append(c)
        rr.append(rng.integers(1, 4, size=length - 1).astype(float))
    if rails == 2:
        ii.append(node[0])
        jj.append(node[1])
        cc.append(numpy.full(length, 1.0))
        rr.append(numpy.full(length, 1.0))
    src_nodes = node[:, -1]
    snk_nodes = node[:, 0]
    tw = [(src_nodes, numpy.full(rails, 50.0), numpy.zeros(rails)), (snk_nodes, numpy.zeros(rails), numpy.full(rails, 50.0))]
    return _graph(n, numpy.concatenate(ii), numpy.concatenate(jj), numpy.concatenate(cc), numpy.concatenate(rr), tw, True,
                  kind="chain", depth=length - 1, sink_end=[int(v) for v in snk_nodes])


def ties_graph(seed, variant):
    """Integer graphs full of equal capacities and degenerate structure."""
    rng = numpy.random.default_rng(seed)
    if variant == "zero_and_reversed":
        # zero-capacity directions, and every pair sent again later in the opposite orientation
        n, m = 3000, 9000
        i = rng.integers(0, n, size=m)
        j = rng.integers(0, n, size=m)
        keep = i != j
        i, j = i[keep], j[keep]
        cap = rng.integers(0, 3, size=i.size).astype(float)
        rev = numpy.where(cap == 0, rng.integers(1, 3, size=i.size), rng.integers(0, 3, size=i.size)).astype(float)
        k = rng.choice(i.size, size=i.size // 2, replace=False)
        i, j, cap, rev = (numpy.concatenate([i, j[k]]), numpy.concatenate([j, i[k]]), numpy.concatenate([cap, rev[k]]),
                          numpy.concatenate([rev, numpy.zeros(k.size)]))
        t = rng.integers(-2, 3, size=n).astype(float)
        tw = [(numpy.arange(n), numpy.maximum(t, 0.0), numpy.maximum(-t, 0.0))]
        return _graph(n, i, j, cap, rev, tw, True)
    if variant == "isolated_and_repeated_tlinks":
        # a third of the nodes have no edge; every node gets three add_tweights calls with either sign
        n = 4000
        i = rng.integers(0, 2 * n // 3, size=6000)
        j = rng.integers(0, 2 * n // 3, size=6000)
        keep = i != j
        i, j = i[keep], j[keep]
        cap = numpy.full(i.size, 2.0)
        rev = numpy.full(i.size, 2.0)
        tw = []
        for _ in range(3):
            nodes = rng.permutation(n)
            tw.append((nodes, rng.integers(-3, 4, size=n).astype(float), rng.integers(-3, 4, size=n).astype(float)))
        return _graph(n, i, j, cap, rev, tw, True)
    if variant == "no_edges":
        n = 5000
        tw = [(numpy.arange(n), rng.integers(0, 3, size=n).astype(float), rng.integers(0, 3, size=n).astype(float))]
        return _graph(n, [], [], [], [], tw, True)
    if variant in ("all_source", "all_sink"):
        n = 20000
        i = numpy.arange(n - 1)
        j = i + 1 + rng.integers(0, 50, size=n - 1) % (n - 1 - i)
        cap = numpy.full(i.size, 1.0)
        rev = numpy.full(i.size, 1.0)
        w = rng.integers(1, 4, size=n).astype(float)
        z = numpy.zeros(n)
        tw = [(numpy.arange(n), w, z)] if variant == "all_source" else [(numpy.arange(n), z, w)]
        return _graph(n, i, j, cap, rev, tw, True)
    assert variant == "huge"
    # capacities up to 2^40 on a random graph: every partial sum of the flow stays below 2^53, so it is exact
    n, m = 20000, 80000
    i = rng.integers(0, n, size=m)
    j = rng.integers(0, n, size=m)
    keep = i != j
    i, j = i[keep], j[keep]
    big = float(2 ** 40)
    cap = numpy.where(rng.random(i.size) < 0.01, big, rng.integers(1, 2 ** 20, size=i.size)).astype(float)
    rev = rng.integers(1, 2 ** 30, size=i.size).astype(float)
    t = numpy.where(rng.random(n) < 0.01, big, rng.integers(1, 2 ** 30, size=n)).astype(float)
    side = rng.random(n) < 0.5
    tw = [(numpy.arange(n), numpy.where(side, t, 0.0), numpy.where(side, 0.0, t))]
    return _graph(n, i, j, cap, rev, tw, True)


GRAPHS = {
    "random-int": lambda: random_graph(11, 200_000, 1_000_000, True),
    "random-float": lambda: random_graph(12, 200_000, 1_000_000, False),
    "wide": lambda: wide_graph(13),
    "grid2d-permuted": lambda: grid_graph(14, (300, 300)),
    "grid3d-permuted": lambda: grid_graph(15, (40, 40, 40)),
    "star": lambda: star_graph(16),
    "bipartite": lambda: bipartite_graph(17),
    "chain-1000-up": lambda: chain_graph(18, 1000, True),
    "chain-5000-down": lambda: chain_graph(19, 5000, False),
    "ladder-2500-up": lambda: chain_graph(20, 2500, True, rails=2),
    "ladder-2500-down": lambda: chain_graph(21, 2500, False, rails=2),
    "ties-zero-reversed": lambda: ties_graph(22, "zero_and_reversed"),
    "ties-isolated-tlinks": lambda: ties_graph(23, "isolated_and_repeated_tlinks"),
    "ties-no-edges": lambda: ties_graph(24, "no_edges"),
    "ties-all-source": lambda: ties_graph(25, "all_source"),
    "ties-all-sink": lambda: ties_graph(26, "all_sink"),
    "ties-huge": lambda: ties_graph(27, "huge"),
}


def graph_case(name):
    return dict(GRAPHS[name](), name=name)


def bk(case):
    """(energy, mask) of the BK solver on the case's call sequence (the reference where built, else its restatement)."""
    from oracle import solvers
    if case["kind"] == "star" and case["n"] > 50_000:
        return star_cut(case)
    flow, mask, _ = solvers.solve_sparse(case["n"], case["i"], case["j"], case["cap"], case["rev"], case["tw"])
    return flow, mask


def cut_capacity(case, mask):
    """Exact capacity of the cut `mask` (1 = source side) of the case's graph, with the add_tweights constants: edges
    from the source side to the sink side plus the t-links each node loses, summed in extended precision."""
    from oracle import energy_label_terms as elt
    lo, hi, a, b = elt.merge_edges(case["i"], case["j"], case["cap"], case["rev"])
    tr, const = elt.add_tweights_replay(case["n"], case["tw"])
    m = numpy.asarray(mask, bool)
    e = math.fsum(a[m[lo] & ~m[hi]].tolist()) + math.fsum(b[m[hi] & ~m[lo]].tolist())
    e += math.fsum(numpy.where(m, numpy.maximum(-tr, 0.0), numpy.maximum(tr, 0.0)).tolist()) + const
    return e
