"""Seeded 3-D lattice instances built to stress the easy-instance schedule of the tile solver: the label window, the capped
first global relabel, lazy materialisation, the partial relabel reset and warm re-solves.  No tests live here
(test_lattice_cases.py checks the generators on the CPU, test_gpu_solver_matrix.py solves them on the GPU).

Every instance is a dict:

* ``name``, ``family``;
* ``kind``: ``"fused"`` -- ``vol`` holds graph_from_voxels' inputs (regional_probability_map when ``vol["prob"]`` is set,
  boundary_difference_exponential always, markers), the path that builds lazily; or ``"dense"`` -- ``src`` / ``snk`` (flat
  t-links) and ``there`` / ``back`` (per axis, extent D-1 along it) for GCGraph.set_tweights_dense / set_nweights_dense,
  the per-term path with the eager push state;
* ``prob``: the oracle.energy_terms.build_problem dict of the same graph (the BK solvers' input);
* ``exact``: every capacity is an integer, so every energy is exact;
* geometry for the CPU checks: ``rungs`` (shell thickness, core slices), ``path`` (voxel ids of a tube / corridor in
  order, sink end last), ``no_sink``;
* ``seeds``: voxel ids for warm refinements (``deep``: inside a core deeper than the first relabel's cap; ``stuck``:
  source-side voxels whose excess never reaches a sink, the tiles the window drops; ``far``: sink-side background).

At least 64 tiles of 8^3 each: below that the solver never classifies an instance as easy and none of this code runs.
"""
import math

import numpy

TILE = 8
WINDOW = 8          # PUSH_WINDOW of the push passes
CAP = 12            # FIRST_RELABEL_CAP of the first global relabel
CORE = 4            # edge of a ladder core; cores start at 7 mod 8, so they straddle tile faces, edges and corners


def _tiles(shape):
    return int(numpy.prod([math.ceil(s / TILE) for s in shape]))


def _check_tiles(shape):
    assert len(shape) == 3 and _tiles(shape) >= 64, (shape, _tiles(shape))


def _sigma(image):
    from medpy_b200 import synthetic
    return synthetic.rms_neighbour_difference(image)


def easy_by_default(prob):
    """How the solver classifies the instance at its first relabel: hard when more than 1/8 of the tiles hold a voxel
    without a sink link (the first relabel's worklist; every voxel here has residual out-arcs), easy otherwise."""
    shape = tuple(prob["shape"])
    unlabelled = numpy.asarray(prob["tr"]).reshape(shape) >= 0
    pad = [(0, -s % TILE) for s in shape]
    u = numpy.pad(unlabelled, pad)
    nt = [u.shape[d] // TILE for d in range(3)]
    per_tile = u.reshape(nt[0], TILE, nt[1], TILE, nt[2], TILE).any(axis=(1, 3, 5))
    return int(per_tile.sum()) <= _tiles(shape) // 8


def _fused(name, family, vol, **extra):
    from oracle import energy_terms as et
    _check_tiles(vol["fg"].shape)
    regional = (vol["prob"], vol["alpha"]) if vol.get("prob") is not None else None
    prob = et.build_problem(vol["fg"], vol["bg"], regional=regional,
                            boundary=("difference_exponential", vol["image"], vol["sigma"], False))
    return dict(dict(rungs=[], path=None, no_sink=False, seeds=None), name=name, family=family, kind="fused", vol=vol,
                prob=prob, exact=False, easy=easy_by_default(prob), **extra)


def _dense(name, family, shape, t, there, back, exact, **extra):
    """t: net t-link per voxel (positive: source link); there / back: per-axis arc capacities p -> p+e_d / p+e_d -> p."""
    from oracle import energy_terms as et
    _check_tiles(shape)
    src = numpy.maximum(t, 0.0).ravel()
    snk = numpy.maximum(-t, 0.0).ravel()
    tr = numpy.zeros(src.size)
    flow = et.add_tweights_pass(tr, 0.0, src, snk)
    zeros = numpy.zeros(src.size, numpy.uint8)
    prob = dict(shape=tuple(shape), wf=et.dense_axis_arrays(shape, there), wb=et.dense_axis_arrays(shape, back),
                tr=tr, flow_const=flow, fg=zeros, bg=zeros, src=src, snk=snk)
    return dict(dict(rungs=[], path=None, no_sink=False, seeds=None), name=name, family=family, kind="dense", src=src,
                snk=snk, there=there, back=back, prob=prob, exact=exact, easy=easy_by_default(prob), **extra)


# ------------------------------------------------------------------------------------------------- track A: fused terms
def _ladder_volume(shape, rungs, seed, image_dtype, prob_dtype):
    """Source cores (p ~ 0.9) of CORE^3 voxels, each inside a shell of the given thickness without t-links (p = 0.5
    exactly), in a background of sink links (p ~ 0.2).  rungs: (shell, core origin); a core's nearest sink link is
    shell + 1 arcs away.  The shell is 30 grey levels above the background and the core 50 above the shell, so each
    core keeps most of its excess and the rest crosses the shell."""
    rng = numpy.random.default_rng(seed)
    image = rng.normal(0.0, 10.0, size=shape)
    p = 0.2 + rng.uniform(-0.05, 0.05, size=shape)
    fg = numpy.zeros(shape, bool)
    boxes = numpy.zeros(shape, numpy.int32)
    out = []
    for shell, origin in rungs:
        assert all(o % TILE == TILE - 1 for o in origin), origin
        box = tuple(slice(o - shell, o + CORE + shell) for o in origin)
        core = tuple(slice(o, o + CORE) for o in origin)
        assert all(b.start >= 1 and b.stop <= s - 1 for b, s in zip(box, shape)), (shell, origin, shape)
        # boxes neither overlap nor touch: a background voxel separates every two
        grown = tuple(slice(b.start - 1, b.stop + 1) for b in box)
        assert not boxes[grown].any(), (shell, origin)
        boxes[box] += 1
        image[box] += 30.0
        image[core] += 50.0
        p[box] = 0.5                        # exact in every float type: src == snk, so the shell has no t-link
        p[core] = 0.9 + rng.uniform(-0.04, 0.04, size=(CORE,) * 3)
        out.append((shell, core))
    kind = numpy.dtype(image_dtype).kind
    if kind == "u":
        image = numpy.clip(numpy.round(image + 100.0), 0, 255)
    elif kind == "i":
        image = numpy.round(image)
    image = image.astype(image_dtype)
    vol = dict(image=image, prob=p.astype(prob_dtype), alpha=0.1, fg=fg, bg=numpy.zeros(shape, bool), sigma=_sigma(image))
    return vol, out


def _ladder_seeds(shape, rungs):
    deepest = max(rungs, key=lambda r: r[0])[1]
    shallow = min(rungs, key=lambda r: r[0])[1]
    ids = numpy.arange(int(numpy.prod(shape)), dtype=numpy.int64).reshape(shape)
    # `stuck`: the shallowest core, which keeps its excess on the source side; its tiles are meant to be the ones the
    # window drops, by design -- the statistics only count dropped tiles, they do not say which
    return dict(deep=ids[deepest].ravel()[::5], stuck=ids[shallow].ravel()[::3], far=ids[-1, -1, -6:])


def ladder(variant):
    """A1: depth ladders.  Shell thicknesses 7, 8, 9 straddle the push window, 11, 12, 13 the first relabel's cap; 24 and
    40 lie far beyond both.  Variants 0 and 2 leave enough sink-linked tiles around their rungs to be easy instances
    under the default options; variant 1 (deep rungs only) is solved as a hard one unless the classification is forced."""
    spec = {
        0: ((96, 96, 224), [(7, (23, 23, 23)), (8, (23, 23, 71)), (9, (23, 71, 23)), (11, (71, 23, 23)),
                           (12, (71, 71, 23)), (13, (71, 71, 71))]),
        1: ((96, 96, 160), [(40, (47, 47, 47)), (24, (47, 47, 127))]),
        2: ((128, 128, 192), [(7, (23, 23, 23)), (12, (23, 23, 47)), (24, (31, 31, 95))]),
    }[variant]
    shape, rungs = spec
    vol, out = _ladder_volume(shape, rungs, seed=100 + variant, image_dtype=numpy.float32, prob_dtype=numpy.float32)
    return _fused("a1-ladder-s%d" % variant, "A1", vol, rungs=out, seeds=_ladder_seeds(shape, out))


_A4 = {
    # name: shape, image dtype, probability dtype
    "oddx": ((64, 64, 61), numpy.float64, numpy.float64),       # odd X: the non-TMA push and the full read-out
    "x4": ((64, 64, 60), numpy.int16, numpy.float32),           # X % 4 == 0, X % 8 != 0: clean read-out over partial tiles
    "ragged": ((61, 53, 64), numpy.uint8, numpy.float64),       # partial tiles along Z and Y
}
A4_RUNGS = [(13, (15, 15, 15)), (9, (47, 39, 15)), (7, (47, 15, 47))]


def ladder_shapes(variant):
    """A4: a three-rung ladder on shapes and dtypes that select other code paths."""
    shape, idt, pdt = _A4[variant]
    vol, out = _ladder_volume(shape, A4_RUNGS, seed=200 + sorted(_A4).index(variant), image_dtype=idt, prob_dtype=pdt)
    return _fused("a4-%s" % variant, "A4", vol, rungs=out, seeds=_ladder_seeds(shape, out))


# waypoints of a serpentine in a 64^3 lattice: every leg runs along one axis, all six directions occur, and every
# centre-line coordinate is 7 mod 8, so the tube straddles tile faces along its legs and tile edges / corners at its turns
SERPENTINE = [(7, 7, 7), (7, 7, 55), (7, 55, 55), (23, 55, 55), (23, 55, 7), (23, 23, 7), (39, 23, 7), (39, 23, 55),
              (55, 23, 55), (55, 47, 55), (39, 47, 55), (39, 47, 23)]


def _polyline(points):
    """Voxel coordinates along the polyline, in order."""
    line = []
    for a, b in zip(points[:-1], points[1:]):
        axis = next(d for d in range(len(a)) if a[d] != b[d])
        step = 1 if b[axis] > a[axis] else -1
        for c in range(a[axis], b[axis], step):
            q = list(a)
            q[axis] = c
            line.append(tuple(q))
    line.append(tuple(points[-1]))
    return line


def _tube_mask(shape, line, width):
    lo = (width - 1) // 2
    m = numpy.zeros(shape, bool)
    for q in line:
        m[tuple(slice(c - lo, c - lo + width) for c in q)] = True
    return m


def serpentine(width):
    """A2: a tube `width` voxels wide along SERPENTINE, 100 grey levels above the background; weak source links along it
    (p ~ 0.51), sink links only around its last 4 centre-line voxels (p = 0.3), sink links everywhere
    outside it.  Once the weak arcs across the wall are saturated the excess has to travel along the tube, through many
    label windows, and more excess arrives than the end's sink links take.  The lattice extends beyond the serpentine's
    64^3 corner so that the instance is an easy one."""
    shape = (128, 128, 64)
    rng = numpy.random.default_rng(300 + width)
    line = _polyline(SERPENTINE)
    tube = _tube_mask(shape, line, width)
    end = _tube_mask(shape, line[-4:], width)
    image = rng.normal(0.0, 10.0, size=shape).astype(numpy.float32)
    image[tube] += 100.0
    p = (0.2 + rng.uniform(-0.05, 0.05, size=shape)).astype(numpy.float32)
    p[tube] = (0.51 + rng.uniform(0.0, 0.02, size=int(tube.sum()))).astype(numpy.float32)
    p[end] = 0.3
    vol = dict(image=image, prob=p, alpha=0.1, fg=numpy.zeros(shape, bool), bg=numpy.zeros(shape, bool),
               sigma=_sigma(image))
    path = numpy.array([numpy.ravel_multi_index(q, shape) for q in line], numpy.int64)
    # `stuck`: the tube's far end, which the design leaves on the source side (its tiles are meant to be dropped once
    # their excess is stuck; the statistics only count dropped tiles, they do not say which)
    seeds = dict(deep=path[len(path) // 2: len(path) // 2 + 4], stuck=path[:6],
                 far=numpy.arange(numpy.ravel_multi_index((60, 2, 2), shape), numpy.ravel_multi_index((60, 2, 2), shape) + 6))
    return _fused("a2-serp-w%d" % width, "A2", vol, path=path, seeds=seeds)


def far_sink(with_sink):
    """A3: source blobs (p ~ 0.9, 40 grey levels up) in a lattice without t-links (p = 0.5), sink links only on the
    x = X-1 face -- or nowhere.  Every source voxel is at least 48 arcs from a sink link, so the capped first relabel
    labels none of them and round 1 pushes nothing."""
    shape = (64, 64, 96)
    rng = numpy.random.default_rng(400 + int(with_sink))
    image = rng.normal(0.0, 10.0, size=shape).astype(numpy.float32)
    p = numpy.full(shape, 0.5, numpy.float32)
    z, y, x = numpy.ogrid[:shape[0], :shape[1], :shape[2]]
    ball = (z - 31) ** 2 + (y - 31) ** 2 + (x - 23) ** 2 <= 64
    cube = numpy.zeros(shape, bool)
    cube[7:15, 47:55, 39:47] = True
    for src in (ball, cube):
        image[src] += 40.0
        p[src] = (0.9 + rng.uniform(-0.04, 0.04, size=int(src.sum()))).astype(numpy.float32)
    if with_sink:
        p[:, :, -1] = (0.2 + rng.uniform(-0.05, 0.05, size=shape[:2])).astype(numpy.float32)
    vol = dict(image=image, prob=p, alpha=0.1, fg=numpy.zeros(shape, bool), bg=numpy.zeros(shape, bool),
               sigma=_sigma(image))
    return _fused("a3-%s" % ("face" if with_sink else "nosink"), "A3", vol, no_sink=not with_sink)


def forced_easy(size):
    """A5: the boundary-only two-blob volume (BASELINE config 2 style: sink links only on the marker shell).  A hard
    instance; run with MEDPY_GC_SWEEP_FRAC=1 it is solved as an easy one, and the capped first relabel leaves most of
    the lattice unlabelled."""
    from medpy_b200 import synthetic
    vol = synthetic.two_blob_volume((size,) * 3, seed=500 + size, with_prob=False)
    vol["prob"] = None
    return _fused("a5-blobs-%d" % size, "A5", vol)


# ------------------------------------------------------------------------------------------------ track B: dense terms
def _random_arcs(rng, shape, draw):
    there, back = [], []
    for d in range(3):
        short = list(shape)
        short[d] -= 1
        there.append(draw(rng, short))
        back.append(draw(rng, short))
    return there, back


def integer_ties(variant):
    """B1: n-weights drawn independently per direction from {1, 2, 3}, t-links from {-3 .. 3}: a graph with many minimum
    cuts.  The set of voxels that cannot reach the sink is the same for every maximum preflow, so the mask must still be
    BK's bit for bit.  Variant 0: inside two balls the t-links are drawn from {-1 .. 3}, outside from {-3 .. 1}.
    Variant 1 keeps the sink links ({-3 .. 2}) in the first tile plane along X; beyond it 5 % of the
    voxels carry a source link of 1, up to 88 arcs from the nearest sink link."""
    shape = ((40, 48, 56), (48, 48, 96))[variant]
    rng = numpy.random.default_rng(600 + variant)
    if variant == 0:
        z, y, x = numpy.ogrid[:shape[0], :shape[1], :shape[2]]
        balls = ((z - 15) ** 2 + (y - 15) ** 2 + (x - 15) ** 2 <= 100) | ((z - 25) ** 2 + (y - 31) ** 2 + (x - 39) ** 2 <= 144)
        t = numpy.where(balls, rng.integers(-1, 4, size=shape), rng.integers(-3, 2, size=shape)).astype(numpy.float64)
    else:
        t = (rng.random(shape) < 0.05).astype(numpy.float64)
        t[:, :, :TILE] = rng.integers(-3, 3, size=shape[:2] + (TILE,))
    there, back = _random_arcs(rng, shape, lambda r, s: r.integers(1, 4, size=s).astype(numpy.float64))
    return _dense("b1-ties-s%d" % variant, "B1", shape, t, there, back, exact=True)


MAZE_BRANCHES = [((7, 7, 31), (7, 15, 31)), ((23, 55, 31), (15, 55, 31)), ((39, 23, 31), (39, 35, 31))]


def integer_maze(embedded):
    """B2: a one-voxel corridor along SERPENTINE with three dead-end branches; arcs between corridor voxels carry 1000,
    every other arc 1.  Sources (3000) sit at the far end and the branches' dead ends, sink links (-1000) on the
    corridor's last 4 voxels; the corridor is 3 times the first relabel's cap long many times over.

    embedded=False: the maze is the whole 64^3 lattice and the corridor's end holds its only sink links -- every tile
    holds a voxel without one, so the solver classifies it as hard.  embedded=True: the maze block sits inside a
    128 x 128 x 160 lattice whose other voxels have a sink link of 1, so it is an easy instance under the default
    options; its sources lie 8, 8, 9 and 17 arcs from the nearest sink link (the last beyond the cap), and the walls
    leak to the sink-linked surroundings as well as to the exit."""
    shape, off = ((128, 128, 160), (32, 32, 48)) if embedded else ((64, 64, 64), (0, 0, 0))

    def shift(points):
        return [tuple(c + o for c, o in zip(q, off)) for q in points]

    line = _polyline(shift(SERPENTINE))
    corridor = _tube_mask(shape, line, 1)
    ends = [line[0]]
    for a, b in MAZE_BRANCHES:
        corridor |= _tube_mask(shape, _polyline(shift([a, b])), 1)
        ends.append(shift([b])[0])
    t = numpy.zeros(shape)
    if embedded:
        t[...] = -1.0
        t[tuple(slice(o, o + 64) for o in off)] = 0.0
    for q in ends:
        t[q] = 3000.0
    for q in line[-4:]:
        t[q] = -1000.0
    there, back = [], []
    for d in range(3):
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[d], hi[d] = slice(0, -1), slice(1, None)
        w = numpy.where(corridor[tuple(lo)] & corridor[tuple(hi)], 1000.0, 1.0)
        there.append(w)
        back.append(w.copy())
    path = numpy.array([numpy.ravel_multi_index(q, shape) for q in line], numpy.int64)
    return _dense("b2-maze-embedded" if embedded else "b2-maze", "B2", shape, t, there, back, exact=True, path=path)


def dynamic_range():
    """B3: capacities 10**U(-9, 6) on every arc and t-link (random sign), and every 27th voxel strongly source linked
    (1e6 .. 2e6) with all its arcs in 10**U(-9, -6): the solver's source clamp and rounded subtractions over fifteen
    decades."""
    shape = (48, 48, 64)
    rng = numpy.random.default_rng(700)
    t = 10.0 ** rng.uniform(-9, 6, size=shape) * rng.choice([-1.0, 1.0], size=shape)
    strong = numpy.zeros(shape, bool)
    strong[1::3, 1::3, 1::3] = True
    t[strong] = rng.uniform(1e6, 2e6, size=int(strong.sum()))
    there, back = _random_arcs(rng, shape, lambda r, s: 10.0 ** r.uniform(-9, 6, size=s))
    for d in range(3):
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[d], hi[d] = slice(0, -1), slice(1, None)
        touch = strong[tuple(lo)] | strong[tuple(hi)]
        for w in (there[d], back[d]):
            w[touch] = 10.0 ** rng.uniform(-9, -6, size=int(touch.sum()))
    return _dense("b3-range", "B3", shape, t, there, back, exact=False)


# ------------------------------------------------------------------------------------------------------------ registry
CASES = {}
for _v in (0, 1, 2):
    CASES["a1-ladder-s%d" % _v] = (lambda v=_v: ladder(v))
for _w in (2, 3):
    CASES["a2-serp-w%d" % _w] = (lambda w=_w: serpentine(w))
CASES["a3-face"] = lambda: far_sink(True)
CASES["a3-nosink"] = lambda: far_sink(False)
for _k in _A4:
    CASES["a4-%s" % _k] = (lambda k=_k: ladder_shapes(k))
for _s in (48, 64):
    CASES["a5-blobs-%d" % _s] = (lambda s=_s: forced_easy(s))
for _v in (0, 1):
    CASES["b1-ties-s%d" % _v] = (lambda v=_v: integer_ties(v))
CASES["b2-maze"] = lambda: integer_maze(False)
CASES["b2-maze-embedded"] = lambda: integer_maze(True)
CASES["b3-range"] = dynamic_range


def make(name):
    return CASES[name]()


def family(name):
    return name.split("-")[0].upper()


# ------------------------------------------------------------------------------------------------------------- oracles
def cut_capacity(prob, mask):
    """Capacity of the cut `mask` (1 = source side) over the float64 capacities of `prob`, correctly rounded (math.fsum):
    the add_tweights constant, the source link of every sink-side voxel, the sink link of every source-side voxel, and
    every arc from the source side to the sink side."""
    shape = tuple(prob["shape"])
    s = numpy.asarray(mask).reshape(shape).astype(bool)
    tr = numpy.asarray(prob["tr"]).reshape(shape)
    terms = [numpy.array([prob["flow_const"]]), tr[~s & (tr > 0)], -tr[s & (tr < 0)]]
    for d in range(len(shape)):
        lo = [slice(None)] * len(shape)
        hi = [slice(None)] * len(shape)
        lo[d], hi[d] = slice(0, -1), slice(1, None)
        lo, hi = tuple(lo), tuple(hi)
        wf = numpy.asarray(prob["wf"][d]).reshape(shape)[lo]
        wb = numpy.asarray(prob["wb"][d]).reshape(shape)[lo]
        terms.append(wf[s[lo] & ~s[hi]])
        terms.append(wb[s[hi] & ~s[lo]])
    return math.fsum(numpy.concatenate([t.ravel() for t in terms]).tolist())


def reversed_problem(prob):
    """The same graph with source and sink exchanged and every arc reversed (for solvers.solve_port, which reads the net
    t-links): its BK mask is 0 exactly on the voxels the source reaches in the residual graph of any maximum flow of
    `prob`, the smallest source side of a minimum cut of `prob`."""
    return dict(prob, tr=-numpy.asarray(prob["tr"]), wf=prob["wb"], wb=prob["wf"], src=None, snk=None)


_BK = {}


def bk(case):
    """(energy, mask) of the BK restatement on the case's problem, cached per instance."""
    from oracle import solvers
    if case["name"] not in _BK:
        e, m, _ = solvers.solve_port(case["prob"])
        _BK[case["name"]] = (e, m)
    return _BK[case["name"]]


_REF = {}


def bk_ref(case):
    """(energy, mask) of the unmodified reference BK where oracle/_ref was built, else None; cached per instance."""
    from oracle import solvers
    if not solvers.have_ref():
        return None
    if case["name"] not in _REF:
        e, m, _ = solvers.solve_ref(case["prob"])
        _REF[case["name"]] = (e, m)
    return _REF[case["name"]]
