"""The instance generators of region_cases.py, checked on the CPU: the label volumes hold the region sizes, the long key
run and the voxel-0 border pairs they are built for, the layouts carry the same values, the case table covers every
layout; the general graphs have the geometry their family claims, and BK solves each one that is small enough to solve
here with a non-trivial cut whose energy is the exact capacity of that cut."""
from collections import deque

import numpy
import pytest

import region_cases as rc

SPARSE_GRID_THREADS = 32 * 132 * 256     # grid_for's cap on 132 SMs


@pytest.fixture(scope="module", params=sorted(rc.VOLUMES))
def vol(request):
    return rc.label_volume(request.param)


def _pair_counts(lab):
    """{(lo, hi): number of border voxel pairs} over all axes."""
    keys = []
    for d in range(lab.ndim):
        a = [slice(None)] * lab.ndim
        b = [slice(None)] * lab.ndim
        a[d], b[d] = slice(None, -1), slice(1, None)
        kf, kt = lab[tuple(a)].ravel().astype(numpy.int64), lab[tuple(b)].ravel().astype(numpy.int64)
        v = kf != kt
        keys.append(numpy.minimum(kf, kt)[v] * (1 << 32) + numpy.maximum(kf, kt)[v])
    k, c = numpy.unique(numpy.concatenate(keys), return_counts=True)
    return k, c


def test_region_sizes(vol):
    lab = vol["label"]
    counts = numpy.bincount(lab.ravel())[1:]
    assert counts.size == vol["regions"] and (counts > 0).all()
    assert 10 ** 4 <= vol["regions"] <= 1.2 * 10 ** 5, vol["regions"]
    for size, region in vol["special"].items():
        assert counts[region - 1] == size, (size, counts[region - 1])
    a, bg = vol["stripe"]
    assert counts[a - 1] > rc.BIG_REGION and counts[bg - 1] > rc.BACKGROUND
    assert counts.argmax() == bg - 1
    if lab.ndim in rc.UINT16_DIMS:
        assert vol["regions"] <= 65535


def test_one_key_run_spans_many_blocks(vol):
    keys, counts = _pair_counts(vol["label"])
    a, bg = vol["stripe"]
    longest = int(counts.max())
    assert keys[counts.argmax()] == min(a, bg) * (1 << 32) + max(a, bg)
    assert longest > rc.LONG_RUN and longest > 256 * 300
    # the pair item count takes several chunks per thread in the single-block scan of the block counts
    items = vol["label"].ndim * vol["label"].size
    assert items >= 262144 and (vol["label"].ndim == 1 or items > 262144)


def test_voxel_zero_is_a_border_pair_on_every_axis(vol):
    lab = vol["label"]
    for d in range(lab.ndim):
        idx = [0] * lab.ndim
        idx[d] = 1
        assert lab.flat[0] != lab[tuple(idx)]


def test_layouts_hold_the_same_values(vol):
    lab = vol["label"]
    for kind in rc.LABEL_LAYOUTS:
        if kind == "c_uint16" and lab.ndim not in rc.UINT16_DIMS:
            continue
        got = rc.label_layout(lab, kind)
        assert numpy.array_equal(got, lab), kind
    assert rc.label_layout(lab, "f_int32").flags.f_contiguous
    view = rc.label_layout(lab, "view")
    assert not view.flags.c_contiguous and all(s > 0 for s in view.strides)
    g = rc.gradient(lab.shape, "int16", 1)
    for kind in rc.VALUE_LAYOUTS:
        v = rc.value_layout(g, kind)
        assert numpy.array_equal(v, g), kind
    assert not rc.value_layout(g, "swapped").dtype.isnative
    assert rc.value_layout(g, "f").flags.f_contiguous and not rc.value_layout(g, "view").flags.c_contiguous


def test_case_table_covers_every_layout():
    cases = rc.volume_cases()
    assert set(cases) == {(d, t) for d in rc.VOLUMES for t in rc.DTYPES}
    assert {c["label_layout"] for c in cases.values()} == set(rc.LABEL_LAYOUTS)
    assert {c["grad_layout"] for c in cases.values()} == set(rc.VALUE_LAYOUTS)
    assert {c["atlas_layout"] for c in cases.values()} == set(rc.VALUE_LAYOUTS)
    assert {c["atlas_dtype"] for c in cases.values()} == {"float32", "float64"}
    assert {numpy.sign(c["directedness"]) for c in cases.values()} == {-1.0, 1.0}
    for (ndim, _), c in cases.items():
        assert c["label_layout"] != "c_uint16" or ndim in rc.UINT16_DIMS


@pytest.mark.parametrize("dtype", rc.DTYPES)
def test_gradients_hold_the_extremes(dtype):
    g = rc.gradient((64, 64), dtype, 3)
    assert g.dtype == numpy.dtype(dtype)
    for v in rc.EXTREMES[dtype]:
        assert (g == numpy.asarray(v, dtype=dtype)).any(), v
    assert g.flat[0] == numpy.asarray(rc.EXTREMES[dtype][0], dtype=dtype)
    if numpy.dtype(dtype).kind == "f":
        h = rc.gradient((64, 64), dtype, 3, nonfinite=True)
        assert numpy.isnan(h).any() and numpy.isposinf(h).any() and numpy.isneginf(h).any() and numpy.isnan(h.flat[1])


def test_markers_mark_both_terminals(vol):
    fg, bg = rc.markers(vol["label"], 0)
    assert fg.any() and bg.any() and not (fg & bg).any()


# ---------------------------------------------------------------------------------------------------------------------
# general graphs
# ---------------------------------------------------------------------------------------------------------------------
CPU_SIZED = sorted(n for n in rc.GRAPHS if not n.startswith(("random", "star")))


@pytest.fixture(scope="module", params=CPU_SIZED)
def graph(request):
    case = rc.graph_case(request.param)
    return case, rc.bk(case)


def test_bk_cut_is_non_trivial_and_exact(graph):
    case, (e, m) = graph
    cap = rc.cut_capacity(case, m)
    if case["exact"]:
        assert e == cap, (e, cap)
    else:
        assert abs(e - cap) <= 1e-9 * abs(cap), (e, cap)
    name = case["name"]
    if name == "ties-all-source":
        assert m.all()
    elif name == "ties-all-sink":
        assert not m.any()
    else:
        assert 0 < int(m.sum()) < m.size, (name, int(m.sum()))


def _bfs_depth(case, start):
    n = case["n"]
    adj = [[] for _ in range(n)]
    for a, b in zip(case["i"].tolist(), case["j"].tolist()):
        adj[a].append(b)
        adj[b].append(a)
    dist = [-1] * n
    dist[start] = 0
    q = deque([start])
    while q:
        v = q.popleft()
        for w in adj[v]:
            if dist[w] < 0:
                dist[w] = dist[v] + 1
                q.append(w)
    return dist


@pytest.mark.parametrize("name", [n for n in rc.GRAPHS if n.startswith(("chain", "ladder"))])
def test_chain_depth_and_id_order(name):
    case = rc.graph_case(name)
    assert 1000 <= case["n"] <= 5000
    for end in case["sink_end"]:
        dist = _bfs_depth(case, end)
        assert max(dist) >= case["depth"] >= 999
    # rail 0 holds ids 0 .. steps-1: its sink end is the first or the last of them
    steps = case["depth"] + 1
    assert case["sink_end"][0] == (0 if name.endswith("up") else steps - 1)
    along = case["i"][:steps - 1] - case["j"][:steps - 1]        # each arc of rail 0 points towards the sink end
    assert (along == (1 if name.endswith("up") else -1)).all()


def test_wide_graph_outgrows_the_sparse_grid():
    case = rc.graph_case("wide")
    assert case["n"] > SPARSE_GRID_THREADS * 1.1
    deg = numpy.bincount(numpy.concatenate([case["i"], case["j"]]), minlength=case["n"])
    assert deg.mean() <= 2.0


def test_grid_ids_are_permuted_and_floored():
    case = rc.graph_case("grid3d-permuted")
    assert (numpy.abs(case["i"] - case["j"]) > 256).mean() > 0.9       # neighbours sit in different blocks
    assert (case["cap"] == numpy.finfo(numpy.float64).tiny).any()
    assert any((numpy.asarray(src) == rc.MARKER).any() for _, src, _ in case["tw"])


def test_ties_graphs_have_their_degeneracies():
    z = rc.graph_case("ties-zero-reversed")
    assert (z["cap"] == 0).any() and (z["rev"] == 0).any()
    fwd = set(zip(z["i"].tolist(), z["j"].tolist()))
    assert any((b, a) in fwd for a, b in fwd)
    iso = rc.graph_case("ties-isolated-tlinks")
    assert numpy.bincount(numpy.concatenate([iso["i"], iso["j"]]), minlength=iso["n"]).min() == 0
    assert len(iso["tw"]) == 3 and all((s < 0).any() and (k < 0).any() for _, s, k in iso["tw"])
    assert rc.graph_case("ties-no-edges")["i"].size == 0
    h = rc.graph_case("ties-huge")
    assert h["cap"].max() == 2.0 ** 40
    # every sum the solvers form stays an integer below 2^53
    assert h["cap"].sum() + h["rev"].sum() + sum(numpy.abs(s).sum() + numpy.abs(k).sum() for _, s, k in h["tw"]) < 2.0 ** 53


def test_star_closed_form_equals_bk():
    """The closed-form cut the big star is checked with equals BK on a star small enough for BK."""
    from oracle import solvers
    case = rc.star_graph(16, leaves=3000)
    flow, mask, _ = solvers.solve_sparse(case["n"], case["i"], case["j"], case["cap"], case["rev"], case["tw"])
    e, m = rc.star_cut(case)
    assert e == flow and numpy.array_equal(m, mask)
    big = rc.graph_case("star")
    e, m = rc.bk(big)
    assert e == rc.cut_capacity(big, m) and 0 < int(m.sum()) < m.size
