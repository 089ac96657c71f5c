"""CPU tests of SlabSolver's warm edits (medpy_b200/distributed.py): the MGC_OPT_WARM plumbing, the mapping of global
arguments to each rank's local calls (its owned t-link entries, the n-link pairs with an owned end, the local slice of a
dense form), and the verdicts on bad arguments, which must be the same on every rank -- a NaN that only one rank's planes
hold included -- with no rank folding anything.  Three gloo ranks drive a recording stand-in for the device handle
defined here."""
import os
import pickle
import socket
import sys

import numpy
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPE = (9, 4, 5)
WORLD = 3


class Recorder:
    """The slab handle calls SlabSolver makes, recorded with their arguments as numpy arrays."""

    def __init__(self, shape, z0, z1):
        self.plane = int(numpy.prod(shape[1:]))
        self.calls = []

    def slab_plane_elems(self):
        return self.plane

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)

        def record(*args):
            self.calls.append((name,) + tuple(None if a is None else numpy.array(a) for a in args))
        return record


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _edits():
    """Global arguments of every warm call, the same on every rank."""
    rng = numpy.random.default_rng(7)
    n = int(numpy.prod(SHAPE))
    P = int(numpy.prod(SHAPE[1:]))
    fg = rng.random(SHAPE) < 0.2
    bg = rng.integers(0, n, 30)
    ids = rng.integers(0, n, 40)
    lo = numpy.concatenate([rng.integers(0, n - P, 30), rng.integers(0, n, 30)])
    lo = lo[numpy.r_[numpy.ones(30, bool), (lo[30:] % SHAPE[-1]) + 1 < SHAPE[-1]]]
    hi = lo + numpy.where(numpy.arange(lo.size) < 30, P, 1)
    flip = rng.random(lo.size) < 0.5
    return dict(
        fg=fg, bg=bg, ids=ids, src=rng.normal(size=40), snk=rng.normal(size=40),
        dsrc=rng.normal(size=SHAPE), dsnk=rng.normal(size=SHAPE),
        i=numpy.where(flip, hi, lo), j=numpy.where(flip, lo, hi), cap=rng.random(lo.size), rev=rng.random(lo.size),
        f0=rng.random(SHAPE), b0=rng.random(SHAPE), f2=rng.random(SHAPE), b2=rng.random(SHAPE))


def _bad_calls(E):
    """(name, call) pairs that every rank must refuse alike."""
    from medpy_b200.distributed import slab_bounds
    z1 = slab_bounds(SHAPE[0], WORLD, 1)
    nan_owned_by_1 = E["dsrc"].copy()
    nan_owned_by_1[(z1[0] + z1[1]) // 2, 1, 1] = numpy.nan     # inside rank 1's planes only
    nan_ghost_of_0 = E["dsrc"].copy()
    nan_ghost_of_0[z1[0], 2, 2] = numpy.nan                    # rank 1's first plane: rank 0's upper ghost plane
    nan_axis0 = E["f0"].copy()
    nan_axis0[z1[1] - 1, 0, 0] = numpy.nan                      # rank 1's last plane, rank 2's lower ghost plane
    neg_axis2 = E["f2"].copy()
    neg_axis2[SHAPE[0] - 1, 3, 1] = -1.0                        # the last rank's planes only
    nan_list = E["src"].copy()
    nan_list[numpy.flatnonzero(E["ids"] >= slab_bounds(SHAPE[0], WORLD, 2)[0] * 20)[0]] = numpy.nan
    n = int(numpy.prod(SHAPE))
    return [
        ("dense_tlink_nan_rank1", lambda s: s.add_tweights_warm(None, nan_owned_by_1, E["dsnk"])),
        ("dense_tlink_nan_ghost", lambda s: s.add_tweights_warm(None, E["dsnk"], nan_ghost_of_0)),
        ("dense_nlink_nan_axis0", lambda s: s.add_nweights_dense_warm(0, nan_axis0, E["b0"])),
        ("dense_nlink_negative", lambda s: s.add_nweights_dense_warm(2, neg_axis2, E["b2"])),
        ("list_tlink_nan", lambda s: s.add_tweights_warm(E["ids"], nan_list, E["snk"])),
        ("seed_range", lambda s: s.add_seeds(numpy.array([0, n]), None)),
        ("pair_not_neighbours", lambda s: s.add_nweights_warm(numpy.array([0, 3]), numpy.array([1, 5]), 1.0, 1.0)),
        ("pair_across_a_row", lambda s: s.add_nweights_warm(numpy.array([SHAPE[-1] - 1]), numpy.array([SHAPE[-1]]), 1.0, 1.0)),
        ("nlink_negative", lambda s: s.add_nweights_warm(E["i"], E["j"], -E["cap"], E["rev"])),
        ("nlink_nan", lambda s: s.add_nweights_warm(E["i"][:3], E["j"][:3], numpy.array([1.0, numpy.nan, 1.0]), 0.0)),
        ("axis", lambda s: s.add_nweights_dense_warm(3, E["f0"], E["b0"])),
        ("shape", lambda s: s.add_nweights_dense_warm(0, E["f0"][1:], E["b0"][1:])),
    ]


def _worker(rank, world, port, out):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from medpy_b200.distributed import SlabSolver
    E = _edits()
    s = SlabSolver(SHAPE, handle_factory=Recorder, warm=True)
    s.add_seeds(E["fg"], E["bg"])
    s.remove_seeds(E["bg"], None)
    s.add_tweights_warm(E["ids"], E["src"], E["snk"])
    s.add_tweights_warm(None, E["dsrc"], E["dsnk"])
    s.add_nweights_warm(E["i"], E["j"], E["cap"], E["rev"])
    s.add_nweights_dense_warm(0, E["f0"], E["b0"])
    s.add_nweights_dense_warm(2, E["f2"], E["b2"])
    good = list(s.handle.calls)
    verdicts = {}
    for name, call in _bad_calls(E):
        before = len(s.handle.calls)
        try:
            call(s)
            verdicts[name] = None
        except ValueError as exc:
            verdicts[name] = str(exc)
        assert len(s.handle.calls) == before, name
    with open(out % rank, "wb") as fh:
        pickle.dump(dict(calls=good, verdicts=verdicts), fh)
    dist.destroy_process_group()


@pytest.fixture(scope="module")
def ranks(tmp_path_factory):
    import torch.multiprocessing as mp
    out = str(tmp_path_factory.mktemp("slab_warm") / "r%d.pkl")
    mp.spawn(_worker, args=(WORLD, _free_port(), out), nprocs=WORLD, join=True)
    res = []
    for r in range(WORLD):
        with open(out % r, "rb") as fh:
            res.append(pickle.load(fh))
    return res


def _expect(rank):
    """The local calls rank `rank` must make, computed from the global arguments."""
    from medpy_b200 import _lib
    from medpy_b200.distributed import slab_bounds
    E = _edits()
    P = int(numpy.prod(SHAPE[1:]))
    z0, z1 = slab_bounds(SHAPE[0], WORLD, rank)
    a, b = z0 - (1 if z0 > 0 else 0), z1 + (1 if z1 < SHAPE[0] else 0)
    own = lambda x: (x >= z0 * P) & (x < z1 * P)  # noqa: E731
    loc = lambda x: x - a * P  # noqa: E731
    fg = numpy.flatnonzero(E["fg"])
    keep = own(E["i"]) | own(E["j"])
    t = own(E["ids"])
    return [
        ("set_option", numpy.array(_lib._mgc.OPT_WARM), numpy.array(1)),
        ("add_seeds", loc(fg[own(fg)]), loc(E["bg"][own(E["bg"])])),
        ("remove_seeds", loc(E["bg"][own(E["bg"])]), None),
        ("add_tweights_warm", loc(E["ids"][t]), E["src"][t], E["snk"][t]),
        ("add_tweights_warm", None, E["dsrc"][a:b].ravel(), E["dsnk"][a:b].ravel()),
        ("add_nweights_warm", loc(E["i"][keep]), loc(E["j"][keep]), E["cap"][keep], E["rev"][keep]),
        ("add_nweights_dense_warm", numpy.array(0), E["f0"][a:b], E["b0"][a:b]),
        ("add_nweights_dense_warm", numpy.array(2), E["f2"][a:b], E["b2"][a:b]),
    ]


@pytest.mark.parametrize("rank", range(WORLD))
def test_each_rank_folds_what_it_owns(ranks, rank):
    got, want = ranks[rank]["calls"], _expect(rank)
    assert [c[0] for c in got] == [c[0] for c in want]
    for g, w in zip(got, want):
        assert len(g) == len(w), g[0]
        for x, y in zip(g[1:], w[1:]):
            assert (x is None) == (y is None), g[0]
            if x is not None:
                assert x.shape == numpy.shape(y) and numpy.array_equal(x, y), g[0]
    # every t-link call lands on exactly one rank, every n-link pair on one or two
    E = _edits()
    t = sum(r["calls"][3][1].size for r in ranks)
    assert t == E["ids"].size


def test_every_rank_gives_the_same_verdict(ranks):
    names = [n for n, _ in _bad_calls(_edits())]
    for name in names:
        v = [r["verdicts"][name] for r in ranks]
        assert v[0] is not None, name
        assert all(x == v[0] for x in v), (name, v)


def test_option_plumbing():
    """warm=True sets MGC_OPT_WARM before anything else reaches the handle; warm=False makes no such call."""
    sys.path.insert(0, ROOT)
    from medpy_b200.distributed import SlabSolver
    s = SlabSolver(SHAPE, rank=0, world=1, handle_factory=Recorder)
    assert s.handle.calls == [] and not s.warm
    s = SlabSolver(SHAPE, rank=0, world=1, handle_factory=Recorder, warm=True)
    assert [c[0] for c in s.handle.calls] == ["set_option"] and s.warm
    assert not hasattr(SlabSolver, "remove_nweights_warm") and not hasattr(SlabSolver, "remove_nweights_dense_warm")
