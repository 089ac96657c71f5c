"""CPU model of the capped global relabel (medpy_b200/csrc/gc_tiles.cuh: relabel_visit with `cap`): tile-wise relaxation
of labels from the sink over a worklist, where no voxel is lowered to a label above the cap and a label at the cap wakes no
neighbouring tile.  Written in plain Python with the kernel's rules (reset labels, the initial list of tiles holding an
unlabelled voxel with residual out-arcs, relaxation inside a tile to its fixed point, the wake test across faces), against
a plain backward BFS.  It pins the claim the first relabel of an easy solve relies on: the capped BFS gives exactly the BFS
distance wherever that distance is <= cap and leaves HINF everywhere else; and the exact relabel that follows, started
from the tiles the capped one wrote (the partial reset), still reaches every voxel through the tiles it left untouched.
The CUDA code itself is checked on the GPU against the reference BK (tests/test_gpu_first_cap.py)."""
import collections
import random

HINF = 0x3FFFFFFF
DIRS = [(-1, 0, 0), (1, 0, 0), (0, -1, 0), (0, 1, 0), (0, 0, -1), (0, 0, 1)]   # arc bit k of rmask


def lattice(rng, dims, p_arc, p_sink):
    vox = [(z, y, x) for z in range(dims[0]) for y in range(dims[1]) for x in range(dims[2])]
    arcs, sink = {}, set()
    for v in vox:
        m = 0
        for k, d in enumerate(DIRS):
            w = (v[0] + d[0], v[1] + d[1], v[2] + d[2])
            if all(0 <= w[a] < dims[a] for a in range(3)) and rng.random() < p_arc:
                m |= 1 << k
        arcs[v] = m
        if rng.random() < p_sink:
            sink.add(v)
    return vox, arcs, sink


def nbr(v, k):
    d = DIRS[k]
    return (v[0] + d[0], v[1] + d[1], v[2] + d[2])


def bfs_distance(vox, arcs, sink):
    """label(v) = 1 at a residual sink link, else 1 + min over residual arcs v -> w of label(w); HINF = no path."""
    into = collections.defaultdict(list)
    for v in vox:
        for k in range(6):
            if arcs[v] >> k & 1:
                into[nbr(v, k)].append(v)
    dist = {v: HINF for v in vox}
    q = collections.deque()
    for s in sink:
        dist[s] = 1
        q.append(s)
    while q:
        w = q.popleft()
        for v in into[w]:
            if dist[v] == HINF:
                dist[v] = dist[w] + 1
                q.append(v)
    return dist


class TileModel:
    def __init__(self, dims, tile, vox, arcs, sink):
        self.dims, self.tile, self.arcs, self.sink = dims, tile, arcs, sink
        self.nt = [(dims[a] + tile - 1) // tile for a in range(3)]
        self.tiles = collections.defaultdict(list)
        for v in vox:
            self.tiles[self.tile_of(v)].append(v)
        self.height = {}
        self.dirty = set()

    def tile_of(self, v):
        return tuple(v[a] // self.tile for a in range(3))

    def reset(self, tiles):
        """k_relabel_reset(_list): labels of `tiles` from the residual mask; returns the tiles that need a label."""
        listed = []
        for t in tiles:
            needs = False
            for v in self.tiles[t]:
                self.height[v] = 1 if v in self.sink else HINF
                needs |= self.arcs[v] != 0 and self.height[v] == HINF
            if needs:
                listed.append(t)
        return listed

    def h(self, w):
        return self.height.get(w, HINF)       # outside the lattice: HINF

    def visit(self, t, cap, nxt):
        """relabel_visit: relax inside the tile to its fixed point (halo read once), write back, wake face neighbours."""
        own = self.tiles[t]
        h0 = {v: self.height[v] for v in own}
        loc = dict(h0)
        while True:
            new = {}
            for v in own:
                m = self.arcs[v]
                hv = loc[v]
                if m and hv > 1:
                    best = hv
                    for k in range(6):
                        if m >> k & 1:
                            w = nbr(v, k)
                            hw = loc[w] if w in loc else self.h(w)
                            best = min(best, hw + 1)
                    if best < hv and best <= cap:
                        new[v] = best
            if not new:
                break
            loc.update(new)       # synchronous round, as the CTA's __syncthreads_or loop
        for v in own:
            hv = loc[v]
            if hv == h0[v]:
                continue
            self.height[v] = hv
            self.dirty.add(t)
            if hv >= cap:
                continue
            for k in range(6):
                w = nbr(v, k)
                if self.tile_of(w) != t and all(0 <= w[a] < self.dims[a] for a in range(3)) and self.h(w) > hv + 1:
                    nxt.add(self.tile_of(w))

    def bfs(self, listed, cap, rng):
        """k_bfs_coop: passes over the current list (in any order; the kernel's tiles race), the woken tiles form the next."""
        cur, passes = list(listed), 0
        while cur:
            rng.shuffle(cur)
            nxt = set()
            for t in cur:
                self.visit(t, cap, nxt)
            cur = sorted(nxt)
            passes += 1
        return passes


def test_capped_relaxation_is_the_bfs_distance_up_to_the_cap():
    rng = random.Random(11)
    for trial in range(60):
        dims = (rng.randrange(3, 13), rng.randrange(3, 13), rng.randrange(3, 13))
        tile = rng.choice([2, 3, 4])
        vox, arcs, sink = lattice(rng, dims, rng.choice([0.4, 0.7, 0.95]), rng.choice([0.005, 0.02, 0.1]))
        dist = bfs_distance(vox, arcs, sink)
        for cap in (2, 3, 5, 8, HINF):
            m = TileModel(dims, tile, vox, arcs, sink)
            m.bfs(m.reset(sorted(m.tiles)), cap, rng)
            for v in vox:
                want = dist[v] if dist[v] <= cap else HINF
                assert m.height[v] == want, (trial, dims, tile, cap, v, m.height[v], dist[v])


def test_exact_relabel_after_a_capped_one_reaches_the_untouched_tiles():
    """Second relabel of an easy solve: only the tiles the capped relabel wrote are reset and listed (partial reset); the
    tiles it left in the reset state are reached by wake-ups.  The labels must be the exact BFS distances."""
    rng = random.Random(5)
    for trial in range(60):
        dims = (rng.randrange(4, 14), rng.randrange(4, 14), rng.randrange(4, 14))
        tile = rng.choice([2, 3, 4])
        vox, arcs, sink = lattice(rng, dims, rng.choice([0.5, 0.8, 1.0]), rng.choice([0.005, 0.02, 0.08]))
        dist = bfs_distance(vox, arcs, sink)
        for cap in (2, 4, 7):
            m = TileModel(dims, tile, vox, arcs, sink)
            m.bfs(m.reset(sorted(m.tiles)), cap, rng)
            dirty, m.dirty = sorted(m.dirty), set()
            m.bfs(m.reset(dirty), HINF, rng)
            assert all(m.height[v] == dist[v] for v in vox), (trial, dims, tile, cap)
