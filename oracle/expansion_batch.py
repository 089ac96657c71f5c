"""oracle/expansion_batch.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

CPU model of the batched alpha-expansion (``medpy_b200.graphcut.expansion_from_voxels_batch``, DESIGN.md §11
"Batches"): B images run through one loop of cycles alpha = 0 .. K-1, each image's move built and cut by
``oracle/expansion.py`` on that image alone.  An image whose cycle switched nothing is frozen: it takes no further moves
and its column of the switch matrix holds 0 from then on.  The loop stops after a cycle in which no image switched a
voxel, or after ``max_cycles`` cycles.

Only tests/ and tools/ may import this module; the product package never does.
"""
import numpy

from . import expansion as ox


def expansion_batch(costs, boundaries=None, markers=None, init=None, max_cycles=20):
    """costs (B, K, *image); boundaries None or one ``(kind, image, sigma, spacing)`` per image (None: no pair term);
    markers / init None or (B, *image).  Returns dict(labels (B, *image) uint8, energies float64 (B,), matrix (moves, B)
    int64 switch counts of the batch loop, batch_moves, batch_cycles, batch_converged, and per image the lists moves,
    cycles, converged, switched)."""
    costs = numpy.asarray(costs)
    B, K = costs.shape[:2]
    shape = costs.shape[2:]
    D, w, lab = [], [], []
    for b in range(B):
        D.append(ox.data_costs(costs[b], None if markers is None else markers[b]))
        w.append(ox.pair_weights(shape, None if boundaries is None else boundaries[b]))
        lab.append(ox.initial_labels(D[b], shape, None if init is None else init[b]))
    active = [True] * B
    cycles = [0] * B
    converged = [False] * B
    rows = []
    batch_cycles = 0
    for _ in range(max_cycles):
        if not any(active):
            break
        changed = [0] * B
        for alpha in range(K):
            row = [0] * B
            for b in range(B):
                if active[b]:
                    lab[b], row[b], _ = ox.move(D[b], w[b], lab[b], alpha)
                    changed[b] += row[b]
            rows.append(row)
        batch_cycles += 1
        for b in range(B):
            if active[b]:
                cycles[b] += 1
                if changed[b] == 0:
                    converged[b] = True
                    active[b] = False
    matrix = numpy.asarray(rows, dtype=numpy.int64).reshape(len(rows), B)
    moves = [K * c for c in cycles]
    return dict(labels=numpy.stack(lab).astype(numpy.uint8),
                energies=numpy.asarray([ox.energy(D[b], w[b], lab[b]) for b in range(B)]),
                matrix=matrix, batch_moves=len(rows), batch_cycles=batch_cycles, batch_converged=not any(active),
                moves=moves, cycles=cycles, converged=converged,
                switched=[matrix[:moves[b], b].tolist() for b in range(B)])
