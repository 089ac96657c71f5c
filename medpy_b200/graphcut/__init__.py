"""``medpy_b200.graphcut`` -- H100-native drop-in for ``medpy.graphcut``'s graph construction and min-cut.

Exports the names the reference package exports (medpy/graphcut/__init__.py:186-222): ``graph_from_voxels`` and the
``energy_voxel`` module (the voxel path, SURVEY.md §8a-e), ``graph_from_voxels_batch`` (many independent images in one build and one
solve, DESIGN.md §3.1), ``expansion_from_voxels`` (a K-label Potts segmentation by alpha-expansion, §11; ``expansion_from_voxels_batch`` for B images in one loop) and ``expansion_from_labels`` (the same over a label image's regions), ``graph_from_labels`` and the ``energy_label`` module (the
region path, §8 row f3), ``graph_from_labels_batch`` (many label images in one region-graph build and one solve, §8), ``GCGraph``, ``split_marker`` and the ``maxflow`` module with ``GraphDouble`` /
``GraphFloat`` / ``GraphInt`` (general sparse graphs: row f4), the plain ``Graph`` record and ``graph_to_dimacs``.  ``graphcut_stawiaski`` / ``graphcut_split`` /
``graphcut_subprocesses`` (wrapper.py:72-329) are provided with the reference's splitting rules; their jobs run back to
back on the GPU instead of in a process pool.
"""
from . import energy_label, energy_voxel, maxflow
from .batch import BatchGraph, graph_from_voxels_batch
from .generate import graph_from_labels, graph_from_voxels, label_cut_mask
from .graph import GCGraph, Graph
from .labels_batch import LabelBatchGraph, graph_from_labels_batch
from .maxflow import GraphDouble, GraphFloat, GraphInt
from .multilabel import expansion_from_labels, expansion_from_voxels, expansion_from_voxels_batch
from .wrapper import graphcut_split, graphcut_stawiaski, graphcut_stawiaski_batch, graphcut_subprocesses, split_marker
from .write import graph_to_dimacs

__all__ = ["graph_from_voxels", "expansion_from_voxels", "expansion_from_voxels_batch", "expansion_from_labels", "graph_from_voxels_batch", "BatchGraph", "graph_from_labels", "graph_from_labels_batch", "LabelBatchGraph", "label_cut_mask", "energy_voxel", "energy_label", "GCGraph", "Graph",
           "graph_to_dimacs", "GraphDouble", "GraphFloat", "GraphInt", "split_marker", "graphcut_split", "graphcut_stawiaski",
           "graphcut_stawiaski_batch", "graphcut_subprocesses", "maxflow"]
