"""Host-side mirror of the reference's SplatTree (src/splattree/SplatTree.js): the octree whose leaves `Viewer.gatherSceneNodesForSort`
(src/Viewer.js:1969-2077) culls against the view frustum to produce the sorter's `indexesToSort` / `splatRenderCount`.

Building the tree is load-time host work in the reference too (a Web Worker, SplatTree.js:81-278); only its leaves matter afterwards.
The per-frame part -- cull every leaf, order the kept ones by distance, lay their index runs out nearest-last -- runs on the GPU
(csrc/cull_kernels.cuh, C ABI gs_upload_splat_tree / gs_gather_for_sort).

    SplatTree(maxDepth=8, maxCentersPerNode=1000)            SplatMesh.js:236
    processSplatMesh: centres of the splats with alpha >= minAlpha, f32, with their global index            SplatTree.js:335-431
    processSplatTreeNode: leaf when count < maxCentersPerNode or depth > maxDepth; otherwise 8 children whose boxes INCLUDE their faces
        (a centre on a shared face goes to several children; the first leaf reached in depth-first child order keeps it)   :132-216
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np


@dataclass
class SplatTreeLeaves:
    """`nodesWithIndexes` of the tree's sub-trees, flattened and concatenated in sub-tree order: leaf i owns indexes[offsets[i]:offsets[i+1]]
    (ascending).  Sub-tree s holds leaves sub_leaf_offsets[s]:sub_leaf_offsets[s+1] and nodes sub_node_offsets[s]:sub_node_offsets[s+1];
    a tree of one sub-tree (every tree but a dynamic mesh's forest) has {0, leaf count} and {0, node count}."""
    node_min: np.ndarray      # f64 [m,3]
    node_max: np.ndarray      # f64 [m,3]
    node_center: np.ndarray   # f64 [m,3]  (max - min) * 0.5 + min                                   SplatTree.js:12
    offsets: np.ndarray       # u32 [m+1]
    indexes: np.ndarray       # u32 [offsets[m]]
    depth: np.ndarray         # i32 [m]
    # every node of the tree, depth first, root first (the raycast's box tests, Raycaster.castRayAtSplatTreeNode)
    all_min: np.ndarray | None = None      # f64 [k,3]
    all_max: np.ndarray | None = None      # f64 [k,3]
    all_parent: np.ndarray | None = None   # i32 [k], -1 for the root
    leaf_node: np.ndarray | None = None    # u32 [m]: the node of leaf i
    sub_leaf_offsets: np.ndarray | None = None   # u32 [sub-trees + 1]
    sub_node_offsets: np.ndarray | None = None   # u32 [sub-trees + 1]

    def __post_init__(self):
        if self.sub_leaf_offsets is None:
            self.sub_leaf_offsets = np.array([0, self.count], np.uint32)
        if self.sub_node_offsets is None:
            self.sub_node_offsets = np.array([0, 0 if self.all_parent is None else self.all_parent.shape[0]], np.uint32)

    @property
    def count(self) -> int:
        return int(self.offsets.shape[0] - 1)

    @property
    def sub_tree_count(self) -> int:
        return int(self.sub_leaf_offsets.shape[0] - 1)


# children boxes in the reference's order (SplatTree.js:164-184): per child, which half along x, y, z (0 = lower, 1 = upper)
_CHILD_HALVES = ((0, 1, 0), (1, 1, 0), (1, 1, 1), (0, 1, 1), (0, 0, 0), (1, 0, 0), (1, 0, 1), (0, 0, 1))


class SplatTree:
    def __init__(self, maxDepth: int = 8, maxCentersPerNode: int = 1000):  # noqa: N803
        self.maxDepth, self.maxCentersPerNode = maxDepth, maxCentersPerNode
        self.leaves: SplatTreeLeaves | None = None

    def processSplatMesh(self, centers: np.ndarray, alphas: np.ndarray | None = None, minAlpha: int = 1,  # noqa: N802,N803
                         scene_ranges=None) -> SplatTreeLeaves:
        """centers: f32 [n,3] as the mesh returns them (scene transform applied for a static mesh); alphas: u8 [n] (splatColor.w).
        scene_ranges: [(splat_offset, splat_count)] of a dynamic mesh's scenes, which the reference gives one sub-tree each over the
        scene's own (untransformed) centres (SplatTree.js:377-390); None: one tree over all splats."""
        if scene_ranges is not None:
            return self._forest(centers, alphas, minAlpha, scene_ranges)
        c32 = np.ascontiguousarray(centers, dtype=np.float32)
        keep = np.arange(c32.shape[0], dtype=np.int64)
        if alphas is not None:
            keep = keep[np.asarray(alphas).astype(np.int64) >= minAlpha]
        c = c32.astype(np.float64)                         # Float32Array elements read as JS numbers
        pts = c[keep]
        if pts.shape[0] == 0:
            self.leaves = SplatTreeLeaves(*(np.zeros((0, 3)) for _ in range(3)), np.zeros(1, np.uint32), np.zeros(0, np.uint32), np.zeros(0, np.int32),
                                          np.zeros((0, 3)), np.zeros((0, 3)), np.zeros(0, np.int32), np.zeros(0, np.uint32))
            return self.leaves
        # the reference's loop (SplatTree.js:233-238): the first centre, then strict comparisons, so a NaN is skipped unless it comes first
        with np.errstate(invalid="ignore"):
            scene_min = np.where(np.isnan(pts[0]), np.nan, np.fmin.reduce(pts, 0))
            scene_max = np.where(np.isnan(pts[0]), np.nan, np.fmax.reduce(pts, 0))
        added = np.zeros(c32.shape[0], bool)
        mins, maxs, depths, runs = [], [], [], []
        all_min, all_max, all_parent, leaf_node = [], [], [], []

        def visit(nmin, nmax, depth, idx, parent=-1):
            me = len(all_parent)
            all_min.append(nmin.copy()); all_max.append(nmax.copy()); all_parent.append(parent)
            if idx.shape[0] < self.maxCentersPerNode or depth > self.maxDepth:
                fresh = idx[~added[idx]]
                added[fresh] = True
                if fresh.shape[0]:
                    mins.append(nmin.copy()); maxs.append(nmax.copy()); depths.append(depth); runs.append(np.sort(fresh)); leaf_node.append(me)
                return
            dims = nmax - nmin
            half = dims * 0.5
            centre = nmin + half
            p = c[idx]
            for hx, hy, hz in _CHILD_HALVES:
                cmin = np.array([centre[0] if hx else centre[0] - half[0], centre[1] if hy else centre[1] - half[1], centre[2] if hz else centre[2] - half[2]])
                cmax = np.array([centre[0] + half[0] if hx else centre[0], centre[1] + half[1] if hy else centre[1], centre[2] + half[2] if hz else centre[2]])
                inside = np.all((p >= cmin) & (p <= cmax), axis=1)          # WorkerBox3.containsPoint: faces included
                visit(cmin, cmax, depth + 1, idx[inside], me)

        visit(scene_min, scene_max, 0, keep)
        m = len(runs)
        offsets = np.zeros(m + 1, np.uint32)
        if m:
            offsets[1:] = np.cumsum([r.shape[0] for r in runs])
        nmin, nmax = np.array(mins, np.float64).reshape(m, 3), np.array(maxs, np.float64).reshape(m, 3)
        self.leaves = SplatTreeLeaves(nmin, nmax, (nmax - nmin) * 0.5 + nmin, offsets,
                                      np.concatenate(runs).astype(np.uint32) if m else np.zeros(0, np.uint32), np.array(depths, np.int32),
                                      np.array(all_min, np.float64).reshape(-1, 3), np.array(all_max, np.float64).reshape(-1, 3),
                                      np.array(all_parent, np.int32), np.array(leaf_node, np.uint32))
        return self.leaves

    def _forest(self, centers, alphas, minAlpha, scene_ranges) -> SplatTreeLeaves:  # noqa: N803
        """One sub-tree per scene, concatenated: indexes shifted by the scene's offset, node numbers by the nodes before it (each root's
        parent stays -1).  A scene without a kept splat contributes nothing and has empty ranges."""
        parts = []
        for off, cnt in scene_ranges:
            off, cnt = int(off), int(cnt)
            parts.append((off, SplatTree(self.maxDepth, self.maxCentersPerNode).processSplatMesh(
                np.asarray(centers)[off:off + cnt], None if alphas is None else np.asarray(alphas)[off:off + cnt], minAlpha)))
        leaf_off, node_off = [0], [0]
        for _, t in parts:
            leaf_off.append(leaf_off[-1] + t.count)
            node_off.append(node_off[-1] + t.all_parent.shape[0])
        cat = lambda xs, dt, shape: np.concatenate(xs).astype(dt) if xs else np.zeros(shape, dt)  # noqa: E731
        offsets = np.zeros(leaf_off[-1] + 1, np.uint32)
        ends = [t.offsets[1:].astype(np.int64) + sum(p.indexes.shape[0] for _, p in parts[:k]) for k, (_, t) in enumerate(parts)]
        if leaf_off[-1]:
            offsets[1:] = np.concatenate(ends)
        self.leaves = SplatTreeLeaves(
            cat([t.node_min for _, t in parts], np.float64, (0, 3)).reshape(-1, 3), cat([t.node_max for _, t in parts], np.float64, (0, 3)).reshape(-1, 3),
            cat([t.node_center for _, t in parts], np.float64, (0, 3)).reshape(-1, 3), offsets,
            cat([t.indexes.astype(np.int64) + off for off, t in parts], np.uint32, (0,)), cat([t.depth for _, t in parts], np.int32, (0,)),
            cat([t.all_min for _, t in parts], np.float64, (0, 3)).reshape(-1, 3), cat([t.all_max for _, t in parts], np.float64, (0, 3)).reshape(-1, 3),
            cat([np.where(t.all_parent < 0, -1, t.all_parent.astype(np.int64) + node_off[k]) for k, (_, t) in enumerate(parts)], np.int32, (0,)),
            cat([t.leaf_node.astype(np.int64) + node_off[k] for k, (_, t) in enumerate(parts)], np.uint32, (0,)),
            np.array(leaf_off, np.uint32), np.array(node_off, np.uint32))
        return self.leaves


def fov_cosines(render_width: float, render_height: float, fov_degrees: float) -> tuple[float, float]:
    """cosFovXOver2, cosFovYOver2 of gatherSceneNodesForSort (Viewer.js:1990-1995)."""
    import math
    focal = (render_height / 2.0) / math.tan(fov_degrees / 2.0 * (math.pi / 180.0))
    return math.cos(math.atan(render_width / 2.0 / focal)), math.cos(math.atan(render_height / 2.0 / focal))
