"""oracle/tree_oracle.py -- TEST INFRASTRUCTURE ONLY.  Imports nothing from the product package.

Scalar restatement (Python floats = JS numbers, plain lists like the reference's arrays) of
  * the octree build of /root/reference/src/splattree/SplatTree.js:132-278 (processSplatTreeNode / buildSubTree / createSplatTree) and the
    leaf list of convertWorkerSubTree (:55-79), and
  * the per-frame cull + ordering + index layout of Viewer.gatherSceneNodesForSort (src/Viewer.js:1969-2077), with three.js's
    Vector3.applyMatrix4 / normalize operation order (three r160, not vendored: restated from its published source),
  * the partial-sort schedule of Viewer.runSplatSort (:1833-1964).
The reference ships no tests or vectors for any of this: pinned by reading the source only ("parity unpinned" in that sense); it is the
checker for the product's vectorised tree build (splat_tree.py), its CUDA gather (csrc/cull_kernels.cuh) and its Viewer mirror."""
from __future__ import annotations

import math

import numpy as np


class _Node:
    __slots__ = ("min", "max", "depth", "children", "indexes")

    def __init__(self, mn, mx, depth):
        self.min, self.max, self.depth, self.children, self.indexes = list(mn), list(mx), depth, [], None


def build_leaves(centers_f32: np.ndarray, alphas=None, min_alpha: int = 1, max_depth: int = 8, max_centers: int = 1000):
    """-> list of (min[3], max[3], depth, indexes[]) in nodesWithIndexes order."""
    c = [[float(v) for v in row] for row in np.asarray(centers_f32, np.float32)]
    ids = [i for i in range(len(c)) if alphas is None or int(alphas[i]) >= min_alpha]
    if not ids:
        return []
    mn = [min(c[i][k] for i in ids) for k in range(3)]
    mx = [max(c[i][k] for i in ids) for k in range(3)]
    root = _Node(mn, mx, 0)
    root.indexes = ids
    added = set()
    leaves = []

    def process(node):
        if len(node.indexes) < max_centers or node.depth > max_depth:
            fresh = []
            for i in node.indexes:
                if i not in added:
                    fresh.append(i)
                    added.add(i)
            node.indexes = sorted(fresh)
            leaves.append(node)
            return
        dims = [node.max[k] - node.min[k] for k in range(3)]
        half = [d * 0.5 for d in dims]
        ctr = [node.min[k] + half[k] for k in range(3)]
        bounds = [
            ([ctr[0] - half[0], ctr[1], ctr[2] - half[2]], [ctr[0], ctr[1] + half[1], ctr[2]]),
            ([ctr[0], ctr[1], ctr[2] - half[2]], [ctr[0] + half[0], ctr[1] + half[1], ctr[2]]),
            ([ctr[0], ctr[1], ctr[2]], [ctr[0] + half[0], ctr[1] + half[1], ctr[2] + half[2]]),
            ([ctr[0] - half[0], ctr[1], ctr[2]], [ctr[0], ctr[1] + half[1], ctr[2] + half[2]]),
            ([ctr[0] - half[0], ctr[1] - half[1], ctr[2] - half[2]], [ctr[0], ctr[1], ctr[2]]),
            ([ctr[0], ctr[1] - half[1], ctr[2] - half[2]], [ctr[0] + half[0], ctr[1], ctr[2]]),
            ([ctr[0], ctr[1] - half[1], ctr[2]], [ctr[0] + half[0], ctr[1], ctr[2] + half[2]]),
            ([ctr[0] - half[0], ctr[1] - half[1], ctr[2]], [ctr[0], ctr[1], ctr[2] + half[2]]),
        ]
        base = [[] for _ in bounds]
        for i in node.indexes:
            p = c[i]
            for j, (bmin, bmax) in enumerate(bounds):
                if bmin[0] <= p[0] <= bmax[0] and bmin[1] <= p[1] <= bmax[1] and bmin[2] <= p[2] <= bmax[2]:
                    base[j].append(i)
        for j, (bmin, bmax) in enumerate(bounds):
            child = _Node(bmin, bmax, node.depth + 1)
            child.indexes = base[j]
            node.children.append(child)
        node.indexes = None
        for child in node.children:
            process(child)

    process(root)
    return [(n.min, n.max, n.depth, n.indexes) for n in leaves if n.indexes]


def _apply_matrix4(v, e):
    """THREE.Vector3.applyMatrix4 (column-major elements e)."""
    x, y, z = v
    w = 1.0 / (e[3] * x + e[7] * y + e[11] * z + e[15])
    return [(e[0] * x + e[4] * y + e[8] * z + e[12]) * w, (e[1] * x + e[5] * y + e[9] * z + e[13]) * w, (e[2] * x + e[6] * y + e[10] * z + e[14]) * w]


def _normalized(v):
    """Vector3.normalize = divideScalar(length() || 1) = multiplyScalar(1 / s)."""
    ln = math.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])
    s = 1.0 / (ln or 1.0)
    return [v[0] * s, v[1] * s, v[2] * s]


def leaf_order_key(dist: float, leaf: int):
    """Where a kept leaf goes in the distance order: ascending distance, a NaN distance after +inf, equal distances (and NaN against NaN)
    by leaf number.  The reference sorts with `(a, b) => a.distanceToNode < b.distanceToNode ? -1 : 1` (Viewer.js:2040-2043): equal
    distances answer 1 both ways, which V8's TimSort reads as "not less" and so keeps them in gather order (= leaf number); a NaN answers
    1 both ways too, which leaves its place to the input order.  The engine fixes that open case: every NaN sorts after every number,
    whatever its bit pattern, and NaNs among themselves by leaf number.  Stated as a key so that list.sort() never compares a NaN."""
    return (dist != dist, 0.0 if dist != dist else dist, leaf)


def gather_for_sort(leaves, model_view16, cos_fov_x_over_2: float, cos_fov_y_over_2: float, gather_all: bool = False):
    """-> (indexesToSort[0:renderCount] as u32 array, renderCount).  Kept leaves ordered by leaf_order_key and laid out from the END
    of the window backwards, i.e. the nearest leaf's indexes come LAST (Viewer.js:2040-2055)."""
    e = [float(v) for v in np.asarray(model_view16, np.float64).reshape(16)]
    kept = []
    for li, (mn, mx, _depth, idx) in enumerate(leaves):
        if not idx:
            continue
        centre = [(mx[k] - mn[k]) * 0.5 + mn[k] for k in range(3)]
        t = _apply_matrix4(centre, e)
        dist = math.sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2])
        t = _normalized(t)
        yz = _normalized([0.0, t[1], t[2]])
        xz = _normalized([t[0], 0.0, t[2]])
        dot_xz = 0.0 * xz[0] + 0.0 * xz[1] + -1.0 * xz[2]          # forward = (0, 0, -1)
        dot_yz = 0.0 * yz[0] + 0.0 * yz[1] + -1.0 * yz[2]
        d = [mx[k] - mn[k] for k in range(3)]
        ns = math.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2])
        out_y = dot_yz < (cos_fov_y_over_2 - 0.6)
        out_x = dot_xz < (cos_fov_x_over_2 - 0.6)
        if not gather_all and ((out_x or out_y) and dist > ns):
            continue
        kept.append((dist, li))
    kept.sort(key=lambda k: leaf_order_key(*k))
    total = sum(len(leaves[li][3]) for _, li in kept)
    out = np.empty(total, np.uint32)
    end = total
    for _, li in kept:
        idx = leaves[li][3]
        out[end - len(idx):end] = idx
        end -= len(idx)
    return out, total


PARTIAL_SORTS = ((0.55, (0.125, 0.33333, 0.75)), (0.65, (0.33333, 0.66667)), (0.8, (0.5,)))      # Viewer.js:1843-1856


class SortSchedule:
    """The state machine of runSplatSort (Viewer.js:1858-1964) reduced to its decisions: given the camera's view direction / position and
    the render count of this call, return the sort count to use, or None when no sort is started."""

    def __init__(self):
        self.last_dir = [0.0, 0.0, -1.0]
        self.last_pos = [0.0, 0.0, 0.0]
        self.queued: list[int] = []

    def step(self, view_dir, position, render_count: int, *, force=False, should_sort_all=False, dynamic=False):
        angle = sum(a * b for a, b in zip(view_dir, self.last_dir))
        pos = math.sqrt(sum((a - b) ** 2 for a, b in zip(position, self.last_pos)))
        if not force and not dynamic and not self.queued:
            if not (angle <= 0.99 or pos >= 1.0):
                return None
        if not self.queued:
            if dynamic or should_sort_all:
                self.queued.append(render_count)
            else:
                for threshold, fractions in PARTIAL_SORTS:
                    if angle < threshold:
                        for f in fractions:
                            self.queued.append(math.floor(render_count * f))
                        break
                self.queued.append(render_count)
        sort_count = min(self.queued.pop(0), render_count)
        if not self.queued:
            self.last_pos = list(position)
            self.last_dir = list(view_dir)
        return sort_count
