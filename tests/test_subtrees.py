"""SplatTree forests: a dynamic mesh of several scenes takes one sub-tree per scene (SplatTree.processSplatMesh, SplatTree.js:377-390),
culled per sub-tree under baseModelView * sceneTransform(s) (Viewer.js:2005-2044) and cast at per sub-tree under matrixWorld *
sceneTransform(s) (Raycaster.js:49-82).  CPU: the host mirror's forest against per-scene trees, and the forest restatements of the
gather and the raycast (forest_gather / forest_raycast, used by the GPU tests too) against oracle/tree_oracle.py and
oracle/ray_oracle.py."""
import math
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from oracle import ray_oracle as RO  # noqa: E402
from oracle import tree_oracle as TO  # noqa: E402


# ---- forest restatements ---------------------------------------------------------------------------------------------------------
def leaves_of(lv, lo=0, hi=None):
    """Leaves [lo, hi) of a splat_tree.SplatTreeLeaves in tree_oracle's format: [(min, max, depth, indexes)]."""
    hi = lv.count if hi is None else hi
    return [(lv.node_min[i].tolist(), lv.node_max[i].tolist(), int(lv.depth[i]), lv.indexes[lv.offsets[i]:lv.offsets[i + 1]].tolist()) for i in range(lo, hi)]


def forest_leaves(lv):
    """Per sub-tree of `lv`, its leaves in tree_oracle's format."""
    o = lv.sub_leaf_offsets
    return [leaves_of(lv, int(o[s]), int(o[s + 1])) for s in range(lv.sub_tree_count)]


def _cull(leaf, e, cx, cy, gather_all):
    """Viewer.js:2013-2033 for one leaf (tree_oracle.gather_for_sort's body): its distance, or None when culled."""
    mn, mx, _depth, _idx = leaf
    centre = [(mx[k] - mn[k]) * 0.5 + mn[k] for k in range(3)]
    t = TO._apply_matrix4(centre, e)
    dist = math.sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2])
    t = TO._normalized(t)
    yz = TO._normalized([0.0, t[1], t[2]])
    xz = TO._normalized([t[0], 0.0, t[2]])
    dot_xz = 0.0 * xz[0] + 0.0 * xz[1] + -1.0 * xz[2]
    dot_yz = 0.0 * yz[0] + 0.0 * yz[1] + -1.0 * yz[2]
    d = [mx[k] - mn[k] for k in range(3)]
    ns = math.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2])
    out_y = dot_yz < (cy - 0.6)
    out_x = dot_xz < (cx - 0.6)
    return None if (not gather_all and ((out_x or out_y) and dist > ns)) else dist


def forest_gather(forest, cos_fov_x_over_2, cos_fov_y_over_2, gather_all=False):
    """gatherSceneNodesForSort over a forest: [(leaves, model_view16)] in sub-tree order, sub-tree s's leaves culled with its own model
    view, the kept leaves of all sub-trees in one list by tree_oracle.leaf_order_key over the forest's leaf numbers (ties and NaN
    distances: sub-tree order, then leaf order; NaN after +inf), laid out nearest last.  -> (indexesToSort[0:renderCount], renderCount)."""
    kept, flat = [], []
    for leaves, mv in forest:
        e = [float(v) for v in np.asarray(mv, np.float64).reshape(16)]
        for leaf in leaves:
            if leaf[3]:
                d = _cull(leaf, e, cos_fov_x_over_2, cos_fov_y_over_2, gather_all)
                if d is not None:
                    kept.append((d, len(flat)))
            flat.append(leaf)
    kept.sort(key=lambda k: TO.leaf_order_key(*k))
    total = sum(len(flat[li][3]) for _, li in kept)
    out = np.empty(total, np.uint32)
    end = total
    for _, li in kept:
        idx = flat[li][3]
        out[end - len(idx):end] = idx
        end -= len(idx)
    return out, total


class Shifted:
    """A ray_oracle scene read through scene-local indexes: local splat i is the scene's splat offset + i."""

    def __init__(self, scene, offset):
        self.scene, self.offset = scene, offset

    def inputs(self, i, ellipsoid):
        return self.scene.inputs(i + self.offset, ellipsoid)


def _index_count(root):
    if root is None:
        return 0
    return len(root.indexes or []) + sum(_index_count(c) for c in root.children)


def forest_raycast(subtrees, scene, origin, direction, *, ellipsoid=False, scene_visible=True):
    """Raycaster.intersectSplatMesh over a forest: [(root over scene-local indexes or None, splat offset, from_local16)] in sub-tree order.
    Each sub-tree is cast at in its local space and its hits mapped back with its own from_local; hits carry global splat indexes and
    positions running across the forest, sorted as ray_oracle sorts them.  -> [(distance, position, splat, world origin, world normal)]."""
    hits, pos = [], 0
    for root, offset, fl in subtrees:
        for dist, p, i, wo, wn in RO.intersect_splat_mesh(root, Shifted(scene, offset), origin, direction, fl, ellipsoid=ellipsoid,
                                                          scene_visible=scene_visible):
            hits.append((dist, p + pos, i + offset, wo, wn))
        pos += _index_count(root)
    hits.sort(key=lambda h: (h[0] != h[0], 0.0 if h[0] != h[0] else h[0], h[1]))
    return hits


# ---- tests -------------------------------------------------------------------------------------------------------------------------
def _scenes(seed=0, counts=(400, 0, 300, 250)):
    """Centres and alphas of consecutive scenes: a Gaussian cloud, an empty scene, one with NaN centres and dropped alphas, and one
    on a grid (centres on split planes)."""
    rng = np.random.default_rng(seed)
    parts, alphas = [], []
    for k, n in enumerate(counts):
        c = rng.normal(0, 1 + k, (n, 3)).astype(np.float32)
        a = rng.integers(0, 256, n).astype(np.uint8)
        if k == 2 and n:
            c[::17, 1] = np.nan
            a[:50] = 0
        if k == 3 and n:
            c = rng.integers(-2, 3, (n, 3)).astype(np.float32)
        parts.append(c)
        alphas.append(a)
    ranges = list(zip(np.cumsum([0] + list(counts[:-1])), counts))
    return np.concatenate(parts), np.concatenate(alphas), ranges


def test_mirror_forest_is_each_scene_alone():
    from gaussiansplats3d_b200.splat_tree import SplatTree
    c, a, ranges = _scenes()
    for max_depth, max_centers in ((8, 1000), (8, 16), (2, 5), (0, 1)):
        f = SplatTree(max_depth, max_centers).processSplatMesh(c, a, 1, scene_ranges=ranges)
        assert f.sub_tree_count == len(ranges)
        assert (f.all_parent[f.sub_node_offsets[:-1][np.diff(f.sub_node_offsets) > 0]] == -1).all()
        assert (f.all_parent == -1).sum() == int((np.diff(f.sub_node_offsets) > 0).sum())
        for s, (off, cnt) in enumerate(ranges):
            one = SplatTree(max_depth, max_centers).processSplatMesh(c[off:off + cnt], a[off:off + cnt], 1)
            l0, l1 = int(f.sub_leaf_offsets[s]), int(f.sub_leaf_offsets[s + 1])
            n0, n1 = int(f.sub_node_offsets[s]), int(f.sub_node_offsets[s + 1])
            assert l1 - l0 == one.count and n1 - n0 == one.all_parent.shape[0], s
            for k in ("node_min", "node_max", "node_center", "depth", "all_min", "all_max"):
                got, want = getattr(f, k), getattr(one, k)
                got = got[l0:l1] if k in ("node_min", "node_max", "node_center", "depth") else got[n0:n1]
                assert np.array_equal(got, want, equal_nan=got.dtype.kind == "f"), (s, k)
            assert np.array_equal(f.indexes[f.offsets[l0]:f.offsets[l1]], one.indexes + off), s
            assert np.array_equal(np.diff(f.offsets[l0:l1 + 1]), np.diff(one.offsets)), s
            assert np.array_equal(f.leaf_node[l0:l1], one.leaf_node + n0), s
            par = f.all_parent[n0:n1]
            assert np.array_equal(np.where(par < 0, -1, par - n0), one.all_parent), s
        assert f.sub_leaf_offsets[1] == f.sub_leaf_offsets[2]    # the empty scene
    # no scene_ranges: the one tree of every splat, one sub-tree
    t = SplatTree(8, 16).processSplatMesh(c, a, 1)
    assert t.sub_tree_count == 1 and list(t.sub_leaf_offsets) == [0, t.count] and list(t.sub_node_offsets) == [0, t.all_parent.shape[0]]


def _view(eye, target=(0.0, 0.0, 0.0)):
    from gaussiansplats3d_b200 import three_math as TM
    return np.asarray(TM.invert(TM.camera_world_matrix(list(eye), list(target), [0.0, 1.0, 0.0])), np.float64).reshape(16)


def test_forest_gather_with_one_sub_tree_is_the_oracle():
    c, a, _ = _scenes(1)
    leaves = TO.build_leaves(c, a, 1, 8, 16)
    for eye in ((0.0, 0.5, 6.0), (3.0, -1.0, 2.0), (0.0, 0.0, 0.5)):
        mv = _view(eye)
        for gather_all in (False, True):
            want = TO.gather_for_sort(leaves, mv, 0.9, 0.95, gather_all)
            got = forest_gather([(leaves, mv)], 0.9, 0.95, gather_all)
            assert got[1] == want[1] and np.array_equal(got[0], want[0])


def test_forest_gather_is_the_concatenation_of_its_sub_trees():
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.splat_tree import SplatTree
    c, a, ranges = _scenes(2)
    f = SplatTree(8, 16).processSplatMesh(c, a, 1, scene_ranges=ranges)
    per = forest_leaves(f)
    base = _view((1.0, 0.5, 7.0))
    xfs = [np.asarray(TM.compose(p, q, s), np.float64).reshape(16) for p, q, s in
           (((0, 0, 0), (0, 0, 0, 1), (1, 1, 1)), ((2, 0, 0), (0, 0.6, 0, 0.8), (1, 1, 1)), ((-2, 1, 0), (0.1, 0.2, -0.3, 0.927), (0.5, 0.5, 0.5)),
            ((0, -1, -3), (0, 0, 0, 1), (2, 2, 2)))]
    views = [TM.multiply(base, x) for x in xfs]
    for gather_all in (False, True):
        got, n = forest_gather(list(zip(per, views)), 0.9, 0.95, gather_all)
        parts = [TO.gather_for_sort(lv, v, 0.9, 0.95, gather_all) for lv, v in zip(per, views)]
        assert n == sum(p[1] for p in parts)
        assert np.array_equal(np.sort(got), np.sort(np.concatenate([p[0] for p in parts])))
        # the same list, placed by hand: every kept leaf of every sub-tree with its distance, ascending, nearest last
        kept = []
        for s, (lv, v) in enumerate(zip(per, views)):
            e = [float(x) for x in v]
            for k, leaf in enumerate(lv):
                d = _cull(leaf, e, 0.9, 0.95, gather_all)
                if d is not None:
                    kept.append((d, s, k, leaf[3]))
        kept.sort(key=lambda t: (t[0], t[1], t[2]))
        want = np.concatenate([np.asarray(t[3], np.uint32) for t in reversed(kept)]) if kept else np.zeros(0, np.uint32)
        assert np.array_equal(got, want)
    # one model view for every sub-tree: the one list of all leaves
    got, n = forest_gather([(lv, base) for lv in per], 0.9, 0.95)
    want = TO.gather_for_sort([leaf for lv in per for leaf in lv], base, 0.9, 0.95)
    assert n == want[1] and np.array_equal(got, want[0])


def _ray_scene(n, seed):
    rng = np.random.default_rng(seed)
    c = rng.normal(0, 1, (n, 3))
    s = np.exp(rng.uniform(-3, -1, (n, 3))).astype(np.float32)
    q = rng.normal(0, 1, (n, 4)).astype(np.float32)
    a = rng.integers(1, 256, n).astype(np.uint8)
    return c, s, q, a


def test_forest_raycast_with_one_sub_tree_is_the_oracle():
    c, s, q, a = _ray_scene(200, 3)
    scene = RO.Scene(c, s, q, a, dynamic=True)
    root = RO.build_tree(c.astype(np.float32), a, max_centers=8)
    fl = list(np.asarray(RO.compose([0.5, 0, 0], [0, 0.6, 0, 0.8], [1.5, 1.5, 1.5]), np.float64))
    for ellipsoid in (False, True):
        for o in ((0.0, 0.0, 8.0), (0.3, -0.2, 6.0)):
            d = RO.normalize([-o[0] * 0.05, -o[1] * 0.05, -1.0])
            want = RO.intersect_splat_mesh(root, scene, o, d, fl, ellipsoid=ellipsoid)
            got = forest_raycast([(root, 0, fl)], scene, o, d, ellipsoid=ellipsoid)
            assert got == want


def test_forest_raycast_merges_its_sub_trees():
    c, s, q, a = _ray_scene(300, 4)
    scene = RO.Scene(c, s, q, a, dynamic=True)
    ranges = ((0, 120), (120, 0), (120, 180))
    roots = [RO.build_tree(c[o:o + n].astype(np.float32), a[o:o + n], max_centers=8) for o, n in ranges]
    fls = [list(np.asarray(RO.compose(p, [0, 0, 0, 1], [1, 1, 1]), np.float64)) for p in ((0, 0, 0), (5, 5, 5), (0.2, 0.1, 0))]
    o, d = (0.1, 0.0, 8.0), RO.normalize([0.0, 0.0, -1.0])
    for ellipsoid in (False, True):
        got = forest_raycast([(r, off, fl) for r, (off, _), fl in zip(roots, ranges, fls)], scene, o, d, ellipsoid=ellipsoid)
        merged, pos = [], 0
        for r, (off, _), fl in zip(roots, ranges, fls):
            for h in RO.intersect_splat_mesh(r, Shifted(scene, off), o, d, fl, ellipsoid=ellipsoid):
                merged.append((h[0], h[1] + pos, h[2] + off, h[3], h[4]))
            pos += _index_count(r)
        merged.sort(key=lambda h: (h[0], h[1]))
        assert got == merged and len(got) > 0
        assert {h[2] for h in got} & set(range(0, 120)) and {h[2] for h in got} & set(range(120, 300))
