"""GPU: SplatTree forests.  gs_build_splat_tree on a dynamic mesh of several scenes builds one sub-tree per scene (SplatTree.js:377-390),
leaf for leaf and node for node the host mirror's forest; gs_gather_for_sort_subtrees culls each sub-tree with its own model view and
is bit-exact against the forest restatement of the gather; gs_raycast casts at each sub-tree with its own from_local and is bit-exact
against the forest restatement of the ray oracle; the Viewer gathers and picks with per-scene matrices."""
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent))
from test_multi_scene_gpu import _count, _mixed, _opts  # noqa: E402
from test_subtrees import forest_gather, forest_leaves, forest_raycast, leaves_of  # noqa: E402

from oracle import file_oracle as FO  # noqa: E402
from oracle import ray_oracle as RO  # noqa: E402
from oracle import tree_oracle as TO  # noqa: E402

pytestmark = pytest.mark.gpu
W, H = 256, 192


def _N():
    from gaussiansplats3d_b200 import _native as N
    return N


def _engine(n, ray=True):
    from gaussiansplats3d_b200 import Engine
    return Engine(max(n, 1), max_width=W, max_height=H, dynamic_mode=True, ray_records=ray)


def _ply(centers, opacity):
    props = [("x", "float"), ("y", "float"), ("z", "float"), ("f_dc_0", "float"), ("f_dc_1", "float"), ("f_dc_2", "float"), ("opacity", "float")] + \
            [(f"scale_{k}", "float") for k in range(3)] + [(f"rot_{k}", "float") for k in range(4)]
    n = centers.shape[0]
    rng = np.random.default_rng(n)
    cols = dict(x=centers[:, 0], y=centers[:, 1], z=centers[:, 2], opacity=opacity, rot_0=np.ones(n),
                **{f"scale_{k}": rng.uniform(-4, -2, n) for k in range(3)}, **{f"f_dc_{k}": rng.normal(0, 1, n) for k in range(3)})
    return FO.write_ply(props, cols, n)


def _special(nan=True):
    """Scenes that exercise the build: every splat below the alpha threshold (an empty sub-tree), NaN centres, and centres on a grid
    (on the split planes)."""
    rng = np.random.default_rng(7)
    with_nan = rng.normal(0, 1, (300, 3))
    with_nan[::13, 0] = np.nan
    with_nan[5::29, 2] = np.nan
    grid = rng.integers(-3, 4, (400, 3)).astype(np.float64)
    return [dict(format=1, data=_ply(rng.normal(0, 1, (200, 3)), np.full(200, -60.0)))] + \
        ([dict(format=1, data=_ply(with_nan, rng.normal(2, 1, 300)))] if nan else []) + [dict(format=1, data=_ply(grid, rng.normal(2, 1, 400)))]


def _upload(e, src):
    infos = e.upload_scenes(src, sh_degree=2)
    n = sum(i["splat_count"] for i in infos)
    cc = e.read_buffer(_N().GS_BUF_CENTERS_COLORS, np.uint32, n * 4).reshape(n, 4)
    return infos, cc[:, 1:4].copy().view(np.float32), (cc[:, 0] >> 24).astype(np.uint8)


def _mirror(centers, alpha, infos, max_depth=8, max_centers=1000):
    from gaussiansplats3d_b200.splat_tree import SplatTree
    return SplatTree(max_depth, max_centers).processSplatMesh(centers, alpha, 1, scene_ranges=[(i["splat_offset"], i["splat_count"]) for i in infos])


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape:
        return False
    if a.dtype.kind == "f":
        return np.array_equal(a.astype(np.float64).view(np.uint64), b.astype(np.float64).view(np.uint64))
    return np.array_equal(a.astype(np.int64), b.astype(np.int64))


KEYS = ("offsets", "indexes", "node_center", "node_min", "node_max", "depth", "all_min", "all_max", "all_parent", "leaf_node",
        "sub_leaf_offsets", "sub_node_offsets")


def _assert_tree(got, want, what=""):
    assert got.count == want.count and got.sub_tree_count == want.sub_tree_count, what
    for k in KEYS:
        assert _same(getattr(got, k), getattr(want, k)), (what, k)


def _sources(nan=True):
    return _mixed(dynamic=True) + _special(nan)


@pytest.mark.parametrize("max_depth,max_centers", [(8, 1000), (8, 4), (2, 3), (0, 1)])
def test_forest_is_the_mirror_and_each_scene_alone(max_depth, max_centers):
    src = _sources()
    e = _engine(sum(_count(s["format"], s["data"]) for s in src))
    try:
        infos, c, a = _upload(e, src)
        info = e.build_splat_tree(max_depth, max_centers, 1)
        assert info["sub_tree_count"] == len(src) and not info["centers_from_ray_records"]
        got, want = e.read_splat_tree(), _mirror(c, a, infos, max_depth, max_centers)
        _assert_tree(got, want)
        empty = len(_mixed(dynamic=True))
        assert not a[infos[empty]["splat_offset"]:][:infos[empty]["splat_count"]].any()
        assert got.sub_leaf_offsets[empty] == got.sub_leaf_offsets[empty + 1] and got.sub_node_offsets[empty] == got.sub_node_offsets[empty + 1]
        # each sub-tree is the tree a one-scene dynamic engine builds of that scene
        for s, sc in enumerate(src):
            one = _engine(_count(sc["format"], sc["data"]))
            try:
                one.upload_scenes([sc], sh_degree=2)
                one.build_splat_tree(max_depth, max_centers, 1)
                t = one.read_splat_tree()
                l0, l1 = int(got.sub_leaf_offsets[s]), int(got.sub_leaf_offsets[s + 1])
                n0, n1 = int(got.sub_node_offsets[s]), int(got.sub_node_offsets[s + 1])
                off = infos[s]["splat_offset"]
                assert t.count == l1 - l0 and t.all_parent.shape[0] == n1 - n0, s
                for k in ("node_center", "node_min", "node_max", "depth"):
                    assert _same(getattr(got, k)[l0:l1], getattr(t, k)), (s, k)
                for k in ("all_min", "all_max"):
                    assert _same(getattr(got, k)[n0:n1], getattr(t, k)), (s, k)
                assert _same(got.indexes[got.offsets[l0]:got.offsets[l1]], t.indexes.astype(np.int64) + off), s
                assert _same(got.leaf_node[l0:l1], t.leaf_node.astype(np.int64) + n0), s
            finally:
                one.close()
    finally:
        e.close()


def test_thirty_two_scenes_and_capacity_keeps_the_forest():
    from gaussiansplats3d_b200 import GsError
    N = _N()
    base = _mixed(dynamic=True)
    src = [base[k % len(base)] for k in range(31)] + [dict(format=1, data=_ply(np.zeros((5000, 3)), np.full(5000, 3.0)))]
    e = _engine(sum(_count(s["format"], s["data"]) for s in src))
    try:
        infos, c, a = _upload(e, src)
        e.build_splat_tree(8, 6000, 1)        # the 5000 coincident centres stay one leaf
        before = e.read_splat_tree()
        _assert_tree(before, _mirror(c, a, infos, 8, 6000))
        assert before.sub_tree_count == 32
        with pytest.raises(GsError) as ei:    # 5000 coincident centres on every split plane: eightfold memberships per level
            e.build_splat_tree(8, 1000, 1)
        assert ei.value.code == N.GS_ERR_CAPACITY
        _assert_tree(e.read_splat_tree(), before)
    finally:
        e.close()


def _xfs(t, count):
    from gaussiansplats3d_b200 import three_math as TM
    out = []
    for s in range(count):
        a = t + 0.7 * s
        out.append(np.asarray(TM.compose([1.5 * np.cos(a) * (s > 0), 0.3 * np.sin(a), 1.5 * np.sin(a) * (s > 0)], [0.0, np.sin(a / 2), 0.0, np.cos(a / 2)],
                                         [1.0 + 0.1 * s] * 3), np.float64).reshape(16))
    return out


def _base(eye):
    from gaussiansplats3d_b200 import three_math as TM
    return np.asarray(TM.invert(TM.camera_world_matrix(list(eye), [0.0, 0.0, 0.0], [0.0, 1.0, 0.0])), np.float64).reshape(16)


def test_gather_is_the_forest_oracle():
    from gaussiansplats3d_b200 import GsError
    from gaussiansplats3d_b200 import three_math as TM
    N = _N()
    src = _sources(nan=False)           # (a NaN distance has no place in an ordered list)
    src = src + [src[0], src[0]]        # two identical scenes: under identical transforms, exact ties across sub-trees
    e = _engine(sum(_count(s["format"], s["data"]) for s in src))
    try:
        infos, c, a = _upload(e, src)
        e.build_splat_tree(8, 4, 1)
        lv = e.read_splat_tree()
        per = forest_leaves(lv)
        k = len(src)
        for step, eye in enumerate(((0.0, 0.5, 6.0), (4.0, 1.0, -2.0), (0.2, 0.1, 0.8), (-3.0, -2.0, 3.0))):
            xfs = _xfs(0.5 * step, k)
            xfs[-1] = xfs[-2]
            views = [TM.multiply(_base(eye), x) for x in xfs]
            for gather_all in (False, True):
                n = e.gather_for_sort_subtrees(views, 0.9, 0.95, gather_all)
                want, wn = forest_gather(list(zip(per, views)), 0.9, 0.95, gather_all)
                assert n == wn, (step, gather_all)
                got = e.read_buffer(N.GS_BUF_INDEXES_TO_SORT, np.uint32, n) if n else np.zeros(0, np.uint32)
                assert np.array_equal(got, want), (step, gather_all)
        with pytest.raises(GsError) as ei:
            e.gather_for_sort_subtrees(views[:-1], 0.9, 0.95)
        assert ei.value.code == N.GS_ERR_BAD_ARG and f"{k - 1} model views" in str(ei.value) and f"{k} sub-trees" in str(ei.value)
        with pytest.raises(GsError) as ei:
            e.gather_for_sort(views[0], 0.9, 0.95)
        assert ei.value.code == N.GS_ERR_BAD_ARG
    finally:
        e.close()
    # one tree: count = 1 is gs_gather_for_sort
    one = _engine(_count(src[0]["format"], src[0]["data"]))
    try:
        one.upload_scenes([src[0]], sh_degree=2)
        one.build_splat_tree(8, 4, 1)
        assert one.splat_tree_info()["sub_tree_count"] == 1
        mv = _base((0.5, 0.5, 5.0))
        n1 = one.gather_for_sort(mv, 0.9, 0.95)
        g1 = one.read_buffer(N.GS_BUF_INDEXES_TO_SORT, np.uint32, n1)
        n2 = one.gather_for_sort_subtrees([mv], 0.9, 0.95)
        assert n1 == n2 and np.array_equal(one.read_buffer(N.GS_BUF_INDEXES_TO_SORT, np.uint32, n2), g1)
        with pytest.raises(GsError) as ei:
            one.gather_for_sort_subtrees([mv, mv], 0.9, 0.95)
        assert ei.value.code == N.GS_ERR_BAD_ARG
    finally:
        one.close()


class _Dynamic:
    """The records of a dynamic mesh for ray_oracle (local centres, stored scale and rotation), with per-scene visibility."""

    def __init__(self, rec, infos, visible):
        self.of = np.repeat(np.arange(len(infos)), [i["splat_count"] for i in infos])
        self.scene = RO.Scene(rec["center"], rec["scale"], rec["rotation"], rec["alpha"], dynamic=True)
        self.visible = visible

    def inputs(self, i, ellipsoid):
        c, s, F, Inv = self.scene.inputs(i, ellipsoid)
        return (c, s, F, Inv) if self.visible[int(self.of[i])] else (c, (0.0, 0.0, 0.0), F, Inv)


def _assert_hits(got, tot, want, what):
    assert tot == len(want) and got.shape[0] == len(want), (what, tot, len(want))
    assert np.array_equal(got["splat_index"], np.array([h[2] for h in want], np.uint32)), what
    assert _same(got["distance"], [h[0] for h in want]), what
    assert _same(got["origin"], np.array([h[3] for h in want]).reshape(-1, 3)), what
    assert _same(got["normal"], np.array([h[4] for h in want]).reshape(-1, 3)), what


def test_raycast_is_the_forest_oracle():
    from gaussiansplats3d_b200 import GsError
    N = _N()
    src = _mixed(dynamic=True)
    src = src + [src[2]]                # a copy of scene 2, placed on it
    e = _engine(sum(_count(s["format"], s["data"]) for s in src))
    try:
        infos, c, a = _upload(e, src)
        e.build_splat_tree(8, 4, 1)
        rec = e.read_buffer(N.GS_BUF_RAY_RECORDS, N.RAY_RECORD_DTYPE, c.shape[0])
        roots = [RO.build_tree(c[i["splat_offset"]:i["splat_offset"] + i["splat_count"]], a[i["splat_offset"]:i["splat_offset"] + i["splat_count"]], max_centers=4)
                 for i in infos]
        from gaussiansplats3d_b200 import three_math as TM
        proj = TM.make_perspective(50, W / H, 0.1, 1000.0)
        ortho = TM.make_orthographic(-4, 4, 3, -3, 0.1, 1000.0)
        cam = TM.camera_world_matrix([0.3, 0.4, 7.0], [0.0, 0.0, 0.0], [0.0, 1.0, 0.0])
        for step in range(3):
            xfs = _xfs(0.6 * step, len(src))
            xfs[-1] = xfs[2]
            rays = []
            for s, i in enumerate(infos):   # through a kept splat of every scene, down -z from above it
                k = i["splat_offset"] + int(np.flatnonzero(a[i["splat_offset"]:i["splat_offset"] + i["splat_count"]] > 0)[0])
                w = RO.apply_matrix4([float(v) for v in rec["center"][k]], [float(v) for v in xfs[s]])
                rays.append(((w[0], w[1], w[2] + 10.0), (0.0, 0.0, -1.0)))
            rays.append(RO.ray_from_camera(proj, cam, (W / 2, H / 2), (W, H)))
            rays.append(RO.ray_from_camera(ortho, cam, (W / 3, H / 2), (W, H), orthographic=True))
            for vis in ([True] * len(src), [s != 2 for s in range(len(src))]):
                scene = _Dynamic(rec, infos, vis)
                subtrees = [(r, i["splat_offset"], [float(v) for v in x]) for r, i, x in zip(roots, infos, xfs)]
                for ellipsoid in (False, True):
                    for o, d in rays:
                        want = forest_raycast(subtrees, scene, o, d, ellipsoid=ellipsoid)
                        got, tot = e.raycast(o, d, None, ellipsoid=ellipsoid, capacity=len(want) + 3, scene_visibility=vis, sub_tree_from_local=xfs)
                        _assert_hits(got, tot, want, (step, vis, ellipsoid, o))
            # the ray above the copy of scene 2 crosses both overlapping scenes
            want = forest_raycast(subtrees, _Dynamic(rec, infos, [True] * len(src)), *rays[2])
            assert {int(scene.of[h[2]]) for h in want} >= {2, len(src) - 1}
        with pytest.raises(GsError) as ei:
            e.raycast(rays[0][0], rays[0][1], None, capacity=1)
        assert ei.value.code == N.GS_ERR_BAD_ARG
        with pytest.raises(GsError) as ei:
            e.raycast(rays[0][0], rays[0][1], None, capacity=1, sub_tree_from_local=xfs[:-1])
        assert ei.value.code == N.GS_ERR_BAD_ARG
    finally:
        e.close()


def _viewer(**kw):
    from gaussiansplats3d_b200.viewer import Viewer
    return Viewer({**dict(width=W, height=H, sphericalHarmonicsDegree=2, initialCameraPosition=(0, 0.5, 6)), **kw})


def _want_gather(v, leaves):
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.splat_tree import fov_cosines
    base = TM.invert(v.camera.matrixWorld)
    mesh = v.splatMesh
    mesh.fillTransformsArray()
    views = [TM.multiply(base, mesh.getSceneTransform(s)) for s in range(leaves.sub_tree_count)]
    o = leaves.sub_leaf_offsets
    per = [leaves_of(leaves, int(o[s]), int(o[s + 1])) for s in range(leaves.sub_tree_count)]
    return forest_gather(list(zip(per, views)), *fov_cosines(v.renderWidth * v.devicePixelRatio, v.renderHeight * v.devicePixelRatio, v.camera.fov))


def test_viewer_gathers_and_picks_per_scene():
    from gaussiansplats3d_b200 import three_math as TM
    N = _N()
    v = _viewer(dynamicScene=True, splatTree=True, raycast=True)
    try:
        v.addSplatScenes([_opts("l2"), _opts("l0"), _opts("ply")])
        lv = v.splatMesh.getSplatTree().leaves
        assert lv.sub_tree_count == 3
        n = v.splatMesh.getSplatCount()
        rec = v.engine.read_buffer(N.GS_BUF_RAY_RECORDS, N.RAY_RECORD_DTYPE, n)
        cc = v.engine.read_buffer(N.GS_BUF_CENTERS_COLORS, np.uint32, n * 4).reshape(n, 4)
        c, a = cc[:, 1:4].copy().view(np.float32), (cc[:, 0] >> 24).astype(np.uint8)
        infos = v.splatMesh.sceneInfos
        roots = [RO.build_tree(c[i["splat_offset"]:i["splat_offset"] + i["splat_count"]], a[i["splat_offset"]:i["splat_offset"] + i["splat_count"]]) for i in infos]
        for step in range(3):
            t = 0.5 * step
            v.getSplatScene(1).position = (1.5 * np.cos(t), 0.0, 1.5 * np.sin(t))
            v.getSplatScene(2).position = (-1.5 * np.cos(t), 0.5 * np.sin(t), 0.0)
            v.update()
            want, wn = _want_gather(v, lv)
            assert v.splatRenderCount == wn, step
            assert np.array_equal(v.engine.read_buffer(N.GS_BUF_INDEXES_TO_SORT, np.uint32, wn) if wn else np.zeros(0, np.uint32), want), step
            p = v.checkForFocalPointChange(W / 2, H / 2)
            ray = v.raycaster.ray
            xfs = [[float(x) for x in TM.multiply(v.splatMesh.matrixWorld, v.splatMesh.getSceneTransform(s))] for s in range(3)]
            hits = forest_raycast([(r, i["splat_offset"], x) for r, i, x in zip(roots, infos, xfs)], _Dynamic(rec, infos, [True] * 3), ray.origin, ray.direction)
            got = v.raycaster.intersectSplatMesh(v.splatMesh)
            assert [h.splatIndex for h in got] == [h[2] for h in hits], step
            assert _same([h.distance for h in got], [h[0] for h in hits]) and _same([h.origin for h in got], [h[3] for h in hits]), step
            if hits:
                far = np.linalg.norm(np.asarray(hits[0][3]) - np.asarray(v.camera.position, np.float64)) > 0.75
                assert (p is not None) == bool(far) and (p is None or _same(p, hits[0][3])), step
    finally:
        v.dispose()


def test_one_scene_dynamic_viewer_culls_under_its_scene_transform():
    """A one-scene dynamic mesh culls its leaves under baseModelView * sceneTransform(0), as the reference does (Viewer.js:2007-2011)."""
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.splat_tree import fov_cosines
    N = _N()
    v = _viewer(dynamicScene=True, splatTree=True)
    try:
        v.addSplatScenes([dict(_opts("l0"), position=(0.5, 0.0, -2.0), rotation=(0.0, 0.6, 0.0, 0.8))])
        lv = v.splatMesh.getSplatTree().leaves
        assert lv.sub_tree_count == 1
        for position in ((0.5, 0.0, -2.0), (0.0, 0.0, 40.0)):     # in front of the camera, then behind it
            v.getSplatScene(0).position = position
            v.update()
            want, wn = _want_gather(v, lv)
            assert v.splatRenderCount == wn, position
            assert np.array_equal(v.engine.read_buffer(N.GS_BUF_INDEXES_TO_SORT, np.uint32, wn) if wn else np.zeros(0, np.uint32), want), position
        # the leaves at their local positions, which the cull used before it applied the scene transform, are in view
        alone = TO.gather_for_sort(leaves_of(lv), TM.invert(v.camera.matrixWorld), *fov_cosines(W, H, v.camera.fov))
        assert alone[1] > wn
    finally:
        v.dispose()


def test_viewer_add_and_remove_rebuild_the_forest():
    a, b, c = (_viewer(dynamicScene=True, splatTree=True) for _ in range(3))
    try:
        a.addSplatScenes([_opts("l2"), _opts("l0")])
        a.addSplatScenes([_opts("ply")])
        b.addSplatScenes([_opts("l2"), _opts("l0"), _opts("ply")])
        _assert_tree(a.engine.read_splat_tree(), b.engine.read_splat_tree(), "add")
        a.removeSplatScenes([0])
        c.addSplatScenes([_opts("l0"), _opts("ply")])
        ta = a.engine.read_splat_tree()
        assert ta.sub_tree_count == 2
        _assert_tree(ta, c.engine.read_splat_tree(), "remove")
    finally:
        a.dispose(); b.dispose(); c.dispose()
