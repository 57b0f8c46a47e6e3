"""gs_build_splat_tree: the SplatTree built on the GPU from the splats the engine holds is, array for array and bit for bit, the tree the
reference's worker builds (SplatTree.js:132-278) -- checked against the scalar restatement (oracle/tree_oracle.build_leaves) for the
leaves and against the host mirror (splat_tree.SplatTree) for all ten arrays.  Covers split-plane duplicates, the alpha filter, NaN and
infinite centres, the capacity refusal, every load path (the f32 centre the engine holds is the centre the reference's tree sees), the
Viewer's `splatTree` option on GPU-decoded scenes, and gs_read_splat_tree."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent / "golden"))

from oracle import file_oracle as FO  # noqa: E402
from oracle import tree_oracle as TO  # noqa: E402

GOLDEN = Path(__file__).resolve().parent / "golden"
ARRAYS = ("node_min", "node_max", "node_center", "offsets", "indexes", "depth", "all_min", "all_max", "all_parent", "leaf_node")
XF = dict(position=(0.5, -1.25, 2.0), rotation=[0.3, -0.5, 0.2, 0.7874007874011811], scale=(1.5, 0.75, 1.25))


# ---- CPU: what needs no device ------------------------------------------------------------------------------------------------------
def test_options_are_validated_before_the_engine():
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200 import build
    build.build()
    lib = N.load()
    for kw, word in ((dict(max_depth=N.GS_TREE_MAX_DEPTH + 1, max_centers_per_node=1000, min_alpha=1), "max_depth"),
                     (dict(max_depth=8, max_centers_per_node=0, min_alpha=1), "max_centers_per_node")):
        o = N.gs_splat_tree_options(struct_size=C.sizeof(N.gs_splat_tree_options), **kw)
        assert lib.gs_build_splat_tree(None, C.byref(o), None) == N.GS_ERR_BAD_ARG
        assert word in lib.gs_last_error_message().decode()
    o = N.gs_splat_tree_options(struct_size=C.sizeof(N.gs_splat_tree_options), max_depth=N.GS_TREE_MAX_DEPTH, max_centers_per_node=1, min_alpha=0)
    assert lib.gs_build_splat_tree(None, C.byref(o), None) == N.GS_ERR_BAD_ARG and "null engine" in lib.gs_last_error_message().decode()
    assert lib.gs_read_splat_tree(None, None, None) == N.GS_ERR_BAD_ARG


def test_tree_struct_sizes_match_header():
    import subprocess
    import tempfile
    from gaussiansplats3d_b200 import _native as N
    root = Path(__file__).resolve().parent.parent
    src = ('#include "gsplat_b200.h"\n#include <stdio.h>\nint main(){printf("%zu %zu %zu %d\\n",sizeof(gs_splat_tree_options),sizeof(gs_splat_tree_info),'
           'sizeof(gs_splat_tree_arrays),GS_TREE_MAX_DEPTH);return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        (Path(d) / "probe.c").write_text(src)
        subprocess.run(["/usr/bin/gcc", "-I", str(root / "include"), str(Path(d) / "probe.c"), "-o", str(Path(d) / "probe")], check=True)
        out = subprocess.run([str(Path(d) / "probe")], capture_output=True, text=True, check=True).stdout.split()
    assert [int(v) for v in out] == [C.sizeof(N.gs_splat_tree_options), C.sizeof(N.gs_splat_tree_info), C.sizeof(N.gs_splat_tree_arrays), N.GS_TREE_MAX_DEPTH]


# ---- GPU ----------------------------------------------------------------------------------------------------------------------------
def _engine(centers, alphas, capacity=None):
    """An engine whose GS_BUF_CENTERS_COLORS holds these f32 centres and alpha bytes."""
    from gaussiansplats3d_b200.engine import Engine
    c = np.ascontiguousarray(centers, np.float32).reshape(-1, 3)
    n = c.shape[0]
    cc = np.zeros((n, 4), np.uint32)
    cc[:, 0] = 0x00808080 | (np.asarray(alphas, np.uint32) << 24)
    cc[:, 1:] = c.view(np.uint32)
    e = Engine(capacity or n, max_width=64, max_height=64)
    e.upload_splat_data(cc, np.zeros((n, 6), np.float32))
    return e


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a, b, equal_nan=a.dtype.kind == "f")


def _assert_equals_mirror(got, centers, alphas, min_alpha, max_depth, max_centers):
    from gaussiansplats3d_b200.splat_tree import SplatTree
    want = SplatTree(max_depth, max_centers).processSplatMesh(centers, alphas, min_alpha)
    for name in ARRAYS:
        assert _same(getattr(got, name), getattr(want, name)), name
    return want


def _assert_equals_oracle(got, centers, alphas, min_alpha, max_depth, max_centers):
    want = TO.build_leaves(centers, alphas, min_alpha, max_depth, max_centers)
    assert got.count == len(want)
    mn, mx = np.array([w[0] for w in want], np.float64).reshape(-1, 3), np.array([w[1] for w in want], np.float64).reshape(-1, 3)
    assert _same(got.node_min, mn) and _same(got.node_max, mx) and _same(got.node_center, (mx - mn) * 0.5 + mn)
    assert _same(got.depth, np.array([w[2] for w in want], np.int32))
    sizes = np.array([len(w[3]) for w in want], np.int64)
    assert _same(got.offsets, np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32))
    assert _same(got.indexes, np.array([i for w in want for i in w[3]], np.uint32))
    return want


def _build_and_check(centers, alphas, *, min_alpha=1, max_depth=8, max_centers=1000, oracle=True):
    e = _engine(centers, alphas)
    info = e.build_splat_tree(max_depth, max_centers, min_alpha)
    got = e.read_splat_tree()
    want = _assert_equals_mirror(got, centers, alphas, min_alpha, max_depth, max_centers)
    if oracle:
        _assert_equals_oracle(got, centers, alphas, min_alpha, max_depth, max_centers)
    assert (info["leaf_count"], info["node_count"], info["index_count"]) == (want.count, want.all_parent.shape[0], want.indexes.shape[0])
    assert info["has_depth"] == 1 and info["has_nodes"] == 1
    assert info["max_leaf_depth"] == (int(want.depth.max()) if want.count else 0)
    e.close()
    return info, want


def _scene(n, seed, kind):
    from gaussiansplats3d_b200.scenes import synthetic_scene
    raw = synthetic_scene(n, seed=seed, kind=kind)
    return raw.centers.astype(np.float32), raw.colors[:, 3].copy()


@pytest.mark.gpu
@pytest.mark.parametrize("n,max_centers,kind", [(6000, 200, "bonsai"), (3000, 50, "garden"), (4000, 100, "uniform"), (900, 1000, "uniform"), (1, 1000, "bonsai")])
def test_built_tree_matches_oracle_and_mirror(gs, n, max_centers, kind):
    centers, alphas = _scene(n, 3, kind)
    info, want = _build_and_check(centers, alphas, max_centers=max_centers)
    if max_centers > n:
        assert info["leaf_count"] == 1 and info["node_count"] == 1 and info["level_count"] == 1      # the root is the only leaf
    else:
        assert info["leaf_count"] > 8 and info["max_leaf_depth"] >= 2


@pytest.mark.gpu
@pytest.mark.parametrize("min_alpha", [1, 16])
def test_grid_snapped_centres_and_alpha_filter(gs, min_alpha):
    """Centres on a 0.25 grid lie on split planes by the hundred: several memberships per splat, one owner.  Two sevenths of the alphas are 0 or 15."""
    centers, alphas = _scene(5000, 7, "garden")
    centers = (np.round(centers * 4) / 4).astype(np.float32)
    alphas[::7] = 0
    alphas[1::7] = 15
    info, want = _build_and_check(centers, alphas, min_alpha=min_alpha, max_centers=50)
    keep = np.nonzero(alphas >= min_alpha)[0]
    assert np.array_equal(np.sort(want.indexes), keep)
    assert info["max_level_memberships"] > keep.shape[0], "the scene must put centres on split planes"


@pytest.mark.gpu
def test_every_splat_filtered_gives_the_empty_tree(gs):
    centers, alphas = _scene(500, 2, "bonsai")
    e = _engine(centers, np.zeros_like(alphas))
    info = e.build_splat_tree()
    assert (info["leaf_count"], info["node_count"], info["index_count"], info["level_count"]) == (0, 0, 0, 0)
    _assert_equals_mirror(e.read_splat_tree(), centers, np.zeros_like(alphas), 1, 8, 1000)
    assert e.gather_for_sort(np.eye(4).reshape(16), 0.9, 0.9) == 0
    e.close()


@pytest.mark.gpu
def test_defaults_at_120k_and_at_1_2m_splats(gs):
    centers, alphas = _scene(120_000, 9, "bonsai")
    info, _ = _build_and_check(centers, alphas)
    assert info["leaf_count"] > 100
    centers, alphas = _scene(1_200_000, 11, "bonsai")
    info, _ = _build_and_check(centers, alphas, oracle=False)      # the scalar restatement takes minutes here; the mirror is pinned to it above
    assert info["leaf_count"] > 1000 and info["build_ms"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["nan_first", "nan_later", "inf", "nan_first_all_axes"])
@pytest.mark.parametrize("n,max_centers", [(300, 1000), (3000, 100)])
def test_non_finite_centres(gs, case, n, max_centers):
    """The scene box starts at the first kept centre and moves on strict comparisons: a NaN there poisons its axis, a NaN later is
    skipped; a root that stays a leaf keeps a NaN centre, a split drops it; infinities take part."""
    centers, alphas = _scene(n, 5, "bonsai")
    alphas[0] = 0                                            # the first KEPT splat is splat 1
    if case == "nan_first":
        centers[1, 1] = np.nan
    elif case == "nan_first_all_axes":
        centers[1] = np.nan
    elif case == "nan_later":
        centers[17, 0] = np.nan; centers[40] = np.nan
    else:
        centers[5, 0] = np.inf; centers[9, 2] = -np.inf; centers[12, 1] = np.inf
    info, want = _build_and_check(centers, alphas, max_centers=max_centers)
    kept = int((alphas >= 1).sum())
    if max_centers > n:
        assert info["index_count"] == kept
    elif case.startswith("nan"):
        assert info["index_count"] < kept


@pytest.mark.gpu
def test_coincident_centres_and_the_capacity_refusal(gs):
    """64 equal centres: every child box contains all of them.  At max_depth 2 that is 8^3 leaves of which the first owns everything; at
    max_depth 8 the level counts grow eightfold until the build refuses -- an error return from the count pass, with the previous tree
    still in place and the engine fit for the next build."""
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200 import GsError
    pts = np.tile(np.array([[0.25, -1.5, 3.0]], np.float32), (64, 1))
    alphas = np.full(64, 255, np.uint8)
    info, want = _build_and_check(pts, alphas, max_depth=2, max_centers=10)
    assert info["node_count"] == 1 + 8 + 64 + 512 and info["leaf_count"] == 1 and info["max_leaf_depth"] == 3
    assert info["max_level_memberships"] == 512 * 64

    centers, a2 = _scene(4000, 6, "bonsai")
    e = _engine(centers, a2, capacity=4000)
    e.build_splat_tree(8, 100)
    before = e.read_splat_tree()
    mv = np.eye(4).reshape(16)
    n0 = e.gather_for_sort(mv, 0.9, 0.95)
    g0 = e.read_buffer(N.GS_BUF_INDEXES_TO_SORT, np.uint32, n0)
    cc = np.zeros((4000, 4), np.uint32)                      # the same engine now holds 4000 coincident centres
    cc[:, 0] = 0xff808080
    cc[:, 1:] = np.tile(pts[:1], (4000, 1)).view(np.uint32)
    e.upload_splat_data(cc, np.zeros((4000, 6), np.float32))
    with pytest.raises(GsError) as ei:
        e.build_splat_tree(8, 100)
    assert ei.value.code == N.GS_ERR_CAPACITY and "level 4" in str(ei.value) and "memberships" in str(ei.value)
    after = e.read_splat_tree()
    for name in ARRAYS:
        assert _same(getattr(after, name), getattr(before, name)), name
    assert e.gather_for_sort(mv, 0.9, 0.95) == n0 and np.array_equal(e.read_buffer(N.GS_BUF_INDEXES_TO_SORT, np.uint32, n0), g0)
    info = e.build_splat_tree(2, 100)                          # and the next valid build succeeds
    assert info["node_count"] == 585 and info["index_count"] == 4000
    e.close()


def _ply_columns(centers, alphas, rng):
    n = centers.shape[0]
    cols = {"x": centers[:, 0], "y": centers[:, 1], "z": centers[:, 2]}
    for k in range(3):
        cols[f"scale_{k}"] = rng.normal(-3.0, 0.3, n)
    q = rng.normal(0, 1, (n, 4))
    for k in range(4):
        cols[f"rot_{k}"] = q[:, k]
    for k in range(3):
        cols[f"f_dc_{k}"] = rng.normal(0, 1, n)
    cols["opacity"] = -np.log(255.0 / np.maximum(alphas.astype(np.float64), 0.5) - 1 + 1e-6)
    return [(k, "float") for k in cols], {k: np.asarray(v, np.float32) for k, v in cols.items()}


def _check_engine_tree_against_records(v, transform16, max_centers):
    """The tree built from GS_BUF_CENTERS_COLORS == the host tree over the centres the reference's tree sees: getSplatCenter's f64
    centre of the ray record, scene transform applied, stored as f32 (raycaster.record_centers_f32)."""
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.raycaster import record_centers_f32
    n = v.splatMesh.getSplatCount()
    recs = v.engine.read_buffer(N.GS_BUF_RAY_RECORDS, N.RAY_RECORD_DTYPE, n)
    centers = record_centers_f32(recs, transform16)
    info = v.engine.build_splat_tree(8, max_centers, 1)
    assert info["centers_from_ray_records"] == 1               # decoded on an engine with ray records
    # the texel centre is that centre too, unless the section was rounded to f32 before its transform or the centre is not finite
    if not (transform16 is not None and v._ksplat_info["compression_level"] >= 1):
        cc = v.engine.read_buffer(N.GS_BUF_CENTERS_COLORS, np.uint32, 4 * n).reshape(-1, 4)
        finite = np.isfinite(recs["center"]).all(1)
        assert _same(cc[finite, 1:].copy().view(np.float32), centers[finite])
    want = _assert_equals_mirror(v.engine.read_splat_tree(), centers, recs["alpha"], 1, 8, max_centers)
    return want


def _viewer(**kw):
    from gaussiansplats3d_b200.viewer import Viewer
    return Viewer(dict(width=320, height=180, **kw))


@pytest.mark.gpu
@pytest.mark.parametrize("xf", [False, True])
@pytest.mark.parametrize("level", [0, 1, 2])
def test_ksplat_load_paths(gs, level, xf):
    from gaussiansplats3d_b200 import ksplat as K
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.scenes import synthetic_scene
    raw = synthetic_scene(5000, seed=8 + level, kind="garden")
    raw.colors[::11, 3] = 0
    data = K.write(raw.centers, raw.scales, raw.rotations, raw.colors, compression_level=level, minimum_alpha=0)
    v = _viewer(raycast=True)
    v.addSplatSceneFromKSplat(data, **(XF if xf else {}))
    want = _check_engine_tree_against_records(v, TM.compose(XF["position"], XF["rotation"], XF["scale"]) if xf else None, 60)
    assert want.count > 50
    v.dispose()
    for name in sorted(p.name for p in GOLDEN.glob(f"ksplat_handmade_l{level}_*.ksplat")):
        v = _viewer(raycast=True)
        v.addSplatSceneFromKSplat((GOLDEN / name).read_bytes(), **(XF if xf else {}))
        _check_engine_tree_against_records(v, TM.compose(XF["position"], XF["rotation"], XF["scale"]) if xf else None, 3)
        v.dispose()


FILES = (sorted(p.name for p in GOLDEN.glob("*_handmade*.ply")) + sorted(p.name for p in GOLDEN.glob("*_handmade*.splat")) +
         sorted(p.name for p in GOLDEN.glob("spz_handmade*.spz") if "empty" not in p.name))


@pytest.mark.gpu
@pytest.mark.parametrize("optimized", [False, True])
@pytest.mark.parametrize("name", FILES)
def test_file_load_paths(gs, name, optimized):
    """INRIA .ply, compressed .ply, .splat and .spz fixtures in file order and through the optimised (generator) load, with a transform."""
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200 import three_math as TM
    fmt = N.GS_FILE_SPLAT if name.endswith(".splat") else (N.GS_FILE_SPZ if name.endswith(".spz") else N.GS_FILE_PLY)
    v = _viewer(raycast=True, inMemoryCompressionLevel=1 if optimized else 0)
    v.addSplatSceneFromFile((GOLDEN / name).read_bytes(), fmt, progressiveLoad=not optimized, **XF)
    if v.splatMesh.getSplatCount():
        _check_engine_tree_against_records(v, TM.compose(XF["position"], XF["rotation"], XF["scale"]), 3)
    v.dispose()


@pytest.mark.gpu
@pytest.mark.parametrize("optimized", [False, True])
def test_larger_ply_load_paths(gs, optimized):
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200 import three_math as TM
    centers, alphas = _scene(6000, 21, "bonsai")
    data = FO.write_ply(*_ply_columns(centers, alphas, np.random.default_rng(2)), centers.shape[0])
    v = _viewer(raycast=True, inMemoryCompressionLevel=2 if optimized else 0)
    v.addSplatSceneFromFile(data, N.GS_FILE_PLY, progressiveLoad=not optimized, **XF)
    want = _check_engine_tree_against_records(v, TM.compose(XF["position"], XF["rotation"], XF["scale"]), 80)
    assert want.count > 50
    v.dispose()


@pytest.mark.gpu
@pytest.mark.parametrize("loader", ["file", "ksplat"])
def test_viewer_splat_tree_without_raycast_on_decoded_scenes(gs, loader):
    """`splatTree` alone builds the tree on the GPU-decoded paths too, and the frame path culls with it."""
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200 import ksplat as K
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.scenes import synthetic_scene
    from gaussiansplats3d_b200.splat_tree import fov_cosines
    raw = synthetic_scene(30_000, seed=4, kind="bonsai")
    v = _viewer(splatTree=True)
    if loader == "file":
        v.addSplatSceneFromFile(FO.write_ply(*_ply_columns(raw.centers, raw.colors[:, 3], np.random.default_rng(3)), raw.count), N.GS_FILE_PLY)
    else:
        v.addSplatSceneFromKSplat(K.write(raw.centers, raw.scales, raw.rotations, raw.colors, compression_level=0, minimum_alpha=0))
    tree = v.splatMesh.getSplatTree()
    assert tree is not None and tree.leaves.count > 20
    lv = tree.leaves
    cc = v.engine.read_buffer(N.GS_BUF_CENTERS_COLORS, np.uint32, 4 * raw.count).reshape(-1, 4)
    _assert_equals_mirror(lv, cc[:, 1:].copy().view(np.float32), (cc[:, 0] >> 24).astype(np.uint8), 1, 8, 1000)
    leaves = [(lv.node_min[i].tolist(), lv.node_max[i].tolist(), int(lv.depth[i]), lv.indexes[lv.offsets[i]:lv.offsets[i + 1]].tolist()) for i in range(lv.count)]
    v.camera.position = np.asarray((-14.0, 0.0, 0.0), np.float64)          # outside, looking away
    v.camera.look_at((-30.0, 0.0, 0.0))
    count, sort_all = v.gatherSceneNodesForSort()
    assert not sort_all and count < int(lv.indexes.shape[0]) // 2
    want, want_n = TO.gather_for_sort(leaves, TM.invert(v.camera.matrixWorld), *fov_cosines(v.renderWidth, v.renderHeight, v.camera.fov))
    assert count == want_n and np.array_equal(v.engine.read_buffer(N.GS_BUF_INDEXES_TO_SORT, np.uint32, count) if count else np.zeros(0, np.uint32), want)
    v.dispose()


@pytest.mark.gpu
def test_gather_and_raycast_equal_those_over_the_uploaded_host_tree(gs):
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.engine import Engine
    from gaussiansplats3d_b200.raycaster import ray_records_from_raw
    from gaussiansplats3d_b200.scenes import pack_scene, synthetic_scene
    from gaussiansplats3d_b200.splat_tree import SplatTree
    import cases
    raw = synthetic_scene(20_000, seed=14, kind="bonsai")
    raw.centers[:5000] = np.round(raw.centers[:5000] * 2) / 2
    p = pack_scene(raw)
    engines = []
    for built in (True, False):
        e = Engine(raw.count, max_width=64, max_height=64, ray_records=True)
        e.upload_splat_data(p.centers_colors, p.covariances, p.sh, p.sh_degree)
        e.upload_ray_records(ray_records_from_raw(raw))
        if built:
            e.build_splat_tree(8, 150)
        else:
            lv = SplatTree(8, 150).processSplatMesh(raw.centers, raw.colors[:, 3], 1)
            e.upload_splat_tree(lv)
            e.upload_splat_tree_nodes(lv)
        engines.append(e)
    a, b = engines
    hits = 0
    for eye, target in (((1.5, 2.7, -6.4), (0.45, 1.95, 1.5)), ((0.2, 0.1, -0.3), (3.0, 0.5, 2.0)), ((-14.0, 0.0, 0.0), (-30.0, 0.0, 0.0))):
        _, view, _ = cases.camera_mvp(eye=eye, target=target, up=(0.02, -0.76, -0.65))
        na, nb = a.gather_for_sort(view, 0.9, 0.95), b.gather_for_sort(view, 0.9, 0.95)
        assert na == nb
        if na:
            assert np.array_equal(a.read_buffer(N.GS_BUF_INDEXES_TO_SORT, np.uint32, na), b.read_buffer(N.GS_BUF_INDEXES_TO_SORT, np.uint32, nb))
        d = np.asarray(target, np.float64) - np.asarray(eye, np.float64)
        d /= np.linalg.norm(d)
        for ell in (False, True):
            ha, ta = a.raycast(eye, d, None, ellipsoid=ell, capacity=256)
            hb, tb = b.raycast(eye, d, None, ellipsoid=ell, capacity=256)
            assert ta == tb and ha.tobytes() == hb.tobytes()
            hits += ta
    assert hits > 0
    a.close(); b.close()


@pytest.mark.gpu
def test_builds_repeat_exactly_and_follow_the_uploaded_scene(gs):
    centers, alphas = _scene(50_000, 30, "garden")
    centers = (np.round(centers * 8) / 8).astype(np.float32)
    e = _engine(centers, alphas)
    e.build_splat_tree(8, 300)
    first = e.read_splat_tree()
    e.build_splat_tree(8, 300)
    second = e.read_splat_tree()
    for name in ARRAYS:
        assert getattr(first, name).tobytes() == getattr(second, name).tobytes(), name
    c2, a2 = _scene(20_000, 31, "bonsai")                     # a second scene in the same engine replaces the tree
    cc = np.zeros((20_000, 4), np.uint32)
    cc[:, 0] = 0x00808080 | (a2.astype(np.uint32) << 24)
    cc[:, 1:] = c2.view(np.uint32)
    e.upload_splat_data(cc, np.zeros((20_000, 6), np.float32))
    e.build_splat_tree(8, 300)
    _assert_equals_mirror(e.read_splat_tree(), c2, a2, 1, 8, 300)
    e.close()


@pytest.mark.gpu
def test_read_splat_tree_skips_null_pointers_and_reports_an_uploaded_tree(gs):
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200 import Engine, GsError
    from gaussiansplats3d_b200.splat_tree import SplatTree
    centers, alphas = _scene(3000, 40, "bonsai")
    e = Engine(3000, max_width=64, max_height=64)
    with pytest.raises(GsError) as ei:
        e.build_splat_tree()
    assert ei.value.code == N.GS_ERR_NOT_READY
    info = e.splat_tree_info()
    assert (info["leaf_count"], info["node_count"], info["has_depth"], info["has_nodes"]) == (0, 0, 0, 0)
    lv = SplatTree(8, 100).processSplatMesh(centers, alphas, 1)
    e.upload_splat_tree(lv)
    info = e.splat_tree_info()
    assert (info["leaf_count"], info["index_count"], info["has_depth"], info["has_nodes"], info["build_ms"]) == (lv.count, lv.indexes.shape[0], 0, 0, 0.0)
    got = e.read_splat_tree()
    assert got.depth is None and got.all_min is None and got.leaf_node is None
    for name in ("node_min", "node_max", "node_center", "offsets", "indexes"):
        assert _same(getattr(got, name), getattr(lv, name)), name
    depth = np.zeros(lv.count, np.int32)
    a = N.gs_splat_tree_arrays(struct_size=C.sizeof(N.gs_splat_tree_arrays), depth=N.ptr(depth))
    assert e._lib.gs_read_splat_tree(e._h, C.byref(a), None) == N.GS_ERR_NOT_READY and "depth" in e._lib.gs_last_error_message().decode()
    parent = np.zeros(lv.all_parent.shape[0], np.int32)
    a = N.gs_splat_tree_arrays(struct_size=C.sizeof(N.gs_splat_tree_arrays), parent=N.ptr(parent))
    assert e._lib.gs_read_splat_tree(e._h, C.byref(a), None) == N.GS_ERR_NOT_READY
    e.upload_splat_tree_nodes(lv)
    got = e.read_splat_tree()
    assert got.depth is None
    for name in ("all_min", "all_max", "all_parent", "leaf_node"):
        assert _same(getattr(got, name), getattr(lv, name)), name
    # only the arrays asked for are written
    offsets = np.full(lv.count + 1, 0xdeadbeef, np.uint32)
    a = N.gs_splat_tree_arrays(struct_size=C.sizeof(N.gs_splat_tree_arrays), node_offsets=N.ptr(offsets))
    N.check(e._lib.gs_read_splat_tree(e._h, C.byref(a), None), "gs_read_splat_tree")
    assert np.array_equal(offsets, lv.offsets)
    e.close()
