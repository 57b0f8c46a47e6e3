"""GPU: gs_raycast (Raycaster.intersectSplatMesh on the GPU) is bit-identical to the scalar oracle (oracle/ray_oracle.py) -- hit count,
splat indexes, world-space origins, normals and distances, in both modes -- for 64 screen positions per scene, on synthetic, file-loaded
(.ply / compressed .ply / .splat), .ksplat (levels 0/1/2) and host-packed scenes, static with and without a scene transform and dynamic,
with perspective and orthographic rays.  Also: the ray records each loader writes, capacities, >1e5 hits on one ray, statuses, stale
records, repeatability, the Viewer's focal-point method, and that ray records leave every existing buffer and frame unchanged."""
import math
import struct
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent / "golden"))

from oracle import file_oracle as FO  # noqa: E402
from oracle import ray_oracle as RO  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden"
W, H = 640, 360
ROT_XF = [0.3, -0.5, 0.2, 0.7874007874011811]


def _transform():
    from gaussiansplats3d_b200 import three_math as TM
    return TM.compose((0.5, -1.25, 2.0), ROT_XF, (1.5, 0.75, 1.25))


def _bits_equal(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint64), b[~nb].view(np.uint64))


def _rays(scene_center, radius, ortho):
    """64 screen positions (8 x 8 grid over the frame) of a camera looking at the scene."""
    from gaussiansplats3d_b200 import three_math as TM
    c = np.asarray(scene_center, np.float64)
    world = TM.camera_world_matrix(c + np.array([0.3, 0.4, 1.0]) * 2.5 * radius, c, [0.0, 1.0, 0.0])
    proj = (TM.make_orthographic(-radius * 1.6, radius * 1.6, radius * 0.9, -radius * 0.9, 0.1, 1000.0) if ortho
            else TM.make_perspective(50, W / H, 0.1, 1000.0))
    out = []
    for iy in range(8):
        for ix in range(8):
            out.append(RO.ray_from_camera(proj, world, ((ix + 0.37) * W / 8, (iy + 0.61) * H / 8), (W, H), orthographic=ortho))
    return out


def _check(engine, root, scene, from_local, *, rays, ellipsoid, capacity=None):
    """Every ray: gs_raycast == oracle, bit for bit."""
    total_hits = 0
    for o, d in rays:
        want = RO.intersect_splat_mesh(root, scene, o, d, from_local, ellipsoid=ellipsoid)
        cap = len(want) + 3 if capacity is None else capacity
        got, total = engine.raycast(o, d, from_local, ellipsoid=ellipsoid, capacity=cap)
        assert total == len(want)
        k = min(cap, len(want))
        assert got.shape[0] == k
        want = want[:k]
        assert np.array_equal(got["splat_index"], np.array([h[2] for h in want], np.uint32))
        assert _bits_equal(got["distance"], [h[0] for h in want])
        assert _bits_equal(got["origin"], np.array([h[3] for h in want]).reshape(-1, 3))
        assert _bits_equal(got["normal"], np.array([h[4] for h in want]).reshape(-1, 3))
        total_hits += total
    return total_hits


def _oracle_tree(recs, transform16, dynamic):
    from gaussiansplats3d_b200.raycaster import record_centers_f32
    return RO.build_tree(record_centers_f32(recs, None if dynamic else transform16), recs["alpha"])


def _read_records(engine, n):
    from gaussiansplats3d_b200 import _native as N
    return engine.read_buffer(N.GS_BUF_RAY_RECORDS, N.RAY_RECORD_DTYPE, n)


def _oracle_scene(recs, transform16, dynamic):
    return RO.Scene(recs["center"], recs["scale"], recs["rotation"], recs["alpha"], dynamic=dynamic, transform16=transform16)


def _check_viewer(v, transform16, *, dynamic=False, modes=(False, True), ortho=(False, True)):
    from gaussiansplats3d_b200 import three_math as TM
    n = v.engine.max_splat_count
    recs = _read_records(v.engine, n)
    root = _oracle_tree(recs, transform16, dynamic)
    scene = _oracle_scene(recs, transform16, dynamic)
    from_local = TM.multiply(TM.identity(), transform16) if dynamic and transform16 is not None else TM.identity()
    pts = np.asarray(recs["center"], np.float64)
    pts = pts[np.isfinite(pts).all(1)]
    center, radius = (pts.mean(0), max(float(np.abs(pts - pts.mean(0)).max()), 0.5)) if pts.size else (np.zeros(3), 1.0)
    hits = 0
    for ell in modes:
        for orth in ortho:
            hits += _check(v.engine, root, scene, from_local, rays=_rays(center, radius, orth), ellipsoid=ell)
    return hits


# ---- records each loader writes ------------------------------------------------------------------------------------------------
def _ksplat_records(data: bytes):
    """SplatBuffer.getSplatCenter / getSplatScaleAndRotation / getSplatColor inputs of every splat (SplatBuffer.js:221-305), restated."""
    f = data
    rd = lambda fmt, off: struct.unpack_from(fmt, f, off)[0]  # noqa: E731
    sections, splats, level = rd("<I", 4), rd("<I", 12), rd("<H", 20)
    kC, kS, kR, kSH, kRange = (12, 6, 6), (12, 6, 6), (16, 8, 8), (4, 2, 1), (1, 32767, 32767)
    half = lambda b: float(np.frombuffer(struct.pack("<H", b), np.float16)[0])  # noqa: E731
    out = []
    base = 4096 + 1024 * sections
    for s in range(sections):
        h = 4096 + 1024 * s
        count, bsize, bcount, block, storage = rd("<I", h + 4), rd("<I", h + 8), rd("<I", h + 12), rd("<f", h + 16), rd("<H", h + 20)
        sr = rd("<I", h + 24) or kRange[level]
        full, partial, deg = rd("<I", h + 32), rd("<I", h + 36), rd("<H", h + 40)
        ncomp = 24 if deg == 2 else (9 if deg == 1 else 0)
        bps = kC[level] + kS[level] + kR[level] + 4 + kSH[level] * ncomp
        lens = [rd("<I", base + 4 * k) for k in range(partial)]
        buckets = base + 4 * partial
        data_base = buckets + storage * bcount
        sf = (block / 2.0) / sr
        for i in range(count):
            r = data_base + i * bps
            if level == 0:
                c = [rd("<f", r + 4 * k) for k in range(3)]
                sc = [rd("<f", r + 12 + 4 * k) for k in range(3)]
                w, x, y, z = (rd("<f", r + 24 + 4 * k) for k in range(4))
                a = f[r + 43]
            else:
                if i < full * bsize:
                    b = i // bsize
                else:
                    rem, b = i - full * bsize, full
                    for ln in lens:
                        if rem < ln:
                            break
                        rem -= ln
                        b += 1
                c = [(rd("<H", r + 2 * k) - sr) * sf + rd("<f", buckets + 12 * b + 4 * k) for k in range(3)]
                sc = [half(rd("<H", r + 6 + 2 * k)) for k in range(3)]
                w, x, y, z = (half(rd("<H", r + 12 + 2 * k)) for k in range(4))
                a = f[r + 23]
            out.append((c, sc, [x, y, z, w], a))
        base = data_base + bps * count
    assert len(out) <= splats
    return out


def _assert_records(recs, want):
    assert recs.shape[0] == len(want)
    assert _bits_equal(recs["center"], np.array([w[0] for w in want], np.float64))
    assert _bits_equal(recs["scale"].astype(np.float64), np.array([w[1] for w in want], np.float32).astype(np.float64))
    assert _bits_equal(recs["rotation"].astype(np.float64), np.array([w[2] for w in want], np.float32).astype(np.float64))
    assert np.array_equal(recs["alpha"], np.array([w[3] for w in want], np.uint8))


def _viewer(**kw):
    from gaussiansplats3d_b200.viewer import Viewer
    return Viewer(dict(width=W, height=H, raycast=True, **kw))


KSPLATS = sorted(p.name for p in GOLDEN.glob("ksplat_handmade_*.ksplat"))
FILES = sorted(p.name for p in GOLDEN.glob("*_handmade*.ply")) + sorted(p.name for p in GOLDEN.glob("*_handmade*.splat"))


@pytest.mark.parametrize("xf", [False, True])
@pytest.mark.parametrize("name", KSPLATS)
def test_ksplat_fixture_raycast_matches_oracle(name, xf):
    data = (GOLDEN / name).read_bytes()
    v = _viewer()
    t = _transform() if xf else None
    if xf:
        v.addSplatSceneFromKSplat(data, position=(0.5, -1.25, 2.0), rotation=ROT_XF, scale=(1.5, 0.75, 1.25))
    else:
        v.addSplatSceneFromKSplat(data)
    _assert_records(_read_records(v.engine, v.engine.max_splat_count), _ksplat_records(data))   # f64 centres at levels 1/2
    _check_viewer(v, t)
    v.dispose()


@pytest.mark.parametrize("name", FILES)
def test_file_fixture_raycast_matches_oracle(name):
    from gaussiansplats3d_b200 import _native as N
    data = (GOLDEN / name).read_bytes()
    fmt = N.GS_FILE_SPLAT if name.endswith(".splat") else N.GS_FILE_PLY
    v = _viewer()
    v.addSplatSceneFromFile(data, fmt)
    if not name.startswith("pcply"):
        rec, _, ambiguous = FO.level0_records(fmt, data, 0)
        r = rec[:, :44].copy()
        want = [(list(r[i, 0:12].view(np.float32).astype(np.float64)), list(r[i, 12:24].view(np.float32)),
                 list(r[i, 24:40].view(np.float32)[[1, 2, 3, 0]]), int(r[i, 43])) for i in range(r.shape[0])]
        got = _read_records(v.engine, len(want))
        ok = ~ambiguous                           # scale / alpha of flagged splats depend on how exp rounds
        assert _bits_equal(got["center"], np.array([w[0] for w in want]))
        assert _bits_equal(got["rotation"].astype(np.float64), np.array([w[2] for w in want], np.float32).astype(np.float64))
        assert _bits_equal(got["scale"][ok].astype(np.float64), np.array([w[1] for w in want], np.float32)[ok].astype(np.float64))
    _check_viewer(v, None)
    v.dispose()


def _synthetic(n, seed, snap=False):
    from gaussiansplats3d_b200.scenes import synthetic_scene
    raw = synthetic_scene(n, seed=seed, kind="bonsai")
    if snap:   # centres on a 0.5 grid: many lie exactly on leaf faces
        raw.centers[: n // 2] = np.round(raw.centers[: n // 2] * 2) / 2
    raw.colors[::97, 3] = 0      # below minAlpha: not in the tree
    raw.colors[1::89, 3] = 1     # the alpha-1 ellipsoid quirk
    raw.scales[2::101] = 0.0     # skipped by the scale epsilon
    return raw


@pytest.mark.parametrize("kind", ["static", "static_xf", "dynamic_xf"])
def test_host_packed_synthetic_matches_oracle(kind):
    raw = _synthetic(6000, 4, snap=True)
    dyn = kind == "dynamic_xf"
    v = _viewer(dynamicScene=dyn)
    if kind == "static":
        v.addSplatScene(raw)
    else:
        v.addSplatScene(raw, position=(0.5, -1.25, 2.0), rotation=ROT_XF, scale=(1.5, 0.75, 1.25))
    t = None if kind == "static" else _transform()
    recs = _read_records(v.engine, raw.count)
    assert _bits_equal(recs["center"], raw.centers.astype(np.float32).astype(np.float64))
    # the viewer's tree (built from the mesh's centres) is the one the oracle builds from the same records
    from gaussiansplats3d_b200 import three_math as TM
    root = RO.build_tree(v.splatMesh.raw.centers if not dyn else raw.centers, raw.colors[:, 3])
    scene = _oracle_scene(recs, t, dyn)
    from_local = t if dyn else TM.identity()
    hits = 0
    for ell in (False, True):
        for orth in (False, True):
            hits += _check(v.engine, root, scene, from_local, rays=_rays(np.zeros(3) if t is None else np.asarray(t[12:15]), 6.0, orth), ellipsoid=ell)
    assert hits > 0
    v.dispose()


def _bare_engine(n, recs, pts, alphas, *, dynamic=True, transform16=None):
    from gaussiansplats3d_b200.engine import Engine
    from gaussiansplats3d_b200.splat_tree import SplatTree
    e = Engine(n, dynamic_mode=dynamic, ray_records=True)
    e.upload_ray_records(recs, 0, transform16)
    lv = SplatTree().processSplatMesh(pts, alphas, 1)
    e.upload_splat_tree(lv)
    e.upload_splat_tree_nodes(lv)
    return e


def test_capacities_and_more_than_1e5_hits_on_one_ray():
    from gaussiansplats3d_b200 import _native as N
    n = 120_000
    rng = np.random.default_rng(9)
    recs = np.zeros(n, N.RAY_RECORD_DTYPE)
    # a line of splats parallel to z at x = y = 0.3 (never on a box face), inside a box widened by four corner splats: the leaves that
    # hold the line contain the ray, so every line splat is a candidate and a hit
    recs["center"] = np.concatenate([np.full((n, 2), 0.3), rng.uniform(-20, 20, (n, 1))], 1).astype(np.float32)
    recs["center"][::5, 2] = np.round(recs["center"][::5, 2])          # equal distances: ties resolved by traversal order
    recs["center"][:4, :2] = [[-1, -1], [-1, 1], [1, -1], [1, 1]]
    recs["scale"] = 1.0
    recs["rotation"] = [0, 0, 0, 1]
    recs["alpha"] = 255
    e = _bare_engine(n, recs, recs["center"].astype(np.float32), recs["alpha"])
    root = RO.build_tree(recs["center"].astype(np.float32), recs["alpha"])
    scene = _oracle_scene(recs, None, True)
    o, d = [float(np.float32(0.3)), float(np.float32(0.3)), 30.0], [0.0, 0.0, -1.0]
    want = RO.intersect_splat_mesh(root, scene, o, d, RO.IDENTITY)
    assert len(want) > 100_000
    for cap in (0, 1, 1000, len(want), len(want) + 10):
        got, total = e.raycast(o, d, None, capacity=cap)
        assert total == len(want) and got.shape[0] == min(cap, total)
        if cap:
            assert np.array_equal(got["splat_index"], [h[2] for h in want[:cap]])
            assert _bits_equal(got["distance"], [h[0] for h in want[:cap]])
            assert _bits_equal(got["origin"], np.array([h[3] for h in want[:cap]]))
    a, _ = e.raycast(o, d, None, capacity=5000)
    b, _ = e.raycast(o, d, None, capacity=5000)
    assert a.tobytes() == b.tobytes()
    got, total = e.raycast([o[0], o[1], 30.0], [0.0, 0.0, 1.0], None, capacity=4)      # away from everything
    assert total == 0 and got.shape[0] == 0
    got, total = e.raycast(o, d, None, capacity=4, scene_visible=False)
    assert total == 0
    e.close()


def test_statuses_and_stale_records():
    import ctypes as C
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.engine import Engine
    from gaussiansplats3d_b200.scenes import pack_scene
    raw = _synthetic(3000, 2)
    e = Engine(raw.count, ray_records=False, max_width=64, max_height=64)
    with pytest.raises(N.GsError) as ei:
        e.raycast([0, 0, 5], [0, 0, -1])
    assert ei.value.code == N.GS_ERR_NOT_READY
    e.close()
    e = Engine(raw.count, ray_records=True, max_width=64, max_height=64)
    with pytest.raises(N.GsError) as ei:                                   # no records yet
        e.raycast([0, 0, 5], [0, 0, -1])
    assert ei.value.code == N.GS_ERR_NOT_READY
    from gaussiansplats3d_b200.raycaster import ray_records_from_raw
    e.upload_ray_records(ray_records_from_raw(raw))
    with pytest.raises(N.GsError) as ei:                                   # no tree
        e.raycast([0, 0, 5], [0, 0, -1])
    assert ei.value.code == N.GS_ERR_NOT_READY
    from gaussiansplats3d_b200.splat_tree import SplatTree
    lv = SplatTree().processSplatMesh(raw.centers, raw.colors[:, 3], 1)
    e.upload_splat_tree(lv)
    with pytest.raises(N.GsError) as ei:                                   # leaves without their nodes
        e.raycast([0, 0, 5], [0, 0, -1])
    assert ei.value.code == N.GS_ERR_NOT_READY
    e.upload_splat_tree_nodes(lv)
    i = int(np.nonzero((raw.colors[:, 3] >= 1) & (raw.scales.min(1) > 1e-3))[0][0])
    c = raw.centers[i].astype(np.float64)
    _, total = e.raycast([c[0], c[1], c[2] + 10], [0, 0, -1], capacity=2)    # along z through a splat's centre: its leaf is reached
    assert total > 0
    p = N.gs_raycast_params()
    p.struct_size = C.sizeof(p)
    cnt = C.c_uint32(0)
    assert e._lib.gs_raycast(e._h, C.byref(p), None, 4, C.byref(cnt)) == N.GS_ERR_BAD_ARG     # capacity > 0 without hits
    assert e._lib.gs_raycast(e._h, None, None, 0, C.byref(cnt)) == N.GS_ERR_BAD_ARG
    assert e._lib.gs_raycast(e._h, C.byref(p), None, 0, None) == N.GS_ERR_BAD_ARG
    assert e._lib.gs_raycast(e._h, C.byref(p), None, 0, C.byref(cnt)) == N.GS_OK
    pk = pack_scene(raw)
    e.upload_splat_data(pk.centers_colors, pk.covariances)                 # refreshes the splats, not the records
    with pytest.raises(N.GsError) as ei:
        e.raycast([0, 0, 5], [0, 0, -1])
    assert ei.value.code == N.GS_ERR_NOT_READY
    e.upload_ray_records(ray_records_from_raw(raw))
    e.raycast([0, 0, 5], [0, 0, -1])
    e.close()


def test_viewer_focal_point_on_ply_matches_oracle():
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.scenes import synthetic_scene
    raw = synthetic_scene(20_000, seed=3, kind="garden")
    data = FO.write_ply(*_ply_columns(raw), raw.count)
    v = _viewer(initialCameraPosition=(1.5, 2.7, -6.4), initialCameraLookAt=(0.4, 1.9, 1.5))
    v.addSplatSceneFromFile(data, N.GS_FILE_PLY)
    recs = _read_records(v.engine, raw.count)
    root = _oracle_tree(recs, None, False)
    scene = _oracle_scene(recs, None, False)
    n_hits = 0
    for x, y in ((320, 180), (100, 50), (600, 300), (10, 350)):
        o, d = RO.ray_from_camera(v.camera.projectionMatrix, v.camera.matrixWorld, (x, y), (W, H))
        want = RO.intersect_splat_mesh(root, scene, o, d, RO.IDENTITY)
        got = v.checkForFocalPointChange(x, y)
        if want and RO.length([want[0][3][k] - v.camera.position[k] for k in range(3)]) > 0.75:
            assert got is not None and _bits_equal(got, want[0][3])
            n_hits += 1
        else:
            assert got is None
    assert n_hits > 0
    v.dispose()


def _ply_columns(raw):
    cols = {"x": raw.centers[:, 0], "y": raw.centers[:, 1], "z": raw.centers[:, 2],
            "scale_0": np.log(raw.scales[:, 0]), "scale_1": np.log(raw.scales[:, 1]), "scale_2": np.log(raw.scales[:, 2]),
            "rot_0": raw.rotations[:, 3], "rot_1": raw.rotations[:, 0], "rot_2": raw.rotations[:, 1], "rot_3": raw.rotations[:, 2],
            "f_dc_0": (raw.colors[:, 0] / 255.0 - 0.5) / 0.28209479177387814, "f_dc_1": (raw.colors[:, 1] / 255.0 - 0.5) / 0.28209479177387814,
            "f_dc_2": (raw.colors[:, 2] / 255.0 - 0.5) / 0.28209479177387814,
            "opacity": -np.log(255.0 / np.maximum(raw.colors[:, 3], 1) - 1 + 1e-6)}
    return [(k, "float") for k in cols], {k: np.asarray(v, np.float32) for k, v in cols.items()}


@pytest.mark.parametrize("loader", ["ksplat", "file"])
def test_ray_records_leave_engine_buffers_and_frames_unchanged(loader):
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.viewer import Viewer
    if loader == "ksplat":
        data, add = (GOLDEN / "ksplat_handmade_l1_sh1.ksplat").read_bytes(), "addSplatSceneFromKSplat"
        args = ()
    else:
        data, add = (GOLDEN / "file_handmade_sh2.ply").read_bytes(), "addSplatSceneFromFile"
        args = (N.GS_FILE_PLY,)
    out = []
    for ray in (False, True):
        v = Viewer(dict(width=W, height=H, raycast=ray, sphericalHarmonicsDegree=2, initialCameraPosition=(0, 1, 6)))
        getattr(v, add)(data, *args, position=(0.5, -1.25, 2.0), rotation=ROT_XF, scale=(1.5, 0.75, 1.25))
        n = v.engine.max_splat_count
        bufs = [v.engine.read_buffer(N.GS_BUF_CENTERS_COLORS, np.uint32, 4 * n), v.engine.read_buffer(N.GS_BUF_COVARIANCES, np.uint32, 6 * n),
                v.engine.read_buffer(N.GS_BUF_CENTERS, np.int32, 4 * n)]
        v.camera.update(); v.updateSplatMesh(); v.update()
        bufs.append(v.frame(frame_format=N.GS_FRAME_RGBA32F, flip_y=False))
        out.append(bufs)
        v.dispose()
    for a, b in zip(*out):
        assert a.tobytes() == b.tobytes()
