"""GPU: gs_compute_bounding_box (SplatMesh.computeBoundingBox on the GPU) is bit-equal to the reference's loop over the reference's
Float32Array centres (tests/test_bounding_box.py: f64 transform, f32 store, strict compares, the seed rule) for .ksplat levels 0/1/2,
.ply SH0-3, compressed .ply, .splat and .spz files (file order and through the generator), host-packed scenes, and mixed multi-scene
meshes, static and dynamic, with and without scene transforms and ray records, every sceneIndex and both applySceneTransforms.  Edge
cases: NaN / +-inf centres, -0/+0 ties in both orders, empty scenes, 1-3 splats, counts past one CTA and one wave, 16 M splats.  The
single-splat getters are checked against the ray oracle's restatement, with their refusals."""
import struct
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent))

from oracle import ray_oracle as RO  # noqa: E402
from test_bounding_box import bits_equal, centers_f32, js_box  # noqa: E402
from test_raycast_gpu import ROT_XF, _ksplat_records, _transform  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden"
I16 = np.eye(4).reshape(16)
POS, SCALE = (0.5, -1.25, 2.0), (1.5, 0.75, 1.25)
KSPLATS = sorted(p.name for p in GOLDEN.glob("ksplat_handmade_*.ksplat"))
FILES = (sorted(p.name for p in GOLDEN.glob("file_handmade_*.ply")) + sorted(p.name for p in GOLDEN.glob("pcply_handmade_*.ply"))
         + ["file_handmade_basic.splat", "spz_handmade_sh1.spz", "spz_handmade_v1.spz", "spz_handmade_scales.spz"])


def _fmt(name):
    from gaussiansplats3d_b200.loaders import SceneFormat
    return {".ply": SceneFormat.Ply, ".splat": SceneFormat.Splat, ".spz": SceneFormat.Spz, ".ksplat": SceneFormat.KSplat}[Path(name).suffix]


def _viewer(**kw):
    from gaussiansplats3d_b200.viewer import Viewer
    return Viewer(dict(width=64, height=32, **kw))


def _records(engine, n):
    from gaussiansplats3d_b200 import _native as N
    return engine.read_buffer(N.GS_BUF_RAY_RECORDS, N.RAY_RECORD_DTYPE, n)


def _held(engine, lo, hi):
    """The f32 centres GS_BUF_CENTERS_COLORS holds for splats [lo, hi)."""
    from gaussiansplats3d_b200 import _native as N
    return engine.read_buffer(N.GS_BUF_CENTERS_COLORS, np.uint32, 4 * (hi - lo), 16 * lo).reshape(-1, 4)[:, 1:].copy().view(np.float32)


def _assert_box(got, want):
    assert bits_equal(got[0], want[0]) and bits_equal(got[1], want[1]), (got, want)


def _load(v, name, xf, opt_level=None):
    data = (GOLDEN / name).read_bytes()
    kw = dict(position=POS, rotation=ROT_XF, scale=SCALE) if xf else {}
    if name.endswith(".ksplat"):
        v.addSplatSceneFromKSplat(data, **kw)
    else:
        v.inMemoryCompressionLevel = opt_level or 0
        v.addSplatSceneFromFile(data, _fmt(name), progressiveLoad=opt_level is None, **kw)


def _check_static_single(name, xf, opt_level=None, c64=None):
    """One static scene, loaded with and without ray records.  c64: the reference's f64 centres (None: the ray records, which
    tests/test_raycast_gpu.py pins to the loaders' restatements)."""
    from gaussiansplats3d_b200._native import GsError
    t = _transform() if xf else I16
    with_rec, without = _viewer(raycast=True), _viewer()
    _load(with_rec, name, xf, opt_level)
    _load(without, name, xf, opt_level)
    n = with_rec.splatMesh.getSplatCount()
    if c64 is None:
        c64 = _records(with_rec.engine, n)["center"]
    level = without._ksplat_info["compression_level"]
    want_raw, want_xf = js_box(centers_f32(c64)), js_box(centers_f32(c64, t))
    for v in (with_rec, without):
        sm = v.splatMesh
        for scene in (None, 0):
            if v is without and xf and level >= 1:
                # without ray records a level-1/2 centre was rounded to f32 before its transform: the box of the centres held
                _assert_box(sm.computeBoundingBox(True, scene), js_box(_held(v.engine, 0, n)))
            else:
                _assert_box(sm.computeBoundingBox(True, scene), want_xf)
            if v is without and xf:
                with pytest.raises(GsError, match="only the transformed centres are kept"):
                    sm.computeBoundingBox(False, scene)
            else:
                _assert_box(sm.computeBoundingBox(False, scene), want_raw)
        with pytest.raises(ValueError, match="Invalid scene index"):
            sm.computeBoundingBox(False, 1)
        with pytest.raises(GsError, match="invalid scene index"):
            v.engine.compute_bounding_box(1)
        v.dispose()


@pytest.mark.parametrize("xf", [False, True])
@pytest.mark.parametrize("name", KSPLATS)
def test_ksplat_box_is_the_references(name, xf):
    data = (GOLDEN / name).read_bytes()
    _check_static_single(name, xf, c64=np.array([r[0] for r in _ksplat_records(data)], np.float64))


@pytest.mark.parametrize("xf", [False, True])
@pytest.mark.parametrize("name", FILES)
def test_file_box_is_the_references(name, xf):
    _check_static_single(name, xf)


@pytest.mark.parametrize("level", [0, 1, 2])
@pytest.mark.parametrize("name", ["file_handmade_sh2.ply", "file_handmade_basic.splat", "spz_handmade_sh2.spz", "pcply_handmade_sh1.ply"])
def test_generated_box_is_the_references(name, level):
    _check_static_single(name, True, opt_level=level)
    _check_static_single(name, False, opt_level=level)


MIXED = [("ksplat_handmade_l1_sh0_many_buckets.ksplat", dict(position=POS, rotation=ROT_XF, scale=SCALE)), ("file_handmade_nonfinite.ply", {}),
         ("spz_handmade_empty.spz", {}), ("file_handmade_basic.splat", dict(position=(-2.0, 0.0, 1.0))),
         ("ksplat_handmade_l2_sh2_two_sections.ksplat", dict(scale=(0.5, 2.0, 1.0))), ("spz_handmade_sh1.spz", {}), ("pcply_handmade_edges.ply", {})]


def _mixed(dynamic, raycast, optimize):
    v = _viewer(dynamicScene=dynamic, raycast=raycast, optimizeSplatData=optimize, inMemoryCompressionLevel=1)
    v.addSplatScenes([dict(format=_fmt(n), data=(GOLDEN / n).read_bytes(), **kw) for n, kw in MIXED])
    return v


@pytest.mark.parametrize("optimize", [False, True])
@pytest.mark.parametrize("dynamic", [False, True])
def test_multi_scene_box_every_scene_both_ways(dynamic, optimize):
    from gaussiansplats3d_b200._native import GsError
    ref = _mixed(dynamic, True, optimize)
    infos = [(i["splat_offset"], i["splat_offset"] + i["splat_count"], i["compression_level"]) for i in ref.splatMesh.sceneInfos]
    total = infos[-1][1]
    c64 = _records(ref.engine, total)["center"]
    T = [sc.transform for sc in ref.splatMesh.scenes]
    has_xf = [not sc.is_identity() for sc in ref.splatMesh.scenes]
    assert any(has_xf) and not all(has_xf) and any(b == a for a, b, _ in infos)
    for raycast in (True, False):
        v = ref if raycast else _mixed(dynamic, False, optimize)
        sm = v.splatMesh
        assert [(i["splat_offset"], i["splat_count"]) for i in sm.sceneInfos] == [(a, b - a) for a, b, _ in infos]
        for apply in (False, True):
            parts, refused = [], []
            for s, (a, b, level) in enumerate(infos):
                c = c64[a:b]
                if not apply:
                    refused.append(not dynamic and not raycast and has_xf[s])
                    parts.append(centers_f32(c))
                elif dynamic:
                    parts.append(centers_f32(c if raycast else centers_f32(c).astype(np.float64), T[s]))
                    refused.append(False)
                elif raycast or not has_xf[s] or level == 0:
                    parts.append(centers_f32(c, T[s]))
                    refused.append(False)
                else:
                    parts.append(_held(v.engine, a, b))   # deviation: transformed after the f32 rounding
                    refused.append(False)
            for scene in [None] + list(range(len(infos))):
                sel = range(len(infos)) if scene is None else [scene]
                if any(refused[s] for s in sel):
                    with pytest.raises(GsError, match="only the transformed centres are kept"):
                        sm.computeBoundingBox(apply, scene)
                    continue
                _assert_box(sm.computeBoundingBox(apply, scene), js_box(np.concatenate([parts[s] for s in sel])))
        with pytest.raises(ValueError, match="Invalid scene index"):
            sm.computeBoundingBox(True, len(infos))
        if v is not ref:
            v.dispose()
    # a dynamic mesh's box follows its scenes' current transforms
    if dynamic:
        ref.getSplatScene(0).position = (3.0, 2.0, 1.0)
        a, b, _ = infos[0]
        _assert_box(ref.splatMesh.computeBoundingBox(True, 0), js_box(centers_f32(c64[a:b], ref.getSplatScene(0).transform)))
    ref.dispose()


def _host_engine(centers, dynamic=False):
    from gaussiansplats3d_b200.engine import Engine
    c = np.ascontiguousarray(centers, np.float32).reshape(-1, 3)
    n = c.shape[0]
    e = Engine(max(n, 1), dynamic_mode=dynamic, max_width=64, max_height=64)
    if n:
        cc = np.empty((n, 4), np.uint32)
        cc[:, 0] = 0xff808080
        cc[:, 1:] = c.view(np.uint32)
        e.upload_splat_data(cc, np.zeros((n, 6), np.float16))
    return e


def _edge_sets():
    rng = np.random.default_rng(11)
    nan, inf = np.float32(np.nan), np.float32(np.inf)
    out = {"one": rng.normal(size=(1, 3)), "two": rng.normal(size=(2, 3)), "three": rng.normal(size=(3, 3)),
           "nan_seed": np.array([[nan, 1, nan], [2, nan, 3], [-1, 5, nan]]),
           "nan_elsewhere": np.array([[1, 2, 3], [nan, nan, nan], [-4, 9, nan], [nan, -7, 0]]),
           "inf": np.array([[0, 0, 0], [inf, -inf, 1], [-inf, inf, nan], [1, 2, -inf]]),
           "zeros_neg_first": np.array([[1, -0.0, 0.0], [-0.0, 1, 1], [0.0, 0.0, -0.0], [2, 3, 4]]),
           "zeros_pos_first": np.array([[1, 0.0, -0.0], [0.0, 1, 1], [-0.0, -0.0, 0.0], [2, 3, 4]])}
    for n in (257, 256 * 132 * 8 + 1000, 3 * 256 * 132 * 8 + 7):   # past one CTA, past one wave of the grid, several waves
        c = rng.normal(size=(n, 3)).astype(np.float32)
        k = rng.integers(1, n, size=12)
        c[k[0:3], 0] = np.nan
        c[k[3], 1], c[k[4], 1] = c[:, 1].min() - 1, c[:, 1].min() - 1          # equal minima: the first stays
        c[k[5], 2], c[k[6], 2] = np.inf, -np.inf
        out[f"n{n}"] = c
    zeros = np.abs(rng.normal(size=(5000, 3))).astype(np.float32) + 1
    zeros[[700, 4100], 0] = [0.0, -0.0]
    zeros[[600, 4200], 1] = [-0.0, 0.0]
    out["zeros_far_apart"] = zeros
    return {k: np.asarray(v, np.float32) for k, v in out.items()}


EDGE = _edge_sets()


@pytest.mark.parametrize("dynamic", [False, True])
@pytest.mark.parametrize("case", sorted(EDGE))
def test_edge_cases(case, dynamic):
    c = EDGE[case]
    e = _host_engine(c, dynamic)
    _assert_box(e.compute_bounding_box(-1, False), js_box(c))
    _assert_box(e.compute_bounding_box(0, False), js_box(c))
    t = _transform() if dynamic else I16        # a static host-packed scene counts as loaded without a transform: the identity applies
    _assert_box(e.compute_bounding_box(-1, True, [t] if dynamic else None), js_box(centers_f32(c, t)))
    e.close()


def test_empty_scene_is_the_zero_vector():
    e = _host_engine(np.zeros((0, 3)))
    for apply in (False, True):
        _assert_box(e.compute_bounding_box(-1, apply), (np.zeros(3, np.float32), np.zeros(3, np.float32)))
    e.close()


def test_16m_splats():
    rng = np.random.default_rng(16)
    n = 1 << 24
    c = (rng.standard_normal((n, 3), np.float32) * np.float32(40.0))
    c[rng.integers(1, n, 64), rng.integers(0, 3, 64)] = np.nan
    e = _host_engine(c)
    _assert_box(e.compute_bounding_box(-1, False), js_box(c))
    _assert_box(e.compute_bounding_box(-1, True), js_box(centers_f32(c, I16)))
    e.close()


@pytest.mark.parametrize("kind", ["static", "static_xf", "dynamic_xf"])
def test_host_packed_viewer_box(kind):
    from gaussiansplats3d_b200.scenes import synthetic_scene
    raw = synthetic_scene(3000, seed=9, kind="bonsai")
    raw.centers[0, 1] = np.nan
    for raycast in (False, True):
        v = _viewer(dynamicScene=kind == "dynamic_xf", raycast=raycast)
        if kind == "static":
            v.addSplatScene(raw)
            _assert_box(v.splatMesh.computeBoundingBox(), js_box(raw.centers))
            _assert_box(v.splatMesh.computeBoundingBox(True), js_box(centers_f32(raw.centers, I16)))
        else:
            v.addSplatScene(raw, position=POS, rotation=ROT_XF, scale=SCALE)
            if kind == "dynamic_xf":
                _assert_box(v.splatMesh.computeBoundingBox(), js_box(raw.centers))
                _assert_box(v.splatMesh.computeBoundingBox(True), js_box(centers_f32(raw.centers, _transform())))
            else:   # the packed centres carry the transform: their box, and no untransformed one
                _assert_box(v.splatMesh.computeBoundingBox(True), js_box(v.splatMesh.raw.centers))
                with pytest.raises(ValueError, match="only the\\s+transformed centres are held"):
                    v.splatMesh.computeBoundingBox(False)
        v.dispose()


def _bits64(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a[~np.isnan(a)].view(np.uint64), b[~np.isnan(b)].view(np.uint64))


@pytest.mark.parametrize("dynamic", [False, True])
def test_getters_match_the_oracle_on_every_scene(dynamic):
    from gaussiansplats3d_b200 import _native as N
    v = _viewer(dynamicScene=dynamic, raycast=True, optimizeSplatData=False)
    kinds = [("ksplat_handmade_l1_sh1.ksplat", dict(position=POS, rotation=ROT_XF, scale=SCALE, splatAlphaRemovalThreshold=100)),
             ("file_handmade_sh1.ply", {}), ("ksplat_handmade_l2_sh2_two_sections.ksplat", dict(rotation=ROT_XF))]
    v.addSplatScenes([dict(format=_fmt(n), data=(GOLDEN / n).read_bytes(), **kw) for n, kw in kinds])
    sm = v.splatMesh
    recs = _records(v.engine, sm.getSplatCount())
    cc = v.engine.read_buffer(N.GS_BUF_CENTERS_COLORS, np.uint32, 4 * sm.getSplatCount()).reshape(-1, 4)
    want_k = _ksplat_records((GOLDEN / kinds[0][0]).read_bytes())
    saw_floored = False
    for s, info in enumerate(sm.sceneInfos):
        T = sm.scenes[s].transform
        for i in range(info["splat_offset"], info["splat_offset"] + info["splat_count"]):
            r = recs[i]
            for apply in (None, False, True):
                on = (not dynamic) if apply is None else apply
                c, sc, q = RO.splat_inputs(r["center"], r["scale"], r["rotation"], not on, T)
                assert _bits64(sm.getSplatCenter(i, apply), c)
                got_s, got_q = sm.getSplatScaleAndRotation(i, apply)
                assert _bits64(got_s, sc) and _bits64(got_q, q)
            rgba = sm.getSplatColor(i)
            assert list(rgba[:3]) == [int(cc[i, 0]) & 255, (int(cc[i, 0]) >> 8) & 255, (int(cc[i, 0]) >> 16) & 255]
            assert rgba[3] == r["alpha"]
            if s == 0:
                assert rgba[3] == want_k[i][3]              # the stored byte, not the floored one (SplatBuffer.js:294-305)
                saw_floored |= (int(cc[i, 0]) >> 24) != rgba[3]
    assert saw_floored
    v.dispose()


def test_getters_without_ray_records():
    from gaussiansplats3d_b200 import _native as N
    v = _viewer(optimizeSplatData=False)
    name = "ksplat_handmade_l1_sh1.ksplat"
    v.addSplatScenes([dict(format=_fmt(name), data=(GOLDEN / name).read_bytes(), splatAlphaRemovalThreshold=100)])
    sm = v.splatMesh
    for getter in ("getSplatCenter", "getSplatScaleAndRotation"):
        with pytest.raises(ValueError, match="raycast"):
            getattr(sm, getter)(0)
    want = _ksplat_records((GOLDEN / name).read_bytes())
    cc = v.engine.read_buffer(N.GS_BUF_CENTERS_COLORS, np.uint32, 4 * sm.getSplatCount()).reshape(-1, 4)
    refused = 0
    for i in range(sm.getSplatCount()):
        if (int(cc[i, 0]) >> 24) == 0:
            with pytest.raises(ValueError, match="raycast"):
                sm.getSplatColor(i)
            refused += 1
        else:
            assert sm.getSplatColor(i)[3] == want[i][3]
    assert refused
    with pytest.raises(IndexError):
        sm.getSplatColor(sm.getSplatCount())
    v.dispose()


def test_box_leaves_frames_unchanged():
    """The call reads the scene and writes only its own buffers: a frame after it is bit-identical to one before."""
    from gaussiansplats3d_b200 import _native as N
    v = _viewer(raycast=True)
    v.addSplatSceneFromKSplat((GOLDEN / "ksplat_handmade_l2_sh2_two_sections.ksplat").read_bytes())
    v.camera.update(); v.updateSplatMesh()
    a = v.frame(frame_format=N.GS_FRAME_RGBA32F, flip_y=False).copy()
    v.splatMesh.computeBoundingBox(True)
    b = v.frame(frame_format=N.GS_FRAME_RGBA32F, flip_y=False)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    v.dispose()


def test_ksplat_level_is_read_from_the_header():
    # the level-dependent expectation above reads the level the engine reports; pin it to the file's
    for name in KSPLATS:
        data = (GOLDEN / name).read_bytes()
        v = _viewer()
        v.addSplatSceneFromKSplat(data)
        assert v._ksplat_info["compression_level"] == struct.unpack_from("<H", data, 20)[0]
        v.dispose()
