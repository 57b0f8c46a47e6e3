"""GPU: the sorter's integer centres on every load path equal JavaScript's `Math.round(f32 * 1000)` stored into an Int32Array
(tests/js_int.py) at NaN, +-inf and products beyond 2^31; a scene with such splats sorts and renders like the reference; and
GS_ERR_BUCKET_RANGE (DESIGN.md §2) is reported at its exact boundary by every entry that sorts, after which the engine works as new.

One engine per case.  Every load is checked twice: an integer-centre engine against js_int of the centres the load's oracle decodes,
and a float-centre engine, whose sorter centres must be the f32 bits of the decoded centres unchanged (NaN as stored)."""
import sys
from pathlib import Path

import numpy as np
import pytest

import blend_f64 as BF
import frame_f64 as FF
import js_int
import spz_oracle as SO
from test_sorter_centers import BUCKET_EDGES, F32_MAX, _edge_centers, _ksplat_level0, edge_bucket_ksplat

sys.path.insert(0, str(Path(__file__).resolve().parent / "golden"))

from oracle import file_oracle as FO  # noqa: E402
from oracle import generate_oracle as GO  # noqa: E402
from oracle import ksplat_oracle as KO  # noqa: E402
from oracle import pcply_oracle as PO  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden"
NAN, INF = float("nan"), float("inf")


def _poisoned(c):
    """Centres whose integer centre a saturating or INT_MIN cast gets wrong: non-finite, or |x * 1000| >= 2^31."""
    c = np.asarray(c, np.float32)
    with np.errstate(all="ignore"):
        return ~np.isfinite(c) | (np.abs(c.astype(np.float64) * 1000.0) >= 2.0**31)


def _check_sorter_centers(gs, n, upload, want_centers):
    """upload(engine) on an integer and a float engine; the sorter centres against the oracle's decoded f32 centres."""
    from gaussiansplats3d_b200 import _native as N
    want_centers = np.asarray(want_centers, np.float32).reshape(n, 3)
    assert _poisoned(want_centers).any(), "the case has no centre where the conversion matters"
    for integer in (True, False):
        with gs.Engine(n, max_width=64, max_height=64, integer_based_sort=integer) as e:
            upload(e)
            cc = e.read_buffer(N.GS_BUF_CENTERS_COLORS, np.uint32, 4 * n).reshape(n, 4)
            got_c = np.ascontiguousarray(cc[:, 1:]).view(np.float32)
            same = (got_c.view(np.uint32) == want_centers.view(np.uint32)) | (np.isnan(got_c) & np.isnan(want_centers))
            assert same.all(), f"decoded centres differ at {np.flatnonzero(~same.all(1))[:8]}"
            cen = e.read_buffer(N.GS_BUF_CENTERS, np.int32 if integer else np.uint32, 4 * n).reshape(n, 4)
            if integer:
                want = js_int.integer_centers(want_centers)
                bad = np.flatnonzero((cen != want).any(1))
                assert bad.size == 0, f"integer centres differ at {bad[:8]}: {cen[bad[:4]].tolist()} != {want[bad[:4]].tolist()}"
            else:
                assert np.array_equal(cen[:, :3], cc[:, 1:]), "float sorter centres are not the decoded f32 bits"
                assert (cen[:, 3] == np.float32(1.0).view(np.uint32)).all()


# ---- gs_upload_ksplat ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("level", [0, 1, 2])
def test_ksplat_sorter_centers(gs, level):
    """Level 0: the edge values stored as centres; levels 1 and 2: the edge values in bucket centres."""
    data = _ksplat_level0(_edge_centers(seed=5)) if level == 0 else edge_bucket_ksplat(level)
    want = KO.decode(data)
    n = want["count"]
    if level:
        assert n > 64 * len(BUCKET_EDGES)
    _check_sorter_centers(gs, n, lambda e: e.upload_ksplat(data), want["centers"])


# ---- gs_upload_file / gs_upload_file_optimized --------------------------------------------------------------------------------------
def _rng_attrs(n, seed):
    rng = np.random.default_rng(seed)
    return rng, rng.uniform(-5.0, -2.0, (n, 3)), rng.normal(0, 1, (n, 4)), rng.uniform(0.1, 0.9, (n, 3))


def _ply_edges():
    c = _edge_centers(seed=6)
    n = len(c)
    rng, ls, q, col = _rng_attrs(n, 7)
    names = ["x", "y", "z", "f_dc_0", "f_dc_1", "f_dc_2", "opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    cols = dict(x=c[:, 0], y=c[:, 1], z=c[:, 2], f_dc_0=col[:, 0], f_dc_1=col[:, 1], f_dc_2=col[:, 2], opacity=rng.uniform(0.5, 4.0, n),
                scale_0=ls[:, 0], scale_1=ls[:, 1], scale_2=ls[:, 2], rot_0=q[:, 0], rot_1=q[:, 1], rot_2=q[:, 2], rot_3=q[:, 3])
    return FO.write_ply([(k, "float") for k in names], cols, n)


def _splat_edges():
    c = _edge_centers(seed=8)
    n = len(c)
    rng, ls, _, _ = _rng_attrs(n, 9)
    rgba = rng.integers(1, 256, (n, 4)).astype(np.uint8)
    rgba[:, 3] = np.maximum(rgba[:, 3], 20)
    return FO.write_splat(c, np.exp(ls).astype(np.float32), rgba, rng.integers(0, 256, (n, 4)).astype(np.uint8))


def _pcply_edges():
    """Six chunks of 256 splats (the last one partial): position extremes of NaN, +-inf, the f32 maximum, +-3e6 and 2^31 / 1000."""
    rng = np.random.default_rng(10)
    nc, n = 6, 5 * 256 + 100
    ext = {k: np.tile(v, nc).astype(np.float64) for k, v in (("min_x", -2.0), ("min_y", -2.0), ("min_z", -2.0), ("max_x", 2.0),
                                                            ("max_y", 2.0), ("max_z", 2.0))}
    ext["min_x"][0] = ext["max_x"][0] = NAN
    ext["min_y"][1], ext["max_y"][1] = INF, INF
    ext["min_z"][2], ext["max_z"][2] = -INF, -1.0
    ext["min_x"][3], ext["max_x"][3] = -3e6, 3e6
    ext["min_y"][4], ext["max_y"][4] = -F32_MAX, F32_MAX
    ext["min_z"][5], ext["max_z"][5] = 2147483.0, 2147484.0
    for a in "xyz":
        ext[f"min_scale_{a}"], ext[f"max_scale_{a}"] = np.full(nc, -6.0), np.full(nc, -2.0)
    chunk_props = [(k, "float") for k in PO.EXTREMES[:12]]
    vcols = {k: rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32) for k in PO.PACKED}
    vcols["packed_color"] |= np.uint32(0x80)                      # alpha well above the removal threshold
    return PO.write_pcply(chunk_props, ext, nc, [(k, "uint") for k in PO.PACKED], vcols, n)


def _spz_edges(version):
    """v1: float16 positions +-inf, NaN, +-65504 and ordinary halves; v2 at fractionalBits 0: 24-bit positions up to +-2^23."""
    rng = np.random.default_rng(11 + version)
    n = 300
    if version == 1:
        pos = np.float16(rng.uniform(-4, 4, (n, 3))).view(np.uint16).copy()
        edges = [0x7C00, 0xFC00, 0x7E00, 0x7BFF, 0xFBFF]
        for k in range(3):
            pos[k * len(edges):(k + 1) * len(edges), k] = edges
    else:
        v = rng.integers(-4000, 4000, (n, 3))
        edges = [8388607, -8388608, 3_000_000, -3_000_000, 2_147_484, -2_147_484, 4_294_968]
        for k in range(3):
            v[k * len(edges):(k + 1) * len(edges), k] = edges
        pos = np.stack([(v & 0xFFFFFF) >> (8 * b) & 0xFF for b in range(3)], 2).reshape(n, 9)
    alphas = rng.integers(30, 256, n)
    return SO.write_spz(pos, alphas, rng.integers(0, 256, (n, 3)), rng.integers(0, 256, (n, 3)), rng.integers(0, 256, (n, 3)),
                        version=version, fractional_bits=0 if version == 2 else 12)


FILE_CASES = {
    "ply-handmade-nonfinite": (FO.PLY, lambda: (GOLDEN / "file_handmade_nonfinite.ply").read_bytes()),
    "ply-edges": (FO.PLY, _ply_edges),
    "splat-edges": (FO.SPLAT, _splat_edges),
    "pcply-handmade-edges": (FO.PLY, lambda: (GOLDEN / "pcply_handmade_edges.ply").read_bytes()),
    "pcply-edges": (FO.PLY, _pcply_edges),
    "spz-handmade-v1": (SO.SPZ, lambda: SO.packed((GOLDEN / "spz_handmade_v1.spz").read_bytes())),
    "spz-handmade-fb0": (SO.SPZ, lambda: SO.packed((GOLDEN / "spz_handmade_fb0.spz").read_bytes())),
    "spz-v1-edges": (SO.SPZ, lambda: _spz_edges(1)),
    "spz-fb0-edges": (SO.SPZ, lambda: _spz_edges(2)),
}


def _level0_image(fmt, data):
    if fmt == SO.SPZ:
        return SO.level0_image(data)[0]
    if fmt == FO.PLY and data.startswith(b"ply") and b"element chunk" in data[:2048]:
        return PO.level0_image(data)[0]
    return FO.level0_image(fmt, data)[0]


@pytest.mark.parametrize("name", sorted(FILE_CASES))
def test_file_sorter_centers(gs, name):
    """gs_upload_file (file order, level 0) against the centres of the oracle's level-0 image."""
    fmt, make = FILE_CASES[name]
    data = make()
    want = KO.decode(_level0_image(fmt, data))
    _check_sorter_centers(gs, want["count"], lambda e: e.upload_file(fmt, data), want["centers"])


@pytest.mark.parametrize("name", ["ply-handmade-nonfinite", "ply-edges", "splat-edges", "pcply-edges", "spz-v1-edges", "spz-fb0-edges"])
def test_file_optimized_sorter_centers(gs, name):
    """gs_upload_file_optimized at level 0 against the centres of oracle/generate_oracle's image: NaN partition keys sort last, so the
    poisoned splats keep their place in that image."""
    fmt, make = FILE_CASES[name]
    data = make()
    if fmt == SO.SPZ:
        rec, c64, sh, deg, _ = SO.generator_inputs(data, 0)
    else:
        rec, c64, sh, deg, _ = GO.generator_inputs(fmt, data, 0)
    want = KO.decode(GO.generate(rec, c64, sh, deg, level=0, minimum_alpha=0))
    _check_sorter_centers(gs, want["count"], lambda e: e.upload_file_optimized(fmt, data, compression_level=0, minimum_alpha=0), want["centers"])


# ---- the host path ------------------------------------------------------------------------------------------------------------------
def test_viewer_host_sorter_centers(gs):
    """Viewer.addSplatScene with raw arrays: the host conversion (scenes.integer_centers) reaches the engine."""
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.scenes import RawScene, synthetic_scene
    from gaussiansplats3d_b200.viewer import Viewer
    c = _edge_centers(seed=12)
    n = len(c)
    base = synthetic_scene(n, 12, "bonsai", 0)
    raw = RawScene(c, base.scales, base.rotations, base.colors, None, 0)
    for integer in (True, False):
        v = Viewer(dict(width=64, height=64, integerBasedSort=integer))
        v.addSplatScene(raw)
        cen = v.engine.read_buffer(N.GS_BUF_CENTERS, np.int32 if integer else np.uint32, 4 * n).reshape(n, 4)
        if integer:
            assert np.array_equal(cen, js_int.integer_centers(c))
        else:
            assert np.array_equal(cen[:, :3], c.view(np.uint32))
        v.dispose()


# ---- end to end ---------------------------------------------------------------------------------------------------------------------
W, H = 1000, 600
# the reference's integer centre of each is 0, +-1294967296 (3e6 wraps) or -204 (-4294967.5 wraps); 2147483.75, which wraps to
# -2147483546, is left out: times any odd row element it lands next to +-2^31, and the reference's own range map would overflow
POISON_VALUES = [NAN, INF, -INF, 1e30, -1e30, 3e6, -3e6, F32_MAX, -F32_MAX, -4294967.5]


def _irow(mvp32):
    m = np.asarray(mvp32, np.float32).reshape(16)
    return np.array([int(np.float64(m[k]) * 1000.0) for k in (2, 6, 10)], np.int64)


def _span(centers_i32, irow):
    d = (centers_i32[:, :3].astype(np.int64) * irow[None, :]).sum(1)
    d = (d + 2**31) % 2**32 - 2**31
    return int(d.max() - d.min())


def _old_device(c):
    """The conversion k_ksplat_decode used before: a saturating cast (NaN -> 0)."""
    with np.errstate(all="ignore"):
        r = np.floor(c.astype(np.float64) * 1000.0 + 0.5)
    return np.where(np.isnan(r), 0, np.clip(np.nan_to_num(r, posinf=2**31 - 1, neginf=-2**31), -2**31, 2**31 - 1)).astype(np.int64)


def _old_host(c):
    """The conversion NumPy's cast gave on x86: INT_MIN for every out-of-range or non-finite value."""
    with np.errstate(all="ignore"):
        r = np.floor(c.astype(np.float64) * 1000.0 + 0.5)
    return np.where(np.isfinite(r) & (np.abs(r) < 2**31), np.nan_to_num(r), -2**31).astype(np.int64)


def _e2e_scene():
    """A 200 K-splat bonsai scene and 30 poisoned splats (one value in one coordinate each), interleaved.  The finite coordinates of a
    poisoned splat put it 50 units behind the camera, so it is culled whatever the poisoned value does to its projection."""
    from gaussiansplats3d_b200.scenes import CAMERAS, RawScene, synthetic_scene
    base = synthetic_scene(200_000, 21, "bonsai", 0)
    cam = CAMERAS["bonsai"]
    pos, look = np.asarray(cam["position"]), np.asarray(cam["look_at"])
    behind = pos - 50.0 * (look - pos) / np.linalg.norm(look - pos)
    rows = []
    for k in range(3):
        for v in POISON_VALUES:
            r = behind.copy()
            r[k] = v
            rows.append(r)
    pc = np.array(rows, np.float32)
    m = len(pc)
    rng = np.random.default_rng(22)
    at = np.sort(rng.choice(base.count + m, m, replace=False))
    keep = np.setdiff1d(np.arange(base.count + m), at)
    centers = np.empty((base.count + m, 3), np.float32)
    centers[keep], centers[at] = base.centers, pc
    def put(a, extra):
        out = np.empty((base.count + m,) + a.shape[1:], a.dtype)
        out[keep], out[at] = a, extra
        return out
    colors = base.colors.copy()
    colors[:, 3] = np.maximum(colors[:, 3], 1)           # every splat survives the .ksplat writer's alpha floor
    raw = RawScene(centers, put(base.scales, np.full((m, 3), 0.05, np.float32)), put(base.rotations, np.tile(np.float32([0, 0, 0, 1]), (m, 1))),
                   put(colors, np.full((m, 4), 200, np.uint8)), None, 0)
    clean = RawScene(base.centers, base.scales, base.rotations, colors, None, 0)
    return raw, clean, at


def _viewer_options(offset):
    from gaussiansplats3d_b200.scenes import CAMERAS
    cam = CAMERAS["bonsai"]
    return dict(width=W, height=H, cameraUp=cam["up"], initialCameraPosition=tuple(np.asarray(cam["position"]) + offset),
                initialCameraLookAt=cam["look_at"])


def _transforms():
    """Scene transforms of the dynamic two-scene case: scene 0 in place, scene 1 moved."""
    from gaussiansplats3d_b200 import three_math as TM
    return np.stack([TM.identity(), TM.compose((0.25, -0.5, 0.75), (0.0, 0.0, 0.0, 1.0), (1.0, 1.0, 1.0))]).astype(np.float32)


def _dynamic_span(centers_i32, mvp, transforms, scene):
    """Distance span of the dynamic integer mode: per scene the third row of mvp * T in f32, left to right, truncated x1000, and the
    four-term wrapping dot product with w = 1000 (sorter.cpp's dynamic branch)."""
    m = np.asarray(mvp, np.float32).reshape(16)
    d = np.zeros(len(scene), np.int64)
    for s, t in enumerate(transforms):
        t = np.asarray(t, np.float32).reshape(16)
        rf = []
        for c in range(4):
            acc = np.float32(m[2] * t[4 * c])
            acc = np.float32(acc + np.float32(m[6] * t[4 * c + 1]))
            acc = np.float32(acc + np.float32(m[10] * t[4 * c + 2]))
            rf.append(np.float32(acc + np.float32(m[14] * t[4 * c + 3])))
        ri = np.array([int(np.float64(v) * 1000.0) for v in rf], np.int64)
        sel = scene == s
        d[sel] = (centers_i32[sel].astype(np.int64) * ri[None, :]).sum(1)
    d = (d + 2**31) % 2**32 - 2**31
    return int(d.max() - d.min())


def _pick_camera(centers):
    """The first of a few nearby bonsai cameras whose integer row has only odd elements (with an even one, INT_MAX or INT_MIN times
    it cancels the wrap), whose reference distances fit the int32 range map (static and dynamic), and where both old conversions
    overflow it."""
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.viewer import Viewer
    good = js_int.integer_centers(centers)
    scene = (np.arange(len(centers)) >= len(centers) // 2).astype(np.uint32)
    for i in range(300):
        offset = 0.01 * np.array([i % 7, (i // 7) % 7, i // 49], np.float64)
        v = Viewer(_viewer_options(offset))
        v.camera.update()
        mvp = TM.multiply(v.camera.projectionMatrix, TM.invert(v.camera.matrixWorld)).astype(np.float32)
        row = _irow(mvp)
        if (row % 2 != 0).all() and _span(good, row) < 2**31 - 1 and _span(_old_device(centers), row) >= 2**31 \
                and _span(_old_host(centers), row) >= 2**31 and _dynamic_span(good, mvp, _transforms(), scene) < 2**31 - 1:
            return offset, mvp, row, scene
    pytest.fail("no camera near the bonsai view meets the conditions")


def _expected_order(oracle_mod, idx, centers_i32, mvp, scene=None, transforms=None):
    n = len(idx)
    dyn = scene is not None
    want = oracle_mod.port_sort_indexes(idx, centers_i32, None, mvp, scene, transforms, 1 << 16, n, n, n, False, True, dyn)
    if oracle_mod.have_ref():
        ref = oracle_mod.ref_sort_indexes(idx, centers_i32, None, mvp, scene, transforms, 1 << 16, n, n, n, False, True, dyn)
        assert np.array_equal(ref, want), "the C restatement and the compiled reference sorter disagree"
    return want


@pytest.mark.parametrize("load", ["host", "ksplat"])
def test_poisoned_scene_sorts_and_renders(gs, oracle_mod, load):
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200 import ksplat as K
    from gaussiansplats3d_b200.viewer import Viewer
    raw, clean, at = _e2e_scene()
    n = raw.count
    offset, mvp, row, scene = _pick_camera(raw.centers)
    print(f"\n[{load}] camera offset {offset.tolist()}, integer row {row.tolist()}")
    assert (row % 2 != 0).all()
    want_c = js_int.integer_centers(raw.centers)
    v = Viewer(_viewer_options(offset))
    if load == "host":
        v.addSplatScene(raw)
    else:
        info = v.addSplatSceneFromKSplat(K.write(raw.centers, raw.scales, raw.rotations, raw.colors, None, 0, compression_level=0))
        assert info["splat_count"] == n
    e = v.engine
    v.camera.update()
    v.updateSplatMesh()
    assert np.array_equal(v.mvp_matrix().astype(np.float32), mvp)
    cen = e.read_buffer(N.GS_BUF_CENTERS, np.int32, 4 * n).reshape(n, 4)
    assert np.array_equal(cen, want_c)
    # the default integer sort: identity and shuffled index lists
    ident = np.arange(n, dtype=np.uint32)
    out, _ = e.sort(mvp, n, n, None)
    assert np.array_equal(out, _expected_order(oracle_mod, ident, want_c, mvp))
    perm = np.random.default_rng(23).permutation(n).astype(np.uint32)
    out, _ = e.sort(mvp, n, n, perm)
    assert np.array_equal(out, _expected_order(oracle_mod, perm, want_c, mvp))
    # the frame: within the f64 blend bound of the GPU's own raw records, poisoned splats culled, same binning load as the clean scene
    u = v.uniforms()
    order = np.empty(n, np.uint32)
    got = e.frame(mvp, u, W, H, n, None, frame_format=N.GS_FRAME_RGBA32F, flip_y=False, sorted_out=order)
    assert np.array_equal(order, _expected_order(oracle_mod, ident, want_c, mvp))
    inst = e.timings()["tile_instances"]
    ps = e.read_projected(n)
    assert (ps["valid"][at] == 0).all(), f"poisoned splats drawn: {at[ps['valid'][at] != 0]}"
    FF.check_blend(f"poisoned scene ({load})", got, BF.read_records(e, n), order, W, H)
    v.dispose()
    vc = Viewer(_viewer_options(offset))
    vc.addSplatScene(clean)
    vc.camera.update()
    vc.updateSplatMesh()
    vc.engine.frame(mvp, vc.uniforms(), W, H, clean.count, None, frame_format=N.GS_FRAME_RGBA32F, flip_y=False)
    assert vc.engine.timings()["tile_instances"] == inst
    vc.dispose()
    # dynamic mode, two scenes: the same sorter centres, the second half in a moved scene
    transforms = _transforms()
    with gs.Engine(n, dynamic_mode=True) as d:
        d.upload_centers(cen, scene)
        for idx in (None, perm):
            out, _ = d.sort(mvp, n, n, idx, transforms=transforms)
            want = _expected_order(oracle_mod, ident if idx is None else idx, want_c, mvp, scene, transforms)
            assert np.array_equal(out, want)


# ---- GS_ERR_BUCKET_RANGE ------------------------------------------------------------------------------------------------------------
BUCKET_MSG = "distances overflow the int32/f32 range map"


def _distances(n, dmin, dmax, seed):
    d = np.random.default_rng(seed).integers(dmin, dmax + 1, n, dtype=np.int64)
    d[[7, n // 2]] = dmin, dmax
    return d.astype(np.int32)


def _sort_args(d, R, idx):
    n = len(d)
    return (idx, None, d, np.eye(4, dtype=np.float32).reshape(16), None, None, R, n, n, n, True, True, False)


def test_bucket_range_boundary_precomputed(gs, oracle_mod):
    """A distance span of exactly 2^31 - 1 sorts (bit-exact, buckets included); a span of 2^31 is GS_ERR_BUCKET_RANGE from gs_sort,
    gs_sort_indexes and the void sortIndexes twin (output left untouched); the engine then sorts as a fresh one does."""
    import ctypes as C
    from gaussiansplats3d_b200 import _native as N
    n = 50_000
    idx = np.random.default_rng(31).permutation(n).astype(np.uint32)
    ok = _distances(n, -2**30 - 1, 2**30 - 2, 32)
    bad = ok.copy()
    bad[n // 2] = 2**30 - 1
    mvp = np.eye(4, dtype=np.float32).reshape(16)
    for R in (1 << 16, 1 << 20):
        want, buckets = oracle_mod.port_sort_indexes(*_sort_args(ok, R, idx), want_buckets=True)
        pos = np.argsort(idx)            # buckets are listed by input position
        # the extremes: rel 0 and rel 2^31 - 1, which f32 rounds to 2^31 = the f32 span, so exactly bucket R - 1
        assert buckets[pos[7]] == 0 and buckets[pos[n // 2]] == R - 1, (buckets[pos[7]], buckets[pos[n // 2]])
        got, mapped, _ = gs.sort_indexes(*_sort_args(ok, R, idx), want_scratch=True)
        assert np.array_equal(got, want) and np.array_equal(mapped, buckets)
        with pytest.raises(RuntimeError):
            oracle_mod.port_sort_indexes(*_sort_args(bad, R, idx))
        with pytest.raises(gs.GsError) as ei:
            gs.sort_indexes(*_sort_args(bad, R, idx))
        assert ei.value.code == N.GS_ERR_BUCKET_RANGE and BUCKET_MSG in str(ei.value)
        # the void twin: the same refusal, nothing written
        lib = gs._native.load()
        lib.sortIndexes.restype = None
        lib.sortIndexes.argtypes = [C.c_void_p] * 9 + [C.c_uint32] * 4 + [C.c_bool] * 3
        sentinel = np.full(n, 123456789, np.uint32)
        mapped, freq = np.zeros(n, np.int32), np.zeros(2 * R, np.uint32)
        p = lambda a: a.ctypes.data_as(C.c_void_p)   # noqa: E731
        lib.sortIndexes(p(idx), None, p(bad), p(mapped), p(freq), p(mvp), p(sentinel), None, None, R, n, n, n, True, True, False)
        assert (sentinel == 123456789).all()
        lib.sortIndexes(p(idx), None, p(ok), p(mapped), p(freq), p(mvp), p(sentinel), None, None, R, n, n, n, True, True, False)
        assert np.array_equal(sentinel, want)
        # the engine entry: error, then the good sort on the same engine equals a fresh engine's
        with gs.Engine(n, distance_map_range=R) as e:
            e.upload_centers(np.zeros((n, 4), np.int32))     # the sort counts clamp to the uploaded splats; distances are precomputed
            with pytest.raises(gs.GsError) as ei:
                e.sort(mvp, n, n, idx, precomputed=bad)
            assert ei.value.code == N.GS_ERR_BUCKET_RANGE and BUCKET_MSG in str(ei.value)
            out, _ = e.sort(mvp, n, n, idx, precomputed=ok)
        with gs.Engine(n, distance_map_range=R) as f:
            f.upload_centers(np.zeros((n, 4), np.int32))
            fresh, _ = f.sort(mvp, n, n, idx, precomputed=ok)
        assert np.array_equal(out, fresh) and np.array_equal(out, want)


def test_bucket_range_on_frame_paths(gs):
    """Finite integer centres whose distances span more than 2^31 (a scene too wide for the int32 range map): gs_frame and the
    pipelined gs_frame_begin / gs_frame_end report GS_ERR_BUCKET_RANGE; the same engine then renders a good frame bit-identical to
    a fresh engine's."""
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.scenes import pack_scene, synthetic_scene
    from test_raster_edges_gpu import _camera
    w, h = 320, 200
    raw = synthetic_scene(20_000, 41, "bonsai", 0)
    p = pack_scene(raw)
    n = raw.count
    u, _, mvp = _camera(w, h, (1.0, 2.0, -9.0), (0.0, 0.0, 0.0))
    row = _irow(mvp)
    k = int(np.argmax(np.abs(row)))
    wide = p.int_centers.copy()
    wide[[3, 4], :3] = 0
    wide[3, k] = int(0.6 * 2**31 / abs(row[k]))
    wide[4, k] = -wide[3, k]
    assert _span(wide, row) > 2**31 and _span(p.int_centers, row) < 2**31
    with gs.Engine(n, max_width=w, max_height=h) as f:
        f.upload_splat_data(p.centers_colors, p.covariances)
        f.upload_centers(p.int_centers)
        fresh = f.frame(mvp, u, w, h, n).copy()
    e = gs.Engine(n, max_width=w, max_height=h)
    e.upload_splat_data(p.centers_colors, p.covariances)
    buf = N.pinned_empty((h, w, 4), np.uint8)
    for path in ("frame", "frame_begin"):
        e.upload_centers(wide)
        with pytest.raises(gs.GsError) as ei:
            if path == "frame":
                e.frame(mvp, u, w, h, n)
            else:
                e.frame_begin(e.prepare_frame(mvp, u, w, h, n), buf)
                e.frame_end()
        assert ei.value.code == N.GS_ERR_BUCKET_RANGE and BUCKET_MSG in str(ei.value), (path, str(ei.value))
        e.upload_centers(p.int_centers)
        assert np.array_equal(e.frame(mvp, u, w, h, n), fresh), f"{path}: the frame after the error differs from a fresh engine's"
        e.frame_begin(e.prepare_frame(mvp, u, w, h, n), buf)
        e.frame_end()
        assert np.array_equal(buf, fresh), f"{path}: the pipelined frame after the error differs from a fresh engine's"
    e.close()

