"""The case matrix of the per-splat vertex-stage checks (tests/test_projection_f64.py on the CPU oracles, tests/test_projection_gpu.py on
k_project): one scene and one set of uniforms per case, each aimed at a branch of SplatMaterial.js / SplatMaterial3D.js, and a check that
the branch really ran (evaluated on projection_f64's result)."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

N_SPLATS = 24_000
W, H = 480, 320
MIN_ALPHA = np.float32(1.0 / 255.0)


@dataclass
class Case:
    name: str
    u: object                       # engine.Uniforms
    cc: np.ndarray
    cov: np.ndarray
    sh: np.ndarray | None = None
    sh_degree: int = 0
    scene_indexes: np.ndarray | None = None
    width: int = W
    height: int = H
    dynamic: bool = False
    ran: object = None              # ran(case, helper_result) -> None: asserts the branch was exercised
    extra: dict = field(default_factory=dict)


def camera_uniforms(w, h, pos, look, up=(0.0, 1.0, 0.0), fov=50.0, focal_adjustment=1.0, **kw):
    """Uniforms of a three.js PerspectiveCamera as Viewer.updateSplatMesh / SplatMesh.updateUniforms define them (Viewer.js:651-677)."""
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.engine import Uniforms
    cam = TM.PerspectiveCamera(fov, w / h, 0.1, 1000.0)
    cam.position = np.asarray(pos, np.float64)
    cam.up = np.asarray(up, np.float64) / np.linalg.norm(up)
    cam.look_at(look)
    P = cam.projectionMatrix
    u = Uniforms(model_view=cam.matrixWorldInverse.astype(np.float32), projection=P.astype(np.float32),
                 camera_position=cam.position.astype(np.float32), focal=(P[0] * 0.5 * w * focal_adjustment, P[5] * 0.5 * h * focal_adjustment),
                 viewport=(w, h), inverse_focal_adjustment=1.0 / focal_adjustment, **kw)
    return u, cam


def bonsai_uniforms(w=W, h=H, **kw):
    from gaussiansplats3d_b200.scenes import CAMERAS
    c = CAMERAS["bonsai"]
    return camera_uniforms(w, h, c["position"], c["look_at"], c["up"], **kw)[0]


def _scene(kind, seed, sh_degree=0, n=N_SPLATS, half=False, sh_format="f16", sh8_range=(-1.5, 1.5)):
    from gaussiansplats3d_b200.scenes import pack_scene, synthetic_scene
    raw = synthetic_scene(n, seed=seed, kind=kind, sh_degree=sh_degree)
    p = pack_scene(raw, half_covariances=half, sh_format=sh_format, sh8_range=sh8_range)
    return raw, p


def _count(label, mask, least=50):
    k = int(np.count_nonzero(mask))
    assert k >= least, f"{label}: {k} splats (want >= {least})"
    return k


# ---- branch checks --------------------------------------------------------------------------------------------------------------------
def _ran_sh(case, h):
    ok = h["valid"]
    base = np.stack([(case.cc[:, 0] >> (8 * k)) & 255 for k in range(3)], 1) / 255.0
    moved = np.abs(np.stack([h["r"], h["g"], h["b"]], 1) - base).max(1) > 1e-3
    if case.u.sh_degree >= 1 and case.sh is not None:
        _count("colour moved by SH", ok & moved, 1000)
    else:
        assert not (ok & moved).any(), "colour moved without SH"


def _ran_min_alpha(case, h):
    _count("cut by minAlpha", h["stats"]["min_alpha_cut"])
    _count("kept by minAlpha", h["valid"] & (h["stats"]["aa_factor"] < 0.9))


def _ran_clamp(case, h):
    _count("clamped by the max size", h["valid"] & h["stats"]["clamped"])
    _count("unclamped", h["valid"] & ~h["stats"]["clamped"])


def _ran_faded(case, h):
    _count("faded", h["valid"] & (h["stats"]["fade"] < 0.99))
    _count("not faded", h["valid"] & (h["stats"]["fade"] == 1.0))


def _ran_point_cloud(case, h):
    q = h["qxx"] + h["qyy"]
    want = 2.0 * 8.0 * np.float32(0.2)
    assert np.allclose(q[h["valid"]], want * case.u.splat_scale ** 2, rtol=1e-5)


def _ran_any(case, h):
    _count("valid", h["valid"], 1000)


# ---- the matrix -----------------------------------------------------------------------------------------------------------------------
def sh_cases():
    """Covariances f32 and f16 x SH: none, f16 degree 1 and 2, u8 degree 2 over (-0.7, 2.3), f32 degree 2, and degree-2 data under
    uniform degree 1 and 0 in each SH format."""
    out = []
    for half in (False, True):
        cv = "cov16" if half else "cov32"
        for fmt, deg, udeg in (("none", 0, 0), ("f16", 1, 1), ("f16", 2, 2), ("u8", 2, 2), ("f32", 2, 2),
                               ("f16", 2, 1), ("f16", 2, 0), ("u8", 2, 1), ("u8", 2, 0), ("f32", 2, 1), ("f32", 2, 0)):
            rng8 = (-0.7, 2.3)
            raw, p = _scene("bonsai", 31, deg, half=half, sh_format="f16" if fmt == "none" else fmt, sh8_range=rng8)
            kw = {}
            if fmt == "u8":
                kw = dict(sh8_min=np.full(32, rng8[0], np.float32), sh8_max=np.full(32, rng8[1], np.float32))
            u = bonsai_uniforms(sh_degree=udeg, **kw)
            out.append(Case(f"{cv}-sh{fmt}{deg}-u{udeg}", u, p.centers_colors, p.covariances, p.sh, p.sh_degree, ran=_ran_sh))
    return out


def option_cases():
    out = []
    raw, p = _scene("bonsai", 32)
    for k2 in (0.3, 0.05, 1.5):
        out.append(Case(f"antialiased-k{k2:g}", bonsai_uniforms(antialiased=1, kernel_2d_size=k2), p.centers_colors, p.covariances, ran=_ran_min_alpha))
    out.append(Case("kernel0.1", bonsai_uniforms(kernel_2d_size=0.1), p.centers_colors, p.covariances, ran=_ran_any))
    out.append(Case("point-cloud", bonsai_uniforms(point_cloud_mode=1), p.centers_colors, p.covariances, ran=_ran_point_cloud))
    for sc in (0.6, 1.7):
        out.append(Case(f"splat-scale{sc:g}-max48", bonsai_uniforms(splat_scale=sc, max_screen_space_splat_size=48.0), p.centers_colors,
                        p.covariances, ran=_ran_clamp))
    out.append(Case("focal-adjustment1.7", bonsai_uniforms(focal_adjustment=1.7), p.centers_colors, p.covariances, ran=_ran_any))
    centre = raw.centers.astype(np.float64).mean(0)
    radius = float(np.median(np.linalg.norm(raw.centers - centre, axis=1)))
    out.append(Case("fade-in", bonsai_uniforms(fade_in_complete=0, scene_center=tuple(centre), visible_region_fade_start_radius=radius),
                    p.centers_colors, p.covariances, ran=_ran_faded))
    return out


def orthographic_uniforms(w, h, zoom, dpr, pos=(30.0, -20.0, 400.0), look=(0.0, 0.0, 0.0), up=(0.0, 1.0, 0.0)):
    """An OrthographicCamera with a pixel-sized frustum, the uniforms as Viewer.updateSplatMesh builds them (Viewer.js:660-673): focal
    multiplier 1 / devicePixelRatio, so inverseFocalAdjustment = devicePixelRatio; viewport = render size x devicePixelRatio
    (SplatMesh.js:1253-1256)."""
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.engine import Uniforms
    _, cam = camera_uniforms(w, h, pos, look, up)
    P = TM.make_orthographic(-w / 2, w / 2, h / 2, -h / 2, 0.1, 1000.0, zoom)
    fa = 1.0 / dpr
    fx, fy = P[0] * 0.5 * dpr * w * fa, P[5] * 0.5 * dpr * h * fa
    return Uniforms(model_view=cam.matrixWorldInverse.astype(np.float32), projection=P.astype(np.float32),
                    camera_position=cam.position.astype(np.float32), focal=(fx, fy), viewport=(w * dpr, h * dpr),
                    inverse_focal_adjustment=1.0 / fa, ortho_zoom=zoom, orthographic_mode=1)


def _pixel_splats(rng, m, spread=(150.0, 110.0, 80.0), rot=True, scales=(0.4, 6.0)):
    from gaussiansplats3d_b200.scenes import compute_covariances, pack_centers_colors
    centers = np.stack([rng.normal(0, spread[0], m), rng.normal(0, spread[1], m), rng.normal(0, spread[2], m)], 1).astype(np.float32)
    s = (np.exp(rng.uniform(np.log(scales[0]), np.log(scales[1]), (m, 1))) * np.exp(rng.uniform(-0.7, 0.7, (m, 3)))).astype(np.float32)
    if rot:
        q = rng.normal(0, 1, (m, 4))
        q /= np.linalg.norm(q, axis=1, keepdims=True)
    else:
        q = np.tile([0.0, 0.0, 0.0, 1.0], (m, 1))
    colors = rng.integers(0, 256, (m, 4)).astype(np.uint8)
    colors[:, 3] = rng.integers(10, 256, m)
    return pack_centers_colors(centers, colors), compute_covariances(s, q.astype(np.float32)), centers


def orthographic_cases():
    out = []
    w, h, dpr = 400, 300, 2
    rng = np.random.default_rng(601)
    cc, cov, _ = _pixel_splats(rng, N_SPLATS)
    for zoom in (1.0, 2.5):
        out.append(Case(f"orthographic-zoom{zoom:g}-dpr2", orthographic_uniforms(w, h, zoom, dpr), cc, cov, width=w * dpr, height=h * dpr,
                        ran=_ran_any))
    return out


def effects_case():
    """Four scenes: opacity 0.6, exactly 0.01f (culled: <= 0.01), 0.0101f, and one with visibility 0."""
    raw, p = _scene("uniform", 33)
    rng = np.random.default_rng(34)
    idx = rng.integers(0, 4, raw.count).astype(np.uint32)
    op = np.ones(32, np.float32)
    op[0], op[1], op[2] = 0.6, np.float32(0.01), np.float32(0.0101)
    vis = np.ones(32, np.int32)
    vis[3] = 0
    u = camera_uniforms(W, H, (0.0, 4.0, 12.0), (0.0, 0.0, 0.0))[0]
    u.scene_count, u.enable_optional_effects, u.scene_opacity, u.scene_visibility = 4, 1, op, vis

    def ran(case, h):
        assert not h["valid"][(idx == 1) | (idx == 3)].any()
        _count("scene 0.6 drawn", h["valid"] & (idx == 0), 1000)
        _count("scene 0.0101 drawn", h["valid"] & (idx == 2), 1000)
    return Case("optional-effects", u, p.centers_colors, p.covariances, scene_indexes=idx, ran=ran)


def dynamic_cases():
    """Three scenes with their own transform (rotation, non-unit scale, translation), SH2 in f16 and u8 with a u8 range per scene."""
    from gaussiansplats3d_b200 import three_math as TM
    out = []
    ranges = [(-1.5, 1.5), (-0.7, 2.3), (-0.4, 0.45)]
    for fmt in ("f16", "u8"):
        raw, _ = _scene("uniform", 35, 2)
        rng = np.random.default_rng(36)
        idx = rng.integers(0, 3, raw.count).astype(np.uint32)
        from gaussiansplats3d_b200.scenes import pack_scene
        p = pack_scene(raw, sh_format="f16")
        sh = p.sh
        if fmt == "u8":     # each scene's coefficients quantised over its own range
            flat = raw.sh.reshape(raw.count, -1).astype(np.float64)
            lo = np.array([r[0] for r in ranges])[idx][:, None]
            hi = np.array([r[1] for r in ranges])[idx][:, None]
            sh = np.floor((np.clip(flat, lo, hi) - lo) / (hi - lo) * 255.0).astype(np.uint8)
        tr = np.tile(np.eye(4, dtype=np.float64).T.reshape(16), (32, 1))
        tr[1] = TM.compose((1.5, 0.0, -1.0), (0.0, np.sin(0.3), 0.0, np.cos(0.3)), (1.3, 0.8, 1.1))
        tr[2] = TM.compose((-2.0, 0.5, 0.5), (np.sin(0.2), 0.1, 0.0, np.cos(0.2)) / np.linalg.norm((np.sin(0.2), 0.1, 0.0, np.cos(0.2))), (0.7, 0.7, 0.7))
        u, cam = camera_uniforms(W, H, (0.0, 4.0, 12.0), (0.0, 0.0, 0.0))
        u.scene_count, u.dynamic_mode, u.sh_degree = 3, 1, 2
        u.scene_transforms = tr.astype(np.float32)
        u.view_matrix = cam.matrixWorldInverse.astype(np.float32)
        u.sh8_min = np.array([r[0] for r in ranges] + [-1.5] * 29, np.float32)
        u.sh8_max = np.array([r[1] for r in ranges] + [1.5] * 29, np.float32)

        def ran(case, h, idx=idx):
            for s in range(3):
                _count(f"scene {s} drawn", h["valid"] & (idx == s), 1000)
        out.append(Case(f"dynamic-sh2-{fmt}", u, p.centers_colors, p.covariances, sh, 2, scene_indexes=idx, dynamic=True, ran=ran))
    return out


def cull_case():
    """Splats behind the camera, between it and the near plane, and on both sides of the 1.2 w guard band, by a relative 1e-3 and by a
    few ulp (the latter ambiguous)."""
    from gaussiansplats3d_b200.scenes import compute_covariances, pack_centers_colors
    rng = np.random.default_rng(37)
    u, cam = camera_uniforms(W, H, (0.0, 0.0, 0.0), (0.0, 0.0, -1.0))
    P = np.asarray(cam.projectionMatrix, np.float64)
    m = 6000
    z = -rng.uniform(0.5, 50.0, m)
    edge_x = 1.2 * (-z) / P[0]
    edge_y = 1.2 * (-z) / P[5]
    k = rng.integers(0, 6, m)
    f = np.where(rng.uniform(0, 1, m) < 0.5, 1.0 - 1e-3, 1.0 + 1e-3)
    f = np.where(rng.uniform(0, 1, m) < 0.1, 1.0 + rng.integers(-3, 4, m) * 1e-7, f)
    sgn = np.where(rng.uniform(0, 1, m) < 0.5, -1.0, 1.0)
    x = np.where(k == 0, sgn * edge_x * f, rng.uniform(-0.5, 0.5, m) * edge_x)
    y = np.where(k == 1, sgn * edge_y * f, rng.uniform(-0.5, 0.5, m) * edge_y)
    z = np.where(k == 2, rng.uniform(0.01, 5.0, m), z)                  # behind the camera
    z = np.where(k == 3, -rng.uniform(0.0, 0.1, m), z)                  # between the camera and the near plane
    centers = np.stack([x, y, z], 1).astype(np.float32)
    s = np.exp(rng.uniform(np.log(0.002), np.log(0.05), (m, 3))).astype(np.float32)
    q = rng.normal(0, 1, (m, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    colors = rng.integers(0, 256, (m, 4)).astype(np.uint8)
    cc, cov = pack_centers_colors(centers, colors), compute_covariances(s, q.astype(np.float32))

    def ran(case, h):
        _count("inside the guard band", h["valid"] & (k <= 1) & (f < 1.0), 100)
        assert not (h["valid"] & (k <= 1) & (f > 1.0 + 1e-4)).any()
        assert not (h["valid"] & ((k == 2) | (k == 3))).any()
        _count("ambiguous at the guard band", h["ambiguous"] & (k <= 1), 1)
    return Case("cull-edges", u, cc, cov, ran=ran, width=W, height=H)


def axis_aligned_case():
    """Unrotated splats under an unrotated orthographic camera: b = 0 exactly, and where a > d + 0.63 px^2 the first eigenvector comes
    from l1 - a, which is pure rounding (often exactly 0)."""
    rng = np.random.default_rng(38)
    w, h = 640, 480
    cc, cov, _ = _pixel_splats(rng, 20_000, spread=(200.0, 150.0, 50.0), rot=False, scales=(0.3, 8.0))
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.engine import Uniforms
    mv = TM.identity().copy()
    mv[14] = -400.0
    P = TM.make_orthographic(-w / 2, w / 2, h / 2, -h / 2, 0.1, 1000.0, 1.0)
    u = Uniforms(model_view=mv.astype(np.float32), projection=P.astype(np.float32), camera_position=np.array([0.0, 0.0, 400.0], np.float32),
                 focal=(1.0, 1.0), viewport=(w, h), orthographic_mode=1)

    def ran(case, hres):
        _count("direction undetermined", hres["stats"]["direction_undetermined"], 1000)
    return Case("axis-aligned", u, cc, cov, width=w, height=h, ran=ran)


def all_cases():
    return sh_cases() + option_cases() + orthographic_cases() + [effects_case()] + dynamic_cases() + [cull_case(), axis_aligned_case()]
