"""The f64 vertex-stage restatement with per-splat error bounds (tests/projection_f64.py), checked on the CPU:

  * the bounds admit legitimate f32 evaluations: oracle/raster_oracle.c unfused (-ffp-contract=off), and compiled a second time with
    FMA contraction, agree with the helper's `valid` on every unambiguous splat and lie inside every bound, on every case of the GPU
    matrix (tests/projection_cases.py);
  * the bounds are not vacuous: ceilings on each field's median bound and on the ambiguous fraction, measured on these cases;
  * two option branches pinned against oracle/raster_independent.py's formulation (finite-difference Jacobian, mass preservation);
  * the Viewer's option semantics against Viewer.js:119-154 and its uniforms against Viewer.updateSplatMesh / SplatMesh.updateUniforms.
Each case prints its worst |oracle - f64| / bound per field (pytest -s)."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import projection_cases as PC
import projection_f64 as P

ROOT = Path(__file__).resolve().parent.parent
CASES = PC.all_cases()
IDS = [c.name for c in CASES]

# Median bounds on the unambiguous valid splats of every case, measured on these cases (worst case in brackets) and set about 2x
# above: centres ~1e-4 px [3.2e-4], ndc z [1.7e-6], SH-free colour at f32 rounding of byte / 255 [6.2e-8], colour with SH [2.1e-6],
# alpha [8.0e-6, antialiased with kernel 0.05], Q relative to its trace [7.5e-5, antialiased with kernel 1.5].
CEIL = dict(cx=6e-4, cy=6e-4, ndc_z=4e-6, rgb_plain=1.2e-7, rgb_sh=5e-6, a=2e-5, q_rel=1.5e-4)
# ambiguous fraction: none in the scene cases; the cull-edge case places 10 % of its edge splats within a few ulp of the guard band;
# the axis-aligned case is built so that the eigenvector direction is undetermined for about 28 % of its splats
AMBIG_CEIL = {"cull-edges": 0.06, "axis-aligned": 0.35}
AMBIG_DEFAULT = 1e-3


def _oracle_project(lib, c):
    from oracle import pyoracle
    from gaussiansplats3d_b200 import _native as N
    d, keep = pyoracle._splat_data(c.cc, c.cov, c.sh, c.sh_degree, c.scene_indexes)
    u = c.u.to_c()
    out = np.empty(d.count, N.PROJECTED_DTYPE)
    lib.gso_project.restype = None
    lib.gso_project.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.gso_project(C.byref(u), C.byref(d), out.ctypes.data)
    del keep
    return out


@pytest.fixture(scope="module")
def helper_results():
    return {c.name: P.project(c.u, c.cc, c.cov, c.sh, c.sh_degree, c.scene_indexes) for c in CASES}


@pytest.fixture(scope="module")
def fma_lib(tmp_path_factory):
    """raster_oracle.c compiled with FMA contraction: another legitimate f32 evaluation order."""
    flags = Path("/proc/cpuinfo").read_text() if Path("/proc/cpuinfo").exists() else ""
    if " fma" not in flags:
        pytest.skip("this CPU has no FMA")
    out = tmp_path_factory.mktemp("fma") / "libgs_oracle_fma.so"
    cmd = ["/usr/bin/gcc", "-std=c11", "-O2", "-fwrapv", "-ffp-contract=fast", "-mfma", "-fPIC", "-shared",
           str(ROOT / "oracle" / "raster_oracle.c"), "-o", str(out), "-lm"]
    try:
        subprocess.run(cmd, check=True, capture_output=True)
    except (OSError, subprocess.CalledProcessError) as e:
        pytest.skip(f"cannot compile the contracted oracle: {e}")
    return C.CDLL(str(out))


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_unfused_oracle_within_bounds(oracle_mod, helper_results, case):
    h = helper_results[case.name]
    rep = P.compare(_oracle_project(oracle_mod.port_lib(), case), h)
    print("\n" + P.format_report(case.name + " unfused", rep))
    P.assert_within(case.name, rep, min_compared=1000)
    case.ran(case, h)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_contracted_oracle_within_bounds(fma_lib, helper_results, case):
    h = helper_results[case.name]
    rep = P.compare(_oracle_project(fma_lib, case), h)
    print("\n" + P.format_report(case.name + " fma", rep))
    P.assert_within(case.name, rep, min_compared=1000)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_bounds_are_not_vacuous(helper_results, case):
    h = helper_results[case.name]
    m = h["valid"] & ~h["ambiguous"]
    med = {k: float(np.median(h[k + "_bound"][m])) for k in P.FIELDS}
    trace = np.abs(h["qxx"][m]) + np.abs(h["qyy"][m])
    q_rel = float(np.median(np.maximum.reduce([h[k + "_bound"][m] for k in ("qxx", "qxy", "qyy")]) / trace))
    sh_used = case.sh is not None and case.u.sh_degree >= 1
    print(f"\n[{case.name}] median bounds " + " ".join(f"{k} {v:.2e}" for k, v in med.items()) + f", Q relative {q_rel:.2e}, ambiguous "
          f"{h['ambiguous'].mean():.4f}")
    assert med["cx"] <= CEIL["cx"] and med["cy"] <= CEIL["cy"], med
    assert med["ndc_z"] <= CEIL["ndc_z"], med
    for k in ("r", "g", "b"):
        assert med[k] <= CEIL["rgb_sh" if sh_used else "rgb_plain"], (k, med[k])
    assert med["a"] <= CEIL["a"], med
    assert q_rel <= CEIL["q_rel"], q_rel
    assert h["ambiguous"].mean() <= AMBIG_CEIL.get(case.name, AMBIG_DEFAULT)


def test_axis_aligned_splats_are_ambiguous_and_the_oracle_drops_degenerate_directions(oracle_mod, helper_results):
    """b = 0 exactly and l1 - a rounded: the helper flags the direction, and where both components round to 0 (normalize(vec2(0)) = NaN,
    no quad in WebGL) the oracle gives an invalid record, never a valid NaN."""
    case = next(c for c in CASES if c.name == "axis-aligned")
    h = helper_results[case.name]
    o = _oracle_project(oracle_mod.port_lib(), case)
    v = o["valid"] == 1
    fields = np.stack([o[k] for k in ("cx", "cy", "b1x", "b1y", "b2x", "b2y", "r", "g", "b", "a", "ndc_z")], 1)
    assert np.isfinite(fields[v]).all()
    undetermined = h["stats"]["direction_undetermined"]
    assert undetermined.sum() > 1000 and (h["ambiguous"] >= undetermined).all()
    assert (~v & h["valid"]).sum() > 0        # the dropped degenerate ones


# ---- two branches pinned by the independent formulation -----------------------------------------------------------------------------
def test_antialias_factor_is_mass_preservation():
    """SplatMaterial3D.js:137-145 multiplies alpha by sqrt(det(S) / det(S + kI)): the factor that keeps the Gaussian's integral when the
    kernel widens it.  S here is the independent formulation's covariance (finite-difference Jacobian), not the shader's det expressions."""
    from oracle import raster_independent as RI
    for k2 in (0.3, 0.05, 1.5):
        case = next(c for c in CASES if c.name == f"antialiased-k{k2:g}")
        u = case.u
        centers = case.cc[:, 1:].copy().view(np.float32)
        rgba = np.stack([(case.cc[:, 0] >> (8 * k)) & 255 for k in range(4)], 1)
        ind = RI.project(u.model_view, u.projection, u.camera_position, u.viewport, centers, rgba, case.cov, kernel2d=0.0)
        S = ind["sigma2"]
        det0 = S[:, 0, 0] * S[:, 1, 1] - S[:, 0, 1] ** 2
        det1 = (S[:, 0, 0] + k2) * (S[:, 1, 1] + k2) - S[:, 0, 1] ** 2
        mass = ind["opacity"] * np.sqrt(np.maximum(det0 / det1, 0.0))
        h = P.project(u, case.cc, case.cov)
        m = h["valid"] & ~h["ambiguous"] & ind["valid"]
        # the finite-difference Jacobian carries ~1e-6 relative error into S; far from the clamp, the factor is well-conditioned
        good = m & (det0 > 1e-3 * det1)
        assert good.sum() > 1000
        err = np.abs(h["a"][good] - mass[good]) / np.maximum(mass[good], 1e-12)
        assert err.max() < 1e-4, (k2, err.max())
        # the minAlpha cut is the mass-preserved alpha against 1/255
        assert not h["valid"][m & (mass < 1.0 / 255 * (1 - 1e-4))].any()


@pytest.mark.parametrize("zoom", [1.0, 2.5])
def test_orthographic_jacobian_is_ortho_zoom(zoom):
    """With a pixel-sized orthographic frustum the projective map is linear and its finite-difference Jacobian is orthoZoom * I (x, y
    rows; the z column is zero): the shader's constant J (SplatMaterial3D.js:117-122) is the exact Jacobian."""
    from oracle import raster_independent as RI
    w, h = 400, 300
    u = PC.orthographic_uniforms(w, h, zoom, dpr=1)
    rng = np.random.default_rng(71)
    v = np.stack([rng.normal(0, 100, 500), rng.normal(0, 80, 500), -rng.uniform(10, 800, 500)], 1)
    J = RI.numeric_jacobian(RI._mat(u.projection), v, u.viewport)
    want = np.zeros((2, 3))
    want[0, 0] = want[1, 1] = zoom
    assert np.abs(J - want[None]).max() < 1e-6 * zoom


# ---- Viewer option semantics (Viewer.js:119-154) and uniforms (Viewer.js:651-677, SplatMesh.js:1253-1264) -----------------------------
def _viewer_without_engine(**opts):
    from gaussiansplats3d_b200.scenes import synthetic_scene
    from gaussiansplats3d_b200.viewer import SplatMesh, Viewer
    v = Viewer(dict(width=320, height=200, **opts))
    sm = SplatMesh(devicePixelRatio=v.devicePixelRatio, maxScreenSpaceSplatSize=v.maxScreenSpaceSplatSize, kernel2DSize=v.kernel2DSize)
    sm.build(synthetic_scene(10, seed=1))
    v.splatMesh = sm
    v.camera.update()
    v.updateSplatMesh()
    return v


@pytest.mark.parametrize("given,want", [(None, 1024.0), (0, 1024.0), (37.9, 37.0), (48, 48.0), (2048.5, 2048.0)])
def test_max_screen_space_splat_size_option(given, want):
    """`options.maxScreenSpaceSplatSize || 1024`, then the material bakes `${parseInt(size)}.0`: the kernel's clamp."""
    v = _viewer_without_engine(**({} if given is None else dict(maxScreenSpaceSplatSize=given)))
    assert v.uniforms().max_screen_space_splat_size == want


@pytest.mark.parametrize("given,want", [(None, 1.0), (0, 1.0), (1.7, 1.7)])
def test_focal_adjustment_option(given, want):
    v = _viewer_without_engine(**({} if given is None else dict(focalAdjustment=given)))
    assert v.focalAdjustment == want
    assert v.uniforms().inverse_focal_adjustment == pytest.approx(1.0 / want)


@pytest.mark.parametrize("given,want", [(None, 0.3), (0, 0.0), (0.1, 0.1)])
def test_kernel2d_size_option(given, want):
    """`(options.kernel2DSize === undefined) ? 0.3 : options.kernel2DSize`: 0 stays 0."""
    v = _viewer_without_engine(**({} if given is None else dict(kernel2DSize=given)))
    assert v.uniforms().kernel_2d_size == want


def test_viewer_uniforms_with_focal_adjustment_and_device_pixel_ratio():
    """Perspective camera, focalAdjustment 1.7, devicePixelRatio 2: focal = projectionMatrix[0|5] * 0.5 * dpr * renderDimensions * 1.7,
    inverseFocalAdjustment = 1 / 1.7, viewport = renderDimensions * dpr."""
    v = _viewer_without_engine(focalAdjustment=1.7, devicePixelRatio=2.0)
    u = v.uniforms()
    Pm = v.camera.projectionMatrix
    assert u.focal[0] == pytest.approx(Pm[0] * 0.5 * 2.0 * 320 * 1.7, rel=1e-12)
    assert u.focal[1] == pytest.approx(Pm[5] * 0.5 * 2.0 * 200 * 1.7, rel=1e-12)
    assert u.inverse_focal_adjustment == pytest.approx(1.0 / 1.7, rel=1e-12)
    assert tuple(u.viewport) == (640.0, 400.0)
    assert u.orthographic_mode == 0 and not v.camera.isOrthographicCamera


def test_orthographic_uniforms_follow_the_reference_definitions():
    """The Python Viewer has no orthographic camera; the GPU cases build its uniforms by hand.  Viewer.js:660-673 for an orthographic
    camera: focal multiplier 1 / devicePixelRatio, so inverseFocalAdjustment = devicePixelRatio; SplatMesh.js:1253-1256: viewport =
    renderDimensions * devicePixelRatio; orthoZoom = camera.zoom."""
    u = PC.orthographic_uniforms(400, 300, 2.5, dpr=2)
    assert u.inverse_focal_adjustment == 2.0 and tuple(u.viewport) == (800, 600) and u.ortho_zoom == 2.5 and u.orthographic_mode == 1
    Pm = np.asarray(u.projection, np.float64)
    assert u.focal[0] == pytest.approx(Pm[0] * 0.5 * 2 * 400 / 2, rel=1e-6)
