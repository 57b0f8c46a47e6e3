"""k_project splat by splat against the f64 restatement with per-splat error bounds (tests/projection_f64.py), for every shader option of
the case matrix (tests/projection_cases.py): one engine per case, one render, the records read back (Engine.read_projected).  Asserted:
  * `valid` equal on every splat the helper does not flag as ambiguous;
  * every field (centre, ndc z, colour, alpha, the quad's quadratic form B1 B1^T + B2 B2^T) within its bound on every splat valid on
    both sides and unambiguous: no quantile exemption;
  * the case's branch really ran (splats cut by minAlpha, clamped by the max size, faded, culled per scene ...);
  * no valid record with a non-finite field, ambiguous splats included.
Each case prints its worst |GPU - f64| / bound per field and its ambiguous count (pytest -s)."""
import dataclasses

import numpy as np
import pytest

import projection_cases as PC
import projection_f64 as P

pytestmark = pytest.mark.gpu

CASES = PC.all_cases()
FIELDS = ("cx", "cy", "b1x", "b1y", "b2x", "b2y", "r", "g", "b", "a", "ndc_z")


def _records(case):
    from gaussiansplats3d_b200.engine import Engine
    n = case.cc.shape[0]
    with Engine(n, max_width=case.width, max_height=case.height, dynamic_mode=case.dynamic or case.scene_indexes is not None) as e:
        e.upload_splat_data(case.cc, case.cov, case.sh, case.sh_degree, scene_indexes=case.scene_indexes)
        e.render(case.u, case.width, case.height, n, np.arange(n, dtype=np.uint32), flip_y=False)
        return e.read_projected(n)


def _finite_when_valid(ps):
    v = ps["valid"] == 1
    return bool(np.isfinite(np.stack([ps[k] for k in FIELDS], 1)[v]).all())


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_k_project_within_per_splat_bounds(gs, case):
    ps = _records(case)
    h = P.project(case.u, case.cc, case.cov, case.sh, case.sh_degree, case.scene_indexes)
    rep = P.compare(ps, h)
    print("\n" + P.format_report(case.name, rep))
    P.assert_within(case.name, rep, min_compared=1000)
    case.ran(case, h)
    assert _finite_when_valid(ps), f"{case.name}: a valid record with a non-finite field"


def test_axis_aligned_degenerate_direction_gives_no_valid_nan(gs):
    """b = 0 exactly: where l1 - a rounds to 0 as well the direction is normalize(vec2(0)) = NaN, which WebGL does not draw.  The GPU gives
    an invalid record there, or a valid one with finite fields; never a valid NaN."""
    case = PC.axis_aligned_case()
    ps = _records(case)
    h = P.project(case.u, case.cc, case.cov)
    amb = h["stats"]["direction_undetermined"]
    assert amb.sum() > 1000
    assert _finite_when_valid(ps)
    dropped = amb & (ps["valid"] == 0)
    print(f"\n[axis-aligned] undetermined direction {int(amb.sum())}, of which dropped as degenerate {int(dropped.sum())}")


def test_viewer_max_screen_space_splat_size_reaches_the_kernel_truncated(gs):
    """Viewer(maxScreenSpaceSplatSize=37.9): the material bakes parseInt -> 37.0; the records are within bounds for 37 and, for the
    clamped splats, outside them for 37.9."""
    from gaussiansplats3d_b200.scenes import CAMERAS, synthetic_scene
    from gaussiansplats3d_b200.viewer import Viewer
    c = CAMERAS["bonsai"]
    raw = synthetic_scene(PC.N_SPLATS, seed=32, kind="bonsai")
    v = Viewer(dict(cameraUp=c["up"], initialCameraPosition=c["position"], initialCameraLookAt=c["look_at"], width=PC.W, height=PC.H,
                    maxScreenSpaceSplatSize=37.9, focalAdjustment=1.7))
    v.addSplatScene(raw)
    v.update()
    v.render(download=False)
    ps = v.engine.read_projected(raw.count)
    u = v.uniforms()
    assert u.max_screen_space_splat_size == 37.0
    p = v.splatMesh.packed
    h = P.project(u, p.centers_colors, p.covariances)
    rep = P.compare(ps, h)
    print("\n" + P.format_report("viewer max size 37.9 -> 37, focalAdjustment 1.7", rep))
    P.assert_within("viewer max size", rep, min_compared=1000)
    assert (h["valid"] & h["stats"]["clamped"]).sum() >= 50
    wrong = P.compare(ps, P.project(dataclasses.replace(u, max_screen_space_splat_size=37.9), p.centers_colors, p.covariances))
    assert wrong["outside"]["qxx"] + wrong["outside"]["qyy"] > 0
    v.dispose()
