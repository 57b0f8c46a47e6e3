"""CPU: the restatement SplatMesh.computeBoundingBox is checked against on the GPU (tests/test_bounding_box_gpu.py), the three.js math the
single-splat getters use (against oracle/ray_oracle.py's independent restatement), and the host-side refusals of the new SplatMesh methods."""
import numpy as np
import pytest

from oracle import ray_oracle as RO


def centers_f32(c64, transform16=None):
    """fillSplatCenterArray (SplatBuffer.js:307-347): the f64 centre, through Vector3.applyMatrix4 when a transform is given (sums left
    to right, the divide by w included; NumPy never fuses), stored into a Float32Array."""
    c = np.asarray(c64, np.float64).reshape(-1, 3)
    if transform16 is None:
        return c.astype(np.float32)
    e = np.asarray(transform16, np.float64).reshape(16)
    x, y, z = c[:, 0], c[:, 1], c[:, 2]
    with np.errstate(all="ignore"):
        w = 1.0 / (((e[3] * x + e[7] * y) + e[11] * z) + e[15])
        return np.stack([(((e[0] * x + e[4] * y) + e[8] * z) + e[12]) * w, (((e[1] * x + e[5] * y) + e[9] * z) + e[13]) * w,
                         (((e[2] * x + e[6] * y) + e[10] * z) + e[14]) * w], 1).astype(np.float32)


def js_box(c32):
    """computeBoundingBox's loop (SplatMesh.js:2080-2091): `if (i === 0 || x < min.x) min.x = x`, and > for max.  -> (min, max) f32."""
    c = np.asarray(c32, np.float32).reshape(-1, 3)
    lo, hi = np.zeros(3, np.float32), np.zeros(3, np.float32)
    if c.shape[0] == 0:
        return lo, hi
    for a in range(3):
        v = c[:, a]
        if np.isnan(v[0]):                       # the seed is never replaced: NaN < x and NaN > x are false
            lo[a] = hi[a] = v[0]
            continue
        ok = v[~np.isnan(v)]
        for out, best in ((lo, ok.min()), (hi, ok.max())):
            out[a] = v[np.flatnonzero(v == best)[0]]   # strict compares: the first of equal values (-0, +0) stays
    return lo, hi


def js_box_loop(c32):
    """The same loop literally, element by element (the reference for js_box on small inputs)."""
    c = np.asarray(c32, np.float32).reshape(-1, 3)
    lo, hi = [0.0] * 3, [0.0] * 3
    for i in range(c.shape[0]):
        for a in range(3):
            x = float(c[i, a])
            if i == 0 or x < lo[a]:
                lo[a] = x
            if i == 0 or x > hi[a]:
                hi[a] = x
    return np.array(lo, np.float32), np.array(hi, np.float32)


def bits_equal(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def test_js_box_matches_the_literal_loop():
    rng = np.random.default_rng(3)
    specials = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, 1.0, -1.0], np.float32)
    for trial in range(400):
        n = int(rng.integers(0, 9))
        c = rng.choice(specials, size=(n, 3)) if trial % 2 else rng.normal(size=(n, 3)).astype(np.float32)
        got, want = js_box(c), js_box_loop(c)
        assert bits_equal(got[0], want[0]) and bits_equal(got[1], want[1]), c


def test_js_box_edge_rules():
    lo, hi = js_box(np.array([[np.nan, 1, -0.0], [2, np.nan, 0.0], [-3, 5, 0.0]], np.float32))
    assert np.isnan(lo[0]) and np.isnan(hi[0])                       # a NaN seed stays
    assert lo[1] == 1 and hi[1] == 5                                 # a later NaN never counts
    assert np.signbit(lo[2]) and np.signbit(hi[2])                   # -0 first: kept against +0
    lo, hi = js_box(np.array([[0.0, -np.inf, 0], [-0.0, np.inf, 0]], np.float32))
    assert not np.signbit(lo[0]) and not np.signbit(hi[0]) and lo[1] == -np.inf and hi[1] == np.inf
    assert bits_equal(js_box(np.zeros((0, 3), np.float32))[0], np.zeros(3)) and bits_equal(js_box(np.zeros((0, 3)))[1], np.zeros(3))


def test_identity_transform_rounds_like_the_reference():
    """applyMatrix4 by the identity turns -0 into +0 and +-inf into NaN (0 * inf), as the reference's static mesh does."""
    c = centers_f32(np.array([[-0.0, 1.0, 2.0], [np.inf, 0.0, 0.0]]), np.eye(4).reshape(16))
    assert not np.signbit(c[0, 0]) and c[0, 1] == 1.0 and c[0, 2] == 2.0 and np.isnan(c[1]).all()


def test_three_math_decompose_matches_the_oracle():
    from gaussiansplats3d_b200 import three_math as TM
    rng = np.random.default_rng(7)
    for _ in range(300):
        q = rng.normal(size=4) * rng.choice([1e-3, 1.0, 10.0])
        s = rng.normal(size=3) * rng.choice([1e-4, 1.0, 100.0])
        T = RO.compose(list(rng.normal(size=3)), list(q / np.linalg.norm(q)), list(rng.normal(size=3)))
        M = RO.multiply(RO.multiply(RO.make_scale(*s), RO.make_rotation_from_quaternion(list(q))), T)
        mine = TM.multiply_elements(TM.multiply_elements(TM.make_scale(*s), TM.compose((0.0, 0.0, 0.0), q, (1.0, 1.0, 1.0))), T)
        assert np.array_equal(np.array(mine).view(np.uint64), np.array(M, np.float64).view(np.uint64))
        p1, q1, s1 = TM.decompose(mine)
        p2, q2, s2 = RO.decompose(M)
        assert np.array_equal(np.array(p1 + q1 + s1).view(np.uint64), np.array(p2 + q2 + s2, np.float64).view(np.uint64))
        v = list(rng.normal(size=3))
        assert np.array_equal(np.array(TM.apply_matrix4(v, T)).view(np.uint64), np.array(RO.apply_matrix4(v, T), np.float64).view(np.uint64))


def _mesh(**kw):
    from gaussiansplats3d_b200.scenes import PackedScene
    from gaussiansplats3d_b200.viewer import SplatMesh
    m = SplatMesh(**kw)
    m.packed = PackedScene(None, None, None, 0, None, 10)
    return m


def test_bounding_box_refuses_an_invalid_scene_index():
    m = _mesh()
    for s in (-1, 1, 5):
        with pytest.raises(ValueError, match="Invalid scene index"):
            m.computeBoundingBox(False, s)


@pytest.mark.parametrize("getter", ["getSplatCenter", "getSplatScaleAndRotation"])
def test_getters_without_ray_records_name_the_raycast_option(getter):
    m = _mesh()
    with pytest.raises(ValueError, match="raycast"):
        getattr(m, getter)(3)
    with pytest.raises(IndexError):
        getattr(m, getter)(10)


def test_scene_of_splat_skips_empty_scenes():
    m = _mesh()
    m.sceneInfos = [dict(splat_offset=0), dict(splat_offset=4), dict(splat_offset=4), dict(splat_offset=9)]
    assert [m._sceneOfSplat(i) for i in range(10)] == [0] * 4 + [2] * 5 + [3]
