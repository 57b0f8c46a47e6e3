"""CPU: the raycast oracle (oracle/ray_oracle.py) against hand-derived cases and independent formulas, the host ray set-up, the log10 table
the kernel embeds, and the C ABI / addon plumbing of gs_raycast."""
import ctypes as C
import math
import re
import subprocess
import tempfile
from decimal import Decimal, getcontext
from pathlib import Path

import numpy as np
import pytest

from oracle import ray_oracle as RO
from oracle import tree_oracle

ROOT = Path(__file__).resolve().parent.parent
I16 = RO.IDENTITY


def test_log10_table_is_correctly_rounded_and_matches_the_kernel():
    getcontext().prec = 80
    src = (ROOT / "gaussiansplats3d_b200" / "csrc" / "ray_kernels.cuh").read_text()
    body = src[src.index("kLog10Byte[256] = {") + 19:]
    body = body[:body.index("};")]
    entries = [e.strip() for e in body.replace("\n", " ").split(",") if e.strip()]
    assert len(entries) == 256 and entries[0] == "-HUGE_VAL"
    for b in range(1, 256):
        v = float.fromhex(entries[b])
        assert v == RO.LOG10_BYTE[b]
        exact = Decimal(b).log10()
        ulp = Decimal(math.ulp(v)) if v != 0 else Decimal(0)
        assert abs(Decimal(v) - exact) <= ulp / 2, b          # within half an ulp: correctly rounded
    assert RO.LOG10_BYTE[0] == -math.inf


def test_three_math_by_property():
    rng = np.random.default_rng(1)
    for _ in range(200):
        p = list(rng.normal(0, 5, 3))
        q = rng.normal(0, 1, 4)
        q = list(q / np.linalg.norm(q))
        if q[3] < 0:
            q = [-v for v in q]
        s = list(rng.uniform(0.1, 4, 3))
        p2, q2, s2 = RO.decompose(RO.compose(p, q, s))
        assert np.allclose(p2, p, rtol=0, atol=1e-12) and np.allclose(s2, s, rtol=0, atol=1e-12)
        assert np.allclose(q2, q, rtol=0, atol=1e-12) or np.allclose(q2, [-v for v in q], rtol=0, atol=1e-12)
        M = RO.compose(p, q, s)
        MI = RO.multiply(RO.invert(M), M)
        assert np.allclose(MI, I16, rtol=0, atol=1e-12)
    assert RO.invert([0.0] * 16) == [0.0] * 16


def test_sphere_axis_aligned_and_inside_and_behind():
    # ray from (0,0,10) down -z at a sphere of radius 2 at the origin: t0 = 8, hit (0,0,2), normal +z
    h = RO.intersect_sphere([0.0, 0.0, 10.0], [0.0, 0.0, -1.0], [0.0, 0.0, 0.0], 2.0)
    assert h[0] == [0.0, 0.0, 2.0] and h[1] == [0.0, 0.0, 1.0] and h[2] == 8.0
    # origin inside the sphere: t0 < 0, t1 = 2 is used -> exit point (0,0,-2)
    h = RO.intersect_sphere([0.0, 0.0, 0.0], [0.0, 0.0, -1.0], [0.0, 0.0, 0.0], 2.0)
    assert h[2] == 2.0 and h[0] == [0.0, 0.0, -2.0]
    # sphere behind the ray: t1 < 0 -> no hit
    assert RO.intersect_sphere([0.0, 0.0, 10.0], [0.0, 0.0, 1.0], [0.0, 0.0, 0.0], 2.0) is None
    # grazing miss
    assert RO.intersect_sphere([3.0, 0.0, 10.0], [0.0, 0.0, -1.0], [0.0, 0.0, 0.0], 2.0) is None


def test_box_inside_zero_component_and_entry_face_only():
    mn, mx = [0.0, 0.0, 0.0], [1.0, 1.0, 1.0]
    assert RO.intersect_box([0.5, 0.5, 0.5], [1.0, 0.0, 0.0], mn, mx)                       # origin inside
    assert RO.intersect_box([1.00005, 0.5, 0.5], [1.0, 0.0, 0.0], mn, mx)                    # within the 1e-4 epsilon counts as inside
    assert not RO.intersect_box([1.001, 0.5, 0.5], [1.0, 0.0, 0.0], mn, mx)                  # outside, moving away
    assert RO.intersect_box([-5.0, 0.5, 0.5], [1.0, 0.0, 0.0], mn, mx)                       # y, z components 0: those axes are skipped
    assert not RO.intersect_box([-5.0, 2.0, 0.5], [1.0, 0.0, 0.0], mn, mx)
    d = RO.normalize([1.0, 1.0, 0.0])
    assert RO.intersect_box([-1.0, -0.5, 0.5], d, mn, mx)                                    # enters through x = 0 at y = 0.5
    assert RO.intersect_box([math.nan, 0.0, 0.0], [1.0, 0.0, 0.0], mn, mx)                   # a NaN origin counts as inside


def test_static_radius_comes_from_decomposed_SRT_not_the_stored_scales():
    # 90 degrees about (1, 1, 0)/sqrt(2): R = [[1/2, 1/2, a], [1/2, 1/2, -a], [-a, a, 0]], a = 1/sqrt(2).  S R with S = diag(1, 2, 4) has
    # columns (1/2, 1, -4a), (1/2, 1, 4a), (a, -2a, 0) of lengths sqrt(37)/2, sqrt(37)/2, sqrt(10)/2, so the sphere radius is
    # (sqrt(37) + sqrt(10)/2) / 3 = 2.5546..., not the mean of the stored scales 7/3.
    q = np.array([0.5, 0.5, 0.0, math.sqrt(0.5)], np.float32)
    c, s, _ = RO.splat_inputs([0.0, 0.0, 0.0], np.array([1, 2, 4], np.float32), q, dynamic=False)
    radius = (s[0] + s[1] + s[2]) / 3
    assert abs(radius - (math.sqrt(37) + math.sqrt(10) / 2) / 3) < 1e-6
    assert abs(radius - 7 / 3) > 0.2
    # dynamic: the stored scales
    _, s, _ = RO.splat_inputs([0.0, 0.0, 0.0], np.array([1, 2, 4], np.float32), q, dynamic=True)
    assert s == [1.0, 2.0, 4.0]


def _one_splat_scene(scale, alpha=255, dynamic=True):
    return RO.Scene(np.zeros((1, 3)), np.array([scale], np.float32), np.array([[0, 0, 0, 1]], np.float32), np.array([alpha], np.uint8),
                    dynamic=dynamic)


def test_alpha_one_ellipsoid_hits_at_the_centre_and_small_scales_are_skipped():
    sc = _one_splat_scene([1, 1, 1], alpha=1)
    # u = log10(1) * 2 = 0: fromSphereSpace is singular and invert returns the zero matrix.  applyMatrix4 by it divides by its w = 0, so the
    # sphere-space ray is NaN, every comparison of intersectSphere fails and the splat "hits" -- even for a ray that passes far away -- with
    # a NaN point (the hit sorts last)
    h = RO.splat_hit(sc, 0, [50.0, 50.0, 10.0], [0.0, 0.0, -1.0], ellipsoid=True)
    assert h is not None and all(v != v for v in h[0] + h[1])
    # u = 2 log10(byte) is in (0, 2) for bytes 2-9 (the ellipsoid is at most twice the stored scales) and grows to 4.81 at 255
    for b in range(2, 10):
        assert 0 < RO.LOG10_BYTE[b] * 2 < 2
        h = RO.splat_hit(_one_splat_scene([1, 1, 1], alpha=b), 0, [0.0, 0.0, 10.0], [0.0, 0.0, -1.0], ellipsoid=True)
        assert h is not None and abs(h[0][2] - RO.LOG10_BYTE[b] * 2) < 1e-12
    # f32(1e-7) = 1.0000000117e-7 > 1e-7 is kept; the largest f32 at or below 1e-7 is skipped
    below = float(np.nextafter(np.float32(1e-7), np.float32(0)))
    assert RO.splat_hit(_one_splat_scene([1e-7, 1, 1]), 0, [0.0, 0.0, 10.0], [0.0, 0.0, -1.0], ellipsoid=False) is not None
    for s in ([below, 1, 1], [1, 1e-8, 1], [1, 1, 0.0], [1, 1, -1.0]):
        assert RO.splat_hit(_one_splat_scene(s), 0, [0.0, 0.0, 10.0], [0.0, 0.0, -1.0], ellipsoid=False) is None
    assert RO.splat_hit(_one_splat_scene([2e-7, 1, 1]), 0, [0.0, 0.0, 10.0], [0.0, 0.0, -1.0], ellipsoid=False) is not None


def _slab(o, d, mn, mx):
    """Independent ray/box test: the slab method (t >= 0)."""
    t0, t1 = 0.0, math.inf
    for k in range(3):
        if d[k] == 0:
            if o[k] < mn[k] or o[k] > mx[k]:
                return False
            continue
        a, b = (mn[k] - o[k]) / d[k], (mx[k] - o[k]) / d[k]
        t0, t1 = max(t0, min(a, b)), min(t1, max(a, b))
    return t0 <= t1


def test_reached_leaves_against_the_slab_method():
    rng = np.random.default_rng(7)
    pts = rng.normal(0, 2, (6000, 3)).astype(np.float32)
    root = RO.build_tree(pts)
    arrays = RO.tree_arrays(root)
    leaves = tree_oracle.build_leaves(pts)
    assert len(leaves) == len(arrays["offsets"]) - 1
    assert np.array_equal(np.concatenate([np.asarray(l[3], np.uint32) for l in leaves]), arrays["indexes"])
    nodes = []

    def walk(n, anc):
        anc = anc + [n]
        if n.indexes:
            nodes.append((n, anc))
        for ch in n.children:
            walk(ch, anc)

    walk(root, [])
    near_face = differ = 0
    for _ in range(300):
        o = list(rng.normal(0, 6, 3))
        d = RO.normalize(list(rng.normal(0, 1, 3)))
        got = {id(n) for n in RO.reached_leaves(root, o, d)}
        for leaf, anc in nodes:
            want = all(_slab(o, d, a.min, a.max) for a in anc)
            if want != (id(leaf) in got):
                # the reference's test uses a 1e-4 containment epsilon and only the entry faces: disagreements must be near a face
                grown = all(_slab(o, d, [v - 2e-4 for v in a.min], [v + 2e-4 for v in a.max]) for a in anc)
                assert grown, "leaf reached/missed far from any face"
                near_face += 1
            differ += 0
    assert near_face < 50


def test_sphere_hits_against_closest_approach():
    rng = np.random.default_rng(3)
    c = rng.normal(0, 1, (2000, 3))
    r = rng.uniform(0.05, 0.5, 2000)
    o = np.array([0.3, -0.2, 8.0])
    d = np.array(RO.normalize([0.01, 0.02, -1.0]))
    v = c - o
    tca = v @ d
    d2 = (v * v).sum(1) - tca * tca
    hit = d2 <= r * r
    thc = np.sqrt(np.maximum(r * r - d2, 0))
    t = np.where(tca - thc < 0, tca + thc, tca - thc)
    for i in range(2000):
        h = RO.intersect_sphere(list(o), list(d), list(c[i]), float(r[i]))
        assert (h is not None) == (bool(hit[i]) and tca[i] + thc[i] >= 0)
        if h is not None:
            assert abs(h[2] - t[i]) <= 1e-12 * max(1.0, abs(t[i]))


@pytest.mark.parametrize("ortho", [False, True])
def test_host_ray_setup_projects_back_to_the_pixel(ortho):
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.raycaster import Raycaster

    class Cam:
        pass

    cam = Cam()
    w, h = 1280, 720
    cam.matrixWorld = TM.camera_world_matrix([1.5, 2.6, -6.3], [0.4, 1.9, 1.5], [0.0, 1.0, 0.0])
    cam.near, cam.far = 0.1, 1000.0
    cam.isOrthographicCamera = ortho
    cam.projectionMatrix = TM.make_orthographic(-8, 8, 4.5, -4.5, 0.1, 1000.0) if ortho else TM.make_perspective(50, w / h, 0.1, 1000.0)
    rc = Raycaster()
    view_proj = TM.multiply(cam.projectionMatrix, TM.invert(cam.matrixWorld))
    for x, y in ((0.0, 0.0), (640.5, 360.25), (1279.0, 719.0), (17.0, 600.0)):
        rc.setFromCameraAndScreenPosition(cam, (x, y), (w, h))
        o, dvec = RO.ray_from_camera(cam.projectionMatrix, cam.matrixWorld, (x, y), (w, h), orthographic=ortho)
        assert rc.ray.origin == o and rc.ray.direction == dvec            # product set-up == oracle bit for bit
        p = [o[k] + dvec[k] * 7.0 for k in range(3)]
        ndc = RO.apply_matrix4(p, list(view_proj))
        px, py = (ndc[0] + 1) / 2 * w, h - (ndc[1] + 1) / 2 * h
        assert abs(px - x) < 1e-9 and abs(py - y) < 1e-9


def test_new_struct_sizes_match_ctypes():
    from gaussiansplats3d_b200 import _native as N
    src = ('#include "gsplat_b200.h"\n#include <stdio.h>\nint main(){printf("%zu %zu %zu %zu\\n",sizeof(gs_ray_record),sizeof(gs_raycast_params),'
           'sizeof(gs_ray_hit),sizeof(gs_config));return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        p = Path(d) / "probe.c"
        p.write_text(src)
        subprocess.run(["/usr/bin/gcc", "-I", str(ROOT / "include"), str(p), "-o", str(Path(d) / "probe")], check=True)
        out = [int(v) for v in subprocess.run([str(Path(d) / "probe")], capture_output=True, text=True, check=True).stdout.split()]
    assert out == [C.sizeof(N.gs_ray_record), C.sizeof(N.gs_raycast_params), C.sizeof(N.gs_ray_hit), C.sizeof(N.gs_config)]
    assert out[0] == 56 == N.RAY_RECORD_DTYPE.itemsize and out[2] == 64 == N.RAY_HIT_DTYPE.itemsize


def test_addon_binds_the_raycast_entries_and_the_shim_uses_only_exports():
    src = (ROOT / "js" / "gsplat_b200_addon.cc").read_text()
    exported = set(re.findall(r'EXPORT\("(\w+)"', src))
    for sym in ("gs_upload_ray_records", "gs_upload_splat_tree_nodes", "gs_raycast"):
        assert re.search(r"\b" + sym + r"\s*\(", src)
    used = set(re.findall(r"\baddon\.(\w+)\(", (ROOT / "js" / "RaycasterB200.js").read_text()))
    assert {"raycast", "uploadSplatTreeNodes", "uploadSplatTree"} <= used <= exported


def test_product_tree_export_matches_the_oracle_nodes():
    from gaussiansplats3d_b200.splat_tree import SplatTree
    rng = np.random.default_rng(11)
    pts = np.concatenate([rng.normal(0, 1, (5000, 3)), np.round(rng.normal(0, 2, (3000, 3)))]).astype(np.float32)   # grid-snapped centres on faces
    alphas = rng.integers(0, 256, pts.shape[0]).astype(np.uint8)
    lv = SplatTree().processSplatMesh(pts, alphas, 1)
    want = RO.tree_arrays(RO.build_tree(pts, alphas))
    assert np.array_equal(lv.all_min, want["node_min"]) and np.array_equal(lv.all_max, want["node_max"])
    assert np.array_equal(lv.all_parent, want["node_parent"]) and np.array_equal(lv.leaf_node, want["leaf_node"])
    assert np.array_equal(lv.offsets, want["offsets"]) and np.array_equal(lv.indexes, want["indexes"])
