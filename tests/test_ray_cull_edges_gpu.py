"""GPU: the raycaster (csrc/ray_kernels.cuh, k_ray_* and their forest variants) and the SplatTree cull and layout (csrc/cull_kernels.cuh)
at their edge geometry, bit for bit against oracle/ray_oracle.py, oracle/tree_oracle.py and the forest restatements of
tests/test_subtrees.py.  Scenes are crafted records: axis-parallel rays (along node faces at the box epsilon), origins inside boxes and
splats, tangent rays, degenerate scales, alpha bytes 0 / 1 / 2 / 255, non-finite centres and rotations, mirrored, non-uniform, near-180
degree and singular transforms, exact duplicates and NaN distances cut by the capacity; leaves at the camera, on the view axes, within a
few ulp of the cull thresholds, one-splat leaves, dist == nodeSize, more than 256 equal keys and non-finite centres.

A bit-exact comparison says nothing about a branch its inputs never reach, so every case counts on the oracle side how often its branch
was taken (the style of projection_cases.ran) and fails when the count is zero.  The oracles follow the kernels' operation order, so every
finite hit is also checked in np.longdouble from the record and the ray alone: on the surface, on the ray, the right root, its distance,
and its normal."""
import collections
import math
import struct
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent))
from test_subtrees import forest_gather, forest_leaves, forest_raycast  # noqa: E402

from oracle import file_oracle as FO  # noqa: E402
from oracle import ray_oracle as RO  # noqa: E402
from oracle import tree_oracle as TO  # noqa: E402

pytestmark = pytest.mark.gpu

# ---- tolerances of the longdouble check (relative to the splat's size L: its radius, or the largest axis of its ellipsoid) -------------
SURFACE_REL = 1e-9            # |hit - c| = r, or |F^-1 (hit - c)| = 1
ON_RAY_REL = 1e-9             # distance of the hit from the ray's line
ROOT_REL = 1e-7               # t against the root the hit must be (a tangent ray loses half the digits in sqrt(r^2 - diff))
NORMAL_SIN = 1e-9             # |n x n_expected|
DIST_REL = 1e-14              # distance against |hit - origin|
COORD_ULPS = 16               # f64 rounding of the coordinates themselves: this many ulps of the largest one involved, added to each bound
CANCEL_ULPS = 16              # Ray.intersectSphere's c2 - tca^2 cancels about this many ulps of |o - c|^2: added to each bound (see _check_hits)
NEAR_SINGULAR_COND = 1e4      # a splat whose S R (T) has a larger condition number is near singular: its decomposition and F^-1 lose digits,
NEAR_SINGULAR_REL = 1e-6      # and it is held to this in place of the four relative bounds above (surface, ray, root, normal); counted
EPS = float(np.finfo(np.float64).eps)
F32_EPS_SCALES = (float(np.nextafter(np.float32(1e-7), np.float32(0))), float(np.float32(1e-7)), 0.0)


def _N():
    from gaussiansplats3d_b200 import _native as N
    return N


def _bits_equal(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint64), b[~nb].view(np.uint64))


def _nan(bits):
    return struct.unpack("<d", struct.pack("<Q", bits))[0]


NANS = (0x7ff8000000000000, 0xfff8000000000000, 0x7ff8000000000123, 0xfff800000000abcd)   # quiet NaNs of both signs, with payloads


# ---- the branch counters ---------------------------------------------------------------------------------------------------------------
class Probe:
    """Wraps the ray oracle's Ray.js / splat / decompose steps and counts the branches the cases are about."""

    def __init__(self, monkeypatch):
        self.n = collections.Counter()
        n = self.n
        box, sphere, splat_hit, decompose, quat = RO.intersect_box, RO.intersect_sphere, RO.splat_hit, RO.decompose, RO.quaternion_from_rotation_matrix
        eps = RO.BOX_EPSILON

        def intersect_box(o, d, mn, mx):
            r = box(o, d, mn, mx)
            if any(v != v for v in o):
                n["nan origin counts as inside"] += r
            elif RO.box_contains(mn, mx, o):
                n["origin inside a node"] += 1
                n["origin inside only by the epsilon"] += not all(mn[k] <= o[k] <= mx[k] for k in range(3))
            elif r and any(v == 0.0 for v in d):
                n["d[a] == 0 skipped, node reached"] += 1
            for k in range(3):
                if d[k] == 0.0 and (o[k] == mn[k] - eps or o[k] == mx[k] + eps):
                    n["ray on a face at the epsilon, reached" if r else "ray on a face at the epsilon, missed"] += 1
                if d[k] == 0.0 and (o[k] == math.nextafter(mn[k] - eps, -math.inf) or o[k] == math.nextafter(mx[k] + eps, math.inf)):
                    n["ray one ulp past the epsilon, reached" if r else "ray one ulp past the epsilon, missed"] += 1
            return r

        def intersect_sphere(o, d, center, radius):
            v = [center[0] - o[0], center[1] - o[1], center[2] - o[2]]
            tca = v[0] * d[0] + v[1] * d[1] + v[2] * d[2]
            diff = (v[0] * v[0] + v[1] * v[1] + v[2] * v[2]) - tca * tca
            r2 = radius * radius
            n["tangent: diff == r2"] += diff == r2
            n["tangent: diff == r2 + 1 ulp"] += diff == math.nextafter(r2, math.inf)
            n["tangent: diff == r2 - 1 ulp"] += diff == math.nextafter(r2, -math.inf)
            if diff <= r2:
                thc = RO.sqrt(r2 - diff)
                t0, t1 = tca - thc, tca + thc
                n["behind: t1 < 0"] += t1 < 0
                n["inside: t0 < 0 <= t1, t1 used"] += t0 < 0 <= t1
            h = sphere(o, d, center, radius)
            n["NaN hit"] += h is not None and h[2] != h[2]
            return h

        def hit(scene, i, o, d, ellipsoid):
            c, s, F, Inv = scene.inputs(i, ellipsoid)
            if s[0] <= RO.SCALE_EPSILON or s[1] <= RO.SCALE_EPSILON or s[2] <= RO.SCALE_EPSILON:
                n["scale epsilon skip"] += 1
                n["scale == 1e-7 exactly, skipped"] += any(v == RO.SCALE_EPSILON for v in s)
                n["negative scale, skipped"] += any(v < 0 for v in s)
            elif ellipsoid:
                n["singular F: inverse is zero"] += all(v == 0.0 for v in Inv)
                n["non-finite F"] += not all(math.isfinite(v) for v in F)
            n["non-finite centre reached"] += not all(math.isfinite(v) for v in c)
            return splat_hit(scene, i, o, d, ellipsoid)

        def dec(te):
            n["decompose: det < 0 flips sx"] += RO.determinant(te) < 0
            return decompose(te)

        def q_from_m(te):
            m11, m22, m33 = te[0], te[5], te[10]
            b = 0 if m11 + m22 + m33 > 0 else 1 if (m11 > m22 and m11 > m33) else 2 if m22 > m33 else 3
            n[f"setFromRotationMatrix branch {b}"] += 1
            return quat(te)

        for name, f in (("intersect_box", intersect_box), ("intersect_sphere", intersect_sphere), ("splat_hit", hit), ("decompose", dec),
                        ("quaternion_from_rotation_matrix", q_from_m)):
            monkeypatch.setattr(RO, name, f)

    def take(self):
        out = dict(self.n)
        self.n.clear()
        return out


def _require(counts, what, *names):
    print(what, {k: counts.get(k, 0) for k in names})
    for k in names:
        assert counts.get(k, 0) > 0, f"{what}: the case no longer reaches '{k}' ({counts})"


# ---- the independent longdouble check --------------------------------------------------------------------------------------------------
LD = np.longdouble


def _rot_ld(q):
    """Matrix4.makeRotationFromQuaternion (x, y, z, w), in longdouble."""
    x, y, z, w = (LD(v) if isinstance(v, LD) else LD(float(v)) for v in q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]], dtype=LD)


def _quat_ld(m):
    """Quaternion.setFromRotationMatrix (x, y, z, w) of a 3x3 matrix, in longdouble: a static splat's S R T is not a rotation once its
    columns are normalised (S is non-uniform and on the left), and the reference's ellipsoid is R of this quaternion, not S R T itself."""
    tr = m[0, 0] + m[1, 1] + m[2, 2]
    if tr > 0:
        s = LD(0.5) / np.sqrt(tr + 1)
        return [(m[2, 1] - m[1, 2]) * s, (m[0, 2] - m[2, 0]) * s, (m[1, 0] - m[0, 1]) * s, LD(0.25) / s]
    if m[0, 0] > m[1, 1] and m[0, 0] > m[2, 2]:
        s = 2 * np.sqrt(1 + m[0, 0] - m[1, 1] - m[2, 2])
        return [s / 4, (m[0, 1] + m[1, 0]) / s, (m[0, 2] + m[2, 0]) / s, (m[2, 1] - m[1, 2]) / s]
    if m[1, 1] > m[2, 2]:
        s = 2 * np.sqrt(1 + m[1, 1] - m[0, 0] - m[2, 2])
        return [(m[0, 1] + m[1, 0]) / s, s / 4, (m[1, 2] + m[2, 1]) / s, (m[0, 2] - m[2, 0]) / s]
    s = 2 * np.sqrt(1 + m[2, 2] - m[0, 0] - m[1, 1])
    return [(m[0, 2] + m[2, 0]) / s, (m[1, 2] + m[2, 1]) / s, s / 4, (m[1, 0] - m[0, 1]) / s]


def _inv3(A):
    """Inverse of a 3x3 longdouble matrix by its adjugate (None when singular)."""
    c = np.empty((3, 3), LD)
    for r in range(3):
        for k in range(3):
            m = np.delete(np.delete(A, r, 0), k, 1)
            c[r, k] = (-1) ** (r + k) * (m[0, 0] * m[1, 1] - m[0, 1] * m[1, 0])
    det = (A[0] * c[0]).sum()
    return None if det == 0 else c.T / det


def _affine_ld(m16):
    m = np.asarray(m16, np.float64).reshape(4, 4).T.astype(LD)          # column-major elements -> rows
    return m[:3, :3], m[:3, 3]


def _norm(v):
    return np.sqrt((v * v).sum())


def _geometry(rec, i, ellipsoid, transform16):
    """Splat i in the mesh's local space from its record alone: centre, and the radius (sphere) or F (ellipsoid), as the reference defines
    them -- a static mesh's splat takes decompose(makeScale(s) R(q) T): its scale is the column lengths of S R T (the first negative when
    det < 0), its radius their mean, and its ellipsoid u R(q') S' with q' the quaternion of the normalised columns; a dynamic mesh's uses s
    and q as stored.  u = 2 log10(alpha)."""
    c = np.asarray(rec["center"][i], np.float64).astype(LD)
    s = np.asarray(rec["scale"][i], np.float64).astype(LD)
    R = _rot_ld(rec["rotation"][i])
    M = R * s[None, :]                                                    # R S: column k scaled by s_k
    if transform16 is not None:
        A, t = _affine_ld(transform16)
        c = A @ c + t
        M = (np.diag(s) @ R) @ A                                          # S R T (Matrix4 products compose left to right)
    cols = s
    if transform16 is not None:
        cols = np.sqrt((M * M).sum(0))
        if np.linalg.det(M.astype(np.float64)) < 0:
            cols[0] = -cols[0]
    sv = np.linalg.svd(M.astype(np.float64), compute_uv=False) if np.isfinite(M.astype(np.float64)).all() else [np.inf, 0.0]
    cond = sv[0] / sv[-1] if sv[-1] > 0 else np.inf
    if not ellipsoid:
        return c, cols.sum() / 3, None, cond
    a = int(rec["alpha"][i])
    u = LD(2) * np.log10(LD(a)) if a else LD(-np.inf)
    if transform16 is not None:
        M = _rot_ld(_quat_ld(M / cols[None, :])) * cols[None, :]
    return c, None, u * M, cond


def _check_hits(got, rec, origin, direction, from_local16, ellipsoid, transform16, stats):
    """Every finite hit against the geometry of its splat (the reference's ray set-up: the local ray is the world ray under
    invert(fromLocal); hits and normals go back through fromLocal -- normals with its translation, Raycaster.js:62-66)."""
    A, t = _affine_ld(from_local16)
    Ai = _inv3(A)
    ow = np.asarray(origin, np.float64).astype(LD)
    dw = np.asarray(direction, np.float64).astype(LD)
    for h in got:
        hw, nw, dist = h["origin"].astype(LD), h["normal"].astype(LD), LD(float(h["distance"]))
        if not (np.isfinite(h["origin"]).all() and np.isfinite(h["normal"]).all() and np.isfinite(h["distance"])):
            continue
        assert Ai is not None, "a finite hit through a singular fromLocal"
        c, r, F, cond = _geometry(rec, int(h["splat_index"]), ellipsoid, transform16)
        hl, ol = Ai @ (hw - t), Ai @ (ow - t)
        dl = Ai @ dw
        dl = dl / _norm(dl)
        big = max(float(np.abs(x).max()) for x in (hw, ow, c, t))
        tol_abs = COORD_ULPS * EPS * big * (1 + float(np.abs(Ai).max()))
        near = cond > NEAR_SINGULAR_COND
        stats["near singular" if near else "regular"] += 1
        stats["finite hits checked"] += 1
        rel = NEAR_SINGULAR_REL if near else 0.0
        if F is None:                                                       # sphere, in local units
            L = r
            oc, dd, rad = ol - c, dl, r
            surface = abs(_norm(hl - c) - r)
            nl = (hl - c) / r
            amp = LD(1)
        else:                                                               # ellipsoid, solved on the unit sphere of F^-1 (x - c)
            Fi = _inv3(F)
            assert Fi is not None
            L = LD(np.linalg.svd(F.astype(np.float64), compute_uv=False)[0])
            oc, dd, rad = Fi @ (ol - c), Fi @ dl, LD(1)
            p = Fi @ (hl - c)
            surface = abs(_norm(p) - 1) * L
            nl = p
            amp = LD(float(np.abs(Fi).max())) * L
        # Ray.intersectSphere's c2 - tca^2 loses CANCEL_ULPS eps |o - c|^2 (in the units it solves in): the hit moves by that over 2 r
        # along the surface normal, and by its square root along the ray next to a tangent
        canc = CANCEL_ULPS * EPS * float((oc * oc).sum())
        unit = L / rad
        assert surface <= (max(SURFACE_REL, rel) * rad + canc / (2 * rad)) * unit + tol_abs * amp, ("off the surface", surface, L, near, h)
        off = hl - ol
        tt = (off * dl).sum()
        assert _norm(off - tt * dl) <= max(ON_RAY_REL, rel) * L + tol_abs * amp, ("off the ray", h)
        a2, b1, c0 = (dd * dd).sum(), (oc * dd).sum(), (oc * oc).sum() - rad * rad
        disc = max(b1 * b1 - a2 * c0, LD(0))
        t0, t1 = (-b1 - np.sqrt(disc)) / a2, (-b1 + np.sqrt(disc)) / a2
        rt = max(ROOT_REL, rel) * L + LD(math.sqrt(canc)) * unit / np.sqrt(a2) * 4 + tol_abs * amp
        assert tt >= -rt and t1 >= -rt, ("behind the origin", tt, t0, t1, h)
        if t0 > rt:
            assert abs(tt - t0) <= rt, ("not the near root", tt, t0, t1, h)
        elif t0 < -rt:
            assert abs(tt - t1) <= rt, ("inside: not the far root", tt, t0, t1, h)
            stats["inside: far root"] += 1
        assert abs(_norm(hw - ow) - dist) <= DIST_REL * dist + tol_abs, ("distance", h)
        ne = A @ nl + t
        ne = ne / _norm(ne)
        cross = np.cross(nw.astype(np.float64), ne.astype(np.float64))
        assert _norm(cross.astype(LD)) <= max(NORMAL_SIN, rel) + 4 * math.sqrt(canc) / float(rad) + tol_abs * amp / float(L) and (nw * ne).sum() > 0, ("normal", h)


# ---- records, trees, engines -----------------------------------------------------------------------------------------------------------
# Rotations that are unit quaternions in f32 exactly: R(q) is then orthogonal, and a static splat's decomposed rotation is R(q) T's
EXACT_Q = np.array([(0, 0, 0, 1), (1, 0, 0, 0), (0, 1, 0, 0), (0, 0, 1, 0)] +
                   [(a * 0.5, b * 0.5, c * 0.5, 0.5) for a in (-1, 1) for b in (-1, 1) for c in (-1, 1)], np.float32)


def _records(n):
    N = _N()
    r = np.zeros(n, N.RAY_RECORD_DTYPE)
    r["rotation"] = [0, 0, 0, 1]
    r["alpha"] = 255
    return r


def _edge_scene(seed=1):
    """-> (records, proxy centres): a jittered 5x5x5 lattice of ordinary splats, then degenerate splats mixed into the same leaves.  The
    tree is built from the proxy centres (f32), so a splat with a non-finite centre still sits in an ordinary leaf."""
    rng = np.random.default_rng(seed)
    g = np.stack(np.meshgrid(*[np.arange(-2, 3)] * 3, indexing="ij"), -1).reshape(-1, 3) * 1.25
    base = g + rng.uniform(-0.3, 0.3, g.shape)
    rows = []                                              # (centre, scale, rotation, alpha, proxy)

    def add(c, s, q=(0, 0, 0, 1), a=255, proxy=None):
        rows.append((c, s, q, a, c if proxy is None else proxy))

    for k, c in enumerate(base):
        add(c, rng.uniform(0.15, 0.45, 3), EXACT_Q[rng.integers(len(EXACT_Q))], int(rng.integers(3, 256)))
    add((0.1, -0.05, 0.07), (0.9, 0.9, 0.9))                                   # a large splat around the origin: rays start inside it
    for k, c in enumerate(base[::7]):
        add(c + 0.02, (1.0, 0.3, 0.3))                                         # scale x exactly 1 and 2: under a (1e-7, 1, 1) transform,
        add(c - 0.02, (2.0, 0.3, 0.3))                                         # exactly 1e-7 (skipped) and 2e-7 (kept)
    for j, v in enumerate(F32_EPS_SCALES + (-0.2,)):
        for a in range(3):
            s = [0.3, 0.3, 0.3]
            s[a] = v
            add(base[(11 * j + 3 * a) % len(base)] + 0.05, s)
    for j, alpha in enumerate((0, 1, 2, 255) * 3):
        add(base[(5 * j + 1) % len(base)] - 0.05, (0.35, 0.25, 0.3), EXACT_Q[j % len(EXACT_Q)], alpha)
    for j, bad in enumerate([_nan(b) for b in NANS] + [math.inf, -math.inf]):
        for a in range(3):
            p = base[(13 * j + 4 * a + 2) % len(base)]
            c = p.copy()
            c[a] = bad
            add(c, (0.3, 0.3, 0.3), proxy=p)
    for j in range(4):
        add(base[(17 * j + 6) % len(base)] + 0.03, (0.3, 0.2, 0.25), (np.nan, 0, 0, 1) if j % 2 else (0.5, np.nan, 0.5, 0.5))
    for j in range(12):                                                        # exact duplicates: in the same leaf ...
        k = int(rng.integers(len(base)))
        rows.append(rows[k])
        rows.append(rows[k])
    for j in range(12):                                                        # ... and in another leaf (proxy one lattice step away)
        k = int(rng.integers(len(base)))
        c, s, q, a, p = rows[k]
        rows.append((c, s, q, a, np.asarray(p) + (1.25 if p[0] < 2 else -1.25, 0.0, 0.0)))
    rec = _records(len(rows))
    rec["center"] = [r[0] for r in rows]
    rec["scale"] = [r[1] for r in rows]
    rec["rotation"] = [r[2] for r in rows]
    rec["alpha"] = [r[3] for r in rows]
    return rec, np.array([r[4] for r in rows], np.float64).astype(np.float32)


MAX_CENTERS = 8


def _engine(rec, proxy32, *, dynamic, transform16=None):
    from gaussiansplats3d_b200.engine import Engine
    from gaussiansplats3d_b200.raycaster import record_centers_f32
    from gaussiansplats3d_b200.splat_tree import SplatTree
    pts = proxy32
    if transform16 is not None:                  # a static mesh's tree holds the transformed centres (SplatTree.js:343-348)
        pr = _records(len(proxy32))
        pr["center"] = proxy32.astype(np.float64)
        pts = record_centers_f32(pr, transform16)
    every = np.full(len(pts), 255, np.uint8)     # alpha 0 splats stay in the tree: the cast, not the build, must meet them
    e = Engine(len(rec), dynamic_mode=dynamic, ray_records=True)
    e.upload_ray_records(rec, 0, transform16)
    lv = SplatTree(8, MAX_CENTERS).processSplatMesh(pts, every, 1)
    e.upload_splat_tree(lv)
    e.upload_splat_tree_nodes(lv)
    return e, RO.build_tree(pts, every, max_centers=MAX_CENTERS)


def _nodes(root):
    out = []

    def visit(n):
        out.append(n)
        for ch in n.children:
            visit(ch)
    visit(root)
    return out


def _axis_rays(root, lo, hi, grid, extra_origins=()):
    """Rays along +-x, +-y, +-z: orthographic (a grid of parallel rays from outside [lo, hi]) and perspective (one eye per axis, rays fanned
    over the grid, the centre one axis-parallel); along faces of nodes at min - 1e-4 and max + 1e-4 (and one ulp further out), in f64;
    from the centres of leaf boxes; and from `extra_origins` (inside splats) along every axis."""
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    mid, span = (lo + hi) / 2, (hi - lo) / 2 + 1.0
    ortho, persp = [], []
    ticks = np.linspace(-1, 1, grid) * 0.93
    leaves = [n for n in _nodes(root) if n.indexes]
    inner = [n for n in _nodes(root)][:: max(1, len(_nodes(root)) // 12)]
    for a in range(3):
        a1, a2 = (a + 1) % 3, (a + 2) % 3
        for sgn in (1.0, -1.0):
            d = [0.0, 0.0, 0.0]
            d[a] = -sgn
            start = mid[a] + sgn * (span[a] + 2.0)
            for u in ticks:
                for v in ticks:
                    o = [0.0, 0.0, 0.0]
                    o[a], o[a1], o[a2] = start, mid[a1] + u * span[a1], mid[a2] + v * span[a2]
                    ortho.append((o, list(d)))
                    eye = [0.0, 0.0, 0.0]
                    eye[a], eye[a1], eye[a2] = start, mid[a1], mid[a2]
                    tgt = list(o)
                    tgt[a] = mid[a] - sgn * span[a]
                    persp.append((eye, RO.normalize([tgt[k] - eye[k] for k in range(3)])))
            for n in inner:                                   # along node faces, at the box epsilon and one ulp past it
                for edge in (n.min[a1] - RO.BOX_EPSILON, n.max[a1] + RO.BOX_EPSILON):
                    for e2 in (edge, math.nextafter(edge, -math.inf if edge < n.min[a1] else math.inf)):
                        o = [0.0, 0.0, 0.0]
                        o[a], o[a1], o[a2] = start, e2, (n.min[a2] + n.max[a2]) / 2
                        ortho.append((o, list(d)))
            for n in leaves[:: max(1, len(leaves) // 10)]:    # from inside leaf boxes
                ortho.append(([(n.min[k] + n.max[k]) / 2 for k in range(3)], list(d)))
            for o in extra_origins:
                ortho.append(([float(v) for v in o], list(d)))
    return ortho, persp


def _cast_and_compare(e, want_fn, rays, ellipsoid, rec, fl, transform16, stats, *, capacities=False, **kw):
    """Every ray: gs_raycast == the oracle bit for bit, at full capacity and (capacities=True) at 0, 1, inside a tie group and the total."""
    hits = 0
    for o, d in rays:
        want = want_fn(o, d)
        got, total = e.raycast(o, d, None if kw.get("sub_tree_from_local") is not None else fl, ellipsoid=ellipsoid, capacity=len(want) + 3, **kw)
        _assert_same(got, total, want, len(want) + 3, (o, d))
        if rec is not None:
            _check_hits(got, rec, o, d, fl if fl is not None else RO.IDENTITY, ellipsoid, transform16, stats)
        hits += total
        stats["NaN-distance hits"] += sum(1 for h in want if h[0] != h[0])
        if capacities and len(want) > 1:
            caps = {0, 1, len(want)}
            for k in range(1, len(want)):
                a, b = want[k - 1][0], want[k][0]
                if (a == b or (a != a and b != b)) and k not in caps:
                    caps.add(k)                                # cuts between two equal distances
                    stats["tie group cut by the capacity"] += 1
                    break
            for cap in sorted(caps):
                got, total = e.raycast(o, d, None if kw.get("sub_tree_from_local") is not None else fl, ellipsoid=ellipsoid, capacity=cap, **kw)
                _assert_same(got, total, want, cap, (o, d, cap))
    return hits


def _assert_same(got, total, want, cap, what):
    assert total == len(want), (what, total, len(want))
    k = min(cap, len(want))
    assert got.shape[0] == k, what
    w = want[:k]
    assert np.array_equal(got["splat_index"], np.array([h[2] for h in w], np.uint32)), what
    assert _bits_equal(got["distance"], [h[0] for h in w]), what
    assert _bits_equal(got["origin"], np.array([h[3] for h in w], np.float64).reshape(-1, 3)), what
    assert _bits_equal(got["normal"], np.array([h[4] for h in w], np.float64).reshape(-1, 3)), what


def _inside_origins(rec):
    big = np.flatnonzero(rec["scale"].min(1) >= 0.3)
    return [rec["center"][i] for i in big[:6]]


# ---- raycaster cases 1-3, 6: dynamic mesh, identity fromLocal ---------------------------------------------------------------------------
@pytest.mark.parametrize("ellipsoid", [False, True], ids=["sphere", "ellipsoid"])
def test_axis_parallel_inside_degenerate_and_ties(monkeypatch, ellipsoid):
    probe = Probe(monkeypatch)
    rec, proxy = _edge_scene()
    e, root = _engine(rec, proxy, dynamic=True)
    scene = RO.Scene(rec["center"], rec["scale"], rec["rotation"], rec["alpha"], dynamic=True)
    stats = collections.Counter()
    try:
        ortho, persp = _axis_rays(root, root.min, root.max, 5, _inside_origins(rec))
        for kind, rays in (("orthographic", ortho), ("perspective", persp)):
            hits = _cast_and_compare(e, lambda o, d: RO.intersect_splat_mesh(root, scene, o, d, RO.IDENTITY, ellipsoid=ellipsoid), rays, ellipsoid,
                                     rec, None, None, stats, capacities=True)
            assert hits > 0, kind
        counts = {**probe.take(), **stats}
        _require(counts, f"axis-parallel / inside / degenerate ({'ellipsoid' if ellipsoid else 'sphere'})",
                 "d[a] == 0 skipped, node reached", "origin inside a node", "ray on a face at the epsilon, reached",
                 "ray one ulp past the epsilon, missed", "inside: t0 < 0 <= t1, t1 used", "behind: t1 < 0", "scale epsilon skip",
                 "negative scale, skipped", "non-finite centre reached", "NaN hit", "NaN-distance hits", "tie group cut by the capacity",
                 "finite hits checked", "inside: far root", *(("singular F: inverse is zero", "non-finite F", "near singular") if ellipsoid else ()))
    finally:
        e.close()


@pytest.mark.parametrize("ellipsoid", [False, True], ids=["sphere", "ellipsoid"])
def test_tangent_rays_at_and_one_ulp_either_side(monkeypatch, ellipsoid):
    """A sphere at the origin and rays along +-z at a distance x from its axis, x chosen in f64 so that the oracle's diff - r2 is 0 and
    +-1 ulp (diff = (x^2 + z0^2) - z0^2 stays in r2's binade, so every ulp is reachable)."""
    probe = Probe(monkeypatch)
    rec = _records(9)
    rec["scale"] = np.float32(0.6)
    rec["center"][1:] = [(sx * 0.7, sy * 0.7, sz * 0.7) for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)]   # corners widen the root
    rec["scale"][1:] = np.float32(0.05)
    s = [float(v) for v in rec["scale"][0]]
    radius = (s[0] + s[1] + s[2]) / 3.0
    r2 = radius * radius
    z0 = 0.25
    want = {r2: [], math.nextafter(r2, math.inf): [], math.nextafter(r2, -math.inf): []}
    x0 = math.sqrt(r2)
    for _ in range(32):
        x0 = math.nextafter(x0, 0.0)
    for y in (0.0, 3e-9, 5e-9, 7e-9, 9e-9, 1.1e-8, 1.3e-8):            # y^2 moves (x^2 + y^2) by a fraction of x^2's step
        x = x0
        for _ in range(64):
            diff = ((-x) * (-x) + (-y) * (-y) + (-z0) * (-z0)) - z0 * z0
            if diff in want:
                want[diff].append((x, y))
            x = math.nextafter(x, math.inf)
    assert all(want.values()), {k: len(v) for k, v in want.items()}
    rays = []
    for xys in want.values():
        for x, y in xys[:3]:
            for sx in (1.0, -1.0):
                for up in (1.0, -1.0):
                    rays.append(([sx * x, y, up * z0], [0.0, 0.0, -up]))
                    rays.append(([y, sx * x, up * z0], [0.0, 0.0, -up]))
    e, root = _engine(rec, rec["center"].astype(np.float32), dynamic=True)
    scene = RO.Scene(rec["center"], rec["scale"], rec["rotation"], rec["alpha"], dynamic=True)
    stats = collections.Counter()
    try:
        _cast_and_compare(e, lambda o, d: RO.intersect_splat_mesh(root, scene, o, d, RO.IDENTITY, ellipsoid=ellipsoid), rays, ellipsoid, rec, None, None,
                          stats)
        counts = {**probe.take(), **stats}
        names = ("tangent: diff == r2", "tangent: diff == r2 + 1 ulp", "tangent: diff == r2 - 1 ulp") if not ellipsoid else ("finite hits checked",)
        _require(counts, f"tangent ({'ellipsoid' if ellipsoid else 'sphere'})", *names)
    finally:
        e.close()


# ---- raycaster cases 4 and 5: static scene transforms, dynamic fromLocal ----------------------------------------------------------------
def _xf(p, q, s):
    return [float(v) for v in RO.compose(p, q, s)]


def _near180(axis):
    h = (math.pi - 1e-3) / 2
    q = [0.0, 0.0, 0.0, math.cos(h)]
    q[axis] = math.sin(h)
    return q


STATIC_XF = {
    "mirror_x": _xf((0.2, -0.1, 0.3), (0, 0, 0, 1), (-1, 1, 1)),
    "mirror_yz": _xf((0.0, 0.5, 0.0), (0, 0, 0, 1), (1, -1, -1)),
    "nonuniform": _xf((0.0, 0.0, 0.0), (0, 0, 0, 1), (1e-3, 1, 1e3)),
    "rot180_x": _xf((0.3, 0.0, -0.2), _near180(0), (1, 1, 1)),
    "rot180_y": _xf((0.0, 0.2, 0.0), _near180(1), (1.5, 1.5, 1.5)),
    "rot180_z": _xf((-0.4, 0.1, 0.0), _near180(2), (1, 1, 1)),
    "singular": _xf((0.0, 0.0, 0.0), (0, 0, 0, 1), (1, 1, 0)),
    "scale_1e-7": _xf((0.0, 0.0, 0.0), (0, 0, 0, 1), (1e-7, 1, 1)),
}
STATIC_BRANCH = {
    "mirror_x": ("decompose: det < 0 flips sx", "negative scale, skipped"), "mirror_yz": ("finite hits checked",), "nonuniform": ("finite hits checked",),
    "rot180_x": ("setFromRotationMatrix branch 1",), "rot180_y": ("setFromRotationMatrix branch 2",), "rot180_z": ("setFromRotationMatrix branch 3",),
    "singular": ("scale epsilon skip",), "scale_1e-7": ("scale == 1e-7 exactly, skipped", "finite hits checked"),
}


@pytest.mark.parametrize("ellipsoid", [False, True], ids=["sphere", "ellipsoid"])
@pytest.mark.parametrize("name", list(STATIC_XF))
def test_static_scene_transforms(monkeypatch, name, ellipsoid):
    probe = Probe(monkeypatch)
    rec, proxy = _edge_scene(2)
    t = STATIC_XF[name]
    e, root = _engine(rec, proxy, dynamic=False, transform16=t)
    scene = RO.Scene(rec["center"], rec["scale"], rec["rotation"], rec["alpha"], dynamic=False, transform16=t)
    stats = collections.Counter()
    try:
        ortho, persp = _axis_rays(root, root.min, root.max, 3)
        _cast_and_compare(e, lambda o, d: RO.intersect_splat_mesh(root, scene, o, d, RO.IDENTITY, ellipsoid=ellipsoid), ortho + persp, ellipsoid,
                          rec, None, t, stats)
        counts = {**probe.take(), **stats}
        names = STATIC_BRANCH[name]
        if name.startswith("rot180") and not ellipsoid:
            names = ("finite hits checked",)      # sphere mode decomposes the scale only
        _require(counts, f"static {name} ({'ellipsoid' if ellipsoid else 'sphere'})", "d[a] == 0 skipped, node reached", *names)
        if name == "singular":
            assert counts.get("finite hits checked", 0) == 0   # every splat is skipped: a zero column
    finally:
        e.close()


FROM_LOCAL = {
    "mirrored": _xf((0.5, -0.25, 0.0), (0.0, 0.6, 0.0, 0.8), (-1, 1, 1)),
    "singular": _xf((0.5, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0), (1, 0, 1)),
    "translated_1e6": _xf((1e6, -2e6, 5e5), (0.1, 0.2, -0.3, 0.927), (1, 1, 1)),
}


def _to_world(rays, fl):
    A, t = _affine_ld(fl)
    if _inv3(A) is None:
        return rays
    out = []
    for o, d in rays:
        ow = (A @ np.asarray(o, np.float64).astype(LD) + t).astype(np.float64)
        dw = (A @ np.asarray(d, np.float64).astype(LD)).astype(np.float64)
        out.append(([float(v) for v in ow], RO.normalize([float(v) for v in dw])))
    return out


@pytest.mark.parametrize("ellipsoid", [False, True], ids=["sphere", "ellipsoid"])
@pytest.mark.parametrize("name", list(FROM_LOCAL))
def test_from_local(monkeypatch, name, ellipsoid):
    probe = Probe(monkeypatch)
    rec, proxy = _edge_scene(3)
    fl = FROM_LOCAL[name]
    e, root = _engine(rec, proxy, dynamic=True)
    scene = RO.Scene(rec["center"], rec["scale"], rec["rotation"], rec["alpha"], dynamic=True)
    stats = collections.Counter()
    try:
        ortho, persp = _axis_rays(root, root.min, root.max, 3)
        rays = _to_world(ortho[::2] + persp, fl)
        _cast_and_compare(e, lambda o, d: RO.intersect_splat_mesh(root, scene, o, d, fl, ellipsoid=ellipsoid), rays, ellipsoid, rec, fl, None, stats,
                          capacities=name == "singular")
        counts = {**probe.take(), **stats}
        names = {"mirrored": ("finite hits checked",), "singular": ("nan origin counts as inside", "NaN-distance hits", "tie group cut by the capacity"),
                 "translated_1e6": ("finite hits checked",)}[name]
        _require(counts, f"fromLocal {name} ({'ellipsoid' if ellipsoid else 'sphere'})", *names)
        if name == "singular":
            assert counts.get("finite hits checked", 0) == 0
    finally:
        e.close()


# ---- raycaster case 7: a forest ----------------------------------------------------------------------------------------------------------
def _ply(rec):
    """A .ply of the records (scale as log, rotation w x y z, opacity as the logit of alpha / 255)."""
    n = len(rec)
    a = np.clip(rec["alpha"].astype(np.float64), 0.5, 254.5) / 255.0
    cols = {"x": rec["center"][:, 0], "y": rec["center"][:, 1], "z": rec["center"][:, 2],
            **{f"scale_{k}": np.log(np.maximum(rec["scale"][:, k], 1e-30)) for k in range(3)},
            "rot_0": rec["rotation"][:, 3], "rot_1": rec["rotation"][:, 0], "rot_2": rec["rotation"][:, 1], "rot_3": rec["rotation"][:, 2],
            "f_dc_0": np.zeros(n), "f_dc_1": np.zeros(n), "f_dc_2": np.zeros(n), "opacity": np.log(a / (1 - a))}
    return FO.write_ply([(k, "float") for k in cols], {k: np.asarray(v, np.float32) for k, v in cols.items()}, n)


def _forest_scene(seed):
    rec, _ = _edge_scene(seed)
    keep = np.isfinite(rec["center"]).all(1) & np.isfinite(rec["rotation"]).all(1) & (rec["scale"].min(1) > 0)
    return rec[keep]


def _forest_engine(parts):
    from gaussiansplats3d_b200.engine import Engine
    N = _N()
    e = Engine(sum(len(p) for p in parts), dynamic_mode=True, ray_records=True, max_width=64, max_height=64)
    infos = e.upload_scenes([dict(format=N.GS_FILE_PLY, data=_ply(p)) for p in parts])
    e.build_splat_tree(8, 4, 1)
    n = sum(i["splat_count"] for i in infos)
    cc = e.read_buffer(N.GS_BUF_CENTERS_COLORS, np.uint32, n * 4).reshape(n, 4)
    return e, infos, cc[:, 1:4].copy().view(np.float32), (cc[:, 0] >> 24).astype(np.uint8)


class _Visible:
    """ray_oracle's view of a dynamic forest's records, a hidden scene's splats skipped (Raycaster.js:112-114)."""

    def __init__(self, rec, infos, visible):
        self.of = np.repeat(np.arange(len(infos)), [i["splat_count"] for i in infos])
        self.scene = RO.Scene(rec["center"], rec["scale"], rec["rotation"], rec["alpha"], dynamic=True)
        self.visible = visible

    def inputs(self, i, ellipsoid):
        c, s, F, Inv = self.scene.inputs(i, ellipsoid)
        return (c, s, F, Inv) if self.visible[int(self.of[i])] else (c, (0.0, 0.0, 0.0), F, Inv)


@pytest.mark.parametrize("ellipsoid", [False, True], ids=["sphere", "ellipsoid"])
def test_forest_mirrored_singular_hidden(monkeypatch, ellipsoid):
    """k_ray_*<true>: a dynamic mesh of four scenes, cast at with fromLocal mirrored, singular, identity (hidden) and identity; the
    axis-parallel rays and the capacities of cases 1 and 6 against forest_raycast."""
    N = _N()
    probe = Probe(monkeypatch)
    base = _forest_scene(4)
    dup = np.concatenate([base, base[:40]])                  # exact duplicates inside one scene
    e, infos, c, a = _forest_engine([dup, base, base, dup])
    try:
        rec = e.read_buffer(N.GS_BUF_RAY_RECORDS, N.RAY_RECORD_DTYPE, c.shape[0])
        roots = [RO.build_tree(c[i["splat_offset"]:i["splat_offset"] + i["splat_count"]], a[i["splat_offset"]:i["splat_offset"] + i["splat_count"]],
                               max_centers=4) for i in infos]
        fls = [FROM_LOCAL["mirrored"], FROM_LOCAL["singular"], RO.IDENTITY, RO.IDENTITY]
        vis = [True, True, False, True]
        scene = _Visible(rec, infos, vis)
        subtrees = [(r, i["splat_offset"], fl) for r, i, fl in zip(roots, infos, fls)]
        ortho, persp = _axis_rays(roots[3], roots[3].min, roots[3].max, 3)
        stats = collections.Counter()
        _cast_and_compare(e, lambda o, d: forest_raycast(subtrees, scene, o, d, ellipsoid=ellipsoid), ortho[::3] + persp[::2], ellipsoid, None, None, None,
                          stats, capacities=True, scene_visibility=vis, sub_tree_from_local=fls)
        counts = {**probe.take(), **stats}
        _require(counts, f"forest ({'ellipsoid' if ellipsoid else 'sphere'})", "d[a] == 0 skipped, node reached", "nan origin counts as inside",
                 "NaN-distance hits", "tie group cut by the capacity", "scale epsilon skip")
    finally:
        e.close()


# ---- the cull and the layout -----------------------------------------------------------------------------------------------------------
def _leaves_lv(boxes, per_leaf=1):
    """SplatTreeLeaves of hand-built leaves [(min, max)], each with its own `per_leaf` indexes; centres (max - min) * 0.5 + min."""
    from gaussiansplats3d_b200.splat_tree import SplatTreeLeaves
    mn = np.array([b[0] for b in boxes], np.float64).reshape(-1, 3)
    mx = np.array([b[1] for b in boxes], np.float64).reshape(-1, 3)
    with np.errstate(invalid="ignore"):
        ctr = (mx - mn) * 0.5 + mn
    m = len(boxes)
    offsets = (np.arange(m + 1) * per_leaf).astype(np.uint32)
    idx = np.arange(m * per_leaf, dtype=np.uint32)[::-1].copy()
    for i in range(m):
        idx[offsets[i]:offsets[i + 1]].sort()
    lv = SplatTreeLeaves(mn, mx, ctr, offsets, idx, np.zeros(m, np.int32))
    tuples = [(mn[i].tolist(), mx[i].tolist(), 0, idx[offsets[i]:offsets[i + 1]].tolist()) for i in range(m)]
    return lv, tuples


def _cull_terms(leaf, e):
    """Viewer.js:2013-2033 for one leaf, restated with tree_oracle's helpers: (dist, dot_xz, dot_yz, nodeSize, t)."""
    mn, mx = leaf[0], leaf[1]
    centre = [(mx[k] - mn[k]) * 0.5 + mn[k] for k in range(3)]
    t = TO._apply_matrix4(centre, e)
    dist = math.sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2])
    u = TO._normalized(t)
    yz, xz = TO._normalized([0.0, u[1], u[2]]), TO._normalized([u[0], 0.0, u[2]])
    d = [mx[k] - mn[k] for k in range(3)]
    return dist, 0.0 * xz[0] + 0.0 * xz[1] + -1.0 * xz[2], 0.0 * yz[0] + 0.0 * yz[1] + -1.0 * yz[2], math.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]), t


def _cull_counts(leaves, e, cx, cy, counts):
    tx, ty = cx - 0.6, cy - 0.6
    dists = []
    for li, leaf in enumerate(leaves):
        dist, dxz, dyz, ns, t = _cull_terms(leaf, e)
        counts["centre at the camera"] += all(v == 0.0 for v in t)
        counts["setX(0) is the zero vector"] += t[1] == 0.0 and t[2] == 0.0 and t[0] != 0.0
        counts["setY(0) is the zero vector"] += t[0] == 0.0 and t[2] == 0.0 and t[1] != 0.0
        for name, dot, thr in (("x", dxz, tx), ("y", dyz, ty)):
            if abs(dot - thr) <= 4 * math.ulp(thr):
                counts[f"{name} within 4 ulp of the threshold, {'out' if dot < thr else 'in'}"] += 1
        counts["one-splat leaf (ns == 0), dist > ns"] += ns == 0.0 and dist > 0
        counts["dist == ns"] += dist == ns and dist > 0
        counts["NaN distance"] += dist != dist
        dists.append((dist, li))
    by = collections.defaultdict(list)
    for dist, li in dists:
        by[struct.pack("<d", dist) if dist == dist else b"nan"].append(li)
    counts["equal keys in different 256-leaf tiles"] += sum(1 for v in by.values() if len({li // 256 for li in v}) > 1)
    return counts


def _sweep_boxes(cx, cy, rng):
    """Leaf centres swept across the x and y thresholds cos - 0.6 in view space (identity model view), a few ulp at a time; half of them
    one-splat leaves (min == max, nodeSize 0, centre exact), half small boxes."""
    boxes = []
    for axis, thr in ((0, cx - 0.6), (1, cy - 0.6)):
        phi = math.acos(thr)
        for R in np.geomspace(2.0, 60.0, 48):
            base = [0.0, 0.0, -R * math.cos(phi)]
            base[axis] = R * math.sin(phi) * (1 if rng.random() < 0.5 else -1)
            for k in range(-10, 11):
                c = list(base)
                for _ in range(abs(k)):
                    c[axis] = math.nextafter(c[axis], math.inf if k > 0 else -math.inf)
                if k % 2:
                    boxes.append((c, c))
                else:
                    h = 1e-3
                    boxes.append(([v - h for v in c], [v + h for v in c]))
    return boxes


def _special_boxes():
    boxes = [([0.0, 0.0, 0.0], [0.0, 0.0, 0.0]), ([-1.0, -1.0, -1.0], [1.0, 1.0, 1.0])]        # centres at the camera
    for p in ((3.0, 0.0, 0.0), (-5.0, 0.0, 0.0), (0.0, 4.0, 0.0), (0.0, -2.5, 0.0), (0.0, 0.0, -7.0), (0.0, 0.0, 6.0)):   # on the view axes
        boxes.append((list(p), list(p)))
        boxes.append(([v - 0.125 for v in p], [v + 0.125 for v in p]))
    # dist == nodeSize to the bit: a 2 x 4 x 4 box (diagonal 6) centred 6 from the camera along each axis
    for a in range(3):
        for sgn in (1.0, -1.0):
            ext = [1.0, 2.0, 2.0]
            ext = ext[-a:] + ext[:-a] if a else ext
            ctr = [0.0, 0.0, 0.0]
            ctr[a] = 6.0 * sgn
            boxes.append(([ctr[k] - ext[k] for k in range(3)], [ctr[k] + ext[k] for k in range(3)]))
    return boxes


def _tie_boxes():
    """More than 256 leaves with exactly equal distances, spread across k_tree_layout's 256-leaf tiles: sign flips of a few centres."""
    boxes = []
    for base in ((0.3, 0.7, -2.0), (1.1, -0.4, -3.5), (0.0, 0.9, -1.0)):
        for rep in range(40):
            for sx in (1, -1):
                for sy in (1, -1):
                    c = [sx * base[0], sy * base[1], base[2]]
                    boxes.append((c, c) if rep % 2 else ([v - 0.25 for v in c], [v + 0.25 for v in c]))
    return boxes


def _nonfinite_boxes():
    boxes = [([0.0, 0.0, -1.0], [math.inf, 1.0, 0.0]), ([-math.inf, 0.0, -2.0], [math.inf, 1.0, -1.0]), ([0.0, -math.inf, -3.0], [1.0, 1.0, -2.0])]
    for b in NANS:
        boxes.append(([_nan(b), 0.0, -1.0], [1.0, 1.0, 0.0]))
    boxes.append(([1.0, 1.0, -1.0], [1.0, 1.0, math.inf]))
    return boxes


CULL_FOVS = {"wide_x": (1080.0, 360.0, 50.0), "demo": (640.0, 360.0, 50.0)}   # wide_x: cos(fovX/2) - 0.6 < 0 < cos(fovY/2) - 0.6


@pytest.mark.parametrize("fov", list(CULL_FOVS))
def test_cull_edges_single_tree(monkeypatch, fov):
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.engine import Engine
    from gaussiansplats3d_b200.splat_tree import fov_cosines
    N = _N()
    cx, cy = fov_cosines(*CULL_FOVS[fov])
    rng = np.random.default_rng(5)
    boxes = _special_boxes() + _sweep_boxes(cx, cy, rng) + _tie_boxes() + _nonfinite_boxes()
    order = rng.permutation(len(boxes))                         # interleave the groups across the layout's tiles
    boxes = [boxes[i] for i in order]
    lv, leaves = _leaves_lv(boxes, 2)
    e = Engine(int(lv.offsets[-1]), ray_records=False, max_width=64, max_height=64)
    counts = collections.Counter()
    try:
        e.upload_splat_tree(lv)
        views = {"identity": RO.IDENTITY,
                 "camera": [float(v) for v in TM.invert(TM.camera_world_matrix([0.5, 0.25, 2.0], [0.5, 0.25, -5.0], [0.0, 1.0, 0.0]))]}
        for vname, mv in views.items():
            for gather_all in (False, True):
                want, wn = TO.gather_for_sort(leaves, mv, cx, cy, gather_all)
                n = e.gather_for_sort(mv, cx, cy, gather_all)
                assert n == wn, (vname, gather_all)
                got = e.read_buffer(N.GS_BUF_INDEXES_TO_SORT, np.uint32, n)
                assert np.array_equal(got, want), (vname, gather_all)
            _cull_counts(leaves, [float(v) for v in mv], cx, cy, counts)
        culled_ids = set(range(int(lv.offsets[-1]))) - set(TO.gather_for_sort(leaves, RO.IDENTITY, cx, cy)[0].tolist())
        counts["leaves culled"] += len(culled_ids) // 2
        names = ["centre at the camera", "setX(0) is the zero vector", "setY(0) is the zero vector", "one-splat leaf (ns == 0), dist > ns",
                 "dist == ns", "NaN distance", "equal keys in different 256-leaf tiles", "leaves culled"]
        names += [f"{a} within 4 ulp of the threshold, {s}" for a in "xy" for s in ("out", "in")]
        _require(counts, f"cull, single tree ({fov})", *names)
        for a in "xy":
            for s in ("out", "in"):
                assert counts[f"{a} within 4 ulp of the threshold, {s}"] >= 200, (a, s, counts)
    finally:
        e.close()


def test_cull_forest_mirrored_copies_and_nonfinite_centres():
    """gs_gather_for_sort_subtrees over a forest: four copies of one scene culled under mirror images of one model view (mirrored in view
    space, so every copy's leaf has the same distance to the bit: ties across sub-trees and layout tiles), a scene with a +inf centre
    (one leaf, infinite box) and one with -inf and +inf on one axis (a NaN leaf centre)."""
    from gaussiansplats3d_b200 import three_math as TM
    N = _N()
    rng = np.random.default_rng(8)
    base = _records(300)
    base["center"] = rng.normal(0, 1.5, (300, 3))
    base["scale"] = 0.05
    inf1 = _records(20)
    inf1["center"] = rng.normal(0, 1, (20, 3))
    inf1["center"][3, 0] = math.inf
    inf2 = inf1.copy()
    inf2["center"][5, 1] = -math.inf
    inf2["center"][6, 1] = math.inf
    parts = [base, base, base, base, inf1, inf2]
    e, infos, c, a = _forest_engine(parts)
    try:
        lv = e.read_splat_tree()
        per = forest_leaves(lv)
        assert lv.count > 256 and len(per) == len(parts)
        mirrors = [np.diag([sx, sy, 1.0, 1.0]).T.reshape(16) for sx, sy in ((1, 1), (-1, 1), (1, -1), (-1, -1))] + [np.eye(4).reshape(16)] * 2
        from gaussiansplats3d_b200.splat_tree import fov_cosines
        cx, cy = fov_cosines(640.0, 360.0, 50.0)
        counts = collections.Counter()
        for eye in ((0.0, 0.5, 6.0), (3.0, -1.0, 2.0), (0.2, 0.1, 0.3)):
            base_mv = TM.invert(TM.camera_world_matrix(list(eye), [0.0, 0.0, 0.0], [0.0, 1.0, 0.0]))
            views = [[float(v) for v in TM.multiply(list(m), base_mv)] for m in mirrors]
            for gather_all in (False, True):
                want, wn = forest_gather(list(zip(per, views)), cx, cy, gather_all)
                n = e.gather_for_sort_subtrees(views, cx, cy, gather_all)
                assert n == wn, (eye, gather_all)
                got = e.read_buffer(N.GS_BUF_INDEXES_TO_SORT, np.uint32, n)
                assert np.array_equal(got, want), (eye, gather_all)
            flat = [leaf for leaves in per for leaf in leaves]
            mv_of = [views[s] for s, leaves in enumerate(per) for _ in leaves]
            dists = [_cull_terms(leaf, mv)[0] for leaf, mv in zip(flat, mv_of)]
            counts["NaN distance"] += sum(d != d for d in dists)
            by = collections.defaultdict(set)
            for li, d in enumerate(dists):
                by[struct.pack("<d", d) if d == d else b"nan"].add(li // 256)
            counts["equal keys in different 256-leaf tiles"] += sum(len(v) > 1 for v in by.values())
        _require(counts, "cull, forest", "NaN distance", "equal keys in different 256-leaf tiles")
        assert counts["NaN distance"] >= 3            # a NaN leaf in every pose
    finally:
        e.close()
