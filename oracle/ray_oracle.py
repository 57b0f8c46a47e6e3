"""oracle/ray_oracle.py -- TEST INFRASTRUCTURE ONLY.  Imports nothing from the product package.

Scalar restatement (Python floats = JS numbers; Python never fuses a multiply-add) of the reference's raycaster:
  * Raycaster.setFromCameraAndScreenPosition / intersectSplatMesh / castRayAtSplatTreeNode  src/raycaster/Raycaster.js:13-165
  * Ray.intersectBox / intersectSphere                                                    src/raycaster/Ray.js:26-113
  * the splat inputs SplatMesh.getSplatCenter / getSplatScaleAndRotation / getSplatColor return  SplatMesh.js:1959-2012, SplatBuffer.js:221-305
  * the SplatTree recursion over EVERY node (the build is tree_oracle's; this module keeps the interior nodes the raycast needs).
three.js (r160) is not vendored: Matrix4.multiplyMatrices / invert / determinant / decompose / compose, Quaternion.setFromRotationMatrix and
Vector3.applyMatrix4 / transformDirection / unproject / normalize are restated from their published source and pinned by property in
tests/test_raycast_oracle.py (decompose(compose(p, q, s)) == (p, q, s), invert(M) M == I).

Hit order: ascending distance, then traversal position (the splat's offset in the depth-first concatenation of the leaves' index runs);
NaN distances last.  The reference's comparator leaves ties to V8's sort (a deliberate deviation)."""
from __future__ import annotations

import math
from decimal import Decimal, getcontext

import numpy as np

SCALE_EPSILON = 0.0000001          # Raycaster.js:97
BOX_EPSILON = 0.0001               # Ray.js:42

# Math.log10 of an alpha byte, correctly rounded (the one libm call of the path)
getcontext().prec = 60
LOG10_BYTE = [-math.inf] + [float(Decimal(b).log10()) for b in range(1, 256)]


# ---- three.js math ----------------------------------------------------------------------------------------------------------
def div(a, b):
    """a / b with IEEE semantics (JS): x / 0 is +-inf or NaN instead of a Python exception."""
    try:
        return a / b
    except ZeroDivisionError:
        if a != a or a == 0:
            return math.nan
        return math.copysign(math.inf, a) * math.copysign(1.0, b)


def sqrt(x):
    """Math.sqrt: NaN for negative arguments."""
    return math.sqrt(x) if x >= 0 or x != x else math.nan


def apply_matrix4(v, e):
    x, y, z = v
    w = div(1.0, e[3] * x + e[7] * y + e[11] * z + e[15])
    return [(e[0] * x + e[4] * y + e[8] * z + e[12]) * w, (e[1] * x + e[5] * y + e[9] * z + e[13]) * w, (e[2] * x + e[6] * y + e[10] * z + e[14]) * w]


def length(v):
    return sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])


def normalize(v):
    """divideScalar(length() || 1): NaN and 0 are falsy in JS (and truthy/falsy differently in Python, hence the explicit test)."""
    ln = length(v)
    s = 1.0 / (1.0 if (ln == 0.0 or ln != ln) else ln)
    return [v[0] * s, v[1] * s, v[2] * s]


def transform_direction(v, e):
    x, y, z = v
    return normalize([e[0] * x + e[4] * y + e[8] * z, e[1] * x + e[5] * y + e[9] * z, e[2] * x + e[6] * y + e[10] * z])


def multiply(a, b):
    """Matrix4.multiplyMatrices(a, b), column-major elements."""
    t = [0.0] * 16
    for c in range(4):
        for r in range(4):
            t[r + 4 * c] = a[r] * b[4 * c] + a[r + 4] * b[4 * c + 1] + a[r + 8] * b[4 * c + 2] + a[r + 12] * b[4 * c + 3]
    return t


def invert(te):
    n11, n21, n31, n41, n12, n22, n32, n42, n13, n23, n33, n43, n14, n24, n34, n44 = te
    t11 = n23 * n34 * n42 - n24 * n33 * n42 + n24 * n32 * n43 - n22 * n34 * n43 - n23 * n32 * n44 + n22 * n33 * n44
    t12 = n14 * n33 * n42 - n13 * n34 * n42 - n14 * n32 * n43 + n12 * n34 * n43 + n13 * n32 * n44 - n12 * n33 * n44
    t13 = n13 * n24 * n42 - n14 * n23 * n42 + n14 * n22 * n43 - n12 * n24 * n43 - n13 * n22 * n44 + n12 * n23 * n44
    t14 = n14 * n23 * n32 - n13 * n24 * n32 - n14 * n22 * n33 + n12 * n24 * n33 + n13 * n22 * n34 - n12 * n23 * n34
    det = n11 * t11 + n21 * t12 + n31 * t13 + n41 * t14
    if det == 0:
        return [0.0] * 16
    d = 1 / det
    return [
        t11 * d,
        (n24 * n33 * n41 - n23 * n34 * n41 - n24 * n31 * n43 + n21 * n34 * n43 + n23 * n31 * n44 - n21 * n33 * n44) * d,
        (n22 * n34 * n41 - n24 * n32 * n41 + n24 * n31 * n42 - n21 * n34 * n42 - n22 * n31 * n44 + n21 * n32 * n44) * d,
        (n23 * n32 * n41 - n22 * n33 * n41 - n23 * n31 * n42 + n21 * n33 * n42 + n22 * n31 * n43 - n21 * n32 * n43) * d,
        t12 * d,
        (n13 * n34 * n41 - n14 * n33 * n41 + n14 * n31 * n43 - n11 * n34 * n43 - n13 * n31 * n44 + n11 * n33 * n44) * d,
        (n14 * n32 * n41 - n12 * n34 * n41 - n14 * n31 * n42 + n11 * n34 * n42 + n12 * n31 * n44 - n11 * n32 * n44) * d,
        (n12 * n33 * n41 - n13 * n32 * n41 + n13 * n31 * n42 - n11 * n33 * n42 - n12 * n31 * n43 + n11 * n32 * n43) * d,
        t13 * d,
        (n14 * n23 * n41 - n13 * n24 * n41 - n14 * n21 * n43 + n11 * n24 * n43 + n13 * n21 * n44 - n11 * n23 * n44) * d,
        (n12 * n24 * n41 - n14 * n22 * n41 + n14 * n21 * n42 - n11 * n24 * n42 - n12 * n21 * n44 + n11 * n22 * n44) * d,
        (n13 * n22 * n41 - n12 * n23 * n41 - n13 * n21 * n42 + n11 * n23 * n42 + n12 * n21 * n43 - n11 * n22 * n43) * d,
        t14 * d,
        (n13 * n24 * n31 - n14 * n23 * n31 + n14 * n21 * n33 - n11 * n24 * n33 - n13 * n21 * n34 + n11 * n23 * n34) * d,
        (n14 * n22 * n31 - n12 * n24 * n31 - n14 * n21 * n32 + n11 * n24 * n32 + n12 * n21 * n34 - n11 * n22 * n34) * d,
        (n12 * n23 * n31 - n13 * n22 * n31 + n13 * n21 * n32 - n11 * n23 * n32 - n12 * n21 * n33 + n11 * n22 * n33) * d,
    ]


def determinant(te):
    n11, n12, n13, n14 = te[0], te[4], te[8], te[12]
    n21, n22, n23, n24 = te[1], te[5], te[9], te[13]
    n31, n32, n33, n34 = te[2], te[6], te[10], te[14]
    n41, n42, n43, n44 = te[3], te[7], te[11], te[15]
    return (n41 * (+n14 * n23 * n32 - n13 * n24 * n32 - n14 * n22 * n33 + n12 * n24 * n33 + n13 * n22 * n34 - n12 * n23 * n34)
            + n42 * (+n11 * n23 * n34 - n11 * n24 * n33 + n14 * n21 * n33 - n13 * n21 * n34 + n13 * n24 * n31 - n14 * n23 * n31)
            + n43 * (+n11 * n24 * n32 - n11 * n22 * n34 - n14 * n21 * n32 + n12 * n21 * n34 + n14 * n22 * n31 - n12 * n24 * n31)
            + n44 * (-n13 * n22 * n31 - n11 * n23 * n32 + n11 * n22 * n33 + n13 * n21 * n32 - n12 * n21 * n33 + n12 * n23 * n31))


def make_scale(x, y, z):
    return [x, 0.0, 0.0, 0.0, 0.0, y, 0.0, 0.0, 0.0, 0.0, z, 0.0, 0.0, 0.0, 0.0, 1.0]


def compose(p, q, s):
    """Matrix4.compose(position, quaternion (x, y, z, w), scale)."""
    x, y, z, w = q
    x2, y2, z2 = x + x, y + y, z + z
    xx, xy, xz = x * x2, x * y2, x * z2
    yy, yz, zz = y * y2, y * z2, z * z2
    wx, wy, wz = w * x2, w * y2, w * z2
    sx, sy, sz = s
    return [(1 - (yy + zz)) * sx, (xy + wz) * sx, (xz - wy) * sx, 0.0,
            (xy - wz) * sy, (1 - (xx + zz)) * sy, (yz + wx) * sy, 0.0,
            (xz + wy) * sz, (yz - wx) * sz, (1 - (xx + yy)) * sz, 0.0,
            p[0], p[1], p[2], 1.0]


def make_rotation_from_quaternion(q):
    return compose((0.0, 0.0, 0.0), q, (1.0, 1.0, 1.0))


def quaternion_from_rotation_matrix(te):
    m11, m12, m13 = te[0], te[4], te[8]
    m21, m22, m23 = te[1], te[5], te[9]
    m31, m32, m33 = te[2], te[6], te[10]
    trace = m11 + m22 + m33
    if trace > 0:
        s = div(0.5, sqrt(trace + 1.0))
        return [(m32 - m23) * s, (m13 - m31) * s, (m21 - m12) * s, div(0.25, s)]
    if m11 > m22 and m11 > m33:
        s = 2.0 * sqrt(1.0 + m11 - m22 - m33)
        return [0.25 * s, div(m12 + m21, s), div(m13 + m31, s), div(m32 - m23, s)]
    if m22 > m33:
        s = 2.0 * sqrt(1.0 + m22 - m11 - m33)
        return [div(m12 + m21, s), 0.25 * s, div(m23 + m32, s), div(m13 - m31, s)]
    s = 2.0 * sqrt(1.0 + m33 - m11 - m22)
    return [div(m13 + m31, s), div(m23 + m32, s), 0.25 * s, div(m21 - m12, s)]


def decompose(te):
    """-> position, quaternion (x, y, z, w), scale."""
    sx = length([te[0], te[1], te[2]])
    sy = length([te[4], te[5], te[6]])
    sz = length([te[8], te[9], te[10]])
    if determinant(te) < 0:
        sx = -sx
    m = list(te)
    ix, iy, iz = div(1.0, sx), div(1.0, sy), div(1.0, sz)
    for k in (0, 1, 2):
        m[k] *= ix
    for k in (4, 5, 6):
        m[k] *= iy
    for k in (8, 9, 10):
        m[k] *= iz
    return [te[12], te[13], te[14]], quaternion_from_rotation_matrix(m), [sx, sy, sz]


def unproject(v, projection, world):
    return apply_matrix4(apply_matrix4(v, invert(projection)), world)


# ---- ray set-up -------------------------------------------------------------------------------------------------------------
def ray_from_camera(projection, world, screen_xy, dims, orthographic=False, near=0.1, far=1000.0):
    """Raycaster.setFromCameraAndScreenPosition -> (origin, direction); screen position in render pixels, y down."""
    ndc_x = screen_xy[0] / dims[0] * 2.0 - 1.0
    ndc_y = (dims[1] - screen_xy[1]) / dims[1] * 2.0 - 1.0
    world = [float(v) for v in world]
    projection = [float(v) for v in projection]
    if orthographic:
        origin = unproject([ndc_x, ndc_y, (near + far) / (near - far)], projection, world)
        return origin, transform_direction([0.0, 0.0, -1.0], world)
    origin = [world[12], world[13], world[14]]
    t = unproject([ndc_x, ndc_y, 0.5], projection, world)
    return origin, normalize([t[0] - origin[0], t[1] - origin[1], t[2] - origin[2]])


# ---- tree with every node -----------------------------------------------------------------------------------------------------
class Node:
    __slots__ = ("min", "max", "children", "indexes")

    def __init__(self, mn, mx):
        self.min, self.max, self.children, self.indexes = list(mn), list(mx), [], None


def build_tree(centers_f32, alphas=None, min_alpha=1, max_depth=8, max_centers=1000):
    """SplatTree.processSplatMesh (SplatTree.js:132-278, 335-431): the root Node, or None without splats.  Same recursion as
    tree_oracle.build_leaves; leaves keep their de-duplicated, sorted indexes."""
    c = [[float(v) for v in row] for row in np.asarray(centers_f32, np.float32)]
    ids = [i for i in range(len(c)) if alphas is None or int(alphas[i]) >= min_alpha]
    if not ids:
        return None
    root = Node([min(c[i][k] for i in ids) for k in range(3)], [max(c[i][k] for i in ids) for k in range(3)])
    added = set()

    def process(node, idx, depth):
        if len(idx) < max_centers or depth > max_depth:
            fresh = [i for i in idx if i not in added]
            added.update(fresh)
            node.indexes = sorted(fresh)
            return
        half = [(node.max[k] - node.min[k]) * 0.5 for k in range(3)]
        ctr = [node.min[k] + half[k] for k in range(3)]
        for hx, hy, hz in ((0, 1, 0), (1, 1, 0), (1, 1, 1), (0, 1, 1), (0, 0, 0), (1, 0, 0), (1, 0, 1), (0, 0, 1)):
            h = (hx, hy, hz)
            bmin = [ctr[k] if h[k] else ctr[k] - half[k] for k in range(3)]
            bmax = [ctr[k] + half[k] if h[k] else ctr[k] for k in range(3)]
            child = Node(bmin, bmax)
            node.children.append(child)
            sub = [i for i in idx if all(bmin[k] <= c[i][k] <= bmax[k] for k in range(3))]
            process(child, sub, depth + 1)

    process(root, ids, 0)
    return root


def tree_arrays(root):
    """The tree in the engine's upload layout: leaves with indexes (nodesWithIndexes order) and every node, depth first.
    -> dict(leaf_min, leaf_max, leaf_center, offsets, indexes, node_min, node_max, node_parent, leaf_node)."""
    nmin, nmax, parent, leaves, leaf_node = [], [], [], [], []

    def visit(n, p):
        me = len(parent)
        nmin.append(n.min); nmax.append(n.max); parent.append(p)
        if n.indexes:
            leaves.append(n); leaf_node.append(me)
        for ch in n.children:
            visit(ch, me)

    if root is not None:
        visit(root, -1)
    m = len(leaves)
    offsets = np.zeros(m + 1, np.uint32)
    if m:
        offsets[1:] = np.cumsum([len(n.indexes) for n in leaves])
    lmin = np.array([n.min for n in leaves], np.float64).reshape(m, 3)
    lmax = np.array([n.max for n in leaves], np.float64).reshape(m, 3)
    return dict(leaf_min=lmin, leaf_max=lmax, leaf_center=(lmax - lmin) * 0.5 + lmin, offsets=offsets,
                indexes=np.array([i for n in leaves for i in n.indexes], np.uint32),
                node_min=np.array(nmin, np.float64).reshape(-1, 3), node_max=np.array(nmax, np.float64).reshape(-1, 3),
                node_parent=np.array(parent, np.int32), leaf_node=np.array(leaf_node, np.uint32))


# ---- the tests of Ray.js -------------------------------------------------------------------------------------------------------
def box_contains(mn, mx, p, eps=BOX_EPSILON):
    return not (p[0] < mn[0] - eps or p[0] > mx[0] + eps or p[1] < mn[1] - eps or p[1] > mx[1] + eps or p[2] < mn[2] - eps or p[2] > mx[2] + eps)


def intersect_box(o, d, mn, mx):
    if box_contains(mn, mx, o):
        return True
    for i in range(3):
        if d[i] == 0.0:
            continue
        extreme = mx if d[i] < 0 else mn
        sign = 1.0 if d[i] > 0 else (-1.0 if d[i] < 0 else math.nan)     # Math.sign
        multiplier = -sign
        to_side = extreme[i] - o[i]
        if to_side * multiplier < 0:
            i1, i2 = (i + 1) % 3, (i + 2) % 3
            p = [0.0, 0.0, 0.0]
            p[i] = extreme[i]
            p[i1] = d[i1] / d[i] * to_side + o[i1]
            p[i2] = d[i2] / d[i] * to_side + o[i2]
            if box_contains(mn, mx, p):
                return True
    return False


def intersect_sphere(o, d, center, radius):
    """-> (hit origin, normal, t) or None."""
    v = [center[0] - o[0], center[1] - o[1], center[2] - o[2]]
    tca = v[0] * d[0] + v[1] * d[1] + v[2] * d[2]
    diff = (v[0] * v[0] + v[1] * v[1] + v[2] * v[2]) - tca * tca
    r2 = radius * radius
    if diff > r2:
        return None
    thc = sqrt(r2 - diff)
    t0, t1 = tca - thc, tca + thc
    if t1 < 0:
        return None
    t = t1 if t0 < 0 else t0
    h = [o[0] + d[0] * t, o[1] + d[1] * t, o[2] + d[2] * t]
    return h, normalize([h[0] - center[0], h[1] - center[1], h[2] - center[2]]), t


# ---- splat inputs ----------------------------------------------------------------------------------------------------------------
IDENTITY = [1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 1.0]


def splat_inputs(center, scale, rotation_xyzw, dynamic, transform16=None, want_rotation=True):
    """getSplatCenter / getSplatScaleAndRotation of one splat: (centre, scale, rotation x y z w).  A static mesh applies scene.transform
    (a Matrix4 even when identity) to the centre, and takes scale and rotation from decompose(makeScale(s) R(q) T)."""
    c = [float(v) for v in center]
    s = [float(v) for v in scale]
    q = [float(v) for v in rotation_xyzw]
    if dynamic:
        return c, s, q
    T = IDENTITY if transform16 is None else [float(v) for v in transform16]
    c = apply_matrix4(c, T)
    M = multiply(multiply(make_scale(*s), make_rotation_from_quaternion(q)), T)
    _, q2, s2 = decompose(M)
    return c, s2, (q2 if want_rotation else q)


class Scene:
    """One scene's records as the raycast reads them: centre (f64), stored scale and rotation (x, y, z, w), alpha byte."""

    def __init__(self, centers64, scales32, rotations_xyzw32, alphas, *, dynamic=False, transform16=None):
        self.c = np.asarray(centers64, np.float64)
        self.s = np.asarray(scales32, np.float32)
        self.q = np.asarray(rotations_xyzw32, np.float32)
        self.a = np.asarray(alphas, np.uint8)
        self.dynamic, self.transform16 = dynamic, transform16
        self._cache: dict = {}

    def inputs(self, i, ellipsoid):
        key = (i, ellipsoid)
        if key not in self._cache:
            c, s, q = splat_inputs(self.c[i], self.s[i], self.q[i], self.dynamic, self.transform16, want_rotation=ellipsoid)
            F = Inv = None
            if ellipsoid:
                u = LOG10_BYTE[int(self.a[i])] * 2.0
                F = multiply(multiply(make_scale(u, u, u), make_rotation_from_quaternion(q)), make_scale(*s))
                Inv = invert(F)
            self._cache[key] = (c, s, F, Inv)
        return self._cache[key]


def splat_hit(scene, i, o, d, ellipsoid):
    """castRayAtSplatTreeNode's per-splat body (Raycaster.js:111-154) -> (local origin, local normal) or None."""
    c, s, F, Inv = scene.inputs(i, ellipsoid)
    if s[0] <= SCALE_EPSILON or s[1] <= SCALE_EPSILON or s[2] <= SCALE_EPSILON:
        return None
    if not ellipsoid:
        r = intersect_sphere(o, d, c, (s[0] + s[1] + s[2]) / 3.0)
        return None if r is None else (r[0], r[1])
    to = apply_matrix4([o[0] - c[0], o[1] - c[1], o[2] - c[2]], Inv)
    td = apply_matrix4([o[0] + d[0] - c[0], o[1] + d[1] - c[1], o[2] + d[2] - c[2]], Inv)
    td = normalize([td[0] - to[0], td[1] - to[1], td[2] - to[2]])
    r = intersect_sphere(to, td, [0.0, 0.0, 0.0], 1.0)
    if r is None:
        return None
    h = apply_matrix4(r[0], F)
    return [h[0] + c[0], h[1] + c[1], h[2] + c[2]], r[1]


def reached_leaves(root, o, d):
    """Depth-first leaves (with indexes) whose box and every ancestor's box pass intersectBox, in traversal order."""
    out = []

    def rec(n):
        if not intersect_box(o, d, n.min, n.max):
            return
        if n.indexes:
            out.append(n)
        for ch in n.children:
            rec(ch)

    if root is not None:
        rec(root)
    return out


def intersect_splat_mesh(root, scene, origin, direction, from_local16, *, ellipsoid=False, scene_visible=True):
    """Raycaster.intersectSplatMesh -> hits [(distance, position, splat index, world origin, world normal)] in the engine's order."""
    fl = [float(v) for v in from_local16]
    to_local = invert(fl)
    lo = apply_matrix4(origin, to_local)
    ld = apply_matrix4([origin[0] + direction[0], origin[1] + direction[1], origin[2] + direction[2]], to_local)
    ld = normalize([ld[0] - lo[0], ld[1] - lo[1], ld[2] - lo[2]])
    hits = []
    if not scene_visible:
        return hits
    pos_of = {}
    pos = 0

    def number(n):
        nonlocal pos
        if n.indexes:
            pos_of[id(n)] = pos
            pos += len(n.indexes)
        for ch in n.children:
            number(ch)

    if root is not None:
        number(root)
    for leaf in reached_leaves(root, lo, ld):
        base = pos_of[id(leaf)]
        for k, i in enumerate(leaf.indexes):
            h = splat_hit(scene, i, lo, ld, ellipsoid)
            if h is None:
                continue
            wo = apply_matrix4(h[0], fl)
            wn = normalize(apply_matrix4(h[1], fl))
            dist = length([wo[0] - origin[0], wo[1] - origin[1], wo[2] - origin[2]])
            hits.append((dist, base + k, i, wo, wn))
    hits.sort(key=lambda h: (h[0] != h[0], 0.0 if h[0] != h[0] else h[0], h[1]))
    return hits
