"""The slice of three.js (r160) math the hot path depends on, restated in float64 NumPy.

three.js is a peer dependency of the reference (package.json:69-71) and is NOT vendored under /root/reference, so
these follow three's documented conventions (column-major `elements`, right-handed, camera looks down -Z) and
algorithms as published in three@0.160.0 -- PARITY UNPINNED against the real library (no JS engine here).
Call sites in the reference: Viewer.js:338 (PerspectiveCamera fov 50, near 0.1, far 1000), :341-343 (position / up /
lookAt), :1888-1891 (mvp = proj * inv(camera.matrixWorld) * mesh.matrixWorld), :662-673 (focal lengths).
"""
from __future__ import annotations

import math

import numpy as np


def identity() -> np.ndarray:
    return np.eye(4, dtype=np.float64).T.reshape(16).copy()


def to_mat(e) -> np.ndarray:
    """column-major elements[16] -> 4x4 ndarray (row, col)."""
    return np.asarray(e, np.float64).reshape(4, 4).T


def to_elements(m) -> np.ndarray:
    return np.asarray(m, np.float64).T.reshape(16).copy()


def multiply(a, b) -> np.ndarray:
    """Matrix4.multiplyMatrices(a, b) = a * b."""
    return to_elements(to_mat(a) @ to_mat(b))


def invert(e) -> np.ndarray:
    """Matrix4.invert(): cofactor expansion (three evaluates the same closed form; a singular matrix gives zeros)."""
    n11, n21, n31, n41, n12, n22, n32, n42, n13, n23, n33, n43, n14, n24, n34, n44 = (float(v) for v in np.asarray(e, np.float64).reshape(16))
    t11 = n23 * n34 * n42 - n24 * n33 * n42 + n24 * n32 * n43 - n22 * n34 * n43 - n23 * n32 * n44 + n22 * n33 * n44
    t12 = n14 * n33 * n42 - n13 * n34 * n42 - n14 * n32 * n43 + n12 * n34 * n43 + n13 * n32 * n44 - n12 * n33 * n44
    t13 = n13 * n24 * n42 - n14 * n23 * n42 + n14 * n22 * n43 - n12 * n24 * n43 - n13 * n22 * n44 + n12 * n23 * n44
    t14 = n14 * n23 * n32 - n13 * n24 * n32 - n14 * n22 * n33 + n12 * n24 * n33 + n13 * n22 * n34 - n12 * n23 * n34
    det = n11 * t11 + n21 * t12 + n31 * t13 + n41 * t14
    if det == 0:
        return np.zeros(16)
    d = 1.0 / det
    out = np.empty(16)
    out[0] = t11 * d
    out[1] = (n24 * n33 * n41 - n23 * n34 * n41 - n24 * n31 * n43 + n21 * n34 * n43 + n23 * n31 * n44 - n21 * n33 * n44) * d
    out[2] = (n22 * n34 * n41 - n24 * n32 * n41 + n24 * n31 * n42 - n21 * n34 * n42 - n22 * n31 * n44 + n21 * n32 * n44) * d
    out[3] = (n23 * n32 * n41 - n22 * n33 * n41 - n23 * n31 * n42 + n21 * n33 * n42 + n22 * n31 * n43 - n21 * n32 * n43) * d
    out[4] = t12 * d
    out[5] = (n13 * n34 * n41 - n14 * n33 * n41 + n14 * n31 * n43 - n11 * n34 * n43 - n13 * n31 * n44 + n11 * n33 * n44) * d
    out[6] = (n14 * n32 * n41 - n12 * n34 * n41 - n14 * n31 * n42 + n11 * n34 * n42 + n12 * n31 * n44 - n11 * n32 * n44) * d
    out[7] = (n12 * n33 * n41 - n13 * n32 * n41 + n13 * n31 * n42 - n11 * n33 * n42 - n12 * n31 * n43 + n11 * n32 * n43) * d
    out[8] = t13 * d
    out[9] = (n14 * n23 * n41 - n13 * n24 * n41 - n14 * n21 * n43 + n11 * n24 * n43 + n13 * n21 * n44 - n11 * n23 * n44) * d
    out[10] = (n12 * n24 * n41 - n14 * n22 * n41 + n14 * n21 * n42 - n11 * n24 * n42 - n12 * n21 * n44 + n11 * n22 * n44) * d
    out[11] = (n13 * n22 * n41 - n12 * n23 * n41 - n13 * n21 * n42 + n11 * n23 * n42 + n12 * n21 * n43 - n11 * n22 * n43) * d
    out[12] = t14 * d
    out[13] = (n13 * n24 * n31 - n14 * n23 * n31 + n14 * n21 * n33 - n11 * n24 * n33 - n13 * n21 * n34 + n11 * n23 * n34) * d
    out[14] = (n14 * n22 * n31 - n12 * n24 * n31 - n14 * n21 * n32 + n11 * n24 * n32 + n12 * n21 * n34 - n11 * n22 * n34) * d
    out[15] = (n12 * n23 * n31 - n13 * n22 * n31 + n13 * n21 * n32 - n11 * n23 * n32 - n12 * n21 * n33 + n11 * n22 * n33) * d
    return out


def make_perspective(fov_deg: float, aspect: float, near: float, far: float, zoom: float = 1.0) -> np.ndarray:
    """PerspectiveCamera.updateProjectionMatrix + Matrix4.makePerspective (WebGL clip space)."""
    top = near * np.tan(np.deg2rad(0.5 * fov_deg)) / zoom
    height = 2.0 * top
    width = aspect * height
    left = -0.5 * width
    right, bottom = left + width, top - height
    e = np.zeros(16)
    e[0] = 2 * near / (right - left)
    e[5] = 2 * near / (top - bottom)
    e[8] = (right + left) / (right - left)
    e[9] = (top + bottom) / (top - bottom)
    e[10] = -(far + near) / (far - near)
    e[11] = -1.0
    e[14] = -2 * far * near / (far - near)
    return e


def make_orthographic(left, right, top, bottom, near, far, zoom: float = 1.0) -> np.ndarray:
    """OrthographicCamera.updateProjectionMatrix + Matrix4.makeOrthographic."""
    dx, dy = (right - left) / (2 * zoom), (top - bottom) / (2 * zoom)
    cx, cy = (right + left) / 2, (top + bottom) / 2
    left, right, top, bottom = cx - dx, cx + dx, cy + dy, cy - dy
    w, h, p = 1.0 / (right - left), 1.0 / (top - bottom), 1.0 / (far - near)
    e = np.zeros(16)
    e[0], e[5], e[10] = 2 * w, 2 * h, -2 * p
    e[12], e[13], e[14], e[15] = -(right + left) * w, -(top + bottom) * h, -(far + near) * p, 1.0
    return e


def camera_world_matrix(position, target, up) -> np.ndarray:
    """Object3D.lookAt for a camera (Matrix4.lookAt(eye=position, target, up)) composed with the position."""
    eye, tgt, upv = (np.asarray(v, np.float64) for v in (position, target, up))
    z = eye - tgt
    if np.dot(z, z) == 0:
        z = np.array([0.0, 0.0, 1.0])
    z = z / np.linalg.norm(z)
    x = np.cross(upv, z)
    if np.dot(x, x) == 0:  # up parallel to view direction: three nudges z
        z = z + np.array([0.0001, 0.0, 0.0]) if abs(upv[2]) == 1 else z + np.array([0.0, 0.0, 0.0001])
        z = z / np.linalg.norm(z)
        x = np.cross(upv, z)
    x = x / np.linalg.norm(x)
    y = np.cross(z, x)
    m = np.eye(4)
    m[:3, 0], m[:3, 1], m[:3, 2], m[:3, 3] = x, y, z, eye
    return to_elements(m)


def compose(position, quaternion_xyzw, scale) -> np.ndarray:
    """Matrix4.compose."""
    x, y, z, w = (float(v) for v in quaternion_xyzw)
    x2, y2, z2 = x + x, y + y, z + z
    xx, xy, xz, yy, yz, zz, wx, wy, wz = x * x2, x * y2, x * z2, y * y2, y * z2, z * z2, w * x2, w * y2, w * z2
    sx, sy, sz = (float(v) for v in scale)
    e = np.zeros(16)
    e[0], e[1], e[2] = (1 - (yy + zz)) * sx, (xy + wz) * sx, (xz - wy) * sx
    e[4], e[5], e[6] = (xy - wz) * sy, (1 - (xx + zz)) * sy, (yz + wx) * sy
    e[8], e[9], e[10] = (xz + wy) * sz, (yz - wx) * sz, (1 - (xx + yy)) * sz
    e[12], e[13], e[14], e[15] = float(position[0]), float(position[1]), float(position[2]), 1.0
    return e


def rotate_about_axis(v, axis, angle_rad) -> np.ndarray:
    """Vector3.applyAxisAngle (Rodrigues)."""
    v, k = np.asarray(v, np.float64), np.asarray(axis, np.float64)
    k = k / np.linalg.norm(k)
    return v * np.cos(angle_rad) + np.cross(k, v) * np.sin(angle_rad) + k * np.dot(k, v) * (1 - np.cos(angle_rad))


class PerspectiveCamera:
    """Just enough of THREE.PerspectiveCamera: position/up/lookAt -> matrixWorld, projectionMatrix."""

    isOrthographicCamera = False

    def __init__(self, fov=50.0, aspect=1.0, near=0.1, far=1000.0):
        self.fov, self.aspect, self.near, self.far, self.zoom = fov, aspect, near, far, 1.0
        self.position = np.zeros(3)
        self.up = np.array([0.0, 1.0, 0.0])
        self.target = np.array([0.0, 0.0, -1.0])
        self.update()

    def look_at(self, target):
        self.target = np.asarray(target, np.float64)
        self.update()

    def update(self):
        self.projectionMatrix = make_perspective(self.fov, self.aspect, self.near, self.far, self.zoom)
        self.matrixWorld = camera_world_matrix(self.position, self.target, self.up)
        self.matrixWorldInverse = invert(self.matrixWorld)


# three.js's per-element arithmetic, in its operation order (Python floats are JS numbers and never fuse): what SplatBuffer.getSplatCenter
# and getSplatScaleAndRotation compute for one splat (SplatBuffer.js:221-290).
def _div(a: float, b: float) -> float:
    if b == 0.0:
        return float("nan") if a != a or a == 0.0 else math.copysign(math.inf, a) * math.copysign(1.0, b)
    return a / b


def _sqrt(x: float) -> float:
    return math.sqrt(x) if x >= 0 or x != x else math.nan


def apply_matrix4(v, e) -> list:
    """Vector3.applyMatrix4: the divide by w included."""
    x, y, z = (float(c) for c in v)
    e = [float(c) for c in np.asarray(e, np.float64).reshape(16)]
    w = _div(1.0, e[3] * x + e[7] * y + e[11] * z + e[15])
    return [(e[0] * x + e[4] * y + e[8] * z + e[12]) * w, (e[1] * x + e[5] * y + e[9] * z + e[13]) * w, (e[2] * x + e[6] * y + e[10] * z + e[14]) * w]


def multiply_elements(a, b) -> list:
    """Matrix4.multiplyMatrices(a, b) element by element, sums left to right (multiply() above goes through a BLAS product)."""
    a = [float(c) for c in np.asarray(a, np.float64).reshape(16)]
    b = [float(c) for c in np.asarray(b, np.float64).reshape(16)]
    return [a[r] * b[4 * c] + a[r + 4] * b[4 * c + 1] + a[r + 8] * b[4 * c + 2] + a[r + 12] * b[4 * c + 3] for c in range(4) for r in range(4)]


def make_scale(x: float, y: float, z: float) -> list:
    return [float(x), 0.0, 0.0, 0.0, 0.0, float(y), 0.0, 0.0, 0.0, 0.0, float(z), 0.0, 0.0, 0.0, 0.0, 1.0]


def _determinant(te) -> float:
    n11, n12, n13, n14 = te[0], te[4], te[8], te[12]
    n21, n22, n23, n24 = te[1], te[5], te[9], te[13]
    n31, n32, n33, n34 = te[2], te[6], te[10], te[14]
    n41, n42, n43, n44 = te[3], te[7], te[11], te[15]
    return (n41 * (+n14 * n23 * n32 - n13 * n24 * n32 - n14 * n22 * n33 + n12 * n24 * n33 + n13 * n22 * n34 - n12 * n23 * n34)
            + n42 * (+n11 * n23 * n34 - n11 * n24 * n33 + n14 * n21 * n33 - n13 * n21 * n34 + n13 * n24 * n31 - n14 * n23 * n31)
            + n43 * (+n11 * n24 * n32 - n11 * n22 * n34 - n14 * n21 * n32 + n12 * n21 * n34 + n14 * n22 * n31 - n12 * n24 * n31)
            + n44 * (-n13 * n22 * n31 - n11 * n23 * n32 + n11 * n22 * n33 + n13 * n21 * n32 - n12 * n21 * n33 + n12 * n23 * n31))


def _quaternion_from_rotation_matrix(te) -> list:
    """Quaternion.setFromRotationMatrix -> (x, y, z, w)."""
    m11, m12, m13, m21, m22, m23, m31, m32, m33 = te[0], te[4], te[8], te[1], te[5], te[9], te[2], te[6], te[10]
    trace = m11 + m22 + m33
    if trace > 0:
        s = _div(0.5, _sqrt(trace + 1.0))
        return [(m32 - m23) * s, (m13 - m31) * s, (m21 - m12) * s, _div(0.25, s)]
    if m11 > m22 and m11 > m33:
        s = 2.0 * _sqrt(1.0 + m11 - m22 - m33)
        return [0.25 * s, _div(m12 + m21, s), _div(m13 + m31, s), _div(m32 - m23, s)]
    if m22 > m33:
        s = 2.0 * _sqrt(1.0 + m22 - m11 - m33)
        return [_div(m12 + m21, s), 0.25 * s, _div(m23 + m32, s), _div(m13 - m31, s)]
    s = 2.0 * _sqrt(1.0 + m33 - m11 - m22)
    return [_div(m13 + m31, s), _div(m23 + m32, s), 0.25 * s, _div(m21 - m12, s)]


def decompose(te) -> tuple[list, list, list]:
    """Matrix4.decompose -> position, quaternion (x, y, z, w), scale."""
    te = [float(c) for c in np.asarray(te, np.float64).reshape(16)]
    sx = _sqrt(te[0] * te[0] + te[1] * te[1] + te[2] * te[2])
    sy = _sqrt(te[4] * te[4] + te[5] * te[5] + te[6] * te[6])
    sz = _sqrt(te[8] * te[8] + te[9] * te[9] + te[10] * te[10])
    if _determinant(te) < 0:
        sx = -sx
    m = list(te)
    for ks, inv in (((0, 1, 2), _div(1.0, sx)), ((4, 5, 6), _div(1.0, sy)), ((8, 9, 10), _div(1.0, sz))):
        for k in ks:
            m[k] *= inv
    return [te[12], te[13], te[14]], _quaternion_from_rotation_matrix(m), [sx, sy, sz]
