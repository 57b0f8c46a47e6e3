"""Mirror of the reference's raycaster (src/raycaster/Ray.js, Hit.js, Raycaster.js): the ray is set up on the host in f64 with three.js
(r160) operation order, and intersectSplatMesh runs on the GPU (Engine.raycast -> gs_raycast, csrc/ray_kernels.cuh).

The engine must hold ray records (Engine(..., ray_records=True)) and the SplatTree's leaves and nodes; Viewer(raycast=True) sets all of
that up for every scene kind."""
from __future__ import annotations

import math

import numpy as np

from . import three_math as TM


def _apply_matrix4(v, e):
    """Vector3.applyMatrix4 (column-major elements e)."""
    x, y, z = (float(c) for c in v)
    e = [float(c) for c in e]
    w = 1.0 / (e[3] * x + e[7] * y + e[11] * z + e[15])
    return [(e[0] * x + e[4] * y + e[8] * z + e[12]) * w, (e[1] * x + e[5] * y + e[9] * z + e[13]) * w, (e[2] * x + e[6] * y + e[10] * z + e[14]) * w]


def _normalize(v):
    """Vector3.normalize = divideScalar(length() || 1); NaN and 0 are both falsy in JS."""
    ln = math.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])
    s = 1.0 / (1.0 if (ln == 0.0 or ln != ln) else ln)
    return [v[0] * s, v[1] * s, v[2] * s]


class Ray:
    def __init__(self, origin=(0.0, 0.0, 0.0), direction=(0.0, 0.0, 0.0)):
        self.origin = [float(c) for c in origin]
        self.direction = _normalize([float(c) for c in direction])


class Hit:
    def __init__(self, origin=(0.0, 0.0, 0.0), normal=(0.0, 0.0, 0.0), distance: float = 0.0, splatIndex: int = 0):  # noqa: N803
        self.origin = np.array(origin, np.float64)
        self.normal = np.array(normal, np.float64)
        self.distance = float(distance)
        self.splatIndex = int(splatIndex)


class Raycaster:
    def __init__(self, origin=(0.0, 0.0, 0.0), direction=(0.0, 0.0, 0.0), raycastAgainstTrueSplatEllipsoid: bool = False):  # noqa: N803
        self.ray = Ray(origin, direction)
        self.raycastAgainstTrueSplatEllipsoid = raycastAgainstTrueSplatEllipsoid

    def setFromCameraAndScreenPosition(self, camera, screenPosition, screenDimensions) -> None:  # noqa: N802,N803  Raycaster.js:13-34
        """screenPosition: render-dimension pixels, y down.  camera: projectionMatrix, matrixWorld (and near / far when orthographic)."""
        ndc_x = float(screenPosition[0]) / float(screenDimensions[0]) * 2.0 - 1.0
        ndc_y = (float(screenDimensions[1]) - float(screenPosition[1])) / float(screenDimensions[1]) * 2.0 - 1.0
        proj_inv = TM.invert(camera.projectionMatrix)
        world = np.asarray(camera.matrixWorld, np.float64).reshape(16)
        if getattr(camera, "isOrthographicCamera", False):
            p = [ndc_x, ndc_y, (camera.near + camera.far) / (camera.near - camera.far)]
            self.ray.origin = _apply_matrix4(_apply_matrix4(p, proj_inv), world)          # Vector3.unproject
            x, y, z, e = 0.0, 0.0, -1.0, [float(c) for c in world]                       # Vector3.transformDirection
            self.ray.direction = _normalize([e[0] * x + e[4] * y + e[8] * z, e[1] * x + e[5] * y + e[9] * z, e[2] * x + e[6] * y + e[10] * z])
        else:
            self.ray.origin = [float(world[12]), float(world[13]), float(world[14])]     # setFromMatrixPosition
            t = _apply_matrix4(_apply_matrix4([ndc_x, ndc_y, 0.5], proj_inv), world)
            self.ray.direction = _normalize([t[0] - self.ray.origin[0], t[1] - self.ray.origin[1], t[2] - self.ray.origin[2]])
        self.camera = camera

    def intersectSplatMesh(self, splatMesh, outHits: list | None = None, capacity: int | None = None) -> list:  # noqa: N802,N803
        """Raycaster.js:36-85 on the GPU: every hit, nearest first (or the nearest `capacity`).  splatMesh: a viewer.SplatMesh whose
        engine holds ray records and the tree's nodes; its matrixWorld [* scene transform when dynamic] maps local to world."""
        if outHits is None:
            outHits = []
        engine = splatMesh.engine
        from_local = np.asarray(splatMesh.matrixWorld, np.float64).reshape(16)
        if splatMesh.dynamicMode:
            from_local = TM.multiply(from_local, splatMesh.getSceneTransform(0))
        cap = 64 if capacity is None else capacity
        hits, total = engine.raycast(self.ray.origin, self.ray.direction, from_local, ellipsoid=self.raycastAgainstTrueSplatEllipsoid,
                                     scene_visible=splatMesh.sceneVisible, capacity=cap)
        if capacity is None and total > cap:
            hits, total = engine.raycast(self.ray.origin, self.ray.direction, from_local, ellipsoid=self.raycastAgainstTrueSplatEllipsoid,
                                         scene_visible=splatMesh.sceneVisible, capacity=total)
        outHits.extend(Hit(h["origin"], h["normal"], h["distance"], h["splat_index"]) for h in hits)
        return outHits


def ray_records_from_raw(raw_scene) -> np.ndarray:
    """gs_ray_record per splat of a RawScene (host-packed scenes): its f32 centre as a JS number, scale, rotation (x, y, z, w), alpha."""
    from ._native import RAY_RECORD_DTYPE
    r = np.zeros(raw_scene.count, RAY_RECORD_DTYPE)
    r["center"] = np.asarray(raw_scene.centers, np.float32).astype(np.float64)
    r["scale"] = np.asarray(raw_scene.scales, np.float32)
    r["rotation"] = np.asarray(raw_scene.rotations, np.float32)
    r["alpha"] = np.asarray(raw_scene.colors, np.uint8)[:, 3]
    return r


def record_centers_f32(records: np.ndarray, transform16=None) -> np.ndarray:
    """The centres the SplatTree is built from (SplatTree.js:343-348): getSplatCenter's f64 centre, with a static mesh's scene transform
    applied in Vector3.applyMatrix4's order, stored into a Float32Array."""
    c = np.asarray(records["center"], np.float64)
    e = np.eye(4).reshape(16) if transform16 is None else np.asarray(transform16, np.float64).reshape(16)
    x, y, z = c[:, 0], c[:, 1], c[:, 2]
    with np.errstate(all="ignore"):
        w = 1.0 / (((e[3] * x + e[7] * y) + e[11] * z) + e[15])
        out = np.stack([(((e[0] * x + e[4] * y) + e[8] * z) + e[12]) * w, (((e[1] * x + e[5] * y) + e[9] * z) + e[13]) * w,
                        (((e[2] * x + e[6] * y) + e[10] * z) + e[14]) * w], 1)
        return out.astype(np.float32)
