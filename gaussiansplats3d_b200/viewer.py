"""Host-side mirror of the slice of the reference's Viewer / SplatMesh that drives the hot path.

    SplatMesh.build(...)                  src/splatmesh/SplatMesh.js:306-405    -> SplatMesh.build
    SplatMesh.getIntegerCenters/Float...  :1912-1948                            -> SplatMesh.getIntegerCenters / getFloatCenters
    SplatMesh.updateRenderIndexes         :1228-1235                            -> SplatMesh.updateRenderIndexes
    SplatMesh.updateUniforms              :1248-1280                            -> SplatMesh.updateUniforms
    Viewer.runSplatSort                   src/Viewer.js:1833-1964               -> Viewer.runSplatSort
    Viewer.updateSplatMesh                :651-677                              -> Viewer.updateSplatMesh
    Viewer.render                         :1599-1623                            -> Viewer.render
    Viewer.update                         :1625-1644                            -> Viewer.update
    WebXRMode                             src/webxr/WebXRMode.js                -> WebXRMode, Viewer(webXRMode=...), render/frame(xrCameras=...)

Only the arithmetic-free orchestration lives here (matrix set-up in float64 like three.js, message passing, option
bag).  Sorting and rasterisation run in libgsplat_b200.so through Engine / SortWorker.  Everything the reference does
around the path (loading UI, controls, the VR/AR buttons and the XR session ...) is out of scope (SURVEY.md section 2).
"""
from __future__ import annotations

import enum
import math

import numpy as np

from . import _native as N
from . import three_math as TM
from .engine import Engine, Eye, Uniforms, View
from .loaders import SceneFormat, decompressGzipped
from .scenes import PackedScene, RawScene, float_centers, integer_centers, pack_scene
from .sort_worker import DefaultSplatSortDistanceMapPrecision, createSortWorker, start
from .splat_tree import SplatTree, fov_cosines

THREE_CAMERA_FOV = 50  # Viewer.js:30
MINIMUM_DISTANCE_TO_NEW_FOCAL_POINT = 0.75  # Viewer.js:31
SCENE_FADEIN_RATE_FAST = 0.012  # SplatMesh.js:30-33
SCENE_FADEIN_RATE_GRADUAL = 0.003
VISIBLE_REGION_EXPANSION_DELTA = 1
PROGRESSIVE_LOAD_SECTION_SIZE = 262144  # Constants.ProgressiveLoadSectionSize, Constants.js:8


class SceneRevealMode(enum.IntEnum):
    """src/SceneRevealMode.js: how loaded splats appear (SplatMesh.updateVisibleRegionFadeDistance)."""
    Default = 0
    Gradual = 1
    Instant = 2


def _js_or(value, default):
    """JavaScript's `value || default`: every falsy value (undefined, null, false, 0, NaN, '') takes the default."""
    return default if not value or value != value else value


def shader_max_splat_size(max_screen_space_splat_size) -> float:
    """The clamp the splat material bakes into its vertex shader, `${parseInt(maxScreenSpaceSplatSize)}.0` (SplatMaterial3D.js:195-196):
    the option truncated toward zero."""
    return float(math.trunc(float(max_screen_space_splat_size)))


class WebXRMode(enum.IntEnum):
    """src/webxr/WebXRMode.js.  The reference's WebXRMode.None is NONE here (None is a Python keyword)."""
    NONE = 0
    VR = 1
    AR = 2


class SplatScene:
    """src/splatmesh/SplatScene.js: one scene of a multi-scene mesh (Viewer.addSplatScenes).  position / quaternion (x, y, z, w) / scale
    give `transform` (updateTransform, SplatScene.js:28-36, without a three.js parent: a caller composes its own matrices).  opacity and
    visible reach the shader with the viewer option enableOptionalEffects; visible also gates the raycaster (Raycaster.js:112-114)."""

    def __init__(self, *, position=(0.0, 0.0, 0.0), quaternion=(0.0, 0.0, 0.0, 1.0), scale=(1.0, 1.0, 1.0), opacity: float = 1.0,
                 visible: bool = True, minimumAlpha: int = 1):  # noqa: N803
        self.position = tuple(float(v) for v in position)
        self.quaternion = tuple(float(v) for v in quaternion)
        self.scale = tuple(float(v) for v in scale)
        self.opacity = float(opacity)
        self.visible = bool(visible)
        self.minimumAlpha = int(minimumAlpha)

    @property
    def transform(self) -> np.ndarray:
        """Column-major f64 Matrix4.compose(position, quaternion, scale)."""
        return np.asarray(TM.compose(self.position, self.quaternion, self.scale), np.float64).reshape(16)

    def is_identity(self) -> bool:
        return self.position == (0.0, 0.0, 0.0) and self.quaternion == (0.0, 0.0, 0.0, 1.0) and self.scale == (1.0, 1.0, 1.0)


class SplatMesh:
    """Owns the GPU-side splat data of one (static) scene, or of the scenes of Viewer.addSplatScenes, and the uniforms of the splat
    material."""

    def __init__(self, *, dynamicMode=False, halfPrecisionCovariancesOnGPU=False, devicePixelRatio=1.0, antialiased=False,
                 maxScreenSpaceSplatSize=1024, splatScale=1.0, pointCloudModeEnabled=False, sphericalHarmonicsDegree=0,
                 kernel2DSize=0.3, enableOptionalEffects=False):
        self.dynamicMode = dynamicMode
        self.halfPrecisionCovariancesOnGPU = halfPrecisionCovariancesOnGPU
        self.devicePixelRatio = devicePixelRatio
        self.antialiased = antialiased
        self.maxScreenSpaceSplatSize = maxScreenSpaceSplatSize
        self.splatScale = splatScale
        self.pointCloudModeEnabled = pointCloudModeEnabled
        self.sphericalHarmonicsDegree = sphericalHarmonicsDegree
        self.kernel2DSize = kernel2DSize
        self.enableOptionalEffects = enableOptionalEffects
        self.matrixWorld = TM.identity()
        self.packed: PackedScene | None = None
        self.raw: RawScene | None = None
        self.uniforms: dict = {}
        self.renderIndexes: np.ndarray | None = None
        self.instanceCount = 0
        self.engine: Engine | None = None
        self.visibleRegionFadeStartRadius = 0.0
        self.fadeInComplete = True
        self.sceneCenter = (0.0, 0.0, 0.0)
        # the reveal (SplatMesh.js:96-110, 1172-1220), driven only by a Viewer with the sceneRevealMode option
        self.sceneFadeInRateMultiplier = 1.0
        self.visibleRegionRadius = 0.0
        self.visibleRegionBufferRadius = 0.0
        self.maxSplatDistanceFromSceneCenter = 0.0
        self.visibleRegionChanging = False
        self.finalBuild = False
        self.lastBuildSplatCount = 0
        # per-scene transforms of a dynamic mesh (SplatScene.transform, SplatScene.js:28-36; uploaded every frame by
        # fillTransformsArray, SplatMesh.js:1660-1673): column-major f64, scene 0 = the one scene this mirror holds
        self.sceneTransforms = np.tile(TM.identity(), (N.GS_MAX_SCENES, 1))
        self.splatTree: SplatTree | None = None
        self.sceneVisible = True      # SplatScene.visible of the one scene (Raycaster.js:117)
        self.scenes: list[SplatScene] = []          # Viewer.addSplatScenes' scenes, in mesh order
        self.sceneInfos: list[dict] = []            # what gs_upload_scenes reported for each (splat_offset, SH range, ...)

    def getSceneTransform(self, sceneIndex: int) -> np.ndarray:  # noqa: N802,N803  SplatMesh.js:1650-1654
        return self.sceneTransforms[sceneIndex]

    def build(self, raw_scene: RawScene, *, sh_format: str = "f16", transform16=None) -> None:
        """Decode + pack the scene like refreshGPUDataFromSplatBuffers (SplatMesh.js:588-603) and keep it for upload.
        `transform16` (column-major 4x4, the SplatScene's position/quaternion/scale): baked into centres, covariances and SH when
        the mesh is static (fillSplatDataArrays' applySceneTransform default, SplatMesh.js:1872-1883); a dynamic mesh keeps the
        data untouched and applies its transforms per frame in the sorter and the vertex stage."""
        if transform16 is not None:
            self.sceneTransforms[0] = np.asarray(transform16, np.float64).reshape(16)     # getSceneTransform(0)
        if transform16 is not None and self.dynamicMode:
            transform16 = None                                                            # applied per frame, not baked
        if transform16 is not None:
            from .scenes import transform_scene
            self.raw = transform_scene(raw_scene, transform16)[0]      # what the sorter's centres are taken from
        else:
            self.raw = raw_scene
        degree = min(self.sphericalHarmonicsDegree, raw_scene.sh_degree)
        if degree < raw_scene.sh_degree:  # minSphericalHarmonicsDegree clamp (SplatMesh.js:680-683)
            ncoef = 0 if degree == 0 else (3 if degree == 1 else 8)
            raw_scene = RawScene(raw_scene.centers, raw_scene.scales, raw_scene.rotations, raw_scene.colors,
                                 None if degree == 0 else raw_scene.sh[:, :ncoef], degree)
        self.packed = pack_scene(raw_scene, half_covariances=self.halfPrecisionCovariancesOnGPU, sh_format=sh_format, transform16=transform16)

    def fillTransformsArray(self) -> np.ndarray:  # noqa: N802  SplatMesh.js:1660-1673
        """f32[32 x 16] for the sorter ('transforms' of the sort message) and the vertex stage (`transforms` uniform)."""
        for i, sc in enumerate(self.scenes):
            self.sceneTransforms[i] = sc.transform
        return self.sceneTransforms.astype(np.float32)

    def getSceneCount(self) -> int:  # noqa: N802
        return max(len(self.scenes), 1 if self.packed is not None else 0)

    def sceneUniformArrays(self) -> dict:  # noqa: N802
        """Per-scene uniforms of a multi-scene mesh (SplatMesh.updateUniforms / SplatMaterial.js:402-409, 124-133): scene_count, each
        scene's 8-bit SH range, opacity and visibility.  Empty for a mesh of one scene loaded any other way."""
        if not self.scenes:
            return {}
        n = len(self.scenes)
        sh_min = np.full(N.GS_MAX_SCENES, -1.5, np.float32)
        sh_max = np.full(N.GS_MAX_SCENES, 1.5, np.float32)
        opacity = np.ones(N.GS_MAX_SCENES, np.float32)
        visible = np.ones(N.GS_MAX_SCENES, np.int32)
        for i, (sc, info) in enumerate(zip(self.scenes, self.sceneInfos)):
            sh_min[i], sh_max[i] = info["min_sh_coeff"], info["max_sh_coeff"]
            opacity[i], visible[i] = sc.opacity, 1 if sc.visible else 0
        return dict(scene_count=n, sh8_min=sh_min, sh8_max=sh_max, scene_opacity=opacity, scene_visibility=visible,
                    enable_optional_effects=1 if self.enableOptionalEffects else 0)

    def buildSplatTree(self, minAlpha: int = 1) -> SplatTree:  # noqa: N802,N803  SplatMesh.js:231-279
        """new SplatTree(8, 1000).processSplatMesh(this, alpha >= minAlpha): the octree over the (transformed) centres."""
        tree = SplatTree(8, 1000)
        tree.processSplatMesh(self.raw.centers, self.raw.colors[:, 3], minAlpha)
        self.splatTree = tree
        return tree

    def updateVisibleRegion(self, sinceLastBuildOnly: bool) -> None:  # noqa: N802,N803  SplatMesh.js:1172-1199
        """After a build: the largest distance of the splats [lastBuildSplatCount or 0, splat count) from the scene centre, on the GPU
        (gs_visible_region, the centres as the engine holds them), then the visible region's radii.  The scene centre is the one scene's
        (the average of one); the engine's centres already carry a static scene's transform, so none is applied again."""
        count = self.getSplatCount()
        start = self.lastBuildSplatCount if sinceLastBuildOnly else 0
        if count > start:
            d = self.engine.visible_region(start, count, None, self.sceneCenter)
            if d > self.maxSplatDistanceFromSceneCenter:
                self.maxSplatDistanceFromSceneCenter = d
        if self.maxSplatDistanceFromSceneCenter - self.visibleRegionBufferRadius > VISIBLE_REGION_EXPANSION_DELTA:
            self.visibleRegionBufferRadius = self.maxSplatDistanceFromSceneCenter
            self.visibleRegionRadius = max(self.visibleRegionBufferRadius - VISIBLE_REGION_EXPANSION_DELTA, 0.0)
        if self.finalBuild:
            self.visibleRegionRadius = self.visibleRegionBufferRadius = self.maxSplatDistanceFromSceneCenter
        self.updateVisibleRegionFadeDistance()

    def updateVisibleRegionFadeDistance(self, sceneRevealMode: int = SceneRevealMode.Default) -> None:  # noqa: N802,N803  SplatMesh.js:1201-1220
        fast = SCENE_FADEIN_RATE_FAST * self.sceneFadeInRateMultiplier
        gradual = SCENE_FADEIN_RATE_GRADUAL * self.sceneFadeInRateMultiplier
        rate = (fast if self.finalBuild else gradual) if sceneRevealMode == SceneRevealMode.Default else gradual
        self.visibleRegionFadeStartRadius = (self.visibleRegionRadius - self.visibleRegionFadeStartRadius) * rate + self.visibleRegionFadeStartRadius
        pct = self.visibleRegionFadeStartRadius / self.visibleRegionBufferRadius if self.visibleRegionBufferRadius > 0 else 0
        complete = pct > 0.99
        self.fadeInComplete = complete or sceneRevealMode == SceneRevealMode.Instant
        self.visibleRegionChanging = not complete

    # -- the scene's bounds and single splats (SplatMesh.js:1827-1834, 1959-2011, 2066-2094) -------------------------------------------
    def computeBoundingBox(self, applySceneTransforms: bool = False, sceneIndex: int | None = None) -> tuple[np.ndarray, np.ndarray]:  # noqa: N802,N803
        """The per-axis (min, max) of the splat centres of scene sceneIndex (None: every scene), f32 as the reference's Float32Array holds
        them, reduced on the GPU (gs_compute_bounding_box) bit for bit as the reference's loop.  applySceneTransforms: through each scene's
        transform (a dynamic mesh's current one).  Of a static scene loaded with a transform the engine keeps the untransformed centres
        only in the ray records of a GPU-decoded scene (the raycast option): otherwise applySceneTransforms=False raises (GsError from
        the engine; ValueError for a host-packed scene)."""
        if sceneIndex is not None and not 0 <= sceneIndex < self.getSceneCount():
            raise ValueError("SplatMesh::computeBoundingBox() -> Invalid scene index.")
        apply = bool(applySceneTransforms)
        if self.packed is not None and self.packed.centers_colors is not None and not self.dynamicMode and not np.array_equal(self.sceneTransforms[0], TM.identity()):
            # host-packed with its transform baked in: the engine holds the transformed centres only (DESIGN.md section 0)
            if not apply:
                raise ValueError("computeBoundingBox(applySceneTransforms=False): the scene was packed with its transform applied, so only the "
                                 "transformed centres are held")
            apply = False
        transforms = None
        if apply and self.dynamicMode:
            transforms = np.stack([self._sceneTransformOf(s) for s in range(self.getSceneCount())])
        return self.engine.compute_bounding_box(-1 if sceneIndex is None else int(sceneIndex), apply, transforms)

    def getSplatCenter(self, globalIndex: int, applySceneTransform: bool | None = None) -> np.ndarray:  # noqa: N802,N803
        """getSplatCenter (SplatBuffer.js:221-245): the f64 centre, through its scene's transform by default on a static mesh
        (getLocalSplatParameters).  Reads the splat's ray record: needs the viewer option raycast."""
        r = self._rayRecord(globalIndex, "getSplatCenter")
        c = [float(v) for v in r["center"]]
        t = self._transformForSplat(globalIndex, applySceneTransform)
        return np.array(c if t is None else TM.apply_matrix4(c, t))

    def getSplatScaleAndRotation(self, globalIndex: int, applySceneTransform: bool | None = None) -> tuple[np.ndarray, np.ndarray]:  # noqa: N802,N803
        """getSplatScaleAndRotation (SplatBuffer.js:247-290): (scale, rotation x y z w); under a scene transform the decomposition of
        makeScale(scale) * makeRotationFromQuaternion(rotation) * transform.  Needs the viewer option raycast, as getSplatCenter."""
        r = self._rayRecord(globalIndex, "getSplatScaleAndRotation")
        scale, rotation = [float(v) for v in r["scale"]], [float(v) for v in r["rotation"]]
        t = self._transformForSplat(globalIndex, applySceneTransform)
        if t is not None:
            m = TM.multiply_elements(TM.multiply_elements(TM.make_scale(*scale), TM.compose((0.0, 0.0, 0.0), rotation, (1.0, 1.0, 1.0))), t)
            _, rotation, scale = TM.decompose(m)
        return np.array(scale), np.array(rotation)

    def getSplatColor(self, globalIndex: int) -> np.ndarray:  # noqa: N802,N803
        """getSplatColor (SplatBuffer.js:294-305): the stored r, g, b, a bytes, before the minimum-alpha floor the data texture applies.
        The colour comes from the engine's centre-colour word; the alpha from the ray record where the engine keeps one, else from that
        word, which zeroes an alpha below its scene's splatAlphaRemovalThreshold: such a splat raises ValueError without the raycast option."""
        self._checkSplatIndex(globalIndex)
        w = int(self.engine.read_buffer(N.GS_BUF_CENTERS_COLORS, np.uint32, 1, 16 * int(globalIndex))[0])
        a = w >> 24
        if self.engine.cfg.ray_records:
            a = int(self._rayRecord(globalIndex, "getSplatColor")["alpha"])
        elif a == 0 and self.scenes and self.scenes[self._sceneOfSplat(globalIndex)].minimumAlpha > 1:
            raise ValueError(f"getSplatColor({globalIndex}): its alpha is below its scene's splatAlphaRemovalThreshold and is stored as 0; the "
                             "stored byte is kept only with the viewer option raycast")
        return np.array([w & 255, (w >> 8) & 255, (w >> 16) & 255, a], np.uint8)

    def _checkSplatIndex(self, i: int) -> None:
        if not 0 <= int(i) < self.getSplatCount():
            raise IndexError(f"splat {i} outside [0, {self.getSplatCount()})")

    def _rayRecord(self, i: int, what: str):
        self._checkSplatIndex(i)
        if self.engine is None or not self.engine.cfg.ray_records:
            raise ValueError(f"SplatMesh.{what} reads the splat's ray record: create the Viewer with the raycast option (raycast=True)")
        return self.engine.read_buffer(N.GS_BUF_RAY_RECORDS, N.RAY_RECORD_DTYPE, 1, int(i) * N.RAY_RECORD_DTYPE.itemsize)[0]

    def _sceneOfSplat(self, i: int) -> int:
        """globalSplatIndexToSceneIndexMap: the last scene starting at or before splat i (an empty scene never holds it)."""
        s = 0
        for k, info in enumerate(self.sceneInfos):
            if info["splat_offset"] <= i:
                s = k
        return s

    def _sceneTransformOf(self, s: int) -> np.ndarray:
        return self.scenes[s].transform if self.scenes else self.sceneTransforms[s]

    def _transformForSplat(self, i: int, applySceneTransform):  # noqa: N803
        """getLocalSplatParameters' rule (SplatMesh.js:1827-1834): by default a static mesh applies the splat's scene transform."""
        if applySceneTransform is None:
            applySceneTransform = not self.dynamicMode
        return self._sceneTransformOf(self._sceneOfSplat(i)) if applySceneTransform else None

    def getSplatTree(self):  # noqa: N802  SplatMesh.js:557-559
        return self.splatTree

    def getSplatCount(self) -> int:  # noqa: N802
        return 0 if self.packed is None else self.packed.count

    def getIntegerCenters(self, start: int, end: int, padFour: bool = False) -> np.ndarray:  # noqa: N802,N803
        c = integer_centers(self.raw.centers[start:end + 1])
        return c if padFour else c[:, :3].copy()

    def getFloatCenters(self, start: int, end: int, padFour: bool = False) -> np.ndarray:  # noqa: N802,N803
        c = float_centers(self.raw.centers[start:end + 1])
        return c if padFour else c[:, :3].copy()

    def setRenderer(self, engine: Engine) -> None:  # noqa: N802
        """The WebGL renderer of the reference (SplatMesh.js:1300-1340) becomes the CUDA engine; uploads the 'textures'."""
        self.engine = engine
        p = self.packed
        engine.upload_splat_data(p.centers_colors, p.covariances, p.sh, p.sh_degree)

    def updateRenderIndexes(self, globalIndexes: np.ndarray | None, renderSplatCount: int) -> None:  # noqa: N802,N803
        """SplatMesh.js:1228-1235.  globalIndexes None = keep the order the engine's last sort left on the device."""
        self.renderIndexes = globalIndexes
        self.instanceCount = int(renderSplatCount)

    def updateUniforms(self, renderDimensions, cameraFocalLengthX, cameraFocalLengthY, orthographicMode, orthographicZoom,  # noqa: N802,N803
                       inverseFocalAdjustment) -> None:
        vw, vh = renderDimensions[0] * self.devicePixelRatio, renderDimensions[1] * self.devicePixelRatio
        self.uniforms.update(viewport=(vw, vh), basisViewport=(1.0 / vw, 1.0 / vh), focal=(cameraFocalLengthX, cameraFocalLengthY),
                             orthographicMode=1 if orthographicMode else 0, orthoZoom=orthographicZoom,
                             inverseFocalAdjustment=inverseFocalAdjustment)


class Viewer:
    """Frame loop of the reference's Viewer reduced to the hot path: update() -> runSplatSort + updateSplatMesh, render()."""

    def __init__(self, options: dict | None = None):
        o = dict(options or {})
        self.cameraUp = np.asarray(o.get("cameraUp", (0, 1, 0)), np.float64)            # Viewer.js:51
        self.initialCameraPosition = np.asarray(o.get("initialCameraPosition", (0, 10, 15)), np.float64)
        self.initialCameraLookAt = np.asarray(o.get("initialCameraLookAt", (0, 0, 0)), np.float64)
        self.renderWidth = int(o.get("width", 1920))
        self.renderHeight = int(o.get("height", 1080))
        self.devicePixelRatio = float(o.get("devicePixelRatio", 1.0))
        # WebXR (Viewer.js webXRMode): width x height are the whole XR framebuffer (both eyes side by side), already in device pixels as
        # three.js sizes it, so devicePixelRatio does not apply; each eye renders one half of it
        self.webXRMode = WebXRMode(int(o.get("webXRMode", WebXRMode.NONE)))
        # frameViews of up to maxViews cameras: the engine holds that many frames of the render size stacked
        self.maxViews = int(o.get("maxViews", 1))
        if not 1 <= self.maxViews <= N.GS_MAX_VIEWS:
            raise ValueError(f"maxViews {self.maxViews} outside [1, {N.GS_MAX_VIEWS}]")
        if self.webXRMode != WebXRMode.NONE:
            if self.renderWidth % 2:
                raise ValueError(f"webXRMode: the XR framebuffer's width must be even (two eyes), got {self.renderWidth}")
            self.devicePixelRatio = 1.0
        self.gpuAcceleratedSort = bool(o.get("gpuAcceleratedSort", False))                  # Viewer.js:90
        self.integerBasedSort = bool(o.get("integerBasedSort", True))                       # Viewer.js:95-98
        self.sharedMemoryForWorkers = bool(o.get("sharedMemoryForWorkers", True))
        self.enableSIMDInSort = bool(o.get("enableSIMDInSort", True))
        self.dynamicScene = bool(o.get("dynamicScene", False))
        self.antialiased = bool(o.get("antialiased", False))
        self.kernel2DSize = float(o.get("kernel2DSize", 0.3))
        self.sphericalHarmonicsDegree = int(o.get("sphericalHarmonicsDegree", 0))
        self.focalAdjustment = float(_js_or(o.get("focalAdjustment"), 1.0))                    # Viewer.js:144
        self.maxScreenSpaceSplatSize = float(_js_or(o.get("maxScreenSpaceSplatSize"), 1024))    # Viewer.js:147
        self.halfPrecisionCovariancesOnGPU = bool(o.get("halfPrecisionCovariancesOnGPU", False))
        prec = int(o.get("splatSortDistanceMapPrecision", DefaultSplatSortDistanceMapPrecision))
        self.splatSortDistanceMapPrecision = int(np.clip(prec, 10, 20 if self.integerBasedSort else 24))  # Viewer.js:207-210
        self.device = int(o.get("device", 0))
        self.rank, self.world_size = int(o.get("rank", 0)), int(o.get("world_size", 1))
        ew, eh = self.renderDimensions()
        self.camera = TM.PerspectiveCamera(THREE_CAMERA_FOV, ew / eh, 0.1, 1000)  # Viewer.js:338
        self.camera.position = self.initialCameraPosition.copy()
        self.camera.up = self.cameraUp / np.linalg.norm(self.cameraUp)
        self.camera.look_at(self.initialCameraLookAt)
        self.splatMesh: SplatMesh | None = None
        self.engine: Engine | None = None
        self.sortWorker = None
        self.sortRunning = False
        self.splatRenderCount = 0
        self.splatSortCount = 0
        self.lastSortTime = 0.0
        self.sortWorkerIndexesToSort: np.ndarray | None = None
        self.sortWorkerSortedIndexes: np.ndarray | None = None
        self._sorted_on_device = False
        self.enableSplatTree = bool(o.get("splatTree", False))   # the reference always builds its tree; the benchmark configs sort all splats, so opt-in
        # the reference always has a Raycaster (Viewer.js:243); here it costs 56 B per splat on the GPU, so opt-in
        self.enableRaycast = bool(o.get("raycast", False))
        # the reference's default load (Viewer.js:171-176, 746-825): SplatBufferGenerator with these settings unless progressiveLoad is asked
        self.optimizeSplatData = bool(o.get("optimizeSplatData", True))
        self.inMemoryCompressionLevel = int(o.get("inMemoryCompressionLevel", 0))
        self.splatAlphaRemovalThreshold = int(o.get("splatAlphaRemovalThreshold", 1))
        self.enableOptionalEffects = bool(o.get("enableOptionalEffects", False))         # Viewer.js: per-scene opacity and visibility
        # Viewer.js:136-140, 205.  None (no option): every load is revealed at once, the reference's Instant (DESIGN.md section 0)
        reveal = o.get("sceneRevealMode")
        self.sceneRevealMode = None if reveal is None else SceneRevealMode(int(reveal))
        self.sceneFadeInRateMultiplier = float(_js_or(o.get("sceneFadeInRateMultiplier"), 1.0))
        self._sceneSources: list[tuple[int, bytes]] = []   # (format, bytes) of each addSplatScenes scene: the reference keeps its SplatBuffers
        self.raycaster = None
        if self.enableRaycast:
            from .raycaster import Raycaster
            self.raycaster = Raycaster()
        # runSplatSort's closure state (Viewer.js:1835-1841)
        self._lastSortViewDir = np.array([0.0, 0.0, -1.0])
        self._lastSortViewPos = np.zeros(3)
        self._queuedSorts: list[int] = []
        self._gathered = False

    # -- scene set-up (addSplatBuffers / setupSortWorker, Viewer.js:1094-1300) ------------------------------------------------
    def addSplatScene(self, raw_scene: RawScene, *, separate_sort_worker: bool = False, position=(0.0, 0.0, 0.0),  # noqa: N802
                      rotation=(0.0, 0.0, 0.0, 1.0), scale=(1.0, 1.0, 1.0)) -> None:
        """Viewer.addSplatScene's `position` / `rotation` (quaternion x, y, z, w) / `scale` options (Viewer.js:736-760): the
        SplatScene transform, baked at load for a static mesh."""
        self.splatMesh = SplatMesh(dynamicMode=self.dynamicScene, halfPrecisionCovariancesOnGPU=self.halfPrecisionCovariancesOnGPU,
                                   devicePixelRatio=self.devicePixelRatio, antialiased=self.antialiased,
                                   maxScreenSpaceSplatSize=self.maxScreenSpaceSplatSize, sphericalHarmonicsDegree=self.sphericalHarmonicsDegree,
                                   kernel2DSize=self.kernel2DSize)
        self._sceneSources = []   # a single-scene mesh replaces any addSplatScenes mesh
        identity = tuple(position) == (0.0, 0.0, 0.0) and tuple(rotation) == (0.0, 0.0, 0.0, 1.0) and tuple(scale) == (1.0, 1.0, 1.0)
        self.splatMesh.build(raw_scene, transform16=None if identity else TM.compose(position, rotation, scale))
        n = self.splatMesh.getSplatCount()
        self.engine = Engine(n, device=self.device, distance_map_range=1 << self.splatSortDistanceMapPrecision,
                             integer_based_sort=self.integerBasedSort, dynamic_mode=self.dynamicScene,
                             max_width=self.renderWidth, max_height=self.renderHeight * self.maxViews, rank=self.rank, world_size=self.world_size,
                             ray_records=self.enableRaycast)
        self.splatMesh.setRenderer(self.engine)
        centers = (self.splatMesh.getIntegerCenters(0, n - 1, True) if self.integerBasedSort else self.splatMesh.getFloatCenters(0, n - 1, True))
        if separate_sort_worker:
            # the reference's topology: a worker with its own memory, sorted indexes travel back through the host
            self.sortWorker = createSortWorker(n, self.sharedMemoryForWorkers, self.enableSIMDInSort, self.integerBasedSort,
                                               self.dynamicScene, self.splatSortDistanceMapPrecision, device=self.device)
            self.sortWorker.onmessage = self._on_worker_message
            start(self.sortWorker)
            self.sortWorker.postMessage({"centers": centers, "sceneIndexes": None, "range": {"from": 0, "to": n - 1, "count": n}})
        else:
            self.engine.upload_centers(centers, np.zeros(n, np.uint32) if self.dynamicScene else None)
        self.splatRenderCount = n
        if self.enableRaycast:
            from .raycaster import ray_records_from_raw
            self.engine.upload_ray_records(ray_records_from_raw(raw_scene), 0, None if identity or self.dynamicScene else TM.compose(position, rotation, scale))
        self._build_splat_tree()

    def _build_splat_tree(self) -> None:
        """SplatMesh.buildSplatTree (SplatMesh.js:231-279, called for every scene at :394) on the GPU, from the centres and alphas the
        engine already holds (gs_build_splat_tree): the frame path culls with it when `splatTree` is on, the raycaster walks it when
        `raycast` is on.  getSplatTree().leaves is the tree read back.  With `raycast` alone the frame path keeps sorting every splat."""
        if not (self.enableSplatTree or self.enableRaycast) or self.splatMesh.getSplatCount() == 0:
            return
        self.engine.build_splat_tree(8, 1000, 1)
        if self.enableSplatTree:
            tree = SplatTree(8, 1000)
            tree.leaves = self.engine.read_splat_tree()
            self.splatMesh.splatTree = tree

    def addSplatSceneFromKSplat(self, data: bytes, *, position=(0.0, 0.0, 0.0), rotation=(0.0, 0.0, 0.0, 1.0), scale=(1.0, 1.0, 1.0)) -> dict:  # noqa: N802
        """Viewer.addSplatScene for a `.ksplat` buffer (KSplatLoader.loadFromFileData -> new SplatBuffer -> SplatMesh.build ->
        'centers' message, Viewer.js:736-868, 1094-1167): header parsing on the host, every per-splat decode on the GPU.
        position / rotation (x, y, z, w) / scale: the SplatScene transform, baked by the decode kernel (static mesh)."""
        from . import ksplat as K
        hdr = K.parse(data)
        return self._add_decoded_scene(hdr.max_splat_count, lambda transform16: self.engine.upload_ksplat(
            data, half_covariances=self.halfPrecisionCovariancesOnGPU, transform16=transform16), position, rotation, scale)

    def addSplatSceneFromFile(self, data: bytes, format: int, *, position=(0.0, 0.0, 0.0), rotation=(0.0, 0.0, 0.0, 1.0),  # noqa: N802,A002
                              scale=(1.0, 1.0, 1.0), progressiveLoad: bool = True) -> dict:  # noqa: N803
        """Viewer.addSplatScene for a `.ply` (format SceneFormat.Ply, INRIA or PlayCanvas-compressed) or `.splat` (SceneFormat.Splat) file,
        every per-splat step on the GPU.  The engine is sized from the file's header (gs_probe_file); SH are loaded up to the viewer's
        sphericalHarmonicsDegree.  position / rotation (x, y, z, w) / scale: the SplatScene transform, baked at load (static mesh).
          progressiveLoad=True (this method's default): as the progressive loader builds it (PlyLoader.js:192-206, SplatLoader.js:108),
            the splats in file order.
          progressiveLoad=False with the viewer option optimizeSplatData (the reference Viewer's default): through
            SplatBufferGenerator.getStandardGenerator (PlyLoader.js:316-330, SplatLoader.js:12-21): splats below
            splatAlphaRemovalThreshold removed, the rest reordered and bucketed, at inMemoryCompressionLevel.
          progressiveLoad=False without optimizeSplatData: file order, as DownloadBeforeProcessing gives it.
        An INRIA v2 (codebook) .ply loads only with progressiveLoad=False and optimizeSplatData, through the generator; otherwise the
        library's GsError says so, as the reference's Viewer throws there.
        A `.spz` file (SceneFormat.Spz) is passed as stored and gunzipped here (SpzLoader.loadFromFileData).  It is not progressively
        loadable (Viewer.isProgressivelyLoadable), so progressiveLoad is ignored: optimizeSplatData alone picks the generator path or
        file order."""
        if format == SceneFormat.Spz:
            data = decompressGzipped(data)
            progressiveLoad = False
        n = Engine.probe_file(format, data)["splat_count"]
        if not progressiveLoad and self.optimizeSplatData:
            return self._add_decoded_scene(n, lambda transform16: self.engine.upload_file_optimized(
                format, data, sh_degree=self.sphericalHarmonicsDegree, compression_level=self.inMemoryCompressionLevel,
                minimum_alpha=self.splatAlphaRemovalThreshold, half_covariances=self.halfPrecisionCovariancesOnGPU, transform16=transform16),
                position, rotation, scale)
        return self._add_decoded_scene(n, lambda transform16: self.engine.upload_file(
            format, data, sh_degree=self.sphericalHarmonicsDegree, half_covariances=self.halfPrecisionCovariancesOnGPU,
            transform16=transform16), position, rotation, scale)

    def _add_decoded_scene(self, n: int, upload, position, rotation, scale) -> dict:
        """Body shared by the loaders that decode on the GPU: a static mesh and an engine for n splats, then upload(transform16)."""
        self._sceneSources = []   # a single-scene mesh replaces any addSplatScenes mesh
        self.splatMesh = SplatMesh(dynamicMode=False, halfPrecisionCovariancesOnGPU=self.halfPrecisionCovariancesOnGPU,
                                   devicePixelRatio=self.devicePixelRatio, antialiased=self.antialiased,
                                   maxScreenSpaceSplatSize=self.maxScreenSpaceSplatSize, sphericalHarmonicsDegree=self.sphericalHarmonicsDegree,
                                   kernel2DSize=self.kernel2DSize)
        self.engine = Engine(n, device=self.device, distance_map_range=1 << self.splatSortDistanceMapPrecision,
                             integer_based_sort=self.integerBasedSort, dynamic_mode=False, max_width=self.renderWidth, max_height=self.renderHeight * self.maxViews,
                             rank=self.rank, world_size=self.world_size, ray_records=self.enableRaycast)
        identity = tuple(position) == (0.0, 0.0, 0.0) and tuple(rotation) == (0.0, 0.0, 0.0, 1.0) and tuple(scale) == (1.0, 1.0, 1.0)
        transform16 = None if identity else TM.compose(position, rotation, scale)
        info = upload(transform16)
        if transform16 is not None:
            self.splatMesh.sceneTransforms[0] = transform16
        self.splatMesh.engine = self.engine
        degree = min(self.sphericalHarmonicsDegree, info["sh_degree"])
        self.splatMesh.packed = PackedScene(None, None, None, degree, None, info["splat_count"])
        self.splatMesh.sceneCenter = info["scene_center"]
        self._ksplat_info = info
        self.splatRenderCount = info["splat_count"]
        self._build_splat_tree()
        self.splatMesh.finalBuild = True
        self._reveal_build(False)
        return info

    def _reveal_build(self, sinceLastBuildOnly: bool) -> None:  # noqa: N803
        """refreshGPUDataFromSplatBuffers' updateVisibleRegion (SplatMesh.js:620-635) after a build, with the sceneRevealMode option."""
        sm = self.splatMesh
        if self.sceneRevealMode is None:
            return
        sm.sceneFadeInRateMultiplier = self.sceneFadeInRateMultiplier
        sm.updateVisibleRegion(sinceLastBuildOnly)
        sm.lastBuildSplatCount = sm.getSplatCount()

    def addSplatSceneProgressive(self, format: int, *, fileSize: int | None = None, position=(0.0, 0.0, 0.0),  # noqa: N802,N803,A002
                                 rotation=(0.0, 0.0, 0.0, 1.0), scale=(1.0, 1.0, 1.0)) -> "ProgressiveSceneLoad":
        """Viewer.addSplatScene with progressiveLoad for a `.ply` (INRIA v1, or PlayCanvas-compressed without SH), `.splat` or `.ksplat` file
        whose bytes arrive in pieces (Viewer.downloadAndBuildSingleSplatSceneProgressiveLoad, Viewer.js:871-946): the returned load takes
        them with append(chunk) and ends with finish().  Splats are rendered as their builds land.  fileSize (the download's length) is
        needed for a `.splat`, which has no header to size the engine from.  A `.spz` or INRIA v2 `.ply` raises GsError, as
        Viewer.isProgressivelyLoadable refuses them."""
        return ProgressiveSceneLoad(self, format, fileSize, position, rotation, scale)

    # -- several scenes in one mesh (Viewer.addSplatScenes / removeSplatScenes, Viewer.js:973-1085, 1326-1430) ------------------------
    def addSplatScenes(self, sceneOptions: list[dict]) -> list[dict]:  # noqa: N802,N803
        """Add scenes to the viewer's multi-scene mesh and rebuild it from all of them, as SplatMesh.build does.  Each option dict has
        `data` and `format` (SceneFormat.Ply / Splat / Spz / KSplat; .spz as stored, gunzipped here), and optionally `position`,
        `rotation` (x, y, z, w), `scale`, `splatAlphaRemovalThreshold`, `opacity` and `visible`.  Files load as the reference's
        non-progressive addSplatScenes loads them: through the generator with optimizeSplatData, else in file order; a .ksplat as stored.
        Scenes already in the mesh keep their current transforms.  Returns the info of every scene of the rebuilt mesh."""
        sources, scenes = [], []
        for opt in sceneOptions:
            fmt, data = int(opt["format"]), opt["data"]
            if fmt == SceneFormat.Spz:
                data = decompressGzipped(data)
            sources.append((fmt, bytes(data)))
            scenes.append(SplatScene(position=opt.get("position", (0.0, 0.0, 0.0)), quaternion=opt.get("rotation", (0.0, 0.0, 0.0, 1.0)),
                                     scale=opt.get("scale", (1.0, 1.0, 1.0)), opacity=opt.get("opacity", 1.0), visible=opt.get("visible", True),
                                     minimumAlpha=_js_or(opt.get("splatAlphaRemovalThreshold"), 1)))
        kept = self.splatMesh.scenes if self.splatMesh is not None and self.splatMesh.scenes else []
        return self._build_scenes(self._sceneSources + sources, kept + scenes)

    def removeSplatScenes(self, indexesToRemove) -> list[dict]:  # noqa: N802,N803
        """Drop scenes and rebuild the mesh from the rest at their current transforms (Viewer.js:1326-1430)."""
        drop = set(int(i) for i in indexesToRemove)
        n = len(self._sceneSources)
        if any(i < 0 or i >= n for i in drop):
            raise IndexError(f"removeSplatScenes: scene indexes {sorted(drop)} outside [0, {n})")
        keep = [i for i in range(n) if i not in drop]
        return self._build_scenes([self._sceneSources[i] for i in keep], [self.splatMesh.scenes[i] for i in keep])

    def removeSplatScene(self, index: int) -> list[dict]:  # noqa: N802
        return self.removeSplatScenes([index])

    def getSplatScene(self, index: int) -> SplatScene:  # noqa: N802
        return self.splatMesh.scenes[index]

    def getSceneCount(self) -> int:  # noqa: N802
        return 0 if self.splatMesh is None else self.splatMesh.getSceneCount()

    def _scene_capacity(self, sources) -> int:
        """The splats the engine must hold for `sources`: each file's header count (the generator keeps at most that many)."""
        from . import ksplat as K
        return sum(K.parse(d).max_splat_count if f == SceneFormat.KSplat else Engine.probe_file(f, d)["splat_count"] for f, d in sources)

    def _build_scenes(self, sources, scenes) -> list[dict]:
        if len(sources) != len(scenes):
            raise ValueError(f"addSplatScenes: {len(sources)} sources for {len(scenes)} scenes")
        if len(sources) > N.GS_MAX_SCENES:
            raise ValueError(f"addSplatScenes: {len(sources)} scenes, a mesh holds at most {N.GS_MAX_SCENES}")
        if len(sources) > 1 and self.world_size > 1:
            raise ValueError(f"addSplatScenes: {len(sources)} scenes with world_size {self.world_size}: multi-scene frames are single-GPU only")
        mesh = SplatMesh(dynamicMode=self.dynamicScene, halfPrecisionCovariancesOnGPU=self.halfPrecisionCovariancesOnGPU,
                         devicePixelRatio=self.devicePixelRatio, antialiased=self.antialiased, maxScreenSpaceSplatSize=self.maxScreenSpaceSplatSize,
                         sphericalHarmonicsDegree=self.sphericalHarmonicsDegree, kernel2DSize=self.kernel2DSize,
                         enableOptionalEffects=self.enableOptionalEffects)
        if not sources:
            self._sceneSources, self.splatMesh, self.splatRenderCount = [], mesh, 0
            return []
        need = self._scene_capacity(sources)
        e = self.engine
        if e is None or e.max_splat_count < need or e.dynamic_mode != self.dynamicScene:
            if e is not None:
                e.close()
            self.engine = Engine(need, device=self.device, distance_map_range=1 << self.splatSortDistanceMapPrecision,
                                 integer_based_sort=self.integerBasedSort, dynamic_mode=self.dynamicScene, max_width=self.renderWidth,
                                 max_height=self.renderHeight * self.maxViews, rank=self.rank, world_size=self.world_size, ray_records=self.enableRaycast)
        src = []
        for (fmt, data), sc in zip(sources, scenes):
            optimized = fmt != SceneFormat.KSplat and self.optimizeSplatData
            src.append(dict(format=fmt, data=data, minimum_alpha=sc.minimumAlpha, optimized=optimized,
                            generate=dict(compression_level=self.inMemoryCompressionLevel, minimum_alpha=sc.minimumAlpha),
                            transform16=None if self.dynamicScene or sc.is_identity() else sc.transform))
        infos = self.engine.upload_scenes(src, sh_degree=self.sphericalHarmonicsDegree, half_covariances=self.halfPrecisionCovariancesOnGPU)
        total = sum(i["splat_count"] for i in infos)
        degree = min([self.sphericalHarmonicsDegree] + [i["sh_degree"] for i in infos])
        mesh.engine = self.engine
        mesh.scenes, mesh.sceneInfos = list(scenes), infos
        mesh.packed = PackedScene(None, None, None, degree, None, total)
        # the mean of the scenes' centres (SplatMesh.js:1176-1182)
        mesh.sceneCenter = tuple(float(np.mean([i["scene_center"][k] for i in infos])) for k in range(3))
        self._sceneSources, self.splatMesh, self.splatRenderCount = list(sources), mesh, total
        self._ksplat_info = None
        self._build_splat_tree()       # a dynamic mesh of several scenes: one sub-tree per scene (SplatTree.js:377-390)
        return infos

    def checkForFocalPointChange(self, x: float, y: float):  # noqa: N802  Viewer.js:555-581
        """Cast a ray through render-dimension pixel (x, y) (y down); the nearest hit's point when it lies farther than
        MINIMUM_DISTANCE_TO_NEW_FOCAL_POINT from the camera (the new focal point), else None.  Needs Viewer(raycast=True)."""
        if self.raycaster is None:
            raise RuntimeError("checkForFocalPointChange needs the viewer option raycast=True")
        self.raycaster.setFromCameraAndScreenPosition(self.camera, (x, y), (self.renderWidth, self.renderHeight))
        hits = self.raycaster.intersectSplatMesh(self.splatMesh, capacity=1)
        if not hits:
            return None
        p = hits[0].origin
        d = [float(p[0]) - float(self.camera.position[0]), float(p[1]) - float(self.camera.position[1]), float(p[2]) - float(self.camera.position[2])]
        import math
        if math.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]) > MINIMUM_DISTANCE_TO_NEW_FOCAL_POINT:
            return p.copy()
        return None

    def _on_worker_message(self, e) -> None:  # Viewer.js:1243-1298
        d = e.data
        if d.get("sortDone"):
            self.sortRunning = False
            self.lastSortTime = d["sortTime"]
            sorted_idx = self.sortWorkerSortedIndexes if self.sharedMemoryForWorkers else d["sortedIndexes"]
            self.splatMesh.updateRenderIndexes(sorted_idx[: d["splatRenderCount"]], d["splatRenderCount"])
        elif d.get("sortSetupPhase1Complete"):
            if self.sharedMemoryForWorkers:
                self.sortWorkerIndexesToSort = d["indexesToSortBuffer"]
                self.sortWorkerSortedIndexes = d["sortedIndexesBuffer"]
                self.sortWorkerIndexesToSort[:] = np.arange(self.sortWorkerIndexesToSort.shape[0], dtype=np.uint32)  # Viewer.js:1282-1284

    # -- matrices ----------------------------------------------------------------------------------------------------------------
    def mvp_matrix(self, camera=None) -> np.ndarray:
        """Viewer.js:1888-1891 in float64: projection * inverse(camera.matrixWorld) * splatMesh.matrixWorld (camera: the viewer's)."""
        camera = self.camera if camera is None else camera
        m = TM.invert(camera.matrixWorld)
        m = TM.multiply(camera.projectionMatrix, m)
        if not self.splatMesh.dynamicMode:
            m = TM.multiply(m, self.splatMesh.matrixWorld)
        return m

    def renderDimensions(self) -> tuple[int, int]:  # noqa: N802
        """What updateSplatMesh sizes the uniforms for: the frame, or in XR mode one eye (half of the XR framebuffer)."""
        return (self.renderWidth // 2 if self.webXRMode != WebXRMode.NONE else self.renderWidth), self.renderHeight

    def updateSplatMesh(self) -> None:  # noqa: N802  Viewer.js:651-677
        if self.sceneRevealMode is not None and self.splatMesh.getSplatCount() > 0:
            self.splatMesh.updateVisibleRegionFadeDistance(self.sceneRevealMode)
        # (XR mode: sized for one eye, so the viewport uniform is the eye's size.  The reference instead rescales a canvas-sized viewport,
        # adjustForWebXRStereo Viewer.js:680-687; see DESIGN.md section 5.x)
        fx, fy, zoom, fa = self._focal(self.camera)
        self.splatMesh.updateUniforms(self.renderDimensions(), fx, fy, self.camera.isOrthographicCamera, zoom, 1.0 / fa)

    def _focal(self, camera) -> tuple[float, float, float, float]:
        """updateSplatMesh's focal lengths for `camera` at the render size (devicePixelRatio, and focalAdjustment as the orthographic
        rule scales it), its orthographic zoom, and that focal adjustment."""
        w, h = self.renderDimensions()
        fx = camera.projectionMatrix[0] * 0.5 * self.devicePixelRatio * w
        fy = camera.projectionMatrix[5] * 0.5 * self.devicePixelRatio * h
        fa = self.focalAdjustment * (1.0 / self.devicePixelRatio if camera.isOrthographicCamera else 1.0)
        return fx * fa, fy * fa, camera.zoom or 1.0, fa

    def uniforms(self) -> Uniforms:
        """What three.js + SplatMesh hand the splat shaders for the current camera."""
        sm = self.splatMesh
        mv = TM.multiply(self.camera.matrixWorldInverse, sm.matrixWorld)
        u = sm.uniforms
        dyn = {}
        if sm.dynamicMode:      # SplatMaterial.js:136-146: transformModelViewMatrix = viewMatrix * transforms[sceneIndex]
            dyn = dict(dynamic_mode=1, scene_transforms=sm.fillTransformsArray(), view_matrix=self.camera.matrixWorldInverse.astype(np.float32), scene_count=1)
        info = getattr(self, "_ksplat_info", None) or {}
        per_scene = dict(sh8_min=np.full(N.GS_MAX_SCENES, info.get("min_sh_coeff", -1.5), np.float32),
                         sh8_max=np.full(N.GS_MAX_SCENES, info.get("max_sh_coeff", 1.5), np.float32))
        per_scene.update(sm.sceneUniformArrays())
        dyn.update(per_scene)
        return Uniforms(**dyn, model_view=mv.astype(np.float32), projection=self.camera.projectionMatrix.astype(np.float32),
                        camera_position=np.asarray(self.camera.position, np.float32), focal=u["focal"], viewport=u["viewport"],
                        inverse_focal_adjustment=u["inverseFocalAdjustment"], ortho_zoom=u["orthoZoom"], orthographic_mode=u["orthographicMode"],
                        splat_scale=sm.splatScale, point_cloud_mode=1 if sm.pointCloudModeEnabled else 0,
                        sh_degree=sm.packed.sh_degree, antialiased=1 if sm.antialiased else 0, kernel_2d_size=sm.kernel2DSize,
                        max_screen_space_splat_size=shader_max_splat_size(sm.maxScreenSpaceSplatSize), fade_in_complete=1 if sm.fadeInComplete else 0,
                        scene_center=sm.sceneCenter, visible_region_fade_start_radius=sm.visibleRegionFadeStartRadius)

    def viewFor(self, camera) -> View:  # noqa: N802
        """The gs_view of `camera` (a three_math camera after update()), built as runSplatSort builds the viewer camera's f32 sort matrix
        and updateSplatMesh / uniforms() its focal lengths, model view, projection, position and view matrix.  Host only."""
        if camera.isOrthographicCamera != self.camera.isOrthographicCamera:
            raise ValueError("frameViews: every camera must be orthographic when the viewer's camera is, and perspective when it is not")
        sm = self.splatMesh
        fx, fy, zoom, _ = self._focal(camera)
        return View(model_view_proj=self.mvp_matrix(camera).astype(np.float32),
                    model_view=TM.multiply(camera.matrixWorldInverse, sm.matrixWorld).astype(np.float32),
                    projection=np.asarray(camera.projectionMatrix, np.float32), camera_position=np.asarray(camera.position, np.float32),
                    focal=(fx, fy), ortho_zoom=zoom,
                    view_matrix=camera.matrixWorldInverse.astype(np.float32) if sm.dynamicMode else None)

    def xrEyes(self, xrCameras) -> tuple[Eye, Eye]:  # noqa: N802,N803
        """The per-eye uniforms of a WebXR frame, as three.js sets its built-ins for each sub-camera of the XR ArrayCamera when it draws
        the splat mesh: modelViewMatrix = eye.matrixWorldInverse * mesh.matrixWorld, projectionMatrix, cameraPosition (the eye's world
        position) and, for a dynamic mesh, viewMatrix.  xrCameras = (left, right), each with matrixWorld, matrixWorldInverse and
        projectionMatrix (three_math.PerspectiveCamera after update()).  Host only: no engine is needed."""
        if len(xrCameras) != 2:
            raise ValueError(f"xrCameras: want (left, right), got {len(xrCameras)} cameras")
        sm = self.splatMesh
        return tuple(Eye(model_view=TM.multiply(c.matrixWorldInverse, sm.matrixWorld).astype(np.float32),
                         projection=np.asarray(c.projectionMatrix, np.float32),
                         camera_position=np.asarray(c.matrixWorld[12:15], np.float32),
                         view_matrix=np.asarray(c.matrixWorldInverse, np.float32) if sm.dynamicMode else None) for c in xrCameras)

    def _xr(self, xrCameras):
        """The eyes of a frame: None for the mono frame; in XR mode the xrCameras' (which are then required)."""
        if self.webXRMode == WebXRMode.NONE:
            if xrCameras is not None:
                raise ValueError("xrCameras: the viewer was not created with webXRMode VR or AR")
            return None
        if xrCameras is None:
            raise ValueError("webXRMode: render / frame need xrCameras=(left, right)")
        return self.xrEyes(xrCameras)

    # -- the per-frame path --------------------------------------------------------------------------------------------------------
    def gatherSceneNodesForSort(self, gatherAllNodes: bool = False) -> tuple[int, bool]:  # noqa: N802,N803  Viewer.js:1969-2077
        """(splatRenderCount, shouldSortAll).  With a SplatTree: every leaf is culled against the frustum and the kept leaves' indexes are
        laid out nearest-last in the sorter's indexesToSort -- on the GPU (gs_gather_for_sort); without one: identity, sort all.  A dynamic
        mesh culls sub-tree s (scene s's) with baseModelView * sceneTransform(s) (Viewer.js:2005-2011)."""
        tree = self.splatMesh.getSplatTree()
        if tree is None or tree.leaves is None:
            self._gathered = False
            return self.splatMesh.getSplatCount(), True
        base = TM.invert(self.camera.matrixWorld)
        if not self.splatMesh.dynamicMode:
            base = TM.multiply(base, self.splatMesh.matrixWorld)
        cx, cy = fov_cosines(self.renderWidth * self.devicePixelRatio, self.renderHeight * self.devicePixelRatio, self.camera.fov)
        if self.splatMesh.dynamicMode:
            self.splatMesh.fillTransformsArray()
            views = [TM.multiply(base, self.splatMesh.getSceneTransform(s)) for s in range(tree.leaves.sub_tree_count)]
            count = self.engine.gather_for_sort_subtrees(views, cx, cy, gatherAllNodes)
        else:
            count = self.engine.gather_for_sort(base, cx, cy, gatherAllNodes)
        self._gathered = True
        return count, False

    def runSplatSort(self, force: bool = False, forceSortAll: bool = False) -> bool:  # noqa: N802,N803  Viewer.js:1833-1964
        """The reference's scheduling: skip while the view has barely changed, gather the visible leaves, and after a large rotation queue
        partial sorts of the nearest 12.5 % / 33 % / 75 % ... before the full one (Viewer.js:1843-1856, 1899-1913)."""
        if self.sortRunning:
            return True
        if self.splatMesh.getSplatCount() <= 0:
            self.splatRenderCount = 0
            return False
        view_dir = -np.asarray(self.camera.matrixWorld[8:11], np.float64)     # (0, 0, -1).applyQuaternion(camera.quaternion)
        angle_diff = float(np.dot(view_dir, self._lastSortViewDir))
        position_diff = float(np.linalg.norm(np.asarray(self.camera.position, np.float64) - self._lastSortViewPos))
        if not force and not self.splatMesh.dynamicMode and not self._queuedSorts:
            if not (angle_diff <= 0.99 or position_diff >= 1.0):
                return False
        render_count, should_sort_all = self.gatherSceneNodesForSort()
        should_sort_all = should_sort_all or forceSortAll
        self.splatRenderCount = render_count
        mvp = self.mvp_matrix()
        if not self._queuedSorts:
            if self.splatMesh.dynamicMode or should_sort_all:
                self._queuedSorts.append(render_count)
            else:
                for threshold, fractions in ((0.55, (0.125, 0.33333, 0.75)), (0.65, (0.33333, 0.66667)), (0.8, (0.5,))):
                    if angle_diff < threshold:
                        self._queuedSorts.extend(int(np.floor(render_count * f)) for f in fractions)
                        break
                self._queuedSorts.append(render_count)
        sort_count = min(self._queuedSorts.pop(0), render_count)
        self.splatSortCount = sort_count
        n = render_count
        if self.sortWorker is not None:
            self.sortRunning = True
            msg = {"modelViewProj": mvp.astype(np.float32), "cameraPosition": list(self.camera.position), "splatRenderCount": n,
                   "splatSortCount": sort_count, "usePrecomputedDistances": False}
            if not self.sharedMemoryForWorkers:
                msg["indexesToSort"] = np.arange(n, dtype=np.uint32)
                msg["transforms"] = self.splatMesh.fillTransformsArray() if self.splatMesh.dynamicMode else None
            self.sortWorker.postMessage({"sort": msg})
        else:
            tr = self.splatMesh.fillTransformsArray() if self.splatMesh.dynamicMode else None
            if self._gathered:
                _, ms = self.engine.sort_gathered(mvp.astype(np.float32), sort_count, n, download=False, transforms=tr)
            else:
                _, ms = self.engine.sort(mvp.astype(np.float32), sort_count, n, None, download=False, transforms=tr)
            self.lastSortTime = ms
            self.splatMesh.updateRenderIndexes(None, n)
        if not self._queuedSorts:
            self._lastSortViewPos = np.asarray(self.camera.position, np.float64).copy()
            self._lastSortViewDir = view_dir.copy()
        return True

    def update(self, force_sort: bool = True) -> None:  # Viewer.js:1625-1644
        """force_sort=True sorts on every call (what the tests and the benchmark want); False applies the reference's view-change
        thresholds like its frame loop does."""
        self.camera.update()
        self.runSplatSort(force=force_sort, forceSortAll=force_sort and self.splatMesh.getSplatTree() is None)
        self.updateSplatMesh()

    def render(self, *, frame_format: int = N.GS_FRAME_RGBA8, flip_y: bool = True, download: bool = True, dest_color=None,
               dest_depth=None, xrCameras=None, depth: bool = False):  # noqa: N803  Viewer.js:1599-1623
        """dest_color / dest_depth: the colour and depth of the opaque pass that Viewer.render draws first (options.threeScene,
        Viewer.js:81-82, 1610-1613); the splat mesh is then drawn into it, depth-tested without depth writes (Engine.render).
        xrCameras (webXRMode VR / AR): the (left, right) eye cameras of the XR ArrayCamera; both eyes are drawn side by side into the
        width x height frame with the draw order of the viewer camera's sort (Engine.render eyes=).
        depth: returns (rgba, depth), the view depth per pixel float32 (height, width) in the frame's row order (Engine.render depth=);
        an addition beyond the reference, whose splat material writes no depth."""
        sm = self.splatMesh
        return self.engine.render(self.uniforms(), self.renderWidth, self.renderHeight, sm.instanceCount, sm.renderIndexes,
                                  frame_format=frame_format, flip_y=flip_y, download=download, dest_color=dest_color, dest_depth=dest_depth,
                                  eyes=self._xr(xrCameras), depth=depth)

    def frame(self, *, frame_format: int = N.GS_FRAME_RGBA8, flip_y: bool = True, download: bool = True, frame_out=None, dest_color=None,
              dest_depth=None, xrCameras=None, depth: bool = False):  # noqa: N803
        """update() + render() fused into one engine call (sort order never leaves the device).  dest_color / dest_depth, xrCameras,
        depth: as for render(); the sort uses the viewer camera."""
        self.camera.update()
        self.updateSplatMesh()
        n = self.splatMesh.getSplatCount()
        return self.engine.frame(self.mvp_matrix().astype(np.float32), self.uniforms(), self.renderWidth, self.renderHeight, n, None,
                                 frame_format=frame_format, flip_y=flip_y, download=download, frame_out=frame_out,
                                 transforms=self.splatMesh.fillTransformsArray() if self.splatMesh.dynamicMode else None,
                                 dest_color=dest_color, dest_depth=dest_depth, eyes=self._xr(xrCameras), depth=depth)

    def frameViews(self, cameras, *, frame_format: int = N.GS_FRAME_RGBA8, flip_y: bool = True, download: bool = True,  # noqa: N802
                   depth: bool = False):
        """Several cameras of the mesh in one engine call (Engine.frame_views): each camera sorted on its own and rendered at the render
        size, as frame() renders the viewer's camera; returns (len(cameras), height, width, 4).  Up to the viewer option maxViews cameras.  The whole mesh in identity order (no
        SplatTree culling per camera).  Every other uniform is the viewer's.  depth: returns (rgba, depth), the view depths float32
        (len(cameras), height, width), each camera's with its own projection (as for render())."""
        if self.webXRMode != WebXRMode.NONE:
            raise ValueError("frameViews: a WebXR viewer renders its eyes with frame(xrCameras=...)")
        self.camera.update()
        self.updateSplatMesh()
        for c in cameras:
            if c is not self.camera:
                c.update()
        n = self.splatMesh.getSplatCount()
        return self.engine.frame_views([self.viewFor(c) for c in cameras], self.uniforms(), self.renderWidth, self.renderHeight, n, None,
                                       frame_format=frame_format, flip_y=flip_y, download=download, depth=depth,
                                       transforms=self.splatMesh.fillTransformsArray() if self.splatMesh.dynamicMode else None)

    def dispose(self) -> None:
        if self.sortWorker is not None:
            self.sortWorker.terminate()
        if self.engine is not None:
            self.engine.close()


def _stream_capacity(format: int, head: bytes, file_size: int | None) -> int | None:  # noqa: A002
    """The splat count a streamed file's header declares, once its bytes are in (None before): the engine is sized from it."""
    if format == SceneFormat.Splat:
        if file_size is None:
            raise ValueError("a progressive .splat load needs fileSize: its splat count is fileSize // 32")
        return int(file_size) // 32
    if format == SceneFormat.KSplat:
        return int.from_bytes(head[12:16], "little") if len(head) >= 16 else None
    end = head.find(b"end_header")
    if end < 0:
        return None
    for line in head[:end].decode("ascii", "replace").split("\n"):
        w = line.split()
        if len(w) == 3 and w[0] == "element" and w[1] == "vertex" and w[2].isdigit():
            return int(w[2])
    return 0


class ProgressiveSceneLoad:
    """One progressive load (Viewer.addSplatSceneProgressive).  append(chunk) takes the next bytes of the file; a build lands when more
    than PROGRESSIVE_LOAD_SECTION_SIZE bytes arrived since the last section (PlyLoader.js:176-272, KSplatLoader.js:131-133: the section
    mark advances by one section size per build; counted here from the file's first byte), and finish() makes the final build.  Each
    build appends the bytes received since the previous one to the engine's stream (gs_stream_append), after which the splats it
    completed render; builds[i] is the splat count after build i."""

    def __init__(self, viewer: Viewer, format: int, file_size, position, rotation, scale):  # noqa: A002
        if format == SceneFormat.Spz:
            raise N.GsError(N.GS_ERR_BAD_ARG, "addSplatSceneProgressive", ".spz is not progressively loadable (Viewer.isProgressivelyLoadable)")
        self.viewer, self.format, self.fileSize = viewer, int(format), file_size
        identity = tuple(position) == (0.0, 0.0, 0.0) and tuple(rotation) == (0.0, 0.0, 0.0, 1.0) and tuple(scale) == (1.0, 1.0, 1.0)
        self.transform16 = None if identity else TM.compose(position, rotation, scale)
        self.received = 0
        self.streamed = 0
        self.builds: list[int] = []
        self._head = b""
        self._pending: list[bytes] = []
        self._stream = None
        self.info: dict | None = None

    def append(self, chunk) -> bool:
        """Take the next bytes; True when they completed a build."""
        chunk = bytes(chunk)
        self.received += len(chunk)
        self._pending.append(chunk)
        if self._stream is None and len(self._head) < (1 << 16):
            self._head += chunk
        if self.received - self.streamed > PROGRESSIVE_LOAD_SECTION_SIZE:
            self.streamed += PROGRESSIVE_LOAD_SECTION_SIZE
            return self._build(False)
        return False

    def finish(self) -> dict:
        """The final build: the rest of the file, the stream closed (GsError when it ended short), the SplatTree built."""
        self._build(True)
        return self.info

    def _open(self) -> bool:
        v = self.viewer
        cap = _stream_capacity(self.format, self._head, self.fileSize)
        if cap is None:
            return False
        v._sceneSources = []   # a single-scene mesh replaces any addSplatScenes mesh
        v.splatMesh = SplatMesh(dynamicMode=False, halfPrecisionCovariancesOnGPU=v.halfPrecisionCovariancesOnGPU, devicePixelRatio=v.devicePixelRatio,
                                antialiased=v.antialiased, maxScreenSpaceSplatSize=v.maxScreenSpaceSplatSize,
                                sphericalHarmonicsDegree=v.sphericalHarmonicsDegree, kernel2DSize=v.kernel2DSize)
        v.engine = Engine(max(cap, 1), device=v.device, distance_map_range=1 << v.splatSortDistanceMapPrecision, integer_based_sort=v.integerBasedSort,
                          dynamic_mode=False, max_width=v.renderWidth, max_height=v.renderHeight * v.maxViews, rank=v.rank, world_size=v.world_size,
                          ray_records=v.enableRaycast)
        v.splatMesh.engine = v.engine
        if self.transform16 is not None:
            v.splatMesh.sceneTransforms[0] = self.transform16
        self._stream = v.engine.open_stream(self.format, sh_degree=v.sphericalHarmonicsDegree, half_covariances=v.halfPrecisionCovariancesOnGPU,
                                            transform16=self.transform16)
        return True

    def _build(self, final: bool) -> bool:
        if self._stream is None and not self._open():
            if not final:
                return False
            raise N.GsError(N.GS_ERR_BAD_ARG, "addSplatSceneProgressive", f"the file ended inside its header ({self.received} bytes)")
        v, sm = self.viewer, self.viewer.splatMesh
        data, self._pending = b"".join(self._pending), []
        loaded = self._stream.append(data)
        info = self._stream.close() if final else self._stream.progress
        if not final and loaded == sm.getSplatCount():
            return False
        self.info = v._ksplat_info = info
        sm.sceneCenter = info["scene_center"]
        first = not self.builds
        sm.packed = PackedScene(None, None, None, min(v.sphericalHarmonicsDegree, info["sh_degree"]), None, loaded)
        v.splatRenderCount = loaded
        self.builds.append(loaded)
        if final:
            v._build_splat_tree()
            sm.finalBuild = True
        v._reveal_build(not first)
        return True
