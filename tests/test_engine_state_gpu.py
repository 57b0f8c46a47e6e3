"""One long-lived engine across scene uploads and frame-parameter changes.  The other frame tests upload one scene once and move the
camera; a Viewer reloads scenes, resizes, switches SH degree, composites, enters XR and moves between partial and full sorts on one
engine, and the frame graph is re-captured only when its key changes.  A seeded script of uploads and frames runs on one dynamic-mode
engine, and after every frame:
  1. the graph frame equals, bit for bit, the same frame with the graph off (and the two draw orders are equal): a kernel argument
     the graph captured that its key does not cover shows up here;
  2. a fresh engine given only the calls that define the current state (the uploads since the last from-0 upload of each buffer, and
     the SplatTree build) renders the same frame eagerly, bit for bit: state left over from an earlier scene shows up here;
  3. each mono frame is held to the f64 projection and blend bounds (tests/frame_f64.py), on windows above 1 Mpx; each half of a
     stereo frame equals the mono frame of its eye bit for bit, and those are held to the f64 bounds.
A CPU tally restates the kernel selection and shows that the script's frames reach every k_project instantiation and the 12 k_blend
instantiations without DEPTH; the view depth, multi-scene meshes and multi-view frames are the second script's
(tests/test_engine_state_mesh_gpu.py, whose tally covers both scripts together).  Small targeted tests beside the script name the
scene-index faults one by one."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np
import pytest

import frame_f64 as FF

N_SPLATS = 150_000
MAX_W, MAX_H = 8200, 2100          # a stereo frame of two radix-binned 4100x2100 eyes
BIG_FRAME = 1 << 20                # frames above this many pixels are blended on windows by the f64 check
N_SCENES = 4

# ---- the script ----------------------------------------------------------------------------------------------------------------------
# Uploads name their data by a seed: the scene of seed s is synthetic_scene(N_SPLATS, s) packed in the step's formats, and a partial
# upload takes rows [start, start + count) of it.  Scene indexes, when given, are seeded by the same seed.


@dataclass(frozen=True)
class Splats:
    """upload_splat_data of rows [start, start + count) of scene `seed` (count None: to the end)"""
    seed: int
    cov: str = "f32"          # f32 | f16
    sh: str = "none"          # none | f16 | u8 | f32
    deg: int = 0
    idx: bool = False         # with scene_indexes
    start: int = 0
    count: int | None = None


@dataclass(frozen=True)
class Centers:
    """upload_centers of rows [start, start + count) of the sorter centres of scene `seed`, with its scene indexes"""
    seed: int
    start: int = 0
    count: int | None = None


@dataclass(frozen=True)
class Ksplat:
    """upload_ksplat of scene `seed` written at a compression level (every splat kept), optionally with a static scene transform"""
    seed: int
    level: int
    deg: int
    half_cov: bool = False
    transform: bool = False


@dataclass(frozen=True)
class PlyFile:
    """upload_file of a handmade .ply from tests/golden"""
    name: str = "file_handmade_sh1.ply"
    deg: int = 1


@dataclass(frozen=True)
class Frame:
    w: int
    h: int
    fmt: str = "rgba8"        # rgba8 | rgba32f
    flip: bool = True
    render: int | None = None  # render_count (None: every uploaded splat)
    sort: int | None = None    # sort_count (None: render_count)
    index: str = "none"       # none | host | device (build_splat_tree + gather_for_sort)
    pre: bool = False         # precomputed distances
    comp: str | None = None   # composite inputs: host | device
    stereo: bool = False      # w is the whole frame: two eyes of w / 2
    scenes: int = 1           # scene_count of the uniforms
    cam: int = 0


# frame sizes: 16-px tiles, 32-px tiles binned by counting sort, radix binning (more than 256 coarse tiles at 32 px)
S16, S32, SRX = (1280, 720), (2600, 1500), (4100, 2100)
ST16, ST32, STRX = (1620, 600), (5200, 1500), (8200, 2100)    # stereo: eyes of 810x600, 2600x1500, 4100x2100
A, B = 90_000, N_SPLATS - 90_000

SCRIPT = [
    Splats(1, "f32", "none", 0, idx=True), Centers(1),
    Frame(*S16, "rgba8", True),
    Frame(*ST16, "rgba32f", False, stereo=True, scenes=4, cam=1),
    # the same count and formats, other contents and no scene indexes: the graph key cannot see this
    Splats(2, "f32", "none", 0),
    Frame(*S16, "rgba8", True, cam=1),
    Frame(*S16, "rgba8", False, cam=2),                       # the same frame but for flip_y
    Frame(*S32, "rgba32f", False, scenes=4, comp="host"),
    # a partial upload, a frame, its continuation and the same frame: only the uploaded count changes (the indexes reach past it)
    Splats(3, "f16", "f16", 1, idx=True, count=A),
    Frame(*S16, "rgba8", True, render=60_000, index="host", scenes=4, cam=2),
    Splats(3, "f16", "f16", 1, idx=True, start=A),
    Frame(*S16, "rgba8", True, render=60_000, index="host", scenes=4, cam=3),
    Centers(3),
    Frame(*ST32, "rgba8", True, stereo=True, scenes=4),
    Frame(*S16, "rgba32f", True, render=120_000, sort=50_000, index="host", scenes=4),
    Splats(4, "f32", "u8", 2, idx=True), Centers(4, count=A), Centers(4, start=A),
    Frame(*STRX, "rgba32f", True, stereo=True, scenes=4, cam=1),
    Frame(*SRX, "rgba8", False, scenes=4, cam=2),
    # the same count and formats again, from 0 without scene indexes: eager and graph frames must drop them
    Splats(5, "f32", "u8", 2),
    Frame(*SRX, "rgba8", False, scenes=4, cam=2),
    Splats(6, "f16", "f32", 2, count=A), Splats(6, "f16", "f32", 2, start=A, count=B),
    Frame(*S32, "rgba8", False, pre=True, scenes=4, comp="device"),
    Frame(*ST16, "rgba8", True, stereo=True, scenes=4, cam=2),
    Splats(7, "f32", "f16", 1),
    Frame(*STRX, "rgba8", False, stereo=True, cam=3),
    Frame(*S16, "rgba8", False, index="device", scenes=4),
    Splats(8, "f16", "u8", 1, idx=True), Centers(8),
    Frame(*ST32, "rgba32f", False, stereo=True, scenes=4, cam=3),
    Frame(*S32, "rgba32f", True, render=100_000, scenes=4, comp="device"),
    Splats(9, "f32", "f32", 1, idx=True, count=A), Splats(9, "f32", "f32", 1, idx=True, start=A),
    Frame(*ST16, "rgba32f", True, stereo=True, scenes=4),
    Frame(*SRX, "rgba32f", True, sort=60_000, scenes=4, cam=1),
    Splats(10, "f16", "none", 0),
    Frame(*STRX, "rgba8", True, stereo=True, scenes=4, cam=2),
    Frame(*S16, "rgba32f", False, comp="host", scenes=4, cam=3),
    # the same contents, count and formats with scene indexes added, and the same frame
    Splats(10, "f16", "none", 0, idx=True),
    Frame(*S16, "rgba32f", False, comp="host", scenes=4, cam=1),
    Ksplat(11, level=2, deg=2, transform=True),
    Frame(*S16, "rgba8", True, scenes=4),
    Ksplat(11, level=1, deg=1, half_cov=True),
    Frame(*ST32, "rgba8", True, stereo=True, cam=1),
    Frame(*S32, "rgba8", True, index="device", cam=2),
    Ksplat(12, level=0, deg=0),
    Frame(*SRX, "rgba32f", False, pre=True),
    Centers(12, start=A, count=B),
    Frame(*S16, "rgba32f", False, render=120_000, sort=30_000, cam=3),
    PlyFile(),
    Frame(*S16, "rgba32f", True, cam=4),
    Splats(13, "f16", "f32", 2, idx=True), Centers(13),
    Frame(*STRX, "rgba32f", False, stereo=True, scenes=4, cam=4),
    Frame(*S16, "rgba8", True, render=140_000, sort=70_000, index="host", scenes=4, comp="host"),
]


# ---- the kernel selection, restated (csrc/raster_kernels.cuh for_each_project / for_each_blend, frame_tiles) ----------------------------
def tile_px(w: int, h: int) -> int:
    """frame_tile_shift: 16-px tiles while the frame has at most 256 coarse tiles of 128x64 px, else 32 px."""
    return 16 if -(-w // 128) * -(-h // 64) <= 256 else 32


def radix_binned(w: int, h: int) -> bool:
    """The binning sorts instances by radix when the frame has more than kBinTiles (256) coarse tiles at its own tile edge."""
    t = tile_px(w, h)
    return -(-w // (8 * t)) * -(-h // (4 * t)) > 256


def raster_formats(script):
    """(cov, sh) storage formats the engine holds at each frame of the script: {frame position: (cov, sh)}"""
    state, out = None, {}
    for k, s in enumerate(script):
        if isinstance(s, Splats):
            state = (s.cov, s.sh if s.deg else "none")
        elif isinstance(s, Ksplat):     # SH kept at 8 bits at level 2, else at 16 (SplatMesh.js:1064-1066)
            state = ("f16" if s.half_cov else "f32", "none" if s.deg == 0 else ("u8" if s.level == 2 else "f16"))
        elif isinstance(s, PlyFile):
            state = ("f32", "f16" if s.deg else "none")
        elif isinstance(s, Frame):
            out[k] = state
    return out


def instantiations(script):
    """{frame position: (k_project key, k_blend key)}: k_project by covariance format, SH format and stereo; k_blend by frame format,
    tile edge of one view, composite (never in a stereo frame) and stereo."""
    out = {}
    for k, (cov, sh) in raster_formats(script).items():
        f = script[k]
        vw = f.w // 2 if f.stereo else f.w
        out[k] = ((cov, sh, f.stereo), (f.fmt, tile_px(vw, f.h), f.comp is not None and not f.stereo, f.stereo))
    return out


def test_script_reaches_every_kernel_instantiation():
    """CPU: the script's frames reach all 16 k_project and the 12 DEPTH = false k_blend instantiations, each binning path and tile edge in mono and
    stereo frames, and every index source, partial sorts, precomputed distances and both composite inputs."""
    got = instantiations(SCRIPT)
    proj = {p for p, _ in got.values()}
    blend = {b for _, b in got.values()}
    want_proj = {(c, s, st) for c in ("f32", "f16") for s in ("none", "f16", "u8", "f32") for st in (False, True)}
    want_blend = {(f, t, comp, st) for f in ("rgba8", "rgba32f") for t in (16, 32) for comp, st in ((False, False), (True, False), (False, True))}
    print(f"\nk_project {len(proj & want_proj)}/{len(want_proj)}, k_blend {len(blend & want_blend)}/{len(want_blend)}")
    assert proj == want_proj, sorted(want_proj - proj)
    assert blend == want_blend, sorted(want_blend - blend)
    frames = [s for s in SCRIPT if isinstance(s, Frame)]
    paths = {(f.stereo, tile_px(f.w // 2 if f.stereo else f.w, f.h), radix_binned(f.w // 2 if f.stereo else f.w, f.h)) for f in frames}
    assert paths == {(st, t, r) for st in (False, True) for t, r in ((16, False), (32, False), (32, True))}, paths
    assert {f.index for f in frames} == {"none", "host", "device"} and {f.comp for f in frames} == {None, "host", "device"}
    assert any(f.pre for f in frames) and any(f.sort is not None for f in frames) and any(f.render is not None for f in frames)
    assert {f.flip for f in frames} == {False, True} and any(f.scenes > 1 and f.stereo for f in frames)
    # every state change the script promises: each storage format from 0 with and without scene indexes, partial continuations that
    # start where the previous upload ended, every .ksplat level, and same-count same-format re-uploads
    ups = [s for s in SCRIPT if isinstance(s, Splats)]
    assert {u.cov for u in ups} == {"f32", "f16"} and {u.sh for u in ups} == {"none", "f16", "u8", "f32"} and {u.deg for u in ups} == {0, 1, 2}
    assert {u.idx for u in ups if u.start == 0} == {False, True} and {u.idx for u in ups if u.start > 0} == {False, True}
    assert {k.level for k in SCRIPT if isinstance(k, Ksplat)} == {0, 1, 2} and {k.transform for k in SCRIPT if isinstance(k, Ksplat)} == {False, True}
    assert any(isinstance(s, Centers) and s.start > 0 for s in SCRIPT) and any(isinstance(s, PlyFile) for s in SCRIPT)
    for i, s in enumerate(SCRIPT):
        if isinstance(s, (Splats, Centers)) and s.start > 0:
            prev = next(p for p in reversed(SCRIPT[:i]) if isinstance(p, (type(s), Ksplat, PlyFile)))
            end = N_SPLATS if isinstance(prev, (Ksplat, PlyFile)) else prev.start + (prev.count or N_SPLATS - prev.start)
            assert end == s.start or isinstance(prev, Ksplat), f"step {i}: a gap after the previous upload"


# ---- GPU side ------------------------------------------------------------------------------------------------------------------------
_raw = {}


def _raw_scene(seed, deg):
    from gaussiansplats3d_b200.scenes import synthetic_scene
    if (seed, deg) not in _raw:
        _raw[(seed, deg)] = synthetic_scene(N_SPLATS, seed=seed, kind="bonsai", sh_degree=deg)
    return _raw[(seed, deg)]


def _packed(s: Splats):
    from gaussiansplats3d_b200.scenes import pack_scene
    p = pack_scene(_raw_scene(s.seed, s.deg), half_covariances=s.cov == "f16", sh_format=s.sh if s.sh != "none" else "f16")
    return p.centers_colors, p.covariances, (p.sh if s.deg else None)


def _scene_indexes(seed, n=N_SPLATS):
    return np.random.default_rng(1000 + seed).integers(0, N_SCENES, n, dtype=np.uint32)


def _int_centers(seed):
    from gaussiansplats3d_b200.scenes import integer_centers
    return integer_centers(_raw_scene(seed, 0).centers)


def _ksplat_bytes(k: Ksplat):
    from gaussiansplats3d_b200 import ksplat as K
    raw = _raw_scene(k.seed, 2)
    sh = None if k.deg == 0 else raw.sh[:, : (3 if k.deg == 1 else 8)]
    return K.write(raw.centers, raw.scales, raw.rotations, raw.colors, sh, k.deg, compression_level=k.level, minimum_alpha=0)


def _static_transform():
    from gaussiansplats3d_b200 import three_math as TM
    return TM.compose((0.2, -0.1, 0.3), (0.0, 0.1305262, 0.0, 0.9914449), (1.1, 1.1, 1.1))


def _scene_transforms(rng):
    """Per-scene rigid transforms (column-major) of a dynamic mesh: small rotations and shifts, scene 0 included"""
    from gaussiansplats3d_b200 import three_math as TM
    xf = np.tile(np.eye(4, dtype=np.float32).reshape(16), 32)
    for s in range(N_SCENES):
        ax = rng.normal(0, 1, 3)
        ax /= np.linalg.norm(ax)
        a = rng.uniform(-0.15, 0.15)
        q = (*(ax * np.sin(a / 2)), np.cos(a / 2))
        xf[16 * s:16 * s + 16] = TM.compose(tuple(rng.normal(0, 0.3, 3)), q, (1.0, 1.0, 1.0)).astype(np.float32)
    return xf


@dataclass
class Model:
    """What the engine holds, kept on the host: the calls that define it and, for host uploads, the arrays it was uploaded from."""
    raster_calls: list = field(default_factory=list)
    sorter_calls: list = field(default_factory=list)
    cc: np.ndarray | None = None
    cov: np.ndarray | None = None
    sh: np.ndarray | None = None
    deg: int = 0
    idx: np.ndarray | None = None
    decoded: bool = False         # the raster state came from a file: the f64 check reads the decoded buffers back
    cov_f16: bool = False         # ... stored at these formats
    sh_u8: bool = False
    uploaded: int = 0
    sorted_splats: int = 0

    def apply(self, e, step, seq):
        """Run one upload step on engine e and record it."""
        from gaussiansplats3d_b200 import _native as N
        if isinstance(step, Splats):
            cc, cov, sh = _packed(step)
            n = (step.count or N_SPLATS - step.start)
            sl = slice(step.start, step.start + n)
            si = _scene_indexes(step.seed)[sl] if step.idx else None
            call = (seq, lambda x: x.upload_splat_data(cc[sl], cov[sl], None if sh is None else sh[sl], step.deg, scene_indexes=si, start=step.start))
            if step.start == 0:
                self.raster_calls = []
                self.cc, self.cov = np.zeros_like(cc), np.zeros_like(cov)
                self.sh = None if sh is None else np.zeros_like(sh)
                self.idx = None if si is None else np.zeros(N_SPLATS, np.uint32)
                self.deg, self.decoded, self.uploaded = step.deg, False, 0
            self.cc[sl], self.cov[sl] = cc[sl], cov[sl]
            if sh is not None:
                self.sh[sl] = sh[sl]
            if si is not None:
                self.idx[sl] = si
            self.uploaded = max(self.uploaded, step.start + n)
            self.raster_calls.append(call)
        elif isinstance(step, Centers):
            n = (step.count or N_SPLATS - step.start)
            sl = slice(step.start, step.start + n)
            c, si = _int_centers(step.seed)[sl], _scene_indexes(step.seed)[sl]
            call = (seq, lambda x: x.upload_centers(c, si, start=step.start))
            if step.start == 0:
                self.sorter_calls = []
            self.sorter_calls.append(call)
            self.sorted_splats = step.start + n
        else:
            if isinstance(step, Ksplat):
                data = _ksplat_bytes(step)
                xf = _static_transform() if step.transform else None
                call = (seq, lambda x: x.upload_ksplat(data, half_covariances=step.half_cov, transform16=xf))
            else:
                from pathlib import Path
                data = (Path(__file__).parent / "golden" / step.name).read_bytes()
                call = (seq, lambda x: x.upload_file(N.GS_FILE_PLY, data, sh_degree=step.deg))
            self.raster_calls, self.sorter_calls = [call], [call]
            self.decoded, self.deg, self.idx = True, step.deg, None
            self.cov_f16, self.sh_u8 = getattr(step, "half_cov", False), getattr(step, "level", 0) == 2
        info = call[1](e)
        if isinstance(step, (Ksplat, PlyFile)):
            self.uploaded = self.sorted_splats = info["splat_count"]

    def sh_is_u8(self):
        return self.deg > 0 and (self.sh_u8 if self.decoded else self.sh.dtype == np.uint8)

    def replay(self, f):
        """The calls that define the current state, in their original order, on a fresh engine f."""
        calls = {seq: c for seq, c in self.raster_calls + self.sorter_calls}
        for seq in sorted(calls):
            calls[seq](f)

    def arrays(self, e):
        """(centers_colors, covariances, sh, sh_degree, scene_indexes) of the scene for the f64 check"""
        from gaussiansplats3d_b200 import _native as N
        if not self.decoded:
            return self.cc, self.cov, self.sh, self.deg, self.idx
        n = self.uploaded
        cc = e.read_buffer(N.GS_BUF_CENTERS_COLORS, np.uint32, 4 * n).reshape(n, 4)
        cov = e.read_buffer(N.GS_BUF_COVARIANCES, np.float16 if self.cov_f16 else np.float32, 6 * n).reshape(n, 6)
        sh = None
        if self.deg:
            ncomp = 9 if self.deg == 1 else 24
            sh = e.read_buffer(N.GS_BUF_SH, np.uint8 if self.sh_u8 else np.float16, ncomp * n).reshape(n, ncomp)
        return cc, cov, sh, self.deg, None


@dataclass
class Rig:
    mvp: np.ndarray
    u: object                     # Uniforms of the frame (one eye's size for a stereo frame)
    eyes: tuple | None
    transforms: np.ndarray
    mv64: np.ndarray
    viewer: object


def _rig(f: Frame, deg: int, sh_u8_ranges: bool):
    """The camera, uniforms, eyes and per-scene parameters of frame f (seeded by its camera number)"""
    import test_stereo_gpu as ST
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.engine import Uniforms
    rng = np.random.default_rng(500 + f.cam)
    head = tuple(rng.normal(0, 0.25, 3)) if f.cam else (0.0, 0.0, 0.0)
    vw = f.w // 2 if f.stereo else f.w
    viewer, cams = ST._rig(vw, f.h, head)
    xf = _scene_transforms(rng)
    P = viewer.projectionMatrix
    kw = {}
    if f.scenes > 1:
        kw = dict(scene_opacity=np.r_[1.0, 0.55, 0.005, 0.8, np.ones(28)].astype(np.float32),
                  scene_visibility=np.r_[1, 1, 1, 0, np.ones(28)].astype(np.int32))
    if sh_u8_ranges:
        kw.update(sh8_min=np.r_[-1.5, -0.6, -0.9, -1.2, np.full(28, -1.5)].astype(np.float32),
                  sh8_max=np.r_[1.5, 0.7, 0.5, 1.1, np.full(28, 1.5)].astype(np.float32))
    u = Uniforms(model_view=viewer.matrixWorldInverse.astype(np.float32), projection=P.astype(np.float32),
                 camera_position=viewer.position.astype(np.float32), focal=(P[0] * 0.5 * vw, P[5] * 0.5 * f.h), viewport=(vw, f.h),
                 sh_degree=deg, dynamic_mode=1, scene_transforms=xf, view_matrix=viewer.matrixWorldInverse.astype(np.float32),
                 scene_count=f.scenes, **kw)
    mvp = TM.multiply(P, viewer.matrixWorldInverse).astype(np.float32)
    eyes = ST._eyes(cams, dynamic=True) if f.stereo else None
    return Rig(mvp, u, eyes, xf, np.asarray(viewer.matrixWorldInverse, np.float64), viewer)


def _composite_inputs(f: Frame, seed):
    """An opaque pass of frame f's shape: a patterned colour and a depth that rises across x through the splats' window depths"""
    rng = np.random.default_rng(seed)
    rgba8 = f.fmt == "rgba8"
    c = rng.random((f.h, f.w, 4), dtype=np.float32)
    c[..., 3] = 1.0
    color = np.floor(c * 255 + 0.5).astype(np.uint8) if rgba8 else c
    depth = np.broadcast_to(np.linspace(0.96, 1.0, f.w, dtype=np.float32), (f.h, f.w)).copy()
    if f.comp == "device":
        import torch
        return color, depth, torch.from_numpy(color).cuda(), torch.from_numpy(depth).cuda()
    return color, depth, color, depth


@dataclass
class FrameArgs:
    f: Frame
    rig: Rig
    render: int
    sort: int
    indexes: np.ndarray | None
    pre: np.ndarray | None
    dest: tuple                   # (host colour, host depth, what the engine is given: colour, depth) or ()


def _gather(e, args_or_rig):
    """build_splat_tree + gather_for_sort on engine e: (device pointer of the gathered list, its length)"""
    from gaussiansplats3d_b200 import _native as N
    e.build_splat_tree()
    n = e.gather_for_sort(args_or_rig.mv64, 0.6, 0.7)
    return e.buffer_dev(N.GS_BUF_INDEXES_TO_SORT)[0], n


def _run_frame(e, a: FrameArgs, graph: bool, index_dev=None):
    """gs_frame of a on engine e with the frame graph on or off: (frame, draw order)"""
    from gaussiansplats3d_b200 import _native as N
    f = a.f
    fmt = N.GS_FRAME_RGBA8 if f.fmt == "rgba8" else N.GS_FRAME_RGBA32F
    e.set_graph_enabled(graph)
    try:
        sp = e._sort_params(a.rig.mvp, a.sort, a.render, a.indexes, a.rig.transforms, a.pre, index_dev)
        dc, dd = (a.dest[2], a.dest[3]) if a.dest else (None, None)
        rp, _ = e._render_params(f.w, f.h, a.render, None, fmt, f.flip, dc, dd, a.rig.eyes)
        u = a.rig.u.to_c()
        frame = np.empty((f.h, f.w, 4), np.uint8 if fmt == N.GS_FRAME_RGBA8 else np.float32)
        order = np.empty(a.render, np.uint32)
        N.check(e._lib.gs_frame(e._h, C.byref(sp), C.byref(u), C.byref(rp), N.ptr(order), N.ptr(frame)), "gs_frame")
        return frame, order
    finally:
        e.set_graph_enabled(True)


def _new_engine():
    from gaussiansplats3d_b200.engine import Engine
    return Engine(N_SPLATS, max_width=MAX_W, max_height=MAX_H, dynamic_mode=True)


def _differ(a, b):
    d = np.flatnonzero(np.any(a.view(np.uint8).reshape(a.shape[0], a.shape[1], -1) != b.view(np.uint8).reshape(b.shape[0], b.shape[1], -1), axis=-1))
    return f"{d.size} pixels differ, first (row, col) {[(int(i // a.shape[1]), int(i % a.shape[1])) for i in d[:3]]}"


def _f64(label, e, a: FrameArgs, u, w, frame, order, arrays):
    cc, cov, sh, deg, idx = arrays
    f = a.f
    dc, dd = (a.dest[0], a.dest[1]) if (a.dest and not f.stereo) else (None, None)
    win = FF.windows(w, f.h) if w * f.h > BIG_FRAME else None
    FF.check_frame(label, e, u, w, f.h, a.render, cc, cov, sh, deg, idx, got=frame if f.fmt == "rgba32f" else None,
                   got8=frame if f.fmt == "rgba8" else None, order=order, windows=win, flip_y=f.flip, dest_color=dc, dest_depth=dd)


@pytest.mark.gpu
def test_scripted_state_sequence_on_one_engine(gs):
    import test_stereo_gpu as ST
    rng = np.random.default_rng(2026)
    model = Model()
    e = _new_engine()
    frames = 0
    try:
        for k, step in enumerate(SCRIPT):
            if not isinstance(step, Frame):
                model.apply(e, step, k)
                continue
            f = step
            label = f"step {k} {f}"
            rig = _rig(f, model.deg, model.sh_is_u8())
            limit = min(model.uploaded, model.sorted_splats)
            render = limit if f.render is None else min(f.render, limit)
            indexes = None
            if f.index == "host":
                indexes = np.sort(rng.choice(limit, render, replace=False)).astype(np.uint32)[rng.permutation(render)]
            pre = rng.integers(-2_000_000, 2_000_000, model.sorted_splats, dtype=np.int64).astype(np.int32) if f.pre else None
            dest = _composite_inputs(f, k) if f.comp else ()
            a = FrameArgs(f, rig, render, render, indexes, pre, dest)
            dev_idx = None
            if f.index == "device":
                dev_idx, a.render = _gather(e, rig)
                assert 0 < a.render < limit, f"{label}: the gather should keep some splats and drop others ({a.render} of {limit})"
            a.sort = a.render if f.sort is None else min(f.sort, a.render)
            # 1. graph frame == eager frame on the same engine
            got, order = _run_frame(e, a, True, dev_idx)
            assert e.timings()["tile_instances"] > 0, label
            eager, eager_order = _run_frame(e, a, False, dev_idx)
            assert np.array_equal(order, eager_order), f"{label}: the graph frame's draw order differs from the eager frame's"
            assert got.tobytes() == eager.tobytes(), f"{label}: the graph frame differs from the eager frame: {_differ(got, eager)}"
            # 2. a fresh engine given only the calls that define the state
            with _new_engine() as fresh:
                model.replay(fresh)
                fdev = None
                if f.index == "device":
                    fdev, n = _gather(fresh, rig)
                    assert n == a.render, f"{label}: a fresh engine gathers {n} splats, this one {a.render}"
                want, want_order = _run_frame(fresh, a, False, fdev)
            assert np.array_equal(order, want_order), f"{label}: the draw order differs from a fresh engine's"
            assert got.tobytes() == want.tobytes(), f"{label}: the frame differs from a fresh engine's: {_differ(got, want)}"
            # 3. f64 bounds (stereo: the halves are the mono eye frames, and those are checked)
            arrays = model.arrays(e)
            fmt = gs._native.GS_FRAME_RGBA8 if f.fmt == "rgba8" else gs._native.GS_FRAME_RGBA32F
            if f.stereo:
                vw = f.w // 2
                for i, eye in enumerate(rig.eyes):
                    ue = ST._substituted(rig.u, eye)
                    mono = e.render(ue, vw, f.h, a.render, order, frame_format=fmt, flip_y=f.flip).copy()
                    half = got[:, i * vw:(i + 1) * vw]
                    assert np.array_equal(half.view(np.uint8), mono.view(np.uint8)), f"{label}: eye {i} differs from its mono frame: {_differ(half, mono)}"
                    _f64(f"{label} eye {i}", e, a, ue, vw, mono, order, arrays)
            else:
                _f64(label, e, a, rig.u, f.w, got, order, arrays)
            frames += 1
    finally:
        e.close()
    assert frames == sum(isinstance(s, Frame) for s in SCRIPT)


# ---- targeted cases ------------------------------------------------------------------------------------------------------------------
T_SPLATS, T_W, T_H = 60_000, 1280, 720


def _t_scene(seed=21):
    from gaussiansplats3d_b200.scenes import integer_centers, pack_scene, synthetic_scene
    raw = synthetic_scene(T_SPLATS, seed=seed, kind="bonsai", sh_degree=1)
    return raw, pack_scene(raw), _scene_indexes(seed, T_SPLATS)


def _t_engine(gs, packed=None, **upload):
    e = gs.Engine(T_SPLATS, max_width=T_W, max_height=T_H, dynamic_mode=True)
    if packed is not None:
        e.upload_splat_data(packed.centers_colors, packed.covariances, packed.sh, packed.sh_degree, **upload)
        e.upload_centers(packed.int_centers, np.zeros(T_SPLATS, np.uint32))
    return e


def _t_frame(e, graph=True, render=T_SPLATS):
    """One 4-scene frame: scene 3 hidden, scene 2 below the opacity cull, scenes 1 and 3 moved: scene indexes change the picture"""
    f = Frame(T_W, T_H, "rgba8", True, scenes=N_SCENES, cam=1)
    a = FrameArgs(f, _rig(f, 1, False), render, render, None, None, ())
    return _run_frame(e, a, graph)


def _same(got, want, what):
    frame, order = got
    wframe, worder = want
    assert np.array_equal(order, worder), f"{what}: draw orders differ"
    assert frame.tobytes() == wframe.tobytes(), f"{what}: {_differ(frame, wframe)}"


@pytest.mark.gpu
def test_graph_frame_sees_scene_indexes_added_by_a_same_format_reupload(gs):
    raw, p, si = _t_scene()
    with _t_engine(gs, p) as e, _t_engine(gs, p, scene_indexes=si) as fresh:
        before = _t_frame(e)
        e.upload_splat_data(p.centers_colors, p.covariances, p.sh, p.sh_degree, scene_indexes=si)
        got = _t_frame(e)
        assert before[0].tobytes() != _t_frame(fresh, False)[0].tobytes(), "scene indexes do not change this frame: the test would see nothing"
        _same(got, _t_frame(e, graph=False), "graph frame after scene indexes were added vs the eager frame")
        _same(got, _t_frame(fresh, False), "graph frame after scene indexes were added vs a fresh engine")


@pytest.mark.gpu
def test_graph_frame_after_a_ksplat_upload_drops_host_scene_indexes(gs):
    from gaussiansplats3d_b200 import ksplat as K
    raw, p, si = _t_scene()
    data = K.write(raw.centers, raw.scales, raw.rotations, raw.colors, raw.sh, 1, compression_level=0, minimum_alpha=0)
    with _t_engine(gs, p, scene_indexes=si) as e, _t_engine(gs) as fresh:
        with_idx = _t_frame(e)
        assert e.upload_ksplat(data)["splat_count"] == T_SPLATS
        fresh.upload_ksplat(data)
        got = _t_frame(e)
        assert with_idx[0].tobytes() != _t_frame(fresh, False)[0].tobytes(), "scene indexes do not change this frame: the test would see nothing"
        _same(got, _t_frame(e, graph=False), "graph frame after the .ksplat upload vs the eager frame")
        _same(got, _t_frame(fresh, False), "graph frame after the .ksplat upload vs a fresh engine")


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_reupload_from_zero_without_scene_indexes_drops_them(gs, graph):
    raw, p, si = _t_scene()
    with _t_engine(gs, p, scene_indexes=si) as e, _t_engine(gs, p) as fresh:
        with_idx = _t_frame(e, graph)
        e.upload_splat_data(p.centers_colors, p.covariances, p.sh, p.sh_degree)
        got = _t_frame(e, graph)
        want = _t_frame(fresh, False)
        assert with_idx[0].tobytes() != want[0].tobytes(), "scene indexes do not change this frame: the test would see nothing"
        _same(got, want, f"{'graph' if graph else 'eager'} frame after a from-0 upload without scene indexes vs a fresh engine")


@pytest.mark.gpu
@pytest.mark.parametrize("first_has_indexes", [True, False], ids=["with-then-without", "without-then-with"])
def test_partial_uploads_must_agree_on_scene_indexes(gs, first_has_indexes):
    N = gs._native
    raw, p, si = _t_scene()
    a = T_SPLATS // 3
    first = dict(scene_indexes=si[:a]) if first_has_indexes else {}
    second = {} if first_has_indexes else dict(scene_indexes=si[a:])
    sh = p.sh
    with _t_engine(gs) as e:
        e.upload_centers(p.int_centers, np.zeros(T_SPLATS, np.uint32))
        e.upload_splat_data(p.centers_colors[:a], p.covariances[:a], sh[:a], 1, **first)
        with pytest.raises(N.GsError) as ei:
            e.upload_splat_data(p.centers_colors[a:], p.covariances[a:], sh[a:], 1, start=a, **second)
        assert ei.value.code == N.GS_ERR_BAD_ARG and "scene_indexes" in str(ei.value), str(ei.value)
        got = _t_frame(e, render=a)
        with _t_engine(gs) as fresh:          # the refused call left the scene as it was: the first upload alone
            fresh.upload_centers(p.int_centers, np.zeros(T_SPLATS, np.uint32))
            fresh.upload_splat_data(p.centers_colors[:a], p.covariances[:a], sh[:a], 1, **first)
            _same(got, _t_frame(fresh, False, render=a), "frame after a refused partial upload vs a fresh engine given the first upload")
        # partial uploads that agree equal one whole upload
        e.upload_splat_data(p.centers_colors[:a], p.covariances[:a], sh[:a], 1, **({"scene_indexes": si[:a]} if first_has_indexes else {}))
        e.upload_splat_data(p.centers_colors[a:], p.covariances[a:], sh[a:], 1, start=a, **({"scene_indexes": si[a:]} if first_has_indexes else {}))
        got = _t_frame(e)
    with _t_engine(gs, p, **({"scene_indexes": si} if first_has_indexes else {})) as whole:
        _same(got, _t_frame(whole, False), "two agreeing partial uploads vs one whole upload")
