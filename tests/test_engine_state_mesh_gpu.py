"""One long-lived engine across multi-scene meshes, optimized and streamed loads, refused uploads, multi-view and pipelined frames and
depth planes: the second state script.  tests/test_engine_state_gpu.py holds one engine to host and single-file uploads with mono and
stereo frames; this script runs the same kind of engine (dynamic mode, 8200x2100 at most, with ray records) through what has joined the
engine since: gs_upload_scenes, gs_upload_file_optimized, gs_stream_*, refused uploads, SplatTree forests, gs_compute_bounding_box,
gs_raycast, gs_frame_views, gs_frame_begin / gs_frame_end, gs_frame_async and the view depth.  After every frame:
  1. the graph frame equals the same frame with the graph off, bit for bit: colour, depth plane and every view's draw order;
  2. a fresh engine given only the calls that define the current state renders the same frame eagerly, bit for bit (an upload_scenes or
     upload_file_optimized call, or an opened stream, restarts both call lists; every append is a call; a refused call is none);
  3. the frame is within the f64 bounds: a mono frame's colour (tests/frame_f64.py) and depth (tests/depth_f64.py); each band of a
     multi-view frame equals gs_render of its camera with its view's draw order (colour and depth), each view's order is the reference
     sorter's, and every band of a multi-view frame up to 1 Mpx (else three) is held to the f64 bounds; each half of a stereo frame is
     the mono frame of its eye.  A multi-scene mesh's scene indexes are restated from its scenes' splat counts, not read back.
A pipelined pair and an asynchronous frame each equal gs_frame of the same inputs, and GS_BUF_DEPTH is the plane of the last frame that
asked for depth.  A refused upload leaves the model unchanged, and the graph frame after it equals the frame before it.
A CPU tally restates the kernel selection of both scripts together against the template parameter lists and instantiation macros read
from the sources."""
from __future__ import annotations

import ctypes as C
import dataclasses
import gzip
import re
from dataclasses import dataclass, field
from pathlib import Path

import numpy as np
import pytest

import test_engine_state_gpu as ST1
from test_engine_state_gpu import Centers, Frame, FrameArgs, Ksplat, Model, PlyFile, Splats, _differ, _rig

HERE = Path(__file__).resolve().parent
GOLDEN = HERE / "golden"
CSRC = HERE.parent / "gaussiansplats3d_b200" / "csrc"
N_SPLATS = ST1.N_SPLATS
PLY, SPLAT, KSPLAT, SPZ = 1, 2, 3, 4


# ---- the script ----------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Src:
    """One scene's file: a synthetic bonsai scene of `n` splats (seed), or rows [lo, hi) of it, written as .ksplat at `level`, INRIA .ply,
    .splat or .spz, or generated on the GPU as a .ksplat of several sections ("gen_ksplat"); a synthetic PlayCanvas .ply ("pcply"); or a
    fixture of tests/golden ("golden", by name).  optimized: load it through the generator."""
    kind: str
    seed: int = 0
    n: int = 0
    deg: int = 0
    level: int = 0
    name: str = ""
    optimized: bool = False
    rows: tuple = ()          # (lo, hi): only rows [lo, hi) of the synthetic scene
    sections: int = 1         # "gen_ksplat": a .ksplat of this many sections generated from the scene's .ply (level `level`)


@dataclass(frozen=True)
class Scenes:
    """upload_scenes(srcs, sh_degree=2)"""
    srcs: tuple


@dataclass(frozen=True)
class Optimized:
    """upload_file_optimized of a synthetic INRIA .ply at a compression level"""
    seed: int
    n: int
    deg: int
    level: int


@dataclass(frozen=True)
class Open:
    """open_stream of a file; Append(upto) then sends its bytes up to the fraction `upto` (cut at a seeded byte), Close() finishes it"""
    src: Src


@dataclass(frozen=True)
class Append:
    upto: float


@dataclass(frozen=True)
class Close:
    pass


@dataclass(frozen=True)
class Refused:
    """An upload that must fail with `code`, leaving the engine as it was"""
    what: str       # ksplat_truncated | scenes_33 | over_capacity | v2_in_file_order | spz_stream | scene0_bad | scene2_bad | transform_dynamic
    code: str


@dataclass(frozen=True)
class Box:
    """compute_bounding_box of the whole mesh and of scene 0, through the frame's scene transforms"""


@dataclass(frozen=True)
class Ray:
    """build_splat_tree + raycast from the bonsai camera"""


@dataclass(frozen=True)
class MFrame(Frame):
    depth: bool = False       # the view depth too
    views: int = 0            # > 0: a gs_frame_views frame of this many w x h cameras, stacked
    mode: str = "sync"        # sync | async (gs_frame_async + gs_synchronize, read back through GS_BUF_FRAME / GS_BUF_DEPTH)


@dataclass(frozen=True)
class Pipe:
    """gs_frame_begin(a), gs_frame_begin(b), gs_frame_end twice: a on one frame-buffer parity, b on the other"""
    a: MFrame
    b: MFrame


S16, S32, SRX = ST1.S16, ST1.S32, ST1.SRX
ST16, ST32, STRX = ST1.ST16, ST1.ST32, ST1.STRX
MV3, MV8, MV16 = (1280, 700), (480, 256), (256, 128)          # multi-view sizes: V bands of w x h within 2100 rows
MV2, MV2RX = (1920, 1050), (8200, 1050)                       # MV2RX: each band radix-binned (297 coarse tiles of 32 px)


def K(seed, n, deg, level):
    return Src("ksplat", seed, n, deg, level)


def P(seed, n, deg):
    return Src("ply", seed, n, deg)


def G(name, optimized=False):
    return Src("golden", name=name, optimized=optimized)


# SH 0 (the .splat and PlayCanvas scenes have none)
MESH3 = (K(31, 40_000, 2, 1), P(32, 50_000, 1), Src("splat", 33, 30_000), Src("pcply", 35, 2048))


def _split(*cuts, seed=45, n=90_000):
    """One synthetic scene's rows as .ply files cut at `cuts`: meshes of the same splats in the same order, split elsewhere"""
    edges = (0, *cuts, n)
    return tuple(Src("ply", seed, n, 1, rows=(lo, hi)) for lo, hi in zip(edges, edges[1:]))


SPLIT_A, SPLIT_B = _split(30_000, 60_000), _split(10_000, 75_000)
GEN_KSPLAT = Src("gen_ksplat", 46, 60_000, 2, 2, sections=2)

SCRIPT = [
    Scenes(MESH3),
    # two frames whose graph keys differ in depth alone: a graph captured without depth must not replay for the second
    MFrame(*S16, "rgba8", True, scenes=4),
    MFrame(*S16, "rgba8", True, scenes=4, depth=True, cam=1),
    MFrame(*MV3, "rgba8", True, scenes=4, views=3, cam=1),
    MFrame(*ST32, "rgba32f", False, stereo=True, scenes=4, depth=True),
    # mesh -> host upload of the same count and formats without scene indexes (the sorter keeps the mesh's centres) -> the mesh again:
    # each frame's graph key differs from the one before it in rs.have_scene_idx alone
    MFrame(*S16, "rgba8", True, scenes=4, cam=3),
    Splats(2, "f32", "none", 0, count=122_048),
    MFrame(*S16, "rgba8", True, scenes=4, cam=1),
    Scenes(MESH3),
    MFrame(*S16, "rgba8", True, scenes=4, cam=2),
    Refused("ksplat_truncated", "GS_ERR_BAD_ARG"),
    # the same splats in the same order, re-uploaded with another scene split: only the scene indexes differ, and the graph replays
    Scenes(SPLIT_A),
    MFrame(*S16, "rgba8", True, scenes=4, comp="host", depth=True, cam=2),
    Scenes(SPLIT_B),
    MFrame(*S16, "rgba8", True, scenes=4, comp="host", depth=True, cam=2),
    Splats(3, "f16", "u8", 2, idx=True), Centers(3),
    MFrame(*MV2, "rgba32f", True, scenes=4, depth=True, views=2, cam=3),
    # a level-2 scene holds the mesh's SH at 8 bits; a .ply at SH 3 and a .spz beside it
    Scenes((K(34, 60_000, 2, 2), G("file_handmade_sh3.ply"), Src("spz", 44, 20_000, 2))),
    MFrame(*SRX, "rgba8", False, scenes=4, depth=True, cam=2),
    Refused("scenes_33", "GS_ERR_BAD_ARG"),
    # a graph on each frame-buffer parity, then the view buffers grow (16 views, more than any frame before), then each parity's key
    # again: both graphs must be re-captured, not replayed on the moved buffers
    Pipe(MFrame(*S16, "rgba8", True, scenes=4, cam=3), MFrame(800, 450, "rgba8", True, scenes=4, depth=True, cam=4)),
    MFrame(*MV16, "rgba8", True, scenes=4, views=16, depth=True),
    Pipe(MFrame(*S16, "rgba8", True, scenes=4, cam=1), MFrame(800, 450, "rgba8", True, scenes=4, depth=True, cam=2)),
    Box(), Ray(),
    MFrame(*S16, "rgba32f", False, scenes=4, index="device", comp="device", depth=True, cam=1),
    Refused("scene0_bad", "GS_ERR_BAD_ARG"),
    Refused("scene2_bad", "GS_ERR_CAPACITY"),
    Refused("transform_dynamic", "GS_ERR_BAD_ARG"),
    MFrame(*ST16, "rgba8", True, stereo=True, scenes=4, cam=4),
    # mesh -> host upload with scene indexes -> one-scene mesh
    Splats(4, "f32", "none", 0, idx=True), Centers(4),
    MFrame(*MV8, "rgba8", True, scenes=4, views=8, cam=2),
    Scenes((P(36, 70_000, 2),)),
    MFrame(*S32, "rgba8", False, scenes=4, comp="host", depth=True, cam=3),
    # pipelined pairs: depth on one parity only, other sizes on the other; then the parities swap keys
    Pipe(MFrame(*S16, "rgba8", True, scenes=4, depth=True, cam=1), MFrame(640, 360, "rgba32f", True, scenes=4, cam=2)),
    Pipe(MFrame(640, 360, "rgba32f", True, scenes=4, cam=3), MFrame(*S16, "rgba8", True, scenes=4, depth=True, cam=4)),
    Optimized(37, 80_000, 2, 1),
    MFrame(*S16, "rgba8", True, scenes=4, depth=True, mode="async", cam=1),
    Refused("over_capacity", "GS_ERR_CAPACITY"),
    MFrame(*MV2RX, "rgba8", True, scenes=4, views=2, depth=True),
    Optimized(38, 60_000, 1, 2),
    MFrame(*STRX, "rgba8", True, stereo=True, scenes=4, depth=True, cam=2),
    Box(), Ray(),
    # streams: a .ply closed, a .splat left open and replaced by a from-0 upload, a two-section .ksplat cut inside section 1 and closed
    Open(P(39, 50_000, 1)), Append(0.3), MFrame(*S16, "rgba8", True, depth=True, cam=1), Append(0.8),
    MFrame(*MV3, "rgba8", True, views=3, cam=2), Append(1.0), Close(),
    MFrame(*S16, "rgba8", True, index="device", cam=3),
    Refused("v2_in_file_order", "GS_ERR_BAD_ARG"),
    Open(Src("splat", 40, 40_000)), Append(0.5), MFrame(*S32, "rgba32f", True, comp="device", depth=True, cam=4),
    Scenes((G("file_handmade_sh2.ply"), G("inriav2_codebook_sh2.ply", True), K(41, 50_000, 1, 0))),
    MFrame(*S16, "rgba8", True, scenes=4, depth=True, cam=1),
    Refused("spz_stream", "GS_ERR_BAD_ARG"),
    Open(GEN_KSPLAT), Append(0.75), MFrame(*S16, "rgba8", True, cam=2), Append(1.0), Close(),
    MFrame(*S16, "rgba32f", False, depth=True, cam=3),
    Scenes(MESH3),
    MFrame(*SRX, "rgba32f", True, scenes=4, index="device", depth=True, cam=4),
    MFrame(*MV3, "rgba8", True, scenes=4, views=3, depth=True, cam=1),
]


# ---- the kernel selection of both scripts, restated against the sources ---------------------------------------------------------------
def _template_params(src: str, kernel: str) -> list:
    """The template parameter names of `kernel`, as declared before its __global__ definition"""
    m = re.search(r"template <([^>]*)>\s*__global__[^\n]*\n\s*" + kernel + r"\(", src)
    assert m, kernel
    return [p.split("=")[0].split()[-1] for p in m.group(1).split(",")]


def _instances():
    """{kernel: set of instantiated template argument tuples} from for_each_project / for_each_blend (GS_PROJ / GS_BLENDS invocations)
    and from decode_section's k_ksplat_decode<...> launches"""
    raster = (CSRC / "raster_kernels.cuh").read_text()
    engine = (CSRC / "engine.cu").read_text()
    ksplat = (CSRC / "ksplat_kernels.cuh").read_text()
    truth = {"true": True, "false": False}
    proj_macro = re.search(r"#define GS_PROJ\(C, ST\)(.*?)\n\s*GS_PROJ\(", raster, re.S).group(1)
    sh_fmts = re.findall(r"k_project<C, (GS_SH_\w+), ST>", proj_macro)
    proj = {(truth[c], {"GS_SH_NONE": "none", "GS_SH_F16": "f16", "GS_SH_U8": "u8", "GS_SH_F32": "f32"}[s], truth[st])
            for c, st in re.findall(r"GS_PROJ\((\w+), (\w+)\);", raster) for s in sh_fmts}
    blend_macro = re.search(r"#define GS_BLEND\(S, COMP, ST, D\)(.*?)#define GS_BLENDS", raster, re.S).group(1)
    fmts = re.findall(r"k_blend<GS_FRAME_(\w+), S, COMP, ST, D>", blend_macro)
    blends_macro = re.search(r"#define GS_BLENDS\(D\)(.*?)\n\s*GS_BLENDS\(", raster, re.S).group(1)
    per = re.findall(r"GS_BLEND\((\d), (\w+), (\w+), D\)", blends_macro)
    blend = {(f.lower(), 16 * int(sc), truth[comp], truth[st], truth[d]) for d in re.findall(r"GS_BLENDS\((\w+)\);", raster)
             for sc, comp, st in per for f in fmts}
    decode = {(truth[x], truth[m]) for x, m in re.findall(r"k_ksplat_decode<(\w+), (\w+)>", engine)}
    params = dict(k_project=_template_params(raster, "k_project"), k_blend=_template_params(raster, "k_blend"),
                  k_ksplat_decode=_template_params(ksplat, "k_ksplat_decode"))
    return params, dict(k_project=proj, k_blend=blend, k_ksplat_decode=decode)


def _raster_state(step, state):
    """(cov, sh storage, k_ksplat_decode key or None) after an upload step"""
    if isinstance(step, Splats):
        return (step.cov, step.sh if step.deg else "none", None)
    if isinstance(step, Ksplat):     # SH kept at 8 bits at level 2, else at 16 (SplatMesh.js:1064-1066)
        return ("f16" if step.half_cov else "f32", "none" if step.deg == 0 else ("u8" if step.level == 2 else "f16"), (step.transform, False))
    if isinstance(step, PlyFile):
        return ("f32", "f16" if step.deg else "none", (False, False))
    if isinstance(step, Scenes):     # the lowest degree, the highest level; several scenes decode with MS
        deg = min(_src_degree(s) for s in step.srcs)
        u8 = any(_src_level(s) == 2 for s in step.srcs)
        return ("f32", "none" if deg == 0 else ("u8" if u8 else "f16"), (False, len(step.srcs) > 1))
    if isinstance(step, Optimized):
        return ("f32", "none" if step.deg == 0 else ("u8" if step.level == 2 else "f16"), (False, False))
    if isinstance(step, Open):
        deg, level = _src_degree(step.src), _src_level(step.src)
        return ("f32", "none" if deg == 0 else ("u8" if level == 2 else "f16"), (False, False))
    return state


_GOLDEN_DEG = {"file_handmade_sh2.ply": 2, "file_handmade_sh3.ply": 2, "inriav2_codebook_sh2.ply": 2}


def _src_degree(s: Src) -> int:
    """The scene's SH degree at sphericalHarmonicsDegree 2"""
    if s.kind == "golden":
        return _GOLDEN_DEG[s.name]
    return 0 if s.kind in ("splat", "pcply") else min(s.deg, 2)


def _src_level(s: Src) -> int:
    if s.kind == "golden":
        return 2 if "_l2_" in s.name else 0
    return s.level if s.kind in ("ksplat", "gen_ksplat") else 0


def _frames(script):
    """(position, frame) of every frame of a script, the two of a pipelined pair at the pair's position"""
    for k, s in enumerate(script):
        if isinstance(s, Pipe):
            yield k, s.a
            yield k, s.b
        elif isinstance(s, Frame):
            yield k, s


def _reached(script):
    """(k_project keys, k_blend keys, k_ksplat_decode keys, binning paths (tile px, radix, depth)) the script's frames reach"""
    state, proj, blend, decode, paths = None, set(), set(), set(), set()
    for s in script:
        new = _raster_state(s, state)
        if new is not state and not isinstance(s, (Centers, Refused, Box, Ray, Append, Close)):
            state = new
            if new[2] is not None:
                decode.add(new[2])
    state = None
    pos = {}
    for k, s in enumerate(script):
        if not isinstance(s, (Centers, Refused, Box, Ray, Append, Close, Frame, Pipe)):
            state = _raster_state(s, state)
        pos[k] = state
    for k, f in _frames(script):
        cov, sh, _ = pos[k]
        views = f.stereo or getattr(f, "views", 0) > 0
        vw = f.w // 2 if f.stereo else f.w
        depth = getattr(f, "depth", False)
        t = ST1.tile_px(vw, f.h)
        proj.add((cov == "f16", sh, views))
        blend.add((f.fmt, t, f.comp is not None and not views, views, depth))
        paths.add((t, ST1.radix_binned(vw, f.h), depth))
    return proj, blend, decode, paths


def test_both_scripts_reach_every_kernel_instantiation():
    """CPU: the two state scripts together reach every k_project (COVF16 x SHFMT x VIEWS), k_blend (format x tile edge x {plain,
    composite, views} x DEPTH) and k_ksplat_decode<XF, MS> instantiation the sources declare, bar k_ksplat_decode<true, true>: a scene
    transform baked into a multi-scene mesh, which a dynamic engine refuses (this script's Refused("transform_dynamic") step).  Each
    binning path is reached with depth on and off, and each upload entry has a graph frame after it."""
    params, inst = _instances()
    assert params == dict(k_project=["COVF16", "SHFMT", "VIEWS"], k_blend=["FORMAT", "S", "COMPOSITE", "VIEWS", "DEPTH"],
                          k_ksplat_decode=["XF", "MS"]), f"a kernel's template parameters changed: restate its selection here: {params}"
    assert (len(inst["k_project"]), len(inst["k_blend"]), len(inst["k_ksplat_decode"])) == (16, 24, 4), {k: len(v) for k, v in inst.items()}
    p1, b1, d1, paths1 = _reached(ST1.SCRIPT)
    p2, b2, d2, paths2 = _reached(SCRIPT)
    # blend keys: (format, tile edge, composite, views, depth); the first script's frames have no depth
    proj, blend, decode = p1 | p2, b1 | b2, d1 | d2
    print(f"\nk_project {len(proj & inst['k_project'])}/{len(inst['k_project'])}, k_blend {len(blend & inst['k_blend'])}/{len(inst['k_blend'])}, "
          f"k_ksplat_decode {len(decode & inst['k_ksplat_decode'])}/{len(inst['k_ksplat_decode'])}")
    assert proj == inst["k_project"], sorted(inst["k_project"] - proj)
    assert blend == inst["k_blend"], sorted(inst["k_blend"] - blend)
    assert decode == inst["k_ksplat_decode"] - {(True, True)}, sorted(inst["k_ksplat_decode"] - decode)
    assert any(isinstance(s, Refused) and s.what == "transform_dynamic" for s in SCRIPT)
    assert {(False, True), (False, False)} <= d2, d2
    paths = paths1 | paths2
    assert paths >= {(t, r, d) for t, r in ((16, False), (32, False), (32, True)) for d in (False, True)}, sorted(paths)
    # every upload entry, with a frame (always a graph frame first) before the next upload
    entries = {Splats: "upload_splat_data", Centers: "upload_centers", Ksplat: "upload_ksplat", PlyFile: "upload_file",
               Scenes: "upload_scenes", Optimized: "upload_file_optimized", Open: "open_stream", Append: "stream append", Close: "stream close"}
    seen = set()
    for script in (ST1.SCRIPT, SCRIPT):
        for i, s in enumerate(script):
            if type(s) in entries:
                # (an opened stream shows nothing before its first append)
                nxt = next((t for t in script[i + 1:] if isinstance(t, (Frame, Pipe)) or (type(t) in entries and not (isinstance(s, Open) and
                                                                                                                   isinstance(t, Append)))), None)
                if isinstance(nxt, (Frame, Pipe)):
                    seen.add(entries[type(s)])
    assert seen == set(entries.values()), sorted(set(entries.values()) - seen)
    # what the script promises beyond the kernels: view counts rising and falling, both frame-buffer parities of a pipelined pair with
    # different keys and then swapped, an asynchronous frame, every refusal, streams closed and left open, multi-scene trees
    vs = [f.views for _, f in _frames(SCRIPT) if f.views]
    assert set(vs) == {2, 3, 8, 16} and any(a > b for a, b in zip(vs, vs[1:])) and any(a < b for a, b in zip(vs, vs[1:])), vs
    key = lambda f: dataclasses.replace(f, cam=0)    # noqa: E731  (what the graph key sees: not the camera)
    pipes = [(k, s) for k, s in enumerate(SCRIPT) if isinstance(s, Pipe)]
    # a pair whose parities take each other's keys next (both slots replaced, then replayed)
    assert any(key(p.a) == key(q.b) and key(p.b) == key(q.a) and key(p.a) != key(p.b) for (_, p), (_, q) in zip(pipes, pipes[1:]))
    # a pair repeated with the same keys on both parities across a frame that grows the view buffers beyond every earlier frame, with
    # no upload between: the slot of the pipelined parity keeps a graph captured before the buffers moved
    most = lambda j: max([2 if f.stereo else f.views for _, f in _frames(SCRIPT[:j])] + [1])    # noqa: E731
    uploads = (Splats, Centers, Ksplat, PlyFile, Scenes, Optimized, Open, Append, Close)
    assert any(key(p.a) == key(q.a) and key(p.b) == key(q.b) and not any(isinstance(t, uploads) for t in SCRIPT[i:j]) and most(j) > most(i)
               for (i, p), (j, q) in zip(pipes, pipes[1:]))
    assert any(f.mode == "async" and f.depth for _, f in _frames(SCRIPT))
    assert {s.what for s in SCRIPT if isinstance(s, Refused)} == {"ksplat_truncated", "scenes_33", "over_capacity", "v2_in_file_order",
                                                                   "spz_stream", "scene0_bad", "scene2_bad", "transform_dynamic"}
    opens = [i for i, s in enumerate(SCRIPT) if isinstance(s, Open)]
    closed = [any(isinstance(t, Close) for t in SCRIPT[i + 1:(opens + [len(SCRIPT)])[j + 1]]) for j, i in enumerate(opens)]
    assert True in closed and False in closed
    kinds = {s.kind for sc in SCRIPT if isinstance(sc, Scenes) for s in sc.srcs} | {s.name.rsplit(".", 1)[1] for sc in SCRIPT
                                                                                   if isinstance(sc, Scenes) for s in sc.srcs if s.kind == "golden"}
    assert kinds >= {"ksplat", "ply", "splat", "pcply", "spz"} and any(s.optimized for sc in SCRIPT if isinstance(sc, Scenes) for s in sc.srcs)
    assert {len(s.srcs) for s in SCRIPT if isinstance(s, Scenes)} >= {1, 3, 4}
    assert {s.level for s in SCRIPT if isinstance(s, Optimized)} == {1, 2}
    # a re-upload of the same rows of one scene in the same order and file type, cut elsewhere, right after the first split
    i = SCRIPT.index(Scenes(SPLIT_A))
    assert SCRIPT[i + 2] == Scenes(SPLIT_B) and isinstance(SCRIPT[i + 1], Frame) and SCRIPT[i + 3] == SCRIPT[i + 1]
    for m in (SPLIT_A, SPLIT_B):
        assert {(x.kind, x.seed, x.n, x.deg) for x in m} == {("ply", 45, 90_000, 1)} and [x.rows[0] for x in m[1:]] == [x.rows[1] for x in m[:-1]]
        assert m[0].rows[0] == 0 and m[-1].rows[1] == 90_000 and len(m) == 3
    assert [x.rows for x in SPLIT_A] != [x.rows for x in SPLIT_B]
    assert any(isinstance(s, Open) and s.src.kind == "gen_ksplat" and s.src.sections >= 2 for s in SCRIPT)
    multi = [k for k, s in enumerate(SCRIPT) if isinstance(s, Scenes) and len(s.srcs) > 1]
    assert any(isinstance(SCRIPT[j], Frame) and SCRIPT[j].index == "device" for j in range(multi[1], len(SCRIPT))
               if max(i for i in multi + [k for k, t in enumerate(SCRIPT) if isinstance(t, (Splats, Scenes, Optimized, Open))] if i < j) in multi)


def test_first_script_tally_is_what_it_reaches_alone():
    """CPU: the first script alone reaches the 16 k_project and the 12 DEPTH = false k_blend instantiations (its docstring's claim)."""
    _, inst = _instances()
    proj, blend, _, _ = _reached(ST1.SCRIPT)
    assert proj == inst["k_project"]
    assert blend == {b for b in inst["k_blend"] if not b[4]}


# ---- GPU side ------------------------------------------------------------------------------------------------------------------------
_bytes_cache = {}


def _inria_ply(raw, deg) -> bytes:
    """An INRIA .ply of a synthetic scene at SH degree deg (f_rest channel-major)"""
    n, rest = raw.count, {0: 0, 1: 9, 2: 24}[deg]
    names = ["x", "y", "z", "f_dc_0", "f_dc_1", "f_dc_2"] + [f"f_rest_{k}" for k in range(rest)] + \
            ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    rec = np.empty((n, len(names)), np.float32)
    rec[:, 0:3] = raw.centers
    rec[:, 3:6] = (raw.colors[:, :3] / 255.0 - 0.5) / 0.28209479177387814
    if rest:
        rec[:, 6:6 + rest] = raw.sh[:, :rest // 3, :].transpose(0, 2, 1).reshape(n, rest)
    a = np.clip(raw.colors[:, 3] / 255.0, 1e-3, 1 - 1e-3)
    rec[:, 6 + rest] = np.log(a / (1 - a))
    rec[:, 7 + rest:10 + rest] = np.log(raw.scales)
    rec[:, 10 + rest:14 + rest] = raw.rotations[:, [3, 0, 1, 2]]
    head = "\n".join(["ply", "format binary_little_endian 1.0", f"element vertex {n}", *[f"property float {k}" for k in names], "end_header"]) + "\n"
    return head.encode() + rec.tobytes()


def _splat_file(raw) -> bytes:
    rec = np.zeros((raw.count, 32), np.uint8)
    rec[:, 0:12] = raw.centers.astype(np.float32).view(np.uint8).reshape(-1, 12)
    rec[:, 12:24] = raw.scales.astype(np.float32).view(np.uint8).reshape(-1, 12)
    rec[:, 24:28] = raw.colors
    rec[:, 28:32] = np.clip(np.round(raw.rotations[:, [3, 0, 1, 2]] * 128 + 128), 0, 255).astype(np.uint8)
    return rec.tobytes()


def _src_bytes(s: Src):
    """(format, bytes) of a scene source (.spz: its gunzipped stream)"""
    if s in _bytes_cache:
        return _bytes_cache[s]
    from gaussiansplats3d_b200 import ksplat as KS
    from gaussiansplats3d_b200.scenes import synthetic_scene
    if s.kind == "golden":
        data = (GOLDEN / s.name).read_bytes()
        ext = s.name.rsplit(".", 1)[1]
        out = ({"ply": PLY, "splat": SPLAT, "ksplat": KSPLAT, "spz": SPZ}[ext], gzip.decompress(data) if ext == "spz" else data)
    elif s.kind == "pcply":
        import test_progressive_gpu as PG
        out = (PLY, PG.pc_ply(s.n, s.seed))
    else:
        raw = synthetic_scene(s.n, seed=s.seed, kind="bonsai", sh_degree=s.deg)
        if s.rows:
            sl = slice(*s.rows)
            raw = dataclasses.replace(raw, centers=raw.centers[sl], scales=raw.scales[sl], rotations=raw.rotations[sl], colors=raw.colors[sl],
                                      sh=None if raw.sh is None else raw.sh[sl])
        if s.kind == "gen_ksplat":     # the generator's sections, partitioned by section_size (on the GPU)
            from gaussiansplats3d_b200.engine import generate_splat_buffer
            out = (KSPLAT, generate_splat_buffer(PLY, _inria_ply(raw, s.deg), sh_degree=s.deg, compression_level=s.level, minimum_alpha=0,
                                                 section_size=-(-s.n // s.sections)))
        elif s.kind == "ksplat":
            out = (KSPLAT, KS.write(raw.centers, raw.scales, raw.rotations, raw.colors, raw.sh, s.deg, compression_level=s.level, minimum_alpha=0))
        elif s.kind == "ply":
            out = (PLY, _inria_ply(raw, s.deg))
        elif s.kind == "spz":
            import spz_oracle as SO
            sh = raw.sh.transpose(0, 2, 1) if s.deg else None
            out = (SPZ, SO.quantize(raw.centers, np.log(raw.scales), raw.rotations, raw.colors / 255.0, sh, sh_degree=s.deg))
        else:
            out = (SPLAT, _splat_file(raw))
    _bytes_cache[s] = out
    return out


def _src_count(s: Src):
    """The splats a scene source holds, known without the engine (None: a fixture, or a file the generator may thin)"""
    if s.kind == "golden" or s.optimized:
        return None
    return s.rows[1] - s.rows[0] if s.rows else s.n


def _source(s: Src) -> dict:
    fmt, data = _src_bytes(s)
    return dict(format=fmt, data=data, optimized=s.optimized)


def _refused_call(what):
    """The call of a Refused step: a function of the engine that must raise"""
    mesh = [_source(s) for s in MESH3]
    ks = _src_bytes(MESH3[0])[1]
    if what == "ksplat_truncated":
        return lambda x: x.upload_ksplat(ks[:len(ks) - 100])
    if what == "scenes_33":
        return lambda x: x.upload_scenes([_source(G("file_handmade_sh1.ply"))] * 33, sh_degree=2)
    if what == "over_capacity":
        return lambda x: x.upload_file(PLY, _src_bytes(P(42, N_SPLATS + 1, 0))[1])
    if what == "v2_in_file_order":
        return lambda x: x.upload_file(PLY, (GOLDEN / "inriav2_codebook_sh2.ply").read_bytes(), sh_degree=2)
    if what == "spz_stream":
        return lambda x: x.open_stream(SPZ, sh_degree=2)
    if what == "scene0_bad":    # scene 0 of a multi-scene call: a truncated .ksplat
        return lambda x: x.upload_scenes([dict(format=KSPLAT, data=ks[:len(ks) - 100])] + mesh[1:], sh_degree=2)
    if what == "scene2_bad":    # scene 2 overflows the engine after scenes 0 and 1
        return lambda x: x.upload_scenes(mesh[:2] + [dict(format=PLY, data=_src_bytes(P(43, N_SPLATS - 80_000, 0))[1])], sh_degree=2)
    if what == "transform_dynamic":   # a static scene transform in a multi-scene call (k_ksplat_decode<true, true>): static engines only
        return lambda x: x.upload_scenes([dict(mesh[0], transform16=ST1._static_transform())] + mesh[1:], sh_degree=2)
    raise AssertionError(what)


def gs_native():
    from gaussiansplats3d_b200 import _native as N
    return N


@dataclass
class MeshModel(Model):
    """Model, plus the new upload steps, the mesh's scenes and the sorter's scene indexes"""
    scene_count: int = 1
    infos: list = field(default_factory=list)
    sort_idx: np.ndarray | None = None      # the sorter's scene indexes (None: all 0)
    stream_data: bytes = b""
    stream_at: int = 0
    stream_src: Src | None = None

    def _decoded(self, info, call, restart, scenes=1, infos=None):
        if restart:
            self.raster_calls, self.sorter_calls = [call], [call]
        else:                     # a stream's appends write the sorter's centres too
            self.raster_calls.append(call)
            self.sorter_calls.append(call)
        self.decoded, self.cov_f16, self.idx = True, False, None
        self.deg, self.sh_u8 = info["sh_degree"], info["compression_level"] == 2
        self.uploaded = self.sorted_splats = info["splat_count"]
        self.scene_count, self.infos, self.sort_idx = scenes, infos or [info], None

    def apply(self, e, step, seq):
        if isinstance(step, (Splats, Centers, Ksplat, PlyFile)):
            super().apply(e, step, seq)
            if isinstance(step, Centers):
                if step.start == 0:
                    self.sort_idx = np.zeros(N_SPLATS, np.uint32)
                n = step.count or N_SPLATS - step.start
                self.sort_idx[step.start:step.start + n] = ST1._scene_indexes(step.seed)[step.start:step.start + n]
            elif isinstance(step, Splats):
                if step.start == 0:
                    self.scene_count = ST1.N_SCENES if step.idx else 1
            else:
                self.scene_count, self.sort_idx = 1, None
        elif isinstance(step, Scenes):
            srcs = [_source(s) for s in step.srcs]
            call = (seq, lambda x: x.upload_scenes(srcs, sh_degree=2))
            infos = call[1](e)
            mesh = dict(splat_count=sum(i["splat_count"] for i in infos), sh_degree=min(i["sh_degree"] for i in infos),
                        compression_level=max(i["compression_level"] for i in infos))
            counts = [i["splat_count"] for i in infos]
            want = [_src_count(x) for x in step.srcs]
            assert all(w is None or w == c for w, c in zip(want, counts)), f"step {seq}: scene splat counts {counts}, sources hold {want}"
            assert [i["splat_offset"] for i in infos] == np.cumsum([0] + counts[:-1]).tolist(), f"step {seq}: scene offsets"
            self._decoded(mesh, call, True, len(infos), infos)
            if len(infos) > 1:
                # scene s's splats follow scene s-1's: the indexes the f64 checks and the reference sorter use are restated here, and the
                # decode's (the rasteriser's copy, GS_BUF_SCENE_INDEXES) must equal them
                self.sort_idx = np.repeat(np.arange(len(counts), dtype=np.uint32), counts)
                got = e.read_buffer(gs_native().GS_BUF_SCENE_INDEXES, np.uint32, self.uploaded)
                assert np.array_equal(got, self.sort_idx), f"step {seq}: the decoded scene indexes differ at {np.flatnonzero(got != self.sort_idx)[:5]}"
        elif isinstance(step, Optimized):
            data = _src_bytes(P(step.seed, step.n, step.deg))[1]
            call = (seq, lambda x: x.upload_file_optimized(PLY, data, sh_degree=2, compression_level=step.level))
            self._decoded(call[1](e), call, True)
        elif isinstance(step, Open):
            fmt, data = _src_bytes(step.src)
            self.stream_data, self.stream_at, self.stream_src = data, 0, step.src
            call = (seq, lambda x: setattr(x, "_stream", x.open_stream(fmt, sh_degree=2)))
            call[1](e)
            self._decoded(dict(splat_count=0, sh_degree=0, compression_level=0), call, True)
        elif isinstance(step, Append):
            data = self.stream_data
            upto = len(data) if step.upto >= 1 else int(len(data) * step.upto) + int(np.random.default_rng(seq).integers(-50, 50))
            chunk = data[self.stream_at:upto]
            self.stream_at = upto
            call = (seq, lambda x: x._stream.append(chunk))
            call[1](e)
            self._decoded(e._stream.progress, call, False)
            src = self.stream_src
            if src.kind == "gen_ksplat" and upto < len(data):     # a cut inside a later section: the sections before it are whole
                per = -(-src.n // src.sections)
                assert per < self.uploaded < src.n and self.uploaded % per, f"step {seq}: {self.uploaded} splats loaded, sections of {per}"
        elif isinstance(step, Close):
            call = (seq, lambda x: x._stream.close())
            self._decoded(call[1](e), call, False)
        else:
            raise AssertionError(step)

    def arrays(self, e):
        cc, cov, sh, deg, idx = super().arrays(e)
        if self.decoded and self.scene_count > 1:
            idx = self.sort_idx
        return cc, cov, sh, deg, idx

    def sh_ranges(self):
        """Each scene's 8-bit SH range (its upload info) of a decoded mesh that stores SH at 8 bits, for the uniforms"""
        if not (self.decoded and self.deg and self.sh_u8):
            return None
        lo, hi = np.full(32, -1.5, np.float32), np.full(32, 1.5, np.float32)
        for s, i in enumerate(self.infos):
            lo[s], hi[s] = i.get("min_sh_coeff", -1.5), i.get("max_sh_coeff", 1.5)
        return lo, hi


def _new_engine():
    from gaussiansplats3d_b200.engine import Engine
    return Engine(N_SPLATS, max_width=ST1.MAX_W, max_height=ST1.MAX_H, dynamic_mode=True, ray_records=True)


def _close(e):
    e._stream = None          # a stream goes before its engine
    e.close()


@dataclass
class Setup:
    """What a frame of the script is rendered from, so that the same frame can be rendered on any engine"""
    a: FrameArgs
    views: list


def _setup(f: MFrame, model: MeshModel, rng, k) -> Setup:
    import test_multi_view_gpu as M
    rig = _rig(f, model.deg, model.sh_is_u8())
    r = model.sh_ranges()
    if r is not None:
        rig.u.sh8_min, rig.u.sh8_max = r
    limit = min(model.uploaded, model.sorted_splats)
    render = limit if f.render is None else min(f.render, limit)
    indexes = np.sort(rng.choice(limit, render, replace=False)).astype(np.uint32)[rng.permutation(render)] if f.index == "host" else None
    pre = rng.integers(-2_000_000, 2_000_000, model.sorted_splats, dtype=np.int64).astype(np.int32) if f.pre else None
    dest = ST1._composite_inputs(f, k) if f.comp else ()
    a = FrameArgs(f, rig, render, render if f.sort is None else min(f.sort, render), indexes, pre, dest)
    views = [M._view(c, f.w, f.h, dynamic=True) for c in M._ring(f.views, f.w, f.h, fovs=[50.0, 62.0, 44.0])] if f.views else []
    return Setup(a, views)


def _gather(e, su: Setup):
    """build_splat_tree + the gather, with one model view per sub-tree of a forest: (device pointer of the list, its length)"""
    from gaussiansplats3d_b200 import three_math as TM
    e.build_splat_tree()
    subs = e.splat_tree_info()["sub_tree_count"]
    if subs > 1:
        xf = su.a.rig.transforms.astype(np.float64)
        n = e.gather_for_sort_subtrees([TM.multiply(su.a.rig.mv64.reshape(16), xf[16 * s:16 * s + 16]) for s in range(subs)], 0.6, 0.7)
    else:
        n = e.gather_for_sort(su.a.rig.mv64, 0.6, 0.7)
    return e.buffer_dev(gs_native().GS_BUF_INDEXES_TO_SORT)[0], n


def _params(e, su: Setup, index_dev=None, depth_out=None):
    """(sort params, uniforms, render params, views array, keep-alive) of the frame on engine e"""
    N = gs_native()
    a, f = su.a, su.a.f
    fmt = N.GS_FRAME_RGBA8 if f.fmt == "rgba8" else N.GS_FRAME_RGBA32F
    sp = e._sort_params(np.zeros(16, np.float32) if f.views else a.rig.mvp, a.sort, a.render, a.indexes, a.rig.transforms, a.pre, index_dev)
    keep = list(e._keep)
    dc, dd = (a.dest[2], a.dest[3]) if a.dest else (None, None)
    rp, _ = e._render_params(f.w, f.h, a.render, None, fmt, f.flip, dc, dd, a.rig.eyes, depth=f.depth, depth_out=depth_out,
                             views=f.views or None)
    cams = (N.gs_view * f.views)(*[v.to_c() for v in su.views]) if f.views else None
    return sp, a.rig.u.to_c(), rp, cams, keep


def _run(e, su: Setup, graph: bool, index_dev=None):
    """The frame on engine e, graph on or off: gs_frame / gs_frame_views, or gs_frame_async + gs_synchronize read back through
    GS_BUF_FRAME / GS_BUF_SORTED_INDEXES / GS_BUF_DEPTH.  (colour, draw order, depth or None); a multi-view frame's with a view axis."""
    N = gs_native()
    a, f = su.a, su.a.f
    dt = np.uint8 if f.fmt == "rgba8" else np.float32
    e.set_graph_enabled(graph)
    try:
        if f.mode == "async":
            sp, u, rp, _, keep = _params(e, su, index_dev)
            N.check(e._lib.gs_frame_async(e._h, C.byref(sp), C.byref(u), C.byref(rp)), "gs_frame_async")
            e.synchronize()
            frame = e.read_buffer(N.GS_BUF_FRAME, dt, f.h * f.w * 4).reshape(f.h, f.w, 4)
            order = e.read_buffer(N.GS_BUF_SORTED_INDEXES, np.uint32, a.render)
            depth = e.read_buffer(N.GS_BUF_DEPTH, np.float32, f.h * f.w).reshape(f.h, f.w) if f.depth else None
            return frame, order, depth
        lead = (f.views,) if f.views else ()
        depth = np.empty(lead + (f.h, f.w), np.float32) if f.depth else None
        sp, u, rp, cams, keep = _params(e, su, index_dev, depth)
        frame = np.empty(lead + (f.h, f.w, 4), dt)
        order = np.empty(lead + (a.render,), np.uint32)
        if f.views:
            N.check(e._lib.gs_frame_views(e._h, C.byref(sp), C.byref(u), C.byref(rp), cams, f.views, N.ptr(order), N.ptr(frame)), "gs_frame_views")
        else:
            N.check(e._lib.gs_frame(e._h, C.byref(sp), C.byref(u), C.byref(rp), N.ptr(order), N.ptr(frame)), "gs_frame")
        return frame, order, depth
    finally:
        e.set_graph_enabled(True)


def _same(got, want, what):
    (gf, go, gd), (wf, wo, wd) = got, want
    assert np.array_equal(go, wo), f"{what}: the draw orders differ"
    assert gf.tobytes() == wf.tobytes(), f"{what}: colour: {_differ(gf.reshape(-1, gf.shape[-2], 4), wf.reshape(-1, wf.shape[-2], 4))}"
    assert (gd is None) == (wd is None), what
    if gd is not None:
        assert gd.tobytes() == wd.tobytes(), f"{what}: depth: {int((gd.view(np.uint32) != wd.view(np.uint32)).sum())} values differ"


def _check_bounds(e, su: Setup, got, model: MeshModel, label, worst):
    """Check 3: the f64 bounds of a mono frame, of each eye of a stereo frame (each half first equal to its eye's gs_render), and of
    bands of a multi-view frame (each band first equal to gs_render of its camera with its view's order, each order the reference
    sorter's): colour and projection through FF.check_frame, depth through depth_f64"""
    import blend_f64 as BF
    import depth_f64 as DF
    import test_multi_view_gpu as M
    import test_stereo_gpu as STG
    FF = ST1.FF
    N = gs_native()
    a, f = su.a, su.a.f
    frame, order, depth = got
    cc, cov, sh, deg, idx = model.arrays(e)
    fmt = N.GS_FRAME_RGBA8 if f.fmt == "rgba8" else N.GS_FRAME_RGBA32F

    def held(lbl, u, w, colour, o, d, dc=None, dd=None):
        win = FF.windows(w, f.h) if w * f.h > ST1.BIG_FRAME else None
        pw, bw = FF.check_frame(lbl, e, u, w, f.h, a.render, cc, cov, sh, deg, idx, got=colour if f.fmt == "rgba32f" else None,
                                got8=colour if f.fmt == "rgba8" else None, order=o, windows=win, flip_y=f.flip, dest_color=dc, dest_depth=dd)
        worst["projection"], worst["blend"] = max(worst["projection"], pw), max(worst["blend"], bw)
        if d is not None:
            rec = BF.read_records(e, int(o.max()) + 1)
            for wn in (win or [(0, 0, w, f.h)]):
                rep = DF.check(f"{lbl} {wn}", DF.restate(rec, o, w, f.h, u.projection, window=wn, dest_depth=dd, flip_y=f.flip), DF.crop(d, wn, f.flip))
                worst["depth"] = max(worst["depth"], rep["worst"])

    if f.views:
        centers = e.read_buffer(N.GS_BUF_CENTERS, np.int32, 4 * model.sorted_splats).reshape(-1, 4)
        sidx = model.sort_idx[:model.sorted_splats] if model.sort_idx is not None else np.zeros(model.sorted_splats, np.uint32)
        xf = np.zeros(16 * 32, np.float32)
        xf[:a.rig.transforms.size] = a.rig.transforms
        # every band of a frame up to 1 Mpx in all, else the first, middle and last
        checked = range(f.views) if f.views <= 3 or f.views * f.w * f.h <= ST1.BIG_FRAME else (0, f.views // 2, f.views - 1)
        for v, view in enumerate(su.views):
            want = FF.reference_order(centers, view.model_view_proj, a.render, indexes=a.indexes, sort_count=a.sort,
                                      splat_count=model.sorted_splats, scene_indexes=sidx, transforms=xf, dynamic=True)
            assert np.array_equal(order[v], want), f"{label}: view {v}'s draw order differs from the reference sorter's"
            uv = M._substituted(a.rig.u, view)
            r = e.render(uv, f.w, f.h, a.render, order[v], frame_format=fmt, flip_y=f.flip, depth=f.depth)
            band, bd = r if f.depth else (r, None)
            assert np.array_equal(band.view(np.uint8), frame[v].view(np.uint8)), f"{label}: band {v} differs from gs_render of its camera: {_differ(frame[v], band)}"
            if f.depth:
                assert bd.tobytes() == depth[v].tobytes(), f"{label}: band {v}'s depth differs from gs_render's"
            if v in checked:
                held(f"{label} view {v}", uv, f.w, frame[v], order[v], depth[v] if f.depth else None)
    elif f.stereo:
        vw = f.w // 2
        for i, eye in enumerate(a.rig.eyes):
            ue = STG._substituted(a.rig.u, eye)
            r = e.render(ue, vw, f.h, a.render, order, frame_format=fmt, flip_y=f.flip, depth=f.depth)
            mono, md = r if f.depth else (r, None)
            half = frame[:, i * vw:(i + 1) * vw]
            assert np.array_equal(half.view(np.uint8), mono.view(np.uint8)), f"{label}: eye {i} differs from its mono frame: {_differ(half, mono)}"
            if f.depth:
                assert np.ascontiguousarray(depth[:, i * vw:(i + 1) * vw]).tobytes() == md.tobytes(), f"{label}: eye {i}'s depth differs from its mono depth"
            held(f"{label} eye {i}", ue, vw, mono, order, md)
    else:
        held(label, a.rig.u, f.w, frame, order, depth, *((a.dest[0], a.dest[1]) if a.dest else (None, None)))


def _pipe(e, step: Pipe, model: MeshModel, rng, k, label):
    """Two pipelined frames in flight, one per frame-buffer parity: each equals gs_frame of the same inputs (graph off), and GS_BUF_DEPTH
    is the plane of the later one that asked for depth"""
    N = gs_native()
    sus = [_setup(f, model, rng, k) for f in (step.a, step.b)]
    outs, douts, keep = [], [], []
    for su in sus:
        f = su.a.f
        out = np.empty((f.h, f.w, 4), np.uint8 if f.fmt == "rgba8" else np.float32)
        dout = np.empty((f.h, f.w), np.float32) if f.depth else None
        sp, u, rp, _, kp = _params(e, su, None, dout)
        keep.append((sp, u, rp, kp))
        N.check(e._lib.gs_frame_begin(e._h, C.byref(sp), C.byref(u), C.byref(rp), N.ptr(out)), "gs_frame_begin")
        outs.append(out)
        douts.append(dout)
    e.frame_end()
    e.frame_end()
    last = max(i for i, su in enumerate(sus) if su.a.f.depth)
    f = sus[last].a.f
    dev = e.read_buffer(N.GS_BUF_DEPTH, np.float32, f.h * f.w).reshape(f.h, f.w)
    assert dev.tobytes() == douts[last].tobytes(), f"{label}: GS_BUF_DEPTH is not the plane of pipelined frame {last}"
    for i, su in enumerate(sus):
        want, _, wd = _run(e, su, False)
        assert outs[i].tobytes() == want.tobytes(), f"{label}: pipelined frame {i} differs from gs_frame: {_differ(outs[i], want)}"
        assert (douts[i] is None) or douts[i].tobytes() == wd.tobytes(), f"{label}: pipelined frame {i}'s depth differs from gs_frame's"


@pytest.mark.gpu
def test_scripted_mesh_sequence_on_one_engine(gs):
    import time
    from gaussiansplats3d_b200.scenes import CAMERAS
    N = gs._native
    t0 = time.time()
    rng = np.random.default_rng(2027)
    model = MeshModel()
    worst = dict(projection=0.0, blend=0.0, depth=0.0)
    e = _new_engine()
    frames, last = 0, None
    try:
        for k, step in enumerate(SCRIPT):
            label = f"step {k} {step}"
            if isinstance(step, Refused):
                with pytest.raises(N.GsError) as ei:
                    _refused_call(step.what)(e)
                assert ei.value.code == getattr(N, step.code), f"{label}: {ei.value}"
                if last is not None:      # not recorded: the frame before the refusal, again, with its graph
                    su, before = last
                    dev = _gather(e, su)[0] if su.a.f.index == "device" else None
                    _same(_run(e, su, True, dev), before, f"{label}: the graph frame after the refusal vs the frame before it")
                continue
            if isinstance(step, Box):
                xf = _setup(MFrame(64, 64), model, rng, k).a.rig.transforms.astype(np.float64)[:16 * model.scene_count].reshape(-1, 16)
                lo, hi = e.compute_bounding_box(-1, True, xf)
                lo0, hi0 = e.compute_bounding_box(0, False)
                assert np.all(lo <= hi) and np.all(lo0 <= hi0), label
                continue
            if isinstance(step, Ray):
                c = CAMERAS["bonsai"]
                xf = _setup(MFrame(64, 64), model, rng, k).a.rig.transforms.astype(np.float64)
                e.build_splat_tree()
                subs = e.splat_tree_info()["sub_tree_count"]
                kw = dict(sub_tree_from_local=xf[:16 * subs].reshape(-1, 16)) if subs > 1 else dict(from_local16=xf[:16])
                _, total = e.raycast(c["position"], np.subtract(c["look_at"], c["position"]), capacity=4, **kw)
                assert total > 0, f"{label}: the ray from the bonsai camera hits nothing"
                continue
            if isinstance(step, Pipe):
                _pipe(e, step, model, rng, k, label)
                frames += 2
                last = None
                continue
            if not isinstance(step, Frame):
                model.apply(e, step, k)
                continue
            f = step
            su = _setup(f, model, rng, k)
            limit = su.a.render
            dev = None
            if f.index == "device":
                dev, n = _gather(e, su)
                assert 0 < n < limit, f"{label}: the gather should keep some splats and drop others ({n} of {limit})"
                su.a.render, su.a.sort = n, n if f.sort is None else min(f.sort, n)
            # 1. graph frame == eager frame on the same engine (colour, depth, every view's order)
            got = _run(e, su, True, dev)
            assert e.timings()["tile_instances"] > 0, label
            _same(got, _run(e, su, False, dev), f"{label}: graph frame vs eager frame")
            # 2. a fresh engine given only the calls that define the state
            fresh = _new_engine()
            try:
                model.replay(fresh)
                fdev = None
                if f.index == "device":
                    fdev, n = _gather(fresh, su)
                    assert n == su.a.render, f"{label}: a fresh engine gathers {n} splats, this one {su.a.render}"
                want = _run(fresh, su, False, fdev)
            finally:
                _close(fresh)
            _same(got, want, f"{label}: this engine vs a fresh engine")
            # 3. f64 bounds
            _check_bounds(e, su, got, model, label, worst)
            last = None if f.views else (su, got)
            frames += 1
    finally:
        _close(e)
    assert frames == sum(2 if isinstance(s, Pipe) else isinstance(s, Frame) for s in SCRIPT)
    print(f"\n{frames} frames in {time.time() - t0:.1f} s; worst |GPU - f64| / bound: projection {worst['projection']:.3f}, "
          f"blend {worst['blend']:.3f}, depth {worst['depth']:.3f}")
