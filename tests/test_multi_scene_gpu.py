"""GPU: several scenes in one mesh (gs_upload_scenes, Viewer.addSplatScenes / removeSplatScenes).

A one-scene call leaves every engine buffer as the matching single-scene entry does; each scene's slot of a multi-scene mesh holds what
that scene alone holds (its SH converted to the mesh's storage where the two differ); multi-scene frames, static and dynamic, are
bit-identical to the frames of an engine fed the same buffers with scene indexes through gs_upload_splat_data and stay within the f64
projection and blend bounds; rejected calls name the scene and leave the frame as it was."""
import gzip
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent))
import frame_f64 as FF  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden"
W, H = 256, 192


def _N():
    from gaussiansplats3d_b200 import _native as N
    return N


def _xf(position, quaternion=(0.0, 0.0, 0.0, 1.0), scale=(1.0, 1.0, 1.0)):
    from gaussiansplats3d_b200 import three_math as TM
    return np.asarray(TM.compose(position, quaternion, scale), np.float64).reshape(16)


T1 = _xf((0.5, -0.25, 1.0), (0.1, 0.2, -0.3, 0.927), (1.5, 0.75, 1.25))
T2 = _xf((-1.0, 0.5, 0.0), (0.0, 0.6, 0.0, 0.8), (0.8, 0.8, 0.8))


def _camera(sh_degree=2):
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.engine import Uniforms
    proj = TM.make_perspective(50, W / H, 0.1, 1000.0)
    view = TM.invert(TM.camera_world_matrix([0.0, 0.5, 6.0], [0.0, 0.0, 0.0], [0.0, 1.0, 0.0]))
    u = Uniforms(model_view=view.astype(np.float32), projection=proj.astype(np.float32), camera_position=np.array([0.0, 0.5, 6.0], np.float32),
                 focal=(proj[0] * 0.5 * W, proj[5] * 0.5 * H), viewport=(W, H), sh_degree=sh_degree)
    return TM.multiply(proj, view).astype(np.float32), u, view


def _engine(n, dynamic=False, ray=True):
    from gaussiansplats3d_b200 import Engine
    return Engine(n, max_width=W, max_height=H, dynamic_mode=dynamic, ray_records=ray)


def _golden(name):
    data = (GOLDEN / name).read_bytes()
    return gzip.decompress(data) if name.endswith(".spz") else data


# (fixture, format, optimized): every single-scene entry and kind the fixtures cover
KINDS = [
    ("ksplat_handmade_l0_sh0.ksplat", 3, False), ("ksplat_handmade_l0_sh2.ksplat", 3, False), ("ksplat_handmade_l1_sh1.ksplat", 3, False),
    ("ksplat_handmade_l1_sh0_many_buckets.ksplat", 3, False), ("ksplat_handmade_l2_sh2_two_sections.ksplat", 3, False),
    ("file_handmade_sh0.ply", 1, False), ("file_handmade_sh1.ply", 1, False), ("file_handmade_sh2.ply", 1, False), ("file_handmade_sh3.ply", 1, False),
    ("pcply_handmade_sh2.ply", 1, False), ("file_handmade_basic.splat", 2, False), ("spz_handmade_sh2.spz", 4, False),
    ("inriav2_codebook_sh2.ply", 1, True), ("file_handmade_sh2.ply", 1, True),
    ("spz_handmade_empty.spz", 4, False), ("inriav2_codebook_empty.ply", 1, True),
]
BUFS = ("GS_BUF_CENTERS_COLORS", "GS_BUF_COVARIANCES", "GS_BUF_SH", "GS_BUF_CENTERS", "GS_BUF_RAY_RECORDS")


def _count(fmt, data):
    from gaussiansplats3d_b200 import Engine, ksplat
    return ksplat.parse(data).max_splat_count if fmt == 3 else Engine.probe_file(fmt, data)["splat_count"]


def _single(e, fmt, data, optimized, transform16, minimum_alpha=1, gen=None):
    if fmt == 3:
        return e.upload_ksplat(data, minimum_alpha=minimum_alpha, transform16=transform16)
    if optimized:
        return e.upload_file_optimized(fmt, data, sh_degree=2, minimum_alpha=minimum_alpha, transform16=transform16, **(gen or {}))
    return e.upload_file(fmt, data, sh_degree=2, minimum_alpha=minimum_alpha, transform16=transform16)


def _bytes(e, buf, n, info):
    """Buffer `buf` of splats [0, n) as bytes, sized by what the mesh stores."""
    N = _N()
    ncomp = {0: 0, 1: 9, 2: 24}[info["sh_degree"]]
    per = {"GS_BUF_CENTERS_COLORS": 16, "GS_BUF_COVARIANCES": 24, "GS_BUF_SH": ncomp * (1 if info["compression_level"] == 2 else 2),
           "GS_BUF_CENTERS": 16, "GS_BUF_RAY_RECORDS": 56, "GS_BUF_SCENE_INDEXES": 4}[buf]
    return e.read_buffer(getattr(N, buf), np.uint8, n * per) if n * per else np.zeros(0, np.uint8)


def _frame(e, n, u, mvp, transforms=None, fmt=None):
    N = _N()
    return e.frame(mvp, u, W, H, n, None, frame_format=N.GS_FRAME_RGBA32F if fmt is None else fmt, transforms=transforms).copy()


@pytest.mark.parametrize("transform", [False, True])
@pytest.mark.parametrize("kind", KINDS, ids=[f"{k[0]}-{'opt' if k[2] else 'plain'}" for k in KINDS])
def test_one_scene_is_its_single_scene_entry(kind, transform):
    from gaussiansplats3d_b200 import GsError
    name, fmt, optimized = kind
    data = _golden(name)
    n0 = _count(fmt, data)
    xf = T1 if transform else None
    mvp, u, _ = _camera()
    a, b = _engine(max(n0, 1)), _engine(max(n0, 1))
    try:
        ia = _single(a, fmt, data, optimized, xf)
        [ib] = b.upload_scenes([dict(format=fmt, data=data, optimized=optimized, transform16=xf)], sh_degree=2)
        assert ib.pop("splat_offset") == 0
        ia.pop("splat_offset")
        assert ia == ib
        n = ia["splat_count"]
        for buf in BUFS:
            assert np.array_equal(_bytes(a, buf, n, ia), _bytes(b, buf, n, ib)), buf
        if n:   # the same frame, or the same refusal (a fixture's out-of-range centres overflow the sort's range map)
            u.sh_degree = ia["sh_degree"]
            got = []
            for x in (a, b):
                try:
                    got.append(_frame(x, n, u, mvp))
                except GsError as err:
                    got.append(err.code)
            assert not isinstance(got[0], int) or got[0] == _N().GS_ERR_BUCKET_RANGE
            assert np.array_equal(got[0], got[1])
    finally:
        a.close(); b.close()


def test_single_scene_entries_write_no_more_than_the_callers_info():
    """A caller built before gs_ksplat_info.splat_offset passes the 40-byte struct (struct_size 0 or 40): the single-scene uploads
    write those 40 bytes and nothing past them."""
    import ctypes as C
    N = _N()
    lib = N.load()
    data = _golden("ksplat_handmade_l1_sh1.ksplat")
    ply = _golden("file_handmade_sh2.ply")
    e = _engine(max(_count(3, data), _count(1, ply)))
    try:
        legacy = N.gs_ksplat_info.splat_offset.offset
        for size in (0, legacy):
            for call in (lambda p: lib.gs_upload_ksplat(e._h, data, len(data), None, p),
                         lambda p: lib.gs_upload_file(e._h, 1, ply, len(ply), 2, None, p),
                         lambda p: lib.gs_upload_file_optimized(e._h, 1, ply, len(ply), 2, None, None, p)):
                buf = (C.c_uint8 * (legacy + 8))(*([0] * legacy + [0xA5] * 8))
                C.memmove(buf, C.byref(C.c_uint32(size)), 4)
                N.check(call(C.cast(buf, C.POINTER(N.gs_ksplat_info))), "upload")
                assert bytes(buf)[legacy:] == b"\xa5" * 8, size
                assert C.cast(buf, C.POINTER(N.gs_ksplat_info)).contents.struct_size == legacy
        full = N.gs_ksplat_info()
        full.struct_size = C.sizeof(N.gs_ksplat_info)
        full.splat_offset = 7
        N.check(lib.gs_upload_ksplat(e._h, data, len(data), None, C.byref(full)), "gs_upload_ksplat")
        assert full.splat_offset == 0 and full.struct_size == C.sizeof(N.gs_ksplat_info)
    finally:
        e.close()


def _raw_sh_f32(data):
    """The f32 SH of a level-0 .ksplat in the mesh's coefficient-major order (SplatBuffer.js:551-734)."""
    from oracle import ksplat_oracle as KO
    h = KO.parse(data)
    buf = np.frombuffer(data, np.uint8)
    out = []
    for s in h.sections:
        n = s.max_splat_count
        rec = buf[s.data_base: s.data_base + n * s.bytes_per_splat].reshape(n, s.bytes_per_splat)
        raw = rec[:, 44:].copy().view(np.float32).reshape(n, -1)
        out.append(np.concatenate([raw[:, :9].reshape(n, 3, 3).transpose(0, 2, 1).reshape(n, 9),
                                   raw[:, 9:24].reshape(n, 3, 5).transpose(0, 2, 1).reshape(n, 15)], 1))
    return np.concatenate(out), float(np.float32(h.min_sh if h.min_sh else -1.5)), float(np.float32(h.max_sh if h.max_sh else 1.5))


def to_uint8(v, lo, hi):
    """SplatBuffer.js toUint8 (:22-26) in f64: clamp = Math.max(Math.min(v, hi), lo); NaN stores as 0."""
    v = np.asarray(v, np.float64)
    q = np.floor((np.maximum(np.minimum(v, hi), lo) - lo) / (hi - lo) * 255)
    q = np.maximum(np.minimum(q, 255), 0)
    return np.where(np.isnan(q), 0, q).astype(np.uint8)


def _rotated_sh(ply, transform16):
    """A .ply's SH2 as its level-0 SplatBuffer holds them (oracle/file_oracle.py), rotated as fillSphericalHarmonicsArray rotates them
    under a scene transform (dot3 / dot5 in f64, SplatBuffer.js:684-772), before the output conversion."""
    from oracle import file_oracle as FO
    from oracle import ksplat_oracle as KO
    raw, _, _ = _raw_sh_f32(FO.level0_image(1, ply, 2)[0])
    n = raw.shape[0]
    m1, m2 = KO.sh_rotation_matrices(KO.rotation_of_transform(transform16))
    tri = raw.astype(np.float64).reshape(n, -1, 3)
    out = np.empty_like(tri)
    for l in range(3):
        out[:, l] = (tri[:, 0] * m1[l, 0] + tri[:, 1] * m1[l, 1]) + tri[:, 2] * m1[l, 2]
    for l in range(5):
        out[:, 3 + l] = (((tri[:, 3] * m2[l, 0] + tri[:, 4] * m2[l, 1]) + tri[:, 5] * m2[l, 2]) + tri[:, 6] * m2[l, 3]) + tri[:, 7] * m2[l, 4]
    return out.reshape(n, 24)


# the mixed static mesh: a level-2 .ksplat (two sections), a level-0 .ksplat, a .ply in file order and a generated level-1 .ply
MIXED = [
    dict(format=3, data="ksplat_handmade_l2_sh2_two_sections.ksplat", transform16=T1, minimum_alpha=1),
    dict(format=3, data="ksplat_handmade_l0_sh2.ksplat", minimum_alpha=40),
    dict(format=1, data="file_handmade_sh2.ply", transform16=T2, minimum_alpha=20),
    dict(format=1, data="file_handmade_sh2.ply", optimized=True, generate=dict(compression_level=1)),
]


def _mixed(dynamic=False):
    out = []
    for s in MIXED:
        s = dict(s, data=_golden(s["data"]))
        if dynamic:
            s.pop("transform16", None)
        out.append(s)
    return out


def _alone(s):
    e = _engine(max(_count(s["format"], s["data"]), 1))
    gen = dict(s.get("generate", {}))
    info = _single(e, s["format"], s["data"], s.get("optimized", False), s.get("transform16"), s.get("minimum_alpha", 1), gen)
    return e, info


def test_each_slot_is_that_scene_alone():
    src = _mixed()
    total = sum(_count(s["format"], s["data"]) for s in src)
    e = _engine(total)
    try:
        infos = e.upload_scenes(src, sh_degree=2)
        mesh = dict(sh_degree=2, compression_level=2)
        n = sum(i["splat_count"] for i in infos)
        assert [i["splat_offset"] for i in infos] == list(np.cumsum([0] + [i["splat_count"] for i in infos[:-1]]))
        idx = e.read_buffer(_N().GS_BUF_SCENE_INDEXES, np.uint32, n)
        sh = _bytes(e, "GS_BUF_SH", n, mesh).reshape(n, 24)
        for s, (sc, info) in enumerate(zip(src, infos)):
            lo, cnt = info["splat_offset"], info["splat_count"]
            assert (idx[lo:lo + cnt] == s).all()
            a, ia = _alone(sc)
            try:
                for buf, per in (("GS_BUF_CENTERS_COLORS", 16), ("GS_BUF_COVARIANCES", 24), ("GS_BUF_CENTERS", 16), ("GS_BUF_RAY_RECORDS", 56)):
                    got = _bytes(e, buf, n, mesh)[lo * per:(lo + cnt) * per]
                    assert np.array_equal(got, _bytes(a, buf, cnt, ia)), (s, buf)
                if s == 0:      # level 2 in a level-2 mesh: stored as it is alone
                    assert np.array_equal(sh[lo:lo + cnt].reshape(-1), _bytes(a, "GS_BUF_SH", cnt, ia)), s
                elif s == 1:    # level 0 without a transform: toUint8 of its f32 values with its own range
                    raw, rlo, rhi = _raw_sh_f32(sc["data"])
                    assert np.array_equal(sh[lo:lo + cnt], to_uint8(raw, rlo, rhi)), s
                elif s == 2:    # level 0 with a transform: toUint8 of its rotated f32 values with its own range (-1.5, 1.5)
                    assert np.array_equal(sh[lo:lo + cnt], to_uint8(_rotated_sh(sc["data"], sc["transform16"]), -1.5, 1.5)), s
                elif s == 3:    # level 1 without a transform: the reference's fromHalfFloatToUint8 stores 0
                    assert not sh[lo:lo + cnt].any()
            finally:
                a.close()
    finally:
        e.close()


def _fed_engine(e, n, dynamic, mesh):
    """An engine fed e's buffers through gs_upload_splat_data(scene_indexes=...) and gs_upload_centers."""
    f = _engine(n, dynamic=dynamic, ray=False)
    cc = e.read_buffer(_N().GS_BUF_CENTERS_COLORS, np.uint32, n * 4).reshape(n, 4)
    cov = e.read_buffer(_N().GS_BUF_COVARIANCES, np.float32, n * 6).reshape(n, 6)
    ncomp = {0: 0, 1: 9, 2: 24}[mesh["sh_degree"]]
    sh = e.read_buffer(_N().GS_BUF_SH, np.uint8 if mesh["compression_level"] == 2 else np.float16, n * ncomp).reshape(n, ncomp) if ncomp else None
    idx = e.read_buffer(_N().GS_BUF_SCENE_INDEXES, np.uint32, n)
    f.upload_splat_data(cc, cov, sh, mesh["sh_degree"], scene_indexes=idx)
    centers = e.read_buffer(_N().GS_BUF_CENTERS, np.int32, n * 4).reshape(n, 4)
    f.upload_centers(centers, idx if dynamic else None)
    return f, cc, cov, sh, idx, centers


@pytest.mark.parametrize("dynamic", [False, True])
def test_frames_match_host_fed_scene_indexes(dynamic):
    N = _N()
    src = _mixed(dynamic)
    total = sum(_count(s["format"], s["data"]) for s in src)
    e = _engine(total, dynamic=dynamic, ray=False)
    try:
        infos = e.upload_scenes(src, sh_degree=2)
        n = sum(i["splat_count"] for i in infos)
        mesh = dict(sh_degree=2, compression_level=2)
        f, cc, cov, sh, idx, centers = _fed_engine(e, n, dynamic, mesh)
        try:
            mvp, u, view = _camera()
            u.scene_count = len(infos)
            u.sh8_min = np.full(N.GS_MAX_SCENES, -1.5, np.float32); u.sh8_max = np.full(N.GS_MAX_SCENES, 1.5, np.float32)
            for s, i in enumerate(infos):
                u.sh8_min[s], u.sh8_max[s] = i["min_sh_coeff"], i["max_sh_coeff"]
            assert len(set(u.sh8_min[:len(infos)].tolist())) > 1 or len(set(u.sh8_max[:len(infos)].tolist())) > 1
            u.enable_optional_effects = 1
            u.scene_opacity = np.ones(N.GS_MAX_SCENES, np.float32); u.scene_opacity[1] = 0.5
            u.scene_visibility = np.ones(N.GS_MAX_SCENES, np.int32); u.scene_visibility[2] = 0
            tr = None
            for step in range(3 if dynamic else 1):
                if dynamic:
                    tr = np.tile(np.eye(4, dtype=np.float32).reshape(16), (N.GS_MAX_SCENES, 1))
                    tr[0] = _xf((0.3 * step, 0.0, 0.0)).astype(np.float32)
                    tr[3] = _xf((0.0, -0.2 * step, 0.1), (0.0, np.sin(0.1 * step), 0.0, np.cos(0.1 * step))).astype(np.float32)
                    u.dynamic_mode, u.scene_transforms, u.view_matrix = 1, tr, view.astype(np.float32)
                for fmt in (N.GS_FRAME_RGBA32F, N.GS_FRAME_RGBA8):
                    got = _frame(e, n, u, mvp, tr, fmt)
                    assert np.array_equal(got, _frame(f, n, u, mvp, tr, fmt)), (step, fmt)
                    assert np.array_equal(e.read_buffer(N.GS_BUF_SORTED_INDEXES, np.uint32, n), f.read_buffer(N.GS_BUF_SORTED_INDEXES, np.uint32, n))
                got = _frame(e, n, u, mvp, tr)
                # the draw order against the reference sorter (the compiled one in oracle/_ref) fed the same sceneIndexes and transforms
                sort = dict(centers=centers, mvp=mvp, scene_indexes=idx if dynamic else None, transforms=tr, dynamic=dynamic)
                FF.check_frame(f"multi-scene dynamic={dynamic} step {step}", e, u, W, H, n, cc, cov, sh, 2, idx, got=got, flip_y=True, sort=sort)
        finally:
            f.close()
    finally:
        e.close()


def test_rejections_name_the_scene_and_keep_the_frame():
    N = _N()
    from gaussiansplats3d_b200 import GsError
    src = _mixed()
    total = sum(_count(s["format"], s["data"]) for s in src)
    e = _engine(total)
    d = _engine(total, dynamic=True, ray=False)
    sharded = None
    try:
        infos = e.upload_scenes(src, sh_degree=2)
        n = sum(i["splat_count"] for i in infos)
        mvp, u, _ = _camera()
        u.scene_count = len(infos)
        before = _frame(e, n, u, mvp)
        ok = dict(format=3, data=_golden("ksplat_handmade_l1_sh1.ksplat"))
        big = dict(format=3, data=_golden("ksplat_handmade_l0_sh2.ksplat"))
        cases = [
            ([ok, dict(format=3, data=b"\0" * 100)], N.GS_ERR_BAD_ARG, "scene 1"),
            ([ok] * 33, N.GS_ERR_BAD_ARG, "33 scenes"),
            ([ok, dict(format=1, data=_golden("inriav2_codebook_sh2.ply"))], N.GS_ERR_BAD_ARG, "scene 1"),
            ([dict(format=1, data=_golden("file_handmade_sh2.ply")), ok, dict(format=3, data=_golden("ksplat_handmade_l2_sh2_two_sections.ksplat"))] + [big] * 8,
             N.GS_ERR_CAPACITY, "scene"),
        ]
        for srcs, code, words in cases:
            with pytest.raises(GsError) as ei:
                e.upload_scenes(srcs, sh_degree=2)
            assert ei.value.code == code and words in str(ei.value), (words, str(ei.value))
            assert np.array_equal(_frame(e, n, u, mvp), before), words
        # a transform on a dynamic engine: refused, the dynamic mesh it holds renders as before
        dn = sum(i["splat_count"] for i in d.upload_scenes([ok, big], sh_degree=2))
        tr = np.tile(np.eye(4, dtype=np.float32).reshape(16), (N.GS_MAX_SCENES, 1))
        du = _camera()[1]
        du.scene_count, du.dynamic_mode, du.scene_transforms, du.sh_degree = 2, 1, tr, 1
        before = _frame(d, dn, du, mvp, tr)
        with pytest.raises(GsError) as ei:
            d.upload_scenes([ok, dict(ok, transform16=T1)], sh_degree=2)
        assert ei.value.code == N.GS_ERR_BAD_ARG and "scene 1" in str(ei.value) and "dynamic" in str(ei.value)
        assert np.array_equal(_frame(d, dn, du, mvp, tr), before)
        # several scenes on a sharded engine: multi-scene frames are single-GPU only
        from gaussiansplats3d_b200 import Engine
        sharded = Engine(total, max_width=W, max_height=H, rank=0, world_size=2)
        with pytest.raises(GsError) as ei:
            sharded.upload_scenes([ok, big], sh_degree=2)
        assert ei.value.code == N.GS_ERR_BAD_ARG and "single-GPU" in str(ei.value)
        sharded.upload_scenes([ok], sh_degree=2)
    finally:
        e.close(); d.close()
        if sharded is not None:
            sharded.close()


class _Scenes:
    """oracle/ray_oracle.py's Scene per scene of a mesh: splat i is read with its own scene's transform, and a splat of an invisible
    scene is skipped (Raycaster.js:112-114) as the oracle skips a splat of zero scale."""

    def __init__(self, rec, infos, transforms, visible):
        from oracle import ray_oracle as RO
        self.of = np.repeat(np.arange(len(infos)), [i["splat_count"] for i in infos])
        self.scenes = [RO.Scene(rec["center"], rec["scale"], rec["rotation"], rec["alpha"], transform16=t) for t in transforms]
        self.visible = visible

    def inputs(self, i, ellipsoid):
        s = int(self.of[i])
        c, sc, F, Inv = self.scenes[s].inputs(i, ellipsoid)
        return (c, sc, F, Inv) if self.visible[s] else (c, (0.0, 0.0, 0.0), F, Inv)


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a, np.float64).view(np.uint64), np.asarray(b, np.float64).view(np.uint64))


def test_tree_and_raycast_over_scenes():
    from oracle import ray_oracle as RO
    from gaussiansplats3d_b200.raycaster import record_centers_f32
    from gaussiansplats3d_b200.splat_tree import SplatTree
    src = _mixed()
    total = sum(_count(s["format"], s["data"]) for s in src)
    e, plain = _engine(total), _engine(total, ray=False)
    try:
        infos = e.upload_scenes(src, sh_degree=2)
        assert plain.upload_scenes(src, sh_degree=2) == infos
        n = sum(i["splat_count"] for i in infos)
        rec = e.read_buffer(_N().GS_BUF_RAY_RECORDS, _N().RAY_RECORD_DTYPE, n)
        cc = e.read_buffer(_N().GS_BUF_CENTERS_COLORS, np.uint32, n * 4).reshape(n, 4)
        alpha = (cc[:, 0] >> 24).astype(np.uint8)
        transforms = [s.get("transform16") for s in src]
        centers = np.concatenate([record_centers_f32(rec[i["splat_offset"]:i["splat_offset"] + i["splat_count"]], t) for t, i in zip(transforms, infos)])
        # with ray records: getSplatCenter's centres, each scene's transform applied to the unrounded centre; without: the f32 texel centres
        for eng, c in ((e, centers), (plain, cc[:, 1:4].copy().view(np.float32))):
            want = SplatTree(8, 1000).processSplatMesh(c, alpha, 1)
            eng.build_splat_tree(8, 1000, 1)
            got = eng.read_splat_tree()
            assert got.count == want.count
            for k in ("offsets", "indexes", "node_center", "node_min", "node_max", "depth"):
                assert np.array_equal(np.asarray(getattr(got, k)), np.asarray(getattr(want, k))), k
        # rays down -z through one kept splat of every scene, against the oracle with per-scene transforms and visibility
        root = RO.build_tree(centers, alpha)
        rays = []
        for i in infos:
            lo, cnt = i["splat_offset"], i["splat_count"]
            k = lo + int(np.flatnonzero(alpha[lo:lo + cnt] > 0)[0])
            rays.append(((float(centers[k, 0]), float(centers[k, 1]), float(centers[k, 2]) + 10.0), (0.0, 0.0, -1.0)))
        for vis in ([True] * len(infos), [s != 1 for s in range(len(infos))], [s in (0, 3) for s in range(len(infos))]):
            scenes = _Scenes(rec, infos, transforms, vis)
            for ellipsoid in (False, True):
                for o, d in rays:
                    want = RO.intersect_splat_mesh(root, scenes, o, d, RO.IDENTITY, ellipsoid=ellipsoid)
                    got, tot = e.raycast(o, d, None, ellipsoid=ellipsoid, capacity=len(want) + 3, scene_visibility=vis)
                    assert tot == len(want) and got.shape[0] == len(want), (vis, ellipsoid)
                    assert np.array_equal(got["splat_index"], np.array([h[2] for h in want], np.uint32))
                    assert _bits_equal(got["distance"], [h[0] for h in want])
                    assert _bits_equal(got["origin"], np.array([h[3] for h in want]).reshape(-1, 3))
                    assert _bits_equal(got["normal"], np.array([h[4] for h in want]).reshape(-1, 3))
                    hidden = np.flatnonzero(~np.asarray(vis))
                    assert not np.isin(scenes.of[got["splat_index"].astype(np.int64)], hidden).any()
        assert any(e.raycast(o, d, None, capacity=1)[1] for o, d in rays)
    finally:
        e.close(); plain.close()


def _viewer(**kw):
    from gaussiansplats3d_b200.viewer import Viewer
    return Viewer({**dict(width=W, height=H, sphericalHarmonicsDegree=2, initialCameraPosition=(0, 0.5, 6)), **kw})


def _viewer_state(v):
    n = v.splatMesh.getSplatCount()
    mesh = dict(sh_degree=v.splatMesh.packed.sh_degree, compression_level=2 if any(i["compression_level"] == 2 for i in v.splatMesh.sceneInfos) else 1)
    bufs = [_bytes(v.engine, b, n, mesh) for b in ("GS_BUF_CENTERS_COLORS", "GS_BUF_COVARIANCES", "GS_BUF_SH", "GS_BUF_CENTERS")]
    return bufs, v.frame(frame_format=_N().GS_FRAME_RGBA32F).copy()


def _opts(kind):
    return {"l2": dict(format=3, data=_golden("ksplat_handmade_l2_sh2_two_sections.ksplat"), position=(0.5, 0, 0)),
            "l0": dict(format=3, data=_golden("ksplat_handmade_l0_sh2.ksplat"), rotation=(0, 0.6, 0, 0.8), opacity=0.5),
            "ply": dict(format=1, data=_golden("file_handmade_sh2.ply"), scale=(0.5, 0.5, 0.5), splatAlphaRemovalThreshold=30)}[kind]


@pytest.mark.parametrize("dynamic", [False, True])
def test_viewer_add_and_remove(dynamic):
    a, b, c = _viewer(dynamicScene=dynamic), _viewer(dynamicScene=dynamic), _viewer(dynamicScene=dynamic)
    try:
        a.addSplatScenes([_opts("l2"), _opts("l0")])
        a.addSplatScenes([_opts("ply")])
        b.addSplatScenes([_opts("l2"), _opts("l0"), _opts("ply")])
        assert a.getSceneCount() == 3
        sa, sb = _viewer_state(a), _viewer_state(b)
        assert all(np.array_equal(x, y) for x, y in zip(sa[0], sb[0])) and np.array_equal(sa[1], sb[1])
        a.getSplatScene(2).position = (0.0, 0.25, 0.0)     # a remaining scene's current transform is kept
        a.removeSplatScenes([0])                           # the only level-2 scene: SH back to f16
        c.addSplatScenes([_opts("l0"), dict(_opts("ply"), position=(0.0, 0.25, 0.0))])
        assert a.getSceneCount() == 2 and all(i["compression_level"] < 2 for i in a.splatMesh.sceneInfos)
        sa, sc = _viewer_state(a), _viewer_state(c)
        assert all(np.array_equal(x, y) for x, y in zip(sa[0], sc[0])) and np.array_equal(sa[1], sc[1])
        sh = a.engine.read_buffer(_N().GS_BUF_SH, np.float16, a.splatMesh.getSplatCount() * 24)
        assert np.isfinite(sh.astype(np.float32)).all()
    finally:
        a.dispose(); b.dispose(); c.dispose()


def test_demo_shape_dynamic_frames_within_f64_bounds():
    """demo/dynamic_scenes.html at test size: a 50 k scene and two 10 k scenes, the two small ones moving over several frames."""
    N = _N()
    from gaussiansplats3d_b200.engine import generate_splat_buffer
    from test_scene_upload_gpu import _synthetic_ply
    imgs = [generate_splat_buffer(N.GS_FILE_PLY, _synthetic_ply(n, seed), sh_degree=1, compression_level=lvl)
            for n, seed, lvl in ((50_000, 1, 2), (10_000, 2, 1), (10_000, 3, 1))]
    v = _viewer(dynamicScene=True, sphericalHarmonicsDegree=1)
    try:
        v.addSplatScenes([dict(format=3, data=imgs[0]), dict(format=3, data=imgs[1], position=(2, 0, 0), scale=(0.3, 0.3, 0.3)),
                          dict(format=3, data=imgs[2], position=(-2, 0, 0), scale=(0.3, 0.3, 0.3))])
        n = v.splatMesh.getSplatCount()
        cc = v.engine.read_buffer(N.GS_BUF_CENTERS_COLORS, np.uint32, n * 4).reshape(n, 4)
        cov = v.engine.read_buffer(N.GS_BUF_COVARIANCES, np.float32, n * 6).reshape(n, 6)
        sh = v.engine.read_buffer(N.GS_BUF_SH, np.uint8, n * 9).reshape(n, 9)
        idx = v.engine.read_buffer(N.GS_BUF_SCENE_INDEXES, np.uint32, n)
        for step in range(3):
            t = 0.4 * step
            v.getSplatScene(1).position = (2 * np.cos(t), 0.0, 2 * np.sin(t))
            v.getSplatScene(2).position = (-2 * np.cos(t), 0.5 * np.sin(t), 0.0)
            got = v.frame(frame_format=N.GS_FRAME_RGBA32F).copy()
            v.updateSplatMesh()
            FF.check_frame(f"demo step {step}", v.engine, v.uniforms(), W, H, n, cc, cov, sh, 1, idx, got=got, flip_y=True)
    finally:
        v.dispose()
