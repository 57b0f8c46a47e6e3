"""GPU: streamed loads (gs_stream_open / gs_stream_append / gs_stream_close), the visible region (gs_visible_region) and the Viewer's
progressive load and scene reveal.  After every append the engine holds the whole-file upload restricted to the loaded prefix; after close
it holds the whole-file upload, bit for bit."""
from __future__ import annotations

import re
from pathlib import Path

import numpy as np
import pytest

from gaussiansplats3d_b200 import Engine, GsError, _native as N
from gaussiansplats3d_b200.loaders import SceneFormat
from gaussiansplats3d_b200.viewer import SceneRevealMode, Viewer

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden"
SIZES = {"float": 4, "uint": 4, "int": 4, "uchar": 1, "char": 1, "short": 2, "ushort": 2, "double": 8}


def inria_ply(n: int, nrest: int, seed: int) -> bytes:
    names = ["x", "y", "z", "f_dc_0", "f_dc_1", "f_dc_2"] + [f"f_rest_{k}" for k in range(nrest)] + \
            ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    rng = np.random.default_rng(seed)
    rec = rng.standard_normal((n, len(names))).astype(np.float32)
    rec[:, 0:3] = rng.uniform(-6, 6, (n, 3))
    rec[:, 7 + nrest:10 + nrest] = rng.uniform(-5, -2, (n, 3))   # scale_0..2
    head = "\n".join(["ply", "format binary_little_endian 1.0", f"element vertex {n}", *[f"property float {k}" for k in names], "end_header"]) + "\n"
    return head.encode() + rec.tobytes()


def pc_ply(n: int, seed: int) -> bytes:
    rng = np.random.default_rng(seed)
    nc = (n + 255) // 256
    ext = ["min_x", "min_y", "min_z", "max_x", "max_y", "max_z", "min_scale_x", "min_scale_y", "min_scale_z",
           "max_scale_x", "max_scale_y", "max_scale_z", "min_r", "min_g", "min_b", "max_r", "max_g", "max_b"]
    lo = np.concatenate([rng.uniform(-5, 0, (nc, 3)), rng.uniform(-6, -4, (nc, 3)), rng.uniform(-0.2, 0.3, (nc, 3))], 1)
    hi = lo + np.concatenate([rng.uniform(1, 5, (nc, 3)), rng.uniform(0.5, 2, (nc, 3)), rng.uniform(0.5, 1, (nc, 3))], 1)
    chunk = np.empty((nc, 18), np.float32)
    chunk[:, [0, 1, 2, 6, 7, 8, 12, 13, 14]], chunk[:, [3, 4, 5, 9, 10, 11, 15, 16, 17]] = lo, hi
    vertex = rng.integers(0, 1 << 32, (n, 4), dtype=np.uint64).astype(np.uint32)
    head = "\n".join(["ply", "format binary_little_endian 1.0", f"element chunk {nc}", *[f"property float {k}" for k in ext],
                      f"element vertex {n}", *[f"property uint packed_{k}" for k in ("position", "rotation", "scale", "color")], "end_header"]) + "\n"
    return head.encode() + chunk.tobytes() + vertex.tobytes()


def splat_rows(n: int, seed: int) -> bytes:
    rng = np.random.default_rng(seed)
    rec = np.empty((n, 8), np.float32)
    rec[:, 0:3] = rng.uniform(-6, 6, (n, 3))
    rec[:, 3:6] = np.exp(rng.uniform(-5, -2, (n, 3)))
    rec[:, 6:8] = rng.integers(0, 256, (n, 8), dtype=np.uint8).view(np.float32)
    return rec.tobytes()


def ply_layout(data: bytes):
    """(offset of the first vertex record, vertex stride, vertex count) of a .ply"""
    end = data.index(b"end_header") + len(b"end_header\n")
    elems = []
    for line in data[:end].decode().split("\n"):
        w = line.split()
        if w[:1] == ["element"]:
            elems.append([w[1], int(w[2]), 0])
        elif w[:1] == ["property"]:
            elems[-1][2] += SIZES[w[1]]
    off = end
    for name, count, stride in elems:
        if name == "vertex":
            return off, stride, count
        off += count * stride
    raise AssertionError("no vertex element")


FILES = {
    "ply_sh0": lambda: (GOLDEN / "file_handmade_sh0.ply").read_bytes(),
    "ply_sh1": lambda: (GOLDEN / "file_handmade_sh1.ply").read_bytes(),
    "ply_sh2": lambda: (GOLDEN / "file_handmade_sh2.ply").read_bytes(),
    "ply_sh3": lambda: (GOLDEN / "file_handmade_sh3.ply").read_bytes(),
    "ply_nonfinite": lambda: (GOLDEN / "file_handmade_nonfinite.ply").read_bytes(),
    "ply_synth_sh1": lambda: inria_ply(1500, 9, 3),
    "pcply_synth": lambda: pc_ply(700, 4),
    "splat_golden": lambda: (GOLDEN / "file_handmade_basic.splat").read_bytes(),
    "splat_synth": lambda: splat_rows(900, 5),
    "ksplat_l0_sh0": lambda: (GOLDEN / "ksplat_handmade_l0_sh0.ksplat").read_bytes(),
    "ksplat_l0_sh2": lambda: (GOLDEN / "ksplat_handmade_l0_sh2.ksplat").read_bytes(),
    "ksplat_l1_sh0": lambda: (GOLDEN / "ksplat_handmade_l1_sh0_many_buckets.ksplat").read_bytes(),
    "ksplat_l1_sh1": lambda: (GOLDEN / "ksplat_handmade_l1_sh1.ksplat").read_bytes(),
    "ksplat_l2_two_sections": lambda: (GOLDEN / "ksplat_handmade_l2_sh2_two_sections.ksplat").read_bytes(),
}


def fmt_of(name: str) -> int:
    return SceneFormat.KSplat if name.startswith("ksplat") else (SceneFormat.Splat if name.startswith("splat") else SceneFormat.Ply)


def engine(cap: int) -> Engine:
    return Engine(max(cap, 1), max_width=64, max_height=64, ray_records=True)


def whole(fmt: int, data: bytes, cap: int):
    e = engine(cap)
    info = e.upload_ksplat(data) if fmt == SceneFormat.KSplat else e.upload_file(fmt, data, sh_degree=2)
    return e, info


def state(e: Engine, n: int, info: dict) -> dict:
    if n == 0:
        return {}
    ncomp = {0: 0, 1: 9, 2: 24}[info["sh_degree"]]
    out = dict(cc=e.read_buffer(N.GS_BUF_CENTERS_COLORS, np.uint32, 4 * n), cov=e.read_buffer(N.GS_BUF_COVARIANCES, np.uint8, 24 * n),
               centers=e.read_buffer(N.GS_BUF_CENTERS, np.int32, 4 * n), ray=e.read_buffer(N.GS_BUF_RAY_RECORDS, np.uint8, 56 * n))
    if ncomp:
        out["sh"] = e.read_buffer(N.GS_BUF_SH, np.uint8, ncomp * (1 if info["compression_level"] == 2 else 2) * n)
    return out


def same(a: dict, b: dict) -> bool:
    return a.keys() == b.keys() and all(np.array_equal(a[k], b[k]) for k in a)


def ksplat_complete(data: bytes, received: int) -> int:
    """Splats of a .ksplat whose records lie in the first `received` bytes (SplatBuffer.js:819-941 layout)"""
    u32 = lambda o: int.from_bytes(data[o:o + 4], "little")  # noqa: E731
    sections, level = u32(4), int.from_bytes(data[20:22], "little")
    kC, kS, kR, kSH = (12, 6, 6), (12, 6, 6), (16, 8, 8), (4, 2, 1)
    if received < 4096 + 1024 * sections:
        return 0
    base, done = 4096 + 1024 * sections, 0
    for i in range(sections):
        h = 4096 + 1024 * i
        count, bucket_count, storage, partial = u32(h + 4), u32(h + 12), int.from_bytes(data[h + 20:h + 22], "little"), u32(h + 36)
        deg = int.from_bytes(data[h + 40:h + 42], "little")
        bps = kC[level] + kS[level] + kR[level] + 4 + kSH[level] * {0: 0, 1: 9, 2: 24}[deg]
        data_base = base + storage * bucket_count + 4 * partial
        k = 0 if received <= data_base else min(count, (received - data_base) // bps)
        done += k
        if k < count:
            break
        base = data_base + bps * count
    return done


def expected_loaded(fmt: int, data: bytes, received: int) -> int:
    if fmt == SceneFormat.KSplat:
        return ksplat_complete(data, received)
    if fmt == SceneFormat.Splat:
        return received // 32
    if b"end_header\n" not in data[:received]:
        return 0
    off, stride, count = ply_layout(data)
    return 0 if received <= off else min(count, (received - off) // stride)


def split_points(name: str, data: bytes, rng) -> dict:
    fmt = fmt_of(name)
    head = 4096 + 1024 * int.from_bytes(data[4:8], "little") if fmt == SceneFormat.KSplat else \
        (0 if fmt == SceneFormat.Splat else data.index(b"end_header") + 11)
    out = {"one": [len(data)], "header": [max(head // 2, 1), len(data)]}
    if len(data) <= 6000:
        out["bytes"] = list(range(1, len(data) + 1))
    if fmt != SceneFormat.KSplat:
        off, stride, count = (0, 32, len(data) // 32) if fmt == SceneFormat.Splat else ply_layout(data)
        cuts = {off + i * stride + d for i in range(0, count + 1, max(1, count // 9)) for d in (-1, 0, 1)}
        out["records"] = sorted(c for c in cuts if 0 < c < len(data)) + [len(data)]
    cuts, at = [], 0
    while at < len(data):
        at = min(len(data), at + int(rng.integers(1, 400)))
        cuts.append(at)
    out["random"] = cuts
    return out


@pytest.mark.parametrize("name", sorted(FILES))
def test_prefix_equality_after_every_append_and_close_equals_whole(name):
    data, fmt = FILES[name](), fmt_of(name)
    cap = 4096
    ref, info = whole(fmt, data, cap)
    n = info["splat_count"]
    want = state(ref, n, info)
    rng = np.random.default_rng(sum(map(ord, name)))
    for split, cuts in split_points(name, data, rng).items():
        e = engine(cap)
        s = e.open_stream(fmt, sh_degree=2)
        at = 0
        for c in cuts:
            loaded = s.append(data[at:c])
            at = c
            assert loaded == expected_loaded(fmt, data, at), (split, at)
            if split != "bytes" or loaded in (0, 1, n) or at == len(data):
                got = state(e, loaded, info)
                assert same(got, {k: v[:len(v) * loaded // n] for k, v in want.items()} if loaded else {}), (split, at)
        got_info = s.close()
        assert got_info == info
        assert same(state(e, n, info), want), split


def test_close_matches_whole_upload_sort_tree_and_raycast():
    data = inria_ply(3000, 24, 11)
    ref, info = whole(SceneFormat.Ply, data, 4096)
    e = engine(4096)
    s = e.open_stream(SceneFormat.Ply, sh_degree=2)
    for k in range(0, len(data), 70001):
        s.append(data[k:k + 70001])
    assert s.close() == info
    mvp = np.array([1.2, 0.1, 0.3, 0.3, 0.0, 1.1, 0.2, 0.2, 0.1, -0.1, 1.0, 1.0, 0.5, 0.2, 9.0, 10.0], np.float32)
    assert np.array_equal(e.sort(mvp, 3000, 3000)[0], ref.sort(mvp, 3000, 3000)[0])
    e.build_splat_tree()
    ref.build_splat_tree()
    assert deep_eq(e.read_splat_tree(), ref.read_splat_tree())
    off, _, _ = ply_layout(data)
    c0 = np.frombuffer(data[off:off + 12], np.float32).astype(np.float64)   # a ray through splat 0's centre
    o = (c0[0], c0[1], c0[2] - 20.0)
    h1, h2 = e.raycast(o, (0.0, 0.0, 1.0), capacity=8), ref.raycast(o, (0.0, 0.0, 1.0), capacity=8)
    assert h2[1] > 0 and deep_eq(h1, h2)


def deep_eq(a, b) -> bool:
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        a, b = np.asarray(a), np.asarray(b)
        return a.shape == b.shape and a.tobytes() == b.tobytes()
    if isinstance(a, (list, tuple)):
        return type(a) is type(b) and len(a) == len(b) and all(deep_eq(x, y) for x, y in zip(a, b))
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(deep_eq(a[k], b[k]) for k in a)
    if hasattr(a, "__dict__"):
        return deep_eq(vars(a), vars(b))
    return a == b


def prefix_ply(data: bytes, k: int) -> bytes:
    off, stride, count = ply_layout(data)
    head = re.sub(rb"element vertex \d+", b"element vertex %d" % k, data[:off])
    return head + data[off:off + k * stride]


def viewer(**extra) -> Viewer:
    return Viewer(dict(width=64, height=48, sphericalHarmonicsDegree=1, initialCameraPosition=(0.5, 1.0, -14.0),
                       initialCameraLookAt=(0.0, 0.0, 0.0), **extra))


@pytest.mark.parametrize("graph", [True, False])
def test_frames_between_appends_equal_a_fresh_load_of_the_prefix(graph):
    data = inria_ply(12000, 9, 21)   # 104 B per splat: a build about every 2500 splats
    v = viewer()
    load = v.addSplatSceneProgressive(SceneFormat.Ply)
    frames = []
    for k in range(0, len(data), 100000):
        if load.append(data[k:k + 100000]):
            v.engine.set_graph_enabled(graph)
            v.camera.update(); v.updateSplatMesh()
            frames.append((v.splatRenderCount, v.frame(frame_format=N.GS_FRAME_RGBA32F)))
    load.finish()
    v.camera.update(); v.updateSplatMesh()
    frames.append((v.splatRenderCount, v.frame(frame_format=N.GS_FRAME_RGBA32F)))
    assert len(frames) >= 4 and frames[-1][0] == 12000
    assert [c for c, _ in frames[:-1]] == load.builds[:-1]
    for count, frame in frames:
        w = viewer()
        w.addSplatSceneFromFile(prefix_ply(data, count), SceneFormat.Ply, progressiveLoad=True)
        w.engine.set_graph_enabled(graph)
        w.camera.update(); w.updateSplatMesh()
        assert np.array_equal(frame, w.frame(frame_format=N.GS_FRAME_RGBA32F)), count


def test_pipelined_frames_across_appends():
    """Frames in flight while the next append decodes: each one pictures the prefix it was begun with."""
    data = inria_ply(30000, 0, 22)   # 56 B per splat
    v = viewer()
    load = v.addSplatSceneProgressive(SceneFormat.Ply)
    inflight, done = [], []
    for k in range(0, len(data), 90000):
        if load.append(data[k:k + 90000]):
            v.camera.update(); v.updateSplatMesh()
            out = np.empty((48, 64, 4), np.uint8)
            prep = v.engine.prepare_frame(v.mvp_matrix().astype(np.float32), v.uniforms(), 64, 48, v.splatRenderCount)
            v.engine.frame_begin(prep, out)
            inflight.append((v.splatRenderCount, out))
            if len(inflight) == 2:
                v.engine.frame_end()
                done.append(inflight.pop(0))
    for _ in inflight:
        v.engine.frame_end()
    done += inflight
    load.finish()
    assert len(done) >= 4
    for count, out in done:
        w = viewer()
        w.addSplatSceneFromFile(prefix_ply(data, count), SceneFormat.Ply, progressiveLoad=True)
        w.camera.update(); w.updateSplatMesh()
        assert np.array_equal(out, w.frame()), count


def region_max(c32: np.ndarray, t=None, center=(0.0, 0.0, 0.0)) -> float:
    """updateVisibleRegion's loop restated in NumPy f64 (getSplatCenter(i, c, true), sub, length, `d > max`)"""
    T = np.eye(4).reshape(16) if t is None else np.asarray(t, np.float64).reshape(16)
    x, y, z = (c32[:, k].astype(np.float64) for k in range(3))
    with np.errstate(all="ignore"):
        w = 1.0 / (((T[3] * x + T[7] * y) + T[11] * z) + T[15])
        c = [(((T[r] * x + T[4 + r] * y) + T[8 + r] * z) + T[12 + r]) * w for r in range(3)]
        d = [c[k] - center[k] for k in range(3)]
        dist = np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])
    dist = dist[dist > 0]
    return float(dist.max()) if dist.size else 0.0


@pytest.mark.parametrize("name", ["ply_synth_sh1", "ply_nonfinite", "ksplat_l1_sh1", "splat_synth"])
def test_visible_region_bit_exact(name):
    data, fmt = FILES[name](), fmt_of(name)
    e, info = whole(fmt, data, 4096)
    n = info["splat_count"]
    c32 = e.read_buffer(N.GS_BUF_CENTERS_COLORS, np.uint32, 4 * n).reshape(n, 4)[:, 1:].copy().view(np.float32)
    t = np.array([0.9, 0.1, 0.0, 0.0, -0.1, 0.9, 0.2, 0.0, 0.0, -0.2, 1.1, 0.001, 0.5, -1.5, 2.0, 1.0])
    for lo, hi in [(0, n), (n // 3, n), (1, 2), (5, 5)]:
        for tr, ctr in [(None, None), (t, None), (t, (0.25, -1.0, 3.0))]:
            got = e.visible_region(lo, hi, tr, ctr)
            want = region_max(c32[lo:hi], tr, (0.0, 0.0, 0.0) if ctr is None else ctr)
            assert got == want or (np.isinf(got) and np.isinf(want)), (lo, hi, tr is None, ctr)
    with pytest.raises(GsError):
        e.visible_region(0, n + 1)


def test_refusals():
    prev = inria_ply(50, 0, 1)
    e = engine(100)
    e.upload_file(SceneFormat.Ply, prev)
    before = state(e, 50, dict(sh_degree=0, compression_level=0))

    def refused(fmt, data, match, code=N.GS_ERR_BAD_ARG, sh=0):
        s = e.open_stream(fmt, sh_degree=sh)
        with pytest.raises(GsError) as ei:
            s.append(data)
        assert ei.value.code == code and re.search(match, str(ei.value)), str(ei.value)
        assert same(state(e, 50, dict(sh_degree=0, compression_level=0)), before)

    with pytest.raises(GsError, match="spz"):
        e.open_stream(SceneFormat.Spz)
    refused(SceneFormat.Ply, (GOLDEN / "inriav2_codebook_sh1.ply").read_bytes(), "INRIA v2")
    refused(SceneFormat.Ply, (GOLDEN / "pcply_handmade_sh1.ply").read_bytes(), "PlayCanvas.*spherical harmonics")
    refused(SceneFormat.Ply, b"ply\nformat ascii 1.0\nelement vertex 3\nend_header\n", "")
    refused(SceneFormat.Ply, inria_ply(101, 0, 2), "capacity", N.GS_ERR_CAPACITY)
    refused(SceneFormat.Splat, splat_rows(101, 2), "capacity", N.GS_ERR_CAPACITY)
    multi = Engine(100, max_width=64, max_height=64, rank=0, world_size=2)
    with pytest.raises(GsError, match="world_size"):
        multi.open_stream(SceneFormat.Ply)
    # short stream: the prefix stays loaded and renderable
    data = inria_ply(80, 0, 3)
    s = e.open_stream(SceneFormat.Ply)
    off, stride, _ = ply_layout(data)
    assert s.append(data[:off + 30 * stride + 5]) == 30
    with pytest.raises(GsError, match="30 of the 80"):
        s.close()
    with pytest.raises(GsError, match="closed"):
        s.append(b"x")
    ref, info = whole(SceneFormat.Ply, data, 100)
    assert same(state(e, 30, info), {k: v[:len(v) * 30 // 80] for k, v in state(ref, 80, info).items()})
    s = e.open_stream(SceneFormat.Splat)
    s.append(splat_rows(3, 4)[:70])
    with pytest.raises(GsError, match="ended short"):
        s.close()


def reveal_restated(dists, mode, frames_per_build, multiplier=1.0):
    """SplatMesh.updateVisibleRegion / updateVisibleRegionFadeDistance over the same builds, restated: (fadeStartRadius, complete) per frame"""
    st = dict(maxd=0.0, buf=0.0, radius=0.0, fade=0.0)
    out = []

    def fade(m, final):
        fast, gradual = 0.012 * multiplier, 0.003 * multiplier
        rate = (fast if final else gradual) if m == SceneRevealMode.Default else gradual
        st["fade"] = (st["radius"] - st["fade"]) * rate + st["fade"]
        pct = st["fade"] / st["buf"] if st["buf"] > 0 else 0
        return (pct > 0.99) or m == SceneRevealMode.Instant

    for i, d in enumerate(dists):
        final = i == len(dists) - 1
        st["maxd"] = max(st["maxd"], d)
        if st["maxd"] - st["buf"] > 1:
            st["buf"] = st["maxd"]
            st["radius"] = max(st["buf"] - 1, 0.0)
        if final:
            st["radius"] = st["buf"] = st["maxd"]
        fade(SceneRevealMode.Default, final)
        for _ in range(frames_per_build):
            c = fade(mode, final)
            out.append((st["fade"], c))
    return out


@pytest.mark.parametrize("mode", [SceneRevealMode.Default, SceneRevealMode.Gradual, SceneRevealMode.Instant])
def test_viewer_reveal_uniforms_follow_the_reference(mode):
    data = inria_ply(9000, 0, 31)
    v = viewer(sceneRevealMode=int(mode), sceneFadeInRateMultiplier=2.0)
    load = v.addSplatSceneProgressive(SceneFormat.Ply)
    got, dists, prev = [], [], 0
    off, stride, _ = ply_layout(data)
    c32 = np.frombuffer(data[off:], np.float32).reshape(9000, -1)[:, :3]

    def frames():   # Viewer.frame runs updateSplatMesh, and with it one updateVisibleRegionFadeDistance(sceneRevealMode)
        for _ in range(3):
            v.frame()
            u = v.uniforms()
            got.append((u.visible_region_fade_start_radius, u.fade_in_complete))

    for k in range(0, len(data), 50000):
        if load.append(data[k:k + 50000]):
            dists.append(region_max(c32[prev:v.splatRenderCount]))
            prev = v.splatRenderCount
            frames()
    load.finish()
    dists.append(region_max(c32[prev:9000]))
    frames()
    want = reveal_restated(dists, mode, 3, 2.0)
    assert len(got) == len(want)
    for (gr, gc), (wr, wc) in zip(got, want):
        assert gr == np.float32(wr) and gc == (1 if wc else 0)


def test_viewer_without_reveal_option_renders_as_before():
    data = inria_ply(4000, 9, 41)
    a, b = viewer(), viewer()
    a.addSplatSceneFromFile(data, SceneFormat.Ply, progressiveLoad=True)
    load = b.addSplatSceneProgressive(SceneFormat.Ply)
    for k in range(0, len(data), 65536):
        if load.append(data[k:k + 65536]):
            b.camera.update(); b.updateSplatMesh()
            assert b.uniforms().fade_in_complete == 1
    load.finish()
    for v in (a, b):
        v.camera.update(); v.updateSplatMesh()
    assert a.uniforms().fade_in_complete == b.uniforms().fade_in_complete == 1
    assert np.array_equal(a.frame(), b.frame())
