"""Every way of enqueueing a frame computes the same frame: gs_frame with and without its CUDA graph, with profiling, gs_frame_async +
gs_synchronize, gs_frame_begin / gs_frame_end two and three deep, and gs_sort + gs_render give byte-identical frames, sorted indexes,
tile-instance and visible-splat counts.  The kernels each entry launches, and their order, are pinned, and so is the rule for which
error a frame that trips several reports."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_SPLATS = 150_000

# Kernel timelines (gs_kernel_timings names) of a 150 K-splat SH1 bonsai scene at 640x360 RGBA8, 16-bit keys.
LAUNCHES = {
    "sort": [
        "k_depth", "k_bucket", "k_radix_scan[depth,0]", "k_radix_scatter[depth,0]", "k_radix_hist[depth,1]", "k_radix_scan[depth,1]",
        "k_radix_scatter[depth,1]",
    ],
    "render": [
        "k_raster_init", "k_project", "k_bin_count", "k_bin_scan", "k_bin_place", "k_blend",
    ],
    "frame": [
        "k_depth", "k_bucket", "k_radix_scan[depth,0]", "k_radix_scatter[depth,0]", "k_radix_hist[depth,1]", "k_radix_scan[depth,1]",
        "k_radix_scatter[depth,1]", "k_raster_init", "k_project", "k_bin_count", "k_bin_scan", "k_bin_place", "k_blend",
    ],
    "subset_frame": [
        "k_raster_init", "k_project", "k_depth", "k_subset_count", "k_subset_emit", "k_bucket", "k_radix_scan[depth,0]",
        "k_radix_scatter[depth,0]", "k_radix_hist[depth,1]", "k_radix_scan[depth,1]", "k_radix_scatter[depth,1]", "k_bin_count",
        "k_bin_scan", "k_bin_place", "k_blend",
    ],
    "graph_kernel_launches": 13,
    # stereo gs_frame of a 150 K-splat SH1 bonsai scene (test_stereo_gpu's) at each eye size: 16-px tiles, 32-px tiles binned by
    # counting sort, radix binning
    "stereo_frame[810x600]": [
        "k_depth", "k_bucket", "k_radix_scan[depth,0]", "k_radix_scatter[depth,0]", "k_radix_hist[depth,1]", "k_radix_scan[depth,1]",
        "k_radix_scatter[depth,1]", "k_raster_init", "k_project", "k_bin_count", "k_bin_scan", "k_bin_place", "k_bin_count", "k_bin_scan",
        "k_bin_place", "k_stereo_join", "k_blend",
    ],
    "stereo_frame[2600x1500]": [
        "k_depth", "k_bucket", "k_radix_scan[depth,0]", "k_radix_scatter[depth,0]", "k_radix_hist[depth,1]", "k_radix_scan[depth,1]",
        "k_radix_scatter[depth,1]", "k_raster_init", "k_project", "k_bin_count", "k_bin_scan", "k_bin_place", "k_bin_count", "k_bin_scan",
        "k_bin_place", "k_stereo_join", "k_blend",
    ],
    "stereo_frame[4100x2100]": [
        "k_depth", "k_bucket", "k_radix_scan[depth,0]", "k_radix_scatter[depth,0]", "k_radix_hist[depth,1]", "k_radix_scan[depth,1]",
        "k_radix_scatter[depth,1]", "k_raster_init", "k_project", "k_tile_count", "k_tile_emit", "k_radix_hist[tile,0]",
        "k_radix_scan[tile,0]", "k_radix_scatter[tile,0]", "k_radix_hist[tile,1]", "k_radix_scan[tile,1]", "k_radix_scatter[tile,1]",
        "k_tile_count", "k_tile_emit", "k_radix_hist[tile,0]", "k_radix_scan[tile,0]", "k_radix_scatter[tile,0]", "k_radix_hist[tile,1]",
        "k_radix_scan[tile,1]", "k_radix_scatter[tile,1]", "k_stereo_join", "k_blend",
    ],
    "stereo_graph_kernel_launches[810x600]": 17,
    "stereo_graph_kernel_launches[2600x1500]": 17,
    "stereo_graph_kernel_launches[4100x2100]": 27,
    # a 20 K-splat garden scene as a .ply, uploaded in file order and through the generator, then its SplatTree built, gathered and
    # raycast (_upload_tree_ray_record)
    "upload_file": ["h2d_file_chunk", "k_ply_to_level0", "k_ksplat_decode"],
    "upload_file_optimized": ["h2d_file_chunk", "k_ply_to_level0", "gen_partition", "gen_sh_range", "gen_alpha", "gen_bucket_sort", "gen_buckets", "gen_write",
                              "k_ksplat_decode"],
    "build_splat_tree_kernel_launches": 105,
    "gather_for_sort_kernel_launches": 3,
    "raycast_kernel_launches": 40,
    # a sharded sort of the 150 K-splat scene over a two-engine group on one device (_sharded_sort_record)
    "sort_sharded[rank0]": [
        "k_depth", "k_shard_exchange_minmax", "k_bucket", "k_radix_scan[shard,0]", "k_radix_scatter[shard,0]", "k_radix_hist[shard,1]",
        "k_radix_scan[shard,1]", "k_radix_scatter[shard,1]", "k_shard_exchange_runs", "k_shard_offsets", "k_shard_place", "k_shard_done",
    ],
    "sort_sharded_kernel_launches[rank0]": 14,
    "sort_sharded[rank1]": [
        "k_depth", "k_shard_exchange_minmax", "k_bucket", "k_radix_scan[shard,0]", "k_radix_scatter[shard,0]", "k_radix_hist[shard,1]",
        "k_radix_scan[shard,1]", "k_radix_scatter[shard,1]", "k_shard_exchange_runs", "k_shard_offsets", "k_shard_place", "k_shard_done",
    ],
    "sort_sharded_kernel_launches[rank1]": 14,
}


def _viewer(w, h, **opts):
    from gaussiansplats3d_b200.scenes import CAMERAS, synthetic_scene
    from gaussiansplats3d_b200.viewer import Viewer
    c = CAMERAS["bonsai"]
    v = Viewer(dict(cameraUp=c["up"], initialCameraPosition=c["position"], initialCameraLookAt=c["look_at"], width=w, height=h,
                    sphericalHarmonicsDegree=1, **opts))
    v.addSplatScene(synthetic_scene(N_SPLATS, seed=8, kind="bonsai", sh_degree=1))
    return v


def _cameras(v, count):
    """(mvp, uniforms) of a camera moving away from the bonsai view"""
    cams = []
    for k in range(count):
        v.camera.position = np.asarray(v.initialCameraPosition) + np.array([0.15 * k, -0.05 * k, 0.1 * k])
        v.camera.look_at(v.initialCameraLookAt)
        v.camera.update(); v.updateSplatMesh()
        cams.append((v.mvp_matrix().astype(np.float32), v.uniforms()))
    return cams


def _stats(e):
    t = e.timings()
    return t["tile_instances"], t["visible_splats"]


def _frame_paths(e, cams, w, h, fmt):
    """{path: [(frame, sorted indexes or None, (tile_instances, visible_splats)) per camera]}"""
    from gaussiansplats3d_b200 import _native as N
    n = N_SPLATS
    shape, dt = (h, w, 4), (np.uint8 if fmt == N.GS_FRAME_RGBA8 else np.float32)
    out = {}

    def blocking(graph, profiling):
        e.set_graph_enabled(graph)
        e.set_profiling(profiling)
        res = []
        for mvp, u in cams:
            frame, order = np.empty(shape, dt), np.empty(n, np.uint32)
            e.frame_prepared(e.prepare_frame(mvp, u, w, h, n, frame_format=fmt), frame, order)
            res.append((frame, order, _stats(e)))
        e.set_graph_enabled(True)
        e.set_profiling(False)
        return res

    out["graph"] = blocking(True, False)
    out["no_graph"] = blocking(False, False)
    out["profiled"] = blocking(True, True)
    res = []
    for mvp, u in cams:
        e.frame_async(mvp, u, w, h, n, frame_format=fmt)
        e.synchronize()
        frame = e.read_buffer(N.GS_BUF_FRAME, dt, h * w * 4).reshape(shape)
        res.append((frame, e.read_buffer(N.GS_BUF_SORTED_INDEXES, np.uint32, n), _stats(e)))
    out["async"] = res
    for depth in (2, 3):
        bufs = [N.pinned_empty(shape, dt) for _ in range(depth)]
        res = []
        for i in range(len(cams) + depth - 1):
            if i < len(cams):
                mvp, u = cams[i]
                e.frame_begin(e.prepare_frame(mvp, u, w, h, n, frame_format=fmt), bufs[i % depth])
            if i >= depth - 1:
                e.frame_end()
                res.append((bufs[(i - depth + 1) % depth].copy(), None, _stats(e)))
        out[f"pipelined{depth}"] = res
    res = []
    for mvp, u in cams:
        order, _ = e.sort(mvp, n, n)
        frame = e.render(u, w, h, n, frame_format=fmt, flip_y=True)
        res.append((frame, order, _stats(e)))
    out["sort_render"] = res
    return out


@pytest.mark.parametrize("w,h,fmt", [(640, 360, "rgba8"), (1920, 1080, "rgba32f")], ids=["640x360-rgba8", "1920x1080-rgba32f"])
def test_every_frame_path_gives_the_same_frame(gs, w, h, fmt):
    from gaussiansplats3d_b200 import _native as N
    v = _viewer(w, h)
    cams = _cameras(v, 4)
    paths = _frame_paths(v.engine, cams, w, h, N.GS_FRAME_RGBA8 if fmt == "rgba8" else N.GS_FRAME_RGBA32F)
    want = paths.pop("graph")
    assert not np.array_equal(want[0][0], want[-1][0]), "the camera should move"
    assert all(s[0] > 0 and s[1] > 0 for _, _, s in want)
    for name, got in paths.items():
        assert len(got) == len(want), name
        for k, ((f, o, s), (wf, wo, ws)) in enumerate(zip(got, want)):
            assert f.dtype == wf.dtype and f.tobytes() == wf.tobytes(), f"{name}: frame {k} differs from the graph frame"
            assert o is None or np.array_equal(o, wo), f"{name}: sorted indexes {k} differ"
            assert s == ws, f"{name}: (tile_instances, visible_splats) {k}: {s} != {ws}"
    v.dispose()


def launch_record():
    """The kernel timelines of gs_sort, gs_render, an eager gs_frame, an eager subset frame (rank 0 of a two-engine group on one
    device) and an eager stereo gs_frame at each of test_stereo_gpu's EYE_SIZES, and the launch counts of a graph gs_frame and graph stereo
    gs_frames."""
    from gaussiansplats3d_b200 import _native as N
    w, h, n = 640, 360, N_SPLATS
    rec = {}
    v = _viewer(w, h)
    e = v.engine
    (mvp, u), = _cameras(v, 1)
    e.frame(mvp, u, w, h, n)
    rec["graph_kernel_launches"] = e.timings()["kernel_launches"]
    e.set_profiling(True)
    e.sort(mvp, n, n)
    rec["sort"] = [k for k, _ in e.kernel_timings()]
    e.render(u, w, h, n, frame_format=N.GS_FRAME_RGBA8, flip_y=True)
    rec["render"] = [k for k, _ in e.kernel_timings()]
    e.frame(mvp, u, w, h, n)
    rec["frame"] = [k for k, _ in e.kernel_timings()]
    v.dispose()
    old = os.environ.get("GS_SUBSET_MIN")
    os.environ["GS_SUBSET_MIN"] = "1"
    try:
        v = _viewer(w, h, rank=0, world_size=2)
        e = v.engine
        (mvp, u), = _cameras(v, 1)
        e.set_profiling(True)
        e.frame(mvp, u, w, h, n)
        rec["subset_frame"] = [k for k, _ in e.kernel_timings()]
        v.dispose()
    finally:
        if old is None:
            del os.environ["GS_SUBSET_MIN"]
        else:
            os.environ["GS_SUBSET_MIN"] = old
    from test_stereo_gpu import EYE_SIZES, _engine, _eyes, _order, _rig, _scene, _shared
    _, packed = _scene(n)
    for eye_w, h in EYE_SIZES:
        viewer, cams = _rig(eye_w, h)
        u, eyes = _shared(viewer, eye_w, h), _eyes(cams)
        with _engine(n, 2 * eye_w, h, packed) as e:
            _, mvp = _order(e, viewer, n)
            e.frame(mvp, u, 2 * eye_w, h, n, eyes=eyes)
            rec[f"stereo_graph_kernel_launches[{eye_w}x{h}]"] = e.timings()["kernel_launches"]
            e.set_profiling(True)
            e.frame(mvp, u, 2 * eye_w, h, n, eyes=eyes)
            rec[f"stereo_frame[{eye_w}x{h}]"] = [k for k, _ in e.kernel_timings()]
    rec.update(_upload_tree_ray_record())
    rec.update(_sharded_sort_record())
    return rec


def _upload_tree_ray_record():
    """The timelines of a .ply gs_upload_file and gs_upload_file_optimized, and the launch counts of gs_build_splat_tree, gs_gather_for_sort
    and a gs_raycast whose hits are sorted."""
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.engine import Engine
    from gaussiansplats3d_b200.scenes import synthetic_scene
    from oracle import file_oracle as FO
    from test_raycast_gpu import _ply_columns
    raw = synthetic_scene(20_000, seed=3, kind="garden")
    data = FO.write_ply(*_ply_columns(raw), raw.count)
    rec = {}
    with Engine(raw.count, max_width=64, max_height=64, ray_records=True) as e:
        e.set_profiling(True)
        e.upload_file(N.GS_FILE_PLY, data, sh_degree=0)
        rec["upload_file"] = [k for k, _ in e.kernel_timings()]
        e.upload_file_optimized(N.GS_FILE_PLY, data, sh_degree=0, compression_level=1)
        rec["upload_file_optimized"] = [k for k, _ in e.kernel_timings()]
        e.set_profiling(False)
        e.build_splat_tree()
        rec["build_splat_tree_kernel_launches"] = e.timings()["kernel_launches"]
        e.gather_for_sort(np.eye(4), 0.9, 0.95, gather_all=True)
        rec["gather_for_sort_kernel_launches"] = e.timings()["kernel_launches"]
        c = raw.centers.mean(axis=0)
        _, hits = e.raycast([c[0], c[1], c[2] + 20.0], [0.0, 0.0, -1.0], capacity=16)
        assert hits > 1, "the ray should hit several splats, so that their order is sorted"
        rec["raycast_kernel_launches"] = e.timings()["kernel_launches"]
    return rec


def _sharded_sort_record():
    """The timeline and launch count of each rank of a sharded sort over a two-engine group on one device."""
    from gaussiansplats3d_b200.engine import Engine
    from gaussiansplats3d_b200.scenes import integer_centers, synthetic_scene
    v = _viewer(640, 360)
    (mvp, _), = _cameras(v, 1)
    v.dispose()
    centers = integer_centers(synthetic_scene(N_SPLATS, seed=8, kind="bonsai").centers)
    old = os.environ.get("GS_SHARD_MIN")
    os.environ["GS_SHARD_MIN"] = "0"
    engines = [Engine(N_SPLATS, rank=g, world_size=2) for g in range(2)]
    rec = {}
    try:
        for e in engines:
            e.upload_centers(centers)
            e.shard_attach_local(engines)
            e.set_profiling(True)
        for e in engines:
            e.sort_sharded_async(mvp, N_SPLATS, N_SPLATS)
        engines[1].sort_sharded_finish(None)
        engines[0].sort_sharded_finish(np.empty(N_SPLATS, np.uint32))
        for g, e in enumerate(engines):
            rec[f"sort_sharded[rank{g}]"] = [k for k, _ in e.kernel_timings()]
            rec[f"sort_sharded_kernel_launches[rank{g}]"] = e.timings()["kernel_launches"]
    finally:
        for e in engines:
            e.close()
        if old is None:
            del os.environ["GS_SHARD_MIN"]
        else:
            os.environ["GS_SHARD_MIN"] = old
    return rec


def test_launch_and_upload_sequences_are_pinned(gs):
    got = launch_record()
    assert "k_subset_count" in got["subset_frame"] and "k_depth" in got["frame"]
    for key, want in LAUNCHES.items():
        assert got[key] == want, f"{key}: {got[key]} != {want}"


def test_bucket_range_wins_over_overflow_on_every_frame_entry(gs, monkeypatch):
    """A frame whose sorter centres span more than the int32 range map AND whose splats overflow the instance list reports
    GS_ERR_BUCKET_RANGE from gs_frame, gs_frame_async -> gs_synchronize and gs_frame_end; each entry's next good frame then equals a
    fresh engine's."""
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.scenes import integer_centers
    from test_raster_edges_gpu import _camera, _cloud
    from test_sorter_centers_gpu import _irow, _span
    monkeypatch.setenv("GS_INSTANCE_FACTOR", "0.05")
    w, h = 1920, 1080
    cc, cov, centers = _cloud(300_000, seed=902)
    n, fit = centers.shape[0], 2000
    u, _, mvp = _camera(w, h, (0.0, 0.0, 12.0), (0.0, 0.0, 0.0))
    good = integer_centers(centers)
    row = _irow(mvp)
    k = int(np.argmax(np.abs(row)))
    wide = good.copy()
    wide[[3, 4], :3] = 0
    wide[3, k] = int(0.6 * 2**31 / abs(row[k]))
    wide[4, k] = -wide[3, k]
    assert _span(wide, row) > 2**31 and _span(good, row) < 2**31

    def engine():
        e = gs.Engine(n, max_width=w, max_height=h)
        e.upload_splat_data(cc, cov)
        e.upload_centers(good)
        return e
    with engine() as f:
        with pytest.raises(N.GsError) as ei:
            f.frame(mvp, u, w, h, n)
        assert ei.value.code == N.GS_ERR_CAPACITY, "the full scene must overflow the instance list"
        fresh = f.frame(mvp, u, w, h, fit).copy()
    buf = N.pinned_empty((h, w, 4), np.uint8)
    e = engine()
    for path in ("frame", "frame_async", "frame_end"):
        e.upload_centers(wide)
        with pytest.raises(N.GsError) as ei:
            if path == "frame":
                e.frame(mvp, u, w, h, n)
            elif path == "frame_async":
                e.frame_async(mvp, u, w, h, n)
                e.synchronize()
            else:
                e.frame_begin(e.prepare_frame(mvp, u, w, h, n), buf)
                e.frame_end()
        assert ei.value.code == N.GS_ERR_BUCKET_RANGE, (path, str(ei.value))
        e.upload_centers(good)
        if path == "frame":
            got = e.frame(mvp, u, w, h, fit)
        elif path == "frame_async":
            e.frame_async(mvp, u, w, h, fit)
            e.synchronize()
            got = e.read_buffer(N.GS_BUF_FRAME, np.uint8, h * w * 4).reshape(h, w, 4)
        else:
            e.frame_begin(e.prepare_frame(mvp, u, w, h, fit), buf)
            e.frame_end()
            got = buf
        assert np.array_equal(got, fresh), f"{path}: the next good frame differs from a fresh engine's"
    e.close()
