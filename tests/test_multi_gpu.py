"""Coarse-tile sharding of the rasteriser: rank r renders the 128x64-px tiles with (cx + cy) % N == r into a full-size frame that is
zero elsewhere; the ranks' frames must SUM to exactly the single-engine frame.  GPU part: N engines on one device (no NCCL needed to
check the arithmetic); CPU part: the reduction plumbing over torch.distributed/gloo with world_size 2 and the ownership map."""
import os
import socket
import sys

import numpy as np
import pytest

import cases


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _gloo_worker(rank, world, port, height, width, q):
    import torch
    import torch.distributed as dist
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from gaussiansplats3d_b200.parallel import ownership_map
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    # the "frame": pixel value encodes its row and column, so any misplacement is visible
    full = np.zeros((height, width, 4), np.int32)
    full[..., 0] = np.arange(height)[:, None] % 251
    full[..., 1] = np.arange(width)[None, :] % 251
    full[..., 3] = 255
    mine = ownership_map(width, height, world) == rank
    part = np.where(mine[..., None], full, 0)
    t = torch.from_numpy(part.copy())
    dist.all_reduce(t, op=dist.ReduceOp.SUM)                            # the final tile gather (NCCL on the GPUs)
    q.put((rank, bool(np.array_equal(t.numpy(), full))))
    dist.destroy_process_group()


@pytest.mark.parametrize("height", [1080, 270, 33])
def test_all_reduce_assembles_frame_gloo_world2(height):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, height, 300, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, True), (1, True)]


def test_ownership_map_is_a_partition():
    from gaussiansplats3d_b200.parallel import COARSE_H, COARSE_W, owner_of_coarse, ownership_map
    for world in (1, 2, 3, 4, 8):
        m = ownership_map(1920, 1080, world)
        assert m.min() == 0 and m.max() == world - 1
        assert m[0, 0] == owner_of_coarse(0, 0, world) and m[1079, 1919] == owner_of_coarse(1919 // COARSE_W, 1079 // COARSE_H, world)
        share = np.bincount(m.ravel(), minlength=world) / m.size
        assert share.max() - share.min() < 0.08, "diagonal interleave should balance the screen area"


@pytest.mark.gpu
@pytest.mark.parametrize("subset_sort", [False, True])
@pytest.mark.parametrize("world", [2, 3, 8])
def test_sharded_frames_sum_to_single_engine_frame(gs, world, subset_sort, monkeypatch):
    # both sort strategies of a sharded frame: replicated full sort (small scenes) and per-rank subset sort (default from 3M splats)
    monkeypatch.setenv("GS_SUBSET_MIN", "1" if subset_sort else "4000000000")
    from gaussiansplats3d_b200.parallel import combine_frames, ownership_map
    from gaussiansplats3d_b200.scenes import CAMERAS, synthetic_scene
    from gaussiansplats3d_b200.viewer import Viewer
    n, w, h = 120_000, 801, 455
    raw = synthetic_scene(n, seed=8, kind="bonsai", sh_degree=1)
    c = CAMERAS["bonsai"]
    opts = dict(cameraUp=c["up"], initialCameraPosition=c["position"], initialCameraLookAt=c["look_at"], width=w, height=h, sphericalHarmonicsDegree=1)
    v1 = Viewer(opts)
    v1.addSplatScene(raw)
    want = v1.frame(frame_format=gs._native.GS_FRAME_RGBA8, flip_y=False)
    v1.dispose()
    own = ownership_map(w, h, world)
    frames = []
    for r in range(world):
        v = Viewer(dict(opts, rank=r, world_size=world))
        v.addSplatScene(raw)
        f = v.frame(frame_format=gs._native.GS_FRAME_RGBA8, flip_y=False).copy()
        assert not f[own != r].any(), "a rank wrote pixels outside its own coarse tiles"
        frames.append(f)
        v.dispose()
    got = combine_frames(frames)
    assert np.array_equal(got, want), "sharded frames do not sum to the single-GPU frame bit for bit"


def _peer_worker(rank, world, port, q):
    """One process per GPU: rank 0 exports its frame through CUDA IPC, the others blend into it (fused tile gather)."""
    import torch
    import torch.distributed as dist
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import gaussiansplats3d_b200 as gs
    from gaussiansplats3d_b200.parallel import PeerGather
    from gaussiansplats3d_b200.scenes import CAMERAS, synthetic_scene
    from gaussiansplats3d_b200.viewer import Viewer
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    n, w, h = 100_000, 801, 455
    raw = synthetic_scene(n, seed=8, kind="bonsai", sh_degree=0)
    c = CAMERAS["bonsai"]
    opts = dict(cameraUp=c["up"], initialCameraPosition=c["position"], initialCameraLookAt=c["look_at"], width=w, height=h, device=rank)
    want = None
    if rank == 0:
        v1 = Viewer(opts)
        v1.addSplatScene(raw)
        want = v1.frame(frame_format=gs._native.GS_FRAME_RGBA8, flip_y=True).copy()
        v1.dispose()
    v = Viewer(dict(opts, rank=rank, world_size=world))
    v.addSplatScene(raw)
    PeerGather(v.engine, rank, world)
    ok = True
    for it in range(3):     # several frames: the release/arrive handshake must hold across frames (graph replay included)
        got = v.frame(frame_format=gs._native.GS_FRAME_RGBA8, flip_y=True)
        if rank == 0:
            ok = ok and bool(np.array_equal(got, want))
    dist.barrier()
    # Pipelined frames on rank 0 (gs_frame_begin / gs_frame_end, three in flight): rank 0's exported allocation holds TWO frames and the
    # half a frame uses travels in the release word, so the peers store frame f+1 while frame f's picture crosses PCIe.  A moving camera:
    # every delivered picture must be that frame's single-GPU picture, in order.
    from gaussiansplats3d_b200 import _native as N
    e = v.engine
    cams, wants = [], []
    for k in range(7):
        v.camera.position = np.asarray(v.initialCameraPosition) + np.array([0.12 * k, -0.04 * k, 0.08 * k])
        v.camera.look_at(v.initialCameraLookAt)
        v.camera.update(); v.updateSplatMesh()
        cams.append(e.prepare_frame(v.mvp_matrix().astype(np.float32), v.uniforms(), w, h, n, frame_format=N.GS_FRAME_RGBA8, flip_y=True))
    if rank == 0:
        v1 = Viewer(opts)
        v1.addSplatScene(raw)
        for k in range(7):
            v1.camera.position = np.asarray(v1.initialCameraPosition) + np.array([0.12 * k, -0.04 * k, 0.08 * k])
            v1.camera.look_at(v1.initialCameraLookAt)
            v1.camera.update(); v1.updateSplatMesh()
            out = N.pinned_empty((h, w, 4), np.uint8)
            v1.engine.frame_prepared(v1.engine.prepare_frame(v1.mvp_matrix().astype(np.float32), v1.uniforms(), w, h, n, frame_format=N.GS_FRAME_RGBA8, flip_y=True), out)
            wants.append(out.copy())
        v1.dispose()
        assert not np.array_equal(wants[0], wants[-1])
    dist.barrier()
    for rep in range(2):
        if rank == 0:
            bufs = [N.pinned_empty((h, w, 4), np.uint8) for _ in range(3)]
            e.frame_begin(cams[0], bufs[0]); e.frame_begin(cams[1], bufs[1])
            for i in range(7):
                if i + 2 < 7:
                    e.frame_begin(cams[i + 2], bufs[(i + 2) % 3])
                e.frame_end()
                ok = ok and bool(np.array_equal(bufs[i % 3], wants[i]))
        else:
            for i in range(7):
                e.frame_async(None, None, w, h, n, prepared=cams[i])
            e.synchronize()
        dist.barrier()
        # and a blocking frame afterwards (half 0 again, whatever half the last pipelined frame used)
        got = v.frame(frame_format=gs._native.GS_FRAME_RGBA8, flip_y=True)
        if rank == 0:
            ok = ok and bool(np.array_equal(got, wants[6]))
        dist.barrier()
    q.put((rank, ok))
    v.dispose()
    dist.destroy_process_group()


@pytest.mark.gpu
def test_fused_peer_gather_two_gpus(gs):
    """Needs 2 GPUs (skipped on a 1-GPU box): the picture assembled in rank 0's memory by peer stores equals the single-GPU frame."""
    if gs._native.load().gs_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_peer_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=240) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, True), (1, True)]


# ---- sort-only sharding by input position (gaussiansplats3d_b200/csrc/shard_kernels.cuh) ---------------------------------------------
def _np_int_static_distances(case, lo, hi):
    """Integer static branch (sorter.cpp:64-74) for positions [lo, hi): wrapping int32 dot with the truncated f64 row."""
    m = case["mvp"].astype(np.float32)
    row = np.array([int(np.float64(m[2]) * 1000.0), int(np.float64(m[6]) * 1000.0), int(np.float64(m[10]) * 1000.0)], np.int64)
    c = case["centers"][case["indexes"][lo:hi].astype(np.int64), :3].astype(np.int64)
    d = (c * row[None, :]).sum(axis=1)
    return ((d + 2**31) % 2**32 - 2**31).astype(np.int32)


def _np_buckets(d, dmin, dmax, R):
    """sorter.cpp:142-146 in f32."""
    span = np.float32(dmax) - np.float32(dmin)
    rm = np.float32(R - 1) / span
    rel = (d.astype(np.int64) - int(dmin)).astype(np.float32)
    return np.minimum((rel * rm).astype(np.int32), R - 1)


@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("kw", [dict(n=20000), dict(n=20000, ties=True), dict(n=5000, sort_frac=0.37, index_kind="octree"), dict(n=5, index_kind="identity")])
def test_sharded_merge_rule_equals_reference_order(world, kw):
    """Per-rank sorted slices + the run-offset rule == the reference's single sort, for any number of ranks (incl. empty slices)."""
    from oracle import pyoracle as O
    from cases import sort_case, call_args
    from gaussiansplats3d_b200.parallel import merge_sharded_order, shard_bounds
    case = sort_case(11, **kw)
    R = 1 << 16
    ref, buckets = O.port_sort_indexes(*call_args(case, R), want_buckets=True)
    rc, sc = case["render_count"], case["sort_count"]
    s0 = rc - sc
    per_rank = [(buckets[lo:hi], case["indexes"][lo:hi]) for lo, hi in shard_bounds(s0, sc, world)]
    got = merge_sharded_order(s0, R, per_rank)
    assert np.array_equal(got, ref[s0:rc])


def _gloo_shard_worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    sys.path.insert(0, os.path.join(root, "tests"))
    from cases import sort_case
    from gaussiansplats3d_b200.parallel import shard_bounds
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    case = sort_case(5, 30000, index_kind="shuffled")
    R, rc = 1 << 16, case["render_count"]
    lo, hi = shard_bounds(0, rc, world)[rank]
    d = _np_int_static_distances(case, lo, hi)
    # C1: global min/max (on the GPUs: 8-byte stores into every peer's block)
    mm = torch.tensor([int(d.min()), -int(d.max())], dtype=torch.int64)
    dist.all_reduce(mm, op=dist.ReduceOp.MIN)
    dmin, dmax = int(mm[0]), -int(mm[1])
    key = (R - 1) - _np_buckets(d, dmin, dmax, R)[::-1].astype(np.int64)
    order = np.argsort(key, kind="stable")
    keys_sorted, vals_sorted = key[order], case["indexes"][lo:hi][::-1][order]
    # C2: everybody's run lengths (on the GPUs: reads of the peers' run tables)
    counts = torch.from_numpy(np.bincount(key, minlength=R))
    allc = [torch.zeros_like(counts) for _ in range(world)]
    dist.all_gather(allc, counts)
    allc = np.stack([c.numpy() for c in allc])
    total = allc.sum(axis=0)
    base = np.concatenate([[0], np.cumsum(total)[:-1]]) + allc[rank + 1:].sum(axis=0) - np.concatenate([[0], np.cumsum(allc[rank])[:-1]])
    # place: my elements into rank 0's buffer (on the GPUs: peer stores); here a SUM of disjoint placements
    out = torch.zeros(rc, dtype=torch.int64)
    out[torch.from_numpy(np.arange(keys_sorted.size) + base[keys_sorted])] = torch.from_numpy(vals_sorted.astype(np.int64))
    dist.all_reduce(out, op=dist.ReduceOp.SUM)
    ok = None
    if rank == 0:
        from oracle import pyoracle as O
        from cases import call_args
        ok = bool(np.array_equal(out.numpy().astype(np.uint32), O.port_sort_indexes(*call_args(case, R))))
    q.put((rank, ok))
    dist.destroy_process_group()


def test_sharded_sort_protocol_gloo_world2():
    """The two exchanges of the sharded sort (min/max, run lengths) and the placement, over torch.distributed/gloo, vs the oracle."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gloo_shard_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=180) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res, key=lambda t: t[0]) == [(0, True), (1, None)]


SHARD_CASES = [
    ("int-static-shuffled", dict(seed=21, n=300_000, index_kind="shuffled")),
    ("int-static-identity", dict(seed=22, n=300_000, index_kind="identity")),
    ("int-partial-octree", dict(seed=23, n=200_000, index_kind="octree", sort_frac=0.37)),
    ("float-dynamic", dict(seed=24, n=120_000, integer=False, dynamic=True, index_kind="shuffled")),
    ("int-precomputed", dict(seed=25, n=120_000, precomputed=True, index_kind="shuffled")),
    ("ties", dict(seed=26, n=150_000, ties=True)),
    ("fewer-splats-than-ranks", dict(seed=27, n=2, index_kind="identity")),
    ("one-tile-plus-one", dict(seed=28, n=4097)),
] + [   # integer precomputed distances whose keys are chosen digit by digit (cases.radix_keys), three radix tiles and one key
    (f"keys-{kind}", dict(seed=50 + i, n=3 * 4096 + 1, keys=kind, index_kind="identity" if i % 2 else "shuffled"))
    for i, kind in enumerate(k for k in cases.KEY_KINDS if k != "random")
]
SHARD_RANGES = (1 << 8, 1 << 16, (1 << 17) + 1, 1 << 24)     # sort plans of one, two and three passes (u16 keys to 16 bits, else u32)


@pytest.mark.gpu
@pytest.mark.parametrize("R", SHARD_RANGES, ids=[f"R{R}" for R in SHARD_RANGES])
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("name,kw", SHARD_CASES)
def test_sharded_sort_engines_on_one_device(gs, oracle_mod, monkeypatch, world, name, kw, R):
    """N engines on one GPU, each sorting its slice of input positions and storing into engine 0's sortedIndexes: the assembled order
    must be bit-identical to the reference's single sort.  (The multi-process variant differs only in how the peers' memory is mapped.)
    Every case runs at ranges of one, two and three radix passes; the run table holds one entry per key (128 MiB per rank at 2^24)."""
    monkeypatch.setenv("GS_SHARD_MIN", "0")     # always split (the default splits only windows of >= 8 M splats)
    if "keys" in kw:
        c = cases.keyed_case(kw["seed"], kw["n"], R, kw["keys"], index_kind=kw["index_kind"])
    else:
        c = cases.sort_case(**kw)
    want = oracle_mod.port_sort_indexes(*cases.call_args(c, R))
    n, rc, sc = c["splat_count"], c["render_count"], c["sort_count"]
    engines = [gs.Engine(n, distance_map_range=R, integer_based_sort=c["integer_sort"], dynamic_mode=c["dynamic_mode"], rank=g, world_size=world) for g in range(world)]
    try:
        for e in engines:
            e.upload_centers(c["centers"], c["scene_indexes"])
        for e in engines:
            e.shard_attach_local(engines)
        idx = None if kw.get("index_kind") == "identity" else c["indexes"]
        for rep in range(3):   # repeated sorts: sequence numbers, run-table reset and the self-cleaning control block must hold
            for e in engines:
                e.sort_sharded_async(c["mvp"], sc, rc, idx, transforms=c["transforms"], precomputed=c["precomputed"])
            out = np.full(rc, 0xFFFFFFFF, np.uint32)
            for g in reversed(range(world)):
                engines[g].sort_sharded_finish(out if g == 0 else None)
            assert np.array_equal(out, want), f"{name} world={world} rep={rep}"
        # the same engines still do an ordinary (unsharded) sort afterwards
        got, _ = engines[1].sort(c["mvp"], sc, rc, idx, transforms=c["transforms"], precomputed=c["precomputed"])
        assert np.array_equal(got, want)
    finally:
        for e in engines:
            e.close()


@pytest.mark.gpu
def test_sharded_sort_below_threshold_is_sorted_by_rank0(gs, oracle_mod, monkeypatch):
    """Default threshold: a small window is not worth the exchange, so rank 0 sorts it alone and the other ranks' calls are no-ops."""
    import cases
    monkeypatch.delenv("GS_SHARD_MIN", raising=False)
    c = cases.sort_case(seed=41, n=100_000, index_kind="shuffled")
    R = 1 << 16
    want = oracle_mod.port_sort_indexes(*cases.call_args(c, R))
    engines = [gs.Engine(c["splat_count"], distance_map_range=R, rank=g, world_size=2) for g in range(2)]
    try:
        for e in engines:
            e.upload_centers(c["centers"])
            e.shard_attach_local(engines)
        for e in engines:
            e.sort_sharded_async(c["mvp"], c["sort_count"], c["render_count"], c["indexes"])
        _, ms1 = engines[1].sort_sharded_finish(None)
        out, ms0 = engines[0].sort_sharded_finish(np.empty(c["render_count"], np.uint32))
        assert np.array_equal(out, want) and ms1 == 0.0 and ms0 > 0.0
    finally:
        for e in engines:
            e.close()


def _shard_worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    sys.path.insert(0, os.path.join(root, "tests"))
    import cases
    import gaussiansplats3d_b200 as gs
    from gaussiansplats3d_b200.parallel import ShardedSort
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    os.environ["GS_SHARD_MIN"] = "0"            # always split
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    ok = True
    R = 1 << 16
    for kw in (dict(seed=31, n=1_000_000, index_kind="shuffled"), dict(seed=32, n=400_000, index_kind="identity"), dict(seed=33, n=250_000, index_kind="octree", sort_frac=0.5)):
        c = cases.sort_case(**kw)
        with gs.Engine(c["splat_count"], device=rank, distance_map_range=R, rank=rank, world_size=world) as e:
            e.upload_centers(c["centers"])
            ss = ShardedSort(e, rank, world)
            idx = None if kw["index_kind"] == "identity" else c["indexes"]
            for rep in range(3):
                got, _ = ss.sort(c["mvp"], c["sort_count"], c["render_count"], idx)
                if rank == 0:
                    single, _ = e.sort(c["mvp"], c["sort_count"], c["render_count"], idx)   # same engine, unsharded
                    ok = ok and bool(np.array_equal(got, single))
                dist.barrier()
    q.put((rank, ok))
    dist.destroy_process_group()


@pytest.mark.gpu
def test_sharded_sort_two_gpus(gs):
    """Needs 2 GPUs (skipped on a 1-GPU box): one process per GPU, peers mapped through CUDA IPC, result in rank 0's memory."""
    if gs._native.load().gs_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_shard_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, True), (1, True)]
