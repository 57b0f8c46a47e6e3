"""GPU: the fused tile gather (gs_peer_attach_local) on one device: N engines with rank r of N, ranks > 0 blending their coarse tiles
straight into rank 0's frame allocation, the handshake kernels (k_peer_release, k_peer_wait_release, k_peer_signal,
k_peer_wait_arrived) running inside the captured frame graphs.

Rank 0's picture must be bit-identical to the single-engine frame of the same scene, camera, format and flip_y, in RGBA8 and RGBA32F,
at 16-px tiles with the counting sort's compacted placement (801x455), 32-px tiles (2600x1500), the radix binning (4097x2049), a
coarse diagonal past 128 (16512x64), at worlds 2 and 3; under the replicated sort and the per-rank subset sort; through
rank 0's graph frame (replayed, and with a moving camera), its eager frame, gs_frame_async and pipelined frames (two and three
in flight, over both halves of the double allocation and over one buffer).  The single-engine frames come from test_sharded_frames_gpu's scenes and are held to the f64 restatements there (tests/frame_f64.py) once per module.

Host order: every frame is enqueued on the peers before rank 0's frame, and nothing is waited for in between, so no host call
waits for a spinning handshake whose partner has not been enqueued yet.  Each group frame must finish well inside the handshake's
~2 s spin bound (FRAME_LIMIT_S), so a stall near that bound fails loudly.

Streams and hardware work queues: the device feeds streams through CUDA_DEVICE_MAX_CONNECTIONS queues (8 by default) and streams
beyond that share queues, where a peer's spinning wait can sit in front of rank 0's release.  A group holds two streams per engine
and rank 0's two pipelining streams, so gs_peer_attach_local takes at most 3 engines with the default 8 queues: the pipelined
world-3 cases use exactly 8, and an engine that gains a stream makes them refuse (or time out, if the count goes wrong).  Larger
groups are refused: world 8 with CUDA_DEVICE_MAX_CONNECTIONS=32 rendered its first frames, then timed out on the first frame after
a format change replaced the frame graphs, for a reason not yet found.  Ranks without tiles: 128x64 at worlds 2 and 3 (one coarse
tile, so every rank but 0 owns none).

Not covered here: NVLink, CUDA IPC mappings and ordering across devices (system scope); those rest on test_multi_gpu's two-GPU
tests and bench.py --gpus N."""
import time

import numpy as np
import pytest

from test_sharded_frames_gpu import PATH_SHAPES, SHAPES, SUBSET_MIN, Singles, _camera, _owner_map, _shape_id

pytestmark = pytest.mark.gpu

GATHER_SHAPES = [s for s in SHAPES if (s[0], s[1]) in {(801, 455), (2600, 1500), (4097, 2049), (16512, 64)}]
PIPE_SHAPE = GATHER_SHAPES[0]     # 801x455
TINY_SHAPE = (128, 64, 16, 1, 0, False)   # one coarse tile (diagonal 0): at worlds 2 and 3 every rank but 0 owns no tile
PIPE_CAMERAS = 7
CAMERAS = 3
FRAME_LIMIT_S = 1.0                # per group frame, against the ~2 s spin bound of kPeerTimeoutCycles


@pytest.fixture(scope="module")
def singles():
    return Singles()


def _fmt_name(fmt):
    from gaussiansplats3d_b200 import _native as N
    return "RGBA8" if fmt == N.GS_FRAME_RGBA8 else "RGBA32F"


def _want(singles, shape, k, fmt):
    from gaussiansplats3d_b200 import _native as N
    got32, got8, inst = singles.get(shape, "default", k)
    return (got8 if fmt == N.GS_FRAME_RGBA8 else got32), inst


class Group:
    """`world` engines of one scene on one device, ranks 1.. attached to rank 0's frame.  Closes peers first, then rank 0."""

    def __init__(self, c, world, engines=None):
        self.c, self.world = c, world
        self.engines = []
        if engines is not None:      # already attached
            self.engines = list(engines)
            return
        try:
            for r in range(world):
                self.engines.append(c.engine(r, world))
            for e in self.engines[1:]:
                e.peer_attach_local(self.engines[0])
        except BaseException:
            self.close()
            raise

    @property
    def root(self):
        return self.engines[0]

    @property
    def peers(self):
        return self.engines[1:]

    def close(self):
        for e in reversed(self.engines):
            e.close()
        self.engines = []

    def prepare(self, k, fmt):
        c = self.c
        u, mvp = _camera(c.w, c.h, k)
        return [e.prepare_frame(mvp, u, c.w, c.h, c.count, frame_format=fmt, flip_y=c.flip_y) for e in self.engines]

    def set_graph(self, on):
        for e in self.engines:
            e.set_graph_enabled(on)

    def enqueue_peers(self, preps):
        for e, p in zip(self.peers, preps[1:]):
            e.frame_async(None, None, self.c.w, self.c.h, self.c.count, prepared=p)

    def frame(self, k, fmt, mode="frame", label=""):
        """One group frame: the peers' frames, then rank 0's (gs_frame, or gs_frame_async + gs_synchronize), then the peers' waits.
        Returns rank 0's picture and every rank's tile instances."""
        from gaussiansplats3d_b200 import _native as N
        c = self.c
        preps = self.prepare(k, fmt)
        shape, dt = _frame_shape(c, fmt)
        out = np.empty(shape, dt)
        t0 = time.perf_counter()
        try:
            self.enqueue_peers(preps)
            if mode == "frame":
                self.root.frame_prepared(preps[0], out)
            else:
                self.root.frame_async(None, None, c.w, c.h, c.count, prepared=preps[0])
                self.root.synchronize()
            for e in self.peers:
                e.synchronize()
        except N.GsError as ex:
            raise AssertionError(f"{label}: {ex}") from ex
        dt_s = time.perf_counter() - t0
        if mode == "async":
            out = self.root.read_buffer(N.GS_BUF_FRAME, dt, out.size).reshape(shape)
        assert dt_s < FRAME_LIMIT_S, f"{label}: the group frame took {dt_s:.3f} s"
        return out, [e.timings()["tile_instances"] for e in self.engines]


def _frame_shape(c, fmt):
    from gaussiansplats3d_b200 import _native as N
    return (c.h, c.w, 4), (np.uint8 if fmt == N.GS_FRAME_RGBA8 else np.float32)


def _check_picture(label, got, want):
    assert got.dtype == want.dtype and got.shape == want.shape, label
    if got.tobytes() != want.tobytes():
        bad = (got != want).any(-1)
        ys, xs = np.nonzero(bad)
        raise AssertionError(f"{label}: {int(bad.sum())} of {bad.size} pixels differ from the single-engine frame "
                             f"(first at x={xs[0]}, y={ys[0]}: {got[ys[0], xs[0]]} vs {want[ys[0], xs[0]]})")


def _check_group_frame(label, got, insts, want, want_inst, owner):
    _check_picture(label, got, want)
    assert sum(insts) == want_inst, f"{label}: tile instances per rank {insts} sum to {sum(insts)}, the single engine drew {want_inst}"
    for r, n in enumerate(insts):
        if not (owner == r).any():
            assert n == 0, f"{label}: rank {r} owns no tile but drew {n} instances"


_CASES = [(s, w) for s in GATHER_SHAPES + [TINY_SHAPE] for w in (2, 3)]


@pytest.mark.parametrize("strategy", list(SUBSET_MIN))
@pytest.mark.parametrize("shape,world", _CASES, ids=[f"{_shape_id(s)}-w{w}" for s, w in _CASES])
def test_gathered_frame_equals_single_engine_frame(gs, oracle_mod, singles, shape, world, strategy, monkeypatch):
    """Rank 0's picture, assembled by the peers' stores, is the single-engine frame bit for bit in RGBA32F and RGBA8: through rank 0's
    graph frame twice in a row (a replay), its eager frame, gs_frame_async + gs_synchronize, and on 801x455 and 4097x2049 three camera
    positions through the graph and eagerly; every rank's instances add up to the single engine's."""
    from gaussiansplats3d_b200 import _native as N
    monkeypatch.setenv("GS_SUBSET_MIN", SUBSET_MIN[strategy])
    c = singles.case(shape, "default")
    for fmt in (N.GS_FRAME_RGBA32F, N.GS_FRAME_RGBA8):
        _want(singles, shape, 0, fmt)
    if (c.w, c.h) in PATH_SHAPES:
        for k in range(CAMERAS):
            _want(singles, shape, k, N.GS_FRAME_RGBA32F)
    if (c.w, c.h) == (TINY_SHAPE[0], TINY_SHAPE[1]):
        assert not (_owner_map(c.w, c.h, world, c.flip_y) > 0).any(), "only rank 0 should own a tile here"
    _gather_sequence(c, world, strategy, lambda k, fmt: _want(singles, shape, k, fmt))


def _gather_sequence(c, world, strategy, want):
    """One group of `world` engines: RGBA32F then RGBA8, each through rank 0's graph frame twice, its eager frame and gs_frame_async;
    on PATH_SHAPES three panned cameras through the graph and eagerly.  want(k, fmt) -> (single-engine frame, its tile instances)."""
    from gaussiansplats3d_b200 import _native as N
    owner = _owner_map(c.w, c.h, world, c.flip_y)
    g = Group(c, world)
    try:
        for fmt in (N.GS_FRAME_RGBA32F, N.GS_FRAME_RGBA8):
            want_frame, want_inst = want(0, fmt)
            steps = [(True, "frame"), (True, "frame"), (False, "frame"), (True, "async")]
            for i, (graph, mode) in enumerate(steps):
                g.set_graph(graph)
                label = f"{c.w}x{c.h} world {world} {strategy} {_fmt_name(fmt)} frame {i} ({'graph' if graph else 'eager'} {mode})"
                got, insts = g.frame(0, fmt, mode, label)
                _check_group_frame(label, got, insts, want_frame, want_inst, owner)
        if (c.w, c.h) in PATH_SHAPES:
            for graph in (True, False):
                g.set_graph(graph)
                for k in range(CAMERAS):
                    want_frame, want_inst = want(k, N.GS_FRAME_RGBA32F)
                    label = f"{c.w}x{c.h} world {world} {strategy} camera {k} ({'graph' if graph else 'eager'})"
                    got, insts = g.frame(k, N.GS_FRAME_RGBA32F, label=label)
                    _check_group_frame(label, got, insts, want_frame, want_inst, owner)
    finally:
        g.close()


@pytest.mark.parametrize("fmt_name", ["RGBA8", "RGBA32F"])
@pytest.mark.parametrize("inflight", [2, 3])
@pytest.mark.parametrize("halves", ["double", "single"])
@pytest.mark.parametrize("strategy", list(SUBSET_MIN))
def test_pipelined_gathered_frames(gs, oracle_mod, singles, strategy, halves, inflight, fmt_name, monkeypatch):
    """Rank 0 pipelines (gs_frame_begin / gs_frame_end, `inflight` frames in flight) over a camera moving through 7 positions, twice,
    with a blocking gs_frame after each pass, at world 3; the peers enqueue each frame (gs_frame_async) just before rank 0 does.  Every
    picture delivered is its own camera's single-engine frame, in order: with the double allocation (the halves alternate, and the
    second pass starts on half 1) and with one buffer (GS_PEER_DOUBLE=0).  The blocking frame goes back to half 0."""
    from gaussiansplats3d_b200 import _native as N
    monkeypatch.setenv("GS_SUBSET_MIN", SUBSET_MIN[strategy])
    if halves == "single":
        monkeypatch.setenv("GS_PEER_DOUBLE", "0")
    else:
        monkeypatch.delenv("GS_PEER_DOUBLE", raising=False)
    fmt = N.GS_FRAME_RGBA8 if fmt_name == "RGBA8" else N.GS_FRAME_RGBA32F
    shape, world = PIPE_SHAPE, 3
    c = singles.case(shape, "default")
    wants = [_want(singles, shape, k, fmt) for k in range(PIPE_CAMERAS)]
    assert wants[0][0].tobytes() != wants[-1][0].tobytes(), "the camera should move"
    owner = _owner_map(c.w, c.h, world, c.flip_y)
    g = Group(c, world)
    try:
        preps = [g.prepare(k, fmt) for k in range(PIPE_CAMERAS)]
        shp, dt = _frame_shape(c, fmt)
        bufs = [N.pinned_empty(shp, dt) for _ in range(inflight)]     # page-locked allocations before any frame is in flight
        for rep in range(2):
            def begin(i):
                g.enqueue_peers(preps[i])
                g.root.frame_begin(preps[i][0], bufs[i % inflight])
            t0 = time.perf_counter()
            for i in range(inflight - 1):
                begin(i)
            for i in range(PIPE_CAMERAS):
                if i + inflight - 1 < PIPE_CAMERAS:
                    begin(i + inflight - 1)
                g.root.frame_end()
                t1 = time.perf_counter()
                assert t1 - t0 < FRAME_LIMIT_S, f"pipelined frame {i} took {t1 - t0:.3f} s"
                t0 = t1
                _check_picture(f"{halves} {inflight} in flight {fmt_name} {strategy} pass {rep} frame {i}", bufs[i % inflight], wants[i][0])
            for e in g.peers:
                e.synchronize()
            # a blocking frame after the pipelined ones: half 0 again, whatever half the last pipelined frame used
            label = f"{halves} {inflight} in flight {fmt_name} {strategy} pass {rep}: blocking frame"
            got, insts = g.frame(PIPE_CAMERAS - 1, fmt, label=label)
            _check_group_frame(label, got, insts, *wants[-1], owner)
    finally:
        g.close()


def test_peer_attach_local_refusals(gs, oracle_mod, singles, monkeypatch):
    """gs_peer_attach_local refuses, before any frame: rank 0 as the peer, a root that is not rank 0, another world_size, a group of
    more engines than the device's default hardware work queues can serve (world 4: 10 streams, 8 queues) and one of more than 3
    engines whatever the queue count (world 8 with 32 queues), engines
    without a framebuffer, another frame size, frames in flight on either engine, and a second attach.  (A root on another device
    needs a second GPU.)  Afterwards the same engines attach and render the single-engine frame."""
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.engine import Engine
    c = singles.case(PIPE_SHAPE, "default")
    want, want_inst = _want(singles, PIPE_SHAPE, 0, N.GS_FRAME_RGBA8)
    made = []

    def engine(rank, world, **kw):
        e = c.engine(rank, world) if not kw else Engine(c.n, rank=rank, world_size=world, **kw)
        made.append(e)
        return e

    def refused(e, root, what):
        with pytest.raises(N.GsError) as ex:
            if root is None:
                N.check(e._lib.gs_peer_attach_local(e._h, None), "gs_peer_attach_local")
            else:
                e.peer_attach_local(root)
        assert ex.value.code == N.GS_ERR_BAD_ARG, f"{what}: {ex.value}"

    try:
        root, peer = engine(0, 2), engine(1, 2)
        refused(peer, None, "null root")
        refused(root, root, "rank 0 as the peer")
        refused(peer, engine(1, 2), "a root of rank 1")
        refused(engine(1, 3), root, "world 3 against world 2")
        monkeypatch.delenv("CUDA_DEVICE_MAX_CONNECTIONS", raising=False)
        refused(engine(1, 4), engine(0, 4), "world 4 with the default 8 hardware work queues")
        monkeypatch.setenv("CUDA_DEVICE_MAX_CONNECTIONS", "32")
        refused(engine(1, 8), engine(0, 8), "world 8 with 32 hardware work queues")
        monkeypatch.delenv("CUDA_DEVICE_MAX_CONNECTIONS")
        refused(engine(1, 2, max_width=0, max_height=0), engine(0, 2, max_width=0, max_height=0), "no framebuffer")
        refused(engine(1, 2, max_width=c.w + 1, max_height=c.h), root, "another frame size")
        u, mvp = _camera(c.w, c.h, 0)
        root.frame_async(mvp, u, c.w, c.h, c.count, frame_format=N.GS_FRAME_RGBA8, flip_y=c.flip_y)
        refused(peer, root, "an asynchronous frame pending on the root")
        root.synchronize()
        peer.frame_async(mvp, u, c.w, c.h, c.count, frame_format=N.GS_FRAME_RGBA8, flip_y=c.flip_y)
        refused(peer, root, "an asynchronous frame pending on the peer")
        peer.synchronize()
        out = N.pinned_empty(want.shape, want.dtype)
        root.frame_begin(root.prepare_frame(mvp, u, c.w, c.h, c.count, frame_format=N.GS_FRAME_RGBA8, flip_y=c.flip_y), out)
        refused(peer, root, "a pipelined frame in flight on the root")
        root.frame_end()
        peer.peer_attach_local(root)
        refused(peer, root, "a second attach")
        got, insts = Group(c, 2, engines=[root, peer]).frame(0, N.GS_FRAME_RGBA8, label="after the refusals")
        _check_group_frame("after the refusals", got, insts, want, want_inst, _owner_map(c.w, c.h, 2, c.flip_y))
    finally:
        for e in reversed(made):
            e.close()


def test_teardown_and_a_fresh_group(gs, oracle_mod, singles):
    """A group renders, its peers and then its root are destroyed, and a fresh group of new engines attaches and renders the same
    single-engine frame; twice, so the second group's teardown is checked by a third."""
    from gaussiansplats3d_b200 import _native as N
    c = singles.case(PIPE_SHAPE, "default")
    want, want_inst = _want(singles, PIPE_SHAPE, 0, N.GS_FRAME_RGBA8)
    owner = _owner_map(c.w, c.h, 3, c.flip_y)
    for generation in range(3):
        g = Group(c, 3)
        try:
            for i in range(2):
                got, insts = g.frame(0, N.GS_FRAME_RGBA8, label=f"group {generation} frame {i}")
                _check_group_frame(f"group {generation} frame {i}", got, insts, want, want_inst, owner)
        finally:
            g.close()
