"""GPU: sharded frames (world_size > 1) on one device, N engines with rank r of N, at every fine-tile size, both binnings, the counting
sort's placement with and without its compaction, coarse diagonals cx + cy past 63 and past 127, ranks that own no tile, both sort
strategies (the replicated full sort and the per-rank subset sort, GS_SUBSET_MIN), the subset sort's key widths, float keys and index
lists, the graph and the eager frame, and graph replays whose subset count changes from frame to frame.

Each frame shape is rendered from one scene that covers it end to end (orthographic, 1 px per world unit: small splats everywhere and
a few that span most of the frame).  The single-engine frame of each scene, camera and sort option set is held to the f64 restatements
(tests/frame_f64.py: draw order, projection, tile-instance count, blend), once per module.  Every rank's frame must then be exactly 0
outside its own coarse tiles and bit-identical to that frame inside them, in RGBA8 and RGBA32F; the ranks' frames must sum to it and
their tile-instance counts to its count."""
import numpy as np
import pytest

import blend_f64 as BF
import frame_f64 as FF

pytestmark = pytest.mark.gpu

# (w, h, fine-tile px, coarse tiles, highest diagonal cx + cy, flip_y): what each frame selects
SHAPES = [
    (801, 455, 16, 56, 13, True),          # counting sort, compacted placement
    (2600, 1500, 32, 132, 21, False),      # 32-px tiles, counting sort
    (4097, 2049, 32, 289, 32, True),       # radix binning: sharded k_tile_count / k_tile_emit and the instance sort
    (8192, 64, 16, 64, 63, False),         # placement without its compaction (512 fine tiles per row), diagonals 0-63
    (8320, 64, 16, 65, 64, True),          # diagonal 64
    (16512, 64, 16, 129, 128, False),      # diagonal 128, 16-px tiles
    (256, 16640, 32, 130, 129, True),      # diagonal 129 along y, 32-px tiles
    (33024, 256, 32, 258, 129, False),     # diagonal 129 under the radix binning
    (640, 120, 16, 10, 5, True),           # world 8: ranks 6 and 7 own no tile
]
PATH_SHAPES = {(801, 455), (4097, 2049)}   # every rank also renders three cameras through its graph and eagerly
CAMERAS = 3
WORLDS = [2, 3, 8]
SUBSET_MIN = {"subset": "1", "replicated": "4000000000"}
BIG_SPLATS = 40
WHOLE_FRAME_PX = 4_300_000                 # blend-checked whole up to this size, on windows above it


def _shape_id(s):
    return f"{s[0]}x{s[1]}"


def _camera(w, h, k=0):
    """Orthographic camera at 1 px per world unit looking down -z at the scene; camera k is panned by (37 k, -23 k) px.  Returns the
    uniforms and the MVP (column-major)."""
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.engine import Uniforms
    cam = TM.PerspectiveCamera(50, w / h, 0.1, 1000)
    x, y = 37.0 * k, -23.0 * k
    cam.position = np.array([x, y, 400.0])
    cam.look_at((x, y, 0.0))
    P = TM.make_orthographic(-w / 2, w / 2, h / 2, -h / 2, 0.1, 1000.0, 1.0)
    mv = cam.matrixWorldInverse
    u = Uniforms(model_view=mv.astype(np.float32), projection=P.astype(np.float32), camera_position=cam.position.astype(np.float32),
                 focal=(1.0, 1.0), viewport=(w, h), ortho_zoom=1.0, orthographic_mode=1, max_screen_space_splat_size=30000.0)
    return u, TM.multiply(P, mv).astype(np.float32)


def _scene(w, h, seed):
    """Small splats (sigma 1.5-8 px, any orientation) spread over the whole frame, and BIG_SPLATS faint ones whose half extents are
    0.4-0.7 of the frame's width and height (nearly axis-aligned): those span more than 32 coarse tiles wherever the frame has them.
    Depths spread over 100 units.  Returns (centers_colors, covariances, centres)."""
    from gaussiansplats3d_b200.scenes import compute_covariances, pack_centers_colors
    rng = np.random.default_rng(seed)
    m = min(60_000, max(4_000, w * h // 120))
    n = m + BIG_SPLATS
    centers = np.empty((n, 3))
    centers[:, 0] = rng.uniform(-0.5, 0.5, n) * w
    centers[:, 1] = rng.uniform(-0.5, 0.5, n) * h
    centers[:, 2] = rng.uniform(-50.0, 50.0, n)
    scales = np.ones((n, 3))
    scales[:m, :2] = np.exp(rng.uniform(np.log(1.5), np.log(8.0), (m, 2)))
    scales[m:, :2] = rng.uniform(0.4, 0.7, (BIG_SPLATS, 2)) * (w, h) / np.sqrt(8.0)      # half extent = sqrt(8) sigma
    angle = np.concatenate([rng.uniform(0.0, np.pi, m), rng.choice([-1.0, 1.0], BIG_SPLATS) * rng.uniform(1e-3, 1e-2, BIG_SPLATS)])
    q = np.zeros((n, 4))                                   # x, y, z, w: a rotation about the view axis
    q[:, 2], q[:, 3] = np.sin(angle / 2), np.cos(angle / 2)
    colors = np.empty((n, 4), np.uint8)
    colors[:, :3] = rng.integers(0, 256, (n, 3))
    colors[:m, 3] = rng.integers(40, 256, m)
    colors[m:, 3] = rng.integers(8, 40, BIG_SPLATS)
    centers = centers.astype(np.float32)
    return pack_centers_colors(centers, colors), compute_covariances(scales.astype(np.float32), q.astype(np.float32)), centers


def _diagonals(w, h, flip_y):
    """[h, w] coarse diagonal cx + cy of every pixel, in the frame's row order."""
    t = BF.tile_px(w, h)
    ys, xs = np.mgrid[0:h, 0:w]
    d = xs // (8 * t) + ys // (4 * t)
    return d[::-1] if flip_y else d


def _owner_map(w, h, world, flip_y):
    from gaussiansplats3d_b200.parallel import ownership_map
    m = ownership_map(w, h, world)
    return m[::-1] if flip_y else m


def _blend_windows(w, h):
    """None (the whole frame) up to WHOLE_FRAME_PX; above it FF.windows plus the frame's last 1024 x 512 px, the highest diagonals."""
    if w * h <= WHOLE_FRAME_PX:
        return None
    x0, y0 = max(0, w - 1024) // 8 * 8, max(0, h - 512) // 8 * 8
    return sorted(set(FF.windows(w, h)) | {(x0, y0, w - x0, h - y0)})


# Sort option sets: Engine keywords, the reference sorter's, and the draw list (None: every splat in input order)
VARIANTS = {
    "default": dict(engine={}, sort={}),
    "keys32": dict(engine=dict(distance_map_range=1 << 20), sort=dict(precision=20)),
    "float22": dict(engine=dict(distance_map_range=1 << 22, integer_based_sort=False), sort=dict(precision=22, integer=False)),
    "indexes": dict(engine={}, sort={}, indexes=True),
}


class Case:
    """One scene at one frame shape under one sort option set: the engine factory and draw arguments that the single engine and every
    rank share."""

    def __init__(self, shape, variant):
        from gaussiansplats3d_b200.scenes import float_centers, integer_centers
        self.w, self.h, self.tile_px, self.ncoarse, self.max_diag, self.flip_y = shape
        self.variant = variant
        v = VARIANTS[variant]
        self.engine_kw, self.sort_kw = v["engine"], v["sort"]
        self.cc, self.cov, centers = _scene(self.w, self.h, seed=self.w * 7 + self.h)
        self.n = centers.shape[0]
        integer = self.engine_kw.get("integer_based_sort", True)
        self.sort_centers = integer_centers(centers) if integer else float_centers(centers)
        self.indexes = None
        if v.get("indexes"):
            rng = np.random.default_rng(self.n)
            self.indexes = rng.permutation(self.n)[: self.n * 7 // 10].astype(np.uint32)      # shuffled, 70 % of the splats
        self.count = self.n if self.indexes is None else len(self.indexes)

    def engine(self, rank=0, world=1):
        from gaussiansplats3d_b200.engine import Engine
        e = Engine(self.n, max_width=self.w, max_height=self.h, rank=rank, world_size=world, **self.engine_kw)
        e.upload_splat_data(self.cc, self.cov)
        e.upload_centers(self.sort_centers)
        return e

    def frame(self, e, k, fmt):
        u, mvp = _camera(self.w, self.h, k)
        return e.frame(mvp, u, self.w, self.h, self.count, self.indexes, frame_format=fmt, flip_y=self.flip_y).copy()


class Singles:
    """Single-engine frames (RGBA32F, RGBA8, tile instances) per (shape, variant, camera), each held to the f64 checks once."""

    def __init__(self):
        self.cases, self.frames = {}, {}

    def case(self, shape, variant):
        key = (shape, variant)
        if key not in self.cases:
            self.cases[key] = Case(shape, variant)
        return self.cases[key]

    def get(self, shape, variant, k):
        from gaussiansplats3d_b200 import _native as N
        key = (shape, variant, k)
        if key in self.frames:
            return self.frames[key]
        c = self.case(shape, variant)
        e = c.engine()
        got = c.frame(e, k, N.GS_FRAME_RGBA32F)
        got8 = c.frame(e, k, N.GS_FRAME_RGBA8)
        inst = e.timings()["tile_instances"]
        u, mvp = _camera(c.w, c.h, k)
        sort = dict(centers=c.sort_centers, mvp=mvp, splat_count=c.n, **c.sort_kw)
        if c.indexes is not None:
            sort["indexes"] = c.indexes
        FF.check_frame(f"{c.w}x{c.h} {variant} camera {k}", e, u, c.w, c.h, c.count, c.cc, c.cov, got=got, got8=got8, sort=sort,
                       windows=_blend_windows(c.w, c.h), flip_y=c.flip_y, min_compared=c.count // 2)
        if k == 0:
            # the scene reaches the frame's highest diagonals, and its big splats span more than 32 coarse tiles where there are that many
            diag = _diagonals(c.w, c.h, c.flip_y)
            for d in range(120, c.max_diag + 1):
                assert (got[..., 3][diag == d] > 0).any(), f"{c.w}x{c.h}: nothing covered on diagonal {d}"
            assert (got[..., 3] > 0).mean() > 0.9, f"{c.w}x{c.h}: only {(got[..., 3] > 0).mean():.3f} of the frame covered"
            if c.ncoarse > 32:
                ps = e.read_projected(c.n)
                spans = FF.coarse_spans(ps, c.w, c.h, 4 if c.tile_px == 16 else 5)
                assert (spans > 32).sum() >= 5, f"{c.w}x{c.h}: only {(spans > 32).sum()} splats span more than 32 coarse tiles"
        e.close()
        self.frames[key] = (got, got8, inst)
        return self.frames[key]


@pytest.fixture(scope="module")
def singles():
    return Singles()


def _check_rank_frame(label, f, want, mine):
    """A rank's frame: exactly 0 outside its own tiles, bit-identical to the single-engine frame inside them."""
    assert f.dtype == want.dtype and f.shape == want.shape, label
    assert not f[~mine].any(), f"{label}: pixels written outside the rank's own coarse tiles"
    assert f[mine].tobytes() == want[mine].tobytes(), \
        f"{label}: {int((f[mine] != want[mine]).any(-1).sum())} of the rank's {int(mine.sum())} pixels differ from the single-engine frame"


def _render_ranks(c, world, singles, shape, variant, subset):
    """Every rank's frames of camera 0 in both formats, checked against the single-engine frames; camera paths on PATH_SHAPES; the
    subset path's kernels.  Returns the per-rank RGBA8 frames and RGBA32F frames."""
    from gaussiansplats3d_b200 import _native as N
    want32, want8, want_inst = singles.get(shape, variant, 0)
    owner = _owner_map(c.w, c.h, world, c.flip_y)
    frames8, frames32, insts = [], [], []
    for r in range(world):
        mine = owner == r
        label = f"{c.w}x{c.h} {variant} world {world} rank {r}"
        e = c.engine(r, world)
        f32 = c.frame(e, 0, N.GS_FRAME_RGBA32F)
        f8 = c.frame(e, 0, N.GS_FRAME_RGBA8)
        t = e.timings()
        insts.append(t["tile_instances"])
        graph_launches = t["kernel_launches"]
        _check_rank_frame(f"{label} RGBA32F", f32, want32, mine)
        _check_rank_frame(f"{label} RGBA8", f8, want8, mine)
        if not mine.any():
            assert insts[-1] == 0 and not f8.any() and not f32.any(), f"{label}: a rank without tiles drew {insts[-1]} instances"
        # which sort ran: a profiled frame runs eagerly and names its kernels
        e.set_profiling(True)
        c.frame(e, 0, N.GS_FRAME_RGBA8)
        names = [k for k, _ in e.kernel_timings()]
        e.set_profiling(False)
        if subset:
            assert "k_subset_count" in names and "k_subset_emit" in names, f"{label}: the eager frame did not sort its subset: {names}"
            assert graph_launches == len(names), f"{label}: the graph frame launched {graph_launches} kernels, the eager frame {len(names)}"
        else:
            assert "k_subset_count" not in names, f"{label}: a replicated sort ran the subset compaction"
        if (c.w, c.h) in PATH_SHAPES and variant == "default":
            # the camera moves: the graph replays with this frame's subset count; then the same frames eagerly
            paths = {}
            for graph in (True, False):
                e.set_graph_enabled(graph)
                paths[graph] = [c.frame(e, k, N.GS_FRAME_RGBA32F) for k in range(CAMERAS)]
            e.set_graph_enabled(True)
            for k in range(CAMERAS):
                assert paths[True][k].tobytes() == paths[False][k].tobytes(), f"{label} camera {k}: graph and eager frames differ"
                _check_rank_frame(f"{label} camera {k}", paths[True][k], singles.get(shape, variant, k)[0], mine)
            assert paths[True][0].tobytes() != paths[True][-1].tobytes() or not mine.any(), f"{label}: the camera should move"
        e.close()
        frames8.append(f8)
        frames32.append(f32)
    from gaussiansplats3d_b200.parallel import combine_frames
    assert np.array_equal(combine_frames(frames8), want8), "the ranks' RGBA8 frames do not sum to the single-engine frame"
    assert np.array_equal(combine_frames(frames32), want32), "the ranks' RGBA32F frames do not sum to the single-engine frame"
    assert sum(insts) == want_inst, f"tile instances per rank {insts} sum to {sum(insts)}, the single engine drew {want_inst}"


@pytest.mark.parametrize("strategy", list(SUBSET_MIN))
@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("shape", SHAPES, ids=_shape_id)
def test_sharded_frame_equals_single_engine_frame(gs, oracle_mod, singles, shape, world, strategy, monkeypatch):
    """Every rank of `world` engines renders its own coarse tiles of the single-engine frame bit for bit and nothing else, in RGBA8 and
    RGBA32F, and the ranks' tile instances add up to the single engine's; on 801x455 and 4097x2049 also for three camera positions,
    through the graph (replayed with a changing subset count) and eagerly."""
    w, h, tile_px, ncoarse, max_diag, _ = shape
    t = BF.tile_px(w, h)
    assert t == tile_px and -(-w // (8 * t)) * -(-h // (4 * t)) == ncoarse
    assert (-(-w // (8 * t)) - 1) + (-(-h // (4 * t)) - 1) == max_diag
    monkeypatch.setenv("GS_SUBSET_MIN", SUBSET_MIN[strategy])
    c = singles.case(shape, "default")
    _render_ranks(c, world, singles, shape, "default", strategy == "subset")


@pytest.mark.parametrize("variant", ["keys32", "float22", "indexes"])
@pytest.mark.parametrize("shape", [s for s in SHAPES if (s[0], s[1]) in PATH_SHAPES], ids=_shape_id)
def test_subset_sort_variants(gs, oracle_mod, singles, shape, variant, monkeypatch):
    """The subset sort at world 3 with 32-bit keys (precision 20), float keys (precision 22) and a shuffled index list of 70 % of the
    splats: every rank's frame is the single engine's with the same options, restricted to its tiles."""
    monkeypatch.setenv("GS_SUBSET_MIN", "1")
    c = singles.case(shape, variant)
    _render_ranks(c, 3, singles, shape, variant, True)
