"""GPU: the radix sort (csrc/sort_kernels.cuh: RadixSort, k_radix_hist / k_radix_scan / k_radix_scatter) at every key width and pass
plan, past one k_radix_scan block of 1024 radix tiles, with keys chosen digit by digit.

The keys are set exactly through integer precomputed distances (cases.keyed_case): 0 and R-1 are both in the sorted window, so every
bucket equals its distance and every key is R-1-distance, for any distance_map_range R up to 2^24.  Every order is held two ways: bit for
bit to the reference sorter (the compiled reference where oracle/_ref has it, else oracle/sort_oracle.c), and to a plain NumPy statement
that shares nothing with either: the head [0, s0) is copied, the window is reversed and stably sorted by key.  The stateless drop-in's
scratch outputs are held to the buckets and their exclusive prefix counts.  The radix binning's instance sort is driven past 1024
radix tiles by a 4097x2049 frame of thin splats, held to the f64 projection and blend bounds (tests/frame_f64.py)."""
import numpy as np
import pytest

import cases
import frame_f64 as FF

TILE = 4096                    # kRadixTile: keys per radix tile (and per k_bucket / k_radix_hist / k_radix_scatter CTA)
BLOCK = 1024 * TILE            # keys per k_radix_scan block: beyond it the scan carries its running offset to the next block
HEAD = 777                     # unsorted head [0, s0) of a partial sort

SWEEP_RANGES = tuple(1 << kb for kb in range(1, 25)) + (3, 200, 257, 1000, 65535, 65537, (1 << 23) + 1)
SWEEP_SIZES = (4095, 4096, 4097, 3 * TILE + 1, 40_000)
ADVERSARIAL_RANGES = (1 << 8, 1 << 13, 1 << 16, (1 << 17) + 1, 1 << 24)   # one, two, two, three, three passes
LARGE_RANGES = (1 << 8, 1 << 16, (1 << 17) + 1, 1 << 24)
LARGE_SIZES = (BLOCK + 1, 2 * BLOCK + TILE + 1)


def _rid(R):
    return f"R{R}" if R & (R - 1) else f"R2^{R.bit_length() - 1}"


def _reference(oracle_mod, c, R):
    sorter = oracle_mod.ref_sort_indexes if oracle_mod.have_ref() else oracle_mod.port_sort_indexes
    return sorter(*cases.call_args(c, R))


def _numpy_order(c, R):
    """out[:s0] = indexes[:s0]; out[s0:] = the window reversed, stably sorted by key R-1-distance."""
    idx, rc = c["indexes"], c["render_count"]
    s0 = rc - c["sort_count"]
    w = idx[s0:rc][::-1]
    key = (R - 1) - c["precomputed"][w].astype(np.int64)
    return np.concatenate([idx[:s0], w[np.argsort(key, kind="stable")]]).astype(np.uint32)


def _same(label, got, want):
    assert got.shape == want.shape, f"{label}: {got.shape} != {want.shape}"
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{label}: {bad.size} positions differ, first at {bad[:5].tolist()}"


def _sort_checked(gs, oracle_mod, e, c, R, label, *, dropin=False):
    """Sort case c on engine e (identity cases pass no index list: the kValIotaReversed values) and, with dropin, through the stateless
    gs_sort_indexes with its scratch outputs; every output against the reference sorter and the NumPy statement."""
    want = _reference(oracle_mod, c, R)
    _same(f"{label}: reference vs NumPy", want, _numpy_order(c, R))
    identity = np.array_equal(c["indexes"], np.arange(c["render_count"], dtype=np.uint32))
    got, _ = e.sort(c["mvp"], c["sort_count"], c["render_count"], None if identity else c["indexes"], precomputed=c["precomputed"])
    _same(f"{label}: Engine.sort", got, want)
    if dropin:
        out, mapped, freq = gs.sort_indexes(*cases.call_args(c, R), want_scratch=True)
        _same(f"{label}: sort_indexes", out, want)
        s0 = c["render_count"] - c["sort_count"]
        buckets = c["precomputed"][c["indexes"][s0:]]
        _same(f"{label}: mappedDistances", mapped[s0:], buckets)
        counts = np.bincount(buckets, minlength=R)
        _same(f"{label}: frequencies", freq, (np.cumsum(counts) - counts).astype(np.uint32))


def _engine(gs, cap, R):
    e = gs.Engine(cap, distance_map_range=R)
    e.upload_centers(np.zeros((cap, 4), np.int32))     # the precomputed branch reads no centres; this sets the uploaded count
    return e


# ---- the plan -------------------------------------------------------------------------------------------------------------------------
def test_sweep_covers_every_plan():
    """The sweep's ranges reach every distinct (passes, digit widths) that key widths 1 to 24 produce, and the plan restated here is
    make_plan_bits' (ceil(kb / 8) passes, wider digits first)."""
    every = {cases.radix_plan(kb) for kb in range(1, 25)}
    swept = {cases.radix_plan(cases.key_bits(R)) for R in SWEEP_RANGES}
    assert every <= swept, every - swept
    assert [cases.key_bits(R) for R in (2, 3, 256, 257, 65535, 65537, (1 << 23) + 1, 1 << 24)] == [1, 2, 8, 9, 16, 17, 24, 24]
    widths = {kb: tuple(b for _, b in cases.radix_plan(kb)) for kb in (1, 8, 9, 13, 16, 17, 20, 21, 23, 24)}
    assert widths == {1: (1,), 8: (8,), 9: (5, 4), 13: (7, 6), 16: (8, 8), 17: (6, 6, 5), 20: (7, 7, 6), 21: (7, 7, 7), 23: (8, 8, 7),
                      24: (8, 8, 8)}
    for kb in range(1, 25):
        plan = cases.radix_plan(kb)
        assert sum(b for _, b in plan) == kb and all(s == sum(b for _, b in plan[:p]) for p, (s, _) in enumerate(plan))
    for R in ADVERSARIAL_RANGES + LARGE_RANGES:
        for kind in cases.KEY_KINDS:
            k = cases.radix_keys(kind, R, 3 * TILE + 1, np.random.default_rng(R))
            assert k.min() == 0 and k.max() == R - 1, (kind, R)


@pytest.mark.gpu
@pytest.mark.parametrize("R", SWEEP_RANGES, ids=[_rid(R) for R in SWEEP_RANGES])
def test_plan_sweep(gs, oracle_mod, R):
    """Every key width 1..24 (R = 2^kb) and ranges that are not powers of two: sizes around one radix tile, three tiles and a tail, and
    ten tiles; identity (kValIotaReversed) and shuffled (kValArrayReversed) index lists; full and partial sorts; random keys."""
    cap = max(SWEEP_SIZES) + HEAD
    with _engine(gs, cap, R) as e:
        for n in SWEEP_SIZES:
            for head in (0, HEAD):
                for kind in ("identity", "shuffled"):
                    c = cases.keyed_case(R + n + head, n, R, "random", index_kind=kind, head=head, splat_count=cap)
                    _sort_checked(gs, oracle_mod, e, c, R, f"R={R} n={n} head={head} {kind}", dropin=(kind == "shuffled"))


@pytest.mark.gpu
@pytest.mark.parametrize("R", ADVERSARIAL_RANGES, ids=[_rid(R) for R in ADVERSARIAL_RANGES])
def test_adversarial_keys(gs, oracle_mod, R):
    """Three radix tiles and one key: one key for all but the extremes, keys that differ only in the first or only in the last pass's
    digit, one key per radix tile, keys already in output order or reversed, only 0 and R-1, digits at their mask's maximum."""
    n = 3 * TILE + 1
    with _engine(gs, n, R) as e:
        for kind in cases.KEY_KINDS:
            for index_kind in ("identity", "shuffled"):
                c = cases.keyed_case(R + 17, n, R, kind, index_kind=index_kind)
                _sort_checked(gs, oracle_mod, e, c, R, f"R={R} {kind} {index_kind}", dropin=(index_kind == "shuffled"))


# ---- past one k_radix_scan block ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("R", LARGE_RANGES, ids=[_rid(R) for R in LARGE_RANGES])
def test_past_1024_radix_tiles(gs, oracle_mod, R):
    """1024 radix tiles and one key, and two blocks of 1024 tiles and a tile and one key, in one plan of each pass count: random keys and
    one key holding all but two, with both value modes."""
    cap = max(LARGE_SIZES)
    with _engine(gs, cap, R) as e:
        for n in LARGE_SIZES:
            for kind in ("random", "single"):
                for index_kind in ("identity", "shuffled"):
                    c = cases.keyed_case(R + n, n, R, kind, index_kind=index_kind, splat_count=cap)
                    _sort_checked(gs, oracle_mod, e, c, R, f"R={R} n={n} {kind} {index_kind}")


@pytest.mark.gpu
def test_float_static_past_1024_radix_tiles(gs, oracle_mod):
    """Float sort mode with static centres at splatSortDistanceMapPrecision 20 (three passes of 7+7+6 bits), past one scan block."""
    R, n = 1 << 20, BLOCK + 1
    c = cases.sort_case(seed=61, n=n, integer=False, index_kind="shuffled")
    with gs.Engine(n, distance_map_range=R, integer_based_sort=False) as e:
        e.upload_centers(c["centers"])
        got, _ = e.sort(c["mvp"], n, n, c["indexes"])
    _same("float static 2^20", got, _reference(oracle_mod, c, R))


@pytest.mark.gpu
def test_engine_reuse_across_sizes(gs, oracle_mod):
    """One engine at 2^24 sorts 1024 tiles and one key, then 4097 keys, then one, then 1024 tiles and one again: the self-cleaning
    scatters leave no digit total or min/max of one sort behind for the next."""
    R, big = 1 << 24, BLOCK + 1
    with _engine(gs, big, R) as e:
        for step, n in enumerate((big, 4097, 1, big)):
            if n == 1:      # one splat: the bucket is 0, so the output is the input (test_sort_gpu.test_edge_cases)
                c = cases.keyed_case(90 + step, 2, R, splat_count=big)
                got, _ = e.sort(c["mvp"], 1, 1, c["indexes"][:1], precomputed=c["precomputed"])
                _same("one key", got, c["indexes"][:1])
                continue
            c = cases.keyed_case(90 + step, n, R, index_kind="shuffled", splat_count=big)
            _sort_checked(gs, oracle_mod, e, c, R, f"step {step} n={n}")


# ---- radix binning past one scan block ------------------------------------------------------------------------------------------------
def _thin_splats(n, w, h, depth, seed):
    """Splats facing a camera at distance `depth`, long in x (about 1300 px at 4097x2049) and a pixel or so across: each touches several
    coarse tiles but covers few pixels, so the f64 blend of the check stays affordable.  They are tilted 0.2-0.5 degrees off the x axis:
    an axis-aligned one leaves the shader's eigenvector undetermined."""
    from gaussiansplats3d_b200.scenes import compute_covariances, pack_centers_colors
    rng = np.random.default_rng(seed)
    t = np.tan(np.deg2rad(25.0))
    centers = np.stack([rng.uniform(-1.1, 1.1, n) * t * depth * w / h, rng.uniform(-1.02, 1.02, n) * t * depth, rng.uniform(-1.0, 1.0, n)], 1)
    scales = np.stack([1.2 * np.exp(rng.uniform(-0.3, 0.3, n)), np.full(n, 1e-4), np.full(n, 1e-4)], 1)
    tilt = np.deg2rad(rng.uniform(0.2, 0.5, n)) * rng.choice([-1.0, 1.0], n)
    quats = np.zeros((n, 4), np.float32)                  # x, y, z, w: a turn about the view axis
    quats[:, 2], quats[:, 3] = np.sin(0.5 * tilt), np.cos(0.5 * tilt)
    colors = np.empty((n, 4), np.uint8)
    colors[:, :3] = rng.integers(0, 256, (n, 3))
    colors[:, 3] = rng.integers(8, 120, n)
    centers = centers.astype(np.float32)
    return pack_centers_colors(centers, colors), compute_covariances(scales.astype(np.float32), quats), centers


@pytest.mark.gpu
def test_radix_binning_past_1024_radix_tiles(gs, oracle_mod, monkeypatch):
    """A 4097x2049 frame (289 coarse tiles: 9-bit tile keys, sorted in passes of 5 + 4 bits) of 800 K thin splats that make more than
    1024 radix tiles of coarse-tile instances.  The draw order is the reference sorter's, and the frame holds to the f64 checks:
    the instance count, every projection, and the blend on FF.windows."""
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.engine import Engine
    from gaussiansplats3d_b200.scenes import integer_centers
    from test_raster_edges_gpu import _camera
    monkeypatch.setenv("GS_INSTANCE_FACTOR", "10")        # room for ~6 instances per splat
    w, h, n, depth = 4097, 2049, 800_000, 10.0
    assert -(-w // 256) * -(-h // 128) == 289 and cases.radix_plan(cases.key_bits(289)) == ((0, 5), (5, 4))
    cc, cov, centers = _thin_splats(n, w, h, depth, seed=71)
    ic = integer_centers(centers)
    u, _, mvp = _camera(w, h, (0.0, 0.0, depth), (0.0, 0.0, 0.0))
    with Engine(n, max_width=w, max_height=h) as e:
        e.upload_splat_data(cc, cov)
        e.upload_centers(ic)
        got = e.frame(mvp, u, w, h, n, frame_format=N.GS_FRAME_RGBA32F, flip_y=False).copy()
        got8 = e.frame(mvp, u, w, h, n, frame_format=N.GS_FRAME_RGBA8, flip_y=False).copy()   # an overflow would raise GS_ERR_CAPACITY
        inst = e.timings()["tile_instances"]
        assert inst > BLOCK, f"{inst} tile instances: not past one k_radix_scan block ({BLOCK})"
        FF.check_frame("radix binning 4097x2049", e, u, w, h, n, cc, cov, got=got, got8=got8, sort=dict(centers=ic, mvp=mvp),
                       windows=FF.windows(w, h), min_compared=n // 2)
