"""GPU: `.spz` files.  gs_upload_file(GS_FILE_SPZ) leaves every engine buffer (centres+colours, covariances, SH, sorter centres, ray
records) bit-identical to gs_upload_ksplat of the level-0 `.ksplat` image SpzLoader builds with optimizeSplatData off
(tests/spz_oracle.py), apart from splats whose scale depends on how `exp` rounds (flagged by the oracle; none of the 256 scale bytes is,
with NumPy's exp).  gs_generate_splat_buffer is byte-identical to oracle/generate_oracle.py fed with the same splats, and the Viewer
loads a `.spz` as stored."""
import gzip
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent / "golden"))
import spz_handmade as SH  # noqa: E402
import spz_oracle as SO  # noqa: E402

from oracle import generate_oracle as GO  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden"
SPZ = 4
ROT_XF = [0.3, -0.5, 0.2, 0.7874007874011811]    # normalised quaternion x, y, z, w
VARIANTS = [dict(integer=True, half_cov=False, xf=False), dict(integer=False, half_cov=True, xf=False),
            dict(integer=True, half_cov=True, xf=True), dict(integer=False, half_cov=False, xf=True)]


def _transform():
    from gaussiansplats3d_b200 import three_math as TM
    return TM.compose((0.5, -1.25, 2.0), ROT_XF, (1.5, 0.75, 1.25))


def _buffers(e, n, *, half_cov, integer, ncomp, level=0):
    from gaussiansplats3d_b200 import _native as N
    out = dict(cc=e.read_buffer(N.GS_BUF_CENTERS_COLORS, np.uint32, 4 * n).reshape(n, 4),
               cov=e.read_buffer(N.GS_BUF_COVARIANCES, np.uint16 if half_cov else np.uint32, 6 * n).reshape(n, 6),
               centers=e.read_buffer(N.GS_BUF_CENTERS, np.int32 if integer else np.uint32, 4 * n).reshape(n, 4),
               ray=e.read_buffer(N.GS_BUF_RAY_RECORDS, np.uint8, 56 * n).reshape(n, 56))
    if ncomp:
        out["sh"] = e.read_buffer(N.GS_BUF_SH, np.uint8 if level == 2 else np.uint16, ncomp * n).reshape(n, ncomp)
    return out


def _compare(got, want, ambiguous, half_cov):
    ok = ~ambiguous
    for k in got:
        assert np.array_equal(got[k][ok], want[k][ok]), f"{k} differs on {np.nonzero((got[k] != want[k]).any(1) & ok)[0][:8]}"
    if ambiguous.any():   # only the scale, hence the covariance and the ray record's scale, may differ
        if half_cov:
            assert (np.abs(got["cov"][ambiguous].astype(int) - want["cov"][ambiguous].astype(int)) <= 1).all()
        else:
            assert np.allclose(got["cov"][ambiguous].view(np.float32), want["cov"][ambiguous].view(np.float32), rtol=1e-6, atol=1e-30)
        gs_, ws_ = got["ray"][ambiguous, 24:36].copy().view(np.int32), want["ray"][ambiguous, 24:36].copy().view(np.int32)
        assert (np.abs(gs_ - ws_) <= 1).all()
        keep = np.r_[0:24, 36:56]
        assert np.array_equal(got["ray"][ambiguous][:, keep], want["ray"][ambiguous][:, keep])
        for k in ("cc", "centers", "sh"):
            if k in got:
                assert np.array_equal(got[k][ambiguous], want[k][ambiguous])


def _load_both(gs, data, sh_degree, *, integer=True, half_cov=False, transform=None):
    """data: a packed stream.  -> number of flagged splats; asserts the two loads agree."""
    img, ambiguous = SO.level0_image(data, sh_degree)
    n = ambiguous.size
    info = gs.Engine.probe_file(SPZ, data)
    assert info["splat_count"] == n
    deg = min(sh_degree, info["sh_degree"])
    ncomp = {0: 0, 1: 9, 2: 24}[deg]
    kw = dict(half_covariances=half_cov, transform16=transform)
    cfg = dict(max_width=64, max_height=64, integer_based_sort=integer, ray_records=True)
    with gs.Engine(n + 5, **cfg) as e:
        got_info = e.upload_file(SPZ, data, sh_degree=sh_degree, **kw)
        assert got_info["splat_count"] == n and got_info["sh_degree"] == deg and got_info["compression_level"] == 0
        got = _buffers(e, n, half_cov=half_cov, integer=integer, ncomp=ncomp) if n else None
    with gs.Engine(n + 5, **cfg) as e:
        want_info = e.upload_ksplat(img, **kw)
        assert want_info == got_info
        want = _buffers(e, n, half_cov=half_cov, integer=integer, ncomp=ncomp) if n else None
    if n:
        _compare(got, want, ambiguous, half_cov)
    return int(ambiguous.sum())


def _synthetic(n, seed, *, sh_degree=3, compress=False):
    rng = np.random.default_rng(seed)
    q = rng.normal(0, 1, (n, 4))
    sh = rng.normal(0, 0.3, (n, 3, SO.DIM[sh_degree])) if sh_degree else None
    return SO.quantize(rng.normal(0, 6, (n, 3)), rng.uniform(-7, -2, (n, 3)), q, rng.uniform(0, 1, (n, 4)), sh, sh_degree=sh_degree,
                       compress=compress)


@pytest.mark.parametrize("variant", range(len(VARIANTS)))
@pytest.mark.parametrize("name", sorted(SH.FIXTURES))
def test_fixture_loads_like_level0_image(gs, name, variant):
    v = VARIANTS[variant]
    data = gzip.decompress((GOLDEN / SH.file_name(name)).read_bytes())
    for deg in (0, 1, 2):
        assert _load_both(gs, data, deg, integer=v["integer"], half_cov=v["half_cov"], transform=_transform() if v["xf"] else None) == 0


@pytest.mark.parametrize("variant", range(len(VARIANTS)))
def test_synthetic_sh3_files_load_like_level0_image(gs, variant):
    """Seeded SH3 files read as degrees 0, 1 and 2, and random bytes in every plane (v1 and v2)."""
    v = VARIANTS[variant]
    kw = dict(integer=v["integer"], half_cov=v["half_cov"], transform=_transform() if v["xf"] else None)
    sh3 = _synthetic(20011, 3)
    for deg in (0, 1, 2):
        _load_both(gs, sh3, deg, **kw)
    rng = np.random.default_rng(7 + variant)
    n = 9001
    for version, fb in ((2, 10), (2, 31), (1, 0)):
        pos = rng.integers(0, 256, (n, 9), dtype=np.uint8) if version == 2 else rng.integers(0, 1 << 16, (n, 3), dtype=np.uint16)
        planes = [rng.integers(0, 256, s, dtype=np.uint8) for s in ((n,), (n, 3), (n, 3), (n, 3), (n, 45))]
        _load_both(gs, SO.write_spz(pos, *planes, version=version, sh_degree=3, fractional_bits=fb), 2, **kw)


def test_large_file_spans_several_chunks(gs):
    """About 2.5 M SH3 splats (64 bytes each in the stream) go through the 64 MiB staging chunks three times."""
    n = 2_500_037
    data = _synthetic(n, 21)
    assert n * 64 > 2 * (64 << 20)
    assert _load_both(gs, data, 2) == 0
    assert _load_both(gs, data, 0, integer=False, half_cov=True) == 0


def _check_image(gs, data, sh_degree, **kw):
    from gaussiansplats3d_b200.engine import generate_splat_buffer
    rec, c64, sh, deg, amb = SO.generator_inputs(data, sh_degree)
    got = generate_splat_buffer(SPZ, data, sh_degree=sh_degree, **kw)
    want, loose = GO.generate(rec, c64, sh, deg, level=kw.get("compression_level", 1), minimum_alpha=kw.get("minimum_alpha", 1),
                              section_size=kw.get("section_size", 0), scene_center=kw.get("scene_center", (0.0, 0.0, 0.0)),
                              block_size=kw.get("block_size", 5.0), bucket_size=kw.get("bucket_size", 256), loose=amb)
    assert len(got) == len(want)
    diff = np.nonzero((np.frombuffer(got, np.uint8) != np.frombuffer(want, np.uint8)) & ~loose)[0]
    assert diff.size == 0, f"{diff.size} bytes differ, first at {diff[:8]}"
    return got


@pytest.mark.parametrize("name", sorted(SH.FIXTURES))
def test_fixture_images_match_generate_oracle(gs, name):
    data = SH.packed_fixture(name)
    for level in (0, 1, 2):
        for deg in (0, 1, 2):
            for alpha in (0, 1, 128):
                _check_image(gs, data, deg, compression_level=level, minimum_alpha=alpha)


def test_synthetic_images_match_generate_oracle(gs):
    data = _synthetic(300_007, 12)
    for level in (0, 1, 2):
        _check_image(gs, data, 2, compression_level=level, section_size=120_000, bucket_size=64)
        _check_image(gs, data, 1, compression_level=level, minimum_alpha=128, block_size=1.5, scene_center=(1.0, -2.0, 0.5))


@pytest.mark.parametrize("level", [0, 1, 2])
def test_optimized_load_equals_ksplat_of_generated_image(gs, level):
    data = _synthetic(50_021, 8)
    for v in (VARIANTS[0], VARIANTS[3]):
        img = _check_image(gs, data, 2, compression_level=level, minimum_alpha=5)
        kw = dict(half_covariances=v["half_cov"], transform16=_transform() if v["xf"] else None, minimum_alpha=5)
        cfg = dict(max_width=64, max_height=64, integer_based_sort=v["integer"], ray_records=True)
        with gs.Engine(50_100, **cfg) as e:
            info = e.upload_file_optimized(SPZ, data, sh_degree=2, compression_level=level, **kw)
            n = info["splat_count"]
            got = _buffers(e, n, half_cov=v["half_cov"], integer=v["integer"], ncomp=24, level=level)
        with gs.Engine(50_100, **cfg) as e:
            assert e.upload_ksplat(img, **kw) == info
            want = _buffers(e, n, half_cov=v["half_cov"], integer=v["integer"], ncomp=24, level=level)
        assert 0 < n < 50_021
        for k in got:
            assert np.array_equal(got[k], want[k]), k


def _viewer(w, h, **extra):
    from gaussiansplats3d_b200.scenes import CAMERAS
    from gaussiansplats3d_b200.viewer import Viewer
    c = CAMERAS["bonsai"]
    return Viewer(dict(cameraUp=c["up"], initialCameraPosition=c["position"], initialCameraLookAt=c["look_at"], width=w, height=h,
                       sphericalHarmonicsDegree=2, **extra))


def test_viewer_loads_spz_as_stored(gs):
    """addSplatSceneFromFile(gz, SceneFormat.Spz): optimizeSplatData on renders the generator's .ksplat frame, off renders the level-0
    image's frame; progressiveLoad changes neither."""
    from gaussiansplats3d_b200.engine import generate_splat_buffer
    from gaussiansplats3d_b200.loaders import SceneFormat
    gz = _synthetic(60_013, 6, compress=True)
    data = gzip.decompress(gz)
    images = {True: generate_splat_buffer(SPZ, data, sh_degree=2, compression_level=0, minimum_alpha=1), False: SO.level0_image(data, 2)[0]}
    w, h = 640, 360
    for optimize in (True, False):
        frames = []
        for kind in ("ksplat", "file", "file_progressive"):
            v = _viewer(w, h, optimizeSplatData=optimize)
            if kind == "ksplat":
                info = v.addSplatSceneFromKSplat(images[optimize])
            else:
                info = v.addSplatSceneFromFile(gz, SceneFormat.Spz, progressiveLoad=kind == "file_progressive")
            frames.append((info["splat_count"], v.frame(frame_format=gs._native.GS_FRAME_RGBA32F, flip_y=False).copy()))
            v.dispose()
        assert frames[0][0] == frames[1][0] == frames[2][0]
        assert (frames[0][0] < 60_013) if optimize else (frames[0][0] == 60_013)
        assert frames[0][1].any()
        assert np.array_equal(frames[0][1], frames[1][1]) and np.array_equal(frames[0][1], frames[2][1]), optimize


def test_malformed_files_leave_previous_scene(gs):
    """Each malformed stream comes back with its error, and the engine still renders the scene it had, bit for bit."""
    from gaussiansplats3d_b200.loaders import SceneFormat
    gz = _synthetic(20_000, 9, sh_degree=1, compress=True)
    v = _viewer(320, 200, optimizeSplatData=False)
    v.addSplatSceneFromFile(gz, SceneFormat.Spz)
    before = v.frame(frame_format=gs._native.GS_FRAME_RGBA32F, flip_y=False).copy()
    assert before.any()
    cases = {k: (blob, SH.BAD_ARG, words) for k, (blob, words) in SH.MALFORMED.items()}
    cases["capacity"] = (_synthetic(20_001, 10, sh_degree=0), 7, "capacity")
    for name, (blob, status, words) in cases.items():
        for upload in (v.engine.upload_file, v.engine.upload_file_optimized):
            with pytest.raises(gs.GsError) as ei:
                upload(SPZ, blob, sh_degree=2)
            assert ei.value.code == status and words in str(ei.value), (name, str(ei.value))
            after = v.frame(frame_format=gs._native.GS_FRAME_RGBA32F, flip_y=False)
            assert np.array_equal(after, before), name
    v.dispose()
