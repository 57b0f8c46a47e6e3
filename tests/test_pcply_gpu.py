"""GPU: PlayCanvas-compressed `.ply` files loaded with gs_upload_file leave every engine buffer (centres+colours, covariances, SH, sorter
centres) bit-identical to gs_upload_ksplat of the level-0 `.ksplat` image the reference builds from the same file
(oracle/pcply_oracle.py), apart from the splats whose scale depends on how `exp` rounds (flagged by the oracle: scale within 1 f32
ulp, so covariances within 1e-6 relative / 1 half ulp)."""
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent / "golden"))
import frame_f64 as FF  # noqa: E402
import pcply_handmade as PH  # noqa: E402

from oracle import pcply_oracle as PO  # noqa: E402

pytestmark = pytest.mark.gpu

PLY = 1
ROT_XF = [0.3, -0.5, 0.2, 0.7874007874011811]    # normalised quaternion x, y, z, w
VARIANTS = [dict(integer=True, half_cov=False, xf=False), dict(integer=False, half_cov=True, xf=False),
            dict(integer=True, half_cov=True, xf=True), dict(integer=False, half_cov=False, xf=True)]


def _transform():
    from gaussiansplats3d_b200 import three_math as TM
    return TM.compose((0.5, -1.25, 2.0), ROT_XF, (1.5, 0.75, 1.25))


def _buffers(e, n, *, half_cov, integer, ncomp):
    from gaussiansplats3d_b200 import _native as N
    out = dict(cc=e.read_buffer(N.GS_BUF_CENTERS_COLORS, np.uint32, 4 * n).reshape(n, 4),
               cov=e.read_buffer(N.GS_BUF_COVARIANCES, np.uint16 if half_cov else np.uint32, 6 * n).reshape(n, 6),
               centers=e.read_buffer(N.GS_BUF_CENTERS, np.int32 if integer else np.uint32, 4 * n).reshape(n, 4))
    if ncomp:
        out["sh"] = e.read_buffer(N.GS_BUF_SH, np.uint16, ncomp * n).reshape(n, ncomp)
    return out


def _compare(got, want, ambiguous, half_cov):
    ok = ~ambiguous
    for k in got:
        assert np.array_equal(got[k][ok], want[k][ok]), f"{k} differs on {np.nonzero((got[k] != want[k]).any(1) & ok)[0][:8]}"
    if ambiguous.any():   # only the scale, hence only the covariance, may differ
        if half_cov:
            assert (np.abs(got["cov"][ambiguous].astype(int) - want["cov"][ambiguous].astype(int)) <= 1).all()
        else:
            gc, wc = got["cov"][ambiguous].view(np.float32), want["cov"][ambiguous].view(np.float32)
            assert np.allclose(gc, wc, rtol=1e-6, atol=1e-30)
        for k in ("cc", "centers", "sh"):
            if k in got:
                assert np.array_equal(got[k][ambiguous], want[k][ambiguous])


def _load_both(gs, data, sh_degree, *, integer=True, half_cov=False, transform=None):
    """-> (number of flagged splats); asserts the two loads agree."""
    img, ambiguous = PO.level0_image(data, sh_degree)
    n = ambiguous.size
    info = gs.Engine.probe_file(PLY, data)
    assert info["splat_count"] == n
    deg = min(sh_degree, info["sh_degree"])
    ncomp = {0: 0, 1: 9, 2: 24}[deg]
    kw = dict(half_covariances=half_cov, transform16=transform)
    with gs.Engine(n + 5, max_width=64, max_height=64, integer_based_sort=integer) as e:
        got_info = e.upload_file(PLY, data, sh_degree=sh_degree, **kw)
        assert got_info["splat_count"] == n and got_info["sh_degree"] == deg and got_info["compression_level"] == 0
        got = _buffers(e, n, half_cov=half_cov, integer=integer, ncomp=ncomp)
    with gs.Engine(n + 5, max_width=64, max_height=64, integer_based_sort=integer) as e:
        want_info = e.upload_ksplat(img, **kw)
        assert want_info == got_info
        want = _buffers(e, n, half_cov=half_cov, integer=integer, ncomp=ncomp)
    _compare(got, want, ambiguous, half_cov)
    return int(ambiguous.sum())


def _synthetic(n, seed, *, nsh=45, color_extremes=True):
    rng = np.random.default_rng(seed)
    sh = rng.normal(0, 0.2, (n, nsh)) if nsh else None
    return PO.quantize(rng.uniform(-4, 4, (n, 3)), rng.uniform(-7, -2, (n, 3)), rng.normal(0, 1, (n, 4)), rng.uniform(0, 1, (n, 4)), sh,
                       color_extremes=color_extremes)


def _raw(n, seed, nsh, pad=1):
    """Random packed words (about 3.6 % NaN rotations) and SH bytes, NaN-free extremes, colour extremes on red only; `pad` uchar
    properties ahead of the packed words (vertex row = pad + 16 bytes)."""
    rng = np.random.default_rng(seed)
    nc = (n + 255) // 256 + 1
    props = [(k, "float") for k in PO.EXTREMES[:12]] + [("min_r", "float"), ("max_r", "float")]
    lo = rng.uniform(-4, 0, (nc, 3))
    slo = rng.uniform(-7, -4, (nc, 3))
    cols = {}
    for i, a in enumerate("xyz"):
        cols[f"min_{a}"], cols[f"max_{a}"] = lo[:, i], lo[:, i] + rng.uniform(0.5, 4, nc)
        cols[f"min_scale_{a}"], cols[f"max_scale_{a}"] = slo[:, i], slo[:, i] + rng.uniform(0.5, 3, nc)
    cols["min_r"], cols["max_r"] = rng.uniform(-0.2, 0.3, nc), rng.uniform(0.7, 1.2, nc)
    vprops = [(f"pad_{k}", "uchar") for k in range(pad)] + [(k, "uint") for k in PO.PACKED]
    vcols = {k: rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32) for k in PO.PACKED}
    vcols.update({f"pad_{k}": rng.integers(0, 256, n) for k in range(pad)})
    sh = rng.integers(0, 256, (n, nsh), dtype=np.uint8) if nsh else None
    return PO.write_pcply(props, cols, nc, vprops, vcols, n, sh)


@pytest.mark.parametrize("variant", range(len(VARIANTS)))
@pytest.mark.parametrize("name", sorted(PH.fixture_files()))
def test_fixture_loads_like_level0_image(gs, name, variant):
    v = VARIANTS[variant]
    data = (Path(__file__).resolve().parent / "golden" / name).read_bytes()
    for deg in (0, 1, 2):
        _load_both(gs, data, deg, integer=v["integer"], half_cov=v["half_cov"], transform=_transform() if v["xf"] else None)


@pytest.mark.parametrize("variant", range(len(VARIANTS)))
def test_synthetic_files_load_like_level0_image(gs, variant):
    v = VARIANTS[variant]
    kw = dict(integer=v["integer"], half_cov=v["half_cov"], transform=_transform() if v["xf"] else None)
    flagged = 0
    sh3 = _synthetic(20011, 3)
    for deg in (0, 1, 2):
        flagged += _load_both(gs, sh3, deg, **kw)
    for nsh in (0, 9, 24):
        flagged += _load_both(gs, _synthetic(5003, 4 + nsh, nsh=nsh, color_extremes=False), 2, **kw)
        flagged += _load_both(gs, _raw(7001, 5 + nsh, nsh), 2, **kw)
    print(f"flagged splats (exp rounding): {flagged}")


# (pad, sh properties, sphericalHarmonicsDegree): the bytes a CTA stages are 256 x (vertex row + loaded sh row); they fit the 48 KiB of
# shared memory less the kernel's 144-byte extremes table up to 191-byte rows, and wider rows are read in place
WIDE = [(175, 0, 0), (176, 0, 0), (152, 24, 0), (152, 24, 2), (300, 45, 2)]


@pytest.mark.parametrize("pad, nsh, deg", WIDE)
def test_wide_rows_load_like_level0_image(gs, pad, nsh, deg):
    """Rows at the edge of the shared-memory staging budget (191 B staged, 192 B in place) and well beyond it."""
    for variant in (VARIANTS[0], VARIANTS[2]):
        _load_both(gs, _raw(3001, pad + nsh, nsh, pad=pad), deg, integer=variant["integer"], half_cov=variant["half_cov"],
                   transform=_transform() if variant["xf"] else None)


def test_large_file_spans_several_chunks(gs):
    """About 4 M SH3 splats (a count that is not a multiple of 256) go through the 64 MiB staging chunks at least three times."""
    n = 4_000_037
    data = _synthetic(n, 21)
    assert n * (16 + 45) > 3 * (64 << 20)
    flagged = _load_both(gs, data, 2)
    print(f"flagged splats (exp rounding): {flagged} of {n}")


def _viewer(w, h):
    from gaussiansplats3d_b200.scenes import CAMERAS
    from gaussiansplats3d_b200.viewer import Viewer
    c = CAMERAS["bonsai"]
    return Viewer(dict(cameraUp=c["up"], initialCameraPosition=c["position"], initialCameraLookAt=c["look_at"], width=w, height=h, sphericalHarmonicsDegree=2))


def test_viewer_frame_from_file_equals_frame_from_level0_image(gs, oracle_mod):
    from oracle import ksplat_oracle as KO
    data = _synthetic(60000, 5)
    img, _ = PO.level0_image(data, 2)
    w, h = 640, 360
    frames = {}
    N = gs._native
    for kind in ("file", "ksplat"):
        v = _viewer(w, h)
        info = v.addSplatSceneFromFile(data, PLY) if kind == "file" else v.addSplatSceneFromKSplat(img)
        assert info["splat_count"] == 60000 and info["sh_degree"] == 2
        for fmt in (N.GS_FRAME_RGBA8, N.GS_FRAME_RGBA32F):
            frames[kind, fmt] = v.frame(frame_format=fmt, flip_y=False).copy()
        if kind == "file":
            FF.check_viewer_frame("frame from file", v, got=frames[kind, N.GS_FRAME_RGBA32F], got8=frames[kind, N.GS_FRAME_RGBA8],
                                  scene=KO.decode(img), min_compared=1000)
        v.dispose()
    for fmt in (gs._native.GS_FRAME_RGBA8, gs._native.GS_FRAME_RGBA32F):
        assert np.array_equal(frames["file", fmt], frames["ksplat", fmt])
        assert frames["file", fmt].any()


def test_malformed_files_leave_previous_scene(gs):
    """Each malformed compressed file comes back with its error, and the engine still renders the scene it had, bit for bit."""
    data = _synthetic(20000, 6, nsh=9)
    v = _viewer(320, 200)
    v.addSplatSceneFromFile(data, PLY)
    before = v.frame(frame_format=gs._native.GS_FRAME_RGBA32F, flip_y=False).copy()
    assert before.any()
    cases = {k: (blob, PH.BAD_ARG, words) for k, (blob, words) in PH.MALFORMED.items()}
    cases["capacity"] = (_synthetic(20001, 7, nsh=0), 7, "capacity")
    for name, (blob, status, words) in cases.items():
        with pytest.raises(gs.GsError) as ei:
            v.engine.upload_file(PLY, blob, sh_degree=2)
        assert ei.value.code == status and words in str(ei.value), (name, str(ei.value))
        after = v.frame(frame_format=gs._native.GS_FRAME_RGBA32F, flip_y=False)
        assert np.array_equal(after, before), name
    v.dispose()
