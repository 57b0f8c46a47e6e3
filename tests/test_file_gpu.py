"""GPU: `.ply` / `.splat` files loaded with gs_upload_file leave every engine buffer (centres+colours, covariances, SH, sorter centres)
bit-identical to gs_upload_ksplat of the level-0 `.ksplat` image the reference's progressive loader builds from the same file
(oracle/file_oracle.py), apart from the splats whose scale or alpha depends on how `exp` rounds (flagged by the oracle: scale within
1 f32 ulp, so covariances within 1e-6 relative / 1 half ulp; alpha within one step)."""
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent / "golden"))
import file_handmade as FH  # noqa: E402
import frame_f64 as FF  # noqa: E402

from oracle import file_oracle as FO  # noqa: E402

pytestmark = pytest.mark.gpu

ROT_XF = [0.3, -0.5, 0.2, 0.7874007874011811]    # normalised quaternion x, y, z, w


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
    if ambiguous.any():
        g, w = got["cc"][ambiguous], want["cc"][ambiguous]
        assert np.array_equal(g[:, 1:], w[:, 1:]) and np.array_equal(g[:, 0] & 0xFFFFFF, w[:, 0] & 0xFFFFFF)
        assert (np.abs((g[:, 0] >> 24).astype(int) - (w[:, 0] >> 24).astype(int)) <= 1).all()
        if half_cov:
            assert (np.abs(got["cov"][ambiguous].astype(int) - want["cov"][ambiguous].astype(int)) <= 1).all()
        else:
            gc, wc = got["cov"][ambiguous].view(np.float32), want["cov"][ambiguous].view(np.float32)
            assert np.allclose(gc, wc, rtol=1e-6, atol=1e-30)
        for k in ("centers", "sh"):
            if k in got:
                assert np.array_equal(got[k][ambiguous], want[k][ambiguous])


def _load_both(gs, fmt, data, sh_degree, *, integer=True, half_cov=False, transform=None):
    """-> (number of flagged splats); asserts the two loads agree."""
    img, ambiguous = FO.level0_image(fmt, data, sh_degree)
    n = ambiguous.size
    info = gs.Engine.probe_file(fmt, data)
    assert info["splat_count"] == n
    deg = min(sh_degree, info["sh_degree"])
    ncomp = {0: 0, 1: 9, 2: 24}[deg]
    kw = dict(half_covariances=half_cov, transform16=transform)
    with gs.Engine(n + 5, max_width=64, max_height=64, integer_based_sort=integer) as e:
        got_info = e.upload_file(fmt, data, sh_degree=sh_degree, **kw)
        assert got_info["splat_count"] == n and got_info["sh_degree"] == deg and got_info["compression_level"] == 0
        got = _buffers(e, n, half_cov=half_cov, integer=integer, ncomp=ncomp)
    with gs.Engine(n + 5, max_width=64, max_height=64, integer_based_sort=integer) as e:
        want_info = e.upload_ksplat(img, **kw)
        assert want_info == got_info
        want = _buffers(e, n, half_cov=half_cov, integer=integer, ncomp=ncomp)
    _compare(got, want, ambiguous, half_cov)
    return int(ambiguous.sum())


VARIANTS = [dict(integer=True, half_cov=False, xf=False), dict(integer=False, half_cov=True, xf=False),
            dict(integer=True, half_cov=True, xf=True), dict(integer=False, half_cov=False, xf=True)]


@pytest.mark.parametrize("variant", range(len(VARIANTS)))
@pytest.mark.parametrize("name", sorted(FH.fixture_files()))
def test_fixture_loads_like_level0_image(gs, name, variant):
    v = VARIANTS[variant]
    data = (Path(__file__).resolve().parent / "golden" / name).read_bytes()
    fmt = FO.SPLAT if name.endswith(".splat") else FO.PLY
    for deg in (0, 1, 2):
        _load_both(gs, fmt, data, deg, integer=v["integer"], half_cov=v["half_cov"], transform=_transform() if v["xf"] else None)


def _synthetic_ply(n, seed, *, nrest=45, odd=False):
    rng = np.random.default_rng(seed)
    props = [("x", "float"), ("y", "float"), ("z", "float"), ("nx", "float"), ("ny", "float"), ("nz", "float"),
             ("f_dc_0", "float"), ("f_dc_1", "float"), ("f_dc_2", "float")] + [(f"f_rest_{k}", "float") for k in range(nrest)] + \
            [("opacity", "float"), ("scale_0", "float"), ("scale_1", "float"), ("scale_2", "float")] + [(f"rot_{k}", "float") for k in range(4)]
    cols = {k: rng.uniform(-4, 4, n) for k in ("x", "y", "z")}
    cols.update({f"f_dc_{k}": rng.normal(0, 1, n) for k in range(3)})
    cols.update({f"f_rest_{k}": rng.normal(0, 0.2, n) for k in range(nrest)})
    cols.update(opacity=rng.normal(0, 3, n), **{f"scale_{k}": rng.uniform(-7, -2, n) for k in range(3)})
    cols.update({f"rot_{k}": rng.normal(0, 1, n) for k in range(4)})
    if odd:   # other scalar types and odd strides: uchar colour, short opacity, ushort / int extras, a double nobody reads
        props = [p for p in props if not p[0].startswith("f_dc")] + [("red", "uchar"), ("green", "uchar"), ("blue", "uchar"), ("tag", "ushort"),
                                                                   ("extra", "double"), ("id", "int")]
        props = [(k, "short") if k == "opacity" else (k, t) for k, t in props]
        cols.update(red=rng.integers(0, 256, n), green=rng.integers(0, 256, n), blue=rng.integers(0, 256, n), opacity=rng.integers(-9, 9, n),
                    tag=rng.integers(0, 65536, n), extra=rng.normal(0, 1, n), id=rng.integers(-2**31, 2**31, n))
        order = rng.permutation(len(props))
        props = [props[i] for i in order]
    return FO.write_ply(props, cols, n, comments=("synthetic",))


@pytest.mark.parametrize("variant", range(len(VARIANTS)))
def test_synthetic_files_load_like_level0_image(gs, variant):
    v = VARIANTS[variant]
    xf = _transform() if v["xf"] else None
    flagged = 0
    sh3 = _synthetic_ply(20011, 3)
    for deg in (0, 1, 2):
        flagged += _load_both(gs, FO.PLY, sh3, deg, integer=v["integer"], half_cov=v["half_cov"], transform=xf)
    for nrest in (0, 9, 24):
        flagged += _load_both(gs, FO.PLY, _synthetic_ply(5003, 4 + nrest, nrest=nrest, odd=True), 2, integer=v["integer"], half_cov=v["half_cov"], transform=xf)
    rng = np.random.default_rng(11)
    n = 30001
    splat = FO.write_splat(rng.uniform(-5, 5, (n, 3)), np.exp(rng.uniform(-6, -1, (n, 3))), rng.integers(0, 256, (n, 4)), rng.integers(0, 256, (n, 4)))
    assert _load_both(gs, FO.SPLAT, splat, 2, integer=v["integer"], half_cov=v["half_cov"], transform=xf) == 0
    print(f"flagged splats (exp rounding): {flagged}")


def test_large_file_spans_several_chunks(gs):
    """2.5 M SH3 splats (about 620 MB, a count that is not a multiple of 128) go through the 64 MiB staging chunks at least three times."""
    n = 2_500_037
    data = _synthetic_ply(n, 21)
    assert len(data) > 3 * (64 << 20)
    flagged = _load_both(gs, FO.PLY, data, 2)
    print(f"flagged splats (exp rounding): {flagged} of {n}")


def _viewer(w, h):
    from gaussiansplats3d_b200.scenes import CAMERAS
    from gaussiansplats3d_b200.viewer import Viewer
    c = CAMERAS["bonsai"]
    return Viewer(dict(cameraUp=c["up"], initialCameraPosition=c["position"], initialCameraLookAt=c["look_at"], width=w, height=h, sphericalHarmonicsDegree=2))


def test_viewer_frame_from_file_equals_frame_from_level0_image(gs, oracle_mod):
    from oracle import ksplat_oracle as KO
    data = _synthetic_ply(60000, 5)
    img, _ = FO.level0_image(FO.PLY, data, 2)
    w, h = 640, 360
    frames = {}
    N = gs._native
    for kind in ("file", "ksplat"):
        v = _viewer(w, h)
        info = v.addSplatSceneFromFile(data, FO.PLY) if kind == "file" else v.addSplatSceneFromKSplat(img)
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
    """Each malformed file comes back with its error, and the engine still renders the scene it had, bit for bit."""
    from gaussiansplats3d_b200.viewer import Viewer  # noqa: F401
    data = _synthetic_ply(20000, 6, nrest=9)
    w, h = 320, 200
    v = _viewer(w, h)
    v.addSplatSceneFromFile(data, FO.PLY)
    before = v.frame(frame_format=gs._native.GS_FRAME_RGBA32F, flip_y=False).copy()
    assert before.any()
    cases = dict(FH.MALFORMED)
    cases["capacity"] = (FO.PLY, _synthetic_ply(20001, 7, nrest=0), FH.CAPACITY, "capacity")
    for name, (fmt, blob, status, words) in cases.items():
        with pytest.raises(gs.GsError) as ei:
            v.engine.upload_file(fmt, blob, sh_degree=2)
        assert ei.value.code == status and words in str(ei.value), (name, str(ei.value))
        after = v.frame(frame_format=gs._native.GS_FRAME_RGBA32F, flip_y=False)
        assert np.array_equal(after, before), name
    v.dispose()
