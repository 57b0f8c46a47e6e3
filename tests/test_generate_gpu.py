"""GPU: gs_generate_splat_buffer's .ksplat image is byte-identical to oracle/generate_oracle.py's, and gs_upload_file_optimized leaves
every engine buffer bit-identical to gs_upload_ksplat of that image."""
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent / "golden"))
import file_handmade as FH  # noqa: E402
import generate_handmade as GH  # noqa: E402
import pcply_handmade as PH  # noqa: E402

from oracle import file_oracle as FO  # noqa: E402
from oracle import generate_oracle as GO  # noqa: E402
from oracle import pcply_oracle as PC  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden"


def _check_image(gs, fmt, data, sh_degree, **kw):
    """-> number of splats flagged for libm exp rounding.  Their own scale and alpha bytes may differ; every other byte must not.  A
    flagged splat must not sit at the alpha threshold, where a flip would change which splats are kept and move the whole layout."""
    from gaussiansplats3d_b200.engine import generate_splat_buffer
    rec, c64, sh, deg, amb = GO.generator_inputs(fmt, data, sh_degree)
    alpha = kw.get("minimum_alpha", 1)
    a = rec[amb, 43].astype(int)
    assert not ((a == alpha) | (a == alpha - 1)).any(), "a flagged splat sits at the alpha threshold"
    got = generate_splat_buffer(fmt, data, sh_degree=sh_degree, **kw)
    want, loose = GO.generate(rec, c64, sh, deg, level=kw.get("compression_level", 1), minimum_alpha=alpha,
                              section_size=kw.get("section_size", 0), scene_center=kw.get("scene_center", (0.0, 0.0, 0.0)),
                              block_size=kw.get("block_size", 5.0), bucket_size=kw.get("bucket_size", 256), loose=amb)
    assert len(got) == len(want)
    diff = np.nonzero((np.frombuffer(got, np.uint8) != np.frombuffer(want, np.uint8)) & ~loose)[0]
    assert diff.size == 0, f"{diff.size} bytes differ, first at {diff[:8]}"
    return int(amb.sum())


@pytest.mark.parametrize("case", range(len(GH.cases())))
def test_hand_derived_images(gs, case):
    from gaussiansplats3d_b200.engine import generate_splat_buffer
    name, data, kw, want = GH.cases()[case]
    assert generate_splat_buffer(FO.SPLAT, data, **kw) == want, name


@pytest.mark.parametrize("name", sorted(PH.fixture_files()))
def test_compressed_fixture_images_match_oracle(gs, name):
    data = PH.fixture_files()[name]
    for level in (0, 1, 2):
        for deg in (0, 1, 2):
            _check_image(gs, FO.PLY, data, deg, compression_level=level, minimum_alpha=1)


@pytest.mark.parametrize("name", sorted(FH.fixture_files()))
def test_fixture_images_match_oracle(gs, name):
    data = (GOLDEN / name).read_bytes()
    fmt = FO.SPLAT if name.endswith(".splat") else FO.PLY
    for level in (0, 1, 2):
        for deg in (0, 1, 2):
            for alpha in (0, 1, 128):
                _check_image(gs, fmt, data, deg, compression_level=level, minimum_alpha=alpha)


def _synthetic_ply(n, seed):
    rng = np.random.default_rng(seed)
    props = [("x", "float"), ("y", "float"), ("z", "float")] + [(f"f_rest_{k}", "float") for k in range(45)] + \
            [("opacity", "float")] + [(f"scale_{k}", "float") for k in range(3)] + [(f"rot_{k}", "float") for k in range(4)] + \
            [(f"f_dc_{k}", "float") for k in range(3)]
    cols = {k: rng.normal(0, 6, n).astype(np.float32) for k in ("x", "y", "z")}
    cols["x"][7] = 3e5                                                  # a floater: its bucket id passes 2^32 - 2
    cols.update({f"f_rest_{k}": rng.normal(0, 0.3, n) for k in range(45)})
    cols.update(opacity=rng.normal(0, 3, n), **{f"scale_{k}": rng.uniform(-6, -2, n) for k in range(3)})
    cols.update({f"rot_{k}": rng.normal(0, 1, n) for k in range(4)}, **{f"f_dc_{k}": rng.normal(0, 1, n) for k in range(3)})
    return FO.write_ply(props, cols, n)


def _synthetic_pcply(n, seed):
    rng = np.random.default_rng(seed)
    centers = rng.normal(0, 6, (n, 3))
    centers[5] = (4e5, 0.0, 0.0)                                        # a floater
    q = rng.normal(0, 1, (n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    return PC.quantize(centers, rng.uniform(-6, -2, (n, 3)), q, rng.uniform(0, 1, (n, 4)), rng.uniform(-1, 1, (n, 45)))


def test_synthetic_compressed_images_match_oracle(gs):
    data = _synthetic_pcply(400_128, 12)
    for level in (0, 1, 2):
        _check_image(gs, FO.PLY, data, 2, compression_level=level, section_size=150_000, bucket_size=64)


def test_million_splat_file_matches_oracle(gs):
    rng = np.random.default_rng(21)
    n = 1_000_003
    c = rng.normal(0, 10, (n, 3))
    c[3] = (0.0, 9e5, 0.0)
    splat = FO.write_splat(c, np.exp(rng.uniform(-6, -1, (n, 3))), rng.integers(0, 256, (n, 4)), rng.integers(0, 256, (n, 4)))
    assert _check_image(gs, FO.SPLAT, splat, 0, compression_level=1, section_size=400_000) == 0


def test_synthetic_images_match_oracle(gs):
    ply = _synthetic_ply(200_003, 5)
    flagged = 0
    for level in (0, 1, 2):
        flagged += _check_image(gs, FO.PLY, ply, 2, compression_level=level)
        flagged += _check_image(gs, FO.PLY, ply, 1, compression_level=level, section_size=70_000, minimum_alpha=20, bucket_size=100,
                                block_size=1.5, scene_center=(1.0, -2.0, 0.5))
    rng = np.random.default_rng(9)
    n = 300_001
    splat = FO.write_splat(rng.normal(0, 8, (n, 3)), np.exp(rng.uniform(-6, -1, (n, 3))), rng.integers(0, 256, (n, 4)), rng.integers(0, 256, (n, 4)))
    for level in (0, 1, 2):
        assert _check_image(gs, FO.SPLAT, splat, 0, compression_level=level, section_size=100_000) == 0
    print(f"flagged .ply splats (exp rounding, allowed in their own scale and alpha bytes): {flagged}")


def _buffers(e, n, *, half_cov, integer, ncomp, level):
    from gaussiansplats3d_b200 import _native as N
    out = dict(cc=e.read_buffer(N.GS_BUF_CENTERS_COLORS, np.uint32, 4 * n),
               cov=e.read_buffer(N.GS_BUF_COVARIANCES, np.uint16 if half_cov else np.uint32, 6 * n),
               centers=e.read_buffer(N.GS_BUF_CENTERS, np.int32 if integer else np.uint32, 4 * n),
               ray=e.read_buffer(N.GS_BUF_RAY_RECORDS, np.uint8, 56 * n))
    if ncomp:
        out["sh"] = e.read_buffer(N.GS_BUF_SH, np.uint8 if level == 2 else np.uint16, ncomp * n)
    return out


@pytest.mark.parametrize("level", [0, 1, 2])
@pytest.mark.parametrize("variant", [dict(integer=True, half_cov=False, xf=None), dict(integer=False, half_cov=True, xf="rot")])
def test_optimized_load_equals_ksplat_of_generated_image(gs, level, variant):
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.engine import generate_splat_buffer
    data = _synthetic_ply(50_021, 8)
    xf = TM.compose((0.5, -1.25, 2.0), [0.3, -0.5, 0.2, 0.7874007874011811], (1.5, 0.75, 1.25)) if variant["xf"] else None
    img = generate_splat_buffer(FO.PLY, data, sh_degree=2, compression_level=level, minimum_alpha=5)
    kw = dict(half_covariances=variant["half_cov"], transform16=xf, minimum_alpha=5)
    cfg = dict(max_width=64, max_height=64, integer_based_sort=variant["integer"], ray_records=True)
    with gs.Engine(50_100, **cfg) as e:
        info = e.upload_file_optimized(FO.PLY, data, sh_degree=2, compression_level=level, **kw)
        n = info["splat_count"]
        got = _buffers(e, n, half_cov=variant["half_cov"], integer=variant["integer"], ncomp=24, level=level)
    with gs.Engine(50_100, **cfg) as e:
        assert e.upload_ksplat(img, **kw) == info
        want = _buffers(e, n, half_cov=variant["half_cov"], integer=variant["integer"], ncomp=24, level=level)
    assert 0 < n < 50_021
    for k in got:
        assert np.array_equal(got[k], want[k]), k


def test_bad_options_and_capacity(gs):
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.engine import generate_splat_buffer
    data = (GOLDEN / "file_handmade_sh1.ply").read_bytes()
    for kw in (dict(compression_level=3), dict(block_size=-1.0), dict(block_size=float("nan")), dict(bucket_size=2**31 + 1)):
        with pytest.raises(N.GsError) as ei:
            generate_splat_buffer(FO.PLY, data, **kw)
        assert ei.value.code == N.GS_ERR_BAD_ARG
    n = FO.parse_ply_header(data)["count"]
    with gs.Engine(max(n - 1, 1), max_width=64, max_height=64) as e:
        with pytest.raises(N.GsError) as ei:
            e.upload_file_optimized(FO.PLY, data)
        assert ei.value.code == N.GS_ERR_CAPACITY


def test_repeated_generation_does_not_leak_device_memory(gs):
    import torch
    from gaussiansplats3d_b200.engine import generate_splat_buffer
    data = _synthetic_ply(100_003, 3)
    generate_splat_buffer(FO.PLY, data, sh_degree=2)
    with gs.Engine(100_100, max_width=64, max_height=64) as e:
        e.upload_file_optimized(FO.PLY, data, sh_degree=2)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info(0)[0]
        for _ in range(3):
            generate_splat_buffer(FO.PLY, data, sh_degree=2, compression_level=2)
            e.upload_file_optimized(FO.PLY, data, sh_degree=2)
        torch.cuda.synchronize()
        free1 = torch.cuda.mem_get_info(0)[0]
    # one generation holds about 600 B per splat (60 MB here); what stays behind must be far less than one generation
    assert free0 - free1 < 8 << 20, f"{(free0 - free1) / 2**20:.1f} MiB not returned"


def _viewer(w, h, **extra):
    from gaussiansplats3d_b200.scenes import CAMERAS
    from gaussiansplats3d_b200.viewer import Viewer
    c = CAMERAS["bonsai"]
    return Viewer(dict(cameraUp=c["up"], initialCameraPosition=c["position"], initialCameraLookAt=c["look_at"], width=w, height=h,
                       sphericalHarmonicsDegree=2, raycast=True, **extra))


@pytest.mark.parametrize("level", [0, 2])
def test_viewer_default_load_equals_generated_ksplat(gs, level):
    from gaussiansplats3d_b200.engine import generate_splat_buffer
    data = _synthetic_ply(60_013, 6)
    img = generate_splat_buffer(FO.PLY, data, sh_degree=2, compression_level=level, minimum_alpha=1)
    w, h = 640, 360
    got = {}
    for kind in ("file", "ksplat", "progressive"):
        v = _viewer(w, h, inMemoryCompressionLevel=level)
        if kind == "file":
            info = v.addSplatSceneFromFile(data, FO.PLY, progressiveLoad=False)
        elif kind == "progressive":
            info = v.addSplatSceneFromFile(data, FO.PLY)
        else:
            info = v.addSplatSceneFromKSplat(img)
        frame = v.frame(frame_format=gs._native.GS_FRAME_RGBA32F, flip_y=False).copy()
        hits = []
        for y in range(0, h, 24):   # a grid of rays: each one's nearest hits as (splat index, distance, point)
            for x in range(0, w, 24):
                v.raycaster.setFromCameraAndScreenPosition(v.camera, (x, y), (w, h))
                hits.append([(r.splatIndex, r.distance, *r.origin.tolist()) for r in v.raycaster.intersectSplatMesh(v.splatMesh, capacity=4)])
        got[kind] = (info["splat_count"], frame, hits)
        v.dispose()
    assert got["file"][0] == got["ksplat"][0] < 60_013 == got["progressive"][0]
    assert np.array_equal(got["file"][1], got["ksplat"][1]) and got["file"][1].any()
    assert got["file"][2] == got["ksplat"][2]
    assert sum(map(len, got["file"][2])) > 0
