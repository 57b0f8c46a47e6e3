"""GPU: INRIA v2 (codebook) `.ply` files, which load only through SplatBufferGenerator.  gs_generate_splat_buffer's image is
byte-identical to oracle/generate_oracle.py fed with what tests/inriav2_oracle.py reads from the file (apart from bytes the oracle marks
as depending on how `exp` rounds); gs_upload_file_optimized leaves every engine buffer bit-identical to gs_upload_ksplat of that image;
gs_upload_file refuses the file and malformed files leave the previous scene; the Viewer and tools/create_ksplat.py load it."""
import importlib.util
import sys
from pathlib import Path

import numpy as np
import pytest

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE / "golden"))
sys.path.insert(0, str(HERE))
import inriav2_handmade as H  # noqa: E402
import inriav2_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = HERE / "golden"
PLY = 1
ROT_XF = [0.3, -0.5, 0.2, 0.7874007874011811]    # normalised quaternion x, y, z, w
VARIANTS = [dict(integer=True, half_cov=False, xf=False), dict(integer=False, half_cov=True, xf=False),
            dict(integer=True, half_cov=True, xf=True), dict(integer=False, half_cov=False, xf=True)]


def _transform():
    from gaussiansplats3d_b200 import three_math as TM
    return TM.compose((0.5, -1.25, 2.0), ROT_XF, (1.5, 0.75, 1.25))


def _buffers(e, n, *, half_cov, integer, ncomp, level):
    from gaussiansplats3d_b200 import _native as N
    out = dict(cc=e.read_buffer(N.GS_BUF_CENTERS_COLORS, np.uint32, 4 * n).reshape(n, 4),
               cov=e.read_buffer(N.GS_BUF_COVARIANCES, np.uint16 if half_cov else np.uint32, 6 * n).reshape(n, 6),
               centers=e.read_buffer(N.GS_BUF_CENTERS, np.int32 if integer else np.uint32, 4 * n).reshape(n, 4),
               ray=e.read_buffer(N.GS_BUF_RAY_RECORDS, np.uint8, 56 * n).reshape(n, 56))
    if ncomp:
        out["sh"] = e.read_buffer(N.GS_BUF_SH, np.uint8 if level == 2 else np.uint16, ncomp * n).reshape(n, ncomp)
    return out


def _check_image(data, sh_degree, **kw):
    from gaussiansplats3d_b200.engine import generate_splat_buffer
    got = generate_splat_buffer(PLY, data, sh_degree=sh_degree, **kw)
    want, loose = O.image(data, sh_degree, level=kw.get("compression_level", 1), minimum_alpha=kw.get("minimum_alpha", 1),
                          section_size=kw.get("section_size", 0), scene_center=kw.get("scene_center", (0.0, 0.0, 0.0)),
                          block_size=kw.get("block_size", 5.0), bucket_size=kw.get("bucket_size", 256))
    assert len(got) == len(want)
    diff = np.nonzero((np.frombuffer(got, np.uint8) != np.frombuffer(want, np.uint8)) & ~loose)[0]
    assert diff.size == 0, f"{diff.size} bytes differ, first at {diff[:8]}"
    return got


@pytest.mark.parametrize("name", sorted(H.FIXTURES))
def test_fixture_images_match_generate_oracle(gs, name):
    data = (GOLDEN / H.file_name(name)).read_bytes()
    for level in (0, 1, 2):
        for deg in (0, 1, 2):
            for alpha in (0, 1, 128):
                _check_image(data, deg, compression_level=level, minimum_alpha=alpha)


@pytest.mark.parametrize("index_type", ["uchar", "short", "int"])
def test_synthetic_images_match_generate_oracle(gs, index_type):
    """Seeded SH3 files with 5 % invalid indices, read at degrees 0, 1 and 2, several sections and a small bucket size."""
    data = O.synthetic(60_011, 12, rows=300 if index_type != "uchar" else 256, index_type=index_type,
                       bad_index_rate=0.05 if index_type != "uchar" else 0.0)
    for level in (0, 1, 2):
        for deg in (0, 1, 2):
            _check_image(data, deg, compression_level=level, section_size=25_000, bucket_size=64)
    _check_image(O.synthetic(20_003, 4, sh_rest=0), 2, compression_level=2, minimum_alpha=128, block_size=1.5, scene_center=(1.0, -2.0, 0.5))


def test_large_file_spans_several_chunks(gs):
    """About 1.2 M SH3 splats of 62 bytes: the splat rows take two 64 MiB staging chunks."""
    n = 1_200_007
    data = O.synthetic(n, 21)
    assert n * 62 > (64 << 20)
    _check_image(data, 2, compression_level=0)


@pytest.mark.parametrize("level", [0, 1, 2])
def test_optimized_load_equals_ksplat_of_generated_image(gs, level):
    data = O.synthetic(50_021, 8, rows=200, index_type="short", bad_index_rate=0.02)
    for v in VARIANTS:
        for deg in (1, 2):
            img = _check_image(data, deg, compression_level=level, minimum_alpha=5)
            kw = dict(half_covariances=v["half_cov"], transform16=_transform() if v["xf"] else None)
            cfg = dict(max_width=64, max_height=64, integer_based_sort=v["integer"], ray_records=True)
            with gs.Engine(50_100, **cfg) as e:
                info = e.upload_file_optimized(PLY, data, sh_degree=deg, compression_level=level, minimum_alpha=5, **kw)
                n = info["splat_count"]
                assert info["sh_degree"] == deg
                got = _buffers(e, n, half_cov=v["half_cov"], integer=v["integer"], ncomp=[0, 9, 24][deg], level=level)
            with gs.Engine(50_100, **cfg) as e:
                assert e.upload_ksplat(img, **kw) == info
                want = _buffers(e, n, half_cov=v["half_cov"], integer=v["integer"], ncomp=[0, 9, 24][deg], level=level)
            assert 0 < n < 50_021
            for k in got:
                assert np.array_equal(got[k], want[k]), (k, v, deg)


def test_degree0_file_asked_for_degree2(gs):
    """The image carries degree 2 with every coefficient 0 and the default +-1.5 range."""
    from gaussiansplats3d_b200.engine import generate_splat_buffer
    data = H.fixture("sh0")
    img = _check_image(data, 2, compression_level=2)
    assert np.frombuffer(img, np.float32, 2, 36).tolist() == [-1.5, 1.5]
    assert np.frombuffer(img, np.uint16, 1, 4096 + 40)[0] == 2
    assert generate_splat_buffer(PLY, data, sh_degree=0) != generate_splat_buffer(PLY, data, sh_degree=2)


def _viewer(w, h, **extra):
    from gaussiansplats3d_b200.scenes import CAMERAS
    from gaussiansplats3d_b200.viewer import Viewer
    c = CAMERAS["bonsai"]
    return Viewer(dict(cameraUp=c["up"], initialCameraPosition=c["position"], initialCameraLookAt=c["look_at"], width=w, height=h,
                       sphericalHarmonicsDegree=2, **extra))


def test_viewer_loads_v2_through_the_generator(gs):
    """addSplatSceneFromFile(v2, Ply, progressiveLoad=False) renders the generator's .ksplat frame; progressive or with
    optimizeSplatData off it raises the library's message."""
    from gaussiansplats3d_b200.engine import generate_splat_buffer
    from gaussiansplats3d_b200.loaders import SceneFormat
    data = O.synthetic(60_013, 6)
    img = generate_splat_buffer(PLY, data, sh_degree=2, compression_level=0, minimum_alpha=1)
    frames = []
    for kind in ("ksplat", "file"):
        v = _viewer(640, 360)
        info = v.addSplatSceneFromKSplat(img) if kind == "ksplat" else v.addSplatSceneFromFile(data, SceneFormat.Ply, progressiveLoad=False)
        frames.append((info["splat_count"], v.frame(frame_format=gs._native.GS_FRAME_RGBA32F, flip_y=False).copy()))
        v.dispose()
    assert frames[0][0] == frames[1][0] and 0 < frames[0][0] <= 60_013
    assert frames[0][1].any() and np.array_equal(frames[0][1], frames[1][1])
    for optimize, progressive in ((True, True), (False, False), (False, True)):
        v = _viewer(64, 64, optimizeSplatData=optimize)
        with pytest.raises(gs.GsError) as ei:
            v.addSplatSceneFromFile(data, SceneFormat.Ply, progressiveLoad=progressive)
        assert ei.value.code == H.BAD_ARG and "loads only through the generator" in str(ei.value)
        v.dispose()


def test_upload_file_refuses_and_malformed_files_leave_previous_scene(gs):
    """gs_upload_file refuses a valid v2 file; each malformed file comes back with its error from both uploads; the engine still
    renders the scene it had, bit for bit."""
    v = _viewer(320, 200)
    v.addSplatSceneFromFile(O.synthetic(20_000, 9, sh_rest=9), 1, progressiveLoad=False)
    before = v.frame(frame_format=gs._native.GS_FRAME_RGBA32F, flip_y=False).copy()
    assert before.any()
    cases = [(v.engine.upload_file, H.fixture(name), H.BAD_ARG, "loads only through the generator") for name in ("sh2", "empty")]
    for blob, words in H.MALFORMED.values():
        cases += [(up, blob, H.BAD_ARG, words) for up in (v.engine.upload_file, v.engine.upload_file_optimized)]
    big = O.synthetic(20_001, 10, sh_rest=0)
    cases.append((v.engine.upload_file_optimized, big, 7, "capacity"))
    cases.append((v.engine.upload_file, big, H.BAD_ARG, "loads only through the generator"))   # refused before the capacity check
    for upload, blob, status, words in cases:
        with pytest.raises(gs.GsError) as ei:
            upload(PLY, blob, sh_degree=2)
        assert ei.value.code == status and words in str(ei.value), str(ei.value)
        after = v.frame(frame_format=gs._native.GS_FRAME_RGBA32F, flip_y=False)
        assert np.array_equal(after, before), words
    v.dispose()


def test_create_ksplat_converts_v2(gs, tmp_path):
    spec = importlib.util.spec_from_file_location("create_ksplat", HERE.parent / "tools" / "create_ksplat.py")
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    src, dst = tmp_path / "scene.ply", tmp_path / "scene.ksplat"
    src.write_bytes(H.fixture("sh3"))
    assert tool.main([str(src), str(dst), "2", "1", "0.5,0,-1", "2.0", "4", "2"]) == 0
    want, loose = O.image(H.fixture("sh3"), 2, level=2, minimum_alpha=1, scene_center=(0.5, 0.0, -1.0), block_size=2.0, bucket_size=4)
    assert not loose.any() and dst.read_bytes() == want
    assert tool.main([str(src), str(dst)]) == 0
    assert dst.read_bytes() == O.image(H.fixture("sh3"), 0)[0]
