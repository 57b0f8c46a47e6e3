"""CPU: the `.ply` / `.splat` loader's host half.  The oracle's restatement of the reference's progressive loader reproduces the
hand-derived level-0 records of every handmade fixture; the committed fixtures are current; gs_probe_file (no device needed) reports
every fixture's count and degree and rejects each malformed file with GS_ERR_BAD_ARG and a message naming the problem."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"
sys.path.insert(0, str(GOLDEN))
import file_handmade as FH  # noqa: E402

from oracle import file_oracle as FO  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    from gaussiansplats3d_b200 import _native, build
    build.build()
    return _native.load()


@pytest.mark.parametrize("name", sorted(FH.PLY_FIXTURES))
@pytest.mark.parametrize("sh_degree", [0, 1, 2])
def test_oracle_reproduces_handmade_ply_records(name, sh_degree):
    data, props, rows = FH.ply_fixture(name)
    want, deg = FH.expected_ply(props, rows, sh_degree)
    rec, got_deg, ambiguous = FO.level0_records(FO.PLY, data, sh_degree)
    assert got_deg == deg == min(sh_degree, FH.FILE_DEGREE[name])
    assert not ambiguous.any()
    assert rec.tobytes() == want


def test_oracle_reproduces_handmade_splat_records():
    data, rows = FH.splat_fixture()
    rec, deg, ambiguous = FO.level0_records(FO.SPLAT, data)
    assert deg == 0 and not ambiguous.any()
    assert rec.tobytes() == FH.expected_splat(rows)
    # the all-128 rotation is the zero quaternion: normalised to (0, 0, 0, 1), stored w, x, y, z
    assert rec[0, 24:40].view(np.float32).tolist() == [1.0, 0.0, 0.0, 0.0]


def test_level0_image_header():
    data, _, rows = FH.ply_fixture("sh3")
    img, _ = FO.level0_image(FO.PLY, data, 2)
    n = len(rows)
    assert len(img) == 4096 + 1024 + n * 140
    hdr = np.frombuffer(img[:4096], np.uint32)
    assert hdr[1:5].tolist() == [1, 1, n, n] and img[20] == 0
    assert np.frombuffer(img[4096 + 40: 4096 + 42], np.uint16)[0] == 2


def test_committed_fixtures_are_current():
    for name, data in FH.fixture_files().items():
        assert (GOLDEN / name).read_bytes() == data, f"{name} is stale: run python tests/golden/file_handmade.py"


def test_handmade_fixtures_cover_the_quirks():
    """uchar red/green/blue are read as u / 255 and written as floor(x 255): in f64 that gives u back for every byte."""
    data, props, rows = FH.ply_fixture("uchar_rgb")
    rec, _, _ = FO.level0_records(FO.PLY, data)
    assert rec[:, 40:43].tolist() == [[r["red"], r["green"], r["blue"]] for r in rows]
    assert rec[0, 24:40].view(np.float32).tolist() == [0.0, 0.0, 0.0, 1.0]         # zero quaternion
    assert (rec[:, 43] == 0).all()                                                    # no opacity property: alpha 0
    assert np.allclose(rec[:, 12:24].view(np.float32), np.float32(0.01))             # no scale properties: 0.01
    nf, _, _ = FO.level0_records(FO.PLY, FH.ply_fixture("nonfinite")[0], 1)
    assert nf[5, 40] == 255 and nf[5, 41] == 0                                        # colour clamped at both ends
    assert nf[0, 40] == 0 and nf[0, 43] == 0                                          # NaN colour / alpha -> 0
    assert nf[1, 43] == 255 and nf[2, 43] == 0


def test_oracle_ply_writer_matches_handmade_writer():
    _, props, rows = FH.ply_fixture("shuffled")
    cols = {n: np.array([r[n] for r in rows]) for n, _ in props}
    data = FO.write_ply(props, cols, len(rows))
    assert data == FH.ply_bytes(props, rows)


@pytest.mark.parametrize("name", sorted(FH.PLY_FIXTURES) + ["splat"])
def test_probe_reports_count_and_degree(lib, name):
    from gaussiansplats3d_b200 import Engine
    if name == "splat":
        data, rows = FH.splat_fixture()
        fmt, deg = FO.SPLAT, 0
    else:
        data, _, rows = FH.ply_fixture(name)
        fmt, deg = FO.PLY, FH.FILE_DEGREE[name]
    info = Engine.probe_file(fmt, data)
    assert info["splat_count"] == len(rows) and info["sh_degree"] == deg


@pytest.mark.parametrize("case", sorted(FH.MALFORMED))
def test_probe_rejects_malformed(lib, case):
    from gaussiansplats3d_b200 import Engine, GsError
    fmt, data, status, words = FH.MALFORMED[case]
    with pytest.raises(GsError) as ei:
        Engine.probe_file(fmt, data)
    assert ei.value.code == status
    assert words in str(ei.value), str(ei.value)


def test_probe_accepts_header_ending_near_eof(lib):
    """The reference throws when end_header lies within its last 100-byte read; the probe accepts any complete file."""
    from gaussiansplats3d_b200 import Engine
    data = FO.write_ply([("x", "float"), ("y", "float"), ("z", "float")] + [(f"rot_{k}", "float") for k in range(4)], {}, 1)
    assert Engine.probe_file(FO.PLY, data)["splat_count"] == 1


def test_probe_rejects_unknown_format(lib):
    from gaussiansplats3d_b200 import Engine, GsError
    with pytest.raises(GsError) as ei:
        Engine.probe_file(7, b"\0" * 64)
    assert ei.value.code == 1 and "format 7" in str(ei.value)


def test_scene_format_from_path():
    from gaussiansplats3d_b200.loaders import SceneFormat, sceneFormatFromPath
    assert sceneFormatFromPath("a/garden.ply") == SceneFormat.Ply == FO.PLY
    assert sceneFormatFromPath("bonsai.splat") == SceneFormat.Splat == FO.SPLAT
    assert sceneFormatFromPath("x.ksplat") == SceneFormat.KSplat
    assert sceneFormatFromPath("x.spz") is None and sceneFormatFromPath("x.obj") is None
