"""CPU: the `.spz` loader's host half.  The oracle (tests/spz_oracle.py) reproduces the hand-derived level-0 records of every handmade
fixture; the committed fixtures are current; gs_probe_file (no device needed) reports every fixture's count and degree and rejects
each malformed packed stream, and a stream still gzipped, with GS_ERR_BAD_ARG and a message naming the problem."""
import gzip
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"
sys.path.insert(0, str(GOLDEN))
import spz_handmade as SH  # noqa: E402
import spz_oracle as SO  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    from gaussiansplats3d_b200 import _native, build
    build.build()
    return _native.load()


@pytest.mark.parametrize("name", sorted(SH.FIXTURES))
@pytest.mark.parametrize("sh_degree", [0, 1, 2])
def test_oracle_reproduces_handmade_records(name, sh_degree):
    want, deg = SH.expected_records(name, sh_degree)
    rec, got_deg, ambiguous = SO.level0_records(SH.packed_fixture(name), sh_degree)
    assert got_deg == deg == min(sh_degree, SH.header_kw(name)["sh_degree"])
    assert not ambiguous.any()
    assert rec.tobytes() == want


def test_committed_fixtures_are_current():
    for name in SH.FIXTURES:
        data = (GOLDEN / SH.file_name(name)).read_bytes()
        assert gzip.decompress(data) == SH.packed_fixture(name), f"{name} is stale: run python tests/golden/spz_handmade.py"


def test_fixtures_cover_the_quirks():
    rec, _, _ = SO.level0_records(SH.packed_fixture("sh0"))
    c = rec[:, 0:12].view(np.float32)
    assert c[0].tolist() == [0.0, 0x7FFFFF / 4096, -0x800000 / 4096] and c[1, 0] == -1 / 4096      # the 24-bit sign boundary
    q = rec[:, 24:40].view(np.float32)
    assert q[1, 0] == 0 and q[4, 0] == 0                                                           # w = sqrt(max(0, 1 - 3)) = 0
    assert np.allclose(np.linalg.norm(q.astype(np.float64), axis=1), 1, atol=1e-6)
    assert rec[0, 40:44].tolist() == [0, 128, 255, 255] and rec[1, 40:44].tolist() == [255, 0, 75, 0]  # colour clamps, raw alpha
    assert rec[4, 40:43].tolist() == [0, 255, 126]                                                 # bytes 1 and 254 clamp too
    fb = {k: SO.level0_records(SH.packed_fixture(f"fb{k}"))[0][:, 0:12].view(np.float32) for k in (0, 31, 32, 33)}
    assert np.array_equal(fb[0], fb[32]) and np.array_equal(fb[33], fb[0] * np.float32(0.5))                  # 1 << 32 = 1, 1 << 33 = 2
    assert np.array_equal(fb[31], fb[0] * np.float32(-2.0 ** -31))                                    # 1 << 31 = -2^31
    v1 = SO.level0_records(SH.packed_fixture("v1"))[0][:, 0:12].view(np.uint32)
    assert {0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0x33800000} <= set(v1.ravel().tolist())   # 2^-24: a subnormal half
    sh = SO.level0_records(SH.packed_fixture("sh3"), 2)[0][:, 44:].view(np.float32)
    assert (sh[0] == 0).all() and (sh[1] == -1).all() and (sh[2] == 127 / 128).all()


def test_flagged_scale_bytes():
    """How many of the 256 scale bytes give an f32 scale that depends on how `exp` rounds."""
    flagged = SO.flagged_scale_bytes()
    print(f"scale bytes flagged for exp rounding: {int(flagged.sum())} of 256")
    assert flagged.sum() < 8


def test_quantizer_round_trips():
    rng = np.random.default_rng(0)
    n = 700
    centers = rng.uniform(-3, 3, (n, 3))
    log_scales = rng.uniform(-6, -2, (n, 3))
    quats = rng.normal(0, 1, (n, 4))
    rgba = rng.uniform(0.2, 0.8, (n, 4))
    sh = rng.normal(0, 0.3, (n, 3, 15)).clip(-0.99, 0.99)
    data = SO.quantize(centers, log_scales, quats, rgba, sh, sh_degree=3, compress=True)
    rec, deg, _ = SO.level0_records(data, 2)
    assert deg == 2
    assert np.abs(rec[:, 0:12].view(np.float32) - centers).max() <= 0.5 / 4096 + 1e-7
    assert np.abs(np.log(rec[:, 12:24].view(np.float32)) - log_scales).max() <= 1 / 32 + 1e-6
    q = rec[:, 24:40].view(np.float32).astype(np.float64)[:, [1, 2, 3, 0]]
    qn = quats / np.linalg.norm(quats, axis=1, keepdims=True)
    assert np.abs(np.abs((q * qn).sum(1)) - 1).max() < 1e-2                        # 8-bit x, y, z
    assert np.abs(rec[:, 40:43] / 255 - rgba[:, :3]).max() < 3 / 255
    assert np.abs(rec[:, 44:80].view(np.float32) - sh[:, :, :3].reshape(n, 9)).max() <= 0.5 / 128 + 1e-7


def test_decompress_gzipped_and_scene_format():
    from gaussiansplats3d_b200.loaders import SceneFormat, decompressGzipped
    assert SceneFormat.Spz == 4 and SceneFormat.KSplat == 3
    data = SH.packed_fixture("sh2")
    assert decompressGzipped(gzip.compress(data)) == data


@pytest.mark.parametrize("name", sorted(SH.FIXTURES))
def test_probe_reports_count_and_degree(lib, name):
    from gaussiansplats3d_b200 import Engine
    info = Engine.probe_file(SH.SPZ, SH.packed_fixture(name))
    assert info["splat_count"] == len(SH.FIXTURES[name][0]) and info["sh_degree"] == min(SH.header_kw(name)["sh_degree"], 2)
    assert info["compression_level"] == 0 and info["section_count"] == 1


@pytest.mark.parametrize("case", sorted(SH.MALFORMED))
def test_probe_rejects_malformed(lib, case):
    from gaussiansplats3d_b200 import Engine, GsError
    data, words = SH.MALFORMED[case]
    with pytest.raises(GsError) as ei:
        Engine.probe_file(SH.SPZ, data)
    assert ei.value.code == SH.BAD_ARG
    msg = str(ei.value)
    assert ".spz: " in msg and words in msg, msg


def test_unknown_format_names_spz(lib):
    from gaussiansplats3d_b200 import Engine, GsError
    with pytest.raises(GsError) as ei:
        Engine.probe_file(5, SH.packed_fixture("sh0"))
    assert "GS_FILE_SPZ = 4" in str(ei.value)
