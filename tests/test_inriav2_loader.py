"""CPU: the INRIA v2 (codebook) `.ply` loader's host half.  The oracle (tests/inriav2_oracle.py) reproduces the hand-derived level-0
records of every handmade fixture at every requested SH degree; the committed fixtures are current; gs_probe_file (no device needed)
reports every fixture's splat count and min(file, 2) SH degree, and rejects each malformed file with GS_ERR_BAD_ARG and a message
naming the problem.  The `exp` pages are enumerated over all 65536 halves for entries whose result depends on how `exp` rounds."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"
sys.path.insert(0, str(GOLDEN))
sys.path.insert(0, str(ROOT / "tests"))
import inriav2_handmade as H  # noqa: E402
import inriav2_oracle as O  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    from gaussiansplats3d_b200 import _native, build
    build.build()
    return _native.load()


@pytest.mark.parametrize("name", sorted(H.FIXTURES))
@pytest.mark.parametrize("sh_degree", [0, 1, 2])
def test_oracle_reproduces_handmade_records(name, sh_degree):
    rec, c64, sh, deg, nread, ambiguous = O.generator_inputs(H.fixture(name), sh_degree)
    assert deg == sh_degree and nread == [0, 9, 24][min(sh_degree, H.file_degree(name))]
    assert sh.shape == (len(H.FIXTURES[name]["splats"]), [0, 9, 24][sh_degree]) and not sh[:, nread:].any()
    assert not ambiguous.any()
    assert rec.tobytes() == H.expected_records(name, sh_degree)


def test_committed_fixtures_are_current():
    for fname, data in H.fixture_files().items():
        assert (GOLDEN / fname).read_bytes() == data, f"{fname} is stale: run python tests/golden/inriav2_handmade.py"


def test_fixtures_cover_the_quirks():
    rec = O.generator_inputs(H.fixture("sh0"))[0]
    assert rec[0, 24:40].view(np.float32).tolist() == [0, 0, 0, 1]                  # zero-length rotation
    assert rec[0, 40:44].tolist() == [128, 128, 128, 128]                           # Math.round(127.5) for dc and opacity
    rec = O.generator_inputs(H.fixture("absent_pages"))[0]
    assert (rec[2:, 12:24].view(np.float32) == 1).all() and (rec[2:, 40:44] == 128).all() and rec[1, 43] == 0
    rec = O.generator_inputs(H.fixture("absent_fields"))[0]
    assert (rec[:, 12:24].view(np.float32) == np.float32(0.01)).all() and (rec[:, 40:43] == 0).all()
    rec, _, sh, _, _, _ = O.generator_inputs(H.fixture("indices"), 1)
    assert np.isnan(sh[:4]).any() and (rec[:4, 24:40].view(np.uint32) == 0x7FC00000).any()   # invalid indices read NaN
    scale = rec[:, 12:24].view(np.float32)
    assert (scale[4] == 0).all() and (scale[7] == 0).all()                        # scale_0 names no row: all three 0
    assert scale[5, 1] == 0 and (scale[5, [0, 2]] > 0).all() and scale[6, 2] == 0 and (scale[6, :2] > 0).all()
    rec = O.generator_inputs(H.fixture("halves"))[0]
    bits = set(rec[:, 0:24].view(np.uint32).ravel().tolist())
    assert {0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0x33800000} <= bits    # centres and scales
    rec, _, sh, deg, nread, _ = O.generator_inputs(H.fixture("sh0"), 2)
    assert deg == 2 and nread == 0 and rec.shape[1] == 140 and not rec[:, 44:].any()      # a degree-0 file asked for degree 2


def test_flagged_halves():
    """How many of the 65536 halves give an f32 scale or an alpha byte that depends on how `exp` rounds (GPU tests skip those bytes)."""
    v = O.half(np.arange(1 << 16))
    scaling, opacity = O.flagged_halves(v)
    print(f"halves flagged for exp rounding: scaling {int(scaling.sum())} {np.nonzero(scaling)[0].tolist()}, opacity {int(opacity.sum())}")
    assert scaling.sum() == 0 and opacity.sum() == 0


def test_synthetic_generator_inputs():
    data = O.synthetic(5000, 3, rows=64, bad_index_rate=0.05)
    rec, c64, sh, deg, nread, amb = O.generator_inputs(data, 2)
    assert deg == 2 and nread == 24 and rec.shape == (5000, 140)
    assert np.isnan(sh).any() and np.isfinite(c64).all()


@pytest.mark.parametrize("name", sorted(H.FIXTURES))
def test_probe_reports_count_and_degree(lib, name):
    from gaussiansplats3d_b200 import Engine
    info = Engine.probe_file(H.PLY, H.fixture(name))
    assert info["splat_count"] == len(H.FIXTURES[name]["splats"]) and info["sh_degree"] == H.file_degree(name)
    assert info["compression_level"] == 0 and info["section_count"] == 1


@pytest.mark.parametrize("case", sorted(H.MALFORMED))
def test_probe_rejects_malformed(lib, case):
    from gaussiansplats3d_b200 import Engine, GsError
    data, words = H.MALFORMED[case]
    with pytest.raises(GsError) as ei:
        Engine.probe_file(H.PLY, data)
    assert ei.value.code == H.BAD_ARG
    msg = str(ei.value)
    assert "] .ply: INRIA v2 (codebook) .ply: " in msg and words in msg, msg
