"""CPU: the PlayCanvas-compressed `.ply` loader's host half.  The oracle reproduces the hand-derived level-0 records of every handmade
fixture; the committed fixtures are current; gs_probe_file (no device needed) reports every fixture's count and degree and rejects each
malformed compressed file with GS_ERR_BAD_ARG and a message naming the problem."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"
sys.path.insert(0, str(GOLDEN))
import pcply_handmade as PH  # noqa: E402

from oracle import pcply_oracle as PO  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    from gaussiansplats3d_b200 import _native, build
    build.build()
    return _native.load()


@pytest.mark.parametrize("name", sorted(PH.PC_FIXTURES))
@pytest.mark.parametrize("sh_degree", [0, 1, 2])
def test_oracle_reproduces_handmade_records(name, sh_degree):
    data, _ = PH.pc_fixture(name)
    want, deg = PH.expected_records(name, sh_degree)
    rec, got_deg, ambiguous = PO.level0_records(data, sh_degree)
    assert got_deg == deg == min(sh_degree, PH.FILE_DEGREE[name])
    assert not ambiguous.any()
    assert rec.tobytes() == want


def test_committed_fixtures_are_current():
    for name, data in PH.fixture_files().items():
        assert (GOLDEN / name).read_bytes() == data, f"{name} is stale: run python tests/golden/pcply_handmade.py"


def test_edge_fixture_covers_the_quirks():
    rec, _, _ = PO.level0_records(PH.pc_fixture("edges")[0])
    q = rec[:, 24:40].view(np.float32)
    slots = [int(np.argmax(np.abs(q[s]))) for s in range(4)]
    assert slots == [0, 1, 2, 3]                                                      # m lands in x, y, z, w
    assert (rec[4:8, 24:40].view(np.uint32) == 0x7FC00000).all()                      # a² + b² + c² > 1: canonical NaN
    assert rec[8, 40:44].tolist() == [128, 0, 255, 128]                               # 127.5 rounds up; clamps at 0 and 255
    assert rec[9, 40:43].tolist() == [191, 0, 255]
    c = rec[256:, 0:12].view(np.uint32)
    assert (c[:, 0] == 0x7FC00000).all()                                              # NaN min_x
    assert c[0, 1] == 0x7FC00000 and c[1, 1] == 0x7F800000                            # inf * 0 in the lerp; inf
    assert 0.00196078431372549 * 255 == 0.5 and 0.00588235294117647 * 255 == 1.5 - 2 ** -52
    assert rec[258, 42] == 1 and rec[259, 42] == 1                                    # Math.round(0.5) = 1 (not half-even 0)
    s = rec[256:258, 12:24].view(np.float32)
    assert s[0, 0] == 0 and s[1, 0] == np.inf and (s[:, 1] == 0).all()                # `|| 0` of NaN; exp(inf); NaN min_scale_y


def test_quantizer_round_trips():
    """The realistic writer packs float splats that the oracle decodes back within the format's quantisation."""
    rng = np.random.default_rng(0)
    n = 700
    centers = rng.uniform(-3, 3, (n, 3))
    log_scales = rng.uniform(-6, -2, (n, 3))
    quats = rng.normal(0, 1, (n, 4))
    rgba = rng.uniform(0, 1, (n, 4))
    sh = rng.normal(0, 0.3, (n, 45))
    data = PO.quantize(centers, log_scales, quats, rgba, sh)
    rec, deg, _ = PO.level0_records(data, 2)
    assert deg == 2
    assert np.abs(rec[:, 0:12].view(np.float32) - centers).max() < 6 / 1023
    q = rec[:, 24:40].view(np.float32).astype(np.float64)
    qn = quats / np.linalg.norm(quats, axis=1, keepdims=True)
    assert np.abs(np.abs((q * qn).sum(1)) - 1).max() < 1e-4 and not np.isnan(q).any()
    assert np.abs(rec[:, 40:43] / 255 - rgba[:, :3]).max() < 2 / 255
    assert np.abs(rec[:, 44:80].view(np.float32) - sh[:, [0, 1, 2, 15, 16, 17, 30, 31, 32]]).max() < 4.1 / 255


@pytest.mark.parametrize("name", sorted(PH.PC_FIXTURES))
def test_probe_reports_count_and_degree(lib, name):
    from gaussiansplats3d_b200 import Engine
    data, d = PH.pc_fixture(name)
    info = Engine.probe_file(PH.PLY, data)
    assert info["splat_count"] == len(d["vertex_rows"]) and info["sh_degree"] == PH.FILE_DEGREE[name]
    assert info["compression_level"] == 0 and info["section_count"] == 1


@pytest.mark.parametrize("case", sorted(PH.MALFORMED))
def test_probe_rejects_malformed(lib, case):
    from gaussiansplats3d_b200 import Engine, GsError
    data, words = PH.MALFORMED[case]
    with pytest.raises(GsError) as ei:
        Engine.probe_file(PH.PLY, data)
    assert ei.value.code == PH.BAD_ARG
    msg = str(ei.value)
    assert PH.PREFIX in msg and words in msg, msg


def test_probe_accepts_trailing_bytes(lib):
    from gaussiansplats3d_b200 import Engine
    rng = np.random.default_rng(1)
    data = PO.quantize(rng.uniform(-1, 1, (10, 3)), rng.uniform(-5, -3, (10, 3)), rng.normal(0, 1, (10, 4)), rng.uniform(0, 1, (10, 4)))
    assert Engine.probe_file(PH.PLY, data + b"\0" * 100)["splat_count"] == 10
