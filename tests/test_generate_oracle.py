"""CPU: oracle/generate_oracle.py, the restatement of SplatBufferGenerator.getStandardGenerator, against hand-derived cases and a round
trip through the existing .ksplat oracle."""
import math
import struct
import sys
from pathlib import Path

import numpy as np
import pytest

from oracle import file_oracle as FO
from oracle import generate_oracle as GO
from oracle import ksplat_oracle as KO

sys.path.insert(0, str(Path(__file__).resolve().parent / "golden"))
import generate_handmade as GH  # noqa: E402


@pytest.mark.parametrize("case", range(len(GH.cases())))
def test_oracle_reproduces_hand_derived_images(case):
    name, data, kw, want = GH.cases()[case]
    rec, c64, sh, deg, _ = GO.generator_inputs(FO.SPLAT, data, 0)
    got = GO.generate(rec, c64, sh, deg, level=kw["compression_level"], minimum_alpha=kw["minimum_alpha"], block_size=kw["block_size"],
                      bucket_size=kw["bucket_size"])
    assert got == want, name


def test_flagged_bytes_mask_covers_scale_and_alpha():
    data = GH.splat_file()
    rec, c64, sh, deg, _ = GO.generator_inputs(FO.SPLAT, data, 0)
    loose = np.zeros(7, bool)
    loose[GH.FILE_ORDER.index("P0")] = True
    img, mask = GO.generate(rec, c64, sh, deg, level=1, block_size=1.0, bucket_size=2, loose=loose)
    base = 4096 + 1024 + 12 + 60 + 24 * GH.OUT_ORDER.index("P0")   # partial lengths, bucket centres, then records
    assert np.nonzero(mask)[0].tolist() == list(range(base + 6, base + 12)) + [base + 23]


def test_sh_range_zero_quirk_and_frc23():
    # `!min || v < min`: a running 0 is replaced by the next value, whatever it is
    assert GO.sh_range([[0.0, 0.5, 0.25]]) == (0.25, 0.5)
    assert GO.sh_range([[-1.0, 0.0, 2.0]]) == (-1.0, 2.0)          # max: -1 -> 0 (falsy) -> 2
    assert GO.sh_range([[2.0, 0.0, 1.0]]) == (1.0, 2.0)            # min: 2 -> 0 -> 1
    assert GO.sh_range([[float("nan"), 0.3]]) == (0.3, 0.3)
    assert GO.sh_range([[0.0, 0.0]]) == (-1.5, 1.5)                 # a final 0 becomes the default
    assert GO.sh_range([]) == (-1.5, 1.5)
    row = [0.1] * 23 + [9.0]                                        # FRC23 is never read
    assert GO.sh_range([row]) == (0.1, 0.1)


def test_partition_order_ties_in_file_order_nan_last():
    c = np.array([[1.2, 0, 0], [float("nan"), 0, 0], [0.1, 0, 0], [1.4, 0, 0], [0.3, 0, 0], [-0.2, 0, 0]])
    # keys: floor(x / 0.5) * 0.5 squared: 1.0, NaN, 0, 1.0, 0, 0.25
    assert GO.partition_order(c).tolist() == [2, 4, 5, 0, 3, 1]


def test_buckets_full_order_partial_keys_and_recreation():
    block = 1.0
    # ids (x blocks, y/z flat: yBlocks = zBlocks = 0 -> id = zBlock = 0 unless the max face...) use x only through a 1-D layout
    c = np.zeros((9, 3))
    c[:, 0] = [2.5, 0.5, 2.6, 0.6, 0.7, 2.7, 2.8, 0.2, 1e12]
    # every id is xBlock * (yBlocks * zBlocks) + ... = 0 here: a flat scene collides everything into key "0"
    out = GO.buckets(c, block, 2)
    assert [b[0] for b in out] == [[0, 1], [2, 3], [4, 5], [6, 7], [8]]
    # the centre of a re-created bucket is its creator's block centre
    assert out[1][1][0] == math.floor((2.6 - 0.2) / block) * block + 0.2 + 0.5


def test_bucket_key_order_index_keys_then_insertion():
    block = 1.0
    # a 3-D scene: yBlocks = zBlocks = 3 (dims 3); ids x * 9 + y * 3 + z
    c = np.array([[0.0, 0.0, 0.0], [3.0, 3.0, 3.0], [2.1, 0.0, 0.0], [0.1, 1.1, 0.0], [1e15, 0.0, 0.0], [0.2, 0.0, 0.0]])
    out = GO.buckets(c[:4], block, 256)
    # ids: 0, 3*9+3*3+3 = 39 (max face), 18, 3 -> partial buckets in ascending id
    assert [b[0] for b in out] == [[0], [3], [2], [1]]
    out = GO.buckets(c, block, 256)
    # with the floater dims grow: yBlocks = zBlocks = 3, its id 1e15 * 9 > 2^32 - 2: enumerated after every index key
    ids = [b[0] for b in out]
    assert ids[-1] == [4] and sorted(sum(ids, [])) == list(range(6))


def test_half_truncates_and_u8_ends():
    assert GO._half(np.array([1.0009765625 + 2 ** -12]))[0] == 0x3C01      # truncation, not rounding
    assert GO._half(np.array([float("nan")]))[0] == 0x7E00
    assert KO.to_half_three(np.array([0.333], np.float32))[0] == GO._half(np.array([0.333]))[0]
    assert GO._u8(np.array([-9.0, 9.0, 0.0]), -1.5, 1.5).tolist() == [0, 255, 127]


def _ply(n, seed, sh=True):
    rng = np.random.default_rng(seed)
    props = [("x", "float"), ("y", "float"), ("z", "float")] + [(f"f_rest_{k}", "float") for k in range(45 if sh else 0)] + \
            [("opacity", "float")] + [(f"scale_{k}", "float") for k in range(3)] + [(f"rot_{k}", "float") for k in range(4)] + \
            [(f"f_dc_{k}", "float") for k in range(3)]
    cols = {k: rng.uniform(-12, 12, n) for k in ("x", "y", "z")}
    cols.update({f"f_rest_{k}": rng.normal(0, 0.3, n) for k in range(45 if sh else 0)})
    cols.update(opacity=rng.normal(0, 3, n), **{f"scale_{k}": rng.uniform(-6, -2, n) for k in range(3)})
    cols.update({f"rot_{k}": rng.normal(0, 1, n) for k in range(4)}, **{f"f_dc_{k}": rng.normal(0, 1, n) for k in range(3)})
    return FO.write_ply(props, cols, n)


@pytest.mark.parametrize("level", [0, 1, 2])
def test_round_trip_through_ksplat_oracle(level):
    data = _ply(3000, 7)
    rec, c64, sh, deg, _ = GO.generator_inputs(FO.PLY, data, 2)
    img = GO.generate(rec, c64, sh, deg, level=level, minimum_alpha=40, section_size=1100, bucket_size=16, block_size=2.0)
    d = KO.decode(img, minimum_alpha=0)
    kept = rec[:, 43] >= 40
    assert d["count"] == kept.sum() and len(d["header"].sections) == 3
    want = c64[kept]
    got = np.asarray(d["centers"], np.float64).reshape(-1, 3)
    got, want = got[np.argsort(got[:, 0], kind="stable")], want[np.argsort(want[:, 0], kind="stable")]   # x values are far apart
    if level == 0:
        assert np.array_equal(got, want.astype(np.float32).astype(np.float64))
    else:   # half a quantisation step of a 2.0 block: 1 / 32767
        assert np.abs(got - want).max() <= 1.0 / 32767 + 1e-6


def test_empty_file_has_no_sections():
    data = _ply(0, 1, sh=False)
    rec, c64, sh, deg, _ = GO.generator_inputs(FO.PLY, data, 0)
    img = GO.generate(rec, c64, sh, deg, level=1)
    assert len(img) == 4096
    assert struct.unpack_from("<4I", img, 4) == (0, 0, 0, 0) and struct.unpack_from("<2f", img, 36) == (-1.5, 1.5)
