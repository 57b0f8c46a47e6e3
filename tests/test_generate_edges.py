"""CPU: the adversarial generator inputs of tests/generate_edge_cases.py reach the branches they are built for (on the oracle side), and
oracle/generate_oracle.py agrees with hand-derived values for the SH range scan, a cross-block id collision and class-1 key order."""
import struct

import numpy as np
import pytest

import generate_edge_cases as EC
from oracle import file_oracle as FO
from oracle import generate_oracle as GO

CASES = EC.all_cases()


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_case_reaches_its_branch(case):
    assert case.ran(case) > 0, case.name


def test_case_names_unique():
    assert len({c.name for c in CASES}) == len(CASES)


def test_sh_boundaries_are_where_the_scan_splits():
    # k_gen_sh_scan: 8 splats per thread, 256 threads per CTA
    assert EC.SH_CTA == EC.SH_THREAD * 256 and EC.N_SH > 10 * EC.SH_CTA
    assert EC._thread_last(3) == 31 and EC._cta_first(2) == 4096 and EC._cta_last(2) == 6143


# ---- hand-derived anchors ------------------------------------------------------------------------------------------------------------
def test_anchor_scan_zero_is_replaced():
    assert GO.sh_range([[3.0, 0.0, 5.0, 2.0]]) == (2.0, 5.0)
    assert np.nanmin([3.0, 0.0, 5.0, 2.0]) == 0.0                       # what a plain min would give
    data = EC.anchor_scan_ply()
    for deg in (1, 2):
        rec, c64, sh, d, _ = GO.generator_inputs(FO.PLY, data, deg)
        assert sh[0, :4].tolist() == [3.0, 0.0, 5.0, 2.0] and np.isnan(sh[0, 4:]).all()
        for level in EC.LEVELS:
            img = GO.generate(rec, c64, sh, d, level=level)
            assert struct.unpack_from("<2f", img, 36) == (2.0, 5.0)
        img = GO.generate(rec, c64, sh, d, level=2)
        # level 2, one splat: header, section header, 4-byte partial length, 12-byte centre, then 24 bytes + ncomp SH bytes
        body = img[4096 + 1024 + 16:]
        # floor((clamp(v, 2, 5) - 2) / 3 * 255): 3 -> 85, 5 -> 255, 2 -> 0; 0 and NaN are written as 0, clamped to 2 -> 0
        assert list(body[24:]) == [85, 0, 255, 0] + [0] * (5 if deg == 1 else 20)


def test_anchor_cross_block_collision_keeps_creator_centre():
    out = GO.buckets(EC.ANCHOR_COLLIDE, 1.0, 256)
    assert [b[0] for b in out] == [[0, 1]] and out[0][1] == list(EC.ANCHOR_COLLIDE_CENTRE)
    _, bid, ctr = EC.block_ids(EC.ANCHOR_COLLIDE, 1.0)
    assert bid.tolist() == [1.0, 1.0] and ctr.tolist() == [[0.5, 0.5, 1.5], [0.5, 1.5, 0.5]]
    data = EC.splat(EC.ANCHOR_COLLIDE)
    rec, c64, sh, d, _ = GO.generator_inputs(FO.SPLAT, data, 0)
    img = GO.generate(rec, c64, sh, d, level=1, block_size=1.0)
    assert struct.unpack_from("<I3f", img, 4096 + 1024) == (2, *EC.ANCHOR_COLLIDE_CENTRE)
    for i, q in enumerate(EC.ANCHOR_COLLIDE_Q):
        assert struct.unpack_from("<3H", img, 4096 + 1024 + 16 + 24 * i) == q


def test_anchor_class1_keys_in_insertion_order():
    out = GO.buckets(EC.ANCHOR_CLASS1, 1.0, 256)
    assert [b[0] for b in out] == EC.ANCHOR_CLASS1_BUCKETS
    # the insertion order NaN, inf, 5e9 is the reverse of the ids' order
    assert [GO._key(b) for b in (float("nan"), float("inf"), 5e9)] == [(1, "NaN"), (1, "inf"), (1, "5000000000.0")]
    data, kw = EC.anchor_class1_splat()
    rec, c64, sh, d, _ = GO.generator_inputs(FO.SPLAT, data, 0)
    img = GO.generate(rec, c64, sh, d, level=1, **kw)
    lens = struct.unpack_from("<5I", img, 4096 + 1024)
    centres = np.array(struct.unpack_from("<15f", img, 4096 + 1024 + 20)).reshape(5, 3)
    assert lens == (1, 1, 1, 1, 2)
    # ids 0 and 2 (block centres (0.5, 0.5, 0.5) and (0.5, 1.5, 1.5)), then 5e9, inf and NaN as inserted
    assert centres[0].tolist() == [0.5, 0.5, 0.5] and centres[1].tolist() == [0.5, 1.5, 1.5]
    assert centres[2].tolist() == [np.float32(5e9 + 0.5), 0.5, 0.5]
    assert centres[3, 0] == np.inf and np.isnan(centres[4, 0]) and centres[4, 1:].tolist() == [0.5, 0.5]
