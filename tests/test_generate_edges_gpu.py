"""GPU: gs_generate_splat_buffer on the adversarial inputs of tests/generate_edge_cases.py, every byte against oracle/generate_oracle.py
(test_generate_gpu._check_image), at every compression level and SH degree the case touches; each case also shows on the oracle side that
its branch ran.  And the hand-derived anchors of tests/test_generate_edges.py against the GPU image."""
import struct

import numpy as np
import pytest

import generate_edge_cases as EC
from oracle import file_oracle as FO
from test_generate_gpu import _check_image

pytestmark = pytest.mark.gpu
CASES = EC.all_cases()


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_generated_image_matches_oracle(gs, case):
    for kw in case.opts:
        assert _check_image(gs, case.fmt, case.data, case.sh_degree, **kw) == 0, f"{case.name} {kw}: a splat flagged for libm exp"
    assert case.ran(case) > 0, case.name


def test_anchor_scan_zero_is_replaced(gs):
    from gaussiansplats3d_b200.engine import generate_splat_buffer
    data = EC.anchor_scan_ply()
    for deg in (1, 2):
        for level in EC.LEVELS:
            img = generate_splat_buffer(FO.PLY, data, sh_degree=deg, compression_level=level)
            assert struct.unpack_from("<2f", img, 36) == (2.0, 5.0)
        img = generate_splat_buffer(FO.PLY, data, sh_degree=deg, compression_level=2)
        assert list(img[4096 + 1024 + 16 + 24:]) == [85, 0, 255, 0] + [0] * (5 if deg == 1 else 20)


def test_anchor_cross_block_collision_keeps_creator_centre(gs):
    from gaussiansplats3d_b200.engine import generate_splat_buffer
    img = generate_splat_buffer(FO.SPLAT, EC.splat(EC.ANCHOR_COLLIDE), compression_level=1, block_size=1.0)
    assert struct.unpack_from("<I3f", img, 4096 + 1024) == (2, *EC.ANCHOR_COLLIDE_CENTRE)
    for i, q in enumerate(EC.ANCHOR_COLLIDE_Q):
        assert struct.unpack_from("<3H", img, 4096 + 1024 + 16 + 24 * i) == q


def test_anchor_class1_keys_in_insertion_order(gs):
    from gaussiansplats3d_b200.engine import generate_splat_buffer
    data, kw = EC.anchor_class1_splat()
    img = generate_splat_buffer(FO.SPLAT, data, compression_level=1, **kw)
    assert struct.unpack_from("<5I", img, 4096 + 1024) == (1, 1, 1, 1, 2)
    centres = np.array(struct.unpack_from("<15f", img, 4096 + 1024 + 20)).reshape(5, 3)
    assert centres[0].tolist() == [0.5, 0.5, 0.5] and centres[1].tolist() == [0.5, 1.5, 1.5]
    assert centres[2].tolist() == [np.float32(5e9 + 0.5), 0.5, 0.5]
    assert centres[3, 0] == np.inf and np.isnan(centres[4, 0]) and centres[4, 1:].tolist() == [0.5, 0.5]
