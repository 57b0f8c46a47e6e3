"""`.ksplat` container: writer/reader round trip (CPU) and the GPU decode (gs_upload_ksplat) against the NumPy restatement of the
reference's SplatBuffer decode (oracle/ksplat_oracle.py).  Bit-exact for centres, colours, sorter centres, covariances and SH."""
import numpy as np
import pytest

import frame_f64 as FF

LEVELS_DEGREES = [(l, d) for l in (0, 1, 2) for d in (0, 1, 2)]


def _scene(n=6000, seed=3, deg=2):
    from gaussiansplats3d_b200.scenes import synthetic_scene
    raw = synthetic_scene(n, seed, "bonsai", 2)
    sh = None if deg == 0 else raw.sh[:, : (3 if deg == 1 else 8)]
    return raw, sh


@pytest.mark.parametrize("level,deg", LEVELS_DEGREES)
def test_writer_reader_round_trip(level, deg):
    from gaussiansplats3d_b200 import ksplat as K
    from oracle import ksplat_oracle as KO
    raw, sh = _scene(deg=deg)
    data = K.write(raw.centers, raw.scales, raw.rotations, raw.colors, sh, deg, compression_level=level)
    h = K.parse(data)
    assert h.compression_level == level and h.sections[0].sh_degree == deg and h.sections[0].bytes_per_splat == K.bytes_per_splat(level, deg)
    assert len(data) == K.HEADER_BYTES + K.SECTION_HEADER_BYTES + h.sections[0].data_base - h.sections[0].base + h.splat_count * h.sections[0].bytes_per_splat
    d = KO.decode(data)
    keep = raw.colors[:, 3] >= 1
    assert d["count"] == keep.sum()
    if level == 0:
        assert np.array_equal(d["centers"], raw.centers[keep]) and np.array_equal(d["scales"], raw.scales[keep])
        assert np.array_equal(d["colors"], raw.colors[keep])
    else:
        # bucket-relative u16 centres: |error| <= half a quantisation step of (blockSize/2)/32767, as a set (buckets reorder the splats)
        step = (K.BUCKET_BLOCK_SIZE / 2) / 32767
        a = np.sort(d["centers"].astype(np.float64), 0); b = np.sort(raw.centers[keep].astype(np.float64), 0)
        assert np.abs(a - b).max() <= 0.5 * step + 1e-6
        assert h.sections[0].full_bucket_count * K.BUCKET_SIZE + sum(np.frombuffer(data, np.uint8)[h.sections[0].base:h.sections[0].buckets_base].view(np.uint32)) == d["count"]
    q = d["rotations"].astype(np.float64)
    assert np.abs(np.linalg.norm(q, axis=1) - 1).max() < 2e-3
    if deg:
        assert d["sh"].shape == (d["count"], 9 if deg == 1 else 24)


def test_to_half_three_truncates():
    from gaussiansplats3d_b200 import ksplat as K
    x = np.array([0.1, -0.1, 1.0009765625, 65504.0, 1e9, 6e-8, 3e-5, 0.0, -2.5], np.float32)
    h = K.to_half_three(x).view(np.float16).astype(np.float32)
    assert np.all(np.abs(h) <= np.abs(np.clip(x, -65504, 65504)))          # truncation toward zero, never rounds up in magnitude
    rne = np.clip(x, -65504, 65504).astype(np.float16).astype(np.float32)
    assert np.all(np.abs(h - rne) <= np.abs(rne) * 2.0 ** -10 + 6e-8)
    assert h[3] == 65504.0 and h[4] == 65504.0 and h[7] == 0.0 and h[8] == -2.5


# integer sorter centres for every (level, degree); the float-centre variant on a subset
_DECODE_CASES = [(lv, dg, True) for lv, dg in LEVELS_DEGREES] + [(lv, dg, False) for lv, dg in LEVELS_DEGREES if (lv, dg) in ((0, 0), (1, 2), (2, 1))]


@pytest.mark.gpu
@pytest.mark.parametrize("level,deg,integer", _DECODE_CASES)
def test_gpu_decode_matches_splatbuffer_semantics(gs, level, deg, integer):
    from gaussiansplats3d_b200 import ksplat as K
    from gaussiansplats3d_b200 import _native as N
    from oracle import ksplat_oracle as KO
    raw, sh = _scene(n=20000, seed=4 + level, deg=deg)
    half_cov = (level == 1)
    data = K.write(raw.centers, raw.scales, raw.rotations, raw.colors, sh, deg, compression_level=level, bucket_size=100 if level else K.BUCKET_SIZE)
    want = KO.decode(data, half_covariances=half_cov)
    n = want["count"]
    with gs.Engine(n + 7, max_width=64, max_height=64, integer_based_sort=integer) as e:
        info = e.upload_ksplat(data, half_covariances=half_cov)
        assert info["splat_count"] == n and info["sh_degree"] == deg and info["compression_level"] == level
        cc = e.read_buffer(N.GS_BUF_CENTERS_COLORS, np.uint32, 4 * n).reshape(n, 4)
        assert np.array_equal(cc, want["centers_colors"])
        cov = e.read_buffer(N.GS_BUF_COVARIANCES, np.float16 if half_cov else np.float32, 6 * n).reshape(n, 6)
        assert np.array_equal(cov.view(np.uint16 if half_cov else np.uint32), want["covariances"].view(np.uint16 if half_cov else np.uint32))
        if deg:
            ncomp = 9 if deg == 1 else 24
            shd = e.read_buffer(N.GS_BUF_SH, np.uint8 if level == 2 else np.uint16, ncomp * n).reshape(n, ncomp)
            assert np.array_equal(shd, want["sh"].view(np.uint8 if level == 2 else np.uint16).reshape(n, ncomp))
        cen = e.read_buffer(N.GS_BUF_CENTERS, np.int32 if integer else np.float32, 4 * n).reshape(n, 4)
        assert np.array_equal(cen, want["int_centers"] if integer else want["float_centers"])


@pytest.mark.gpu
def test_frame_from_ksplat_equals_frame_from_arrays(gs, oracle_mod):
    """End to end: a level-1 SH2 .ksplat decoded on the GPU renders exactly like the same data uploaded as arrays."""
    from gaussiansplats3d_b200 import ksplat as K
    from gaussiansplats3d_b200.scenes import CAMERAS
    from gaussiansplats3d_b200.viewer import Viewer
    from oracle import ksplat_oracle as KO
    raw, sh = _scene(n=60000, seed=9, deg=2)
    data = K.write(raw.centers, raw.scales, raw.rotations, raw.colors, sh, 2, compression_level=1)
    d = KO.decode(data)
    n, w, h = d["count"], 640, 360
    c = CAMERAS["bonsai"]
    v = Viewer(dict(cameraUp=c["up"], initialCameraPosition=c["position"], initialCameraLookAt=c["look_at"], width=w, height=h, sphericalHarmonicsDegree=2))
    info = v.addSplatSceneFromKSplat(data)
    assert info["splat_count"] == n
    got = v.frame(frame_format=gs._native.GS_FRAME_RGBA32F, flip_y=False)
    FF.check_viewer_frame("frame from .ksplat", v, got=got, scene=d, min_compared=1000)
    v.dispose()


@pytest.mark.parametrize("level,deg", [(0, 2), (1, 2), (2, 2), (1, 1), (0, 0)])
def test_oracle_decode_with_scene_transform(level, deg):
    """The .ksplat restatement with a baked scene transform (the specification the GPU decode will follow): per splat it must agree
    with the scalar restatement of SplatBuffer.js (oracle/pack_oracle.py) applied to the values the identity decode produced, and an
    identity transform must reproduce the identity decode bit for bit in centres and covariances."""
    from oracle import ksplat_oracle as KO
    from oracle import pack_oracle as PO
    from gaussiansplats3d_b200 import ksplat as K
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.scenes import rotation_of_transform, synthetic_scene
    raw = synthetic_scene(400, seed=12, kind="bonsai", sh_degree=deg)
    data = K.write(raw.centers, raw.scales, raw.rotations, raw.colors, raw.sh, deg, compression_level=level)
    plain = KO.decode(data)
    q = np.array([0.21, 0.43, -0.36, 0.8]); q /= np.linalg.norm(q)
    T = TM.compose((0.4, -0.9, 1.3), q, (1.3, 1.3, 1.3))
    baked = KO.decode(data, transform16=T)
    ident = KO.decode(data, transform16=TM.identity())
    assert np.array_equal(ident["centers"], plain["centers"]) and np.array_equal(ident["covariances"], plain["covariances"])
    R = rotation_of_transform(T).tolist()
    lo, hi = plain["header"].min_sh, plain["header"].max_sh
    n = plain["count"]
    sh_plain = None
    if deg:
        sp = plain["sh"]
        sh_plain = (sp.astype(np.float64) / 255 * (hi - lo) + lo) if sp.dtype == np.uint8 else sp.astype(np.float64)
        if level == 0:      # the identity decode already rounded level-0 SH to half; the transform path rotates the f32 values
            sh_plain = None
    for i in range(0, n, 7):
        tri = [] if sh_plain is None else [[float(v) for v in t] for t in sh_plain[i].reshape(-1, 3)]
        c, cov6, sh = PO.bake_one([float(v) for v in plain["centers"][i]], [float(v) for v in plain["scales"][i]], [float(v) for v in plain["rotations"][i]],
                                  tri, deg if sh_plain is not None else 0, [float(v) for v in T], R)
        assert np.array_equal(baked["centers"][i], np.array(c, np.float32))
        assert np.allclose(baked["covariances"][i], np.array(cov6, np.float32), rtol=3e-7, atol=0)
        if sh_plain is not None:
            got = baked["sh"][i]
            if got.dtype == np.uint8:
                want = np.clip(np.floor((np.clip(np.array(sh).reshape(-1), lo, hi) - lo) / (hi - lo) * 255), 0, 255)
                assert np.abs(got.astype(np.int32) - want.astype(np.int32)).max() <= 0
            else:
                assert np.array_equal(got.view(np.uint16), K.to_half_three(np.array(sh, np.float32).reshape(-1)).view(np.uint16))
    # the sorter's integer centres follow the transformed centres
    assert np.array_equal(baked["int_centers"][:, :3], np.floor(baked["centers"].astype(np.float64) * 1000.0 + 0.5).astype(np.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("level,deg", [(0, 2), (1, 2), (2, 2), (1, 1), (0, 0)])
def test_gpu_decode_with_scene_transform(gs, level, deg):
    """gs_upload_ksplat with a static scene transform vs the restatement (bit-exact: both follow the reference's operation order)."""
    from gaussiansplats3d_b200 import ksplat as K
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200 import three_math as TM
    from oracle import ksplat_oracle as KO
    raw, sh = _scene(n=20000, seed=14 + level, deg=deg)
    q = np.array([0.21, 0.43, -0.36, 0.8]); q /= np.linalg.norm(q)
    T = TM.compose((0.4, -0.9, 1.3), q, (1.3, 1.3, 1.3))
    data = K.write(raw.centers, raw.scales, raw.rotations, raw.colors, sh, deg, compression_level=level, bucket_size=100 if level else K.BUCKET_SIZE)
    want = KO.decode(data, transform16=T)
    n = want["count"]
    with gs.Engine(n, max_width=64, max_height=64) as e:
        e.upload_ksplat(data, transform16=T)
        cc = e.read_buffer(N.GS_BUF_CENTERS_COLORS, np.uint32, 4 * n).reshape(n, 4)
        assert np.array_equal(cc, want["centers_colors"])
        cov = e.read_buffer(N.GS_BUF_COVARIANCES, np.float32, 6 * n).reshape(n, 6)
        assert np.array_equal(cov.view(np.uint32), want["covariances"].view(np.uint32))
        if deg:
            ncomp = 9 if deg == 1 else 24
            shd = e.read_buffer(N.GS_BUF_SH, np.uint8 if level == 2 else np.uint16, ncomp * n).reshape(n, ncomp)
            assert np.array_equal(shd, want["sh"].view(np.uint8 if level == 2 else np.uint16).reshape(n, ncomp))
        cen = e.read_buffer(N.GS_BUF_CENTERS, np.int32, 4 * n).reshape(n, 4)
        assert np.array_equal(cen, want["int_centers"])


def test_host_transform_parameters_match_python(tmp_path):
    """csrc/ksplat_transform.h (what gs_upload_ksplat hands the decode kernel) against scenes.sh_rotation_matrices, incl. a mirrored
    and a non-uniformly scaled transform (decompose's sign / scale handling)."""
    import subprocess
    from pathlib import Path
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.scenes import rotation_of_transform, sh_rotation_matrices
    root = Path(__file__).resolve().parent.parent
    exe = tmp_path / "ktc"
    subprocess.run(["/usr/bin/g++", "-O1", "-std=c++17", "-ffp-contract=off", "-o", str(exe), str(root / "oracle" / "ksplat_transform_check.cpp")], check=True)
    rng = np.random.default_rng(6)
    for trial in range(12):
        q = rng.normal(size=4); q /= np.linalg.norm(q)
        scale = (1.7, 1.7, 1.7) if trial % 3 == 0 else tuple(rng.uniform(0.4, 2.5, 3))
        if trial % 4 == 3:
            scale = (-scale[0], scale[1], scale[2])
        T = TM.compose(rng.normal(size=3), q, scale)
        out = subprocess.run([str(exe)] + [repr(float(v)) for v in T], capture_output=True, text=True, check=True)
        vals = np.array([float(v) for v in out.stdout.split()])
        m1, m2 = sh_rotation_matrices(rotation_of_transform(T))
        assert np.allclose(vals[:9].reshape(3, 3), m1, rtol=0, atol=1e-15)
        assert np.allclose(vals[9:].reshape(5, 5), m2, rtol=0, atol=1e-15)


# ---- hand-assembled byte fixtures (tests/golden/ksplat_handmade.py): built with struct.pack from the format tables, expected values from
# scalar arithmetic; imports neither the product nor oracle/ -- the third party that pins both ------------------------------------------------
def _handmade(name):
    import sys
    from pathlib import Path
    sys.path.insert(0, str(Path(__file__).resolve().parent / "golden"))
    import ksplat_handmade as HM
    data, exp = HM.fixture(name)
    return HM, data, exp


def _handmade_names():
    import sys
    from pathlib import Path
    sys.path.insert(0, str(Path(__file__).resolve().parent / "golden"))
    import ksplat_handmade as HM
    return list(HM.FIXTURES)


def _expected_arrays(exp):
    n = exp["count"]
    centers = np.array(exp["centers"], np.float32).reshape(n, 3)
    cc = np.empty((n, 4), np.uint32)
    cc[:, 0] = np.array(exp["rgba"], np.uint32)
    cc[:, 1:] = centers.view(np.uint32)
    cov = np.array(exp["cov"], np.float32).reshape(n, 6)
    ic = np.array(exp["int_centers"], np.int64).astype(np.int32).reshape(n, 4)
    sh = None
    if exp["sh_degree"]:
        sh = np.array(exp["sh"], np.uint8 if exp["level"] == 2 else np.uint16)
    return centers, cc, cov, ic, sh


@pytest.mark.parametrize("name", _handmade_names())
def test_committed_handmade_fixture_is_current(name):
    from pathlib import Path
    _, data, _ = _handmade(name)
    assert (Path(__file__).resolve().parent / "golden" / f"ksplat_handmade_{name}.ksplat").read_bytes() == data


@pytest.mark.parametrize("name", _handmade_names())
def test_oracle_decodes_handmade_fixture(name):
    """Pins oracle/ksplat_oracle.py (the decoder the GPU tests compare against) to bytes and values it did not produce."""
    from oracle import ksplat_oracle as KO
    _, data, exp = _handmade(name)
    centers, cc, cov, ic, sh = _expected_arrays(exp)
    d = KO.decode(data)
    assert d["count"] == exp["count"] and d["sh_degree"] == exp["sh_degree"]
    assert np.array_equal(d["centers"].view(np.uint32), centers.view(np.uint32))
    assert np.array_equal(d["centers_colors"], cc)
    assert np.array_equal(d["int_centers"], ic)
    assert np.array_equal(d["covariances"].view(np.uint32), cov.view(np.uint32))
    assert np.allclose(d["scales"], np.array(exp["scales"], np.float32), rtol=0, atol=0)
    assert np.allclose(d["rotations"], np.array(exp["rot_xyzw"], np.float32), rtol=0, atol=0)
    if sh is not None:
        assert np.array_equal(d["sh"].view(sh.dtype).reshape(sh.shape), sh)
    h = d["header"]
    assert (h.min_sh, h.max_sh) == exp["sh_range"] and tuple(h.scene_center) == exp["scene_center"] and len(h.sections) == exp["sections"]
    # half covariances: THREE toHalfFloat (truncation) of the f32 values, via the fixture's own IEEE-based truncation
    HM, _, _ = _handmade(name)
    dh = KO.decode(data, half_covariances=True)
    want = np.array([[HM.half_bits_truncated(float(v)) for v in row] for row in cov], np.uint16)
    ok = (np.abs(cov) >= 6.2e-5) | (cov == 0)            # the fixture's truncation helper covers the normal half range
    assert np.array_equal(dh["covariances"].view(np.uint16)[ok], want[ok])


@pytest.mark.parametrize("name", _handmade_names())
def test_product_parser_reads_handmade_fixture(name):
    from gaussiansplats3d_b200 import ksplat as K
    _, data, exp = _handmade(name)
    h = K.parse(data)
    assert h.compression_level == exp["level"] and h.max_splat_count == exp["count"] and h.splat_count == exp["count"]
    assert len(h.sections) == exp["sections"] and all(s.sh_degree == exp["sh_degree"] and s.bytes_per_splat == exp["bytes_per_splat"] for s in h.sections)
    assert (h.min_sh, h.max_sh) == exp["sh_range"] and tuple(h.scene_center) == exp["scene_center"]
    assert h.sections[-1].data_base + h.sections[-1].max_splat_count * exp["bytes_per_splat"] == len(data)
    assert sum(s.max_splat_count for s in h.sections) == exp["count"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", _handmade_names())
@pytest.mark.parametrize("half_cov", [False, True])
def test_gpu_decodes_handmade_fixture(gs, name, half_cov):
    """gs_upload_ksplat on bytes assembled by hand, against values computed by hand (no product writer, no oracle in the loop)."""
    from gaussiansplats3d_b200 import _native as N
    HM, data, exp = _handmade(name)
    centers, cc, cov, ic, sh = _expected_arrays(exp)
    n = exp["count"]
    with gs.Engine(n + 3, max_width=64, max_height=64) as e:
        info = e.upload_ksplat(data, half_covariances=half_cov)
        assert info["splat_count"] == n and info["sh_degree"] == exp["sh_degree"] and info["compression_level"] == exp["level"]
        assert info["section_count"] == exp["sections"]
        assert (np.float32(info["min_sh_coeff"]), np.float32(info["max_sh_coeff"])) == tuple(np.float32(v) for v in exp["sh_range"])
        assert np.array_equal(e.read_buffer(N.GS_BUF_CENTERS_COLORS, np.uint32, 4 * n).reshape(n, 4), cc)
        assert np.array_equal(e.read_buffer(N.GS_BUF_CENTERS, np.int32, 4 * n).reshape(n, 4), ic)
        if half_cov:
            got = e.read_buffer(N.GS_BUF_COVARIANCES, np.uint16, 6 * n).reshape(n, 6)
            want = np.array([[HM.half_bits_truncated(float(v)) for v in row] for row in cov], np.uint16)
            ok = (np.abs(cov) >= 6.2e-5) | (cov == 0)
            assert np.array_equal(got[ok], want[ok])
        else:
            assert np.array_equal(e.read_buffer(N.GS_BUF_COVARIANCES, np.uint32, 6 * n).reshape(n, 6), cov.view(np.uint32))
        if sh is not None:
            got = e.read_buffer(N.GS_BUF_SH, sh.dtype, sh.size).reshape(sh.shape)
            assert np.array_equal(got, sh)


@pytest.mark.gpu
def test_malformed_ksplat_is_rejected_before_any_kernel_runs(gs):
    """An untrusted file: section counts beyond the header's, zero bucket size, bucket tables that do not cover the splats, partial-bucket
    lengths past the section, truncated data -- every one must come back as an error code, not as out-of-bounds device accesses."""
    import struct
    from gaussiansplats3d_b200 import _native as N
    HM, data, exp = _handmade("l1_sh1")
    n = exp["count"]

    def patched(off, fmt, *vals):
        b = bytearray(data)
        struct.pack_into(fmt, b, off, *vals)
        return bytes(b)

    sec = 4096
    bad = {
        "section count > header": patched(sec + 4, "<I", n + 1000),
        "zero bucket size": patched(sec + 8, "<I", 0),
        "bucket storage": patched(sec + 20, "<H", 8),
        "more buckets than centres": patched(sec + 32, "<I", 1000),
        "partial length huge": patched(4096 + 1024, "<I", 1 << 30),
        "buckets do not cover": patched(sec + 32, "<I", 0),
        "truncated": data[:-40],
        "header count small": patched(12, "<I", 3),
    }
    with gs.Engine(n + 8, max_width=64, max_height=64) as e:
        for name, blob in bad.items():
            with pytest.raises(RuntimeError):
                e.upload_ksplat(blob)
        info = e.upload_ksplat(data)            # the engine is still usable afterwards
        assert info["splat_count"] == n
