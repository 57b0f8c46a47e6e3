"""GPU: a rejected scene upload leaves the scene the engine had, for each of the three upload entries (gs_upload_ksplat, gs_upload_file,
gs_upload_file_optimized).  Each malformed or over-capacity input comes back with its error code, the next frame is bit-identical to the
one before it, and a valid upload through the same entry afterwards renders that frame again."""
import struct
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent / "golden"))
import file_handmade as FH  # noqa: E402

from oracle import file_oracle as FO  # noqa: E402

pytestmark = pytest.mark.gpu
W, H = 256, 192
N_SPLATS = 20_000


def _synthetic_ply(n, seed):
    rng = np.random.default_rng(seed)
    props = [("x", "float"), ("y", "float"), ("z", "float"), ("f_dc_0", "float"), ("f_dc_1", "float"), ("f_dc_2", "float")] + \
            [(f"f_rest_{k}", "float") for k in range(9)] + [("opacity", "float")] + [(f"scale_{k}", "float") for k in range(3)] + \
            [(f"rot_{k}", "float") for k in range(4)]
    cols = {k: rng.uniform(-4, 4, n) for k in ("x", "y", "z")}
    cols.update({f"f_dc_{k}": rng.normal(0, 1, n) for k in range(3)})
    cols.update({f"f_rest_{k}": rng.normal(0, 0.2, n) for k in range(9)})
    cols.update(opacity=rng.normal(0, 3, n), **{f"scale_{k}": rng.uniform(-7, -2, n) for k in range(3)})
    cols.update({f"rot_{k}": rng.normal(0, 1, n) for k in range(4)})
    return FO.write_ply(props, cols, n)


def _camera():
    """(mvp, uniforms) of a camera 15 units in front of the scene, looking at its centre."""
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.engine import Uniforms
    proj = TM.make_perspective(50, W / H, 0.1, 1000.0)
    view = TM.invert(TM.camera_world_matrix([0.0, 0.0, 15.0], [0.0, 0.0, 0.0], [0.0, 1.0, 0.0]))
    u = Uniforms(model_view=view.astype(np.float32), projection=proj.astype(np.float32), camera_position=np.array([0.0, 0.0, 15.0], np.float32),
                 focal=(proj[0] * 0.5 * W, proj[5] * 0.5 * H), viewport=(W, H), sh_degree=1)
    return TM.multiply(proj, view).astype(np.float32), u


def _patched(data, off, fmt, *vals):
    b = bytearray(data)
    struct.pack_into(fmt, b, off, *vals)
    return bytes(b)


def _ksplat_cases(img, capacity):
    """name -> (image, status, words) for gs_upload_ksplat; `img` is a one-section level-1 image with partial buckets."""
    from gaussiansplats3d_b200 import _native as N
    sections, partial = struct.unpack_from("<I", img, 4)[0], struct.unpack_from("<I", img, 4096 + 36)[0]
    assert sections == 1 and partial > 0
    return {
        "short": (img[:4000], N.GS_ERR_BAD_ARG, "4096-byte header"),
        "version": (_patched(img, 0, "<BB", 0, 0), N.GS_ERR_BAD_ARG, "version"),
        "level": (_patched(img, 20, "<H", 3), N.GS_ERR_BAD_ARG, "compression level"),
        "header capacity": (_patched(img, 12, "<I", capacity + 1), N.GS_ERR_CAPACITY, "engine capacity"),
        "section headers": (img[:4096 + 512], N.GS_ERR_BAD_ARG, "section headers"),
        "truncated": (img[:-40], N.GS_ERR_BAD_ARG, "truncated"),
        "sh degree": (_patched(img, 4096 + 40, "<H", 3), N.GS_ERR_BAD_ARG, "SH degree"),
        "partial length": (_patched(img, 4096 + 1024, "<I", 1 << 30), N.GS_ERR_BAD_ARG, "partial bucket"),
        "buckets do not cover": (_patched(img, 4096 + 32, "<I", 0), N.GS_ERR_BAD_ARG, "do not cover"),
        "more than declared": (_patched(img, 12, "<I", 3), N.GS_ERR_CAPACITY, "its header declares"),
    }


def _file_cases(capacity):
    """name -> (format, file, status, words) for the file entries."""
    cases = dict(FH.MALFORMED)
    cases["capacity"] = (FO.PLY, _synthetic_ply(capacity + 1, 5), FH.CAPACITY, "capacity")
    return cases


@pytest.mark.parametrize("entry", ["upload_ksplat", "upload_file", "upload_file_optimized"])
def test_rejected_upload_keeps_previous_scene(gs, entry):
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.engine import generate_splat_buffer
    data = _synthetic_ply(N_SPLATS, 3)
    mvp, u = _camera()
    if entry == "upload_ksplat":
        img = generate_splat_buffer(FO.PLY, data, sh_degree=1, bucket_size=64)
        good = dict(data=img)
        bad = {k: (dict(data=blob), status, words) for k, (blob, status, words) in _ksplat_cases(img, N_SPLATS).items()}
    else:
        good = dict(format=FO.PLY, data=data, sh_degree=1)
        bad = {k: (dict(format=fmt, data=blob, sh_degree=1), status, words) for k, (fmt, blob, status, words) in _file_cases(N_SPLATS).items()}
        bad["sh_degree"] = (dict(good, sh_degree=3), N.GS_ERR_BAD_ARG, "sphericalHarmonicsDegree")
        if entry == "upload_file_optimized":
            bad["generate options"] = (dict(good, compression_level=3), N.GS_ERR_BAD_ARG, "compression level")
    with gs.Engine(N_SPLATS, max_width=W, max_height=H) as e:
        upload = getattr(e, entry)
        n = upload(**good)["splat_count"]
        assert 0 < n <= N_SPLATS
        before = e.frame(mvp, u, W, H, n, frame_format=N.GS_FRAME_RGBA32F)
        assert before.any()
        for name, (kw, status, words) in bad.items():
            with pytest.raises(N.GsError) as ei:
                upload(**kw)
            assert ei.value.code == status and words in str(ei.value), (name, str(ei.value))
            assert np.array_equal(e.frame(mvp, u, W, H, n, frame_format=N.GS_FRAME_RGBA32F), before), name
        assert upload(**good)["splat_count"] == n
        assert np.array_equal(e.frame(mvp, u, W, H, n, frame_format=N.GS_FRAME_RGBA32F), before)
