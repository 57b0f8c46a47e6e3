"""GPU: an engine gives back all of its device memory when it is destroyed, whatever it allocated on the way: file and generator
uploads, a rejected upload, blocking and pipelined frames, a SplatTree with its nodes and a raycast, profiling and the L2 flush
buffer.  Static and dynamic engines, each created and destroyed three times in one process."""
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent / "golden"))
import file_handmade as FH  # noqa: E402

from oracle import file_oracle as FO  # noqa: E402

pytestmark = pytest.mark.gpu
W, H = 320, 240


def _synthetic_ply(n, seed):
    """-> (file bytes, f32 centres)."""
    rng = np.random.default_rng(seed)
    props = [("x", "float"), ("y", "float"), ("z", "float"), ("f_dc_0", "float"), ("f_dc_1", "float"), ("f_dc_2", "float")] + \
            [(f"f_rest_{k}", "float") for k in range(9)] + [("opacity", "float")] + [(f"scale_{k}", "float") for k in range(3)] + \
            [(f"rot_{k}", "float") for k in range(4)]
    cols = {k: rng.uniform(-4, 4, n) for k in ("x", "y", "z")}
    cols.update({f"f_dc_{k}": rng.normal(0, 1, n) for k in range(3)})
    cols.update({f"f_rest_{k}": rng.normal(0, 0.2, n) for k in range(9)})
    cols.update(opacity=rng.normal(0, 3, n), **{f"scale_{k}": rng.uniform(-7, -2, n) for k in range(3)})
    cols.update({f"rot_{k}": rng.normal(0, 1, n) for k in range(4)})
    return FO.write_ply(props, cols, n), np.stack([cols["x"], cols["y"], cols["z"]], 1).astype(np.float32)


def _camera(dynamic):
    """(mvp, uniforms) of a camera 15 units in front of the scene, looking at its centre."""
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.engine import Uniforms
    proj = TM.make_perspective(50, W / H, 0.1, 1000.0)
    view = TM.invert(TM.camera_world_matrix([0.0, 0.0, 15.0], [0.0, 0.0, 0.0], [0.0, 1.0, 0.0]))
    dyn = dict(dynamic_mode=1, view_matrix=view.astype(np.float32)) if dynamic else {}
    u = Uniforms(model_view=view.astype(np.float32), projection=proj.astype(np.float32), camera_position=np.array([0.0, 0.0, 15.0], np.float32),
                 focal=(proj[0] * 0.5 * W, proj[5] * 0.5 * H), viewport=(W, H), sh_degree=1, **dyn)
    return TM.multiply(proj, view).astype(np.float32), u


def _cycle(data, count, tree, bad, pinned, **cfg):
    """Create an engine, use every path that allocates on it, destroy it."""
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.engine import Engine
    dynamic = cfg.get("dynamic_mode", False)
    mvp, u = _camera(dynamic)
    transforms = np.tile(np.eye(4, dtype=np.float32).reshape(16), N.GS_MAX_SCENES) if dynamic else None
    e = Engine(count, max_width=W, max_height=H, **cfg)
    e.upload_file(FO.PLY, data, sh_degree=1)
    n = e.upload_file_optimized(FO.PLY, data, sh_degree=1)["splat_count"]
    with pytest.raises(N.GsError) as ei:
        e.upload_file(FO.PLY, bad, sh_degree=1)
    assert ei.value.code == N.GS_ERR_BAD_ARG
    first = e.frame(mvp, u, W, H, n, transforms=transforms)
    assert first.any()
    cam = e.prepare_frame(mvp, u, W, H, n)
    e.frame_begin(cam, pinned[0])
    e.frame_begin(cam, pinned[1])
    e.frame_end()
    e.frame_end()
    assert np.array_equal(pinned[0], first) and np.array_equal(pinned[1], first)
    e.upload_splat_tree(tree)
    e.upload_splat_tree_nodes(tree)
    e.raycast([0.0, 0.0, 15.0], [0.0, 0.0, -1.0], capacity=4)
    e.set_profiling(True)
    e.frame(mvp, u, W, H, n, transforms=transforms)
    assert e.kernel_timings()
    e.set_profiling(False)
    e.flush_l2()
    e.close()


def test_destroyed_engines_return_their_device_memory(gs):
    import torch
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.engine import generate_splat_buffer
    from gaussiansplats3d_b200.splat_tree import SplatTree
    n = 50_000
    data, centers = _synthetic_ply(n, 3)
    bad = FH.MALFORMED["no_end_header"][1]
    tree = SplatTree().processSplatMesh(centers, np.full(n, 255, np.uint8), 1)
    pinned = [N.pinned_empty((H, W, 4), np.uint8) for _ in range(2)]
    configs = (dict(ray_records=True), dict(dynamic_mode=True, ray_records=True))
    for cfg in configs:          # warm-up: module loading and context set-up stay out of the count
        _cycle(data, n, tree, bad, pinned, **cfg)
    generate_splat_buffer(FO.PLY, data, sh_degree=1)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(0)[0]
    for _ in range(3):
        for cfg in configs:
            _cycle(data, n, tree, bad, pinned, **cfg)
        generate_splat_buffer(FO.PLY, data, sh_degree=1)
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info(0)[0]
    # one engine here holds hundreds of MiB (the L2 flush buffer alone is 4 x L2); what stays behind must be far less than one engine
    assert free0 - free1 < 8 << 20, f"{(free0 - free1) / 2**20:.1f} MiB not returned"
