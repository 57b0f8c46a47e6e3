"""Host-only checks of multi-view frames (gs_frame_views): the C struct's layout and the gs_view the Viewer builds for a camera."""
import ctypes as C

import numpy as np


def test_gs_view_layout():
    from gaussiansplats3d_b200 import _native as N
    assert N.GS_MAX_VIEWS == 16
    off = {name: getattr(N.gs_view, name).offset for name, _ in N.gs_view._fields_}
    assert off == dict(model_view_proj=0, model_view=64, projection=128, camera_position=192, view_matrix=204, focal=268, ortho_zoom=276)
    assert C.sizeof(N.gs_view) == 280
    assert "gs_frame_views" in N.EXPORTED_SYMBOLS


def _viewer(**opts):
    from gaussiansplats3d_b200.viewer import Viewer
    o = dict(width=640, height=360, cameraUp=(0.01933, -0.7583, -0.65161), initialCameraPosition=(1.54163, 2.68515, -6.37228),
             initialCameraLookAt=(0.45622, 1.95338, 1.51278))
    o.update(opts)
    return Viewer(o)


def _with_mesh(v, dynamic=False):
    """The uniform state updateSplatMesh sets, on a mesh without an engine."""
    from gaussiansplats3d_b200.scenes import pack_scene, synthetic_scene
    from gaussiansplats3d_b200.viewer import SplatMesh
    v.splatMesh = SplatMesh(dynamicMode=dynamic, devicePixelRatio=v.devicePixelRatio)
    v.splatMesh.packed = pack_scene(synthetic_scene(16, seed=1))
    v.camera.update()
    v.updateSplatMesh()
    return v


def test_view_of_the_viewer_camera_is_its_mono_uniforms():
    """The gs_view built for the viewer's camera carries, bit for bit, the f32 sort matrix frame() sorts with and the camera fields of
    the uniforms frame() renders with, at devicePixelRatio 1 and 2, static and dynamic."""
    for dpr in (1.0, 2.0):
        for dynamic in (False, True):
            v = _with_mesh(_viewer(devicePixelRatio=dpr), dynamic)
            view = v.viewFor(v.camera).to_c()
            uc = v.uniforms().to_c()
            mvp = v.mvp_matrix().astype(np.float32)
            assert np.array_equal(np.frombuffer(bytes(view.model_view_proj), np.float32), mvp.reshape(16))
            su = v.splatMesh.uniforms
            focal = np.array([su["focal"][0], su["focal"][1]], np.float32)
            assert np.array_equal(np.frombuffer(bytes(view.focal), np.float32), focal)
            assert np.float32(view.ortho_zoom) == np.float32(su["orthoZoom"])
            for name in ("model_view", "projection", "camera_position", "focal") + (("view_matrix",) if dynamic else ()):
                assert bytes(getattr(view, name)) == bytes(getattr(uc, name)), (dpr, dynamic, name)
            assert view.ortho_zoom == uc.ortho_zoom


def test_another_cameras_focal_follows_its_projection():
    """A camera of another fov gets the focal length updateSplatMesh would give it at the render size."""
    from gaussiansplats3d_b200 import three_math as TM
    v = _with_mesh(_viewer(devicePixelRatio=1.5))
    cam = TM.PerspectiveCamera(80.0, 640 / 360, 0.1, 1000.0)
    cam.position = np.array([0.0, 1.0, -5.0])
    cam.look_at((0.0, 0.0, 0.0))
    view = v.viewFor(cam)
    assert np.isclose(view.focal[0], cam.projectionMatrix[0] * 0.5 * 1.5 * 640)
    assert np.isclose(view.focal[1], cam.projectionMatrix[5] * 0.5 * 1.5 * 360)
    assert np.array_equal(view.model_view_proj, v.mvp_matrix(cam).astype(np.float32))
