"""CPU: the uniforms a WebXR Viewer hands the engine, against three.js's definitions worked by hand in numpy.  Per eye (what three.js sets
for each sub-camera of the XR ArrayCamera): modelViewMatrix = eye.matrixWorldInverse * mesh.matrixWorld, projectionMatrix, cameraPosition
= the eye's world position, viewMatrix = eye.matrixWorldInverse (dynamic meshes).  Shared (Viewer.updateSplatMesh for one eye's size): the
viewport is the eye's size in device pixels and the focal lengths are the viewer camera's at that size."""
import numpy as np
import pytest


def _col(m16):
    return np.asarray(m16, np.float64).reshape(4, 4).T      # three.js elements are column-major


def _viewer(dynamic=False, w=2 * 1440, h=1600):
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.scenes import synthetic_scene
    from gaussiansplats3d_b200.viewer import SplatMesh, Viewer, WebXRMode
    v = Viewer(dict(webXRMode=WebXRMode.VR, width=w, height=h, devicePixelRatio=2.0, dynamicScene=dynamic, sphericalHarmonicsDegree=1,
                    initialCameraPosition=(0.3, 1.6, 2.5), initialCameraLookAt=(0.0, 1.0, 0.0)))
    v.splatMesh = SplatMesh(dynamicMode=dynamic, sphericalHarmonicsDegree=1)        # no engine: host-side only
    v.splatMesh.build(synthetic_scene(100, seed=3, sh_degree=1))
    v.splatMesh.matrixWorld = TM.compose((0.5, -0.25, 1.0), (0.0, 0.3826834, 0.0, 0.9238795), (2.0, 2.0, 2.0))
    v.camera.update()
    v.updateSplatMesh()
    return v


def _eye_cameras(v, ipd=0.064):
    from gaussiansplats3d_b200 import three_math as TM
    cams = []
    right = v.camera.matrixWorld[0:3]
    for s in (-0.5, 0.5):
        c = TM.PerspectiveCamera(v.camera.fov, v.camera.aspect, v.camera.near, v.camera.far)
        c.position = v.camera.position + s * ipd * right
        c.up = v.camera.up
        c.look_at(v.camera.target + s * ipd * right)
        c.update()
        cams.append(c)
    return cams


@pytest.mark.parametrize("dynamic", [False, True])
def test_per_eye_uniforms_follow_threejs(dynamic):
    v = _viewer(dynamic)
    cams = _eye_cameras(v)
    eyes = v.xrEyes(cams)
    mesh = _col(v.splatMesh.matrixWorld)
    for eye, cam in zip(eyes, cams):
        world = _col(cam.matrixWorld)
        mv = np.linalg.inv(world) @ mesh
        np.testing.assert_allclose(_col(eye.model_view), mv, rtol=1e-6, atol=1e-6)
        np.testing.assert_array_equal(eye.projection, np.asarray(cam.projectionMatrix, np.float32))
        np.testing.assert_allclose(eye.camera_position, world[:3, 3], rtol=1e-6)
        if dynamic:
            np.testing.assert_allclose(_col(eye.view_matrix), np.linalg.inv(world), rtol=1e-6, atol=1e-6)
        else:
            assert eye.view_matrix is None
    # the eyes are the ipd apart along the viewer camera's right axis
    assert np.isclose(np.linalg.norm(eyes[1].camera_position - eyes[0].camera_position), 0.064, rtol=1e-5)
    c = eyes[0].to_c()
    assert list(c.model_view) == [float(x) for x in np.asarray(eyes[0].model_view, np.float32).reshape(16)]


def test_shared_uniforms_are_sized_for_one_eye():
    v = _viewer(w=2 * 1440, h=1600)
    u = v.uniforms()
    assert v.renderDimensions() == (1440, 1600)
    assert tuple(u.viewport) == (1440.0, 1600.0), "the viewport uniform must be the eye's size in device pixels"
    P = _col(v.camera.projectionMatrix)
    assert u.focal == pytest.approx((P[0, 0] * 0.5 * 1440, P[1, 1] * 0.5 * 1600), rel=1e-12)
    # the sort and the shared model-view stay the viewer camera's
    np.testing.assert_allclose(_col(u.model_view), np.linalg.inv(_col(v.camera.matrixWorld)) @ _col(v.splatMesh.matrixWorld), rtol=1e-6, atol=1e-6)


def test_webxr_mode_option_and_arguments():
    from gaussiansplats3d_b200.viewer import Viewer, WebXRMode
    assert (WebXRMode.NONE, WebXRMode.VR, WebXRMode.AR) == (0, 1, 2)
    with pytest.raises(ValueError, match="even"):
        Viewer(dict(webXRMode=WebXRMode.AR, width=1001, height=600))
    v = _viewer()
    with pytest.raises(ValueError, match="xrCameras"):
        v._xr(None)
    mono = Viewer(dict(width=800, height=600))
    assert mono.renderDimensions() == (800, 600) and mono._xr(None) is None
    with pytest.raises(ValueError, match="webXRMode"):
        mono._xr(_eye_cameras(v))
