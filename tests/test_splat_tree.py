"""SURVEY 8(f) N2: the SplatTree cull -> index gather -> partial-sort schedule (Viewer.gatherSceneNodesForSort, Viewer.js:1969-2077;
runSplatSort :1833-1964; SplatTree.js:132-278).  CPU: the vectorised tree build against the scalar restatement.  GPU: gs_gather_for_sort
against the restatement of the reference's per-frame loop (bit-exact index list), partial sorts over the gathered list against the
reference sorter, and the Viewer mirror's sort schedule against the restated state machine."""
import numpy as np
import pytest

import frame_f64 as FF

from oracle import tree_oracle as TO


def _leaf_tuples(leaves):
    return [(leaves.node_min[i].tolist(), leaves.node_max[i].tolist(), int(leaves.depth[i]),
             leaves.indexes[leaves.offsets[i]:leaves.offsets[i + 1]].tolist()) for i in range(leaves.count)]


@pytest.mark.parametrize("n,max_centers,kind", [(6000, 200, "bonsai"), (3000, 50, "garden"), (900, 1000, "uniform")])
def test_tree_build_matches_scalar_restatement(n, max_centers, kind):
    from gaussiansplats3d_b200.scenes import synthetic_scene
    from gaussiansplats3d_b200.splat_tree import SplatTree
    raw = synthetic_scene(n, seed=3, kind=kind)
    # grid-snapped centres put many points exactly on split planes (the inclusive-box / first-leaf-wins rule matters)
    centers = (np.round(raw.centers * 4) / 4).astype(np.float32) if kind == "garden" else raw.centers
    alphas = raw.colors[:, 3]
    got = _leaf_tuples(SplatTree(8, max_centers).processSplatMesh(centers, alphas, 1))
    want = TO.build_leaves(centers, alphas, 1, 8, max_centers)
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g[0] == w[0] and g[1] == w[1] and g[2] == w[2] and g[3] == w[3]
    allidx = np.concatenate([np.asarray(g[3]) for g in got])
    keep = np.nonzero(alphas >= 1)[0]
    assert np.array_equal(np.sort(allidx), keep), "every splat with alpha >= minAlpha sits in exactly one leaf"
    if max_centers < n:
        assert max(g[2] for g in got) >= 1 and len(got) > 8


def test_gather_restatement_layout_properties():
    """The restated gather itself: kept leaves nearest-LAST, every leaf's run ascending, gatherAllNodes keeps everything."""
    from gaussiansplats3d_b200.scenes import synthetic_scene
    import cases
    raw = synthetic_scene(4000, seed=5, kind="bonsai")
    leaves = TO.build_leaves(raw.centers, raw.colors[:, 3], 1, 8, 100)
    _, view, _ = cases.camera_mvp(eye=(1.5, 2.7, -6.4), target=(0.45, 1.95, 1.5), up=(0.02, -0.76, -0.65))
    out_all, n_all = TO.gather_for_sort(leaves, view, 0.9, 0.95, gather_all=True)
    assert n_all == sum(len(l[3]) for l in leaves) and np.array_equal(np.sort(out_all), np.sort(np.concatenate([l[3] for l in leaves])))
    out, n = TO.gather_for_sort(leaves, view, 0.9, 0.95)
    assert 0 < n <= n_all
    # the last run belongs to the leaf nearest to the camera
    V = np.asarray(view).reshape(4, 4).T
    best = min((np.linalg.norm(V[:3, :3] @ ((np.array(l[1]) - np.array(l[0])) * 0.5 + np.array(l[0])) + V[:3, 3]), i) for i, l in enumerate(leaves))
    assert out[-len(leaves[best[1]][3]):].tolist() == leaves[best[1]][3]


def test_gather_orders_nan_after_inf_and_ties_by_leaf_number():
    """The restated gather's order rule (tree_oracle.leaf_order_key), stated where list.sort() over NaN would leave it to the input: a NaN
    distance -- of any sign or payload -- after every number, NaNs and equal distances by leaf number."""
    nan_pos, nan_neg = float("nan"), -float("nan")
    inf = float("inf")
    assert np.signbit(nan_neg) and not np.signbit(nan_pos)
    # leaf centres: NaN (-inf .. +inf), NaN by payload, a far finite leaf, two equal near leaves, +inf centre (dist NaN via 0 * inf)
    leaves = [([-inf, 0.0, -1.0], [inf, 1.0, 0.0], 0, [0]), ([nan_pos, 0.0, -1.0], [1.0, 1.0, 0.0], 0, [1]),
              ([0.0, 0.0, -9.0], [1.0, 1.0, -8.0], 0, [2]), ([0.0, 0.0, -3.0], [1.0, 1.0, -2.0], 0, [3]),
              ([nan_neg, 0.0, -1.0], [1.0, 1.0, 0.0], 0, [4]), ([-1.0, 0.0, -3.0], [0.0, 1.0, -2.0], 0, [5]),
              ([0.0, 0.0, 0.0], [1.0, 1.0, inf], 0, [6])]
    ident = np.eye(4).reshape(16)
    out, n = TO.gather_for_sort(leaves, ident, 0.9, 0.95, gather_all=True)
    assert n == 7
    # nearest last: the two equal leaves 3 and 5 (leaf 3 first in order, so placed last), then leaf 2, then the NaNs 0, 1, 4, 6 in leaf
    # order from the front of the window
    assert out.tolist() == [6, 4, 1, 0, 2, 5, 3]
    assert TO.leaf_order_key(nan_neg, 9) > TO.leaf_order_key(inf, 10) and TO.leaf_order_key(nan_pos, 1) < TO.leaf_order_key(nan_neg, 2)
    # the same leaves in another order keep the rule (only leaf numbers decide among NaNs)
    perm = [4, 6, 0, 3, 2, 5, 1]
    out2, _ = TO.gather_for_sort([leaves[i] for i in perm], ident, 0.9, 0.95, gather_all=True)
    assert out2.tolist() == [1, 0, 6, 4, 2, 5, 3]


# ---- GPU ----------------------------------------------------------------------------------------------------------------------------
def _viewer_with_tree(gs, n=120_000, w=640, h=360, seed=9, **opts):
    from gaussiansplats3d_b200.scenes import CAMERAS, synthetic_scene
    from gaussiansplats3d_b200.viewer import Viewer
    raw = synthetic_scene(n, seed=seed, kind="bonsai")
    c = CAMERAS["bonsai"]
    v = Viewer(dict(cameraUp=c["up"], initialCameraPosition=c["position"], initialCameraLookAt=c["look_at"], width=w, height=h, splatTree=True, **opts))
    v.addSplatScene(raw)
    return v, raw


CAMERA_POSES = [((1.54163, 2.68515, -6.37228), (0.45622, 1.95338, 1.51278)),      # the demo camera
                ((0.2, 0.1, -0.3), (3.0, 0.5, 2.0)),                               # inside the cloud, looking sideways
                ((0.0, 9.0, 0.5), (0.0, 0.0, 0.0)),                                # above, looking down
                ((-14.0, 0.0, 0.0), (-30.0, 0.0, 0.0)),                            # outside, looking AWAY: almost everything culled
                ((4.0, -1.0, 5.0), (0.0, 0.0, 0.0))]


@pytest.mark.gpu
@pytest.mark.parametrize("pose", range(len(CAMERA_POSES)))
def test_gpu_gather_matches_reference_loop(gs, pose):
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.splat_tree import fov_cosines
    v, raw = _viewer_with_tree(gs)
    leaves = _leaf_tuples(v.splatMesh.getSplatTree().leaves)
    assert len(leaves) > 100
    eye, target = CAMERA_POSES[pose]
    v.camera.position = np.asarray(eye, np.float64)
    v.camera.look_at(target)
    mv = TM.invert(v.camera.matrixWorld)
    cx, cy = fov_cosines(v.renderWidth, v.renderHeight, v.camera.fov)
    for gather_all in (False, True):
        want, want_n = TO.gather_for_sort(leaves, mv, cx, cy, gather_all)
        got_n = v.engine.gather_for_sort(mv, cx, cy, gather_all)
        assert got_n == want_n
        got = v.engine.read_buffer(N.GS_BUF_INDEXES_TO_SORT, np.uint32, got_n) if got_n else np.zeros(0, np.uint32)
        assert np.array_equal(got, want)
    n_all = sum(len(l[3]) for l in leaves)
    if pose == 3:
        assert want_n == n_all and TO.gather_for_sort(leaves, mv, cx, cy, False)[1] < n_all // 2      # culling really happens
    v.dispose()


@pytest.mark.gpu
def test_partial_sorts_over_the_gathered_list(gs, oracle_mod):
    """sort_count < render_count driven end to end: the gathered list (nearest leaves last) -> gs_sort with the partial counts the
    schedule produces -> bit-exact against the reference sorter on the same list; the head is copied through (sorter.cpp:158-160)."""
    from gaussiansplats3d_b200 import _native as N
    v, raw = _viewer_with_tree(gs, n=150_000)
    n = raw.count
    eye, target = CAMERA_POSES[1]
    v.camera.position = np.asarray(eye, np.float64)
    v.camera.look_at(target)
    render_count, sort_all = v.gatherSceneNodesForSort()
    assert not sort_all and 0 < render_count < n
    gathered = v.engine.read_buffer(N.GS_BUF_INDEXES_TO_SORT, np.uint32, render_count)
    centers = v.splatMesh.getIntegerCenters(0, n - 1, True)
    mvp = v.mvp_matrix().astype(np.float32)
    sorter = oracle_mod.ref_sort_indexes if oracle_mod.have_ref() else oracle_mod.port_sort_indexes
    for frac in (0.125, 0.33333, 0.75, 1.0):
        sort_count = int(np.floor(render_count * frac))
        got, _ = v.engine.sort_gathered(mvp, sort_count, render_count)
        want = sorter(gathered, centers, None, mvp, None, None, 1 << 16, sort_count, render_count, n, False, True, False)
        assert np.array_equal(got, want), frac
        assert np.array_equal(got[:render_count - sort_count], gathered[:render_count - sort_count])
    # and the frame of the culled, fully sorted list draws that order and passes the f64 checks
    v.updateSplatMesh()
    v.splatMesh.updateRenderIndexes(None, render_count)
    frame = v.render(frame_format=N.GS_FRAME_RGBA32F, flip_y=False)
    FF.check_viewer_frame("culled, fully sorted list", v, got=frame, render_count=render_count,
                          sort=dict(centers=centers, mvp=mvp, indexes=gathered, splat_count=n), min_compared=1000)
    v.dispose()


@pytest.mark.gpu
def test_viewer_sort_schedule_follows_reference_state_machine(gs):
    """Viewer.runSplatSort over a camera path: skipped sorts below the view-change thresholds, queued partial sorts after large rotations
    (12.5 % / 33 % / 75 % / all ...), render counts from the gather -- against the restated state machine fed with the restated gather."""
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.splat_tree import fov_cosines
    v, raw = _viewer_with_tree(gs, n=60_000)
    leaves = _leaf_tuples(v.splatMesh.getSplatTree().leaves)
    sched = TO.SortSchedule()
    cx, cy = fov_cosines(v.renderWidth, v.renderHeight, v.camera.fov)
    rng = np.random.default_rng(4)
    path = [CAMERA_POSES[0]] * 3 + [CAMERA_POSES[1]] * 5 + [((0.25, 0.1, -0.3), (3.0, 0.5, 2.0))] * 2 + [CAMERA_POSES[4]] * 4 + [CAMERA_POSES[2]] * 4
    partial_seen = False
    for step, (eye, target) in enumerate(path):
        v.camera.position = np.asarray(eye, np.float64) + (rng.normal(0, 1e-3, 3) if step % 2 else 0)
        v.camera.look_at(target)
        view_dir = (-np.asarray(v.camera.matrixWorld[8:11])).tolist()
        started = v.runSplatSort()
        # the restated machine decides first whether a sort starts; the gather only runs when it does
        angle = float(np.dot(view_dir, sched.last_dir)); moved = float(np.linalg.norm(np.asarray(v.camera.position) - np.asarray(sched.last_pos)))
        if not sched.queued and not (angle <= 0.99 or moved >= 1.0):
            assert started is False
            continue
        _, rc = TO.gather_for_sort(leaves, TM.invert(v.camera.matrixWorld), cx, cy)
        want = sched.step(view_dir, list(v.camera.position), rc)
        assert started is True and want is not None
        assert (v.splatSortCount, v.splatRenderCount) == (want, rc), step
        partial_seen = partial_seen or want < rc
    assert partial_seen, "the path must exercise the partial-sort queue"
    v.dispose()


def test_cull_decision_against_an_angle_formulation():
    """Independent check of the restated cull rule (Viewer.js:2010-2037): the reference tests dot products of normalised in-plane
    projections against cos(fov/2) - 0.6; here the same geometry is decided with angles (atan2 / acos on numpy vectors, none of the
    restatement's helpers).  A leaf survives unless it is farther away than its own diagonal AND outside the widened frustum in x or y."""
    from gaussiansplats3d_b200.scenes import synthetic_scene
    from gaussiansplats3d_b200.splat_tree import fov_cosines
    import cases
    raw = synthetic_scene(20000, seed=12, kind="bonsai")
    leaves = TO.build_leaves(raw.centers, raw.colors[:, 3], 1, 8, 150)
    cx, cy = fov_cosines(1280.0, 720.0, 50.0)
    checked = culled = 0
    for eye, target in (((1.5, 2.7, -6.4), (0.45, 1.95, 1.5)), ((0.2, 0.1, -0.3), (3.0, 0.5, 2.0)), ((-14.0, 0.0, 0.0), (-30.0, 0.0, 0.0))):
        _, view, _ = cases.camera_mvp(eye=eye, target=target, up=(0.02, -0.76, -0.65))
        out, n = TO.gather_for_sort(leaves, view, cx, cy)
        kept_ids = set(out.tolist())
        V = np.asarray(view, np.float64).reshape(4, 4).T
        for mn, mx, _d, idx in leaves:
            mn, mx = np.asarray(mn), np.asarray(mx)
            t = V[:3, :3] @ ((mx - mn) * 0.5 + mn) + V[:3, 3]
            dist, diag = np.linalg.norm(t), np.linalg.norm(mx - mn)
            ang_x, ang_y = np.arctan2(abs(t[0]), -t[2]), np.arctan2(abs(t[1]), -t[2])          # angle from the view direction (0, 0, -1)
            lim_x = np.arccos(np.clip(cx - 0.6, -1.0, 1.0)) if cx - 0.6 > -1.0 else np.inf
            lim_y = np.arccos(np.clip(cy - 0.6, -1.0, 1.0)) if cy - 0.6 > -1.0 else np.inf
            margins = [abs(ang_x - lim_x), abs(ang_y - lim_y), abs(dist - diag)]
            if min(margins) < 1e-6:
                continue                                          # on a threshold: rounding may decide either way
            want_culled = (ang_x > lim_x or ang_y > lim_y) and dist > diag
            is_kept = idx[0] in kept_ids
            assert is_kept == (not want_culled), (eye, mn.tolist(), ang_x, lim_x, ang_y, lim_y, dist, diag)
            checked += 1
            culled += int(want_culled)
    assert checked > 300 and 0 < culled < checked
