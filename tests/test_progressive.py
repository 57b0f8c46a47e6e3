"""CPU: the progressive load's section cadence, the reveal recurrence of SplatMesh.updateVisibleRegion /
updateVisibleRegionFadeDistance (src/splatmesh/SplatMesh.js:1172-1220) and the Viewer options that drive it, without a device."""
from __future__ import annotations

import math

import pytest

from gaussiansplats3d_b200.loaders import SceneFormat
from gaussiansplats3d_b200.viewer import (PROGRESSIVE_LOAD_SECTION_SIZE, ProgressiveSceneLoad, SceneRevealMode, SplatMesh, Viewer,
                                          _stream_capacity)


class _Region:
    """An engine whose gs_visible_region answers from a list of per-splat distances."""

    def __init__(self, dists):
        self.dists = dists

    def visible_region(self, start, end, transform16=None, scene_center=None):
        return max([0.0] + [d for d in self.dists[start:end] if d > 0])


def _mesh(dists, multiplier=1.0):
    sm = SplatMesh()
    sm.engine = _Region(dists)
    sm.sceneFadeInRateMultiplier = multiplier
    return sm


def _build(sm, count, final, since):
    sm.packed = type("P", (), {"count": count})()
    sm.finalBuild = final
    sm.updateVisibleRegion(since)
    sm.lastBuildSplatCount = count


def test_section_cadence_follows_the_loader():
    """A build when more than one section size arrived since the section mark; the mark advances by one section per build."""
    load = ProgressiveSceneLoad.__new__(ProgressiveSceneLoad)
    load.received, load.streamed, load._pending, load._head, load._stream = 0, 0, [], b"", object()
    builds = []
    load._build = lambda final: builds.append((load.received, final)) or True
    for size in [100000, 100000, 100000, 600000, 1, 1, 262144]:
        load.append(b"\0" * size)
    S = PROGRESSIVE_LOAD_SECTION_SIZE
    assert S == 262144
    assert builds == [(300000, False), (900000, False), (900001, False), (1162146, False)]
    assert load.streamed == 4 * S


def test_reveal_recurrence():
    sm = _mesh([0.5, 3.0, 2.0, 7.5, float("nan"), 9.25])
    _build(sm, 2, False, False)
    # maxDistance 3 exceeds the buffer radius 0 by more than VISIBLE_REGION_EXPANSION_DELTA = 1: radius 2, buffer 3
    assert (sm.maxSplatDistanceFromSceneCenter, sm.visibleRegionBufferRadius, sm.visibleRegionRadius) == (3.0, 3.0, 2.0)
    assert sm.visibleRegionFadeStartRadius == 2.0 * 0.003      # the build's own Default-mode step: gradual before the final build
    r = sm.visibleRegionFadeStartRadius
    sm.updateVisibleRegionFadeDistance(SceneRevealMode.Gradual)
    assert sm.visibleRegionFadeStartRadius == (2.0 - r) * 0.003 + r and not sm.fadeInComplete
    sm.updateVisibleRegionFadeDistance(SceneRevealMode.Instant)
    assert sm.fadeInComplete and sm.visibleRegionChanging
    _build(sm, 4, False, True)
    assert (sm.visibleRegionBufferRadius, sm.visibleRegionRadius) == (7.5, 6.5)
    _build(sm, 6, True, True)
    assert sm.visibleRegionRadius == sm.visibleRegionBufferRadius == 9.25
    for _ in range(2000):
        r = sm.visibleRegionFadeStartRadius
        sm.updateVisibleRegionFadeDistance(SceneRevealMode.Default)
        assert sm.visibleRegionFadeStartRadius == (9.25 - r) * 0.012 + r
        if sm.fadeInComplete:
            break
    assert sm.fadeInComplete and sm.visibleRegionFadeStartRadius / 9.25 > 0.99 and not sm.visibleRegionChanging


def test_fade_rate_multiplier_and_empty_region():
    sm = _mesh([0.0, float("inf")], multiplier=2.5)
    _build(sm, 1, False, False)
    assert sm.visibleRegionBufferRadius == 0 and not sm.fadeInComplete   # nothing loaded far from the centre yet: 0 %, not complete
    _build(sm, 2, True, True)
    assert math.isinf(sm.visibleRegionRadius)
    sm2 = _mesh([4.0], multiplier=2.5)
    _build(sm2, 1, True, False)
    assert sm2.visibleRegionFadeStartRadius == 4.0 * (0.012 * 2.5)


def test_viewer_options():
    v = Viewer(dict(width=8, height=8))
    assert v.sceneRevealMode is None and v.sceneFadeInRateMultiplier == 1.0
    v = Viewer(dict(width=8, height=8, sceneRevealMode=SceneRevealMode.Gradual, sceneFadeInRateMultiplier=0))
    assert v.sceneRevealMode == SceneRevealMode.Gradual and v.sceneFadeInRateMultiplier == 1.0   # `|| 1.0`, Viewer.js:205


def test_stream_capacity_from_headers():
    ply = b"ply\nformat binary_little_endian 1.0\nelement vertex 77\nproperty float x\nend_header\n"
    assert _stream_capacity(SceneFormat.Ply, ply[:20], None) is None
    assert _stream_capacity(SceneFormat.Ply, ply, None) == 77
    assert _stream_capacity(SceneFormat.KSplat, b"\0" * 12 + (1234).to_bytes(4, "little"), None) == 1234
    assert _stream_capacity(SceneFormat.Splat, b"", 32 * 5 + 3) == 5
    with pytest.raises(ValueError):
        _stream_capacity(SceneFormat.Splat, b"", None)
