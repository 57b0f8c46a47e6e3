"""Scene file formats (src/loaders/SceneFormat.js, src/loaders/Utils.js).

`.ply` and `.splat` files load through Viewer.addSplatSceneFromFile (gs_upload_file, whose format codes SceneFormat.Ply / .Splat are);
`.ksplat` files through Viewer.addSplatSceneFromKSplat (gs_upload_ksplat)."""
from __future__ import annotations

from . import _native as N


class SceneFormat:
    Ply = N.GS_FILE_PLY
    Splat = N.GS_FILE_SPLAT
    KSplat = 3


def sceneFormatFromPath(path: str) -> int | None:  # noqa: N802  src/loaders/Utils.js:3-9
    """The format a file name's extension names, or None (`.spz` is not supported)."""
    path = str(path)
    if path.endswith(".ply"):
        return SceneFormat.Ply
    if path.endswith(".splat"):
        return SceneFormat.Splat
    if path.endswith(".ksplat"):
        return SceneFormat.KSplat
    return None
