"""Scene file formats (src/loaders/SceneFormat.js, src/loaders/Utils.js).

`.ply`, `.splat` and `.spz` files load through Viewer.addSplatSceneFromFile (gs_upload_file, whose format codes SceneFormat.Ply /
.Splat / .Spz are); `.ksplat` files through Viewer.addSplatSceneFromKSplat (gs_upload_ksplat).  A `.spz` file is gzip-compressed:
the library takes its packed stream, which decompressGzipped returns (Compression.js)."""
from __future__ import annotations

import gzip

from . import _native as N


class SceneFormat:
    Ply = N.GS_FILE_PLY
    Splat = N.GS_FILE_SPLAT
    KSplat = 3
    Spz = N.GS_FILE_SPZ


def decompressGzipped(data) -> bytes:  # noqa: N802  src/loaders/Compression.js
    """The gunzipped bytes of a `.spz` file as stored: the packed stream gs_upload_file(GS_FILE_SPZ) reads."""
    return gzip.decompress(bytes(data))


def sceneFormatFromPath(path: str) -> int | None:  # noqa: N802  src/loaders/Utils.js:3-9
    """The format a file name's extension names, or None.  `.spz` is not mapped here: pass SceneFormat.Spz explicitly."""
    path = str(path)
    if path.endswith(".ply"):
        return SceneFormat.Ply
    if path.endswith(".splat"):
        return SceneFormat.Splat
    if path.endswith(".ksplat"):
        return SceneFormat.KSplat
    return None
