"""Convert a `.ply` (INRIA or PlayCanvas-compressed) or `.splat` file to `.ksplat` on the GPU, with the positional arguments of the
reference's util/create-ksplat.js:

    python tools/create_ksplat.py <input .ply | .splat> <output .ksplat> [compression level] [alpha removal threshold]
                                  [scene center "x,y,z"] [block size] [bucket size] [spherical harmonics degree]

An omitted argument takes the value create-ksplat.js really ends up with: it passes `undefined`, so SplatBufferGenerator's defaults apply
(compression level 1, alpha removal threshold 1, centre 0,0,0, block size 5.0, bucket size 256) and the parser's SH degree 0.  Its usage
line says level 0; the generated file is level 1.
"""
from __future__ import annotations

import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from gaussiansplats3d_b200 import _native as N  # noqa: E402
from gaussiansplats3d_b200.engine import generate_splat_buffer  # noqa: E402


def main(argv: list[str]) -> int:
    if len(argv) < 2:
        print("Expected at least 2 arguments!")
        print("Usage: create_ksplat.py [path to .PLY or .SPLAT] [output file name] [compression level = 1] [alpha removal threshold = 1] "
              "[scene center = \"0,0,0\"] [block size = 5.0] [bucket size = 256] [spherical harmonics level = 0]")
        return 1
    src, dst = argv[0], argv[1]
    level = int(argv[2]) if len(argv) >= 3 else 1
    alpha = int(argv[3]) if len(argv) >= 4 else 1
    center = tuple(float(v) for v in argv[4].split(",")) if len(argv) >= 5 else (0.0, 0.0, 0.0)
    block = float(argv[5]) if len(argv) >= 6 else 5.0
    bucket = int(argv[6]) if len(argv) >= 7 else 256
    degree = int(argv[7]) if len(argv) >= 8 else 0
    path = src.lower().strip()
    if path.endswith(".ply"):
        fmt = N.GS_FILE_PLY
    elif path.endswith(".splat"):
        fmt = N.GS_FILE_SPLAT
    else:
        print(f"{src}: not a .ply or .splat file")
        return 1
    image = generate_splat_buffer(fmt, Path(src).read_bytes(), sh_degree=degree, compression_level=level, minimum_alpha=alpha,
                                  scene_center=center, block_size=block, bucket_size=bucket)
    Path(dst).write_bytes(image)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
