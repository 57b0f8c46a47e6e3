"""tests/inriav2_oracle.py -- TEST INFRASTRUCTURE ONLY.  Imports nothing from the product package.

NumPy restatement of what the reference builds from an INRIA v2 (codebook) `.ply` through SplatBufferGenerator, the only way it loads
one (PlyParser.parseToUncompressedSplatBuffer throws for this flavour):
  header    INRIAV2PlyParser.decodeSectionHeadersFromHeaderLines / findVertexData: elements in header order, each one's rows after the
            previous one's; one codebook_centers element and one splat element
  codebook  decodeCodeBook (:128-160): fromHalfFloat of each entry (0 when the row lacks it), then opacity Math.round(sigmoid(v) 255),
            features_dc Math.round((0.5 + SH_C0 v) 255), scaling Math.exp(v), every other page v
  splat     parseToUncompressedSplat (:202-269, readVertex with normalize = false): half-bit centres, codebook lookups for everything
            else; an index that names no codebook row reads `undefined`, which every later step treats as NaN, except one: the writer
            zeroes all three scales when scale_0 is `undefined` (SplatBuffer.js:1099-1105), and each NaN scale on its own
  image     the unified array is built at the requested SH degree (:300), so the image carries that degree with 0 past the file's
            coefficients; the SH range scan sees only the file's coefficients (SplatBuffer.js:1193)

`generator_inputs` gives the level-0 records, f64 centres and raw SH for oracle.generate_oracle.generate; `image` runs it.  Every step is
exact JavaScript-number arithmetic except the two `exp` pages: a splat is flagged `ambiguous` when it reads a scaling or opacity entry
whose f32 scale or rounded alpha an `exp` 2 f64 ulps away would change (`flagged_halves` enumerates all 65536 halves).
"""
from __future__ import annotations

import re

import numpy as np

from oracle import generate_oracle as GO
from oracle.file_oracle import SH_C0, _exp_band, _f32, _normalize, _u8_floor

PLY = 1
PAGES = ["features_dc"] + [f"features_rest_{k}" for k in range(15)] + ["opacity", "scaling", "rotation_re", "rotation_im"]
DC, REST0, REST3, OPACITY, SCALING, ROT_RE, ROT_IM = 0, 1, 4, 16, 17, 18, 19
_TYPES = {"double": "<f8", "int": "<i4", "uint": "<u4", "float": "<f4", "short": "<i2", "ushort": "<u2", "uchar": "u1"}


# ---- reader (reference semantics on files the library accepts) -----------------------------------------------------------------------
def parse(data) -> dict:
    """-> dict(codebook=structured rows, splats=structured rows, sh_degree, sh_per_channel) of a v2 file."""
    data = bytes(data)
    end = data.index(b"end_header")
    at = end + 11
    elements = []
    for ln in (s.strip() for s in data[:end].decode("ascii").split("\n")):
        if ln.startswith("element"):
            w = ln.split()
            elements.append([w[1], int(w[2]), []])
        elif ln.startswith("property") and elements:
            m = re.match(r"(\w+)\s+(\w+)\s+(\w+)", ln)
            elements[-1][2].append((m.group(3), _TYPES[m.group(2)]))
    out = {}
    for name, count, props in elements:
        dt = np.dtype(props)
        rows = np.frombuffer(data, dt, count, at)
        at += count * dt.itemsize
        out["codebook" if name == "codebook_centers" else "splats"] = rows
    nrest = sum(1 for n in out["splats"].dtype.names if n.startswith("f_rest"))
    cpc = nrest // 3
    out["sh_per_channel"] = cpc
    out["sh_degree"] = 2 if cpc >= 8 else (1 if cpc >= 3 else 0)
    return out


def half(bits) -> np.ndarray:
    """fromHalfFloat of 16-bit patterns (ushort or short), exactly, as f64."""
    return (np.asarray(bits).astype(np.int64) & 0xFFFF).astype(np.uint16).view(np.float16).astype(np.float64)


def _js_round(v):
    with np.errstate(invalid="ignore"):
        r = np.floor(v)
        return np.where(np.isfinite(v), np.where(v - r >= 0.5, r + 1, r), v)


def _opacity(v):
    with np.errstate(over="ignore"):
        return _js_round((1 / (1 + np.exp(-v))) * 255)


def codebook_table(cb) -> np.ndarray:
    """f64[20, rows]: decodeCodeBook's pages."""
    rows = len(cb)
    t = np.zeros((len(PAGES), rows))
    for p, name in enumerate(PAGES):
        if name in cb.dtype.names:
            t[p] = half(cb[name])
    with np.errstate(over="ignore", invalid="ignore"):
        t[OPACITY] = _opacity(t[OPACITY])
        t[DC] = _js_round((0.5 + SH_C0 * t[DC]) * 255)
        t[SCALING] = np.exp(t[SCALING])
    return t


def flagged_halves(v) -> tuple[np.ndarray, np.ndarray]:
    """-> (scaling, opacity) bool masks over the halves v: whether an `exp` 2 f64 ulps away changes the f32 scale / the rounded alpha.
    exp(+-0) = 1 is exact in every libm and is not flagged (it is the opacity tie 127.5)."""
    v = np.asarray(v, np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        lo, hi = _exp_band(np.exp(v))
        lo = np.maximum(lo, 0.0)                         # exp is never negative: the band of the least subnormal stops at +0
        scaling = _f32(lo).view(np.uint32) != _f32(hi).view(np.uint32)
        lo, hi = _exp_band(np.exp(-v))
        a, b = _js_round((1 / (1 + lo)) * 255), _js_round((1 / (1 + hi)) * 255)
        opacity = (_u8_floor(a) != _u8_floor(b)) & (v != 0)
    return scaling, opacity


def _index(col) -> np.ndarray:
    return np.asarray(col).astype(np.int64)


def generator_inputs(data, sh_degree: int = 0):
    """-> (records u8[n, 44 | 80 | 140], centres f64[n, 3], raw SH f64[n, image ncomp], image SH degree, SH components read,
    ambiguous bool[n]).  The records and SH are at the requested degree; the SH columns past the file's are 0."""
    p = parse(data)
    cb, s = p["codebook"], p["splats"]
    rows, n = len(cb), len(s)
    names = s.dtype.names
    t = codebook_table(cb)
    flag_s, flag_o = flagged_halves(half(cb["scaling"]) if "scaling" in cb.dtype.names else np.zeros(rows))[0], \
        flagged_halves(half(cb["opacity"]) if "opacity" in cb.dtype.names else np.zeros(rows))[1]

    def look(page, field):
        i = _index(s[field])
        ok = (i >= 0) & (i < rows)
        return np.where(ok, t[page][np.where(ok, i, 0)] if rows else np.nan, np.nan), ok

    ambiguous = np.zeros(n, bool)
    rec_deg, read = sh_degree, min(sh_degree, p["sh_degree"])
    ncomp, nread = {0: 0, 1: 9, 2: 24}[rec_deg], {0: 0, 1: 9, 2: 24}[read]
    rec = np.zeros((n, 44 + 4 * ncomp), np.uint8)
    with np.errstate(all="ignore"):
        c64 = np.stack([half(s[k]) for k in "xyz"], 1)
        rec[:, 0:12] = _f32(c64).view(np.uint8).reshape(n, 12)
        if "scale_0" in names:
            # the writer: `scale_0 !== undefined ? (s_k || 0) : 0` -- an undefined scale_0 zeroes all three, a NaN value only itself
            read0 = look(SCALING, "scale_0")[1]
            sc = []
            for k in range(3):
                v, ok = look(SCALING, f"scale_{k}")
                sc.append(np.where(read0 & ~np.isnan(v), v, 0.0))
                ambiguous |= read0 & ok & flag_s[np.where(ok, _index(s[f"scale_{k}"]), 0)] if rows else False
            sc = np.stack(sc, 1)
        else:
            sc = np.full((n, 3), 0.01)
        rec[:, 12:24] = _f32(sc).view(np.uint8).reshape(n, 12)
        q = [look(ROT_RE, "rot_0")[0]] + [look(ROT_IM, f"rot_{k}")[0] for k in (1, 2, 3)]
        q = _normalize(*_normalize(*q))                                           # parser, then writer
        rec[:, 24:40] = _f32(np.stack(q, 1)).view(np.uint8).reshape(n, 16)
        for k in range(3):
            rec[:, 40 + k] = _u8_floor(look(DC, f"f_dc_{k}")[0]) if "f_dc_0" in names else 0
        if "opacity" in names:
            v, ok = look(OPACITY, "opacity")
            rec[:, 43] = _u8_floor(v)
            ambiguous |= ok & flag_o[np.where(ok, _index(s["opacity"]), 0)] if rows else False
        sh = np.zeros((n, ncomp))
        c = p["sh_per_channel"]
        for k in range(nread):
            src = (k % 3) + c * (k // 3) if k < 9 else 3 + (k - 9) % 5 + c * ((k - 9) // 5)
            sh[:, k] = look(REST0 + k % 3 if k < 9 else REST3 + (k - 9) % 5, f"f_rest_{src}")[0]
        if ncomp:
            rec[:, 44:] = _f32(np.where(np.isnan(sh) | (sh == 0), 0.0, sh)).view(np.uint8).reshape(n, 4 * ncomp)
    return rec, c64, sh, rec_deg, nread, ambiguous


def image(data, sh_degree: int = 0, **kw):
    """-> (.ksplat image, loose byte mask) of SplatBufferGenerator for the file: oracle.generate_oracle.generate on generator_inputs.
    The SH past the file's coefficients go in as NaN: the range scan's `!min ||` passes over NaN exactly as if the scan stopped at
    the file's coefficients, and the level-2 writer's `|| 0` writes NaN as 0, as it writes the missing coefficients."""
    rec, c64, sh, deg, nread, amb = generator_inputs(data, sh_degree)
    sh = sh.copy()
    sh[:, nread:] = np.nan
    return GO.generate(rec, c64, sh, deg, loose=amb, **kw)


# ---- writer (test inputs) ------------------------------------------------------------------------------------------------------------
def write_inriav2(splat_props, splat_cols: dict, count: int, cb_props, cb_cols: dict, rows: int, *, codebook_first=True) -> bytes:
    """props: [(name, type)] in file order; cols[name]: values (cast to the property's type; absent = zeros)."""
    def block(props, cols, m):
        dt = np.dtype([(k, _TYPES[t]) for k, t in props])
        r = np.zeros(m, dt)
        for k, _ in props:
            if k in cols:
                r[k] = np.asarray(cols[k]).astype(np.int64).astype(dt[k]) if dt[k].kind in "iu" else np.asarray(cols[k]).astype(dt[k])
        return r.tobytes()
    cb = [f"element codebook_centers {rows}", *[f"property {t} {k}" for k, t in cb_props]]
    sp = [f"element vertex {count}", *[f"property {t} {k}" for k, t in splat_props]]
    head = ["ply", "format binary_little_endian 1.0", *(cb + sp if codebook_first else sp + cb), "end_header"]
    body = [block(cb_props, cb_cols, rows), block(splat_props, splat_cols, count)]
    return ("\n".join(head) + "\n").encode("ascii") + b"".join(body if codebook_first else body[::-1])


def synthetic(n: int, seed: int, *, rows: int = 256, sh_rest: int = 45, index_type: str = "uchar", bad_index_rate: float = 0.0) -> bytes:
    """A v2 file like a compressed capture: half centres, a `rows`-row codebook of all 20 entries, every index field present."""
    rng = np.random.default_rng(seed)
    cb_props = [(k, "ushort") for k in PAGES]
    pages = {
        "features_dc": rng.normal(0, 1.0, rows), "opacity": rng.normal(0, 3.0, rows), "scaling": rng.uniform(-7, -2, rows),
        "rotation_re": rng.normal(0, 1, rows), "rotation_im": rng.normal(0, 1, rows),
        **{f"features_rest_{k}": rng.normal(0, 0.3, rows) for k in range(15)},
    }
    cb_cols = {k: v.astype(np.float16).view(np.uint16) for k, v in pages.items()}
    fields = ["scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3", "f_dc_0", "f_dc_1", "f_dc_2", "opacity"] + \
        [f"f_rest_{k}" for k in range(sh_rest)]
    props = [(k, "ushort") for k in "xyz"] + [(k, index_type) for k in fields]
    hi = rows + (int(rows * bad_index_rate / (1 - bad_index_rate)) + 1 if bad_index_rate else 0)
    cols = {k: rng.normal(0, 6, n).astype(np.float16).view(np.uint16) for k in "xyz"}
    cols.update({k: rng.integers(0, hi, n) for k in fields})
    return write_inriav2(props, cols, n, cb_props, cb_cols, rows)
