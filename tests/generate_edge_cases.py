"""Adversarial inputs for the SplatBuffer generator (gs_generate_splat_buffer) and the oracle-side checks that each one reaches the
branch it is built for.  Shared by tests/test_generate_edges.py (CPU: the checks and hand-derived anchors) and
tests/test_generate_edges_gpu.py (every byte of the GPU image against oracle/generate_oracle.py).

The generator restates sequential JavaScript loops (SplatBuffer.js:1177-1399) as parallel scans and stable sorts; these inputs put the
data where those restatements join their pieces:
  * SH range: k_gen_sh_scan gives each thread 8 splats and each CTA 2048; ShRun summaries join across threads (an ordered tree) and
    CTAs (k_gen_sh_final).  The values that make `if (!min || v < min)` differ from a plain min (0, -0, NaN, +-inf) sit at the first and
    last splat of a thread, of a CTA and of the file.
  * buckets: ids that collide across blocks (extents that are exact multiples of the block size), ids 2^32 - 2 and 2^32 - 1, many
    class-1 keys whose insertion order is not their key order, and groups of 50 000 identical centres at several bucket sizes.
  * sections: section sizes around the 2048 boundaries, whole sections emptied by alpha, a NaN first kept centre, and kept counts of
    4096 k +- 1 (the scan tile).
  * level-1 quantisers: a scale factor of exactly 1024 so that centre offsets land on .5 ties and past the [0, 65535] clamp, and half
    floats at every branch of three's toHalfFloat.
Each Case's `ran` asserts, on the oracle side only, that its branch was reached, and returns a count for the report."""
from __future__ import annotations

import dataclasses
import zlib
from typing import Callable

import numpy as np

from oracle import file_oracle as FO
from oracle import generate_oracle as GO

LEVELS = (0, 1, 2)
SH_THREAD, SH_CTA = 8, 2048                  # k_gen_sh_scan: splats per thread, per CTA
N_SH = 10 * SH_CTA + 37                      # ten full CTAs and a partial one
Q_BLOCK = 65534.0 / 1024.0                   # scale factor 32767 / (block / 2) = 1024 exactly


@dataclasses.dataclass
class Case:
    name: str
    fmt: int
    data: bytes
    sh_degree: int
    opts: list                               # generator options per run (compression_level, minimum_alpha, ...)
    ran: Callable[["Case"], int]             # oracle-side: asserts the case reaches its branch; -> how often


def inputs(case: Case):
    return GO.generator_inputs(case.fmt, case.data, case.sh_degree)


def levels(**kw):
    return [dict(kw, compression_level=lv) for lv in LEVELS]


# ---- writers --------------------------------------------------------------------------------------------------------------------------
_PLY_PROPS = [("x", "float"), ("y", "float"), ("z", "float")] + [(f"f_rest_{k}", "float") for k in range(45)] + \
             [("opacity", "float")] + [(f"scale_{k}", "float") for k in range(3)] + [(f"rot_{k}", "float") for k in range(4)] + \
             [(f"f_dc_{k}", "float") for k in range(3)]
# scan component s (FRC s of UncompressedSplatArray) of a degree-2 INRIA file (15 f_rest per channel): its f_rest column
_SRC = [(s % 3) + 15 * (s // 3) for s in range(9)] + [3 + (s % 5) + 15 * (s // 5) for s in range(15)]


def sh_ply(centers, frc, rot=None) -> bytes:
    """A degree-2 .ply: frc[n, 24] in FRC order; scale exp(0) = 1 and opacity 10 (alpha 254) for every splat, so no value depends on
    libm's exp; rotation (1, 0, 0, 0) unless given."""
    n = len(centers)
    cols = {"x": centers[:, 0], "y": centers[:, 1], "z": centers[:, 2], "opacity": np.full(n, 10.0), "rot_0": np.ones(n)}
    for s in range(24):
        cols[f"f_rest_{_SRC[s]}"] = frc[:, s]
    for k in range(45):
        cols.setdefault(f"f_rest_{k}", np.full(n, 0.75))
    if rot is not None:
        cols.update({f"rot_{k}": rot[:, k] for k in range(4)})
    cols.update({f"f_dc_{k}": np.linspace(-1, 1, n) * (k + 1) for k in range(3)})
    return FO.write_ply(_PLY_PROPS, cols, n)


def splat(centers, *, scales=None, alpha=None, seed=0) -> bytes:
    """A .splat whose colour bytes tell the splats apart (the file index in RGB) so that any reordering changes the image."""
    n = len(centers)
    i = np.arange(n)
    rgba = np.stack([i & 255, (i >> 8) & 255, (i >> 16) & 255, np.full(n, 255) if alpha is None else alpha], 1)
    rng = np.random.default_rng(seed)
    if scales is None:
        scales = rng.uniform(0.01, 0.5, (n, 3))
    return FO.write_splat(centers, scales, rgba, rng.integers(0, 256, (n, 4)))


# ---- section geometry and ids, restated for the checks (computeBucketsForUncompressedSplatArray's first loop) --------------------------
def geometry(c, block):
    """-> (min[3], yBlocks, zBlocks) of one section's centres in section order (strict comparisons from the first centre)."""
    mn, mx = [float(v) for v in c[0]], [float(v) for v in c[0]]
    for k in range(3):
        if mn[k] == mn[k]:
            col = c[:, k][~np.isnan(c[:, k])]
            mn[k], mx[k] = float(col.min()), float(col.max())
    with np.errstate(all="ignore"):
        return mn, float(np.ceil((mx[1] - mn[1]) / block)), float(np.ceil((mx[2] - mn[2]) / block))


def block_ids(c, block):
    """-> (xBlock/yBlock/zBlock f64[m, 3], bucketId f64[m], block centre f64[m, 3]) for one section's centres."""
    mn, yb, zb = geometry(c, block)
    with np.errstate(all="ignore"):
        b = np.floor((c - np.asarray(mn)) / block)
        ctr = (b * block + np.asarray(mn)) + block / 2.0
        bid = (b[:, 0] * (yb * zb) + b[:, 1] * zb) + b[:, 2]
    return b, bid, ctr


def sections(case: Case, kw):
    """-> [(section rows kept, in section order)] as GO.generate forms them."""
    rec, c64, _, _, _ = inputs(case)
    n = len(rec)
    order = GO.partition_order(c64, kw.get("scene_center", (0.0, 0.0, 0.0)))
    size = n if kw.get("section_size", 0) <= 0 else min(n, kw["section_size"])
    out = []
    for s in range(0 if n == 0 else -(-n // size)):
        rows = order[s * size:(s + 1) * size]
        out.append(rows[rec[rows, 43] >= kw.get("minimum_alpha", 1)])
    return out


def key_class(bid: float) -> int:
    return GO._key(bid)[0]


# ---- 1. SH range scan at thread and CTA boundaries ------------------------------------------------------------------------------------
def _sh_centers(n):
    c = np.zeros((n, 3))
    c[:, 0] = 0.5 * np.arange(n) + 0.25          # partition keys (0.5 i)^2: strictly increasing, so section order = file order
    return c


def _thread_last(t):
    return SH_THREAD * t + SH_THREAD - 1


def _cta_first(c):
    return SH_CTA * c


def _cta_last(c):
    return SH_CTA * c + SH_CTA - 1


def _sh_patterns():
    """name -> (degrees, fill(v, last) that edits the scan values v[n, nscan] in place, check(lo, hi, v) -> bool: the point of the case).
    `last` is the last scanned component (8 at degree 1, 22 at degree 2)."""
    def nanmin(v):
        return float(np.nanmin(v))

    def nanmax(v):
        return float(np.nanmax(v))

    def nonzero_min(v):
        w = v[~np.isnan(v) & (v != 0)]
        return float(w.min())

    P = {}

    def zero_at(at_splat, comp_last, neg=False):
        def fill(v, last):
            v[SH_CTA + 5, 3] = 0.01                                              # the least value, before the 0
            v[at_splat, last if comp_last else 0] = -0.0 if neg else 0.0
        return fill

    # a single 0 in an all-positive run: the running min falls to 0 and restarts from the next value
    sh_after_zero = (lambda lo, hi, v: lo != nanmin(v) and lo != nonzero_min(v) and lo >= 0.5)
    P["zero_thread_last"] = ((1, 2), zero_at(_thread_last(2 * SH_CTA // SH_THREAD + 9), True), sh_after_zero)
    P["negzero_thread_first"] = ((1, 2), zero_at(SH_THREAD * 301, False, neg=True), sh_after_zero)
    P["zero_cta_last"] = ((1, 2), zero_at(_cta_last(3), True), sh_after_zero)
    P["negzero_cta_first"] = ((1, 2), zero_at(_cta_first(5), False, neg=True), sh_after_zero)

    def zero_file_first(v, last):
        v[0, 0] = 0.0
        v[SH_CTA * 4 + 17, 2] = 0.01
    P["zero_file_first"] = ((1, 2), zero_file_first, lambda lo, hi, v: lo == np.float32(0.01) and nanmin(v) == 0.0)

    def zero_file_last(v, last):
        v[SH_CTA + 5, 3] = 0.01
        v[-1, last] = 0.0
    P["zero_file_last"] = ((1, 2), zero_file_last, lambda lo, hi, v: lo == -1.5 and nanmin(v) == 0.0)

    # 0, then smaller positives: the run after the 0 carries its own minimum (ShRun.C), within a thread and into the next CTA
    def zero_then_smaller_thread(v, last):
        v[5, 1] = 0.001
        t = 2 * 40                                                                # an even thread: joined as a left operand
        v[SH_THREAD * t + 2, 4] = 0.0
        v[SH_THREAD * t + 5, 1] = 0.02
        v[SH_THREAD * (t + 1) + 3, 0] = 0.03
    P["zero_then_smaller_thread"] = ((1, 2), zero_then_smaller_thread, lambda lo, hi, v: lo == np.float32(0.02) and nanmin(v) == 0.0)

    def zero_then_smaller_cta(v, last):
        v[5, 1] = 0.001
        v[_cta_last(3), last] = 0.0
        v[_cta_first(4):_cta_first(5)] = np.linspace(0.1, 0.05, SH_CTA)[:, None]
    P["zero_then_smaller_cta"] = ((1, 2), zero_then_smaller_cta, lambda lo, hi, v: lo == np.float32(0.05) and nanmin(v) == 0.0)

    # 0, then a negative (the running value restarts at the negative), and a negative, then 0 (a negative running value ignores the 0)
    def zero_then_negative(v, last):
        v[5, 1] = 0.001
        v[_cta_last(5), last] = 0.0
        v[_cta_first(6), 0] = -0.25
        v[SH_THREAD * 1601 + 3, 1] = -0.125
    P["zero_then_negative"] = ((1, 2), zero_then_negative, lambda lo, hi, v: lo == -0.25)

    def negative_then_zero_thread(v, last):
        t = 2 * SH_CTA // SH_THREAD + 127                                         # the last thread of a CTA's left half
        v[_thread_last(t), last] = -0.25
        v[_thread_last(t) + 1, 0] = 0.0
        v[_thread_last(t) + 1, 1] = 0.6
    P["negative_then_zero_thread"] = ((1, 2), negative_then_zero_thread, lambda lo, hi, v: lo == -0.25)

    def negative_then_zero_pair(v, last):
        t = 2 * 37 + 1                                                            # an odd thread, then the next (even) one
        v[_thread_last(t), last] = -0.25
        v[_thread_last(t) + 1, 0] = 0.0
    P["negative_then_zero_pair"] = ((1, 2), negative_then_zero_pair, lambda lo, hi, v: lo == -0.25)

    # the max side: a 0 inside an all-negative run
    def zero_in_negatives(v, last):
        v[:] = -v
        v[SH_CTA + 7, 2] = -0.01
        v[_thread_last(700), last] = 0.0
    P["max_zero_in_negatives"] = ((1, 2), zero_in_negatives,
                                  lambda lo, hi, v: hi != nanmax(v) and hi <= -0.5)

    # a whole CTA of NaN after a 0: the running value stays falsy across the CTA
    def nan_cta(v, last):
        v[SH_CTA + 5, 3] = 0.01
        v[_cta_last(2), last] = 0.0
        v[_cta_first(3):_cta_first(4)] = np.nan
        v[_cta_first(4):] = np.maximum(v[_cta_first(4):], 0.6)
    P["nan_cta"] = ((1, 2), nan_cta, lambda lo, hi, v: lo >= np.float32(0.6) and lo != nonzero_min(v))

    # a CTA whose only non-NaN value is a 0
    def zero_only_cta(v, last):
        v[SH_CTA + 5, 3] = 0.01
        v[_cta_first(5):_cta_first(6)] = np.nan
        v[_cta_first(5) + 1000, 3] = 0.0
        v[_cta_first(6):] = np.maximum(v[_cta_first(6):], 0.7)
    P["zero_only_cta"] = ((1, 2), zero_only_cta, lambda lo, hi, v: lo >= np.float32(0.7) and lo != nonzero_min(v))

    def infinities(v, last):
        v[_cta_first(2), 0] = np.inf
        v[_thread_last(1000), last] = -np.inf
        v[_cta_last(7), last] = 0.0
    P["infinities"] = ((1, 2), infinities, lambda lo, hi, v: lo == -np.inf and hi == np.inf)

    def subnormals(v, last):
        v[_cta_last(6), last] = 1e-45                                             # f32's least subnormal
        v[_cta_first(8), 0] = 3e-39
        v[_thread_last(2000), 2] = -1e-45
    P["subnormals"] = ((1, 2), subnormals, lambda lo, hi, v: lo == -np.float32(1e-45))

    def subnormal_after_zero(v, last):
        v[SH_CTA + 5, 3] = 0.01
        v[_cta_last(1), last] = 0.0
        v[_cta_first(2), 0] = 1e-45
    P["subnormal_after_zero"] = ((1, 2), subnormal_after_zero, lambda lo, hi, v: lo == np.float32(1e-45))
    return P


def _frc23_ply():
    """FRC23 (the last degree-2 coefficient) holds the extremes; the reference's scan stops before it."""
    n = N_SH
    rng = np.random.default_rng(23)
    frc = rng.uniform(0.5, 1.0, (n, 24)).astype(np.float32)
    frc[_cta_first(3), 23] = -100.0
    frc[_cta_last(9), 23] = 100.0
    frc[7, 12] = -50.0                                                            # read at degree 2, never at degree 1
    return sh_ply(_sh_centers(n), frc)


def sh_cases() -> list[Case]:
    out = []
    for name, (degrees, fill, check) in _sh_patterns().items():
        for deg in degrees:
            nscan = 9 if deg == 1 else 23
            rng = np.random.default_rng(zlib.crc32(name.encode()))
            frc = rng.uniform(0.5, 1.0, (N_SH, 24)).astype(np.float32).astype(np.float64)
            v = frc[:, :nscan]
            fill(v, nscan - 1)
            frc[:, :nscan] = v
            data = sh_ply(_sh_centers(N_SH), frc)

            def ran(case, check=check, nscan=nscan):
                _, c64, sh, _, _ = inputs(case)
                assert np.array_equal(GO.partition_order(c64), np.arange(len(c64))), "section order is not the file order"
                v = sh[:, :nscan]
                lo, hi = GO.sh_range(v)
                assert check(lo, hi, v), f"{case.name}: oracle range ({lo}, {hi}) does not show the pattern"
                return 1
            out.append(Case(f"sh_{name}_deg{deg}", FO.PLY, data, deg, levels(), ran))

    def ran23(case):
        _, _, sh, _, _ = inputs(case)
        lo, hi = GO.sh_range(sh)
        if case.sh_degree == 2:     # FRC12 is scanned, FRC23 is not
            assert lo == -50.0 and hi < 1.0 and np.nanmin(sh[:, 23]) == -100.0 and np.nanmax(sh[:, 23]) == 100.0
        else:                       # neither is read
            assert sh.shape[1] == 9 and 0.5 <= lo and hi < 1.0
        return 1
    data = _frc23_ply()
    for deg in (1, 2):
        out.append(Case(f"sh_frc23_unread_deg{deg}", FO.PLY, data, deg, levels(), ran23))
    return out


# ---- 2. bucket ids and order ---------------------------------------------------------------------------------------------------------
def _bucket_stats(case: Case, kw):
    """-> dict of counts over every section: cross-block collisions (a member whose own block centre is not its bucket's), groups whose
    buckets have different centres, class-1 partial buckets, and class-1 partial buckets out of key order."""
    _, c64, _, _, _ = inputs(case)
    block, bsize = kw.get("block_size", 5.0), kw.get("bucket_size", 256)
    st = dict(collide=0, recreated_elsewhere=0, class1_partial=0, class1_out_of_key_order=0, full=0, full_interleaved=0, class0_top=0,
              class1_first=0)
    for rows in sections(case, kw):
        if not len(rows):
            continue
        c = c64[rows]
        _, bid, ctr = block_ids(c, block)
        bl = GO.buckets(c, block, bsize)
        centres_by_key, partial_c1 = {}, []
        prev = None
        for members, centre in bl:
            key = GO._key(float(bid[members[0]]))
            own = ctr[members]
            st["collide"] += int((~np.all((own == np.asarray(centre)) | (np.isnan(own) & np.isnan(centre)), 1)).sum())
            centres_by_key.setdefault(key, set()).add(tuple(np.nan_to_num(centre, nan=1e300)))
            if len(members) >= bsize:
                st["full"] += 1
                st["full_interleaved"] += prev is not None and prev != key
                prev = key
            elif key[0] == 1:
                partial_c1.append(float(bid[members[0]]))
            st["class0_top"] += key == (0, 4294967294)
            st["class1_first"] += key == (1, repr(4294967295.0))
        st["recreated_elsewhere"] += sum(len(v) > 1 for v in centres_by_key.values())
        st["class1_partial"] += len(partial_c1)
        bits = [np.float64(b).view(np.uint64) if b == b else np.uint64(0x7FF8000000000000) for b in partial_c1]
        st["class1_out_of_key_order"] += sum(int(a > b) for a, b in zip(bits, bits[1:]))
    return st


def _lattice(flat_y: bool, reps: int, seed: int):
    """Integer lattice, block 1: extents are exact multiples of the block, so zBlock == zBlocks on the max face and ids collide across
    blocks ((x, y, zBlocks) is (x, y + 1, 0)).  flat_y: every y = 0, yBlocks = 0, and every x collides."""
    g = np.stack(np.meshgrid(np.arange(5.0), [0.0] if flat_y else np.arange(4.0), np.arange(5.0), indexing="ij"), -1).reshape(-1, 3)
    c = np.repeat(g, reps, 0)
    rng = np.random.default_rng(seed)
    return c[rng.permutation(len(c))]


def _class1_scene():
    """Corners (0, 0, 0) and (0, 65535, 65535) at block 1 make yBlocks zBlocks = 65535^2, so every splat with xBlock >= 1 has an id above
    2^32 - 2 (class 1).  Group k (k = 1..300, three identical members) sits at (k, 0, 40000 - 100 k): its id grows with k but its distance
    from the scene centre falls, so the partition inserts the groups in the reverse of their key order.  20 000 class-0 splats on the
    x = 0 face interleave with them, spreading the groups' first members over many CTAs.  Two +inf x (id +inf) and three NaN x (id NaN)
    join the class-1 keys; two splats sit on ids 2^32 - 2 (class 0, the largest index key) and 2^32 - 1 (class 1)."""
    rng = np.random.default_rng(31)
    rows = [(0.0, 0.0, 0.0), (0.0, 65535.0, 65535.0)]
    rows += [(0.0, float(y), float(z)) for y, z in rng.integers(0, 65536, (20_000, 2))]
    for k in range(1, 301):
        rows += [(float(k) + 0.25, 0.5, 40000.0 - 100 * k)] * 3
    rows += [(np.inf, 1.0, 1.0)] * 2 + [(np.nan, 1.0, 2.0)] * 3
    rows += [(1.0, 1.0, 65534.0), (1.0, 1.0, 65535.0), (1.5, 1.25, 65534.5)]
    c = np.asarray(rows)
    return c[rng.permutation(len(c))]


def _identical_groups():
    """Three groups of 50 000 identical centres, (1.1, 0, 0), (0, 1.1, 0) and (0, 0, 1.1): equal partition keys, so their members
    interleave in file order, and their buckets complete interleaved.  2 000 other splats in [0, 1.5)^3."""
    rng = np.random.default_rng(50)
    c = np.concatenate([np.repeat(np.eye(3) * 1.1, 50_000, 0), rng.uniform(0, 1.5, (2000, 3))])
    return c[rng.permutation(len(c))]


def bucket_cases() -> list[Case]:
    out = []

    def need(**want):
        """Each count, summed over the case's option sets (one bucket size may not show a collision another does), reaches its floor."""
        def ran(case):
            sums = dict.fromkeys(want, 0)
            for kw in case.opts:
                st = _bucket_stats(case, kw)
                for k in want:
                    sums[k] += st[k]
            for k, lowest in want.items():
                assert sums[k] >= lowest, f"{case.name}: {k} = {sums[k]} < {lowest}"
            return sum(sums.values())
        return ran

    lat = _lattice(False, 3, 1)
    out.append(Case("lattice_collisions", FO.SPLAT, splat(lat), 0,
                    [dict(o, block_size=1.0, bucket_size=b) for b in (2, 3, 255) for o in levels()],
                    need(collide=1, recreated_elsewhere=1)))
    flat = _lattice(True, 4, 2)
    out.append(Case("lattice_flat_y", FO.SPLAT, splat(flat), 0,
                    [dict(o, block_size=1.0, bucket_size=b) for b in (1, 2, 7) for o in levels()], need(collide=1, recreated_elsewhere=1)))
    c1 = _class1_scene()
    out.append(Case("class1_many", FO.SPLAT, splat(c1), 0,
                    [dict(o, block_size=1.0, bucket_size=b) for b in (2, 4, 1) for o in levels()[1:]] + [dict(compression_level=0, block_size=1.0, bucket_size=2)],
                    need(class1_partial=0, class0_top=1, class1_first=1)))
    out[-1].ran = _class1_ran(out[-1].ran)
    ig = _identical_groups()
    out.append(Case("identical_groups", FO.SPLAT, splat(ig), 0,
                    [dict(compression_level=lv, block_size=1.0, bucket_size=b) for b in (256, 4097) for lv in LEVELS] +
                    [dict(compression_level=1, block_size=1.0, bucket_size=b) for b in (1, 2, 255, 2**31)],
                    need(full=0)))
    out[-1].ran = _identical_ran(out[-1].ran)
    return out


def _class1_ran(base):
    def ran(case):
        total = base(case)
        st = _bucket_stats(case, dict(block_size=1.0, bucket_size=4))
        assert st["class1_partial"] >= 300 and st["class1_out_of_key_order"] >= 250, st
        rows = sections(case, dict())[0]
        _, bid, _ = block_ids(inputs(case)[1][rows], 1.0)
        first = {}
        for j, b in enumerate(bid):
            if key_class(b) == 1:
                first.setdefault(GO._key(float(b)), j)
        ctas = {j // 256 for j in first.values()}
        assert len(ctas) >= 20, f"class-1 first members in only {len(ctas)} CTAs"
        return total + st["class1_out_of_key_order"] + len(ctas)
    return ran


def _identical_ran(base):
    def ran(case):
        total = base(case)
        st = _bucket_stats(case, dict(block_size=1.0, bucket_size=256))
        assert st["full"] >= 3 * 195 and st["full_interleaved"] >= 100, st
        st1 = _bucket_stats(case, dict(block_size=1.0, bucket_size=2**31))
        assert st1["full"] == 0
        return total + st["full_interleaved"]
    return ran


# ---- 3. sections and alpha -----------------------------------------------------------------------------------------------------------
def _line(n, seed):
    """Centres x = 0.5 i + 0.25 (section order = file order) with y, z in [0, 0.5) (no effect on the partition key) for varied ids."""
    rng = np.random.default_rng(seed)
    c = rng.uniform(0.0, 0.5, (n, 3)).astype(np.float32).astype(np.float64)
    c[:, 0] = 0.5 * np.arange(n) + 0.25
    return c


def section_cases() -> list[Case]:
    out = []
    n = 6 * 2049 + 5
    for size in (1, 7, 2047, 2048, 2049):
        nsec = -(-n // size)
        rng = np.random.default_rng(size)
        alpha = rng.integers(100, 256, n)
        alpha[rng.random(n) < 0.05] = 40                                          # scattered removals
        sec = np.arange(n) // size
        empty = {0, 1, nsec // 2, nsec - 1} if size <= 7 else {0, nsec // 2, nsec - 1}
        alpha[np.isin(sec, list(empty))] = 99
        c = _line(n, size)

        def ran(case, size=size, empty=empty):
            secs = sections(case, case.opts[0])
            got = {s for s, rows in enumerate(secs) if len(rows) == 0}
            assert empty <= got and len(got) < len(secs), (sorted(got)[:8], sorted(empty))
            return len(got)
        out.append(Case(f"sections_{size}", FO.SPLAT, splat(c, alpha=alpha), 0,
                        [dict(o, section_size=size, minimum_alpha=100, block_size=0.125, bucket_size=3) for o in levels()], ran))

    # kept counts 4096 k +- 1 at four minimum alphas
    n = 8300
    alpha = np.concatenate([np.full(4095, 220), np.full(2, 160), np.full(4094, 120), np.full(2, 60), np.full(n - 8193, 10)])
    rng = np.random.default_rng(4096)
    alpha = alpha[rng.permutation(n)]

    def ran_kept(case):
        rec = inputs(case)[0]
        got = [int((rec[:, 43] >= kw["minimum_alpha"]).sum()) for kw in case.opts]
        assert sorted(set(got)) == [4095, 4097, 8191, 8193], got
        return len(got)
    out.append(Case("kept_4096k_pm1", FO.SPLAT, splat(_line(n, 7), alpha=alpha), 0,
                    [dict(compression_level=lv, minimum_alpha=a, block_size=0.1, bucket_size=b) for a in (200, 150, 100, 50)
                     for lv, b in ((1, 1), (2, 5), (0, 256))], ran_kept))

    # a section whose first kept centre has x = NaN, and later kept centres a finite x (and NaN y): the x bounds stay NaN
    fin = _line(300, 9)
    nanrows = np.zeros((40, 3))
    nanrows[:, 0] = np.arange(40) * 0.75 + 0.5
    nanrows[:, 1] = np.nan
    nanrows[:, 2] = np.arange(40) * 0.125
    nanrows[3, :] = (np.nan, 1.0, 0.25)                  # the first NaN-keyed splat alpha keeps
    nanrows[9, :] = (np.nan, 2.0, np.nan)
    c = np.concatenate([fin, nanrows])
    alpha = np.full(len(c), 200)
    alpha[300:303] = 5                                     # NaN-keyed splats removed ahead of it

    def ran_nan(case):
        kw = case.opts[0]
        rows = sections(case, kw)[1]
        c64 = inputs(case)[1]
        assert np.isnan(c64[rows[0], 0]) and np.isfinite(c64[rows[1:], 0]).sum() >= 30
        assert np.isnan(geometry(c64[rows], 1.0)[0][0])
        return 1
    out.append(Case("nan_first_kept", FO.SPLAT, splat(c, alpha=alpha), 0,
                    [dict(o, section_size=300, minimum_alpha=100, block_size=1.0, bucket_size=2) for o in levels()], ran_nan))
    return out


# ---- 4. level-1 quantisers -----------------------------------------------------------------------------------------------------------
def _offset_stats(case: Case, kw):
    """-> (ties, negative ties, clamped low, clamped high, exactly at 65535) of (c - bucketCentre) * 1024 + 32767 over every splat."""
    _, c64, _, _, _ = inputs(case)
    sf = GO.SCALE_RANGE / (kw["block_size"] * 0.5)
    t = [0] * 5
    for rows in sections(case, kw):
        for members, centre in GO.buckets(c64[rows], kw["block_size"], kw["bucket_size"]):
            d = (c64[rows][members] - np.asarray(centre)) * sf
            d = d[np.isfinite(d)]
            frac = d - np.floor(d)
            v = GO._js_round(d) + GO.SCALE_RANGE
            t[0] += int((frac == 0.5).sum())
            t[1] += int(((frac == 0.5) & (d < 0)).sum())
            t[2] += int((v < 0).sum())
            t[3] += int((v > 65535).sum())
            t[4] += int((v == 65535).sum())
    return t


def _quant_scene():
    """Block 65534 / 1024 (scale factor 1024), min (0, 0, 0), extents (2 block, block, 2 block): yBlocks = 1, zBlocks = 2.  Block (0, 0, 0)
    has centre h = 32767 / 1024 on each axis; x = h + k / 2048 puts the offset on k / 2 (a tie for odd k), both signs.  Splats at
    (x, 0, 2 block) and (x, block, 0) share id 2, so one bucket holds both blocks: offsets of +-1.5 blocks, past the clamp.  Offsets of
    The id-3 family sits on the clamp: P0 = (0, B, B + 1) creates the bucket (centre (h, B + h, B + h)); (x, 0, B + 1) with x in x-block 1
    has the same id (the y-max face of x-block 0 is x-block 1's y = 0) and x offsets of 32767.5, 32768 and 32768.5 / 1024 (65535 after a
    tie, exactly 65535, and 65536 clamped)."""
    B, h = Q_BLOCK, 32767.0 / 1024.0
    rows = [(0.0, 0.0, 0.0), (2 * B, B, 2 * B)]
    ks = np.concatenate([np.arange(-65533, 65534, 911), [-1, 1, -3, 3, -5, 5, 65533, -65533, 65532]])
    rows += [(h + k / 2048.0, h, h - k / 2048.0) for k in ks]
    for k in range(0, 64, 3):
        rows += [(k / 16.0, 0.0, 2 * B), (k / 16.0 + 1 / 2048.0, B, 0.0)]
    c = np.asarray(rows, np.float32).astype(np.float64)
    rng = np.random.default_rng(1024)
    edge = [(0.0, B, B + 1.0), (65534.5 / 1024.0, 0.0, B + 1.0), (65535.0 / 1024.0, 0.0, B + 1.0), (65535.5 / 1024.0, 0.0, B + 1.0)]
    return np.concatenate([np.asarray(edge, np.float32), c[rng.permutation(len(c))]])     # equal partition keys: P0 first


_HALF_VALUES = np.array([2.0**-25, 2.0**-24, 3 * 2.0**-26, 2.0**-14, np.nextafter(np.float32(2.0**-14), np.float32(0)),
                         np.nextafter(np.float32(2.0**-14), np.float32(1)), 65504.0, 65505.0, 65519.0, 65520.0, np.inf, np.nan, 0.0,
                         2.0**-26, 2.0**-27, 2.0**-28, 1e-45, 1.0, 1 + 2.0**-11, 1 + 2.0**-11 + 2.0**-23, 1 + 2.0**-10 - 2.0**-23,
                         2.0**15 + 2.0**4 - 2.0**-8, 0.333, 3 * 2.0**-25, 5 * 2.0**-26, 2.0**-15 + 2.0**-24 + 2.0**-25], np.float64)


def _rn_half_bits(v):
    with np.errstate(all="ignore"):
        return np.clip(np.asarray(v, np.float32), -65504, 65504).astype(np.float16).view(np.uint16)


def quant_cases() -> list[Case]:
    out = []

    def ran_offsets(case):
        t = _offset_stats(case, case.opts[0])
        assert t[0] >= 20 and t[1] >= 10 and t[2] >= 10 and t[3] >= 10 and t[4] >= 1, t
        return sum(t)
    qc = _quant_scene()
    out.append(Case("quant_ties_and_clamp", FO.SPLAT, splat(qc), 0,
                    [dict(compression_level=lv, block_size=Q_BLOCK, bucket_size=b) for lv in (1, 2) for b in (256, 3)] +
                    [dict(compression_level=0, block_size=Q_BLOCK, bucket_size=256)], ran_offsets))

    # .splat scales: every toHalfFloat branch, both signs (the writer's `|| 0` makes NaN 0)
    v = np.concatenate([_HALF_VALUES, -_HALF_VALUES])
    n = len(v)
    scales = np.stack([v, np.roll(v, 7), np.roll(v, 19)], 1)
    c = np.stack([np.arange(n) * 0.5 + 0.25, np.zeros(n), np.zeros(n)], 1)

    def ran_half(case):
        rec = inputs(case)[0]
        f = rec[:, 12:24].copy().view(np.float32).astype(np.float64).ravel()
        trunc, rn = GO._half(f), _rn_half_bits(f)
        differ = int((trunc != rn).sum())
        assert differ >= 10, differ
        return differ
    out.append(Case("half_scales", FO.SPLAT, splat(c, scales=scales), 0, levels(), ran_half))

    # .ply: SH coefficients at the same values (level-1 halves; the writer's `|| 0` makes NaN 0) and NaN rotations (the NaN half)
    m = 64
    frc = np.resize(np.concatenate([_HALF_VALUES, -_HALF_VALUES]), (m, 24))
    rot = np.tile([1.0, 0.0, 0.0, 0.0], (m, 1))
    rot[::5, 0] = np.nan
    rot[1::7, 2] = np.inf

    def ran_half_ply(case):
        rec = inputs(case)[0]
        q = rec[:, 24:40].copy().view(np.float32)
        assert np.isnan(q).any()
        if case.sh_degree == 0:
            return int(np.isnan(q).sum())
        sh = rec[:, 44:].copy().view(np.float32).astype(np.float64).ravel()
        differ = int((GO._half(sh) != _rn_half_bits(sh)).sum())
        assert differ >= 10, differ
        return differ
    data = sh_ply(_sh_centers(m), frc, rot=rot)
    for deg in (0, 1, 2):
        out.append(Case(f"half_sh_rot_deg{deg}", FO.PLY, data, deg, levels(), ran_half_ply))
    return out


def all_cases() -> list[Case]:
    return sh_cases() + bucket_cases() + section_cases() + quant_cases()


# ---- 5. hand-derived anchors ---------------------------------------------------------------------------------------------------------
def anchor_scan_ply() -> bytes:
    """One degree-1 splat whose nine scanned values are 3, 0, 5, 2 and five NaN: min 3 -> 0 -> 5 (replaces the falsy 0) -> 2; max 3 -> 5.
    The range is (2, 5); a nanmin would give 0."""
    frc = np.full((1, 24), np.nan)
    frc[0, :4] = (3.0, 0.0, 5.0, 2.0)
    return sh_ply(np.zeros((1, 3)), frc)


# Two splats whose ids collide across blocks: block 1, extents (0, 1, 1) so yBlocks = zBlocks = 1.  A = (0, 0, 1) is in block (0, 0, 1),
# id 0 + 0 + 1 = 1; B = (0, 1, 0) is in block (0, 1, 0), id 0 + 1 + 0 = 1.  Both keys are 1.0 (a tie: file order A, B), so A creates the
# bucket and its centre is A's block centre (0.5, 0.5, 1.5).  Level 1 (scale factor 65534): A's offsets (-0.5, -0.5, -0.5) become
# -32767 + 32767 = 0 on each axis; B's (-0.5, 0.5, -1.5) become 0, 32767 + 32767 = 65534 and clamp(-98301 + 32767) = 0.
ANCHOR_COLLIDE = np.array([[0.0, 0.0, 1.0], [0.0, 1.0, 0.0]])
ANCHOR_COLLIDE_CENTRE = (0.5, 0.5, 1.5)
ANCHOR_COLLIDE_Q = [(0, 0, 0), (0, 65534, 0)]

# Class-1 keys come out in insertion order.  Block 1; the section's centres (in section order) with min (0, 0, 0), max y = z = 1, so
# yBlocks = zBlocks = 1 and id = xBlock + yBlock + zBlock:
#   (0, 0, 0) id 0; (nan, 0, 0) id NaN; (inf, 0, 0) id inf; (5e9, 0, 0) id 5e9 (above 2^32 - 2); (0, 1, 1) id 2; (nan, 1, 0) id NaN again
# Partial buckets: index keys ascending (0, 2), then NaN, inf, 5e9 as first inserted; NaN holds rows 1 and 5.
ANCHOR_CLASS1 = np.array([[0.0, 0.0, 0.0], [np.nan, 0.0, 0.0], [np.inf, 0.0, 0.0], [5e9, 0.0, 0.0], [0.0, 1.0, 1.0], [np.nan, 1.0, 0.0]])
ANCHOR_CLASS1_BUCKETS = [[0], [4], [1, 5], [2], [3]]


def anchor_class1_splat():
    """The class-1 anchor through the partition: scene centre (5e9, 0, 0) puts the 5e9 splat first (key 0), then the three finite splats
    near the origin (keys 2.5e19 in file order), the inf splat (key inf) and the NaN splats last.  Insertion order of the class-1 keys:
    5e9, inf, NaN; partial buckets: ids 0, 2, then 5e9, inf, NaN."""
    c = np.array([[0.0, 0.0, 0.0], [np.nan, 0.0, 0.0], [np.inf, 0.0, 0.0], [5e9, 0.0, 0.0], [0.0, 1.0, 1.0], [np.nan, 1.0, 0.0]])
    return splat(c), dict(block_size=1.0, bucket_size=256, scene_center=(5e9, 0.0, 0.0))
