"""The vertex stage (SplatMaterial.js:112-341, SplatMaterial3D.js:83-216, fade-in SplatMaterial.js:347-363) restated in float64, with a
per-splat bound on the error of ANY float32 evaluation of the same expressions.  Test infrastructure: nothing here is imported from the
product or from oracle/raster_oracle.c.

Every intermediate is an `Ev`: the f64 value of the expression on the f32 inputs, and an absolute bound on how far an f32 evaluation
can be from it.  The bound is first-order running error analysis with u = 2^-24:
  * sums and dot products of n terms: gamma_n * sum |terms| -- holds for any summation order and for FMA contraction;
  * multiply, divide, sqrt: correctly rounded (no fast-math), one u each; a division is charged as reciprocal + multiply, which also
    covers the shader's x / w written as x * (1 / w);
  * rsqrt: 2 ulp (CUDA maths accuracy table), charged as 4 u of the result;
  * constants enter as their f32 values; half and 8-bit inputs widen exactly;
  * min, max, clamp are 1-Lipschitz: they pass the larger bound on;
  * inverse(transform): cofactors bounded by gamma_7 times the permanent of the absolute minor, then the determinant and scaling.
Input errors propagate first order plus the product of the bounds.

Discontinuous decisions (the cull planes, minAlpha, l2 <= 0, ndc z in [-1, 1]) are evaluated on the f64 value; a splat whose operand
lies within its bound of the threshold is `ambiguous`, and so is a splat whose first eigenvector is undetermined: normalize(b, l1 - a)
when the bound on (b, l1 - a) reaches its length (b ~ 0 with a > d + 0.63 px^2: an f32 evaluation, the reference's included, gets a
direction decided by rounding).

`project` returns, per splat, value and bound of cx, cy, ndc_z, r, g, b, a and of the quad's quadratic form Q = B1 B1^T + B2 B2^T
(qxx, qxy, qyy: free of e1's sign), the expected `valid` and `ambiguous`.  The quad fields include the export's reconstruction
B = g / |g|^2 from g = e / s (k_export_projected)."""
from __future__ import annotations

import numpy as np

U = 2.0 ** -24
MAX_SCENES = 32
F = np.float32


def gamma(n: int) -> float:
    return n * U / (1.0 - n * U)


class Ev:
    """f64 value and absolute error bound of one intermediate, elementwise over splats."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=0.0):
        self.v = np.asarray(v, np.float64)
        self.e = np.asarray(e, np.float64)

    @property
    def mag(self):
        return np.abs(self.v) + self.e

    def take(self, idx):
        return Ev(self.v[idx], self.e[idx] if self.e.ndim else self.e)

    def neg(self):
        return Ev(-self.v, self.e)


def const(c) -> Ev:
    """A literal as the f32 value it has in the kernel."""
    return Ev(np.float64(F(c)), 0.0)


def _round(v, prop, k=1.0):
    return prop + k * U * (np.abs(v) + prop)


def add(a: Ev, b: Ev, sign: float = 1.0) -> Ev:
    v = a.v + sign * b.v
    return Ev(v, _round(v, a.e + b.e))


def mul(a: Ev, b: Ev) -> Ev:
    v = a.v * b.v
    return Ev(v, _round(v, np.abs(a.v) * b.e + np.abs(b.v) * a.e + a.e * b.e))


def dot(xs, ys) -> Ev:
    """sum x_i y_i over n terms, any order, fused or not."""
    v = sum(x.v * y.v for x, y in zip(xs, ys))
    prop = sum(np.abs(x.v) * y.e + np.abs(y.v) * x.e + x.e * y.e for x, y in zip(xs, ys))
    return Ev(v, prop + gamma(len(xs)) * sum(x.mag * y.mag for x, y in zip(xs, ys)))


def recip(a: Ev) -> Ev:
    with np.errstate(divide="ignore", invalid="ignore"):
        v = 1.0 / a.v
        lo = np.abs(a.v) - a.e
        prop = np.where(lo > 0, a.e / (np.abs(a.v) * np.where(lo > 0, lo, 1.0)), np.inf)
    return Ev(v, _round(v, prop))


def div(a: Ev, b: Ev) -> Ev:
    return mul(a, recip(b))


def sqrt(a: Ev) -> Ev:
    x = np.maximum(a.v, 0.0)
    v = np.sqrt(x)
    den = v + np.sqrt(np.maximum(x - a.e, 0.0))
    with np.errstate(divide="ignore", invalid="ignore"):
        prop = np.minimum(np.sqrt(a.e), np.where(den > 0, a.e / np.where(den > 0, den, 1.0), np.inf))
    return Ev(v, _round(v, prop))


def rsqrt(a: Ev) -> Ev:
    with np.errstate(divide="ignore", invalid="ignore"):
        v = 1.0 / np.sqrt(a.v)
        lo = a.v - a.e
        prop = np.where(lo > 0, 1.0 / np.sqrt(np.where(lo > 0, lo, 1.0)) - v, np.inf)
    return Ev(v, _round(v, prop, 4.0))


def fmin(a: Ev, b: Ev) -> Ev:
    return Ev(np.minimum(a.v, b.v), np.maximum(a.e, b.e))


def fmax(a: Ev, b: Ev) -> Ev:
    return Ev(np.maximum(a.v, b.v), np.maximum(a.e, b.e))


def clamp01(a: Ev) -> Ev:
    return Ev(np.clip(a.v, 0.0, 1.0), a.e)


def near(x: Ev, t: Ev):
    """The decision x < t (or <=) is not determined by an f32 evaluation."""
    return np.abs(x.v - t.v) <= x.e + t.e


# ---- 4x4 matrices, column-major lists of 16 Ev --------------------------------------------------------------------------------------
def _mat_in(m16) -> list:
    m = np.asarray(m16, np.float32).reshape(-1, 16).astype(np.float64)
    return [Ev(m[:, k], 0.0) for k in range(16)]


def _mat_mul(a, b) -> list:
    return [dot([a[r], a[4 + r], a[8 + r], a[12 + r]], [b[4 * c], b[4 * c + 1], b[4 * c + 2], b[4 * c + 3]]) for c in range(4) for r in range(4)]


def _perm3(m):
    return (m[..., 0, 0] * (m[..., 1, 1] * m[..., 2, 2] + m[..., 1, 2] * m[..., 2, 1])
            + m[..., 0, 1] * (m[..., 1, 0] * m[..., 2, 2] + m[..., 1, 2] * m[..., 2, 0])
            + m[..., 0, 2] * (m[..., 1, 0] * m[..., 2, 1] + m[..., 1, 1] * m[..., 2, 0]))


def _mat_inverse(m16) -> list:
    """GLSL inverse() of [S, 16] column-major f32 matrices: cofactor expansion, determinant from the first column, scaled by 1 / det."""
    m = np.asarray(m16, np.float32).reshape(-1, 16).astype(np.float64)
    M = m.reshape(-1, 4, 4).transpose(0, 2, 1)                     # M[s, row, col]
    cof = [None] * 16
    for r in range(4):
        for c in range(4):
            minor = np.delete(np.delete(M, c, axis=1), r, axis=2)  # adj[r][c] = (-1)^(r+c) det(M without row c, column r)
            val = (-1.0) ** (r + c) * np.linalg.det(minor)
            cof[4 * c + r] = Ev(val, gamma(7) * _perm3(np.abs(minor)))
    mcol = [Ev(m[:, k], 0.0) for k in range(16)]
    det = dot([mcol[0], mcol[1], mcol[2], mcol[3]], [cof[0], cof[4], cof[8], cof[12]])
    idet = recip(det)
    return [mul(x, idet) for x in cof]


def _transform_point(m, p) -> list:
    one = Ev(1.0, 0.0)
    return [dot([m[r], m[4 + r], m[8 + r], m[12 + r]], [p[0], p[1], p[2], one]) for r in range(4)]


def _half_or_f32(a):
    return np.asarray(a).astype(np.float64) if np.asarray(a).dtype == np.float16 else np.asarray(a, np.float32).astype(np.float64)


def _get(u, name, default):
    x = getattr(u, name, None)
    return default if x is None else x


# ---- the vertex stage ---------------------------------------------------------------------------------------------------------------
def project(u, centers_colors, covariances, sh=None, sh_degree=0, scene_indexes=None) -> dict:
    """`u`: the uniforms as plain attributes (the names of engine.Uniforms).  centers_colors u32 [n,4], covariances f32 / f16 [n,6], sh
    f16 / u8 / f32 [n, 9 or 24] of data degree `sh_degree`, scene_indexes u32 [n] or None.  `stats` says which branches each splat took:
    min_alpha_cut, aa_factor, clamped (a basis length at the max size), fade (the fade-in factor), direction_undetermined."""
    with np.errstate(all="ignore"):          # culled splats run through the arithmetic too; their values are never used
        return _project(u, centers_colors, covariances, sh, sh_degree, scene_indexes)


def _project(u, centers_colors, covariances, sh, sh_degree, scene_indexes) -> dict:
    cc = np.ascontiguousarray(centers_colors, np.uint32).reshape(-1, 4)
    n = cc.shape[0]
    ctr = cc[:, 1:].copy().view(np.float32).astype(np.float64)
    c = [Ev(ctr[:, k], 0.0) for k in range(3)]
    scene_count = int(_get(u, "scene_count", 1))
    scene = np.zeros(n, np.int64)
    if scene_count > 1 and scene_indexes is not None:
        scene = np.asarray(scene_indexes, np.int64) & (MAX_SCENES - 1)
    valid = np.ones(n, bool)
    amb = np.zeros(n, bool)
    stats = dict(min_alpha_cut=np.zeros(n, bool), aa_factor=np.ones(n), clamped=np.zeros(n, bool), fade=np.ones(n),
                 direction_undetermined=np.zeros(n, bool))

    opacity = np.asarray(_get(u, "scene_opacity", np.ones(MAX_SCENES)), np.float32).astype(np.float64)
    visibility = np.asarray(_get(u, "scene_visibility", np.ones(MAX_SCENES)), np.int64)
    effects = bool(_get(u, "enable_optional_effects", 0))
    if effects:                                                     # SplatMaterial.js:124-133: exact f32 comparison of a uniform
        valid &= ~((opacity[scene] <= np.float64(F(0.01))) | (visibility[scene] == 0))

    dynamic = bool(_get(u, "dynamic_mode", 0))
    transforms = np.asarray(_get(u, "scene_transforms", np.tile(np.eye(4, dtype=np.float32).reshape(16), MAX_SCENES)), np.float32).reshape(MAX_SCENES, 16)
    if dynamic:                                                     # SplatMaterial.js:136-146: viewMatrix * transforms[scene]
        view_m = _mat_in(_get(u, "view_matrix", np.eye(4, dtype=np.float32)))
        mv_s = _mat_mul(view_m, _mat_in(transforms))
        mv = [x.take(scene) for x in mv_s]
    else:
        mv = [Ev(x.v[0], 0.0) for x in _mat_in(u.model_view)]
    proj = [Ev(x.v[0], 0.0) for x in _mat_in(u.projection)]

    view = _transform_point(mv, c)
    clip = [dot([proj[r], proj[4 + r], proj[8 + r], proj[12 + r]], view) for r in range(4)]
    lim = mul(const(1.2), clip[3])                                  # SplatMaterial.js:160-164
    mlim = lim.neg()
    cull = (clip[2].v < mlim.v) | (clip[0].v < mlim.v) | (clip[0].v > lim.v) | (clip[1].v < mlim.v) | (clip[1].v > lim.v)
    amb |= valid & (near(clip[2], mlim) | near(clip[0], mlim) | near(clip[0], lim) | near(clip[1], mlim) | near(clip[1], lim))
    valid &= ~cull
    iw = recip(clip[3])
    ndcx, ndcy, ndcz = mul(clip[0], iw), mul(clip[1], iw), mul(clip[2], iw)

    rgba = np.stack([(cc[:, 0] >> (8 * k)) & 255 for k in range(4)], 1).astype(np.float64)
    col = [Ev(rgba[:, k] / 255.0, 2.0 * U * rgba[:, k] / 255.0) for k in range(4)]     # byte * (1/255): constant + product rounding

    udeg = int(_get(u, "sh_degree", 0))
    if sh is not None and sh_degree >= 1 and udeg >= 1:
        s = np.asarray(sh)
        nuse = 24 if (sh_degree >= 2 and udeg >= 2) else 9
        if s.dtype == np.uint8:                                     # SplatMaterial.js: sh * range + min, per scene
            lo = np.asarray(_get(u, "sh8_min", np.full(MAX_SCENES, -1.5)), np.float32).astype(np.float64)
            hi = np.asarray(_get(u, "sh8_max", np.full(MAX_SCENES, 1.5)), np.float32).astype(np.float64)
            rng = add(Ev(hi, 0.0), Ev(lo, 0.0), -1.0).take(scene)
            shv = [add(mul(div(Ev(s[:, k].astype(np.float64), 0.0), const(255.0)), rng), Ev(lo[scene], 0.0)) for k in range(nuse)]
        else:
            w = _half_or_f32(s)
            shv = [Ev(w[:, k], 0.0) for k in range(nuse)]
        cam = [Ev(np.float64(F(x)), 0.0) for x in np.asarray(u.camera_position, np.float32).reshape(3)]
        if dynamic:                                                 # SplatMaterial.js:181-183: inverse(transform) * cameraPosition
            inv = _mat_inverse(transforms)
            camt = _transform_point(inv, [Ev(np.full(MAX_SCENES, x.v), 0.0) for x in cam])
            cam = [x.take(scene) for x in camt[:3]]
        d = [add(c[k], cam[k], -1.0) for k in range(3)]
        il = rsqrt(dot(d, d))
        x, y, z = (mul(d[k], il) for k in range(3))
        C1 = const(0.4886025119029199)
        for ch in range(3):
            col[ch] = add(col[ch], mul(C1, dot([shv[ch], shv[3 + ch], shv[6 + ch]], [y.neg(), z, x.neg()])))
        if nuse == 24:
            xx, yy, zz, xy, yz, xz = mul(x, x), mul(y, y), mul(z, z), mul(x, y), mul(y, z), mul(x, z)
            two_zz = mul(const(2.0), zz)
            w6 = dot([two_zz, xx, yy], [const(1.0), const(-1.0), const(-1.0)])
            w8 = add(xx, yy, -1.0)
            k = [mul(const(1.0925484), xy), mul(const(-1.0925484), yz), mul(const(0.3153916), w6), mul(const(-1.0925484), xz), mul(const(0.5462742), w8)]
            for ch in range(3):
                col[ch] = add(col[ch], dot(k, [shv[9 + ch], shv[12 + ch], shv[15 + ch], shv[18 + ch], shv[21 + ch]]))
        for ch in range(3):
            col[ch] = clamp01(col[ch])

    V = _half_or_f32(covariances)
    Vk = [Ev(V[:, k], 0.0) for k in range(6)]
    if int(_get(u, "orthographic_mode", 0)) == 1:                   # SplatMaterial3D.js:117-122
        j00 = j11 = const(_get(u, "ortho_zoom", 1.0))
        j02 = j12 = Ev(0.0, 0.0)
    else:
        iz = recip(view[2])
        sc = mul(iz, iz)
        f0, f1 = const(u.focal[0]), const(u.focal[1])
        j00, j11 = mul(f0, iz), mul(f1, iz)
        j02, j12 = mul(mul(f0, view[0]), sc).neg(), mul(mul(f1, view[1]), sc).neg()
    T0 = [dot([mv[4 * k], mv[4 * k + 2]], [j00, j02]) for k in range(3)]           # T = transpose(mat3(MV)) * J, columns 0 and 1
    T1 = [dot([mv[4 * k + 1], mv[4 * k + 2]], [j11, j12]) for k in range(3)]
    S = [[Vk[0], Vk[1], Vk[2]], [Vk[1], Vk[3], Vk[4]], [Vk[2], Vk[4], Vk[5]]]
    VT0 = [dot(S[r], T0) for r in range(3)]
    VT1 = [dot(S[r], T1) for r in range(3)]
    a, b, dd = dot(T0, VT0), dot(T0, VT1), dot(T1, VT1)

    k2 = const(_get(u, "kernel_2d_size", 0.3))
    min_alpha = const(1.0 / 255.0)
    if int(_get(u, "antialiased", 0)):                              # SplatMaterial3D.js:137-145
        det0 = dot([a, b], [dd, b.neg()])
        a, dd = add(a, k2), add(dd, k2)
        det1 = dot([a, b], [dd, b.neg()])
        factor = sqrt(fmax(div(det0, det1), Ev(0.0, 0.0)))
        col[3] = mul(col[3], factor)
        amb |= valid & near(col[3], min_alpha)
        stats["aa_factor"] = factor.v
        stats["min_alpha_cut"] = valid & (col[3].v < min_alpha.v)
        valid &= ~(col[3].v < min_alpha.v)
    else:
        a, dd = add(a, k2), add(dd, k2)

    D = dot([a, b], [dd, b.neg()])                                   # :174-196 eigen split
    half_tr = mul(const(0.5), add(a, dd))
    term2 = sqrt(fmax(const(0.1), dot([half_tr, D], [half_tr, const(-1.0)])))
    l1, l2 = add(half_tr, term2), add(half_tr, term2, -1.0)
    if int(_get(u, "point_cloud_mode", 0)) == 1:
        l1 = l2 = const(0.2)
    zero = Ev(0.0, 0.0)
    amb |= valid & near(l2, zero)
    valid &= ~(l2.v <= 0.0)

    ex_, ey_ = b, add(l1, a, -1.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        length = np.hypot(ex_.v, ey_.v)
        dlen = np.hypot(ex_.e, ey_.e)
        undetermined = ~(dlen < length)
        amb |= valid & undetermined
        stats["direction_undetermined"] = valid & undetermined
        e_dir = np.where(undetermined, np.inf, np.minimum(2.0 * dlen / np.where(length > 0, length, 1.0), 2.0)) + 8.0 * U
        ex = Ev(ex_.v / length, e_dir)
        ey = Ev(ey_.v / length, e_dir)

    sqrt8 = const(2.8284271247461903)
    mx = const(_get(u, "max_screen_space_splat_size", 1024.0))
    scale = const(_get(u, "splat_scale", 1.0))
    ifa = const(_get(u, "inverse_focal_adjustment", 1.0))
    r1, r2 = mul(sqrt8, sqrt(l1)), mul(sqrt8, sqrt(l2))
    stats["clamped"] = valid & (r1.v > mx.v)
    s1 = mul(mul(scale, fmin(r1, mx)), ifa)
    s2 = mul(mul(scale, fmin(r2, mx)), ifa)
    if effects:                                                     # SplatMaterial3D.js:198-202
        col[3] = mul(col[3], Ev(opacity[scene], 0.0))
    if not int(_get(u, "fade_in_complete", 1)):                     # SplatMaterial.js:347-363
        sc3 = [const(x) for x in _get(u, "scene_center", (0.0, 0.0, 0.0))]
        q = [add(c[k], sc3[k], -1.0) for k in range(3)]
        dist = sqrt(dot(q, q))
        fs = const(_get(u, "visible_region_fade_start_radius", 0.0))
        ramp = add(const(1.0), clamp01(div(add(dist, fs, -1.0), const(0.75))), -1.0)
        st = dist.v >= fs.v                                         # the factor is 1 on both sides of the step: no decision to flag
        col[3] = mul(col[3], Ev(np.where(st, ramp.v, 1.0), np.where(st, ramp.e, 0.0)))
        stats["fade"] = np.where(st, ramp.v, 1.0)

    vp = [const(x) for x in u.viewport]
    half = const(0.5)
    cx = mul(mul(add(ndcx, const(1.0)), half), vp[0])
    cy = mul(mul(add(ndcy, const(1.0)), half), vp[1])

    b1x, b1y, b2x, b2y = mul(ex, s1), mul(ey, s1), mul(ey, s2), mul(ex.neg(), s2)
    qxx, qxy, qyy = dot([b1x, b2x], [b1x, b2x]), dot([b1x, b2x], [b1y, b2y]), dot([b1y, b2y], [b1y, b2y])
    # the record stores g = e / s and the export rebuilds B = g / |g|^2: a few u on every component of B, twice that on Q's terms
    ex_u = 24.0 * U
    qxx.e = qxx.e + ex_u * (b1x.mag ** 2 + b2x.mag ** 2)
    qxy.e = qxy.e + ex_u * (b1x.mag * b1y.mag + b2x.mag * b2y.mag)
    qyy.e = qyy.e + ex_u * (b1y.mag ** 2 + b2y.mag ** 2)

    amb |= valid & (near(ndcz, const(-1.0)) | near(ndcz, const(1.0)))
    valid &= (ndcz.v >= -1.0) & (ndcz.v <= 1.0)
    with np.errstate(invalid="ignore"):
        valid &= np.isfinite(s1.v) & np.isfinite(s2.v) & (s1.v > 0) & (s2.v > 0)     # the kernel's extra drop of degenerate quads

    out = dict(valid=valid, ambiguous=amb, stats=stats)
    for name, x in (("cx", cx), ("cy", cy), ("ndc_z", ndcz), ("r", col[0]), ("g", col[1]), ("b", col[2]), ("a", col[3]),
                    ("qxx", qxx), ("qxy", qxy), ("qyy", qyy)):
        out[name] = np.broadcast_to(x.v, (n,)).astype(np.float64)
        out[name + "_bound"] = np.broadcast_to(x.e, (n,)).astype(np.float64)
    return out


FIELDS = ("cx", "cy", "ndc_z", "r", "g", "b", "a", "qxx", "qxy", "qyy")


def quad_form(ps) -> dict:
    """Q = B1 B1^T + B2 B2^T of exported records (gs_projected_splat), in f64."""
    b1x, b1y, b2x, b2y = (np.asarray(ps[k], np.float64) for k in ("b1x", "b1y", "b2x", "b2y"))
    return dict(qxx=b1x * b1x + b2x * b2x, qxy=b1x * b1y + b2x * b2y, qyy=b1y * b1y + b2y * b2y)


def compare(ps, want) -> dict:
    """Check exported records against `project`'s result.  Returns a report: mismatched `valid` among unambiguous splats, and per field
    the worst |got - f64| / bound over splats valid on both sides and unambiguous (fields out of bound counted)."""
    got_valid = np.asarray(ps["valid"]) == 1
    unamb = ~want["ambiguous"]
    both = got_valid & want["valid"] & unamb
    q = quad_form(ps)
    rep = dict(valid_mismatch=int((got_valid != want["valid"])[unamb].sum()), compared=int(both.sum()),
               ambiguous=int(want["ambiguous"].sum()), worst={}, outside={})
    for k in FIELDS:
        g = q[k] if k in q else np.asarray(ps[k], np.float64)
        err = np.abs(g[both] - want[k][both])
        bound = want[k + "_bound"][both]
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = np.where(bound > 0, err / bound, np.where(err > 0, np.inf, 0.0))
        rep["worst"][k] = float(ratio.max(initial=0.0))
        rep["outside"][k] = int((~(err <= bound)).sum())
    return rep


def format_report(label, rep) -> str:
    w = " ".join(f"{k} {rep['worst'][k]:.3f}" for k in FIELDS)
    return f"[{label}] compared {rep['compared']}, ambiguous {rep['ambiguous']}, valid mismatches {rep['valid_mismatch']}; worst |err|/bound: {w}"


def assert_within(label, rep, min_compared=1):
    assert rep["compared"] >= min_compared, f"{label}: only {rep['compared']} splats compared"
    assert rep["valid_mismatch"] == 0, f"{label}: {rep['valid_mismatch']} unambiguous splats with the wrong `valid`"
    bad = {k: v for k, v in rep["outside"].items() if v}
    assert not bad, f"{label}: fields outside their bound {bad}; worst ratios {rep['worst']}"
