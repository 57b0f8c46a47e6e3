/* oracle/raster_oracle.c -- TEST INFRASTRUCTURE ONLY (never linked into or called by the product path).
 *
 * CPU restatement of the reference's splat rasteriser (3D mode): the GLSL vertex + fragment shaders and the
 * fixed-function blend, evaluated per splat in draw order exactly as WebGL would:
 *   vertex base  : /root/reference/src/splatmesh/SplatMaterial.js:112-170   (fetch, transform, cull)
 *   SH colour    : SplatMaterial.js:173-341
 *   projection   : src/splatmesh/SplatMaterial3D.js:83-216                  (cov3D -> cov2D, eigen basis, quad)
 *   fade-in      : SplatMaterial.js:347-363
 *   fragment     : SplatMaterial3D.js:234-252
 *   blend state  : SplatMaterial3D.js:65-75 (NormalBlending), clear (0,0,0,0) Viewer.js:353-360
 *
 * PINNING: the reference has no golden frames and its WebGL/three.js output cannot be produced in this environment (no
 * browser, three@0.160.0 not vendored), so no reference-made artefact pins this file ("parity unpinned" in that strict sense).
 * It is pinned by an INDEPENDENT FORMULATION instead -- oracle/raster_independent.py, checked in
 * tests/test_oracle_raster_independent.py -- that shares no code or algebra with this file or with the CUDA kernels:
 * finite-difference Jacobian of the actual projection, conic exp(-1/2 d^T Sigma'^-1 d) where the shader's clamps are inactive,
 * scipy's real spherical harmonics, and a triangle rasteriser of the 4-vertex quad with interpolated vPosition.
 * The blend-function mapping of THREE.NormalBlending is three.js behaviour restated from knowledge of
 * WebGLState.setBlending (SRC_ALPHA, ONE_MINUS_SRC_ALPHA, ONE, ONE_MINUS_SRC_ALPHA).
 *
 * All arithmetic is f32, unfused, in GLSL expression order (-ffp-contract=off).  Coverage: a fragment exists for
 * every pixel whose centre lies in the quad; since the fragment shader discards A > 8 and the unit disc is
 * inscribed in the quad, coverage reduces to A <= 8 with A from the exact inverse of the affine quad map.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "../include/gsplat_b200.h"

#define GS_ORACLE_API __attribute__((visibility("default")))

static inline float clamp01(float v) { return v < 0.f ? 0.f : (v > 1.f ? 1.f : v); }

/* column-major 4x4 times (x,y,z,1) */
static inline void mat4_mul_point(const float *m, float x, float y, float z, float out[4]) {
    for (int r = 0; r < 4; ++r) out[r] = m[r] * x + m[4 + r] * y + m[8 + r] * z + m[12 + r];
}
static inline void mat4_mul_vec4(const float *m, const float v[4], float out[4]) {
    for (int r = 0; r < 4; ++r) out[r] = m[r] * v[0] + m[4 + r] * v[1] + m[8 + r] * v[2] + m[12 + r] * v[3];
}
static void mat4_mul(const float *a, const float *b, float *o) { /* o = a*b, column-major */
    for (int c = 0; c < 4; ++c)
        for (int r = 0; r < 4; ++r)
            o[4 * c + r] = a[r] * b[4 * c] + a[4 + r] * b[4 * c + 1] + a[8 + r] * b[4 * c + 2] + a[12 + r] * b[4 * c + 3];
}
/* general 4x4 inverse (GLSL inverse()); f32 cofactor expansion */
static void mat4_inverse(const float *m, float *o) {
    float inv[16];
    inv[0] = m[5] * m[10] * m[15] - m[5] * m[11] * m[14] - m[9] * m[6] * m[15] + m[9] * m[7] * m[14] + m[13] * m[6] * m[11] - m[13] * m[7] * m[10];
    inv[4] = -m[4] * m[10] * m[15] + m[4] * m[11] * m[14] + m[8] * m[6] * m[15] - m[8] * m[7] * m[14] - m[12] * m[6] * m[11] + m[12] * m[7] * m[10];
    inv[8] = m[4] * m[9] * m[15] - m[4] * m[11] * m[13] - m[8] * m[5] * m[15] + m[8] * m[7] * m[13] + m[12] * m[5] * m[11] - m[12] * m[7] * m[9];
    inv[12] = -m[4] * m[9] * m[14] + m[4] * m[10] * m[13] + m[8] * m[5] * m[14] - m[8] * m[6] * m[13] - m[12] * m[5] * m[10] + m[12] * m[6] * m[9];
    inv[1] = -m[1] * m[10] * m[15] + m[1] * m[11] * m[14] + m[9] * m[2] * m[15] - m[9] * m[3] * m[14] - m[13] * m[2] * m[11] + m[13] * m[3] * m[10];
    inv[5] = m[0] * m[10] * m[15] - m[0] * m[11] * m[14] - m[8] * m[2] * m[15] + m[8] * m[3] * m[14] + m[12] * m[2] * m[11] - m[12] * m[3] * m[10];
    inv[9] = -m[0] * m[9] * m[15] + m[0] * m[11] * m[13] + m[8] * m[1] * m[15] - m[8] * m[3] * m[13] - m[12] * m[1] * m[11] + m[12] * m[3] * m[9];
    inv[13] = m[0] * m[9] * m[14] - m[0] * m[10] * m[13] - m[8] * m[1] * m[14] + m[8] * m[2] * m[13] + m[12] * m[1] * m[10] - m[12] * m[2] * m[9];
    inv[2] = m[1] * m[6] * m[15] - m[1] * m[7] * m[14] - m[5] * m[2] * m[15] + m[5] * m[3] * m[14] + m[13] * m[2] * m[7] - m[13] * m[3] * m[6];
    inv[6] = -m[0] * m[6] * m[15] + m[0] * m[7] * m[14] + m[4] * m[2] * m[15] - m[4] * m[3] * m[14] - m[12] * m[2] * m[7] + m[12] * m[3] * m[6];
    inv[10] = m[0] * m[5] * m[15] - m[0] * m[7] * m[13] - m[4] * m[1] * m[15] + m[4] * m[3] * m[13] + m[12] * m[1] * m[7] - m[12] * m[3] * m[5];
    inv[14] = -m[0] * m[5] * m[14] + m[0] * m[6] * m[13] + m[4] * m[1] * m[14] - m[4] * m[2] * m[13] - m[12] * m[1] * m[6] + m[12] * m[2] * m[5];
    inv[3] = -m[1] * m[6] * m[11] + m[1] * m[7] * m[10] + m[5] * m[2] * m[11] - m[5] * m[3] * m[10] - m[9] * m[2] * m[7] + m[9] * m[3] * m[6];
    inv[7] = m[0] * m[6] * m[11] - m[0] * m[7] * m[10] - m[4] * m[2] * m[11] + m[4] * m[3] * m[10] + m[8] * m[2] * m[7] - m[8] * m[3] * m[6];
    inv[11] = -m[0] * m[5] * m[11] + m[0] * m[7] * m[9] + m[4] * m[1] * m[11] - m[4] * m[3] * m[9] - m[8] * m[1] * m[7] + m[8] * m[3] * m[5];
    inv[15] = m[0] * m[5] * m[10] - m[0] * m[6] * m[9] - m[4] * m[1] * m[10] + m[4] * m[2] * m[9] + m[8] * m[1] * m[6] - m[8] * m[2] * m[5];
    float det = m[0] * inv[0] + m[1] * inv[4] + m[2] * inv[8] + m[3] * inv[12];
    float id = 1.0f / det;
    for (int i = 0; i < 16; ++i) o[i] = inv[i] * id;
}

/* IEEE half -> float (exact) */
static float half_to_float(uint16_t h) {
    uint32_t s = (uint32_t)(h >> 15) << 31, e = (h >> 10) & 31u, m = h & 1023u, bits;
    if (e == 0) {
        if (m == 0) bits = s;
        else {
            int sh = 0;
            while (!(m & 1024u)) { m <<= 1; ++sh; }
            m &= 1023u;
            bits = s | ((uint32_t)(127 - 15 - sh + 1) << 23) | (m << 13);
        }
    } else if (e == 31) bits = s | 0x7f800000u | (m << 13);
    else bits = s | ((e + 112u) << 23) | (m << 13);
    float f;
    memcpy(&f, &bits, 4);
    return f;
}

/* One vertex-shader evaluation per splat (the 4 corner invocations differ only in `position`). */
static void project_one(const gs_uniforms *u, const gs_splat_data *d, uint32_t s, gs_projected_splat *o) {
    memset(o, 0, sizeof(*o));
    const uint32_t *cc = d->centers_colors + 4 * (size_t)s;
    float c[3];
    memcpy(c, cc + 1, 12);
    uint32_t scene = 0;
    if (u->scene_count > 1 && d->scene_indexes) scene = d->scene_indexes[s];

    if (u->enable_optional_effects) { /* SplatMaterial.js:124-133 */
        if (u->scene_opacity[scene] <= 0.01f || u->scene_visibility[scene] == 0) return;
    }
    /* SplatMaterial.js:136-146: dynamic -> viewMatrix * transforms[scene] */
    float mv_dyn[16];
    const float *mv = u->model_view;
    const int dynamic = u->dynamic_mode != 0;
    if (dynamic) {
        mat4_mul(u->view_matrix, u->scene_transforms + 16 * scene, mv_dyn);
        mv = mv_dyn;
    }
    float view[4], clip[4];
    mat4_mul_point(mv, c[0], c[1], c[2], view);
    mat4_mul_vec4(u->projection, view, clip);
    const float lim = 1.2f * clip[3]; /* :160-164 */
    if (clip[2] < -lim || clip[0] < -lim || clip[0] > lim || clip[1] < -lim || clip[1] > lim) return;
    const float ndc[3] = {clip[0] / clip[3], clip[1] / clip[3], clip[2] / clip[3]};

    const uint32_t packed = cc[0]; /* :169, uintToRGBAVec :84-91 */
    float col[4];
    for (int k = 0; k < 4; ++k) col[k] = (float)((packed >> (8 * k)) & 255u) * (1.0f / 255.0f);

    if (d->sh_degree >= 1 && u->sh_degree >= 1 && d->spherical_harmonics) { /* :173-341 */
        const uint32_t ncomp = d->sh_degree >= 2 ? 24u : 9u;
        float sh[24];
        const float lo = u->sh8_min[scene], range = u->sh8_max[scene] - u->sh8_min[scene];
        for (uint32_t k = 0; k < ncomp; ++k) {
            const size_t at = (size_t)s * ncomp + k;
            if (d->sh_format == GS_SH_F16) sh[k] = half_to_float(((const uint16_t *)d->spherical_harmonics)[at]);
            else if (d->sh_format == GS_SH_U8) sh[k] = ((float)((const uint8_t *)d->spherical_harmonics)[at] / 255.0f) * range + lo;
            else sh[k] = ((const float *)d->spherical_harmonics)[at];
        }
        float cam[3] = {u->camera_position[0], u->camera_position[1], u->camera_position[2]};
        if (dynamic) { /* :181-183 */
            float inv[16], cp[4];
            mat4_inverse(u->scene_transforms + 16 * scene, inv);
            mat4_mul_point(inv, cam[0], cam[1], cam[2], cp);
            cam[0] = cp[0]; cam[1] = cp[1]; cam[2] = cp[2];
        }
        float dir[3] = {c[0] - cam[0], c[1] - cam[1], c[2] - cam[2]};
        const float il = 1.0f / sqrtf(dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2]);
        const float x = dir[0] * il, y = dir[1] * il, z = dir[2] * il;
        const float C1 = 0.4886025119029199f;
        for (int ch = 0; ch < 3; ++ch) col[ch] += C1 * (-sh[0 + ch] * y + sh[3 + ch] * z - sh[6 + ch] * x);
        if (d->sh_degree >= 2 && u->sh_degree >= 2) {
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            for (int ch = 0; ch < 3; ++ch)
                col[ch] += (1.0925484f * xy) * sh[9 + ch] + (-1.0925484f * yz) * sh[12 + ch] +
                           (0.3153916f * (2.0f * zz - xx - yy)) * sh[15 + ch] + (-1.0925484f * xz) * sh[18 + ch] +
                           (0.5462742f * (xx - yy)) * sh[21 + ch];
        }
        for (int ch = 0; ch < 3; ++ch) col[ch] = clamp01(col[ch]);
    }

    /* SplatMaterial3D.js:85-109: covariance fetch */
    float V[6];
    if (d->cov_format == GS_COV_F16)
        for (int k = 0; k < 6; ++k) V[k] = half_to_float(((const uint16_t *)d->covariances)[6 * (size_t)s + k]);
    else
        memcpy(V, (const float *)d->covariances + 6 * (size_t)s, 24);

    /* M = transpose(T) = Jstd * mat3(MV) : rows m0, m1 (third row is zero)   :111-134 */
    float j00, j02, j11, j12;
    if (u->orthographic_mode == 1) { j00 = u->ortho_zoom; j11 = u->ortho_zoom; j02 = 0.f; j12 = 0.f; }
    else {
        const float sc = 1.0f / (view[2] * view[2]);
        j00 = u->focal[0] / view[2]; j11 = u->focal[1] / view[2];
        j02 = -(u->focal[0] * view[0]) * sc; j12 = -(u->focal[1] * view[1]) * sc;
    }
    /* T = W*J with W = transpose(mat3(mv)):  T[k][col j] = sum_i mv(i,k) ... written out: T_col0 = W * J_col0 */
    float T0[3], T1[3]; /* columns 0 and 1 of T (column 2 is zero) */
    for (int k = 0; k < 3; ++k) {
        /* W[row k] = (mv[4k+0], mv[4k+1], mv[4k+2])  (transpose of the upper 3x3)  -> W*(a,b,c) row k */
        const float w0 = mv[4 * k + 0], w1 = mv[4 * k + 1], w2 = mv[4 * k + 2];
        T0[k] = w0 * j00 + w1 * 0.0f + w2 * j02;
        T1[k] = w0 * 0.0f + w1 * j11 + w2 * j12;
    }
    /* Vrk * T columns */
    const float S[3][3] = {{V[0], V[1], V[2]}, {V[1], V[3], V[4]}, {V[2], V[4], V[5]}};
    float VT0[3], VT1[3];
    for (int r = 0; r < 3; ++r) {
        VT0[r] = S[r][0] * T0[0] + S[r][1] * T0[1] + S[r][2] * T0[2];
        VT1[r] = S[r][0] * T1[0] + S[r][1] * T1[1] + S[r][2] * T1[2];
    }
    float a = T0[0] * VT0[0] + T0[1] * VT0[1] + T0[2] * VT0[2];
    float b = T0[0] * VT1[0] + T0[1] * VT1[1] + T0[2] * VT1[2]; /* cov2Dm[0][1] */
    float dd = T1[0] * VT1[0] + T1[1] * VT1[1] + T1[2] * VT1[2];

    if (u->antialiased) { /* :137-145 */
        const float det0 = a * dd - b * b;
        a += u->kernel_2d_size; dd += u->kernel_2d_size;
        const float det1 = a * dd - b * b;
        col[3] *= sqrtf(fmaxf(det0 / det1, 0.0f));
        if (col[3] < 1.0f / 255.0f) return;
    } else { a += u->kernel_2d_size; dd += u->kernel_2d_size; }

    /* :174-196 eigen decomposition */
    const float D = a * dd - b * b, half_tr = 0.5f * (a + dd);
    const float term2 = sqrtf(fmaxf(0.1f, half_tr * half_tr - D));
    float l1 = half_tr + term2, l2 = half_tr - term2;
    if (u->point_cloud_mode == 1) l1 = l2 = 0.2f;
    if (l2 <= 0.0f) return;
    float ex = b, ey = l1 - a;
    const float en = 1.0f / sqrtf(ex * ex + ey * ey);
    if (!isfinite(en)) return; /* normalize(vec2(0)) is NaN: the quad's vertices are NaN and GL draws nothing */
    ex *= en; ey *= en;
    const float sqrt8 = sqrtf(8.0f);
    const float s1 = u->splat_scale * fminf(sqrt8 * sqrtf(l1), u->max_screen_space_splat_size);
    const float s2 = u->splat_scale * fminf(sqrt8 * sqrtf(l2), u->max_screen_space_splat_size);
    /* e1*splatScale*min(...) evaluates left to right in GLSL: (e1 * splatScale) * min(..) ; products commute up
       to rounding -- tolerance-level. */
    float b1x = ex * s1, b1y = ey * s1, b2x = ey * s2, b2y = -ex * s2;

    if (u->enable_optional_effects) col[3] *= u->scene_opacity[scene]; /* :198-202 */

    if (!u->fade_in_complete) { /* SplatMaterial.js:347-363 */
        const float dx = c[0] - u->scene_center[0], dy = c[1] - u->scene_center[1], dz = c[2] - u->scene_center[2];
        const float dist = sqrtf(dx * dx + dy * dy + dz * dz);
        const float st = dist >= u->visible_region_fade_start_radius ? 1.0f : 0.0f;
        const float f = (1.0f - st) + (1.0f - clamp01((dist - u->visible_region_fade_start_radius) / 0.75f)) * st;
        col[3] *= f;
    }

    /* ndcOffset = (q.x*B1 + q.y*B2) * basisViewport * 2 * invFocalAdj ; pixels = ndc * viewport/2 */
    const float k = u->inverse_focal_adjustment;
    o->b1x = b1x * k; o->b1y = b1y * k; o->b2x = b2x * k; o->b2y = b2y * k;
    o->cx = (ndc[0] + 1.0f) * 0.5f * u->viewport[0];
    o->cy = (ndc[1] + 1.0f) * 0.5f * u->viewport[1];
    o->r = col[0]; o->g = col[1]; o->b = col[2]; o->a = col[3];
    o->ndc_z = ndc[2];
    o->valid = (ndc[2] >= -1.0f && ndc[2] <= 1.0f) ? 1u : 0u; /* GL near/far clipping of the quad (w = 1) */
}

GS_ORACLE_API void gso_project(const gs_uniforms *u, const gs_splat_data *d, gs_projected_splat *out) {
#pragma omp parallel for schedule(static)
    for (int64_t s = 0; s < (int64_t)d->count; ++s) project_one(u, d, (uint32_t)s, out + s);
}

/* Blend the projected splats in draw order (sorted_indexes[0] first = farthest) into a float RGBA frame
 * (GL window orientation: row 0 = bottom).  quantize8 != 0 models an RGBA8 render target: the destination is
 * rounded to 8 bits after every blend (informational second oracle, SURVEY 8c).
 * Rows are distributed over threads; every pixel still sees the splats in exactly the draw order. */
static void blend_region(const gs_projected_splat *ps, const uint32_t *sorted_indexes, uint32_t render_count, uint32_t width, uint32_t height,
                         uint32_t cx0, uint32_t cy0, uint32_t cw, uint32_t chh, int quantize8, float *frame);

GS_ORACLE_API void gso_blend(const gs_projected_splat *ps, const uint32_t *sorted_indexes, uint32_t render_count,
                             uint32_t width, uint32_t height, int quantize8, float *frame) {
    blend_region(ps, sorted_indexes, render_count, width, height, 0, 0, width, height, quantize8, frame);
}

/* The same blend restricted to the window [cx0, cx0+cw) x [cy0, cy0+chh) of a width x height frame (GL window coordinates, row 0 =
 * bottom); `frame` is cw x chh x 4.  Lets the tests check parts of frames that are too large to restate whole (16 M splats at 4K). */
GS_ORACLE_API void gso_blend_crop(const gs_projected_splat *ps, const uint32_t *sorted_indexes, uint32_t render_count, uint32_t width,
                                  uint32_t height, uint32_t cx0, uint32_t cy0, uint32_t cw, uint32_t chh, int quantize8, float *frame) {
    blend_region(ps, sorted_indexes, render_count, width, height, cx0, cy0, cw, chh, quantize8, frame);
}

/* The same blends plus a coverage-boundary map: flags[pixel] = 1 where the GPU's own f32 evaluation of q = A/8 may fall on the other
 * side of the discard test (A > 8) than this one AND that could matter.  A splat (a >= 1/255) is "on the boundary" of a pixel when
 * |A/8 - 1| <= delta; flipping its coverage there moves the pixel by at most T a e^-4 (T = transmittance in front of it, colours in
 * [0,1]).  The pixel is flagged when that bound, summed over its boundary splats, exceeds `min_weight`.
 * delta = 4e-3 is twice kEllipseSlack (csrc/ellipse_mask.h), chosen for a blend that evaluated q at absolute pixel coordinates (~1e-3
 * of rounding at 8K for |g| <= 0.65 px^-1).  k_blend now evaluates q relative to the tile's first pixel centre (~1e-5 wherever the tile
 * lies), and the GPU's blend is held to the per-pixel f64 bounds of tests/blend_f64.c, not to this map; the map is kept as a
 * diagnostic of the oracle's own blend, and k_export_projected's basis b = g / |g|^2 adds about one ulp to it.  min_weight = 1/4 of
 * an 8-bit step: with the 1/512 cutoff (< 1/2 step) an unflagged pixel then stays within one step of this frame. */
static void flag_region(const gs_projected_splat *ps, const uint32_t *sorted_indexes, uint32_t render_count, uint32_t cx0, uint32_t cy0,
                        uint32_t cw, uint32_t chh, float delta, float min_weight, uint8_t *flags);

GS_ORACLE_API void gso_blend_flags(const gs_projected_splat *ps, const uint32_t *sorted_indexes, uint32_t render_count, uint32_t width,
                                   uint32_t height, int quantize8, float delta, float min_weight, float *frame, uint8_t *flags) {
    blend_region(ps, sorted_indexes, render_count, width, height, 0, 0, width, height, quantize8, frame);
    flag_region(ps, sorted_indexes, render_count, 0, 0, width, height, delta, min_weight, flags);
}

GS_ORACLE_API void gso_blend_crop_flags(const gs_projected_splat *ps, const uint32_t *sorted_indexes, uint32_t render_count, uint32_t width,
                                        uint32_t height, uint32_t cx0, uint32_t cy0, uint32_t cw, uint32_t chh, int quantize8, float delta,
                                        float min_weight, float *frame, uint8_t *flags) {
    blend_region(ps, sorted_indexes, render_count, width, height, cx0, cy0, cw, chh, quantize8, frame);
    flag_region(ps, sorted_indexes, render_count, cx0, cy0, cw, chh, delta, min_weight, flags);
}

/* Pixel-window bounds of a splat's quad (the blend's own, 1 px of margin); 0 if it misses the window. */
static int splat_window(const gs_projected_splat *p, uint32_t cx0, uint32_t cy0, uint32_t cw, uint32_t chh, int *x0, int *x1, int *y0, int *y1) {
    if (!p->valid) return 0;
    const float n1 = p->b1x * p->b1x + p->b1y * p->b1y, n2 = p->b2x * p->b2x + p->b2y * p->b2y;
    if (!(n1 > 0.f) || !(n2 > 0.f)) return 0;
    const float ex = fabsf(p->b1x) + fabsf(p->b2x), ey = fabsf(p->b1y) + fabsf(p->b2y);
    float fx0 = floorf(p->cx - ex - 1.0f), fx1 = ceilf(p->cx + ex + 1.0f), fy0 = floorf(p->cy - ey - 1.0f), fy1 = ceilf(p->cy + ey + 1.0f);
    if (fx0 < (float)cx0) fx0 = (float)cx0;
    if (fx1 > (float)(cx0 + cw) - 1.f) fx1 = (float)(cx0 + cw) - 1.f;
    if (fy0 < (float)cy0) fy0 = (float)cy0;
    if (fy1 > (float)(cy0 + chh) - 1.f) fy1 = (float)(cy0 + chh) - 1.f;
    if (!(fx0 <= fx1) || !(fy0 <= fy1)) return 0;
    *x0 = (int)fx0; *x1 = (int)fx1; *y0 = (int)fy0; *y1 = (int)fy1;
    return 1;
}

/* Front to back (the draw order reversed), one row at a time: transmittance in front of each splat, boundary weights summed. */
static void flag_region(const gs_projected_splat *ps, const uint32_t *sorted_indexes, uint32_t render_count, uint32_t cx0, uint32_t cy0,
                        uint32_t cw, uint32_t chh, float delta, float min_weight, uint8_t *flags) {
#pragma omp parallel
    {
        float *T = (float *)malloc(sizeof(float) * cw), *E = (float *)malloc(sizeof(float) * cw);
#pragma omp for schedule(dynamic, 1)
        for (int y = (int)cy0; y < (int)(cy0 + chh); ++y) {
            for (uint32_t k = 0; k < cw; ++k) { T[k] = 1.f; E[k] = 0.f; }
            const float dy = ((float)y + 0.5f);
            for (uint32_t i = render_count; i-- > 0;) {
                const gs_projected_splat *p = ps + sorted_indexes[i];
                int x0, x1, y0, y1;
                if (!splat_window(p, cx0, cy0, cw, chh, &x0, &x1, &y0, &y1) || y < y0 || y > y1) continue;
                const float n1 = p->b1x * p->b1x + p->b1y * p->b1y, n2 = p->b2x * p->b2x + p->b2y * p->b2y;
                for (int x = x0; x <= x1; ++x) {
                    const float dx = ((float)x + 0.5f) - p->cx, ddy = dy - p->cy;
                    const float qu = (dx * p->b1x + ddy * p->b1y) / n1, qw = (dx * p->b2x + ddy * p->b2y) / n2;
                    const float A = 8.0f * (qu * qu + qw * qw);
                    const uint32_t k = (uint32_t)(x - (int)cx0);
                    if (p->a >= 1.0f / 255.0f && fabsf(A * 0.125f - 1.0f) <= delta) E[k] += T[k] * p->a * 0.01831564f;   /* e^-4 */
                    if (A <= 8.0f) T[k] *= 1.0f - expf(-0.5f * A) * p->a;
                }
            }
            for (uint32_t k = 0; k < cw; ++k) flags[(size_t)(y - (int)cy0) * cw + k] = E[k] > min_weight;
        }
        free(T);
        free(E);
    }
}

static void blend_region(const gs_projected_splat *ps, const uint32_t *sorted_indexes, uint32_t render_count, uint32_t width, uint32_t height,
                         uint32_t cx0, uint32_t cy0, uint32_t cw, uint32_t chh, int quantize8, float *frame) {
    (void)width; (void)height;
    memset(frame, 0, (size_t)cw * chh * 4 * sizeof(float));
    /* per-splat row extents so each row band can skip quickly */
    int32_t *ylo = (int32_t *)malloc(sizeof(int32_t) * (size_t)render_count);
    int32_t *yhi = (int32_t *)malloc(sizeof(int32_t) * (size_t)render_count);
    for (uint32_t i = 0; i < render_count; ++i) {
        const gs_projected_splat *p = ps + sorted_indexes[i];
        if (!p->valid) { ylo[i] = 1; yhi[i] = 0; continue; }
        const float ey = fabsf(p->b1y) + fabsf(p->b2y);
        float lo = floorf(p->cy - ey - 1.0f), hi = ceilf(p->cy + ey + 1.0f);
        if (lo < (float)cy0) lo = (float)cy0;
        if (hi > (float)(cy0 + chh) - 1.f) hi = (float)(cy0 + chh) - 1.f;
        if (!(lo <= hi)) { ylo[i] = 1; yhi[i] = 0; continue; }
        ylo[i] = (int32_t)lo; yhi[i] = (int32_t)hi;
    }
    const int band = 8;
    const int nbands = ((int)chh + band - 1) / band;
#pragma omp parallel for schedule(dynamic, 1)
    for (int bi = 0; bi < nbands; ++bi) {
        const int y0 = (int)cy0 + bi * band, y1 = (y0 + band < (int)(cy0 + chh) ? y0 + band : (int)(cy0 + chh)) - 1;
        for (uint32_t i = 0; i < render_count; ++i) {
            if (yhi[i] < y0 || ylo[i] > y1) continue;
            const gs_projected_splat *p = ps + sorted_indexes[i];
            const float n1 = p->b1x * p->b1x + p->b1y * p->b1y, n2 = p->b2x * p->b2x + p->b2y * p->b2y;
            if (!(n1 > 0.f) || !(n2 > 0.f)) continue;
            const float ex = fabsf(p->b1x) + fabsf(p->b2x);
            float fx0 = floorf(p->cx - ex - 1.0f), fx1 = ceilf(p->cx + ex + 1.0f);
            if (fx0 < (float)cx0) fx0 = (float)cx0;
            if (fx1 > (float)(cx0 + cw) - 1.f) fx1 = (float)(cx0 + cw) - 1.f;
            if (!(fx0 <= fx1)) continue;
            const int x0 = (int)fx0, x1 = (int)fx1;
            const int ya = ylo[i] > y0 ? ylo[i] : y0, yb = yhi[i] < y1 ? yhi[i] : y1;
            for (int y = ya; y <= yb; ++y) {
                const float dy = ((float)y + 0.5f) - p->cy;
                for (int x = x0; x <= x1; ++x) {
                    const float dx = ((float)x + 0.5f) - p->cx;
                    /* inverse of the affine map (orthogonal basis): quad-local coordinates in [-1,1] */
                    const float qu = (dx * p->b1x + dy * p->b1y) / n1;
                    const float qw = (dx * p->b2x + dy * p->b2y) / n2;
                    /* vPosition = q * sqrt8 ; A = dot(vPosition, vPosition) */
                    const float A = 8.0f * (qu * qu + qw * qw);
                    if (A > 8.0f) continue;
                    const float alpha = expf(-0.5f * A) * p->a;
                    float *px = frame + ((size_t)(y - (int)cy0) * cw + (size_t)(x - (int)cx0)) * 4;
                    const float om = 1.0f - alpha;
                    px[0] = p->r * alpha + px[0] * om;
                    px[1] = p->g * alpha + px[1] * om;
                    px[2] = p->b * alpha + px[2] * om;
                    px[3] = alpha + px[3] * om;
                    if (quantize8)
                        for (int k = 0; k < 4; ++k) px[k] = floorf(clamp01(px[k]) * 255.0f + 0.5f) / 255.0f;
                }
            }
        }
    }
    free(ylo);
    free(yhi);
}

/* Convenience: project + blend. */
GS_ORACLE_API void gso_render(const gs_uniforms *u, const gs_splat_data *d, const uint32_t *sorted_indexes,
                              uint32_t render_count, uint32_t width, uint32_t height, int quantize8, float *frame,
                              gs_projected_splat *projected /* d->count entries, caller-owned */) {
    gso_project(u, d, projected);
    gso_blend(projected, sorted_indexes, render_count, width, height, quantize8, frame);
}
