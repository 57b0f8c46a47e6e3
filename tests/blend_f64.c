/* The fragment stage and blend of the splat mesh restated in f64, with a bound on every channel of every pixel that the f32 blend
 * kernel must meet, and an f32 emulation of that kernel to test the bound with.  TEST INFRASTRUCTURE ONLY; includes nothing from the
 * product.
 *
 * Input: the engine's 48-byte projected records (cx, cy, g1, g2, half2 hx/hy, a, rgb, ndc_z), a draw order (back to front), the frame
 * size and a window of it aligned to 8 px.  A record is drawn iff ndc_z is in [-1, 1].  Semantics: the reference's fragment stage and
 * NormalBlending over a zero clear.  A pixel centre p = (x + 1/2, y + 1/2) is covered when q = (g1.(p - c))^2 + (g2.(p - c))^2 <= 1,
 * alpha = a e^(-4 q), C = sum T_i alpha_i c_i, A = 1 - prod(1 - alpha_i).  Composite: zw = f32(0.5 ndc_z + 0.5) passes iff zw <= d (NaN d
 * passes nothing, no depth = +inf), then C += T Cd, A += T Ad.
 *
 * Which splats reach an 8x8 block is decided here from f64 extents of q <= kExtQ, not from the engine's rects or masks, so a fault in
 * those is an error and not a shared assumption.
 *
 * The bound has three parts:
 *  - rounding of the kernel's operation sequence, first order: one u per rounded operation on the magnitude of its exact result;
 *  - coverage ambiguity: a (splat, pixel) term with |q - 1| <= dq (dq: the rounding bound of the kernel's q) may go either way and adds
 *    its largest effect, T a e^(-4 (1 - dq)) (|c| + the most the rest can contribute); every other term must match in or out;
 *  - the early stop: per 8x8 block (in-frame pixels), the first position in its front-to-back list at which every pixel may be below the
 *    cutoff; from there the kernel may stop, and the allowance is what T can still be there times the most the rest can contribute.
 *    Where no such position exists the kernel cannot have stopped and the allowance is 0. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
    float cx, cy, g1x, g1y, g2x, g2y;
    uint32_t hh;                    /* half2 hx, hy: not read, the extents here are the restatement's own */
    float a, r, g, b, z;
} bf_rec;

#define U32 0x1p-24                 /* unit roundoff of f32 round-to-nearest */
/* ex2.approx.f32 (PTX ISA, "ex2"): maximum relative error 2 ulp over the full range of inputs, i.e. <= 2^-22 relative; the .ftz form
 * flushes subnormal results, at most 2^-126 absolute */
#define EX2_REL 0x1p-22
#define FTZ 0x1p-126
#define CUTOFF (1.0 / 512.0)        /* the kernel's transmittance cutoff */
#define KEXP (-5.770780163555854f)  /* the kernel's -4/ln2 rounded to f32 */
static const double kExtQ = 1.01;   /* candidate extents: q <= kExtQ; a term's dq must stay below kExtQ - 1 */

enum { FORM_TILE = 0, FORM_ABS = 1 };   /* quad coordinates relative to the tile's first pixel centre / absolute (the earlier kernel) */

typedef struct {
    int width, height, x0, y0, w, h, nbx, nby, tile;
} win_t;

static int drawn(const bf_rec *r) { return r->z >= -1.0f && r->z <= 1.0f; }
static int finite_rec(const bf_rec *r) {
    return isfinite(r->cx) && isfinite(r->cy) && isfinite(r->g1x) && isfinite(r->g1y) && isfinite(r->g2x) && isfinite(r->g2y) && isfinite(r->a) &&
           isfinite(r->r) && isfinite(r->g) && isfinite(r->b);
}

/* the window's blocks that the ellipse q <= kExtQ reaches (its AABB); 0 = none */
static int block_range(const bf_rec *r, const win_t *wd, int *bx0, int *bx1, int *by0, int *by1) {
    const double g1x = r->g1x, g1y = r->g1y, g2x = r->g2x, g2y = r->g2y;
    const double qxx = g1x * g1x + g2x * g2x, qyy = g1y * g1y + g2y * g2y, dt = g1x * g2y - g1y * g2x, det = dt * dt;
    int px0 = wd->x0, px1 = wd->x0 + wd->w - 1, py0 = wd->y0, py1 = wd->y0 + wd->h - 1;
    if (det > 0.0) {
        const double hx = sqrt(kExtQ * qyy / det) * (1.0 + 1e-9) + 1e-9, hy = sqrt(kExtQ * qxx / det) * (1.0 + 1e-9) + 1e-9;
        const double fx0 = ceil(r->cx - hx - 0.5), fx1 = floor(r->cx + hx - 0.5), fy0 = ceil(r->cy - hy - 0.5), fy1 = floor(r->cy + hy - 0.5);
        if (fx1 < px0 || fy1 < py0 || fx0 > px1 || fy0 > py1 || fx0 > fx1 || fy0 > fy1) return 0;
        if (fx0 > px0) px0 = (int)fx0;
        if (fx1 < px1) px1 = (int)fx1;
        if (fy0 > py0) py0 = (int)fy0;
        if (fy1 < py1) py1 = (int)fy1;
    }
    *bx0 = (px0 - wd->x0) >> 3; *bx1 = (px1 - wd->x0) >> 3; *by0 = (py0 - wd->y0) >> 3; *by1 = (py1 - wd->y0) >> 3;
    return 1;
}

/* per-block lists (CSR) of the records that may reach each block, front to back; returns the number of drawn records with a non-finite
 * field (skipped), or -1 when out of memory */
static long build_lists(const bf_rec *rec, const uint32_t *order, uint32_t count, const win_t *wd, int64_t drop, int64_t **off_out,
                        uint32_t **ent_out) {
    const int64_t nb = (int64_t)wd->nbx * wd->nby;
    int64_t *off = calloc((size_t)nb + 1, sizeof(int64_t));
    if (!off) return -1;
    long bad = 0;
    for (int pass = 0; pass < 2; ++pass) {
        uint32_t *ent = pass ? *ent_out : NULL;
        int64_t *fill = NULL;
        if (pass) {
            fill = malloc((size_t)nb * sizeof(int64_t));
            if (!fill) return -1;
            memcpy(fill, off, (size_t)nb * sizeof(int64_t));
        }
        for (int64_t k = (int64_t)count - 1; k >= 0; --k) {
            const uint32_t i = order[k];
            if ((int64_t)i == drop) continue;
            const bf_rec *r = rec + i;
            if (!drawn(r)) continue;
            if (!finite_rec(r)) { bad += pass == 0; continue; }
            if (!(r->a > 0.0f)) continue;
            int bx0, bx1, by0, by1;
            if (!block_range(r, wd, &bx0, &bx1, &by0, &by1)) continue;
            for (int by = by0; by <= by1; ++by)
                for (int bx = bx0; bx <= bx1; ++bx) {
                    const int64_t b = (int64_t)by * wd->nbx + bx;
                    if (pass) ent[fill[b]++] = i; else off[b + 1]++;
                }
        }
        if (!pass) {
            for (int64_t b = 0; b < nb; ++b) off[b + 1] += off[b];
            *ent_out = malloc((size_t)(off[nb] ? off[nb] : 1) * sizeof(uint32_t));
            if (!*ent_out) return -1;
        } else {
            free(fill);
        }
    }
    *off_out = off;
    return bad;
}

static int init_window(win_t *wd, int width, int height, int x0, int y0, int w, int h, int tile) {
    if (x0 % 8 || y0 % 8 || w <= 0 || h <= 0 || x0 + w > width || y0 + h > height) return 0;
    if ((w % 8 && x0 + w != width) || (h % 8 && y0 + h != height)) return 0;
    *wd = (win_t){width, height, x0, y0, w, h, (w + 7) / 8, (h + 7) / 8, tile};
    return 1;
}

/* rounding bound of the kernel's U = g . (p - c) for one of the two rows (gx, gy) of the inverse quad map */
static double quad_err(int form, double gx, double gy, double cx, double cy, double px, double py, double tx0, double ty0) {
    if (form == FORM_TILE) {     /* X0 = tile_x0 - cx; u0 = fma(X0, gx, Y0 gy); t = fma(dx, gx, u0); U = fma(dy, gy, t) */
        const double X0 = tx0 - cx, Y0 = ty0 - cy, s = Y0 * gy, u0 = X0 * gx + s, t = (px - tx0) * gx + u0, U = (py - ty0) * gy + t;
        return fabs(gx) * U32 * fabs(X0) + fabs(gy) * U32 * fabs(Y0) + U32 * (fabs(s) + fabs(u0) + fabs(t) + fabs(U));
    }
    /* u0 = -fma(cx, gx, cy gy); t = fma(px, gx, u0); U = fma(py, gy, t) */
    const double s = cy * gy, u0 = -(cx * gx + s), t = px * gx + u0, U = py * gy + t;
    return U32 * (fabs(s) + fabs(u0) + fabs(t) + fabs(U));
}

static double f32_ulp(double v) {
    const float f = (float)fabs(v);
    return (double)nextafterf(f, INFINITY) - (double)f;
}

/* The f64 frame of the window and its per-channel bound.  Outputs (window rows, pixel y = row + y0, bottom-up): val[h][w][4],
 * bound[h][w][4], amb[h][w] (number of ambiguous terms), and stats[0] = the largest dq of a term with q <= 1.1, stats[1] = the largest dq of a
 * term with |q - 1| <= 0.05.  dest_color (RGBA, f32 as the kernel reads it) and dest_depth are whole frames in pixel-y order, or NULL.
 * Returns the number of drawn records with non-finite fields, -1 on bad arguments or memory, -2 when some dq reaches kExtQ - 1. */
long bf_reference(const bf_rec *rec, const uint32_t *order, uint32_t count, int width, int height, int x0, int y0, int w, int h, int tile,
                  int form, const float *dest_color, const float *dest_depth, double *val, double *bound, int32_t *amb, double *stats) {
    win_t wd;
    if (!init_window(&wd, width, height, x0, y0, w, h, tile)) return -1;
    int64_t *off = NULL;
    uint32_t *ent = NULL;
    const long bad = build_lists(rec, order, count, &wd, -1, &off, &ent);
    if (bad < 0) return -1;
    double M[4] = {0.0, 0.0, 0.0, 1.0};    /* the most a splat's colour can be */
    for (uint32_t k = 0; k < count; ++k) {
        const bf_rec *r = rec + order[k];
        if (!drawn(r) || !finite_rec(r)) continue;
        M[0] = fmax(M[0], fabs(r->r)); M[1] = fmax(M[1], fabs(r->g)); M[2] = fmax(M[2], fabs(r->b));
    }
    const double K = (double)KEXP, Kx = -4.0 / log(2.0);
    double dq_max = 0.0, dq_near = 0.0;
    int over = 0;
    const int64_t nb = (int64_t)wd.nbx * wd.nby;
#pragma omp parallel for schedule(dynamic, 4) reduction(max : dq_max, dq_near) reduction(| : over)
    for (int64_t blk = 0; blk < nb; ++blk) {
        const int bxw = (int)(blk % wd.nbx), byw = (int)(blk / wd.nbx);
        const int bx = wd.x0 + 8 * bxw, by = wd.y0 + 8 * byw;
        const double tx0 = (double)(bx / tile * tile) + 0.5, ty0 = (double)(by / tile * tile) + 0.5;
        double T[64], Tup[64], Tlo[64], eT[64], Cc[64][3], eC[64][3], am[64][4], Tstop[64], cd[64][4], dd[64];
        int act[64], namb[64], stopped = 0;
        for (int p = 0; p < 64; ++p) {
            const int x = bx + (p & 7), y = by + (p >> 3);
            act[p] = x < width && y < height;
            T[p] = Tup[p] = Tlo[p] = act[p] ? 1.0 : 0.0;
            eT[p] = 0.0; Tstop[p] = 0.0; namb[p] = 0;
            for (int c = 0; c < 3; ++c) Cc[p][c] = eC[p][c] = 0.0;
            for (int c = 0; c < 4; ++c) { am[p][c] = 0.0; cd[p][c] = 0.0; }
            dd[p] = INFINITY;
            if (act[p]) {
                const size_t at = (size_t)y * width + x;
                if (dest_color) for (int c = 0; c < 4; ++c) cd[p][c] = dest_color[4 * at + c];
                if (dest_depth) dd[p] = dest_depth[at];
            }
        }
        for (int64_t e = off[blk]; e < off[blk + 1]; ++e) {
            const bf_rec *r = rec + ent[e];
            const double cx = r->cx, cy = r->cy, g1x = r->g1x, g1y = r->g1y, g2x = r->g2x, g2y = r->g2y, a = r->a;
            const double col[3] = {r->r, r->g, r->b};
            const float zw = fmaf(0.5f, r->z, 0.5f);
            const double L = log2(a), eL = f32_ulp(L);    /* log2f: 1 ulp */
            for (int p = 0; p < 64; ++p) {
                if (!act[p]) continue;
                const double px = bx + (p & 7) + 0.5, py = by + (p >> 3) + 0.5, dx = px - cx, dy = py - cy;
                const double U = g1x * dx + g1y * dy, W = g2x * dx + g2y * dy, q = U * U + W * W;
                const double eU = quad_err(form, g1x, g1y, cx, cy, px, py, tx0, ty0), eW = quad_err(form, g2x, g2y, cx, cy, px, py, tx0, ty0);
                const double dq = (2.0 * fabs(U) * eU + 2.0 * fabs(W) * eW + eU * eU + eW * eW + U32 * (U * U + q)) * (1.0 + 1e-6) + 1e-15;
                if (fabs(q - 1.0) <= 0.05 && dq > dq_near) dq_near = dq;
                if (q <= 1.1 && dq > dq_max) dq_max = dq;
                if (q <= 1.1 && dq >= kExtQ - 1.0) over = 1;   /* terms outside the extents are taken as out */
                if (!(zw <= dd[p])) continue;              /* depth test: exact on both sides */
                if (q > 1.0 + dq) continue;                /* out, certainly */
                if (q >= 1.0 - dq) {                       /* ambiguous: either way */
                    const double amax = a * exp(-4.0 * (1.0 - dq)) * (1.0 + 2.0 * EX2_REL) + FTZ;
                    for (int c = 0; c < 3; ++c) am[p][c] += Tup[p] * amax * (fabs(col[c]) + M[c] + fabs(cd[p][c]));
                    am[p][3] += Tup[p] * amax * (1.0 + fabs(cd[p][3]));
                    namb[p]++;
                    Tlo[p] *= 1.0 - amax;
                    eT[p] += 2.0 * U32 * Tup[p];
                    for (int c = 0; c < 3; ++c) eC[p][c] += 2.0 * U32 * Tup[p] * (1.0 + fabs(col[c]));
                    if (q > 1.0) continue;                 /* the f64 value follows q <= 1 */
                }
                /* X = fma(Q, K, log2f(a)), alpha = ex2(X) */
                const double xs = Kx * q + L;
                const double eX = fabs(K - Kx) * q + fabs(K) * dq + eL + U32 * fabs(xs);
                const double al = a * exp(-4.0 * q);
                const double g = exp(log(2.0) * eX);
                const double eal = al * ((g - 1.0) + EX2_REL * g) * (1.0 + 1e-6) + FTZ;
                const double wgt = T[p] * al, ew = al * eT[p] + T[p] * eal + U32 * wgt;
                for (int c = 0; c < 3; ++c) {
                    Cc[p][c] += wgt * col[c];
                    eC[p][c] += fabs(col[c]) * ew + U32 * fabs(Cc[p][c]);
                }
                const double Tn = T[p] - wgt;
                eT[p] = eT[p] * (1.0 - al + eal) + T[p] * eal + U32 * wgt + U32 * Tn;
                T[p] = Tn;
                Tup[p] *= 1.0 - al;
                Tlo[p] *= 1.0 - al;
            }
            if (!stopped) {
                int can = 1;
                for (int p = 0; p < 64 && can; ++p) can = !act[p] || Tlo[p] - eT[p] < CUTOFF;
                if (can) {
                    stopped = 1;
                    for (int p = 0; p < 64; ++p) Tstop[p] = act[p] ? Tup[p] + eT[p] : 0.0;
                }
            }
        }
        for (int p = 0; p < 64; ++p) {
            const int x = bx + (p & 7), y = by + (p >> 3);
            if (x >= wd.x0 + wd.w || y >= wd.y0 + wd.h) continue;
            const size_t o = (size_t)(y - wd.y0) * wd.w + (x - wd.x0);
            const double Tp = T[p];
            double v[4], bd[4];
            for (int c = 0; c < 3; ++c) {
                v[c] = Cc[p][c] + Tp * cd[p][c];
                bd[c] = eC[p][c] + fabs(cd[p][c]) * eT[p] + (dest_color ? U32 * fabs(v[c]) : 0.0);
            }
            v[3] = 1.0 - Tp + Tp * cd[p][3];
            bd[3] = eT[p] * (1.0 + fabs(cd[p][3])) + U32 * fabs(1.0 - Tp) + (dest_color ? U32 * fabs(v[3]) : 0.0);
            for (int c = 0; c < 4; ++c) {
                const double Mc = c < 3 ? M[c] : 1.0;
                bd[c] += am[p][c] + Tstop[p] * (Mc + fabs(cd[p][c]));
                val[4 * o + c] = v[c];
                bound[4 * o + c] = bd[c] * (1.0 + 1e-3) + 1e-12;
            }
            amb[o] = namb[p];
        }
    }
    free(off);
    free(ent);
    stats[0] = dq_max;
    stats[1] = dq_near;
    return over ? -2 : bad;
}

/* ---- f32 emulation of the blend kernel ------------------------------------------------------------------------------------------- */
static uint64_t rng_next(uint64_t *s) {
    uint64_t x = *s;
    x ^= x << 13; x ^= x >> 7; x ^= x << 17;
    return *s = x;
}
static double rng_unit(uint64_t *s) { return (double)(rng_next(s) >> 11) * 0x1p-53; }

/* ex2.approx.ftz.f32 within its stated error: 2^x perturbed by up to 3/4 of 2^-22 relative, plus the rounding to f32, then flushed */
static float ex2_emul(float x, uint64_t *s) {
    const double e = (2.0 * rng_unit(s) - 1.0) * 0.75 * EX2_REL;
    float y = (float)(exp2((double)x) * (1.0 + e));
    return y < 0x1p-126f ? 0.0f : y;
}

static float sat(float v) { return v > 0.0f ? (v < 1.0f ? v : 1.0f) : 0.0f; }

/* The window as the kernel computes it: per-block lists (this file's own, front to back) walked in record pairs (an odd tail pairs with
 * a null record), fmaf in the kernel's order, ex2 perturbed within its error; the block may stop after any pair at which all its
 * in-frame pixels are below `cutoff` (each such pair stops it with probability 1/2).  out32[h][w][4] and out8[h][w][4] (bytes:
 * sat(x) * 255 + round_add, truncated), bottom-up rows.  `drop` (record index, or -1) is left out of every list. */
long bf_emulate(const bf_rec *rec, const uint32_t *order, uint32_t count, int width, int height, int x0, int y0, int w, int h, int tile,
                int form, const float *dest_color, const float *dest_depth, float cutoff, float round_add, int64_t drop, uint64_t seed,
                float *out32, uint8_t *out8) {
    win_t wd;
    if (!init_window(&wd, width, height, x0, y0, w, h, tile)) return -1;
    int64_t *off = NULL;
    uint32_t *ent = NULL;
    const long bad = build_lists(rec, order, count, &wd, drop, &off, &ent);
    if (bad < 0) return -1;
    const int64_t nb = (int64_t)wd.nbx * wd.nby;
#pragma omp parallel for schedule(dynamic, 4)
    for (int64_t blk = 0; blk < nb; ++blk) {
        const int bx = wd.x0 + 8 * (int)(blk % wd.nbx), by = wd.y0 + 8 * (int)(blk / wd.nbx);
        const float tile_x0 = (float)(bx / tile * tile) + 0.5f, tile_y0 = (float)(by / tile * tile) + 0.5f;
        uint64_t s = (seed + 1) * 0x9E3779B97F4A7C15ull ^ (uint64_t)(blk + 1) * 0xD1B54A32D192ED03ull;
        if (!s) s = 1;
        float T[64], R[64][3], dd[64];
        for (int p = 0; p < 64; ++p) {
            const int x = bx + (p & 7), y = by + (p >> 3);
            T[p] = (x < width && y < height) ? 1.0f : 0.0f;
            R[p][0] = R[p][1] = R[p][2] = 0.0f;
            dd[p] = INFINITY;
            if (dest_depth && x < width && y < height) dd[p] = dest_depth[(size_t)y * width + x];
        }
        const int64_t n = off[blk + 1] - off[blk];
        for (int64_t k = 0; k < n; k += 2) {
            for (int j = 0; j < 2; ++j) {
                if (k + j >= n) break;                 /* the null record adds exactly nothing */
                const bf_rec *r = rec + ent[off[blk] + k + j];
                const float zw = fmaf(0.5f, r->z, 0.5f), la = log2f(r->a);
                float u0, w0;
                if (form == FORM_TILE) {
                    const float X0 = tile_x0 - r->cx, Y0 = tile_y0 - r->cy;
                    u0 = fmaf(X0, r->g1x, Y0 * r->g1y); w0 = fmaf(X0, r->g2x, Y0 * r->g2y);
                } else {
                    u0 = -fmaf(r->cx, r->g1x, r->cy * r->g1y); w0 = -fmaf(r->cx, r->g2x, r->cy * r->g2y);
                }
                for (int p = 0; p < 64; ++p) {
                    const int x = bx + (p & 7), y = by + (p >> 3);
                    const float qx = form == FORM_TILE ? (float)x - (tile_x0 - 0.5f) : (float)x + 0.5f;
                    const float qy = form == FORM_TILE ? (float)y - (tile_y0 - 0.5f) : (float)y + 0.5f;
                    const float U = fmaf(qy, r->g1y, fmaf(qx, r->g1x, u0)), W = fmaf(qy, r->g2y, fmaf(qx, r->g2x, w0));
                    const float Q = fmaf(W, W, U * U);
                    const float X = fmaf(Q, KEXP, la);
                    const float e = (Q <= 1.0f && zw <= dd[p]) ? ex2_emul(X, &s) : 0.0f;
                    const float wgt = T[p] * e;
                    R[p][0] = fmaf(wgt, r->r, R[p][0]); R[p][1] = fmaf(wgt, r->g, R[p][1]); R[p][2] = fmaf(wgt, r->b, R[p][2]);
                    T[p] = fmaf(wgt, -1.0f, T[p]);
                }
            }
            int below = 1;
            for (int p = 0; p < 64 && below; ++p) below = T[p] < cutoff;
            if (below && (rng_next(&s) & 1)) break;
        }
        for (int p = 0; p < 64; ++p) {
            const int x = bx + (p & 7), y = by + (p >> 3);
            if (x >= wd.x0 + wd.w || y >= wd.y0 + wd.h) continue;
            const size_t o = (size_t)(y - wd.y0) * wd.w + (x - wd.x0), at = (size_t)y * width + x;
            float v[4] = {R[p][0], R[p][1], R[p][2], 1.0f - T[p]};
            if (dest_color) {
                for (int c = 0; c < 3; ++c) v[c] = fmaf(T[p], dest_color[4 * at + c], v[c]);
                v[3] = fmaf(T[p], dest_color[4 * at + 3], v[3]);
            }
            for (int c = 0; c < 4; ++c) {
                out32[4 * o + c] = v[c];
                out8[4 * o + c] = (uint8_t)(uint32_t)(sat(v[c]) * 255.0f + round_add);
            }
        }
    }
    free(off);
    free(ent);
    return bad;
}
