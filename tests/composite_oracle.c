/* tests/composite_oracle.c -- TEST INFRASTRUCTURE ONLY (never linked into or called by the product path).
 *
 * The CPU blend of oracle/raster_oracle.c (blend_region: fragment shader + NormalBlending per splat, in draw order) drawn into a
 * framebuffer that already holds an opaque pass, as the reference's Viewer draws its threeScene first and then the splat mesh with
 * autoClear off (Viewer.js:1599-1620).  Two changes to that blend, nothing else:
 *   - the frame starts from the destination colour instead of (0,0,0,0);
 *   - a fragment is skipped unless its window depth 0.5 * ndc_z + 0.5 (SplatMaterial3D.js:208-210, glDepthRange(0, 1)) is <= the
 *     destination depth at the pixel (three's default LessEqualDepth; depthTest: true, depthWrite: false, SplatMaterial3D.js:65-75).
 *     A NaN depth passes nothing.
 * Compiled and loaded by tests/composite_oracle.py with the flags of oracle/Makefile (f32, unfused, in the same expression order), so
 * with depth 1 everywhere and a zero destination it returns gso_blend's frame bit for bit.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "../include/gsplat_b200.h"

#define GS_ORACLE_API __attribute__((visibility("default")))

static inline float clamp01(float v) { return v < 0.f ? 0.f : (v > 1.f ? 1.f : v); }

/* The window [cx0, cx0+cw) x [cy0, cy0+chh) of a width x height frame (GL window coordinates, row 0 = bottom); `frame` is cw x chh x 4.
 * dest_color (RGBA float, may be NULL = zero) and dest_depth (may be NULL = no test) are whole width x height frames in the same
 * orientation. */
GS_ORACLE_API void gso_blend_composite_crop(const gs_projected_splat *ps, const uint32_t *sorted_indexes, uint32_t render_count, uint32_t width,
                                            uint32_t height, uint32_t cx0, uint32_t cy0, uint32_t cw, uint32_t chh, int quantize8,
                                            const float *dest_color, const float *dest_depth, float *frame) {
    (void)height;
    for (uint32_t y = 0; y < chh; ++y)
        for (uint32_t x = 0; x < cw; ++x)
            for (int k = 0; k < 4; ++k)
                frame[((size_t)y * cw + x) * 4 + k] = dest_color ? dest_color[((size_t)(y + cy0) * width + (x + cx0)) * 4 + k] : 0.0f;
    int32_t *ylo = (int32_t *)malloc(sizeof(int32_t) * (size_t)(render_count ? render_count : 1));
    int32_t *yhi = (int32_t *)malloc(sizeof(int32_t) * (size_t)(render_count ? render_count : 1));
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
            const float zw = 0.5f * p->ndc_z + 0.5f;
            for (int y = ya; y <= yb; ++y) {
                const float dy = ((float)y + 0.5f) - p->cy;
                for (int x = x0; x <= x1; ++x) {
                    if (dest_depth && !(zw <= dest_depth[(size_t)y * width + (size_t)x])) continue;   /* LessEqualDepth */
                    const float dx = ((float)x + 0.5f) - p->cx;
                    const float qu = (dx * p->b1x + dy * p->b1y) / n1;
                    const float qw = (dx * p->b2x + dy * p->b2y) / n2;
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

GS_ORACLE_API void gso_blend_composite(const gs_projected_splat *ps, const uint32_t *sorted_indexes, uint32_t render_count, uint32_t width,
                                       uint32_t height, int quantize8, const float *dest_color, const float *dest_depth, float *frame) {
    gso_blend_composite_crop(ps, sorted_indexes, render_count, width, height, 0, 0, width, height, quantize8, dest_color, dest_depth, frame);
}
