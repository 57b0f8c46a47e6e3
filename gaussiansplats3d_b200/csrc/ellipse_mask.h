// ellipse_mask.h -- can a rectangle of pixel centres (an 8x8-px block of a tile) contain a pixel a splat covers?  (host + device, no CUDA dependency)
//
// A splat covers pixel p iff q(p) = (g1.(p-c))^2 + (g2.(p-c))^2 <= 1 at the pixel CENTRE (the fragment shader's `A > 8 -> discard`,
// SplatMaterial3D.js:240-243, with A = 8 q).  q is a convex quadratic, so its minimum over a tile's rectangle of pixel centres is 0
// when the rectangle contains c and otherwise lies on one of the four edges, where it is a clamped 1-D minimisation: exact, no sampling.
// A block is kept when that minimum is <= 1 + kEllipseSlack; the slack covers the rounding of this test and of the blend kernel's own
// evaluation of q in f32 (taken relative to the tile's first pixel centre, so it rounds q by ~1e-5 wherever the tile lies in the
// frame), so a block holding a covered pixel is never dropped (the blend kernel applies it per 8x8-px block).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define GS_HD __host__ __device__ __forceinline__
#else
#define GS_HD static inline
#endif
// The position of an edge's minimiser only has to be close: q evaluated next to its minimum differs from it to second order, far
// inside kEllipseSlack.  On the device that allows the approximate divide (no slow-path subroutine).
#if defined(__CUDA_ARCH__)
#define GS_EDGE_DIV(a, b) __fdividef((a), (b))
#else
#define GS_EDGE_DIV(a, b) ((a) / (b))
#endif

constexpr float kEllipseSlack = 2e-3f;

GS_HD float gs_clampf(float v, float lo, float hi) { return v < lo ? lo : (v > hi ? hi : v); }

// minimum of q(x, y) = qxx x^2 + 2 qxy x y + qyy y^2 over the rectangle [x0, x1] x [y0, y1] (coordinates relative to the centre)
GS_HD float ellipse_min_q(float x0, float x1, float y0, float y1, float qxx, float qxy, float qyy) {
    if (x0 <= 0.f && x1 >= 0.f && y0 <= 0.f && y1 >= 0.f) return 0.f;
    float best = 3.0e38f;
    for (int e = 0; e < 2; ++e) {                       // edges x = x0, x = x1
        const float X = e ? x1 : x0;
        const float y = gs_clampf(GS_EDGE_DIV(-qxy * X, qyy), y0, y1);
        const float q = qxx * X * X + 2.f * qxy * X * y + qyy * y * y;
        best = q < best ? q : best;
    }
    for (int e = 0; e < 2; ++e) {                       // edges y = y0, y = y1
        const float Y = e ? y1 : y0;
        const float x = gs_clampf(GS_EDGE_DIV(-qxy * Y, qxx), x0, x1);
        const float q = qxx * x * x + 2.f * qxy * x * Y + qyy * Y * Y;
        best = q < best ? q : best;
    }
    return best;
}
