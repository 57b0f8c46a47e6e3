// region_kernels.cuh -- reductions over a splat range: its largest distance from the scene centre (k_visible_region) and its bounding
// box (k_bounding_box, below).  The distance is the loop of SplatMesh.updateVisibleRegion
// (src/splatmesh/SplatMesh.js:1172-1199), which drives the fade-in of SplatMaterial.getVertexShaderFadeIn.
//   centre    getSplatCenter(i, c, true): the stored f32 centre through the scene transform by three.js Vector3.applyMatrix4 (f64,
//             divide by w included); the reference multiplies by the identity too, so 0 * inf = NaN there as here
//   distance  tempCenter.sub(sceneCenter).length() = Math.sqrt(x * x + y * y + z * z), f64, unfused, correctly rounded sqrt
//   maximum   `if (d > max) max = d` from 0: a NaN distance never counts.  The distances are >= 0, so their order is the order of their
//             bit patterns and one 64-bit atomicMax gives the same maximum whatever the order the splats are visited in.
#pragma once
#include "common.cuh"
#include "ray_kernels.cuh"    // m4_apply
#include "tree_kernels.cuh"   // f32_ordered

namespace gs {

struct RegionParams {
    double t[16];         // column-major Matrix4
    double center[3];
};

__global__ void __launch_bounds__(256) k_visible_region(const uint4 *__restrict__ cc, uint32_t from, uint32_t to, RegionParams P,
                                                          unsigned long long *__restrict__ max_bits) {
    double m = 0.0;
    for (uint32_t i = from + blockIdx.x * blockDim.x + threadIdx.x; i < to; i += gridDim.x * blockDim.x) {
        const uint4 v = cc[i];
        const double x = __uint_as_float(v.y), y = __uint_as_float(v.z), z = __uint_as_float(v.w);
        const double *T = P.t;
        const double w = __ddiv_rn(1.0, __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[3], x), __dmul_rn(T[7], y)), __dmul_rn(T[11], z)), T[15]));
        const double cx = __dmul_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[0], x), __dmul_rn(T[4], y)), __dmul_rn(T[8], z)), T[12]), w);
        const double cy = __dmul_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[1], x), __dmul_rn(T[5], y)), __dmul_rn(T[9], z)), T[13]), w);
        const double cz = __dmul_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[2], x), __dmul_rn(T[6], y)), __dmul_rn(T[10], z)), T[14]), w);
        const double dx = __dadd_rn(cx, -P.center[0]), dy = __dadd_rn(cy, -P.center[1]), dz = __dadd_rn(cz, -P.center[2]);
        const double d = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
        if (d > m) m = d;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double n = __shfl_down_sync(0xffffffffu, m, o);
        if (n > m) m = n;
    }
    if ((threadIdx.x & 31) == 0 && m > 0.0) atomicMax(max_bits, (unsigned long long)__double_as_longlong(m));
}


// SplatMesh.computeBoundingBox (src/splatmesh/SplatMesh.js:2066-2094) over splats [from, to):
//   centre    the Float32Array value fillSplatCenterArray writes (SplatBuffer.js:307-347): the f64 centre, through the scene transform
//             by Vector3.applyMatrix4 (m4_apply, the ray kernels' restatement) when the scene's bit of `apply` is set, stored as f32
//   compare   `if (i === 0 || x < min.x) min.x = x` and likewise for max: element `from` seeds both, a NaN seed stays, a NaN never
//             replaces anything after it, and of equal values (-0 and +0) the lowest index wins.  So each candidate is a 64-bit key, the
//             f32's order in the high half (-0 counted as +0) and the index in the low half (inverted for the maximum); NaN gets the
//             key that never wins.  The winners' values are then read again by index, so the sign of a winning zero is its own.
// k_bounding_box reduces a grid-stride slice per CTA into 6 keys (min x y z, max x y z); k_bounding_box_final, one CTA, reduces the CTAs'
// keys and writes the box.  Neither depends on the order in which threads run.
struct BoundsParams {
    uint32_t from, to;
    uint32_t apply;                  // bit s: scene s's centres go through xf[16 s .. 16 s + 16)
    const double *xf;                // device f64[16 * GS_MAX_SCENES], column-major
    const uint32_t *scene_idx;       // device scene index per splat, or nullptr: every splat is scene 0
};
constexpr int kBoundsThreads = 256;
__device__ __forceinline__ unsigned long long bounds_none(bool max) { return max ? 0ull : ~0ull; }   // the key that never wins

// kRecords: src is gs_ray_record[] (getSplatCenter's unrounded centre), else the uint4 {colour, x, y, z} of GS_BUF_CENTERS_COLORS
template <bool kRecords>
__device__ __forceinline__ void bounds_center(const void *__restrict__ src, const BoundsParams &P, uint32_t i, float c[3]) {
    double x, y, z;
    if (kRecords) {
        const gs_ray_record *r = static_cast<const gs_ray_record *>(src) + i;
        x = r->center[0]; y = r->center[1]; z = r->center[2];
    } else {
        const uint4 v = static_cast<const uint4 *>(src)[i];
        x = __uint_as_float(v.y); y = __uint_as_float(v.z); z = __uint_as_float(v.w);
    }
    const uint32_t s = P.scene_idx ? P.scene_idx[i] & (GS_MAX_SCENES - 1) : 0u;
    if ((P.apply >> s) & 1u) m4_apply(P.xf + 16 * s, x, y, z);
    c[0] = (float)x; c[1] = (float)y; c[2] = (float)z;
}

__device__ __forceinline__ unsigned long long bounds_key(float v, uint32_t i, bool max) {
    if (v != v) return bounds_none(max);
    const uint32_t ord = f32_ordered(v == 0.0f ? 0u : __float_as_uint(v));
    return ((unsigned long long)ord << 32) | (max ? ~i : i);
}
__device__ __forceinline__ unsigned long long bounds_pick(unsigned long long a, unsigned long long b, bool max) {
    return max ? (a > b ? a : b) : (a < b ? a : b);
}

// The CTA's 6 keys, reduced over its warps; valid in thread 0
__device__ __forceinline__ void bounds_block_reduce(unsigned long long k[6], unsigned long long (*smem)[6]) {
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) k[a] = bounds_pick(k[a], __shfl_down_sync(0xffffffffu, k[a], o), a >= 3);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0)
#pragma unroll
        for (int a = 0; a < 6; ++a) smem[warp][a] = k[a];
    __syncthreads();
    if (threadIdx.x == 0)
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
#pragma unroll
            for (int a = 0; a < 6; ++a) k[a] = bounds_pick(k[a], smem[w][a], a >= 3);
}

template <bool kRecords>
__global__ void __launch_bounds__(kBoundsThreads) k_bounding_box(const void *__restrict__ src, BoundsParams P, unsigned long long *__restrict__ partial) {
    __shared__ unsigned long long smem[kBoundsThreads / 32][6];
    unsigned long long k[6];
#pragma unroll
    for (int a = 0; a < 6; ++a) k[a] = bounds_none(a >= 3);
    for (uint32_t i = P.from + blockIdx.x * blockDim.x + threadIdx.x; i < P.to; i += gridDim.x * blockDim.x) {
        float c[3];
        bounds_center<kRecords>(src, P, i, c);
#pragma unroll
        for (int a = 0; a < 6; ++a) k[a] = bounds_pick(k[a], bounds_key(c[a % 3], i, a >= 3), a >= 3);
    }
    bounds_block_reduce(k, smem);
    if (threadIdx.x == 0)
#pragma unroll
        for (int a = 0; a < 6; ++a) partial[6 * blockIdx.x + a] = k[a];
}

// out: f32[6] = min x y z, max x y z
template <bool kRecords>
__global__ void __launch_bounds__(kBoundsThreads) k_bounding_box_final(const void *__restrict__ src, BoundsParams P, const unsigned long long *__restrict__ partial,
                                                                      uint32_t blocks, float *__restrict__ out) {
    __shared__ unsigned long long smem[kBoundsThreads / 32][6];
    unsigned long long k[6];
#pragma unroll
    for (int a = 0; a < 6; ++a) k[a] = bounds_none(a >= 3);
    for (uint32_t b = threadIdx.x; b < blocks; b += blockDim.x)
#pragma unroll
        for (int a = 0; a < 6; ++a) k[a] = bounds_pick(k[a], partial[6 * b + a], a >= 3);
    bounds_block_reduce(k, smem);
    if (threadIdx.x != 0) return;
    float seed[3];
    bounds_center<kRecords>(src, P, P.from, seed);
    for (int a = 0; a < 6; ++a) {
        const int axis = a % 3;
        float v = seed[axis];
        if (v == v) {   // a finite or infinite seed: some candidate won (the seed itself at least)
            float c[3];
            bounds_center<kRecords>(src, P, a >= 3 ? ~(uint32_t)k[a] : (uint32_t)k[a], c);
            v = c[axis];
        }
        out[a] = v;
    }
}

} // namespace gs
