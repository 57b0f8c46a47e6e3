// region_kernels.cuh -- the largest distance of a splat range from the scene centre: the loop of SplatMesh.updateVisibleRegion
// (src/splatmesh/SplatMesh.js:1172-1199), which drives the fade-in of SplatMaterial.getVertexShaderFadeIn.
//   centre    getSplatCenter(i, c, true): the stored f32 centre through the scene transform by three.js Vector3.applyMatrix4 (f64,
//             divide by w included); the reference multiplies by the identity too, so 0 * inf = NaN there as here
//   distance  tempCenter.sub(sceneCenter).length() = Math.sqrt(x * x + y * y + z * z), f64, unfused, correctly rounded sqrt
//   maximum   `if (d > max) max = d` from 0: a NaN distance never counts.  The distances are >= 0, so their order is the order of their
//             bit patterns and one 64-bit atomicMax gives the same maximum whatever the order the splats are visited in.
#pragma once
#include "common.cuh"

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

} // namespace gs
