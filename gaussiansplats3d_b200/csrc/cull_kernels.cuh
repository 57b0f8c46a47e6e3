// cull_kernels.cuh -- the per-frame half of Viewer.gatherSceneNodesForSort (src/Viewer.js:1969-2077) on the GPU (SURVEY.md 8(f) N2):
// which leaves of the SplatTree are in (or near) the view frustum, the kept leaves ordered by distance to the camera, and their index
// runs laid out from the END of the sorter's window backwards -- the nearest leaf LAST (Viewer.js:2040-2055) -- so that a partial sort
// (sortCount < renderCount, Viewer.js:1843-1856, sorter.cpp:158-160) re-sorts exactly the nearest splats.
//   k_tree_cull    one thread per leaf: centre -> view space, distance, the two angle tests          Viewer.js:2013-2033
//   k_tree_layout  one thread per kept leaf: splats of all kept leaves that are nearer (ties: lower leaf number first) -> start of its run
//   k_tree_copy    one CTA per kept leaf: its (ascending) indexes -> indexesToSort[start ...]
// All arithmetic is f64 in the operation order of three.js's Vector3.applyMatrix4 / normalize (JS numbers are doubles), unfused.
#pragma once
#include "common.cuh"

namespace gs {

struct CullParams {
    double mv[16];            // baseModelView: inverse(camera.matrixWorld) [* mesh.matrixWorld], column-major   Viewer.js:2003-2004
    double cos_fov_x_over_2, cos_fov_y_over_2;
    int gather_all;
};

__device__ __forceinline__ void normalize3(double &x, double &y, double &z) {   // Vector3.normalize(): multiplyScalar(1 / (length() || 1))
    const double ln = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
    const double s = __ddiv_rn(1.0, ln != 0.0 ? ln : 1.0);
    x = __dmul_rn(x, s); y = __dmul_rn(y, s); z = __dmul_rn(z, s);
}

constexpr unsigned long long kCulledKey = ~0ull;
constexpr unsigned long long kNaNKey = 0x7ff0000000000001ull;   // every NaN distance, whatever its sign and payload: just above +inf

// kForest: leaf i culls with model view mvs[16 * s] of its sub-tree s (the range of i in sub_leaf[0..subs]): baseModelView *
// sceneTransform(s) (Viewer.js:2005-2011); P.mv is unused
template <bool kForest>
__global__ void k_tree_cull(const double *__restrict__ center, const double *__restrict__ nmin, const double *__restrict__ nmax, uint32_t m, CullParams P,
                            const double *__restrict__ mvs, const uint32_t *__restrict__ sub_leaf, uint32_t subs, unsigned long long *__restrict__ key) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const double x = center[3 * i], y = center[3 * i + 1], z = center[3 * i + 2];
    const double *e = kForest ? mvs + 16 * range_of(sub_leaf, subs, i) : P.mv;
    // Vector3.applyMatrix4: w = 1 / (e3 x + e7 y + e11 z + e15); components (e0 x + e4 y + e8 z + e12) * w, sums left to right
    const double w = __ddiv_rn(1.0, __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e[3], x), __dmul_rn(e[7], y)), __dmul_rn(e[11], z)), e[15]));
    double tx = __dmul_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e[0], x), __dmul_rn(e[4], y)), __dmul_rn(e[8], z)), e[12]), w);
    double ty = __dmul_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e[1], x), __dmul_rn(e[5], y)), __dmul_rn(e[9], z)), e[13]), w);
    double tz = __dmul_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e[2], x), __dmul_rn(e[6], y)), __dmul_rn(e[10], z)), e[14]), w);
    const double dist = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(tx, tx), __dmul_rn(ty, ty)), __dmul_rn(tz, tz)));
    normalize3(tx, ty, tz);
    double ax = 0.0, ay = ty, az = tz;      // tempVectorYZ = copy(t).setX(0).normalize()
    normalize3(ax, ay, az);
    double bx = tx, by = 0.0, bz = tz;      // tempVectorXZ = copy(t).setY(0).normalize()
    normalize3(bx, by, bz);
    // forward.dot(v) with forward = (0, 0, -1): 0 * vx + 0 * vy + (-1) * vz
    const double dot_xz = __dadd_rn(__dadd_rn(__dmul_rn(0.0, bx), __dmul_rn(0.0, by)), __dmul_rn(-1.0, bz));
    const double dot_yz = __dadd_rn(__dadd_rn(__dmul_rn(0.0, ax), __dmul_rn(0.0, ay)), __dmul_rn(-1.0, az));
    const double dx = __dadd_rn(nmax[3 * i], -nmin[3 * i]), dy = __dadd_rn(nmax[3 * i + 1], -nmin[3 * i + 1]), dz = __dadd_rn(nmax[3 * i + 2], -nmin[3 * i + 2]);
    const double ns = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));   // nodeSize: |max - min|
    const bool out_y = dot_yz < __dadd_rn(P.cos_fov_y_over_2, -0.6);
    const bool out_x = dot_xz < __dadd_rn(P.cos_fov_x_over_2, -0.6);
    const bool culled = !P.gather_all && ((out_x || out_y) && dist > ns);
    // distances are >= 0 or NaN: their bit patterns order like the numbers, and one key for every NaN puts them after +inf, among
    // themselves by leaf number (k_tree_layout's tie rule; tree_oracle.leaf_order_key)
    key[i] = culled ? kCulledKey : dist != dist ? kNaNKey : (unsigned long long)__double_as_longlong(dist);
}

constexpr int kLayoutThreads = 256;
__global__ void __launch_bounds__(kLayoutThreads)
k_tree_layout(const unsigned long long *__restrict__ key, const uint32_t *__restrict__ offsets, uint32_t m, uint32_t *__restrict__ start,
              unsigned long long *__restrict__ render_count) {
    __shared__ unsigned long long s_key[kLayoutThreads];
    __shared__ uint32_t s_size[kLayoutThreads];
    const uint32_t i = blockIdx.x * kLayoutThreads + threadIdx.x;
    const unsigned long long ki = i < m ? key[i] : kCulledKey;
    unsigned long long before = 0, total = 0;
    for (uint32_t base = 0; base < m; base += kLayoutThreads) {
        const uint32_t j = base + threadIdx.x;
        s_key[threadIdx.x] = j < m ? key[j] : kCulledKey;
        s_size[threadIdx.x] = j < m ? offsets[j + 1] - offsets[j] : 0u;
        __syncthreads();
        const uint32_t lim = min((uint32_t)kLayoutThreads, m - base);
        for (uint32_t t = 0; t < lim; ++t) {
            const unsigned long long kj = s_key[t];
            if (kj == kCulledKey) continue;
            const uint32_t sz = s_size[t];
            total += sz;
            if (kj < ki || (kj == ki && base + t < i)) before += sz;
        }
        __syncthreads();
    }
    if (i < m) {
        const uint32_t mine = offsets[i + 1] - offsets[i];
        start[i] = ki == kCulledKey ? 0xffffffffu : (uint32_t)(total - before - mine);   // nearest leaf (before = 0) ends the window
    }
    if (i == 0) *render_count = total;
}

__global__ void __launch_bounds__(128)
k_tree_copy(const uint32_t *__restrict__ start, const uint32_t *__restrict__ offsets, const uint32_t *__restrict__ indexes, uint32_t *__restrict__ out) {
    const uint32_t i = blockIdx.x;
    const uint32_t at = start[i];
    if (at == 0xffffffffu) return;
    const uint32_t lo = offsets[i], n = offsets[i + 1] - lo;
    for (uint32_t k = threadIdx.x; k < n; k += blockDim.x) out[at + k] = indexes[lo + k];
}

} // namespace gs
