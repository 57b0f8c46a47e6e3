// sort_kernels.cuh -- depth + bucket + histogram/scan/scatter radix kernels (sm_90a).
//
// Replaces the reference's sortIndexes() (src/worker/sorter.cpp:17-168) stage by stage:
//   k_depth      : distance pass, all six branches            sorter.cpp:29-140   (+ running min/max :24-25)
//   k_bucket     : f32 range map + bucket                      sorter.cpp:142-149  (+ per-digit histograms)
//   k_radix_*    : stable LSD radix sort (hist/scan/scatter)   sorter.cpp:151-167  (prefix sum + backward scatter)
// The reference's output is reverse(stable ascending by bucket); we sort key = (R-1-bucket) ascending, stably,
// over the REVERSED input sequence, which is the same permutation (SURVEY.md Appendix B).
//
// Bit-exactness: all float steps use explicit round-to-nearest intrinsics (no FMA contraction), the *1000.0 and
// *4096.0 products are f64 and truncate toward zero, int32 products wrap (done in uint32).
#pragma once
#include "common.cuh"
#include <utility>

namespace gs {

enum DepthMode : int {
    kIntStatic = 0, kIntDynamic = 1, kIntPrecomputed = 2, kFloatStatic = 3, kFloatDynamic = 4, kFloatPrecomputed = 5
};

struct DepthParams {
    int32_t irow[4];   // static integer mode: trunc(mvp[2,6,10] * 1000.0), 1       sorter.cpp:64
    float frow[4];     // static float mode: mvp[2], mvp[6], mvp[10]                 sorter.cpp:130-133
    float mvp[16];     // dynamic modes: full matrix                                  sorter.cpp:48, :114
};

// ---------------------------------------------------------------------------------------------------------------
__global__ void k_sort_init(SortControl *ctl) {
    pdl_enter();
    const uint32_t tid = threadIdx.x;
    if (tid == 0) {
        ctl->dmin = 2147483640;
        ctl->dmax = -2147483640;
        ctl->error = 0;
    }
    uint32_t *h = &ctl->hist[0][0];
    for (uint32_t i = tid; i < 4 * kRadix; i += blockDim.x) h[i] = 0;
}

// third row of (mvp * T_scene), f32, left-to-right, unfused (sorter.cpp:11-15)
__device__ __forceinline__ void scene_row(const float *mvp, const float *t, float out[4]) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        float acc = __fmul_rn(mvp[2], t[4 * c + 0]);
        acc = __fadd_rn(acc, __fmul_rn(mvp[6], t[4 * c + 1]));
        acc = __fadd_rn(acc, __fmul_rn(mvp[10], t[4 * c + 2]));
        acc = __fadd_rn(acc, __fmul_rn(mvp[14], t[4 * c + 3]));
        out[c] = acc;
    }
}
__device__ __forceinline__ int32_t trunc_scaled(float f, double scale) { return __double2int_rz((double)f * scale); }

template <int MODE>
__device__ __forceinline__ int32_t splat_distance(uint32_t g, const void *__restrict__ centers, const void *__restrict__ pre,
                                                  const uint32_t *__restrict__ scene_idx, const DepthParams &P,
                                                  const int32_t (*s_irow)[4], const float (*s_frow)[4]) {
    if (MODE == kIntPrecomputed) return (int32_t)ld_nc_u32((const uint32_t *)pre + g);
    if (MODE == kFloatPrecomputed) return trunc_scaled(__uint_as_float(ld_nc_u32((const uint32_t *)pre + g)), 4096.0);
    const int4 c = ld_nc_v4((const int4 *)centers + g);
    if (MODE == kIntStatic) {
        return (int32_t)((uint32_t)P.irow[0] * (uint32_t)c.x + (uint32_t)P.irow[1] * (uint32_t)c.y + (uint32_t)P.irow[2] * (uint32_t)c.z);
    } else if (MODE == kIntDynamic) {
        const int32_t *r = s_irow[ld_nc_u32(scene_idx + g) & (GS_MAX_SCENES_DEV - 1)];
        return (int32_t)((uint32_t)r[0] * (uint32_t)c.x + (uint32_t)r[1] * (uint32_t)c.y + (uint32_t)r[2] * (uint32_t)c.z +
                         (uint32_t)r[3] * (uint32_t)c.w);
    } else if (MODE == kFloatStatic) {
        float acc = __fmul_rn(P.frow[0], __int_as_float(c.x));
        acc = __fadd_rn(acc, __fmul_rn(P.frow[1], __int_as_float(c.y)));
        acc = __fadd_rn(acc, __fmul_rn(P.frow[2], __int_as_float(c.z)));
        return trunc_scaled(acc, 4096.0);
    } else { // kFloatDynamic
        const float *r = s_frow[ld_nc_u32(scene_idx + g) & (GS_MAX_SCENES_DEV - 1)];
        float acc = __fmul_rn(r[0], __int_as_float(c.x));
        acc = __fadd_rn(acc, __fmul_rn(r[1], __int_as_float(c.y)));
        acc = __fadd_rn(acc, __fmul_rn(r[2], __int_as_float(c.z)));
        acc = __fadd_rn(acc, __fmul_rn(r[3], __int_as_float(c.w)));
        return trunc_scaled(acc, 4096.0);
    }
}

constexpr int kDepthThreads = 256;
constexpr int kDepthItems = 4;

// dist[i] for i in [s0, rc); indexes == nullptr means identity.  One min/max atomic pair per block.
// VIEWS: the depth of every view of a multi-view frame in one launch, blockIdx.y = view v, with camera Pp[v], distances
// dist[v rc + i] and min/max in ctl[v].
template <int MODE, bool IDENTITY, bool VIEWS = false>
__global__ void __launch_bounds__(kDepthThreads)
k_depth(const uint32_t *__restrict__ indexes, const void *__restrict__ centers, const void *__restrict__ pre,
        const uint32_t *__restrict__ scene_idx, const float *__restrict__ transforms, const DepthParams *__restrict__ Pp, uint32_t s0,
        uint32_t rc, int32_t *__restrict__ dist, SortControl *ctl) {
    pdl_enter();
    if (VIEWS) { Pp += blockIdx.y; dist += (size_t)blockIdx.y * rc; ctl += blockIdx.y; }
    // per-frame parameters live in device memory so that a captured CUDA graph of the frame can be replayed unchanged
    DepthParams P;
#pragma unroll
    for (int i = 0; i < 4; ++i) { P.irow[i] = __ldg(&Pp->irow[i]); P.frow[i] = __ldg(&Pp->frow[i]); }
    if (MODE == kIntDynamic || MODE == kFloatDynamic) {
#pragma unroll
        for (int i = 0; i < 16; ++i) P.mvp[i] = __ldg(&Pp->mvp[i]);
    }
    __shared__ int32_t s_irow[GS_MAX_SCENES_DEV][4];
    __shared__ float s_frow[GS_MAX_SCENES_DEV][4];
    __shared__ int s_min[kDepthThreads / 32], s_max[kDepthThreads / 32];
    if (MODE == kIntDynamic || MODE == kFloatDynamic) {
        if (threadIdx.x < GS_MAX_SCENES_DEV) {
            float row[4];
            scene_row(P.mvp, transforms + 16 * threadIdx.x, row);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                s_frow[threadIdx.x][k] = row[k];
                s_irow[threadIdx.x][k] = trunc_scaled(row[k], 1000.0);
            }
        }
        __syncthreads();
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) ctl->error = 0;   // only k_bucket (a later kernel) raises error bits
    int32_t lmin = 2147483640, lmax = -2147483640;
    const uint32_t tile = kDepthThreads * kDepthItems;
    for (uint64_t base = (uint64_t)s0 + (uint64_t)blockIdx.x * tile; base < rc; base += (uint64_t)gridDim.x * tile) {
        uint32_t g[kDepthItems];
#pragma unroll
        for (int k = 0; k < kDepthItems; ++k) {
            const uint64_t i = base + (uint64_t)k * kDepthThreads + threadIdx.x;
            g[k] = (i < rc) ? (IDENTITY ? (uint32_t)i : ld_nc_u32(indexes + i)) : 0xffffffffu;
        }
        int32_t d[kDepthItems];
#pragma unroll
        for (int k = 0; k < kDepthItems; ++k)
            if (g[k] != 0xffffffffu) d[k] = splat_distance<MODE>(g[k], centers, pre, scene_idx, P, s_irow, s_frow);
#pragma unroll
        for (int k = 0; k < kDepthItems; ++k) {
            const uint64_t i = base + (uint64_t)k * kDepthThreads + threadIdx.x;
            if (i < rc) {
                dist[i] = d[k];
                lmin = min(lmin, d[k]);
                lmax = max(lmax, d[k]);
            }
        }
    }
    lmin = warp_min(lmin);
    lmax = warp_max(lmax);
    if ((threadIdx.x & 31) == 0) { s_min[threadIdx.x >> 5] = lmin; s_max[threadIdx.x >> 5] = lmax; }
    __syncthreads();
    if (threadIdx.x < 32) {
        lmin = threadIdx.x < kDepthThreads / 32 ? s_min[threadIdx.x] : 2147483640;
        lmax = threadIdx.x < kDepthThreads / 32 ? s_max[threadIdx.x] : -2147483640;
        lmin = warp_min(lmin);
        lmax = warp_max(lmax);
        if (threadIdx.x == 0) {
            atomicMin(&ctl->dmin, lmin);
            atomicMax(&ctl->dmax, lmax);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Stable LSD radix sort, 8-bit digits, three kernels per pass and NO cross-CTA dependency chain:
//   H  k_radix_hist    per-tile digit histogram            -> tile_hist[digit][tile]   (+ global digit totals)
//   S  k_radix_scan    per digit: exclusive scan over tiles + global digit base (in place: counts become offsets)
//   P  k_radix_scatter rank inside the tile (peer masks from warp votes), reorder through shared memory, coalesced scatter
// A one-sweep (decoupled look-back) variant was measured first: at the sizes of this path (1M-16M keys, ~300 co-resident
// CTAs) the look-back chain of the first wave costs ~k/2 L2 round trips for tile k and dominated the pass (profiles/).
//   tile = kRadixThreads * kRadixItems consecutive elements; warp w owns a contiguous 32*ITEMS run, item k of lane l
//   is element run_base + 32k + l, so (warp, k, lane) order == sequence order and ranks are stable.
struct PassPlan {
    int npasses;
    int shift[4];
    int bits[4];
};

constexpr int kRadixThreads = 512;
constexpr int kRadixItems = 8;
constexpr int kRadixTile = kRadixThreads * kRadixItems;
constexpr int kRadixWarps = kRadixThreads / 32;

enum ValMode : int { kValArray = 0, kValArrayReversed = 1, kValIotaReversed = 2 };

// Lanes of the warp holding the same (<= NB-bit) value, from NB warp votes (8 for a full tile, 9 when tail items use the private bin 256).  MATCH.ANY does this in one instruction but is a
// low-throughput instruction (it limited the scatter kernel when it was used); VOTE is full rate.
template <int NB>
__device__ __forceinline__ uint32_t warp_peers(uint32_t d) {
    uint32_t peers = 0xffffffffu;
#pragma unroll
    for (int b = 0; b < NB; ++b) {
        const bool bit = (d >> b) & 1u;
        const uint32_t vote = __ballot_sync(0xffffffffu, bit);
        peers &= bit ? vote : ~vote;
    }
    return peers;
}

// Bucket + key (sorter.cpp:142-149), one CTA per radix tile of the REVERSED sequence: key[j] = (R-1) - bucket(dist[i]) with
// j = rc-1-i.  Also the pass-0 tile histogram and pass-0 global digit totals (H of pass 0 fused here).
// Optionally leaves the bucket in dist[i] (the reference's mappedDistances).
template <typename KeyT>
__global__ void __launch_bounds__(kRadixThreads)
k_bucket(int32_t *__restrict__ dist /* distances of the n sorted positions (dist + sortStart) */, KeyT *__restrict__ keys, uint32_t n_host,
         const unsigned long long *__restrict__ n_dev, uint32_t R, PassPlan plan, int write_buckets, SortControl *ctl,
         uint32_t *__restrict__ tile_hist, uint32_t stride) {
    pdl_enter();
    __shared__ uint32_t s_hist[kRadix];
    if (threadIdx.x < kRadix) s_hist[threadIdx.x] = 0;
    __syncthreads();
    const int32_t dmin = ctl->dmin, dmax = ctl->dmax;
    const float span = __fsub_rn(__int2float_rn(dmax), __int2float_rn(dmin)); // sorter.cpp:142
    const float range_map = __fdiv_rn(__uint2float_rn(R - 1u), span);          // sorter.cpp:143
    const bool degenerate = (dmax == dmin);
    uint32_t err = 0;
    const uint32_t n = n_dev ? (uint32_t)*n_dev : n_host;   // device-side count: the per-GPU subset of a sharded frame
    const uint64_t jbase = (uint64_t)blockIdx.x * kRadixTile;
    int32_t d[kRadixItems];
#pragma unroll
    for (int k = 0; k < kRadixItems; ++k) {
        const uint64_t j = jbase + (uint64_t)k * kRadixThreads + threadIdx.x;
        d[k] = (j < n) ? dist[(uint64_t)n - 1u - j] : 0;
    }
#pragma unroll
    for (int k = 0; k < kRadixItems; ++k) {
        const uint64_t j = jbase + (uint64_t)k * kRadixThreads + threadIdx.x;
        if (j < n) {
            const int32_t rel = (int32_t)((uint32_t)d[k] - (uint32_t)dmin);
            int32_t b = __float2int_rz(__fmul_rn(__int2float_rn(rel), range_map)); // sorter.cpp:146
            if (degenerate) b = 0;               // defined deviation: the reference traps / writes out of bounds
            // f32 rounding can push the farthest splat's bucket to exactly R at 2^22..2^24 ranges (the reference then writes
            // frequencies[R], outside its prefix sum): clamp.  A negative (d - min) means int32 wrap-around: report.
            if (rel < 0 || b < 0) { err |= kErrBucketRange; b = 0; }
            else if ((uint32_t)b >= R) b = (int32_t)(R - 1u);
            if (write_buckets) dist[(uint64_t)n - 1u - j] = b;
            const uint32_t key = (R - 1u) - (uint32_t)b;
            keys[j] = (KeyT)key;
            // shared-memory atomics: measured faster here than grouping equal digits with MATCH.ANY (2x slower) or ballots (1.4x)
            atomicAdd(&s_hist[(key >> plan.shift[0]) & ((1u << plan.bits[0]) - 1u)], 1u);
        }
    }
    __syncthreads();
    if (threadIdx.x < kRadix) {
        const uint32_t v = s_hist[threadIdx.x];
        tile_hist[(size_t)threadIdx.x * stride + blockIdx.x] = v;
        if (v) atomicAdd(&ctl->hist[0][threadIdx.x], v);
    }
    if (err) atomicOr(&ctl->error, err);
    if (degenerate && blockIdx.x == 0 && threadIdx.x == 0) atomicOr(&ctl->error, kErrDegenerate);
}

// Multi-view frames: k_bucket for every view at once, over the concatenation of the views' REVERSED sort windows.  Element J = v n + j
// (n = rc - s0) is view v's position i = rc-1-j, bucketed with view v's own min/max (ctl[v]); its key is (v << key_bits) | (R-1 - bucket)
// and its value the index at i.  One stable sort of the nviews x n keys then leaves view v's order in [v n, (v + 1) n), the
// permutation gs_sort gives for that view alone.  Pass 0's tile histogram and global digit totals go to ctl[0], as do the error bits.
__global__ void __launch_bounds__(kRadixThreads)
k_bucket_views(const int32_t *__restrict__ dist /* [nviews][rc] */, uint32_t s0, uint32_t rc, const uint32_t *__restrict__ indexes, uint32_t nviews,
               uint32_t R, int key_bits, PassPlan plan, SortControl *ctl, uint32_t *__restrict__ keys, uint32_t *__restrict__ vals,
               uint32_t *__restrict__ tile_hist, uint32_t stride) {
    __shared__ uint32_t s_hist[kRadix];
    __shared__ int32_t s_min[GS_MAX_VIEWS];
    __shared__ float s_map[GS_MAX_VIEWS];
    __shared__ uint32_t s_degenerate[GS_MAX_VIEWS];
    if (threadIdx.x < kRadix) s_hist[threadIdx.x] = 0;
    if (threadIdx.x < nviews) {   // sorter.cpp:142-143, per view
        const int32_t dmin = ctl[threadIdx.x].dmin, dmax = ctl[threadIdx.x].dmax;
        const float span = __fsub_rn(__int2float_rn(dmax), __int2float_rn(dmin));
        s_min[threadIdx.x] = dmin;
        s_map[threadIdx.x] = __fdiv_rn(__uint2float_rn(R - 1u), span);
        s_degenerate[threadIdx.x] = dmax == dmin;
    }
    __syncthreads();
    uint32_t err = 0;
    const uint32_t n = rc - s0, total = n * nviews;
    const uint32_t jbase = blockIdx.x * kRadixTile;
#pragma unroll
    for (int k = 0; k < kRadixItems; ++k) {
        const uint32_t J = jbase + (uint32_t)k * kRadixThreads + threadIdx.x;
        if (J < total) {
            const uint32_t v = J / n, i = rc - 1u - (J - v * n);
            const int32_t rel = (int32_t)((uint32_t)dist[(size_t)v * rc + i] - (uint32_t)s_min[v]);
            int32_t b = __float2int_rz(__fmul_rn(__int2float_rn(rel), s_map[v]));   // sorter.cpp:146
            if (s_degenerate[v]) b = 0;
            if (rel < 0 || b < 0) { err |= kErrBucketRange; b = 0; }
            else if ((uint32_t)b >= R) b = (int32_t)(R - 1u);
            const uint32_t key = (v << key_bits) | ((R - 1u) - (uint32_t)b);
            keys[J] = key;
            vals[J] = indexes ? ld_nc_u32(indexes + i) : i;
            atomicAdd(&s_hist[(key >> plan.shift[0]) & ((1u << plan.bits[0]) - 1u)], 1u);
        }
    }
    __syncthreads();
    if (threadIdx.x < kRadix) {
        const uint32_t h = s_hist[threadIdx.x];
        tile_hist[(size_t)threadIdx.x * stride + blockIdx.x] = h;
        if (h) atomicAdd(&ctl->hist[0][threadIdx.x], h);
    }
    if (err) atomicOr(&ctl->error, err);
    if (blockIdx.x == 0 && threadIdx.x < nviews && s_degenerate[threadIdx.x]) atomicOr(&ctl->error, kErrDegenerate);
}

// Multi-view frames: every view's control block as k_sort_init leaves one.  One CTA per view.
// (This kernel, k_bucket_views and k_views_assemble are ordinary launches: they wait for their predecessors to finish.)
__global__ void k_sort_init_views(SortControl *ctl) {
    SortControl *c = ctl + blockIdx.x;
    if (threadIdx.x == 0) { c->dmin = 2147483640; c->dmax = -2147483640; c->error = 0; }
    uint32_t *h = &c->hist[0][0];
    for (uint32_t i = threadIdx.x; i < 4 * kRadix; i += blockDim.x) h[i] = 0;
}

// Multi-view partial sorts: view v's draw order out[v rc, (v + 1) rc) = the unsorted head [0, s0) of the index list (sorter.cpp:158-160)
// followed by the view's sorted window sorted[v n, (v + 1) n).  blockIdx.y = view.
__global__ void k_views_assemble(const uint32_t *__restrict__ indexes, const uint32_t *__restrict__ sorted, uint32_t s0, uint32_t rc, uint32_t *__restrict__ out) {
    const uint32_t v = blockIdx.y, n = rc - s0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < rc; i += gridDim.x * blockDim.x)
        out[(size_t)v * rc + i] = i < s0 ? (indexes ? indexes[i] : i) : sorted[(size_t)v * n + i - s0];
}

// H: per-tile digit histogram; `add_global` also accumulates the pass's global digit totals.
template <typename KeyT>
__global__ void __launch_bounds__(kRadixThreads)
k_radix_hist(const KeyT *__restrict__ keys, uint32_t n_host, const unsigned long long *__restrict__ n_dev, unsigned long long n_cap,
             int shift, int bits, uint32_t *__restrict__ tile_hist, uint32_t stride, uint32_t *global_hist, int add_global) {
    pdl_enter();
    const uint32_t n = n_dev ? (uint32_t)min(*n_dev, n_cap) : n_host;
    const uint64_t base = (uint64_t)blockIdx.x * kRadixTile;
    if (base >= n) return;
    __shared__ uint32_t s_hist[kRadix];
    if (threadIdx.x < kRadix) s_hist[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t dmask = (1u << bits) - 1u;
    uint32_t kk[kRadixItems];
#pragma unroll
    for (int k = 0; k < kRadixItems; ++k) {
        const uint64_t e = base + (uint64_t)k * kRadixThreads + threadIdx.x;
        kk[k] = (e < n) ? (((uint32_t)keys[e] >> shift) & dmask) : 0xffffffffu;
    }
#pragma unroll
    for (int k = 0; k < kRadixItems; ++k)
        if (kk[k] != 0xffffffffu) atomicAdd(&s_hist[kk[k]], 1u);
    __syncthreads();
    if (threadIdx.x < kRadix) {
        const uint32_t v = s_hist[threadIdx.x];
        tile_hist[(size_t)threadIdx.x * stride + blockIdx.x] = v;
        if (add_global && v) atomicAdd(global_hist + threadIdx.x, v);
    }
}

// S: one CTA per digit.  tile_hist[d][t] (count) -> global output offset of tile t's first element with digit d.
constexpr int kScanColThreads = 1024;
__global__ void __launch_bounds__(kScanColThreads)
k_radix_scan(uint32_t *__restrict__ tile_hist, uint32_t stride, uint32_t n_host, const unsigned long long *__restrict__ n_dev,
             unsigned long long n_cap, const uint32_t *__restrict__ global_hist) {
    pdl_enter();
    __shared__ uint32_t s_scan[40];
    __shared__ uint32_t s_carry;
    const uint32_t n = n_dev ? (uint32_t)min(*n_dev, n_cap) : n_host;
    const uint32_t ntiles = (uint32_t)(((uint64_t)n + kRadixTile - 1) / kRadixTile);
    const uint32_t d = blockIdx.x;
    {   // global base of this digit = total of all smaller digits
        uint32_t total;
        const uint32_t c = (threadIdx.x < kRadix && threadIdx.x < d) ? global_hist[threadIdx.x] : 0u;
        (void)block_exclusive_scan<kScanColThreads>(c, s_scan, total);
        if (threadIdx.x == 0) s_carry = total;
    }
    __syncthreads();
    uint32_t *col = tile_hist + (size_t)d * stride;
    for (uint32_t base = 0; base < ntiles; base += kScanColThreads) {
        const uint32_t t = base + threadIdx.x;
        const uint32_t v = t < ntiles ? col[t] : 0u;
        uint32_t total;
        const uint32_t ex = block_exclusive_scan<kScanColThreads>(v, s_scan, total);
        const uint32_t carry = s_carry;
        if (t < ntiles) col[t] = ex + carry;
        __syncthreads();
        if (threadIdx.x == 0) s_carry = carry + total;
        __syncthreads();
    }
}

// P: stable scatter of one tile.  RANGES (final pass of the tile-instance sort): the tile's reorder buffer is fully sorted by
// key, so [first, last+1) of every key's run is found from neighbours; runs may continue in other tiles -> atomicMin/Max.
// Register diet (3 CTAs/SM): values are loaded only after ranking, element indices are 32-bit, full tiles skip bounds checks,
// and the peer masks of a thread's 8 items are computed back to back before the serial counter updates that consume them.
template <typename KeyT, typename ValT, int VALMODE, bool WRITE_KEYS, bool RANGES, bool FULL>
__device__ __forceinline__ void radix_scatter_tile(const KeyT *__restrict__ keys_in, const ValT *__restrict__ vals_in, uint32_t iota_top,
                                                   KeyT *__restrict__ keys_out, ValT *__restrict__ vals_out, uint32_t n, uint32_t tile,
                                                   int shift, uint32_t dmask, const uint32_t *__restrict__ tile_offsets, uint32_t stride,
                                                   uint2 *ranges, unsigned char *s_raw, uint32_t *s_tile_count, uint32_t *s_tile_start,
                                                   uint32_t *s_gbase, uint32_t *s_scan) {
    uint32_t(*s_whist)[kRadix + 1] = reinterpret_cast<uint32_t(*)[kRadix + 1]>(s_raw);
    ValT *s_vals = reinterpret_cast<ValT *>(s_raw);
    KeyT *s_keys = reinterpret_cast<KeyT *>(s_raw + (size_t)kRadixTile * sizeof(ValT));
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t tile_base = tile * (uint32_t)kRadixTile;
    const uint32_t run_base = tile_base + (uint32_t)warp * (32 * kRadixItems) + lane;
    for (int i = tid; i < kRadixWarps * (kRadix + 1); i += kRadixThreads) (&s_whist[0][0])[i] = 0;

    uint32_t key[kRadixItems];
#pragma unroll
    for (int k = 0; k < kRadixItems; ++k) {
        const uint32_t e = run_base + (uint32_t)k * 32;
        key[k] = (FULL || e < n) ? (uint32_t)keys_in[e] : 0xffffffffu;
    }
    const uint32_t my_offset = tid < kRadix ? tile_offsets[(size_t)tid * stride + tile] : 0u;
    uint32_t peers[kRadixItems];
#pragma unroll
    for (int k = 0; k < kRadixItems; ++k) {
        const uint32_t d = (FULL || key[k] != 0xffffffffu) ? ((key[k] >> shift) & dmask) : (uint32_t)kRadix; // tail items: private bin
        peers[k] = warp_peers<FULL ? 8 : 9>(d);
    }
    __syncthreads();
    uint32_t rank[kRadixItems];
    const uint32_t lt = lanemask_lt();
#pragma unroll
    for (int k = 0; k < kRadixItems; ++k) {
        const uint32_t d = (FULL || key[k] != 0xffffffffu) ? ((key[k] >> shift) & dmask) : (uint32_t)kRadix;
        const uint32_t before = s_whist[warp][d];
        rank[k] = before + __popc(peers[k] & lt);
        __syncwarp();
        if ((peers[k] & lt) == 0) s_whist[warp][d] = before + __popc(peers[k]);
        __syncwarp();
    }
    __syncthreads();
    // ---- per digit: exclusive scan over warps, tile totals -------------------------------------------------------
    if (tid < kRadix) {
        uint32_t run = 0;
#pragma unroll
        for (int w = 0; w < kRadixWarps; ++w) {
            const uint32_t c = s_whist[w][tid];
            s_whist[w][tid] = run;
            run += c;
        }
        s_tile_count[tid] = run;
    }
    __syncthreads();
    {
        uint32_t total;
        const uint32_t c = tid < kRadix ? s_tile_count[tid] : 0u;
        const uint32_t ex = block_exclusive_scan<kRadixThreads>(c, s_scan, total);
        if (tid < kRadix) { s_tile_start[tid] = ex; s_gbase[tid] = my_offset - ex; }
    }
    __syncthreads();
    // reorder slots for my items (read the counters before the reorder buffers overwrite them)
#pragma unroll
    for (int k = 0; k < kRadixItems; ++k) {
        const uint32_t d = (key[k] >> shift) & dmask;
        rank[k] = (FULL || key[k] != 0xffffffffu) ? (s_tile_start[d] + s_whist[warp][d] + rank[k]) : 0xffffffffu;
    }
    __syncthreads();
    // ---- values are fetched only now (keeps 8 registers free during ranking), then reordered through shared memory -------------
#pragma unroll
    for (int k = 0; k < kRadixItems; ++k) {
        const uint32_t e = run_base + (uint32_t)k * 32;
        if (FULL || rank[k] != 0xffffffffu) {
            ValT v;
            if (VALMODE == kValArray) v = __ldg(vals_in + e);
            else if (VALMODE == kValArrayReversed) v = __ldg(vals_in + (n - 1u - e));
            else v = (ValT)(iota_top - e);
            s_vals[rank[k]] = v;
            s_keys[rank[k]] = (KeyT)key[k];
        }
    }
    __syncthreads();
    const uint32_t valid = FULL ? (uint32_t)kRadixTile : (n - tile_base);
#pragma unroll
    for (int k = 0; k < kRadixItems; ++k) {
        const uint32_t q = (uint32_t)k * kRadixThreads + tid;
        if (FULL || q < valid) {
            const KeyT kk = s_keys[q];
            const uint32_t d = ((uint32_t)kk >> shift) & dmask;
            const uint32_t dst = s_gbase[d] + q;
            vals_out[dst] = s_vals[q];
            if (WRITE_KEYS) keys_out[dst] = kk;
            if (RANGES) {
                if (q == 0 || s_keys[q - 1] != kk) atomicMin(&ranges[(uint32_t)kk].x, dst);
                if (q + 1 == valid || s_keys[q + 1] != kk) atomicMax(&ranges[(uint32_t)kk].y, dst + 1u);
            }
        }
    }
}

template <typename KeyT, typename ValT, int VALMODE, bool WRITE_KEYS, bool RANGES>
__global__ void __launch_bounds__(kRadixThreads, 2)
k_radix_scatter(const KeyT *__restrict__ keys_in, const ValT *__restrict__ vals_in, uint32_t iota_top,
                KeyT *__restrict__ keys_out, ValT *__restrict__ vals_out, uint32_t n_host,
                const unsigned long long *__restrict__ n_dev, unsigned long long n_cap, int shift, int bits,
                const uint32_t *__restrict__ tile_offsets, uint32_t stride, uint2 *ranges, uint32_t *clear_hist, SortControl *reset_ctl) {
    pdl_enter();
    const uint32_t n = n_dev ? (uint32_t)min(*n_dev, n_cap) : n_host;
    const uint32_t tile = blockIdx.x;
    // self-cleaning control block (no init kernel on the frame's critical path): this pass's digit totals were consumed by the
    // scan that ran before this kernel; the final pass also re-seeds min/max (sorter.cpp:24-25) for the next sort
    if (tile == 0) {
        if (clear_hist && threadIdx.x < kRadix) clear_hist[threadIdx.x] = 0;
        if (reset_ctl && threadIdx.x == 0) { reset_ctl->dmin = 2147483640; reset_ctl->dmax = -2147483640; }
    }
    const uint64_t tile_base = (uint64_t)tile * kRadixTile;
    if (tile_base >= n) return; // surplus CTA of a capacity-sized grid (uniform exit)
    // phase A: per-warp digit counters; phase B: reorder buffers (aliased)
    __shared__ __align__(16) unsigned char s_raw[kRadixTile * (sizeof(KeyT) + sizeof(ValT)) > kRadixWarps * (kRadix + 1) * 4
                                                     ? kRadixTile * (sizeof(KeyT) + sizeof(ValT))
                                                     : kRadixWarps * (kRadix + 1) * 4];
    __shared__ uint32_t s_tile_count[kRadix];  // digit totals of this tile
    __shared__ uint32_t s_tile_start[kRadix];  // exclusive scan of the above (slot in the reorder buffer)
    __shared__ uint32_t s_gbase[kRadix];       // global slot of reorder-slot 0 for each digit (wrapping arithmetic)
    __shared__ uint32_t s_scan[40];
    const uint32_t dmask = (1u << bits) - 1u;
    if (tile_base + kRadixTile <= n)
        radix_scatter_tile<KeyT, ValT, VALMODE, WRITE_KEYS, RANGES, true>(keys_in, vals_in, iota_top, keys_out, vals_out, n, tile, shift, dmask, tile_offsets, stride,
                                                                          ranges, s_raw, s_tile_count, s_tile_start, s_gbase, s_scan);
    else
        radix_scatter_tile<KeyT, ValT, VALMODE, WRITE_KEYS, RANGES, false>(keys_in, vals_in, iota_top, keys_out, vals_out, n, tile, shift, dmask, tile_offsets, stride,
                                                                           ranges, s_raw, s_tile_count, s_tile_start, s_gbase, s_scan);
}

// out[0..s0) = indexes[0..s0)   (sorter.cpp:158-160)
__global__ void k_copy_head(const uint32_t *__restrict__ indexes, uint32_t *__restrict__ out, uint32_t s0) {
    pdl_enter();
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < s0; i += (uint64_t)gridDim.x * blockDim.x)
        out[i] = indexes ? indexes[i] : (uint32_t)i;
}

// ---- scratch reproduction for the stateless drop-in: frequencies[b] = #sorted splats in buckets < b --------------------
__global__ void k_bucket_counts(const int32_t *__restrict__ buckets, uint32_t s0, uint32_t rc, uint32_t *counts) {
    for (uint64_t i = (uint64_t)s0 + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < rc; i += (uint64_t)gridDim.x * blockDim.x)
        atomicAdd(&counts[buckets[i]], 1u);
}
__global__ void __launch_bounds__(1024) k_exclusive_scan_single_block(uint32_t *data, uint32_t n) {
    __shared__ uint32_t s_scan[40];
    __shared__ uint32_t s_carry;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < n; base += 1024) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t v = i < n ? data[i] : 0u;
        uint32_t total;
        const uint32_t ex = block_exclusive_scan<1024>(v, s_scan, total);
        const uint32_t carry = s_carry;
        if (i < n) data[i] = ex + carry;
        __syncthreads();
        if (threadIdx.x == 0) s_carry = carry + total;
        __syncthreads();
    }
}

// Calls f(mode, identity, views, kernel) for each k_depth instantiation: the launch picks one, the preloads take them all.  Multi-view
// frames compute their distances (precomputed distances belong to one camera).
template <typename F> static void for_each_depth(F &&f) {
#define GS_DEPTH(M, V) f(M, false, V, k_depth<M, false, V>); f(M, true, V, k_depth<M, true, V>)
    GS_DEPTH(kIntStatic, false); GS_DEPTH(kIntDynamic, false); GS_DEPTH(kIntPrecomputed, false); GS_DEPTH(kFloatStatic, false); GS_DEPTH(kFloatDynamic, false);
    GS_DEPTH(kFloatPrecomputed, false);
    GS_DEPTH(kIntStatic, true); GS_DEPTH(kIntDynamic, true); GS_DEPTH(kFloatStatic, true); GS_DEPTH(kFloatDynamic, true);
#undef GS_DEPTH
}

// ---- D1: SplatMesh.computeDistancesOnGPU (SplatMesh.js:1451-1502): distances in SPLAT order ---------------------------
template <bool INTEGER, bool DYNAMIC>
__global__ void k_distances_splat_order(const void *__restrict__ centers, const uint32_t *__restrict__ scene_idx,
                                        const int32_t *__restrict__ irows /*[scenes][4]*/, const float *__restrict__ frows,
                                        uint32_t count, void *__restrict__ out) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (uint64_t)gridDim.x * blockDim.x) {
        const int4 c = ld_nc_v4((const int4 *)centers + i);
        const uint32_t sc = DYNAMIC ? (scene_idx[i] & (GS_MAX_SCENES_DEV - 1)) : 0u;
        if (INTEGER) {
            const int32_t *r = irows + 4 * sc;
            uint32_t d = (uint32_t)c.x * (uint32_t)r[0] + (uint32_t)c.y * (uint32_t)r[1] + (uint32_t)c.z * (uint32_t)r[2];
            if (DYNAMIC) d += (uint32_t)r[3] * (uint32_t)c.w;
            ((int32_t *)out)[i] = (int32_t)d;
        } else {
            const float *r = frows + 4 * sc;
            float acc = __fmul_rn(__int_as_float(c.x), r[0]);
            acc = __fadd_rn(acc, __fmul_rn(__int_as_float(c.y), r[1]));
            acc = __fadd_rn(acc, __fmul_rn(__int_as_float(c.z), r[2]));
            if (DYNAMIC) acc = __fadd_rn(acc, r[3]);
            ((float *)out)[i] = acc;
        }
    }
}


// ---------------------------------------------------------------------------------------------------------------
// Host side of the radix sort
static inline PassPlan make_plan_bits(int key_bits) {
    PassPlan pl{};
    int np = (key_bits + kRadixBits - 1) / kRadixBits;
    if (np < 1) np = 1;
    pl.npasses = np;
    int done = 0;
    for (int p = 0; p < np; ++p) {
        const int left = key_bits - done, b = (left + (np - p) - 1) / (np - p);
        pl.shift[p] = done;
        pl.bits[p] = b < 1 ? 1 : b;
        done += b;
    }
    return pl;
}

// Calls f(valmode, write_keys, ranges, kernel) for each k_radix_scatter variant a sort of (KeyT, ValT) can launch: the only ones
// compiled.  valmode is the first pass's (later passes read an array); a one-pass sort is first and last at once.
template <typename KeyT, typename ValT, typename F> static void for_each_scatter(F &&f) {
#define GS_SCATTER(VM, WK, RG) f(VM, WK, RG, k_radix_scatter<KeyT, ValT, VM, WK, RG>)
    if constexpr (sizeof(ValT) == 8) {          // tile-instance sort (radix binning): two passes, the last writes ranges and no keys
        GS_SCATTER(kValArray, true, false); GS_SCATTER(kValArray, false, true);
    } else if constexpr (sizeof(KeyT) == 2) {   // depth and sharded sorts of <= 16-bit keys: one or two passes
        GS_SCATTER(kValArrayReversed, false, false); GS_SCATTER(kValIotaReversed, false, false);   // depth, one pass
        GS_SCATTER(kValArrayReversed, true, true); GS_SCATTER(kValIotaReversed, true, true);       // sharded, one pass
        GS_SCATTER(kValArrayReversed, true, false); GS_SCATTER(kValIotaReversed, true, false);     // first of two
        GS_SCATTER(kValArray, false, false); GS_SCATTER(kValArray, true, true);                    // last of two: depth, sharded
    } else {   // depth and sharded sorts of 17..24-bit keys (three passes); raycast and generator pieces (one to four, from an array)
        GS_SCATTER(kValArrayReversed, true, false); GS_SCATTER(kValIotaReversed, true, false);     // first of the depth and sharded sorts
        GS_SCATTER(kValArray, true, false);                                                        // any but the last
        GS_SCATTER(kValArray, false, false); GS_SCATTER(kValArray, true, true);                    // last: depth, raycast, generator; sharded
    }
#undef GS_SCATTER
}

// Loads every kernel a sort of (KeyT, ValT) may launch.  CUDA loads a kernel's code on its first launch (lazy module loading) and that
// load can wait for running kernels to finish; cudaFuncGetAttributes forces it.
template <typename F> static inline void preload_kernel(F f) { cudaFuncAttributes a; (void)cudaFuncGetAttributes(&a, f); }
template <typename KeyT, typename ValT> static void radix_preload() {
    preload_kernel(k_radix_hist<KeyT>); preload_kernel(k_radix_scan);
    for_each_scatter<KeyT, ValT>([](int, bool, bool, auto kernel) { preload_kernel(kernel); });
}

// Profiler names [tag][hist, scan, scatter][pass]: k_radix_hist[depth,0] ... k_radix_scatter[tile,3]; a PiecewiseSort's are unnamed
enum RadixTag : int { kTagDepth = 0, kTagShard = 1, kTagTile = 2, kTagPiece = 3 };
#define GS_RADIX_STAGE(S, T) {"k_radix_" S "[" T ",0]", "k_radix_" S "[" T ",1]", "k_radix_" S "[" T ",2]", "k_radix_" S "[" T ",3]"}
#define GS_RADIX_NAMES(T) {GS_RADIX_STAGE("hist", T), GS_RADIX_STAGE("scan", T), GS_RADIX_STAGE("scatter", T)}
static const char *const kRadixNames[4][3][4] = {GS_RADIX_NAMES("depth"), GS_RADIX_NAMES("shard"), GS_RADIX_NAMES("tile"), {}};

// One sort.  Its keys are in the sorter's first key buffer; the sorted values land in `out`.  The first pass's values are `vals` read
// forwards (kValArray) or backwards (kValArrayReversed), or iota_top - i (kValIotaReversed).  The count is n, or *n_dev <= n_cap on the
// device (grids sized for n_cap, surplus CTAs exit).  ctl holds the per-pass global digit totals: zero, or counted by bucket() with pass
// 0's tile histogram (hist0_done).  ranges: per key, [first, last+1) of the output.  self_clean: the scatters zero the totals they
// consumed and the last one re-seeds min/max.  keep_final_keys: the last pass writes the sorted keys too (final_keys()).
template <typename ValT> struct RadixJob {
    const ValT *vals = nullptr; int valmode = kValArray; uint32_t iota_top = 0;
    ValT *out = nullptr;
    uint32_t n = 0; const unsigned long long *n_dev = nullptr; unsigned long long n_cap = 0;
    PassPlan plan{};
    SortControl *ctl = nullptr;
    uint2 *ranges = nullptr;
    bool hist0_done = false, self_clean = false, keep_final_keys = false;
    RadixTag tag = kTagDepth;   // names each kernel (k_bucket, then kRadixNames[tag])
    unsigned long long grid_n() const { return n_dev ? n_cap : n; }
};

// A radix sort's scratch: key and value ping-pong buffers and the tile histograms [pass][digit][tile] (tile columns padded to 32).
// KeyT is the key storage; a sort may read it as a narrower key.  reserve() alone sizes them: a sort never allocates, so it may be
// enqueued inside a graph capture or behind a spinning wait kernel (cudaFree synchronises the device), and one larger than the
// reservation fails with GS_ERR_CAPACITY.
template <typename KeyT, typename ValT> struct RadixSort {
    DevBuf<KeyT> keys[2];
    DevBuf<ValT> vals[2];
    DevBuf<uint32_t> tile_hist;

    static uint32_t stride(unsigned long long n) { return (uint32_t)(((n + kRadixTile - 1) / kRadixTile + 31) & ~31ull); }
    int reserve(unsigned long long capacity, int npasses) {
        const size_t n = std::max(capacity, 1ull);
        int rc;
        if ((rc = keys[0].ensure(n)) || (rc = keys[1].ensure(n)) || (rc = vals[0].ensure(n)) || (rc = vals[1].ensure(n))) return rc;
        return tile_hist.ensure((size_t)stride(n) * kRadix * npasses);
    }
    int check(const RadixJob<ValT> &j) const {
        const unsigned long long n = j.grid_n();
        if (n <= keys[0].n && n <= vals[0].n && (size_t)stride(n) * kRadix * j.plan.npasses <= tile_hist.n) return GS_OK;
        return fail(GS_ERR_CAPACITY, "radix sort of %llu keys in %d passes exceeds its reservation (%zu keys)", n, j.plan.npasses, keys[0].n);
    }
    template <typename K = KeyT> K *final_keys(const RadixJob<ValT> &j) const { return (K *)keys[j.plan.npasses & 1].p; }

    // k_bucket for a job with hist0_done: the depth sort's keys (R-1 - bucket of the reversed distances) in keys[0], pass 0's tile
    // histogram and every pass's global digit totals
    template <typename K> int bucket(const RadixJob<ValT> &j, int32_t *dist, uint32_t R, bool write_buckets, const Launch &launch) {
        if (int rc = check(j)) return rc;
        launch.pdl("k_bucket", k_bucket<K>, (uint32_t)((j.grid_n() + kRadixTile - 1) / kRadixTile), kRadixThreads, 0, dist, (K *)keys[0].p, j.n, j.n_dev, R, j.plan,
                   write_buckets ? 1 : 0, j.ctl, tile_hist.p, stride(j.grid_n()));
        return GS_OK;
    }

    template <typename K = KeyT> int sort(const RadixJob<ValT> &j, const Launch &launch) {
        static_assert(sizeof(K) <= sizeof(KeyT), "keys wider than their storage");
        const uint32_t tiles = (uint32_t)((j.grid_n() + kRadixTile - 1) / kRadixTile), hs = stride(j.grid_n());
        if (!tiles) return GS_OK;
        if (int rc = check(j)) return rc;
        K *kin = (K *)keys[0].p, *kout = (K *)keys[1].p;
        const ValT *vin = j.vals;
        for (int p = 0; p < j.plan.npasses; ++p) {
            const bool last = (p == j.plan.npasses - 1);
            ValT *vout = last ? j.out : (vin == vals[0].p ? vals[1].p : vals[0].p);
            uint32_t *th = tile_hist.p + (size_t)p * kRadix * hs, *global = &j.ctl->hist[p][0];
            const int shift = j.plan.shift[p], bits = j.plan.bits[p];
            if (!(p == 0 && j.hist0_done))
                launch.pdl(kRadixNames[j.tag][0][p], k_radix_hist<K>, tiles, kRadixThreads, 0, kin, j.n, j.n_dev, j.n_cap, shift, bits, th, hs, global, 1);
            launch.pdl(kRadixNames[j.tag][1][p], k_radix_scan, 1u << bits, kScanColThreads, 0, th, hs, j.n, j.n_dev, j.n_cap, global);
            const int vm = p ? kValArray : j.valmode;
            const bool wk = !last || j.keep_final_keys, rg = last && j.ranges;
            bool found = false;
            for_each_scatter<K, ValT>([&](int v, bool w, bool r, auto kernel) {
                if (v != vm || w != wk || r != rg) return;
                launch.pdl(kRadixNames[j.tag][2][p], kernel, tiles, kRadixThreads, 0, (const K *)kin, vin, j.iota_top, kout, vout, j.n, j.n_dev, j.n_cap, shift, bits,
                           (const uint32_t *)th, hs, j.ranges, j.self_clean ? global : nullptr, (j.self_clean && last) ? j.ctl : nullptr);
                found = true;
            });
            if (!found) return fail(GS_ERR_BAD_ARG, "radix sort: no scatter variant for value mode %d, keys %d, ranges %d", vm, (int)wk, (int)rg);
            vin = vout;
            std::swap(kin, kout);
        }
        return GS_OK;
    }
};

// Stable sort of an order (n entries; nullptr: the identity) by a key wider than one radix sort, one piece at a time, least significant
// first.  piece(launch, r, order, keys, vals) launches the caller's kernel that writes piece r's keys and the order's entries into the radix
// sort's first buffers.  It consumes the order before the passes write the next one, so `out` may be the input order.
struct PiecewiseSort {
    RadixSort<uint32_t, uint32_t> radix;
    DevBuf<uint32_t> order;    // between pieces
    DevBuf<SortControl> ctl;   // zero: the self-cleaning scatters leave it so

    int reserve(uint32_t capacity, int max_piece_bits, cudaStream_t st) {
        const bool fresh = !ctl.p;
        int rc;
        if ((rc = radix.reserve(capacity, make_plan_bits(max_piece_bits).npasses)) || (rc = order.ensure(capacity)) || (rc = ctl.ensure(1))) return rc;
        if (fresh) CU(cudaMemsetAsync(ctl.p, 0, sizeof(SortControl), st));
        return GS_OK;
    }
    template <typename Piece>
    int sort(const uint32_t *in, uint32_t n, const int *piece_bits, int pieces, uint32_t *out, Piece &&piece, const Launch &launch) {
        RadixJob<uint32_t> j;
        j.vals = radix.vals[0].p; j.n = n; j.ctl = ctl.p; j.self_clean = true; j.tag = kTagPiece;
        for (int r = 0; r < pieces && n; ++r, in = j.out) {
            j.plan = make_plan_bits(piece_bits[r]);
            j.out = (r == pieces - 1) ? out : order.p;
            piece(launch, r, in, radix.keys[0].p, radix.vals[0].p);
            if (int rc = radix.sort(j, launch)) return rc;
        }
        return GS_OK;
    }
};

} // namespace gs
