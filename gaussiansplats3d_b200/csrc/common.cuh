// common.cuh -- shared device/host helpers for libgsplat_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/gsplat_b200.h"   // GS_OK, GS_ERR_CUDA

// last error text of the calling host thread (defined in engine.cu)
extern thread_local char g_gs_err[512];

#include <vector>
#include <string.h>
#include <stdlib.h>

namespace gs {

// Owning, grow-only allocation of T elements: device memory (DevBuf) or page-locked host memory (PinBuf), freed by the destructor.
// ensure(count) keeps the allocation when it already holds `count` elements, else replaces it with one of max(count, 1) elements
// (contents are not preserved).  It returns GS_OK, or GS_ERR_CUDA with the error text in g_gs_err.
template <typename T, bool PINNED> struct GpuBuf {
    T *p = nullptr;
    size_t n = 0;
    GpuBuf() = default;
    GpuBuf(const GpuBuf &) = delete;
    GpuBuf &operator=(const GpuBuf &) = delete;
    ~GpuBuf() { release(); }
    int ensure(size_t count) {
        if (count <= n) return GS_OK;
        release();
        const size_t bytes = (count ? count : 1) * sizeof(T);
        const cudaError_t e = PINNED ? cudaHostAlloc((void **)&p, bytes, cudaHostAllocDefault) : cudaMalloc((void **)&p, bytes);
        if (e != cudaSuccess) {
            p = nullptr;
            snprintf(g_gs_err, sizeof(g_gs_err), "%s(%zu bytes) -> %s", PINNED ? "cudaHostAlloc" : "cudaMalloc", count * sizeof(T), cudaGetErrorString(e));
            return GS_ERR_CUDA;
        }
        n = count;
        return GS_OK;
    }
    void release() {
        if (p) { if (PINNED) cudaFreeHost(p); else cudaFree(p); }
        p = nullptr; n = 0;
    }
};
template <typename T> using DevBuf = GpuBuf<T, false>;
template <typename T> using PinBuf = GpuBuf<T, true>;

// Programmatic dependent launch (PDL): every kernel of the frame chain starts with pdl_enter() -- "my dependents may be scheduled
// now" followed by "wait until the grids I depend on have completed and their memory is visible" -- and is launched through
// gs_launch() with the programmatic-stream-serialization attribute.  The next kernel's CTAs are then already resident (spinning at
// their own wait) when this one drains, which removes the launch latency and ramp-up from every kernel boundary of the frame;
// the data dependence itself is unchanged (griddepcontrol.wait returns only after FULL completion of the predecessor).
// A kernel launched without the attribute sees both instructions as no-ops.  GS_PDL=0 disables the attribute (A/B measurements).
__device__ __forceinline__ void pdl_enter() {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
}
inline bool pdl_enabled() {
    static int on = -1;
    if (on < 0) { const char *v = getenv("GS_PDL"); on = (v && v[0] == '0') ? 0 : 1; }
    return on != 0;
}
template <typename... KArgs, typename... Args>
static inline void gs_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    cfg.attrs = attr; cfg.numAttrs = 1;
    (void)cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);   // errors surface through cudaGetLastError() like a <<<>>> launch
}

// Optional per-kernel timeline: one CUDA event after every kernel launch (gs_set_profiling).  Durations are the gaps
// between consecutive events on the engine's stream, i.e. device time of each kernel including its launch gap.
struct Profiler {
    bool on = false;
    std::vector<cudaEvent_t> ev;
    std::vector<const char *> names;
    size_t used = 0;
    Profiler() = default;
    Profiler(const Profiler &) = delete;
    Profiler &operator=(const Profiler &) = delete;
    ~Profiler() { for (auto e : ev) cudaEventDestroy(e); }
    void begin(cudaStream_t st) { used = 0; names.clear(); mark("<begin>", st); }
    void mark(const char *name, cudaStream_t st) {
        if (!on) return;
        if (used == ev.size()) { cudaEvent_t e; cudaEventCreate(&e); ev.push_back(e); }
        cudaEventRecord(ev[used++], st);
        names.push_back(name);
    }
};

#define GS_MAX_SCENES_DEV 32 /* == GS_MAX_SCENES (power of two: used as a mask) */

constexpr int kRadixBits = 8;
constexpr int kRadix = 1 << kRadixBits;

// ---- cache-hinted vector loads / stores (streaming data is read once: keep it out of L1) -------------------
__device__ __forceinline__ int4 ld_nc_v4(const void *p) {
    int4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ uint32_t ld_nc_u32(const void *p) {
    uint32_t r;
    asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}
__device__ __forceinline__ uint32_t ld_volatile_u32(const uint32_t *p) {
    uint32_t r;
    asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(r) : "l"(p) : "memory");
    return r;
}
__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t *p) {
    uint32_t r;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(r) : "l"(p) : "memory");
    return r;
}
__device__ __forceinline__ void st_release_u32(uint32_t *p, uint32_t v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t lanemask_lt() {
    uint32_t m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}
__device__ __forceinline__ int warp_min(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ int warp_max(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ uint32_t warp_inclusive_scan(uint32_t v) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
    }
    return v;
}

// Block-wide exclusive scan of one value per thread (THREADS multiple of 32, <= 1024).  `total` gets the sum.
template <int THREADS>
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t *smem_warp /* >= 33 */, uint32_t &total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int NW = THREADS / 32;
    const uint32_t inc = warp_inclusive_scan(v);
    if (lane == 31) smem_warp[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = lane < NW ? smem_warp[lane] : 0u;
        uint32_t wi = warp_inclusive_scan(w);
        smem_warp[lane] = wi - w;
        if (lane == 31) smem_warp[32] = wi;
    }
    __syncthreads();
    const uint32_t r = inc - v + smem_warp[warp];
    total = smem_warp[32];
    __syncthreads();
    return r;
}

// ---- control block shared by the sort kernels (device memory, one per engine) ------------------------------
struct SortControl {
    int32_t dmin, dmax;          // running min / max of the distances (seeds +-2147483640, sorter.cpp:24-25)
    uint32_t error;              // sticky error bits (see kErr*)
    uint32_t hist[4][kRadix];    // per-pass global digit histograms
};
constexpr uint32_t kErrDegenerate = 1u;   // dmax == dmin  (reference: NaN bucket -> wasm trap)
constexpr uint32_t kErrBucketRange = 2u;  // bucket outside [0, R)
constexpr uint32_t kErrCapacity = 4u;     // tile-instance buffer overflow

} // namespace gs
