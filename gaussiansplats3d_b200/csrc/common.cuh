// common.cuh -- shared device/host helpers for libgsplat_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/gsplat_b200.h"   // GS_OK, GS_ERR_CUDA

// last error text of the calling host thread (defined in engine.cu)
extern thread_local char g_gs_err[512];

#include <stdarg.h>
#include <vector>
#include <string.h>
#include <stdlib.h>

namespace gs {

// Every host entry reports an error the same way: the status code, with its text in g_gs_err.
static inline int fail(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_gs_err, sizeof(g_gs_err), fmt, ap);
    va_end(ap);
    return code;
}
#define CU(call)                                                                                                  \
    do {                                                                                                          \
        cudaError_t _e = (call);                                                                                  \
        if (_e != cudaSuccess) return fail(GS_ERR_CUDA, "%s -> %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)

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

// Programmatic dependent launch (PDL): a kernel of the frame chain starts with pdl_enter() -- "my dependents may be scheduled
// now" followed by "wait until the grids I depend on have completed and their memory is visible" -- and is launched by
// Launch::pdl() with the programmatic-stream-serialization attribute.  The next kernel's CTAs are then already resident (spinning at
// their own wait) when this one drains, which removes the launch latency and ramp-up from every kernel boundary of the frame;
// the data dependence itself is unchanged (griddepcontrol.wait returns only after FULL completion of the predecessor).
// A kernel launched without the attribute sees both instructions as no-ops.  GS_PDL=0 disables the attribute (A/B measurements).
// The pairing is a rule (tests/test_launch_rules.py): a PDL launch without the wait would race its predecessor.
__device__ __forceinline__ void pdl_enter() {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
}
inline bool pdl_enabled() {
    static int on = -1;
    if (on < 0) { const char *v = getenv("GS_PDL"); on = (v && v[0] == '0') ? 0 : 1; }
    return on != 0;
}

// Optional timeline of marks (gs_set_profiling): one CUDA event after each named kernel or stage.  Durations are the gaps
// between consecutive events on the engine's stream, i.e. device time of each kernel or stage including its launch gap.
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

// Every kernel launch of the library goes through a Launch: a stream, the timeline (or none) and the calling entry's launch total
// (or none).  Each launch adds one to the total and, when it has a name, marks the timeline right after it.  A frame captured on two
// streams counts into one total through on().  The arguments convert to the kernel's parameters implicitly, as in a <<<>>> launch, so a
// mismatched pointer stays a compile error.  Launch errors surface through cudaGetLastError(), as for any launch.
class Launch {
public:
    explicit Launch(cudaStream_t st, Profiler *prof = nullptr, uint32_t *total = nullptr) : st_(st), prof_(prof), total_(total) {}
    cudaStream_t stream() const { return st_; }
    Launch on(cudaStream_t st) const { return Launch(st, prof_, total_); }
    void mark(const char *name) const { if (name && prof_) prof_->mark(name, st_); }
    template <typename... KArgs, typename... Args>
    void plain(const char *name, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, Args... args) const {
        kernel<<<grid, block, smem, st_>>>(args...);
        done(name);
    }
    // The same with programmatic stream serialization: the kernel must begin with pdl_enter()
    template <typename... KArgs, typename... Args>
    void pdl(const char *name, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, Args... args) const {
        cudaLaunchAttribute attr{cudaLaunchAttributeProgrammaticStreamSerialization};
        attr.val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
        const cudaLaunchConfig_t cfg{grid, block, smem, st_, &attr, 1};
        (void)cudaLaunchKernelEx(&cfg, kernel, args...);
        done(name);
    }
private:
    void done(const char *name) const { if (total_) ++*total_; mark(name); }
    cudaStream_t st_;
    Profiler *prof_;
    uint32_t *total_;
};

#define GS_MAX_SCENES_DEV 32 /* == GS_MAX_SCENES (power of two: used as a mask) */

// The range of `x` among `count` consecutive ranges [start[s], start[s + 1]): the last s with start[s] <= x, so that empty ranges
// (start[s] == start[s + 1]) are never returned for an x inside the union.  A SplatTree forest's sub-tree of a leaf or node, a scene's
// of a splat.
__device__ __forceinline__ uint32_t range_of(const uint32_t *__restrict__ start, uint32_t count, uint32_t x) {
    uint32_t lo = 0, hi = count - 1;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (start[mid] <= x) lo = mid; else hi = mid - 1;
    }
    return lo;
}

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
