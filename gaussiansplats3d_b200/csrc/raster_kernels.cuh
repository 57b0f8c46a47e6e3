// raster_kernels.cuh -- tile-binned forward rasteriser (sm_90a) replacing the reference's WebGL path:
//   k_project      : vertex shader, once per splat (not x4)    SplatMaterial.js:112-341, SplatMaterial3D.js:83-216
//   binning        : per-coarse-tile lists of {fine mask, splat} in draw order.  Frames of at most 256 coarse tiles (kBinTiles): a
//                    counting sort, k_bin_count -> k_bin_scan -> k_bin_place.  Larger frames: k_tile_count -> k_tile_emit, then a
//                    stable radix sort of the instances by coarse tile id (sort_kernels.cuh)
//   k_blend        : fragment shader + blend, front-to-back      SplatMaterial3D.js:234-252, :65-75
// Draw order is the reference's (sorted_indexes[0] first = farthest).  We composite front-to-back over the REVERSED
// list with a transmittance accumulator, which is algebraically the same "over" chain (SURVEY.md Appendix C).
#pragma once
#include "common.cuh"
#include "sort_kernels.cuh"
#include "../../include/gsplat_b200.h"
#include <cuda_fp16.h>
#include "ellipse_mask.h"

namespace gs {

constexpr int kTile = 16;              // tile edge in pixels
constexpr int kTileShift = 4;
constexpr float kTransmittanceCutoff = 1.0f / 512.0f;  // stop compositing below this: what is left adds < 0.5/255 (half an RGBA8 step); stated deviation

struct __align__(16) SplatRecord {     // 48 bytes, read as 3 x 16 B
    float cx, cy;                      // quad centre in pixels, GL window coordinates (y up)
    float g1x, g1y;                    // g1 = B1 / |B1|^2 : u = dot(d, g1) is the quad-local coordinate in [-1,1]
    float g2x, g2y;                    // g2 = B2 / |B2|^2
    uint32_t hxhy;                     // half2: half extents of the ellipse's pixel AABB, rounded UP (culling only)
    float a;
    float r, g, b;
    float ndc_z;                       // outside [-1,1] (2.0 for culled splats) <=> not drawn
};

constexpr int kVisibleSlots = 64;
struct RasterControl {
    unsigned long long total_instances;
    uint32_t overflow;
    uint32_t visible;
    uint32_t reserved0;
    uint32_t frame_seq;      // frames rendered so far (never reset): the peer-gather handshake counts in frames
    uint32_t peer_timeout;   // a peer handshake gave up waiting
    uint32_t peer_parity;    // ranks > 0: which half of rank 0's (double) frame buffer this frame's tiles go to (from the release word)
    unsigned long long subset_count;   // sharded frames: splats whose rect touches one of this rank's coarse tiles
    // visible-splat statistic, spread over 64 counters 32 B apart: same-address atomics serialise, and with one counter the atomics
    // (one per warp) set the duration of k_project
    uint32_t visible_slots[kVisibleSlots * 8];
};

// Block in rank 0's memory that the other ranks map through CUDA IPC: the fused tile gather's handshake.
//   released = 2 f + b : rank 0 has finished with the picture that last occupied half b of its frame allocation; peers may write
//                  frame f's tiles into that half (b = 0 always unless rank 0 pipelines its frames over two halves)
//   arrived      : += 1 by every peer once its tiles of the current frame are in rank 0's buffer
struct PeerSync { uint32_t released; uint32_t arrived; uint32_t pad[2]; };

__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t *p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
constexpr long long kPeerTimeoutCycles = 4000000000ll;   // ~2 s: a missing peer must never hang the GPU

// rank 0, start of frame f: the picture of frame f-1 has been consumed (stream order) -> peers may overwrite the buffer
__global__ void k_peer_release(PeerSync *sync, const RasterControl *rctl, uint32_t half) {
    __threadfence_system();
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(&sync->released), "r"(rctl->frame_seq * 2u + (half & 1u)) : "memory");
}
// rank r > 0, before its blend of frame f: wait until rank 0 released frame f
__global__ void k_peer_wait_release(const PeerSync *sync, RasterControl *rctl) {
    // rank 0 cannot release frame f+1 before every peer has signalled frame f, so the word read here is frame f's
    const uint32_t f = rctl->frame_seq;
    const long long t0 = clock64();
    uint32_t v = ld_acquire_sys_u32(&sync->released);
    while ((int32_t)((v >> 1) - f) < 0) {
        if (clock64() - t0 > kPeerTimeoutCycles) { rctl->peer_timeout = 1; v = 0; break; }
        __nanosleep(200);
        v = ld_acquire_sys_u32(&sync->released);
    }
    rctl->peer_parity = v & 1u;
}
// rank r > 0, after its blend: tiles are in rank 0's frame
__global__ void k_peer_signal(PeerSync *sync) {
    __threadfence_system();
    atomicAdd_system(&sync->arrived, 1u);
}
// rank 0, end of frame f: wait for the tiles of all world-1 peers
__global__ void k_peer_wait_arrived(const PeerSync *sync, RasterControl *rctl, uint32_t peers) {
    const uint32_t want = rctl->frame_seq * peers;
    const long long t0 = clock64();
    while ((int32_t)(ld_acquire_sys_u32(&sync->arrived) - want) < 0) {
        if (clock64() - t0 > kPeerTimeoutCycles) { rctl->peer_timeout = 1; break; }
        __nanosleep(200);
    }
    __threadfence_system();
}

struct ProjParams {
    float mv[16], proj[16];
    float cam[3];
    float focal[2], viewport[2];
    float inv_focal_adj, ortho_zoom;
    int orthographic;
    float splat_scale;
    int point_cloud, sh_degree, antialiased;
    float kernel2d, max_size;
    int fade_in_complete;
    float scene_center[3], fade_start;
    int dynamic, optional_effects, scene_count;
    int tiles_x, tiles_y;
    uint32_t rank, world;
    int width, height;
    int tile_shift;                    // log2 of the fine-tile edge in pixels: 4 (16 px) or 5 (32 px, frames beyond ~2048x1024)
};

struct DynamicUniforms {               // only read in dynamic / optional-effects / 8-bit SH modes
    float view[16];
    float transforms[16 * GS_MAX_SCENES_DEV];
    float sh8_min[GS_MAX_SCENES_DEV], sh8_max[GS_MAX_SCENES_DEV];
    float opacity[GS_MAX_SCENES_DEV];
    int visibility[GS_MAX_SCENES_DEV];
};

// Multi-GPU ownership: COARSE tile (cx, cy) belongs to rank (cx + cy) % world -- a diagonal interleave, so every rank gets tiles from
// all over the picture (dense centre and empty border alike) and any `world` horizontally adjacent coarse tiles cover every rank.
__host__ __device__ __forceinline__ bool owns_coarse(int cx, int cy, uint32_t rank, uint32_t world) {
    return world <= 1 || (uint32_t)(cx + cy) % world == rank;
}

__device__ __forceinline__ void mat4_mul_dev(const float *a, const float *b, float *o) {
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int r = 0; r < 4; ++r)
            o[4 * c + r] = a[r] * b[4 * c] + a[4 + r] * b[4 * c + 1] + a[8 + r] * b[4 * c + 2] + a[12 + r] * b[4 * c + 3];
}
__device__ inline void mat4_inverse_dev(const float *m, float *o) {
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
    const float det = m[0] * inv[0] + m[1] * inv[4] + m[2] * inv[8] + m[3] * inv[12];
    const float id = 1.0f / det;
#pragma unroll
    for (int i = 0; i < 16; ++i) o[i] = inv[i] * id;
}

// ---------------------------------------------------------------------------------------------------------------
// Projection: one thread per splat, splat order (coalesced 16 B + 24 B + SH loads).
//   COVF16: covariances stored as 6 halfs;  SHFMT: gs_sh_format
//   VIEWS: one launch projects every view of a stereo or multi-view frame, blockIdx.y = view; view v > 0 reads and writes the blocks of
//   views[v].
constexpr int kProjThreads = 128;

// One view's buffers as the kernels of a stereo or multi-view frame find them: RasterState::view_table, one row of GS_MAX_VIEWS entries
// per frame-buffer parity (the parameter blocks are that parity's).  The mono instantiations never read it.
struct ViewEntry {
    const ProjParams *P;
    const DynamicUniforms *dyn;
    SplatRecord *rec;
    ushort4 *rects;
    const unsigned long long *list;
    RasterControl *rctl;
    SortControl *sctl;
    uint32_t *bin_totals;
    uint32_t *super_sums;
};

template <bool COVF16, int SHFMT, bool VIEWS = false>
__global__ void __launch_bounds__(kProjThreads)
k_project(const uint4 *__restrict__ cc, const void *__restrict__ cov, const void *__restrict__ sh, int sh_data_degree,
          const uint32_t *__restrict__ scene_idx, const DynamicUniforms *__restrict__ dyn, const ProjParams *__restrict__ Pp, uint32_t count,
          SplatRecord *__restrict__ rec, ushort4 *__restrict__ rects, RasterControl *rctl, const ViewEntry *__restrict__ views) {
    pdl_enter();
    if (VIEWS && blockIdx.y) { const ViewEntry &E = views[blockIdx.y]; dyn = E.dyn; Pp = E.P; rec = E.rec; rects = E.rects; }
    // per-frame parameters: device memory -> shared memory once per CTA (graph-replayable, broadcast reads afterwards)
    __shared__ ProjParams s_P;
    {
        const uint32_t *src = reinterpret_cast<const uint32_t *>(Pp);
        uint32_t *dst = reinterpret_cast<uint32_t *>(&s_P);
        for (int i = threadIdx.x; i < (int)(sizeof(ProjParams) / 4); i += kProjThreads) dst[i] = __ldg(src + i);
    }
    __syncthreads();
    const ProjParams &P = s_P;
    __shared__ float4 s_out[kProjThreads / 32][96];
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t s = blockIdx.x * kProjThreads + threadIdx.x;
    uint32_t visible = 0;
    if (s < count) {
        SplatRecord o;
        o.cx = o.cy = o.g1x = o.g1y = o.g2x = o.g2y = o.a = o.r = o.g = o.b = 0.f;
        o.ndc_z = 2.0f;
        o.hxhy = 0;
        ushort4 rect = make_ushort4(1, 1, 0, 0); // empty
        // all of the splat's loads are issued up front (also for splats that turn out to be culled): the kernel is bound by load
        // latency, so memory-level parallelism matters more than the ~30% of bytes that culled splats would not have needed
        const int4 c4 = ld_nc_v4(cc + s);
        float V[6];
        if (COVF16) {
            const uint32_t *h32 = (const uint32_t *)cov + (size_t)s * 3;
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const uint32_t w = ld_nc_u32(h32 + k);
                const __half2 hh = *reinterpret_cast<const __half2 *>(&w);
                V[2 * k] = __low2float(hh); V[2 * k + 1] = __high2float(hh);
            }
        } else {
            const float2 *f2 = (const float2 *)cov + (size_t)s * 3;
            const float2 a0 = __ldg(f2), a1 = __ldg(f2 + 1), a2 = __ldg(f2 + 2);
            V[0] = a0.x; V[1] = a0.y; V[2] = a1.x; V[3] = a1.y; V[4] = a2.x; V[5] = a2.y;
        }
        int4 shq[3];
        if (SHFMT == GS_SH_F16 && sh_data_degree >= 2 && P.sh_degree >= 1) {
            const uint4 *h4 = (const uint4 *)((const __half *)sh + (size_t)s * 24);
#pragma unroll
            for (int q = 0; q < 3; ++q) shq[q] = ld_nc_v4(h4 + q);
        }
        const float cx = __int_as_float(c4.y), cy = __int_as_float(c4.z), cz = __int_as_float(c4.w);
        uint32_t scene = 0;
        if (P.scene_count > 1 && scene_idx) scene = scene_idx[s] & (GS_MAX_SCENES_DEV - 1);
        bool alive = true;
        if (P.optional_effects) alive = !(dyn->opacity[scene] <= 0.01f || dyn->visibility[scene] == 0);

        float mvd[16];
        const float *mv = P.mv;
        if (P.dynamic) { mat4_mul_dev(dyn->view, dyn->transforms + 16 * scene, mvd); mv = mvd; }
        float view[4], clip[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) view[r] = mv[r] * cx + mv[4 + r] * cy + mv[8 + r] * cz + mv[12 + r];
#pragma unroll
        for (int r = 0; r < 4; ++r) clip[r] = P.proj[r] * view[0] + P.proj[4 + r] * view[1] + P.proj[8 + r] * view[2] + P.proj[12 + r] * view[3];
        const float lim = 1.2f * clip[3];
        if (clip[2] < -lim || clip[0] < -lim || clip[0] > lim || clip[1] < -lim || clip[1] > lim) alive = false;
        if (alive) {
            const float iw = 1.0f / clip[3];
            const float ndcx = clip[0] * iw, ndcy = clip[1] * iw, ndcz = clip[2] * iw;
            const uint32_t packed = (uint32_t)c4.x;
            float col[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) col[k] = (float)((packed >> (8 * k)) & 255u) * (1.0f / 255.0f);

            if (SHFMT != GS_SH_NONE && sh_data_degree >= 1 && P.sh_degree >= 1) {
                const int ncomp = sh_data_degree >= 2 ? 24 : 9;
                float shv[24];
                const int nuse = (sh_data_degree >= 2 && P.sh_degree >= 2) ? 24 : 9;
                if (SHFMT == GS_SH_F16) {
                    const __half *h = (const __half *)sh + (size_t)s * ncomp;
                    if (ncomp == 24) {
#pragma unroll
                        for (int q = 0; q < 3; ++q) {
                            const int4 v = shq[q];
                            const uint32_t w[4] = {(uint32_t)v.x, (uint32_t)v.y, (uint32_t)v.z, (uint32_t)v.w};
#pragma unroll
                            for (int k = 0; k < 4; ++k) {
                                const __half2 hh = *reinterpret_cast<const __half2 *>(&w[k]);
                                shv[q * 8 + 2 * k] = __low2float(hh);
                                shv[q * 8 + 2 * k + 1] = __high2float(hh);
                            }
                        }
                    } else {
#pragma unroll
                        for (int k = 0; k < 9; ++k) shv[k] = __half2float(h[k]);
                    }
                } else if (SHFMT == GS_SH_U8) {
                    const unsigned char *b = (const unsigned char *)sh + (size_t)s * ncomp;
                    const float lo = dyn->sh8_min[scene], range = dyn->sh8_max[scene] - dyn->sh8_min[scene];
                    for (int k = 0; k < nuse; ++k) shv[k] = ((float)b[k] / 255.0f) * range + lo;
                } else {
                    const float *f = (const float *)sh + (size_t)s * ncomp;
                    for (int k = 0; k < nuse; ++k) shv[k] = f[k];
                }
                float camx = P.cam[0], camy = P.cam[1], camz = P.cam[2];
                if (P.dynamic) {
                    float inv[16];
                    mat4_inverse_dev(dyn->transforms + 16 * scene, inv);
                    const float tx = inv[0] * camx + inv[4] * camy + inv[8] * camz + inv[12];
                    const float ty = inv[1] * camx + inv[5] * camy + inv[9] * camz + inv[13];
                    const float tz = inv[2] * camx + inv[6] * camy + inv[10] * camz + inv[14];
                    camx = tx; camy = ty; camz = tz;
                }
                float dx = cx - camx, dy = cy - camy, dz = cz - camz;
                const float il = rsqrtf(dx * dx + dy * dy + dz * dz);
                const float x = dx * il, y = dy * il, z = dz * il;
                const float C1 = 0.4886025119029199f;
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) col[ch] += C1 * (-shv[ch] * y + shv[3 + ch] * z - shv[6 + ch] * x);
                if (nuse == 24) {
                    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
#pragma unroll
                    for (int ch = 0; ch < 3; ++ch)
                        col[ch] += (1.0925484f * xy) * shv[9 + ch] + (-1.0925484f * yz) * shv[12 + ch] +
                                   (0.3153916f * (2.0f * zz - xx - yy)) * shv[15 + ch] + (-1.0925484f * xz) * shv[18 + ch] +
                                   (0.5462742f * (xx - yy)) * shv[21 + ch];
                }
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) col[ch] = __saturatef(col[ch]);
            }

            float j00, j02, j11, j12;
            if (P.orthographic == 1) { j00 = P.ortho_zoom; j11 = P.ortho_zoom; j02 = 0.f; j12 = 0.f; }
            else {
                const float iz = 1.0f / view[2], sc = iz * iz;
                j00 = P.focal[0] * iz; j11 = P.focal[1] * iz;
                j02 = -(P.focal[0] * view[0]) * sc; j12 = -(P.focal[1] * view[1]) * sc;
            }
            float T0[3], T1[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const float w0 = mv[4 * k + 0], w1 = mv[4 * k + 1], w2 = mv[4 * k + 2];
                T0[k] = w0 * j00 + w2 * j02;
                T1[k] = w1 * j11 + w2 * j12;
            }
            const float VT0x = V[0] * T0[0] + V[1] * T0[1] + V[2] * T0[2];
            const float VT0y = V[1] * T0[0] + V[3] * T0[1] + V[4] * T0[2];
            const float VT0z = V[2] * T0[0] + V[4] * T0[1] + V[5] * T0[2];
            const float VT1x = V[0] * T1[0] + V[1] * T1[1] + V[2] * T1[2];
            const float VT1y = V[1] * T1[0] + V[3] * T1[1] + V[4] * T1[2];
            const float VT1z = V[2] * T1[0] + V[4] * T1[1] + V[5] * T1[2];
            float a = T0[0] * VT0x + T0[1] * VT0y + T0[2] * VT0z;
            const float b = T0[0] * VT1x + T0[1] * VT1y + T0[2] * VT1z;
            float d = T1[0] * VT1x + T1[1] * VT1y + T1[2] * VT1z;
            if (P.antialiased) {
                const float det0 = a * d - b * b;
                a += P.kernel2d; d += P.kernel2d;
                const float det1 = a * d - b * b;
                col[3] *= sqrtf(fmaxf(det0 / det1, 0.0f));
                if (col[3] < 1.0f / 255.0f) alive = false;
            } else { a += P.kernel2d; d += P.kernel2d; }
            const float D = a * d - b * b, half_tr = 0.5f * (a + d);
            const float term2 = sqrtf(fmaxf(0.1f, half_tr * half_tr - D));
            float l1 = half_tr + term2, l2 = half_tr - term2;
            if (P.point_cloud == 1) l1 = l2 = 0.2f;
            if (l2 <= 0.0f) alive = false;
            if (alive) {
                float ex = b, ey = l1 - a;
                const float en = rsqrtf(ex * ex + ey * ey);
                ex *= en; ey *= en;
                const float sqrt8 = 2.8284271247461903f;
                const float s1 = P.splat_scale * fminf(sqrt8 * sqrtf(l1), P.max_size) * P.inv_focal_adj;
                const float s2 = P.splat_scale * fminf(sqrt8 * sqrtf(l2), P.max_size) * P.inv_focal_adj;
                if (P.optional_effects) col[3] *= dyn->opacity[scene];
                if (!P.fade_in_complete) {
                    const float qx = cx - P.scene_center[0], qy = cy - P.scene_center[1], qz = cz - P.scene_center[2];
                    const float dist = sqrtf(qx * qx + qy * qy + qz * qz);
                    const float st = dist >= P.fade_start ? 1.0f : 0.0f;
                    col[3] *= (1.0f - st) + (1.0f - __saturatef((dist - P.fade_start) / 0.75f)) * st;
                }
                // B1 = e1*s1, B2 = (e1.y,-e1.x)*s2 ; g = B/|B|^2 = e/s
                const float is1 = 1.0f / s1, is2 = 1.0f / s2;
                o.cx = (ndcx + 1.0f) * 0.5f * P.viewport[0];
                o.cy = (ndcy + 1.0f) * 0.5f * P.viewport[1];
                o.g1x = ex * is1; o.g1y = ey * is1;
                o.g2x = ey * is2; o.g2y = -ex * is2;
                o.ndc_z = ndcz; o.a = col[3];
                o.r = col[0]; o.g = col[1]; o.b = col[2];
                // en = inf: b and l1 - a both rounded to 0 (an axis-aligned splat with a > d), normalize(vec2(0)) is NaN and WebGL drops
                // the quad; so do we, rather than export a valid record with a NaN basis
                const bool in_depth = (ndcz >= -1.0f && ndcz <= 1.0f) && isfinite(s1) && isfinite(s2) && s1 > 0.f && s2 > 0.f && isfinite(en);
                if (!in_depth && ndcz >= -1.0f && ndcz <= 1.0f) o.ndc_z = 2.0f;
                if (in_depth) {
                    // tight AABB of the ellipse u^2+w^2<=1 : half extents sqrt(B1x^2+B2x^2), sqrt(B1y^2+B2y^2)
                    const float b1x = ex * s1, b1y = ey * s1, b2x = ey * s2, b2y = -ex * s2;
                    const float hx = sqrtf(b1x * b1x + b2x * b2x) * 1.0005f + 0.01f;
                    const float hy = sqrtf(b1y * b1y + b2y * b2y) * 1.0005f + 0.01f;
                    const __half2 hh = __halves2half2(__float2half_ru(fminf(hx, 60000.f)), __float2half_ru(fminf(hy, 60000.f)));
                    o.hxhy = *reinterpret_cast<const uint32_t *>(&hh);
                    // pixel centres (px+0.5) inside [c-h, c+h]
                    const float fx0 = ceilf(o.cx - hx - 0.5f), fx1 = floorf(o.cx + hx - 0.5f);
                    const float fy0 = ceilf(o.cy - hy - 0.5f), fy1 = floorf(o.cy + hy - 0.5f);
                    const float W1 = (float)(P.width - 1), H1 = (float)(P.height - 1);
                    if (fx1 >= 0.f && fy1 >= 0.f && fx0 <= W1 && fy0 <= H1 && fx0 <= fx1 && fy0 <= fy1) {
                        const int px0 = (int)fmaxf(fx0, 0.f), px1 = (int)fminf(fx1, W1);
                        const int py0 = (int)fmaxf(fy0, 0.f), py1 = (int)fminf(fy1, H1);
                        rect = make_ushort4((unsigned short)(px0 >> P.tile_shift), (unsigned short)(py0 >> P.tile_shift),
                                            (unsigned short)(px1 >> P.tile_shift), (unsigned short)(py1 >> P.tile_shift));
                        visible = 1;
                    }
                }
            }
        }
        // stage the 48-byte record so that the warp stores its 1536 contiguous bytes with three fully coalesced 16-byte stores
        float4 *stage = s_out[threadIdx.x >> 5];
        stage[lane * 3 + 0] = make_float4(o.cx, o.cy, o.g1x, o.g1y);
        stage[lane * 3 + 1] = make_float4(o.g2x, o.g2y, __uint_as_float(o.hxhy), o.a);
        stage[lane * 3 + 2] = make_float4(o.r, o.g, o.b, o.ndc_z);
        rects[s] = rect;
    }
    __syncwarp();
    {
        const uint32_t warp_first = blockIdx.x * kProjThreads + (threadIdx.x & ~31u);
        if (warp_first < count) {
            const uint32_t nrec = min(32u, count - warp_first);
            float4 *gdst = reinterpret_cast<float4 *>(rec + warp_first);
            const float4 *stage = s_out[threadIdx.x >> 5];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const uint32_t idx = (uint32_t)k * 32 + lane;
                if (idx < nrec * 3) gdst[idx] = stage[idx];
            }
        }
    }
    const uint32_t nvis = __popc(__ballot_sync(0xffffffffu, visible));
    if ((threadIdx.x & 31) == 0 && nvis) atomicAdd(&rctl->visible_slots[((blockIdx.x * (kProjThreads / 32) + (threadIdx.x >> 5)) & (kVisibleSlots - 1)) * 8], nvis);
}

// ---------------------------------------------------------------------------------------------------------------
// Hierarchical binning.  Splats are binned (in draw order) into COARSE tiles of kCoarseW x kCoarseH fine tiles (128 x 64 px at
// 16-px fine tiles, 256 x 128 px at 32 px).  Each instance carries a 32-bit mask of the fine tiles it touches inside that coarse
// tile; the blend CTA of a fine tile streams its coarse tile's list and keeps the entries whose mask bit is set.  Order inside a
// list = draw order (both binnings are stable over a sequence generated in draw order), so filtering preserves it.
// What an instance is lives in one place for both binnings: coarse_instances() counts a splat's instances, round_instances() visits
// them, fine_mask_in_coarse() gives each its mask.
constexpr int kCoarseW = 8, kCoarseH = 4, kCoarseShiftX = 3, kCoarseShiftY = 2;
constexpr int kFinePerCoarse = kCoarseW * kCoarseH;   // 32 = bits of the mask

// Ownership of a sharded frame's coarse tiles by their diagonal d = cx + cy, the same test as owns_coarse: d % world == rank, for every
// diagonal a frame of up to 65 536 coarse tiles (raster_check) can have, i.e. d <= 65 535.  The owned diagonals in a window [d0, d1] are
// counted as f(d1) - f(d0 - 1) with f(D) = owned diagonals in [0, D], so counting a window needs no walk.  Only sharded frames evaluate
// these, once or twice per coarse tile or row a splat touches: d / world is a multiply-high by magic = ceil(2^32 / world) instead of a
// division by a run-time value, which is exact for d < 2^32 / world.  A world above 65 536 is replaced by 65 536: both exceed every
// diagonal, so d / world = 0 and d % world = d either way, and the multiply stays exact.
struct Ownership { uint32_t rank, world, magic; };
__device__ __forceinline__ uint32_t own_div(const Ownership &o, uint32_t d) { return __umulhi(d, o.magic); }
__device__ __forceinline__ bool own_diag(const Ownership &o, int diag) {
    return (uint32_t)diag - own_div(o, (uint32_t)diag) * o.world == o.rank;
}
__device__ __forceinline__ uint32_t own_upto(const Ownership &o, int d) {   // owned diagonals in [0, d]; 0 for d < 0
    return d < (int)o.rank ? 0u : own_div(o, (uint32_t)d - o.rank) + 1u;
}
__device__ __forceinline__ uint32_t own_count_range(const Ownership &o, int d0, int d1) {   // 0 <= d0 <= d1
    return own_upto(o, d1) - own_upto(o, d0 - 1);
}
static inline Ownership make_ownership(uint32_t rank, uint32_t world) {     // world <= 1: never consulted
    const uint32_t w = std::min(std::max(world, 2u), 65536u);
    return Ownership{rank, w, (uint32_t)(((1ull << 32) + w - 1) / w)};
}

__device__ __forceinline__ uint32_t coarse_instances(ushort4 r, const Ownership &own, bool sharded) {
    if (r.z < r.x || r.w < r.y) return 0;
    const int cx0 = r.x >> kCoarseShiftX, cx1 = r.z >> kCoarseShiftX, cy0 = r.y >> kCoarseShiftY, cy1 = r.w >> kCoarseShiftY;
    if (!sharded) return (uint32_t)(cx1 - cx0 + 1) * (uint32_t)(cy1 - cy0 + 1);
    if (cx0 == cx1 && cy0 == cy1) return own_diag(own, cx0 + cy0) ? 1u : 0u;
    uint32_t n = 0;   // per coarse row: owned diagonals in [cx0 + cy, cx1 + cy]
    for (int cy = cy0; cy <= cy1; ++cy) n += own_count_range(own, cx0 + cy, cx1 + cy);
    return n;
}

__device__ __forceinline__ uint32_t fine_mask_in_coarse(int rx0, int ry0, int rx1, int ry1, int cx, int cy) {
    const int fx0 = max(rx0, cx * kCoarseW) - cx * kCoarseW, fx1 = min(rx1, cx * kCoarseW + kCoarseW - 1) - cx * kCoarseW;
    const int fy0 = max(ry0, cy * kCoarseH) - cy * kCoarseH, fy1 = min(ry1, cy * kCoarseH + kCoarseH - 1) - cy * kCoarseH;
    const uint32_t rowsel = (0x01010101u >> (8 * (kCoarseH - 1 - (fy1 - fy0)))) << (8 * fy0);
    return (((1u << (fx1 - fx0 + 1)) - 1u) << fx0) * rowsel;
}

// Calls f(owner lane, owner's splat id, coarse tile id, fine mask) for every instance of this warp round: as many calls per splat
// as coarse_instances() counts.  Splats over a handful of coarse tiles are walked by their own lane; the few huge ones (> 32 coarse
// tiles, some cover the whole screen) by the whole warp, 32 tiles per step.
// Must be called by all 32 lanes.  f must not contain warp-synchronous operations.
template <typename F>
__device__ __forceinline__ void round_instances(bool valid, uint32_t sid, ushort4 r, int coarse_x, const Ownership &own, bool sharded, F f) {
    const int lane = threadIdx.x & 31;
    const bool nonempty = valid && r.z >= r.x && r.w >= r.y;
    const int cx0 = r.x >> kCoarseShiftX, cx1 = r.z >> kCoarseShiftX, cy0 = r.y >> kCoarseShiftY, cy1 = r.w >> kCoarseShiftY;
    const bool big = nonempty && (uint32_t)(cx1 - cx0 + 1) * (uint32_t)(cy1 - cy0 + 1) > 32u;
    if (nonempty && !big) {
#pragma unroll 1
        for (int cy = cy0; cy <= cy1; ++cy)
#pragma unroll 1
            for (int cx = cx0; cx <= cx1; ++cx) {      // one iteration for most splats
                if (sharded && !own_diag(own, cx + cy)) continue;
                f(lane, sid, cy * coarse_x + cx, fine_mask_in_coarse((int)r.x, (int)r.y, (int)r.z, (int)r.w, cx, cy));
            }
    }
    uint32_t multi = __ballot_sync(0xffffffffu, big);
    while (multi) {
        const int src = __ffs(multi) - 1;
        multi &= multi - 1;
        const uint32_t bsid = __shfl_sync(0xffffffffu, sid, src);
        const int bx0 = __shfl_sync(0xffffffffu, (int)r.x, src), by0 = __shfl_sync(0xffffffffu, (int)r.y, src);
        const int bx1 = __shfl_sync(0xffffffffu, (int)r.z, src), by1 = __shfl_sync(0xffffffffu, (int)r.w, src);
        const int ccx0 = bx0 >> kCoarseShiftX, ccy0 = by0 >> kCoarseShiftY;
        const int cw = (bx1 >> kCoarseShiftX) - ccx0 + 1, ntile = cw * ((by1 >> kCoarseShiftY) - ccy0 + 1);
        for (int i = lane; i < ntile; i += 32) {
            const int cy = ccy0 + i / cw, cx = ccx0 + i % cw;
            if (sharded && !own_diag(own, cx + cy)) continue;
            f(src, bsid, cy * coarse_x + cx, fine_mask_in_coarse(bx0, by0, bx1, by1, cx, cy));
        }
    }
}

// Does a fine-tile rect reach a coarse tile of this rank?  The coarse tiles of a rect cover EVERY diagonal index cx + cy in
// [cx0 + cy0, cx1 + cy1], and ownership depends on the diagonal only: one count over that window, no loop.
__device__ __forceinline__ bool rect_touches_owned(ushort4 r, const Ownership &own) {
    if (r.z < r.x || r.w < r.y) return false;
    const int d0 = (r.x >> kCoarseShiftX) + (r.y >> kCoarseShiftY), d1 = (r.z >> kCoarseShiftX) + (r.w >> kCoarseShiftY);
    return own_count_range(own, d0, d1) != 0u;
}

constexpr int kBinThreads = 256;
constexpr int kBinItems = 2;
constexpr int kBinTile = kBinThreads * kBinItems;   // draw ranks per CTA

// This thread's share of "instances of all chunks before mine": whole groups of kBinThreads chunks from the second-level sums,
// the chunks of my own group one per thread.
__device__ __forceinline__ unsigned long long chunk_prefix(const uint32_t *__restrict__ block_sums, const uint32_t *__restrict__ super_sums) {
    const uint32_t grp = blockIdx.x / kBinThreads;
    unsigned long long before = 0;
    for (uint32_t g = threadIdx.x; g < grp; g += kBinThreads) before += super_sums[g];
    const uint32_t b = grp * kBinThreads + threadIdx.x;
    if (b < blockIdx.x) before += block_sums[b];
    return before;
}

// Count and emit passes over chunks of kBinTile items (the radix binning's instances, the sharded sort's subset) share their sums:
// the count pass ends in chunk_sums_store(), the emit pass starts with warp_first_slot().
// Tail of a count pass, `mine` = what this thread counted: sums per warp, per CTA chunk and per group of kBinThreads chunks.
__device__ __forceinline__ void chunk_sums_store(uint32_t mine, uint32_t *__restrict__ block_sums, uint32_t *__restrict__ warp_sums, uint32_t *__restrict__ super_sums) {
    __shared__ uint32_t s_w[kBinThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
    if (lane == 0) { s_w[warp] = mine; warp_sums[blockIdx.x * (kBinThreads / 32) + warp] = mine; }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t total = 0;
#pragma unroll
        for (int w = 0; w < kBinThreads / 32; ++w) total += s_w[w];
        block_sums[blockIdx.x] = total;
        if (total) atomicAdd(&super_sums[blockIdx.x / kBinThreads], total);   // second level: one counter per kBinThreads chunks
    }
}

// Head of an emit pass: the first output slot of this warp = everything counted in earlier chunks and in the earlier warps of this
// one.  The last CTA's thread 0 also stores the count of all chunks to *total.  T = width of a slot number.
// Two levels (a flat sum over all earlier chunks is quadratic in the chunk count: 16 M splats = 31 K chunks = 0.5 G reads).
template <typename T>
__device__ __forceinline__ T warp_first_slot(const uint32_t *__restrict__ block_sums, const uint32_t *__restrict__ warp_sums, const uint32_t *__restrict__ super_sums,
                                             unsigned long long *total) {
    __shared__ T s_prefix;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T before = (T)chunk_prefix(block_sums, super_sums);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) before += __shfl_xor_sync(0xffffffffu, before, o);
    if (threadIdx.x == 0) s_prefix = 0;
    __syncthreads();
    if (lane == 0 && before) atomicAdd(&s_prefix, before);
    __syncthreads();
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) *total = (unsigned long long)s_prefix + block_sums[blockIdx.x];
    T w0 = s_prefix;
    for (int w = 0; w < warp; ++w) w0 += warp_sums[blockIdx.x * (kBinThreads / 32) + w];
    return w0;
}

// Binning of frames above kBinTiles coarse tiles (the counting sort below has 8-bit bins): emit every instance with its coarse
// tile id as the key, then a stable radix sort of the (key, value) pairs by key.
// pass 1: instances per warp (256 consecutive draw ranks) and per CTA chunk (rank p = 0 is the NEAREST splat = last in the
// reference's draw order).  Warp-striped like pass 2: warp w of a CTA owns ranks [chunk + 256 w, +256), item k of lane l = +32k + l.
__global__ void __launch_bounds__(kBinThreads)
k_tile_count(const uint32_t *__restrict__ order, uint32_t render_count_host, const unsigned long long *__restrict__ n_dev,
             const ushort4 *__restrict__ rects, uint32_t *__restrict__ block_sums, uint32_t *__restrict__ warp_sums, uint32_t *__restrict__ super_sums,
             Ownership own, int sharded) {
    pdl_enter();
    const uint32_t render_count = n_dev ? (uint32_t)*n_dev : render_count_host;
    const uint32_t run = blockIdx.x * kBinTile + (threadIdx.x >> 5) * (32 * kBinItems) + (threadIdx.x & 31);
    uint32_t mine = 0;
#pragma unroll
    for (int k = 0; k < kBinItems; ++k) {
        const uint32_t p = run + (uint32_t)k * 32;
        if (p < render_count) mine += coarse_instances(rects[ld_nc_u32(order + (render_count - 1u - p))], own, sharded != 0);
    }
    chunk_sums_store(mine, block_sums, warp_sums, super_sums);
}

// pass 2: write (coarse tile id, {fine mask, splat id}) for every instance, in draw order.  One item at a time (rolled loop, no
// per-thread arrays): the warp's base offset comes from pass 1's sums, the first slot of each lane's splat from a warp scan.
// Instances of one splat land in different lists, so their mutual order is free: each takes the next slot of its splat's range
// from a per-lane counter in shared memory, which the lanes of a warp-walked splat share.
__global__ void __launch_bounds__(kBinThreads)
k_tile_emit(const uint32_t *__restrict__ order, uint32_t render_count_host, const unsigned long long *__restrict__ n_dev,
            const ushort4 *__restrict__ rects, const uint32_t *__restrict__ block_sums, const uint32_t *__restrict__ warp_sums,
            const uint32_t *__restrict__ super_sums, int coarse_x,
            uint16_t *__restrict__ keys, unsigned long long *__restrict__ vals, unsigned long long capacity, RasterControl *rctl, Ownership own,
            int sharded) {
    pdl_enter();
    const uint32_t render_count = n_dev ? (uint32_t)*n_dev : render_count_host;
    __shared__ uint32_t s_next[kBinThreads / 32][32];   // next free slot of each lane's splat, relative to the warp's w0
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long w0 = warp_first_slot<unsigned long long>(block_sums, warp_sums, super_sums, &rctl->total_instances);   // read by the tile sort
    uint32_t *next = s_next[warp];
    const uint32_t run = blockIdx.x * kBinTile + (uint32_t)warp * (32 * kBinItems) + lane;
    bool overflow = false;
#pragma unroll 2
    for (int k = 0; k < kBinItems; ++k) {
        const uint32_t p = run + (uint32_t)k * 32;
        uint32_t sid = 0, cnt = 0;
        ushort4 r = make_ushort4(1, 1, 0, 0);
        if (p < render_count) {
            sid = ld_nc_u32(order + (render_count - 1u - p));
            r = rects[sid];
            cnt = coarse_instances(r, own, sharded != 0);
        }
        const uint32_t inc = warp_inclusive_scan(cnt);
        next[lane] = inc - cnt;
        __syncwarp();
        round_instances(p < render_count, sid, r, coarse_x, own, sharded != 0, [&](int owner, uint32_t sid_o, int t, uint32_t fmask) {
            const unsigned long long at = w0 + atomicAdd(&next[owner], 1u);
            if (at < capacity) {
                keys[at] = (uint16_t)t;
                vals[at] = ((unsigned long long)fmask << 32) | sid_o;
            } else overflow = true;
        });
        w0 += __shfl_sync(0xffffffffu, inc, 31);
        __syncwarp();
    }
    if (overflow) rctl->overflow = 1;
}

// ---------------------------------------------------------------------------------------------------------------
// Binning of frames with at most kBinTiles coarse tiles: a COUNTING SORT of the coarse-tile instances straight from the draw order
// -- count, scan, place.  One instance is written once (8 B) at its final slot of its coarse tile's list.
//   k_bin_count : per chunk of draw ranks, instances per coarse tile            -> hist[tile][chunk], totals[tile]
//   k_bin_scan  : per tile: exclusive scan over chunks + base of the tile's list -> hist becomes offsets, ranges[tile]
//   k_bin_place : per chunk: stable rank of every instance inside the chunk (per-warp lane masks in shared memory: a splat touches a
//                 coarse tile at most once, so the instances of one tile in one warp round ARE a 32-bit lane mask and the rank of lane l
//                 is popc(mask & lanes_below(l))) + the chunk's offset -> list[slot] = {fine mask, splat id}
// Rank order inside a chunk = (warp, round, lane) = draw-rank order (warp-striped, as in the radix kernels).
constexpr int kBinTiles = 256;      // coarse tiles per frame in this path (8-bit bins)
constexpr int kBinWarps = 16;       // warps per CTA of k_bin_count / k_bin_place (32 KB shared in k_bin_place)
constexpr int kBinRankItems = 4;    // draw ranks per lane
constexpr int kBinRanks = kBinWarps * 32 * kBinRankItems;     // draw ranks per CTA: 2048

__global__ void __launch_bounds__(kBinWarps * 32)
k_bin_count(const uint32_t *__restrict__ order, uint32_t render_count_host, const unsigned long long *__restrict__ n_dev, const ushort4 *__restrict__ rects,
            int coarse_x, uint32_t nt, uint32_t *__restrict__ hist, uint32_t stride, uint32_t *__restrict__ totals, ushort4 *__restrict__ rect_by_rank,
            Ownership own, int sharded) {
    pdl_enter();
    constexpr int W = kBinWarps, ITEMS = kBinRankItems, NT = kBinTiles;
    const uint32_t n = n_dev ? (uint32_t)*n_dev : render_count_host;
    const uint32_t base = blockIdx.x * (uint32_t)(W * 32 * ITEMS);
    if (base >= n) return;
    __shared__ uint32_t s_hist[NT];
    for (uint32_t t = threadIdx.x; t < nt; t += W * 32) s_hist[t] = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t run = base + (uint32_t)warp * (32 * ITEMS) + lane;
    uint32_t sid[ITEMS];
    ushort4 rc[ITEMS];
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
        const uint32_t p = run + (uint32_t)k * 32;
        sid[k] = p < n ? ld_nc_u32(order + (n - 1u - p)) : 0xffffffffu;
    }
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) rc[k] = sid[k] != 0xffffffffu ? rects[sid[k]] : make_ushort4(1, 1, 0, 0);
    // the gathered rects are left in DRAW-RANK order for k_bin_place: its reads are then streams, not a second random gather
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
        const uint32_t p = run + (uint32_t)k * 32;
        if (p < n) rect_by_rank[p] = rc[k];
    }
#pragma unroll 1
    for (int k = 0; k < ITEMS; ++k) {
        uint32_t id = 0; ushort4 r = make_ushort4(1, 1, 0, 0);
#pragma unroll
        for (int j = 0; j < ITEMS; ++j) if (j == k) { id = sid[j]; r = rc[j]; }      // register select (no local-memory indexing)
        round_instances(id != 0xffffffffu, id, r, coarse_x, own, sharded != 0, [&](int, uint32_t, int t, uint32_t) { atomicAdd(&s_hist[t], 1u); });
    }
    __syncthreads();
    for (uint32_t t = threadIdx.x; t < nt; t += W * 32) {
        const uint32_t v = s_hist[t];
        hist[(size_t)t * stride + blockIdx.x] = v;
        if (v) atomicAdd(&totals[t], v);
    }
}

// One CTA per coarse tile: where its list starts (all smaller tiles' totals) and the running offset of every chunk inside it.
// k_bin_place drops the instances that fall at or past `capacity`, so the blend may only read the slots below it: both ends of every
// range are clamped there (an overflowing frame is reported as GS_ERR_CAPACITY; total_instances keeps the unclamped count).
__global__ void __launch_bounds__(1024)
k_bin_scan(uint32_t *__restrict__ hist, uint32_t stride, uint32_t ranks_per_chunk, uint32_t render_count_host, const unsigned long long *__restrict__ n_dev,
           const uint32_t *__restrict__ totals, uint32_t nt, uint2 *__restrict__ ranges, RasterControl *rctl, uint32_t *__restrict__ tile_order,
           unsigned long long capacity) {
    pdl_enter();
    __shared__ uint32_t s_scan[40];
    __shared__ uint32_t s_carry;
    {   // longest list first: the blend's duration is bounded below by its densest tiles, so their CTAs must start first.
        // rank of this tile among all tiles by list length, descending (ties: lower tile id first)
        const uint32_t mine = totals[blockIdx.x];
        bool ahead = false;
        if (threadIdx.x < nt) { const uint32_t o = totals[threadIdx.x]; ahead = o > mine || (o == mine && threadIdx.x < blockIdx.x); }
        const int rank = __syncthreads_count(ahead);
        if (threadIdx.x == 0) tile_order[rank] = blockIdx.x;
    }
    const uint32_t n = n_dev ? (uint32_t)*n_dev : render_count_host;
    const uint32_t nchunks = (uint32_t)(((uint64_t)n + ranks_per_chunk - 1) / ranks_per_chunk);
    const uint32_t d = blockIdx.x;
    {
        uint32_t total;
        const uint32_t c = threadIdx.x < d ? totals[threadIdx.x] : 0u;
        (void)block_exclusive_scan<1024>(c, s_scan, total);
        if (threadIdx.x == 0) {
            s_carry = total;
            const uint32_t mine = totals[d];
            const unsigned long long lo = total, hi = lo + mine;
            ranges[d] = make_uint2((uint32_t)min(lo, capacity), (uint32_t)min(hi, capacity));
            if (d == nt - 1) rctl->total_instances = hi;
        }
    }
    __syncthreads();
    uint32_t *col = hist + (size_t)d * stride;
    for (uint32_t b = 0; b < nchunks; b += 1024) {
        const uint32_t t = b + threadIdx.x;
        const uint32_t v = t < nchunks ? col[t] : 0u;
        uint32_t total;
        const uint32_t ex = block_exclusive_scan<1024>(v, s_scan, total);
        const uint32_t carry = s_carry;
        if (t < nchunks) col[t] = ex + carry;
        __syncthreads();
        if (threadIdx.x == 0) s_carry = carry + total;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kBinWarps * 32)
k_bin_place(const uint32_t *__restrict__ order, uint32_t render_count_host, const unsigned long long *__restrict__ n_dev, const ushort4 *__restrict__ rect_by_rank,
            int coarse_x, uint32_t nt, const uint32_t *__restrict__ offsets, uint32_t stride, unsigned long long *__restrict__ list, unsigned long long capacity,
            RasterControl *rctl, Ownership own, int sharded, int pack_ok) {
    pdl_enter();
    constexpr int W = kBinWarps, ITEMS = kBinRankItems, NT = kBinTiles;
    const uint32_t n = n_dev ? (uint32_t)*n_dev : render_count_host;
    const uint32_t base = blockIdx.x * (uint32_t)(W * 32 * ITEMS);
    if (base >= n) return;
    __shared__ uint32_t s_pre[W][NT];      // instances of this warp per tile, then: END of the slots this warp has handed out in the tile's list
    __shared__ __align__(8) uint32_t s_mask[W][NT];     // lanes of the current round that touch the tile (first: staging of the compaction)
    static_assert(NT * 4 >= 32 * ITEMS * 8, "the mask row of a warp doubles as the staging buffer of its compacted items");
    for (uint32_t i = threadIdx.x; i < (uint32_t)(W * NT); i += W * 32) (&s_pre[0][0])[i] = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t run = base + (uint32_t)warp * (32 * ITEMS) + lane;
    uint32_t sid[ITEMS];
    ushort4 rc[ITEMS];
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
        const uint32_t p = run + (uint32_t)k * 32;
        sid[k] = p < n ? ld_nc_u32(order + (n - 1u - p)) : 0xffffffffu;
        rc[k] = p < n ? rect_by_rank[p] : make_ushort4(1, 1, 0, 0);
    }
    uint32_t *my_pre = s_pre[warp], *my_mask = s_mask[warp];
    // Culled splats (empty rect) and, on a sharded frame, splats that reach none of this rank's tiles leave most lanes idle in the
    // rounds below (ncu: 9-13 of 32 lanes active).  The warp's 32 * ITEMS items are therefore compacted first, order preserved
    // (item k of lane l is draw rank run + 32 k + l, so (k, lane) order is draw order): fewer rounds, full lanes.  A compacted item is
    // 8 bytes, {rect as 4 x u8, splat id}, which needs the frame to be at most 256 tiles wide and high (pack_ok).
    uint32_t nvalid = 32u * ITEMS;
    if (pack_ok) {
        const uint32_t lt = lanemask_lt();
        unsigned long long *stage = reinterpret_cast<unsigned long long *>(my_mask);
        uint32_t before = 0;
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) {
            const bool keep = sid[k] != 0xffffffffu && (sharded ? rect_touches_owned(rc[k], own) : (rc[k].z >= rc[k].x && rc[k].w >= rc[k].y));
            const uint32_t bal = __ballot_sync(0xffffffffu, keep);
            if (keep) stage[before + __popc(bal & lt)] = ((unsigned long long)((uint32_t)rc[k].x | ((uint32_t)rc[k].y << 8) | ((uint32_t)rc[k].z << 16) | ((uint32_t)rc[k].w << 24)) << 32) | sid[k];
            before += __popc(bal);
        }
        nvalid = before;
        __syncwarp();
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) {
            const uint32_t j = (uint32_t)k * 32u + (uint32_t)lane;
            sid[k] = 0xffffffffu;
            rc[k] = make_ushort4(1, 1, 0, 0);
            if (j < nvalid) {
                const unsigned long long v = stage[j];
                const uint32_t pr = (uint32_t)(v >> 32);
                sid[k] = (uint32_t)v;
                rc[k] = make_ushort4((unsigned short)(pr & 255u), (unsigned short)((pr >> 8) & 255u), (unsigned short)((pr >> 16) & 255u), (unsigned short)(pr >> 24));
            }
        }
        __syncwarp();
#pragma unroll
        for (int i = 0; i < NT / 32; ++i) my_mask[i * 32 + lane] = 0u;      // (rounds clear it again; keeps the buffer's two uses apart)
        __syncwarp();
    }
#pragma unroll
    for (int k = 0; k < ITEMS; ++k)
        if ((uint32_t)k * 32u < nvalid)      // warp-uniform
            round_instances(sid[k] != 0xffffffffu, sid[k], rc[k], coarse_x, own, sharded != 0, [&](int, uint32_t, int t, uint32_t) { atomicAdd(&my_pre[t], 1u); });
    __syncthreads();
    for (uint32_t t = threadIdx.x; t < nt; t += W * 32) {   // counts -> first slot of each warp (chunk offset + earlier warps)
        uint32_t at = offsets[(size_t)t * stride + blockIdx.x];
#pragma unroll
        for (int w = 0; w < W; ++w) {
            const uint32_t c = s_pre[w][t];
            s_pre[w][t] = at;
            at += c;
        }
    }
    __syncthreads();
    bool overflow = false;
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
        if ((uint32_t)k * 32u >= nvalid) break;      // warp-uniform: the compacted items fill the first rounds
        const bool valid = sid[k] != 0xffffffffu;
        // a round: (1) clear the warp's lane masks, (2) every instance sets its owner's bit in its tile's mask and takes one slot of the
        // tile's list, (3) with all bits in place, the instance of lane l sits popc(mask & lanes below l) after the round's first slot,
        // which is the tile's new end minus the round's population.
#pragma unroll
        for (int i = 0; i < NT / 32; ++i) my_mask[i * 32 + lane] = 0u;
        __syncwarp();
        round_instances(valid, sid[k], rc[k], coarse_x, own, sharded != 0, [&](int owner, uint32_t, int t, uint32_t) {
            atomicOr(&my_mask[t], 1u << owner);
            atomicAdd(&my_pre[t], 1u);
        });
        __syncwarp();
        round_instances(valid, sid[k], rc[k], coarse_x, own, sharded != 0, [&](int owner, uint32_t sid_o, int t, uint32_t fmask) {
            const uint32_t m = my_mask[t];
            const unsigned long long at = (unsigned long long)(my_pre[t] - (uint32_t)__popc(m)) + __popc(m & ((1u << owner) - 1u));
            if (at < capacity) list[at] = ((unsigned long long)fmask << 32) | sid_o;
            else overflow = true;
        });
        __syncwarp();
    }
    if (overflow) rctl->overflow = 1;
}

// ---------------------------------------------------------------------------------------------------------------
// Sharded frames (world_size > 1): the depth sort of a rank covers only the splats whose screen rect touches one of ITS coarse tiles.
// Any subset, bucketed with the GLOBAL min/max and kept in input order, sorts into exactly the global order restricted to that subset
// (ties are broken by input position) -- SURVEY.md 8(e) -- so no keys or splats are exchanged between GPUs.
// pass 1: survivors per warp / chunk of input positions;  pass 2: order-preserving compaction of (index, distance).
__global__ void __launch_bounds__(kBinThreads)
k_subset_count(const uint32_t *__restrict__ indexes, uint32_t count, const ushort4 *__restrict__ rects, Ownership own,
               uint32_t *__restrict__ block_sums, uint32_t *__restrict__ warp_sums, uint32_t *__restrict__ super_sums) {
    pdl_enter();
    const uint32_t run = blockIdx.x * kBinTile + (threadIdx.x >> 5) * (32 * kBinItems) + (threadIdx.x & 31);
    uint32_t mine = 0;
#pragma unroll
    for (int k = 0; k < kBinItems; ++k) {
        const uint32_t i = run + (uint32_t)k * 32;
        if (i < count) mine += rect_touches_owned(rects[indexes ? ld_nc_u32(indexes + i) : i], own) ? 1u : 0u;
    }
    chunk_sums_store(mine, block_sums, warp_sums, super_sums);
}
__global__ void __launch_bounds__(kBinThreads)
k_subset_emit(const uint32_t *__restrict__ indexes, uint32_t count, const ushort4 *__restrict__ rects, Ownership own,
              const uint32_t *__restrict__ block_sums, const uint32_t *__restrict__ warp_sums, const uint32_t *__restrict__ super_sums,
              const int32_t *__restrict__ dist, uint32_t *__restrict__ sub_idx, int32_t *__restrict__ sub_dist, RasterControl *rctl) {
    pdl_enter();
    uint32_t w0 = warp_first_slot<uint32_t>(block_sums, warp_sums, super_sums, &rctl->subset_count);   // n of this rank's sort
    const uint32_t run = blockIdx.x * kBinTile + (threadIdx.x >> 5) * (32 * kBinItems) + (threadIdx.x & 31);
#pragma unroll 2
    for (int k = 0; k < kBinItems; ++k) {
        const uint32_t i = run + (uint32_t)k * 32;
        uint32_t g = 0;
        bool keep = false;
        if (i < count) {
            g = indexes ? ld_nc_u32(indexes + i) : i;
            keep = rect_touches_owned(rects[g], own);
        }
        const uint32_t bal = __ballot_sync(0xffffffffu, keep);
        if (keep) {
            const uint32_t at = w0 + __popc(bal & lanemask_lt());
            sub_idx[at] = g;
            sub_dist[at] = dist[i];
        }
        w0 += __popc(bal);
    }
}

__global__ void k_raster_init(RasterControl *rctl, SortControl *ctl, uint2 *ranges, uint32_t ntiles, uint32_t *super_sums, uint32_t nsuper, uint32_t *bin_totals, uint32_t *tile_order) {
    pdl_enter();
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    if (tid == 0) {
        rctl->total_instances = 0; rctl->overflow = 0; rctl->visible = 0; rctl->subset_count = 0;
        rctl->frame_seq += 1;
        ctl->error = 0;
    }
    uint32_t *h = &ctl->hist[0][0];
    for (size_t i = tid; i < 4 * kRadix; i += stride) h[i] = 0;
    for (size_t i = tid; i < ntiles; i += stride) ranges[i] = make_uint2(0xffffffffu, 0u); // empty: first > last
    for (size_t i = tid; i < (size_t)kVisibleSlots * 8; i += stride) rctl->visible_slots[i] = 0;
    for (size_t i = tid; i < nsuper; i += stride) super_sums[i] = 0;
    if (bin_totals) for (size_t i = tid; i < kBinTiles; i += stride) bin_totals[i] = 0;
    for (size_t i = tid; i < ntiles; i += stride) tile_order[i] = (uint32_t)i;     // blend schedule: identity unless the counting-sort binning ranks the tiles
}

// Stereo and multi-view frames, after every view is binned: the instance count and overflow flag of view blockIdx.x + 1 join the frame's
// (view 0's control block, which the host reads back), and that view's binning state is left empty for the next frame (view 0's is
// reset by k_raster_init): instance count and overflow flag, counting-sort tile totals, radix-binning histograms and group sums.
// raster_reserve_view leaves a new view empty.  One CTA per view after the first.
__global__ void k_views_join(const ViewEntry *__restrict__ views, uint32_t super_words) {
    pdl_enter();
    const ViewEntry &E = views[blockIdx.x + 1];
    if (threadIdx.x == 0) {
        RasterControl *rctl = views[0].rctl;
        atomicAdd(&rctl->total_instances, E.rctl->total_instances);
        if (E.rctl->overflow) rctl->overflow = 1;
        E.rctl->total_instances = 0; E.rctl->overflow = 0; E.sctl->error = 0;
    }
    uint32_t *h = &E.sctl->hist[0][0];
    for (uint32_t i = threadIdx.x; i < 4 * kRadix; i += blockDim.x) h[i] = 0;
    for (uint32_t i = threadIdx.x; i < (uint32_t)kBinTiles; i += blockDim.x) E.bin_totals[i] = 0;
    for (uint32_t i = threadIdx.x; i < super_words; i += blockDim.x) E.super_sums[i] = 0;
}

// ---------------------------------------------------------------------------------------------------------------
// Blend: one CTA per fine tile; warp w owns an 8x8-px BLOCK of it, a lane owns two vertically adjacent pixels.  The fine tile is
// 16 px (S = 1: 4 warps) or 32 px (S = 2: 16 warps, frames beyond 256 coarse tiles of 128x64 px).  The blend is bound by FP32 issue,
// not by HBM, so its structure aims at issuing fewer instructions:
//   * the thread that stages a splat record into shared memory also decides EXACTLY which of the tile's blocks the ellipse can
//     reach (minimum of the quadratic over the block's rectangle of pixel centres, ellipse_mask.h) -- no AABB-corner work at all;
//   * a warp then walks only the records that touch ITS block (one 32-bit word of touch bits per staging warp), ~45 instructions per
//     record for its 64 pixels, and stops on its own as soon as its 64 pixels are saturated;
//   * opacity is folded into the exponent (ex2(q * k + log2 a)), one multiply less per pixel.
// q = u^2 + w^2 from the inverse quad map, alpha = exp(-4 q) a for q <= 1 (A = 8 q <= 8), front to back.
__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// ---- a lane's two pixels as a pair of f32 (sm_90 has no packed f32x2 FMA: two scalar FFMA / FMUL per pair).  Each half is rounded once
// (fma.rn / mul.rn, no contraction of the multiply into a later add), so the results are the IEEE fp32 values of the per-pixel formulas.
struct f32x2 { float lo, hi; };
__device__ __forceinline__ f32x2 pack2(float lo, float hi) { return f32x2{lo, hi}; }
__device__ __forceinline__ f32x2 bcast2(float v) { return pack2(v, v); }
__device__ __forceinline__ float lo2(f32x2 v) { return v.lo; }
__device__ __forceinline__ float hi2(f32x2 v) { return v.hi; }
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) { return f32x2{__fmaf_rn(a.lo, b.lo, c.lo), __fmaf_rn(a.hi, b.hi, c.hi)}; }
__device__ __forceinline__ f32x2 mul2(f32x2 a, f32x2 b) { return f32x2{__fmul_rn(a.lo, b.lo), __fmul_rn(a.hi, b.hi)}; }

// Which of a tile's 8x8-px blocks can hold a pixel the splat covers: exact minimum of q over each block's rectangle of pixel
// centres (ellipse_mask.h), only for the blocks the ellipse's AABB reaches.  a0 = cx, cy, g1x, g1y; a1 = g2x, g2y, half2(hx, hy), alpha.
// NBX x NBY = blocks per tile row / column.  Not inlined: the caller's composite loop is register-bound and this runs once per staged record.
template <int NBX, int NBY>
__device__ __noinline__ uint32_t block_touch_mask(float4 a0, float4 a1, float tile_x0, float tile_y0) {
    if (!(a1.w > 0.0f)) return 0u;
    const uint32_t hb = __float_as_uint(a1.z);
    const __half2 hh = *reinterpret_cast<const __half2 *>(&hb);
    const float hx = __low2float(hh), hy = __high2float(hh);
    const float qxx = a0.z * a0.z + a1.x * a1.x, qxy = a0.z * a0.w + a1.x * a1.y, qyy = a0.w * a0.w + a1.y * a1.y;
    const float X0 = tile_x0 - a0.x, Y0 = tile_y0 - a0.y;      // first pixel centre of the tile, relative to the splat centre
    // block i spans [X0 + 8 i, X0 + 8 i + 7]; it meets [-hx, hx] iff  (-hx - X0 - 7) / 8 <= i <= (hx - X0) / 8
    const int ix0 = max(0, (int)ceilf((-hx - X0 - 7.0f) * 0.125f)), ix1 = min(NBX - 1, (int)floorf((hx - X0) * 0.125f));
    const int iy0 = max(0, (int)ceilf((-hy - Y0 - 7.0f) * 0.125f)), iy1 = min(NBY - 1, (int)floorf((hy - Y0) * 0.125f));
    // The AABB (exact extents of the ellipse) inside ONE block: that block holds the whole ellipse, nothing to decide.  (A block without
    // a pixel centre inside the ellipse can still pass here; it costs one visit that adds nothing.)
    if (ix0 == ix1 && iy0 == iy1) return 1u << (iy0 * NBX + ix0);
    uint32_t bm = 0;
#pragma unroll 1
    for (int iy = iy0; iy <= iy1; ++iy) {
        const float by0 = Y0 + (float)(8 * iy), by1 = by0 + 7.0f;
#pragma unroll 1
        for (int ix = ix0; ix <= ix1; ++ix) {
            const float bx0 = X0 + (float)(8 * ix), bx1 = bx0 + 7.0f;
            if (ellipse_min_q(bx0, bx1, by0, by1, qxx, qxy, qyy) <= 1.0f + kEllipseSlack) bm |= 1u << (iy * NBX + ix);
        }
    }
    return bm;
}

struct StatusSnapshot {
    const uint32_t *sort_ctl;     // SortControl head: 3 words (dmin, dmax, error)
    const uint32_t *raster_ctl;   // RasterControl
    uint32_t *dst;                // [0, 3) sort head, [4, 4 + sizeof(RasterControl) / 4) raster control; nullptr = no snapshot
    // multi-GPU peers: the frame pointer is rank 0's allocation; *half_src (0 / 1, RasterControl::peer_parity) selects its half
    const uint32_t *half_src;
    unsigned long long half_bytes;
};

// What the host reads back about a sort and a frame.  A status snapshot slot is one FrameStatus: the layout above.
struct FrameStatus {
    uint32_t sort[4];         // SortControl head: dmin, dmax, error (word 3 is not written)
    RasterControl raster;
};
constexpr size_t kSortHeadBytes = 3 * 4;
static_assert(offsetof(SortControl, error) + 4 == kSortHeadBytes, "the SortControl head is its words 0-2");
static_assert(offsetof(FrameStatus, raster) == 4 * 4 && sizeof(FrameStatus) == (4 + sizeof(RasterControl) / 4) * 4,
              "StatusSnapshot writes the sort head to words 0-2 and the RasterControl from word 4");

// The caller's opaque pass that a frame is composited into (gs_render_params dest_color / dest_depth): device pointers to width x height
// pixels in the frame's format and row order, nullptr where that input is absent.  One block per frame-buffer parity, uploaded with the
// frame's other parameter blocks, so a captured frame graph reads each frame's own inputs.
struct CompositeParams {
    const void *color;      // RGBA8 or RGBA32F, as the frame
    const float *depth;     // window depth per pixel (glDepthRange(0, 1))
};
static inline bool has_composite_inputs(const gs_render_params &p) { return p.dest_color || p.dest_color_dev || p.dest_depth || p.dest_depth_dev; }

// A stereo or multi-view frame to the blend: every view's coarse tiles in one grid, view v's are slots [v ncoarse, (v + 1) ncoarse) of
// `ranges` and `tile_order` (k_bin_scan leaves each view's own schedule there, or k_raster_init the identity); the views' lists and
// records; where each view's pixels go in the frame.
struct ViewBlend {
    const ViewEntry *views;
    uint32_t nviews;
    uint32_t ncoarse;              // coarse tiles of one view
    int frame_width;               // pixels per row of the frame: 2 x the eye width (stereo, side by side), the view width (stacked)
    unsigned long long view_stride;   // pixels from one view's first pixel to the next's: the eye width, or width x height
};

// A frame's depth plane (gs_render_params.depth): one f32 per pixel, indexed as the frame's pixels, and the projection whose z row turns
// a record's ndc_z back into view depth -- the mono frame's ProjParams block of this parity; a stereo or multi-view frame reads each
// view's own from ViewBlend instead.
struct DepthTarget {
    float *plane;
    const ProjParams *P;
};

// View depth d = -z_view of a splat centre from its ndc_z and the projection's z row (column-major, as three.js stores it):
// z_view = (P[14] - ndc P[15]) / (ndc P[11] - P[10]), which covers perspective (P[11] = -1, P[15] = 0) and orthographic projections.
// Each step rounds once; tests/depth_f64.py restates it.
__device__ __forceinline__ float view_depth(float ndc, float p10, float p11, float p14, float p15) {
    return __fdiv_rn(fmaf(-ndc, p15, p14), fmaf(-ndc, p11, p10));
}

// COMPOSITE: the blend of a splat mesh drawn into a framebuffer that already holds an opaque pass (Viewer.js:1599-1620, the material's
// depthTest: true, depthWrite: false, NormalBlending, SplatMaterial3D.js:65-75).  Every fragment of a splat has the window depth
// zw = 0.5 ndc_z + 0.5 of its centre (SplatMaterial3D.js:208-210) and passes where zw <= d (three's LessEqualDepth; a NaN d passes
// nothing); the splats never test against each other.  What is left of the transmittance then shows the caller's colour:
// C = C_acc + T Cd, A = A_acc + T Ad.  Each warp keeps the largest depth of its 8x8 block, and the staging thread drops the blocks
// where zw exceeds it -- no pixel there can pass -- so an occluded splat never enters the compositing loop.
// VIEWS: the tiles of every view of a stereo or multi-view frame in one grid (ViewBlend); tiles_x ... height are one view's.  The
// schedule takes the views' own schedules in turn (the longest list of each view, then the second longest of each, ...), and a tile of
// view v reads that view's lists and records and stores its pixels v view strides further into the frame.
// DEPTH: the frame's view depth beside its colour (gs_render_params.depth): sum w_i d_i / (1 - T) over the same weights w_i = T_i alpha_i
// the colour is blended with, d_i the view depth of splat i's centre (view_depth, once per staged splat), +inf where 1 - T == 0.  The
// depth is staged in the record's ndc_z slot, or beside the records where COMPOSITE still needs the window depth there.
template <int FORMAT, int S, bool COMPOSITE, bool VIEWS = false, bool DEPTH = false>
__global__ void __launch_bounds__(128 * S * S, S == 1 ? 8 : 2)
k_blend(const uint2 *__restrict__ ranges, const unsigned long long *__restrict__ list, const SplatRecord *__restrict__ rec, int tiles_x,
        int tiles_y, int coarse_x, uint32_t rank, uint32_t world, int width, int height, int flip_y, void *__restrict__ frame_base, const uint32_t *__restrict__ tile_order,
        StatusSnapshot snap, const CompositeParams *__restrict__ comp, ViewBlend views, DepthTarget dt) {
    static_assert(!(VIEWS && COMPOSITE), "stereo and multi-view frames are not composited");
    pdl_enter();
    void *__restrict__ frame = snap.half_src ? (void *)((unsigned char *)frame_base + (size_t)(*snap.half_src & 1u) * snap.half_bytes) : frame_base;
    // Everything the host reads back about a frame (sort error bits, instance / visibility counters, overflow flag) is final before the
    // blend starts; CTA 0 copies it into a per-frame-buffer slot so that the read-back can run on the copy stream, off this stream.
    if (snap.dst && blockIdx.x == 0) {
        if (threadIdx.x < 3) snap.dst[threadIdx.x] = snap.sort_ctl[threadIdx.x];
        for (uint32_t i = threadIdx.x; i < (uint32_t)(sizeof(RasterControl) / 4); i += blockDim.x) snap.dst[4 + i] = snap.raster_ctl[i];
    }
    // (A CTA covering TWO fine tiles side by side -- one scan of the coarse list for 32x16 px -- was measured: fewer instructions, but
    // the per-round barrier then waits for the densest of 8 blocks instead of 4 and the blend got 5-18 % slower.  Not kept.)
    constexpr int THREADS = 128 * S * S, WARPS = THREADS / 32, NBX = 2 * S, NBY = 2 * S, TILE = 16 * S;
    constexpr int ROUNDS = S == 1 ? 4 : 1;       // filter rounds per batch
    constexpr int BATCH = ROUNDS * THREADS;      // list entries per batch
    __shared__ float4 s_rec[THREADS + 1][3];    // [THREADS] = the null record (alpha 0) that pairs with an odd tail
    __shared__ uint32_t s_ids[BATCH];
    __shared__ uint32_t s_cnt[ROUNDS * WARPS + 1];   // [round][warp] survivors of the filter -> exclusive offsets; last = total
    __shared__ uint8_t s_list[WARPS][THREADS];  // [block][staging warp * 32 + k] indices of the staged records that reach the block, in order
    __shared__ uint8_t s_nlist[WARPS][WARPS];   // [block][staging warp] how many
    static_assert(THREADS <= 256 || sizeof(uint8_t) == 1, "");
    const uint32_t sub = blockIdx.x % kFinePerCoarse;
    uint32_t slot, view = 0, coarse;   // slot: index into ranges
    if constexpr (VIEWS) {
        const uint32_t pos = blockIdx.x / kFinePerCoarse;
        view = pos % views.nviews;
        coarse = tile_order[view * views.ncoarse + pos / views.nviews] % views.ncoarse;   // the identity schedule holds slots, k_bin_scan's tiles
        slot = view * views.ncoarse + coarse;
        if (view) { list = views.views[view].list; rec = views.views[view].rec; }
    } else {
        slot = coarse = tile_order[blockIdx.x / kFinePerCoarse];
    }
    const int ccx = (int)(coarse % (uint32_t)coarse_x), ccy = (int)(coarse / (uint32_t)coarse_x);
    const int tx = ccx * kCoarseW + (int)(sub & (kCoarseW - 1)), ty = ccy * kCoarseH + (int)(sub >> kCoarseShiftX);
    if (tx >= tiles_x || ty >= tiles_y) return;
    if (!owns_coarse(ccx, ccy, rank, world)) return;   // another GPU's tile
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int lx = (warp % NBX) * 8 + (lane & 7), ly = (warp / NBX) * 8 + (lane >> 3) * 2;   // the lane's offset in the tile
    const int x = tx * TILE + lx, y0 = ty * TILE + ly;
    const float tile_x0 = (float)(tx * TILE) + 0.5f, tile_y0 = (float)(ty * TILE) + 0.5f;    // first pixel centre of the tile
    // pixels outside the frame start saturated so that they never keep a warp alive
    f32x2 T = pack2((x < width && y0 < height) ? 1.0f : 0.0f, (x < width && y0 + 1 < height) ? 1.0f : 0.0f);
    f32x2 Rr = pack2(0.f, 0.f), Gg = Rr, Bb = Rr, Dd = Rr;
    // pixel centres relative to the tile's first one: exact small integers, so the rounding of q does not grow with the distance from
    // the frame origin (with absolute coordinates the first-order bound on q's rounding near the q = 1 contour is ~4e-3 at 8K for
    // |g| up to 3 px^-1; an f32 emulation of that form reaches ~2e-3)
    const float DX = (float)lx;
    const f32x2 DY = pack2((float)ly, (float)(ly + 1));
    bool wdone = !__any_sync(0xffffffffu, fmaxf(lo2(T), hi2(T)) >= kTransmittanceCutoff);
    const uint2 rg = ranges[slot];
    const uint32_t lt = lanemask_lt();
    // COMPOSITE: the caller's depth at the lane's two pixels (no depth input: +inf, every fragment passes); pixels outside the frame are
    // NaN, which passes nothing and drops out of the block maximum (fmaxf returns the other operand)
    __shared__ float s_bmax[COMPOSITE ? WARPS : 1];
    float d0 = 0.0f, d1 = 0.0f;
    if constexpr (COMPOSITE) {
        const float *depth = comp->depth;
        d0 = d1 = __int_as_float(0x7fffffff);
        if (x < width) {
            if (y0 < height) d0 = depth ? depth[(size_t)(flip_y ? height - 1 - y0 : y0) * width + x] : __int_as_float(0x7f800000);
            if (y0 + 1 < height) d1 = depth ? depth[(size_t)(flip_y ? height - 2 - y0 : y0 + 1) * width + x] : __int_as_float(0x7f800000);
        }
        float m = fmaxf(d0, d1);
#pragma unroll
        for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (lane == 0) s_bmax[warp] = m;
    }
    if (threadIdx.x < 3) s_rec[THREADS][threadIdx.x] = (threadIdx.x == 1) ? make_float4(0.f, 0.f, 0.f, __int_as_float(0xff800000)) : make_float4(0.f, 0.f, 0.f, 0.f);   // log2(alpha) = -inf
    // DEPTH: the view's projection z row P[10], P[11], P[14], P[15] for the staging threads; under COMPOSITE the staged view depths sit
    // in s_d, the null record's at [THREADS].  (Shared, not registers: nothing of it stays live across the compositing loop.)
    __shared__ float s_pz[DEPTH ? 4 : 1];
    __shared__ float s_d[DEPTH && COMPOSITE ? THREADS + 1 : 1];
    if constexpr (DEPTH) {
        const ProjParams *P = VIEWS ? views.views[view].P : dt.P;
        if (threadIdx.x < 4) s_pz[threadIdx.x] = P->proj[threadIdx.x < 2 ? 10 + threadIdx.x : 12 + threadIdx.x];
        if (COMPOSITE && threadIdx.x == 0) s_d[THREADS] = 0.0f;
    }
    __syncthreads();      // the null record (and the block depths) are visible to every warp from here on
    // the tile's list is consumed in batches of BATCH entries
    const uint32_t nbatch = (rg.y - rg.x + BATCH - 1) / BATCH;
    for (uint32_t b = 0; b < nbatch; ++b) {
        const uint32_t base = rg.x + b * (uint32_t)BATCH;
        if (__syncthreads_and(wdone)) break;
        const unsigned long long *chunk = list + base;
        // ---- filter ROUNDS x THREADS list entries by this tile's mask bit; order-preserving compaction (order: round, warp, lane) --
        uint32_t ids[ROUNDS], bal[ROUNDS];
#pragma unroll
        for (int k = 0; k < ROUNDS; ++k) {
            const uint32_t i = base + (uint32_t)k * THREADS + threadIdx.x;
            bool hit = false;
            ids[k] = 0;
            if (i < rg.y) {
                const unsigned long long e = __ldg(chunk + (uint32_t)k * THREADS + threadIdx.x);
                hit = ((uint32_t)(e >> 32) >> sub) & 1u;
                ids[k] = (uint32_t)e;
            }
            bal[k] = __ballot_sync(0xffffffffu, hit);
            if (lane == 0) s_cnt[k * WARPS + warp] = __popc(bal[k]);
        }
        __syncthreads();
        if (warp == 0) {      // exclusive scan of the ROUNDS * WARPS counts
            uint32_t run = 0;
#pragma unroll
            for (int c = 0; c < ROUNDS * WARPS; c += 32) {
                const uint32_t v = (c + lane < ROUNDS * WARPS) ? s_cnt[c + lane] : 0u;
                const uint32_t inc = warp_inclusive_scan(v);
                if (c + lane < ROUNDS * WARPS) s_cnt[c + lane] = run + inc - v;
                run += __shfl_sync(0xffffffffu, inc, 31);
            }
            if (lane == 0) s_cnt[ROUNDS * WARPS] = run;
        }
        __syncthreads();
        const uint32_t nsurv = s_cnt[ROUNDS * WARPS];
#pragma unroll
        for (int k = 0; k < ROUNDS; ++k)
            if ((bal[k] >> lane) & 1u) s_ids[s_cnt[k * WARPS + warp] + __popc(bal[k] & lt)] = ids[k];
        __syncthreads();
        // ---- stage up to THREADS survivors at a time, then every warp composites the ones that reach its block -------------------
        for (uint32_t c0 = 0; c0 < nsurv; c0 += THREADS) {
            const uint32_t j = c0 + threadIdx.x;
            uint32_t bm = 0;
            if (j < nsurv) {
                const float4 *src = reinterpret_cast<const float4 *>(rec + s_ids[j]);
                float4 a0 = __ldg(src), a1 = __ldg(src + 1);
                float4 a2 = __ldg(src + 2);
                // a0 = cx, cy, g1x, g1y ; a1 = g2x, g2y, half2(hx, hy), alpha ; a2 = r, g, b, ndc z
                bm = block_touch_mask<NBX, NBY>(a0, a1, tile_x0, tile_y0);
                if constexpr (DEPTH) {
                    const float d = view_depth(a2.w, s_pz[0], s_pz[1], s_pz[2], s_pz[3]);
                    if constexpr (COMPOSITE) s_d[threadIdx.x] = d; else a2.w = d;
                }
                if constexpr (COMPOSITE) {
                    // window depth; 0.5 ndc_z is exact, so this is 0.5 ndc_z + 0.5 rounded once, fused or not.  Blocks whose every pixel
                    // is nearer than the splat drop out (also blocks without a depth that passes anything: NaN maximum)
                    a2.w = fmaf(0.5f, a2.w, 0.5f);
#pragma unroll
                    for (int b = 0; b < WARPS; ++b)
                        if (!(a2.w <= s_bmax[b])) bm &= ~(1u << b);
                }
                // staged form: u(p) = g1 . (p - t) + u0, w(p) = g2 . (p - t) + w0 at a pixel centre p, t = the tile's first pixel
                // centre (two FMAs each in the loop below); u0 = g1 . (t - c), w0 = g2 . (t - c)
                const float X0 = tile_x0 - a0.x, Y0 = tile_y0 - a0.y;
                const float u0 = fmaf(X0, a0.z, Y0 * a0.w), w0 = fmaf(X0, a1.x, Y0 * a1.y);
                a1.z = a0.w * a0.w + a1.y * a1.y;     // h = |d(u,w)/dy|^2
                a1.w = log2f(a1.w);                   // opacity folded into the exponent
                a0.x = u0; a0.y = w0;
                s_rec[threadIdx.x][0] = a0;           // u0, w0, g1x, g1y
                s_rec[threadIdx.x][1] = a1;           // g2x, g2y, h, log2(alpha)
                s_rec[threadIdx.x][2] = a2;
            }
            // per block: the indices of this staging warp's records that reach it, compacted in order
#pragma unroll
            for (int b = 0; b < WARPS; ++b) {
                const uint32_t v = __ballot_sync(0xffffffffu, (bm >> b) & 1u);
                if ((bm >> b) & 1u) s_list[b][warp * 32 + __popc(v & lt)] = (uint8_t)(threadIdx.x & 255);
                if (lane == 0) s_nlist[b][warp] = (uint8_t)__popc(v);
            }
            __syncthreads();
            if (!wdone) {
#pragma unroll 1
                for (int sw = 0; sw < WARPS && !wdone; ++sw) {
                    const int cnt = s_nlist[warp][sw];
                    const uint8_t *lst = &s_list[warp][sw * 32];
                    const int jbase = (THREADS > 256 ? (sw & ~7) * 32 : 0);      // 8-bit index inside the group of 8 staging warps
                    // Two records per iteration: their quad coordinates and exponentials are independent, only the transmittance chain is
                    // serial.  The blend's duration is set by the longest per-warp chain (the densest block), not by issue slots, so the
                    // instruction-level parallelism matters more than the instruction count.  An odd tail pairs with the null record.
#pragma unroll 1
                    for (int k = 0; k < cnt; k += 2) {
                        const int ja = jbase + lst[k];
                        const int jb = (k + 1 < cnt) ? jbase + lst[k + 1] : THREADS;
                        const float4 A = s_rec[ja][0], B = s_rec[ja][1], C = s_rec[ja][2];
                        const float4 D = s_rec[jb][0], E = s_rec[jb][1], F = s_rec[jb][2];
                        // the lane's two pixels ride in the halves of an f32x2 pair; per-record scalars enter as broadcast operands
                        const float tua = fmaf(DX, A.z, A.x), twa = fmaf(DX, B.x, A.y);
                        const float tub = fmaf(DX, D.z, D.x), twb = fmaf(DX, E.x, D.y);
                        const f32x2 Ua = fma2(DY, bcast2(A.w), bcast2(tua)), Wa = fma2(DY, bcast2(B.y), bcast2(twa));
                        const f32x2 Ub = fma2(DY, bcast2(D.w), bcast2(tub)), Wb = fma2(DY, bcast2(E.y), bcast2(twb));
                        const f32x2 Qa = fma2(Wa, Wa, mul2(Ua, Ua)), Qb = fma2(Wb, Wb, mul2(Ub, Ub));
                        // exp(-0.5 A) * vColor.a with A = 8 q, zero outside the quad's inscribed disc (COMPOSITE: and where the
                        // splat's window depth, staged in C.w / F.w, fails the caller's depth test)
                        const f32x2 Xa = fma2(Qa, bcast2(-5.770780163555854f), bcast2(B.w)), Xb = fma2(Qb, bcast2(-5.770780163555854f), bcast2(E.w));
                        const float ea0 = (lo2(Qa) <= 1.0f && (!COMPOSITE || C.w <= d0)) ? ex2_approx(lo2(Xa)) : 0.0f;
                        const float ea1 = (hi2(Qa) <= 1.0f && (!COMPOSITE || C.w <= d1)) ? ex2_approx(hi2(Xa)) : 0.0f;
                        const float eb0 = (lo2(Qb) <= 1.0f && (!COMPOSITE || F.w <= d0)) ? ex2_approx(lo2(Xb)) : 0.0f;
                        const float eb1 = (hi2(Qb) <= 1.0f && (!COMPOSITE || F.w <= d1)) ? ex2_approx(hi2(Xb)) : 0.0f;
                        f32x2 wgt = mul2(T, pack2(ea0, ea1));
                        Rr = fma2(wgt, bcast2(C.x), Rr); Gg = fma2(wgt, bcast2(C.y), Gg); Bb = fma2(wgt, bcast2(C.z), Bb);
                        if constexpr (DEPTH) Dd = fma2(wgt, bcast2(COMPOSITE ? s_d[ja] : C.w), Dd);
                        T = fma2(wgt, bcast2(-1.0f), T);                                   // T *= (1 - alpha)
                        wgt = mul2(T, pack2(eb0, eb1));
                        Rr = fma2(wgt, bcast2(F.x), Rr); Gg = fma2(wgt, bcast2(F.y), Gg); Bb = fma2(wgt, bcast2(F.z), Bb);
                        if constexpr (DEPTH) Dd = fma2(wgt, bcast2(COMPOSITE ? s_d[jb] : F.w), Dd);
                        T = fma2(wgt, bcast2(-1.0f), T);
                        if (!__any_sync(0xffffffffu, fmaxf(lo2(T), hi2(T)) >= kTransmittanceCutoff)) { wdone = true; break; }
                    }
                }
            }
            if (__syncthreads_and(wdone)) break;      // every pixel of the tile is saturated: the rest of the batch cannot change it
        }
    }
    const float T0 = lo2(T), T1 = hi2(T), r0 = lo2(Rr), r1 = hi2(Rr), g0 = lo2(Gg), g1 = hi2(Gg), b0 = lo2(Bb), b1 = hi2(Bb);
    if (x < width) {
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const int y = y0 + k;
            if (y < height) {
                const float Tk = k ? T1 : T0;
                float Rk = k ? r1 : r0, Gk = k ? g1 : g0, Bk = k ? b1 : b0;
                float A = 1.0f - Tk;            // alpha accumulates as 1 - prod(1 - alpha_i)
                const int out_row = flip_y ? (height - 1 - y) : y;   // every rank writes its tiles into a full-size frame
                const size_t at = VIEWS ? view * views.view_stride + (size_t)out_row * views.frame_width + x : (size_t)out_row * width + x;
                if constexpr (DEPTH) {          // (before the destination enters A)
                    const float Dk = k ? hi2(Dd) : lo2(Dd);
                    dt.plane[at] = A == 0.0f ? __int_as_float(0x7f800000) : __fdiv_rn(Dk, A);
                }
                if constexpr (COMPOSITE) {      // the caller's colour under what the splats left of the transmittance
                    if (const void *dst = comp->color) {
                        float4 cd;
                        if (FORMAT == GS_FRAME_RGBA32F) {
                            cd = reinterpret_cast<const float4 *>(dst)[at];
                        } else {
                            const uint32_t v = reinterpret_cast<const uint32_t *>(dst)[at];
                            cd = make_float4((float)(v & 255u) * (1.0f / 255.0f), (float)((v >> 8) & 255u) * (1.0f / 255.0f),
                                             (float)((v >> 16) & 255u) * (1.0f / 255.0f), (float)(v >> 24) * (1.0f / 255.0f));
                        }
                        Rk = fmaf(Tk, cd.x, Rk); Gk = fmaf(Tk, cd.y, Gk); Bk = fmaf(Tk, cd.z, Bk); A = fmaf(Tk, cd.w, A);
                    }
                }
                if (FORMAT == GS_FRAME_RGBA32F) {
                    reinterpret_cast<float4 *>(frame)[at] = make_float4(Rk, Gk, Bk, A);
                } else {
                    const uint32_t r8 = (uint32_t)(__saturatef(Rk) * 255.0f + 0.5f), g8 = (uint32_t)(__saturatef(Gk) * 255.0f + 0.5f);
                    const uint32_t b8 = (uint32_t)(__saturatef(Bk) * 255.0f + 0.5f), a8 = (uint32_t)(__saturatef(A) * 255.0f + 0.5f);
                    reinterpret_cast<uint32_t *>(frame)[at] = r8 | (g8 << 8) | (b8 << 16) | (a8 << 24);
                }
            }
        }
    }
    if (world > 1) __threadfence_system();   // the frame may live in a peer GPU's memory (fused tile gather): publish before the signal
}

// records -> the ABI's gs_projected_splat (basis vectors recovered from g = B/|B|^2)
__global__ void k_export_projected(const SplatRecord *__restrict__ rec, const ushort4 *__restrict__ rects, uint32_t count, gs_projected_splat *out) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= count) return;
    const SplatRecord r = rec[s];
    gs_projected_splat o;
    o.cx = r.cx; o.cy = r.cy;
    const float n1 = r.g1x * r.g1x + r.g1y * r.g1y, n2 = r.g2x * r.g2x + r.g2y * r.g2y;
    o.b1x = n1 > 0.f ? r.g1x / n1 : 0.f; o.b1y = n1 > 0.f ? r.g1y / n1 : 0.f;
    o.b2x = n2 > 0.f ? r.g2x / n2 : 0.f; o.b2y = n2 > 0.f ? r.g2y / n2 : 0.f;
    o.r = r.r; o.g = r.g; o.b = r.b; o.a = r.a;
    o.ndc_z = r.ndc_z;
    o.valid = (r.ndc_z >= -1.0f && r.ndc_z <= 1.0f) ? 1u : 0u;
    if (!o.valid) o.ndc_z = 0.f;
    out[s] = o;
}

// ---------------------------------------------------------------------------------------------------------------
// Host side of the rasteriser

// Calls f(cov_f16, sh_format, views, kernel) for each k_project instantiation: the launch picks one, the preloads take them all
template <typename F> static void for_each_project(F &&f) {
#define GS_PROJ(C, ST) f(C, GS_SH_NONE, ST, k_project<C, GS_SH_NONE, ST>); f(C, GS_SH_F16, ST, k_project<C, GS_SH_F16, ST>); \
                       f(C, GS_SH_U8, ST, k_project<C, GS_SH_U8, ST>); f(C, GS_SH_F32, ST, k_project<C, GS_SH_F32, ST>)
    GS_PROJ(false, false); GS_PROJ(true, false); GS_PROJ(false, true); GS_PROJ(true, true);
#undef GS_PROJ
}

// Calls f(format, tile_scale, composite, views, depth, kernel) for each k_blend instantiation (a stereo or multi-view frame composites
// nothing)
template <typename F> static void for_each_blend(F &&f) {
#define GS_BLEND(S, COMP, ST, D) f(GS_FRAME_RGBA8, S, COMP, ST, D, k_blend<GS_FRAME_RGBA8, S, COMP, ST, D>); \
                                 f(GS_FRAME_RGBA32F, S, COMP, ST, D, k_blend<GS_FRAME_RGBA32F, S, COMP, ST, D>)
#define GS_BLENDS(D) GS_BLEND(1, false, false, D); GS_BLEND(2, false, false, D); GS_BLEND(1, true, false, D); GS_BLEND(2, true, false, D); \
                     GS_BLEND(1, false, true, D); GS_BLEND(2, false, true, D)
    GS_BLENDS(false); GS_BLENDS(true);
#undef GS_BLENDS
#undef GS_BLEND
}

// What one view's projection and binning read and write: the mono frame's, one eye's of a stereo frame (gs_render_params.eyes), or
// one camera's of a multi-view frame (gs_frame_views).  view[0].rctl is also the frame's control block: frame_seq, the peer words,
// subset_count, the visibility slots of every view, and the block the host reads back.  The rctl of a later view carries only its
// instance count and overflow flag until k_views_join folds them in.
struct View {
    DevBuf<ProjParams> projp;          // per-frame projection parameters read by k_project, one block per frame-buffer parity
    DevBuf<DynamicUniforms> dyn;       // ... and the uniforms of dynamic / optional-effects / 8-bit SH frames
    DevBuf<SplatRecord> records;
    DevBuf<ushort4> rects;
    DevBuf<unsigned long long> list;   // per-coarse-tile lists (instance_capacity entries)
    DevBuf<uint32_t> bin_totals;       // counting-sort binning: instances per coarse tile (kBinTiles words, zero at the start of a frame)
    DevBuf<RasterControl> rctl;
    DevBuf<SortControl> sctl;          // the instance sort's digit histograms (radix binning), zero at the start of a frame
    DevBuf<uint32_t> super_own;        // views > 0: their own per-group instance counts
    uint32_t *super_sums = nullptr;    // the radix binning's per-group instance counts (view 0: RasterState::super_sums; else super_own)
};

// The views of a frame: the mono frame, the two eyes of a stereo frame side by side from one draw order (gs_render_params.eyes), or the
// cameras of a multi-view frame stacked top to bottom, each with its own draw order (gs_frame_views).  A view is width x height (one
// eye: width / 2).
struct FrameViews {
    uint32_t count = 1;
    const gs_view *cams = nullptr;     // a multi-view frame's cameras
    bool stacked() const { return cams != nullptr; }
};
static inline FrameViews frame_views(const gs_render_params &p) { FrameViews v; if (p.eyes) v.count = 2; return v; }

struct RasterState {
    DevBuf<uint4> cc;
    DevBuf<unsigned char> cov, sh;
    DevBuf<uint32_t> scene_idx;
    int cov_format = GS_COV_F32, sh_format = GS_SH_NONE;
    uint32_t sh_degree = 0, uploaded = 0;
    uint64_t generation = 0;     // counts the uploads that replaced the scene: a streamed upload (gs_stream_append) checks it is still its own
    bool have_scene_idx = false;
    // view[0]: the mono frame, a stereo frame's left eye or a multi-view frame's first camera.  Later views are reserved by the first
    // frame that has them (before any graph capture), so a mono engine allocates nothing for them and view[0]'s buffers stay where the
    // frame graphs captured them
    View view[GS_MAX_VIEWS];
    uint32_t views_reserved = 1;
    DevBuf<ViewEntry> view_table;  // [parity][GS_MAX_VIEWS]: the reserved views' buffers, for the kernels of stereo and multi-view frames
    DevBuf<uint32_t> block_sums; // coarse instances per chunk of draw ranks
    DevBuf<uint32_t> warp_sums;  // ... and per warp (256 draw ranks) inside the chunk
    DevBuf<uint32_t> super_sums; // ... and per group of kBinThreads chunks: [0, S) view 0's binning, [S, 2S) subset compaction
    uint32_t super_stride = 0;
    RadixSort<uint16_t, unsigned long long> isort;   // radix binning: instances {coarse tile id; fine-tile mask, splat id}
    // the frame's coarse tiles, indexed by slot: view v's tiles are [v ncoarse, (v + 1) ncoarse)
    DevBuf<uint2> ranges;         // each tile's range of its view's list
    DevBuf<uint32_t> tile_order;  // blend schedule: slots by list length, longest first
    DevBuf<uint32_t> bin_hist;    // counting-sort binning: [coarse tile][chunk] instance counts -> offsets
    DevBuf<ushort4> rect_by_rank; // counting-sort binning: the rects gathered in draw-rank order by k_bin_count
    uint32_t bin_stride = 0;
    // composited frames (first use allocates): per parity, the blend's CompositeParams and the device copies of host inputs
    DevBuf<CompositeParams> comp;
    DevBuf<unsigned char> dest_color[2];
    DevBuf<float> dest_depth[2];
    // frames with depth (gs_render_params.depth; first use allocates): one max_width x max_height f32 plane per frame-buffer parity, and
    // the plane and bytes of the last frame enqueued with depth (GS_BUF_DEPTH; -1: none yet).  Host code that runs on every frame sets
    // them, graph replays included
    DevBuf<float> depth[2];
    int last_depth_parity = -1;
    size_t last_depth_bytes = 0;
    DevBuf<unsigned char> frame;
    DevBuf<unsigned char> frame_alt;   // second device frame: pipelined frames (gs_frame_begin) alternate so a D2H copy can overlap the next frame
    unsigned char *frame_half2 = nullptr;   // multi-GPU rank 0 with a double-size exported frame allocation: its second half (instead of frame_alt)
    size_t frame_half_bytes = 0;
    int frame_parity = 0;
    // status snapshot taken by the blend kernel (see StatusSnapshot): one destination slot per frame-buffer parity, source sort control
    FrameStatus *snap_slots = nullptr;
    const uint32_t *snap_sort_ctl = nullptr;
    bool snapshot_taken = false;   // the last raster_bin_blend launched a blend that wrote the snapshot
    DevBuf<gs_projected_splat> exported;
    // fused tile gather over NVLink peer memory (world_size > 1)
    DevBuf<PeerSync> peer_sync_local;      // rank 0 owns the block
    PeerSync *peer_sync = nullptr;       // rank 0: local block; others: rank 0's block mapped through CUDA IPC (or rank 0's, see peer_local)
    void *peer_frame = nullptr;          // others: rank 0's frame buffer mapped through CUDA IPC (or rank 0's, see peer_local)
    bool peer_root = false, peer_attached = false;
    bool peer_local = false;             // the group shares this process and device (gs_peer_attach_local): peer_frame / peer_sync are
                                         // rank 0's own pointers, not mappings
    unsigned long long instance_capacity = 0;
    int sm_count = 132;
    int last_format = GS_FRAME_RGBA32F;
    size_t last_frame_bytes = 0;
};

// Fine-tile edge for a frame: 16 px while that gives at most kBinTiles coarse tiles (8 x 4 fine tiles each, the counting-sort binning's
// 8-bit bins: 1920x1080 = 255), else 32 px (3840x2160 = 255 coarse tiles of 256 x 128 px).  Frames with more than kBinTiles coarse
// tiles at 32 px keep 32 px and take the radix binning.
static inline int frame_tile_shift(uint32_t width, uint32_t height) {
    const uint32_t cx = (width + kTile * kCoarseW - 1) / (kTile * kCoarseW), cy = (height + kTile * kCoarseH - 1) / (kTile * kCoarseH);
    return (cx * cy <= (uint32_t)kBinTiles) ? kTileShift : kTileShift + 1;
}

// The tiles of a frame at its own fine-tile edge
struct FrameTiles {
    int shift;              // fine-tile edge, log2 px
    int x, y;               // fine tiles across, down
    int coarse_x;           // coarse tiles across
    uint32_t ncoarse;       // coarse tiles
};
static inline FrameTiles frame_tiles(uint32_t width, uint32_t height) {
    FrameTiles t;
    t.shift = frame_tile_shift(width, height);
    const int tpx = 1 << t.shift;
    t.x = (width + tpx - 1) / tpx;
    t.y = (height + tpx - 1) / tpx;
    t.coarse_x = (t.x + kCoarseW - 1) / kCoarseW;
    t.ncoarse = (uint32_t)t.coarse_x * (uint32_t)((t.y + kCoarseH - 1) / kCoarseH);
    return t;
}

// Reserves view v's buffers once: view 0 when the engine is created, later views on the first frame that has them.  An engine created
// without a framebuffer keeps only view 0's parameter and control blocks, which sort-only and peer calls use.
static int raster_reserve_view(RasterState &rs, const gs_config &c, int v) {
    View &w = rs.view[v];
    if (w.rctl.p) return GS_OK;
    const size_t n = c.max_splat_count ? c.max_splat_count : 1;
    int rc;
    // per-frame parameter blocks: one per frame-buffer parity (pipelined frames upload them off-stream)
    if ((rc = w.projp.ensure(2)) || (rc = w.dyn.ensure(2)) || (rc = w.sctl.ensure(1))) return rc;
    CU(cudaMemset(w.dyn.p, 0, 2 * sizeof(DynamicUniforms)));
    if (c.max_width && c.max_height) {
        if ((rc = w.records.ensure(n)) || (rc = w.rects.ensure(n)) || (rc = w.list.ensure(rs.instance_capacity)) || (rc = w.bin_totals.ensure(kBinTiles)))
            return rc;
        CU(cudaMemset(w.bin_totals.p, 0, kBinTiles * 4));
    }
    if (v) {   // a later view starts empty; after each frame k_views_join empties it again
        if ((rc = w.super_own.ensure(rs.super_stride))) return rc;
        CU(cudaMemset(w.super_own.p, 0, w.super_own.n * sizeof(uint32_t)));
        CU(cudaMemset(w.sctl.p, 0, sizeof(SortControl)));
    }
    w.super_sums = v ? w.super_own.p : rs.super_sums.p;
    if ((rc = w.rctl.ensure(1))) return rc;      // last: its presence says the rest is there
    // k_raster_init resets only the per-frame counters; peer_timeout, which the host checks after every frame, is written by the
    // multi-GPU kernels alone, so it must start at zero (cudaMalloc can hand back memory that a freed allocation left non-zero)
    CU(cudaMemset(w.rctl.p, 0, sizeof(RasterControl)));
    return GS_OK;
}

// Grows a buffer that frames index by slot without losing it when the allocation fails: the engine keeps rendering the frames it could.
template <typename T> static int grow_keeping(DevBuf<T> &b, size_t count) {
    if (count <= b.n) return GS_OK;
    DevBuf<T> t;
    if (int rc = t.ensure(count)) return rc;
    std::swap(b.p, t.p); std::swap(b.n, t.n);
    return GS_OK;
}

// Reserves views [1, count) for a stereo or multi-view frame (before any graph capture) and lists every reserved view in view_table.
// Frames of more than two stacked views may need more tile slots than the engine was created with: *moved reports that the slots
// were reallocated, so that frame graphs holding the old ones are dropped.  A failed reservation leaves the views reserved so far.
static int raster_reserve_views(RasterState &rs, const gs_config &c, uint32_t count, bool *moved) {
    *moved = false;
    if (count <= rs.views_reserved) return GS_OK;
    int rc;
    if ((rc = rs.view_table.ensure(2 * GS_MAX_VIEWS))) return rc;
    if (c.max_width && c.max_height) {   // V stacked views of width x height, V height <= max_height: see raster_init
        const uint32_t view_coarse = std::max(frame_tiles(c.max_width, std::max(c.max_height / count, 1u)).ncoarse, (uint32_t)kBinTiles);
        const size_t slots = (size_t)count * std::min(view_coarse, 65536u);
        *moved = slots > rs.ranges.n;
        if ((rc = grow_keeping(rs.ranges, slots)) || (rc = grow_keeping(rs.tile_order, slots))) return rc;
    }
    for (uint32_t v = rs.views_reserved; v < count; ++v) {
        if ((rc = raster_reserve_view(rs, c, (int)v))) return rc;
        for (uint32_t u = v == 1 ? 0 : v; u <= v; ++u) {   // view 0's entries go in with the first table
            const View &w = rs.view[u];
            for (int parity = 0; parity < 2; ++parity) {
                const ViewEntry E{w.projp.p + parity, w.dyn.p + parity, w.records.p, w.rects.p, w.list.p, w.rctl.p, w.sctl.p, w.bin_totals.p, w.super_sums};
                CU(cudaMemcpy(rs.view_table.p + parity * GS_MAX_VIEWS + u, &E, sizeof(E), cudaMemcpyHostToDevice));
            }
        }
        rs.views_reserved = v + 1;
    }
    return GS_OK;
}

static int raster_init(RasterState &rs, const gs_config &c, int sm_count) {
    rs.sm_count = sm_count;
    const size_t n = c.max_splat_count ? c.max_splat_count : 1;
    const bool framebuffer = c.max_width && c.max_height;
    int rc;
    if (framebuffer) {   // what view 0's reservation reads: the list's capacity and super_sums
        rs.super_stride = (uint32_t)(((n + kBinTile - 1) / kBinTile) / kBinThreads + 2);
        if ((rc = rs.cc.ensure(n)) || (rc = rs.block_sums.ensure((n + kBinTile - 1) / kBinTile + 1)) ||
            (rc = rs.warp_sums.ensure(((n + kBinTile - 1) / kBinTile + 1) * (kBinThreads / 32))) || (rc = rs.super_sums.ensure(2 * (size_t)rs.super_stride)))
            return rc;
        const char *f = getenv("GS_INSTANCE_FACTOR");
        const double factor = f ? atof(f) : 4.0;
        const size_t tiles = (size_t)((c.max_width + kTile - 1) / kTile) * ((c.max_height + kTile - 1) / kTile);
        rs.instance_capacity = (unsigned long long)(factor * (double)n) + 4ull * tiles + 65536ull;
        if (rs.instance_capacity > 0xfffffff0ull) rs.instance_capacity = 0xfffffff0ull;
    }
    if ((rc = raster_reserve_view(rs, c, 0)) || !framebuffer) return rc;
    // Slots for two views of the most coarse tiles any frame up to the maximum can have.  A frame at 16-px tiles has at most kBinTiles;
    // at 32 px the count grows with width and height, so it is at most the maximum frame's.  (Across the switch the count drops:
    // 1920x1080 has 255 coarse tiles at 16 px, 2048x1080 has 72 at 32 px.)  raster_check refuses views of more than 65536.  Every writer
    // indexes by a coarse tile of the current frame: k_raster_init the first views x ncoarse slots, k_bin_scan its ncoarse CTAs' tiles,
    // the radix binning's scatters the tile keys present in the view, all below ncoarse.
    const FrameTiles most = frame_tiles(c.max_width, c.max_height);
    const size_t slots = 2 * (size_t)std::min(std::max(most.ncoarse, (uint32_t)kBinTiles), 65536u);
    if ((rc = rs.ranges.ensure(slots)) || (rc = rs.tile_order.ensure(slots)) || (rc = rs.frame.ensure((size_t)c.max_width * (c.max_height + kTile) * 16)))
        return rc;
    // The radix binning runs only for frames with more than kBinTiles coarse tiles at their own tile edge, i.e. at 32 px (a frame with
    // that many at 16 px switches to 32 px).  The count at 32 px grows with width and height separately and no frame exceeds the
    // engine's maximum in either, so an engine whose maximum frame stays within kBinTiles never needs the instance sort's buffers
    // (20 B per instance slot).
    if (most.ncoarse > (uint32_t)kBinTiles && (rc = rs.isort.reserve(rs.instance_capacity, 2))) return rc;
    // counting-sort binning: one column of chunk counts per coarse tile (kBinRanks draw ranks per chunk)
    const size_t coarse = (size_t)((c.max_width + kTile * kCoarseW - 1) / (kTile * kCoarseW)) * ((c.max_height + kTile * kCoarseH - 1) / (kTile * kCoarseH));
    const size_t chunks = (n + kBinRanks - 1) / kBinRanks + 1;
    rs.bin_stride = (uint32_t)((chunks + 31) & ~(size_t)31);
    if ((rc = rs.bin_hist.ensure(std::max<size_t>(coarse, 1) * rs.bin_stride))) return rc;
    return rs.rect_by_rank.ensure(n);
}

static int raster_upload(RasterState &rs, const gs_config &c, const gs_splat_data &d, cudaStream_t st) {
    if (!c.max_width || !c.max_height) return fail(GS_ERR_NOT_READY, "engine created without a framebuffer (max_width/max_height = 0)");
    if ((uint64_t)d.from + d.count > c.max_splat_count) return fail(GS_ERR_CAPACITY, "splat data [%u,%u) exceeds max_splat_count %u", d.from, d.from + d.count, c.max_splat_count);
    if (!d.centers_colors || !d.covariances) return fail(GS_ERR_BAD_ARG, "gs_upload_splat_data: null centers_colors/covariances");
    if (d.sh_degree > 2) return fail(GS_ERR_BAD_ARG, "sh_degree %u > 2", d.sh_degree);
    const size_t n = c.max_splat_count;
    const size_t cov_elt = d.cov_format == GS_COV_F16 ? 12 : 24;
    const size_t ncomp = d.sh_degree == 2 ? 24 : (d.sh_degree == 1 ? 9 : 0);
    const size_t sh_elt = ncomp * (d.sh_format == GS_SH_F16 ? 2 : (d.sh_format == GS_SH_U8 ? 1 : 4));
    if (d.from == 0) { rs.uploaded = 0; ++rs.generation; } // a (re)upload from splat 0 may change the storage formats and drop the scene indexes
    if (rs.uploaded && (rs.cov_format != d.cov_format || (rs.sh_degree != d.sh_degree) || (ncomp && rs.sh_format != d.sh_format)))
        return fail(GS_ERR_BAD_ARG, "splat data format changed between partial uploads");
    // every splat of a scene has a scene index or none has: a range uploaded without them would read whatever the buffer held
    if (rs.uploaded && (d.scene_indexes != nullptr) != rs.have_scene_idx)
        return fail(GS_ERR_BAD_ARG, "scene_indexes %s in this partial upload but %s in the first", d.scene_indexes ? "given" : "absent",
                    rs.have_scene_idx ? "given" : "absent");
    rs.cov_format = d.cov_format;
    rs.sh_degree = d.sh_degree;
    rs.sh_format = ncomp ? d.sh_format : GS_SH_NONE;
    int rc;
    if ((rc = rs.cov.ensure(n * cov_elt + 16))) return rc;
    if (ncomp) {
        if (!d.spherical_harmonics) return fail(GS_ERR_BAD_ARG, "sh_degree %u without spherical_harmonics", d.sh_degree);
        if ((rc = rs.sh.ensure(n * sh_elt + 16))) return rc;
    }
    CU(cudaMemcpyAsync(rs.cc.p + d.from, d.centers_colors, (size_t)d.count * 16, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(rs.cov.p + (size_t)d.from * cov_elt, d.covariances, (size_t)d.count * cov_elt, cudaMemcpyHostToDevice, st));
    if (ncomp) CU(cudaMemcpyAsync(rs.sh.p + (size_t)d.from * sh_elt, d.spherical_harmonics, (size_t)d.count * sh_elt, cudaMemcpyHostToDevice, st));
    if (d.scene_indexes) {
        if ((rc = rs.scene_idx.ensure(n))) return rc;
        CU(cudaMemcpyAsync(rs.scene_idx.p + d.from, d.scene_indexes, (size_t)d.count * 4, cudaMemcpyHostToDevice, st));
    }
    rs.have_scene_idx = d.scene_indexes != nullptr;
    rs.uploaded = std::max<uint32_t>(rs.uploaded, d.from + d.count);
    return GS_OK;
}

static unsigned char *raster_second_frame(RasterState &rs) { return rs.frame_alt.p ? rs.frame_alt.p : rs.frame_half2; }
static void *raster_frame_ptr(RasterState &rs, int) { return (rs.frame_parity && raster_second_frame(rs)) ? raster_second_frame(rs) : rs.frame.p; }

// The width of one view: the frame's, or one eye's of a stereo frame
static inline uint32_t view_width(const gs_render_params &p, const FrameViews &fv) { return fv.count > 1 && !fv.stacked() ? p.width / 2 : p.width; }

// View v's parameter blocks: the frame's uniforms, with the fields of the same names replaced by eye v's gs_eye (stereo) or camera v's
// gs_view (multi-view).
static int raster_upload_view_params(RasterState &rs, const gs_config &c, const gs_uniforms &frame_u, const gs_render_params &p, const FrameViews &fv, int v,
                                     cudaStream_t st) {
    gs_uniforms u = frame_u;
    if (fv.stacked()) {
        const gs_view &V = fv.cams[v];
        memcpy(u.model_view, V.model_view, 64); memcpy(u.projection, V.projection, 64);
        memcpy(u.camera_position, V.camera_position, 12); memcpy(u.view_matrix, V.view_matrix, 64);
        u.focal[0] = V.focal[0]; u.focal[1] = V.focal[1]; u.ortho_zoom = V.ortho_zoom;
    } else if (p.eyes) {
        const gs_eye &E = p.eyes[v];
        memcpy(u.model_view, E.model_view, 64); memcpy(u.projection, E.projection, 64);
        memcpy(u.camera_position, E.camera_position, 12); memcpy(u.view_matrix, E.view_matrix, 64);
    }
    const uint32_t width = view_width(p, fv);
    const FrameTiles t = frame_tiles(width, p.height);
    ProjParams P{};
    memcpy(P.mv, u.model_view, 64); memcpy(P.proj, u.projection, 64);
    memcpy(P.cam, u.camera_position, 12);
    P.focal[0] = u.focal[0]; P.focal[1] = u.focal[1]; P.viewport[0] = u.viewport[0]; P.viewport[1] = u.viewport[1];
    P.inv_focal_adj = u.inverse_focal_adjustment; P.ortho_zoom = u.ortho_zoom; P.orthographic = u.orthographic_mode;
    P.splat_scale = u.splat_scale; P.point_cloud = u.point_cloud_mode; P.sh_degree = u.sh_degree; P.antialiased = u.antialiased;
    P.kernel2d = u.kernel_2d_size; P.max_size = u.max_screen_space_splat_size; P.fade_in_complete = u.fade_in_complete;
    memcpy(P.scene_center, u.scene_center, 12); P.fade_start = u.visible_region_fade_start_radius;
    P.dynamic = u.dynamic_mode; P.optional_effects = u.enable_optional_effects; P.scene_count = (int)u.scene_count;
    P.tiles_x = t.x; P.tiles_y = t.y; P.rank = c.rank; P.world = c.world_size; P.width = (int)width; P.height = (int)p.height;
    P.tile_shift = t.shift;
    CU(cudaMemcpyAsync(rs.view[v].projp.p + rs.frame_parity, &P, sizeof(P), cudaMemcpyHostToDevice, st)); // pageable source: staged before return
    if (u.dynamic_mode || u.enable_optional_effects || rs.sh_format == GS_SH_U8) {
        DynamicUniforms du;
        memcpy(du.view, u.view_matrix, 64);
        memcpy(du.transforms, u.scene_transforms, sizeof(du.transforms));
        memcpy(du.sh8_min, u.sh8_min, sizeof(du.sh8_min)); memcpy(du.sh8_max, u.sh8_max, sizeof(du.sh8_max));
        memcpy(du.opacity, u.scene_opacity, sizeof(du.opacity)); memcpy(du.visibility, u.scene_visibility, sizeof(du.visibility));
        CU(cudaMemcpyAsync(rs.view[v].dyn.p + rs.frame_parity, &du, sizeof(du), cudaMemcpyHostToDevice, st)); // pageable source: staged before return
    }
    return GS_OK;
}

// The frame's parameter blocks.  The frame's views must be reserved (raster_reserve_views): callers upload the blocks before any graph capture.
static int raster_upload_params(RasterState &rs, const gs_config &c, const gs_uniforms &u, const gs_render_params &p, const FrameViews &fv, cudaStream_t st) {
    int rc;
    if (fv.count > rs.views_reserved) return fail(GS_ERR_NOT_READY, "a frame of %u views on an engine with %u reserved", fv.count, rs.views_reserved);
    for (uint32_t v = 0; v < fv.count; ++v) {
        if ((rc = raster_upload_view_params(rs, c, u, p, fv, (int)v, st))) return rc;
    }
    if (has_composite_inputs(p)) {     // the caller's opaque pass: host inputs are copied into this parity's buffers
        const size_t px = (size_t)p.width * p.height, color_bytes = px * (p.frame_format == GS_FRAME_RGBA8 ? 4 : 16);
        CompositeParams cp{p.dest_color_dev, p.dest_depth_dev};
        if ((rc = rs.comp.ensure(2))) return rc;
        if (p.dest_color) {
            if ((rc = rs.dest_color[rs.frame_parity].ensure(color_bytes))) return rc;
            CU(cudaMemcpyAsync(rs.dest_color[rs.frame_parity].p, p.dest_color, color_bytes, cudaMemcpyHostToDevice, st));
            cp.color = rs.dest_color[rs.frame_parity].p;
        }
        if (p.dest_depth) {
            if ((rc = rs.dest_depth[rs.frame_parity].ensure(px))) return rc;
            CU(cudaMemcpyAsync(rs.dest_depth[rs.frame_parity].p, p.dest_depth, px * sizeof(float), cudaMemcpyHostToDevice, st));
            cp.depth = rs.dest_depth[rs.frame_parity].p;
        }
        CU(cudaMemcpyAsync(rs.comp.p + rs.frame_parity, &cp, sizeof(cp), cudaMemcpyHostToDevice, st)); // pageable source: staged before return
    }
    return GS_OK;
}

// What every frame must satisfy before any of it is enqueued
static int raster_check(const RasterState &rs, const gs_config &c, const gs_uniforms &u, const gs_render_params &p, const FrameViews &fv) {
    if (fv.stacked()) {
        if (p.eyes) return fail(GS_ERR_BAD_ARG, "gs_frame_views: eyes cannot be set (each view is one camera)");
        if (has_composite_inputs(p)) return fail(GS_ERR_BAD_ARG, "gs_frame_views: multi-view frames cannot be composited (dest_color / dest_depth)");
        if (c.world_size > 1) return fail(GS_ERR_BAD_ARG, "gs_frame_views: multi-view frames are single-GPU (world_size %u)", c.world_size);
        if ((uint64_t)p.height * fv.count > c.max_height)
            return fail(GS_ERR_BAD_ARG, "gs_frame_views: %u views of height %u stack to %llu rows, more than the engine's max_height %u", fv.count, p.height,
                        (unsigned long long)p.height * fv.count, c.max_height);
    }
    if (!rs.uploaded) return fail(GS_ERR_NOT_READY, "gs_render before gs_upload_splat_data");
    if (p.width == 0 || p.height == 0 || p.width > c.max_width || p.height > c.max_height)
        return fail(GS_ERR_BAD_ARG, "frame %ux%u outside the engine's %ux%u", p.width, p.height, c.max_width, c.max_height);
    if ((p.dest_color && p.dest_color_dev) || (p.dest_depth && p.dest_depth_dev))
        return fail(GS_ERR_BAD_ARG, "dest_color / dest_depth: set the host or the device pointer of an input, not both");
    if (has_composite_inputs(p) && c.world_size > 1)
        return fail(GS_ERR_BAD_ARG, "dest_color / dest_depth: composited frames are single-GPU (world_size %u)", c.world_size);
    if (p.depth != 0 && p.depth != 1) return fail(GS_ERR_BAD_ARG, "depth %d: 0 (colour only) or 1 (view depth beside the colour)", (int)p.depth);
    if (p.depth && c.world_size > 1) return fail(GS_ERR_BAD_ARG, "depth: frames with depth are single-GPU (world_size %u)", c.world_size);
    if (p.render_count > rs.uploaded) return fail(GS_ERR_CAPACITY, "render_count %u > uploaded splats %u", p.render_count, rs.uploaded);
    const uint32_t ncoarse = frame_tiles(p.width, p.height).ncoarse;
    if (ncoarse > 65536u) return fail(GS_ERR_BAD_ARG, "frame %ux%u needs %u coarse tiles (> 65536)", p.width, p.height, ncoarse);
    if (p.eyes) {
        if (p.width & 1u) return fail(GS_ERR_BAD_ARG, "eyes: a stereo frame needs an even width, got %u", p.width);
        if (has_composite_inputs(p)) return fail(GS_ERR_BAD_ARG, "eyes: stereo frames cannot be composited (dest_color / dest_depth)");
        if (c.world_size > 1) return fail(GS_ERR_BAD_ARG, "eyes: stereo frames are single-GPU (world_size %u)", c.world_size);
        // the engine places splat centres with the viewport uniform, where WebGL uses the GL viewport: the two agree at the eye's size
        if (u.viewport[0] != (float)(p.width / 2) || u.viewport[1] != (float)p.height)
            return fail(GS_ERR_BAD_ARG, "eyes: the viewport uniform (%g, %g) must be one eye's size (%u, %u)", u.viewport[0], u.viewport[1], p.width / 2, p.height);
        const uint32_t eye_coarse = frame_tiles(p.width / 2, p.height).ncoarse;
        if (eye_coarse > 65536u) return fail(GS_ERR_BAD_ARG, "eyes: an eye of %ux%u needs %u coarse tiles (> 65536)", p.width / 2, p.height, eye_coarse);
    }
    return GS_OK;
}

// First half of a frame (it does not depend on the draw order): reset the frame's counters, let the peers store into rank 0's frame
// buffer, project every splat.  The frame's parameter blocks are on the device (raster_upload_params).
// A stereo or multi-view frame projects every view in one launch and resets every view's slots of the ranges and schedule.
static int raster_project(RasterState &rs, const gs_config &c, const gs_render_params &p, const FrameViews &fv, const Launch &launch) {
    const bool views = fv.count > 1;
    const uint32_t ncoarse = frame_tiles(view_width(p, fv), p.height).ncoarse;
    View &v = rs.view[0];
    const ViewEntry *table = views ? rs.view_table.p + rs.frame_parity * GS_MAX_VIEWS : nullptr;
    launch.pdl("k_raster_init", k_raster_init, 8, 256, 0, v.rctl.p, v.sctl.p, rs.ranges.p, fv.count * ncoarse, rs.super_sums.p, 2 * rs.super_stride,
               v.bin_totals.p, rs.tile_order.p);
    // rank 0 frees its frame buffer for the peers' stores right at the START of the frame (everything that consumed the previous
    // picture is earlier in stream order), so their blends never wait for rank 0's own sort + binning
    if (c.world_size > 1 && rs.peer_root) launch.plain(nullptr, k_peer_release, 1, 1, 0, rs.peer_sync, v.rctl.p, (uint32_t)(rs.frame_parity && rs.frame_half2));
    const dim3 grid((rs.uploaded + kProjThreads - 1) / kProjThreads, fv.count);
    const uint32_t *sc = rs.have_scene_idx ? rs.scene_idx.p : nullptr;
    const bool cov_f16 = rs.cov_format == GS_COV_F16;
    const int sh = (rs.sh_format == GS_SH_F16 || rs.sh_format == GS_SH_U8 || rs.sh_format == GS_SH_F32) ? (int)rs.sh_format : GS_SH_NONE;
    bool found = false;
    for_each_project([&](bool f16, int s, bool vw, auto kernel) {
        if (f16 != cov_f16 || s != sh || vw != views) return;
        launch.pdl("k_project", kernel, grid, kProjThreads, 0, rs.cc.p, rs.cov.p, rs.sh.p, (int)rs.sh_degree, sc, v.dyn.p + rs.frame_parity, v.projp.p + rs.frame_parity,
                   rs.uploaded, v.records.p, v.rects.p, v.rctl.p, table);
        found = true;
    });
    return found ? GS_OK : fail(GS_ERR_BAD_ARG, "no k_project for covariance format %d, SH format %d, %u views", (int)rs.cov_format, sh, fv.count);
}

// Bin the first render_count splats of the draw order d_order (or the device-side count at order_count_dev) into view v's per-coarse-
// tile lists, and its coarse tiles' slots [v ncoarse, (v + 1) ncoarse) of the ranges and schedule.
static int raster_bin(RasterState &rs, const gs_config &c, const FrameTiles &t, uint32_t render_count, const uint32_t *d_order,
                       const unsigned long long *order_count_dev, int v, const Launch &launch) {
    const int tiles_x = t.x, tiles_y = t.y, coarse_x = t.coarse_x;
    const uint32_t ncoarse = t.ncoarse, world = c.world_size, rank = c.rank;
    View &w = rs.view[v];
    uint2 *const ranges = rs.ranges.p + (size_t)v * ncoarse;
    uint32_t *const tile_order = rs.tile_order.p + (size_t)v * ncoarse;
    const uint32_t local_tiles = (uint32_t)tiles_x * (uint32_t)tiles_y;
    const bool counting_sort = ncoarse <= (uint32_t)kBinTiles;
    if (render_count && local_tiles && counting_sort) {
        const Ownership own = make_ownership(rank, world);
        const int sharded = world > 1 ? 1 : 0;
        const uint32_t chunks = (render_count + kBinRanks - 1u) / kBinRanks;
        launch.pdl("k_bin_count", k_bin_count, chunks, kBinWarps * 32, 0, d_order, render_count, order_count_dev, w.rects.p, coarse_x, ncoarse, rs.bin_hist.p,
                   rs.bin_stride, w.bin_totals.p, rs.rect_by_rank.p, own, sharded);
        launch.pdl("k_bin_scan", k_bin_scan, ncoarse, 1024, 0, rs.bin_hist.p, rs.bin_stride, (uint32_t)kBinRanks, render_count, order_count_dev, w.bin_totals.p, ncoarse,
                   ranges, w.rctl.p, tile_order, rs.instance_capacity);
        launch.pdl("k_bin_place", k_bin_place, chunks, kBinWarps * 32, 0, d_order, render_count, order_count_dev, rs.rect_by_rank.p, coarse_x, ncoarse, rs.bin_hist.p,
                   rs.bin_stride, w.list.p, rs.instance_capacity, w.rctl.p, own, sharded, (tiles_x <= 256 && tiles_y <= 256) ? 1 : 0);
    }
    if (render_count && local_tiles && !counting_sort) {
        const uint32_t chunks = (render_count + kBinTile - 1) / kBinTile;
        launch.pdl("k_tile_count", k_tile_count, chunks, kBinThreads, 0, d_order, render_count, order_count_dev, w.rects.p, rs.block_sums.p, rs.warp_sums.p, w.super_sums,
                   make_ownership(rank, world), world > 1 ? 1 : 0);
        launch.pdl("k_tile_emit", k_tile_emit, chunks, kBinThreads, 0, d_order, render_count, order_count_dev, w.rects.p, rs.block_sums.p, rs.warp_sums.p, w.super_sums,
                   coarse_x, rs.isort.keys[0].p, rs.isort.vals[0].p, rs.instance_capacity, w.rctl.p, make_ownership(rank, world), world > 1 ? 1 : 0);
        int tile_bits = 1;
        while ((1u << tile_bits) < std::max(ncoarse, 2u)) ++tile_bits;
        RadixJob<unsigned long long> j;   // the instance count lives on the device only
        j.vals = rs.isort.vals[0].p; j.out = w.list.p; j.n_dev = &w.rctl.p->total_instances; j.n_cap = rs.instance_capacity;
        j.plan = make_plan_bits(tile_bits); j.ctl = w.sctl.p; j.ranges = ranges; j.tag = kTagTile;
        return rs.isort.sort(j, launch);
    }
    return GS_OK;
}

// Second half of a frame: bin the draw order d_order (see raster_bin) into per-coarse-tile lists, blend them into the frame, and run the
// multi-GPU handshake.  ev_bin, if given, is recorded before the blend.  A stereo or multi-view frame bins each view on its own fine-tile
// grid (one grid over the whole frame would let tiles straddle the views' boundaries), then blends every view's tiles in one launch.
// View v's draw order is d_order + v order_stride: one shared order (stereo, 0) or one per view (multi-view, the render count).
static int raster_bin_blend(RasterState &rs, const gs_config &c, const gs_render_params &p, const FrameViews &fv, const uint32_t *d_order, size_t order_stride,
                            const unsigned long long *order_count_dev, cudaEvent_t ev_bin, const Launch &launch) {
    cudaStream_t st = launch.stream();
    const bool views = fv.count > 1;
    const uint32_t width = view_width(p, fv);
    const FrameTiles t = frame_tiles(width, p.height);
    const int tiles_x = t.x, tiles_y = t.y, coarse_x = t.coarse_x;
    const uint32_t ncoarse = t.ncoarse, world = c.world_size, rank = c.rank;
    const uint32_t local_tiles = (uint32_t)tiles_x * (uint32_t)tiles_y;
    rs.snapshot_taken = false;
    const View &v = rs.view[0];
    const ViewEntry *table = views ? rs.view_table.p + rs.frame_parity * GS_MAX_VIEWS : nullptr;
    for (uint32_t i = 0; i < fv.count; ++i) {
        const int rc = raster_bin(rs, c, t, p.render_count, d_order + i * order_stride, order_count_dev, (int)i, launch);
        if (rc) return rc;
    }
    // (a stereo frame's timeline keeps the name its join has always had)
    if (views) launch.pdl(fv.stacked() ? "k_views_join" : "k_stereo_join", k_views_join, fv.count - 1, 256, 0, table, rs.super_stride);
    if (ev_bin) CU(cudaEventRecord(ev_bin, st));
    if (local_tiles) {
        const bool peer_mode = world > 1 && (rs.peer_root || rs.peer_attached);
        // multi-GPU without the peer path: pixels of other ranks' tiles must be zero so that the frames can be summed (all-reduce)
        void *target = raster_frame_ptr(rs, p.frame_format);
        if (world > 1 && !peer_mode) CU(cudaMemsetAsync(target, 0, (size_t)p.width * p.height * (p.frame_format == GS_FRAME_RGBA8 ? 4 : 16), st));
        if (peer_mode && rs.peer_attached) {   // fused tile gather: blend straight into rank 0's frame over NVLink
            launch.plain(nullptr, k_peer_wait_release, 1, 1, 0, rs.peer_sync, v.rctl.p);
            target = rs.peer_frame;
        }
        const uint32_t grid = fv.count * ncoarse * kFinePerCoarse;
        const bool to_peer = peer_mode && rs.peer_attached;
        const StatusSnapshot snap{rs.snap_sort_ctl, reinterpret_cast<const uint32_t *>(v.rctl.p),
                                  (rs.snap_slots && rs.snap_sort_ctl) ? reinterpret_cast<uint32_t *>(rs.snap_slots + rs.frame_parity) : nullptr,
                                  to_peer ? &v.rctl.p->peer_parity : nullptr, to_peer ? (unsigned long long)rs.frame.n : 0ull};
        rs.snapshot_taken = snap.dst != nullptr;
        const int format = p.frame_format == GS_FRAME_RGBA8 ? GS_FRAME_RGBA8 : GS_FRAME_RGBA32F;
        const bool tile16 = t.shift == kTileShift, composite = !views && has_composite_inputs(p);
        // stereo: the eyes side by side in rows of the whole width; multi-view: the views stacked, one band of rows each
        const ViewBlend vb = !views ? ViewBlend{} : fv.stacked() ? ViewBlend{table, fv.count, ncoarse, (int)width, (unsigned long long)width * p.height}
                                                                 : ViewBlend{table, fv.count, ncoarse, (int)p.width, (unsigned long long)width};
        const bool depth = p.depth == 1;
        const DepthTarget dt{depth ? rs.depth[rs.frame_parity].p : nullptr, v.projp.p + rs.frame_parity};
        bool found = false;
        for_each_blend([&](int f, int s, bool comp, bool vw, bool dp, auto kernel) {
            if (f != format || s != (tile16 ? 1 : 2) || comp != composite || vw != views || dp != depth) return;
            launch.pdl("k_blend", kernel, grid, tile16 ? 128 : 512, 0, rs.ranges.p, v.list.p, v.records.p, tiles_x, tiles_y, coarse_x, rank, world, (int)width,
                       (int)p.height, p.flip_y, target, rs.tile_order.p, snap, has_composite_inputs(p) ? (const CompositeParams *)(rs.comp.p + rs.frame_parity) : nullptr,
                       vb, dt);
            found = true;
        });
        if (!found)
            return fail(GS_ERR_BAD_ARG, "no k_blend for frame format %d, %d-px tiles, composite %d, %u views, depth %d", format, tile16 ? 16 : 32, (int)composite,
                        fv.count, (int)depth);
        if (peer_mode && rs.peer_attached) launch.plain(nullptr, k_peer_signal, 1, 1, 0, rs.peer_sync);
        if (peer_mode && rs.peer_root) launch.plain("k_peer_wait_arrived", k_peer_wait_arrived, 1, 1, 0, rs.peer_sync, v.rctl.p, world - 1);
    }
    rs.last_format = p.frame_format;
    const size_t rows = fv.stacked() ? (size_t)fv.count * p.height : p.height;
    rs.last_frame_bytes = rows * p.width * (p.frame_format == GS_FRAME_RGBA8 ? 4 : 16);
    return GS_OK;
}

// order-preserving compaction of the sort input to this rank's splats (needs k_project's rects of THIS frame)
static int raster_subset(RasterState &rs, const gs_config &c, const uint32_t *d_indexes, uint32_t count, const int32_t *dist, uint32_t *sub_idx,
                         int32_t *sub_dist, const Launch &launch) {
    const uint32_t chunks = (count + kBinTile - 1) / kBinTile;
    const Ownership own = make_ownership(c.rank, c.world_size);
    launch.pdl("k_subset_count", k_subset_count, chunks, kBinThreads, 0, d_indexes, count, rs.view[0].rects.p, own, rs.block_sums.p, rs.warp_sums.p,
               rs.super_sums.p + rs.super_stride);
    launch.pdl("k_subset_emit", k_subset_emit, chunks, kBinThreads, 0, d_indexes, count, rs.view[0].rects.p, own, rs.block_sums.p, rs.warp_sums.p,
               rs.super_sums.p + rs.super_stride, dist, sub_idx, sub_dist, rs.view[0].rctl.p);
    return GS_OK;
}

static int raster_read_projected(RasterState &rs, gs_projected_splat *out, uint32_t count, const Launch &launch) {
    cudaStream_t st = launch.stream();
    if (count > rs.uploaded) return fail(GS_ERR_CAPACITY, "count %u > uploaded %u", count, rs.uploaded);
    int rc = rs.exported.ensure(count);
    if (rc) return rc;
    if (count) launch.plain(nullptr, k_export_projected, (count + 255) / 256, 256, 0, rs.view[0].records.p, rs.view[0].rects.p, count, rs.exported.p);
    CU(cudaMemcpyAsync(out, rs.exported.p, (size_t)count * sizeof(gs_projected_splat), cudaMemcpyDeviceToHost, st));
    return GS_OK;
}

} // namespace gs
