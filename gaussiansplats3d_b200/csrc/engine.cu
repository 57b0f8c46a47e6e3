// engine.cu -- host side of libgsplat_b200.so: the C ABI declared in include/gsplat_b200.h.
//
// One gs_engine = the device-resident state of one sort Worker (src/worker/SortWorker.js) plus one SplatMesh
// (src/splatmesh/SplatMesh.js) on one H100: persistent centres, splat data, scratch, one CUDA stream.
// There is no CPU implementation of any stage in this library: without a device every entry fails.
#include "../../include/gsplat_b200.h"
#include "common.cuh"
#include "sort_kernels.cuh"
#include "raster_kernels.cuh"
#include "shard_kernels.cuh"
#include "ksplat_transform.h"
#include "ksplat_kernels.cuh"
#include "file_kernels.cuh"
#include "cull_kernels.cuh"
#include "ray_kernels.cuh"
#include "generate_kernels.cuh"

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <new>
#include <type_traits>
#include <vector>

using namespace gs;

// ---------------------------------------------------------------------------------------------------------------
thread_local char g_gs_err[512] = "";
#define g_err g_gs_err
static int fail(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}
#define CU(call)                                                                                                  \
    do {                                                                                                          \
        cudaError_t _e = (call);                                                                                  \
        if (_e != cudaSuccess) return fail(GS_ERR_CUDA, "%s -> %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)

extern "C" int gs_abi_version(void) { return GS_ABI_VERSION; }
extern "C" const char *gs_last_error_message(void) { return g_err; }
extern "C" const char *gs_status_string(int s) {
    switch (s) {
        case GS_OK: return "ok";
        case GS_ERR_BAD_ARG: return "bad argument";
        case GS_ERR_NO_DEVICE: return "no CUDA device";
        case GS_ERR_CUDA: return "CUDA error";
        case GS_ERR_DEGENERATE: return "all distances equal";
        case GS_ERR_BUCKET_RANGE: return "bucket index out of range";
        case GS_ERR_NOT_READY: return "not ready";
        case GS_ERR_CAPACITY: return "capacity exceeded";
        default: return "unknown";
    }
}
extern "C" int gs_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

// ---------------------------------------------------------------------------------------------------------------
enum { EV_SORT0, EV_DEPTH, EV_BUCKET, EV_SORT1, EV_R0, EV_PROJECT, EV_BIN, EV_R1, EV_H2D0, EV_H2D1, EV_D2H0, EV_D2H1, EV_COUNT };

// one status slot of a pipelined frame: SortControl head (3 words, padded to 4) + RasterControl + slack
constexpr size_t kPipeSlotWords = 4 + (sizeof(RasterControl) + 3) / 4 + 12;   // SortControl head (3 words) + RasterControl
struct gs_engine {
    gs_config cfg{};
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[EV_COUNT]{};
    int sm_count = 132;
    size_t l2_bytes = 50u << 20;
    int key_bits = 16;

    // --- sorter state (SortWorker.js:125-178 memory regions, device side) ---
    DevBuf<int4> centers;            // int32x4 or f32x4 per splat
    DevBuf<uint32_t> scene_idx;      // dynamic mode
    DevBuf<uint32_t> indexes;        // indexesToSort
    DevBuf<uint32_t> precomputed;    // precomputedDistances (i32 or f32 bits)
    DevBuf<int32_t> dist;            // mappedDistances
    DevBuf<uint32_t> keys[2];        // radix keys ping/pong (u16 or u32 elements, sized in u32 words)
    DevBuf<uint32_t> vals[2];        // radix values ping/pong
    DevBuf<uint32_t> sorted;         // sortedIndexes
    DevBuf<float> transforms;        // 32 x mat4
    DevBuf<SortControl> ctl;
    DevBuf<DepthParams> depthp;      // per-frame depth parameters (device copy read by k_depth)
    DevBuf<uint32_t> tile_hist;       // radix tile histograms / offsets [pass][digit][tile]
    DevBuf<uint32_t> freq;           // scratch reproduction for gs_sort_indexes
    DevBuf<int32_t> dist_rows_i;     // gs_compute_distances: per-scene integer / float rows
    DevBuf<float> dist_rows_f;
    DevBuf<uint32_t> sub_idx;        // sharded frames: this rank's subset of the sort input (index, distance)
    DevBuf<int32_t> sub_dist;
    uint32_t uploaded_splats = 0;    // 'uploadedSplatCount' SortWorker.js:97
    uint32_t last_render_count = 0;
    bool have_sorted = false;
    bool ctl_dirty = true;           // SortControl needs k_sort_init (first sort / after a failed one); otherwise the sort leaves it clean

    // pinned staging (the shared-memory views of SortWorker.js:180-191)
    PinBuf<uint32_t> h_indexes, h_sorted;
    PinBuf<uint32_t> h_ctl;
    PinBuf<unsigned char> h_frame;

    // --- rasteriser state ---
    RasterState rs;

    gs_timings tm{};
    Profiler prof;
    // CUDA graph of one frame (sort + render), replayed while its shape key is unchanged
    cudaGraphExec_t graph_exec = nullptr;
    cudaStream_t stream2 = nullptr;  // second capture branch (projection beside the depth sort)
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    unsigned long long graph_key[8] = {0};
    bool graph_enabled = true;
    bool last_frame_was_graph = false;
    bool no_subset = false;          // gs_frame with sorted_out on a sharded engine needs the full order: replicated sort
    uint32_t graph_launches = 0;
    bool have_prof_begin = false;    // true while a frame's sort already opened the timeline
    bool pending_async = false;
    gs_render_params pending_rp{};
    DevBuf<uint32_t> flush;          // L2 flush scratch (bench hygiene)
    // SplatTree leaves (gs_upload_splat_tree) and the scratch of gs_gather_for_sort
    struct Tree {
        DevBuf<double> center, nmin, nmax;
        DevBuf<uint32_t> offsets, indexes, start;
        DevBuf<unsigned long long> key, total;
        uint32_t count = 0, splats = 0;
        // every node (gs_upload_splat_tree_nodes): the raycast's box tests
        DevBuf<double> all_min, all_max;
        DevBuf<int32_t> parent;
        DevBuf<uint32_t> leaf_node;
        uint32_t node_count = 0;
        bool have_nodes = false;     // nodes uploaded for the current leaves
    } tree;
    // gs_raycast: per-splat records (ray_records engines only) and the call's scratch, allocated on first use
    struct Ray {
        DevBuf<gs_ray_record> rec;
        bool valid = false;          // the records describe the current scene
        double xf[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};   // static mesh: the SplatScene transform
        DevBuf<RaySetup> setup;
        DevBuf<uint8_t> pass;
        DevBuf<uint32_t> reached, list, counts;
        DevBuf<RayHit> hits;
        DevBuf<uint32_t> keys[2], vals[4], tile_hist;
        DevBuf<SortControl> ctl;
        DevBuf<gs_ray_hit> out;
    } ray;
    // pipelined frames (gs_frame_begin / gs_frame_end): device frames alternate between two buffers, the D2H copy of frame i runs on
    // copy_stream while frame i+1 computes on `stream`
    cudaStream_t copy_stream = nullptr;
    // ring of per-frame events / host status slots (more entries than frames in flight); the DEVICE frame buffers stay two
    static constexpr int kPipeRing = 4, kPipeMaxInflight = 3;
    cudaEvent_t ev_frame_done[kPipeRing] = {nullptr}, ev_copy_done[kPipeRing] = {nullptr};
    // per-frame parameter blocks are double buffered by frame-buffer parity and uploaded on their own stream, and the frame's status words
    // are snapshotted by the blend kernel into a per-parity device slot that the copy stream reads: a pipelined frame then puts NO copy
    // operation on the compute stream (each small copy there costs a few microseconds of serialisation between two frame graphs)
    cudaStream_t param_stream = nullptr;
    cudaEvent_t ev_params[2] = {nullptr, nullptr};
    bool param_side = false;                       // upload_frame_params goes through param_stream (set by gs_frame_begin)
    bool graph_snapshot[2] = {false, false};       // the captured frame graph of this parity ends in a blend that writes the status snapshot
    DevBuf<uint32_t> status_dev;                   // 2 x kPipeSlotWords
    cudaGraphExec_t graph_exec_alt = nullptr;     // the same frame graph with the alternate frame buffer as target
    unsigned long long graph_key_alt[8] = {0};
    PinBuf<uint32_t> h_pipe;                       // kPipeRing slots x (SortControl head + RasterControl) read back per pipelined frame
    uint64_t pipe_begun = 0, pipe_ended = 0;       // frames begun / ended; in flight = the difference
    uint32_t pipe_inflight() const { return (uint32_t)(pipe_begun - pipe_ended); }

    // --- sort-only sharding by input position (shard_kernels.cuh) ---
    struct Shard {
        DevBuf<unsigned char> block;                 // ShardHeader + runs[R] (exported through CUDA IPC)
        DevBuf<uint32_t> total, ahead, block_total, delta, local_sorted;
        ShardPeers peers{};
        uint32_t *root_out = nullptr;                // rank 0's sortedIndexes as mapped here
        void *opened[kMaxShardRanks + 1] = {nullptr};// IPC mappings to close
        uint32_t world = 0, seq = 0;
        uint32_t pending_render_count = 0;
        bool attached = false, pending = false;
        bool pending_unsplit = false;                // the pending call was below the split threshold: rank 0 sorted alone
    } shard;

    // Releases what is not a buffer; the buffers then free themselves, on the device selected here.
    ~gs_engine() {
        cudaSetDevice(cfg.device);
        if (stream) cudaStreamSynchronize(stream);
        for (void *m : shard.opened) if (m) cudaIpcCloseMemHandle(m);
        if (rs.peer_attached) { if (rs.peer_frame) cudaIpcCloseMemHandle(rs.peer_frame); if (rs.peer_sync) cudaIpcCloseMemHandle(rs.peer_sync); }
        if (graph_exec) cudaGraphExecDestroy(graph_exec);
        if (graph_exec_alt) cudaGraphExecDestroy(graph_exec_alt);
        for (cudaEvent_t x : ev) if (x) cudaEventDestroy(x);
        for (int i = 0; i < kPipeRing; ++i) { if (ev_frame_done[i]) cudaEventDestroy(ev_frame_done[i]); if (ev_copy_done[i]) cudaEventDestroy(ev_copy_done[i]); }
        for (cudaEvent_t x : {ev_params[0], ev_params[1], ev_fork, ev_join}) if (x) cudaEventDestroy(x);
        for (cudaStream_t x : {stream, stream2, copy_stream, param_stream}) if (x) cudaStreamDestroy(x);
    }
};

static int check_engine(gs_engine *e) {
    if (!e) return fail(GS_ERR_BAD_ARG, "null engine");
    cudaError_t ce = cudaSetDevice(e->cfg.device);
    if (ce != cudaSuccess) return fail(GS_ERR_CUDA, "cudaSetDevice(%d) -> %s", e->cfg.device, cudaGetErrorString(ce));
    return GS_OK;
}

// A caller's versioned struct over `defaults`: its first struct_size bytes (0: all of it), no more than this library's struct holds.
template <typename T> static T read_options(const T *in, T defaults) {
    if (in) memcpy(&defaults, in, std::min<size_t>(in->struct_size ? in->struct_size : sizeof(T), sizeof(T)));
    return defaults;
}

extern "C" int gs_create(const gs_config *cfg, gs_engine **out) {
    if (!cfg || !out) return fail(GS_ERR_BAD_ARG, "gs_create: null argument");
    *out = nullptr;
    gs_config c = read_options(cfg, gs_config{});
    if (c.distance_map_range == 0) c.distance_map_range = 1u << 16; // Constants.DefaultSplatSortDistanceMapPrecision
    if (c.distance_map_range < 2 || c.distance_map_range > (1u << 24)) return fail(GS_ERR_BAD_ARG, "distance_map_range %u outside [2, 2^24]", c.distance_map_range);
    if (c.world_size == 0) { c.world_size = 1; c.rank = 0; }
    if (c.rank >= c.world_size) return fail(GS_ERR_BAD_ARG, "rank %u >= world_size %u", c.rank, c.world_size);
    int ndev = gs_device_count();
    if (ndev <= 0) return fail(GS_ERR_NO_DEVICE, "no CUDA device visible: libgsplat_b200 has no CPU path");
    if (c.device < 0 || c.device >= ndev) return fail(GS_ERR_BAD_ARG, "device %d not in [0,%d)", c.device, ndev);
    CU(cudaSetDevice(c.device));
    std::unique_ptr<gs_engine> e(new (std::nothrow) gs_engine());   // freed by every return before the end
    if (!e) return fail(GS_ERR_BAD_ARG, "out of host memory");
    e->cfg = c;
    cudaDeviceProp prop{};
    CU(cudaGetDeviceProperties(&prop, c.device));
    e->sm_count = prop.multiProcessorCount;
    if (prop.l2CacheSize > 0) e->l2_bytes = (size_t)prop.l2CacheSize;
    CU(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
    CU(cudaStreamCreateWithFlags(&e->stream2, cudaStreamNonBlocking));
    CU(cudaEventCreateWithFlags(&e->ev_fork, cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&e->ev_join, cudaEventDisableTiming));
    for (int i = 0; i < EV_COUNT; ++i) CU(cudaEventCreate(&e->ev[i]));
    int kb = 0;
    while ((1u << kb) < c.distance_map_range) ++kb;
    e->key_bits = kb;
    int rc = GS_OK;
    const size_t n = std::max<uint32_t>(c.max_splat_count, 1);
    if ((rc = e->centers.ensure(n)) || (rc = e->indexes.ensure(n)) || (rc = e->dist.ensure(n)) || (rc = e->sorted.ensure(n)) ||
        (rc = e->vals[0].ensure(n)) || (rc = e->vals[1].ensure(n)) || (rc = e->keys[0].ensure(n)) || (rc = e->keys[1].ensure(n)) ||
        (rc = e->ctl.ensure(1)) || (rc = e->depthp.ensure(2)) || (rc = e->transforms.ensure(16 * GS_MAX_SCENES)) || (rc = e->h_ctl.ensure(sizeof(SortControl) / 4 + 64 + sizeof(RasterControl) / 4 + sizeof(ShardHeader) / 4)))
        return rc;
    if (c.dynamic_mode && (rc = e->scene_idx.ensure(n))) return rc;
    if (c.ray_records && (rc = e->ray.rec.ensure(n))) return rc;
    if (e->scene_idx.p) CU(cudaMemsetAsync(e->scene_idx.p, 0, e->scene_idx.n * 4, e->stream));
    {   // identity transforms until the caller provides some
        std::vector<float> id(16 * GS_MAX_SCENES, 0.f);
        for (int s = 0; s < GS_MAX_SCENES; ++s) id[16 * s] = id[16 * s + 5] = id[16 * s + 10] = id[16 * s + 15] = 1.f;
        CU(cudaMemcpy(e->transforms.p, id.data(), id.size() * 4, cudaMemcpyHostToDevice));
    }
    CU(cudaMemset(e->ctl.p, 0, sizeof(SortControl)));
    rc = raster_init(e->rs, c, e->sm_count);
    if (rc) return fail(rc, "raster_init failed: %s", g_err);
    if ((rc = e->status_dev.ensure(2 * kPipeSlotWords))) return rc;
    CU(cudaMemset(e->status_dev.p, 0, 2 * kPipeSlotWords * 4));
    e->rs.snap_base = e->status_dev.p;
    e->rs.snap_stride = (uint32_t)kPipeSlotWords;
    e->rs.snap_sort_ctl = reinterpret_cast<const uint32_t *>(e->ctl.p);
    CU(cudaStreamSynchronize(e->stream));
    *out = e.release();
    return GS_OK;
}

extern "C" void gs_destroy(gs_engine *e) { delete e; }

extern "C" int gs_upload_centers(gs_engine *e, const void *centers, const uint32_t *sceneIndexes, uint32_t from, uint32_t count) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!centers && count) return fail(GS_ERR_BAD_ARG, "gs_upload_centers: null centers");
    if ((uint64_t)from + count > e->cfg.max_splat_count) return fail(GS_ERR_CAPACITY, "centres [%u,%u) exceed max_splat_count %u", from, from + count, e->cfg.max_splat_count);
    e->ray.valid = false;
    if (count) CU(cudaMemcpyAsync(e->centers.p + from, centers, (size_t)count * 16, cudaMemcpyHostToDevice, e->stream));
    if (e->cfg.dynamic_mode && sceneIndexes && count)
        CU(cudaMemcpyAsync(e->scene_idx.p + from, sceneIndexes, (size_t)count * 4, cudaMemcpyHostToDevice, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    e->uploaded_splats = from + count; // SortWorker.js:97
    return GS_OK;
}

// ---------------------------------------------------------------------------------------------------------------
template <int MODE>
static void launch_depth(bool identity, int blocks, cudaStream_t st, const uint32_t *idx, const void *centers, const void *pre,
                         const uint32_t *scene, const float *tr, const DepthParams *P, uint32_t s0, uint32_t rc, int32_t *dist, SortControl *ctl) {
    if (identity) gs_launch(k_depth<MODE, true>, blocks, kDepthThreads, 0, st, idx, centers, pre, scene, tr, P, s0, rc, dist, ctl);
    else gs_launch(k_depth<MODE, false>, blocks, kDepthThreads, 0, st, idx, centers, pre, scene, tr, P, s0, rc, dist, ctl);
}

// Distance pass (sorter.cpp:29-140) over positions [lo, hi) of the index list: dist[i] and the running min/max in the control block.
static int enqueue_depth(gs_engine *e, const uint32_t *d_indexes, const float *mvp, bool use_pre, uint32_t lo, uint32_t hi, bool capturing) {
    cudaStream_t st = e->stream;
    const uint32_t n = hi - lo;
    DepthParams P{};
    memcpy(P.mvp, mvp, 64);
    P.irow[0] = (int32_t)((double)mvp[2] * 1000.0);   // sorter.cpp:64 -- f64 product, truncation toward zero
    P.irow[1] = (int32_t)((double)mvp[6] * 1000.0);
    P.irow[2] = (int32_t)((double)mvp[10] * 1000.0);
    P.irow[3] = 1;
    P.frow[0] = mvp[2]; P.frow[1] = mvp[6]; P.frow[2] = mvp[10]; P.frow[3] = 0.f;
    if (!capturing) CU(cudaMemcpyAsync(e->depthp.p + e->rs.frame_parity, &P, sizeof(P), cudaMemcpyHostToDevice, st)); // pageable source: staged before return
    const bool integer = e->cfg.integer_based_sort, dyn = e->cfg.dynamic_mode;
    const int mode = use_pre ? (integer ? kIntPrecomputed : kFloatPrecomputed)
                             : (integer ? (dyn ? kIntDynamic : kIntStatic) : (dyn ? kFloatDynamic : kFloatStatic));
    const int dblocks = (int)std::max<uint64_t>(1, std::min<uint64_t>(((uint64_t)n + kDepthThreads * kDepthItems - 1) / (kDepthThreads * kDepthItems), (uint64_t)e->sm_count * 8));
    const bool identity = (d_indexes == nullptr);
    const void *pre = e->precomputed.p;
    switch (mode) {
        case kIntStatic: launch_depth<kIntStatic>(identity, dblocks, st, d_indexes, e->centers.p, pre, e->scene_idx.p, e->transforms.p, e->depthp.p + e->rs.frame_parity, lo, hi, e->dist.p, e->ctl.p); break;
        case kIntDynamic: launch_depth<kIntDynamic>(identity, dblocks, st, d_indexes, e->centers.p, pre, e->scene_idx.p, e->transforms.p, e->depthp.p + e->rs.frame_parity, lo, hi, e->dist.p, e->ctl.p); break;
        case kIntPrecomputed: launch_depth<kIntPrecomputed>(identity, dblocks, st, d_indexes, e->centers.p, pre, e->scene_idx.p, e->transforms.p, e->depthp.p + e->rs.frame_parity, lo, hi, e->dist.p, e->ctl.p); break;
        case kFloatStatic: launch_depth<kFloatStatic>(identity, dblocks, st, d_indexes, e->centers.p, pre, e->scene_idx.p, e->transforms.p, e->depthp.p + e->rs.frame_parity, lo, hi, e->dist.p, e->ctl.p); break;
        case kFloatDynamic: launch_depth<kFloatDynamic>(identity, dblocks, st, d_indexes, e->centers.p, pre, e->scene_idx.p, e->transforms.p, e->depthp.p + e->rs.frame_parity, lo, hi, e->dist.p, e->ctl.p); break;
        default: launch_depth<kFloatPrecomputed>(identity, dblocks, st, d_indexes, e->centers.p, pre, e->scene_idx.p, e->transforms.p, e->depthp.p + e->rs.frame_parity, lo, hi, e->dist.p, e->ctl.p); break;
    }
    return GS_OK;
}

// The sort proper, everything already on the device.  d_indexes == nullptr: identity.
static int sort_on_device(gs_engine *e, const uint32_t *d_indexes, const float *mvp, uint32_t sort_count, uint32_t render_count,
                          bool use_pre, bool write_buckets, bool capturing = false, bool subset = false, cudaEvent_t wait_for_rects = nullptr) {
    if (sort_count > render_count) return fail(GS_ERR_BAD_ARG, "sortCount %u > renderCount %u", sort_count, render_count);
    if (render_count > e->cfg.max_splat_count) return fail(GS_ERR_CAPACITY, "renderCount %u > max_splat_count %u", render_count, e->cfg.max_splat_count);
    cudaStream_t st = e->stream;
    const uint32_t s0 = render_count - sort_count, n = sort_count;
    const PassPlan pl = make_plan_bits(e->key_bits);
    uint32_t launches = 0;
    uint32_t stride = 0;
    int rc = e->tile_hist.ensure(radix_tile_hist_words(std::max(n, 1u), pl.npasses, &stride));
    if (rc) return rc;
    if (!capturing) CU(cudaEventRecord(e->ev[EV_SORT0], st));
    if (!e->have_prof_begin) e->prof.begin(st);
    if (e->ctl_dirty && !capturing) {   // first sort, or the previous one failed part-way; a completed sort leaves the block clean
        gs_launch(k_sort_init, 1, 256, 0, st, e->ctl.p);
        ++launches;
    }
    if (!capturing) e->ctl_dirty = true;
    if (s0 > 0) { gs_launch(k_copy_head, std::min<uint32_t>((s0 + 255) / 256, e->sm_count * 8), 256, 0, st, d_indexes, e->sorted.p, s0); ++launches; e->prof.mark("k_copy_head", st); }
    if (n > 0) {
        if ((rc = enqueue_depth(e, d_indexes, mvp, use_pre, s0, render_count, capturing))) return rc;
        const bool identity = (d_indexes == nullptr);
        ++launches;
        e->prof.mark("k_depth", st);
        if (!capturing) CU(cudaEventRecord(e->ev[EV_DEPTH], st));
        const uint32_t tiles = (n + kRadixTile - 1) / kRadixTile;
        const uint32_t R = e->cfg.distance_map_range;
        const uint32_t *vsrc = identity ? nullptr : d_indexes + s0;
        int vmode = identity ? kValIotaReversed : kValArrayReversed;
        int32_t *dist_sorted = e->dist.p + s0;
        const unsigned long long *n_dev = nullptr;
        if (subset) {   // this rank sorts only the splats that reach its tiles; bucketed with the GLOBAL min/max found by k_depth above
            if (wait_for_rects) CU(cudaStreamWaitEvent(st, wait_for_rects, 0));
            int rcs = raster_subset(e->rs, e->cfg, d_indexes, render_count, e->dist.p, e->sub_idx.p, e->sub_dist.p, st, e->prof, launches);
            if (rcs) return rcs;
            vsrc = e->sub_idx.p; vmode = kValArrayReversed;
            dist_sorted = e->sub_dist.p;
            n_dev = &e->rs.rctl.p->subset_count;
        }
        static const RadixNames names = {{"k_radix_hist[depth,0]", "k_radix_hist[depth,1]", "k_radix_hist[depth,2]", "k_radix_hist[depth,3]"},
                                         {"k_radix_scan[depth,0]", "k_radix_scan[depth,1]", "k_radix_scan[depth,2]", "k_radix_scan[depth,3]"},
                                         {"k_radix_scatter[depth,0]", "k_radix_scatter[depth,1]", "k_radix_scatter[depth,2]", "k_radix_scatter[depth,3]"}};
        if (e->key_bits <= 16) {
            gs_launch(k_bucket<uint16_t>, tiles, kRadixThreads, 0, st, dist_sorted, (uint16_t *)e->keys[0].p, n, n_dev, R, pl, write_buckets ? 1 : 0, e->ctl.p, e->tile_hist.p, stride);
            ++launches;
            e->prof.mark("k_bucket", st);
            if (!capturing) CU(cudaEventRecord(e->ev[EV_BUCKET], st));
            radix_sort_pairs<uint16_t, uint32_t>((uint16_t *)e->keys[0].p, (uint16_t *)e->keys[1].p, vsrc, render_count - 1u, vmode, e->vals[0].p, e->vals[1].p,
                                       e->sorted.p + s0, n, n_dev, (unsigned long long)n, pl, e->ctl.p, e->tile_hist.p, stride, true, nullptr, st, launches, &e->prof, names, true);
        } else {
            gs_launch(k_bucket<uint32_t>, tiles, kRadixThreads, 0, st, dist_sorted, e->keys[0].p, n, n_dev, R, pl, write_buckets ? 1 : 0, e->ctl.p, e->tile_hist.p, stride);
            ++launches;
            e->prof.mark("k_bucket", st);
            if (!capturing) CU(cudaEventRecord(e->ev[EV_BUCKET], st));
            radix_sort_pairs<uint32_t, uint32_t>(e->keys[0].p, e->keys[1].p, vsrc, render_count - 1u, vmode, e->vals[0].p, e->vals[1].p, e->sorted.p + s0, n,
                                       n_dev, (unsigned long long)n, pl, e->ctl.p, e->tile_hist.p, stride, true, nullptr, st, launches, &e->prof, names, true);
        }
    } else if (!capturing) {
        CU(cudaEventRecord(e->ev[EV_DEPTH], st));
        CU(cudaEventRecord(e->ev[EV_BUCKET], st));
    }
    if (!capturing) CU(cudaEventRecord(e->ev[EV_SORT1], st));
    CU(cudaGetLastError());
    e->tm.kernel_launches = launches;
    e->last_render_count = render_count;
    e->have_sorted = true;
    if (!capturing) e->ctl_dirty = false;
    return GS_OK;
}

// after a stream sync: fold the device-side error bits and stage timings into the engine
static int finish_sort(gs_engine *e, float *sort_time_ms) {
    CU(cudaMemcpyAsync(e->h_ctl.p, e->ctl.p, 12, cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    float ms = 0.f;
    if (e->last_frame_was_graph) {   // one graph launch: only the whole-frame time is observable
        e->tm.depth_ms = e->tm.bucket_ms = e->tm.scatter_ms = 0.f;
        cudaEventElapsedTime(&ms, e->ev[EV_SORT0], e->ev[EV_R1]);
    } else {
        cudaEventElapsedTime(&e->tm.depth_ms, e->ev[EV_SORT0], e->ev[EV_DEPTH]);
        cudaEventElapsedTime(&e->tm.bucket_ms, e->ev[EV_DEPTH], e->ev[EV_BUCKET]);
        cudaEventElapsedTime(&e->tm.scatter_ms, e->ev[EV_BUCKET], e->ev[EV_SORT1]);
        cudaEventElapsedTime(&ms, e->ev[EV_SORT0], e->ev[EV_SORT1]);
    }
    e->tm.sort_total_ms = ms;
    if (sort_time_ms) *sort_time_ms = ms;
    const uint32_t err = e->h_ctl.p[2];
    if (err & kErrBucketRange) return fail(GS_ERR_BUCKET_RANGE, "a bucket index fell outside [0,%u): distances overflow the int32/f32 range map", e->cfg.distance_map_range);
    return GS_OK;
}

static int stage_sort_inputs(gs_engine *e, const gs_sort_params *p, const uint32_t **d_indexes) {
    cudaStream_t st = e->stream;
    *d_indexes = nullptr;
    CU(cudaEventRecord(e->ev[EV_H2D0], st));
    if (p->indexes_to_sort_dev) *d_indexes = p->indexes_to_sort_dev;
    else if (p->indexes_to_sort) {
        CU(cudaMemcpyAsync(e->indexes.p, p->indexes_to_sort, (size_t)p->render_count * 4, cudaMemcpyHostToDevice, st));
        *d_indexes = e->indexes.p;
    }
    if (e->cfg.dynamic_mode && p->transforms) CU(cudaMemcpyAsync(e->transforms.p, p->transforms, 16 * GS_MAX_SCENES * 4, cudaMemcpyHostToDevice, st));
    if (p->use_precomputed_distances) {
        if (!p->precomputed_distances) return fail(GS_ERR_BAD_ARG, "use_precomputed_distances without precomputed_distances");
        int rc = e->precomputed.ensure(e->cfg.max_splat_count);
        if (rc) return rc;
        CU(cudaMemcpyAsync(e->precomputed.p, p->precomputed_distances, (size_t)e->uploaded_splats * 4, cudaMemcpyHostToDevice, st));
    }
    CU(cudaEventRecord(e->ev[EV_H2D1], st));
    return GS_OK;
}

extern "C" int gs_sort(gs_engine *e, const gs_sort_params *p, uint32_t *sorted_out, float *sort_time_ms) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!p) return fail(GS_ERR_BAD_ARG, "gs_sort: null params");
    // SortWorker.js:99-100: counts are clamped to what has been uploaded
    gs_sort_params q = *p;
    q.render_count = std::min(q.render_count, e->uploaded_splats);
    q.sort_count = std::min(q.sort_count, e->uploaded_splats);
    if (q.sort_count > q.render_count) return fail(GS_ERR_BAD_ARG, "sortCount %u > renderCount %u", q.sort_count, q.render_count);
    const uint32_t *d_idx = nullptr;
    e->last_frame_was_graph = false;
    if ((rc = stage_sort_inputs(e, &q, &d_idx))) return rc;
    if ((rc = sort_on_device(e, d_idx, q.model_view_proj, q.sort_count, q.render_count, q.use_precomputed_distances != 0, false))) return rc;
    CU(cudaEventRecord(e->ev[EV_D2H0], e->stream));
    if (sorted_out && q.render_count) CU(cudaMemcpyAsync(sorted_out, e->sorted.p, (size_t)q.render_count * 4, cudaMemcpyDeviceToHost, e->stream));
    CU(cudaEventRecord(e->ev[EV_D2H1], e->stream));
    rc = finish_sort(e, sort_time_ms);
    cudaEventElapsedTime(&e->tm.h2d_ms, e->ev[EV_H2D0], e->ev[EV_H2D1]);
    cudaEventElapsedTime(&e->tm.d2h_ms, e->ev[EV_D2H0], e->ev[EV_D2H1]);
    return rc;
}


// ---------------------------------------------------------------------------------------------------------------
// Sort-only on N GPUs (SURVEY.md 8(e) "depth + sort"): rank g sorts the input positions [lo_g, hi_g) of the sort window and the
// ranks assemble the reference's global order in rank 0's sortedIndexes over peer memory.  See shard_kernels.cuh.
static int shard_prepare(gs_engine *e) {
    const uint32_t R = e->cfg.distance_map_range;
    int rc;
    const size_t bytes = sizeof(ShardHeader) + (size_t)R * sizeof(uint2);
    if (e->shard.block.n < bytes) {
        if ((rc = e->shard.block.ensure(bytes))) return rc;
        CU(cudaMemset(e->shard.block.p, 0, bytes));
    }
    const size_t blocks = ((size_t)R + kShardScanThreads - 1) / kShardScanThreads;
    if ((rc = e->shard.total.ensure(R)) || (rc = e->shard.ahead.ensure(R)) || (rc = e->shard.delta.ensure(R)) || (rc = e->shard.block_total.ensure(blocks)) ||
        (rc = e->shard.local_sorted.ensure(e->cfg.max_splat_count)))
        return rc;
    // everything the per-sort path could otherwise grow (cudaFree synchronises the device: not while a peer's wait kernel may be spinning)
    const PassPlan pl = make_plan_bits(e->key_bits);
    if ((rc = e->tile_hist.ensure(radix_tile_hist_words(std::max(e->cfg.max_splat_count, 1u), pl.npasses, nullptr))) || (rc = e->precomputed.ensure(e->cfg.max_splat_count))) return rc;
    return GS_OK;
}
// CUDA loads a kernel's code on its first launch (lazy module loading) and that load can wait for running kernels to finish.  The
// sharded sort keeps bounded spin-wait kernels in flight while the host enqueues the rest of the chain, so every kernel of the chain
// is loaded up front (cudaFuncGetAttributes forces the load); otherwise a first sort could stall on its own wait kernel.
template <typename F> static inline void preload_kernel(F f) { cudaFuncAttributes a; (void)cudaFuncGetAttributes(&a, f); }
template <typename KeyT> static void shard_preload_keyed() {
    preload_kernel(k_bucket<KeyT>);
    preload_kernel(k_radix_hist<KeyT>);
    preload_kernel(k_shard_place<KeyT>);
    preload_kernel(k_radix_scatter<KeyT, uint32_t, kValArray, true, false>);
    preload_kernel(k_radix_scatter<KeyT, uint32_t, kValArrayReversed, true, false>);
    preload_kernel(k_radix_scatter<KeyT, uint32_t, kValIotaReversed, true, false>);
    preload_kernel(k_radix_scatter<KeyT, uint32_t, kValArray, true, true>);
    preload_kernel(k_radix_scatter<KeyT, uint32_t, kValArrayReversed, true, true>);
    preload_kernel(k_radix_scatter<KeyT, uint32_t, kValIotaReversed, true, true>);
}
template <int MODE> static void shard_preload_depth() { preload_kernel(k_depth<MODE, true>); preload_kernel(k_depth<MODE, false>); }
static void shard_preload(gs_engine *e) {
    preload_kernel(k_sort_init); preload_kernel(k_copy_head); preload_kernel(k_radix_scan);
    preload_kernel(k_shard_exchange_minmax); preload_kernel(k_shard_exchange_runs); preload_kernel(k_shard_totals); preload_kernel(k_shard_delta); preload_kernel(k_shard_done);
    shard_preload_depth<kIntStatic>(); shard_preload_depth<kIntDynamic>(); shard_preload_depth<kIntPrecomputed>();
    shard_preload_depth<kFloatStatic>(); shard_preload_depth<kFloatDynamic>(); shard_preload_depth<kFloatPrecomputed>();
    if (e->key_bits <= 16) shard_preload_keyed<uint16_t>(); else shard_preload_keyed<uint32_t>();
    (void)cudaGetLastError();
}
static inline ShardHeader *shard_hdr(void *block) { return (ShardHeader *)block; }
static inline const uint2 *shard_runs(void *block) { return (const uint2 *)((unsigned char *)block + sizeof(ShardHeader)); }

extern "C" int gs_shard_export(gs_engine *e, void *block_handle, void *sorted_handle) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!block_handle || !sorted_handle) return fail(GS_ERR_BAD_ARG, "gs_shard_export: null");
    if ((rc = shard_prepare(e))) return rc;
    cudaIpcMemHandle_t h;
    CU(cudaIpcGetMemHandle(&h, e->shard.block.p));
    memcpy(block_handle, &h, sizeof(h));
    CU(cudaIpcGetMemHandle(&h, e->sorted.p));
    memcpy(sorted_handle, &h, sizeof(h));
    return GS_OK;
}
static int shard_bind(gs_engine *e, uint32_t world, void *const *blocks, uint32_t *root_out) {
    for (uint32_t g = 0; g < world; ++g) {
        e->shard.peers.hdr[g] = shard_hdr(blocks[g]);
        e->shard.peers.runs[g] = shard_runs(blocks[g]);
    }
    shard_preload(e);
    e->shard.root_out = root_out;
    e->shard.world = world;
    e->shard.seq = 0;
    e->shard.attached = true;
    return GS_OK;
}
static int shard_check_group(gs_engine *e, uint32_t world, const char *who) {
    if (world < 1 || world > (uint32_t)kMaxShardRanks) return fail(GS_ERR_BAD_ARG, "%s: world %u outside [1, %d]", who, world, kMaxShardRanks);
    if (e->cfg.world_size != world || e->cfg.rank >= world) return fail(GS_ERR_BAD_ARG, "%s: engine was created as rank %u of %u, not of %u", who, e->cfg.rank, e->cfg.world_size, world);
    return GS_OK;
}
extern "C" int gs_shard_attach(gs_engine *e, uint32_t world, const void *block_handles, const void *root_sorted_handle) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!block_handles || !root_sorted_handle) return fail(GS_ERR_BAD_ARG, "gs_shard_attach: null");
    if ((rc = shard_check_group(e, world, "gs_shard_attach")) || (rc = shard_prepare(e))) return rc;
    void *blocks[kMaxShardRanks] = {nullptr};
    for (uint32_t g = 0; g < world; ++g) {
        if (g == e->cfg.rank) { blocks[g] = e->shard.block.p; continue; }
        cudaIpcMemHandle_t h;
        memcpy(&h, (const unsigned char *)block_handles + (size_t)g * GS_IPC_HANDLE_BYTES, sizeof(h));
        CU(cudaIpcOpenMemHandle(&blocks[g], h, cudaIpcMemLazyEnablePeerAccess));
        e->shard.opened[g] = blocks[g];
    }
    uint32_t *root_out = e->sorted.p;
    if (e->cfg.rank != 0) {
        cudaIpcMemHandle_t h;
        void *m = nullptr;
        memcpy(&h, root_sorted_handle, sizeof(h));
        CU(cudaIpcOpenMemHandle(&m, h, cudaIpcMemLazyEnablePeerAccess));
        e->shard.opened[kMaxShardRanks] = m;
        root_out = (uint32_t *)m;
    }
    return shard_bind(e, world, blocks, root_out);
}
// Same process, same device (several engines sharing one GPU, or a test without a second GPU): plain pointers instead of IPC mappings.
extern "C" int gs_shard_attach_local(gs_engine *e, uint32_t world, gs_engine *const *engines) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!engines) return fail(GS_ERR_BAD_ARG, "gs_shard_attach_local: null");
    if ((rc = shard_check_group(e, world, "gs_shard_attach_local"))) return rc;
    void *blocks[kMaxShardRanks] = {nullptr};
    for (uint32_t g = 0; g < world; ++g) {
        gs_engine *pe = engines[g];
        if (!pe || pe->cfg.device != e->cfg.device || pe->cfg.rank != g || pe->cfg.world_size != world ||
            pe->cfg.distance_map_range != e->cfg.distance_map_range)
            return fail(GS_ERR_BAD_ARG, "gs_shard_attach_local: engines[%u] must be rank %u of %u on device %d with the same distance_map_range", g, g, world, e->cfg.device);
        if ((rc = shard_prepare(pe))) return rc;
        blocks[g] = pe->shard.block.p;
    }
    return shard_bind(e, world, blocks, engines[0]->sorted.p);
}

template <typename KeyT>
static int shard_local_sort(gs_engine *e, const uint32_t *d_indexes, uint32_t s0, uint32_t lo, uint32_t hi, uint32_t &launches) {
    cudaStream_t st = e->stream;
    const uint32_t n = hi - lo, R = e->cfg.distance_map_range;
    const PassPlan pl = make_plan_bits(e->key_bits);
    uint32_t stride = 0;
    int rc = e->tile_hist.ensure(radix_tile_hist_words(std::max(n, 1u), pl.npasses, &stride));
    if (rc) return rc;
    const bool identity = (d_indexes == nullptr);
    static const RadixNames names = {{"k_radix_hist[shard,0]", "k_radix_hist[shard,1]", "k_radix_hist[shard,2]", "k_radix_hist[shard,3]"},
                                     {"k_radix_scan[shard,0]", "k_radix_scan[shard,1]", "k_radix_scan[shard,2]", "k_radix_scan[shard,3]"},
                                     {"k_radix_scatter[shard,0]", "k_radix_scatter[shard,1]", "k_radix_scatter[shard,2]", "k_radix_scatter[shard,3]"}};
    const uint32_t me = e->cfg.rank, world = e->shard.world, seq = e->shard.seq;
    uint2 *runs = (uint2 *)shard_runs(e->shard.block.p);
    KeyT *final_keys = nullptr;
    if (n) {   // slice -> keys with the GLOBAL range map -> local order + per-key runs of that order
        const uint32_t tiles = (n + kRadixTile - 1) / kRadixTile;
        gs_launch(k_bucket<KeyT>, tiles, kRadixThreads, 0, st, e->dist.p + lo, (KeyT *)e->keys[0].p, n, nullptr, R, pl, 0, e->ctl.p, e->tile_hist.p, stride);
        ++launches;
        e->prof.mark("k_bucket", st);
        radix_sort_pairs<KeyT, uint32_t>((KeyT *)e->keys[0].p, (KeyT *)e->keys[1].p, identity ? nullptr : d_indexes + lo, hi - 1u,
                                         identity ? kValIotaReversed : kValArrayReversed, e->vals[0].p, e->vals[1].p, e->shard.local_sorted.p, n, nullptr,
                                         (unsigned long long)n, pl, e->ctl.p, e->tile_hist.p, stride, true, runs, st, launches, &e->prof, names, true, true, &final_keys);
    }
    // C2: publish my runs, wait for everybody's, turn them into the offsets of my runs in the global order
    k_shard_exchange_runs<<<1, 32, 0, st>>>(e->shard.peers, me, world, seq);
    ++launches;
    e->prof.mark("k_shard_exchange_runs", st);
    if (n) {
        const uint32_t sblocks = (R + kShardScanThreads - 1) / kShardScanThreads;
        k_shard_totals<<<sblocks, kShardScanThreads, 0, st>>>(e->shard.peers, me, world, R, e->shard.total.p, e->shard.ahead.p, e->shard.block_total.p);
        k_shard_delta<<<sblocks, kShardScanThreads, 0, st>>>(runs, R, e->shard.total.p, e->shard.ahead.p, e->shard.block_total.p, e->shard.delta.p);
        e->prof.mark("k_shard_offsets", st);
        k_shard_place<KeyT><<<std::min<uint32_t>((n + 255) / 256, e->sm_count * 16), 256, 0, st>>>(final_keys, e->shard.local_sorted.p, n, e->shard.delta.p, e->shard.root_out + s0);
        e->prof.mark("k_shard_place", st);
        launches += 3;
    }
    return GS_OK;
}

// Position slice of rank g: [sortStart + n*g/G, sortStart + n*(g+1)/G)
static inline uint32_t shard_bound(uint32_t s0, uint32_t n, uint32_t g, uint32_t world) { return s0 + (uint32_t)(((uint64_t)n * g) / world); }

extern "C" int gs_sort_sharded_async(gs_engine *e, const gs_sort_params *p) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!p) return fail(GS_ERR_BAD_ARG, "gs_sort_sharded: null params");
    if (!e->shard.attached) return fail(GS_ERR_NOT_READY, "gs_sort_sharded: call gs_shard_attach (or gs_shard_attach_local) first");
    if (e->shard.pending) return fail(GS_ERR_NOT_READY, "gs_sort_sharded_async: the previous sharded sort has not been finished");
    gs_sort_params q = *p;
    q.render_count = std::min(q.render_count, e->uploaded_splats);   // SortWorker.js:99-100
    q.sort_count = std::min(q.sort_count, e->uploaded_splats);
    if (q.sort_count > q.render_count) return fail(GS_ERR_BAD_ARG, "sortCount %u > renderCount %u", q.sort_count, q.render_count);
    const uint32_t *d_idx = nullptr;
    e->last_frame_was_graph = false;
    const uint32_t me = e->cfg.rank, world = e->shard.world;
    // The split pays only for large windows (DESIGN.md 6.1: three NVLink handshakes + offsets + placement vs a single sort that is
    // latency bound below ~8 M splats).  Smaller calls are sorted by rank 0 alone; the decision depends only on the call's arguments,
    // so every rank takes the same branch.  GS_SHARD_MIN overrides the threshold (0 = always split).
    uint32_t split_min = 8000000u;
    if (const char *sv = getenv("GS_SHARD_MIN")) split_min = (uint32_t)strtoul(sv, nullptr, 10);
    if (world == 1 || q.sort_count < split_min) {
        e->shard.pending = true;
        e->shard.pending_unsplit = true;
        e->shard.pending_render_count = q.render_count;
        if (me != 0) return GS_OK;
        if ((rc = stage_sort_inputs(e, &q, &d_idx)) ||
            (rc = sort_on_device(e, d_idx, q.model_view_proj, q.sort_count, q.render_count, q.use_precomputed_distances != 0, false))) {
            e->shard.pending = false;
            return rc;
        }
        return GS_OK;
    }
    e->shard.pending_unsplit = false;
    if ((rc = stage_sort_inputs(e, &q, &d_idx))) return rc;
    cudaStream_t st = e->stream;
    const uint32_t s0 = q.render_count - q.sort_count;
    const uint32_t lo = shard_bound(s0, q.sort_count, me, world), hi = shard_bound(s0, q.sort_count, me + 1, world);
    const uint32_t seq = ++e->shard.seq;
    uint32_t launches = 0;
    CU(cudaEventRecord(e->ev[EV_SORT0], st));
    e->prof.begin(st);
    if (e->ctl_dirty) { gs_launch(k_sort_init, 1, 256, 0, st, e->ctl.p); ++launches; }
    e->ctl_dirty = true;
    if (me == 0 && s0 > 0) { gs_launch(k_copy_head, std::min<uint32_t>((s0 + 255) / 256, e->sm_count * 8), 256, 0, st, d_idx, e->sorted.p, s0); ++launches; e->prof.mark("k_copy_head", st); }
    if (hi > lo) {
        if ((rc = enqueue_depth(e, d_idx, q.model_view_proj, q.use_precomputed_distances != 0, lo, hi, false))) return rc;
        ++launches;
        e->prof.mark("k_depth", st);
    }
    // C1: global min/max over peer memory
    k_shard_exchange_minmax<<<1, kShardSyncThreads, 0, st>>>(e->shard.peers, e->ctl.p, me, world, seq, hi > lo ? 0 : 1, (uint2 *)shard_runs(e->shard.block.p),
                                                             e->cfg.distance_map_range);
    ++launches;
    e->prof.mark("k_shard_exchange_minmax", st);
    CU(cudaEventRecord(e->ev[EV_DEPTH], st));
    CU(cudaEventRecord(e->ev[EV_BUCKET], st));
    rc = (e->key_bits <= 16) ? shard_local_sort<uint16_t>(e, d_idx, s0, lo, hi, launches) : shard_local_sort<uint32_t>(e, d_idx, s0, lo, hi, launches);
    if (rc) return rc;
    k_shard_done<<<1, 32, 0, st>>>(e->shard.peers, me, world, seq);
    ++launches;
    e->prof.mark("k_shard_done", st);
    CU(cudaEventRecord(e->ev[EV_SORT1], st));
    CU(cudaGetLastError());
    e->tm.kernel_launches = launches;
    e->last_render_count = q.render_count;
    e->have_sorted = (me == 0);     // the assembled order lives in rank 0's sortedIndexes
    e->ctl_dirty = !(hi > lo);      // an empty slice ran no final radix pass, which is what re-seeds the control block
    e->shard.pending = true;
    e->shard.pending_render_count = q.render_count;
    return GS_OK;
}

extern "C" int gs_sort_sharded_finish(gs_engine *e, uint32_t *sorted_out, float *sort_time_ms) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!e->shard.pending) return fail(GS_ERR_NOT_READY, "gs_sort_sharded_finish: nothing pending");
    e->shard.pending = false;
    const uint32_t rcnt = e->shard.pending_render_count;
    if (e->shard.pending_unsplit && e->cfg.rank != 0) {   // rank 0 sorted alone
        if (sort_time_ms) *sort_time_ms = 0.f;
        return GS_OK;
    }
    CU(cudaEventRecord(e->ev[EV_D2H0], e->stream));
    if (sorted_out && rcnt && e->cfg.rank == 0) CU(cudaMemcpyAsync(sorted_out, e->sorted.p, (size_t)rcnt * 4, cudaMemcpyDeviceToHost, e->stream));
    CU(cudaEventRecord(e->ev[EV_D2H1], e->stream));
    if (e->shard.pending_unsplit) {
        rc = finish_sort(e, sort_time_ms);
        cudaEventElapsedTime(&e->tm.h2d_ms, e->ev[EV_H2D0], e->ev[EV_H2D1]);
        cudaEventElapsedTime(&e->tm.d2h_ms, e->ev[EV_D2H0], e->ev[EV_D2H1]);
        return rc;
    }
    CU(cudaMemcpyAsync(e->h_ctl.p + 640, e->shard.block.p, sizeof(ShardHeader), cudaMemcpyDeviceToHost, e->stream));
    rc = finish_sort(e, sort_time_ms);
    cudaEventElapsedTime(&e->tm.h2d_ms, e->ev[EV_H2D0], e->ev[EV_H2D1]);
    cudaEventElapsedTime(&e->tm.d2h_ms, e->ev[EV_D2H0], e->ev[EV_D2H1]);
    ShardHeader hd;
    memcpy(&hd, e->h_ctl.p + 640, sizeof(hd));
    if (hd.timeout) {
        cudaMemsetAsync(&shard_hdr(e->shard.block.p)->timeout, 0, 4, e->stream);
        e->ctl_dirty = true;
        return fail(GS_ERR_CUDA, "sharded sort: a peer rank did not reach the exchange within the time limit (are all %u ranks calling gs_sort_sharded?)", e->shard.world);
    }
    return rc;
}

extern "C" int gs_sort_sharded(gs_engine *e, const gs_sort_params *p, uint32_t *sorted_out, float *sort_time_ms) {
    int rc = gs_sort_sharded_async(e, p);
    if (rc) return rc;
    return gs_sort_sharded_finish(e, sorted_out, sort_time_ms);
}

// ---------------------------------------------------------------------------------------------------------------
// Stateless drop-in (sorter.cpp:17-22).  A private engine per (device 0, splatCount, mode, range) is cached so repeated
// calls do not re-allocate; inputs are uploaded on every call like a non-shared-memory worker copies them
// (SortWorker.js:35-51).
static gs_engine *g_dropin = nullptr;
#include <mutex>
static std::mutex g_dropin_mutex;   // the stateless entry shares one cached engine: calls are serialised, not rejected

extern "C" void gs_dropin_release(void) {
    std::lock_guard<std::mutex> lock(g_dropin_mutex);
    if (g_dropin) { gs_destroy(g_dropin); g_dropin = nullptr; }
}

extern "C" int gs_sort_indexes(const uint32_t *indexes, const void *centers, const void *precomputedDistances, int32_t *mappedDistances,
                               uint32_t *frequencies, const float *modelViewProj, uint32_t *indexesOut, const uint32_t *sceneIndexes,
                               const float *transforms, uint32_t distanceMapRange, uint32_t sortCount, uint32_t renderCount,
                               uint32_t splatCount, bool usePrecomputedDistances, bool useIntegerSort, bool dynamicMode) {
    if (!indexes || !modelViewProj || !indexesOut) return fail(GS_ERR_BAD_ARG, "gs_sort_indexes: null indexes/modelViewProj/indexesOut");
    if (!usePrecomputedDistances && !centers) return fail(GS_ERR_BAD_ARG, "gs_sort_indexes: null centers");
    if (usePrecomputedDistances && !precomputedDistances) return fail(GS_ERR_BAD_ARG, "gs_sort_indexes: null precomputedDistances");
    if (dynamicMode && !usePrecomputedDistances && (!sceneIndexes || !transforms)) return fail(GS_ERR_BAD_ARG, "gs_sort_indexes: dynamic mode needs sceneIndexes and transforms");
    if (sortCount > renderCount || renderCount > splatCount) return fail(GS_ERR_BAD_ARG, "need sortCount <= renderCount <= splatCount");
    if (distanceMapRange < 2 || distanceMapRange > (1u << 24)) return fail(GS_ERR_BAD_ARG, "distanceMapRange %u outside [2, 2^24]", distanceMapRange);
    std::lock_guard<std::mutex> lock(g_dropin_mutex);
    int cur_dev = 0;
    if (cudaGetDevice(&cur_dev) != cudaSuccess) { cudaGetLastError(); cur_dev = 0; }     // the caller's current device, like any CUDA library
    gs_engine *e = g_dropin;
    if (!e || e->cfg.device != cur_dev || e->cfg.max_splat_count < splatCount || e->cfg.distance_map_range != distanceMapRange ||
        (bool)e->cfg.integer_based_sort != useIntegerSort || (bool)e->cfg.dynamic_mode != dynamicMode) {
        if (e) gs_destroy(e);
        g_dropin = nullptr;
        gs_config c{};
        c.struct_size = sizeof(c);
        c.device = cur_dev;
        c.max_splat_count = std::max(splatCount, 1u);
        c.distance_map_range = distanceMapRange;
        c.integer_based_sort = useIntegerSort;
        c.dynamic_mode = dynamicMode;
        int rc = gs_create(&c, &e);
        if (rc) return rc;
        g_dropin = e;
    }
    int rc = check_engine(e);
    if (rc) return rc;
    cudaStream_t st = e->stream;
    if (centers && splatCount) CU(cudaMemcpyAsync(e->centers.p, centers, (size_t)splatCount * 16, cudaMemcpyHostToDevice, st));
    if (dynamicMode && sceneIndexes && splatCount) CU(cudaMemcpyAsync(e->scene_idx.p, sceneIndexes, (size_t)splatCount * 4, cudaMemcpyHostToDevice, st));
    if (dynamicMode && transforms) CU(cudaMemcpyAsync(e->transforms.p, transforms, 16 * GS_MAX_SCENES * 4, cudaMemcpyHostToDevice, st));
    if (usePrecomputedDistances) {
        if ((rc = e->precomputed.ensure(e->cfg.max_splat_count))) return rc;
        CU(cudaMemcpyAsync(e->precomputed.p, precomputedDistances, (size_t)splatCount * 4, cudaMemcpyHostToDevice, st));
    }
    if (renderCount) CU(cudaMemcpyAsync(e->indexes.p, indexes, (size_t)renderCount * 4, cudaMemcpyHostToDevice, st));
    e->uploaded_splats = splatCount;
    e->last_frame_was_graph = false;
    const bool want_scratch = (mappedDistances != nullptr) || (frequencies != nullptr);
    if ((rc = sort_on_device(e, e->indexes.p, modelViewProj, sortCount, renderCount, usePrecomputedDistances, want_scratch))) return rc;
    // wasm-trap emulation: results are only written back when the device reported no range error
    if ((rc = finish_sort(e, nullptr))) return rc;
    if (renderCount) CU(cudaMemcpyAsync(indexesOut, e->sorted.p, (size_t)renderCount * 4, cudaMemcpyDeviceToHost, st));
    const uint32_t s0 = renderCount - sortCount;
    if (mappedDistances && sortCount) CU(cudaMemcpyAsync(mappedDistances + s0, e->dist.p + s0, (size_t)sortCount * 4, cudaMemcpyDeviceToHost, st));
    if (frequencies) {
        if ((rc = e->freq.ensure(distanceMapRange))) return rc;
        CU(cudaMemsetAsync(e->freq.p, 0, (size_t)distanceMapRange * 4, st));
        if (sortCount) k_bucket_counts<<<std::min<uint32_t>((sortCount + 255) / 256, e->sm_count * 8), 256, 0, st>>>(e->dist.p, s0, renderCount, e->freq.p);
        k_exclusive_scan_single_block<<<1, 1024, 0, st>>>(e->freq.p, distanceMapRange);
        CU(cudaMemcpyAsync(frequencies, e->freq.p, (size_t)distanceMapRange * 4, cudaMemcpyDeviceToHost, st));
    }
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    return GS_OK;
}

extern "C" void sortIndexes(unsigned int *indexes, void *centers, void *precomputedDistances, int *mappedDistances,
                            unsigned int *frequencies, float *modelViewProj, unsigned int *indexesOut, unsigned int *sceneIndexes,
                            float *transforms, unsigned int distanceMapRange, unsigned int sortCount, unsigned int renderCount,
                            unsigned int splatCount, bool usePrecomputedDistances, bool useIntegerSort, bool dynamicMode) {
    (void)gs_sort_indexes(indexes, centers, precomputedDistances, mappedDistances, frequencies, modelViewProj, indexesOut, sceneIndexes,
                          transforms, distanceMapRange, sortCount, renderCount, splatCount, usePrecomputedDistances, useIntegerSort, dynamicMode);
}

// ---------------------------------------------------------------------------------------------------------------
// D1: SplatMesh.computeDistancesOnGPU.  mvp is f64 because three.js Matrix4 elements are JS numbers and the integer rows
// are Math.round(element * 1000) on those doubles (SplatMesh.js:2057-2064).
extern "C" int gs_compute_distances(gs_engine *e, const double *mvp, const double *scene_transforms, uint32_t count, void *out) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!mvp || !out) return fail(GS_ERR_BAD_ARG, "gs_compute_distances: null argument");
    if (count > e->uploaded_splats) return fail(GS_ERR_CAPACITY, "count %u > uploaded splats %u", count, e->uploaded_splats);
    const bool integer = e->cfg.integer_based_sort, dyn = e->cfg.dynamic_mode;
    if (dyn && !scene_transforms) return fail(GS_ERR_BAD_ARG, "dynamic mode needs scene_transforms (f64[16*32])");
    std::vector<int32_t> irows(4 * GS_MAX_SCENES, 0);
    std::vector<float> frows(4 * GS_MAX_SCENES, 0.f);
    auto jsround = [](double v) { return (int32_t)std::floor(v + 0.5); }; // Math.round
    for (int s = 0; s < (dyn ? GS_MAX_SCENES : 1); ++s) {
        double m[16];
        if (dyn) { // tempMatrix = mvp * transform_s (three.js Matrix4.multiply, f64)   SplatMesh.js:1722-1724
            const double *t = scene_transforms + 16 * s;
            for (int c = 0; c < 4; ++c)
                for (int r = 0; r < 4; ++r) m[4 * c + r] = mvp[r] * t[4 * c] + mvp[4 + r] * t[4 * c + 1] + mvp[8 + r] * t[4 * c + 2] + mvp[12 + r] * t[4 * c + 3];
        } else memcpy(m, mvp, sizeof(m));
        for (int k = 0; k < 4; ++k) {
            irows[4 * s + k] = jsround(m[2 + 4 * k] * 1000.0);
            frows[4 * s + k] = (float)m[2 + 4 * k];
        }
    }
    DevBuf<int32_t> &d_ir = e->dist_rows_i;   // engine-owned: repeated calls allocate nothing
    DevBuf<float> &d_fr = e->dist_rows_f;
    if ((rc = d_ir.ensure(irows.size())) || (rc = d_fr.ensure(frows.size()))) return rc;
    cudaStream_t st = e->stream;
    CU(cudaMemcpyAsync(d_ir.p, irows.data(), irows.size() * 4, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d_fr.p, frows.data(), frows.size() * 4, cudaMemcpyHostToDevice, st));
    if ((rc = e->precomputed.ensure(e->cfg.max_splat_count))) return rc;
    const int blocks = std::max(1, (int)std::min<uint32_t>((count + 255) / 256, e->sm_count * 8));
    if (integer && dyn) k_distances_splat_order<true, true><<<blocks, 256, 0, st>>>(e->centers.p, e->scene_idx.p, d_ir.p, d_fr.p, count, e->precomputed.p);
    else if (integer) k_distances_splat_order<true, false><<<blocks, 256, 0, st>>>(e->centers.p, e->scene_idx.p, d_ir.p, d_fr.p, count, e->precomputed.p);
    else if (dyn) k_distances_splat_order<false, true><<<blocks, 256, 0, st>>>(e->centers.p, e->scene_idx.p, d_ir.p, d_fr.p, count, e->precomputed.p);
    else k_distances_splat_order<false, false><<<blocks, 256, 0, st>>>(e->centers.p, e->scene_idx.p, d_ir.p, d_fr.p, count, e->precomputed.p);
    CU(cudaMemcpyAsync(out, e->precomputed.p, (size_t)count * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    return GS_OK;
}

// ---------------------------------------------------------------------------------------------------------------
extern "C" int gs_upload_splat_data(gs_engine *e, const gs_splat_data *d) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!d) return fail(GS_ERR_BAD_ARG, "gs_upload_splat_data: null");
    e->ray.valid = false;   // host-packed splats: their ray records come from gs_upload_ray_records
    rc = raster_upload(e->rs, e->cfg, *d, e->stream);
    if (rc) return rc;
    CU(cudaStreamSynchronize(e->stream));
    return GS_OK;
}

static int render_on_device(gs_engine *e, const gs_uniforms *u, const gs_render_params *p, const uint32_t *d_order, bool capturing = false, int phases = 3,
                            const unsigned long long *order_count_dev = nullptr) {
    cudaStream_t st = e->stream;
    if (!capturing && (phases & 1)) CU(cudaEventRecord(e->ev[EV_R0], st));
    if (!e->have_prof_begin) e->prof.begin(st);
    int rc = raster_render(e->rs, e->cfg, *u, *p, d_order, st, e->ev[EV_PROJECT], e->ev[EV_BIN], e->tm, e->prof, !capturing, !capturing, phases, order_count_dev);
    if (rc) return rc;
    if (!capturing && (phases & 2)) CU(cudaEventRecord(e->ev[EV_R1], st));
    CU(cudaGetLastError());
    return GS_OK;
}

static size_t frame_bytes(const gs_render_params *p) { return (size_t)p->width * p->height * (p->frame_format == GS_FRAME_RGBA8 ? 4 : 16); }

static int finish_render(gs_engine *e, const gs_render_params *p, void *frame_out) {
    cudaStream_t st = e->stream;
    CU(cudaEventRecord(e->ev[EV_D2H0], st));
    // world_size > 1: a full-size frame whose pixels outside this rank's coarse tiles are zero
    if (frame_out) CU(cudaMemcpyAsync(frame_out, raster_frame_ptr(e->rs, p->frame_format), frame_bytes(p), cudaMemcpyDeviceToHost, st));
    CU(cudaEventRecord(e->ev[EV_D2H1], st));
    CU(cudaMemcpyAsync(e->h_ctl.p + 16, e->rs.rctl.p, sizeof(RasterControl), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (e->last_frame_was_graph) {
        e->tm.project_ms = e->tm.bin_ms = e->tm.blend_ms = 0.f;
        cudaEventElapsedTime(&e->tm.render_total_ms, e->ev[EV_SORT0], e->ev[EV_R1]);   // whole frame (sort + render) in graph mode
    } else {
        cudaEventElapsedTime(&e->tm.project_ms, e->ev[EV_R0], e->ev[EV_PROJECT]);
        cudaEventElapsedTime(&e->tm.bin_ms, e->ev[EV_PROJECT], e->ev[EV_BIN]);
        cudaEventElapsedTime(&e->tm.blend_ms, e->ev[EV_BIN], e->ev[EV_R1]);
        cudaEventElapsedTime(&e->tm.render_total_ms, e->ev[EV_R0], e->ev[EV_R1]);
    }
    cudaEventElapsedTime(&e->tm.d2h_ms, e->ev[EV_D2H0], e->ev[EV_D2H1]);
    RasterControl rc;
    memcpy(&rc, e->h_ctl.p + 16, sizeof(rc));
    e->tm.tile_instances = rc.total_instances;
    uint32_t vis = 0;
    for (int i = 0; i < kVisibleSlots; ++i) vis += rc.visible_slots[i * 8];
    e->tm.visible_splats = vis;
    if (rc.peer_timeout) return fail(GS_ERR_CUDA, "multi-GPU tile gather: a peer did not arrive within the time limit (ranks must render the same frames)");
    if (rc.overflow) return fail(GS_ERR_CAPACITY, "tile-instance buffer overflow: %llu instances needed, capacity %llu (raise GS_INSTANCE_FACTOR)",
                                 (unsigned long long)rc.total_instances, (unsigned long long)e->rs.instance_capacity);
    return GS_OK;
}

static int stage_order(gs_engine *e, const gs_render_params *p, const uint32_t **d_order) {
    *d_order = nullptr;
    if (p->render_count > e->cfg.max_splat_count) return fail(GS_ERR_CAPACITY, "render_count %u > max_splat_count %u", p->render_count, e->cfg.max_splat_count);
    if (p->sorted_indexes_dev) *d_order = p->sorted_indexes_dev;
    else if (p->sorted_indexes) { // SplatMesh.updateRenderIndexes: upload of the splatIndex attribute
        CU(cudaMemcpyAsync(e->sorted.p, p->sorted_indexes, (size_t)p->render_count * 4, cudaMemcpyHostToDevice, e->stream));
        *d_order = e->sorted.p;
        e->have_sorted = true;
        e->last_render_count = p->render_count;
    } else {
        if (!e->have_sorted || e->last_render_count < p->render_count) return fail(GS_ERR_NOT_READY, "gs_render without sorted indexes: call gs_sort first or pass sorted_indexes");
        *d_order = e->sorted.p;
    }
    return GS_OK;
}

extern "C" int gs_render(gs_engine *e, const gs_uniforms *u, const gs_render_params *p, void *frame_out) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!u || !p) return fail(GS_ERR_BAD_ARG, "gs_render: null argument");
    if (e->pipe_inflight()) return fail(GS_ERR_NOT_READY, "gs_render: pipelined frames are in flight (gs_frame_end first)");
    const uint32_t *d_order = nullptr;
    e->last_frame_was_graph = false;
    if ((rc = stage_order(e, p, &d_order))) return rc;
    if ((rc = render_on_device(e, u, p, d_order))) return rc;
    return finish_render(e, p, frame_out);
}

// host-side parameter blocks of one frame -> device (outside any graph; pageable sources are staged by the driver before return)
static int upload_frame_params(gs_engine *e, const float *mvp, const gs_uniforms &u, const gs_render_params &p) {
    DepthParams P{};
    memcpy(P.mvp, mvp, 64);
    P.irow[0] = (int32_t)((double)mvp[2] * 1000.0);
    P.irow[1] = (int32_t)((double)mvp[6] * 1000.0);
    P.irow[2] = (int32_t)((double)mvp[10] * 1000.0);
    P.irow[3] = 1;
    P.frow[0] = mvp[2]; P.frow[1] = mvp[6]; P.frow[2] = mvp[10]; P.frow[3] = 0.f;
    cudaStream_t st = e->param_side ? e->param_stream : e->stream;
    CU(cudaMemcpyAsync(e->depthp.p + e->rs.frame_parity, &P, sizeof(P), cudaMemcpyHostToDevice, st));
    int rc = raster_upload_params(e->rs, e->cfg, u, p, st);
    if (rc) return rc;
    if (e->param_side) {      // the frame graph (and nothing else on the compute stream) waits for the side upload
        CU(cudaEventRecord(e->ev_params[e->rs.frame_parity], st));
        CU(cudaStreamWaitEvent(e->stream, e->ev_params[e->rs.frame_parity], 0));
    }
    return GS_OK;
}

static int enqueue_frame(gs_engine *e, const gs_sort_params *s, const gs_uniforms *u, const gs_render_params *p, gs_sort_params &q, gs_render_params &rp) {
    q = *s;
    q.render_count = std::min(q.render_count, e->uploaded_splats);
    q.sort_count = std::min(q.sort_count, e->uploaded_splats);
    const uint32_t *d_idx = nullptr;
    int rc;
    if ((rc = stage_sort_inputs(e, &q, &d_idx))) return rc;
    rp = *p;
    rp.sorted_indexes = nullptr; rp.sorted_indexes_dev = nullptr;
    rp.render_count = std::min(rp.render_count, q.render_count);
    cudaStream_t st = e->stream;
    e->last_frame_was_graph = false;
    // sharded frame: sort only this rank's subset (full sorts only; a partial sort keeps the replicated path)
    // The subset path adds two compaction kernels (~35 us at 1M splats) and only shrinks kernels that are already at their latency
    // floor there; it pays off from a few million splats (measured: 1.2M slower, 16M faster).  GS_SUBSET_MIN overrides the threshold.
    const uint32_t subset_min = getenv("GS_SUBSET_MIN") ? (uint32_t)atoll(getenv("GS_SUBSET_MIN")) : 3000000u;
    const bool subset = e->cfg.world_size > 1 && q.sort_count == q.render_count && q.render_count >= subset_min && q.render_count > 0 && !e->no_subset;
    if (subset) {
        if ((rc = e->sub_idx.ensure(e->cfg.max_splat_count)) || (rc = e->sub_dist.ensure(e->cfg.max_splat_count))) return rc;
    }
    const unsigned long long *order_count = subset ? &e->rs.rctl.p->subset_count : nullptr;
    const bool use_graph = e->graph_enabled && !e->prof.on && q.sort_count <= q.render_count && q.render_count <= e->cfg.max_splat_count && e->rs.uploaded;
    if (use_graph) {
        const unsigned long long key[8] = {q.render_count, q.sort_count, ((unsigned long long)rp.width << 32) | rp.height,
                                           ((unsigned long long)rp.frame_format << 8) | (unsigned long long)(rp.flip_y ? 1 : 0) | ((unsigned long long)q.use_precomputed_distances << 4),
                                           (unsigned long long)(uintptr_t)d_idx, ((unsigned long long)e->rs.cov_format << 16) | ((unsigned long long)e->rs.sh_format << 8) | e->rs.sh_degree,
                                           e->rs.uploaded, ((unsigned long long)rp.render_count << 1) | (subset ? 1ull : 0ull)};
        if ((rc = upload_frame_params(e, q.model_view_proj, *u, rp))) return rc;
        cudaGraphExec_t &gexec = e->rs.frame_parity ? e->graph_exec_alt : e->graph_exec;      // one instantiated graph per target frame buffer
        unsigned long long *gkey = e->rs.frame_parity ? e->graph_key_alt : e->graph_key;
        if (!gexec || memcmp(key, gkey, sizeof(key)) != 0) {
            if (gexec) { cudaGraphExecDestroy(gexec); gexec = nullptr; }
            // buffers that the enqueue path may grow must be sized BEFORE capture (no allocation inside a capture)
            uint32_t stride = 0;
            const PassPlan pl = make_plan_bits(e->key_bits);
            if ((rc = e->tile_hist.ensure(radix_tile_hist_words(std::max(q.sort_count, 1u), pl.npasses, &stride)))) return rc;
            CU(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
            struct CaptureGuard {   // an early error return must not leave the stream capturing
                cudaStream_t st; bool armed;
                ~CaptureGuard() { if (armed) { cudaGraph_t g = nullptr; cudaStreamEndCapture(st, &g); if (g) cudaGraphDestroy(g); (void)cudaGetLastError(); } }
            } guard{st, true};
            // fork: the projection does not depend on the draw order, so it runs beside the (latency-bound) depth sort
            CU(cudaEventRecord(e->ev_fork, st));
            CU(cudaStreamWaitEvent(e->stream2, e->ev_fork, 0));
            int rc2 = GS_OK;
            uint32_t proj_launches = 0;
            {
                cudaStream_t keep = e->stream;
                e->stream = e->stream2;
                rc2 = render_on_device(e, u, &rp, e->sorted.p, true, 1);
                proj_launches = e->tm.kernel_launches;
                e->stream = keep;
            }
            CU(cudaEventRecord(e->ev_join, e->stream2));
            rc = sort_on_device(e, d_idx, q.model_view_proj, q.sort_count, q.render_count, q.use_precomputed_distances != 0, false, true, subset, e->ev_join);
            const uint32_t sort_launches = e->tm.kernel_launches;
            CU(cudaStreamWaitEvent(st, e->ev_join, 0));
            if (!rc2) rc2 = rc ? rc : render_on_device(e, u, &rp, e->sorted.p, true, 2, order_count);
            e->graph_launches = e->tm.kernel_launches + sort_launches + proj_launches;
            cudaGraph_t g = nullptr;
            guard.armed = false;
            cudaError_t ce = cudaStreamEndCapture(st, &g);
            if (rc2) { if (g) cudaGraphDestroy(g); return rc2; }
            if (ce != cudaSuccess) return fail(GS_ERR_CUDA, "cudaStreamEndCapture -> %s", cudaGetErrorString(ce));
            ce = cudaGraphInstantiate(&gexec, g, 0);
            cudaGraphDestroy(g);
            if (ce != cudaSuccess) { gexec = nullptr; return fail(GS_ERR_CUDA, "cudaGraphInstantiate -> %s", cudaGetErrorString(ce)); }
            memcpy(gkey, key, sizeof(key));
            e->graph_snapshot[e->rs.frame_parity ? 1 : 0] = e->rs.snapshot_taken;
        }
        if (e->ctl_dirty) gs_launch(k_sort_init, 1, 256, 0, st, e->ctl.p);   // the captured sort assumes (and leaves) a clean control block
        e->ctl_dirty = true;
        CU(cudaEventRecord(e->ev[EV_SORT0], st));
        CU(cudaGraphLaunch(gexec, st));
        e->ctl_dirty = false;
        CU(cudaEventRecord(e->ev[EV_R1], st));
        e->tm.kernel_launches = e->graph_launches;
        e->last_render_count = q.render_count;
        e->have_sorted = !subset;   // a subset order is not a draw order for gs_render
        e->last_frame_was_graph = true;
        return GS_OK;
    }
    if (subset) {   // one stream: projection first (its rects select the subset), then depth + subset sort, then binning + blend
        e->prof.begin(st);
        e->have_prof_begin = true;
        if ((rc = render_on_device(e, u, &rp, e->sorted.p, false, 1))) { e->have_prof_begin = false; return rc; }
        const uint32_t proj_launches = e->tm.kernel_launches;
        if ((rc = sort_on_device(e, d_idx, q.model_view_proj, q.sort_count, q.render_count, q.use_precomputed_distances != 0, false, false, true, nullptr))) { e->have_prof_begin = false; return rc; }
        const uint32_t sort_launches = e->tm.kernel_launches;
        rc = render_on_device(e, u, &rp, e->sorted.p, false, 2, order_count);
        e->have_prof_begin = false;
        if (rc) return rc;
        e->tm.kernel_launches += sort_launches + proj_launches;
        e->have_sorted = false;
        return GS_OK;
    }
    if ((rc = sort_on_device(e, d_idx, q.model_view_proj, q.sort_count, q.render_count, q.use_precomputed_distances != 0, false))) return rc;
    const uint32_t sort_launches = e->tm.kernel_launches;
    e->have_prof_begin = true;
    rc = render_on_device(e, u, &rp, e->sorted.p);
    e->have_prof_begin = false;
    if (rc) return rc;
    e->tm.kernel_launches += sort_launches;
    return GS_OK;
}

extern "C" int gs_frame(gs_engine *e, const gs_sort_params *s, const gs_uniforms *u, const gs_render_params *p, uint32_t *sorted_out, void *frame_out) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!s || !u || !p) return fail(GS_ERR_BAD_ARG, "gs_frame: null argument");
    if (e->pipe_inflight()) return fail(GS_ERR_NOT_READY, "gs_frame: pipelined frames are in flight (gs_frame_end first)");
    e->rs.frame_parity = 0;
    gs_sort_params q; gs_render_params rp;
    e->no_subset = (sorted_out != nullptr);
    rc = enqueue_frame(e, s, u, p, q, rp);
    e->no_subset = false;
    if (rc) return rc;
    if (sorted_out && q.render_count) CU(cudaMemcpyAsync(sorted_out, e->sorted.p, (size_t)q.render_count * 4, cudaMemcpyDeviceToHost, e->stream));
    int rc2 = finish_render(e, &rp, frame_out);
    rc = finish_sort(e, nullptr);
    cudaEventElapsedTime(&e->tm.h2d_ms, e->ev[EV_H2D0], e->ev[EV_H2D1]);
    return rc ? rc : rc2;
}

// Enqueue one frame and return without waiting: the frame stays on the device (gs_buffer_dev(GS_BUF_FRAME)), errors and
// timings are collected by the next gs_synchronize().  Lets a caller keep several frames in flight on the stream.
extern "C" int gs_frame_async(gs_engine *e, const gs_sort_params *s, const gs_uniforms *u, const gs_render_params *p) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!s || !u || !p) return fail(GS_ERR_BAD_ARG, "gs_frame_async: null argument");
    if (e->pipe_inflight()) return fail(GS_ERR_NOT_READY, "gs_frame_async: pipelined frames are in flight (gs_frame_end first): their pictures are still being copied out of the frame buffers");
    gs_sort_params q; gs_render_params rp;
    if ((rc = enqueue_frame(e, s, u, p, q, rp))) return rc;
    e->pending_async = true;
    e->pending_rp = rp;
    return GS_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Pipelined frames: gs_frame_begin enqueues frame i (camera H2D, sort, render) and a D2H copy of its picture on a separate copy
// stream; gs_frame_end waits for the OLDEST frame in flight and reports its errors.  Up to three frames may be in flight over TWO
// device frame buffers: frame i+1 renders while frame i's picture crosses PCIe, and frame i+2 is already queued behind it (it
// starts only when frame i's copy has left its buffer), so the GPU never waits for the host between frames
// (begin(0); begin(1); loop { begin(i+2); end(i); }).  Every frame in flight needs its own `frame_out`.  Per-frame latency is that of
// gs_frame; throughput approaches max(compute, copy).  With two buffers a frame graph is the ONLY thing a frame puts on the compute
// stream: the parameter blocks go up on `param_stream` into the block of the frame buffer's parity, and the status words are
// snapshotted by the blend kernel and read back on the copy stream.  Multi-GPU engines that gather tiles into rank 0's exported
// frame keep ONE buffer (the peers store into it), so there the copy only overlaps the host side.
static int pipe_init(gs_engine *e) {
    if (e->copy_stream) return GS_OK;
    CU(cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking));
    CU(cudaStreamCreateWithFlags(&e->param_stream, cudaStreamNonBlocking));
    for (int i = 0; i < gs_engine::kPipeRing; ++i) {
        CU(cudaEventCreateWithFlags(&e->ev_frame_done[i], cudaEventDisableTiming));
        CU(cudaEventCreateWithFlags(&e->ev_copy_done[i], cudaEventDisableTiming));
    }
    for (int i = 0; i < 2; ++i) CU(cudaEventCreateWithFlags(&e->ev_params[i], cudaEventDisableTiming));
    int rc = e->h_pipe.ensure(gs_engine::kPipeRing * kPipeSlotWords);
    if (rc) return rc;
    const bool single = e->cfg.world_size > 1;      // (rank 0 of a peer group may hold a double allocation instead: rs.frame_half2)
    if (!single && !e->rs.frame_alt.p) return e->rs.frame_alt.ensure(e->rs.frame.n);
    return GS_OK;
}

extern "C" int gs_frame_begin(gs_engine *e, const gs_sort_params *s, const gs_uniforms *u, const gs_render_params *p, void *frame_out) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!s || !u || !p) return fail(GS_ERR_BAD_ARG, "gs_frame_begin: null argument");
    if (e->pipe_inflight() >= (uint32_t)gs_engine::kPipeMaxInflight) return fail(GS_ERR_NOT_READY, "gs_frame_begin: %d frames already in flight (call gs_frame_end)", gs_engine::kPipeMaxInflight);
    if (e->pending_async) return fail(GS_ERR_NOT_READY, "gs_frame_begin: an asynchronous frame is pending (gs_synchronize first)");
    if ((rc = pipe_init(e))) return rc;
    constexpr uint64_t R = gs_engine::kPipeRing;
    const uint64_t seq = e->pipe_begun;
    const uint32_t ring = (uint32_t)(seq % R);
    const bool two = raster_second_frame(e->rs) != nullptr;
    // the buffer this frame renders into must have been copied out: frame seq-2 with two buffers, seq-1 with one
    if (two) { if (seq >= 2) CU(cudaStreamWaitEvent(e->stream, e->ev_copy_done[(seq - 2) % R], 0)); }
    else if (seq >= 1) CU(cudaStreamWaitEvent(e->stream, e->ev_copy_done[(seq - 1) % R], 0));
    e->rs.frame_parity = two ? (int)(seq & 1) : 0;
    // parameter blocks of this parity were last read by frame seq-2: its graph must have finished before they are overwritten
    e->param_side = two;
    if (two && seq >= 2) CU(cudaStreamWaitEvent(e->param_stream, e->ev_frame_done[(seq - 2) % R], 0));
    gs_sort_params q; gs_render_params rp;
    rc = enqueue_frame(e, s, u, p, q, rp);
    e->param_side = false;
    if (rc) { e->rs.frame_parity = 0; return rc; }
    cudaStream_t st = e->stream;
    uint32_t *hs = e->h_pipe.p + ring * kPipeSlotWords;
    // (multi-GPU: rank 0's peer_timeout flag is raised AFTER the blend, by k_peer_wait_arrived -- the snapshot would miss it)
    const bool snapshot = two && e->cfg.world_size == 1 && e->last_frame_was_graph && e->graph_snapshot[e->rs.frame_parity];
    if (!snapshot) {      // status read-back in stream order (frames outside a graph, blend generations without the snapshot, one buffer)
        CU(cudaMemcpyAsync(hs, e->ctl.p, 12, cudaMemcpyDeviceToHost, st));
        CU(cudaMemcpyAsync(hs + 4, e->rs.rctl.p, sizeof(RasterControl), cudaMemcpyDeviceToHost, st));
    }
    CU(cudaEventRecord(e->ev_frame_done[ring], st));
    CU(cudaStreamWaitEvent(e->copy_stream, e->ev_frame_done[ring], 0));
    if (snapshot)
        CU(cudaMemcpyAsync(hs, e->status_dev.p + (size_t)e->rs.frame_parity * kPipeSlotWords, (4 + sizeof(RasterControl) / 4) * 4, cudaMemcpyDeviceToHost, e->copy_stream));
    if (frame_out) CU(cudaMemcpyAsync(frame_out, raster_frame_ptr(e->rs, rp.frame_format), frame_bytes(&rp), cudaMemcpyDeviceToHost, e->copy_stream));
    CU(cudaEventRecord(e->ev_copy_done[ring], e->copy_stream));
    ++e->pipe_begun;
    return GS_OK;
}

extern "C" int gs_frame_end(gs_engine *e) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (e->pipe_inflight() == 0) return fail(GS_ERR_NOT_READY, "gs_frame_end: no frame in flight");
    const uint32_t ring = (uint32_t)(e->pipe_ended % (uint64_t)gs_engine::kPipeRing);
    CU(cudaEventSynchronize(e->ev_copy_done[ring]));
    ++e->pipe_ended;
    const uint32_t *hs = e->h_pipe.p + ring * kPipeSlotWords;
    RasterControl rctl;
    memcpy(&rctl, hs + 4, sizeof(rctl));
    e->tm.tile_instances = rctl.total_instances;
    uint32_t vis = 0;
    for (int i = 0; i < kVisibleSlots; ++i) vis += rctl.visible_slots[i * 8];
    e->tm.visible_splats = vis;
    if (hs[2] & kErrBucketRange) return fail(GS_ERR_BUCKET_RANGE, "a bucket index fell outside [0,%u): distances overflow the int32/f32 range map", e->cfg.distance_map_range);
    if (rctl.peer_timeout) return fail(GS_ERR_CUDA, "multi-GPU tile gather: a peer did not arrive within the time limit (ranks must render the same frames)");
    if (rctl.overflow) return fail(GS_ERR_CAPACITY, "tile-instance buffer overflow: %llu instances needed, capacity %llu (raise GS_INSTANCE_FACTOR)",
                                   (unsigned long long)rctl.total_instances, (unsigned long long)e->rs.instance_capacity);
    return GS_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// SplatTree leaves -> device, and the per-frame cull + index gather (SURVEY 8(f) N2; cull_kernels.cuh).
extern "C" int gs_upload_splat_tree(gs_engine *e, const double *node_center, const double *node_min, const double *node_max, const uint32_t *node_offsets,
                                    const uint32_t *indexes, uint32_t node_count) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (node_count && (!node_center || !node_min || !node_max || !node_offsets || !indexes)) return fail(GS_ERR_BAD_ARG, "gs_upload_splat_tree: null argument");
    const uint32_t total = node_count ? node_offsets[node_count] : 0;
    if (total > e->cfg.max_splat_count) return fail(GS_ERR_CAPACITY, "the tree's leaves hold %u indexes, engine capacity %u", total, e->cfg.max_splat_count);
    for (uint32_t i = 0; i < node_count; ++i)
        if (node_offsets[i + 1] < node_offsets[i]) return fail(GS_ERR_BAD_ARG, "gs_upload_splat_tree: node_offsets must be non-decreasing");
    auto &t = e->tree;
    const size_t m = std::max<uint32_t>(node_count, 1);
    if ((rc = t.center.ensure(3 * m)) || (rc = t.nmin.ensure(3 * m)) || (rc = t.nmax.ensure(3 * m)) || (rc = t.offsets.ensure(m + 1)) || (rc = t.indexes.ensure(std::max<uint32_t>(total, 1))) ||
        (rc = t.start.ensure(m)) || (rc = t.key.ensure(m)) || (rc = t.total.ensure(1)))
        return rc;
    cudaStream_t st = e->stream;
    if (node_count) {
        CU(cudaMemcpyAsync(t.center.p, node_center, 24 * (size_t)node_count, cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync(t.nmin.p, node_min, 24 * (size_t)node_count, cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync(t.nmax.p, node_max, 24 * (size_t)node_count, cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync(t.offsets.p, node_offsets, 4 * ((size_t)node_count + 1), cudaMemcpyHostToDevice, st));
        if (total) CU(cudaMemcpyAsync(t.indexes.p, indexes, 4 * (size_t)total, cudaMemcpyHostToDevice, st));
    }
    CU(cudaStreamSynchronize(st));
    t.count = node_count; t.splats = total;
    t.have_nodes = false;   // gs_upload_splat_tree_nodes describes these leaves next
    return GS_OK;
}

extern "C" int gs_gather_for_sort(gs_engine *e, const double *model_view, double cos_fov_x_over_2, double cos_fov_y_over_2, int gather_all_nodes,
                                  uint32_t *render_count_out) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!model_view || !render_count_out) return fail(GS_ERR_BAD_ARG, "gs_gather_for_sort: null argument");
    auto &t = e->tree;
    if (!t.count) { *render_count_out = 0; return GS_OK; }
    CullParams P;
    memcpy(P.mv, model_view, sizeof(P.mv));
    P.cos_fov_x_over_2 = cos_fov_x_over_2; P.cos_fov_y_over_2 = cos_fov_y_over_2; P.gather_all = gather_all_nodes;
    cudaStream_t st = e->stream;
    k_tree_cull<<<(t.count + 127) / 128, 128, 0, st>>>(t.center.p, t.nmin.p, t.nmax.p, t.count, P, t.key.p);
    k_tree_layout<<<(t.count + kLayoutThreads - 1) / kLayoutThreads, kLayoutThreads, 0, st>>>(t.key.p, t.offsets.p, t.count, t.start.p, t.total.p);
    k_tree_copy<<<t.count, 128, 0, st>>>(t.start.p, t.offsets.p, t.indexes.p, e->indexes.p);
    CU(cudaMemcpyAsync(e->h_ctl.p + 8, t.total.p, 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    unsigned long long total;
    memcpy(&total, e->h_ctl.p + 8, 8);
    *render_count_out = (uint32_t)total;
    e->tm.kernel_launches = 3;
    return GS_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Raycaster.intersectSplatMesh on the GPU (ray_kernels.cuh).
// The ray records now describe the current scene; a static mesh's are placed by `xf` (column-major 4x4, nullptr: identity).
static void set_ray_transform(gs_engine *e, const double *xf) {
    static const double kIdentity[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    memcpy(e->ray.xf, xf ? xf : kIdentity, sizeof(e->ray.xf));
    e->ray.valid = true;
}

extern "C" int gs_upload_ray_records(gs_engine *e, const gs_ray_record *records, uint32_t from, uint32_t count, const double *scene_transform) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!e->ray.rec.p) return fail(GS_ERR_NOT_READY, "gs_upload_ray_records: engine created without ray_records");
    if (!records && count) return fail(GS_ERR_BAD_ARG, "gs_upload_ray_records: null records");
    if ((uint64_t)from + count > e->cfg.max_splat_count) return fail(GS_ERR_CAPACITY, "ray records [%u,%u) exceed max_splat_count %u", from, from + count, e->cfg.max_splat_count);
    if (count) CU(cudaMemcpyAsync(e->ray.rec.p + from, records, (size_t)count * sizeof(gs_ray_record), cudaMemcpyHostToDevice, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    set_ray_transform(e, scene_transform);
    return GS_OK;
}

extern "C" int gs_upload_splat_tree_nodes(gs_engine *e, const double *node_min, const double *node_max, const int32_t *node_parent, uint32_t node_count,
                                          const uint32_t *leaf_node, uint32_t leaf_count) {
    int rc = check_engine(e);
    if (rc) return rc;
    auto &t = e->tree;
    if (leaf_count != t.count) return fail(GS_ERR_BAD_ARG, "gs_upload_splat_tree_nodes: %u leaves, the uploaded tree has %u", leaf_count, t.count);
    if ((node_count && (!node_min || !node_max || !node_parent)) || (leaf_count && !leaf_node)) return fail(GS_ERR_BAD_ARG, "gs_upload_splat_tree_nodes: null argument");
    // a parent precedes its children (depth-first, root first), so every walk up the tree ends at the root
    for (uint32_t i = 0; i < node_count; ++i)
        if (node_parent[i] >= (int32_t)i || (i == 0) != (node_parent[i] < 0)) return fail(GS_ERR_BAD_ARG, "gs_upload_splat_tree_nodes: node %u has parent %d", i, node_parent[i]);
    for (uint32_t i = 0; i < leaf_count; ++i)
        if (leaf_node[i] >= node_count) return fail(GS_ERR_BAD_ARG, "gs_upload_splat_tree_nodes: leaf %u -> node %u of %u", i, leaf_node[i], node_count);
    const size_t m = std::max<uint32_t>(node_count, 1);
    if ((rc = t.all_min.ensure(3 * m)) || (rc = t.all_max.ensure(3 * m)) || (rc = t.parent.ensure(m)) || (rc = t.leaf_node.ensure(std::max<uint32_t>(leaf_count, 1))))
        return rc;
    cudaStream_t st = e->stream;
    if (node_count) {
        CU(cudaMemcpyAsync(t.all_min.p, node_min, 24 * (size_t)node_count, cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync(t.all_max.p, node_max, 24 * (size_t)node_count, cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync(t.parent.p, node_parent, 4 * (size_t)node_count, cudaMemcpyHostToDevice, st));
    }
    if (leaf_count) CU(cudaMemcpyAsync(t.leaf_node.p, leaf_node, 4 * (size_t)leaf_count, cudaMemcpyHostToDevice, st));
    CU(cudaStreamSynchronize(st));
    t.node_count = node_count;
    t.have_nodes = true;
    return GS_OK;
}

extern "C" int gs_raycast(gs_engine *e, const gs_raycast_params *p, gs_ray_hit *hits, uint32_t capacity, uint32_t *hit_count) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!p || !hit_count || (capacity && !hits)) return fail(GS_ERR_BAD_ARG, "gs_raycast: null argument");
    const gs_raycast_params q = read_options(p, gs_raycast_params{});
    auto &t = e->tree;
    auto &R = e->ray;
    if (!R.rec.p) return fail(GS_ERR_NOT_READY, "gs_raycast: engine created without ray_records");
    if (!R.valid) return fail(GS_ERR_NOT_READY, "gs_raycast: the ray records are stale (upload the scene or gs_upload_ray_records)");
    if (!t.have_nodes) return fail(GS_ERR_NOT_READY, "gs_raycast: no SplatTree (gs_upload_splat_tree + gs_upload_splat_tree_nodes)");
    *hit_count = 0;
    if (!t.count || !t.node_count || !q.scene_visible) return GS_OK;   // no leaves, or every splat skipped (Raycaster.js:117)
    RayParams P{};
    memcpy(P.origin, q.origin, sizeof(P.origin)); memcpy(P.dir, q.direction, sizeof(P.dir));
    memcpy(P.from_local, q.from_local, sizeof(P.from_local)); memcpy(P.xf, R.xf, sizeof(P.xf));
    P.ellipsoid = q.mode == GS_RAYCAST_ELLIPSOID; P.dynamic = e->cfg.dynamic_mode;
    const uint32_t m = t.count, nn = t.node_count, n = std::max<uint32_t>(t.splats, 1);
    if ((rc = R.setup.ensure(1)) || (rc = R.pass.ensure(nn)) || (rc = R.reached.ensure(m)) || (rc = R.list.ensure(m)) || (rc = R.counts.ensure(4)) ||
        (rc = R.hits.ensure(n)))
        return rc;
    cudaStream_t st = e->stream;
    uint32_t launches = 0;
    k_ray_setup<<<1, 1, 0, st>>>(P, R.setup.p);
    k_ray_nodes<<<(nn + 127) / 128, 128, 0, st>>>(t.all_min.p, t.all_max.p, nn, R.setup.p, R.pass.p);
    k_ray_leaves<<<(m + 127) / 128, 128, 0, st>>>(t.leaf_node.p, t.parent.p, R.pass.p, m, R.reached.p);
    k_ray_compact<<<1, kRayCompactThreads, 0, st>>>(R.reached.p, m, R.list.p, R.counts.p);   // also zeroes the hit counter counts[1]
    const uint32_t grid = std::min<uint32_t>((m + kRaySplatThreads / 32 - 1) / (kRaySplatThreads / 32), (uint32_t)e->sm_count * 16);
    k_ray_splats<<<grid, kRaySplatThreads, 0, st>>>(R.list.p, R.counts.p, t.offsets.p, t.indexes.p, R.rec.p, P, R.setup.p, R.hits.p, R.counts.p + 1);
    launches += 5;
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(e->h_ctl.p + 8, R.counts.p, 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    const uint32_t total = e->h_ctl.p[9];
    *hit_count = total;
    const uint32_t k = std::min(capacity, total);
    if (!k) { e->tm.kernel_launches = launches; return GS_OK; }
    const uint32_t *perm = nullptr;
    if (total > 1) {   // stable LSD radix sort by (distance, traversal position): position first, then the distance's three pieces
        uint32_t stride = 0;
        int pos_bits = 1;
        while (pos_bits < 32 && (1ull << pos_bits) < (unsigned long long)t.splats) ++pos_bits;
        if ((rc = R.keys[0].ensure(n)) || (rc = R.keys[1].ensure(n)) || (rc = R.vals[0].ensure(n)) || (rc = R.vals[1].ensure(n)) || (rc = R.vals[2].ensure(n)) ||
            (rc = R.vals[3].ensure(n)) || (rc = R.tile_hist.ensure(radix_tile_hist_words(total, 4, &stride))))
            return rc;
        if (!R.ctl.p) {
            if ((rc = R.ctl.ensure(1))) return rc;
            CU(cudaMemsetAsync(R.ctl.p, 0, sizeof(SortControl), st));   // the scatter passes clear their histograms again (self_clean)
        }
        static const RadixNames names{{"ray_hist0", "ray_hist1", "ray_hist2", "ray_hist3"}, {"ray_scan0", "ray_scan1", "ray_scan2", "ray_scan3"},
                                      {"ray_scatter0", "ray_scatter1", "ray_scatter2", "ray_scatter3"}};
        uint32_t *order = nullptr;
        for (int which = 0; which < 4; ++which) {
            const PassPlan pl = make_plan_bits(which == 0 ? pos_bits : kRayKeyBits[which]);
            uint32_t *dst = R.vals[2 + (which & 1)].p;
            k_ray_keys<<<(total + 255) / 256, 256, 0, st>>>(R.hits.p, order, total, which, R.keys[0].p, R.vals[0].p);
            ++launches;
            radix_sort_pairs<uint32_t, uint32_t>(R.keys[0].p, R.keys[1].p, R.vals[0].p, 0, kValArray, R.vals[1].p, R.vals[0].p, dst, total, nullptr, 0, pl,
                                                 R.ctl.p, R.tile_hist.p, stride, false, nullptr, st, launches, nullptr, names, true);
            order = dst;
        }
        perm = order;
    }
    if ((rc = R.out.ensure(k))) return rc;
    k_ray_out<<<(k + 127) / 128, 128, 0, st>>>(R.hits.p, perm, k, R.out.p);
    ++launches;
    CU(cudaMemcpyAsync(hits, R.out.p, (size_t)k * sizeof(gs_ray_hit), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    e->tm.kernel_launches = launches;
    return GS_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Scene uploads: .ksplat images (gs_upload_ksplat, gs_upload_file_optimized's generated image) and files (gs_upload_file).  Each one
//   1. validates the engine, its arguments and the source's header;
//   2. allocates this call's transient buffers and uploads the scene transform: a failure up to here leaves the previous scene;
//   3. marks the scene empty before any scene buffer may be reallocated, then sets the storage formats (clear_scene);
//   4. decodes level-N SplatBuffer sections on the GPU (decode_section);
//   5. commits the scene and reports it (commit_scene).
// .ksplat header/section parsing is host logic (SplatBuffer.js:819-941); the decode runs on the GPU (SURVEY 8f N1).
static gs_ksplat_options ksplat_options(const gs_ksplat_options *opt) {
    gs_ksplat_options o{};
    o.minimum_alpha = 1; o.upload_sort_centers = 1;
    return read_options(opt, o);
}

// What a scene upload reports, for a level-`level` image of `sections` sections.  The scene centre and SH range are those of a level-0
// SplatBuffer header (SplatBuffer.js:873-874); a .ksplat's own header replaces them.
static gs_ksplat_info scene_info(uint32_t splats, uint32_t sh_degree, uint32_t level, uint32_t sections) {
    gs_ksplat_info S{};
    S.struct_size = sizeof(S);
    S.splat_count = splats; S.sh_degree = sh_degree; S.compression_level = level; S.section_count = sections;
    S.min_sh_coeff = -1.5f; S.max_sh_coeff = 1.5f;
    return S;
}

// Step 1, the engine's part.  `entry` names the caller in the messages; sh_degree is the Viewer's sphericalHarmonicsDegree.
static int check_scene_engine(gs_engine *e, const char *entry, uint32_t sh_degree) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!e->cfg.max_width || !e->cfg.max_height) return fail(GS_ERR_NOT_READY, "engine created without a framebuffer (max_width/max_height = 0)");
    if (sh_degree > 2) return fail(GS_ERR_BAD_ARG, "%s: sphericalHarmonicsDegree %u (0..2)", entry, sh_degree);
    return GS_OK;
}

// Step 2's transform (none unless o.has_transform): the doubles k_ksplat_decode<true> bakes into the scene, for the scene's SH range.
static int upload_transform(gs_engine *e, const gs_ksplat_options &o, const gs_ksplat_info &S, DevBuf<KTransform> &d_xf) {
    if (!o.has_transform) return GS_OK;
    KTransform K;
    ksplat_transform_params(o.transform, S.min_sh_coeff, S.max_sh_coeff, K);
    int rc = d_xf.ensure(1);
    if (rc) return rc;
    CU(cudaMemcpyAsync(d_xf.p, &K, sizeof(K), cudaMemcpyHostToDevice, e->stream));
    CU(cudaStreamSynchronize(e->stream));   // pageable source
    return GS_OK;
}

// Step 3: storage formats of the "textures" (SplatMesh.js:1064-1066: SH kept at compression level max(1, file level)).
static int clear_scene(gs_engine *e, const gs_ksplat_options &o, const gs_ksplat_info &S) {
    RasterState &rs = e->rs;
    rs.uploaded = 0;
    e->ray.valid = false;
    rs.cov_format = o.half_covariances ? GS_COV_F16 : GS_COV_F32;
    rs.sh_degree = S.sh_degree;
    rs.sh_format = S.sh_degree ? (S.compression_level == 2 ? GS_SH_U8 : GS_SH_F16) : GS_SH_NONE;
    const size_t n = e->cfg.max_splat_count, ncomp = S.sh_degree == 2 ? 24 : (S.sh_degree == 1 ? 9 : 0);
    int rc;
    if ((rc = rs.cov.ensure(n * (o.half_covariances ? 12 : 24) + 16)) || (ncomp && (rc = rs.sh.ensure(n * ncomp * (rs.sh_format == GS_SH_U8 ? 1 : 2) + 16))))
        return rc;
    return GS_OK;
}

// Step 4: one section of a SplatBuffer image in device memory.  `prefix`: its partial-bucket prefixes (level >= 1); `xf`: the transform
// or nullptr.
static void decode_section(gs_engine *e, const gs_ksplat_options &o, const unsigned char *image, KSectionParams P, const uint32_t *prefix,
                           const KTransform *xf) {
    if (!P.count) return;
    RasterState &rs = e->rs;
    P.sh_degree_out = (int)rs.sh_degree;
    P.minimum_alpha = o.minimum_alpha; P.half_cov = o.half_covariances; P.integer_centers = e->cfg.integer_based_sort; P.write_sort_centers = o.upload_sort_centers;
    const uint32_t grid = (P.count + 127) / 128;
    if (xf) k_ksplat_decode<true><<<grid, 128, 0, e->stream>>>(image, P, prefix, rs.cc.p, rs.cov.p, rs.sh.p, e->centers.p, xf, e->ray.rec.p);
    else k_ksplat_decode<false><<<grid, 128, 0, e->stream>>>(image, P, prefix, rs.cc.p, rs.cov.p, rs.sh.p, e->centers.p, nullptr, e->ray.rec.p);
}

// Step 5, once the decode has completed.  A static mesh's ray records are placed by the scene transform.
static void commit_scene(gs_engine *e, const gs_ksplat_options &o, const gs_ksplat_info &S, gs_ksplat_info *info) {
    e->rs.uploaded = S.splat_count;
    e->rs.have_scene_idx = false;
    if (o.upload_sort_centers) e->uploaded_splats = S.splat_count;
    if (e->ray.rec.p) set_ray_transform(e, o.has_transform ? o.transform : nullptr);
    if (info) *info = S;
}

static uint32_t rd32(const unsigned char *p) { uint32_t v; memcpy(&v, p, 4); return v; }
static uint16_t rd16(const unsigned char *p) { uint16_t v; memcpy(&v, p, 2); return v; }
static float rdf(const unsigned char *p) { float v; memcpy(&v, p, 4); return v; }

struct KsplatLayout {
    gs_ksplat_info info;                // splats, lowest section SH degree, level, sections, centre, SH range
    uint32_t max_splats = 0;            // the header's declared splat count
    std::vector<KSectionParams> secs;   // byte offsets into the image, splat offsets
};

// .ksplat, part 1: the header and the section headers, the first 4096 + 1024 x sections bytes of `f`, checked against the image's size
// `bytes` and the engine's capacity.  The partial-bucket lengths are not read here.
static int parse_ksplat_head(const unsigned char *f, size_t bytes, uint32_t capacity, KsplatLayout &K) {
    if (!f || bytes < 4096) return fail(GS_ERR_BAD_ARG, "gs_upload_ksplat: buffer shorter than the 4096-byte header");
    const uint32_t max_sections = rd32(f + 4), max_splats = rd32(f + 12), level = rd16(f + 20);
    if (f[0] == 0 && f[1] < 1) return fail(GS_ERR_BAD_ARG, "unsupported .ksplat version %u.%u", f[0], f[1]);
    if (level > 2) return fail(GS_ERR_BAD_ARG, ".ksplat compression level %u unknown", level);
    if (max_splats > capacity) return fail(GS_ERR_CAPACITY, ".ksplat holds %u splats, engine capacity %u", max_splats, capacity);
    if (4096ull + 1024ull * max_sections > bytes) return fail(GS_ERR_BAD_ARG, ".ksplat truncated (section headers)");
    static const uint32_t kC[3] = {12, 6, 6}, kS[3] = {12, 6, 6}, kR[3] = {16, 8, 8}, kSH[3] = {4, 2, 1}, kRange[3] = {1, 32767, 32767};
    unsigned long long base = 4096ull + 1024ull * max_sections;
    uint32_t offset = 0, min_degree = 2;
    K.secs.clear();
    for (uint32_t i = 0; i < max_sections; ++i) {
        const unsigned char *h = f + 4096 + 1024ull * i;
        KSectionParams P{};
        P.count = rd32(h + 4);
        P.bucket_size = rd32(h + 8);
        const uint32_t bucket_count = rd32(h + 12);
        const float block = rdf(h + 16);
        const uint32_t storage = rd16(h + 20);
        P.scale_range = rd32(h + 24) ? rd32(h + 24) : kRange[level];
        P.full_bucket_count = rd32(h + 32);
        P.partial_count = rd32(h + 36);
        P.sh_degree_file = rd16(h + 40);
        if (P.sh_degree_file > 2) return fail(GS_ERR_BAD_ARG, ".ksplat section %u: SH degree %d", i, P.sh_degree_file);
        const uint32_t ncomp = P.sh_degree_file == 2 ? 24 : (P.sh_degree_file == 1 ? 9 : 0);
        P.bytes_per_splat = kC[level] + kS[level] + kR[level] + 4 + kSH[level] * ncomp;
        const unsigned long long meta = 4ull * P.partial_count, buckets_bytes = (unsigned long long)storage * bucket_count + meta;
        P.base = base; P.buckets_base = base + meta; P.data_base = base + buckets_bytes;
        P.splat_offset = offset; P.level = (int)level;
        P.scale_factor = ((double)block / 2.0) / (double)P.scale_range;
        if (P.data_base + (unsigned long long)P.bytes_per_splat * P.count > bytes) return fail(GS_ERR_BAD_ARG, ".ksplat truncated (section %u data)", i);
        // an untrusted file must not make the decode kernel read bucket centres or write splats outside its buffers
        if (level >= 1 && P.count) {
            if (P.bucket_size == 0 || storage != 12) return fail(GS_ERR_BAD_ARG, ".ksplat section %u: bucket size %u / bucket storage %u bytes (expected > 0 / 12)", i, P.bucket_size, storage);
            if ((unsigned long long)P.full_bucket_count + P.partial_count > bucket_count) return fail(GS_ERR_BAD_ARG, ".ksplat section %u: %u full + %u partial buckets exceed its %u bucket centres", i, P.full_bucket_count, P.partial_count, bucket_count);
        }
        if (P.data_base > bytes || P.buckets_base > P.data_base) return fail(GS_ERR_BAD_ARG, ".ksplat truncated (section %u buckets)", i);
        min_degree = std::min<uint32_t>(min_degree, (uint32_t)P.sh_degree_file);
        base += (unsigned long long)P.bytes_per_splat * P.count + buckets_bytes;
        offset += P.count;
        K.secs.push_back(P);
    }
    K.max_splats = max_splats;
    K.info = scene_info(offset, K.secs.empty() ? 0 : min_degree, level, (uint32_t)K.secs.size());
    K.info.scene_center[0] = rdf(f + 24); K.info.scene_center[1] = rdf(f + 28); K.info.scene_center[2] = rdf(f + 32);
    const float lo = rdf(f + 36), hi = rdf(f + 40);
    if (lo != 0.f) K.info.min_sh_coeff = lo;   // SplatBuffer.js:833-834
    if (hi != 0.f) K.info.max_sh_coeff = hi;
    return GS_OK;
}

// .ksplat, part 2: lens[i] holds section i's partial_count partial-bucket lengths (u32).  Each section's prefixes [0, l0, l0+l1, ...] are
// appended to `pre`, after checking that its buckets cover its splats and that the sections fit the header's count and the engine.
static int ksplat_prefixes(const KsplatLayout &K, const std::vector<const unsigned char *> &lens, uint32_t capacity, std::vector<uint32_t> &pre) {
    pre.clear();
    for (uint32_t i = 0; i < K.secs.size(); ++i) {
        const KSectionParams &P = K.secs[i];
        const size_t at = pre.size();
        pre.resize(at + P.partial_count + 1, 0);
        uint32_t *q = pre.data() + at;
        for (uint32_t k = 0; k < P.partial_count; ++k) {
            const unsigned long long len = rd32(lens[i] + 4ull * k);
            if (len > P.count) return fail(GS_ERR_BAD_ARG, ".ksplat section %u: partial bucket %u claims %llu splats", i, k, len);
            q[k + 1] = q[k] + (uint32_t)len;
        }
        if (P.level >= 1 && (unsigned long long)P.full_bucket_count * P.bucket_size + q[P.partial_count] < P.count) return fail(GS_ERR_BAD_ARG, ".ksplat section %u: buckets do not cover its splats", i);
        if ((unsigned long long)P.splat_offset + P.count > K.max_splats || (unsigned long long)P.splat_offset + P.count > capacity)
            return fail(GS_ERR_CAPACITY, ".ksplat sections hold more than the %u splats its header declares (engine capacity %u)", K.max_splats, capacity);
    }
    return GS_OK;
}

// Steps 2-5 for a parsed .ksplat image with bucket prefixes `pre`: `d_image` is the image in device memory, else `data` is staged there.
static int upload_ksplat_image(gs_engine *e, const gs_ksplat_options &o, const KsplatLayout &K, const std::vector<uint32_t> &pre, const void *data,
                               size_t bytes, const unsigned char *d_image, gs_ksplat_info *info) {
    int rc;
    cudaStream_t st = e->stream;
    DevBuf<unsigned char> d_file; DevBuf<uint32_t> d_pre; DevBuf<KTransform> d_xf;   // the staged image, the prefixes: this call only
    if ((!d_image && (rc = d_file.ensure(bytes))) || (rc = d_pre.ensure(pre.size())) || (rc = upload_transform(e, o, K.info, d_xf))) return rc;
    if (!d_image) {
        CU(cudaMemcpyAsync(d_file.p, data, bytes, cudaMemcpyHostToDevice, st));   // pageable source: staged before return
        d_image = d_file.p;
    }
    if (!pre.empty()) CU(cudaMemcpyAsync(d_pre.p, pre.data(), pre.size() * 4, cudaMemcpyHostToDevice, st));
    if ((rc = clear_scene(e, o, K.info))) return rc;
    size_t at = 0;
    for (const KSectionParams &P : K.secs) {
        decode_section(e, o, d_image, P, d_pre.p + at, d_xf.p);
        at += P.partial_count + 1;
    }
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    commit_scene(e, o, K.info, info);
    return GS_OK;
}

extern "C" int gs_upload_ksplat(gs_engine *e, const void *data, size_t bytes, const gs_ksplat_options *opt, gs_ksplat_info *info) {
    int rc;
    KsplatLayout K;
    if ((rc = check_scene_engine(e, "gs_upload_ksplat", 0)) || (rc = parse_ksplat_head((const unsigned char *)data, bytes, e->cfg.max_splat_count, K)))
        return rc;
    std::vector<const unsigned char *> lens;
    for (const KSectionParams &P : K.secs) lens.push_back((const unsigned char *)data + P.base);
    std::vector<uint32_t> pre;
    if ((rc = ksplat_prefixes(K, lens, e->cfg.max_splat_count, pre))) return rc;
    return upload_ksplat_image(e, ksplat_options(opt), K, pre, data, bytes, nullptr, info);
}

// ---------------------------------------------------------------------------------------------------------------
// .ply / .splat -> engine (file_parse.h, file_kernels.cuh).  The file is parsed and validated on the host; its records then go through the
// device in chunks: file chunk -> staging buffer -> k_ply_to_level0 / k_splat_to_level0 -> level-0 SplatBuffer records -> k_ksplat_decode.
// Chunking bounds the transient device memory to about 2 x kFileChunkBytes whatever the file's size.
static constexpr size_t kFileChunkBytes = 64u << 20;

extern "C" int gs_probe_file(int format, const void *data, size_t bytes, gs_ksplat_info *info) {
    FileLayout L;
    if (parse_file(format, data, bytes, L, g_err, sizeof(g_err))) return GS_ERR_BAD_ARG;
    if (info) *info = scene_info(L.count, (uint32_t)L.sh_degree, 0, 1);
    return GS_OK;
}

// Step 1 for a file, after check_scene_engine: its header, then its splat count against the engine's capacity.
static int parse_scene_file(const gs_engine *e, int format, const void *data, size_t bytes, FileLayout &L) {
    if (parse_file(format, data, bytes, L, g_err, sizeof(g_err))) return GS_ERR_BAD_ARG;
    if (L.count > e->cfg.max_splat_count) return fail(GS_ERR_CAPACITY, "the file holds %u splats, engine capacity %u", L.count, e->cfg.max_splat_count);
    return GS_OK;
}

// The file's records through the device in chunks: file chunk -> staging buffer -> k_ply_to_level0 / k_pcply_to_level0 / k_splat_to_level0 /
// k_spz_to_level0.
// Level-0 records of `degree` land in the chunk buffer, or (generate mode: `whole` set) at their splat index in `whole` with the
// JavaScript numbers beside them in G.  `prepare()` runs once the transient buffers exist (a failure before it leaves the caller's state
// alone); `after(first, n, records)` runs on the stream after each chunk's parse.
template <typename Prepare, typename After>
static int parse_file_chunks(const FileLayout &L, const void *data, uint32_t degree, cudaStream_t st, Profiler &prof, unsigned char *whole, GenOut G,
                             Prepare prepare, After after) {
    int rc;
    const uint32_t ncomp = degree == 2 ? 24 : (degree == 1 ? 9 : 0), out_bytes = 44 + 4 * ncomp;
    // PlayCanvas-compressed .ply: a splat's sh row lies in a later block than its vertex row.  Chunks are splat ranges of a multiple of
    // 256 splats (whole PLY chunks); each is staged as its vertex rows, then (16-byte aligned) its sh rows when SH are loaded.
    // .spz: chunks are splat ranges too; each plane's slice of the range is staged at a 16-byte-aligned offset (the SH plane only when SH
    // are loaded), so a chunk takes at most SPZ_PLANES x 15 bytes of padding beyond its rows.
    const bool spz = L.format == GS_FILE_SPZ;
    const uint32_t sh_bytes = (L.pc || spz) && degree ? (spz ? 3 * L.spz_sh_coeff : L.pc_sh_stride) : 0;
    const uint32_t row_bytes = L.stride + sh_bytes;
    const size_t pad = spz ? SPZ_PLANES * 16 : 0;
    const size_t unit = L.pc ? kPcChunkSplats : 1;
    const size_t cap = std::max<size_t>(unit, (kFileChunkBytes - pad) / row_bytes / unit * unit);
    const uint32_t chunk_records = (uint32_t)std::min<size_t>(cap, ((size_t)std::max<uint32_t>(L.count, 1) + unit - 1) / unit * unit);
    const size_t chunk_bytes = (size_t)chunk_records * row_bytes + pad;

    DevBuf<unsigned char> d_in, d_l0; DevBuf<double> d_tab; PinBuf<unsigned char> h_in[2];
    struct Events { cudaEvent_t ev[2] = {nullptr, nullptr}; ~Events() { for (cudaEvent_t x : ev) if (x) cudaEventDestroy(x); } } copied;
    if ((rc = d_in.ensure(chunk_bytes + 16)) || (!whole && (rc = d_l0.ensure((size_t)chunk_records * out_bytes)))) return rc;
    if (L.count && ((rc = h_in[0].ensure(chunk_bytes)) || (L.count > chunk_records && (rc = h_in[1].ensure(chunk_bytes))))) return rc;
    for (int i = 0; i < 2; ++i) CU(cudaEventCreateWithFlags(&copied.ev[i], cudaEventDisableTiming));
    if (L.pc && L.count) {   // the chunk table: 18 extremes per 256 splats, as f64
        const std::vector<double> tab = file_detail::pc_chunk_table((const unsigned char *)data, L);
        if ((rc = d_tab.ensure(tab.size()))) return rc;
        CU(cudaMemcpyAsync(d_tab.p, tab.data(), tab.size() * sizeof(double), cudaMemcpyHostToDevice, st));
        CU(cudaStreamSynchronize(st));   // pageable source
    }
    const size_t pc_smem = (size_t)kPcChunkSplats * row_bytes;   // a CTA's vertex + sh rows
    // the dynamic shared memory a launch may request without opting in: 48 KiB less the kernel's static extremes table
    cudaFuncAttributes pc_fa{};
    if (L.pc) CU(cudaFuncGetAttributes(&pc_fa, k_pcply_to_level0<true>));
    const bool pc_staged = pc_smem <= (size_t)pc_fa.maxDynamicSharedSizeBytes;
    rc = prepare();
    if (rc) return rc;

    PlyKernelParams PP{};
    PP.stride = L.stride; PP.out_bytes = out_bytes; PP.sh_out = (int)degree; PP.sh_per_channel = L.sh_per_channel;
    memcpy(PP.offset, L.offset, sizeof(PP.offset)); memcpy(PP.type, L.type, sizeof(PP.type));
    // records per CTA: the largest of 128 / 64 / 32 whose block fits the default 48 KiB of shared memory; larger records are read in place
    uint32_t cta = 128;
    while (cta > 32 && (size_t)cta * L.stride > (48u << 10)) cta >>= 1;
    const bool ply_smem = (size_t)cta * L.stride <= (48u << 10);
    if (!ply_smem) cta = 128;
    PcKernelParams CP{};
    CP.stride = L.stride; CP.sh_stride = sh_bytes; CP.out_bytes = out_bytes; CP.sh_out = (int)degree; CP.color_mask = L.pc_color_mask;
    static const uint32_t kShCoeff[4] = {0, 3, 8, 15};   // decompressSphericalHarmonics' shCoeffMap
    CP.read_coeff = kShCoeff[L.pc_sh_file_degree];
    memcpy(CP.packed, L.pc_packed, sizeof(CP.packed));
    SpzKernelParams SP{};
    SP.out_bytes = out_bytes; SP.sh_out = (int)degree; SP.sh_coeff = L.spz_sh_coeff; SP.version = L.spz_version; SP.pos_scale = L.spz_pos_scale;
    const uint32_t spz_bytes[SPZ_PLANES] = {L.stride - 10, 1, 3, 3, 3, sh_bytes};   // per splat and plane; no SH plane when none are loaded
    const unsigned char *src_sh = (const unsigned char *)data + L.pc_sh_offset;
    const unsigned char *src = (const unsigned char *)data + L.data_offset;
    for (uint32_t first = 0, k = 0; first < L.count; first += chunk_records, ++k) {
        const uint32_t n = std::min(chunk_records, L.count - first);
        const size_t split = L.pc ? ((size_t)n * L.stride + 15) & ~(size_t)15 : (size_t)n * L.stride;   // PlayCanvas: sh rows start here
        size_t nb = split + (size_t)n * sh_bytes;
        PinBuf<unsigned char> &h = h_in[k & 1];
        // the pinned buffer is refilled on the host while the device works on the previous chunk
        if (k >= 2) CU(cudaEventSynchronize(copied.ev[k & 1]));
        if (spz) {
            nb = 0;
            for (int p = 0; p < SPZ_PLANES; ++p) {
                SP.plane[p] = (uint32_t)nb;
                memcpy(h.p + nb, (const unsigned char *)data + L.spz_plane[p] + (size_t)first * spz_bytes[p], (size_t)n * spz_bytes[p]);
                nb = (nb + (size_t)n * spz_bytes[p] + 15) & ~(size_t)15;
            }
        } else {
            memcpy(h.p, src + (size_t)first * L.stride, (size_t)n * L.stride);
            if (sh_bytes) memcpy(h.p + split, src_sh + (size_t)first * sh_bytes, (size_t)n * sh_bytes);
        }
        CU(cudaMemcpyAsync(d_in.p, h.p, nb, cudaMemcpyHostToDevice, st));
        CU(cudaEventRecord(copied.ev[k & 1], st));
        prof.mark("h2d_file_chunk", st);
        const uint32_t grid = (n + cta - 1) / cta;
        PP.count = n;
        CP.count = n; CP.chunk_base = first / kPcChunkSplats;
        SP.count = n;
        const uint32_t pc_grid = (n + kPcChunkSplats - 1) / kPcChunkSplats;
        // GEN (std::true_type / std::false_type): generate mode, the records of the whole scene in `whole` with the numbers beside them
        auto to_level0 = [&](auto gen, unsigned char *o, GenOut g) {
            constexpr bool GEN = decltype(gen)::value;
            if (spz) k_spz_to_level0<GEN><<<(n + 127) / 128, 128, 0, st>>>(d_in.p, SP, o, g);
            else if (L.format == GS_FILE_SPLAT) k_splat_to_level0<GEN><<<(n + 127) / 128, 128, 0, st>>>(d_in.p, n, o, g);
            else if (L.pc && pc_staged) k_pcply_to_level0<true, GEN><<<pc_grid, kPcChunkSplats, pc_smem, st>>>(d_in.p, d_in.p + split, d_tab.p, CP, o, g);
            else if (L.pc) k_pcply_to_level0<false, GEN><<<pc_grid, kPcChunkSplats, 0, st>>>(d_in.p, d_in.p + split, d_tab.p, CP, o, g);
            else if (ply_smem) k_ply_to_level0<true, GEN><<<grid, cta, cta * L.stride, st>>>(d_in.p, PP, o, g);
            else k_ply_to_level0<false, GEN><<<grid, cta, 0, st>>>(d_in.p, PP, o, g);
        };
        if (whole) to_level0(std::true_type{}, whole + (size_t)first * out_bytes, GenOut{G.center + (size_t)first * 3, G.sh ? G.sh + (size_t)first * ncomp : nullptr});
        else to_level0(std::false_type{}, d_l0.p, GenOut{});
        prof.mark(spz ? "k_spz_to_level0" : L.format == GS_FILE_SPLAT ? "k_splat_to_level0" : (L.pc ? "k_pcply_to_level0" : "k_ply_to_level0"), st);
        CU(cudaGetLastError());
        if ((rc = after(first, n, whole ? whole + (size_t)first * out_bytes : d_l0.p))) return rc;
    }
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    return GS_OK;
}

extern "C" int gs_upload_file(gs_engine *e, int format, const void *data, size_t bytes, uint32_t sh_degree, const gs_ksplat_options *opt,
                              gs_ksplat_info *info) {
    int rc;
    FileLayout L;
    if ((rc = check_scene_engine(e, "gs_upload_file", sh_degree)) || (rc = parse_scene_file(e, format, data, bytes, L))) return rc;
    const gs_ksplat_options o = ksplat_options(opt);
    const uint32_t degree = std::min<uint32_t>(sh_degree, (uint32_t)L.sh_degree);   // min(sphericalHarmonicsDegree, file degree)
    const gs_ksplat_info S = scene_info(L.count, degree, 0, 1);
    KSectionParams KP{};   // each chunk of records is one level-0 section
    KP.level = 0; KP.bytes_per_splat = 44 + 4 * (degree == 2 ? 24 : (degree == 1 ? 9 : 0)); KP.sh_degree_file = (int)degree; KP.scale_range = 1;
    DevBuf<KTransform> d_xf;
    cudaStream_t st = e->stream;
    // parse_file_chunks allocates the transient buffers before it calls `prepare`
    auto prepare = [&]() -> int {
        int r;
        if ((r = upload_transform(e, o, S, d_xf)) || (r = clear_scene(e, o, S))) return r;
        e->prof.begin(st);   // gs_set_profiling: per-chunk timeline of the copy and the two kernels (tools/load_bench.py)
        return GS_OK;
    };
    rc = parse_file_chunks(L, data, degree, st, e->prof, nullptr, GenOut{}, prepare, [&](uint32_t first, uint32_t n, const unsigned char *d_l0) -> int {
        KP.count = n; KP.splat_offset = first;
        decode_section(e, o, d_l0, KP, nullptr, d_xf.p);
        e->prof.mark("k_ksplat_decode", st);
        CU(cudaGetLastError());
        return GS_OK;
    });
    if (rc) return rc;
    commit_scene(e, o, S, info);
    return GS_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// SplatBufferGenerator.getStandardGenerator on the device (generate_kernels.cuh): the file is parsed in generate mode into whole-scene
// level-0 records plus f64 centres and SH, then partitioned, filtered, bucketed and written as a .ksplat image in device memory.  The
// host writes only the 4096-byte header and the 1024-byte section headers, from scalars the device reduced.
struct GenImage {
    DevBuf<unsigned char> image;
    size_t bytes = 0;
    uint32_t splats = 0, sections = 0, level = 0;
    std::vector<unsigned char> head;                        // header + section headers, as written into the image
};

// Stable LSD sort of `order` (n entries, nullptr = identity) by a 64-bit key indexed by element, `bits` low bits, in 24-bit rounds.
struct GenSort {
    DevBuf<uint32_t> keys[2], vals[3], tile_hist;
    DevBuf<SortControl> ctl;
    int run(const unsigned long long *key, const uint32_t *order, uint32_t n, int bits, uint32_t *out, cudaStream_t st, uint32_t &launches) {
        int rc;
        uint32_t stride = 0;
        if ((rc = keys[0].ensure(n)) || (rc = keys[1].ensure(n)) || (rc = vals[0].ensure(n)) || (rc = vals[1].ensure(n)) || (rc = vals[2].ensure(n)) ||
            (rc = tile_hist.ensure(radix_tile_hist_words(std::max(n, 1u), 3, &stride))))
            return rc;
        if (!ctl.p) {
            if ((rc = ctl.ensure(1))) return rc;
            CU(cudaMemsetAsync(ctl.p, 0, sizeof(SortControl), st));   // the scatter passes clear their histograms again (self_clean)
        }
        static const RadixNames names{{"gen_hist0", "gen_hist1", "gen_hist2", "gen_hist3"}, {"gen_scan0", "gen_scan1", "gen_scan2", "gen_scan3"},
                                      {"gen_scatter0", "gen_scatter1", "gen_scatter2", "gen_scatter3"}};
        if (n == 0) return GS_OK;
        const int rounds = std::max(1, (bits + 23) / 24);
        for (int r = 0; r < rounds; ++r) {
            const PassPlan pl = make_plan_bits(std::min(24, bits - 24 * r));
            // k_gen_sort_piece consumes `order` before the passes write `dst`, so the two may be the same buffer
            uint32_t *dst = (r == rounds - 1) ? out : vals[2].p;
            k_gen_sort_piece<<<(n + 255) / 256, 256, 0, st>>>(key, order, n, 24 * r, keys[0].p, vals[0].p);
            ++launches;
            radix_sort_pairs<uint32_t, uint32_t>(keys[0].p, keys[1].p, vals[0].p, 0, kValArray, vals[1].p, vals[0].p, dst, n, nullptr, 0, pl,
                                                 ctl.p, tile_hist.p, stride, false, nullptr, st, launches, nullptr, names, true);
            order = dst;
        }
        return GS_OK;
    }
};

// out[0..n]: exclusive scan of in[0..n), out[n] = total
static int gen_scan(const uint32_t *in, uint32_t n, uint32_t *out, DevBuf<uint32_t> &sums, cudaStream_t st, uint32_t &launches) {
    int rc;
    const uint32_t tiles = (uint32_t)(((uint64_t)n + kScanTile - 1) / kScanTile);
    if ((rc = sums.ensure(tiles + 1))) return rc;
    CU(cudaMemsetAsync(sums.p + tiles, 0, 4, st));
    if (tiles) k_gen_scan_reduce<<<tiles, kScanThreads, 0, st>>>(in, n, sums.p);
    k_exclusive_scan_single_block<<<1, 1024, 0, st>>>(sums.p, tiles + 1);
    if (tiles) k_gen_scan_apply<<<tiles, kScanThreads, 0, st>>>(in, n, sums.p, tiles, out);
    else CU(cudaMemsetAsync(out, 0, 4, st));
    launches += tiles ? 3 : 1;
    return GS_OK;
}

static int check_generate_options(const gs_generate_options *gen, gs_generate_options &g) {
    gs_generate_options d{};
    d.compression_level = 1; d.minimum_alpha = 1;   // SplatBufferGenerator.getStandardGenerator's defaults
    g = read_options(gen, d);
    if (g.bucket_size == 0) g.bucket_size = 256;
    if (g.block_size == 0.0) g.block_size = 5.0;
    if (g.compression_level > 2) return fail(GS_ERR_BAD_ARG, "generate: compression level %u (0..2)", g.compression_level);
    if (!(g.block_size > 0.0) || !std::isfinite(g.block_size)) return fail(GS_ERR_BAD_ARG, "generate: block size %g (finite, > 0)", g.block_size);
    if (g.bucket_size > 0x80000000u) return fail(GS_ERR_BAD_ARG, "generate: bucket size %u (<= 2^31)", g.bucket_size);
    return GS_OK;
}

static void put32(unsigned char *p, uint32_t v) { memcpy(p, &v, 4); }
static void put16(unsigned char *p, uint16_t v) { memcpy(p, &v, 2); }
static void putf(unsigned char *p, float v) { memcpy(p, &v, 4); }

static int generate_image(const FileLayout &L, const void *data, uint32_t sh_degree, const gs_generate_options &g, cudaStream_t st, Profiler &prof,
                          GenImage &out, uint32_t &launches) {
    int rc;
    const uint32_t degree = std::min<uint32_t>(sh_degree, (uint32_t)L.sh_degree);
    const uint32_t ncomp = degree == 2 ? 24 : (degree == 1 ? 9 : 0), rec_bytes = 44 + 4 * ncomp, n = L.count;
    const uint32_t level = g.compression_level, B = g.bucket_size;
    static const uint32_t kBytes[3] = {44, 24, 24}, kSH[3] = {4, 2, 1};
    const uint32_t bps = kBytes[level] + kSH[level] * ncomp;
    // SplatPartitioner: sections of section_size splats in partition order (0 or more than the splats: one); no splats, no sections
    const uint32_t S = (g.section_size == 0 || g.section_size > n) ? n : g.section_size;
    const uint32_t nsec = n ? (uint32_t)(((uint64_t)n + S - 1) / S) : 0;

    DevBuf<unsigned char> rec0; DevBuf<double> c64, sh64, bcenter, bucket_center, range;
    DevBuf<unsigned long long> key, lo, hi, bmin, bmax, pkey_lo, pkey_hi, offs;
    DevBuf<uint32_t> perm, keep, kscan, src, sec, sec_base, nanf, order, head, gscan, gstart, complete, fscan, fbase, pflag, pscan, plist, porder, pinv,
        plen, pcount, pbase, pprefix, bbase, out_src, out_bucket, sums;
    DevBuf<GenGeom> geom; DevBuf<ShRun> runs;
    GenSort sorter;
    if ((rc = rec0.ensure((size_t)n * rec_bytes)) || (rc = c64.ensure((size_t)n * 3)) || (ncomp && (rc = sh64.ensure((size_t)n * ncomp)))) return rc;
    rc = parse_file_chunks(L, data, degree, st, prof, rec0.p, GenOut{c64.p, ncomp ? sh64.p : nullptr}, [] { return GS_OK; },
                           [](uint32_t, uint32_t, const unsigned char *) { return GS_OK; });
    if (rc) return rc;
    const uint32_t grid_n = (n + kGenThreads - 1) / kGenThreads;
    // ---- partition order
    if ((rc = key.ensure(n)) || (rc = perm.ensure(n))) return rc;
    if (n) k_gen_partition_key<<<grid_n, kGenThreads, 0, st>>>(c64.p, n, g.scene_center[0], g.scene_center[1], g.scene_center[2], key.p);
    if ((rc = sorter.run(key.p, nullptr, n, 64, perm.p, st, launches))) return rc;
    prof.mark("gen_partition", st);
    // ---- SH range over FRC0..FRC22 of every splat, partition order
    const uint32_t sh_blocks = (uint32_t)(((uint64_t)n + kGenThreads * kGenShItems - 1) / (kGenThreads * kGenShItems));
    if ((rc = range.ensure(2)) || (rc = runs.ensure(2 * (size_t)std::max(sh_blocks, 1u)))) return rc;
    if (ncomp && sh_blocks) k_gen_sh_scan<<<sh_blocks, kGenThreads, 0, st>>>(sh64.p, (int)ncomp, (int)std::min(ncomp, 23u), perm.p, n, runs.p);
    k_gen_sh_final<<<1, 1, 0, st>>>(runs.p, ncomp ? sh_blocks : 0, range.p);
    prof.mark("gen_sh_range", st);
    // ---- alpha removal
    if ((rc = keep.ensure(n)) || (rc = kscan.ensure((size_t)n + 1)) || (rc = src.ensure(n)) || (rc = sec.ensure(n)) || (rc = sec_base.ensure((size_t)nsec + 1)))
        return rc;
    if (n) k_gen_keep<<<grid_n, kGenThreads, 0, st>>>(rec0.p, rec_bytes, perm.p, n, g.minimum_alpha, keep.p);
    if ((rc = gen_scan(keep.p, n, kscan.p, sums, st, launches))) return rc;
    if (n) k_gen_compact<<<grid_n, kGenThreads, 0, st>>>(perm.p, keep.p, kscan.p, n, std::max(S, 1u), src.p, sec.p);
    k_gen_section_base<<<nsec / 256 + 1, 256, 0, st>>>(kscan.p, n, std::max(S, 1u), nsec, sec_base.p);
    uint32_t m = 0;
    CU(cudaMemcpyAsync(&m, kscan.p + n, 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    prof.mark("gen_alpha", st);
    const uint32_t grid_m = (m + kGenThreads - 1) / kGenThreads, grid_s = nsec / 256 + 1;
    // ---- bounds and bucket keys per section
    if ((rc = bmin.ensure((size_t)nsec * 3 + 1)) || (rc = bmax.ensure((size_t)nsec * 3 + 1)) || (rc = nanf.ensure((size_t)nsec * 3 + 1)) ||
        (rc = geom.ensure((size_t)nsec + 1)) || (rc = lo.ensure(m)) || (rc = hi.ensure(m)) || (rc = bcenter.ensure((size_t)m * 3)) || (rc = order.ensure(m)))
        return rc;
    CU(cudaMemsetAsync(bmin.p, 0xff, ((size_t)nsec * 3 + 1) * 8, st));
    CU(cudaMemsetAsync(bmax.p, 0, ((size_t)nsec * 3 + 1) * 8, st));
    CU(cudaMemsetAsync(nanf.p, 0, ((size_t)nsec * 3 + 1) * 4, st));
    if (m) {
        k_gen_bounds<<<grid_m, kGenThreads, 0, st>>>(c64.p, src.p, sec.p, sec_base.p, m, bmin.p, bmax.p, nanf.p);
        k_gen_geometry<<<grid_s, 256, 0, st>>>(bmin.p, bmax.p, nanf.p, sec_base.p, nsec, g.block_size, geom.p);
        k_gen_bucket_key<<<grid_m, kGenThreads, 0, st>>>(c64.p, src.p, sec.p, geom.p, m, g.block_size, lo.p, hi.p, bcenter.p);
    }
    int sec_bits = 1;
    while (sec_bits < 40 && (1ull << sec_bits) < 2ull * nsec) ++sec_bits;
    if ((rc = sorter.run(lo.p, nullptr, m, 64, order.p, st, launches)) || (rc = sorter.run(hi.p, order.p, m, sec_bits, order.p, st, launches))) return rc;
    prof.mark("gen_bucket_sort", st);
    // ---- groups of equal (section, key), bucket fill
    if ((rc = head.ensure(m)) || (rc = gscan.ensure((size_t)m + 1)) || (rc = complete.ensure(m)) || (rc = fscan.ensure((size_t)m + 1)) ||
        (rc = fbase.ensure((size_t)nsec + 1)))
        return rc;
    if (m) k_gen_heads<<<grid_m, kGenThreads, 0, st>>>(lo.p, hi.p, order.p, m, head.p);
    if ((rc = gen_scan(head.p, m, gscan.p, sums, st, launches))) return rc;
    uint32_t groups = 0;
    CU(cudaMemcpyAsync(&groups, gscan.p + m, 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if ((rc = gstart.ensure((size_t)groups + 1)) || (rc = pflag.ensure(groups)) || (rc = pscan.ensure((size_t)groups + 1)) || (rc = pkey_lo.ensure(groups)) ||
        (rc = pkey_hi.ensure(groups)) || (rc = pinv.ensure(groups)))
        return rc;
    k_gen_group_start<<<grid_m + 1, kGenThreads, 0, st>>>(head.p, gscan.p, m, gstart.p);
    if (m) k_gen_complete<<<grid_m, kGenThreads, 0, st>>>(order.p, gscan.p, gstart.p, m, B, complete.p);
    if ((rc = gen_scan(complete.p, m, fscan.p, sums, st, launches))) return rc;
    k_gen_gather_base<<<grid_s, 256, 0, st>>>(fscan.p, sec_base.p, nsec, fbase.p);
    // ---- partial buckets: order within each section, lengths, counts
    const uint32_t grid_g = (groups + kGenThreads - 1) / kGenThreads;
    if (groups) k_gen_partial_keys<<<grid_g, kGenThreads, 0, st>>>(order.p, gstart.p, groups, B, hi.p, pflag.p, pkey_lo.p, pkey_hi.p);
    if ((rc = gen_scan(pflag.p, groups, pscan.p, sums, st, launches))) return rc;
    uint32_t np = 0;
    CU(cudaMemcpyAsync(&np, pscan.p + groups, 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if ((rc = plist.ensure(np)) || (rc = porder.ensure(np)) || (rc = plen.ensure(np)) || (rc = pprefix.ensure((size_t)np + 1)) || (rc = pcount.ensure((size_t)nsec + 1)) ||
        (rc = pbase.ensure((size_t)nsec + 1)) || (rc = bbase.ensure((size_t)nsec + 1)))
        return rc;
    if (groups) k_gen_partial_list<<<grid_g, kGenThreads, 0, st>>>(pflag.p, pscan.p, groups, plist.p);
    if ((rc = sorter.run(pkey_lo.p, plist.p, np, 32, porder.p, st, launches)) || (rc = sorter.run(pkey_hi.p, porder.p, np, sec_bits, porder.p, st, launches))) return rc;
    CU(cudaMemsetAsync(pcount.p, 0, ((size_t)nsec + 1) * 4, st));
    if (np) k_gen_partial_info<<<(np + kGenThreads - 1) / kGenThreads, kGenThreads, 0, st>>>(porder.p, np, gstart.p, B, pkey_hi.p, pinv.p, plen.p, pcount.p);
    if ((rc = gen_scan(pcount.p, nsec, pbase.p, sums, st, launches)) || (rc = gen_scan(plen.p, np, pprefix.p, sums, st, launches))) return rc;
    const GenLayout GL{sec_base.p, fbase.p, pbase.p, pprefix.p};
    k_gen_bucket_base<<<grid_s, 256, 0, st>>>(GL, nsec, bbase.p);
    // ---- output slots and bucket centres
    std::vector<uint32_t> h_sec((size_t)nsec + 1), h_f((size_t)nsec + 1), h_p((size_t)nsec + 1);
    CU(cudaMemcpyAsync(h_sec.data(), sec_base.p, h_sec.size() * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(h_f.data(), fbase.p, h_f.size() * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(h_p.data(), pbase.p, h_p.size() * 4, cudaMemcpyDeviceToHost, st));
    double h_range[2] = {0, 0};
    CU(cudaMemcpyAsync(h_range, range.p, 16, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    const uint32_t nbuckets = h_f[nsec] + h_p[nsec];
    if ((rc = out_src.ensure(m)) || (rc = out_bucket.ensure(m)) || (rc = bucket_center.ensure((size_t)nbuckets * 3))) return rc;
    if (m) k_gen_slots<<<grid_m, kGenThreads, 0, st>>>(order.p, gscan.p, gstart.p, fscan.p, pinv.p, src.p, sec.p, bcenter.p, m, B, GL, out_src.p, out_bucket.p,
                                                       bucket_center.p);
    prof.mark("gen_buckets", st);
    // ---- layout (SplatBuffer.js:1228-1243, 1297-1324): header, section headers, then per section [partial lengths, bucket centres] and splats
    std::vector<unsigned long long> h_offs(2 * (size_t)nsec + 1);   // [data offset per section][metadata offset per section]
    std::vector<unsigned char> head_bytes(4096 + 1024 * (size_t)nsec, 0);
    unsigned long long at = head_bytes.size();
    for (uint32_t s = 0; s < nsec; ++s) {
        const uint32_t ms = h_sec[s + 1] - h_sec[s], fs = h_f[s + 1] - h_f[s], ps = h_p[s + 1] - h_p[s];
        const unsigned long long meta = level >= 1 ? 12ull * (fs + ps) + 4ull * ps : 0ull, size = meta + (unsigned long long)ms * bps;
        if (size > 0xffffffffull) return fail(GS_ERR_CAPACITY, "generate: section %u would hold %llu bytes (its header stores 32 bits)", s, size);
        h_offs[nsec + s] = at;
        h_offs[s] = at + meta;
        at += size;
        unsigned char *h = head_bytes.data() + 4096 + 1024ull * s;   // writeSectionHeaderToBuffer
        put32(h + 0, ms); put32(h + 4, ms);
        if (level >= 1) {
            put32(h + 8, B); put32(h + 12, fs + ps); putf(h + 16, (float)g.block_size); put16(h + 20, 12); put32(h + 24, 32767);
            put32(h + 32, fs); put32(h + 36, ps);
        }
        put32(h + 28, (uint32_t)size);
        put16(h + 40, (uint16_t)degree);
    }
    unsigned char *h = head_bytes.data();   // writeHeaderToBuffer
    h[0] = 0; h[1] = 1;
    put32(h + 4, nsec); put32(h + 8, nsec); put32(h + 12, m); put32(h + 16, m); put16(h + 20, (uint16_t)level);
    putf(h + 24, (float)g.scene_center[0]); putf(h + 28, (float)g.scene_center[1]); putf(h + 32, (float)g.scene_center[2]);
    putf(h + 36, (float)h_range[0]); putf(h + 40, (float)h_range[1]);
    if ((rc = out.image.ensure(at)) || (rc = offs.ensure(h_offs.size()))) return rc;
    CU(cudaMemcpyAsync(out.image.p, head_bytes.data(), head_bytes.size(), cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(offs.p, h_offs.data(), h_offs.size() * 8, cudaMemcpyHostToDevice, st));
    GenWriteParams WP{};
    WP.m = m; WP.nsec = nsec; WP.level = level; WP.ncomp = ncomp; WP.in_bytes = rec_bytes; WP.out_bytes = bps;
    WP.scale_range = 32767.0; WP.scale_factor = 32767.0 / (g.block_size * 0.5);
    if (m) k_gen_write<<<grid_m, kGenThreads, 0, st>>>(rec0.p, c64.p, ncomp ? sh64.p : nullptr, out_src.p, out_bucket.p, bucket_center.p, sec_base.p, offs.p,
                                                       range.p, WP, out.image.p);
    const uint32_t nmeta = std::max(nbuckets, h_p[nsec]);
    if (level >= 1 && nmeta)
        k_gen_bucket_meta<<<(nmeta + 255) / 256, 256, 0, st>>>(bucket_center.p, plen.p, GL, nsec, nbuckets, h_p[nsec], offs.p + nsec, bbase.p, out.image.p);
    prof.mark("gen_write", st);
    CU(cudaStreamSynchronize(st));   // the host buffers above are pageable
    CU(cudaGetLastError());
    out.bytes = at; out.splats = m; out.sections = nsec; out.level = level;
    out.head = std::move(head_bytes);
    return GS_OK;
}

static int generate_to_host(const FileLayout &L, const void *data, uint32_t sh_degree, const gs_generate_options &g, void **image, size_t *image_bytes) {
    cudaStream_t st = nullptr;
    CU(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    struct Stream { cudaStream_t s; ~Stream() { cudaStreamDestroy(s); } } stream{st};
    GenImage out;
    Profiler prof;
    uint32_t launches = 0;
    int rc = generate_image(L, data, sh_degree, g, st, prof, out, launches);
    if (rc) return rc;
    void *h = nullptr;
    CU(cudaHostAlloc(&h, std::max<size_t>(out.bytes, 1), cudaHostAllocDefault));
    cudaError_t ce = cudaMemcpyAsync(h, out.image.p, out.bytes, cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
    if (ce != cudaSuccess) { cudaFreeHost(h); return fail(GS_ERR_CUDA, "gs_generate_splat_buffer: image read-back -> %s", cudaGetErrorString(ce)); }
    *image = h; *image_bytes = out.bytes;
    return GS_OK;
}

extern "C" int gs_generate_splat_buffer(int device, int format, const void *data, size_t bytes, uint32_t sh_degree, const gs_generate_options *gen,
                                        void **image, size_t *image_bytes) {
    if (!image || !image_bytes) return fail(GS_ERR_BAD_ARG, "gs_generate_splat_buffer: null output");
    *image = nullptr; *image_bytes = 0;
    if (sh_degree > 2) return fail(GS_ERR_BAD_ARG, "gs_generate_splat_buffer: sphericalHarmonicsDegree %u (0..2)", sh_degree);
    gs_generate_options g;
    int rc;
    if ((rc = check_generate_options(gen, g))) return rc;
    FileLayout L;
    if (parse_file(format, data, bytes, L, g_err, sizeof(g_err))) return GS_ERR_BAD_ARG;
    if (device < 0 || device >= gs_device_count()) return fail(GS_ERR_NO_DEVICE, "gs_generate_splat_buffer: no CUDA device %d", device);
    int prev = 0;
    CU(cudaGetDevice(&prev));   // the caller's current device is restored on every return
    CU(cudaSetDevice(device));
    rc = generate_to_host(L, data, sh_degree, g, image, image_bytes);
    cudaSetDevice(prev);
    return rc;
}

extern "C" int gs_upload_file_optimized(gs_engine *e, int format, const void *data, size_t bytes, uint32_t sh_degree, const gs_ksplat_options *opt,
                                        const gs_generate_options *gen, gs_ksplat_info *info) {
    int rc;
    gs_generate_options g;
    FileLayout L;
    if ((rc = check_scene_engine(e, "gs_upload_file_optimized", sh_degree)) || (rc = check_generate_options(gen, g)) ||
        (rc = parse_scene_file(e, format, data, bytes, L)))
        return rc;
    GenImage out;
    uint32_t launches = 0;
    e->prof.begin(e->stream);   // gs_set_profiling: the generation's timeline (tools/load_bench.py --optimize)
    if ((rc = generate_image(L, data, sh_degree, g, e->stream, e->prof, out, launches))) return rc;
    // The image is decoded in place; of its bytes the host reads only the headers, which it wrote, and the partial-bucket lengths.
    KsplatLayout K;
    if ((rc = parse_ksplat_head(out.head.data(), out.bytes, e->cfg.max_splat_count, K))) return rc;
    size_t nlens = 0;
    for (const KSectionParams &P : K.secs) nlens += P.partial_count;
    std::vector<uint32_t> h_lens(nlens);
    std::vector<const unsigned char *> lens;
    size_t at = 0;
    for (const KSectionParams &P : K.secs) {
        if (P.partial_count) CU(cudaMemcpyAsync(h_lens.data() + at, out.image.p + P.base, 4ull * P.partial_count, cudaMemcpyDeviceToHost, e->stream));
        lens.push_back((const unsigned char *)(h_lens.data() + at));
        at += P.partial_count;
    }
    CU(cudaStreamSynchronize(e->stream));
    std::vector<uint32_t> pre;
    if ((rc = ksplat_prefixes(K, lens, e->cfg.max_splat_count, pre))) return rc;
    return upload_ksplat_image(e, ksplat_options(opt), K, pre, nullptr, out.bytes, out.image.p, info);
}

// Debug / test read-back of an engine buffer (see gs_buffer_id) into host memory.
extern "C" int gs_read_buffer(gs_engine *e, int id, void *out, size_t offset, size_t bytes) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!out) return fail(GS_ERR_BAD_ARG, "gs_read_buffer: null");
    const unsigned char *p = nullptr; size_t cap = 0;
    switch (id) {
        case GS_BUF_CENTERS_COLORS: p = (const unsigned char *)e->rs.cc.p; cap = e->rs.cc.n * 16; break;
        case GS_BUF_COVARIANCES: p = e->rs.cov.p; cap = e->rs.cov.n; break;
        case GS_BUF_SH: p = e->rs.sh.p; cap = e->rs.sh.n; break;
        case GS_BUF_RAY_RECORDS: p = (const unsigned char *)e->ray.rec.p; cap = e->ray.rec.n * sizeof(gs_ray_record); break;
        default: { void *q = nullptr; if ((rc = gs_buffer_dev(e, id, &q, &cap))) return rc; p = (const unsigned char *)q; }
    }
    if (!p || offset + bytes > cap) return fail(GS_ERR_CAPACITY, "gs_read_buffer: [%zu,%zu) outside the %zu-byte buffer", offset, offset + bytes, cap);
    CU(cudaMemcpyAsync(out, p + offset, bytes, cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    return GS_OK;
}

extern "C" int gs_read_projected(gs_engine *e, gs_projected_splat *out, uint32_t count) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!out) return fail(GS_ERR_BAD_ARG, "gs_read_projected: null");
    rc = raster_read_projected(e->rs, out, count, e->stream);
    if (rc) return rc;
    CU(cudaStreamSynchronize(e->stream));
    return GS_OK;
}

extern "C" int gs_buffer_dev(gs_engine *e, int id, void **ptr, size_t *bytes) {
    if (!e || !ptr) return fail(GS_ERR_BAD_ARG, "gs_buffer_dev: null");
    size_t b = 0;
    switch (id) {
        case GS_BUF_SORTED_INDEXES: *ptr = e->sorted.p; b = e->sorted.n * 4; break;
        case GS_BUF_FRAME: *ptr = raster_frame_ptr(e->rs, e->rs.last_format); b = e->rs.last_frame_bytes; break;
        case GS_BUF_CENTERS: *ptr = e->centers.p; b = e->centers.n * 16; break;
        case GS_BUF_DISTANCES: *ptr = e->dist.p; b = e->dist.n * 4; break;
        case GS_BUF_SPLAT_RECORDS: *ptr = e->rs.records.p; b = e->rs.records.n * sizeof(SplatRecord); break;
        case GS_BUF_INDEXES_TO_SORT: *ptr = e->indexes.p; b = e->indexes.n * 4; break;
        default: return fail(GS_ERR_BAD_ARG, "unknown buffer id %d", id);
    }
    if (bytes) *bytes = b;
    return GS_OK;
}
extern "C" int gs_stream(gs_engine *e, void **s) {
    if (!e || !s) return fail(GS_ERR_BAD_ARG, "gs_stream: null");
    *s = (void *)e->stream;
    return GS_OK;
}
extern "C" int gs_synchronize(gs_engine *e) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (e->pending_async) { // collect errors + timings of the last asynchronous frame
        e->pending_async = false;
        int rc2 = finish_render(e, &e->pending_rp, nullptr);
        rc = finish_sort(e, nullptr);
        return rc ? rc : rc2;
    }
    CU(cudaStreamSynchronize(e->stream));
    return GS_OK;
}

// ---- measurement helpers (bench hygiene; no effect on results) -------------------------------------------------------
__global__ void k_flush_l2(uint32_t *buf, size_t words, uint32_t v) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += (size_t)gridDim.x * blockDim.x) buf[i] = v;
}
extern "C" int gs_flush_l2(gs_engine *e) { // overwrite a buffer of 4x the device's L2 on the engine's stream
    int rc = check_engine(e);
    if (rc) return rc;
    const size_t words = 4 * e->l2_bytes / 4;
    if ((rc = e->flush.ensure(words))) return rc;
    static uint32_t tick = 0;
    k_flush_l2<<<e->sm_count * 8, 512, 0, e->stream>>>(e->flush.p, words, ++tick);
    CU(cudaGetLastError());
    return GS_OK;
}
// ---- fused tile gather: rank 0's frame buffer + handshake block shared with the other ranks through CUDA IPC -------------------------
extern "C" int gs_peer_export(gs_engine *e, void *frame_handle, void *sync_handle) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!frame_handle || !sync_handle) return fail(GS_ERR_BAD_ARG, "gs_peer_export: null");
    if (e->cfg.world_size < 2 || e->cfg.rank != 0) return fail(GS_ERR_BAD_ARG, "gs_peer_export: only rank 0 of a multi-GPU group exports");
    if (!e->rs.frame.p) return fail(GS_ERR_NOT_READY, "engine created without a framebuffer");
    if ((rc = e->rs.peer_sync_local.ensure(1))) return rc;
    CU(cudaMemset(e->rs.peer_sync_local.p, 0, sizeof(PeerSync)));
    // Double the exported allocation: pipelined frames (gs_frame_begin) then alternate between its halves, so the picture of frame f
    // leaves over PCIe while the peers already store frame f+1 into the other half.  Which half a frame uses travels in the release
    // word.  Every rank sizes its own frame buffer from the same gs_config, so the peers know where the second half starts.
    // GS_PEER_DOUBLE=0 keeps one buffer.
    const char *pd = getenv("GS_PEER_DOUBLE");
    if (!(pd && pd[0] == '0') && !e->rs.frame_half2 && !e->pipe_inflight()) {
        CU(cudaStreamSynchronize(e->stream));
        const size_t half = e->rs.frame.n;
        e->rs.frame.release();
        if ((rc = e->rs.frame.ensure(2 * half))) return rc;
        CU(cudaMemset(e->rs.frame.p, 0, 2 * half));
        e->rs.frame_half2 = e->rs.frame.p + half;
        e->rs.frame_half_bytes = half;
    }
    static_assert(sizeof(cudaIpcMemHandle_t) == GS_IPC_HANDLE_BYTES, "IPC handle size");
    cudaIpcMemHandle_t h;
    CU(cudaIpcGetMemHandle(&h, e->rs.frame.p));
    memcpy(frame_handle, &h, sizeof(h));
    CU(cudaIpcGetMemHandle(&h, e->rs.peer_sync_local.p));
    memcpy(sync_handle, &h, sizeof(h));
    CU(cudaMemset(&e->rs.rctl.p->frame_seq, 0, 4));   // ranks count frames in lockstep from here on
    e->rs.peer_sync = e->rs.peer_sync_local.p;
    e->rs.peer_root = true;
    if (e->graph_exec) { cudaGraphExecDestroy(e->graph_exec); e->graph_exec = nullptr; }
    if (e->graph_exec_alt) { cudaGraphExecDestroy(e->graph_exec_alt); e->graph_exec_alt = nullptr; }
    return GS_OK;
}
extern "C" int gs_peer_attach(gs_engine *e, const void *frame_handle, const void *sync_handle) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!frame_handle || !sync_handle) return fail(GS_ERR_BAD_ARG, "gs_peer_attach: null");
    if (e->cfg.world_size < 2 || e->cfg.rank == 0) return fail(GS_ERR_BAD_ARG, "gs_peer_attach: only ranks > 0 of a multi-GPU group attach");
    cudaIpcMemHandle_t h;
    void *pf = nullptr, *ps = nullptr;
    memcpy(&h, frame_handle, sizeof(h));
    CU(cudaIpcOpenMemHandle(&pf, h, cudaIpcMemLazyEnablePeerAccess));
    memcpy(&h, sync_handle, sizeof(h));
    CU(cudaIpcOpenMemHandle(&ps, h, cudaIpcMemLazyEnablePeerAccess));
    CU(cudaMemset(&e->rs.rctl.p->frame_seq, 0, 4));
    e->rs.peer_frame = pf;
    e->rs.peer_sync = (PeerSync *)ps;
    e->rs.peer_attached = true;
    if (e->graph_exec) { cudaGraphExecDestroy(e->graph_exec); e->graph_exec = nullptr; }
    return GS_OK;
}

extern "C" int gs_set_graph_enabled(gs_engine *e, int on) {
    if (!e) return fail(GS_ERR_BAD_ARG, "gs_set_graph_enabled: null");
    e->graph_enabled = on != 0;
    return GS_OK;
}
extern "C" int gs_set_profiling(gs_engine *e, int on) {
    if (!e) return fail(GS_ERR_BAD_ARG, "gs_set_profiling: null");
    e->prof.on = on != 0;
    return GS_OK;
}
// Per-kernel device times of the last sort / render / frame (call after gs_synchronize or a blocking entry).
extern "C" int gs_kernel_timings(gs_engine *e, gs_kernel_time *out, uint32_t capacity, uint32_t *count) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!count) return fail(GS_ERR_BAD_ARG, "gs_kernel_timings: null");
    CU(cudaStreamSynchronize(e->stream));
    uint32_t n = 0;
    for (size_t i = 1; i < e->prof.used; ++i) {
        if (n < capacity && out) {
            float ms = 0.f;
            cudaEventElapsedTime(&ms, e->prof.ev[i - 1], e->prof.ev[i]);
            strncpy(out[n].name, e->prof.names[i], sizeof(out[n].name) - 1);
            out[n].name[sizeof(out[n].name) - 1] = 0;
            out[n].ms = ms;
        }
        ++n;
    }
    *count = n;
    return GS_OK;
}
extern "C" int gs_event_create(void **ev) {
    if (!ev) return fail(GS_ERR_BAD_ARG, "gs_event_create: null");
    cudaEvent_t x;
    CU(cudaEventCreate(&x));
    *ev = (void *)x;
    return GS_OK;
}
extern "C" int gs_event_record(gs_engine *e, void *ev) {
    int rc = check_engine(e);
    if (rc) return rc;
    CU(cudaEventRecord((cudaEvent_t)ev, e->stream));
    return GS_OK;
}
extern "C" int gs_event_elapsed_ms(void *ev0, void *ev1, float *ms) {
    if (!ms) return fail(GS_ERR_BAD_ARG, "gs_event_elapsed_ms: null");
    CU(cudaEventSynchronize((cudaEvent_t)ev1));
    CU(cudaEventElapsedTime(ms, (cudaEvent_t)ev0, (cudaEvent_t)ev1));
    return GS_OK;
}
extern "C" int gs_event_destroy(void *ev) {
    if (ev) CU(cudaEventDestroy((cudaEvent_t)ev));
    return GS_OK;
}
extern "C" int gs_last_timings(gs_engine *e, gs_timings *t) {
    if (!e || !t) return fail(GS_ERR_BAD_ARG, "gs_last_timings: null");
    *t = e->tm;
    return GS_OK;
}

// pinned host memory for callers (the SharedArrayBuffer views a shared-memory worker hands out, SortWorker.js:180-191)
extern "C" int gs_host_alloc(void **ptr, size_t bytes) {
    if (!ptr) return fail(GS_ERR_BAD_ARG, "gs_host_alloc: null");
    if (gs_device_count() <= 0) return fail(GS_ERR_NO_DEVICE, "no CUDA device");
    CU(cudaHostAlloc(ptr, std::max<size_t>(bytes, 1), cudaHostAllocDefault));
    return GS_OK;
}
extern "C" int gs_host_free(void *ptr) {
    if (ptr) CU(cudaFreeHost(ptr));
    return GS_OK;
}
