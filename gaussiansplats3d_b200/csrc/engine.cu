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
#include "tree_kernels.cuh"
#include "ray_kernels.cuh"
#include "generate_kernels.cuh"
#include "region_kernels.cuh"

#include <algorithm>
#include <cmath>
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

// Pinned host memory that the blocking calls read their device-side results back into
struct HostStatus {
    FrameStatus frame;                 // gs_sort, gs_render, gs_frame, gs_synchronize
    unsigned long long gather_total;   // gs_gather_for_sort: indexes gathered
    uint32_t ray_counts[2];            // gs_raycast: leaves reached, hits
    ShardHeader shard;                 // gs_sort_sharded_finish: this rank's exchange block
};

// What a frame graph's kernels were captured with (enqueue_frame): a frame replays its parity's graph only when every field is equal
struct GraphKey {
    const void *indexes, *cov, *sh;   // the sort's index list (nullptr: identity) and the splats' covariance and SH buffers
    uint32_t render_count, sort_count;                  // the sort's
    uint32_t frame_render_count, width, height, frame_format, flip_y;
    uint32_t precomputed, eyes, scene_idx, depth, composite, subset;
    uint32_t views;                                     // a multi-view frame's view count; 0: mono or stereo
    uint32_t cov_format, sh_format, sh_degree, uploaded;
    bool operator==(const GraphKey &o) const { return memcmp(this, &o, sizeof(*this)) == 0; }
};
static_assert(std::has_unique_object_representations_v<GraphKey>, "GraphKey is compared bytewise: it must have no padding");

// The CUDA graph of one frame (sort + render), one per frame-buffer parity (the target frame buffer is captured), replayed while its key
// is unchanged
struct FrameGraph {
    struct Slot {
        cudaGraphExec_t exec = nullptr;
        GraphKey key{};
        bool snapshot = false;        // its blend writes the status snapshot (gs_frame_begin)
    } slot[2];
    uint32_t launches = 0;            // kernels in the graph captured last
    std::vector<cudaGraphExec_t> retired;   // graphs replaced while in a peer group on one device (see capture)
    cudaStream_t side = nullptr;      // second capture branch (projection beside the depth sort)
    cudaEvent_t fork = nullptr, join = nullptr;

    FrameGraph() = default;
    FrameGraph(const FrameGraph &) = delete;
    FrameGraph &operator=(const FrameGraph &) = delete;
    ~FrameGraph() {
        drop();
        for (cudaGraphExec_t g : retired) cudaGraphExecDestroy(g);
        for (cudaEvent_t x : {fork, join}) if (x) cudaEventDestroy(x);
        if (side) cudaStreamDestroy(side);
    }
    bool current(int parity, const GraphKey &key) const { return slot[parity].exec && slot[parity].key == key; }
    // Captures enqueue(side, join), forked onto `side` and joined back through `join`, on st as the graph of `parity`.  retire: a peer
    // group on one device keeps the replaced graph (destroying it frees device memory, which waits for the whole device, and the peers
    // enqueued before this engine may be spinning in their handshake until this frame releases them).
    template <typename F> int capture(int parity, const GraphKey &key, bool retire, cudaStream_t st, F &&enqueue) {
        Slot &s = slot[parity];
        if (s.exec) { if (retire) retired.push_back(s.exec); else cudaGraphExecDestroy(s.exec); s.exec = nullptr; }
        CU(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        struct Guard {   // an early error return ends the capture and discards it
            cudaStream_t st; bool armed;
            ~Guard() { if (armed) { cudaGraph_t g = nullptr; cudaStreamEndCapture(st, &g); if (g) cudaGraphDestroy(g); (void)cudaGetLastError(); } }
        } guard{st, true};
        CU(cudaEventRecord(fork, st));
        CU(cudaStreamWaitEvent(side, fork, 0));
        if (int rc = enqueue(side, join)) return rc;
        CU(cudaGetLastError());
        guard.armed = false;
        cudaGraph_t g = nullptr;
        cudaError_t ce = cudaStreamEndCapture(st, &g);
        if (ce != cudaSuccess) return fail(GS_ERR_CUDA, "cudaStreamEndCapture -> %s", cudaGetErrorString(ce));
        ce = cudaGraphInstantiate(&s.exec, g, 0);
        cudaGraphDestroy(g);
        if (ce != cudaSuccess) { s.exec = nullptr; return fail(GS_ERR_CUDA, "cudaGraphInstantiate -> %s", cudaGetErrorString(ce)); }
        s.key = key;
        return GS_OK;
    }
    // Destroys both graphs, for a change their keys do not see (buffers they captured are replaced)
    void drop() { for (Slot &s : slot) if (s.exec) { cudaGraphExecDestroy(s.exec); s.exec = nullptr; } }
};

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
    RadixSort<uint32_t, uint32_t> sorter;   // depth-sort scratch: keys sized in u32 words, read as u16 or u32 by key_bits
    DevBuf<uint32_t> sorted;         // sortedIndexes
    DevBuf<float> transforms;        // 32 x mat4
    DevBuf<SortControl> ctl;
    DevBuf<DepthParams> depthp;      // per-frame depth parameters (device copy read by k_depth)
    DevBuf<uint32_t> freq;           // scratch reproduction for gs_sort_indexes
    DevBuf<int32_t> dist_rows_i;     // gs_compute_distances: per-scene integer / float rows
    DevBuf<float> dist_rows_f;
    DevBuf<uint32_t> sub_idx;        // sharded frames: this rank's subset of the sort input (index, distance)
    DevBuf<int32_t> sub_dist;
    uint32_t uploaded_splats = 0;    // 'uploadedSplatCount' SortWorker.js:97
    bool scenes_multi = false;       // the mesh holds several scenes of one gs_upload_scenes
    std::vector<uint32_t> scene_start;   // with scenes_multi: scene s holds splats [scene_start[s], scene_start[s + 1])
    uint32_t baked_xf = 0;           // bit s: scene s was decoded with a transform, which its f32 centres carry (has_transform)
    uint32_t last_render_count = 0;
    bool have_sorted = false;
    bool ctl_dirty = true;           // SortControl needs k_sort_init (first sort / after a failed one); otherwise the sort leaves it clean

    // pinned staging (the shared-memory views of SortWorker.js:180-191)
    PinBuf<uint32_t> h_indexes, h_sorted;
    PinBuf<HostStatus> h_status;
    PinBuf<unsigned char> h_frame;

    // --- rasteriser state ---
    RasterState rs;

    // Multi-view frames (gs_frame_views): every view's camera, distances and min/max, and the views' draw orders [view][render_count]
    // from one sort of all views' keys.  Sized for `views` views by the first frame that has that many.
    struct ViewSort {
        uint32_t views = 0;
        DevBuf<DepthParams> depthp;      // [GS_MAX_VIEWS]
        DevBuf<SortControl> ctl;         // [views]: view v's min/max; ctl[0] also the sort's digit totals and error bits
        DevBuf<int32_t> dist;            // [views][max_splat_count]
        DevBuf<uint32_t> sorted;         // [views][render_count]: the draw orders
        DevBuf<uint32_t> window;         // partial sorts: the views' sorted windows before k_views_assemble
        RadixSort<uint32_t, uint32_t> sorter;
    };
    std::unique_ptr<ViewSort> vsort;

    gs_timings tm{};
    Profiler prof;
    FrameGraph graph;
    bool graph_enabled = true;
    bool last_frame_was_graph = false;
    bool pending_async = false;
    DevBuf<uint32_t> flush;          // L2 flush scratch (bench hygiene)
    DevBuf<unsigned long long> region_max;   // gs_visible_region's result
    DevBuf<double> bounds_xf;                // gs_compute_bounding_box: the call's transforms, its CTAs' keys and the box
    DevBuf<unsigned long long> bounds_partial;
    DevBuf<float> bounds_out;
    // SplatTree leaves (gs_upload_splat_tree / gs_build_splat_tree) and the scratch of gs_gather_for_sort
    struct Tree {
        DevBuf<double> center, nmin, nmax;
        DevBuf<uint32_t> offsets, indexes, start;
        DevBuf<unsigned long long> key, total;
        uint32_t count = 0, splats = 0;
        DevBuf<int32_t> depth;       // per leaf; only a tree built here has it
        bool have_depth = false;
        gs_splat_tree_info built{};  // what the last gs_build_splat_tree reported (zero for an uploaded tree)
        // The scene's ray records were written by the GPU decode.  The build then takes its centres from them: getSplatCenter's value
        // exactly, which the texel centre is not for a level-1/2 section under a transform (rounded to f32 before the transform) nor for
        // a non-finite centre without one (the reference still multiplies by the identity: 0 * inf = NaN).
        bool decoded_ray_records = false;
        // every node (gs_upload_splat_tree_nodes): the raycast's box tests
        DevBuf<double> all_min, all_max;
        DevBuf<int32_t> parent;
        DevBuf<uint32_t> leaf_node;
        uint32_t node_count = 0;
        bool have_nodes = false;     // nodes uploaded for the current leaves
        // A forest (gs_build_splat_tree on a dynamic mesh of several scenes): sub-tree s, scene s's, holds leaves
        // [sub_leaf[s], sub_leaf[s + 1]) and nodes [sub_node[s], sub_node[s + 1]) (host copies; device copies for the cull and the
        // raycast).  Any other tree is one sub-tree and keeps neither.
        uint32_t sub_trees = 1;
        std::vector<uint32_t> h_sub_leaf, h_sub_node;
        DevBuf<uint32_t> sub_leaf, sub_node;
        DevBuf<double> mvs;          // gs_gather_for_sort_subtrees: the call's model views
    } tree;
    // gs_raycast: per-splat records (ray_records engines only) and the call's scratch, allocated on first use
    struct Ray {
        DevBuf<gs_ray_record> rec;
        bool valid = false;          // the records describe the current scene
        DevBuf<double> xf;           // static mesh: each SplatScene's transform, f64[16 * GS_MAX_SCENES]
        bool per_scene = false;      // a record's scene is its splat's rasteriser scene index (else every record is scene 0)
        DevBuf<RaySetup> setup;      // one per sub-tree
        DevBuf<double> fl;           // a forest cast's sub_tree_from_local
        DevBuf<uint8_t> pass;
        DevBuf<uint32_t> reached, list, counts;
        DevBuf<RayHit> hits;
        PiecewiseSort sort;          // by (distance, traversal position); the final order stays in sort.order
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
    DevBuf<FrameStatus> status_dev;                // one snapshot slot per frame-buffer parity
    PinBuf<FrameStatus> h_pipe;                    // kPipeRing slots, one read back per pipelined frame
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
        if (rs.peer_attached && !rs.peer_local) { if (rs.peer_frame) cudaIpcCloseMemHandle(rs.peer_frame); if (rs.peer_sync) cudaIpcCloseMemHandle(rs.peer_sync); }
        for (cudaEvent_t x : ev) if (x) cudaEventDestroy(x);
        for (int i = 0; i < kPipeRing; ++i) { if (ev_frame_done[i]) cudaEventDestroy(ev_frame_done[i]); if (ev_copy_done[i]) cudaEventDestroy(ev_copy_done[i]); }
        for (cudaEvent_t x : {ev_params[0], ev_params[1]}) if (x) cudaEventDestroy(x);
        for (cudaStream_t x : {stream, copy_stream, param_stream}) if (x) cudaStreamDestroy(x);
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
    CU(cudaStreamCreateWithFlags(&e->graph.side, cudaStreamNonBlocking));
    CU(cudaEventCreateWithFlags(&e->graph.fork, cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&e->graph.join, cudaEventDisableTiming));
    for (int i = 0; i < EV_COUNT; ++i) CU(cudaEventCreate(&e->ev[i]));
    int kb = 0;
    while ((1u << kb) < c.distance_map_range) ++kb;
    e->key_bits = kb;
    int rc = GS_OK;
    const size_t n = std::max<uint32_t>(c.max_splat_count, 1);
    if ((rc = e->centers.ensure(n)) || (rc = e->indexes.ensure(n)) || (rc = e->dist.ensure(n)) || (rc = e->sorted.ensure(n)) ||
        (rc = e->sorter.reserve(n, make_plan_bits(kb).npasses)) || (rc = e->ctl.ensure(1)) || (rc = e->depthp.ensure(2)) || (rc = e->transforms.ensure(16 * GS_MAX_SCENES)) || (rc = e->h_status.ensure(1)))
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
    if ((rc = e->status_dev.ensure(2))) return rc;
    CU(cudaMemset(e->status_dev.p, 0, 2 * sizeof(FrameStatus)));
    e->rs.snap_slots = e->status_dev.p;
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
    e->scenes_multi = false;
    e->scene_start.clear();
    if (count) CU(cudaMemcpyAsync(e->centers.p + from, centers, (size_t)count * 16, cudaMemcpyHostToDevice, e->stream));
    if (e->cfg.dynamic_mode && sceneIndexes && count)
        CU(cudaMemcpyAsync(e->scene_idx.p + from, sceneIndexes, (size_t)count * 4, cudaMemcpyHostToDevice, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    e->uploaded_splats = from + count; // SortWorker.js:97
    return GS_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// SortWorker.js:99-100: the counts are clamped to what has been uploaded
static int clamp_counts(const gs_engine *e, gs_sort_params &q) {
    q.render_count = std::min(q.render_count, e->uploaded_splats);
    q.sort_count = std::min(q.sort_count, e->uploaded_splats);
    if (q.sort_count > q.render_count) return fail(GS_ERR_BAD_ARG, "sortCount %u > renderCount %u", q.sort_count, q.render_count);
    return GS_OK;
}

// The camera rows every depth mode reads
static DepthParams depth_params(const float *mvp) {
    DepthParams P{};
    memcpy(P.mvp, mvp, 64);
    P.irow[0] = (int32_t)((double)mvp[2] * 1000.0);   // sorter.cpp:64 -- f64 product, truncation toward zero
    P.irow[1] = (int32_t)((double)mvp[6] * 1000.0);
    P.irow[2] = (int32_t)((double)mvp[10] * 1000.0);
    P.irow[3] = 1;
    P.frow[0] = mvp[2]; P.frow[1] = mvp[6]; P.frow[2] = mvp[10]; P.frow[3] = 0.f;
    return P;
}

// The mono sort's camera -> the depth parameters of the frame's parity (pageable source: staged before return)
static int upload_camera(gs_engine *e, const float *mvp, cudaStream_t st) {
    const DepthParams P = depth_params(mvp);
    CU(cudaMemcpyAsync(e->depthp.p + e->rs.frame_parity, &P, sizeof(P), cudaMemcpyHostToDevice, st));
    return GS_OK;
}

// A sort's launches, eager or captured into a frame graph.  An eager sort records the stage events (mark), uploads its cameras and runs
// k_sort_init when the control block is dirty; a captured sort leaves all three to the code that launches its graph (enqueue_frame,
// upload_frame_params).
struct SortLaunch {
    Launch launch;
    cudaEvent_t *ev;                  // the engine's stage events; nullptr: the sort is being captured
    bool eager() const { return ev != nullptr; }
    cudaError_t mark(int stage) const { return ev ? cudaEventRecord(ev[stage], launch.stream()) : cudaSuccess; }
    // a sort without keys (sort_count 0) still closes its depth and bucket stages
    cudaError_t no_keys() const { const cudaError_t ce = mark(EV_DEPTH); return ce != cudaSuccess ? ce : mark(EV_BUCKET); }
};

// The depth pass (sorter.cpp:29-140) over positions [lo, hi) of the index list: dist[i] and the running min/max in the control block.
// views = 0: the mono sort's; otherwise the multi-view sort's, every view at once (blockIdx.y) into its own distances and control block.
static int depth_pass(gs_engine *e, const Launch &launch, const uint32_t *d_indexes, const gs_sort_params &q, uint32_t lo, uint32_t hi, uint32_t views) {
    const bool integer = e->cfg.integer_based_sort, dyn = e->cfg.dynamic_mode;
    const int mode = q.use_precomputed_distances ? (integer ? kIntPrecomputed : kFloatPrecomputed)
                                                 : (integer ? (dyn ? kIntDynamic : kIntStatic) : (dyn ? kFloatDynamic : kFloatStatic));
    const int dblocks = (int)std::max<uint64_t>(1, std::min<uint64_t>(((uint64_t)(hi - lo) + kDepthThreads * kDepthItems - 1) / (kDepthThreads * kDepthItems), (uint64_t)e->sm_count * 8));
    gs_engine::ViewSort *w = views ? e->vsort.get() : nullptr;
    bool found = false;
    for_each_depth([&](int m, bool identity, bool multi, auto kernel) {
        if (m != mode || identity != (d_indexes == nullptr) || multi != (w != nullptr)) return;
        launch.pdl("k_depth", kernel, dim3(dblocks, w ? views : 1), kDepthThreads, 0, d_indexes, e->centers.p, e->precomputed.p, e->scene_idx.p, e->transforms.p,
                   w ? w->depthp.p : e->depthp.p + e->rs.frame_parity, lo, hi, w ? w->dist.p : e->dist.p, w ? w->ctl.p : e->ctl.p);
        found = true;
    });
    return found ? GS_OK : fail(GS_ERR_BAD_ARG, "depth pass: no k_depth variant for mode %d, %u views", mode, views);
}

// The start of every mono sort: EV_SORT0, the profiler timeline, k_sort_init when the control block is dirty (first sort, or the
// previous one failed part-way; a completed sort leaves it clean), and k_copy_head for the unsorted positions [0, s0)
static int sort_prologue(gs_engine *e, const SortLaunch &sl, const uint32_t *d_indexes, uint32_t s0, bool open_timeline = true) {
    CU(sl.mark(EV_SORT0));
    if (open_timeline) e->prof.begin(sl.launch.stream());
    if (sl.eager()) {
        if (e->ctl_dirty) sl.launch.pdl(nullptr, k_sort_init, 1, 256, 0, e->ctl.p);
        e->ctl_dirty = true;
    }
    if (s0 > 0) sl.launch.pdl("k_copy_head", k_copy_head, std::min<uint32_t>((s0 + 255) / 256, e->sm_count * 8), 256, 0, d_indexes, e->sorted.p, s0);
    return GS_OK;
}

// The depth sort of positions [lo, hi) of the index list (nullptr: identity) by k_bucket's keys: values from the end of the slice
static RadixJob<uint32_t> depth_job(gs_engine *e, const uint32_t *d_indexes, uint32_t lo, uint32_t hi, uint32_t *out, RadixTag tag) {
    RadixJob<uint32_t> j;
    j.vals = d_indexes ? d_indexes + lo : nullptr; j.valmode = d_indexes ? kValArrayReversed : kValIotaReversed; j.iota_top = hi - 1u;
    j.out = out; j.n_cap = j.n = hi - lo; j.plan = make_plan_bits(e->key_bits); j.ctl = e->ctl.p;
    j.hist0_done = j.self_clean = true; j.tag = tag;
    return j;
}

// What a mono sort does beyond gs_sort's
struct SortOptions {
    bool write_buckets = false;             // keep every key in dist (gs_sort_indexes' mappedDistances and frequencies)
    bool open_timeline = true;              // false: the caller has opened the profiler timeline
    bool subset = false;                    // this rank sorts only the splats that reach its tiles, which needs this frame's projection
    cudaEvent_t wait_for_rects = nullptr;   // subset: the event after that projection, when it runs on another stream
};

// The sort proper on the launch's stream, everything already on the device.  d_indexes == nullptr: identity.
template <typename KeyT>
static int sort_keyed(gs_engine *e, const SortLaunch &sl, const uint32_t *d_indexes, const gs_sort_params &q, const SortOptions &o) {
    const Launch &launch = sl.launch;
    cudaStream_t st = launch.stream();
    const uint32_t render_count = q.render_count, n = q.sort_count, s0 = render_count - n;
    if (render_count > e->cfg.max_splat_count) return fail(GS_ERR_CAPACITY, "renderCount %u > max_splat_count %u", render_count, e->cfg.max_splat_count);
    int rc = sort_prologue(e, sl, d_indexes, s0, o.open_timeline);
    if (rc) return rc;
    if (n > 0) {
        if ((sl.eager() && (rc = upload_camera(e, q.model_view_proj, st))) || (rc = depth_pass(e, launch, d_indexes, q, s0, render_count, 0))) return rc;
        CU(sl.mark(EV_DEPTH));
        RadixJob<uint32_t> j = depth_job(e, d_indexes, s0, render_count, e->sorted.p + s0, kTagDepth);
        int32_t *dist_sorted = e->dist.p + s0;
        if (o.subset) {   // bucketed with the GLOBAL min/max found by k_depth above
            if (o.wait_for_rects) CU(cudaStreamWaitEvent(st, o.wait_for_rects, 0));
            if ((rc = raster_subset(e->rs, e->cfg, d_indexes, render_count, e->dist.p, e->sub_idx.p, e->sub_dist.p, launch))) return rc;
            j.vals = e->sub_idx.p; j.valmode = kValArrayReversed;
            dist_sorted = e->sub_dist.p;
            j.n_dev = &e->rs.view[0].rctl.p->subset_count;
        }
        if ((rc = e->sorter.bucket<KeyT>(j, dist_sorted, e->cfg.distance_map_range, o.write_buckets, launch))) return rc;
        CU(sl.mark(EV_BUCKET));
        if ((rc = e->sorter.sort<KeyT>(j, launch))) return rc;
    } else CU(sl.no_keys());
    CU(sl.mark(EV_SORT1));
    CU(cudaGetLastError());
    e->last_render_count = render_count;
    e->have_sorted = true;
    if (sl.eager()) e->ctl_dirty = false;
    return GS_OK;
}
static int sort_on_device(gs_engine *e, const SortLaunch &sl, const uint32_t *d_indexes, const gs_sort_params &q, const SortOptions &o = {}) {
    return e->key_bits <= 16 ? sort_keyed<uint16_t>(e, sl, d_indexes, q, o) : sort_keyed<uint32_t>(e, sl, d_indexes, q, o);
}

// The multi-view sort's passes: the depth sort's over the bucket bits, then one over the view index above them
static PassPlan views_plan(int key_bits, uint32_t nviews) {
    PassPlan pl = make_plan_bits(key_bits);
    int view_bits = 0;
    while ((1u << view_bits) < nviews) ++view_bits;
    if (view_bits) { pl.shift[pl.npasses] = key_bits; pl.bits[pl.npasses] = view_bits; ++pl.npasses; }
    return pl;
}

// Sizes the multi-view sort for `views` views.  The buffers are replaced as a whole, so a failed reservation leaves the previous ones;
// frame graphs captured with those are dropped.
static int reserve_view_sort(gs_engine *e, uint32_t views) {
    if (e->vsort && e->vsort->views >= views) return GS_OK;
    std::unique_ptr<gs_engine::ViewSort> w(new (std::nothrow) gs_engine::ViewSort());
    if (!w) return fail(GS_ERR_BAD_ARG, "out of host memory");
    const size_t n = std::max<uint32_t>(e->cfg.max_splat_count, 1), vn = views * n;
    int rc;
    if ((rc = w->depthp.ensure(GS_MAX_VIEWS)) || (rc = w->ctl.ensure(views)) || (rc = w->dist.ensure(vn)) || (rc = w->sorted.ensure(vn)) ||
        (rc = w->window.ensure(vn)) || (rc = w->sorter.reserve(vn, views_plan(e->key_bits, views).npasses)))
        return rc;
    w->views = views;
    e->graph.drop();
    e->vsort = std::move(w);
    return GS_OK;
}

// The depth plane of the frame's parity, on the first frame that asks for depth (before any graph is captured with it): a stereo frame
// is at most max_width wide and a multi-view frame's stacked bands at most max_height tall
static int reserve_depth(gs_engine *e, const gs_render_params &p) {
    return p.depth ? e->rs.depth[e->rs.frame_parity].ensure((size_t)e->cfg.max_width * e->cfg.max_height) : GS_OK;
}

// After a frame with depth is enqueued (a replayed graph as well as a captured or eager one): GS_BUF_DEPTH is its plane
static void note_depth(gs_engine *e, const gs_render_params &p, const FrameViews &fv) {
    if (!p.depth) return;
    e->rs.last_depth_parity = e->rs.frame_parity;
    e->rs.last_depth_bytes = (fv.stacked() ? (size_t)fv.count : 1u) * p.width * p.height * sizeof(float);
}

// Reserves the views of a stereo or multi-view frame before anything of it is enqueued (see raster_reserve_views)
static int reserve_views(gs_engine *e, const FrameViews &fv) {
    bool moved = false;
    int rc = raster_reserve_views(e->rs, e->cfg, fv.count, &moved);
    if (moved) e->graph.drop();
    if (rc || !fv.stacked()) return rc;
    return reserve_view_sort(e, fv.count);
}

// Every view's sort camera (gs_view.model_view_proj) -> the multi-view depth pass's parameter blocks (pageable source: staged before return)
static int upload_view_cameras(gs_engine *e, const FrameViews &fv, cudaStream_t st) {
    DepthParams P[GS_MAX_VIEWS];
    for (uint32_t v = 0; v < fv.count; ++v) P[v] = depth_params(fv.cams[v].model_view_proj);
    CU(cudaMemcpyAsync(e->vsort->depthp.p, P, fv.count * sizeof(DepthParams), cudaMemcpyHostToDevice, st));
    return GS_OK;
}

// The multi-view sort (gs_frame_views): for every view, what sort_keyed computes for that view's camera alone, in one set of launches.
// The depth pass runs every view (blockIdx.y), k_bucket_views keys each view's window with its own range and the view index above the
// bucket, and one stable radix sort of the views' keys leaves view v's order in sorted[v render_count ...].  The control blocks start
// every sort fresh (k_sort_init_views).  A captured sort's cameras are uploaded before its graph runs (upload_frame_params).
static int sort_views(gs_engine *e, const SortLaunch &sl, const uint32_t *d_indexes, const gs_sort_params &q, const FrameViews &fv) {
    const Launch &launch = sl.launch;
    gs_engine::ViewSort &w = *e->vsort;
    const uint32_t nviews = fv.count, render_count = q.render_count, n = q.sort_count, s0 = render_count - n;
    int rc;
    if (sl.eager() && (rc = upload_view_cameras(e, fv, launch.stream()))) return rc;
    CU(sl.mark(EV_SORT0));
    launch.plain("k_sort_init_views", k_sort_init_views, nviews, 256, 0, w.ctl.p);
    if (n > 0) {
        if ((rc = depth_pass(e, launch, d_indexes, q, s0, render_count, nviews))) return rc;
        CU(sl.mark(EV_DEPTH));
        RadixJob<uint32_t> j;
        j.vals = w.sorter.vals[0].p; j.valmode = kValArray;
        j.out = s0 ? w.window.p : w.sorted.p; j.n_cap = j.n = n * nviews; j.plan = views_plan(e->key_bits, nviews); j.ctl = w.ctl.p;
        j.hist0_done = j.self_clean = true; j.tag = kTagDepth;
        if ((rc = w.sorter.check(j))) return rc;
        const uint32_t tiles = (n * nviews + kRadixTile - 1) / kRadixTile;
        launch.plain("k_bucket_views", k_bucket_views, tiles, kRadixThreads, 0, w.dist.p, s0, render_count, d_indexes, nviews, e->cfg.distance_map_range, e->key_bits,
                   j.plan, w.ctl.p, w.sorter.keys[0].p, w.sorter.vals[0].p, w.sorter.tile_hist.p, RadixSort<uint32_t, uint32_t>::stride(j.n));
        CU(sl.mark(EV_BUCKET));
        if ((rc = w.sorter.sort<uint32_t>(j, launch))) return rc;
    } else CU(sl.no_keys());
    if (s0 > 0)
        launch.plain("k_views_assemble", k_views_assemble, dim3(std::min<uint32_t>((render_count + 255) / 256, e->sm_count * 8), nviews), 256, 0, d_indexes, w.window.p, s0,
                   render_count, w.sorted.p);
    CU(sl.mark(EV_SORT1));
    CU(cudaGetLastError());
    return GS_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// The end of a blocking call.  `parts` says what it enqueued: a sort, a render, or both (a frame), and whether it staged inputs
// between EV_H2D0 and EV_H2D1 (stage_sort_inputs).
enum { kSortPart = 1, kRenderPart = 2, kCopyIn = 4 };

// Folds a read-back status into the engine's counters and returns the call's status.  A bucket index out of range is reported
// before a peer timeout, and that before an instance-list overflow.
static int frame_status(gs_engine *e, const FrameStatus &s, int parts) {
    if (parts & kRenderPart) {
        e->tm.tile_instances = s.raster.total_instances;
        uint32_t vis = 0;
        for (int i = 0; i < kVisibleSlots; ++i) vis += s.raster.visible_slots[i * 8];
        e->tm.visible_splats = vis;
    }
    if ((parts & kSortPart) && (s.sort[2] & kErrBucketRange))
        return fail(GS_ERR_BUCKET_RANGE, "a bucket index fell outside [0,%u): distances overflow the int32/f32 range map", e->cfg.distance_map_range);
    if (!(parts & kRenderPart)) return GS_OK;
    if (s.raster.peer_timeout) return fail(GS_ERR_CUDA, "multi-GPU tile gather: a peer did not arrive within the time limit (ranks must render the same frames)");
    if (s.raster.overflow) return fail(GS_ERR_CAPACITY, "tile-instance buffer overflow: %llu instances needed, capacity %llu (raise GS_INSTANCE_FACTOR)",
                                       (unsigned long long)s.raster.total_instances, (unsigned long long)e->rs.instance_capacity);
    return GS_OK;
}

// Reads the status back, waits for the stream, and folds the stage and copy timings and the status into the engine.  The call has
// copied its results back through copy_out.  sort_ctl: the control block whose error bits the sort left (a multi-view sort's; nullptr:
// the engine's).
static int finish_call(gs_engine *e, int parts, float *sort_time_ms = nullptr, const SortControl *sort_ctl = nullptr) {
    cudaStream_t st = e->stream;
    FrameStatus &s = e->h_status.p->frame;
    if (parts & kRenderPart) CU(cudaMemcpyAsync(&s.raster, e->rs.view[0].rctl.p, sizeof(RasterControl), cudaMemcpyDeviceToHost, st));
    if (parts & kSortPart) CU(cudaMemcpyAsync(s.sort, sort_ctl ? sort_ctl : e->ctl.p, kSortHeadBytes, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    gs_timings &t = e->tm;
    const bool graph = e->last_frame_was_graph;   // one graph launch: only the whole-frame time is observable
    if (parts & kRenderPart) {
        if (graph) {
            t.project_ms = t.bin_ms = t.blend_ms = 0.f;
            cudaEventElapsedTime(&t.render_total_ms, e->ev[EV_SORT0], e->ev[EV_R1]);   // whole frame (sort + render)
        } else {
            cudaEventElapsedTime(&t.project_ms, e->ev[EV_R0], e->ev[EV_PROJECT]);
            cudaEventElapsedTime(&t.bin_ms, e->ev[EV_PROJECT], e->ev[EV_BIN]);
            cudaEventElapsedTime(&t.blend_ms, e->ev[EV_BIN], e->ev[EV_R1]);
            cudaEventElapsedTime(&t.render_total_ms, e->ev[EV_R0], e->ev[EV_R1]);
        }
    }
    if (parts & kSortPart) {
        float ms = 0.f;
        if (graph) {
            t.depth_ms = t.bucket_ms = t.scatter_ms = 0.f;
            cudaEventElapsedTime(&ms, e->ev[EV_SORT0], e->ev[EV_R1]);
        } else {
            cudaEventElapsedTime(&t.depth_ms, e->ev[EV_SORT0], e->ev[EV_DEPTH]);
            cudaEventElapsedTime(&t.bucket_ms, e->ev[EV_DEPTH], e->ev[EV_BUCKET]);
            cudaEventElapsedTime(&t.scatter_ms, e->ev[EV_BUCKET], e->ev[EV_SORT1]);
            cudaEventElapsedTime(&ms, e->ev[EV_SORT0], e->ev[EV_SORT1]);
        }
        t.sort_total_ms = ms;
        if (sort_time_ms) *sort_time_ms = ms;
    }
    if (parts & kCopyIn) cudaEventElapsedTime(&t.h2d_ms, e->ev[EV_H2D0], e->ev[EV_H2D1]);
    cudaEventElapsedTime(&t.d2h_ms, e->ev[EV_D2H0], e->ev[EV_D2H1]);
    return frame_status(e, s, parts);
}

// A blocking call's picture copied back between the D2H timing events (none: the events alone), and its depth where the caller asked for
// it (rp: the call's parameters, views: a multi-view frame's count)
static int copy_out(gs_engine *e, void *dst, const void *src, size_t bytes, const gs_render_params *rp = nullptr, uint32_t views = 1) {
    CU(cudaEventRecord(e->ev[EV_D2H0], e->stream));
    if (dst && bytes) CU(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, e->stream));
    if (rp && rp->depth && rp->depth_out)
        CU(cudaMemcpyAsync(rp->depth_out, e->rs.depth[e->rs.frame_parity].p, (size_t)views * rp->width * rp->height * sizeof(float), cudaMemcpyDeviceToHost, e->stream));
    CU(cudaEventRecord(e->ev[EV_D2H1], e->stream));
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
    gs_sort_params q = *p;
    const uint32_t *d_idx = nullptr;
    uint32_t launches = 0;
    if ((rc = clamp_counts(e, q))) return rc;
    e->last_frame_was_graph = false;
    if ((rc = stage_sort_inputs(e, &q, &d_idx)) || (rc = sort_on_device(e, {Launch(e->stream, &e->prof, &launches), e->ev}, d_idx, q))) return rc;
    e->tm.kernel_launches = launches;
    if ((rc = copy_out(e, sorted_out, e->sorted.p, (size_t)q.render_count * 4))) return rc;
    return finish_call(e, kSortPart | kCopyIn, sort_time_ms);
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
    return e->precomputed.ensure(e->cfg.max_splat_count);
}
// The sharded sort keeps bounded spin-wait kernels in flight while the host enqueues the rest of the chain, so every kernel of the
// chain is loaded up front (preload_kernel); otherwise a first sort could stall on its own wait kernel.
template <typename KeyT> static void shard_preload_keyed() { preload_kernel(k_bucket<KeyT>); preload_kernel(k_shard_place<KeyT>); radix_preload<KeyT, uint32_t>(); }
static void shard_preload(gs_engine *e) {
    preload_kernel(k_sort_init); preload_kernel(k_copy_head);
    preload_kernel(k_shard_exchange_minmax); preload_kernel(k_shard_exchange_runs); preload_kernel(k_shard_totals); preload_kernel(k_shard_delta); preload_kernel(k_shard_done);
    for_each_depth([](int, bool, bool views, auto kernel) { if (!views) preload_kernel(kernel); });
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
static int shard_local_sort(gs_engine *e, const Launch &launch, const uint32_t *d_indexes, uint32_t s0, uint32_t lo, uint32_t hi) {
    const uint32_t n = hi - lo, R = e->cfg.distance_map_range;
    const uint32_t me = e->cfg.rank, world = e->shard.world, seq = e->shard.seq;
    uint2 *runs = (uint2 *)shard_runs(e->shard.block.p);
    RadixJob<uint32_t> j = depth_job(e, d_indexes, lo, hi, e->shard.local_sorted.p, kTagShard);
    j.keep_final_keys = true; j.ranges = runs;
    if (n) {   // slice -> keys with the GLOBAL range map -> local order + per-key runs of that order
        int rc;
        if ((rc = e->sorter.bucket<KeyT>(j, e->dist.p + lo, R, false, launch)) || (rc = e->sorter.sort<KeyT>(j, launch))) return rc;
    }
    // C2: publish my runs, wait for everybody's, turn them into the offsets of my runs in the global order
    launch.plain("k_shard_exchange_runs", k_shard_exchange_runs, 1, 32, 0, e->shard.peers, me, world, seq);
    if (n) {
        const uint32_t sblocks = (R + kShardScanThreads - 1) / kShardScanThreads;
        launch.plain(nullptr, k_shard_totals, sblocks, kShardScanThreads, 0, e->shard.peers, me, world, R, e->shard.total.p, e->shard.ahead.p, e->shard.block_total.p);
        launch.plain(nullptr, k_shard_delta, sblocks, kShardScanThreads, 0, runs, R, e->shard.total.p, e->shard.ahead.p, e->shard.block_total.p, e->shard.delta.p);
        launch.mark("k_shard_offsets");
        launch.plain("k_shard_place", k_shard_place<KeyT>, std::min<uint32_t>((n + 255) / 256, e->sm_count * 16), 256, 0, e->sorter.final_keys<KeyT>(j),
                     e->shard.local_sorted.p, n, e->shard.delta.p, e->shard.root_out + s0);
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
    if ((rc = clamp_counts(e, q))) return rc;
    const uint32_t *d_idx = nullptr;
    uint32_t launches = 0;
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
        if ((rc = stage_sort_inputs(e, &q, &d_idx)) || (rc = sort_on_device(e, {Launch(e->stream, &e->prof, &launches), e->ev}, d_idx, q))) {
            e->shard.pending = false;
            return rc;
        }
        e->tm.kernel_launches = launches;
        return GS_OK;
    }
    e->shard.pending_unsplit = false;
    if ((rc = stage_sort_inputs(e, &q, &d_idx))) return rc;
    cudaStream_t st = e->stream;
    const SortLaunch sl{Launch(st, &e->prof, &launches), e->ev};
    const Launch &launch = sl.launch;
    const uint32_t s0 = q.render_count - q.sort_count;
    const uint32_t lo = shard_bound(s0, q.sort_count, me, world), hi = shard_bound(s0, q.sort_count, me + 1, world);
    const uint32_t seq = ++e->shard.seq;
    if ((rc = sort_prologue(e, sl, d_idx, me == 0 ? s0 : 0))) return rc;
    if (hi > lo && ((rc = upload_camera(e, q.model_view_proj, st)) || (rc = depth_pass(e, launch, d_idx, q, lo, hi, 0)))) return rc;
    // C1: global min/max over peer memory
    launch.plain("k_shard_exchange_minmax", k_shard_exchange_minmax, 1, kShardSyncThreads, 0, e->shard.peers, e->ctl.p, me, world, seq, hi > lo ? 0 : 1,
                 (uint2 *)shard_runs(e->shard.block.p), e->cfg.distance_map_range);
    CU(sl.mark(EV_DEPTH));
    CU(sl.mark(EV_BUCKET));
    rc = (e->key_bits <= 16) ? shard_local_sort<uint16_t>(e, launch, d_idx, s0, lo, hi) : shard_local_sort<uint32_t>(e, launch, d_idx, s0, lo, hi);
    if (rc) return rc;
    launch.plain("k_shard_done", k_shard_done, 1, 32, 0, e->shard.peers, me, world, seq);
    CU(sl.mark(EV_SORT1));
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
    if ((rc = copy_out(e, e->cfg.rank == 0 ? sorted_out : nullptr, e->sorted.p, (size_t)rcnt * 4))) return rc;
    const bool split = !e->shard.pending_unsplit;
    ShardHeader &hd = e->h_status.p->shard;
    if (split) CU(cudaMemcpyAsync(&hd, e->shard.block.p, sizeof(ShardHeader), cudaMemcpyDeviceToHost, e->stream));
    rc = finish_call(e, kSortPart | kCopyIn, sort_time_ms);
    if (split && hd.timeout) {
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
    gs_sort_params q{};
    memcpy(q.model_view_proj, modelViewProj, sizeof(q.model_view_proj));
    q.sort_count = sortCount;
    q.render_count = renderCount;
    q.use_precomputed_distances = usePrecomputedDistances;
    SortOptions o;
    o.write_buckets = (mappedDistances != nullptr) || (frequencies != nullptr);
    uint32_t launches = 0;
    if ((rc = sort_on_device(e, {Launch(st, &e->prof, &launches), e->ev}, e->indexes.p, q, o))) return rc;
    e->tm.kernel_launches = launches;
    // wasm-trap emulation: results are only written back when the device reported no range error (copy_out: its timing events alone)
    if ((rc = copy_out(e, nullptr, nullptr, 0)) || (rc = finish_call(e, kSortPart))) return rc;
    if (renderCount) CU(cudaMemcpyAsync(indexesOut, e->sorted.p, (size_t)renderCount * 4, cudaMemcpyDeviceToHost, st));
    const uint32_t s0 = renderCount - sortCount;
    if (mappedDistances && sortCount) CU(cudaMemcpyAsync(mappedDistances + s0, e->dist.p + s0, (size_t)sortCount * 4, cudaMemcpyDeviceToHost, st));
    if (frequencies) {
        if ((rc = e->freq.ensure(distanceMapRange))) return rc;
        CU(cudaMemsetAsync(e->freq.p, 0, (size_t)distanceMapRange * 4, st));
        const Launch uncounted(st);   // the reference's scratch output, not part of the sort: kernel_launches counts the sort alone
        if (sortCount)
            uncounted.plain(nullptr, k_bucket_counts, std::min<uint32_t>((sortCount + 255) / 256, e->sm_count * 8), 256, 0, e->dist.p, s0, renderCount, e->freq.p);
        uncounted.plain(nullptr, k_exclusive_scan_single_block, 1, 1024, 0, e->freq.p, distanceMapRange);
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
    using DistanceKernel = decltype(&k_distances_splat_order<false, false>);
    static const DistanceKernel kernels[2][2] = {{k_distances_splat_order<false, false>, k_distances_splat_order<false, true>},   // [integer][dynamic]
                                                 {k_distances_splat_order<true, false>, k_distances_splat_order<true, true>}};
    Launch(st).plain(nullptr, kernels[integer][dyn], blocks, 256, 0, e->centers.p, e->scene_idx.p, d_ir.p, d_fr.p, count, e->precomputed.p);
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
    e->scenes_multi = false;
    e->scene_start.clear();
    e->baked_xf = 0;
    e->tree.decoded_ray_records = false;
    rc = raster_upload(e->rs, e->cfg, *d, e->stream);
    if (rc) return rc;
    CU(cudaStreamSynchronize(e->stream));
    return GS_OK;
}

// A frame's bytes: width x height, or a multi-view frame's `views` stacked bands of that size
static size_t frame_bytes(const gs_render_params *p, uint32_t views = 1) {
    return (size_t)p->width * p->height * views * (p->frame_format == GS_FRAME_RGBA8 ? 4 : 16);
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

// The two halves of a frame outside a graph, with their timing events: the parameter upload and the projection, then the binning
// and the blend of the draw order d_order (view v's at d_order + v order_stride).
static int project_eager(gs_engine *e, const gs_uniforms &u, const gs_render_params &p, const FrameViews &fv, const Launch &launch) {
    CU(cudaEventRecord(e->ev[EV_R0], launch.stream()));
    int rc = raster_upload_params(e->rs, e->cfg, u, p, fv, launch.stream());
    if (rc || (rc = raster_project(e->rs, e->cfg, p, fv, launch))) return rc;
    CU(cudaEventRecord(e->ev[EV_PROJECT], launch.stream()));
    return GS_OK;
}
static int bin_blend_eager(gs_engine *e, const gs_render_params &p, const FrameViews &fv, const uint32_t *d_order, size_t order_stride,
                           const unsigned long long *order_count_dev, const Launch &launch) {
    int rc = raster_bin_blend(e->rs, e->cfg, p, fv, d_order, order_stride, order_count_dev, e->ev[EV_BIN], launch);
    if (rc) return rc;
    CU(cudaEventRecord(e->ev[EV_R1], launch.stream()));
    CU(cudaGetLastError());
    return GS_OK;
}

extern "C" int gs_render(gs_engine *e, const gs_uniforms *u, const gs_render_params *p, void *frame_out) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!u || !p) return fail(GS_ERR_BAD_ARG, "gs_render: null argument");
    if (e->pipe_inflight()) return fail(GS_ERR_NOT_READY, "gs_render: pipelined frames are in flight (gs_frame_end first)");
    const gs_render_params rp = read_options(p, gs_render_params{});
    const uint32_t *d_order = nullptr;
    uint32_t launches = 0;
    e->last_frame_was_graph = false;
    const FrameViews fv = frame_views(rp);
    if ((rc = stage_order(e, &rp, &d_order)) || (rc = raster_check(e->rs, e->cfg, *u, rp, fv)) || (rc = reserve_views(e, fv)) || (rc = reserve_depth(e, rp)))
        return rc;
    e->prof.begin(e->stream);
    const Launch launch(e->stream, &e->prof, &launches);
    if ((rc = project_eager(e, *u, rp, fv, launch)) || (rc = bin_blend_eager(e, rp, fv, d_order, 0, nullptr, launch))) return rc;
    e->tm.kernel_launches = launches;
    note_depth(e, rp, fv);
    if ((rc = copy_out(e, frame_out, raster_frame_ptr(e->rs, rp.frame_format), frame_bytes(&rp), &rp))) return rc;
    return finish_call(e, kRenderPart);
}

// host-side parameter blocks of one frame -> device (outside any graph; pageable sources are staged by the driver before return).
// A multi-view frame sorts with each view's camera.
static int upload_frame_params(gs_engine *e, const float *mvp, const gs_uniforms &u, const gs_render_params &p, const FrameViews &fv) {
    cudaStream_t st = e->param_side ? e->param_stream : e->stream;
    int rc = fv.stacked() ? upload_view_cameras(e, fv, st) : upload_camera(e, mvp, st);
    if (rc || (rc = raster_upload_params(e->rs, e->cfg, u, p, fv, st))) return rc;
    if (e->param_side) {      // the frame graph (and nothing else on the compute stream) waits for the side upload
        CU(cudaEventRecord(e->ev_params[e->rs.frame_parity], st));
        CU(cudaStreamWaitEvent(e->stream, e->ev_params[e->rs.frame_parity], 0));
    }
    return GS_OK;
}

// Enqueues one frame (sort + render) on the engine's stream; q and rp receive the call's clamped parameters.  no_subset: the caller
// reads the sorted indexes back, so a sharded engine sorts the full order instead of its subset.  multi: the cameras of a multi-view
// frame (gs_frame_views), each sorted on its own; nullptr: the mono or stereo frame of p.
static int enqueue_frame(gs_engine *e, const gs_sort_params *s, const gs_uniforms *u, const gs_render_params *p, bool no_subset, gs_sort_params &q,
                         gs_render_params &rp, const FrameViews *multi = nullptr) {
    q = *s;
    int rc;
    if ((rc = clamp_counts(e, q))) return rc;
    const uint32_t *d_idx = nullptr;
    if ((rc = stage_sort_inputs(e, &q, &d_idx))) return rc;
    rp = read_options(p, gs_render_params{});     // a caller built before the composite inputs or the eyes renders the plain mono frame
    rp.sorted_indexes = nullptr; rp.sorted_indexes_dev = nullptr;
    rp.render_count = std::min(rp.render_count, q.render_count);
    const FrameViews fv = multi ? *multi : frame_views(rp);
    if ((rc = raster_check(e->rs, e->cfg, *u, rp, fv)) || (rc = reserve_views(e, fv)) || (rc = reserve_depth(e, rp))) return rc;
    // a multi-view frame bins view v's draw order at sorted[v render_count]
    const uint32_t *order = fv.stacked() ? e->vsort->sorted.p : e->sorted.p;
    const size_t order_stride = fv.stacked() ? q.render_count : 0;
    cudaStream_t st = e->stream;
    e->last_frame_was_graph = false;
    // sharded frame: sort only this rank's subset (full sorts only; a partial sort keeps the replicated path)
    // The subset path adds two compaction kernels (~35 us at 1M splats) and only shrinks kernels that are already at their latency
    // floor there; it pays off from a few million splats (measured: 1.2M slower, 16M faster).  GS_SUBSET_MIN overrides the threshold.
    const uint32_t subset_min = getenv("GS_SUBSET_MIN") ? (uint32_t)atoll(getenv("GS_SUBSET_MIN")) : 3000000u;
    const bool subset = e->cfg.world_size > 1 && q.sort_count == q.render_count && q.render_count >= subset_min && q.render_count > 0 && !no_subset;
    if (subset) {
        if ((rc = e->sub_idx.ensure(e->cfg.max_splat_count)) || (rc = e->sub_dist.ensure(e->cfg.max_splat_count))) return rc;
    }
    const unsigned long long *order_count = subset ? &e->rs.view[0].rctl.p->subset_count : nullptr;
    uint32_t launches = 0;
    const Launch launch(st, &e->prof, &launches);
    if (e->graph_enabled && !e->prof.on) {
        // (the composite inputs, the eyes and the depth enter the key as one flag each, a multi-view frame as its view count: their
        // pointers and matrices are read from the frame's parameter blocks, not captured, and a parity's depth plane never moves, so a
        // moving head replays the same graph.  k_project reads the scene indexes only when the scene has them, from a buffer allocated
        // once; the covariance and SH buffers grow when a format needs more bytes per splat, so a later upload in the captured formats
        // can leave them elsewhere: their addresses are part of the key)
        const RasterState &rs = e->rs;
        GraphKey key{};
        key.indexes = d_idx; key.cov = rs.cov.p; key.sh = rs.sh.p;
        key.render_count = q.render_count; key.sort_count = q.sort_count; key.precomputed = q.use_precomputed_distances;
        key.frame_render_count = rp.render_count; key.width = rp.width; key.height = rp.height; key.frame_format = (uint32_t)rp.frame_format;
        key.flip_y = rp.flip_y != 0; key.eyes = rp.eyes != nullptr; key.depth = rp.depth != 0; key.composite = has_composite_inputs(rp);
        key.scene_idx = rs.have_scene_idx; key.subset = subset; key.views = fv.stacked() ? fv.count : 0;
        key.cov_format = (uint32_t)rs.cov_format; key.sh_format = (uint32_t)rs.sh_format; key.sh_degree = rs.sh_degree; key.uploaded = rs.uploaded;
        if ((rc = upload_frame_params(e, q.model_view_proj, *u, rp, fv))) return rc;
        FrameGraph &g = e->graph;
        const int parity = e->rs.frame_parity;
        if (!g.current(parity, key)) {
            rc = g.capture(parity, key, e->rs.peer_local, st, [&](cudaStream_t side, cudaEvent_t join) {
                // fork: the projection does not depend on the draw order, so it runs beside the (latency-bound) depth sort
                int r = raster_project(e->rs, e->cfg, rp, fv, launch.on(side));
                if (r) return r;
                CU(cudaEventRecord(join, side));
                const SortLaunch captured{launch, nullptr};
                SortOptions o; o.subset = subset; o.wait_for_rects = join;
                if ((r = fv.stacked() ? sort_views(e, captured, d_idx, q, fv) : sort_on_device(e, captured, d_idx, q, o))) return r;
                CU(cudaStreamWaitEvent(st, join, 0));
                return raster_bin_blend(e->rs, e->cfg, rp, fv, order, order_stride, order_count, nullptr, launch);
            });
            if (rc) return rc;
            g.launches = launches;
            g.slot[parity].snapshot = e->rs.snapshot_taken;
        }
        // the captured mono sort assumes (and leaves) a clean control block; a multi-view sort resets its own
        const bool mono_sort = !fv.stacked();
        if (mono_sort && e->ctl_dirty) launch.pdl(nullptr, k_sort_init, 1, 256, 0, e->ctl.p);
        if (mono_sort) e->ctl_dirty = true;
        CU(cudaEventRecord(e->ev[EV_SORT0], st));
        CU(cudaGraphLaunch(g.slot[parity].exec, st));
        if (mono_sort) e->ctl_dirty = false;
        CU(cudaEventRecord(e->ev[EV_R1], st));
        launches = g.launches;   // (the k_sort_init above is not the frame's)
        if (mono_sort) {
            e->last_render_count = q.render_count;
            e->have_sorted = !subset;   // a subset order is not a draw order for gs_render
        }
        e->last_frame_was_graph = true;
    } else if (subset) {   // one stream: projection first (its rects select the subset), then depth + subset sort, then binning + blend
        e->prof.begin(st);
        SortOptions o; o.open_timeline = false; o.subset = true;
        if ((rc = project_eager(e, *u, rp, fv, launch)) || (rc = sort_on_device(e, {launch, e->ev}, d_idx, q, o)) ||
            (rc = bin_blend_eager(e, rp, fv, e->sorted.p, 0, order_count, launch)))
            return rc;
        e->have_sorted = false;
    } else {
        if (fv.stacked()) e->prof.begin(st);
        const SortLaunch eager{launch, e->ev};
        if ((rc = fv.stacked() ? sort_views(e, eager, d_idx, q, fv) : sort_on_device(e, eager, d_idx, q)) ||
            (rc = project_eager(e, *u, rp, fv, launch)) || (rc = bin_blend_eager(e, rp, fv, order, order_stride, nullptr, launch)))
            return rc;
    }
    e->tm.kernel_launches = launches;
    note_depth(e, rp, fv);
    return GS_OK;
}

// The end of a blocking frame: its draw order (a multi-view frame's, multi: its views, one order after another) and its picture copied
// back, then finish_call
static int finish_frame(gs_engine *e, const gs_sort_params &q, const gs_render_params &rp, const FrameViews *multi, uint32_t *sorted_out, void *frame_out) {
    const uint32_t views = multi ? multi->count : 1;
    if (sorted_out && q.render_count)
        CU(cudaMemcpyAsync(sorted_out, multi ? e->vsort->sorted.p : e->sorted.p, (size_t)views * q.render_count * 4, cudaMemcpyDeviceToHost, e->stream));
    const int rc = copy_out(e, frame_out, raster_frame_ptr(e->rs, rp.frame_format), frame_bytes(&rp, views), &rp, views);
    return rc ? rc : finish_call(e, kSortPart | kRenderPart | kCopyIn, nullptr, multi ? e->vsort->ctl.p : nullptr);
}

extern "C" int gs_frame(gs_engine *e, const gs_sort_params *s, const gs_uniforms *u, const gs_render_params *p, uint32_t *sorted_out, void *frame_out) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!s || !u || !p) return fail(GS_ERR_BAD_ARG, "gs_frame: null argument");
    if (e->pipe_inflight()) return fail(GS_ERR_NOT_READY, "gs_frame: pipelined frames are in flight (gs_frame_end first)");
    e->rs.frame_parity = 0;
    gs_sort_params q; gs_render_params rp;
    if ((rc = enqueue_frame(e, s, u, p, sorted_out != nullptr, q, rp))) return rc;
    return finish_frame(e, q, rp, nullptr, sorted_out, frame_out);
}

// Enqueue one frame and return without waiting: the frame stays on the device (gs_buffer_dev(GS_BUF_FRAME)), errors and
// timings are collected by the next gs_synchronize().  Lets a caller keep several frames in flight on the stream.
extern "C" int gs_frame_async(gs_engine *e, const gs_sort_params *s, const gs_uniforms *u, const gs_render_params *p) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!s || !u || !p) return fail(GS_ERR_BAD_ARG, "gs_frame_async: null argument");
    if (e->pipe_inflight()) return fail(GS_ERR_NOT_READY, "gs_frame_async: pipelined frames are in flight (gs_frame_end first): their pictures are still being copied out of the frame buffers");
    gs_sort_params q; gs_render_params rp;
    if ((rc = enqueue_frame(e, s, u, p, false, q, rp))) return rc;
    e->pending_async = true;
    return GS_OK;
}

// Several cameras of one mesh in one frame: every view sorted with its own camera (one batched sort), projected, binned and blended in
// shared launches, the views stacked top to bottom.  See the header.
extern "C" int gs_frame_views(gs_engine *e, const gs_sort_params *s, const gs_uniforms *u, const gs_render_params *p, const gs_view *views,
                              uint32_t view_count, uint32_t *sorted_out, void *frame_out) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!s || !u || !p || !views) return fail(GS_ERR_BAD_ARG, "gs_frame_views: null argument");
    if (view_count == 0 || view_count > GS_MAX_VIEWS) return fail(GS_ERR_BAD_ARG, "gs_frame_views: view_count %u outside [1, %d]", view_count, GS_MAX_VIEWS);
    if (s->use_precomputed_distances) return fail(GS_ERR_BAD_ARG, "gs_frame_views: precomputed distances belong to one camera (use_precomputed_distances)");
    if (e->pipe_inflight()) return fail(GS_ERR_NOT_READY, "gs_frame_views: pipelined frames are in flight (gs_frame_end first)");
    if ((uint64_t)view_count * std::min(s->render_count, e->uploaded_splats) > 0xffffffffull)
        return fail(GS_ERR_CAPACITY, "gs_frame_views: %u views of %u splats exceed 2^32 sort keys", view_count, s->render_count);
    e->rs.frame_parity = 0;
    const FrameViews fv{view_count, views};
    gs_sort_params q; gs_render_params rp;
    if ((rc = enqueue_frame(e, s, u, p, true, q, rp, &fv))) return rc;
    return finish_frame(e, q, rp, &fv, sorted_out, frame_out);
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
    int rc = e->h_pipe.ensure(gs_engine::kPipeRing);
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
    rc = enqueue_frame(e, s, u, p, false, q, rp);
    e->param_side = false;
    if (rc) { e->rs.frame_parity = 0; return rc; }
    cudaStream_t st = e->stream;
    FrameStatus *hs = e->h_pipe.p + ring;
    // (multi-GPU: rank 0's peer_timeout flag is raised AFTER the blend, by k_peer_wait_arrived -- the snapshot would miss it)
    const bool snapshot = two && e->cfg.world_size == 1 && e->last_frame_was_graph && e->graph.slot[e->rs.frame_parity].snapshot;
    if (!snapshot) {      // status read-back in stream order (frames outside a graph, blend generations without the snapshot, one buffer)
        CU(cudaMemcpyAsync(hs->sort, e->ctl.p, kSortHeadBytes, cudaMemcpyDeviceToHost, st));
        CU(cudaMemcpyAsync(&hs->raster, e->rs.view[0].rctl.p, sizeof(RasterControl), cudaMemcpyDeviceToHost, st));
    }
    CU(cudaEventRecord(e->ev_frame_done[ring], st));
    CU(cudaStreamWaitEvent(e->copy_stream, e->ev_frame_done[ring], 0));
    if (snapshot) CU(cudaMemcpyAsync(hs, e->status_dev.p + e->rs.frame_parity, sizeof(FrameStatus), cudaMemcpyDeviceToHost, e->copy_stream));
    if (frame_out) CU(cudaMemcpyAsync(frame_out, raster_frame_ptr(e->rs, rp.frame_format), frame_bytes(&rp), cudaMemcpyDeviceToHost, e->copy_stream));
    if (rp.depth && rp.depth_out)
        CU(cudaMemcpyAsync(rp.depth_out, e->rs.depth[e->rs.frame_parity].p, (size_t)rp.width * rp.height * sizeof(float), cudaMemcpyDeviceToHost, e->copy_stream));
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
    return frame_status(e, e->h_pipe.p[ring], kSortPart | kRenderPart);
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
    t.sub_trees = 1;
    t.have_nodes = false;   // gs_upload_splat_tree_nodes describes these leaves next
    t.have_depth = false;
    t.built = gs_splat_tree_info{};
    return GS_OK;
}

// One model view per sub-tree (count = the tree's sub-tree count); the one-matrix case is the kernel a single tree has always run.
static int gather_for_sort(gs_engine *e, const char *entry, const double *model_views, uint32_t count, double cos_fov_x_over_2, double cos_fov_y_over_2,
                           int gather_all_nodes, uint32_t *render_count_out) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!model_views || !render_count_out) return fail(GS_ERR_BAD_ARG, "%s: null argument", entry);
    auto &t = e->tree;
    if (count != t.sub_trees) return fail(GS_ERR_BAD_ARG, "%s: %u model views for a tree of %u sub-trees", entry, count, t.sub_trees);
    if (!t.count) { *render_count_out = 0; return GS_OK; }
    CullParams P;
    memcpy(P.mv, model_views, sizeof(P.mv));
    P.cos_fov_x_over_2 = cos_fov_x_over_2; P.cos_fov_y_over_2 = cos_fov_y_over_2; P.gather_all = gather_all_nodes;
    cudaStream_t st = e->stream;
    uint32_t launches = 0;
    const Launch launch(st, nullptr, &launches);
    if (count == 1) {
        launch.plain(nullptr, k_tree_cull<false>, (t.count + 127) / 128, 128, 0, t.center.p, t.nmin.p, t.nmax.p, t.count, P, nullptr, nullptr, 1u, t.key.p);
    } else {
        if ((rc = t.mvs.ensure(16 * (size_t)count))) return rc;
        CU(cudaMemcpyAsync(t.mvs.p, model_views, 128 * (size_t)count, cudaMemcpyHostToDevice, st));
        launch.plain(nullptr, k_tree_cull<true>, (t.count + 127) / 128, 128, 0, t.center.p, t.nmin.p, t.nmax.p, t.count, P, t.mvs.p, t.sub_leaf.p, count,
                     t.key.p);
    }
    launch.plain(nullptr, k_tree_layout, (t.count + kLayoutThreads - 1) / kLayoutThreads, kLayoutThreads, 0, t.key.p, t.offsets.p, t.count, t.start.p, t.total.p);
    launch.plain(nullptr, k_tree_copy, t.count, 128, 0, t.start.p, t.offsets.p, t.indexes.p, e->indexes.p);
    CU(cudaMemcpyAsync(&e->h_status.p->gather_total, t.total.p, 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    *render_count_out = (uint32_t)e->h_status.p->gather_total;
    e->tm.kernel_launches = launches;
    return GS_OK;
}

extern "C" int gs_gather_for_sort(gs_engine *e, const double *model_view, double cos_fov_x_over_2, double cos_fov_y_over_2, int gather_all_nodes,
                                  uint32_t *render_count_out) {
    return gather_for_sort(e, "gs_gather_for_sort", model_view, 1, cos_fov_x_over_2, cos_fov_y_over_2, gather_all_nodes, render_count_out);
}

extern "C" int gs_gather_for_sort_subtrees(gs_engine *e, const double *model_views, uint32_t count, double cos_fov_x_over_2, double cos_fov_y_over_2,
                                           int gather_all_nodes, uint32_t *render_count_out) {
    return gather_for_sort(e, "gs_gather_for_sort_subtrees", model_views, count, cos_fov_x_over_2, cos_fov_y_over_2, gather_all_nodes, render_count_out);
}

// ---------------------------------------------------------------------------------------------------------------
// Raycaster.intersectSplatMesh on the GPU (ray_kernels.cuh).
// The ray records now describe the current scene.  A static mesh places scene s's records by xf[s] (column-major 4x4 each, nullptr:
// identity); `per_scene`: a record's scene is its splat's scene index, else every record is scene 0.
static int set_ray_transforms(gs_engine *e, const double (*xf)[16], uint32_t count, bool per_scene) {
    std::vector<double> t(16 * GS_MAX_SCENES, 0.0);
    for (int s = 0; s < GS_MAX_SCENES; ++s) t[16 * s] = t[16 * s + 5] = t[16 * s + 10] = t[16 * s + 15] = 1.0;
    if (xf) memcpy(t.data(), xf, sizeof(double) * 16 * count);
    int rc = e->ray.xf.ensure(t.size());
    if (rc) return rc;
    CU(cudaMemcpyAsync(e->ray.xf.p, t.data(), t.size() * sizeof(double), cudaMemcpyHostToDevice, e->stream));
    CU(cudaStreamSynchronize(e->stream));   // pageable source
    e->ray.per_scene = per_scene;
    e->ray.valid = true;
    return GS_OK;
}
static int set_ray_transform(gs_engine *e, const double *xf) {
    return set_ray_transforms(e, reinterpret_cast<const double (*)[16]>(xf), xf ? 1 : 0, false);
}

extern "C" int gs_upload_ray_records(gs_engine *e, const gs_ray_record *records, uint32_t from, uint32_t count, const double *scene_transform) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!e->ray.rec.p) return fail(GS_ERR_NOT_READY, "gs_upload_ray_records: engine created without ray_records");
    if (!records && count) return fail(GS_ERR_BAD_ARG, "gs_upload_ray_records: null records");
    if ((uint64_t)from + count > e->cfg.max_splat_count) return fail(GS_ERR_CAPACITY, "ray records [%u,%u) exceed max_splat_count %u", from, from + count, e->cfg.max_splat_count);
    if (count) CU(cudaMemcpyAsync(e->ray.rec.p + from, records, (size_t)count * sizeof(gs_ray_record), cudaMemcpyHostToDevice, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    return set_ray_transform(e, scene_transform);
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
    gs_raycast_params defaults{};
    for (int32_t &v : defaults.scene_visibility) v = 1;
    const gs_raycast_params q = read_options(p, defaults);
    auto &t = e->tree;
    auto &R = e->ray;
    if (!R.rec.p) return fail(GS_ERR_NOT_READY, "gs_raycast: engine created without ray_records");
    if (!R.valid) return fail(GS_ERR_NOT_READY, "gs_raycast: the ray records are stale (upload the scene or gs_upload_ray_records)");
    if (!t.have_nodes) return fail(GS_ERR_NOT_READY, "gs_raycast: no SplatTree (gs_build_splat_tree, or gs_upload_splat_tree + gs_upload_splat_tree_nodes)");
    const uint32_t subs = t.sub_trees;
    const bool forest = subs > 1;
    if (q.sub_tree_count && q.sub_tree_count != subs)
        return fail(GS_ERR_BAD_ARG, "gs_raycast: sub_tree_count %u for a tree of %u sub-trees", q.sub_tree_count, subs);
    if (q.sub_tree_count && !q.sub_tree_from_local) return fail(GS_ERR_BAD_ARG, "gs_raycast: sub_tree_count %u with sub_tree_from_local NULL", q.sub_tree_count);
    if (forest && !q.sub_tree_count)
        return fail(GS_ERR_BAD_ARG, "gs_raycast: the tree is a forest of %u sub-trees (one per scene): pass one from_local per sub-tree", subs);
    *hit_count = 0;
    if (!t.count || !t.node_count || !q.scene_visible) return GS_OK;   // no leaves, or every splat skipped (Raycaster.js:117)
    RayParams P{};
    memcpy(P.origin, q.origin, sizeof(P.origin)); memcpy(P.dir, q.direction, sizeof(P.dir));
    memcpy(P.from_local, q.sub_tree_count ? q.sub_tree_from_local : q.from_local, sizeof(P.from_local));
    P.xf = R.xf.p; P.scene_idx = R.per_scene ? e->rs.scene_idx.p : nullptr; P.scenes = P.scene_idx ? GS_MAX_SCENES : 1;
    for (int s = 0; s < GS_MAX_SCENES; ++s) P.visible |= q.scene_visibility[s] ? 1u << s : 0u;
    P.ellipsoid = q.mode == GS_RAYCAST_ELLIPSOID; P.dynamic = e->cfg.dynamic_mode;
    const uint32_t m = t.count, nn = t.node_count, n = std::max<uint32_t>(t.splats, 1);
    if ((rc = R.setup.ensure(subs)) || (rc = R.pass.ensure(nn)) || (rc = R.reached.ensure(m)) || (rc = R.list.ensure(m)) || (rc = R.counts.ensure(4)) ||
        (rc = R.hits.ensure(n)))
        return rc;
    cudaStream_t st = e->stream;
    uint32_t launches = 0;
    const Launch launch(st, nullptr, &launches);
    if (forest) {
        if ((rc = R.fl.ensure(16 * (size_t)subs))) return rc;
        CU(cudaMemcpyAsync(R.fl.p, q.sub_tree_from_local, 128 * (size_t)subs, cudaMemcpyHostToDevice, st));
        P.sub_from_local = R.fl.p; P.sub_leaf = t.sub_leaf.p; P.sub_node = t.sub_node.p; P.sub_trees = subs;
        launch.plain(nullptr, k_ray_setup<true>, 1, 32, 0, P, R.setup.p);
        launch.plain(nullptr, k_ray_nodes<true>, (nn + 127) / 128, 128, 0, t.all_min.p, t.all_max.p, nn, R.setup.p, t.sub_node.p, subs, R.pass.p);
    } else {
        launch.plain(nullptr, k_ray_setup<false>, 1, 1, 0, P, R.setup.p);
        launch.plain(nullptr, k_ray_nodes<false>, (nn + 127) / 128, 128, 0, t.all_min.p, t.all_max.p, nn, R.setup.p, nullptr, 1u, R.pass.p);
    }
    launch.plain(nullptr, k_ray_leaves, (m + 127) / 128, 128, 0, t.leaf_node.p, t.parent.p, R.pass.p, m, R.reached.p);
    launch.plain(nullptr, k_ray_compact, 1, kRayCompactThreads, 0, R.reached.p, m, R.list.p, R.counts.p);   // also zeroes the hit counter counts[1]
    const uint32_t grid = std::min<uint32_t>((m + kRaySplatThreads / 32 - 1) / (kRaySplatThreads / 32), (uint32_t)e->sm_count * 16);
    launch.plain(nullptr, forest ? k_ray_splats<true> : k_ray_splats<false>, grid, kRaySplatThreads, 0, R.list.p, R.counts.p, t.offsets.p, t.indexes.p, R.rec.p,
                 P, R.setup.p, R.hits.p, R.counts.p + 1);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(e->h_status.p->ray_counts, R.counts.p, 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    const uint32_t total = e->h_status.p->ray_counts[1];
    *hit_count = total;
    const uint32_t k = std::min(capacity, total);
    if (!k) { e->tm.kernel_launches = launches; return GS_OK; }
    const uint32_t *perm = nullptr;
    if (total > 1) {   // stable LSD radix sort by (distance, traversal position): position first, then the distance's three pieces
        int bits[4] = {1, kRayKeyBits[1], kRayKeyBits[2], kRayKeyBits[3]};
        while (bits[0] < 32 && (1ull << bits[0]) < (unsigned long long)t.splats) ++bits[0];
        auto keys = [&](const Launch &launch, int which, const uint32_t *order, uint32_t *keys, uint32_t *vals) {
            launch.plain(nullptr, k_ray_keys, (total + 255) / 256, 256, 0, R.hits.p, order, total, which, keys, vals);
        };
        if ((rc = R.sort.reserve(n, 32, st)) || (rc = R.sort.sort(nullptr, total, bits, 4, R.sort.order.p, keys, launch))) return rc;
        perm = R.sort.order.p;
    }
    if ((rc = R.out.ensure(k))) return rc;
    launch.plain(nullptr, k_ray_out, (k + 127) / 128, 128, 0, R.hits.p, perm, k, R.out.p);
    CU(cudaMemcpyAsync(hits, R.out.p, (size_t)k * sizeof(gs_ray_hit), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    e->tm.kernel_launches = launches;
    return GS_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Scene uploads: .ksplat images (gs_upload_ksplat, gs_upload_file_optimized's generated image) and files (gs_upload_file), each a mesh
// of one scene, and meshes of several (gs_upload_scenes).  Each one
//   1. validates the engine, its arguments and each scene's header (parse_scene);
//   2. allocates a scene's transient buffers and uploads its transform: a failure up to here in the first scene leaves the previous scene;
//   3. marks the scene empty before any scene buffer may be reallocated, then sets the mesh's storage formats (clear_scene);
//   4. decodes each scene's level-N SplatBuffer sections on the GPU (decode_section);
//   5. commits the mesh and reports each scene (commit_scenes).
// load_scenes runs steps 2-5.
// .ksplat header/section parsing is host logic (SplatBuffer.js:819-941); the decode runs on the GPU (SURVEY 8f N1).
// A scene upload's report into the caller's gs_ksplat_info: no more than its struct_size bytes, and struct_size = the bytes written.  A
// struct_size of 0 (or one that does not cover a field) is a caller built before that field was appended: its struct ends before it.
static void write_info(gs_ksplat_info *info, const gs_ksplat_info &S) {
    if (!info) return;
    const size_t n = info->struct_size >= sizeof(gs_ksplat_info) ? sizeof(gs_ksplat_info) : offsetof(gs_ksplat_info, splat_offset);
    memcpy(info, &S, n);
    info->struct_size = (uint32_t)n;
}

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
    ++rs.generation;
    e->ray.valid = false;
    e->scenes_multi = false;
    e->scene_start.clear();
    e->baked_xf = 0;
    rs.cov_format = o.half_covariances ? GS_COV_F16 : GS_COV_F32;
    rs.sh_degree = S.sh_degree;
    rs.sh_format = S.sh_degree ? (S.compression_level == 2 ? GS_SH_U8 : GS_SH_F16) : GS_SH_NONE;
    const size_t n = e->cfg.max_splat_count, ncomp = S.sh_degree == 2 ? 24 : (S.sh_degree == 1 ? 9 : 0);
    int rc;
    if ((rc = rs.cov.ensure(n * (o.half_covariances ? 12 : 24) + 16)) || (ncomp && (rc = rs.sh.ensure(n * ncomp * (rs.sh_format == GS_SH_U8 ? 1 : 2) + 16))))
        return rc;
    return GS_OK;
}

// Step 4: the splats [first, P.count) of one section of a SplatBuffer image in device memory.  `prefix`: its partial-bucket prefixes
// (level >= 1); `xf`: the transform or nullptr; `ms`: the scene of a multi-scene mesh the section belongs to, or nullptr.  A one-scene
// mesh needs no scene work: the rasteriser has no scene indexes, the commit zeroes the sorter's, and the mesh's SH level is the scene's.
static void decode_section(gs_engine *e, const gs_ksplat_options &o, const unsigned char *image, KSectionParams P, uint32_t first, const uint32_t *prefix,
                           const KTransform *xf, const KSceneParams *ms, const Launch &launch) {
    if (first >= P.count) return;
    RasterState &rs = e->rs;
    if (ms) P.splat_offset += ms->offset;
    P.sh_degree_out = (int)rs.sh_degree;
    P.minimum_alpha = o.minimum_alpha; P.half_cov = o.half_covariances; P.integer_centers = e->cfg.integer_based_sort; P.write_sort_centers = o.upload_sort_centers;
    const KSceneParams S = ms ? *ms : KSceneParams{};
    const uint32_t grid = (P.count - first + 127) / 128;
    auto go = [&](auto kernel) {
        launch.plain("k_ksplat_decode", kernel, grid, 128, 0, image, P, first, prefix, rs.cc.p, rs.cov.p, rs.sh.p, e->centers.p, xf, e->ray.rec.p, S);
    };
    if (xf) ms ? go(k_ksplat_decode<true, true>) : go(k_ksplat_decode<true, false>);
    else ms ? go(k_ksplat_decode<false, true>) : go(k_ksplat_decode<false, false>);
}

// A chunk of level-0 records of SH degree `degree`, as parse_file_chunks writes them: one level-0 section
static KSectionParams level0_section(uint32_t degree) {
    KSectionParams P{};
    P.level = 0; P.bytes_per_splat = 44 + 4 * (degree == 2 ? 24 : (degree == 1 ? 9 : 0)); P.sh_degree_file = (int)degree; P.scale_range = 1;
    return P;
}

static uint32_t rd32(const unsigned char *p) { uint32_t v; memcpy(&v, p, 4); return v; }
static uint16_t rd16(const unsigned char *p) { uint16_t v; memcpy(&v, p, 2); return v; }
static float rdf(const unsigned char *p) { float v; memcpy(&v, p, 4); return v; }

struct KsplatLayout {
    gs_ksplat_info info;                // splats, lowest section SH degree, level, sections, centre, SH range
    uint32_t max_splats = 0;            // the header's declared splat count
    std::vector<KSectionParams> secs;   // byte offsets into the image, splat offsets
};

// One scene of an upload: its source, its options, and what step 1 found.
struct SceneLoad {
    gs_scene_source src{};                         // format, data, bytes, optimized
    gs_ksplat_options o{};
    gs_generate_options g{};                       // an optimized file's generator options
    gs_ksplat_info S{};                            // the scene's report (an optimized file's is its generated image's once generated)
    KsplatLayout K; std::vector<uint32_t> pre;     // a .ksplat, or an optimized file's generated image
    FileLayout L;                                  // files
};

// Step 5, once the decode has completed: the mesh of `count` scenes, each at S.splat_offset.  A static mesh's ray records are placed by
// each scene's transform.  One scene needs no scene indexes: the rasteriser drops them, and the sorter's, when it takes the scene's
// centres, become scene 0.  Several keep the indexes their decode wrote, and where each scene starts.
static int commit_scenes(gs_engine *e, const SceneLoad *sc, uint32_t count) {
    const bool multi = count > 1;
    const uint32_t total = sc[count - 1].S.splat_offset + sc[count - 1].S.splat_count;
    e->rs.uploaded = total;
    e->rs.have_scene_idx = multi;
    if (sc[0].o.upload_sort_centers) {
        e->uploaded_splats = total;
        if (!multi && e->scene_idx.p && total) {
            CU(cudaMemsetAsync(e->scene_idx.p, 0, (size_t)total * 4, e->stream));
            CU(cudaStreamSynchronize(e->stream));
        }
    }
    std::vector<double> xf(16 * count, 0.0);
    uint32_t baked = 0;
    for (uint32_t s = 0; s < count; ++s) {
        double *t = xf.data() + 16 * s;
        if (sc[s].o.has_transform) { memcpy(t, sc[s].o.transform, sizeof(sc[s].o.transform)); baked |= 1u << s; }
        else t[0] = t[5] = t[10] = t[15] = 1.0;
    }
    int rc;
    if (e->ray.rec.p && (rc = set_ray_transforms(e, reinterpret_cast<const double (*)[16]>(xf.data()), count, multi))) return rc;
    e->tree.decoded_ray_records = e->ray.rec.p != nullptr;
    e->baked_xf = baked;
    if (multi) {
        e->scenes_multi = true;
        e->scene_start.resize(count + 1);
        for (uint32_t s = 0; s < count; ++s) e->scene_start[s] = sc[s].S.splat_offset;
        e->scene_start[count] = total;
    }
    return GS_OK;
}

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

// Steps 2 and 4 for a scene's parsed .ksplat image c.K with bucket prefixes c.pre: `d_image` is the image in device memory, else the
// source's bytes are staged there.  `prepare()` runs once the transient buffers exist, before the first decode; `ms`: the scene's place
// in a multi-scene mesh, or nullptr.
template <typename Prepare>
static int decode_ksplat_image(gs_engine *e, const SceneLoad &c, const unsigned char *d_image, const KSceneParams *ms, Prepare prepare) {
    int rc;
    cudaStream_t st = e->stream;
    const std::vector<uint32_t> &pre = c.pre;
    DevBuf<unsigned char> d_file; DevBuf<uint32_t> d_pre; DevBuf<KTransform> d_xf;   // the staged image, the prefixes: this call only
    if ((!d_image && (rc = d_file.ensure(c.src.bytes))) || (rc = d_pre.ensure(pre.size())) || (rc = upload_transform(e, c.o, c.S, d_xf))) return rc;
    if (!d_image) {
        CU(cudaMemcpyAsync(d_file.p, c.src.data, c.src.bytes, cudaMemcpyHostToDevice, st));   // pageable source: staged before return
        d_image = d_file.p;
    }
    if (!pre.empty()) CU(cudaMemcpyAsync(d_pre.p, pre.data(), pre.size() * 4, cudaMemcpyHostToDevice, st));
    KSceneParams m{};
    if (ms) { m = *ms; m.sh_lo = c.S.min_sh_coeff; m.sh_hi = c.S.max_sh_coeff; }
    if ((rc = prepare())) return rc;
    const Launch launch(st, &e->prof);
    size_t at = 0;
    for (const KSectionParams &P : c.K.secs) {
        decode_section(e, c.o, d_image, P, 0, d_pre.p + at, d_xf.p, ms ? &m : nullptr, launch);
        at += P.partial_count + 1;
    }
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    return GS_OK;
}

// Step 1 for a .ksplat image in host memory: its header, sections and bucket prefixes, against `capacity` splats
static int parse_ksplat(const void *data, size_t bytes, uint32_t capacity, KsplatLayout &K, std::vector<uint32_t> &pre) {
    int rc;
    if ((rc = parse_ksplat_head((const unsigned char *)data, bytes, capacity, K))) return rc;
    std::vector<const unsigned char *> lens;
    for (const KSectionParams &P : K.secs) lens.push_back((const unsigned char *)data + P.base);
    return ksplat_prefixes(K, lens, capacity, pre);
}

// ---------------------------------------------------------------------------------------------------------------
// .ply / .splat -> engine (file_parse.h, file_kernels.cuh).  The file is parsed and validated on the host; its records then go through the
// device in chunks: file chunk -> staging buffer -> k_ply_to_level0 / k_splat_to_level0 -> level-0 SplatBuffer records -> k_ksplat_decode.
// Chunking bounds the transient device memory to about 2 x kFileChunkBytes whatever the file's size.
static constexpr size_t kFileChunkBytes = 64u << 20;

extern "C" int gs_probe_file(int format, const void *data, size_t bytes, gs_ksplat_info *info) {
    FileLayout L;
    if (parse_file(format, data, bytes, L, g_err, sizeof(g_err))) return GS_ERR_BAD_ARG;
    write_info(info, scene_info(L.count, (uint32_t)L.sh_degree, 0, 1));
    return GS_OK;
}

// Step 1 for a file, after check_scene_engine: its header, then its splat count against the engine's capacity.  In file order
// (generate = false) an INRIA v2 file is refused first: PlyParser.parseToUncompressedSplatBuffer throws for it, and the reference loads
// it through the generator only.
static int parse_scene_file(const gs_engine *e, int format, const void *data, size_t bytes, bool generate, FileLayout &L, bool header_only = false) {
    if (parse_file(format, data, bytes, L, g_err, sizeof(g_err), header_only)) return GS_ERR_BAD_ARG;
    if (L.v2 && !generate)
        return fail(GS_ERR_BAD_ARG, ".ply: INRIA v2 (codebook) .ply: loads only through the generator (gs_upload_file_optimized, "
                                    "gs_generate_splat_buffer), not in file order");
    if (L.count > e->cfg.max_splat_count) return fail(GS_ERR_CAPACITY, "the file holds %u splats, engine capacity %u", L.count, e->cfg.max_splat_count);
    return GS_OK;
}

// The file's records through the device in chunks: file chunk -> staging buffer -> k_ply_to_level0 / k_pcply_to_level0 / k_splat_to_level0 /
// k_spz_to_level0 / k_inriav2_to_level0.
// Level-0 records of `degree` land in the chunk buffer, or (generate mode: `whole` set) at their splat index in `whole` with the
// JavaScript numbers beside them in G.  The SH read from the file are min(degree, file degree); only INRIA v2 (generate mode only) is
// called with a larger degree, whose extra components are 0.  `prepare()` runs once the transient buffers exist (a failure before it
// leaves the caller's state alone); `after(first, n, records)` runs on the stream after each chunk's parse.  Only the records
// [begin, end) are read (a PlayCanvas file's `begin` is a multiple of 256: its chunks are converted whole).
template <typename Prepare, typename After>
static int parse_file_chunks(const FileLayout &L, const void *data, uint32_t degree, const Launch &launch, unsigned char *whole, GenOut G,
                             uint32_t begin, uint32_t end, Prepare prepare, After after) {
    cudaStream_t st = launch.stream();
    int rc;
    const uint32_t ncomp = degree == 2 ? 24 : (degree == 1 ? 9 : 0), out_bytes = 44 + 4 * ncomp;
    const uint32_t read_degree = std::min<uint32_t>(degree, (uint32_t)L.sh_degree);
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
    const uint32_t chunk_records = (uint32_t)std::min<size_t>(cap, ((size_t)std::max<uint32_t>(end - begin, 1) + unit - 1) / unit * unit);
    const size_t chunk_bytes = (size_t)chunk_records * row_bytes + pad;

    DevBuf<unsigned char> d_in, d_l0; DevBuf<double> d_tab; PinBuf<unsigned char> h_in[2];
    struct Events { cudaEvent_t ev[2] = {nullptr, nullptr}; ~Events() { for (cudaEvent_t x : ev) if (x) cudaEventDestroy(x); } } copied;
    if ((rc = d_in.ensure(chunk_bytes + 16)) || (!whole && (rc = d_l0.ensure((size_t)chunk_records * out_bytes)))) return rc;
    if (end > begin && ((rc = h_in[0].ensure(chunk_bytes)) || (end - begin > chunk_records && (rc = h_in[1].ensure(chunk_bytes))))) return rc;
    for (int i = 0; i < 2; ++i) CU(cudaEventCreateWithFlags(&copied.ev[i], cudaEventDisableTiming));
    if (L.pc && L.count) {   // the chunk table: 18 extremes per 256 splats, as f64
        const std::vector<double> tab = file_detail::pc_chunk_table((const unsigned char *)data, L);
        if ((rc = d_tab.ensure(tab.size()))) return rc;
        CU(cudaMemcpyAsync(d_tab.p, tab.data(), tab.size() * sizeof(double), cudaMemcpyHostToDevice, st));
        CU(cudaStreamSynchronize(st));   // pageable source
    }
    if (L.v2 && L.count && L.v2_rows) {   // INRIA v2: the codebook block, copied once and decoded to the f64 table [V2_PAGES][rows]
        DevBuf<unsigned char> d_cb;
        const size_t cb_bytes = (size_t)L.v2_rows * L.v2_row_stride;
        if ((rc = d_cb.ensure(std::max<size_t>(cb_bytes, 1))) || (rc = d_tab.ensure((size_t)V2_PAGES * L.v2_rows))) return rc;
        CU(cudaMemcpyAsync(d_cb.p, (const unsigned char *)data + L.v2_codebook_offset, cb_bytes, cudaMemcpyHostToDevice, st));
        V2CodebookParams CB{};
        CB.rows = L.v2_rows; CB.stride = L.v2_row_stride; CB.mask = L.v2_page_mask;
        memcpy(CB.offset, L.v2_page_offset, sizeof(CB.offset));
        launch.plain("k_inriav2_codebook", k_inriav2_codebook, (L.v2_rows + 127) / 128, 128, 0, d_cb.p, CB, d_tab.p);
        CU(cudaGetLastError());
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
    V2KernelParams VP{};
    VP.stride = L.stride; VP.out_bytes = out_bytes; VP.rows = L.v2_rows; VP.ncomp_out = (int)ncomp; VP.sh_per_channel = L.sh_per_channel;
    VP.ncomp_read = read_degree == 2 ? 24 : (read_degree == 1 ? 9 : 0); VP.staged = ply_smem;
    memcpy(VP.offset, L.offset, sizeof(VP.offset)); memcpy(VP.type, L.type, sizeof(VP.type));
    const unsigned char *src_sh = (const unsigned char *)data + L.pc_sh_offset;
    const unsigned char *src = (const unsigned char *)data + L.data_offset;
    for (uint32_t first = begin, k = 0; first < end; first += chunk_records, ++k) {
        const uint32_t n = std::min(chunk_records, end - first);
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
        launch.mark("h2d_file_chunk");
        const uint32_t grid = (n + cta - 1) / cta;
        PP.count = n;
        CP.count = n; CP.chunk_base = first / kPcChunkSplats;
        SP.count = n;
        VP.count = n;
        const uint32_t pc_grid = (n + kPcChunkSplats - 1) / kPcChunkSplats;
        // GEN (std::true_type / std::false_type): generate mode, the records of the whole scene in `whole` with the numbers beside them
        auto to_level0 = [&](auto gen, unsigned char *o, GenOut g) {
            constexpr bool GEN = decltype(gen)::value;
            if (L.v2) {
                if constexpr (GEN) launch.plain("k_inriav2_to_level0", k_inriav2_to_level0, grid, cta, ply_smem ? cta * L.stride : 0, d_in.p, d_tab.p, VP, o, g);
            } else if (spz) launch.plain("k_spz_to_level0", k_spz_to_level0<GEN>, (n + 127) / 128, 128, 0, d_in.p, SP, o, g);
            else if (L.format == GS_FILE_SPLAT) launch.plain("k_splat_to_level0", k_splat_to_level0<GEN>, (n + 127) / 128, 128, 0, d_in.p, n, o, g);
            else if (L.pc && pc_staged) launch.plain("k_pcply_to_level0", k_pcply_to_level0<true, GEN>, pc_grid, kPcChunkSplats, pc_smem, d_in.p, d_in.p + split, d_tab.p,
                                                     CP, o, g);
            else if (L.pc) launch.plain("k_pcply_to_level0", k_pcply_to_level0<false, GEN>, pc_grid, kPcChunkSplats, 0, d_in.p, d_in.p + split, d_tab.p, CP, o, g);
            else if (ply_smem) launch.plain("k_ply_to_level0", k_ply_to_level0<true, GEN>, grid, cta, cta * L.stride, d_in.p, PP, o, g);
            else launch.plain("k_ply_to_level0", k_ply_to_level0<false, GEN>, grid, cta, 0, d_in.p, PP, o, g);
        };
        if (whole) to_level0(std::true_type{}, whole + (size_t)first * out_bytes, GenOut{G.center + (size_t)first * 3, G.sh ? G.sh + (size_t)first * ncomp : nullptr});
        else to_level0(std::false_type{}, d_l0.p, GenOut{});
        CU(cudaGetLastError());
        if ((rc = after(first, n, whole ? whole + (size_t)first * out_bytes : d_l0.p))) return rc;
    }
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    return GS_OK;
}

// Steps 2 and 4 for a scene's parsed file in file order; `prepare` and `ms` as for decode_ksplat_image.
template <typename Prepare>
static int decode_file(gs_engine *e, const SceneLoad &c, const KSceneParams *ms, Prepare prepare) {
    const uint32_t degree = c.S.sh_degree;
    KSceneParams m{};
    if (ms) { m = *ms; m.sh_lo = c.S.min_sh_coeff; m.sh_hi = c.S.max_sh_coeff; }
    KSectionParams KP = level0_section(degree);   // each chunk of records is one level-0 section
    DevBuf<KTransform> d_xf;
    const Launch launch(e->stream, &e->prof);
    // parse_file_chunks allocates the transient buffers before it calls the hook
    auto hook = [&]() -> int {
        const int rc = upload_transform(e, c.o, c.S, d_xf);
        return rc ? rc : prepare();
    };
    return parse_file_chunks(c.L, c.src.data, degree, launch, nullptr, GenOut{}, 0, c.L.count, hook, [&](uint32_t first, uint32_t n, const unsigned char *d_l0) -> int {
        KP.count = n; KP.splat_offset = first;
        decode_section(e, c.o, d_l0, KP, 0, nullptr, d_xf.p, ms ? &m : nullptr, launch);
        CU(cudaGetLastError());
        return GS_OK;
    });
}

// ---------------------------------------------------------------------------------------------------------------
// Streamed uploads: the reference's progressive load (PlyLoader / SplatLoader / KSplatLoader.loadFromURL with progressiveLoadToSplatBuffer,
// Viewer.downloadAndBuildSingleSplatSceneProgressiveLoad).  The stream keeps every byte it has received on the host; each append converts
// and decodes the records it completes, with the kernels of gs_upload_file / gs_upload_ksplat, and commits the prefix.  So the engine
// holds, after every append, the whole-file upload restricted to the loaded prefix, and after close the whole-file upload itself.
struct gs_file_stream {
    gs_engine *e = nullptr;
    int format = 0;
    uint32_t sh_degree = 0;
    gs_ksplat_options o{};
    std::vector<unsigned char> bytes;    // everything received: a record split across appends waits here for its rest
    bool have_header = false, closed = false, broken = false;
    uint64_t generation = 0;             // the engine's scene generation since this stream's first commit (0: nothing committed yet)
    uint32_t loaded = 0, total = 0;      // splats committed; splats the header declares (.splat: whole rows received)
    gs_ksplat_info S{};                  // the whole file's report
    FileLayout L;                        // .ply / .splat
    KsplatLayout K;                      // .ksplat: the headers,
    std::vector<uint32_t> pre;           //   each section's partial-bucket prefixes at pre_at[i], read once its first record is complete
    std::vector<size_t> pre_at;
    std::vector<bool> pre_ready;
    size_t image_bytes = 0, copied = 0;  //   the image's size, and how much of it is on the device
    DevBuf<unsigned char> d_image;
    DevBuf<uint32_t> d_pre;
    DevBuf<KTransform> d_xf;
};

extern "C" int gs_stream_open(gs_engine *e, int format, uint32_t sh_degree, const gs_ksplat_options *opt, gs_file_stream **out) {
    if (!out) return fail(GS_ERR_BAD_ARG, "gs_stream_open: out is NULL");
    *out = nullptr;
    int rc;
    if ((rc = check_scene_engine(e, "gs_stream_open", sh_degree))) return rc;
    if (e->cfg.world_size > 1)
        return fail(GS_ERR_BAD_ARG, "gs_stream_open: engine with world_size %u: a streamed scene loads on one GPU only", e->cfg.world_size);
    if (format == GS_FILE_SPZ) return fail(GS_ERR_BAD_ARG, "gs_stream_open: .spz is not progressively loadable (Viewer.isProgressivelyLoadable)");
    if (format != GS_FILE_PLY && format != GS_FILE_SPLAT && format != GS_FILE_KSPLAT)
        return fail(GS_ERR_BAD_ARG, "gs_stream_open: file format %d unknown (GS_FILE_PLY = 1, GS_FILE_SPLAT = 2, GS_FILE_KSPLAT = 3)", format);
    gs_file_stream *s = new (std::nothrow) gs_file_stream;
    if (!s) return fail(GS_ERR_CAPACITY, "gs_stream_open: out of host memory");
    s->e = e; s->format = format; s->sh_degree = sh_degree; s->o = ksplat_options(opt);
    *out = s;
    return GS_OK;
}

extern "C" void gs_stream_destroy(gs_file_stream *s) { delete s; }

// The header, once its bytes are complete (have_header stays false until then): parsed and checked against the engine's capacity with the
// whole-file parsers, before the engine's scene is touched.
static int stream_header(gs_file_stream *s) {
    gs_engine *e = s->e;
    const unsigned char *f = s->bytes.data();
    const size_t n = s->bytes.size();
    int rc;
    if (s->format == GS_FILE_PLY) {
        const size_t end = ply_header_end(f, n);
        if (!end || end >= n) return GS_OK;   // the last header line or the byte after it is to come
        if ((rc = parse_scene_file(e, GS_FILE_PLY, f, n, false, s->L, true))) return rc;
        if (s->L.pc && s->L.pc_sh_file_degree)
            return fail(GS_ERR_BAD_ARG, ".ply: a PlayCanvas-compressed .ply with spherical harmonics is not progressively loadable (PlyLoader.js "
                                        "DirectLoadError)");
        s->total = s->L.count;
        s->S = scene_info(s->L.count, std::min<uint32_t>(s->sh_degree, (uint32_t)s->L.sh_degree), 0, 1);
        s->bytes.reserve(s->L.data_offset + (size_t)s->L.count * s->L.stride);
    } else if (s->format == GS_FILE_SPLAT) {
        s->L.format = GS_FILE_SPLAT; s->L.stride = 32;
        s->S = scene_info(0, 0, 0, 1);
    } else {
        if (n < 4096 || n < 4096ull + 1024ull * rd32(f + 4)) return GS_OK;
        // only the headers are read here (hence no size to check them against); each section's data is checked as it arrives
        if ((rc = parse_ksplat_head(f, SIZE_MAX, e->cfg.max_splat_count, s->K))) return rc;
        if (s->K.info.splat_count > s->K.max_splats)
            return fail(GS_ERR_CAPACITY, ".ksplat sections hold %u splats, more than the %u its header declares", s->K.info.splat_count, s->K.max_splats);
        s->total = s->K.info.splat_count;
        s->S = s->K.info;
        s->image_bytes = 4096ull + 1024ull * s->K.secs.size();
        for (const KSectionParams &P : s->K.secs) {
            s->pre_at.push_back(s->pre.size());
            s->pre.resize(s->pre.size() + P.partial_count + 1, 0);
            s->image_bytes = std::max<size_t>(s->image_bytes, P.data_base + (size_t)P.bytes_per_splat * P.count);
        }
        s->pre_ready.assign(s->K.secs.size(), false);
        if ((rc = s->d_image.ensure(s->image_bytes)) || (rc = s->d_pre.ensure(std::max<size_t>(s->pre.size(), 1)))) return rc;
    }
    if ((rc = upload_transform(e, s->o, s->S, s->d_xf))) return rc;
    s->have_header = true;
    return GS_OK;
}

// Splats whose records are complete in the bytes received
static uint32_t stream_complete(const gs_file_stream *s) {
    const size_t n = s->bytes.size();
    if (s->format != GS_FILE_KSPLAT) return n <= s->L.data_offset ? 0 : (uint32_t)std::min<size_t>(s->total, (n - s->L.data_offset) / s->L.stride);
    uint32_t done = 0;
    for (const KSectionParams &P : s->K.secs) {
        const uint32_t k = n <= P.data_base ? 0 : (uint32_t)std::min<size_t>(P.count, (n - P.data_base) / P.bytes_per_splat);
        done += k;
        if (k < P.count) break;
    }
    return done;
}

// .ply / .splat: records [s->loaded, upto) through parse_file_chunks and k_ksplat_decode, as decode_file runs them.  A PlayCanvas chunk
// (256 splats) shares one row of quantisation extremes, so the chunk holding s->loaded is converted from its start; its splats before
// s->loaded are not decoded again.
static int stream_decode_file(gs_file_stream *s, uint32_t upto) {
    gs_engine *e = s->e;
    const uint32_t degree = s->S.sh_degree, a = s->loaded;
    KSectionParams KP = level0_section(degree);
    const Launch launch(e->stream, &e->prof);
    const uint32_t begin = s->L.pc ? a / kPcChunkSplats * kPcChunkSplats : a;
    return parse_file_chunks(s->L, s->bytes.data(), degree, launch, nullptr, GenOut{}, begin, upto, [] { return GS_OK; },
                             [&](uint32_t first, uint32_t n, const unsigned char *d_l0) -> int {
        KP.count = n; KP.splat_offset = first;
        decode_section(e, s->o, d_l0, KP, first < a ? a - first : 0, nullptr, s->d_xf.p, nullptr, launch);
        CU(cudaGetLastError());
        return GS_OK;
    });
}

// .ksplat: the new bytes to the device image, then each section's records in [s->loaded, upto) through k_ksplat_decode
static int stream_decode_ksplat(gs_file_stream *s, uint32_t upto) {
    gs_engine *e = s->e;
    cudaStream_t st = e->stream;
    int rc;
    const size_t to = std::min(s->bytes.size(), s->image_bytes);
    if (to > s->copied) {
        CU(cudaMemcpyAsync(s->d_image.p + s->copied, s->bytes.data() + s->copied, to - s->copied, cudaMemcpyHostToDevice, st));
        s->copied = to;
    }
    const Launch launch(st, &e->prof);
    for (size_t i = 0; i < s->K.secs.size(); ++i) {
        KSectionParams P = s->K.secs[i];
        if (upto <= P.splat_offset || s->loaded >= P.splat_offset + P.count) continue;
        const uint32_t a = std::max(s->loaded, P.splat_offset) - P.splat_offset, b = std::min(upto, P.splat_offset + P.count) - P.splat_offset;
        if (!s->pre_ready[i]) {   // its partial-bucket lengths precede its records, so they are complete
            KsplatLayout one;
            one.max_splats = s->K.max_splats; one.secs = {P};
            std::vector<uint32_t> q;
            if ((rc = ksplat_prefixes(one, {s->bytes.data() + P.base}, e->cfg.max_splat_count, q))) return rc;
            std::copy(q.begin(), q.end(), s->pre.begin() + s->pre_at[i]);
            CU(cudaMemcpyAsync(s->d_pre.p + s->pre_at[i], s->pre.data() + s->pre_at[i], q.size() * 4, cudaMemcpyHostToDevice, st));
            s->pre_ready[i] = true;
        }
        P.count = b;
        decode_section(e, s->o, s->d_image.p, P, a, s->d_pre.p + s->pre_at[i], s->d_xf.p, nullptr, launch);
        CU(cudaGetLastError());
    }
    CU(cudaStreamSynchronize(st));   // pageable sources
    CU(cudaGetLastError());
    return GS_OK;
}

// The prefix [0, upto) committed as a whole one-scene upload is; the first commit replaces the engine's scene.
static int stream_commit(gs_file_stream *s, uint32_t upto) {
    gs_engine *e = s->e;
    int rc;
    if (!s->generation) {
        if ((rc = clear_scene(e, s->o, s->S))) return rc;
        s->generation = e->rs.generation;
    }
    if (upto > s->loaded && (rc = s->format == GS_FILE_KSPLAT ? stream_decode_ksplat(s, upto) : stream_decode_file(s, upto))) return rc;
    s->loaded = upto;
    SceneLoad c;
    c.o = s->o; c.S = s->S;
    c.S.splat_count = upto;
    return commit_scenes(e, &c, 1);
}

static int stream_advance(gs_file_stream *s) {
    int rc;
    if (!s->have_header && ((rc = stream_header(s)) || !s->have_header)) return rc;
    gs_engine *e = s->e;
    if (s->generation && s->generation != e->rs.generation)
        return fail(GS_ERR_NOT_READY, "gs_stream_append: the engine's scene was replaced after this stream's first splats");
    if (s->format == GS_FILE_SPLAT) {
        const size_t rows = s->bytes.size() / 32;
        if (rows > e->cfg.max_splat_count) return fail(GS_ERR_CAPACITY, "the stream holds %zu splats, engine capacity %u", rows, e->cfg.max_splat_count);
        s->total = (uint32_t)rows;
    }
    const uint32_t upto = stream_complete(s);
    return upto > s->loaded ? stream_commit(s, upto) : GS_OK;
}

// What the stream reports after an append or at close: the file's report with the loaded count (zero until the header is in)
static void stream_info(const gs_file_stream *s, gs_ksplat_info *info) {
    gs_ksplat_info S = s->S;
    S.struct_size = sizeof(S);
    S.splat_count = s->loaded;
    write_info(info, S);
}

extern "C" int gs_stream_append(gs_file_stream *s, const void *data, size_t bytes, gs_ksplat_info *progress) {
    if (!s) return fail(GS_ERR_BAD_ARG, "gs_stream_append: null stream");
    if (s->closed) return fail(GS_ERR_BAD_ARG, "gs_stream_append: the stream is closed");
    if (s->broken) return fail(GS_ERR_BAD_ARG, "gs_stream_append: an earlier append failed; the stream stopped at %u splats", s->loaded);
    if (!data && bytes) return fail(GS_ERR_BAD_ARG, "gs_stream_append: null data");
    int rc = check_engine(s->e);
    if (!rc) {
        s->bytes.insert(s->bytes.end(), (const unsigned char *)data, (const unsigned char *)data + bytes);
        rc = stream_advance(s);
        s->broken = rc != GS_OK;
    }
    stream_info(s, progress);
    return rc;
}

extern "C" int gs_stream_close(gs_file_stream *s, gs_ksplat_info *info) {
    if (!s) return fail(GS_ERR_BAD_ARG, "gs_stream_close: null stream");
    if (s->closed) return fail(GS_ERR_BAD_ARG, "gs_stream_close: the stream is already closed");
    s->closed = true;
    if (s->broken) return fail(GS_ERR_BAD_ARG, "gs_stream_close: an earlier append failed; the stream stopped at %u splats", s->loaded);
    int rc;
    if ((rc = check_engine(s->e))) return rc;
    if (!s->have_header)
        return fail(GS_ERR_BAD_ARG, "gs_stream_close: the stream ended inside the file's header (%zu bytes received)", s->bytes.size());
    if (s->generation && s->generation != s->e->rs.generation)
        return fail(GS_ERR_NOT_READY, "gs_stream_close: the engine's scene was replaced after this stream's first splats");
    if (s->format == GS_FILE_SPLAT && s->bytes.size() % 32)
        return fail(GS_ERR_BAD_ARG, "gs_stream_close: the stream ended short: %u splats loaded, %zu bytes of splat %u (32-byte rows) received",
                    s->loaded, s->bytes.size() % 32, s->loaded + 1);
    if (s->loaded < s->total)
        return fail(GS_ERR_BAD_ARG, "gs_stream_close: the stream ended short: %u of the %u splats its header declares were loaded", s->loaded, s->total);
    if (!s->generation && (rc = stream_commit(s, 0))) return rc;   // a file without splats still replaces the scene, as gs_upload_file does
    stream_info(s, info);
    return GS_OK;
}

extern "C" int gs_visible_region(gs_engine *e, uint32_t from, uint32_t to, const double *transform, const double *scene_center, double *max_distance) {
    int rc;
    if ((rc = check_engine(e))) return rc;
    if (!max_distance) return fail(GS_ERR_BAD_ARG, "gs_visible_region: max_distance is NULL");
    if (from > to || to > e->rs.uploaded) return fail(GS_ERR_BAD_ARG, "gs_visible_region: splats [%u, %u) outside the %u uploaded", from, to, e->rs.uploaded);
    RegionParams P{};
    for (int k = 0; k < 16; ++k) P.t[k] = transform ? transform[k] : (k % 5 == 0 ? 1.0 : 0.0);
    for (int k = 0; k < 3; ++k) P.center[k] = scene_center ? scene_center[k] : 0.0;
    if ((rc = e->region_max.ensure(1))) return rc;
    cudaStream_t st = e->stream;
    CU(cudaMemsetAsync(e->region_max.p, 0, sizeof(unsigned long long), st));
    if (to > from) {
        const uint32_t grid = std::min<uint32_t>((to - from + 255) / 256, (uint32_t)e->sm_count * 8);
        Launch(st, &e->prof).plain("k_visible_region", k_visible_region, grid, 256, 0, e->rs.cc.p, from, to, P, e->region_max.p);
    }
    unsigned long long bits = 0;
    CU(cudaMemcpyAsync(&bits, e->region_max.p, sizeof(bits), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    memcpy(max_distance, &bits, sizeof(bits));
    return GS_OK;
}

// SplatMesh.computeBoundingBox on the GPU (region_kernels.cuh).  Centres: the ray records where the decode wrote them (getSplatCenter's
// unrounded centre), else the f32 centres, as gs_build_splat_tree takes them.  `apply` marks the scenes whose centres go through xf.
extern "C" int gs_compute_bounding_box(gs_engine *e, const gs_bounding_box_params *p, float out_min[3], float out_max[3]) {
    int rc;
    if ((rc = check_engine(e))) return rc;
    if (!out_min || !out_max) return fail(GS_ERR_BAD_ARG, "gs_compute_bounding_box: null output");
    gs_bounding_box_params defaults{};
    defaults.scene_index = -1;
    const gs_bounding_box_params q = read_options(p, defaults);
    const uint32_t scenes = e->scenes_multi ? (uint32_t)e->scene_start.size() - 1 : 1;
    if (q.scene_index < -1 || q.scene_index >= (int32_t)scenes)
        return fail(GS_ERR_BAD_ARG, "gs_compute_bounding_box: invalid scene index %d (the mesh has %u scene%s)", q.scene_index, scenes, scenes == 1 ? "" : "s");
    BoundsParams P{};
    P.from = 0; P.to = e->rs.uploaded;
    if (q.scene_index >= 0 && e->scenes_multi) { P.from = e->scene_start[q.scene_index]; P.to = e->scene_start[q.scene_index + 1]; }
    const uint32_t range_scenes = q.scene_index < 0 ? (scenes == 32 ? ~0u : (1u << scenes) - 1) : 1u << q.scene_index;
    const bool records = e->tree.decoded_ray_records && e->ray.valid;
    std::vector<double> xf(16 * GS_MAX_SCENES, 0.0);
    for (int s = 0; s < GS_MAX_SCENES; ++s) xf[16 * s] = xf[16 * s + 5] = xf[16 * s + 10] = xf[16 * s + 15] = 1.0;
    bool ray_xf = false;                   // the static mesh's transforms the ray records keep
    if (!q.apply_scene_transforms) {
        // only the transformed centres are kept of a scene decoded with a transform
        if (!records && (e->baked_xf & range_scenes))
            return fail(GS_ERR_BAD_ARG, "gs_compute_bounding_box: apply_scene_transforms 0, but scene %d was loaded with its transform baked into its centres "
                        "and the engine has no ray records: only the transformed centres are kept", __builtin_ctz(e->baked_xf & range_scenes));
    } else if (e->cfg.dynamic_mode) {
        P.apply = ~0u;
        if (q.scene_transforms) memcpy(xf.data(), q.scene_transforms, sizeof(double) * 16 * scenes);
    } else if (records) {
        P.apply = ~0u;
        ray_xf = true;                     // each scene's transform, the identity for a scene without one
    } else {
        P.apply = ~e->baked_xf;            // the identity for the others: the reference multiplies by it too (0 * inf = NaN)
    }
    P.scene_idx = e->rs.have_scene_idx ? e->rs.scene_idx.p : nullptr;
    if (P.to == P.from) {   // new THREE.Vector3()
        for (int a = 0; a < 3; ++a) out_min[a] = out_max[a] = 0.0f;
        return GS_OK;
    }
    const uint32_t blocks = std::min<uint32_t>((P.to - P.from + kBoundsThreads - 1) / kBoundsThreads, (uint32_t)e->sm_count * (2048 / kBoundsThreads));
    if ((rc = e->bounds_xf.ensure(xf.size())) || (rc = e->bounds_partial.ensure(6 * (size_t)blocks)) || (rc = e->bounds_out.ensure(6))) return rc;
    cudaStream_t st = e->stream;
    if (!ray_xf) CU(cudaMemcpyAsync(e->bounds_xf.p, xf.data(), xf.size() * sizeof(double), cudaMemcpyHostToDevice, st));
    P.xf = ray_xf ? e->ray.xf.p : e->bounds_xf.p;
    const Launch launch(st, &e->prof);
    if (records) {
        launch.plain("k_bounding_box", k_bounding_box<true>, blocks, kBoundsThreads, 0, (const void *)e->ray.rec.p, P, e->bounds_partial.p);
        launch.plain("k_bounding_box_final", k_bounding_box_final<true>, 1, kBoundsThreads, 0, (const void *)e->ray.rec.p, P, e->bounds_partial.p, blocks, e->bounds_out.p);
    } else {
        launch.plain("k_bounding_box", k_bounding_box<false>, blocks, kBoundsThreads, 0, (const void *)e->rs.cc.p, P, e->bounds_partial.p);
        launch.plain("k_bounding_box_final", k_bounding_box_final<false>, 1, kBoundsThreads, 0, (const void *)e->rs.cc.p, P, e->bounds_partial.p, blocks, e->bounds_out.p);
    }
    float box[6];
    CU(cudaMemcpyAsync(box, e->bounds_out.p, sizeof(box), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    memcpy(out_min, box, 12);
    memcpy(out_max, box + 3, 12);
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

// Stable sort of `order` (n entries, nullptr = identity; `out` may be `order`) by a 64-bit key indexed by element, `bits` low bits, in 24-bit rounds.
static int gen_sort(PiecewiseSort &sorter, const unsigned long long *key, const uint32_t *order, uint32_t n, int bits, uint32_t *out, const Launch &launch) {
    int widths[3], rounds = 0;
    for (int left = bits; rounds == 0 || left > 0; left -= 24) widths[rounds++] = std::min(24, left);
    return sorter.sort(order, n, widths, rounds, out, [&](const Launch &launch, int r, const uint32_t *in, uint32_t *keys, uint32_t *vals) {
        launch.plain(nullptr, k_gen_sort_piece, (n + 255) / 256, 256, 0, key, in, n, 24 * r, keys, vals);
    }, launch);
}

// out[0..n]: exclusive scan of in[0..n), out[n] = total
static int gen_scan(const uint32_t *in, uint32_t n, uint32_t *out, DevBuf<uint32_t> &sums, const Launch &launch) {
    cudaStream_t st = launch.stream();
    int rc;
    const uint32_t tiles = (uint32_t)(((uint64_t)n + kScanTile - 1) / kScanTile);
    if ((rc = sums.ensure(tiles + 1))) return rc;
    CU(cudaMemsetAsync(sums.p + tiles, 0, 4, st));
    if (tiles) launch.plain(nullptr, k_gen_scan_reduce, tiles, kScanThreads, 0, in, n, sums.p);
    launch.plain(nullptr, k_exclusive_scan_single_block, 1, 1024, 0, sums.p, tiles + 1);
    if (tiles) launch.plain(nullptr, k_gen_scan_apply, tiles, kScanThreads, 0, in, n, sums.p, tiles, out);
    else CU(cudaMemsetAsync(out, 0, 4, st));
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

static int generate_image(const FileLayout &L, const void *data, uint32_t sh_degree, const gs_generate_options &g, const Launch &launch, GenImage &out) {
    cudaStream_t st = launch.stream();
    int rc;
    // The image's SH degree is min(sh_degree, file degree), except for INRIA v2: its unified UncompressedSplatArray is built at the
    // requested degree, so the image carries sh_degree with 0 past the file's coefficients, and the SH range scan sees only the latter.
    const uint32_t read_degree = std::min<uint32_t>(sh_degree, (uint32_t)L.sh_degree), degree = L.v2 ? sh_degree : read_degree;
    const uint32_t ncomp = degree == 2 ? 24 : (degree == 1 ? 9 : 0), rec_bytes = 44 + 4 * ncomp, n = L.count;
    const uint32_t read_ncomp = read_degree == 2 ? 24 : (read_degree == 1 ? 9 : 0);
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
    PiecewiseSort sorter;   // every sort below orders at most n entries
    if ((rc = sorter.reserve(n, 24, st)) || (rc = rec0.ensure((size_t)n * rec_bytes)) || (rc = c64.ensure((size_t)n * 3)) || (ncomp && (rc = sh64.ensure((size_t)n * ncomp)))) return rc;
    rc = parse_file_chunks(L, data, degree, launch, rec0.p, GenOut{c64.p, ncomp ? sh64.p : nullptr}, 0, L.count, [] { return GS_OK; },
                           [](uint32_t, uint32_t, const unsigned char *) { return GS_OK; });
    if (rc) return rc;
    const uint32_t grid_n = (n + kGenThreads - 1) / kGenThreads;
    // ---- partition order
    if ((rc = key.ensure(n)) || (rc = perm.ensure(n))) return rc;
    if (n) launch.plain(nullptr, k_gen_partition_key, grid_n, kGenThreads, 0, c64.p, n, g.scene_center[0], g.scene_center[1], g.scene_center[2], key.p);
    if ((rc = gen_sort(sorter, key.p, nullptr, n, 64, perm.p, launch))) return rc;
    launch.mark("gen_partition");
    // ---- SH range over FRC0..FRC22 of every splat, partition order
    const uint32_t sh_blocks = (uint32_t)(((uint64_t)n + kGenThreads * kGenShItems - 1) / (kGenThreads * kGenShItems));
    if ((rc = range.ensure(2)) || (rc = runs.ensure(2 * (size_t)std::max(sh_blocks, 1u)))) return rc;
    if (read_ncomp && sh_blocks)
        launch.plain(nullptr, k_gen_sh_scan, sh_blocks, kGenThreads, 0, sh64.p, (int)ncomp, (int)std::min(read_ncomp, 23u), perm.p, n, runs.p);
    launch.plain(nullptr, k_gen_sh_final, 1, 1, 0, runs.p, read_ncomp ? sh_blocks : 0, range.p);
    launch.mark("gen_sh_range");
    // ---- alpha removal
    if ((rc = keep.ensure(n)) || (rc = kscan.ensure((size_t)n + 1)) || (rc = src.ensure(n)) || (rc = sec.ensure(n)) || (rc = sec_base.ensure((size_t)nsec + 1)))
        return rc;
    if (n) launch.plain(nullptr, k_gen_keep, grid_n, kGenThreads, 0, rec0.p, rec_bytes, perm.p, n, g.minimum_alpha, keep.p);
    if ((rc = gen_scan(keep.p, n, kscan.p, sums, launch))) return rc;
    if (n) launch.plain(nullptr, k_gen_compact, grid_n, kGenThreads, 0, perm.p, keep.p, kscan.p, n, std::max(S, 1u), src.p, sec.p);
    launch.plain(nullptr, k_gen_section_base, nsec / 256 + 1, 256, 0, kscan.p, n, std::max(S, 1u), nsec, sec_base.p);
    uint32_t m = 0;
    CU(cudaMemcpyAsync(&m, kscan.p + n, 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    launch.mark("gen_alpha");
    const uint32_t grid_m = (m + kGenThreads - 1) / kGenThreads, grid_s = nsec / 256 + 1;
    // ---- bounds and bucket keys per section
    if ((rc = bmin.ensure((size_t)nsec * 3 + 1)) || (rc = bmax.ensure((size_t)nsec * 3 + 1)) || (rc = nanf.ensure((size_t)nsec * 3 + 1)) ||
        (rc = geom.ensure((size_t)nsec + 1)) || (rc = lo.ensure(m)) || (rc = hi.ensure(m)) || (rc = bcenter.ensure((size_t)m * 3)) || (rc = order.ensure(m)))
        return rc;
    CU(cudaMemsetAsync(bmin.p, 0xff, ((size_t)nsec * 3 + 1) * 8, st));
    CU(cudaMemsetAsync(bmax.p, 0, ((size_t)nsec * 3 + 1) * 8, st));
    CU(cudaMemsetAsync(nanf.p, 0, ((size_t)nsec * 3 + 1) * 4, st));
    if (m) {
        launch.plain(nullptr, k_gen_bounds, grid_m, kGenThreads, 0, c64.p, src.p, sec.p, sec_base.p, m, bmin.p, bmax.p, nanf.p);
        launch.plain(nullptr, k_gen_geometry, grid_s, 256, 0, bmin.p, bmax.p, nanf.p, sec_base.p, nsec, g.block_size, geom.p);
        launch.plain(nullptr, k_gen_bucket_key, grid_m, kGenThreads, 0, c64.p, src.p, sec.p, geom.p, m, g.block_size, lo.p, hi.p, bcenter.p);
    }
    int sec_bits = 1;
    while (sec_bits < 40 && (1ull << sec_bits) < 2ull * nsec) ++sec_bits;
    if ((rc = gen_sort(sorter, lo.p, nullptr, m, 64, order.p, launch)) || (rc = gen_sort(sorter, hi.p, order.p, m, sec_bits, order.p, launch))) return rc;
    launch.mark("gen_bucket_sort");
    // ---- groups of equal (section, key), bucket fill
    if ((rc = head.ensure(m)) || (rc = gscan.ensure((size_t)m + 1)) || (rc = complete.ensure(m)) || (rc = fscan.ensure((size_t)m + 1)) ||
        (rc = fbase.ensure((size_t)nsec + 1)))
        return rc;
    if (m) launch.plain(nullptr, k_gen_heads, grid_m, kGenThreads, 0, lo.p, hi.p, order.p, m, head.p);
    if ((rc = gen_scan(head.p, m, gscan.p, sums, launch))) return rc;
    uint32_t groups = 0;
    CU(cudaMemcpyAsync(&groups, gscan.p + m, 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if ((rc = gstart.ensure((size_t)groups + 1)) || (rc = pflag.ensure(groups)) || (rc = pscan.ensure((size_t)groups + 1)) || (rc = pkey_lo.ensure(groups)) ||
        (rc = pkey_hi.ensure(groups)) || (rc = pinv.ensure(groups)))
        return rc;
    launch.plain(nullptr, k_gen_group_start, grid_m + 1, kGenThreads, 0, head.p, gscan.p, m, gstart.p);
    if (m) launch.plain(nullptr, k_gen_complete, grid_m, kGenThreads, 0, order.p, gscan.p, gstart.p, m, B, complete.p);
    if ((rc = gen_scan(complete.p, m, fscan.p, sums, launch))) return rc;
    launch.plain(nullptr, k_gen_gather_base, grid_s, 256, 0, fscan.p, sec_base.p, nsec, fbase.p);
    // ---- partial buckets: order within each section, lengths, counts
    const uint32_t grid_g = (groups + kGenThreads - 1) / kGenThreads;
    if (groups) launch.plain(nullptr, k_gen_partial_keys, grid_g, kGenThreads, 0, order.p, gstart.p, groups, B, hi.p, pflag.p, pkey_lo.p, pkey_hi.p);
    if ((rc = gen_scan(pflag.p, groups, pscan.p, sums, launch))) return rc;
    uint32_t np = 0;
    CU(cudaMemcpyAsync(&np, pscan.p + groups, 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if ((rc = plist.ensure(np)) || (rc = porder.ensure(np)) || (rc = plen.ensure(np)) || (rc = pprefix.ensure((size_t)np + 1)) || (rc = pcount.ensure((size_t)nsec + 1)) ||
        (rc = pbase.ensure((size_t)nsec + 1)) || (rc = bbase.ensure((size_t)nsec + 1)))
        return rc;
    if (groups) launch.plain(nullptr, k_gen_partial_list, grid_g, kGenThreads, 0, pflag.p, pscan.p, groups, plist.p);
    if ((rc = gen_sort(sorter, pkey_lo.p, plist.p, np, 32, porder.p, launch)) || (rc = gen_sort(sorter, pkey_hi.p, porder.p, np, sec_bits, porder.p, launch))) return rc;
    CU(cudaMemsetAsync(pcount.p, 0, ((size_t)nsec + 1) * 4, st));
    if (np) launch.plain(nullptr, k_gen_partial_info, (np + kGenThreads - 1) / kGenThreads, kGenThreads, 0, porder.p, np, gstart.p, B, pkey_hi.p, pinv.p, plen.p,
                         pcount.p);
    if ((rc = gen_scan(pcount.p, nsec, pbase.p, sums, launch)) || (rc = gen_scan(plen.p, np, pprefix.p, sums, launch))) return rc;
    const GenLayout GL{sec_base.p, fbase.p, pbase.p, pprefix.p};
    launch.plain(nullptr, k_gen_bucket_base, grid_s, 256, 0, GL, nsec, bbase.p);
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
    if (m) launch.plain(nullptr, k_gen_slots, grid_m, kGenThreads, 0, order.p, gscan.p, gstart.p, fscan.p, pinv.p, src.p, sec.p, bcenter.p, m, B, GL, out_src.p,
                        out_bucket.p, bucket_center.p);
    launch.mark("gen_buckets");
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
    if (m) launch.plain(nullptr, k_gen_write, grid_m, kGenThreads, 0, rec0.p, c64.p, ncomp ? sh64.p : nullptr, out_src.p, out_bucket.p, bucket_center.p, sec_base.p,
                        offs.p, range.p, WP, out.image.p);
    const uint32_t nmeta = std::max(nbuckets, h_p[nsec]);
    if (level >= 1 && nmeta)
        launch.plain(nullptr, k_gen_bucket_meta, (nmeta + 255) / 256, 256, 0, bucket_center.p, plen.p, GL, nsec, nbuckets, h_p[nsec], offs.p + nsec, bbase.p,
                     out.image.p);
    launch.mark("gen_write");
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
    int rc = generate_image(L, data, sh_degree, g, Launch(st), out);
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

// Steps 2 and 4 for a file through the generator: its image is generated, c.K, c.pre and c.S become the image's, and the image is decoded
// in place; `prepare` and `ms` as for decode_ksplat_image.  c.S.sh_degree is the degree generate_image is asked for: the scene's degree
// (min(sphericalHarmonicsDegree, file degree), or sphericalHarmonicsDegree for INRIA v2) leads it to the same image.
template <typename Prepare>
static int decode_generated(gs_engine *e, SceneLoad &c, const KSceneParams *ms, Prepare prepare) {
    int rc;
    GenImage out;
    if ((rc = generate_image(c.L, c.src.data, c.S.sh_degree, c.g, Launch(e->stream, &e->prof), out))) return rc;
    // The image is decoded in place; of its bytes the host reads only the headers, which it wrote, and the partial-bucket lengths.
    const uint32_t room = e->cfg.max_splat_count - (ms ? ms->offset : 0u);
    if ((rc = parse_ksplat_head(out.head.data(), out.bytes, room, c.K))) return rc;
    size_t nlens = 0;
    for (const KSectionParams &P : c.K.secs) nlens += P.partial_count;
    std::vector<uint32_t> h_lens(nlens);
    std::vector<const unsigned char *> lens;
    size_t at = 0;
    for (const KSectionParams &P : c.K.secs) {
        if (P.partial_count) CU(cudaMemcpyAsync(h_lens.data() + at, out.image.p + P.base, 4ull * P.partial_count, cudaMemcpyDeviceToHost, e->stream));
        lens.push_back((const unsigned char *)(h_lens.data() + at));
        at += P.partial_count;
    }
    CU(cudaStreamSynchronize(e->stream));
    if ((rc = ksplat_prefixes(c.K, lens, room, c.pre))) return rc;
    c.S = c.K.info;
    return decode_ksplat_image(e, c, out.image.p, ms, prepare);
}

// Step 1 for one scene, after its entry's own checks: its header, and its splats against the room left after `before` splats of the
// mesh; c.S = what it reports at `sh_degree` (an optimized file's: before generation).
static int parse_scene(const gs_engine *e, SceneLoad &c, uint32_t sh_degree, uint32_t before) {
    const gs_scene_source &q = c.src;
    const uint32_t room = e->cfg.max_splat_count - before;
    int rc;
    if (q.format == GS_FILE_KSPLAT) {
        if ((rc = parse_ksplat(q.data, q.bytes, room, c.K, c.pre))) return rc;
        c.S = c.K.info;
        c.S.sh_degree = std::min(c.S.sh_degree, sh_degree);
        return GS_OK;
    }
    if ((rc = parse_scene_file(e, q.format, q.data, q.bytes, q.optimized, c.L))) return rc;
    if (c.L.count > room) return fail(GS_ERR_CAPACITY, "%u splats after %u, engine capacity %u", c.L.count, before, e->cfg.max_splat_count);
    const uint32_t d = std::min<uint32_t>(sh_degree, (uint32_t)c.L.sh_degree);   // min(sphericalHarmonicsDegree, file degree)
    c.S = scene_info(c.L.count, q.optimized && c.L.v2 ? sh_degree : d, q.optimized ? c.g.compression_level : 0, 1);
    return GS_OK;
}

// Steps 2-5 for `count` >= 1 scenes parsed by step 1, as one mesh in order; infos[s] (infos may be nullptr) gets scene s's report.  On a
// failure in a scene's steps 2-4, *failed = that scene.
static int load_scenes(gs_engine *e, SceneLoad *sc, uint32_t count, gs_ksplat_info *infos, uint32_t *failed = nullptr) {
    const bool multi = count > 1;
    int rc;
    // several scenes' formats (SplatMesh.js:324-331, 1064-1078): the lowest SH degree, the highest level
    uint32_t total = 0, degree = 2, level = 0;
    for (uint32_t s = 0; s < count; ++s) {
        total += sc[s].S.splat_count;
        degree = std::min(degree, sc[s].S.sh_degree);
        level = std::max(level, sc[s].S.compression_level);
    }
    if (multi && (rc = e->rs.scene_idx.ensure(std::max<uint32_t>(e->cfg.max_splat_count, 1)))) return rc;
    e->prof.begin(e->stream);   // gs_set_profiling: the upload's timeline (tools/load_bench.py)
    uint32_t offset = 0;
    for (uint32_t s = 0; s < count; ++s) {
        SceneLoad &c = sc[s];
        KSceneParams ms{};
        ms.scene = s; ms.offset = offset; ms.sh_u8 = level == 2;
        ms.raster_scene_idx = e->rs.scene_idx.p;
        ms.sort_scene_idx = e->scene_idx.p;   // dynamic engines only
        const KSceneParams *m = multi ? &ms : nullptr;
        // step 3 for the mesh, in the first scene; one scene's formats are its own (an optimized file's: its generated image's)
        auto prepare = [&]() -> int { return s ? GS_OK : clear_scene(e, c.o, multi ? scene_info(total, degree, level, 0) : c.S); };
        if (c.src.format == GS_FILE_KSPLAT) rc = decode_ksplat_image(e, c, nullptr, m, prepare);
        else if (c.src.optimized) rc = decode_generated(e, c, m, prepare);
        else rc = decode_file(e, c, m, prepare);
        if (rc) {
            if (failed) *failed = s;
            return rc;
        }
        c.S.splat_offset = offset;
        offset += c.S.splat_count;
    }
    if ((rc = commit_scenes(e, sc, count))) return rc;
    if (infos)
        for (uint32_t s = 0; s < count; ++s) write_info(&infos[s], sc[s].S);
    return GS_OK;
}

extern "C" int gs_upload_ksplat(gs_engine *e, const void *data, size_t bytes, const gs_ksplat_options *opt, gs_ksplat_info *info) {
    int rc;
    if ((rc = check_scene_engine(e, "gs_upload_ksplat", 0))) return rc;
    SceneLoad c;
    c.src.format = GS_FILE_KSPLAT; c.src.data = data; c.src.bytes = bytes;
    c.o = ksplat_options(opt);
    // sphericalHarmonicsDegree 2: the file's own degree is kept
    if ((rc = parse_scene(e, c, 2, 0))) return rc;
    return load_scenes(e, &c, 1, info);
}

// A .ksplat given to a file entry is refused as parse_file refuses every format it does not know.
extern "C" int gs_upload_file(gs_engine *e, int format, const void *data, size_t bytes, uint32_t sh_degree, const gs_ksplat_options *opt,
                              gs_ksplat_info *info) {
    int rc;
    if ((rc = check_scene_engine(e, "gs_upload_file", sh_degree))) return rc;
    SceneLoad c;
    c.src.format = format; c.src.data = data; c.src.bytes = bytes;
    c.o = ksplat_options(opt);
    if ((rc = format == GS_FILE_KSPLAT ? parse_scene_file(e, format, data, bytes, false, c.L) : parse_scene(e, c, sh_degree, 0))) return rc;
    return load_scenes(e, &c, 1, info);
}

extern "C" int gs_upload_file_optimized(gs_engine *e, int format, const void *data, size_t bytes, uint32_t sh_degree, const gs_ksplat_options *opt,
                                        const gs_generate_options *gen, gs_ksplat_info *info) {
    int rc;
    if ((rc = check_scene_engine(e, "gs_upload_file_optimized", sh_degree))) return rc;
    SceneLoad c;
    c.src.format = format; c.src.data = data; c.src.bytes = bytes; c.src.optimized = 1;
    c.o = ksplat_options(opt);
    if ((rc = check_generate_options(gen, c.g)) ||
        (rc = format == GS_FILE_KSPLAT ? parse_scene_file(e, format, data, bytes, true, c.L) : parse_scene(e, c, sh_degree, 0)))
        return rc;
    return load_scenes(e, &c, 1, info);
}

// ---------------------------------------------------------------------------------------------------------------
// Several scenes in one mesh (SplatMesh.build, SplatMesh.js:306-405), each loaded as its single-scene entry loads it.  A failing scene
// is named (in front of the parser's or the loader's message).
static int scene_fail(int rc, uint32_t s) {
    if (rc) {
        char t[sizeof(g_err)];
        snprintf(t, sizeof(t), "gs_upload_scenes: scene %u: %s", s, g_err);
        memcpy(g_err, t, sizeof(t));
    }
    return rc;
}

extern "C" int gs_upload_scenes(gs_engine *e, const gs_scene_source *scenes, uint32_t scene_count, uint32_t sh_degree, const gs_ksplat_options *mesh_opt,
                                gs_ksplat_info *infos) {
    int rc;
    if ((rc = check_scene_engine(e, "gs_upload_scenes", sh_degree))) return rc;
    if (!scenes || scene_count < 1 || scene_count > GS_MAX_SCENES)
        return fail(GS_ERR_BAD_ARG, "gs_upload_scenes: %u scenes%s (1..%d)", scene_count, scenes ? "" : " at NULL", GS_MAX_SCENES);
    if (scene_count > 1 && e->cfg.world_size > 1)
        return fail(GS_ERR_BAD_ARG, "gs_upload_scenes: %u scenes on an engine with world_size %u: multi-scene frames are single-GPU only", scene_count,
                    e->cfg.world_size);
    const gs_ksplat_options mo = ksplat_options(mesh_opt);
    std::vector<SceneLoad> sc(scene_count);
    // Step 1: every scene, before anything is touched
    uint32_t total = 0;
    for (uint32_t s = 0; s < scene_count; ++s) {
        SceneLoad &c = sc[s];
        c.src = read_options(&scenes[s], gs_scene_source{});
        const gs_scene_source &q = c.src;
        c.o = mo;   // with this scene's minimum_alpha and transform
        c.o.minimum_alpha = q.minimum_alpha ? q.minimum_alpha : 1;
        c.o.has_transform = q.has_transform;
        memcpy(c.o.transform, q.transform, sizeof(c.o.transform));
        if (!q.data) return scene_fail(fail(GS_ERR_BAD_ARG, "null data"), s);
        if (q.has_transform && e->cfg.dynamic_mode)
            return scene_fail(fail(GS_ERR_BAD_ARG, "has_transform on a dynamic engine (its transform is applied per frame: scene_transforms)"), s);
        if (q.format == GS_FILE_KSPLAT && q.optimized) return scene_fail(fail(GS_ERR_BAD_ARG, "a .ksplat is loaded as stored (optimized applies to files)"), s);
        if (q.optimized && (rc = check_generate_options(q.generate.struct_size ? &q.generate : nullptr, c.g))) return scene_fail(rc, s);
        if ((rc = parse_scene(e, c, sh_degree, total))) return scene_fail(rc, s);
        total += c.S.splat_count;
    }
    uint32_t failed = scene_count;
    rc = load_scenes(e, sc.data(), scene_count, infos, &failed);
    return failed < scene_count ? scene_fail(rc, failed) : rc;
}

// ---------------------------------------------------------------------------------------------------------------
// The SplatTree built on the device from the uploaded scene (tree_kernels.cuh), one level of the octree at a time.
namespace {
struct TreeLevel {
    uint32_t nodes = 0, memb = 0, splits = 0, chunks = 0;
    DevBuf<double> box;                                            // min xyz, max xyz per node
    DevBuf<uint32_t> parent, seg, list;                            // node of the level above; runs of `list` (nodes + 1); member splats
    DevBuf<uint32_t> split, split_rank, chunk_count, chunk_base;   // k_tree_classify and its exclusive scans (nodes + 1)
    DevBuf<uint32_t> size, leaves, dfs, lrank;                     // k_tree_sizes / k_tree_ranks
};
struct TreeEvents {
    cudaEvent_t begin = nullptr, end = nullptr;
    ~TreeEvents() { if (begin) cudaEventDestroy(begin); if (end) cudaEventDestroy(end); }
};
// ensure() that adds what it allocated to `bytes`
template <typename T> int tree_take(DevBuf<T> &b, size_t count, uint64_t &bytes) {
    const size_t before = b.n;
    const int rc = b.ensure(count);
    if (!rc && b.n != before) bytes += (uint64_t)(b.n - before) * sizeof(T);
    return rc;
}
template <typename T> void tree_swap(DevBuf<T> &a, DevBuf<T> &b) { std::swap(a.p, b.p); std::swap(a.n, b.n); }
}

static gs_splat_tree_info tree_info(const gs_engine *e) {
    const auto &t = e->tree;
    gs_splat_tree_info I = t.built;
    I.struct_size = sizeof(I);
    I.leaf_count = t.count; I.node_count = t.have_nodes ? t.node_count : 0; I.index_count = t.splats;
    I.has_depth = t.have_depth; I.has_nodes = t.have_nodes;
    I.sub_tree_count = t.sub_trees;
    return I;
}
// No more than the caller's struct_size (0: a caller built before sub_tree_count, whose struct ends before it), as write_info
static void write_tree_info(gs_splat_tree_info *info, const gs_engine *e) {
    if (!info) return;
    const gs_splat_tree_info I = tree_info(e);
    const size_t n = info->struct_size >= sizeof(I) ? sizeof(I) : offsetof(gs_splat_tree_info, sub_tree_count);
    memcpy(info, &I, n);
    info->struct_size = (uint32_t)n;
}

extern "C" int gs_build_splat_tree(gs_engine *e, const gs_splat_tree_options *opt, gs_splat_tree_info *info) {
    gs_splat_tree_options defaults{};
    defaults.max_depth = 8; defaults.max_centers_per_node = 1000; defaults.min_alpha = 1;   // SplatMesh.js:236
    const gs_splat_tree_options o = read_options(opt, defaults);
    if (o.max_depth > GS_TREE_MAX_DEPTH) return fail(GS_ERR_BAD_ARG, "gs_build_splat_tree: max_depth %u (0..%d)", o.max_depth, GS_TREE_MAX_DEPTH);
    if (!o.max_centers_per_node) return fail(GS_ERR_BAD_ARG, "gs_build_splat_tree: max_centers_per_node 0 (every node would split, the empty ones too)");
    int rc = check_engine(e);
    if (rc) return rc;
    const uint32_t n = e->rs.uploaded;
    if (!n) return fail(GS_ERR_NOT_READY, "gs_build_splat_tree: no scene uploaded");
    // a dynamic mesh of several scenes takes one sub-tree per scene, over that scene's (untransformed) centres (SplatTree.js:377-390)
    const bool forest = e->scenes_multi && e->cfg.dynamic_mode;
    const uint32_t scenes = forest ? (uint32_t)e->scene_start.size() - 1 : 1;
    const uint4 *cc = e->rs.cc.p;
    cudaStream_t st = e->stream;
    uint32_t launches = 0;
    const Launch launch(st, nullptr, &launches);
    uint64_t scratch = 0, max_memb = 0;
    // the centres the reference's tree sees (SplatTree.js:343-353: getSplatCenter, scene transform applied, stored as f32): rebuilt from
    // the ray records where the decode wrote them, else the f32 centres of GS_BUF_CENTERS_COLORS
    DevBuf<uint4> record_centers;
    const bool from_records = e->tree.decoded_ray_records && e->ray.valid && !e->cfg.dynamic_mode;
    TreeEvents ev;
    CU(cudaEventCreate(&ev.begin)); CU(cudaEventCreate(&ev.end));
    PinBuf<unsigned long long> h;      // read-backs of this call
    if ((rc = h.ensure(2 * GS_MAX_SCENES + 2))) return rc;
    CU(cudaEventRecord(ev.begin, st));
    if (from_records) {
        if ((rc = tree_take(record_centers, n, scratch))) return rc;
        launch.plain(nullptr, k_tree_record_centers, (n + 255) / 256, 256, 0, cc, e->ray.rec.p, e->ray.xf.p, e->ray.per_scene ? e->rs.scene_idx.p : nullptr, n,
                     record_centers.p);
        cc = record_centers.p;
    }

    // the splats with alpha >= minAlpha, in splat order
    DevBuf<uint32_t> keep, kscan, sums, bounds, counts, pos, owner, owned, nonempty, leaf_index, leaf_offset, deepest, scene_start, root_seg;
    DevBuf<unsigned char> mask;
    DevBuf<unsigned long long> total;
    if ((rc = tree_take(keep, n, scratch)) || (rc = tree_take(kscan, (size_t)n + 1, scratch)) || (rc = tree_take(bounds, 6 * (size_t)scenes, scratch)) ||
        (rc = tree_take(total, 1, scratch)) || (rc = tree_take(deepest, 1, scratch)))
        return rc;
    launch.plain(nullptr, k_tree_keep, (n + 255) / 256, 256, 0, cc, n, o.min_alpha, keep.p);
    if ((rc = gen_scan(keep.p, n, kscan.p, sums, launch))) return rc;
    uint32_t *h32 = (uint32_t *)h.p;
    // forest: the kept splats before each scene (scenes are contiguous in splat order, so each scene's kept splats are one run of the list)
    std::vector<uint32_t> kept_before(scenes + 1);
    if (forest) {
        if ((rc = tree_take(scene_start, scenes + 1, scratch))) return rc;
        CU(cudaMemcpyAsync(scene_start.p, e->scene_start.data(), 4 * ((size_t)scenes + 1), cudaMemcpyHostToDevice, st));
        for (uint32_t s = 0; s < scenes; ++s) CU(cudaMemcpyAsync(h32 + s, kscan.p + e->scene_start[s], 4, cudaMemcpyDeviceToHost, st));
    }
    CU(cudaMemcpyAsync(h32 + scenes, kscan.p + n, 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    const uint32_t kept = h32[scenes];
    if (forest) memcpy(kept_before.data(), h32, 4 * ((size_t)scenes + 1));
    // forest roots: root r is scene root_scene[r]'s, the scenes with kept splats in scene order
    std::vector<uint32_t> root_scene;
    for (uint32_t s = 0; forest && s < scenes; ++s)
        if (kept_before[s + 1] > kept_before[s]) root_scene.push_back(s);
    const uint32_t roots = forest ? (uint32_t)root_scene.size() : 1;
    std::vector<uint32_t> sub_leaf(scenes + 1, 0), sub_node(scenes + 1, 0);   // forest: each scene's leaf and node ranges

    std::vector<std::unique_ptr<TreeLevel>> levels;
    uint32_t leaf_count = 0, node_count = 0, index_count = 0, all_leaves = 0;
    if (kept) {
        // one level may hold this many memberships; see GS_ERR_CAPACITY in the header
        const uint64_t level_cap = std::min<uint64_t>(std::max<uint64_t>(8ull * kept, GS_TREE_MIN_LEVEL_CAPACITY), 0xffffffffull);
        levels.emplace_back(new TreeLevel());
        TreeLevel &root = *levels[0];
        root.nodes = roots; root.memb = kept; max_memb = kept;
        if ((rc = tree_take(root.box, 6 * (size_t)roots, scratch)) || (rc = tree_take(root.parent, roots, scratch)) ||
            (rc = tree_take(root.seg, (size_t)roots + 1, scratch)) || (rc = tree_take(root.list, kept, scratch)))
            return rc;
        CU(cudaMemsetAsync(bounds.p, 0xff, 12 * (size_t)scenes, st));
        CU(cudaMemsetAsync(bounds.p + 3 * scenes, 0, 12 * (size_t)scenes, st));
        if (!forest) {
            launch.plain(nullptr, k_tree_root_list<false>, (n + kTreeThreads - 1) / kTreeThreads, kTreeThreads, 0, cc, keep.p, kscan.p, n, root.list.p, bounds.p,
                         nullptr, 1u);
            launch.plain(nullptr, k_tree_root, 1, 1, 0, cc, root.list.p, bounds.p, kept, root.box.p, root.seg.p);
        } else {
            // root r's run: [kept_before[s], kept_before[s + 1]) of its scene s; root_seg = seg (roots + 1), then root_scene (roots)
            std::vector<uint32_t> rs(2 * (size_t)roots + 1);
            for (uint32_t r = 0; r < roots; ++r) { rs[r] = kept_before[root_scene[r]]; rs[roots + 1 + r] = root_scene[r]; }
            rs[roots] = kept;
            if ((rc = tree_take(root_seg, rs.size(), scratch))) return rc;
            CU(cudaMemcpyAsync(root_seg.p, rs.data(), 4 * rs.size(), cudaMemcpyHostToDevice, st));
            CU(cudaMemcpyAsync(root.seg.p, rs.data(), 4 * ((size_t)roots + 1), cudaMemcpyHostToDevice, st));
            launch.plain(nullptr, k_tree_root_list<true>, (n + kTreeThreads - 1) / kTreeThreads, kTreeThreads, 0, cc, keep.p, kscan.p, n, root.list.p, bounds.p,
                         scene_start.p, scenes);
            launch.plain(nullptr, k_tree_roots, 1, 32, 0, cc, root.list.p, bounds.p, scenes, root_seg.p, root_seg.p + roots + 1, roots, root.box.p);
            CU(cudaStreamSynchronize(st));   // pageable sources
        }
        for (uint32_t depth = 0;; ++depth) {
            TreeLevel &c = *levels[depth];
            const size_t nn = (size_t)c.nodes + 1;
            if ((rc = tree_take(c.split, nn, scratch)) || (rc = tree_take(c.split_rank, nn, scratch)) || (rc = tree_take(c.chunk_count, nn, scratch)) ||
                (rc = tree_take(c.chunk_base, nn, scratch)))
                return rc;
            launch.plain(nullptr, k_tree_classify, (c.nodes + 255) / 256, 256, 0, c.seg.p, c.nodes, o.max_centers_per_node, depth > o.max_depth, c.split.p,
                         c.chunk_count.p);
            if ((rc = gen_scan(c.split.p, c.nodes, c.split_rank.p, sums, launch)) || (rc = gen_scan(c.chunk_count.p, c.nodes, c.chunk_base.p, sums, launch)))
                return rc;
            CU(cudaMemcpyAsync(h32, c.split_rank.p + c.nodes, 4, cudaMemcpyDeviceToHost, st));
            CU(cudaMemcpyAsync(h32 + 1, c.chunk_base.p + c.nodes, 4, cudaMemcpyDeviceToHost, st));
            CU(cudaStreamSynchronize(st));
            c.splits = h32[0]; c.chunks = h32[1];
            if (!c.splits) break;
            const uint64_t child_nodes = 8ull * c.splits;
            if (child_nodes > (1ull << 28))
                return fail(GS_ERR_CAPACITY, "gs_build_splat_tree: level %u would have %llu nodes (at most 2^28)", depth + 1, (unsigned long long)child_nodes);
            std::unique_ptr<TreeLevel> next(new TreeLevel());
            next->nodes = (uint32_t)child_nodes;
            const size_t slots = 8 * (size_t)c.chunks;
            if ((rc = tree_take(next->box, 6 * (size_t)child_nodes, scratch)) || (rc = tree_take(next->parent, child_nodes, scratch)) ||
                (rc = tree_take(next->seg, child_nodes + 1, scratch)) || (rc = tree_take(mask, c.memb, scratch)) || (rc = tree_take(counts, slots, scratch)) ||
                (rc = tree_take(pos, slots + 1, scratch)))
                return rc;
            launch.plain(nullptr, k_tree_children, (uint32_t)((8ull * c.nodes + 255) / 256), 256, 0, c.box.p, c.split.p, c.split_rank.p, c.nodes, next->box.p,
                         next->parent.p);
            CU(cudaMemsetAsync(total.p, 0, 8, st));
            // count the level before placing it: the capacity check comes before anything is written into the next list
            launch.plain(nullptr, k_tree_count, c.chunks, kTreeThreads, 0, c.list.p, c.seg.p, c.chunk_base.p, c.chunk_count.p, c.split_rank.p, c.nodes, cc, next->box.p,
                         mask.p, counts.p, total.p);
            CU(cudaMemcpyAsync(h.p, total.p, 8, cudaMemcpyDeviceToHost, st));
            CU(cudaStreamSynchronize(st));
            CU(cudaGetLastError());
            const unsigned long long memb = h.p[0];
            if (memb > level_cap)
                return fail(GS_ERR_CAPACITY, "gs_build_splat_tree: level %u would hold %llu memberships of %u splats (at most %llu): centres coincide on split planes",
                            depth + 1, memb, kept, (unsigned long long)level_cap);
            next->memb = (uint32_t)memb;
            max_memb = std::max<uint64_t>(max_memb, memb);
            if ((rc = tree_take(next->list, std::max<size_t>(next->memb, 1), scratch))) return rc;
            if ((rc = gen_scan(counts.p, (uint32_t)slots, pos.p, sums, launch))) return rc;
            launch.plain(nullptr, k_tree_child_seg, (uint32_t)((8ull * c.nodes + 255) / 256), 256, 0, c.split.p, c.split_rank.p, c.chunk_base.p, c.chunk_count.p, c.nodes,
                         pos.p, next->nodes, next->memb, next->seg.p);
            launch.plain(nullptr, k_tree_place, c.chunks, kTreeThreads, 0, c.list.p, c.seg.p, c.chunk_base.p, c.chunk_count.p, c.nodes, mask.p, pos.p, next->list.p);
            levels.push_back(std::move(next));
        }
        // sub-tree sizes bottom-up, depth-first places top-down
        const int L = (int)levels.size();
        for (int l = L - 1; l >= 0; --l) {
            TreeLevel &c = *levels[l];
            TreeLevel *below = l + 1 < L ? levels[l + 1].get() : nullptr;
            if ((rc = tree_take(c.size, c.nodes, scratch)) || (rc = tree_take(c.leaves, c.nodes, scratch)) || (rc = tree_take(c.dfs, c.nodes, scratch)) ||
                (rc = tree_take(c.lrank, c.nodes, scratch)))
                return rc;
            launch.plain(nullptr, k_tree_sizes, (c.nodes + 255) / 256, 256, 0, c.split.p, c.split_rank.p, c.nodes, below ? below->size.p : nullptr,
                         below ? below->leaves.p : nullptr, c.size.p, c.leaves.p);
        }
        // level 0: the roots' depth-first places and leaf ranks, exclusive sums of their sub-trees' sizes (0 for the one root)
        std::vector<uint32_t> root_dfs(roots), root_lrank(roots);
        if (!forest) {
            CU(cudaMemsetAsync(levels[0]->dfs.p, 0, 4, st));
            CU(cudaMemsetAsync(levels[0]->lrank.p, 0, 4, st));
        } else {
            std::vector<uint32_t> sz(2 * (size_t)roots);
            CU(cudaMemcpyAsync(sz.data(), levels[0]->size.p, 4 * (size_t)roots, cudaMemcpyDeviceToHost, st));
            CU(cudaMemcpyAsync(sz.data() + roots, levels[0]->leaves.p, 4 * (size_t)roots, cudaMemcpyDeviceToHost, st));
            CU(cudaStreamSynchronize(st));
            uint32_t d = 0, l = 0;
            for (uint32_t r = 0; r < roots; ++r) { root_dfs[r] = d; root_lrank[r] = l; d += sz[r]; l += sz[roots + r]; }
            CU(cudaMemcpyAsync(levels[0]->dfs.p, root_dfs.data(), 4 * (size_t)roots, cudaMemcpyHostToDevice, st));
            CU(cudaMemcpyAsync(levels[0]->lrank.p, root_lrank.data(), 4 * (size_t)roots, cudaMemcpyHostToDevice, st));
            CU(cudaStreamSynchronize(st));   // pageable sources
            h32[0] = d; h32[1] = l;
        }
        for (int l = 0; l + 1 < L; ++l) {
            TreeLevel &c = *levels[l], &b = *levels[l + 1];
            launch.plain(nullptr, k_tree_ranks, (c.nodes + 255) / 256, 256, 0, c.split.p, c.split_rank.p, c.dfs.p, c.lrank.p, c.nodes, b.size.p, b.leaves.p, b.dfs.p,
                         b.lrank.p);
        }
        if (!forest) {
            CU(cudaMemcpyAsync(h32, levels[0]->size.p, 4, cudaMemcpyDeviceToHost, st));
            CU(cudaMemcpyAsync(h32 + 1, levels[0]->leaves.p, 4, cudaMemcpyDeviceToHost, st));
            CU(cudaStreamSynchronize(st));
        }
        node_count = h32[0]; all_leaves = h32[1];
        // which leaf keeps a splat that several hold, how many each leaf keeps, and which leaves keep any
        const size_t na = (size_t)all_leaves + 1;
        if ((rc = tree_take(owner, n, scratch)) || (rc = tree_take(owned, na, scratch)) || (rc = tree_take(nonempty, na, scratch)) ||
            (rc = tree_take(leaf_index, na, scratch)) || (rc = tree_take(leaf_offset, na, scratch)))
            return rc;
        CU(cudaMemsetAsync(owner.p, 0xff, 4 * (size_t)n, st));
        for (auto &lv : levels) launch.plain(nullptr, k_tree_own, lv->nodes, kTreeLeafThreads, 0, lv->split.p, lv->seg.p, lv->list.p, lv->lrank.p, owner.p);
        for (auto &lv : levels)
            launch.plain(nullptr, k_tree_owned_count, lv->nodes, kTreeLeafThreads, 0, lv->split.p, lv->seg.p, lv->list.p, lv->lrank.p, owner.p, owned.p, nonempty.p);
        if ((rc = gen_scan(nonempty.p, all_leaves, leaf_index.p, sums, launch)) || (rc = gen_scan(owned.p, all_leaves, leaf_offset.p, sums, launch)))
            return rc;
        CU(cudaMemcpyAsync(h32, leaf_index.p + all_leaves, 4, cudaMemcpyDeviceToHost, st));
        CU(cudaMemcpyAsync(h32 + 1, leaf_offset.p + all_leaves, 4, cudaMemcpyDeviceToHost, st));
        // forest: the kept leaves before each root's sub-tree (the kept leaves are numbered in depth-first order across the forest)
        for (uint32_t r = 0; forest && r < roots; ++r) CU(cudaMemcpyAsync(h32 + 2 + r, leaf_index.p + root_lrank[r], 4, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        leaf_count = h32[0]; index_count = h32[1];
        if (forest) {   // an empty scene's ranges are empty, at the next sub-tree's start
            for (uint32_t s = 0, r = 0; s <= scenes; ++s) {
                const bool at_root = r < roots && root_scene[r] == s;
                sub_leaf[s] = r < roots ? h32[2 + r] : leaf_count;
                sub_node[s] = r < roots ? root_dfs[r] : node_count;
                r += at_root ? 1 : 0;
            }
        }
    }

    // the arrays, built beside the engine's current tree and swapped in at the end: a failure up to there leaves that tree as it was
    gs_engine::Tree out;
    const size_t m = std::max<uint32_t>(leaf_count, 1), k = std::max<uint32_t>(node_count, 1);
    if ((rc = out.center.ensure(3 * m)) || (rc = out.nmin.ensure(3 * m)) || (rc = out.nmax.ensure(3 * m)) || (rc = out.offsets.ensure(m + 1)) ||
        (rc = out.indexes.ensure(std::max<uint32_t>(index_count, 1))) || (rc = out.depth.ensure(m)) || (rc = out.start.ensure(m)) || (rc = out.key.ensure(m)) ||
        (rc = out.total.ensure(1)) || (rc = out.all_min.ensure(3 * k)) || (rc = out.all_max.ensure(3 * k)) || (rc = out.parent.ensure(k)) ||
        (rc = out.leaf_node.ensure(m)))
        return rc;
    CU(cudaMemsetAsync(out.offsets.p, 0, 4, st));
    CU(cudaMemsetAsync(deepest.p, 0, 4, st));
    if (kept) {
        const TreeOut O{out.center.p, out.nmin.p, out.nmax.p, out.offsets.p, out.indexes.p, out.depth.p, out.all_min.p, out.all_max.p, out.parent.p, out.leaf_node.p,
                        deepest.p};
        for (size_t l = 0; l < levels.size(); ++l) {
            TreeLevel &c = *levels[l];
            launch.plain(nullptr, k_tree_write_leaves, c.nodes, kTreeLeafThreads, 0, c.split.p, c.seg.p, c.list.p, c.lrank.p, c.dfs.p, c.box.p, (int)l, owner.p, owned.p,
                         leaf_index.p, leaf_offset.p, O);
            launch.plain(nullptr, k_tree_write_nodes, (c.nodes + 255) / 256, 256, 0, c.box.p, c.parent.p, c.dfs.p, l ? levels[l - 1]->dfs.p : nullptr, c.nodes, O);
        }
        CU(cudaMemcpyAsync(out.offsets.p + leaf_count, leaf_offset.p + all_leaves, 4, cudaMemcpyDeviceToDevice, st));
    }
    if (forest) {
        if ((rc = out.sub_leaf.ensure(scenes + 1)) || (rc = out.sub_node.ensure(scenes + 1))) return rc;
        CU(cudaMemcpyAsync(out.sub_leaf.p, sub_leaf.data(), 4 * ((size_t)scenes + 1), cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync(out.sub_node.p, sub_node.data(), 4 * ((size_t)scenes + 1), cudaMemcpyHostToDevice, st));
    }
    CU(cudaEventRecord(ev.end, st));
    CU(cudaMemcpyAsync(h.p, deepest.p, 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    float ms = 0.f;
    CU(cudaEventElapsedTime(&ms, ev.begin, ev.end));

    auto &t = e->tree;
    tree_swap(t.center, out.center); tree_swap(t.nmin, out.nmin); tree_swap(t.nmax, out.nmax); tree_swap(t.offsets, out.offsets);
    tree_swap(t.indexes, out.indexes); tree_swap(t.depth, out.depth); tree_swap(t.start, out.start); tree_swap(t.key, out.key); tree_swap(t.total, out.total);
    tree_swap(t.all_min, out.all_min); tree_swap(t.all_max, out.all_max); tree_swap(t.parent, out.parent); tree_swap(t.leaf_node, out.leaf_node);
    tree_swap(t.sub_leaf, out.sub_leaf); tree_swap(t.sub_node, out.sub_node);
    t.count = leaf_count; t.splats = index_count; t.node_count = node_count;
    t.sub_trees = scenes;
    t.h_sub_leaf = forest ? sub_leaf : std::vector<uint32_t>();
    t.h_sub_node = forest ? sub_node : std::vector<uint32_t>();
    t.have_nodes = true; t.have_depth = true;
    t.built = gs_splat_tree_info{};
    t.built.max_leaf_depth = *(const uint32_t *)h.p;
    t.built.level_count = (uint32_t)levels.size();
    t.built.max_level_memberships = max_memb;
    t.built.scratch_bytes = scratch + sums.n * sizeof(uint32_t);
    t.built.build_ms = ms;
    t.built.centers_from_ray_records = from_records;
    e->tm.kernel_launches = launches;
    write_tree_info(info, e);
    return GS_OK;
}

extern "C" int gs_read_splat_tree(gs_engine *e, const gs_splat_tree_arrays *out, gs_splat_tree_info *info) {
    int rc = check_engine(e);
    if (rc) return rc;
    const auto &t = e->tree;
    write_tree_info(info, e);
    if (!out) return GS_OK;
    const gs_splat_tree_arrays a = read_options(out, gs_splat_tree_arrays{});
    if (a.depth && !t.have_depth) return fail(GS_ERR_NOT_READY, "gs_read_splat_tree: the tree was uploaded without leaf depths (only gs_build_splat_tree records them)");
    if ((a.all_min || a.all_max || a.parent || a.leaf_node) && !t.have_nodes)
        return fail(GS_ERR_NOT_READY, "gs_read_splat_tree: the engine holds leaves without nodes (gs_upload_splat_tree_nodes was not called for them)");
    cudaStream_t st = e->stream;
    const size_t m = t.count, k = t.node_count;
    struct Copy { void *dst; const void *src; size_t bytes; };
    const Copy copies[] = {{a.node_center, t.center.p, 24 * m}, {a.node_min, t.nmin.p, 24 * m}, {a.node_max, t.nmax.p, 24 * m},
                           {a.node_offsets, t.offsets.p, t.offsets.p ? 4 * (m + 1) : 0}, {a.indexes, t.indexes.p, 4 * (size_t)t.splats},
                           {a.depth, t.depth.p, 4 * m}, {a.all_min, t.all_min.p, 24 * k}, {a.all_max, t.all_max.p, 24 * k}, {a.parent, t.parent.p, 4 * k},
                           {a.leaf_node, t.leaf_node.p, 4 * m}};
    for (const Copy &c : copies)
        if (c.dst && c.bytes) CU(cudaMemcpyAsync(c.dst, c.src, c.bytes, cudaMemcpyDeviceToHost, st));
    if (a.node_offsets && !t.offsets.p) a.node_offsets[0] = 0;   // no tree yet: no leaves
    // u32[sub_tree_count + 1] each; one sub-tree: all leaves, all nodes
    const std::vector<uint32_t> one_leaf{0u, (uint32_t)m}, one_node{0u, t.have_nodes ? (uint32_t)k : 0u};
    if (a.sub_tree_leaf_offsets) memcpy(a.sub_tree_leaf_offsets, (t.sub_trees > 1 ? t.h_sub_leaf : one_leaf).data(), 4 * ((size_t)t.sub_trees + 1));
    if (a.sub_tree_node_offsets) memcpy(a.sub_tree_node_offsets, (t.sub_trees > 1 ? t.h_sub_node : one_node).data(), 4 * ((size_t)t.sub_trees + 1));
    CU(cudaStreamSynchronize(st));
    return GS_OK;
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
        case GS_BUF_SCENE_INDEXES: p = (const unsigned char *)e->rs.scene_idx.p; cap = e->rs.scene_idx.n * 4; break;
        default: { void *q = nullptr; if ((rc = gs_buffer_dev(e, id, &q, &cap))) return rc; p = (const unsigned char *)q; }
    }
    if (!p || offset + bytes > cap) return fail(GS_ERR_CAPACITY, "gs_read_buffer: [%zu,%zu) outside the %zu-byte buffer", offset, offset + bytes, cap);
    CU(cudaMemcpyAsync(out, p + offset, bytes, cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    return GS_OK;
}

// After a stereo frame: the left eye's records (the right eye's are view[1]'s)
extern "C" int gs_read_projected(gs_engine *e, gs_projected_splat *out, uint32_t count) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!out) return fail(GS_ERR_BAD_ARG, "gs_read_projected: null");
    rc = raster_read_projected(e->rs, out, count, Launch(e->stream));
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
        case GS_BUF_SPLAT_RECORDS: *ptr = e->rs.view[0].records.p; b = e->rs.view[0].records.n * sizeof(SplatRecord); break;
        case GS_BUF_INDEXES_TO_SORT: *ptr = e->indexes.p; b = e->indexes.n * 4; break;
        case GS_BUF_DEPTH:
            *ptr = e->rs.last_depth_parity >= 0 ? e->rs.depth[e->rs.last_depth_parity].p : nullptr;
            b = e->rs.last_depth_parity >= 0 ? e->rs.last_depth_bytes : 0;
            break;
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
        if ((rc = copy_out(e, nullptr, nullptr, 0))) return rc;
        return finish_call(e, kSortPart | kRenderPart);
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
    Launch(e->stream).plain(nullptr, k_flush_l2, e->sm_count * 8, 512, 0, e->flush.p, words, ++tick);
    CU(cudaGetLastError());
    return GS_OK;
}
// ---- fused tile gather: rank 0's frame buffer + handshake block shared with the other ranks through CUDA IPC -------------------------
// A frame graph captures the frame buffer and the handshake pointers: attaching drops both graphs.
// A peer group on one device keeps bounded spin-wait kernels in flight while the host enqueues the other engines' frames, so every
// kernel a frame with world_size > 1 can launch is loaded up front (preload_kernel): the depth sort, the projection, both binnings,
// the subset compaction, the blend and the handshake.
template <typename KeyT> static void peer_preload_sort() { preload_kernel(k_bucket<KeyT>); radix_preload<KeyT, uint32_t>(); }
static void peer_preload() {
    preload_kernel(k_sort_init); preload_kernel(k_copy_head);
    for_each_depth([](int, bool, bool views, auto kernel) { if (!views) preload_kernel(kernel); });
    peer_preload_sort<uint16_t>(); peer_preload_sort<uint32_t>();    // the group's engines may sort keys of either width
    // a peer group renders neither stereo, multi-view nor composited frames
    preload_kernel(k_raster_init);
    for_each_project([](bool, int, bool views, auto kernel) { if (!views) preload_kernel(kernel); });
    preload_kernel(k_subset_count); preload_kernel(k_subset_emit);
    preload_kernel(k_bin_count); preload_kernel(k_bin_scan); preload_kernel(k_bin_place);
    preload_kernel(k_tile_count); preload_kernel(k_tile_emit); radix_preload<uint16_t, unsigned long long>();
    for_each_blend([](int, int, bool composite, bool views, bool depth, auto kernel) { if (!composite && !views && !depth) preload_kernel(kernel); });
    preload_kernel(k_peer_release); preload_kernel(k_peer_wait_release); preload_kernel(k_peer_signal); preload_kernel(k_peer_wait_arrived);
    (void)cudaGetLastError();
}
// What a frame could otherwise allocate once the group renders (cudaMalloc / cudaFree may wait for the device): the subset sort's input.
static int peer_reserve(gs_engine *e) {
    int rc;
    if ((rc = e->sub_idx.ensure(e->cfg.max_splat_count)) || (rc = e->sub_dist.ensure(e->cfg.max_splat_count))) return rc;
    return GS_OK;
}
// Rank 0's side of the gather (gs_peer_export, gs_peer_attach_local): the handshake block, the double frame allocation, the frame count.
static int peer_root_setup(gs_engine *e) {
    int rc;
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
    CU(cudaMemset(&e->rs.view[0].rctl.p->frame_seq, 0, 4));   // ranks count frames in lockstep from here on
    e->rs.peer_sync = e->rs.peer_sync_local.p;
    e->rs.peer_root = true;
    e->graph.drop();
    return GS_OK;
}
extern "C" int gs_peer_export(gs_engine *e, void *frame_handle, void *sync_handle) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!frame_handle || !sync_handle) return fail(GS_ERR_BAD_ARG, "gs_peer_export: null");
    if (e->cfg.world_size < 2 || e->cfg.rank != 0) return fail(GS_ERR_BAD_ARG, "gs_peer_export: only rank 0 of a multi-GPU group exports");
    if (!e->rs.frame.p) return fail(GS_ERR_NOT_READY, "engine created without a framebuffer");
    if ((rc = peer_root_setup(e))) return rc;
    static_assert(sizeof(cudaIpcMemHandle_t) == GS_IPC_HANDLE_BYTES, "IPC handle size");
    cudaIpcMemHandle_t h;
    CU(cudaIpcGetMemHandle(&h, e->rs.frame.p));
    memcpy(frame_handle, &h, sizeof(h));
    CU(cudaIpcGetMemHandle(&h, e->rs.peer_sync_local.p));
    memcpy(sync_handle, &h, sizeof(h));
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
    CU(cudaMemset(&e->rs.view[0].rctl.p->frame_seq, 0, 4));
    e->rs.peer_frame = pf;
    e->rs.peer_sync = (PeerSync *)ps;
    e->rs.peer_attached = true;
    e->graph.drop();
    return GS_OK;
}
// Same process, same device: rank 0's own frame allocation and handshake block instead of IPC mappings.  A peer finds the second half
// of rank 0's allocation at its own frame size, so both engines must have the same one (the IPC path cannot check this).
// The device feeds streams through CUDA_DEVICE_MAX_CONNECTIONS hardware work queues (8 unless the process sets it, at most 32), and
// streams beyond that share queues: a peer's spinning k_peer_wait_release can then sit in front of rank 0's k_peer_release in one
// queue until the spin gives up.  A group holds two streams per engine (stream, graph.side) and rank 0's two pipelining streams, so it
// must have at most that many.  Beyond that, groups of more than kPeerLocalMaxWorld engines are refused: a group of 8 with 32 queues
// renders its first frames but times out on the first frame after a frame graph is replaced, for a reason not yet found.
constexpr uint32_t kPeerLocalMaxWorld = 3;
static int peer_local_queues() {
    const char *v = getenv("CUDA_DEVICE_MAX_CONNECTIONS");
    const int n = v ? atoi(v) : 8;
    return n < 1 ? 8 : std::min(n, 32);
}
extern "C" int gs_peer_attach_local(gs_engine *e, gs_engine *root) {
    int rc = check_engine(e);
    if (rc) return rc;
    if (!root) return fail(GS_ERR_BAD_ARG, "gs_peer_attach_local: null root");
    const gs_config &c = e->cfg, &r = root->cfg;
    if (c.world_size < 2 || c.rank == 0) return fail(GS_ERR_BAD_ARG, "gs_peer_attach_local: only ranks > 0 of a multi-GPU group attach");
    if (r.rank != 0 || r.world_size != c.world_size || r.device != c.device)
        return fail(GS_ERR_BAD_ARG, "gs_peer_attach_local: root must be rank 0 of %u on device %d (it is rank %u of %u on device %d)", c.world_size, c.device,
                    r.rank, r.world_size, r.device);
    if (c.world_size > kPeerLocalMaxWorld || 2 * c.world_size + 2 > (uint32_t)peer_local_queues())
        return fail(GS_ERR_BAD_ARG, "gs_peer_attach_local: a group of %u engines on one device: at most %u, and at most (queues - 2) / 2 for the "
                    "device's %d hardware work queues (CUDA_DEVICE_MAX_CONNECTIONS)", c.world_size, kPeerLocalMaxWorld, peer_local_queues());
    if (!e->rs.frame.p || !root->rs.frame.p) return fail(GS_ERR_BAD_ARG, "gs_peer_attach_local: engines created without a framebuffer");
    const size_t root_half = root->rs.frame_half2 ? root->rs.frame_half_bytes : root->rs.frame.n;
    if (e->rs.frame.n != root_half)
        return fail(GS_ERR_BAD_ARG, "gs_peer_attach_local: frame buffers of %zu and %zu bytes (max_width / max_height must match)", e->rs.frame.n, root_half);
    if (e->pipe_inflight() || e->pending_async || root->pipe_inflight() || root->pending_async)
        return fail(GS_ERR_BAD_ARG, "gs_peer_attach_local: frames in flight (gs_frame_end / gs_synchronize first)");
    if (e->rs.peer_attached) return fail(GS_ERR_BAD_ARG, "gs_peer_attach_local: engine already attached to a root");
    if ((rc = peer_reserve(e))) return rc;
    if (!root->rs.peer_root && ((rc = peer_root_setup(root)) || (rc = peer_reserve(root)))) return rc;
    peer_preload();
    CU(cudaMemset(&e->rs.view[0].rctl.p->frame_seq, 0, 4));
    e->rs.peer_frame = root->rs.frame.p;
    e->rs.peer_sync = root->rs.peer_sync_local.p;
    e->rs.peer_attached = e->rs.peer_local = root->rs.peer_local = true;
    e->graph.drop();
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
