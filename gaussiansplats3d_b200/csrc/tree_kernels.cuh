// tree_kernels.cuh -- the SplatTree build of the reference's tree worker (src/splattree/SplatTree.js:132-278, createSplatTree /
// buildSubTree / processSplatTreeNode) and the flattening of convertWorkerSubTree (:55-79) on the GPU, level by level.
//
// The reference recurses depth first.  Here one level of the octree is built at a time from a list of (node, splat) memberships that is
// kept sorted by node and, inside a node, by splat index:
//   k_tree_record_centers   (scenes decoded on an engine with ray records) the centres as getSplatCenter gives them
//   k_tree_keep / k_tree_root_list / k_tree_root   the splats with alpha >= minAlpha in splat order, and the scene box       :222-248
//                     (a dynamic mesh of several scenes: one root per scene with kept splats, k_tree_roots; the roots are level 0 of
//                     one forest, numbered depth first sub-tree after sub-tree, as the reference's subTrees loop visits them :377-390)
//   k_tree_classify   a node is a leaf when its count < maxCentersPerNode or its depth > maxDepth                            :141
//   k_tree_children   the eight child boxes of every node that splits, in the reference's child order                       :152-182
//   k_tree_count      every membership of a splitting node against its eight child boxes (faces included: a centre on a split
//                     plane is a member of several children, and is COUNTED in each)                                      :184-197
//   k_tree_child_seg / k_tree_place   the next level's list: a stable eight-way split of every node's run
// and once no node splits any more:
//   k_tree_sizes / k_tree_ranks   sub-tree sizes bottom-up, then every node's depth-first index and every leaf's depth-first rank
//   k_tree_own        a splat that is a member of several leaves belongs to the one the depth-first walk reaches first (addedIndexes)
//   k_tree_owned_count / k_tree_write_leaves / k_tree_write_nodes   leaves left empty are dropped; the arrays of gs_upload_splat_tree
//                     and gs_upload_splat_tree_nodes in the reference's order
// Box arithmetic is f64 in the reference's operation order, unfused.  Nothing here depends on the order in which threads run: counts
// are integer sums, ownership is an integer minimum, placement is by exclusive scans.
#pragma once
#include "common.cuh"

namespace gs {

constexpr int kTreeThreads = 256;
constexpr int kTreeChunk = 2048;          // memberships one CTA of k_tree_count / k_tree_place handles
constexpr int kTreeLeafThreads = 128;

// f32 bit patterns in an order that matches the numbers' (for integer atomicMin / atomicMax)
__device__ __forceinline__ uint32_t f32_ordered(uint32_t bits) { return bits ^ ((bits >> 31) ? 0xffffffffu : 0x80000000u); }
__device__ __forceinline__ float f32_from_ordered(uint32_t u) { return __uint_as_float(u ^ ((u >> 31) ? 0x80000000u : 0xffffffffu)); }

// The centre SplatMesh.getSplatCenter hands the tree (SplatBuffer.js:221-245): the ray record's unrounded centre under the static mesh's
// scene transform (Vector3.applyMatrix4, sums left to right), stored as f32; the colour word (alpha) as GS_BUF_CENTERS_COLORS has it.
// xf: f64[16 * GS_MAX_SCENES], one transform per scene; scene_idx: the splat's scene, or nullptr for scene 0.
__global__ void k_tree_record_centers(const uint4 *__restrict__ cc, const gs_ray_record *__restrict__ rec, const double *__restrict__ xf,
                                      const uint32_t *__restrict__ scene_idx, uint32_t n, uint4 *__restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double *e = xf + 16 * (scene_idx ? scene_idx[i] & (GS_MAX_SCENES - 1) : 0u);
    const double x = rec[i].center[0], y = rec[i].center[1], z = rec[i].center[2];
    const double w = __ddiv_rn(1.0, __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e[3], x), __dmul_rn(e[7], y)), __dmul_rn(e[11], z)), e[15]));
    const float tx = (float)__dmul_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e[0], x), __dmul_rn(e[4], y)), __dmul_rn(e[8], z)), e[12]), w);
    const float ty = (float)__dmul_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e[1], x), __dmul_rn(e[5], y)), __dmul_rn(e[9], z)), e[13]), w);
    const float tz = (float)__dmul_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e[2], x), __dmul_rn(e[6], y)), __dmul_rn(e[10], z)), e[14]), w);
    out[i] = make_uint4(cc[i].x, __float_as_uint(tx), __float_as_uint(ty), __float_as_uint(tz));
}

__global__ void k_tree_keep(const uint4 *__restrict__ cc, uint32_t n, uint32_t min_alpha, uint32_t *__restrict__ keep) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) keep[i] = (cc[i].x >> 24) >= min_alpha ? 1u : 0u;
}

// list[scan[i]] = i for the kept splats; bounds[0..2] / [3..5]: minimum / maximum of their coordinates that are not NaN (ordered bits;
// seeded 0xffffffff / 0 by the caller).  kForest: one box per scene, scene s = the range of splat i in scene_start[0..scenes];
// bounds[3 s + a] / bounds[3 scenes + 3 s + a].  A warp that straddles two scenes updates the bounds lane by lane.
template <bool kForest>
__global__ void __launch_bounds__(kTreeThreads)
k_tree_root_list(const uint4 *__restrict__ cc, const uint32_t *__restrict__ keep, const uint32_t *__restrict__ scan, uint32_t n, uint32_t *__restrict__ list,
                 uint32_t *__restrict__ bounds, const uint32_t *__restrict__ scene_start, uint32_t scenes) {
    const uint32_t i = blockIdx.x * kTreeThreads + threadIdx.x;
    uint32_t lo[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, hi[3] = {0u, 0u, 0u};
    if (i < n && keep[i]) {
        list[scan[i]] = i;
        const uint4 c = cc[i];
        const uint32_t b[3] = {c.y, c.z, c.w};
#pragma unroll
        for (int a = 0; a < 3; ++a)
            if ((b[a] & 0x7fffffffu) <= 0x7f800000u) lo[a] = hi[a] = f32_ordered(b[a]);
    }
    uint32_t *bmin = bounds, *bmax = bounds + 3;
    if (kForest) {
        const uint32_t s = range_of(scene_start, scenes, min(i, n - 1));
        bmin = bounds + 3 * s; bmax = bounds + 3 * (scenes + s);
        if (!__all_sync(0xffffffffu, s == __shfl_sync(0xffffffffu, s, 0))) {
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                if (lo[a] != 0xffffffffu) atomicMin(&bmin[a], lo[a]);
                if (hi[a] != 0u) atomicMax(&bmax[a], hi[a]);
            }
            return;
        }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const uint32_t wlo = __reduce_min_sync(0xffffffffu, lo[a]), whi = __reduce_max_sync(0xffffffffu, hi[a]);
        if ((threadIdx.x & 31) == 0) {
            if (wlo != 0xffffffffu) atomicMin(&bmin[a], wlo);
            if (whi != 0u) atomicMax(&bmax[a], whi);
        }
    }
}

// The scene box (SplatTree.js:233-238): min and max start at the first kept centre and move on strict < / >, so a NaN coordinate is
// skipped unless the first kept splat has it, and then that axis stays NaN.  box: min xyz, max xyz of node 0; seg: its run [0, kept).
__global__ void k_tree_root(const uint4 *__restrict__ cc, const uint32_t *__restrict__ list, const uint32_t *__restrict__ bounds, uint32_t kept,
                            double *__restrict__ box, uint32_t *__restrict__ seg) {
    const uint4 c = cc[list[0]];
    const float first[3] = {__uint_as_float(c.y), __uint_as_float(c.z), __uint_as_float(c.w)};
    for (int a = 0; a < 3; ++a) {
        const bool nan = first[a] != first[a];
        box[a] = nan ? (double)first[a] : (double)f32_from_ordered(bounds[a]);
        box[3 + a] = nan ? (double)first[a] : (double)f32_from_ordered(bounds[3 + a]);
    }
    seg[0] = 0; seg[1] = kept;
}

// The roots of a forest (SplatTree.processSplatMesh of a dynamic mesh, SplatTree.js:377-390: one sub-tree per scene): root r is scene
// root_scene[r]'s, over its kept splats list[seg[r] .. seg[r + 1]) (seg uploaded by the caller), with k_tree_root's box from that
// scene's bounds (k_tree_root_list<true>).  Scenes without a kept splat have no root.
__global__ void k_tree_roots(const uint4 *__restrict__ cc, const uint32_t *__restrict__ list, const uint32_t *__restrict__ bounds, uint32_t scenes,
                             const uint32_t *__restrict__ seg, const uint32_t *__restrict__ root_scene, uint32_t roots, double *__restrict__ box) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= roots) return;
    const uint32_t s = root_scene[r];
    const uint4 c = cc[list[seg[r]]];
    const float first[3] = {__uint_as_float(c.y), __uint_as_float(c.z), __uint_as_float(c.w)};
    for (int a = 0; a < 3; ++a) {
        const bool nan = first[a] != first[a];
        box[6 * (size_t)r + a] = nan ? (double)first[a] : (double)f32_from_ordered(bounds[3 * s + a]);
        box[6 * (size_t)r + 3 + a] = nan ? (double)first[a] : (double)f32_from_ordered(bounds[3 * (scenes + s) + a]);
    }
}

// split[i] = 1 when node i gets children; chunks[i] = the CTAs of k_tree_count / k_tree_place its run takes
__global__ void k_tree_classify(const uint32_t *__restrict__ seg, uint32_t nodes, uint32_t max_centers, int past_max_depth, uint32_t *__restrict__ split,
                                uint32_t *__restrict__ chunks) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nodes) return;
    const uint32_t count = seg[i + 1] - seg[i];
    const bool leaf = count < max_centers || past_max_depth;
    split[i] = leaf ? 0u : 1u;
    chunks[i] = leaf ? 0u : (count + kTreeChunk - 1) / kTreeChunk;
}

// Child j of a splitting node (SplatTree.js:152-182): dims = max - min, half = dims * 0.5, c = min + half, bounds from c, c - half and
// c + half.  Which half along x, y, z each child takes, in the reference's child order:
__device__ __constant__ unsigned char kChildHalves[8] = {0b010, 0b011, 0b111, 0b110, 0b000, 0b001, 0b101, 0b100};   // bit 0 = x upper, 1 = y, 2 = z
__global__ void k_tree_children(const double *__restrict__ box, const uint32_t *__restrict__ split, const uint32_t *__restrict__ split_rank, uint32_t nodes,
                                double *__restrict__ child_box, uint32_t *__restrict__ child_parent) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t p = t >> 3, j = t & 7;
    if (p >= nodes || !split[p]) return;
    const uint32_t c = 8 * split_rank[p] + j;
    const unsigned char h = kChildHalves[j];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const double mn = box[6 * (size_t)p + a], mx = box[6 * (size_t)p + 3 + a];
        const double half = __dmul_rn(__dadd_rn(mx, -mn), 0.5);
        const double ctr = __dadd_rn(mn, half);
        const bool upper = (h >> a) & 1;
        child_box[6 * (size_t)c + a] = upper ? ctr : __dadd_rn(ctr, -half);
        child_box[6 * (size_t)c + 3 + a] = upper ? __dadd_rn(ctr, half) : ctr;
    }
    child_parent[c] = p;
}

// The node whose run CTA `b` works on: the last p with chunk_base[p] <= b (nodes without chunks share their successor's base)
__device__ __forceinline__ uint32_t tree_chunk_node(const uint32_t *__restrict__ chunk_base, uint32_t nodes, uint32_t b) {
    uint32_t lo = 0, hi = nodes;       // first index in [0, nodes] with chunk_base > b
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (chunk_base[mid] > b) hi = mid; else lo = mid + 1;
    }
    return lo - 1;
}

// One CTA per chunk of a splitting node's run: mask[i] = the children whose box contains membership i's centre (WorkerBox3.containsPoint,
// >= and <=, on the f32 centre widened to f64); counts[8 * chunk_base[p] + j * chunks[p] + k] = members of child j in chunk k of node p, so
// that ONE exclusive scan of `counts` gives every (child, chunk) its place in the next level's list; *total += all of them.
__global__ void __launch_bounds__(kTreeThreads)
k_tree_count(const uint32_t *__restrict__ list, const uint32_t *__restrict__ seg, const uint32_t *__restrict__ chunk_base, const uint32_t *__restrict__ chunks,
             const uint32_t *__restrict__ split_rank, uint32_t nodes, const uint4 *__restrict__ cc, const double *__restrict__ child_box,
             unsigned char *__restrict__ mask, uint32_t *__restrict__ counts, unsigned long long *__restrict__ total) {
    __shared__ double s_box[48];
    __shared__ uint32_t s_cnt[8];
    const uint32_t p = tree_chunk_node(chunk_base, nodes, blockIdx.x);
    const uint32_t k = blockIdx.x - chunk_base[p];
    if (threadIdx.x < 48) s_box[threadIdx.x] = child_box[48 * (size_t)split_rank[p] + threadIdx.x];
    if (threadIdx.x < 8) s_cnt[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t lo = seg[p] + k * kTreeChunk, hi = min(seg[p + 1], lo + kTreeChunk);
    uint32_t mine[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (uint32_t i = lo + threadIdx.x; i < hi; i += kTreeThreads) {
        const uint4 c = cc[list[i]];
        const double x = (double)__uint_as_float(c.y), y = (double)__uint_as_float(c.z), z = (double)__uint_as_float(c.w);
        uint32_t m = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const double *b = s_box + 6 * j;
            const bool in = x >= b[0] && x <= b[3] && y >= b[1] && y <= b[4] && z >= b[2] && z <= b[5];
            m |= in ? (1u << j) : 0u;
            mine[j] += in ? 1u : 0u;
        }
        mask[i] = (unsigned char)m;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const uint32_t w = __reduce_add_sync(0xffffffffu, mine[j]);
        if ((threadIdx.x & 31) == 0 && w) atomicAdd(&s_cnt[j], w);
    }
    __syncthreads();
    if (threadIdx.x < 8) counts[8 * (size_t)chunk_base[p] + (size_t)threadIdx.x * chunks[p] + k] = s_cnt[threadIdx.x];
    if (threadIdx.x == 0) {
        unsigned long long sum = 0;
        for (int j = 0; j < 8; ++j) sum += s_cnt[j];
        atomicAdd(total, sum);
    }
}

// seg of the next level: child j of node p starts where its first chunk does
__global__ void k_tree_child_seg(const uint32_t *__restrict__ split, const uint32_t *__restrict__ split_rank, const uint32_t *__restrict__ chunk_base,
                                 const uint32_t *__restrict__ chunks, uint32_t nodes, const uint32_t *__restrict__ pos, uint32_t child_nodes, uint32_t child_total,
                                 uint32_t *__restrict__ child_seg) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t == 0) child_seg[child_nodes] = child_total;
    const uint32_t p = t >> 3, j = t & 7;
    if (p >= nodes || !split[p]) return;
    child_seg[8 * split_rank[p] + j] = pos[8 * (size_t)chunk_base[p] + (size_t)j * chunks[p]];
}

// The stable eight-way split: membership i goes, for every child in mask[i], behind the members of that child that precede it in its
// node's run.  pos = exclusive scan of k_tree_count's counts.
__global__ void __launch_bounds__(kTreeThreads)
k_tree_place(const uint32_t *__restrict__ list, const uint32_t *__restrict__ seg, const uint32_t *__restrict__ chunk_base, const uint32_t *__restrict__ chunks,
             uint32_t nodes, const unsigned char *__restrict__ mask, const uint32_t *__restrict__ pos, uint32_t *__restrict__ child_list) {
    constexpr int NW = kTreeThreads / 32;
    __shared__ uint32_t s_base[8];
    __shared__ uint32_t s_warp[NW][8];
    const uint32_t p = tree_chunk_node(chunk_base, nodes, blockIdx.x);
    const uint32_t k = blockIdx.x - chunk_base[p];
    if (threadIdx.x < 8) s_base[threadIdx.x] = pos[8 * (size_t)chunk_base[p] + (size_t)threadIdx.x * chunks[p] + k];
    const uint32_t lo = seg[p] + k * kTreeChunk, hi = min(seg[p + 1], lo + kTreeChunk);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint32_t base = lo; base < hi; base += kTreeThreads) {      // uniform trip count: every thread reaches the barriers
        const uint32_t i = base + threadIdx.x;
        const uint32_t m = i < hi ? mask[i] : 0u;
        const uint32_t splat = i < hi ? list[i] : 0u;
        uint32_t before[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const uint32_t b = __ballot_sync(0xffffffffu, (m >> j) & 1);
            before[j] = __popc(b & lanemask_lt());
            if (lane == 0) s_warp[warp][j] = __popc(b);
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (!((m >> j) & 1)) continue;
            uint32_t at = s_base[j] + before[j];
            for (int w = 0; w < warp; ++w) at += s_warp[w][j];
            child_list[at] = splat;
        }
        __syncthreads();
        if (threadIdx.x < 8) {
            uint32_t sum = 0;
            for (int w = 0; w < NW; ++w) sum += s_warp[w][threadIdx.x];
            s_base[threadIdx.x] += sum;
        }
        __syncthreads();
    }
}

// Bottom-up: nodes and leaves in the sub-tree of node i (children of a splitting node: 8 * split_rank[i] + j of the level below)
__global__ void k_tree_sizes(const uint32_t *__restrict__ split, const uint32_t *__restrict__ split_rank, uint32_t nodes, const uint32_t *__restrict__ child_size,
                             const uint32_t *__restrict__ child_leaves, uint32_t *__restrict__ size, uint32_t *__restrict__ leaves) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nodes) return;
    uint32_t s = 1, l = 1;
    if (split[i]) {
        l = 0;
        for (uint32_t c = 8 * split_rank[i]; c < 8 * split_rank[i] + 8; ++c) { s += child_size[c]; l += child_leaves[c]; }
    }
    size[i] = s; leaves[i] = l;
}

// Top-down: dfs[i] = node i's place in the depth-first, root-first order; lrank[i] = leaves that order reaches before node i's
__global__ void k_tree_ranks(const uint32_t *__restrict__ split, const uint32_t *__restrict__ split_rank, const uint32_t *__restrict__ dfs,
                             const uint32_t *__restrict__ lrank, uint32_t nodes, const uint32_t *__restrict__ child_size, const uint32_t *__restrict__ child_leaves,
                             uint32_t *__restrict__ child_dfs, uint32_t *__restrict__ child_lrank) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nodes || !split[i]) return;
    uint32_t d = dfs[i] + 1, l = lrank[i];
    for (uint32_t c = 8 * split_rank[i]; c < 8 * split_rank[i] + 8; ++c) {
        child_dfs[c] = d; child_lrank[c] = l;
        d += child_size[c]; l += child_leaves[c];
    }
}

// One CTA per node of a level; leaves only.  owner[splat] = the lowest depth-first rank among the leaves the splat is a member of.
__global__ void __launch_bounds__(kTreeLeafThreads)
k_tree_own(const uint32_t *__restrict__ split, const uint32_t *__restrict__ seg, const uint32_t *__restrict__ list, const uint32_t *__restrict__ lrank,
           uint32_t *__restrict__ owner) {
    const uint32_t i = blockIdx.x;
    if (split[i]) return;
    const uint32_t r = lrank[i];
    for (uint32_t k = seg[i] + threadIdx.x; k < seg[i + 1]; k += kTreeLeafThreads) atomicMin(&owner[list[k]], r);
}

// owned[lrank] = the members leaf `lrank` keeps; nonempty[lrank] = whether it keeps any (convertWorkerSubTree drops the others)
__global__ void __launch_bounds__(kTreeLeafThreads)
k_tree_owned_count(const uint32_t *__restrict__ split, const uint32_t *__restrict__ seg, const uint32_t *__restrict__ list, const uint32_t *__restrict__ lrank,
                   const uint32_t *__restrict__ owner, uint32_t *__restrict__ owned, uint32_t *__restrict__ nonempty) {
    __shared__ uint32_t s_sum;
    const uint32_t i = blockIdx.x;
    if (split[i]) return;
    if (threadIdx.x == 0) s_sum = 0;
    __syncthreads();
    const uint32_t r = lrank[i];
    uint32_t mine = 0;
    for (uint32_t k = seg[i] + threadIdx.x; k < seg[i + 1]; k += kTreeLeafThreads) mine += owner[list[k]] == r ? 1u : 0u;
    mine = __reduce_add_sync(0xffffffffu, mine);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(&s_sum, mine);
    __syncthreads();
    if (threadIdx.x == 0) { owned[r] = s_sum; nonempty[r] = s_sum ? 1u : 0u; }
}

struct TreeOut {          // the arrays of gs_upload_splat_tree (+ depth) and gs_upload_splat_tree_nodes
    double *center, *nmin, *nmax;
    uint32_t *offsets, *indexes;
    int32_t *depth;
    double *all_min, *all_max;
    int32_t *parent;
    uint32_t *leaf_node;
    uint32_t *deepest;    // one word: the greatest depth of a kept leaf
};

// One CTA per node of a level; leaves that keep members only.  leaf_index / leaf_offset: exclusive scans of nonempty / owned.
__global__ void __launch_bounds__(kTreeLeafThreads)
k_tree_write_leaves(const uint32_t *__restrict__ split, const uint32_t *__restrict__ seg, const uint32_t *__restrict__ list, const uint32_t *__restrict__ lrank,
                    const uint32_t *__restrict__ dfs, const double *__restrict__ box, int depth, const uint32_t *__restrict__ owner,
                    const uint32_t *__restrict__ owned, const uint32_t *__restrict__ leaf_index, const uint32_t *__restrict__ leaf_offset, TreeOut out) {
    constexpr int NW = kTreeLeafThreads / 32;
    __shared__ uint32_t s_warp[NW];
    __shared__ uint32_t s_base;
    const uint32_t i = blockIdx.x;
    if (split[i]) return;
    const uint32_t r = lrank[i];
    if (!owned[r]) return;
    const uint32_t li = leaf_index[r];
    if (threadIdx.x < 3) {
        const int a = threadIdx.x;
        const double mn = box[6 * (size_t)i + a], mx = box[6 * (size_t)i + 3 + a];
        out.nmin[3 * (size_t)li + a] = mn; out.nmax[3 * (size_t)li + a] = mx;
        out.center[3 * (size_t)li + a] = __dadd_rn(__dmul_rn(__dadd_rn(mx, -mn), 0.5), mn);      // SplatTree.js:121-123
    }
    if (threadIdx.x == 0) {
        out.offsets[li] = leaf_offset[r];
        out.depth[li] = depth;
        out.leaf_node[li] = dfs[i];
        atomicMax(out.deepest, (uint32_t)depth);
        s_base = leaf_offset[r];
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint32_t base = seg[i]; base < seg[i + 1]; base += kTreeLeafThreads) {
        const uint32_t k = base + threadIdx.x;
        const uint32_t splat = k < seg[i + 1] ? list[k] : 0u;
        const bool keep = k < seg[i + 1] && owner[splat] == r;
        const uint32_t b = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) s_warp[warp] = __popc(b);
        __syncthreads();
        uint32_t at = s_base + __popc(b & lanemask_lt());
        for (int w = 0; w < warp; ++w) at += s_warp[w];
        if (keep) out.indexes[at] = splat;
        __syncthreads();
        if (threadIdx.x == 0) { uint32_t sum = 0; for (int w = 0; w < NW; ++w) sum += s_warp[w]; s_base += sum; }
        __syncthreads();
    }
}

// Every node of a level at its depth-first place; parent_dfs: dfs of the level above (nullptr for the root's level)
__global__ void k_tree_write_nodes(const double *__restrict__ box, const uint32_t *__restrict__ parent, const uint32_t *__restrict__ dfs,
                                   const uint32_t *__restrict__ parent_dfs, uint32_t nodes, TreeOut out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nodes) return;
    const uint32_t d = dfs[i];
#pragma unroll
    for (int a = 0; a < 3; ++a) { out.all_min[3 * (size_t)d + a] = box[6 * (size_t)i + a]; out.all_max[3 * (size_t)d + a] = box[6 * (size_t)i + 3 + a]; }
    out.parent[d] = parent_dfs ? (int32_t)parent_dfs[parent[i]] : -1;
}

} // namespace gs
