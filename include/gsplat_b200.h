/* gsplat_b200.h -- C ABI of libgsplat_b200.so: the H100 (sm_90a) depth -> sort -> rasterise engine that
 * sits behind the GaussianSplats3D sort-worker / SplatMesh boundary.
 *
 * Every entry point cites the reference interface (file:line under mkkellogg/GaussianSplats3D @ v0.4.7)
 * it replaces.  Plain pointers and sizes only; no torch / C++ types.  All functions return 0 (GS_OK) or a
 * gs_status error code unless stated otherwise; nothing in this library falls back to the CPU: without a
 * CUDA device every compute entry returns GS_ERR_NO_DEVICE.
 *
 * Memory kinds: pointers are HOST pointers unless the parameter name ends in `_dev`.
 *
 * Threading: like the reference's worker (one sort in flight, SortWorker.js `sortRunning`), an engine handle is driven by one
 * thread at a time; different handles may be used from different threads.  The stateless drop-in (section 1) keeps one cached
 * private engine; concurrent calls are serialised.  gs_last_error_message() is per thread.
 */
#ifndef GSPLAT_B200_H
#define GSPLAT_B200_H

#include <stdint.h>
#include <stdbool.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GS_API __attribute__((visibility("default")))
#define GS_ABI_VERSION 1
#define GS_MAX_SCENES 32 /* Constants.MaxScenes, src/Constants.js:7 */

typedef enum gs_status {
    GS_OK = 0,
    GS_ERR_BAD_ARG = 1,       /* null pointer, sortCount > renderCount, range < 2, ...                        */
    GS_ERR_NO_DEVICE = 2,     /* no CUDA device / CUDA runtime error at init                                   */
    GS_ERR_CUDA = 3,          /* a CUDA call failed; gs_last_error_message() has the text                      */
    GS_ERR_DEGENERATE = 4,    /* all distances equal (reference: rangeMap = inf -> NaN -> wasm trap)           */
    GS_ERR_BUCKET_RANGE = 5,  /* a bucket index fell outside [0, distanceMapRange) (reference: OOB write)      */
    GS_ERR_NOT_READY = 6,     /* render before upload / sort                                                   */
    GS_ERR_CAPACITY = 7       /* splat range outside the capacity given at create time                         */
} gs_status;

GS_API int gs_abi_version(void);
GS_API const char *gs_status_string(int status);
GS_API const char *gs_last_error_message(void); /* thread-local text of the last failing call */
GS_API int gs_device_count(void);

/* ------------------------------------------------------------------------------------------------------------
 * 1. Stateless drop-in for the reference's only native symbol
 *      extern "C" void sortIndexes(...16 args...)                     src/worker/sorter.cpp:17-22
 *    Same argument order and meaning.  HOST pointers, as the wasm module sees its linear memory
 *    (SortWorker.js:56-60).  The two scratch outputs are reproduced too when their pointers are non-NULL:
 *    `mappedDistances[sortStart..renderCount)` = bucket of each position, `frequencies[b]` = number of
 *    sorted splats in buckets < b (what the reference's in-place counters hold on return).
 *    Every call uploads its inputs, runs the CUDA pipeline and downloads indexesOut: this is the
 *    parity-test boundary; the persistent-state path (section 2) is the fast one.
 * ---------------------------------------------------------------------------------------------------------- */
GS_API int gs_sort_indexes(const uint32_t *indexes, const void *centers, const void *precomputedDistances,
                           int32_t *mappedDistances, uint32_t *frequencies, const float *modelViewProj,
                           uint32_t *indexesOut, const uint32_t *sceneIndexes, const float *transforms,
                           uint32_t distanceMapRange, uint32_t sortCount, uint32_t renderCount, uint32_t splatCount,
                           bool usePrecomputedDistances, bool useIntegerSort, bool dynamicMode);

/* The stateless entry keeps ONE private engine cached (sized for the largest call so far, on the caller's current CUDA device) so that
 * repeated calls do not re-allocate; concurrent callers are serialised by a mutex.  gs_dropin_release() frees it (call it before
 * unloading the library or tearing the CUDA context down; it is re-created on demand). */
GS_API void gs_dropin_release(void);

/* void twin with the reference's exact symbol name and signature; errors are swallowed like a wasm trap
 * would abort the call (indexesOut untouched on failure). */
GS_API void sortIndexes(unsigned int *indexes, void *centers, void *precomputedDistances, int *mappedDistances,
                        unsigned int *frequencies, float *modelViewProj, unsigned int *indexesOut,
                        unsigned int *sceneIndexes, float *transforms, unsigned int distanceMapRange,
                        unsigned int sortCount, unsigned int renderCount, unsigned int splatCount,
                        bool usePrecomputedDistances, bool useIntegerSort, bool dynamicMode);

/* ------------------------------------------------------------------------------------------------------------
 * 2. Engine handle: the state a sort Worker + SplatMesh pair keeps on the device.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct gs_engine gs_engine;

typedef struct gs_config {
    uint32_t struct_size;           /* sizeof(gs_config), for ABI growth                                        */
    int32_t device;                 /* CUDA device ordinal                                                       */
    uint32_t max_splat_count;       /* 'splatCount' of createSortWorker          SortWorker.js:202               */
    uint32_t distance_map_range;    /* 1 << splatSortDistanceMapPrecision        SortWorker.js:243, Constants.js:3 */
    uint8_t integer_based_sort;     /* Viewer option integerBasedSort            Viewer.js:95-98                 */
    uint8_t dynamic_mode;           /* Viewer option dynamicScene                SortWorker.js:120               */
    uint8_t ray_records;            /* keep one gs_ray_record per splat for gs_raycast (56 B per splat; 0 = none)   */
    uint8_t reserved0[1];
    uint32_t max_width, max_height; /* largest framebuffer gs_render will be asked for (0,0: sort only)          */
    /* multi-GPU sharding (one engine per process per GPU): this engine rasterises the 128x64-pixel coarse tiles
     * (cx, cy) with (cx + cy) % world_size == rank and leaves every other pixel of its frame zero, so the ranks'
     * frames SUM to the picture (one NCCL all-reduce).  world_size 0 or 1 = everything.                         */
    uint32_t rank, world_size;
} gs_config;

GS_API int gs_create(const gs_config *cfg, gs_engine **out);
GS_API void gs_destroy(gs_engine *e); /* worker.terminate()  Viewer.js:1311 */

/* 'centers' message: persistent sorter centres for splats [from, from+count)      SortWorker.js:84-98
 * centers: int32x4 (integer_based_sort) or f32x4 per splat, exactly what SplatMesh.getIntegerCenters /
 * getFloatCenters(padFour=true) produce (SplatMesh.js:1912-1948).  sceneIndexes may be NULL unless dynamic. */
GS_API int gs_upload_centers(gs_engine *e, const void *centers, const uint32_t *sceneIndexes, uint32_t from,
                             uint32_t count);

typedef struct gs_sort_params {
    uint32_t struct_size;
    float model_view_proj[16];           /* column-major, Viewer.js:1888-1891                                    */
    uint32_t sort_count, render_count;   /* 'splatSortCount' / 'splatRenderCount'    SortWorker.js:99-101         */
    const uint32_t *indexes_to_sort;     /* HOST u32[render_count]; NULL = identity (gatherSceneNodesForSort's
                                            no-tree case, Viewer.js:2061-2074)                                    */
    const uint32_t *indexes_to_sort_dev; /* or DEVICE pointer (takes precedence)                                  */
    const float *transforms;             /* HOST f32[16*GS_MAX_SCENES] when dynamic  SortWorker.js:38-39          */
    const void *precomputed_distances;   /* HOST i32/f32[splat_count] when use_precomputed (SortWorker.js:40-50)  */
    uint8_t use_precomputed_distances;
    uint8_t reserved[3];
} gs_sort_params;

/* 'sort' message -> 'sortDone'.  Runs asynchronously on the engine's stream; the sorted order stays on the
 * device for gs_render.  sorted_out (HOST u32[render_count], may be NULL) receives 'sortedIndexes'
 * (SortWorker.js:68-75); sort_time_ms (may be NULL) the device time of the sort kernels.                       */
GS_API int gs_sort(gs_engine *e, const gs_sort_params *p, uint32_t *sorted_out, float *sort_time_ms);

/* The SplatTree's leaves (`nodesWithIndexes`, src/splattree/SplatTree.js:55-79; uploaded here from a tree built elsewhere, e.g. the
 * reference's own tree worker, or built on the device by gs_build_splat_tree below) and the per-frame half of Viewer.gatherSceneNodesForSort (src/Viewer.js:1969-2077) on the GPU: every leaf is tested against the view
 * frustum (the two angle tests and the `distance > nodeSize` exemption of Viewer.js:2013-2033, f64), the kept leaves are ordered by their
 * distance to the camera and their index runs are written into the engine's indexesToSort (GS_BUF_INDEXES_TO_SORT) from the END of the
 * window backwards -- nearest leaf last -- exactly the layout the reference builds (Viewer.js:2040-2055).  *render_count = splatRenderCount.
 * Follow with gs_sort(indexes_to_sort_dev = GS_BUF_INDEXES_TO_SORT, render_count, sort_count <= render_count): a partial sort
 * (Viewer.js:1843-1856) re-sorts the nearest sort_count splats and copies the rest through (sorter.cpp:158-160).
 * node_center / node_min / node_max: f64[3 * node_count]; node_offsets: u32[node_count + 1]; indexes: u32[node_offsets[node_count]].
 * model_view: f64[16] column-major = inverse(camera.matrixWorld) [* mesh.matrixWorld]; cos_fov_*: Viewer.js:1990-1995.                 */
GS_API int gs_upload_splat_tree(gs_engine *e, const double *node_center, const double *node_min, const double *node_max,
                                const uint32_t *node_offsets, const uint32_t *indexes, uint32_t node_count);
GS_API int gs_gather_for_sort(gs_engine *e, const double *model_view, double cos_fov_x_over_2, double cos_fov_y_over_2, int gather_all_nodes,
                              uint32_t *render_count);
/* The same over a forest (gs_build_splat_tree on a dynamic mesh of several scenes, gs_splat_tree_info.sub_tree_count > 1): every leaf of
 * sub-tree s is culled with model_views[16 s .. 16 s + 16) = baseModelView * sceneTransform(s) (Viewer.js:2005-2011), and the kept leaves
 * of all sub-trees are laid out as one list (ascending distance; ties by leaf number, i.e. sub-tree order, then depth-first order).
 * count must be the tree's sub-tree count, else GS_ERR_BAD_ARG naming both; count = 1 on a tree of one sub-tree is gs_gather_for_sort,
 * and gs_gather_for_sort on a forest is GS_ERR_BAD_ARG.  model_views: f64[16 * count], column-major.                               */
GS_API int gs_gather_for_sort_subtrees(gs_engine *e, const double *model_views, uint32_t count, double cos_fov_x_over_2, double cos_fov_y_over_2,
                                       int gather_all_nodes, uint32_t *render_count);

/* The tree worker's build (SplatTree.js:132-278: createSplatTree / buildSubTree / processSplatTreeNode, flattened as convertWorkerSubTree
 * :55-79 does) on the GPU, from the scene the engine holds: the f32 centre and the alpha byte of GS_BUF_CENTERS_COLORS for splats
 * [0, uploaded splat count).  For a static mesh the scene transform is baked into those centres, which is the Float32Array the reference
 * hands its worker (SplatTree.js:343-353).  The result is bit-exact with the reference's recursion (a centre on a split plane is counted in
 * every child that contains it and kept by the first leaf the depth-first walk reaches; leaves left empty are dropped; indexes ascend inside
 * a leaf) and lands where gs_upload_splat_tree + gs_upload_splat_tree_nodes would have put it: gs_gather_for_sort and gs_raycast work
 * right after.  One sub-tree over all of a static mesh's scenes (SplatTree.processSplatMesh, SplatTree.js:378-390).  A dynamic mesh of
 * several scenes (gs_upload_scenes) gets a forest, as the reference's: one sub-tree per scene over that scene's kept centres in scene-local
 * space, each with its own root box, and each sub-tree exactly the tree of its scene alone (indexes shifted by the scene's splat
 * offset).  The arrays are the concatenation of the sub-trees in scene order (leaves and nodes depth first inside each; every root's
 * parent is -1); sub_tree_count is the scene count, and a scene without a kept splat has an empty sub-tree (no node, no leaf).  Cull a
 * forest with gs_gather_for_sort_subtrees and cast at it with gs_raycast_params.sub_tree_from_local.  gs_upload_splat_tree /
 * gs_upload_splat_tree_nodes take one tree; a forest is only built here.
 *   Two cases differ.  A level-1/2 section decoded WITH a scene transform has the transform baked into its f32-rounded centre, where the
 *     reference transforms the unrounded one (SplatBuffer.js:307-347); and a scene decoded without a transform keeps a non-finite centre
 *     as stored, where the reference's static mesh still multiplies by the identity (0 * inf = NaN).  So on an engine with ray_records
 *     whose scene was decoded on the GPU (gs_upload_ksplat / gs_upload_file / gs_upload_file_optimized) the build takes its centres from
 *     the ray records (unrounded centre, transform, f32: exactly getSplatCenter's) and info->centers_from_ray_records is 1.  Otherwise
 *     it uses the uploaded f32 centres and is the exact tree of those, which is the reference's tree outside these two cases.
 *   min_alpha: a splat takes part when its stored alpha byte >= min_alpha.  The scene uploads zero an alpha below THEIR minimum_alpha, so
 *     this equals the reference's test on the raw byte whenever min_alpha >= the upload's minimum_alpha (the Viewer passes one threshold
 *     to both, SplatMesh.js:236, 394).  For a gs_upload_scenes mesh, min_alpha = 1 is the reference's per-scene test: each scene's
 *     alphas below its minimum_alpha are zeroed at decode, and the reference's thresholds are >= 1 (`splatAlphaRemovalThreshold || 1`).
 *   max_depth <= GS_TREE_MAX_DEPTH and max_centers_per_node >= 1, else GS_ERR_BAD_ARG (the options are checked before the engine).
 *   GS_ERR_NOT_READY without an uploaded scene.
 *   GS_ERR_CAPACITY, naming the level and the count, when one level of the tree would hold more (node, splat) memberships than
 *     max(8 * kept splats, GS_TREE_MIN_LEVEL_CAPACITY): centres exactly on split planes multiply memberships, eightfold per level
 *     when at least max_centers_per_node centres coincide, and the reference then recurses until it runs out of memory.  The level is
 *     counted before it is placed; a failed build leaves the engine's previous tree in place.
 * Scratch is allocated by the call and released when it returns; it runs on the engine's stream and returns synchronised.           */
#define GS_TREE_MAX_DEPTH 20                     /* one membership list is kept per level until the leaves are written          */
#define GS_TREE_MIN_LEVEL_CAPACITY (1u << 22)
typedef struct gs_splat_tree_options {
    uint32_t struct_size;
    uint32_t max_depth;               /* SplatTree maxDepth, default 8 (SplatMesh.js:236)                                           */
    uint32_t max_centers_per_node;    /* SplatTree maxCentersPerNode, default 1000                                                   */
    uint32_t min_alpha;               /* default 1                                                                                   */
} gs_splat_tree_options;
typedef struct gs_splat_tree_info {
    uint32_t struct_size;
    uint32_t leaf_count;              /* leaves that keep at least one splat (nodesWithIndexes)                                      */
    uint32_t node_count;              /* every node, 0 when the engine holds leaves without nodes                                    */
    uint32_t index_count;             /* splats in the leaves = node_offsets[leaf_count]                                             */
    uint8_t has_depth;                /* the leaves carry their depth (built trees; an uploaded tree does not)                       */
    uint8_t has_nodes;                /* all_min / all_max / parent / leaf_node describe the current leaves                          */
    uint8_t centers_from_ray_records; /* the last build took its centres from the ray records (see gs_build_splat_tree)              */
    uint8_t reserved[1];
    /* of the last gs_build_splat_tree, 0 for an uploaded tree */
    uint32_t max_leaf_depth;          /* depth of the deepest kept leaf                                                              */
    uint32_t level_count;             /* levels of the tree (root = 1)                                                               */
    uint64_t max_level_memberships;   /* the largest (node, splat) membership count of one level                                     */
    uint64_t scratch_bytes;           /* device memory the build allocated and released                                              */
    float build_ms;                   /* device time of the build                                                                    */
    uint32_t reserved1;
    /* Appended: written only when struct_size covers it (a caller built before it passes a smaller struct_size, or 0).               */
    uint32_t sub_tree_count;          /* sub-trees: the scene count of a forest (see gs_build_splat_tree), else 1                     */
    uint32_t reserved2;
} gs_splat_tree_info;
GS_API int gs_build_splat_tree(gs_engine *e, const gs_splat_tree_options *opt, gs_splat_tree_info *info /* may be NULL */);
/* The current tree's arrays, built or uploaded, copied to the host.  Any pointer may be NULL and is then skipped; `out` itself may be NULL
 * to ask only for *info (the sizes).  Sizes: node_center / node_min / node_max f64[3 * leaf_count], node_offsets u32[leaf_count + 1],
 * indexes u32[index_count], depth i32[leaf_count], all_min / all_max f64[3 * node_count], parent i32[node_count], leaf_node
 * u32[leaf_count], sub_tree_leaf_offsets / sub_tree_node_offsets u32[sub_tree_count + 1] (sub-tree s holds leaves
 * [sub_tree_leaf_offsets[s], sub_tree_leaf_offsets[s + 1]) and nodes [sub_tree_node_offsets[s], ...[s + 1]); one sub-tree: {0, leaf_count}
 * and {0, node_count}).  Asking for `depth` of a tree that was uploaded, or for a node array when has_nodes is 0, is GS_ERR_NOT_READY:
 * the engine does not hold them.                                                                                                   */
typedef struct gs_splat_tree_arrays {
    uint32_t struct_size;
    uint32_t reserved;
    double *node_center, *node_min, *node_max;
    uint32_t *node_offsets, *indexes;
    int32_t *depth;
    double *all_min, *all_max;
    int32_t *parent;
    uint32_t *leaf_node;
    uint32_t *sub_tree_leaf_offsets, *sub_tree_node_offsets;   /* appended (read only when struct_size covers them)                 */
} gs_splat_tree_arrays;
GS_API int gs_read_splat_tree(gs_engine *e, const gs_splat_tree_arrays *out, gs_splat_tree_info *info /* may be NULL */);

/* D1: the transform-feedback distance pre-pass, SplatMesh.computeDistancesOnGPU (SplatMesh.js:1701-1814): distances
 * in SPLAT order from the uploaded centres.  model_view_proj is f64 because three.js matrices are JS numbers and the
 * integer rows are Math.round(element * 1000) of those doubles (getIntegerMatrixArray, SplatMesh.js:2057-2064);
 * scene_transforms (f64[16*GS_MAX_SCENES], dynamic mode only, else NULL) are the per-scene matrices multiplied in at
 * SplatMesh.js:1722-1724.  out: HOST i32[count] (integer mode) or f32[count] (float mode, SplatMesh.js:1473-1502).   */
GS_API int gs_compute_distances(gs_engine *e, const double *model_view_proj, const double *scene_transforms,
                                uint32_t count, void *out);

/* ------------------------------------------------------------------------------------------------------------
 * 3. Rasteriser: the data textures SplatMesh uploads (setupDataTextures, SplatMesh.js:637-898) and the uniforms
 *    it sets per frame (updateUniforms :1248-1280, Viewer.updateSplatMesh Viewer.js:651-677, three.js camera
 *    matrices).
 * ---------------------------------------------------------------------------------------------------------- */
typedef enum gs_cov_format { GS_COV_F32 = 0, GS_COV_F16 = 1 } gs_cov_format;
typedef enum gs_sh_format { GS_SH_NONE = 0, GS_SH_F16 = 1, GS_SH_U8 = 2, GS_SH_F32 = 3 } gs_sh_format;

typedef struct gs_splat_data {
    uint32_t struct_size;
    uint32_t from, count;             /* splat range being (re)uploaded                                          */
    const uint32_t *centers_colors;   /* u32x4: {r|g<<8|b<<16|a<<24, bits(x), bits(y), bits(z)}  SplatMesh.js:1143-1153 */
    const void *covariances;          /* 6 x f32 (GS_COV_F32) or 6 x f16 (GS_COV_F16, tightly packed) per splat:
                                         [m00 m01 m02 m11 m12 m22]                     SplatBuffer.js:440-486       */
    int32_t cov_format;
    const void *spherical_harmonics;  /* sh_components values per splat, coefficient-major RGB triples
                                         (sh1.rgb, sh2.rgb, ...)                        SplatBuffer.js:551-734      */
    int32_t sh_format;                /* gs_sh_format                                                             */
    uint32_t sh_degree;               /* 0, 1 (9 values) or 2 (24 values)                                         */
    const uint32_t *scene_indexes;    /* u32 per splat or NULL (single scene)                                     */
} gs_splat_data;
/* An upload from splat 0 sets whether the scene has scene indexes: NULL there drops those of any earlier upload, as a fresh engine
 * would have none.  Later partial uploads (from > 0) must agree with it, as they must on the formats: one that gives scene_indexes
 * when the first did not, or omits them when it gave them, is GS_ERR_BAD_ARG and leaves the scene as it was.  gs_upload_ksplat and
 * gs_upload_file load one scene without indexes.                                                                                      */

GS_API int gs_upload_splat_data(gs_engine *e, const gs_splat_data *d);

/* `.ksplat` buffer (the SplatBuffer container, src/loaders/SplatBuffer.js:819-941, KSplatLoader.loadFromFileData) decoded ON THE
 * GPU into everything above at once: centres+colours, covariances, spherical harmonics AND the sorter's centres
 * (= new SplatBuffer(fileData) + SplatMesh.build + the 'centers' message).  Compression levels 0/1/2, SH degree 0/1/2.        */
typedef struct gs_ksplat_options {
    uint32_t struct_size;
    uint32_t minimum_alpha;          /* splatAlphaRemovalThreshold (Viewer.js), default 1: alpha below it renders as 0            */
    uint8_t half_covariances;        /* halfPrecisionCovariancesOnGPU                                                            */
    uint8_t upload_sort_centers;     /* also fill the sorter's centres (integer or float per gs_config), default 1              */
    uint8_t has_transform;           /* bake `transform` into centres, covariances and SH (static scene: SplatMesh.js:1872-1897)  */
    uint8_t reserved[1];
    double transform[16];            /* column-major Matrix4 of the SplatScene (position, quaternion, scale), JS doubles          */
} gs_ksplat_options;
typedef struct gs_ksplat_info {
    uint32_t struct_size;
    uint32_t splat_count, sh_degree, compression_level, section_count;
    float scene_center[3];
    float min_sh_coeff, max_sh_coeff; /* 8-bit SH range -> gs_uniforms.sh8_min/max                                                */
    uint32_t splat_offset;            /* gs_upload_scenes: the scene's first splat in the mesh (0 for the single-scene uploads)      */
} gs_ksplat_info;
/* gs_ksplat_info is filled up to the caller's struct_size: set struct_size = sizeof(gs_ksplat_info) to receive splat_offset.  A
 * struct_size of 0, or one that ends before splat_offset, is a caller built before that field: only the fields up to max_sh_coeff are
 * written.  On return struct_size holds the bytes written.                                                                         */
GS_API int gs_upload_ksplat(gs_engine *e, const void *data, size_t bytes, const gs_ksplat_options *opt, gs_ksplat_info *info);

/* `.ply` (INRIA v1, binary_little_endian 1.0) and `.splat` (32-byte rows) files, loaded the way the reference's progressive loader
 * does (PlyLoader.js:192-206 -> INRIAV1PlyParser.parseToUncompressedSplat; SplatLoader.js:108 -> SplatParser): the splats in FILE ORDER
 * as one compression-level-0 SplatBuffer section, decoded exactly like gs_upload_ksplat decodes that level-0 image.  The header is
 * parsed and validated on the host; a rejected file (GS_ERR_BAD_ARG with the reason, GS_ERR_CAPACITY beyond max_splat_count) leaves
 * the engine's previous scene untouched.  The records are converted on the GPU in fixed-size chunks, so the transient device memory
 * stays small whatever the file's size.  A PlayCanvas-compressed .ply (an `element chunk` line or `packed_` in the header, as the
 * reference detects it) goes through the same call: PlayCanvasCompressedPlyParser.parseToUncompressedSplatBuffer's records, SH
 * included, in file order.  An INRIA v2 (codebook) .ply (an `element codebook_centers` line) loads only through
 * gs_upload_file_optimized / gs_generate_splat_buffer, as the reference loads it only through SplatBufferGenerator;
 * gs_upload_file refuses it with GS_ERR_BAD_ARG and leaves the previous scene.
 * GS_FILE_SPZ takes a `.spz` file's packed stream AFTER gunzip (the library does not inflate; Python's gzip and Node's
 * zlib.gunzipSync do): SpzLoader.unpackGaussians' records, versions 1 (float16 positions) and 2 (24-bit fixed point), SH degree
 * min(file, 2) as for .ply.  A gzip stream (starting 1f 8b) is rejected with a message saying so.  The antialiased flag is ignored,
 * as the reference ignores it.  Through gs_upload_file the splats come in file order (the reference with optimizeSplatData off),
 * through gs_upload_file_optimized / gs_generate_splat_buffer as its default optimizeSplatData load builds them.                  */
typedef enum gs_file_format { GS_FILE_PLY = 1, GS_FILE_SPLAT = 2, GS_FILE_KSPLAT = 3, GS_FILE_SPZ = 4 } gs_file_format;   /* SceneFormat.Ply / .Splat / .KSplat / .Spz */
/* Header parse and validation only: no engine and no device needed.  info->splat_count and info->sh_degree (the file's degree,
 * min(file, 2); for INRIA v2 too, so that the Viewer can size its engine).                                                       */
GS_API int gs_probe_file(int format, const void *data, size_t bytes, gs_ksplat_info *info);
/* Decode on the GPU into centres+colours, covariances, SH and (opt->upload_sort_centers) the sorter's centres.
 * sh_degree = Viewer option sphericalHarmonicsDegree (0..2). opt = the gs_ksplat_options used by gs_upload_ksplat.
 * info->sh_degree = the uploaded degree, min(sh_degree, file degree).                                                             */
GS_API int gs_upload_file(gs_engine *e, int format, const void *data, size_t bytes, uint32_t sh_degree,
                          const gs_ksplat_options *opt, gs_ksplat_info *info);

/* Streamed load: the reference's progressive load (PlyLoader / SplatLoader / KSplatLoader.loadFromURL with progressiveLoadToSplatBuffer,
 * Viewer.downloadAndBuildSingleSplatSceneProgressiveLoad, Viewer.js:871-946), fed with the file's bytes as they arrive.
 *   Formats: INRIA v1 .ply (SH degree min(file, sh_degree, 2)), PlayCanvas-compressed .ply without SH, .splat, and .ksplat (sh_degree
 *     is ignored, as gs_upload_ksplat has none).  Refused by gs_stream_open or, once the header shows it, by gs_stream_append, with
 *     GS_ERR_BAD_ARG and the reason, as Viewer.isProgressivelyLoadable and PlyLoader's DirectLoadError refuse them: .spz, INRIA v2
 *     .ply, a compressed .ply with SH.  An engine with world_size > 1 is refused (one scene on one GPU).
 *   The header is parsed and checked by the whole-file parsers once its bytes are complete; a bad header or more splats than
 *     max_splat_count fails there (GS_ERR_BAD_ARG / GS_ERR_CAPACITY) and leaves the previous scene untouched.  The previous scene is
 *     replaced when the first splats are committed.
 *   Each append converts and decodes the records it completes, [loaded, loaded + k), with the kernels of gs_upload_file /
 *     gs_upload_ksplat, sorter centres included (opt->upload_sort_centers), and commits the prefix: after it the engine holds exactly
 *     what gs_upload_file (gs_upload_ksplat) of the whole file holds over [0, loaded), and gs_render / gs_frame / gs_frame_async /
 *     gs_frame_begin render that prefix (render_count <= loaded).  A record split across appends waits in the stream's host copy of
 *     the bytes, which holds the whole file until gs_stream_destroy.  A PlayCanvas chunk of 256 splats is converted from its start
 *     each time it grows (its splats share one row of quantisation extremes); no splat is decoded twice.
 *   gs_stream_close: after it every engine buffer is that of the whole-file upload and *info is its report.  A stream that ended short
 *     (inside the header, or before the header's splat count, or inside a .splat row) fails with GS_ERR_BAD_ARG naming the loaded and
 *     expected counts; the loaded prefix stays renderable.  The SplatTree is not built here: build it after close
 *     (gs_build_splat_tree), as the reference builds it on the final build only.
 *   A failed append ends the stream: later appends and close return GS_ERR_BAD_ARG.  An append or close after another upload replaced
 *     the stream's scene is GS_ERR_NOT_READY.  Append after close is GS_ERR_BAD_ARG.  gs_stream_destroy frees the stream (before its
 *     engine), closed or not.  One thread drives a stream and its engine.                                                              */
typedef struct gs_file_stream gs_file_stream;
GS_API int gs_stream_open(gs_engine *e, int format, uint32_t sh_degree, const gs_ksplat_options *opt, gs_file_stream **out);
/* progress (may be NULL): the report of the loaded prefix, as gs_ksplat_info (struct_size rules as for gs_upload_ksplat):
 * splat_count = the splats loaded so far, the rest as gs_stream_close will report them (all zero until the header is complete).   */
GS_API int gs_stream_append(gs_file_stream *s, const void *data, size_t bytes, gs_ksplat_info *progress);
GS_API int gs_stream_close(gs_file_stream *s, gs_ksplat_info *info /* may be NULL */);
GS_API void gs_stream_destroy(gs_file_stream *s);

/* SplatMesh.updateVisibleRegion's loop (SplatMesh.js:1172-1199) on the GPU: the largest distance from scene_center (f64[3], NULL =
 * the origin, a progressive buffer's centre) of the uploaded splats [from, to), each centre being the f32 centre of
 * GS_BUF_CENTERS_COLORS through `transform` (f64[16] column-major, NULL = identity, applied all the same as getSplatCenter(i, c, true)
 * applies the scene transform: three.js applyMatrix4 with its divide by w).  f64, unfused, correctly rounded sqrt; a NaN distance
 * never counts and the maximum starts at 0, so the result is the reference's whatever the order.  GS_ERR_BAD_ARG outside [0, uploaded). */
GS_API int gs_visible_region(gs_engine *e, uint32_t from, uint32_t to, const double *transform, const double *scene_center, double *max_distance);

/* SplatMesh.computeBoundingBox(applySceneTransforms, sceneIndex) (SplatMesh.js:2066-2094) on the GPU: the per-axis min and max of the
 * centres fillSplatDataArrays writes into its Float32Array, for one scene or the whole mesh, bit for bit the reference's loop:
 *   compare   `if (i === 0 || x < min.x) min.x = x` (and > for max): the range's first splat seeds both, so a NaN there stays NaN; after
 *             it a NaN never counts; +-inf count as any value; of equal values (-0 and +0) the first splat's is kept.  An empty range
 *             gives (0,0,0)-(0,0,0), new THREE.Vector3().
 *   centres   as gs_build_splat_tree takes them.  On an engine with ray_records whose scene was decoded on the GPU (gs_upload_ksplat,
 *             gs_upload_file(_optimized), gs_upload_scenes, a stream): the record's unrounded centre, through the scene transform (f64,
 *             Vector3.applyMatrix4 with its divide by w) when applied, stored as f32 -- exactly the reference's, both ways.  Otherwise the
 *             f32 centres of GS_BUF_CENTERS_COLORS: a static mesh's scene has its transform baked into them when it was loaded with one
 *             (has_transform), and the identity is applied to the others, as the reference applies it (0 * inf = NaN); a dynamic mesh's
 *             are scene-local and go through scene_transforms.  A scene uploaded with gs_upload_splat_data counts as loaded without a
 *             transform.  Deviation: without ray records a level-1/2 section's centre is rounded to f32 before its transform, where the
 *             reference transforms the unrounded centre (as for gs_build_splat_tree).
 *   scene_index  -1: every splat of the mesh; else scene s of a gs_upload_scenes mesh (any other mesh is one scene, 0).  Outside the
 *             mesh's scenes: GS_ERR_BAD_ARG (the reference throws 'Invalid scene index').
 *   apply_scene_transforms  0 (the reference's default): the centres before any scene transform.  Deviation: 0 on a static mesh whose
 *             scene was loaded with a transform, on an engine without ray records, is GS_ERR_BAD_ARG naming the scene: only the
 *             transformed centres are kept.
 *   scene_transforms  f64[16 * scene count], column-major, each scene's current SplatScene transform: read by a dynamic mesh when
 *             apply_scene_transforms is set (NULL = identity), ignored otherwise (a static mesh keeps its own).
 * Runs on the engine's stream and returns once out_min / out_max (HOST f32[3] each) are written.  A struct_size of 0 reads the whole
 * struct; params = NULL is scene_index -1 without transforms.                                                                       */
typedef struct gs_bounding_box_params {
    uint32_t struct_size;
    int32_t scene_index;
    uint8_t apply_scene_transforms;
    uint8_t reserved[7];
    const double *scene_transforms;
} gs_bounding_box_params;
GS_API int gs_compute_bounding_box(gs_engine *e, const gs_bounding_box_params *params, float out_min[3], float out_max[3]);

/* The reference's default (non-progressive) load and its .ply -> .ksplat converter: SplatBufferGenerator.getStandardGenerator
 * (SplatPartitioner.js:46-99, SplatBuffer.generateFromUncompressedSplatArrays :1177-1399) on the GPU.  Splats are ordered by their
 * clamped distance from scene_center and split into sections, those below minimum_alpha are REMOVED, the rest are grouped into
 * spatial buckets and written at compression level 0, 1 or 2.  Equal partition keys keep file order (DESIGN.md section 2).
 * gen = NULL: getStandardGenerator's defaults (level 1, minimum alpha 1).  Level > 2, a block size that is not finite and > 0, or a
 * bucket size above 2^31 is GS_ERR_BAD_ARG; the file is validated as gs_upload_file validates it.  The image's SH degree is
 * min(sh_degree, file degree), except for an INRIA v2 .ply: the reference builds its array at the requested degree, so the image
 * (and info->sh_degree of gs_upload_file_optimized) carries sh_degree, with 0 in every coefficient the file lacks.                */
typedef struct gs_generate_options {
    uint32_t struct_size;
    uint32_t compression_level;      /* 0..2 (inMemoryCompressionLevel / create-ksplat)                                           */
    uint32_t minimum_alpha;          /* splatAlphaRemovalThreshold: splats below it are removed                                   */
    uint32_t section_size;           /* 0 = one section                                                                           */
    uint32_t bucket_size;            /* 0 = 256                                                                                   */
    double block_size;               /* 0 = 5.0                                                                                   */
    double scene_center[3];
} gs_generate_options;
/* Loads the file as the reference's default path does: the same result as gs_upload_ksplat of gs_generate_splat_buffer's image.
 * GS_ERR_CAPACITY when the file holds more splats than max_splat_count; a rejected call leaves the previous scene in place.       */
GS_API int gs_upload_file_optimized(gs_engine *e, int format, const void *data, size_t bytes, uint32_t sh_degree,
                                    const gs_ksplat_options *opt, const gs_generate_options *gen, gs_ksplat_info *info);
/* create-ksplat: the .ksplat image in page-locked host memory (free with gs_host_free).  Needs a device, not an engine.            */
GS_API int gs_generate_splat_buffer(int device, int format, const void *data, size_t bytes, uint32_t sh_degree,
                                    const gs_generate_options *gen, void **image, size_t *image_bytes);

/* Several scenes in one mesh: Viewer.addSplatScenes -> SplatMesh.build(splatBuffers, sceneOptions) (Viewer.js:973-1085,
 * SplatMesh.js:306-405), up to GS_MAX_SCENES.  Each scene is loaded as its single-scene entry loads it: GS_FILE_KSPLAT as
 * gs_upload_ksplat, a file with `optimized` as gs_upload_file_optimized (with `generate`), without it as gs_upload_file.  Scene s's
 * splats are [splat_offset_s, splat_offset_s + count_s), in scene order, and carry scene index s (SplatMesh.js:203-220, 881-897).
 *   Mesh-level formats, over all scenes: SH degree = min(sh_degree, each scene's degree); SH storage = u8 when some scene is level 2,
 *     else f16 (max(1, max level), SplatMesh.js:1064-1078).  A level-0 scene in a u8 mesh is stored with toUint8 over its own SH
 *     range, as is a level-0/1 scene with a transform (SplatBuffer.js:639-672); a level-1 scene without one stores 0 in every SH
 *     byte, because the reference's fromHalfFloatToUint8 passes toUint8 no range.  gs_uniforms.sh8_min/max[s] = infos[s].min/max_sh_coeff.
 *   Static engines bake each scene's transform and minimum_alpha as the single-scene entries do; a dynamic engine takes the
 *     transforms per frame (gs_uniforms.scene_transforms, gs_sort_params.transforms), and has_transform there is GS_ERR_BAD_ARG.
 *   1 <= scene_count <= GS_MAX_SCENES.  Every source is validated and the splat total checked against max_splat_count before the mesh
 *     is touched (an optimized scene counts with its file's splat count, an upper bound of what the generator keeps).  A rejected
 *     call returns GS_ERR_BAD_ARG or GS_ERR_CAPACITY with a message naming the scene index, and leaves the previous mesh in place.
 *     An INRIA v2 .ply without `optimized` is refused, as gs_upload_file refuses it.
 *   With more than one scene the rasteriser and (dynamic) the sorter get the scene indexes (GS_BUF_SCENE_INDEXES), and the ray records
 *     one transform per scene; one scene leaves the engine exactly as its single-scene entry does.
 *   mesh_opt: half_covariances and upload_sort_centers (minimum_alpha and the transform come from each source); NULL = defaults.
 *   Transient device memory is that of one scene at a time.  More than one scene on an engine with world_size > 1 is GS_ERR_BAD_ARG:
 *     multi-scene frames are single-GPU only.                                                                                          */
typedef struct gs_scene_source {
    uint32_t struct_size;            /* sizeof(gs_scene_source), for ABI growth                                                     */
    int32_t format;                  /* GS_FILE_PLY / GS_FILE_SPLAT / GS_FILE_SPZ (after gunzip) / GS_FILE_KSPLAT                      */
    const void *data;                /* HOST bytes of the file                                                                      */
    size_t bytes;
    uint8_t optimized;               /* files only: load through the generator (optimizeSplatData), with `generate`                  */
    uint8_t has_transform;           /* static engines: bake `transform` into this scene                                            */
    uint8_t reserved[2];
    uint32_t minimum_alpha;          /* splatAlphaRemovalThreshold of this scene (0 reads as 1, the reference's `|| 1`)              */
    gs_generate_options generate;    /* when optimized (struct_size 0 = getStandardGenerator's defaults)                            */
    double transform[16];            /* column-major Matrix4 of the SplatScene                                                       */
} gs_scene_source;
GS_API int gs_upload_scenes(gs_engine *e, const gs_scene_source *scenes, uint32_t scene_count, uint32_t sh_degree,
                            const gs_ksplat_options *mesh_opt, gs_ksplat_info *infos /* [scene_count], may be NULL */);

typedef struct gs_uniforms {
    uint32_t struct_size;
    float model_view[16];             /* three: modelViewMatrix = camera.matrixWorldInverse * mesh.matrixWorld    */
    float projection[16];             /* camera.projectionMatrix                                                  */
    float camera_position[3];         /* cameraPosition uniform (world)                                           */
    float focal[2];                   /* SplatMesh.js:1262                                                        */
    float viewport[2];                /* render dimensions * devicePixelRatio, SplatMesh.js:1257-1259             */
    float inverse_focal_adjustment;   /* SplatMesh.js:1265                                                        */
    float ortho_zoom;                 /* SplatMesh.js:1264                                                        */
    int32_t orthographic_mode;        /* SplatMesh.js:1263                                                        */
    float splat_scale;                /* SplatMaterial.js:469                                                     */
    int32_t point_cloud_mode;         /* SplatMaterial.js:473                                                     */
    int32_t sh_degree;                /* sphericalHarmonicsDegree uniform (<= uploaded degree)                    */
    int32_t antialiased;              /* SplatMaterial3D.js:137-145                                               */
    float kernel_2d_size;             /* default 0.3, SplatMaterial3D.js:21                                       */
    float max_screen_space_splat_size;/* the constant the material bakes into its shader, ${parseInt(maxScreenSpaceSplatSize)}.0
                                         (SplatMaterial3D.js:195-196): callers pass the option truncated toward zero; Viewer.js:147
                                         reads `options.maxScreenSpaceSplatSize || 1024`                           */
    float sh8_min[GS_MAX_SCENES];     /* sphericalHarmonics8BitCompressionRangeMin/Max, SplatMaterial.js:402-409  */
    float sh8_max[GS_MAX_SCENES];
    uint32_t scene_count;
    float scene_transforms[16 * GS_MAX_SCENES]; /* dynamic mode `transforms` uniform                              */
    float view_matrix[16];            /* three: viewMatrix (dynamic mode only)                                    */
    float scene_opacity[GS_MAX_SCENES];   /* enableOptionalEffects                                                */
    int32_t scene_visibility[GS_MAX_SCENES];
    int32_t enable_optional_effects;  /* SplatMaterial.js:23-28,124-133; SplatMaterial3D.js:198-202           */
    int32_t dynamic_mode;             /* per-scene transforms in the vertex stage, SplatMaterial.js:136-146       */
    /* fade-in (SplatMaterial.js:347-363) */
    int32_t fade_in_complete;
    float scene_center[3];
    float visible_region_fade_start_radius;
} gs_uniforms;

typedef enum gs_frame_format {
    GS_FRAME_RGBA32F = 0, /* float accumulators, premultiplied colour + coverage alpha                            */
    GS_FRAME_RGBA8 = 1    /* the canvas format: round(clamp(v,0,1)*255) once at the end                           */
} gs_frame_format;

/* One eye of a WebXR stereo frame (gs_render_params.eyes): what three.js sets per sub-camera of the XR ArrayCamera when it draws the
 * splat mesh once per eye (Viewer.js:1599-1620 under renderer.xr; WebXRMode, src/webxr/WebXRMode.js).  These four replace the fields of
 * gs_uniforms with the same names; every other uniform is shared by both eyes, as the material's are (Viewer.updateSplatMesh,
 * Viewer.js:651-687).                                                                                                                */
typedef struct gs_eye {
    float model_view[16];             /* eye.matrixWorldInverse * mesh.matrixWorld                                                   */
    float projection[16];             /* eye.projectionMatrix                                                                         */
    float camera_position[3];         /* cameraPosition uniform of that eye (world)                                                   */
    float view_matrix[16];            /* viewMatrix of that eye (dynamic mode only)                                                   */
} gs_eye;

typedef struct gs_render_params {
    uint32_t struct_size;
    uint32_t width, height;
    uint32_t render_count;              /* geometry.instanceCount, SplatMesh.js:1233-1234                         */
    const uint32_t *sorted_indexes;     /* HOST u32[render_count] = the splatIndex attribute
                                           (SplatMesh.updateRenderIndexes :1228-1235); NULL = use the order of
                                           the engine's last gs_sort                                              */
    const uint32_t *sorted_indexes_dev; /* or DEVICE pointer                                                      */
    int32_t frame_format;               /* gs_frame_format                                                        */
    int32_t flip_y;                     /* 0: row 0 = bottom (GL window coords); 1: row 0 = top (image order)     */
    /* Composite into the caller's opaque pass: Viewer's options.threeScene (Viewer.js:81-82), drawn first, and the splat mesh
     * drawn into the same framebuffer with autoClear off (Viewer.js:1599-1620); DropInViewer's group beside ordinary meshes
     * (DropInViewer.js:8-30).  The splat material tests depth and writes none, with NormalBlending (SplatMaterial3D.js:65-75), and
     * every fragment of a splat has the window depth of its centre, zw = 0.5 * ndc_z + 0.5 (SplatMaterial3D.js:208-210,
     * glDepthRange(0, 1)).  So:
     *   - a fragment passes where zw <= d (three's default LessEqualDepth), d = dest_depth at the pixel; a NaN d passes nothing.
     *     Splats are never tested against each other.
     *   - over the destination (Cd, Ad): C = C_splats + T * Cd, A = A_splats + T * Ad, T = the transmittance the splats leave
     *     (below 1/512 the blend stops early, as without a destination, and T then also scales the destination).
     *   - dest_color: width * height pixels in the frame's own format (RGBA8: 4 bytes, RGBA32F: 4 floats); dest_depth: width *
     *     height floats (window depth in [0, 1]).  Both in the frame's row order (flip_y).  Depth alone composites over
     *     (0,0,0,0); colour alone is an "over" with no depth test; neither is the plain frame.
     *   - D24 deviation: WebGL's default depth buffer is 24-bit fixed point.  The test here is f32 against f32, so a caller that
     *     converts D24 depths to float may see splats that tie the buffer to within 2^-24 go the other way.
     * Each input is a HOST pointer or a DEVICE pointer (`_dev`), not both (GS_ERR_BAD_ARG).  Host inputs are copied in stream
     * order: like frame_out, they must stay valid and unchanged until the frame is complete -- gs_render / gs_frame returned,
     * gs_synchronize after gs_frame_async, gs_frame_end of that frame after gs_frame_begin -- and so must device inputs, which
     * must also be complete when the frame is enqueued (the engine's stream waits for no other stream).
     * Engines with world_size > 1 refuse them (GS_ERR_BAD_ARG).  Callers built before these fields (smaller struct_size) render
     * the plain frame.                                                                                                */
    const void *dest_color;             /* HOST destination colour, or NULL                                       */
    const void *dest_color_dev;         /* or DEVICE pointer                                                      */
    const float *dest_depth;            /* HOST destination depth, or NULL                                        */
    const float *dest_depth_dev;        /* or DEVICE pointer                                                      */
    /* WebXR stereo (WebXRMode.VR / .AR): both eyes of an XR framebuffer side by side in one width x height frame, from ONE draw order
     * (the reference sorts once per frame, with the viewer camera: Viewer.js:1833-1964).  Eye e covers columns [e * width/2,
     * (e+1) * width/2) at (width/2) x height, on its own tile grid; flip_y flips the rows of the whole frame.  Each half is bit-identical to
     * the mono frame of (width/2) x height with the same draw order and gs_uniforms, and that eye's gs_eye fields substituted.
     * gs_render, gs_frame, gs_frame_async and gs_frame_begin accept it; gs_frame sorts with gs_sort_params.model_view_proj (the viewer
     * camera's).  The engine must be created for the whole frame (max_width x max_height), and its first stereo frame allocates the right
     * eye's buffers.  GS_ERR_BAD_ARG: an odd width, dest_* inputs, world_size > 1, or a viewport uniform other than (width/2, height)
     * (splat centres are placed with the viewport uniform, where WebGL uses the GL viewport: they agree at the eye's size).
     * An instance-list overflow in either eye is GS_ERR_CAPACITY, with both eyes' instance count and one eye's capacity.
     * gs_read_projected / GS_BUF_SPLAT_RECORDS after a stereo frame hold the LEFT eye's records; gs_timings.visible_splats counts both
     * eyes' and tile_instances both eyes' instances.  Callers built before this field (smaller struct_size) render the mono frame. */
    const gs_eye *eyes;                 /* HOST gs_eye[2] (left, right), or NULL: the mono frame                  */
    /* View depth beside the colour: for RGB-D output, post effects (fog, depth of field, SSAO), and chaining the frame into another
     * renderer's depth test.  An addition beyond the reference, whose splat material writes no depth (SplatMaterial3D.js:65-75).
     * At pixel p the splats blend front to back exactly as the colour does (same list, same early stop at T < 1/512, in a composited
     * frame only the fragments that pass the caller's depth test); splat i contributes the weight w_i = T_i * alpha_i(p) its colour is
     * multiplied by.
     *   - d_i = -z_view of splat i's centre, recovered from its f32 ndc_z through the z row of the frame's projection (column-major):
     *     z_view = (P[14] - ndc * P[15]) / (ndc * P[11] - P[10]), perspective (d = P[14] / (ndc + P[10])) and orthographic alike.
     *   - depth(p) = sum_i w_i d_i / (1 - T), T the final transmittance before any destination is added (the frame's alpha is 1 - T in a
     *     plain frame); +inf where 1 - T == 0 (no splat reaches the pixel).
     *   - One f32 per pixel whatever the frame format, in the frame's row order (flip_y).  Stereo: width x height, eye e's columns
     *     with eye e's projection.  Multi-view (gs_frame_views): width x (view_count * height), stacked like the colour, band v with
     *     views[v].projection.  Composited: only the splat fragments that pass zw <= d count; where the caller's pass hides every splat
     *     the depth is +inf -- the caller's depth is not merged in.
     *   - Precision: d is limited by ndc_z in f32.  In perspective dd/dndc ~ d^2 / (2 near): at near = 0.1 one ulp of ndc_z near 1
     *     (2^-24) is ~3e-3 units of depth at d = 100 and ~3e-5 at d = 10.
     * depth: 0 = the colour frame alone; 1 = the depth too; anything else, or 1 with world_size > 1, is GS_ERR_BAD_ARG.  The engine
     * allocates its depth planes (max_width x max_height f32, a second one for pipelined frames) on the first frame that asks for them.
     * depth_out: HOST width * height floats (multi-view: * view_count), written as frame_out is (gs_render / gs_frame / gs_frame_views
     * on return, gs_frame_begin on the copy stream by gs_frame_end); NULL (and always for gs_frame_async) leaves the depth on the device,
     * in GS_BUF_DEPTH.  Callers built before these fields (smaller struct_size) render the colour frame alone.                          */
    int32_t depth;
    float *depth_out;
} gs_render_params;

/* renderer.render(splatMesh, camera)  Viewer.js:1616.  frame_out: HOST buffer of width*height*4 floats or bytes
 * (may be NULL: the frame stays on the device, see gs_frame_dev).                                               */
GS_API int gs_render(gs_engine *e, const gs_uniforms *u, const gs_render_params *p, void *frame_out);

/* One viewer frame: Viewer.update() -> runSplatSort (full sort) + render  (Viewer.js:1625-1644, 1599-1623).    */
GS_API int gs_frame(gs_engine *e, const gs_sort_params *s, const gs_uniforms *u, const gs_render_params *p,
                    uint32_t *sorted_out, void *frame_out);

/* Same, but only enqueued on the engine's stream: returns without waiting, the frame stays on the device
 * (gs_buffer_dev(GS_BUF_FRAME)); device-side errors and timings are collected by the next gs_synchronize().         */
GS_API int gs_frame_async(gs_engine *e, const gs_sort_params *s, const gs_uniforms *u, const gs_render_params *p);

/* Pipelined frames: the frame loop of Viewer.selfDrivenUpdate (Viewer.js:1543-1555) with up to three frames in flight.  gs_frame_begin
 * enqueues one frame exactly like gs_frame (camera host -> device, full sort, render) plus the copy of its picture into frame_out (HOST,
 * ideally page-locked: gs_host_alloc; every frame in flight needs its own) on a separate copy stream, and returns at once; gs_frame_end
 * waits for the OLDEST frame in flight, after which its frame_out is complete, and returns that frame's status.  Device frames alternate
 * between two buffers, so frame i+1 is computed while frame i crosses PCIe and frame i+2 is already queued behind it:
 *   begin(0); begin(1); for (i...) { begin(i+2); end(i); }       (begin(0); for (i...) { begin(i+1); end(i); } also works)
 * A fourth gs_frame_begin without a gs_frame_end returns GS_ERR_NOT_READY.                                                            */
GS_API int gs_frame_begin(gs_engine *e, const gs_sort_params *s, const gs_uniforms *u, const gs_render_params *p, void *frame_out);
GS_API int gs_frame_end(gs_engine *e);

/* Several cameras of one splat mesh in one frame: a server rendering for several clients, every camera of a capture, cube-map faces,
 * several viewports of a page.  Each view is one gs_frame of its own camera -- its own depth sort and draw order, unlike a stereo
 * frame's eyes -- but the views share the mesh and their kernels: the view_count depth sorts run as one batched sort (one stable radix
 * sort of every view's keys, the view index above the bucket), and every view is projected, binned and blended in shared launches.
 *   Sort      view v is sorted with views[v].model_view_proj.  The index list, sort_count, render_count and the dynamic-mode transforms
 *             come from s and are shared; s->model_view_proj is not read.
 *   Order     sorted_out (HOST, may be NULL) receives view_count x render_count entries, view by view: view v's block is exactly what
 *             gs_sort returns for that view's matrix, partial sorts (sort_count < render_count) included.
 *   Frame     p->width x p->height is ONE view.  The frame is width x (view_count * height): view v occupies rows [v height, (v+1) height)
 *             and each band is byte for byte the frame gs_frame produces with that view's fields substituted into u and s.  flip_y flips
 *             the rows within each band.  frame_out follows gs_render's rules: HOST memory, or NULL to leave the frame in GS_BUF_FRAME.
 *             The engine must hold the whole stacked frame: view_count * height <= max_height.
 *   Refused   with GS_ERR_BAD_ARG: view_count 0 or above GS_MAX_VIEWS, p->eyes set, any dest_* input, world_size > 1,
 *             use_precomputed_distances (precomputed distances belong to one camera), a stacked frame taller than max_height.
 *   Status    an instance-list overflow in any view is GS_ERR_CAPACITY, with the instance count of all views, as for a stereo frame; the
 *             engine's next frame that fits renders as a fresh engine's would.  After a multi-view frame gs_read_projected returns view
 *             0's records, and gs_timings sums over the views (visible_splats, tile_instances).
 *   Memory    the first frame of V views reserves views up to V (before any frame graph is captured): per view the projected records,
 *             the tile lists and the batched sort's buffers (DESIGN.md has the bytes per view).  A failed reservation returns its error
 *             and leaves the engine rendering the frames it could before.
 * Blocking, like gs_frame: it returns once frame_out and sorted_out are written.  A captured frame graph is replayed only for the same
 * view count.                                                                                                                           */
#define GS_MAX_VIEWS 16
typedef struct gs_view {
    float model_view_proj[16];  /* this camera's sort matrix, as gs_sort_params.model_view_proj (Viewer.js:1888-1891)                */
    float model_view[16];       /* these replace the gs_uniforms fields of the same names for this view                              */
    float projection[16];
    float camera_position[3];
    float view_matrix[16];      /* dynamic mode                                                                                     */
    float focal[2];             /* cameras may differ in fov (SplatMesh.js:1262)                                                     */
    float ortho_zoom;
} gs_view;
GS_API int gs_frame_views(gs_engine *e, const gs_sort_params *s, const gs_uniforms *u, const gs_render_params *p, const gs_view *views,
                          uint32_t view_count, uint32_t *sorted_out, void *frame_out);

/* ------------------------------------------------------------------------------------------------------------
 * 3b. Raycasting: Raycaster.intersectSplatMesh (src/raycaster/Raycaster.js:36-85) against the engine's scene, on the GPU.
 *     Needs an engine created with gs_config.ray_records = 1 and the SplatTree's leaves and nodes (gs_build_splat_tree, or
 *     gs_upload_splat_tree + gs_upload_splat_tree_nodes).  All arithmetic is f64 in three.js (r160) operation order, unfused.
 * ---------------------------------------------------------------------------------------------------------- */
/* What the Raycaster reads of one splat (SplatMesh.getSplatCenter / getSplatScaleAndRotation / getSplatColor, SplatMesh.js:1959-2012,
 * SplatBuffer.js:221-305), before any scene transform: the centre as a JS number (levels 1/2: (u16 - sr) * sf + bucket, not rounded to
 * f32), the stored scale and rotation, and the stored alpha byte (not the minimum_alpha-clamped texel).                          56 B */
typedef struct gs_ray_record {
    double center[3];
    float scale[3];
    float rotation[4];                /* x, y, z, w (THREE.Quaternion order; not normalised)                                        */
    uint8_t alpha;
    uint8_t reserved[3];
} gs_ray_record;
/* gs_upload_ksplat, gs_upload_file and gs_upload_scenes write the records of a ray_records engine (gs_upload_scenes: each scene
 * placed by its own transform on a static mesh; a dynamic mesh of several scenes casts at its forest, one from_local per scene).
 * A scene uploaded with gs_upload_splat_data gets its records here; any other upload (gs_upload_splat_data, gs_upload_centers) marks the records stale until this call refreshes them.
 * scene_transform: f64[16] column-major SplatScene transform a static mesh applies to centre, scale and rotation (SplatMesh.js:1959-1987),
 * NULL = identity (the reference still multiplies by it).  Ignored by dynamic engines, whose transform is part of from_local.          */
GS_API int gs_upload_ray_records(gs_engine *e, const gs_ray_record *records, uint32_t from, uint32_t count, const double *scene_transform);
/* Every node of the SplatTree (SplatTree.js:132-278), depth first, root first: its box (f64[3 * node_count] each), its parent node
 * (-1 for the root) and, for leaf i of gs_upload_splat_tree, leaf_node[i] = its node.  Call after gs_upload_splat_tree.              */
GS_API int gs_upload_splat_tree_nodes(gs_engine *e, const double *node_min, const double *node_max, const int32_t *node_parent, uint32_t node_count,
                                      const uint32_t *leaf_node, uint32_t leaf_count);
typedef enum gs_raycast_mode { GS_RAYCAST_SPHERE = 0, GS_RAYCAST_ELLIPSOID = 1 } gs_raycast_mode;  /* raycastAgainstTrueSplatEllipsoid */
typedef struct gs_raycast_params {
    uint32_t struct_size;
    int32_t mode;                     /* gs_raycast_mode                                                                            */
    double origin[3], direction[3];   /* the world ray (Raycaster.ray; direction normalised, Raycaster.js:13-34)                     */
    double from_local[16];            /* mesh.matrixWorld [* sceneTransform when dynamic], column-major              Raycaster.js:50-54 */
    int32_t scene_visible;            /* SplatScene.visible: 0 = no hits                                             Raycaster.js:117  */
    int32_t reserved;
    /* per scene of a gs_upload_scenes mesh: 0 = no hits from that scene's splats (Raycaster.js:112-114); a splat of a one-scene mesh
     * is scene 0.  Callers built before this field (smaller struct_size) see every scene visible.                                   */
    int32_t scene_visibility[GS_MAX_SCENES];
    /* Per sub-tree of the tree (Raycaster.js:49-82): sub-tree s casts with from_local = sub_tree_from_local[16 s .. 16 s + 16) =
     * mesh.matrixWorld * sceneTransform(s), column-major, and its hits are mapped back with it; the hits of all sub-trees are sorted
     * together.  sub_tree_count 0 (or a caller built before these fields): from_local is sub-tree 0's.  Otherwise sub_tree_count must be
     * the tree's sub-tree count (gs_splat_tree_info) and replaces from_local.  A forest cast with sub_tree_count 0 is GS_ERR_BAD_ARG.      */
    const double *sub_tree_from_local;
    uint32_t sub_tree_count;
    uint32_t reserved2;
} gs_raycast_params;
typedef struct gs_ray_hit {           /* Hit (src/raycaster/Hit.js), world space                                                    */
    double origin[3], normal[3];
    double distance;
    uint32_t splat_index;
    uint32_t reserved;
} gs_ray_hit;
/* intersectSplatMesh: the recursion of castRayAtSplatTreeNode (Raycaster.js:87-165; Ray.intersectBox / intersectSphere, Ray.js:26-113)
 * over the uploaded tree, every hit mapped back to world space, sorted by distance.  *hit_count = the number of hits; the nearest
 * min(capacity, *hit_count) are written to hits in ascending distance (ties: traversal order; NaN distances last).  Runs on the engine's
 * stream (behind any frames in flight) and returns when done.  GS_ERR_NOT_READY: no tree / nodes, or no valid ray records.            */
GS_API int gs_raycast(gs_engine *e, const gs_raycast_params *p, gs_ray_hit *hits, uint32_t capacity, uint32_t *hit_count);

/* ------------------------------------------------------------------------------------------------------------
 * 4. Device-side access for zero-copy callers and for the multi-GPU plumbing (tile gather over NCCL).
 * ---------------------------------------------------------------------------------------------------------- */
typedef enum gs_buffer_id {
    GS_BUF_SORTED_INDEXES = 0, /* u32[render_count]                                                               */
    GS_BUF_FRAME = 1,          /* last rendered frame in the requested format                                     */
    GS_BUF_CENTERS = 2,
    GS_BUF_DISTANCES = 3,      /* i32[render_count] scratch (= mappedDistances)                                   */
    GS_BUF_SPLAT_RECORDS = 4,  /* per-splat projected records (engine-internal 48-byte layout)                    */
    GS_BUF_INDEXES_TO_SORT = 5,/* u32[max_splat_count] staging for indexesToSort                                  */
    GS_BUF_CENTERS_COLORS = 6, GS_BUF_COVARIANCES = 7, GS_BUF_SH = 8,  /* the uploaded / decoded splat data (gs_read_buffer only) */
    GS_BUF_RAY_RECORDS = 9,    /* gs_ray_record per splat (gs_read_buffer only; ray_records engines)                            */
    GS_BUF_SCENE_INDEXES = 10, /* u32 scene index per splat of a multi-scene mesh (gs_read_buffer only; as written by the last upload
                                  that had scene indexes: gs_upload_scenes of > 1 scene, gs_upload_splat_data with scene_indexes)   */
    GS_BUF_DEPTH = 11          /* f32 view depth per pixel of the last frame rendered with gs_render_params.depth = 1              */
} gs_buffer_id;
GS_API int gs_buffer_dev(gs_engine *e, int buffer_id, void **ptr_dev, size_t *bytes);
GS_API int gs_read_buffer(gs_engine *e, int buffer_id, void *out, size_t offset, size_t bytes); /* D2H copy, for tests / tools */
GS_API int gs_stream(gs_engine *e, void **cuda_stream); /* cudaStream_t of the engine */
GS_API int gs_synchronize(gs_engine *e);

/* Fused tile gather (multi-GPU, one process per GPU).  Rank 0 exports CUDA-IPC handles of its frame buffer and of a small handshake
 * block; every other rank attaches, after which its blend kernel stores finished pixels STRAIGHT INTO RANK 0'S FRAME over NVLink
 * and rank 0's frame is complete when gs_frame / gs_synchronize returns -- no NCCL call, no staging copy.  All ranks must render
 * the same sequence of frames.  (Without these calls the ranks' frames are zero outside their own tiles and can be summed.)
 * The exported allocation holds TWO frames (all ranks size it from the same gs_config): rank 0's pipelined frames (gs_frame_begin)
 * alternate between the halves, the half in use travels in the handshake, so frame f+1 is assembled while frame f's picture is
 * copied to the host.  Environment GS_PEER_DOUBLE=0 on rank 0 keeps a single frame.
 * gs_peer_attach_local: the same gather between engines of one process on one device (several engines sharing one GPU, or a test
 * without a second GPU), with plain pointers instead of IPC mappings.  It sets `root` (rank 0 of the same world_size, device and
 * frame size) up as gs_peer_export would if that has not been done, and refuses engines with frames in flight.  Attach every peer
 * before the group's first frame.  `root` must outlive the engines attached to it: destroy the peers first.  On one device every
 * engine's spinning handshake kernel shares the context, so a host call that waits for the whole device (a kernel's first load, a
 * cudaFree) stalls until the peers it waits for arrive: enqueue each frame on the peers before rank 0's, and wait after both.
 * The group's streams (two per engine, two more on rank 0) must each have a hardware work queue of their own, else a peer's
 * spinning wait can block rank 0's release: at most (CUDA_DEVICE_MAX_CONNECTIONS - 2) / 2 engines, 3 with the default 8 queues.
 * Groups of more than 3 engines are refused whatever the queue count (8 engines with 32 queues time out after a graph change).  A group on one
 * device keeps each frame graph it replaces (a new draw count, format or frame size) until the engine is destroyed, because
 * destroying one waits for the whole device while peers may be spinning: a group whose draw count changes every frame grows by
 * one graph per frame.                                                                                                             */
#define GS_IPC_HANDLE_BYTES 64
GS_API int gs_peer_export(gs_engine *e, void *frame_handle /*64 B out*/, void *sync_handle /*64 B out*/);      /* rank 0     */
GS_API int gs_peer_attach(gs_engine *e, const void *frame_handle, const void *sync_handle);                    /* ranks > 0  */
GS_API int gs_peer_attach_local(gs_engine *e, gs_engine *root);                                                /* ranks > 0  */

/* Sort-only on N GPUs (SURVEY.md 8(e) "depth + sort"): ONE sortIndexes call (sorter.cpp:17-168) split by input position.  Every
 * rank holds all centres; rank g computes distances for, and sorts, positions [sortStart + n*g/N, sortStart + n*(g+1)/N) of the
 * sort window.  Two exchanges over peer memory (NVLink), no NCCL, no host round trip: the global min/max before the range map
 * (8 B per rank pair), and the per-bucket run lengths (8 B per bucket per rank pair) from which every rank derives where its runs
 * sit in the reference's order (buckets descending, inside a bucket higher input positions first = rank N-1 ... 0).  Each rank
 * then stores its 4 B/splat straight into RANK 0's sortedIndexes, which is bit-exact with the single-GPU gs_sort.
 *   setup    every rank: gs_shard_export -> exchange the handles (any transport) -> gs_shard_attach with all N block handles
 *            (index = rank) and rank 0's sorted handle.  gs_shard_attach_local: engines of one process on one device (as with
 *            gs_peer_attach_local, every engine of the group must outlive the others' sorts that read its memory).
 *   per sort every rank calls gs_sort_sharded with the SAME parameters; sorted_out is filled on rank 0 only (may be NULL elsewhere).
 *            _async enqueues and returns; _finish waits, copies, reports errors (a missing peer gives GS_ERR_CUDA after ~2 s).
 *   Windows below 8 M splats (env GS_SHARD_MIN overrides; 0 = always split) are sorted by rank 0 alone -- the single-GPU sort is
 *   latency bound there and the exchange would cost more than it saves; the other ranks' calls then return at once.            */
#define GS_MAX_SHARD_RANKS 8
GS_API int gs_shard_export(gs_engine *e, void *block_handle /*64 B out*/, void *sorted_handle /*64 B out*/);
GS_API int gs_shard_attach(gs_engine *e, uint32_t world, const void *block_handles /* world x 64 B */, const void *root_sorted_handle);
GS_API int gs_shard_attach_local(gs_engine *e, uint32_t world, gs_engine *const *engines /* [world], index = rank */);
GS_API int gs_sort_sharded(gs_engine *e, const gs_sort_params *p, uint32_t *sorted_out /* host, rank 0 */, float *sort_time_ms);
GS_API int gs_sort_sharded_async(gs_engine *e, const gs_sort_params *p);
GS_API int gs_sort_sharded_finish(gs_engine *e, uint32_t *sorted_out /* host, rank 0 */, float *sort_time_ms);

/* Page-locked host memory for callers: the counterpart of the SharedArrayBuffer views a shared-memory sort worker
 * hands to the main thread (SortWorker.js:180-191).  Buffers passed to gs_sort / gs_render from such memory are
 * copied asynchronously without an extra staging copy. */
GS_API int gs_host_alloc(void **ptr, size_t bytes);
GS_API int gs_host_free(void *ptr);

/* Per-splat output of the projection stage (what the vertex shader hands to rasterisation), for parity tests. */
typedef struct gs_projected_splat {
    float cx, cy;        /* quad centre, pixels, GL window coordinates (y up, pixel centres at +0.5)              */
    float b1x, b1y;      /* basisVector1 * inverseFocalAdjustment, pixels    SplatMaterial3D.js:193,206-207        */
    float b2x, b2y;      /* basisVector2 ...                                                                      */
    float r, g, b, a;    /* vColor                                                                                */
    float ndc_z;
    uint32_t valid;      /* 0 = culled / dropped                                                                  */
} gs_projected_splat;
GS_API int gs_read_projected(gs_engine *e, gs_projected_splat *out, uint32_t count); /* splat order; the left eye after a stereo frame */

typedef struct gs_timings {
    float depth_ms, bucket_ms, scatter_ms, sort_total_ms;
    float project_ms, bin_ms, blend_ms, render_total_ms;
    float h2d_ms, d2h_ms;
    uint64_t tile_instances;   /* (splat, tile) pairs binned in the last render                                   */
    uint32_t kernel_launches;  /* kernels launched by the last gs_sort, gs_render, gs_frame / gs_frame_async /
                                  gs_frame_begin (a graph frame: the captured frame's), gs_sort_sharded(_async),
                                  gs_gather_for_sort, gs_raycast or gs_build_splat_tree                              */
    uint32_t visible_splats;
} gs_timings;
GS_API int gs_last_timings(gs_engine *e, gs_timings *t);

/* Measurement helpers for bench.py (no effect on results): L2 flush on the engine's stream (writes a scratch buffer
 * of four times the device's L2 size) and CUDA events recorded on that stream, so per-step device times can be taken without touching torch.     */
GS_API int gs_flush_l2(gs_engine *e);
/* Per-kernel timeline: when on, a CUDA event is recorded after each named kernel or stage (a stage may span several
 * kernels, e.g. k_shard_offsets, gen_*, h2d_file_chunk; some kernels, such as the multi-GPU handshake's, are not
 * named); gs_kernel_timings returns {name, device ms since the previous mark} for the last eager gs_sort / gs_render /
 * gs_frame / gs_sort_sharded / gs_upload_file / gs_upload_file_optimized in launch order.                          */
typedef struct gs_kernel_time { char name[40]; float ms; } gs_kernel_time;
GS_API int gs_set_profiling(gs_engine *e, int on);
/* gs_frame / gs_frame_async replay a captured CUDA graph of the frame while its shape is unchanged (default on).      */
GS_API int gs_set_graph_enabled(gs_engine *e, int on);
GS_API int gs_kernel_timings(gs_engine *e, gs_kernel_time *out, uint32_t capacity, uint32_t *count);
GS_API int gs_event_create(void **event);
GS_API int gs_event_record(gs_engine *e, void *event);
GS_API int gs_event_elapsed_ms(void *event0, void *event1, float *ms); /* waits for event1 */
GS_API int gs_event_destroy(void *event);

#ifdef __cplusplus
}
#endif
#endif /* GSPLAT_B200_H */
