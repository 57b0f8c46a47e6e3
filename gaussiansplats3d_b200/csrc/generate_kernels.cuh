// generate_kernels.cuh -- SplatBufferGenerator.getStandardGenerator on the GPU: partition, SH range, alpha removal, buckets and the
// SplatBuffer writer at compression levels 0-2.  The restated JavaScript:
//   SplatPartitioner.getStandardPartitioner (SplatPartitioner.js:46-99)
//   SplatBuffer.generateFromUncompressedSplatArrays (SplatBuffer.js:1177-1326), computeBucketsForUncompressedSplatArray (:1328-1399)
//   SplatBuffer.writeSplatDataToSectionBuffer (:1069-1172)
// Inputs are the level-0 records the parse kernels write in generate mode plus the JavaScript numbers beside them (GenOut): the f64
// centre and the f64 SH.  Every f64 step is explicit and unfused.  The order-dependent steps (the SH range scan, bucket filling, the
// order of partially filled buckets) are restated as associative scans and stable sorts; see DESIGN.md section 2.
#pragma once
#include "common.cuh"
#include "ksplat_kernels.cuh"   // to_half_three
#include "file_kernels.cuh"     // js_round

namespace gs {

constexpr int kGenThreads = 256;

// ---- partition key: lengthSq(floor((c - sceneCenter) / 0.5) * 0.5), ascending; NaN keys last --------------------------------------
__global__ void k_gen_partition_key(const double *__restrict__ c64, uint32_t n, double cx, double cy, double cz, unsigned long long *__restrict__ key) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double o[3] = {cx, cy, cz};
    double v[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) v[k] = __dmul_rn(floor(__ddiv_rn(__dsub_rn(c64[(size_t)i * 3 + k], o[k]), 0.5)), 0.5);
    const double d = __dadd_rn(__dadd_rn(__dmul_rn(v[0], v[0]), __dmul_rn(v[1], v[1])), __dmul_rn(v[2], v[2]));
    // d >= +0 or NaN: non-negative doubles order like their bits; every NaN goes after +inf
    key[i] = d != d ? 0xffffffffffffffffull : (unsigned long long)__double_as_longlong(d);
}

// One 24-bit piece of a 64-bit key for a stable LSD radix round, gathered through the current order (pieces stay below 2^32 - 1, which
// the radix kernels reserve for tail slots).
__global__ void k_gen_sort_piece(const unsigned long long *__restrict__ key, const uint32_t *__restrict__ order, uint32_t n, int shift,
                                 uint32_t *__restrict__ keys, uint32_t *__restrict__ vals) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t v = order ? order[i] : i;
    keys[i] = (uint32_t)((key[v] >> shift) & 0xffffffull);
    vals[i] = v;
}

// ---- SH range: `if (!min || v < min) min = v` over FRC0..FRC22 of every splat in partition order -------------------------------------
// The running value m is either falsy (undefined, 0 or NaN: all behave alike, and all end as the default) or a non-zero number.  A run
// of values acts on m as:
//   m falsy -> R (NaN stands for falsy);   m < 0 -> min(m, smin);   m > 0 -> Z ? C : min(m, smin)
// smin: the least non-NaN value (+inf if none); Z: the first non-NaN value <= 0 is a 0 (a positive m falls to 0 there, then the rest
// runs from falsy and gives C).  These summaries compose associatively, so the scan is an ordered reduction.  The max is the min of
// the negated values, negated.
struct ShRun {
    double R, smin, C;
    int Z;
};
__device__ __forceinline__ bool js_falsy(double v) { return v != v || v == 0.0; }
__device__ __forceinline__ double sh_apply(const ShRun &f, double m) {
    if (js_falsy(m)) return f.R;
    if (m > 0.0 && f.Z) return f.C;
    return fmin(m, f.smin);
}
__device__ __forceinline__ ShRun sh_identity() { return ShRun{__longlong_as_double(0x7ff8000000000000ll), __longlong_as_double(0x7ff0000000000000ll), 0.0, 0}; }
__device__ __forceinline__ ShRun sh_compose(const ShRun &a, const ShRun &b) {   // a, then b
    ShRun r;
    r.R = sh_apply(b, a.R);
    r.smin = fmin(a.smin, b.smin);
    r.Z = a.Z || (a.smin > 0.0 && b.Z);
    r.C = a.Z ? sh_apply(b, a.C) : b.C;
    return r;
}
__device__ __forceinline__ ShRun sh_step(const ShRun &a, double v) {
    ShRun b;
    b.R = js_falsy(v) ? __longlong_as_double(0x7ff8000000000000ll) : v;
    b.smin = v != v ? __longlong_as_double(0x7ff0000000000000ll) : v;
    b.Z = v == 0.0;
    b.C = __longlong_as_double(0x7ff8000000000000ll);
    return sh_compose(a, b);
}

constexpr int kGenShItems = 8;   // consecutive splats per thread
__global__ void __launch_bounds__(kGenThreads) k_gen_sh_scan(const double *__restrict__ sh64, int ncomp, int nscan, const uint32_t *__restrict__ perm,
                                                             uint32_t n, ShRun *__restrict__ out /* [block][2]: min, max of negated */) {
    __shared__ ShRun s_min[kGenThreads], s_max[kGenThreads];
    ShRun mn = sh_identity(), mx = sh_identity();
    const uint64_t first = ((uint64_t)blockIdx.x * kGenThreads + threadIdx.x) * kGenShItems;
    for (int it = 0; it < kGenShItems; ++it) {
        if (first + it >= n) break;
        const double *v = sh64 + (size_t)perm[first + it] * ncomp;
        for (int s = 0; s < nscan; ++s) { const double x = v[s]; mn = sh_step(mn, x); mx = sh_step(mx, -x); }
    }
    s_min[threadIdx.x] = mn; s_max[threadIdx.x] = mx;
    __syncthreads();
    for (int st = 1; st < kGenThreads; st <<= 1) {   // ordered pairwise tree: left operand first
        if ((threadIdx.x & (2 * st - 1)) == 0) {
            s_min[threadIdx.x] = sh_compose(s_min[threadIdx.x], s_min[threadIdx.x + st]);
            s_max[threadIdx.x] = sh_compose(s_max[threadIdx.x], s_max[threadIdx.x + st]);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) { out[2 * blockIdx.x] = s_min[0]; out[2 * blockIdx.x + 1] = s_max[0]; }
}
// Blocks in order; `|| DefaultSphericalHarmonics8BitCompressionHalfRange` at the end.  range[0] = min, range[1] = max (f64).
__global__ void k_gen_sh_final(const ShRun *__restrict__ runs, uint32_t blocks, double *__restrict__ range) {
    ShRun mn = sh_identity(), mx = sh_identity();
    for (uint32_t b = 0; b < blocks; ++b) { mn = sh_compose(mn, runs[2 * b]); mx = sh_compose(mx, runs[2 * b + 1]); }
    const double lo = mn.R, hi = -mx.R;
    range[0] = js_falsy(lo) ? -1.5 : lo;
    range[1] = js_falsy(hi) ? 1.5 : hi;
}

// ---- exclusive scan of u32 flags: out[0..n] (out[n] = total) ---------------------------------------------------------------------------
constexpr int kScanThreads = 1024, kScanItems = 4, kScanTile = kScanThreads * kScanItems;
__global__ void __launch_bounds__(kScanThreads) k_gen_scan_reduce(const uint32_t *__restrict__ in, uint32_t n, uint32_t *__restrict__ sums) {
    __shared__ uint32_t s_scan[40];
    uint32_t v = 0;
    const uint64_t base = (uint64_t)blockIdx.x * kScanTile + (uint64_t)threadIdx.x * kScanItems;
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) if (base + k < n) v += in[base + k];
    uint32_t total;
    (void)block_exclusive_scan<kScanThreads>(v, s_scan, total);
    if (threadIdx.x == 0) sums[blockIdx.x] = total;
}
__global__ void __launch_bounds__(kScanThreads) k_gen_scan_apply(const uint32_t *__restrict__ in, uint32_t n, const uint32_t *__restrict__ sums,
                                                                uint32_t ntiles, uint32_t *__restrict__ out) {
    __shared__ uint32_t s_scan[40];
    uint32_t v[kScanItems], t = 0;
    const uint64_t base = (uint64_t)blockIdx.x * kScanTile + (uint64_t)threadIdx.x * kScanItems;
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) { v[k] = base + k < n ? in[base + k] : 0u; t += v[k]; }
    uint32_t total;
    uint32_t run = block_exclusive_scan<kScanThreads>(t, s_scan, total) + sums[blockIdx.x];
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) if (base + k < n) { out[base + k] = run; run += v[k]; }
    if (blockIdx.x == 0 && threadIdx.x == 0) out[n] = sums[ntiles];
}

// ---- alpha removal: `(opacity || 0) >= minimumAlpha`, per section, keeping order ----------------------------------------------------
__global__ void k_gen_keep(const unsigned char *__restrict__ rec0, uint32_t out_bytes, const uint32_t *__restrict__ perm, uint32_t n, uint32_t min_alpha,
                           uint32_t *__restrict__ keep) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    keep[p] = rec0[(size_t)perm[p] * out_bytes + 43] >= min_alpha ? 1u : 0u;
}
// kept splat j (section order): its source splat and its section
__global__ void k_gen_compact(const uint32_t *__restrict__ perm, const uint32_t *__restrict__ keep, const uint32_t *__restrict__ scan, uint32_t n,
                              uint32_t section_size, uint32_t *__restrict__ src, uint32_t *__restrict__ sec) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n || !keep[p]) return;
    src[scan[p]] = perm[p];
    sec[scan[p]] = p / section_size;
}
// sec_base[s] = kept splats in sections < s, s = 0..nsec
__global__ void k_gen_section_base(const uint32_t *__restrict__ scan, uint32_t n, uint32_t section_size, uint32_t nsec, uint32_t *__restrict__ sec_base) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s > nsec) return;
    sec_base[s] = scan[min((unsigned long long)s * section_size, (unsigned long long)n)];
}

// ---- bounds: min / max from the section's first centre with strict comparisons (a NaN first centre poisons the axis) -------------
__device__ __forceinline__ unsigned long long order_key(double d) {   // monotonic in d for non-NaN d; -0 counts as +0
    if (d == 0.0) d = 0.0;
    const unsigned long long b = (unsigned long long)__double_as_longlong(d);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double from_order_key(unsigned long long k) {
    return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}
__global__ void k_gen_bounds(const double *__restrict__ c64, const uint32_t *__restrict__ src, const uint32_t *__restrict__ sec,
                             const uint32_t *__restrict__ sec_base, uint32_t m, unsigned long long *__restrict__ bmin, unsigned long long *__restrict__ bmax,
                             uint32_t *__restrict__ nan_first) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const uint32_t s = sec[j];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double c = c64[(size_t)src[j] * 3 + k];
        if (c != c) { if (j == sec_base[s]) nan_first[3 * s + k] = 1u; continue; }
        atomicMin(bmin + 3 * s + k, order_key(c));
        atomicMax(bmax + 3 * s + k, order_key(c));
    }
}
struct GenGeom {
    double min[3];
    double yblocks, zblocks;
};
__global__ void k_gen_geometry(const unsigned long long *__restrict__ bmin, const unsigned long long *__restrict__ bmax, const uint32_t *__restrict__ nan_first,
                               const uint32_t *__restrict__ sec_base, uint32_t nsec, double block, GenGeom *__restrict__ geom) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= nsec || sec_base[s + 1] == sec_base[s]) return;
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    double lo[3], hi[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        lo[k] = nan_first[3 * s + k] ? nan : from_order_key(bmin[3 * s + k]);
        hi[k] = nan_first[3 * s + k] ? nan : from_order_key(bmax[3 * s + k]);
    }
    GenGeom g;
    g.min[0] = lo[0]; g.min[1] = lo[1]; g.min[2] = lo[2];
    g.yblocks = ceil(__ddiv_rn(__dsub_rn(hi[1], lo[1]), block));
    g.zblocks = ceil(__ddiv_rn(__dsub_rn(hi[2], lo[2]), block));
    geom[s] = g;
}

// ---- buckets ---------------------------------------------------------------------------------------------------------------------
// bucketId = xBlock (yBlocks zBlocks) + yBlock zBlocks + zBlock.  Its JS object key String(bucketId): an integer 0 <= id <= 2^32 - 2 is
// an array index (class 0, enumerated ascending); any other id (class 1: larger, negative, fractional, NaN, +-inf) enumerates in
// insertion order.  Key identity is the value (-0 and 0 are one key, all NaNs are one key).
//   lo = class 0 ? id : the id's bits, hi = section * 2 + class; the block centre of the splat is kept for the bucket it may create.
__global__ void k_gen_bucket_key(const double *__restrict__ c64, const uint32_t *__restrict__ src, const uint32_t *__restrict__ sec,
                                 const GenGeom *__restrict__ geom, uint32_t m, double block, unsigned long long *__restrict__ lo,
                                 unsigned long long *__restrict__ hi, double *__restrict__ bcenter) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const uint32_t s = sec[j];
    const GenGeom g = geom[s];
    const double half = __ddiv_rn(block, 2.0);
    double b[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        b[k] = floor(__ddiv_rn(__dsub_rn(c64[(size_t)src[j] * 3 + k], g.min[k]), block));
        bcenter[(size_t)j * 3 + k] = __dadd_rn(__dadd_rn(__dmul_rn(b[k], block), g.min[k]), half);
    }
    const double id = __dadd_rn(__dadd_rn(__dmul_rn(b[0], __dmul_rn(g.yblocks, g.zblocks)), __dmul_rn(b[1], g.zblocks)), b[2]);
    const bool index = id >= 0.0 && id <= 4294967294.0 && id == floor(id);
    unsigned long long bits;
    if (index) bits = (unsigned long long)id;
    else bits = id != id ? 0x7ff8000000000000ull : (unsigned long long)__double_as_longlong(id);
    lo[j] = bits;
    hi[j] = (unsigned long long)s * 2u + (index ? 0u : 1u);
}
// head[t] = 1 where a new (section, key) group starts in the sorted order
__global__ void k_gen_heads(const unsigned long long *__restrict__ lo, const unsigned long long *__restrict__ hi, const uint32_t *__restrict__ order,
                            uint32_t m, uint32_t *__restrict__ head) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= m) return;
    const uint32_t j = order[t];
    head[t] = t == 0 || lo[j] != lo[order[t - 1]] || hi[j] != hi[order[t - 1]];
}
// gstart[g] = sorted position of group g's first member; gstart[G] = m
__global__ void k_gen_group_start(const uint32_t *__restrict__ head, const uint32_t *__restrict__ gscan, uint32_t m, uint32_t *__restrict__ gstart) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t == 0) gstart[gscan[m]] = m;
    if (t < m && head[t]) gstart[gscan[t]] = t;
}
// A group's members fill its buckets in section order: ranks [kB, kB + B) form its k-th bucket.  complete[j] = 1 where a member
// completes a bucket (rank = B - 1 mod B); full buckets are numbered in section order of their completion.
__global__ void k_gen_complete(const uint32_t *__restrict__ order, const uint32_t *__restrict__ gscan, const uint32_t *__restrict__ gstart, uint32_t m,
                               uint32_t bucket, uint32_t *__restrict__ complete) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= m) return;
    const uint32_t g = gscan[t + 1] - 1u, r = t - gstart[g], size = gstart[g + 1] - gstart[g];
    complete[order[t]] = (r < size / bucket * bucket && r % bucket == bucket - 1u) ? 1u : 0u;
}
// Groups that end with a partially filled bucket: flag, and the order key among a section's partial buckets (class-0 keys keep their
// ascending sorted order, class-1 keys go by the position of the group's first member).
__global__ void k_gen_partial_keys(const uint32_t *__restrict__ order, const uint32_t *__restrict__ gstart, uint32_t groups, uint32_t bucket,
                                   const unsigned long long *__restrict__ hi, uint32_t *__restrict__ pflag, unsigned long long *__restrict__ pkey_lo,
                                   unsigned long long *__restrict__ pkey_hi) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= groups) return;
    const uint32_t first = order[gstart[g]];
    const unsigned long long h = hi[first];
    pflag[g] = (gstart[g + 1] - gstart[g]) % bucket ? 1u : 0u;
    pkey_hi[g] = h;
    pkey_lo[g] = (h & 1u) ? first : 0u;
}
__global__ void k_gen_partial_list(const uint32_t *__restrict__ pflag, const uint32_t *__restrict__ pscan, uint32_t groups, uint32_t *__restrict__ plist) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g < groups && pflag[g]) plist[pscan[g]] = g;
}
// For partial bucket q (sorted): its group's inverse index, its length, and the per-section count
__global__ void k_gen_partial_info(const uint32_t *__restrict__ porder, uint32_t np, const uint32_t *__restrict__ gstart, uint32_t bucket,
                                   const unsigned long long *__restrict__ pkey_hi, uint32_t *__restrict__ pinv, uint32_t *__restrict__ plen,
                                   uint32_t *__restrict__ pcount) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= np) return;
    const uint32_t g = porder[q];
    pinv[g] = q;
    plen[q] = (gstart[g + 1] - gstart[g]) % bucket;
    atomicAdd(pcount + (pkey_hi[g] >> 1), 1u);
}

// Section layout from the scans: sec_base (kept splats before s), fbase (full buckets before s), pbase (partial buckets before s).
// A section's buckets are its full buckets in completion order, then its partial buckets; bucket numbers are global (fbase + pbase).
struct GenLayout {
    const uint32_t *sec_base, *fbase, *pbase, *pprefix;
};
// Output slot, bucket and (for the member that creates a bucket) the bucket centre of every kept splat
__global__ void k_gen_slots(const uint32_t *__restrict__ order, const uint32_t *__restrict__ gscan, const uint32_t *__restrict__ gstart,
                            const uint32_t *__restrict__ fscan, const uint32_t *__restrict__ pinv, const uint32_t *__restrict__ src,
                            const uint32_t *__restrict__ sec, const double *__restrict__ bcenter, uint32_t m, uint32_t bucket, GenLayout L,
                            uint32_t *__restrict__ out_src, uint32_t *__restrict__ out_bucket, double *__restrict__ bucket_center) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= m) return;
    const uint32_t j = order[t], s = sec[j];
    const uint32_t g = gscan[t + 1] - 1u, r = t - gstart[g], size = gstart[g + 1] - gstart[g], nfull = size / bucket * bucket;
    const uint32_t fb = L.fbase[s], nf = L.fbase[s + 1] - fb, pb = L.pbase[s];
    uint32_t slot, b;
    if (r < nfull) {
        const uint32_t jc = order[gstart[g] + r / bucket * bucket + bucket - 1u];
        const uint32_t f = fscan[jc] - fb;
        slot = f * bucket + r % bucket;
        b = f;
    } else {
        const uint32_t q = pinv[g];
        slot = nf * bucket + (L.pprefix[q] - L.pprefix[pb]) + (r - nfull);
        b = nf + (q - pb);
    }
    b += fb + pb;
    const uint32_t o = L.sec_base[s] + slot;
    out_src[o] = src[j];
    out_bucket[o] = b;
    if (r % bucket == 0u) {
#pragma unroll
        for (int k = 0; k < 3; ++k) bucket_center[(size_t)b * 3 + k] = bcenter[(size_t)j * 3 + k];
    }
}

// last s in [0, count) with a[s] <= v
__device__ __forceinline__ uint32_t gen_find(const uint32_t *a, uint32_t count, uint32_t v) {
    uint32_t lo = 0, hi = count;
    while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (a[mid] <= v) lo = mid; else hi = mid; }
    return lo;
}

// three's toHalfFloat: clamp (NaN passes through), Float32Array store, table lookup (to_half_three)
__device__ __forceinline__ uint16_t to_half_js(float v) { return v != v ? (uint16_t)0x7e00u : to_half_three(v); }
// toUint8(v, min, max) = clamp(floor((clamp(v, min, max) - min) / (max - min) * 255), 0, 255), stored in a Uint8Array (NaN -> 0)
__device__ __forceinline__ unsigned char to_u8_js(double v, double lo, double hi) {
    v = fmax(fmin(v, hi), lo);
    const double q = floor(__dmul_rn(__ddiv_rn(__dsub_rn(v, lo), __dsub_rn(hi, lo)), 255.0));
    return q != q ? 0 : (unsigned char)fmax(fmin(q, 255.0), 0.0);
}

struct GenWriteParams {
    uint32_t m, nsec, level, ncomp, in_bytes, out_bytes;
    double scale_factor;                 // compressionScaleRange / (blockSize * 0.5)
    double scale_range;
};
// One thread per output splat: the record at level 0 (the generate-mode level-0 record as it is), 1 or 2.
__global__ void __launch_bounds__(kGenThreads) k_gen_write(const unsigned char *__restrict__ rec0, const double *__restrict__ c64, const double *__restrict__ sh64,
                                                          const uint32_t *__restrict__ out_src, const uint32_t *__restrict__ out_bucket,
                                                          const double *__restrict__ bucket_center, const uint32_t *__restrict__ sec_base,
                                                          const unsigned long long *__restrict__ data_off, const double *__restrict__ sh_range,
                                                          GenWriteParams P, unsigned char *__restrict__ image) {
    const uint32_t o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= P.m) return;
    const uint32_t s = gen_find(sec_base, P.nsec, o), i = out_src[o];
    const unsigned char *in = rec0 + (size_t)i * P.in_bytes;
    unsigned char *out = image + data_off[s] + (size_t)(o - sec_base[s]) * P.out_bytes;
    if (P.level == 0) {
        for (uint32_t k = 0; k < P.out_bytes; k += 4) *reinterpret_cast<uint32_t *>(out + k) = *reinterpret_cast<const uint32_t *>(in + k);
        return;
    }
    uint16_t h[10];
    const double *bc = bucket_center + (size_t)out_bucket[o] * 3;
    const double top = __dadd_rn(__dmul_rn(P.scale_range, 2.0), 1.0);
#pragma unroll
    for (int k = 0; k < 3; ++k) {   // clamp(Math.round((c - bucketCentre) * factor) + range, 0, 2 range + 1) into a Uint16Array
        const double v = __dadd_rn(js_round(__dmul_rn(__dsub_rn(c64[(size_t)i * 3 + k], bc[k]), P.scale_factor)), P.scale_range);
        h[k] = v != v ? 0 : (uint16_t)fmax(fmin(v, top), 0.0);
    }
#pragma unroll
    for (int k = 0; k < 7; ++k) h[3 + k] = to_half_js(*reinterpret_cast<const float *>(in + 12 + 4 * k));   // scale x3, rotation x4
    for (int k = 0; k < 10; ++k) { out[2 * k] = (unsigned char)h[k]; out[2 * k + 1] = (unsigned char)(h[k] >> 8); }
    for (int k = 0; k < 4; ++k) out[20 + k] = in[40 + k];
    if (P.level == 1) {
        for (uint32_t c = 0; c < P.ncomp; ++c) {
            const uint16_t v = to_half_js(*reinterpret_cast<const float *>(in + 44 + 4 * c));
            out[24 + 2 * c] = (unsigned char)v; out[25 + 2 * c] = (unsigned char)(v >> 8);
        }
    } else {
        const double lo = sh_range[0], hi = sh_range[1];
        for (uint32_t c = 0; c < P.ncomp; ++c) {
            double v = sh64[(size_t)i * P.ncomp + c];
            if (js_falsy(v)) v = 0.0;
            out[24 + c] = to_u8_js(v, lo, hi);
        }
    }
}
// Bucket metadata of levels 1/2: the partial-bucket lengths (u32) and every bucket's centre (f32 x 3).  Sections need not start 4-byte
// aligned (a level-1 degree-1 record is 42 bytes): byte stores.
__device__ __forceinline__ void put_bytes(unsigned char *p, uint32_t v) { p[0] = (unsigned char)v; p[1] = (unsigned char)(v >> 8); p[2] = (unsigned char)(v >> 16); p[3] = (unsigned char)(v >> 24); }
__global__ void k_gen_bucket_meta(const double *__restrict__ bucket_center, const uint32_t *__restrict__ plen, GenLayout L, uint32_t nsec,
                                  uint32_t nbuckets, uint32_t npartial, const unsigned long long *__restrict__ meta_off, const uint32_t *__restrict__ bbase,
                                  unsigned char *__restrict__ image) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < nbuckets) {
        const uint32_t s = gen_find(bbase, nsec, b);
        unsigned char *c = image + meta_off[s] + 4ull * (L.pbase[s + 1] - L.pbase[s]) + 12ull * (b - bbase[s]);
#pragma unroll
        for (int k = 0; k < 3; ++k) put_bytes(c + 4 * k, __float_as_uint(f32_store(bucket_center[(size_t)b * 3 + k])));   // NaN as 0x7fc00000
    }
    if (b < npartial) {
        const uint32_t s = gen_find(L.pbase, nsec, b);
        put_bytes(image + meta_off[s] + 4ull * (b - L.pbase[s]), plen[b]);
    }
}
// bbase[s] = fbase[s] + pbase[s]
__global__ void k_gen_bucket_base(GenLayout L, uint32_t nsec, uint32_t *__restrict__ bbase) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s <= nsec) bbase[s] = L.fbase[s] + L.pbase[s];
}
// fbase[s] = fscan[sec_base[s]]
__global__ void k_gen_gather_base(const uint32_t *__restrict__ scan, const uint32_t *__restrict__ sec_base, uint32_t nsec, uint32_t *__restrict__ out) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s <= nsec) out[s] = scan[sec_base[s]];
}

} // namespace gs
