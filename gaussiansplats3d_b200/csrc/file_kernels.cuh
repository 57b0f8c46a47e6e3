// file_kernels.cuh -- `.ply` (INRIA v1) and `.splat` records -> compression-level-0 SplatBuffer records on the GPU.
// This is the reference's own load structure (file -> level-0 SplatBuffer section -> SplatMesh): the records written here are decoded by
// the unchanged k_ksplat_decode, so everything downstream of the level-0 image is the `.ksplat` path.
//   .ply    INRIAV1PlyParser.parseToUncompressedSplat (:143-207) + PlyParserUtils.readVertex (:278-302, normalize = true)
//           -> SplatBuffer.writeSplatDataToSectionBuffer, compression level 0 (SplatBuffer.js:1092-1124, 1168-1172)
//   .splat  SplatParser.parseToUncompressedSplatBufferSection (SplatParser.js:13-56)
//   .spz    SpzLoader.unpackGaussians (:160-250) on the gunzipped packed stream, level-0 writer
//   .ply    INRIA v2 (codebook): INRIAV2PlyParser.decodeCodeBook + parseToUncompressedSplat, level-0 writer (generate mode only)
// Level-0 record: centre f32x3 @0, scale f32x3 @12, rotation f32x4 @24, RGBA u8x4 @40, SH f32 x {0, 9, 24} @44.
// float64 steps use explicit __dmul_rn/__dadd_rn/__ddiv_rn/__dsqrt_rn (JavaScript numbers, no FMA contraction); exp is CUDA's f64 exp.
// NaN is stored as 0x7fc00000 wherever a value lands in a Float32Array (JavaScript leaves NaN bit patterns to the engine).
#pragma once
#include "common.cuh"
#include "file_parse.h"

namespace gs {

struct PlyKernelParams {
    uint32_t count, stride, out_bytes;   // records in this chunk, file bytes per record, level-0 bytes per record
    int sh_out;                          // output SH degree (0..2)
    uint32_t sh_per_channel;             // f_rest count / 3
    uint16_t offset[PF_COUNT];
    uint8_t type[PF_COUNT];
};

__device__ __forceinline__ float f32_store(double v) {   // Float32Array element assignment
    const float f = (float)v;
    return f != f ? __uint_as_float(0x7fc00000u) : f;
}
// Generate mode (SplatBufferGenerator): the JavaScript numbers the generator reads beside each level-0 record, at the record's index.
// center: f64 x 3; sh: f64 x ncomp, the raw UncompressedSplatArray values (NaN kept, no `|| 0`).
struct GenOut {
    double *center, *sh;
};

// level-0 records are 44, 80 or 140 bytes in a cudaMalloc'd buffer: every field is 4-byte aligned
__device__ __forceinline__ void put_f32(unsigned char *rec, int at, float v) { *reinterpret_cast<float *>(rec + at) = v; }

// readVertex: the value a DataView getter gives, as a JavaScript number; uchar is normalised (u / 255.0)
__device__ __forceinline__ double ply_value(const unsigned char *r, uint8_t type, uint16_t off) {
    const unsigned char *p = r + off;
    switch (type) {
        case PT_FLOAT: { float v; memcpy(&v, p, 4); return (double)v; }
        case PT_INT: { int32_t v; memcpy(&v, p, 4); return (double)v; }
        case PT_UINT: { uint32_t v; memcpy(&v, p, 4); return (double)v; }
        case PT_SHORT: { int16_t v; memcpy(&v, p, 2); return (double)v; }
        case PT_USHORT: { uint16_t v; memcpy(&v, p, 2); return (double)v; }
        case PT_UCHAR: return __ddiv_rn((double)p[0], 255.0);
        default: return 0.0;
    }
}

// clamp(Math.floor(v), 0, 255) followed by `|| 0` at write time: NaN -> 0.  Math.min/max propagate NaN, fmin/fmax do not: test first.
__device__ __forceinline__ uint32_t to_u8_floor(double v) {
    if (v != v) return 0u;
    return (uint32_t)fmax(fmin(floor(v), 255.0), 0.0);
}

// three.js Quaternion.normalize on JavaScript numbers: l = sqrt(x x + y y + z z + w w); l == 0 -> (0, 0, 0, 1), else multiply by 1 / l
__device__ __forceinline__ void quat_normalize(double &x, double &y, double &z, double &w) {
    const double l = __dsqrt_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)), __dmul_rn(w, w)));
    if (l == 0.0) { x = 0.0; y = 0.0; z = 0.0; w = 1.0; return; }
    const double il = __ddiv_rn(1.0, l);
    x = __dmul_rn(x, il); y = __dmul_rn(y, il); z = __dmul_rn(z, il); w = __dmul_rn(w, il);
}

// Copy a CTA's block of `bytes` (a multiple of 16 unless it is the chunk's last block; the staging buffer is padded so rounding up is
// safe) from global into shared memory with 16-byte loads.  The block starts 16-byte aligned: R * stride is a multiple of 16 for R >= 16.
__device__ __forceinline__ void stage_block(unsigned char *smem, const unsigned char *src, uint32_t bytes) {
    const uint4 *s = reinterpret_cast<const uint4 *>(src);
    uint4 *d = reinterpret_cast<uint4 *>(smem);
    for (uint32_t k = threadIdx.x; k < (bytes + 15) / 16; k += blockDim.x) d[k] = __ldg(s + k);
    __syncthreads();
}

// One thread per record; blockDim.x records per CTA.  SMEM: stage the CTA's records in shared memory first (coalesced), else read them
// straight from global memory (records too large for the shared-memory budget).
template <bool SMEM, bool GEN = false>
__global__ void __launch_bounds__(128) k_ply_to_level0(const unsigned char *__restrict__ in, PlyKernelParams P, unsigned char *__restrict__ out,
                                                       GenOut G = GenOut{}) {
    extern __shared__ uint4 smem_raw[];
    const uint32_t first = blockIdx.x * blockDim.x;
    const uint32_t n_here = min((uint32_t)blockDim.x, P.count - first);
    const unsigned char *r;
    if (SMEM) {
        unsigned char *smem = reinterpret_cast<unsigned char *>(smem_raw);
        stage_block(smem, in + (size_t)first * P.stride, n_here * P.stride);
        r = smem + (size_t)threadIdx.x * P.stride;
    } else r = in + (size_t)(first + threadIdx.x) * P.stride;
    if (threadIdx.x >= n_here) return;
    unsigned char *o = out + (size_t)(first + threadIdx.x) * P.out_bytes;
    auto val = [&](int f) { return ply_value(r, P.type[f], P.offset[f]); };
    // centre: raw x, y, z into a Float32Array
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double c = val(PF_X + k);
        put_f32(o, 4 * k, f32_store(c));
        if (GEN) G.center[(size_t)(first + threadIdx.x) * 3 + k] = c;
    }
    // scale: exp in f64 (0.01 when the file has none), `|| 0` at write time
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        double s = 0.01;
        if (P.type[PF_SCALE0]) { s = exp(val(PF_SCALE0 + k)); if (s != s) s = 0.0; }
        put_f32(o, 12 + 4 * k, f32_store(s));
    }
    // rotation: Quaternion(rot_0, rot_1, rot_2, rot_3) normalised by the parser, set again and normalised by the writer; stored x, y, z, w
    double qx = val(PF_ROT0), qy = val(PF_ROT1), qz = val(PF_ROT2), qw = val(PF_ROT3);
    quat_normalize(qx, qy, qz, qw);
    quat_normalize(qx, qy, qz, qw);
    put_f32(o, 24, f32_store(qx)); put_f32(o, 28, f32_store(qy)); put_f32(o, 32, f32_store(qz)); put_f32(o, 36, f32_store(qw));
    // colour: (0.5 + SH_C0 f_dc) 255, else red 255, else 0; alpha = sigmoid(opacity) 255, else 0 (createSplat's default)
    uint32_t rgba = 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        double c = 0.0;
        if (P.type[PF_DC0]) c = __dmul_rn(__dadd_rn(0.5, __dmul_rn(0.28209479177387814, val(PF_DC0 + k))), 255.0);
        else if (P.type[PF_RED]) c = __dmul_rn(val(PF_RED + k), 255.0);
        rgba |= to_u8_floor(c) << (8 * k);
    }
    if (P.type[PF_OPACITY]) rgba |= to_u8_floor(__dmul_rn(__ddiv_rn(1.0, __dadd_rn(1.0, exp(-val(PF_OPACITY)))), 255.0)) << 24;
    *reinterpret_cast<uint32_t *>(o + 40) = rgba;
    // SH: degree-1 fields f_rest_{i + c rgb}, degree-2 fields f_rest_{3 + i + c rgb} (c = f_rest count / 3), `|| 0` at write time
    if (P.sh_out >= 1) {
        const int ncomp = P.sh_out >= 2 ? 24 : 9;
        for (int s = 0; s < ncomp; ++s) {
            const int src = s < 9 ? (s % 3) + (int)P.sh_per_channel * (s / 3) : 3 + (s - 9) % 5 + (int)P.sh_per_channel * ((s - 9) / 5);
            double v = val(PF_REST0 + src);
            if (GEN) G.sh[(size_t)(first + threadIdx.x) * ncomp + s] = v;
            if (v != v || v == 0.0) v = 0.0;
            put_f32(o, 44 + 4 * s, f32_store(v));
        }
    }
}

// .splat: 32-byte rows (centre f32x3, scale f32x3, RGBA u8x4, rotation u8x4 as (w, x, y, z) around 128).  Rows are staged in shared
// memory like the .ply records (128 x 32 bytes per CTA).
// GEN: the generator's record (SplatParser.parseStandardSplatToUncompressedSplatArray -> writeSplatDataToSectionBuffer): scale `|| 0`,
// and the writer normalises the parser's normalised quaternion a second time.
template <bool GEN = false>
__global__ void __launch_bounds__(128) k_splat_to_level0(const unsigned char *__restrict__ in, uint32_t count, unsigned char *__restrict__ out,
                                                         GenOut G = GenOut{}) {
    __shared__ uint4 smem[128 * 2];
    const uint32_t first = blockIdx.x * blockDim.x;
    const uint32_t n_here = min((uint32_t)blockDim.x, count - first);
    stage_block(reinterpret_cast<unsigned char *>(smem), in + (size_t)first * 32, n_here * 32);
    if (threadIdx.x >= n_here) return;
    const unsigned char *r = reinterpret_cast<const unsigned char *>(smem) + threadIdx.x * 32;
    unsigned char *o = out + (size_t)(first + threadIdx.x) * 44;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        float v;
        memcpy(&v, r + 4 * k, 4);
        if (GEN && k < 3) G.center[(size_t)(first + threadIdx.x) * 3 + k] = (double)v;
        if (GEN && k >= 3 && (v != v || v == 0.0f)) v = 0.0f;
        put_f32(o, 4 * k, f32_store((double)v));
    }
    // Quaternion((r1 - 128) / 128, (r2 - 128) / 128, (r3 - 128) / 128, (r0 - 128) / 128).normalize(), stored w, x, y, z
    double qx = __ddiv_rn((double)r[29] - 128.0, 128.0), qy = __ddiv_rn((double)r[30] - 128.0, 128.0);
    double qz = __ddiv_rn((double)r[31] - 128.0, 128.0), qw = __ddiv_rn((double)r[28] - 128.0, 128.0);
    quat_normalize(qx, qy, qz, qw);
    if (GEN) quat_normalize(qw, qx, qy, qz);   // Quaternion(w, x, y, z): the sum of squares in that order
    put_f32(o, 24, f32_store(qw)); put_f32(o, 28, f32_store(qx)); put_f32(o, 32, f32_store(qy)); put_f32(o, 36, f32_store(qz));
    *reinterpret_cast<uint32_t *>(o + 40) = *reinterpret_cast<const uint32_t *>(r + 24);
}

// ---- PlayCanvas-compressed .ply ------------------------------------------------------------------------------------------------------
//   PlayCanvasCompressedPlyParser.decompressBaseSplat (:379-432) + decompressSphericalHarmonics (:434-460), driven by
//   parseToUncompressedSplatBuffer (:547-585) -> SplatBuffer.writeSplatDataToSectionBuffer, level 0
struct PcKernelParams {
    uint32_t count;                      // splats in this staging chunk
    uint32_t chunk_base;                 // PLY chunk row of its first splat (the staging chunk starts on a multiple of 256)
    uint32_t stride, sh_stride;          // bytes per vertex row, per sh row (uchar f_rest_*)
    uint32_t out_bytes;                  // level-0 bytes per record
    int sh_out;                          // output SH degree (0..2)
    uint32_t read_coeff;                 // {0, 3, 8, 15}[file SH degree]: channel stride of the f_rest_* bytes
    uint32_t color_mask;                 // bit c: chunk extremes for colour channel c
    uint16_t packed[4];                  // offsets of packed_position, packed_rotation, packed_scale, packed_color
};

// unpackUnorm(v, bits) = (v & (2^bits - 1)) / (2^bits - 1)
__device__ __forceinline__ double pc_unorm(uint32_t v, uint32_t mask) { return __ddiv_rn((double)(v & mask), (double)mask); }
// lerp(a, b, t) = a * (1 - t) + b * t
__device__ __forceinline__ double pc_lerp(double a, double b, double t) {
    return __dadd_rn(__dmul_rn(a, __dadd_rn(1.0, -t)), __dmul_rn(b, t));
}
// Math.round: the integer closest to v, ties towards +inf (not floor(v + 0.5), which gives 1 for 0.49999999999999994).  v - floor(v) is
// exact for v >= 0; for v < 0 the result is <= 0 and the caller clamps it to 0 anyway.
__device__ __forceinline__ double js_round(double v) {
    const double r = floor(v);
    return __dadd_rn(v, -r) >= 0.5 ? __dadd_rn(r, 1.0) : r;
}
__device__ __forceinline__ uint32_t pc_u32(const unsigned char *p) { uint32_t v; memcpy(&v, p, 4); return v; }

// One CTA of 256 threads per PLY chunk: the chunk's 18 extremes go to shared memory once.  SMEM: the CTA's 256 vertex rows and 256 sh
// rows are staged in shared memory with 16-byte loads (256 x stride is a multiple of 16), else read in place.
template <bool SMEM, bool GEN = false>
__global__ void __launch_bounds__(kPcChunkSplats) k_pcply_to_level0(const unsigned char *__restrict__ in, const unsigned char *__restrict__ in_sh,
                                                                    const double *__restrict__ table, PcKernelParams P,
                                                                    unsigned char *__restrict__ out, GenOut G = GenOut{}) {
    extern __shared__ uint4 smem_raw[];
    __shared__ double ext[PC_EXTREMES];
    const uint32_t first = blockIdx.x * kPcChunkSplats;
    const uint32_t n_here = min(kPcChunkSplats, P.count - first);
    if (threadIdx.x < PC_EXTREMES) ext[threadIdx.x] = table[(size_t)(P.chunk_base + blockIdx.x) * PC_EXTREMES + threadIdx.x];
    const unsigned char *r, *rs;
    if (SMEM) {
        unsigned char *smem = reinterpret_cast<unsigned char *>(smem_raw);
        unsigned char *smem_sh = smem + kPcChunkSplats * P.stride;
        if (P.sh_out) stage_block(smem_sh, in_sh + (size_t)first * P.sh_stride, n_here * P.sh_stride);
        stage_block(smem, in + (size_t)first * P.stride, n_here * P.stride);
        r = smem + threadIdx.x * P.stride;
        rs = smem_sh + threadIdx.x * P.sh_stride;
    } else {
        __syncthreads();
        r = in + (size_t)(first + threadIdx.x) * P.stride;
        rs = in_sh + (size_t)(first + threadIdx.x) * P.sh_stride;
    }
    if (threadIdx.x >= n_here) return;
    unsigned char *o = out + (size_t)(first + threadIdx.x) * P.out_bytes;
    const uint32_t pos = pc_u32(r + P.packed[0]), rot = pc_u32(r + P.packed[1]), scl = pc_u32(r + P.packed[2]), col = pc_u32(r + P.packed[3]);
    // centre and scale: 11-10-11 unorm, lerp between the chunk's extremes; scale = Math.exp(lerp), `|| 0` at write time
    const uint32_t shift[3] = {21, 11, 0}, mask[3] = {2047, 1023, 2047};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double c = pc_lerp(ext[PC_MIN_X + k], ext[PC_MAX_X + k], pc_unorm(pos >> shift[k], mask[k]));
        put_f32(o, 4 * k, f32_store(c));
        if (GEN) G.center[(size_t)(first + threadIdx.x) * 3 + k] = c;
        double s = exp(pc_lerp(ext[PC_MIN_SX + k], ext[PC_MAX_SX + k], pc_unorm(scl >> shift[k], mask[k])));
        if (s != s) s = 0.0;
        put_f32(o, 12 + 4 * k, f32_store(s));
    }
    // rotation: 2-10-10-10 smallest three, norm = 1 / (sqrt(2) * 0.5) as JavaScript computes it; m is NaN when a² + b² + c² > 1.
    // The writer normalises once and stores x, y, z, w.
    const double norm = 0x1.6a09e667f3bccp+0;
    const double a = __dmul_rn(__dadd_rn(pc_unorm(rot >> 20, 1023), -0.5), norm);
    const double b = __dmul_rn(__dadd_rn(pc_unorm(rot >> 10, 1023), -0.5), norm);
    const double c = __dmul_rn(__dadd_rn(pc_unorm(rot, 1023), -0.5), norm);
    const double m = __dsqrt_rn(__dadd_rn(1.0, -__dadd_rn(__dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b)), __dmul_rn(c, c))));
    double q[4];
    const uint32_t slot = rot >> 30;
    q[0] = slot == 0 ? m : a;
    q[1] = slot == 0 ? a : (slot == 1 ? m : b);
    q[2] = slot <= 1 ? b : (slot == 2 ? m : c);
    q[3] = slot <= 2 ? c : m;
    quat_normalize(q[0], q[1], q[2], q[3]);
#pragma unroll
    for (int k = 0; k < 4; ++k) put_f32(o, 24 + 4 * k, f32_store(q[k]));
    // colour: 8888 unorm; clamp(Math.round(lerp(min, max, c) 255)) with both extremes, else clamp(floor(c 255)); alpha floor(c.w 255)
    uint32_t rgba = 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double ck = pc_unorm(col >> (24 - 8 * k), 255);
        const uint32_t u = (P.color_mask >> k) & 1u ? to_u8_floor(js_round(__dmul_rn(pc_lerp(ext[PC_MIN_R + k], ext[PC_MAX_R + k], ck), 255.0)))
                                                    : to_u8_floor(__dmul_rn(ck, 255.0));
        rgba |= u << (8 * k);
    }
    rgba |= to_u8_floor(__dmul_rn(pc_unorm(col, 255), 255.0)) << 24;
    *reinterpret_cast<uint32_t *>(o + 40) = rgba;
    // SH: u8 (8 / 255) - 4 from f_rest_{j readCoeff + k} into the level-0 slot of (channel j, coefficient k), as k_ply_to_level0 lays it out
    if (P.sh_out >= 1) {
        const int ncomp = P.sh_out >= 2 ? 24 : 9;
        for (int s = 0; s < ncomp; ++s) {
            const int j = s < 9 ? s / 3 : (s - 9) / 5, k = s < 9 ? s % 3 : 3 + (s - 9) % 5;
            double v = __dadd_rn(__dmul_rn((double)rs[j * (int)P.read_coeff + k], 8.0 / 255.0), -4.0);
            if (GEN) G.sh[(size_t)(first + threadIdx.x) * ncomp + s] = v;
            if (v == 0.0) v = 0.0;
            put_f32(o, 44 + 4 * s, f32_store(v));
        }
    }
}

// ---- .spz (the gunzipped packed stream) ----------------------------------------------------------------------------------------------
//   SpzLoader.unpackGaussians (:160-250) + unpackedSplatToUncompressedSplat (:84-145) -> SplatBuffer.writeSplatDataToSectionBuffer,
//   level 0.  Every step is exact f64 arithmetic except the scale's exp.
struct SpzKernelParams {
    uint32_t count;                      // splats in this chunk
    uint32_t out_bytes;                  // level-0 bytes per record
    int sh_out;                          // output SH degree (0..2)
    uint32_t sh_coeff;                   // the file's SH coefficients per channel (0, 3, 8, 15)
    uint32_t version;                    // 1: float16 positions, 2: 24-bit fixed point
    double pos_scale;                    // 1.0 / (1 << fractionalBits), JavaScript int32 shift
    uint32_t plane[SPZ_PLANES];          // offset of each plane's slice of this chunk in the staging buffer (16-byte aligned)
};

// halfToFloat: exact in f64, subnormals and -0 included; exponent 31 gives +-Infinity or NaN
__device__ __forceinline__ double spz_half(uint32_t h) {
    const uint32_t e = (h >> 10) & 31u, m = h & 1023u;
    const double sign = (h >> 15) & 1u ? -1.0 : 1.0;
    if (e == 0) return __ddiv_rn(__dmul_rn(__dmul_rn(sign, 0x1p-14), (double)m), 1024.0);
    if (e == 31) return m ? __longlong_as_double(0x7ff8000000000000ll) : __dmul_rn(sign, __longlong_as_double(0x7ff0000000000000ll));
    return __dmul_rn(__dmul_rn(sign, ldexp(1.0, (int)e - 15)), __dadd_rn(1.0, __ddiv_rn((double)m, 1024.0)));
}

// One thread per splat, reading its bytes from each plane of the chunk (consecutive threads read consecutive bytes).
template <bool GEN = false>
__global__ void __launch_bounds__(128) k_spz_to_level0(const unsigned char *__restrict__ in, SpzKernelParams P, unsigned char *__restrict__ out,
                                                       GenOut G = GenOut{}) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.count) return;
    unsigned char *o = out + (size_t)i * P.out_bytes;
    // centre: v2 sign-extends each 24-bit value and multiplies by the position scale; v1 is float16
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        double c;
        if (P.version == 1) {
            const unsigned char *p = in + P.plane[SPZ_POS] + (size_t)i * 6 + 2 * k;
            c = spz_half((uint32_t)p[0] | ((uint32_t)p[1] << 8));
        } else {
            const unsigned char *p = in + P.plane[SPZ_POS] + (size_t)i * 9 + 3 * k;
            const int32_t v = (int32_t)(((uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16)) ^ 0x800000u) - 0x800000;
            c = __dmul_rn((double)v, P.pos_scale);
        }
        put_f32(o, 4 * k, f32_store(c));
        if (GEN) G.center[(size_t)i * 3 + k] = c;
    }
    // scale: Math.exp(b / 16 - 10)
    const unsigned char *sc = in + P.plane[SPZ_SCALE] + (size_t)i * 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) put_f32(o, 12 + 4 * k, f32_store(exp(__dadd_rn(__ddiv_rn((double)sc[k], 16.0), -10.0))));
    // rotation: xyz = b / 127.5 - 1, w = sqrt(max(0, 1 - |xyz|²)); Quaternion.set(w, x, y, z).normalize() by the loader, normalised again
    // by the writer; stored w, x, y, z
    const unsigned char *r = in + P.plane[SPZ_ROT] + (size_t)i * 3;
    double x = __dadd_rn(__ddiv_rn((double)r[0], 127.5), -1.0), y = __dadd_rn(__ddiv_rn((double)r[1], 127.5), -1.0);
    double z = __dadd_rn(__ddiv_rn((double)r[2], 127.5), -1.0);
    double w = __dsqrt_rn(fmax(0.0, __dadd_rn(1.0, -__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)))));
    quat_normalize(w, x, y, z);
    quat_normalize(w, x, y, z);
    put_f32(o, 24, f32_store(w)); put_f32(o, 28, f32_store(x)); put_f32(o, 32, f32_store(y)); put_f32(o, 36, f32_store(z));
    // colour: floor(((c / 255 - 0.5) / 0.15 SH_C0 + 0.5) 255), clamped; alpha: the byte
    const unsigned char *cl = in + P.plane[SPZ_COLOR] + (size_t)i * 3;
    uint32_t rgba = (uint32_t)in[P.plane[SPZ_ALPHA] + i] << 24;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double t = __ddiv_rn(__dadd_rn(__ddiv_rn((double)cl[k], 255.0), -0.5), 0.15);
        rgba |= to_u8_floor(__dmul_rn(__dadd_rn(__dmul_rn(t, 0.28209479177387814), 0.5), 255.0)) << (8 * k);
    }
    *reinterpret_cast<uint32_t *>(o + 40) = rgba;
    // SH: (b - 128) / 128 from sh[i][k][j] (coefficient-major, channel-minor) into the level-0 slot of (channel j, coefficient k)
    if (P.sh_out >= 1) {
        const int ncomp = P.sh_out >= 2 ? 24 : 9;
        const unsigned char *sh = in + P.plane[SPZ_SH] + (size_t)i * 3 * P.sh_coeff;
        for (int s = 0; s < ncomp; ++s) {
            const int j = s < 9 ? s / 3 : (s - 9) / 5, k = s < 9 ? s % 3 : 3 + (s - 9) % 5;
            const double v = __ddiv_rn((double)sh[3 * k + j] - 128.0, 128.0);
            if (GEN) G.sh[(size_t)i * ncomp + s] = v;
            put_f32(o, 44 + 4 * s, f32_store(v));
        }
    }
}

// ---- INRIA v2 .ply (codebook) ---------------------------------------------------------------------------------------------------------
//   INRIAV2PlyParser.decodeCodeBook (:128-160) + parseToUncompressedSplat (:202-269, readVertex with normalize = false), reached only
//   through SplatBufferGenerator (generate mode).  An index that names no codebook row reads `undefined`, restated as NaN.
struct V2CodebookParams {
    uint32_t rows, stride;               // codebook rows, bytes per codebook row
    uint32_t mask;                       // bit p: the row has entry p (V2Page)
    uint16_t offset[V2_PAGES];           // byte offset of each entry in the row
};

// One thread per codebook row -> table[page][row] (f64): fromHalfFloat of the entry (0 when the file lacks it), then per page
// opacity Math.round(sigmoid(v) 255), features_dc Math.round((0.5 + SH_C0 v) 255), scaling Math.exp(v), every other page v.
__global__ void __launch_bounds__(128) k_inriav2_codebook(const unsigned char *__restrict__ in, V2CodebookParams P, double *__restrict__ table) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= P.rows) return;
    const unsigned char *row = in + (size_t)r * P.stride;
#pragma unroll
    for (int p = 0; p < V2_PAGES; ++p) {
        double v = 0.0;
        if ((P.mask >> p) & 1u) v = spz_half((uint32_t)row[P.offset[p]] | ((uint32_t)row[P.offset[p] + 1] << 8));
        if (p == V2_OPACITY) v = js_round(__dmul_rn(__ddiv_rn(1.0, __dadd_rn(1.0, exp(-v))), 255.0));
        else if (p == V2_DC) v = js_round(__dmul_rn(__dadd_rn(0.5, __dmul_rn(0.28209479177387814, v)), 255.0));
        else if (p == V2_SCALING) v = exp(v);
        table[(size_t)p * P.rows + r] = v;
    }
}

struct V2KernelParams {
    uint32_t count, stride, out_bytes;   // splats in this chunk, file bytes per splat, level-0 bytes per record
    uint32_t rows;                       // codebook rows
    int ncomp_out;                       // SH components of the image (the requested degree: 0, 9, 24)
    int ncomp_read;                      // SH components read from the file (min(requested, file degree)); the rest are 0
    uint32_t sh_per_channel;             // f_rest count / 3
    bool staged;                         // the CTA's rows are staged in shared memory
    uint16_t offset[PF_COUNT];
    uint8_t type[PF_COUNT];
};

// The codebook index in the field at `off`, as readVertex(normalize = false) reads it
__device__ __forceinline__ int64_t v2_index(const unsigned char *r, uint8_t type, uint16_t off) {
    const unsigned char *p = r + off;
    switch (type) {
        case PT_UCHAR: return p[0];
        case PT_USHORT: { uint16_t v; memcpy(&v, p, 2); return v; }
        case PT_SHORT: { int16_t v; memcpy(&v, p, 2); return v; }
        case PT_UINT: { uint32_t v; memcpy(&v, p, 4); return v; }
        case PT_INT: { int32_t v; memcpy(&v, p, 4); return v; }
        default: return 0;
    }
}
__device__ __forceinline__ bool v2_names_row(int64_t i, uint32_t rows) { return i >= 0 && i < (int64_t)rows; }
// codeBook[page][index]: NaN when the index names no row (negative, or >= rows), where the reference reads `undefined`
__device__ __forceinline__ double v2_lookup(const double *__restrict__ table, uint32_t rows, int page, int64_t i) {
    return v2_names_row(i, rows) ? __ldg(table + (size_t)page * rows + i) : __longlong_as_double(0x7ff8000000000000ll);
}

// One thread per splat; blockDim.x splats per CTA, staged in shared memory like k_ply_to_level0 when they fit.  Writes the level-0 record
// at the image's SH width, the f64 centre and the raw f64 SH (NaN kept; 0 past the components read).
__global__ void __launch_bounds__(128) k_inriav2_to_level0(const unsigned char *__restrict__ in, const double *__restrict__ table, V2KernelParams P,
                                                           unsigned char *__restrict__ out, GenOut G) {
    extern __shared__ uint4 smem_raw[];
    const uint32_t first = blockIdx.x * blockDim.x;
    const uint32_t n_here = min((uint32_t)blockDim.x, P.count - first);
    const unsigned char *r;
    if (P.staged) {
        unsigned char *smem = reinterpret_cast<unsigned char *>(smem_raw);
        stage_block(smem, in + (size_t)first * P.stride, n_here * P.stride);
        r = smem + (size_t)threadIdx.x * P.stride;
    } else r = in + (size_t)(first + threadIdx.x) * P.stride;
    if (threadIdx.x >= n_here) return;
    const size_t i = first + threadIdx.x;
    unsigned char *o = out + i * P.out_bytes;
    auto index = [&](int f) { return v2_index(r, P.type[f], P.offset[f]); };
    auto look = [&](int page, int f) { return v2_lookup(table, P.rows, page, index(f)); };
    // centre: fromHalfFloat(x | y | z)
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        uint16_t h;
        memcpy(&h, r + P.offset[PF_X + k], 2);
        const double c = spz_half(h);
        put_f32(o, 4 * k, f32_store(c));
        G.center[i * 3 + k] = c;
    }
    // scale: codeBook[scaling][scale_k] (0.01 when the file has none).  The writer tests `scale_0 !== undefined`: when the scale_0
    // index names no row all three scales are 0, otherwise each gets `|| 0` (a NaN table value included)
    const bool scale_read = P.type[PF_SCALE0] && v2_names_row(index(PF_SCALE0), P.rows);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        double s = 0.01;
        if (P.type[PF_SCALE0]) { s = scale_read ? look(V2_SCALING, PF_SCALE0 + k) : 0.0; if (s != s) s = 0.0; }
        put_f32(o, 12 + 4 * k, f32_store(s));
    }
    // rotation: Quaternion.set(re[rot_0], im[rot_1], im[rot_2], im[rot_3]) normalised by the parser, again by the writer; stored x, y, z, w
    double qx = look(V2_ROT_RE, PF_ROT0), qy = look(V2_ROT_IM, PF_ROT1), qz = look(V2_ROT_IM, PF_ROT2), qw = look(V2_ROT_IM, PF_ROT3);
    quat_normalize(qx, qy, qz, qw);
    quat_normalize(qx, qy, qz, qw);
    put_f32(o, 24, f32_store(qx)); put_f32(o, 28, f32_store(qy)); put_f32(o, 32, f32_store(qz)); put_f32(o, 36, f32_store(qw));
    // colour: codeBook[features_dc][f_dc_k] else 0 (red/green/blue alias f_dc_*); alpha: codeBook[opacity][opacity] else 0; clamp(floor)
    uint32_t rgba = 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) rgba |= (P.type[PF_DC0] ? to_u8_floor(look(V2_DC, PF_DC0 + k)) : 0u) << (8 * k);
    if (P.type[PF_OPACITY]) rgba |= to_u8_floor(look(V2_OPACITY, PF_OPACITY)) << 24;
    *reinterpret_cast<uint32_t *>(o + 40) = rgba;
    // SH: degree-1 slot s from page features_rest_(s % 3), degree-2 slot 9 + s from features_rest_(3 + s % 5), at the fields
    // k_ply_to_level0 reads; `|| 0` at write time
    for (int s = 0; s < P.ncomp_out; ++s) {
        double v = 0.0;
        if (s < P.ncomp_read) {
            const int src = s < 9 ? (s % 3) + (int)P.sh_per_channel * (s / 3) : 3 + (s - 9) % 5 + (int)P.sh_per_channel * ((s - 9) / 5);
            v = look(s < 9 ? V2_REST0 + s % 3 : V2_REST3 + (s - 9) % 5, PF_REST0 + src);
        }
        G.sh[i * P.ncomp_out + s] = v;
        if (v != v || v == 0.0) v = 0.0;
        put_f32(o, 44 + 4 * s, f32_store(v));
    }
}

} // namespace gs
