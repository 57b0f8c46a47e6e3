// ray_kernels.cuh -- Raycaster.intersectSplatMesh (src/raycaster/Raycaster.js:36-165, Ray.js:26-113) on the GPU.
//   k_ray_setup    one thread (per sub-tree of a forest): toLocal = invert(fromLocal), the local ray    Raycaster.js:50-60
//   k_ray_nodes    one thread per SplatTree node: Ray.intersectBox                                      Ray.js:26-82
//   k_ray_leaves   one thread per leaf: reached = the leaf and every ancestor pass (castRayAtSplatTreeNode's recursion, :87-165)
//   k_ray_compact  one CTA: the reached leaves in depth-first order, and their count
//   k_ray_splats   one warp per reached leaf: the per-splat test (:111-154), the hit mapped back to world space (:62-66)
//   k_ray_keys     sort keys of the hits (traversal position, then the distance's two halves) for the engine's stable radix sort
//   k_ray_out      the nearest hits in order -> gs_ray_hit
// Every f64 step follows three.js (r160) operation order with explicit __dmul_rn / __dadd_rn / __ddiv_rn / __dsqrt_rn: JS numbers are
// doubles and JS never fuses.  Matrix helpers restate Matrix4.multiplyMatrices / invert / determinant / decompose / compose,
// Quaternion.setFromRotationMatrix, Vector3.applyMatrix4 / length / normalize.
#pragma once
#include "../../include/gsplat_b200.h"
#include "common.cuh"

namespace gs {

struct RayParams {
    double origin[3], dir[3];   // world ray
    double from_local[16];
    const double *xf;           // device f64[16 * GS_MAX_SCENES]: static mesh, each SplatScene's transform (identity when none)
    const uint32_t *scene_idx;  // device scene index per splat, or nullptr: every splat is scene 0
    uint32_t scenes;            // transforms k_ray_splats stages in shared memory: 1 without scene_idx, else GS_MAX_SCENES
    uint32_t visible;           // bit s: scene s is visible (Raycaster.js:112-114)
    int ellipsoid, dynamic;
    // a forest (one sub-tree per scene of a dynamic mesh): sub-tree s casts with from_local = sub_from_local[16 s]; its leaves and
    // nodes are the ranges [sub_leaf[s], sub_leaf[s + 1]) and [sub_node[s], sub_node[s + 1])                    Raycaster.js:49-82
    const double *sub_from_local;
    const uint32_t *sub_leaf, *sub_node;
    uint32_t sub_trees;
};
struct RaySetup {               // written by k_ray_setup, read by the other kernels
    double o[3], d[3];          // local ray
};
struct RayHit {                 // 64 B; pos = the splat's offset in the concatenated leaf index runs (depth-first traversal order)
    double o[3], n[3], dist;
    uint32_t splat, pos;
};

// Math.log10(byte) correctly rounded (the only libm call of the path; tests/test_raycast_oracle.py checks every entry against decimal)
__constant__ double kLog10Byte[256] = {
    -HUGE_VAL, 0x0.0p+0, 0x1.34413509f79ffp-2, 0x1.e8927964fd5fdp-2,
    0x1.34413509f79ffp-1, 0x1.65df657b04301p-1, 0x1.8e69d7377a7fep-1, 0x1.b0b0b0b78cc3fp-1,
    0x1.ce61cf8ef36fep-1, 0x1.e8927964fd5fdp-1, 0x1.0000000000000p+0, 0x1.0a98b6050c56fp+0,
    0x1.144538de3b27fp+0, 0x1.1d2b643bc124fp+0, 0x1.2568a59e4449fp+0, 0x1.2d145116c1700p+0,
    0x1.34413509f79ffp+0, 0x1.3afeb354b7d97p+0, 0x1.415989f4fc97ep+0, 0x1.475c655fbc110p+0,
    0x1.4d104d427de80p+0, 0x1.527cf6b505b9fp+0, 0x1.57a903478a3eep+0, 0x1.5c9a3209bf97fp+0,
    0x1.61558620b90fep+0, 0x1.65df657b04301p+0, 0x1.6a3bb17e3f0cfp+0, 0x1.6e6ddb0bbe07ep+0,
    0x1.7278f2e0c231fp+0, 0x1.765fb716b63eap+0, 0x1.7a249e593f57fp+0, 0x1.7dc9e145867e6p+0,
    0x1.8151824c7587fp+0, 0x1.84bd545e4baeep+0, 0x1.880f009735c17p+0, 0x1.8b480b19487a0p+0,
    0x1.8e69d7377a7fep+0, 0x1.9175ab0e66080p+0, 0x1.946cb2a239f90p+0, 0x1.97500295007cep+0,
    0x1.9a209a84fbcffp+0, 0x1.9cdf672020c58p+0, 0x1.9f8d43f783a1fp+0, 0x1.a22afd1bc30f5p+0,
    0x1.a4b9508a0826ep+0, 0x1.a738ef7000c7fp+0, 0x1.a9aa7f4c3d7ffp+0, 0x1.ac0e9aef8ba9ep+0,
    0x1.ae65d36336f7ep+0, 0x1.b0b0b0b78cc3fp+0, 0x1.b2efb2bd82180p+0, 0x1.b52351adf7316p+0,
    0x1.b74bfec0bcf4fp+0, 0x1.b96a24b537a43p+0, 0x1.bb7e284e3befep+0, 0x1.bd8868c28e6efp+0,
    0x1.bf8940234019fp+0, 0x1.c18103b8fb690p+0, 0x1.c37004593426ap+0, 0x1.c5568eb40f0eep+0,
    0x1.c734eb9bbd3ffp+0, 0x1.c90b6045f1bf0p+0, 0x1.cada2e8804666p+0, 0x1.cca1950e4511ep+0,
    0x1.ce61cf8ef36fep+0, 0x1.d01b16f9433cfp+0, 0x1.d1cda1a0c996ep+0, 0x1.d379a365a652ep+0,
    0x1.d51f4dd9b3a97p+0, 0x1.d6bed062feefep+0, 0x1.d858585bc6620p+0, 0x1.d9ec113032053p+0,
    0x1.db7a2479f867ep+0, 0x1.dd02ba1a1b464p+0, 0x1.de85f850e3f00p+0, 0x1.e00403d443880p+0,
    0x1.e17cffe4b7e10p+0, 0x1.e2f10e60d2b8ep+0, 0x1.e4604fd77e64ep+0, 0x1.e5cae3991896ep+0,
    0x1.e730e7c779b7fp+0, 0x1.e8927964fd5fdp+0, 0x1.e9efb4629ead8p+0, 0x1.eb48b3ad39ad9p+0,
    0x1.ec9d913a0189ep+0, 0x1.edee661239f17p+0, 0x1.ef3b4a5e40f75p+0, 0x1.f084556ff5969p+0,
    0x1.f1c99dcc860eep+0, 0x1.f30b3935b06a6p+0, 0x1.f4493cb27eaffp+0, 0x1.f583bc978786fp+0,
    0x1.f6bacc8ebb67fp+0, 0x1.f7ee7f9ec5d65p+0, 0x1.f91ee8320991dp+0, 0x1.fa4c181d3e291p+0,
    0x1.fb7620a5b4dfep+0, 0x1.fc9d12874a6cep+0, 0x1.fdc0fdfa0aabfp+0, 0x1.fee1f2b78b06dp+0,
    0x1.0000000000000p+1, 0x1.008d9a4f88fdbp+1, 0x1.0119cf783a8cbp+1, 0x1.01a4a67223daep+1,
    0x1.022e26019d6e7p+1, 0x1.02b654b943e90p+1, 0x1.033d38fbdac62p+1, 0x1.03c2d8fe186fcp+1,
    0x1.04473ac85cebfp+1, 0x1.04ca643854534p+1, 0x1.054c5b02862b7p+1, 0x1.05cd24b3d2b00p+1,
    0x1.064cc6b2df00fp+1, 0x1.06cb46417122bp+1, 0x1.0748a87dbca88p+1, 0x1.07c4f263a0d80p+1,
    0x1.084028cdd9075p+1, 0x1.08ba50771fea7p+1, 0x1.09336dfb467b7p+1, 0x1.09ab85d83f1dbp+1,
    0x1.0a229c6f1d93fp+1, 0x1.0a98b6050c56fp+1, 0x1.0b0dd6c437d38p+1, 0x1.0b8202bcb00ecp+1,
    0x1.0bf53de541273p+1, 0x1.0c678c1c43240p+1, 0x1.0cd8f128617cfp+1, 0x1.0d4970b95abebp+1,
    0x1.0db90e68b8abfp+1, 0x1.0e27cdba8133ap+1, 0x1.0e95b21de0928p+1, 0x1.0f02beedccef6p+1,
    0x1.0f6ef771a3bf7p+1, 0x1.0fda5eddc1398p+1, 0x1.1044f854121d7p+1, 0x1.10aec6e4a00ffp+1,
    0x1.1117cd8e18c8bp+1, 0x1.11800f3e504cap+1, 0x1.11e78ed2be6bfp+1, 0x1.124e4f18f7b84p+1,
    0x1.12b452cf22250p+1, 0x1.13199ca46580ep+1, 0x1.137e2f3957f69p+1, 0x1.13e20d2066bdfp+1,
    0x1.144538de3b27fp+1, 0x1.14a7b4ea1c2b5p+1, 0x1.150983ae4c972p+1, 0x1.156aa788660dfp+1,
    0x1.15cb22c9b0ec0p+1, 0x1.162af7b779372p+1, 0x1.168a288b60b80p+1, 0x1.16e8b773ae589p+1,
    0x1.1746a6939ae48p+1, 0x1.17a3f8039b44bp+1, 0x1.1800add1a8507p+1, 0x1.185cca01844b3p+1,
    0x1.18b84e8cfe267p+1, 0x1.19133d64329d5p+1, 0x1.196d986dcb3f7p+1, 0x1.19c761873b7e1p+1,
    0x1.1a209a84fbcffp+1, 0x1.1a794532c2fcfp+1, 0x1.1ad16353bda3ep+1, 0x1.1b28f6a2c40afp+1,
    0x1.1b8000d28e4acp+1, 0x1.1bd6838de6e37p+1, 0x1.1c2c8077dbcacp+1, 0x1.1c81f92bee00cp+1,
    0x1.1cd6ef3e3fb8fp+1, 0x1.1d2b643bc124fp+1, 0x1.1d7f59aa5beccp+1, 0x1.1dd2d1091d607p+1,
    0x1.1e25cbd05f6fap+1, 0x1.1e784b71f0701p+1, 0x1.1eca515939bf5p+1, 0x1.1f1bdeeb65490p+1,
    0x1.1f6cf58781fb7p+1, 0x1.1fbd9686a7337p+1, 0x1.200dc33c17293p+1, 0x1.205d7cf560662p+1,
    0x1.20acc4fa7e4bfp+1, 0x1.20fb9c8df8b56p+1, 0x1.214a04ed02b77p+1, 0x1.2197ff4f988b7p+1,
    0x1.21e58ce89ca7fp+1, 0x1.2232aee5f4100p+1, 0x1.227f6670a1df3p+1, 0x1.22cbb4ace2183p+1,
    0x1.23179aba43bcfp+1, 0x1.236319b3c234fp+1, 0x1.23ae32afde088p+1, 0x1.23f8e6c0b4f5bp+1,
    0x1.244336f41963fp+1, 0x1.248d2453a93c6p+1, 0x1.24d6afe4e42a7p+1, 0x1.251fdaa9414a7p+1,
    0x1.2568a59e4449fp+1, 0x1.25b111bd91fe9p+1, 0x1.25f91ffd04776p+1, 0x1.2640d14ebe8d1p+1,
    0x1.268826a13ef40p+1, 0x1.26cf20df72d57p+1, 0x1.2715c0f0c7f1bp+1, 0x1.275c07b93e505p+1,
    0x1.27a1f6197980bp+1, 0x1.27e78ceed16ecp+1, 0x1.282ccd1362ceep+1, 0x1.2871b75e1f23fp+1,
    0x1.28b64ca2dc627p+1, 0x1.28fa8db264340p+1, 0x1.293e7b5a82dcfp+1, 0x1.2982166615c83p+1,
    0x1.29c55f9d19ba1p+1, 0x1.2a0857c4b8ae9p+1, 0x1.2a4aff9f5763cp+1, 0x1.2a8d57eca293bp+1,
    0x1.2acf61699bdfep+1, 0x1.2b111cd0a6703p+1, 0x1.2b528ad993473p+1, 0x1.2b93ac39ad4f2p+1,
    0x1.2bd481a3c51f7p+1, 0x1.2c150bc83c7f3p+1, 0x1.2c554b5511a40p+1, 0x1.2c9540f5ea30ap+1,
    0x1.2cd4ed541df4fp+1, 0x1.2d145116c1700p+1, 0x1.2d536ce2b016bp+1, 0x1.2d92415a9660cp+1,
    0x1.2dd0cf1efb9c8p+1, 0x1.2e0f16ce4b8bdp+1, 0x1.2e4d1904dfcc0p+1, 0x1.2e8ad65d09087p+1,
    0x1.2ec84f6f17fb5p+1, 0x1.2f0584d1663c2p+1, 0x1.2f4277185ede7p+1, 0x1.2f7f26d686e0fp+1,
    0x1.2fbb949c856f7p+1, 0x1.2ff7c0f92bf77p+1, 0x1.3033ac797e11bp+1, 0x1.306f57a8b9411p+1,
    0x1.30aac3105c87fp+1, 0x1.30e5ef382fd56p+1, 0x1.3120dca64b4aep+1, 0x1.315b8bdf1e5bep+1,
    0x1.3195fd6576c77p+1, 0x1.31d031ba876e0p+1, 0x1.320a295def02cp+1, 0x1.3243e4cdbe9b0p+1,
    0x1.327d6486801b3p+1, 0x1.32b6a9033c82cp+1, 0x1.32efb2bd82180p+1, 0x1.3328822d6a743p+1,
    0x1.336117c9a070fp+1, 0x1.3399740765f77p+1, 0x1.33d1975a99b2bp+1, 0x1.34098235bca4bp+1,
};

__device__ __forceinline__ double js_len(double x, double y, double z) {   // Vector3.length
    return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
}
// Vector3.normalize = divideScalar(length() || 1): NaN and 0 are falsy in JS, so both divide by 1
__device__ __forceinline__ void js_normalize(double &x, double &y, double &z) {
    const double ln = js_len(x, y, z);
    const double s = __ddiv_rn(1.0, (ln == 0.0 || ln != ln) ? 1.0 : ln);
    x = __dmul_rn(x, s); y = __dmul_rn(y, s); z = __dmul_rn(z, s);
}
__device__ __forceinline__ void m4_apply(const double *e, double &x, double &y, double &z) {   // Vector3.applyMatrix4
    const double X = x, Y = y, Z = z;
    const double w = __ddiv_rn(1.0, __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e[3], X), __dmul_rn(e[7], Y)), __dmul_rn(e[11], Z)), e[15]));
    x = __dmul_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e[0], X), __dmul_rn(e[4], Y)), __dmul_rn(e[8], Z)), e[12]), w);
    y = __dmul_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e[1], X), __dmul_rn(e[5], Y)), __dmul_rn(e[9], Z)), e[13]), w);
    z = __dmul_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e[2], X), __dmul_rn(e[6], Y)), __dmul_rn(e[10], Z)), e[14]), w);
}
// Matrix4.multiplyMatrices(a, b): te[r + 4c] = a[r][0] b[0][c] + a[r][1] b[1][c] + a[r][2] b[2][c] + a[r][3] b[3][c], left to right
__device__ __forceinline__ void m4_mul(const double *a, const double *b, double *t) {
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int r = 0; r < 4; ++r)
            t[r + 4 * c] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(a[r], b[4 * c]), __dmul_rn(a[r + 4], b[4 * c + 1])), __dmul_rn(a[r + 8], b[4 * c + 2])),
                                     __dmul_rn(a[r + 12], b[4 * c + 3]));
}
__device__ __forceinline__ double m3(double a, double b, double c) { return __dmul_rn(__dmul_rn(a, b), c); }
// Matrix4.invert: cofactors in three's order; det === 0 -> the zero matrix
__device__ __forceinline__ void m4_invert(const double *te, double *o) {
    const double n11 = te[0], n21 = te[1], n31 = te[2], n41 = te[3], n12 = te[4], n22 = te[5], n32 = te[6], n42 = te[7];
    const double n13 = te[8], n23 = te[9], n33 = te[10], n43 = te[11], n14 = te[12], n24 = te[13], n34 = te[14], n44 = te[15];
    auto s6 = [](double a, double b, double c, double d, double e, double f) {   // a - b + c - d - e + f  (signs as written in each line)
        return __dadd_rn(__dsub_rn(__dsub_rn(__dadd_rn(__dsub_rn(a, b), c), d), e), f);
    };
    auto s6b = [](double a, double b, double c, double d, double e, double f) {  // a - b - c + d + e - f
        return __dsub_rn(__dadd_rn(__dadd_rn(__dsub_rn(__dsub_rn(a, b), c), d), e), f);
    };
    const double t11 = s6(m3(n23, n34, n42), m3(n24, n33, n42), m3(n24, n32, n43), m3(n22, n34, n43), m3(n23, n32, n44), m3(n22, n33, n44));
    const double t12 = s6b(m3(n14, n33, n42), m3(n13, n34, n42), m3(n14, n32, n43), m3(n12, n34, n43), m3(n13, n32, n44), m3(n12, n33, n44));
    const double t13 = s6(m3(n13, n24, n42), m3(n14, n23, n42), m3(n14, n22, n43), m3(n12, n24, n43), m3(n13, n22, n44), m3(n12, n23, n44));
    const double t14 = s6b(m3(n14, n23, n32), m3(n13, n24, n32), m3(n14, n22, n33), m3(n12, n24, n33), m3(n13, n22, n34), m3(n12, n23, n34));
    const double det = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(n11, t11), __dmul_rn(n21, t12)), __dmul_rn(n31, t13)), __dmul_rn(n41, t14));
    if (det == 0.0) {
#pragma unroll
        for (int k = 0; k < 16; ++k) o[k] = 0.0;
        return;
    }
    const double di = __ddiv_rn(1.0, det);
    o[0] = __dmul_rn(t11, di);
    o[1] = __dmul_rn(s6b(m3(n24, n33, n41), m3(n23, n34, n41), m3(n24, n31, n43), m3(n21, n34, n43), m3(n23, n31, n44), m3(n21, n33, n44)), di);
    o[2] = __dmul_rn(s6(m3(n22, n34, n41), m3(n24, n32, n41), m3(n24, n31, n42), m3(n21, n34, n42), m3(n22, n31, n44), m3(n21, n32, n44)), di);
    o[3] = __dmul_rn(s6b(m3(n23, n32, n41), m3(n22, n33, n41), m3(n23, n31, n42), m3(n21, n33, n42), m3(n22, n31, n43), m3(n21, n32, n43)), di);
    o[4] = __dmul_rn(t12, di);
    o[5] = __dmul_rn(s6(m3(n13, n34, n41), m3(n14, n33, n41), m3(n14, n31, n43), m3(n11, n34, n43), m3(n13, n31, n44), m3(n11, n33, n44)), di);
    o[6] = __dmul_rn(s6b(m3(n14, n32, n41), m3(n12, n34, n41), m3(n14, n31, n42), m3(n11, n34, n42), m3(n12, n31, n44), m3(n11, n32, n44)), di);
    o[7] = __dmul_rn(s6(m3(n12, n33, n41), m3(n13, n32, n41), m3(n13, n31, n42), m3(n11, n33, n42), m3(n12, n31, n43), m3(n11, n32, n43)), di);
    o[8] = __dmul_rn(t13, di);
    o[9] = __dmul_rn(s6b(m3(n14, n23, n41), m3(n13, n24, n41), m3(n14, n21, n43), m3(n11, n24, n43), m3(n13, n21, n44), m3(n11, n23, n44)), di);
    o[10] = __dmul_rn(s6(m3(n12, n24, n41), m3(n14, n22, n41), m3(n14, n21, n42), m3(n11, n24, n42), m3(n12, n21, n44), m3(n11, n22, n44)), di);
    o[11] = __dmul_rn(s6b(m3(n13, n22, n41), m3(n12, n23, n41), m3(n13, n21, n42), m3(n11, n23, n42), m3(n12, n21, n43), m3(n11, n22, n43)), di);
    o[12] = __dmul_rn(t14, di);
    o[13] = __dmul_rn(s6(m3(n13, n24, n31), m3(n14, n23, n31), m3(n14, n21, n33), m3(n11, n24, n33), m3(n13, n21, n34), m3(n11, n23, n34)), di);
    o[14] = __dmul_rn(s6b(m3(n14, n22, n31), m3(n12, n24, n31), m3(n14, n21, n32), m3(n11, n24, n32), m3(n12, n21, n34), m3(n11, n22, n34)), di);
    o[15] = __dmul_rn(s6(m3(n12, n23, n31), m3(n13, n22, n31), m3(n13, n21, n32), m3(n11, n23, n32), m3(n12, n21, n33), m3(n11, n22, n33)), di);
}
// Matrix4.determinant, three's grouping: n41 (...) + n42 (...) + n43 (...) + n44 (...)
__device__ __forceinline__ double m4_det(const double *te) {
    const double n11 = te[0], n12 = te[4], n13 = te[8], n14 = te[12], n21 = te[1], n22 = te[5], n23 = te[9], n24 = te[13];
    const double n31 = te[2], n32 = te[6], n33 = te[10], n34 = te[14], n41 = te[3], n42 = te[7], n43 = te[11], n44 = te[15];
    auto sum6 = [](double a, double b, double c, double d, double e, double f) {   // a + b + c + d + e + f, left to right (signs folded in)
        return __dadd_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dadd_rn(a, b), c), d), e), f);
    };
    const double g1 = sum6(m3(n14, n23, n32), -m3(n13, n24, n32), -m3(n14, n22, n33), m3(n12, n24, n33), m3(n13, n22, n34), -m3(n12, n23, n34));
    const double g2 = sum6(m3(n11, n23, n34), -m3(n11, n24, n33), m3(n14, n21, n33), -m3(n13, n21, n34), m3(n13, n24, n31), -m3(n14, n23, n31));
    const double g3 = sum6(m3(n11, n24, n32), -m3(n11, n22, n34), -m3(n14, n21, n32), m3(n12, n21, n34), m3(n14, n22, n31), -m3(n12, n24, n31));
    const double g4 = sum6(-m3(n13, n22, n31), -m3(n11, n23, n32), m3(n11, n22, n33), m3(n13, n21, n32), -m3(n12, n21, n33), m3(n12, n23, n31));
    return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(n41, g1), __dmul_rn(n42, g2)), __dmul_rn(n43, g3)), __dmul_rn(n44, g4));
}
__device__ __forceinline__ void m4_scale(double *t, double x, double y, double z) {   // Matrix4.makeScale
#pragma unroll
    for (int k = 0; k < 16; ++k) t[k] = 0.0;
    t[0] = x; t[5] = y; t[10] = z; t[15] = 1.0;
}
// Matrix4.makeRotationFromQuaternion = compose(0, q, (1, 1, 1)); the `* 1` of compose is exact and left out
__device__ __forceinline__ void m4_rotation(double *te, double x, double y, double z, double w) {
    const double x2 = __dadd_rn(x, x), y2 = __dadd_rn(y, y), z2 = __dadd_rn(z, z);
    const double xx = __dmul_rn(x, x2), xy = __dmul_rn(x, y2), xz = __dmul_rn(x, z2), yy = __dmul_rn(y, y2), yz = __dmul_rn(y, z2), zz = __dmul_rn(z, z2);
    const double wx = __dmul_rn(w, x2), wy = __dmul_rn(w, y2), wz = __dmul_rn(w, z2);
    te[0] = __dsub_rn(1.0, __dadd_rn(yy, zz)); te[1] = __dadd_rn(xy, wz); te[2] = __dsub_rn(xz, wy); te[3] = 0.0;
    te[4] = __dsub_rn(xy, wz); te[5] = __dsub_rn(1.0, __dadd_rn(xx, zz)); te[6] = __dadd_rn(yz, wx); te[7] = 0.0;
    te[8] = __dadd_rn(xz, wy); te[9] = __dsub_rn(yz, wx); te[10] = __dsub_rn(1.0, __dadd_rn(xx, yy)); te[11] = 0.0;
    te[12] = 0.0; te[13] = 0.0; te[14] = 0.0; te[15] = 1.0;
}
// Matrix4.decompose -> scale (sign of x from the determinant) and, when want_q, Quaternion.setFromRotationMatrix of the
// column-normalised matrix
__device__ __forceinline__ void m4_decompose(const double *te, double *s, double *q, bool want_q) {
    double sx = js_len(te[0], te[1], te[2]);
    const double sy = js_len(te[4], te[5], te[6]), sz = js_len(te[8], te[9], te[10]);
    if (m4_det(te) < 0.0) sx = -sx;
    s[0] = sx; s[1] = sy; s[2] = sz;
    if (!want_q) return;
    const double ix = __ddiv_rn(1.0, sx), iy = __ddiv_rn(1.0, sy), iz = __ddiv_rn(1.0, sz);
    const double m11 = __dmul_rn(te[0], ix), m21 = __dmul_rn(te[1], ix), m31 = __dmul_rn(te[2], ix);
    const double m12 = __dmul_rn(te[4], iy), m22 = __dmul_rn(te[5], iy), m32 = __dmul_rn(te[6], iy);
    const double m13 = __dmul_rn(te[8], iz), m23 = __dmul_rn(te[9], iz), m33 = __dmul_rn(te[10], iz);
    const double trace = __dadd_rn(__dadd_rn(m11, m22), m33);
    if (trace > 0.0) {
        const double r = __ddiv_rn(0.5, __dsqrt_rn(__dadd_rn(trace, 1.0)));
        q[3] = __ddiv_rn(0.25, r);
        q[0] = __dmul_rn(__dsub_rn(m32, m23), r); q[1] = __dmul_rn(__dsub_rn(m13, m31), r); q[2] = __dmul_rn(__dsub_rn(m21, m12), r);
    } else if (m11 > m22 && m11 > m33) {
        const double r = __dmul_rn(2.0, __dsqrt_rn(__dsub_rn(__dsub_rn(__dadd_rn(1.0, m11), m22), m33)));
        q[3] = __ddiv_rn(__dsub_rn(m32, m23), r); q[0] = __dmul_rn(0.25, r);
        q[1] = __ddiv_rn(__dadd_rn(m12, m21), r); q[2] = __ddiv_rn(__dadd_rn(m13, m31), r);
    } else if (m22 > m33) {
        const double r = __dmul_rn(2.0, __dsqrt_rn(__dsub_rn(__dsub_rn(__dadd_rn(1.0, m22), m11), m33)));
        q[3] = __ddiv_rn(__dsub_rn(m13, m31), r); q[0] = __ddiv_rn(__dadd_rn(m12, m21), r);
        q[1] = __dmul_rn(0.25, r); q[2] = __ddiv_rn(__dadd_rn(m23, m32), r);
    } else {
        const double r = __dmul_rn(2.0, __dsqrt_rn(__dsub_rn(__dsub_rn(__dadd_rn(1.0, m33), m11), m22)));
        q[3] = __ddiv_rn(__dsub_rn(m21, m12), r); q[0] = __ddiv_rn(__dadd_rn(m13, m31), r);
        q[1] = __ddiv_rn(__dadd_rn(m23, m32), r); q[2] = __dmul_rn(0.25, r);
    }
}
// Ray.intersectSphere (Ray.js:84-113): t = t0, or t1 when t0 < 0; no hit when t1 < 0.  Hit origin o + d t, normal (hit - c).normalize()
__device__ __forceinline__ bool ray_sphere(const double *o, const double *d, double cx, double cy, double cz, double radius, double *ho, double *hn) {
    const double vx = __dsub_rn(cx, o[0]), vy = __dsub_rn(cy, o[1]), vz = __dsub_rn(cz, o[2]);
    const double tca = __dadd_rn(__dadd_rn(__dmul_rn(vx, d[0]), __dmul_rn(vy, d[1])), __dmul_rn(vz, d[2]));
    const double tca2 = __dmul_rn(tca, tca);
    const double c2 = __dadd_rn(__dadd_rn(__dmul_rn(vx, vx), __dmul_rn(vy, vy)), __dmul_rn(vz, vz));
    const double diff = __dsub_rn(c2, tca2), r2 = __dmul_rn(radius, radius);
    if (diff > r2) return false;
    const double thc = __dsqrt_rn(__dsub_rn(r2, diff));
    const double t0 = __dsub_rn(tca, thc), t1 = __dadd_rn(tca, thc);
    if (t1 < 0.0) return false;
    const double t = t0 < 0.0 ? t1 : t0;
    ho[0] = __dadd_rn(o[0], __dmul_rn(d[0], t)); ho[1] = __dadd_rn(o[1], __dmul_rn(d[1], t)); ho[2] = __dadd_rn(o[2], __dmul_rn(d[2], t));
    hn[0] = __dsub_rn(ho[0], cx); hn[1] = __dsub_rn(ho[1], cy); hn[2] = __dsub_rn(ho[2], cz);
    js_normalize(hn[0], hn[1], hn[2]);
    return true;
}

// kForest: one thread per sub-tree, S[s] = sub-tree s's local ray
template <bool kForest>
__global__ void k_ray_setup(RayParams P, RaySetup *S) {
    double to_local[16];
    if (kForest) {
        if (threadIdx.x >= P.sub_trees) return;
        double fl[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) fl[k] = P.sub_from_local[16 * threadIdx.x + k];
        m4_invert(fl, to_local);
        S += threadIdx.x;
    } else {
        m4_invert(P.from_local, to_local);
    }
    double ox = P.origin[0], oy = P.origin[1], oz = P.origin[2];
    m4_apply(to_local, ox, oy, oz);
    double dx = __dadd_rn(P.origin[0], P.dir[0]), dy = __dadd_rn(P.origin[1], P.dir[1]), dz = __dadd_rn(P.origin[2], P.dir[2]);
    m4_apply(to_local, dx, dy, dz);
    dx = __dsub_rn(dx, ox); dy = __dsub_rn(dy, oy); dz = __dsub_rn(dz, oz);
    js_normalize(dx, dy, dz);
    S->o[0] = ox; S->o[1] = oy; S->o[2] = oz;
    S->d[0] = dx; S->d[1] = dy; S->d[2] = dz;
}

// Ray.boxContainsPoint: a NaN coordinate fails every comparison and so counts as inside
__device__ __forceinline__ bool box_contains(const double *mn, const double *mx, const double *p) {
    constexpr double eps = 0.0001;
    return !(p[0] < __dsub_rn(mn[0], eps) || p[0] > __dadd_rn(mx[0], eps) || p[1] < __dsub_rn(mn[1], eps) || p[1] > __dadd_rn(mx[1], eps) ||
             p[2] < __dsub_rn(mn[2], eps) || p[2] > __dadd_rn(mx[2], eps));
}
// kForest: node i is tested against the ray of its sub-tree (the range of i in sub_node[0..subs])
template <bool kForest>
__global__ void k_ray_nodes(const double *__restrict__ nmin, const double *__restrict__ nmax, uint32_t n, const RaySetup *__restrict__ S,
                            const uint32_t *__restrict__ sub_node, uint32_t subs, uint8_t *__restrict__ pass) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (kForest) S += range_of(sub_node, subs, i);
    const double mn[3] = {nmin[3 * i], nmin[3 * i + 1], nmin[3 * i + 2]}, mx[3] = {nmax[3 * i], nmax[3 * i + 1], nmax[3 * i + 2]};
    const double o[3] = {S->o[0], S->o[1], S->o[2]}, d[3] = {S->d[0], S->d[1], S->d[2]};
    bool hit = box_contains(mn, mx, o);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        if (hit || d[a] == 0.0) continue;
        const double mult = d[a] > 0.0 ? -1.0 : (d[a] < 0.0 ? 1.0 : __longlong_as_double(0x7ff8000000000000ll));   // -Math.sign(d)
        const double plane = d[a] < 0.0 ? mx[a] : mn[a];
        const double to_side = __dsub_rn(plane, o[a]);
        if (__dmul_rn(to_side, mult) < 0.0) {
            const int a1 = (a + 1) % 3, a2 = (a + 2) % 3;
            double p[3];
            p[a] = plane;
            p[a1] = __dadd_rn(__dmul_rn(__ddiv_rn(d[a1], d[a]), to_side), o[a1]);
            p[a2] = __dadd_rn(__dmul_rn(__ddiv_rn(d[a2], d[a]), to_side), o[a2]);
            hit = box_contains(mn, mx, p);
        }
    }
    pass[i] = hit;
}

__global__ void k_ray_leaves(const uint32_t *__restrict__ leaf_node, const int32_t *__restrict__ parent, const uint8_t *__restrict__ pass,
                             uint32_t m, uint32_t *__restrict__ reached) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    int32_t v = (int32_t)leaf_node[i];
    bool ok = true;
    while (v >= 0) { ok = ok && pass[v]; v = parent[v]; }
    reached[i] = ok;
}

constexpr int kRayCompactThreads = 1024;
// counts[0] = reached leaves; list = their numbers in ascending (= depth-first) order
__global__ void __launch_bounds__(kRayCompactThreads) k_ray_compact(const uint32_t *__restrict__ reached, uint32_t m, uint32_t *__restrict__ list,
                                                                     uint32_t *__restrict__ counts) {
    __shared__ uint32_t s_scan[40];
    uint32_t carry = 0;
    for (uint32_t base = 0; base < m; base += kRayCompactThreads) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t f = i < m ? reached[i] : 0u;
        uint32_t total;
        const uint32_t ex = block_exclusive_scan<kRayCompactThreads>(f, s_scan, total);
        if (f) list[carry + ex] = i;
        carry += total;
    }
    if (threadIdx.x == 0) { counts[0] = carry; counts[1] = 0; }
}

constexpr int kRaySplatThreads = 128;
// kForest: the leaf's sub-tree s (the range of the leaf in P.sub_leaf) gives the local ray S[s] and from_local P.sub_from_local[16 s]
template <bool kForest>
__global__ void __launch_bounds__(kRaySplatThreads)
k_ray_splats(const uint32_t *__restrict__ list, const uint32_t *__restrict__ counts, const uint32_t *__restrict__ offsets, const uint32_t *__restrict__ indexes,
             const gs_ray_record *__restrict__ recs, RayParams P, const RaySetup *__restrict__ S, RayHit *__restrict__ hits, uint32_t *__restrict__ hit_count) {
    const uint32_t nreached = counts[0];
    const uint32_t lane = threadIdx.x & 31, warps = gridDim.x * (kRaySplatThreads / 32);
    double o[3] = {S->o[0], S->o[1], S->o[2]}, d[3] = {S->d[0], S->d[1], S->d[2]};
    __shared__ double s_xf[16 * GS_MAX_SCENES];   // the scene transforms, read by every splat
    __shared__ double s_fl[kForest ? 16 * GS_MAX_SCENES : 1];   // forest: every sub-tree's from_local
    for (uint32_t k = threadIdx.x; k < 16 * P.scenes; k += kRaySplatThreads) s_xf[k] = P.xf[k];
    if (kForest)
        for (uint32_t k = threadIdx.x; k < 16 * P.sub_trees; k += kRaySplatThreads) s_fl[k] = P.sub_from_local[k];
    __syncthreads();
    const double *fl = P.from_local;
    for (uint32_t w = blockIdx.x * (kRaySplatThreads / 32) + (threadIdx.x >> 5); w < nreached; w += warps) {
        const uint32_t leaf = list[w], lo = offsets[leaf], hi = offsets[leaf + 1];
        if (kForest) {
            const uint32_t sub = range_of(P.sub_leaf, P.sub_trees, leaf);
            const RaySetup &T = S[sub];
            o[0] = T.o[0]; o[1] = T.o[1]; o[2] = T.o[2];
            d[0] = T.d[0]; d[1] = T.d[1]; d[2] = T.d[2];
            fl = s_fl + 16 * sub;
        }
        for (uint32_t pos = lo + lane; pos < hi; pos += 32) {
            const uint32_t idx = indexes[pos];
            const uint32_t sc = P.scene_idx ? P.scene_idx[idx] & (GS_MAX_SCENES - 1) : 0u;
            if (!((P.visible >> sc) & 1u)) continue;
            const double *xf = s_xf + 16 * sc;
            const gs_ray_record r = recs[idx];
            double c[3] = {r.center[0], r.center[1], r.center[2]};
            double s[3] = {(double)r.scale[0], (double)r.scale[1], (double)r.scale[2]};
            double q[4] = {(double)r.rotation[0], (double)r.rotation[1], (double)r.rotation[2], (double)r.rotation[3]};
            if (!P.dynamic) {   // static mesh: getSplatCenter(.., scene.transform); decompose(makeScale(s) * R(q) * T)   SplatBuffer.js:242, 276-280
                m4_apply(xf, c[0], c[1], c[2]);
                double A[16], B[16], M[16];
                m4_scale(A, s[0], s[1], s[2]);
                m4_rotation(B, q[0], q[1], q[2], q[3]);
                m4_mul(A, B, M);
                m4_mul(M, xf, A);
                m4_decompose(A, s, q, P.ellipsoid);
            }
            constexpr double kScaleEps = 0.0000001;
            if (s[0] <= kScaleEps || s[1] <= kScaleEps || s[2] <= kScaleEps) continue;
            double ho[3], hn[3];
            if (!P.ellipsoid) {
                const double radius = __ddiv_rn(__dadd_rn(__dadd_rn(s[0], s[1]), s[2]), 3.0);
                if (!ray_sphere(o, d, c[0], c[1], c[2], radius, ho, hn)) continue;
            } else {
                const double u = __dmul_rn(kLog10Byte[r.alpha], 2.0);
                double U[16], R[16], F[16], Inv[16];
                m4_scale(U, u, u, u);
                m4_rotation(R, q[0], q[1], q[2], q[3]);
                m4_mul(U, R, Inv);
                m4_scale(U, s[0], s[1], s[2]);
                m4_mul(Inv, U, F);
                m4_invert(F, Inv);
                double to[3] = {__dsub_rn(o[0], c[0]), __dsub_rn(o[1], c[1]), __dsub_rn(o[2], c[2])};
                m4_apply(Inv, to[0], to[1], to[2]);
                double td[3] = {__dsub_rn(__dadd_rn(o[0], d[0]), c[0]), __dsub_rn(__dadd_rn(o[1], d[1]), c[1]), __dsub_rn(__dadd_rn(o[2], d[2]), c[2])};
                m4_apply(Inv, td[0], td[1], td[2]);
                td[0] = __dsub_rn(td[0], to[0]); td[1] = __dsub_rn(td[1], to[1]); td[2] = __dsub_rn(td[2], to[2]);
                js_normalize(td[0], td[1], td[2]);
                if (!ray_sphere(to, td, 0.0, 0.0, 0.0, 1.0, ho, hn)) continue;
                m4_apply(F, ho[0], ho[1], ho[2]);
                ho[0] = __dadd_rn(ho[0], c[0]); ho[1] = __dadd_rn(ho[1], c[1]); ho[2] = __dadd_rn(ho[2], c[2]);
            }
            // back to world space (Raycaster.js:62-66)
            m4_apply(fl, ho[0], ho[1], ho[2]);
            m4_apply(fl, hn[0], hn[1], hn[2]);
            js_normalize(hn[0], hn[1], hn[2]);
            RayHit h;
            h.o[0] = ho[0]; h.o[1] = ho[1]; h.o[2] = ho[2];
            h.n[0] = hn[0]; h.n[1] = hn[1]; h.n[2] = hn[2];
            h.dist = js_len(__dsub_rn(ho[0], P.origin[0]), __dsub_rn(ho[1], P.origin[1]), __dsub_rn(ho[2], P.origin[2]));
            h.splat = idx; h.pos = pos;
            hits[atomicAdd(hit_count, 1u)] = h;
        }
    }
}

// Keys for the stable LSD radix sort by (distance, traversal position): the position, then the distance's bits 0-23, 24-47 and 48-63
// (pieces below 2^32 - 1, which the radix kernels reserve for tail slots).  A distance is >= 0 or NaN: non-negative doubles order like
// their bits, and every NaN becomes 0x7ff0000000000001, just above +inf.
constexpr int kRayKeyBits[4] = {0, 24, 24, 16};   // [0]: the position's bits, set per call
__global__ void k_ray_keys(const RayHit *__restrict__ hits, const uint32_t *__restrict__ perm, uint32_t n, int which, uint32_t *__restrict__ keys,
                           uint32_t *__restrict__ vals) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t v = perm ? perm[i] : i;
    const RayHit &h = hits[v];
    const unsigned long long bits = h.dist != h.dist ? 0x7ff0000000000001ull : (unsigned long long)__double_as_longlong(h.dist);
    keys[i] = which == 0 ? h.pos : (uint32_t)((bits >> (24 * (which - 1))) & 0xffffffull);
    vals[i] = v;
}

__global__ void k_ray_out(const RayHit *__restrict__ hits, const uint32_t *__restrict__ perm, uint32_t n, gs_ray_hit *__restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const RayHit &h = hits[perm ? perm[i] : i];
    gs_ray_hit g;
    g.origin[0] = h.o[0]; g.origin[1] = h.o[1]; g.origin[2] = h.o[2];
    g.normal[0] = h.n[0]; g.normal[1] = h.n[1]; g.normal[2] = h.n[2];
    g.distance = h.dist; g.splat_index = h.splat; g.reserved = 0;
    out[i] = g;
}

} // namespace gs
