// ppg_device.cuh -- device-side building blocks of the H100 guided path tracer.
//
// Everything here is net-new sm_90a code; the *behaviour* follows the reference
// integrator mitsuba/src/integrators/path/guided_path.cpp ("GP") and the Mitsuba
// services it calls -- each function cites the lines it has to agree with.
// No tensor cores on this path (no dense contraction anywhere); the work is
// gather/scatter + fp32 ALU, so the rules that matter are coalesced float4 state
// traffic, shared-memory staging of the hot read-only data, and warp-aggregated atomics.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include "ppg_scene_layout.h"     // SceneView, EnvLight, Camera: the packed scene

namespace ppg {

#define PPG_PI 3.14159265358979323846f            // M_PI, single-precision build (core/constants.h:63,80)
#define PPG_INV_PI 0.31830988618379067154f
#define PPG_EPSILON 1e-4f                          // core/constants.h:28

// ------------------------------------------------------------------ float3 helpers
__device__ __forceinline__ float3 f3(float x, float y, float z) { return make_float3(x, y, z); }
__device__ __forceinline__ float3 operator+(float3 a, float3 b) { return f3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ float3 operator-(float3 a, float3 b) { return f3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ float3 operator*(float3 a, float s) { return f3(a.x * s, a.y * s, a.z * s); }
__device__ __forceinline__ float3 operator*(float3 a, float3 b) { return f3(a.x * b.x, a.y * b.y, a.z * b.z); }
__device__ __forceinline__ float3 operator-(float3 a) { return f3(-a.x, -a.y, -a.z); }
__device__ __forceinline__ float dot(float3 a, float3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ float3 cross(float3 a, float3 b) { return f3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
__device__ __forceinline__ float3 normalize(float3 a) { return a * (1.0f / sqrtf(dot(a, a))); }   // TVector3::operator/ multiplies by the reciprocal
__device__ __forceinline__ bool is_zero(float3 a) { return a.x == 0.f && a.y == 0.f && a.z == 0.f; }
__device__ __forceinline__ bool is_valid(float3 a) {   // Spectrum::isValid: finite and non-negative
    return isfinite(a.x) && isfinite(a.y) && isfinite(a.z) && a.x >= 0.f && a.y >= 0.f && a.z >= 0.f;
}
__device__ __forceinline__ float max3(float3 a) { return fmaxf(fmaxf(a.x, a.y), a.z); }
__device__ __forceinline__ float comp(float3 a, int i) { return i == 0 ? a.x : (i == 1 ? a.y : a.z); }
// sincosf of an angle the caller bounds (|x| <= 2 pi, or NaN): the same result, without sincosf's large-argument reduction
// (|x| >= 105615), whose scratch array would give every thread of the kernel a local-memory frame
__device__ __forceinline__ void sincosf_bounded(float x, float *s, float *c) {
#ifdef __CUDA_ARCH__
    __builtin_assume(!(fabsf(x) >= 105615.0f));
#endif
    sincosf(x, s, c);
}

// ------------------------------------------------------------------ PCG32 path sampler
// One stream per path, keyed by (seed, global sample index); numbers are consumed in the
// reference's order (SURVEY A.1).  Must match oracle/ppg_cpu_tracer.h bit for bit.
__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}
struct Pcg32 {
    uint64_t state, inc;
    __device__ __forceinline__ uint32_t nextU32() {
        const uint64_t old = state;
        state = old * 6364136223846793005ull + inc;
        const uint32_t xs = (uint32_t) (((old >> 18u) ^ old) >> 27u);
        const uint32_t rot = (uint32_t) (old >> 59u);
        return __funnelshift_r(xs, xs, rot);
    }
    __device__ __forceinline__ float next1D() { return (float) (nextU32() >> 8) * (1.0f / 16777216.0f); }
    __device__ __forceinline__ void seed(uint64_t initstate, uint64_t initseq) {
        state = 0; inc = (initseq << 1) | 1u;
        nextU32(); state += initstate; nextU32();
    }
};
__device__ __forceinline__ void seed_path_rng(Pcg32 &r, uint64_t seed, uint64_t sampleIndex) {
    r.seed(splitmix64(seed ^ splitmix64(sampleIndex)), sampleIndex);
}
__device__ __forceinline__ void seed_vertex_rng(Pcg32 &r, uint64_t seed, uint64_t sampleIndex, uint32_t ordinal) {
    r.seed(splitmix64((seed + 0x5851F42D4C957F2Dull) ^ splitmix64(sampleIndex * 64 + ordinal)), sampleIndex * 64 + ordinal);
}

#define PPG_ENV_EMITTER (-2)    // "dRec.object is the environment emitter" in the emitter-pdf queries

struct Hit { float t, u, v; uint32_t tri; uint32_t prim; };

// Scene access.  Small scenes are staged into dynamic shared memory; the accessor indexes the extern __shared__ symbol
// directly so that the compiler KNOWS the address space (a generic pointer that may hold either a shared or a global
// address was once compiled to LDG and faulted).  SMEM == false reads HBM through the read-only path.
extern __shared__ float4 ppg_scene_smem[];
template <bool SMEM> struct SceneAccess {
    static constexpr bool kStaged = SMEM;
    const SceneView &g;
    uint32_t oGeom, oMeta, oBvh, oBsdf, oRadiance, oGroups;      // float4 offsets of the staged sections (accel at 0)
    __device__ __forceinline__ SceneAccess(const SceneView &v) : g(v) {
        oGeom = 3 * v.nTris; oMeta = oGeom + 6 * v.nTris; oBvh = oMeta + v.nTris; oBsdf = oBvh + 2 * v.nBvhNodes;
        oRadiance = oBsdf + PPG_BSDF_F4 * v.nBsdfs; oGroups = oRadiance + v.nEmitters;
    }
    __device__ __forceinline__ float4 accel(uint32_t i) const { return SMEM ? ppg_scene_smem[i] : __ldg(&g.accel[i]); }
    __device__ __forceinline__ float4 geom(uint32_t i) const { return SMEM ? ppg_scene_smem[oGeom + i] : __ldg(&g.geom[i]); }
    __device__ __forceinline__ int4 meta(uint32_t i) const {
        if (SMEM) { const float4 m = ppg_scene_smem[oMeta + i]; return make_int4(__float_as_int(m.x), __float_as_int(m.y), __float_as_int(m.z), __float_as_int(m.w)); }
        return __ldg(&g.meta[i]);
    }
    __device__ __forceinline__ float4 bvh(uint32_t i) const { return SMEM ? ppg_scene_smem[oBvh + i] : __ldg(&g.bvh[i]); }
    __device__ __forceinline__ float4 bsdf(uint32_t i) const { return SMEM ? ppg_scene_smem[oBsdf + i] : __ldg(&g.bsdf[i]); }
    __device__ __forceinline__ float4 radiance(uint32_t i) const { return SMEM ? ppg_scene_smem[oRadiance + i] : __ldg(&g.radiance[i]); }
    __device__ __forceinline__ float4 groups(uint32_t i) const { return SMEM ? ppg_scene_smem[oGroups + i] : __ldg(&g.groups[i]); }
    // block-cooperative staging (call once, all threads): accel | geom | meta | bvh | bsdf | radiance | groups
    __device__ __forceinline__ void stage() const {
        if (!SMEM) return;
        auto copy = [&](uint32_t off, const float4 *src, uint32_t n) { for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) ppg_scene_smem[off + i] = src[i]; };
        copy(0, g.accel, 3 * g.nTris); copy(oGeom, g.geom, 6 * g.nTris); copy(oMeta, reinterpret_cast<const float4 *>(g.meta), g.nTris);
        copy(oBvh, g.bvh, 2 * g.nBvhNodes); copy(oBsdf, g.bsdf, PPG_BSDF_F4 * g.nBsdfs); copy(oRadiance, g.radiance, g.nEmitters); copy(oGroups, g.groups, 2 * g.nGroups);
        __syncthreads();
    }
};

__device__ __forceinline__ bool tri_intersect(const float4 A, const float4 B, const float4 C, float3 o, float3 d, float mint, float maxt,
                                              float &u, float &v, float &t) {
    const int k = __float_as_int(A.w);
    float o_u, o_v, o_k, d_u, d_v, d_k;
    if (k == 0) { o_u = o.y; o_v = o.z; o_k = o.x; d_u = d.y; d_v = d.z; d_k = d.x; }
    else if (k == 1) { o_u = o.z; o_v = o.x; o_k = o.y; d_u = d.z; d_v = d.x; d_k = d.y; }
    else if (k == 2) { o_u = o.x; o_v = o.y; o_k = o.z; d_u = d.x; d_v = d.y; d_k = d.z; }
    else return false;
    t = (A.z - o_u * A.x - o_v * A.y - o_k) / (d_u * A.x + d_v * A.y + d_k);
    if (!(t >= mint && t <= maxt)) return false;
    const float hu = o_u + t * d_u - B.x;
    const float hv = o_v + t * d_v - B.y;
    u = hv * B.z + hu * B.w;
    v = hu * C.x + hv * C.y;
    return u >= 0.f && v >= 0.f && u + v <= 1.0f;
}

// exact Wald test (triaccel.h:95-158) of every triangle of coplanar group q, ray components already permuted for the group's axis
template <class Acc>
__device__ __forceinline__ void tri_group_exact(const Acc &A_, uint32_t q, float o_u, float o_v, float o_k, float d_u, float d_v, float d_k,
                                                float mint, float maxt, Hit &hit) {
    const uint32_t fc = __float_as_uint(A_.groups(2 * q).w), last = (fc & 0xffffu) + (fc >> 16);
    for (uint32_t i = fc & 0xffffu; i < last; ++i) {
        const float4 A = A_.accel(3 * i), B = A_.accel(3 * i + 1), C = A_.accel(3 * i + 2);
        const float t = (A.z - o_u * A.x - o_v * A.y - o_k) / (d_u * A.x + d_v * A.y + d_k);
        if (t >= mint && t <= maxt) {
            const float hu = o_u + t * d_u - B.x, hv = o_v + t * d_v - B.y;
            const float u = hv * B.z + hu * B.w, v = hu * C.x + hv * C.y;
            if (u >= 0.f && v >= 0.f && u + v <= 1.0f) {
                const uint32_t prim = __float_as_uint(C.z);
                if (t < hit.t || (t == hit.t && prim < hit.prim)) { hit.t = t; hit.u = u; hit.v = v; hit.prim = prim; hit.tri = i; }
            }
        }
    }
}

// Sphere::rayIntersect (src/shapes/sphere.cpp:163-187) with solveQuadraticDouble (src/libcore/util.cpp:487-525): double precision like the reference
__device__ __forceinline__ bool sphere_intersect(float4 cr, float3 ro, float3 rd, float mint, float maxt, float &t) {
    const double ox = (double) ro.x - (double) cr.x, oy = (double) ro.y - (double) cr.y, oz = (double) ro.z - (double) cr.z;
    const double dx = rd.x, dy = rd.y, dz = rd.z;
    const double A = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
    const double B = __dmul_rn(2.0, __dadd_rn(__dadd_rn(__dmul_rn(ox, dx), __dmul_rn(oy, dy)), __dmul_rn(oz, dz)));
    const double C = __dsub_rn(__dadd_rn(__dadd_rn(__dmul_rn(ox, ox), __dmul_rn(oy, oy)), __dmul_rn(oz, oz)), (double) (cr.w * cr.w));
    double nearT, farT;
    if (A == 0.0) { if (B != 0.0) nearT = farT = -C / B; else return false; }
    else {
        const double discrim = __dsub_rn(__dmul_rn(B, B), __dmul_rn(__dmul_rn(4.0, A), C));
        if (discrim < 0.0) return false;
        const double sqrtDiscrim = sqrt(discrim);
        const double temp = B < 0.0 ? __dmul_rn(-0.5, __dsub_rn(B, sqrtDiscrim)) : __dmul_rn(-0.5, __dadd_rn(B, sqrtDiscrim));
        nearT = temp / A; farT = C / temp;
        if (nearT > farT) { const double s = nearT; nearT = farT; farT = s; }
    }
    if (!(nearT <= (double) maxt && farT >= (double) mint)) return false;
    if (nearT < (double) mint) { if (farT > (double) maxt) return false; t = (float) farT; }
    else t = (float) nearT;
    return true;
}
// Ray / box test of the BVH walks: entry distance in tEntry; `tmax` = min(maxt, nearest hit so far).
// fmaxf / fminf drop NaN operands (0 * inf when the ray lies in a box plane); widening once after the reductions equals widening every axis.
// The widening is multiplicative: `x -+ |x| * 1e-6` is inf - inf = NaN for an infinite bound, which fmaxf / fminf then DROP -- a ray with an
// exactly zero direction component was never culled on that axis and walked ~450 000 nodes of KITCHEN: 300 ms for one lane.
__device__ __forceinline__ bool bvh_slab(float3 o, float3 inv, float mint, float tmax, const float4 n0, const float4 n1, float &tEntry) {
    float ta = (n0.x - o.x) * inv.x, tb = (n1.x - o.x) * inv.x; if (ta > tb) { const float s_ = ta; ta = tb; tb = s_; }
    float nearMax = fmaxf(__int_as_float(0xff800000), ta), farMin = fminf(__int_as_float(0x7f800000), tb);
    ta = (n0.y - o.y) * inv.y; tb = (n1.y - o.y) * inv.y; if (ta > tb) { const float s_ = ta; ta = tb; tb = s_; }
    nearMax = fmaxf(nearMax, ta); farMin = fminf(farMin, tb);
    ta = (n0.z - o.z) * inv.z; tb = (n1.z - o.z) * inv.z; if (ta > tb) { const float s_ = ta; ta = tb; tb = s_; }
    nearMax = fmaxf(nearMax, ta); farMin = fminf(farMin, tb);
    const float t0 = fmaxf(mint, nearMax * (nearMax > 0.f ? 1.0f - 1e-6f : 1.0f + 1e-6f)), t1 = fminf(tmax, farMin * (farMin > 0.f ? 1.0f + 1e-6f : 1.0f - 1e-6f));
    tEntry = t0;
    return t0 <= t1;
}
// Not inlined: the walk's two stacks and its registers stay out of the callers' frames (the tiny-scene path of the bounce
// kernel never calls it and keeps its register allocation).  Arguments and result are values: an object whose address is passed to
// a call that is not inlined has to live in the caller's local memory.  Only the HBM variants walk (staged scenes have coplanar groups).
static __device__ __noinline__ Hit bvh_walk(const float4 *__restrict__ accel, const float4 *__restrict__ bvh, float3 o, float3 d, float mint, float maxt) {
    Hit hit; hit.t = __int_as_float(0x7f800000); hit.u = hit.v = 0.f; hit.prim = 0xFFFFFFFFu; hit.tri = 0;
    // BVH walk, near child first.  A node is 2 float4 {min.xyz, bits(left)}, {max.xyz, bits(count)}; siblings are adjacent, so one
    // 64-byte fetch brings both children's boxes.  The far child is pushed with its entry distance and skipped on pop when
    // a closer hit has been found since.  The slab test is widened by 1 ulp-ish factors so that flat boxes and NaNs (0 * inf)
    // never cull; results do not depend on the visiting order (ties on t go to the lower original triangle index).
    const float3 inv = f3(1.0f / d.x, 1.0f / d.y, 1.0f / d.z);
    auto slab = [&](const float4 n0, const float4 n1, float &tEntry) -> bool { return bvh_slab(o, inv, mint, fminf(maxt, hit.t), n0, n1, tEntry); };
    auto node = [&](uint32_t i) { return __ldg(&bvh[i]); };
    auto tri = [&](uint32_t i) { return __ldg(&accel[i]); };
    uint32_t stackN[PPG_BVH_STACK]; float stackT[PPG_BVH_STACK]; int sp = 0;
    uint32_t left, count;      // the current node: children left, left+1 (count == 0) or leaf slots [left, left+count)
    {
        const float4 r0 = node(0), r1 = node(1);
        float te;
        if (!slab(r0, r1, te)) return hit;
        left = __float_as_uint(r0.w); count = __float_as_uint(r1.w);
    }
    auto pop = [&]() -> bool {
        while (sp > 0) {
            --sp;
            if (stackT[sp] <= hit.t) { left = stackN[sp] & 0x0fffffffu; count = stackN[sp] >> 28; return true; }
        }
        return false;
    };
    // "while-while" (Aila & Laine): every lane first descends inner nodes until it HOLDS a leaf (or is done); the warp reconverges
    // behind that loop, so the triangle tests of all lanes run together instead of one lane's leaf serialising against the other
    // lanes' box tests in every iteration (ncu, KITCHEN: 3.7 of 32 lanes in the box test, 1.5 in the triangle test before).
    bool done = false;
    for (;;) {
        while (count == 0u && !done) {
            const float4 a0 = node(2 * left), a1 = node(2 * left + 1), b0 = node(2 * left + 2), b1 = node(2 * left + 3);
            float ta, tb;
            const bool ha = slab(a0, a1, ta), hb = slab(b0, b1, tb);
            if (ha && hb) {
                const bool aFirst = ta <= tb;
                const float4 f0 = aFirst ? b0 : a0, f1 = aFirst ? b1 : a1, n0 = aFirst ? a0 : b0, n1 = aFirst ? a1 : b1;
                stackN[sp] = __float_as_uint(f0.w) | (__float_as_uint(f1.w) << 28); stackT[sp] = aFirst ? tb : ta; ++sp;
                left = __float_as_uint(n0.w); count = __float_as_uint(n1.w);
            } else if (ha) { left = __float_as_uint(a0.w); count = __float_as_uint(a1.w); }
            else if (hb) { left = __float_as_uint(b0.w); count = __float_as_uint(b1.w); }
            else done = !pop();
        }
        if (done) break;
        for (uint32_t i = left; i < left + count; ++i) {
            const float4 A = tri(3 * i), B = tri(3 * i + 1), C = tri(3 * i + 2);
            float u, v, t;
            if (tri_intersect(A, B, C, o, d, mint, maxt, u, v, t)) {
                const uint32_t prim = __float_as_uint(C.z);
                if (t < hit.t || (t == hit.t && prim < hit.prim)) { hit.t = t; hit.u = u; hit.v = v; hit.prim = prim; hit.tri = i; }
            }
        }
        if (!pop()) break;
    }
    return hit;
}
template <class Acc> __device__ __forceinline__ bool tri_scene_intersect(const Acc &A_, float3 o, float3 d, float mint, float maxt, Hit &hit);

// Nearest hit in [mint, maxt]; ties on t go to the lower ORIGINAL triangle index so that the
// result does not depend on the traversal order (same rule as the oracle).  Spheres are tested after the triangles.
// SPHERES == false: the scene holds triangles only (host-checked; the sphere code compiles away).
template <bool SPHERES, class Acc>
__device__ __forceinline__ bool bvh_intersect(const Acc &A_, float3 o, float3 d, float mint, float maxt, Hit &hit) {
    bool found = tri_scene_intersect(A_, o, d, mint, maxt, hit);
    if (!SPHERES) return found;
    const SceneView &sc = A_.g;
    for (uint32_t k = 0; k < sc.nSpheres; ++k) {
        float t;
        if (sphere_intersect(__ldg(&sc.spheres[2 * k]), o, d, mint, maxt, t) && t < hit.t) { hit.t = t; hit.u = hit.v = 0.f; hit.prim = PPG_SPHERE_BIT | k; hit.tri = 0; found = true; }
    }
    return found;
}
template <class Acc>
__device__ __forceinline__ bool tri_scene_intersect(const Acc &A_, float3 o, float3 d, float mint, float maxt, Hit &hit) {
    const SceneView &sc = A_.g;
    hit.t = __int_as_float(0x7f800000); hit.prim = 0xFFFFFFFFu; hit.tri = 0;
    if (sc.nTris == 0u) return false;
    if (Acc::kStaged || sc.nGroups != 0u) {      // host sets nGroups only for tiny scenes (<= PPG_BRUTE_FORCE_TRIS triangles in <= 32 coplanar groups), and stages only those
        // Tiny scenes (CBOX: 36 triangles in 18 coplanar groups, staged in shared memory).  A BVH walk makes every lane
        // of a warp reach its leaves at different times (measured: 2.5 of 32 lanes active in the triangle test), so
        // instead all lanes visit every coplanar group in lock step (shared-memory broadcasts; groups are ordered by
        // projection axis k so that the component selection is a uniform branch).  Per group a cheap conservative
        // filter -- approximate plane distance, hit point against the group's padded bounding rectangle -- rejects
        // clear misses; only the triangles of surviving groups (1-2 per ray) run the exact reference test with its
        // IEEE division, so the hit set is identical to testing every triangle exactly.
        // Pass 1 (converged): filter every group, remember the survivors in a bit mask (<= 32 groups).  Pass 2: every lane pops its candidates one at a time, so the expensive exact
        // tests run with most lanes active instead of being scattered over the 18 filter iterations (measured: 3.2 of
        // 32 lanes active and 36 % of all warp instructions when the exact test sat inside the filter loop).
        const float tlo = mint * (1.0f - 1e-4f), thi = maxt * (1.0f + 1e-4f);
        uint32_t cand = 0, nearQ = 0xFFFFFFFFu; float nearT = __int_as_float(0x7f800000);
#pragma unroll 1
        for (int g = 0; g < 3; ++g) {
            float o_u, o_v, o_k, d_u, d_v, d_k;
            if (g == 0) { o_u = o.y; o_v = o.z; o_k = o.x; d_u = d.y; d_v = d.z; d_k = d.x; }
            else if (g == 1) { o_u = o.z; o_v = o.x; o_k = o.y; d_u = d.z; d_v = d.x; d_k = d.y; }
            else { o_u = o.x; o_v = o.y; o_k = o.z; d_u = d.x; d_v = d.y; d_k = d.z; }
            const uint32_t end = sc.kBegin[g + 1];
#pragma unroll 1
            for (uint32_t q = sc.kBegin[g]; q < end; ++q) {
                const float4 G0 = A_.groups(2 * q);
                const float ta = __fdividef(G0.z - o_u * G0.x - o_v * G0.y - o_k, d_u * G0.x + d_v * G0.y + d_k);
                if (ta >= tlo && ta <= thi) {
                    const float4 G1 = A_.groups(2 * q + 1);
                    const float pu = o_u + ta * d_u, pv = o_v + ta * d_v;
                    if (pu >= G1.x && pv >= G1.y && pu <= G1.z && pv <= G1.w) {
                        cand |= 1u << q; if (ta < nearT) { nearT = ta; nearQ = q; }
                    }
                }
            }
        }
        // Pass 2a (converged): every lane tests its NEAREST candidate group exactly -- almost always the true hit.
        if (nearQ != 0xFFFFFFFFu) {
            const uint32_t q = nearQ; cand &= ~(1u << q);
            const int k = (q >= sc.kBegin[1]) + (q >= sc.kBegin[2]);
            const float o_u = k == 0 ? o.y : (k == 1 ? o.z : o.x), o_v = k == 0 ? o.z : (k == 1 ? o.x : o.y), o_k = k == 0 ? o.x : (k == 1 ? o.y : o.z);
            const float d_u = k == 0 ? d.y : (k == 1 ? d.z : d.x), d_v = k == 0 ? d.z : (k == 1 ? d.x : d.y), d_k = k == 0 ? d.x : (k == 1 ? d.y : d.z);
            tri_group_exact(A_, q, o_u, o_v, o_k, d_u, d_v, d_k, mint, maxt, hit);
        }
        // Pass 2b (rare): remaining candidates that are not clearly behind the hit found so far
        while (cand) {
            const uint32_t q = __ffs(cand) - 1; cand &= cand - 1u;
            const int k = (q >= sc.kBegin[1]) + (q >= sc.kBegin[2]);
            const float o_u = k == 0 ? o.y : (k == 1 ? o.z : o.x), o_v = k == 0 ? o.z : (k == 1 ? o.x : o.y), o_k = k == 0 ? o.x : (k == 1 ? o.y : o.z);
            const float d_u = k == 0 ? d.y : (k == 1 ? d.z : d.x), d_v = k == 0 ? d.z : (k == 1 ? d.x : d.y), d_k = k == 0 ? d.x : (k == 1 ? d.y : d.z);
            const float4 G0 = A_.groups(2 * q);
            const float ta = __fdividef(G0.z - o_u * G0.x - o_v * G0.y - o_k, d_u * G0.x + d_v * G0.y + d_k);
            if (ta <= hit.t * (1.0f + 1e-4f)) tri_group_exact(A_, q, o_u, o_v, o_k, d_u, d_v, d_k, mint, maxt, hit);
        }
        return hit.prim != 0xFFFFFFFFu;
    }
    hit = bvh_walk(sc.accel, sc.bvh, o, d, mint, maxt);
    return hit.prim != 0xFFFFFFFFu;
}

// Intersection record (render/shape.h:36), the fields the path uses
struct Its {
    float3 p, geoN, shN, shS, shT, wi;
    int bsdf, emitter;
    __device__ __forceinline__ float3 toLocal(float3 v) const { return f3(dot(v, shS), dot(v, shT), dot(v, shN)); }
    __device__ __forceinline__ float3 toWorld(float3 v) const { return shS * v.x + shT * v.y + shN * v.z; }
};

// fillIntersectionRecord (render/skdtree.h:343-428) + computeShadingFrame (libcore/util.cpp:603-608)
template <bool SPHERES, class Acc>
__device__ __forceinline__ void fill_its(const Acc &A_, const Hit &h, float3 o, float3 d, Its &its) {
    if (SPHERES && (h.prim & PPG_SPHERE_BIT)) {        // Sphere::fillIntersectionRecord (src/shapes/sphere.cpp:209-255), identity rotation
        const uint32_t k = h.prim & ~PPG_SPHERE_BIT;
        const float4 cr = __ldg(&A_.g.spheres[2 * k]), mt = __ldg(&A_.g.spheres[2 * k + 1]);
        const float3 c = f3(cr.x, cr.y, cr.z);
        its.p = o + d * h.t;
        its.p = c + normalize(its.p - c) * cr.w;
        const float3 local = its.p - c;
        const float3 dpdu = f3(-local.y, local.x, 0.f) * (2.f * PPG_PI);
        its.geoN = normalize(its.p - c);
        if (__float_as_uint(mt.z)) its.geoN = its.geoN * -1.0f;
        its.shN = its.geoN;
        its.shS = normalize(dpdu - its.shN * dot(its.shN, dpdu));
        its.shT = cross(its.shN, its.shS);
        its.wi = its.toLocal(-d);
        its.bsdf = __float_as_int(mt.x); its.emitter = __float_as_int(mt.y);
        return;
    }
    const float4 g0 = A_.geom(6 * h.tri), g1 = A_.geom(6 * h.tri + 1), g2 = A_.geom(6 * h.tri + 2);
    const int4 m = A_.meta(h.tri);
    const float3 p0 = f3(g0.x, g0.y, g0.z), p1 = f3(g1.x, g1.y, g1.z), p2 = f3(g2.x, g2.y, g2.z);
    const float3 b = f3(1 - h.u - h.v, h.u, h.v);
    its.p = p0 * b.x + p1 * b.y + p2 * b.z;
    const float3 side1 = p1 - p0, side2 = p2 - p0;
    float3 faceN = cross(side1, side2);
    const float len = sqrtf(dot(faceN, faceN));
    if (!is_zero(faceN)) faceN = faceN * (1.0f / len);
    if (m.z & 1) {
        const float4 h0 = A_.geom(6 * h.tri + 3), h1 = A_.geom(6 * h.tri + 4), h2 = A_.geom(6 * h.tri + 5);
        const float3 n0 = f3(g0.w, h0.x, h0.y), n1 = f3(g1.w, h1.x, h1.y), n2 = f3(g2.w, h2.x, h2.y);
        its.shN = normalize(n0 * b.x + n1 * b.y + n2 * b.z);
        if (dot(faceN, its.shN) < 0.f) faceN = -faceN;
    } else its.shN = faceN;
    its.geoN = faceN;
    const float3 dpdu = side1;
    its.shS = normalize(dpdu - its.shN * dot(its.shN, dpdu));
    its.shT = cross(its.shN, its.shS);
    its.wi = its.toLocal(-d);
    its.bsdf = m.x; its.emitter = m.y;
}

// ------------------------------------------------------------------ BSDF: diffuse (+ twosided)
// src/libcore/warp.cpp:81-102 (concentric disk) then :43-52
__device__ __forceinline__ float3 square_to_cosine_hemisphere(float sx, float sy) {
    const float r1 = 2.0f * sx - 1.0f, r2 = 2.0f * sy - 1.0f;
    float phi, r;
    if (r1 == 0.f && r2 == 0.f) { r = phi = 0.f; }
    else if (r1 * r1 > r2 * r2) { r = r1; phi = (PPG_PI / 4.0f) * (r2 / r1); }
    else { r = r2; phi = (PPG_PI / 2.0f) - (r1 / r2) * (PPG_PI / 4.0f); }
    float s, c; sincosf_bounded(phi, &s, &c);                                  // |r1 / r2| <= 1: |phi| <= 3 pi / 4
    const float px = r * c, py = r * s;
    float z = sqrtf(fmaxf(0.0f, 1.0f - px * px - py * py));
    if (z == 0.f) z = 1e-10f;
    return f3(px, py, z);
}
#define PPG_BSDF_TWOSIDED 1u
#define PPG_BSDF_T_DIFFUSE 0u
#define PPG_BSDF_T_DIELECTRIC 2u
#define PPG_BSDF_T_CONDUCTOR 3u
#define PPG_BSDF_T_ROUGHCONDUCTOR 4u
#define PPG_BSDF_T_ROUGHPLASTIC 5u
#define PPG_BSDF_T_ROUGHDIELECTRIC 6u
#define PPG_BSDF_T_PLASTIC 7u
#define PPG_BSDF_T_THINDIELECTRIC 8u
#define PPG_BSDF_NONLINEAR 2u
#define PPG_BSDF_MASK 4u
#define PPG_BSDF_BUMPMAP 8u
struct Bsdf { float3 refl, trans, etaRgb, k, specRefl, opacity; float eta, invEta, alpha, fdrInt, ssw, maskProb; uint32_t type, flags; int distr; const float *lut;
              uint32_t reflTex, bumpTex; };     // 1 + texture index, 0 = none (ppg_bsdf.reflectance_texture / bump_texture)
// FULL == false: the scene holds diffuse BSDFs and triangles only (host-checked); every other model compiles away
template <bool FULL, class Acc>
__device__ __forceinline__ Bsdf load_bsdf(const Acc &A_, int idx) {
    const float4 a = A_.bsdf(PPG_BSDF_F4 * idx);
    Bsdf b; b.refl = f3(a.x, a.y, a.z);
    const uint32_t tf = __float_as_uint(a.w); b.type = FULL ? (tf & 0xffu) : PPG_BSDF_T_DIFFUSE; b.flags = tf >> 8;
    b.trans = b.etaRgb = b.k = b.specRefl = f3(0, 0, 0); b.eta = b.invEta = 1.f; b.alpha = 0.1f; b.distr = 1; b.fdrInt = b.ssw = 0.f; b.lut = nullptr;
    b.opacity = f3(1, 1, 1); b.maskProb = 1.f; b.reflTex = b.bumpTex = 0u;
    if (FULL) { const float4 w = A_.bsdf(PPG_BSDF_F4 * idx + 5); b.reflTex = __float_as_uint(w.z); b.bumpTex = (b.flags & PPG_BSDF_BUMPMAP) ? __float_as_uint(w.w) : 0u; }
    if (FULL && (b.flags & PPG_BSDF_MASK)) { const float4 m = A_.bsdf(PPG_BSDF_F4 * idx + 6); b.opacity = f3(m.x, m.y, m.z); b.maskProb = m.w; }
    if (!FULL) b.flags &= PPG_BSDF_TWOSIDED;
    if (FULL && b.type != PPG_BSDF_T_DIFFUSE) {
        const float4 t = A_.bsdf(PPG_BSDF_F4 * idx + 1), e = A_.bsdf(PPG_BSDF_F4 * idx + 2), k = A_.bsdf(PPG_BSDF_F4 * idx + 3);
        b.trans = f3(t.x, t.y, t.z); b.eta = t.w; b.etaRgb = f3(e.x, e.y, e.z); b.invEta = e.w; b.k = f3(k.x, k.y, k.z);
        b.alpha = fabsf(k.w); b.distr = k.w < 0.f ? 0 : 1;
        if (b.type == PPG_BSDF_T_ROUGHPLASTIC || b.type == PPG_BSDF_T_PLASTIC) {
            const float4 s = A_.bsdf(PPG_BSDF_F4 * idx + 4), w = A_.bsdf(PPG_BSDF_F4 * idx + 5);
            b.specRefl = f3(s.x, s.y, s.z); b.fdrInt = s.w; b.ssw = w.x; b.lut = A_.g.bsdfTables + (size_t) __float_as_uint(w.y) * PPG_BSDF_LUT;
        }
    }
    return b;
}
__device__ __forceinline__ bool bsdf_has_smooth(const Bsdf &b) { return b.type == PPG_BSDF_T_DIFFUSE || b.type == PPG_BSDF_T_ROUGHCONDUCTOR || b.type == PPG_BSDF_T_ROUGHPLASTIC || b.type == PPG_BSDF_T_ROUGHDIELECTRIC || b.type == PPG_BSDF_T_PLASTIC; }   // type & ESmooth = diffuse | glossy (bsdf.h:224-285)
__device__ __forceinline__ bool bsdf_has_transmission_or_backside(const Bsdf &b) { return (b.flags & (PPG_BSDF_TWOSIDED | PPG_BSDF_MASK)) || b.type == PPG_BSDF_T_DIELECTRIC || b.type == PPG_BSDF_T_ROUGHDIELECTRIC || b.type == PPG_BSDF_T_THINDIELECTRIC; }
__device__ __forceinline__ bool bsdf_has_null(const Bsdf &b) { return b.type == PPG_BSDF_T_THINDIELECTRIC || (b.flags & PPG_BSDF_MASK); }                     // type & ENull

// fresnelDielectricExt, src/libcore/util.cpp:651-683
__device__ __forceinline__ float fresnel_dielectric_ext(float cosThetaI_, float &cosThetaT_, float eta) {
    if (eta == 1.f) { cosThetaT_ = -cosThetaI_; return 0.0f; }
    const float scale = (cosThetaI_ > 0.f) ? 1.f / eta : eta, cosThetaTSqr = 1.f - (1.f - cosThetaI_ * cosThetaI_) * (scale * scale);
    if (cosThetaTSqr <= 0.0f) { cosThetaT_ = 0.0f; return 1.0f; }
    const float cosThetaI = fabsf(cosThetaI_), cosThetaT = sqrtf(cosThetaTSqr);
    const float Rs = (cosThetaI - eta * cosThetaT) / (cosThetaI + eta * cosThetaT);
    const float Rp = (eta * cosThetaI - cosThetaT) / (eta * cosThetaI + cosThetaT);
    cosThetaT_ = (cosThetaI_ > 0.f) ? -cosThetaT : cosThetaT;
    return 0.5f * (Rs * Rs + Rp * Rp);
}
// fresnelConductorExact, src/libcore/util.cpp:715-738 (per channel)
__device__ __forceinline__ float fresnel_conductor_exact(float cosThetaI, float eta, float k) {
    const float cosThetaI2 = cosThetaI * cosThetaI, sinThetaI2 = 1.f - cosThetaI2, sinThetaI4 = sinThetaI2 * sinThetaI2;
    const float temp1 = eta * eta - k * k - sinThetaI2;
    const float a2pb2 = sqrtf(fmaxf(0.0f, temp1 * temp1 + k * k * eta * eta * 4.f));
    const float a = sqrtf(fmaxf(0.0f, (a2pb2 + temp1) * 0.5f));
    const float term1 = a2pb2 + cosThetaI2, term2 = a * (2.f * cosThetaI);
    const float Rs2 = (term1 - term2) / (term1 + term2);
    const float term3 = a2pb2 * cosThetaI2 + sinThetaI4, term4 = term2 * sinThetaI2;
    const float Rp2 = Rs2 * (term3 - term4) / (term3 + term4);
    return 0.5f * (Rp2 + Rs2);
}
// ---- MicrofacetDistribution (isotropic Beckmann / GGX, visible-normal sampling), src/bsdfs/microfacet.h
__device__ __forceinline__ float mts_erfinv(float x) {       // math::erfinv, src/libcore/math.cpp:25-53
    float w = -logf((1.0f - x) * (1.0f + x)), p;
    if (w < 5.0f) {
        w = w - 2.5f; p = 2.81022636e-08f; p = 3.43273939e-07f + p * w; p = -3.5233877e-06f + p * w; p = -4.39150654e-06f + p * w;
        p = 0.00021858087f + p * w; p = -0.00125372503f + p * w; p = -0.00417768164f + p * w; p = 0.246640727f + p * w; p = 1.50140941f + p * w;
    } else {
        w = sqrtf(w) - 3.0f; p = -0.000200214257f; p = 0.000100950558f + p * w; p = 0.00134934322f + p * w; p = -0.00367342844f + p * w;
        p = 0.00573950773f + p * w; p = -0.0076224613f + p * w; p = 0.00943887047f + p * w; p = 1.00167406f + p * w; p = 2.83297682f + p * w;
    }
    return p * x;
}
__device__ __forceinline__ float mts_erf(float x) {          // math::erf, src/libcore/math.cpp:55-72
    const float a1 = 0.254829592f, a2 = -0.284496736f, a3 = 1.421413741f, a4 = -1.453152027f, a5 = 1.061405429f, p = 0.3275911f;
    const float sign = copysignf(1.0f, x); x = fabsf(x);
    const float t = 1.0f / (1.0f + p * x);
    const float y = 1.0f - (((((a5 * t + a4) * t) + a3) * t + a2) * t + a1) * t * expf(-x * x);
    return sign * y;
}
__device__ __forceinline__ float mts_hypot2(float a, float b) {   // math::hypot2, src/libcore/math.cpp:74-86
    float r;
    if (fabsf(a) > fabsf(b)) { r = b / a; r = fabsf(a) * sqrtf(1.0f + r * r); }
    else if (b != 0.0f) { r = a / b; r = fabsf(b) * sqrtf(1.0f + r * r); }
    else r = 0.0f;
    return r;
}
__device__ __forceinline__ float mf_eval(int type, float alpha, float3 m) {                      // microfacet.h:191-236
    if (m.z <= 0.f) return 0.0f;
    const float cosTheta2 = m.z * m.z;
    const float beckmannExponent = ((m.x * m.x) / (alpha * alpha) + (m.y * m.y) / (alpha * alpha)) / cosTheta2;
    float result;
    if (type == 0) result = expf(-beckmannExponent) / (PPG_PI * alpha * alpha * cosTheta2 * cosTheta2);
    else { const float root = (1.0f + beckmannExponent) * cosTheta2; result = 1.0f / (PPG_PI * alpha * alpha * root * root); }
    if (result * m.z < 1e-20f) result = 0.f;
    return result;
}
__device__ __forceinline__ float mf_smithG1(int type, float alpha, float3 v, float3 m) {         // microfacet.h:477-517
    if (dot(v, m) * v.z <= 0.f) return 0.0f;
    const float temp = 1.f - v.z * v.z;
    const float tanTheta = fabsf(temp <= 0.0f ? 0.0f : sqrtf(temp) / v.z);
    if (tanTheta == 0.0f) return 1.0f;
    if (type == 0) {
        const float a = 1.0f / (alpha * tanTheta);
        if (a >= 1.6f) return 1.0f;
        const float aSqr = a * a;
        return (3.535f * a + 2.181f * aSqr) / (1.0f + 2.276f * a + 2.577f * aSqr);
    }
    return 2.0f / (1.0f + mts_hypot2(1.0f, alpha * tanTheta));
}
__device__ __forceinline__ float mf_pdfVisible(int type, float alpha, float3 wi, float3 m) {     // microfacet.h:462-466
    if (wi.z == 0.f) return 0.0f;
    return mf_smithG1(type, alpha, wi, m) * fabsf(dot(wi, m)) * mf_eval(type, alpha, m) / fabsf(wi.z);
}
__device__ __forceinline__ void mf_sampleVisible11(int type, float thetaI, float sx, float sy, float &slopeX, float &slopeY) {   // microfacet.h:573-690
    const float SQRT_PI_INV = 1.f / sqrtf(PPG_PI);
    if (type == 0) {
        if (thetaI < 1e-4f) { const float r = sqrtf(-logf(1.0f - sx)); float s, c; sincosf(2.f * PPG_PI * sy, &s, &c); slopeX = r * c; slopeY = r * s; return; }
        const float tanThetaI = tanf(thetaI), cotThetaI = 1.f / tanThetaI;
        float a = -1.f, c = mts_erf(cotThetaI);
        const float sample_x = fmaxf(sx, 1e-6f);
        const float fit = 1.f + thetaI * (-0.876f + thetaI * (0.4265f - 0.0594f * thetaI));
        float b = c - (1.f + c) * powf(1.f - sample_x, fit);
        const float normalization = 1.f / (1.f + c + SQRT_PI_INV * tanThetaI * expf(-cotThetaI * cotThetaI));
        int it = 0;
        while (++it < 10) {
            if (!(b >= a && b <= c)) b = 0.5f * (a + c);
            const float invErf = mts_erfinv(b);
            const float value = normalization * (1.f + b + SQRT_PI_INV * tanThetaI * expf(-invErf * invErf)) - sample_x;
            const float derivative = normalization * (1.f - invErf * tanThetaI);
            if (fabsf(value) < 1e-5f) break;
            if (value > 0.f) c = b; else a = b;
            b -= value / derivative;
        }
        slopeX = mts_erfinv(b);
        slopeY = mts_erfinv(2.0f * fmaxf(sy, 1e-6f) - 1.0f);
        return;
    }
    if (thetaI < 1e-4f) { const float r = sqrtf(fmaxf(0.0f, sx / (1.f - sx))); float s, c; sincosf(2.f * PPG_PI * sy, &s, &c); slopeX = r * c; slopeY = r * s; return; }
    const float tanThetaI = tanf(thetaI), a = 1.f / tanThetaI;
    const float G1 = 2.0f / (1.0f + sqrtf(fmaxf(0.0f, 1.0f + 1.0f / (a * a))));
    float A = 2.0f * sx / G1 - 1.0f;
    if (fabsf(A) == 1.f) A -= copysignf(1.0f, A) * PPG_EPSILON;
    const float tmp = 1.0f / (A * A - 1.0f), B = tanThetaI;
    const float D = sqrtf(fmaxf(0.0f, B * B * tmp * tmp - (A * A - B * B) * tmp));
    const float slope_x_1 = B * tmp - D, slope_x_2 = B * tmp + D;
    slopeX = (A < 0.0f || slope_x_2 > 1.0f / tanThetaI) ? slope_x_1 : slope_x_2;
    float S;
    if (sy > 0.5f) { S = 1.0f; sy = 2.0f * (sy - 0.5f); } else { S = -1.0f; sy = 2.0f * (0.5f - sy); }
    const float z = (sy * (sy * (sy * (-0.365728915865723f) + 0.790235037209296f) - 0.424965825137544f) + 0.000152998850436920f) /
                    (sy * (sy * (sy * (sy * 0.169507819808272f - 0.397203533833404f) - 0.232500544458471f) + 1.0f) - 0.539825872510702f);
    slopeY = S * z * sqrtf(1.0f + slopeX * slopeX);
}
__device__ __forceinline__ float3 mf_sampleVisible(int type, float alpha, float3 _wi, float sx, float sy) {   // microfacet.h:421-459
    const float3 wi = normalize(f3(alpha * _wi.x, alpha * _wi.y, _wi.z));
    float theta = 0.f, phi = 0.f;
    if (wi.z < 0.99999f) { theta = acosf(wi.z); phi = atan2f(wi.y, wi.x); }
    float sinPhi, cosPhi; sincosf(phi, &sinPhi, &cosPhi);
    float slx, sly; mf_sampleVisible11(type, theta, sx, sy, slx, sly);
    float rx = cosPhi * slx - sinPhi * sly, ry = sinPhi * slx + cosPhi * sly;
    rx *= alpha; ry *= alpha;
    const float normalization = 1.0f / sqrtf(rx * rx + ry * ry + 1.0f);
    return f3(-rx * normalization, -ry * normalization, normalization);
}
__device__ __forceinline__ float3 fresnel_conductor_rgb(float c, const Bsdf &b) {
    return f3(b.refl.x * fresnel_conductor_exact(c, b.etaRgb.x, b.k.x), b.refl.y * fresnel_conductor_exact(c, b.etaRgb.y, b.k.y), b.refl.z * fresnel_conductor_exact(c, b.etaRgb.z, b.k.z));
}
// roughconductor.cpp:257-283 (eval), :285-312 (pdf), :355-404 (sample)
__device__ __forceinline__ float3 roughconductor_eval(const Bsdf &b, float3 wi, float3 wo) {
    if (wi.z <= 0.f || wo.z <= 0.f) return f3(0, 0, 0);
    const float3 H = normalize(wo + wi);
    const float D = mf_eval(b.distr, b.alpha, H);
    if (D == 0.f) return f3(0, 0, 0);
    const float3 F = fresnel_conductor_rgb(dot(wi, H), b);
    const float G = mf_smithG1(b.distr, b.alpha, wi, H) * mf_smithG1(b.distr, b.alpha, wo, H);
    return F * (D * G / (4.0f * wi.z));
}
__device__ __forceinline__ float roughconductor_pdf(const Bsdf &b, float3 wi, float3 wo) {
    if (wi.z <= 0.f || wo.z <= 0.f) return 0.0f;
    const float3 H = normalize(wo + wi);
    return mf_eval(b.distr, b.alpha, H) * mf_smithG1(b.distr, b.alpha, wi, H) / (4.0f * wi.z);
}
__device__ __forceinline__ float3 roughconductor_sample(const Bsdf &b, float3 wi, float sx, float sy, float3 &wo, float &pdf) {
    pdf = 0.f;
    if (wi.z < 0.f) return f3(0, 0, 0);
    const float3 m = mf_sampleVisible(b.distr, b.alpha, wi, sx, sy);
    pdf = mf_pdfVisible(b.distr, b.alpha, wi, m);
    if (pdf == 0.f) return f3(0, 0, 0);
    wo = m * (2.f * dot(wi, m)) - wi;
    if (wo.z <= 0.f) return f3(0, 0, 0);
    const float3 F = fresnel_conductor_rgb(dot(wi, m), b);
    const float weight = mf_smithG1(b.distr, b.alpha, wo, m);
    pdf /= 4.0f * dot(wo, m);
    return F * weight;
}

// ---- roughplastic (src/bsdfs/roughplastic.cpp).  RoughTransmittance::eval with alpha and eta fixed (src/bsdfs/rtrans.h:183-193, 233):
// evalCubicInterp1D (src/libcore/spline.cpp:23-60) of the material's table over cos(theta)^(1/4), clamped to [0,1].
__device__ __forceinline__ float rough_transmittance(const float *__restrict__ values, float cosTheta) {
    if (!(cosTheta >= 0.f)) return 0.0f;
    const float x = powf(fabsf(cosTheta), 0.25f);
    const int size = PPG_BSDF_LUT;
    float result = 0.0f;
    if (x >= 0.0f && x <= 1.0f) {
        float t = ((x - 0.0f) * (float) (size - 1)) / (1.0f - 0.0f);
        const int k = max(0, min((int) t, size - 2));
        const float f0 = __ldg(&values[k]), f1 = __ldg(&values[k + 1]);
        const float d0 = k > 0 ? 0.5f * (f1 - __ldg(&values[k - 1])) : f1 - f0;
        const float d1 = k + 2 < size ? 0.5f * (__ldg(&values[k + 2]) - f0) : f1 - f0;
        t = t - (float) k;
        const float t2 = t * t, t3 = t2 * t;
        result = (2.f * t3 - 3.f * t2 + 1.f) * f0 + (-2.f * t3 + 3.f * t2) * f1 + (t3 - 2.f * t2 + t) * d0 + (t3 - t2) * d1;
    }
    return fminf(1.0f, fmaxf(0.0f, result));
}
__device__ __forceinline__ float roughplastic_prob_specular(const Bsdf &b, float cosThetaI) {   // roughplastic.cpp:403-409 = :446-452
    const float probSpecular = 1.f - rough_transmittance(b.lut, cosThetaI);
    return (probSpecular * b.ssw) / (probSpecular * b.ssw + (1.f - probSpecular) * (1.f - b.ssw));
}
__device__ __forceinline__ float3 roughplastic_eval(const Bsdf &b, float3 wi, float3 wo) {     // roughplastic.cpp:326-380
    if (wi.z <= 0.f || wo.z <= 0.f) return f3(0, 0, 0);
    const float3 H = normalize(wo + wi);
    const float D = mf_eval(b.distr, b.alpha, H);
    float cosThetaT; const float F = fresnel_dielectric_ext(dot(wi, H), cosThetaT, b.eta);
    const float G = mf_smithG1(b.distr, b.alpha, wi, H) * mf_smithG1(b.distr, b.alpha, wo, H);
    const float value = F * D * G / (4.0f * wi.z);
    const float3 result = b.specRefl * value;
    float3 diff = b.refl;
    const float T12 = rough_transmittance(b.lut, wi.z), T21 = rough_transmittance(b.lut, wo.z), Fdr = b.fdrInt;
    if (b.flags & PPG_BSDF_NONLINEAR) diff = f3(diff.x / (1.0f - diff.x * Fdr), diff.y / (1.0f - diff.y * Fdr), diff.z / (1.0f - diff.z * Fdr));
    else diff = diff * (1.0f / (1.f - Fdr));                   // Spectrum /= Float multiplies by the reciprocal (core/spectrum.h:447-456)
    const float invEta2 = 1.f / (b.eta * b.eta);
    return result + diff * (PPG_INV_PI * wo.z * T12 * T21 * invEta2);
}
__device__ __forceinline__ float roughplastic_pdf(const Bsdf &b, float3 wi, float3 wo) {       // roughplastic.cpp:382-430
    if (wi.z <= 0.f || wo.z <= 0.f) return 0.0f;
    const float3 H = normalize(wo + wi);
    const float probSpecular = roughplastic_prob_specular(b, wi.z), probDiffuse = 1.f - probSpecular;
    const float dwh_dwo = 1.0f / (4.0f * dot(wo, H));
    const float prob = mf_pdfVisible(b.distr, b.alpha, wi, H);
    float result = prob * dwh_dwo * probSpecular;
    result += probDiffuse * (PPG_INV_PI * wo.z);
    return result;
}
__device__ __forceinline__ float3 roughplastic_sample(const Bsdf &b, float3 wi, float sx, float sy, float3 &wo, float &pdf) {   // roughplastic.cpp:432-497
    pdf = 0.f;
    if (wi.z <= 0.f) return f3(0, 0, 0);
    bool choseSpecular = true;
    const float probSpecular = roughplastic_prob_specular(b, wi.z);
    if (sy < probSpecular) sy /= probSpecular;
    else { sy = (sy - probSpecular) / (1.f - probSpecular); choseSpecular = false; }
    if (choseSpecular) {
        const float3 m = mf_sampleVisible(b.distr, b.alpha, wi, sx, sy);
        wo = m * (2.f * dot(wi, m)) - wi;
        if (wo.z <= 0.f) return f3(0, 0, 0);
    } else wo = square_to_cosine_hemisphere(sx, sy);
    pdf = roughplastic_pdf(b, wi, wo);
    if (pdf == 0.f) return f3(0, 0, 0);
    return roughplastic_eval(b, wi, wo) * (1.0f / pdf);       // Spectrum / Float, core/spectrum.h:415-425
}

// ---- thindielectric (src/bsdfs/thindielectric.cpp): R' = R + T R T + T R^3 T + ... (:160-165)
__device__ __forceinline__ float thindielectric_reflectance(float cosThetaI, float eta) {
    float ct; float R = fresnel_dielectric_ext(fabsf(cosThetaI), ct, eta); const float T = 1.f - R;
    if (R < 1.f) R += T * T * R / (1.f - R * R);
    return R;
}
// bsdf->eval(bRec, EDiscrete) with typeMask == ENull and wo == -wi (thindielectric.cpp:153-176): what a straight-through ray keeps
__device__ __forceinline__ float3 bsdf_eval_null(const Bsdf &b, float cosThetaI) {
    if (b.flags & PPG_BSDF_MASK) return f3(1.f - b.opacity.x, 1.f - b.opacity.y, 1.f - b.opacity.z);       // mask.cpp:118-119
    if (b.type != PPG_BSDF_T_THINDIELECTRIC) return f3(0, 0, 0);
    return b.trans * (1.f - thindielectric_reflectance(cosThetaI, b.eta));
}
// ---- plastic (src/bsdfs/plastic.cpp): delta reflection off the coat + diffuse base; eval / pdf in the solid-angle measure see the diffuse part only
__device__ __forceinline__ float3 plastic_diffuse(const Bsdf &b) {                                       // plastic.cpp:266-271
    const float3 diff = b.refl;
    if (b.flags & PPG_BSDF_NONLINEAR) return f3(diff.x / (1.0f - diff.x * b.fdrInt), diff.y / (1.0f - diff.y * b.fdrInt), diff.z / (1.0f - diff.z * b.fdrInt));
    return diff * (1.0f / (1.f - b.fdrInt));
}
__device__ __forceinline__ float plastic_prob_specular(const Bsdf &b, float Fi) {                        // plastic.cpp:292-294
    return (Fi * b.ssw) / (Fi * b.ssw + (1.f - Fi) * (1.f - b.ssw));
}
__device__ __forceinline__ float3 plastic_eval(const Bsdf &b, float3 wi, float3 wo) {                    // plastic.cpp:245-278
    if (wo.z <= 0.f || wi.z <= 0.f) return f3(0, 0, 0);
    float ct; const float Fi = fresnel_dielectric_ext(wi.z, ct, b.eta), Fo = fresnel_dielectric_ext(wo.z, ct, b.eta);
    const float invEta2 = 1.f / (b.eta * b.eta);
    return plastic_diffuse(b) * ((PPG_INV_PI * wo.z) * invEta2 * (1.f - Fi) * (1.f - Fo));
}
__device__ __forceinline__ float plastic_pdf(const Bsdf &b, float3 wi, float3 wo) {                      // plastic.cpp:280-308
    if (wo.z <= 0.f || wi.z <= 0.f) return 0.0f;
    float ct; const float Fi = fresnel_dielectric_ext(wi.z, ct, b.eta);
    return (PPG_INV_PI * wo.z) * (1.f - plastic_prob_specular(b, Fi));
}
__device__ __forceinline__ float3 plastic_sample(const Bsdf &b, float3 wi, float sx, float sy, float3 &wo, bool &delta, float &pdf) {   // plastic.cpp:374-441
    pdf = 0.f; delta = false;
    if (wi.z <= 0.f) return f3(0, 0, 0);
    float ct; const float Fi = fresnel_dielectric_ext(wi.z, ct, b.eta);
    const float probSpecular = plastic_prob_specular(b, Fi);
    if (sx < probSpecular) {
        delta = true; wo = f3(-wi.x, -wi.y, wi.z); pdf = probSpecular;
        return (b.specRefl * Fi) * (1.0f / probSpecular);
    }
    wo = square_to_cosine_hemisphere((sx - probSpecular) / (1.f - probSpecular), sy);
    const float Fo = fresnel_dielectric_ext(wo.z, ct, b.eta);
    const float invEta2 = 1.f / (b.eta * b.eta);
    pdf = (1.f - probSpecular) * (PPG_INV_PI * wo.z);
    return plastic_diffuse(b) * (invEta2 * (1.f - Fi) * (1.f - Fo) / (1.f - probSpecular));
}
// ---- roughdielectric (src/bsdfs/roughdielectric.cpp), visible-normal sampling.  sample() takes ONE extra number `su` of the path's
// sampler to choose reflection / refraction (EUsesSampler, :536-543).
__device__ __forceinline__ float mts_signum(float v) { return copysignf(1.0f, v); }                     // core/math.h:269-278
__device__ __forceinline__ float3 roughdielectric_eval(const Bsdf &b, float3 wi, float3 wo) {            // roughdielectric.cpp:270-350
    if (wi.z == 0.f) return f3(0, 0, 0);
    const bool reflect = wi.z * wo.z > 0.f;
    float3 H;
    if (reflect) H = normalize(wo + wi);
    else { const float eta = wi.z > 0.f ? b.eta : b.invEta; H = normalize(wi + wo * eta); }
    H = H * mts_signum(H.z);
    const float D = mf_eval(b.distr, b.alpha, H);
    if (D == 0.f) return f3(0, 0, 0);
    float cosThetaT; const float F = fresnel_dielectric_ext(dot(wi, H), cosThetaT, b.eta);
    const float G = mf_smithG1(b.distr, b.alpha, wi, H) * mf_smithG1(b.distr, b.alpha, wo, H);
    if (reflect) {
        const float value = F * D * G / (4.0f * fabsf(wi.z));
        return b.refl * value;
    }
    const float eta = wi.z > 0.0f ? b.eta : b.invEta;
    const float sqrtDenom = dot(wi, H) + eta * dot(wo, H);
    const float value = ((1.f - F) * D * G * eta * eta * dot(wi, H) * dot(wo, H)) / (wi.z * sqrtDenom * sqrtDenom);
    const float factor = wi.z > 0.f ? b.invEta : b.eta;                                                  // ERadiance
    return b.trans * fabsf(value * factor * factor);
}
__device__ __forceinline__ float roughdielectric_pdf(const Bsdf &b, float3 wi, float3 wo) {              // roughdielectric.cpp:352-422
    const bool reflect = wi.z * wo.z > 0.f;
    float3 H; float dwh_dwo;
    if (reflect) { H = normalize(wo + wi); dwh_dwo = 1.0f / (4.0f * dot(wo, H)); }
    else {
        const float eta = wi.z > 0.f ? b.eta : b.invEta;
        H = normalize(wi + wo * eta);
        const float sqrtDenom = dot(wi, H) + eta * dot(wo, H);
        dwh_dwo = (eta * eta * dot(wo, H)) / (sqrtDenom * sqrtDenom);
    }
    H = H * mts_signum(H.z);
    float prob = mf_pdfVisible(b.distr, b.alpha, wi * mts_signum(wi.z), H);
    float cosThetaT; const float F = fresnel_dielectric_ext(dot(wi, H), cosThetaT, b.eta);
    prob *= reflect ? F : (1.f - F);
    return fabsf(prob * dwh_dwo);
}
__device__ __forceinline__ float3 roughdielectric_sample(const Bsdf &b, float3 wi, float sx, float sy, float su, float3 &wo, float &etaOut, float &pdf) {   // :502-600
    pdf = 0.f;
    const float3 wiUp = wi * mts_signum(wi.z);
    const float3 m = mf_sampleVisible(b.distr, b.alpha, wiUp, sx, sy);
    const float microfacetPDF = mf_pdfVisible(b.distr, b.alpha, wiUp, m);
    if (microfacetPDF == 0.f) return f3(0, 0, 0);
    pdf = microfacetPDF;
    float cosThetaT; const float F = fresnel_dielectric_ext(dot(wi, m), cosThetaT, b.eta);
    float3 weight = f3(1, 1, 1);
    bool sampleReflection = true;
    if (su > F) { sampleReflection = false; pdf *= 1.f - F; } else pdf *= F;
    float dwh_dwo;
    if (sampleReflection) {
        wo = m * (2.f * dot(wi, m)) - wi; etaOut = 1.0f;
        if (wi.z * wo.z <= 0.f) return f3(0, 0, 0);
        weight = weight * b.refl;
        dwh_dwo = 1.0f / (4.0f * dot(wo, m));
    } else {
        if (cosThetaT == 0.f) return f3(0, 0, 0);
        { const float eta = cosThetaT < 0.f ? 1.f / b.eta : b.eta; wo = m * (dot(wi, m) * eta + cosThetaT) - wi * eta; }   // refract(), util.cpp:767-772
        etaOut = cosThetaT < 0.f ? b.eta : b.invEta;
        if (wi.z * wo.z >= 0.f) return f3(0, 0, 0);
        const float factor = cosThetaT < 0.f ? b.invEta : b.eta;
        weight = weight * (b.trans * (factor * factor));
        const float sqrtDenom = dot(wi, m) + etaOut * dot(wo, m);
        dwh_dwo = (etaOut * etaOut * dot(wo, m)) / (sqrtDenom * sqrtDenom);
    }
    weight = weight * mf_smithG1(b.distr, b.alpha, wo, m);
    pdf *= fabsf(dwh_dwo);
    return weight;
}

// eval / pdf in the solid-angle measure (delta models: 0); sample per src/bsdfs/{diffuse.cpp:110-150, dielectric.cpp:277-334, conductor.cpp:262-277};
// twosided per src/bsdfs/twosided.cpp:108-184
__device__ __forceinline__ float3 bsdf_eval_inner(const Bsdf &b, float3 wi, float3 wo) {
    if (!bsdf_has_smooth(b)) return f3(0, 0, 0);
    if ((b.flags & PPG_BSDF_TWOSIDED) && wi.z < 0.f) { wi.z = -wi.z; wo.z = -wo.z; }
    if (b.type == PPG_BSDF_T_ROUGHCONDUCTOR) return roughconductor_eval(b, wi, wo);
    if (b.type == PPG_BSDF_T_ROUGHDIELECTRIC) return roughdielectric_eval(b, wi, wo);
    if (b.type == PPG_BSDF_T_PLASTIC) return plastic_eval(b, wi, wo);
    if (b.type == PPG_BSDF_T_ROUGHPLASTIC) return roughplastic_eval(b, wi, wo);
    if (wi.z <= 0.f || wo.z <= 0.f) return f3(0, 0, 0);
    return b.refl * (PPG_INV_PI * wo.z);
}
__device__ __forceinline__ float bsdf_pdf_inner(const Bsdf &b, float3 wi, float3 wo) {
    if (!bsdf_has_smooth(b)) return 0.0f;
    if ((b.flags & PPG_BSDF_TWOSIDED) && wi.z < 0.f) { wi.z = -wi.z; wo.z = -wo.z; }
    if (b.type == PPG_BSDF_T_ROUGHCONDUCTOR) return roughconductor_pdf(b, wi, wo);
    if (b.type == PPG_BSDF_T_ROUGHDIELECTRIC) return roughdielectric_pdf(b, wi, wo);
    if (b.type == PPG_BSDF_T_PLASTIC) return plastic_pdf(b, wi, wo);
    if (b.type == PPG_BSDF_T_ROUGHPLASTIC) return roughplastic_pdf(b, wi, wo);
    if (wi.z <= 0.f || wo.z <= 0.f) return 0.0f;
    return PPG_INV_PI * wo.z;
}
// `rng`: the path's sampler, consumed only by models that draw from it themselves (roughdielectric)
// isNull: sampledType == ENull (index-matched transition straight through the surface)
__device__ __forceinline__ float3 bsdf_sample_inner(const Bsdf &b, float3 wi, float sx, float sy, float3 &wo, float &eta, bool &delta, float &pdf, Pcg32 &rng, bool &isNull) {
    isNull = false;
    if (b.type == PPG_BSDF_T_THINDIELECTRIC) {                                                 // thindielectric.cpp:206-240
        const float R = thindielectric_reflectance(wi.z, b.eta);
        delta = true; eta = 1.0f;
        if (sx <= R) { wo = f3(-wi.x, -wi.y, wi.z); pdf = R; return b.refl; }
        isNull = true; wo = f3(-wi.x, -wi.y, -wi.z); pdf = 1.f - R;
        return b.trans;
    }
    bool flip = false;
    if ((b.flags & PPG_BSDF_TWOSIDED) && wi.z < 0.f) { wi.z = -wi.z; flip = true; }
    eta = 1.0f; delta = false; pdf = 0.f;
    if (b.type == PPG_BSDF_T_DIELECTRIC) {
        float cosThetaT; const float F = fresnel_dielectric_ext(wi.z, cosThetaT, b.eta);
        delta = true;
        if (sx <= F) { wo = f3(-wi.x, -wi.y, wi.z); pdf = F; return b.refl; }
        const float scale = -(cosThetaT < 0.f ? b.invEta : b.eta);
        wo = f3(scale * wi.x, scale * wi.y, cosThetaT); eta = cosThetaT < 0.f ? b.eta : b.invEta; pdf = 1.f - F;
        const float factor = cosThetaT < 0.f ? b.invEta : b.eta;
        return b.trans * (factor * factor);
    }
    if (b.type == PPG_BSDF_T_CONDUCTOR) {
        if (wi.z <= 0.f) return f3(0, 0, 0);
        delta = true; wo = f3(-wi.x, -wi.y, wi.z); pdf = 1.f;
        if (flip) wo.z = -wo.z;
        return f3(b.refl.x * fresnel_conductor_exact(wi.z, b.etaRgb.x, b.k.x), b.refl.y * fresnel_conductor_exact(wi.z, b.etaRgb.y, b.k.y),
                  b.refl.z * fresnel_conductor_exact(wi.z, b.etaRgb.z, b.k.z));
    }
    if (b.type == PPG_BSDF_T_ROUGHCONDUCTOR) {
        const float3 w = roughconductor_sample(b, wi, sx, sy, wo, pdf);
        if (flip) wo.z = -wo.z;
        return w;
    }
    if (b.type == PPG_BSDF_T_ROUGHDIELECTRIC) { const float su = rng.next1D(); return roughdielectric_sample(b, wi, sx, sy, su, wo, eta, pdf); }
    if (b.type == PPG_BSDF_T_PLASTIC) {
        const float3 w = plastic_sample(b, wi, sx, sy, wo, delta, pdf);
        if (flip) wo.z = -wo.z;
        return w;
    }
    if (b.type == PPG_BSDF_T_ROUGHPLASTIC) {
        const float3 w = roughplastic_sample(b, wi, sx, sy, wo, pdf);
        if (flip) wo.z = -wo.z;
        return w;
    }
    if (wi.z <= 0.f) return f3(0, 0, 0);
    wo = square_to_cosine_hemisphere(sx, sy);
    pdf = PPG_INV_PI * wo.z;
    if (flip) wo.z = -wo.z;
    return b.refl;
}

// ---- mask (src/bsdfs/mask.cpp:113-220), the outermost wrapper: nested model scaled by the opacity, or a straight-through null transition
__device__ __forceinline__ float3 bsdf_eval(const Bsdf &b, float3 wi, float3 wo) {
    const float3 v = bsdf_eval_inner(b, wi, wo);
    return (b.flags & PPG_BSDF_MASK) ? v * b.opacity : v;
}
__device__ __forceinline__ float bsdf_pdf(const Bsdf &b, float3 wi, float3 wo) {
    const float p = bsdf_pdf_inner(b, wi, wo);
    return (b.flags & PPG_BSDF_MASK) ? p * b.maskProb : p;
}
__device__ __forceinline__ float3 bsdf_sample(const Bsdf &b, float3 wi, float sx, float sy, float3 &wo, float &eta, bool &delta, float &pdf, Pcg32 &rng, bool &isNull) {
    const bool mask = b.flags & PPG_BSDF_MASK;                                                // mask.cpp:186-207
    if (mask) {
        if (!(sx < b.maskProb)) {
            wo = f3(-wi.x, -wi.y, -wi.z); eta = 1.0f; delta = true; isNull = true;
            pdf = 1.f - b.maskProb;
            return f3(1.f - b.opacity.x, 1.f - b.opacity.y, 1.f - b.opacity.z) * (1.0f / pdf);
        }
        sx /= b.maskProb;
    }
    float3 result = bsdf_sample_inner(b, wi, sx, sy, wo, eta, delta, pdf, rng, isNull);
    if (mask) { result = (result * b.opacity) * (1.0f / b.maskProb); pdf *= b.maskProb; }
    return result;
}

// ------------------------------------------------------------------ bitmap textures, bump mapping, environment map (full-feature variants only)
// Not inlined: rare paths that must not cost the main shading code registers.
__device__ __forceinline__ int tex_wrap(int x, int size, uint32_t mode) {                    // TMIPMap::evalTexel boundary handling, render/mipmap.h:503-563
    if (x >= 0 && x < size) return x;
    if (mode == 0u) { const int r = x % size; return r < 0 ? r + size : r; }                 // repeat (math::modulo)
    if (mode == 1u) return min(max(x, 0), size - 1);                                          // clamp
    int r = x % (2 * size); if (r < 0) r += 2 * size;                                         // mirror
    return r >= size ? 2 * size - r - 1 : r;
}
__device__ __forceinline__ float3 tex_texel(const uint2 *__restrict__ base, int W, int H, uint32_t wu, uint32_t wv, int x, int y) {
    x = tex_wrap(x, W, wu); y = tex_wrap(y, H, wv);
    const uint2 t = __ldg(&base[(size_t) y * (size_t) W + (size_t) x]);
    return f3(__half2float(__ushort_as_half((unsigned short) (t.x & 0xffffu))), __half2float(__ushort_as_half((unsigned short) (t.x >> 16))),
              __half2float(__ushort_as_half((unsigned short) (t.y & 0xffffu))));
}
// TMIPMap::evalBilinear(0, uv), render/mipmap.h:575-596 (same operation order as the oracle: ((texel * wx) * wy), summed left to right)
__device__ __forceinline__ float3 tex_bilinear(const uint2 *__restrict__ base, int W, int H, uint32_t wu, uint32_t wv, float uu, float vv) {
    if (!isfinite(uu) || !isfinite(vv)) return f3(0, 0, 0);
    const float u = uu * (float) W - 0.5f, v = vv * (float) H - 0.5f;
    const int xPos = (int) floorf(u), yPos = (int) floorf(v);
    const float dx1 = u - (float) xPos, dx2 = 1.0f - dx1, dy1 = v - (float) yPos, dy2 = 1.0f - dy1;
    float3 r = tex_texel(base, W, H, wu, wv, xPos, yPos) * dx2 * dy2;
    r = r + tex_texel(base, W, H, wu, wv, xPos, yPos + 1) * dx2 * dy1;
    r = r + tex_texel(base, W, H, wu, wv, xPos + 1, yPos) * dx1 * dy2;
    r = r + tex_texel(base, W, H, wu, wv, xPos + 1, yPos + 1) * dx1 * dy1;
    return r;
}
// Texture2D::eval(its) without UV partials (librender/texture.cpp:112-121) -> BitmapTexture::eval(uv) (textures/bitmap.cpp:431-453)
static __device__ __noinline__ float3 tex_eval(const SceneView &sc, uint32_t idx, float2 uv) {
    const float4 m0 = __ldg(&sc.texMeta[2 * idx]), m1 = __ldg(&sc.texMeta[2 * idx + 1]);
    const uint32_t wr = __float_as_uint(m0.z);
    return tex_bilinear(sc.texels + __float_as_uint(m0.w), (int) __float_as_uint(m0.x), (int) __float_as_uint(m0.y), wr & 0xffu, wr >> 8, uv.x * m1.x + m1.z, uv.y * m1.y + m1.w);
}
// Texture2D::evalGradient(its) (texture.cpp:123-130) -> evalGradientBilinear (mipmap.h:601-626), reduced to the luminances BumpMap::getFrame uses
static __device__ __noinline__ float2 tex_gradient_lum(const SceneView &sc, uint32_t idx, float2 uv) {
    const float4 m0 = __ldg(&sc.texMeta[2 * idx]), m1 = __ldg(&sc.texMeta[2 * idx + 1]);
    const uint32_t wr = __float_as_uint(m0.z), wu = wr & 0xffu, wv = wr >> 8;
    const int W = (int) __float_as_uint(m0.x), H = (int) __float_as_uint(m0.y);
    const uint2 *base = sc.texels + __float_as_uint(m0.w);
    const float uu = uv.x * m1.x + m1.z, vv = uv.y * m1.y + m1.w;
    float3 g0 = f3(0, 0, 0), g1 = f3(0, 0, 0);
    if (isfinite(uu) && isfinite(vv)) {
        const float u = uu * (float) W - 0.5f, v = vv * (float) H - 0.5f;
        const int xPos = (int) floorf(u), yPos = (int) floorf(v);
        const float dx = u - (float) xPos, dy = v - (float) yPos;
        const float3 p00 = tex_texel(base, W, H, wu, wv, xPos, yPos), p10 = tex_texel(base, W, H, wu, wv, xPos + 1, yPos),
                     p01 = tex_texel(base, W, H, wu, wv, xPos, yPos + 1), p11 = tex_texel(base, W, H, wu, wv, xPos + 1, yPos + 1);
        const float3 tmp = p01 + p10 - p11;
        g0 = (p10 + p00 * (dy - 1.f) - tmp * dy) * (float) W;
        g1 = (p01 + p00 * (dx - 1.f) - tmp * dx) * (float) H;
    }
    g0 = g0 * m1.x; g1 = g1 * m1.y;
    return make_float2(g0.x * 0.212671f + g0.y * 0.715160f + g0.z * 0.072169f, g1.x * 0.212671f + g1.y * 0.715160f + g1.z * 0.072169f);
}
// EnvironmentMap::evalEnvironment without ray differentials (src/emitters/envmap.cpp:380-410): u repeats, v clamps (:176-178)
static __device__ __noinline__ float3 env_eval(const SceneView &sc, float3 d) {
    const float3 v = f3(sc.worldToEnv[0] * d.x + sc.worldToEnv[1] * d.y + sc.worldToEnv[2] * d.z, sc.worldToEnv[3] * d.x + sc.worldToEnv[4] * d.y + sc.worldToEnv[5] * d.z,
                        sc.worldToEnv[6] * d.x + sc.worldToEnv[7] * d.y + sc.worldToEnv[8] * d.z);
    const float uu = atan2f(v.x, -v.z) * 0.15915494309189533577f;                     // INV_TWOPI
    const float vv = acosf(fminf(1.0f, fmaxf(-1.0f, v.y))) * PPG_INV_PI;               // math::safe_acos * INV_PI
    return tex_bilinear(sc.envTexels, (int) sc.envW, (int) sc.envH, 0u, 1u, uu, vv) * sc.envScale;
}
// ---- light sampling of the environment emitter (full-feature NEE variants only; rare path, not inlined)
// EnvironmentMap::sampleReuse (envmap.cpp:657-662): std::lower_bound over cdf[0..size], clamp, rescale the sample
__device__ __forceinline__ uint32_t env_sample_reuse(const float *__restrict__ cdf, uint32_t size, float &sample) {
    uint32_t lo = 0, hi = size + 1;                   // first index with !(cdf[idx] < sample)
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (__ldg(&cdf[mid]) < sample) lo = mid + 1; else hi = mid; }
    int index = (int) lo - 1; if (index < 0) index = 0; if ((uint32_t) index > size - 1) index = (int) size - 1;
    const float c0 = __ldg(&cdf[index]), c1 = __ldg(&cdf[index + 1]);
    sample = (sample - c0) / (c1 - c0);
    return (uint32_t) index;
}
__device__ __forceinline__ float interval_to_tent(float sample) {                     // libcore/warp.cpp:143-155
    float sign;
    if (sample < 0.5f) { sign = 1.f; sample *= 2.f; } else { sign = -1.f; sample = 2.f * (sample - 0.5f); }
    return sign * (1.f - sqrtf(sample));
}
__device__ __forceinline__ float luminance(float3 c) { return c.x * 0.212671f + c.y * 0.715160f + c.z * 0.072169f; }
// the bilinear, luminance- and row-weighted density shared by internalSampleDirection / internalPdfDirection (envmap.cpp:577-591, 619-632), before the 1 / sin(theta)
static __device__ __noinline__ float env_density(const SceneView &sc, float px, float py, float3 *valueOut) {
    const int W = (int) sc.envW, H = (int) sc.envH;
    const int xPos = (int) floorf(px), yPos = (int) floorf(py);
    const float dx1 = px - (float) xPos, dx2 = 1.0f - dx1, dy1 = py - (float) yPos, dy2 = 1.0f - dy1;
    const float3 value1 = tex_texel(sc.envTexels, W, H, 0u, 1u, xPos, yPos) * dx2 * dy2 + tex_texel(sc.envTexels, W, H, 0u, 1u, xPos + 1, yPos) * dx1 * dy2;
    const float3 value2 = tex_texel(sc.envTexels, W, H, 0u, 1u, xPos, yPos + 1) * dx2 * dy1 + tex_texel(sc.envTexels, W, H, 0u, 1u, xPos + 1, yPos + 1) * dx1 * dy1;
    if (valueOut) *valueOut = (value1 + value2) * sc.envScale;
    const int y0 = min(max(yPos, 0), H - 1), y1 = min(max(yPos + 1, 0), H - 1);
    const float *rowWeights = sc.env->rowWeights;
    return (luminance(value1) * __ldg(&rowWeights[y0]) + luminance(value2) * __ldg(&rowWeights[y1])) * sc.env->normalization;
}
// EnvironmentMap::internalSampleDirection (envmap.cpp:567-600): direction in the emitter's frame, radiance there, solid-angle density
static __device__ __noinline__ void env_sample_direction(const SceneView &sc, float sx, float sy, float3 &d, float3 &value, float &pdf) {
    const uint32_t row = env_sample_reuse(sc.env->cdfRows, sc.envH, sy);
    const uint32_t col = env_sample_reuse(sc.env->cdfCols + (size_t) row * (sc.envW + 1u), sc.envW, sx);
    const float px = (float) col + interval_to_tent(sx), py = (float) row + interval_to_tent(sy);
    pdf = env_density(sc, px, py, &value);
    float sinPhi, cosPhi, sinTheta, cosTheta;
    sincosf(sc.env->pixelX * (px + 0.5f), &sinPhi, &cosPhi);
    sincosf(sc.env->pixelY * (py + 0.5f), &sinTheta, &cosTheta);
    d = f3(sinPhi * sinTheta, cosTheta, -cosPhi * sinTheta);
    pdf /= fmaxf(fabsf(sinTheta), PPG_EPSILON);
}
// EnvironmentMap::pdfDirect in the solid-angle measure -> internalPdfDirection (envmap.cpp:545-548, 603-633) for a WORLD direction
static __device__ __noinline__ float env_pdf_direction(const SceneView &sc, float3 dw) {
    const float3 d = f3(sc.worldToEnv[0] * dw.x + sc.worldToEnv[1] * dw.y + sc.worldToEnv[2] * dw.z, sc.worldToEnv[3] * dw.x + sc.worldToEnv[4] * dw.y + sc.worldToEnv[5] * dw.z,
                        sc.worldToEnv[6] * dw.x + sc.worldToEnv[7] * dw.y + sc.worldToEnv[8] * dw.z);
    const float uu = atan2f(d.x, -d.z) * 0.15915494309189533577f, vv = acosf(fminf(1.0f, fmaxf(-1.0f, d.y))) * PPG_INV_PI;
    if (!isfinite(uu) || !isfinite(vv)) return 0.0f;
    const float u = uu * (float) sc.envW - 0.5f, v = vv * (float) sc.envH - 0.5f;
    const float sinTheta = sqrtf(fmaxf(0.0f, 1.f - d.y * d.y));                        // math::safe_sqrt
    return env_density(sc, u, v, nullptr) / fmaxf(fabsf(sinTheta), PPG_EPSILON);
}
__device__ __forceinline__ void coordinate_system(float3 a, float3 &b, float3 &c);
// Texture coordinates of a triangle hit (skdtree.h:398-405), the textured BSDF parameters there, and BumpMap::getFrame (src/bsdfs/bumpmap.cpp:139-159)
// with the per-triangle UV tangents of TriMesh::computeUVTangents (src/librender/trimesh.cpp:683-743).  With a bump map the shading frame of `its`
// is REPLACED by the perturbed one: the wrapper (bumpmap.cpp:161-236) evaluates the nested model there on the same world-space directions; what the
// integrator and the wrapper still need of the original frame is its normal (the caller keeps it): cos(theta) signs for the strict-normal tests
// (GP:1929-1932, 2028-2032) and for the wrapper's own `cosTheta(wo) * cosTheta(perturbed wo) <= 0` rejection.
template <class Acc>
__device__ __noinline__ void apply_textures(const Acc &A_, const Hit &h, float3 rayD, Its &its, Bsdf &b) {
    const float4 g0 = A_.geom(6 * h.tri), g1 = A_.geom(6 * h.tri + 1), g2 = A_.geom(6 * h.tri + 2);
    const float4 h0 = A_.geom(6 * h.tri + 3), h1 = A_.geom(6 * h.tri + 4), h2 = A_.geom(6 * h.tri + 5);
    const bool hasUv = A_.meta(h.tri).z & 2;
    const float3 bc = f3(1 - h.u - h.v, h.u, h.v);
    float2 uv;
    if (hasUv) { uv.x = h0.z * bc.x + h1.z * bc.y + h2.z * bc.z; uv.y = h0.w * bc.x + h1.w * bc.y + h2.w * bc.z; }
    else { uv.x = bc.y; uv.y = bc.z; }
    if (b.reflTex) b.refl = tex_eval(A_.g, b.reflTex - 1u, uv);
    if (b.bumpTex) {
        const float2 grad = tex_gradient_lum(A_.g, b.bumpTex - 1u, uv);
        const float3 dP1 = f3(g1.x - g0.x, g1.y - g0.y, g1.z - g0.z), dP2 = f3(g2.x - g0.x, g2.y - g0.y, g2.z - g0.z);
        float3 dpdu0 = dP1, dpdv0 = dP2;
        if (hasUv) {
            const float du1 = h1.z - h0.z, dv1 = h1.w - h0.w, du2 = h2.z - h0.z, dv2 = h2.w - h0.w;
            const float3 n = cross(dP1, dP2); const float len = sqrtf(dot(n, n));
            if (len == 0.f) dpdu0 = dpdv0 = f3(0, 0, 0);
            else {
                const float determinant = du1 * dv2 - dv1 * du2;
                if (determinant == 0.f) coordinate_system(n * (1.0f / len), dpdu0, dpdv0);
                else { const float invDet = 1.0f / determinant; dpdu0 = (dP1 * dv2 - dP2 * dv1) * invDet; dpdv0 = (dP1 * (-du2) + dP2 * du1) * invDet; }
            }
        }
        const float3 dpdu = dpdu0 + its.shN * (grad.x - dot(its.shN, dpdu0)), dpdv = dpdv0 + its.shN * (grad.y - dot(its.shN, dpdv0));
        float3 n = normalize(cross(dpdu, dpdv));
        its.shS = normalize(dpdu - n * dot(n, dpdu));
        its.shT = cross(n, its.shS);
        if (dot(n, its.geoN) < 0.f) n = n * -1.0f;
        its.shN = n;
        its.wi = its.toLocal(-rayD);
    }
}

// ------------------------------------------------------------------ SD-tree views
// S-tree node: uint2 {child0, child1}; child0 == 0 marks a leaf (node 0 is the root, never a child; GP:844).
// Axis cycles x,y,z with depth (root 0, children (axis+1)%3, GP:889), so it is not stored.
// Per-node leaf record (valid for leaves):
//   leafA[n] = {bits(samplingBase), bits(buildingBase), theta (Adam variable), bits(flags)}  flags bit0: sampling mean()>0
// Sampling quadtree node: 32 B = float4 sums + uint2 children (4 x uint16, 0 = leaf; GP:368-370) + pad,
// read with one 16 B and one 8 B load from the same 32 B sector.
struct SampNode { float4 sums; uint2 children; uint2 pad; };
struct TreeView {
    const uint2 *snodes;
    const uint32_t *stable;       // S-tree prefix table (see stree_lookup), or nullptr
    const float4 *leafA;
    const SampNode *samp;         // sampling pool
    const uint2 *bchildren;       // building pool topology (4 x uint16 per node)
    float4 *bsums;                // building pool sums (atomics target)
    float *bweight;               // per S-tree node: building statistical weight (atomics target)
    float3 aabbMin, extent;       // cubified scene box (GP:850-860)
};

// DTree::mean() (GP:387-393) of a tree whose m_atomic holds `sum` and statistical weight `weight`; mean > 0 is the flag bit of leafA
__host__ __device__ __forceinline__ float dtree_mean(float sum, float weight) {
    float mean = 0.f;
    if (weight != 0.f) { const float factor = 1.f / (PPG_PI * 4.f * weight); mean = factor * sum; }
    return mean;
}

__device__ __forceinline__ uint32_t child16(uint2 c, int i) { return ((i & 2) ? c.y : c.x) >> ((i & 1) * 16) & 0xffffu; }
__device__ __forceinline__ float sum4(float4 s, int i) { return i == 0 ? s.x : (i == 1 ? s.y : (i == 2 ? s.z : s.w)); }

// STree::dTreeWrapper(p, size) -- GP:897-905 + 761-769 + 747-755.  Returns the leaf node index and the
// number of levels descended (the voxel size follows from it: size[axis] halves once per level on that axis).
//
// The reference walks one node per level (~18 dependent loads on CBOX).  Because every split is at the midpoint and
// the axes cycle x,y,z, the first 3*B levels of the walk are exactly the B leading binary digits of each normalised
// coordinate (p < 0.5 ? 2p : 2p-1 is exact in fp32), so a prefix table indexed by the interleaved digits replaces them
// with ONE load; the walk then continues from the table's node with the exact remainders 2^B*p - floor(2^B*p).
// Table entry: node | levels<<24 | leaf<<31 (built by stree_table_kernel after every refine).  The node number has 24 bits, so the
// table serves S-trees of at most 0xFFFFFF nodes (stree_table_usable); a larger tree is looked up with table == nullptr, the plain
// walk from the root, which is the reference's walk and returns the same leaf bit for bit.
constexpr int PPG_STREE_TABLE_BITS = 7;     // digits per axis -> 3*7 = 21 levels, 2^21 entries (8 MB, L2 resident; CBOX 1024^2 descends 18.5 levels on average)
// whether stree_table_kernel's entries can hold every node number of an S-tree of n_nodes nodes (host side: pass the table or nullptr)
inline bool stree_table_usable(size_t n_nodes) { return n_nodes <= 0x00ffffffu; }
__device__ __forceinline__ uint32_t spread3(uint32_t v) {   // bit i -> bit 3i (7 bits)
    return (v & 1u) | ((v & 2u) << 2) | ((v & 4u) << 4) | ((v & 8u) << 6) | ((v & 16u) << 8) | ((v & 32u) << 10) | ((v & 64u) << 12);
}
__device__ __forceinline__ uint32_t stree_lookup(const uint2 *__restrict__ snodes, const uint32_t *__restrict__ table, float3 aabbMin, float3 extent,
                                                 float3 pw, int &levels) {
    // p0 is the coordinate of the current split axis; the triple rotates with the axis (no dynamic indexing)
    float p0 = (pw.x - aabbMin.x) / extent.x, p1 = (pw.y - aabbMin.y) / extent.y, p2 = (pw.z - aabbMin.z) / extent.z;
    uint32_t n = 0; int depth = 0;
    if (table) {
        const float S = (float) (1 << PPG_STREE_TABLE_BITS), M = S - 1.0f;
        // digits: clamp(floor(S*p), 0, S-1); p >= 1 keeps taking the upper child and p < 0 the lower one, exactly like the walk
        const float f0 = fminf(fmaxf(floorf(p0 * S), 0.f), M), f1 = fminf(fmaxf(floorf(p1 * S), 0.f), M), f2 = fminf(fmaxf(floorf(p2 * S), 0.f), M);
        const uint32_t key = (spread3((uint32_t) f0) << 2) | (spread3((uint32_t) f1) << 1) | spread3((uint32_t) f2);
        const uint32_t e = __ldg(&table[key]);
        n = e & 0x00ffffffu; depth = (int) ((e >> 24) & 0x7fu);
        if (e >> 31) { levels = depth; return n; }
        p0 = p0 * S - f0; p1 = p1 * S - f1; p2 = p2 * S - f2;       // exact remainders; depth == 3*BITS here, next axis is x again
    }
    for (;;) {
        const uint2 c = __ldg(&snodes[n]);
        if (c.x == 0u) break;
        if (p0 < 0.5f) { p0 *= 2.f; n = c.x; } else { p0 = (p0 - 0.5f) * 2.f; n = c.y; }
        const float t = p0; p0 = p1; p1 = p2; p2 = t;
        ++depth;
    }
    levels = depth;
    return n;
}
__device__ __forceinline__ float3 voxel_size(float3 extent, int levels) {
    // size[a] /= 2 once per level whose axis is a (exact powers of two)
    const int nx = (levels + 2) / 3, ny = (levels + 1) / 3, nz = levels / 3;
    return f3(ldexpf(extent.x, -nx), ldexpf(extent.y, -ny), ldexpf(extent.z, -nz));
}

// DTreeWrapper::dirToCanonical -- GP:597-608
__device__ __forceinline__ float2 dir_to_canonical(float3 d) {
    if (!isfinite(d.x) || !isfinite(d.y) || !isfinite(d.z)) return make_float2(0.f, 0.f);
    const float cosTheta = fminf(fmaxf(d.z, -1.0f), 1.0f);
    float phi = atan2f(d.y, d.x);
    while (phi < 0.f) phi += 2.0f * PPG_PI;   // == the reference's double add rounded to float (both addends are floats)
    return make_float2((cosTheta + 1.f) / 2.f, phi / (2.f * PPG_PI));
}
// DTreeWrapper::canonicalToDir -- GP:586-595
__device__ __forceinline__ float3 canonical_to_dir(float2 p) {
    const float cosTheta = 2.f * p.x - 1.f;
    const float phi = 2.f * PPG_PI * p.y;
    const float sinTheta = sqrtf(1.f - cosTheta * cosTheta);
    float s, c; sincosf_bounded(phi, &s, &c);                                  // p.y in [0, 1]
    return f3(sinTheta * c, sinTheta * s, cosTheta);
}

// QuadTreeNode::childIndex -- GP:205-217
__device__ __forceinline__ int quad_child_index(float2 &p) {
    int res = 0;
    if (p.x < 0.5f) p.x *= 2.f; else { p.x = (p.x - 0.5f) * 2.f; res |= 1; }
    if (p.y < 0.5f) p.y *= 2.f; else { p.y = (p.y - 0.5f) * 2.f; res |= 2; }
    return res;
}

// DTree::pdf -- GP:415-421 + 232-245 (valid == mean() > 0).  Product accumulated top-down.
template <class NodeT>
__device__ __forceinline__ float dtree_pdf(const NodeT *__restrict__ tree, bool valid, float2 p) {
    if (!valid) return 1.0f / (4.0f * PPG_PI);
    float result = 1.0f; uint32_t n = 0;
    for (;;) {
        const float4 s = __ldg(&tree[n].sums);
        const uint2 ch = __ldg(&tree[n].children);
        const int c = quad_child_index(p);
        const float sc = sum4(s, c);
        if (!(sc > 0.f)) return 0.f;
        result *= 4.f * sc / (s.x + s.y + s.z + s.w);
        const uint32_t next = child16(ch, c);
        if (next == 0u) break;
        n = next;
    }
    return result / (4.0f * PPG_PI);
}

// DTree::sample -- GP:431-442 + 257-301.  One uniform per level, re-stretched; two at the leaf.
// The reference evaluates origin_0 + 0.5*(origin_1 + 0.5*(... + 0.5*next2D)) from the leaf upward;
// the per-level origin bits are kept in two masks and folded in that same order.
template <class NodeT, class RngT>
__device__ __forceinline__ float2 dtree_sample(const NodeT *__restrict__ tree, bool valid, RngT &rng) {
    float2 res;
    if (!valid) { res.x = rng.next1D(); res.y = rng.next1D(); return res; }
    uint32_t bx = 0, by = 0; int levels = 0; uint32_t n = 0;
    for (;;) {
        const float4 s = __ldg(&tree[n].sums);
        const uint2 ch = __ldg(&tree[n].children);
        int index = 0;
        const float topLeft = s.x, topRight = s.y;
        float partial = topLeft + s.z;
        const float total = partial + topRight + s.w;
        if (!(total > 0.0f)) { res.x = rng.next1D(); res.y = rng.next1D(); break; }
        float boundary = partial / total;
        float smp = rng.next1D();
        if (smp < boundary) {
            smp /= boundary;
            boundary = topLeft / partial;
        } else {
            partial = total - partial;
            smp = (smp - boundary) / (1.0f - boundary);
            boundary = topRight / partial;
            index |= 1;
        }
        if (smp < boundary) {
            smp /= boundary;
        } else {
            smp = (smp - boundary) / (1.0f - boundary);
            index |= 2;
        }
        bx |= (uint32_t) (index & 1) << levels; by |= (uint32_t) ((index >> 1) & 1) << levels; ++levels;
        const uint32_t next = child16(ch, index);
        if (next == 0u) { res.x = rng.next1D(); res.y = rng.next1D(); break; }
        n = next;
    }
    for (int i = levels - 1; i >= 0; --i) {
        res.x = ((bx >> i) & 1u ? 0.5f : 0.0f) + 0.5f * res.x;
        res.y = ((by >> i) & 1u ? 0.5f : 0.0f) + 0.5f * res.y;
    }
    res.x = fminf(fmaxf(res.x, 0.0f), 1.0f);
    res.y = fminf(fmaxf(res.y, 0.0f), 1.0f);
    return res;
}

// red.global.add.f32 without a return value
__device__ __forceinline__ void red_add(float *addr, float v) { atomicAdd(addr, v); }

// Add `w` to counters[key] with one atomic per distinct key per warp (the statistical-weight counter of
// a D-tree is a single address that every vertex of that leaf hits: in iteration 0 that is ONE address
// for the whole wavefront).  Lanes with equal (key, w) are merged: leader adds popc * w.
__device__ __forceinline__ void warp_aggregated_add(float *counters, uint32_t key, float w, bool active) {
    const unsigned m = __ballot_sync(0xffffffffu, active);
    if (!active) return;
    const unsigned long long k = ((unsigned long long) key << 32) | __float_as_uint(w);
    const unsigned peers = __match_any_sync(m, k);
    const int leader = __ffs(peers) - 1;
    if ((threadIdx.x & 31) == leader) red_add(&counters[key], w * (float) __popc(peers));
}

// QuadTreeNode::record (nearest) -- GP:303-312
__device__ __forceinline__ void dtree_record_nearest(const uint2 *__restrict__ bchildren, float4 *bsums, uint32_t base, float2 p, float value) {
    uint32_t n = 0;
    for (;;) {
        const int c = quad_child_index(p);
        const uint32_t next = child16(__ldg(&bchildren[base + n]), c);
        if (next == 0u) { red_add(reinterpret_cast<float *>(&bsums[base + n]) + c, value); return; }
        n = next;
    }
}
// DTree::depthAt -- GP:423-425 + 247-255
__device__ __forceinline__ int dtree_depth_at(const uint2 *__restrict__ bchildren, uint32_t base, float2 p) {
    int d = 1; uint32_t n = 0;
    for (;;) {
        const int c = quad_child_index(p);
        const uint32_t next = child16(__ldg(&bchildren[base + n]), c);
        if (next == 0u) return d;
        n = next; ++d;
    }
}
// QuadTreeNode::record (box footprint) -- GP:322-338 + 314-320; explicit stack, no wrap-around, no clamping
__device__ __forceinline__ void dtree_record_box(const uint2 *__restrict__ bchildren, float4 *bsums, uint32_t base, float2 origin, float size, float value) {
    struct E { uint32_t n; float ox, oy, s; };
    E st[48]; int sp = 0;
    st[sp++] = E{0u, 0.f, 0.f, 1.0f};
    while (sp) {
        const E e = st[--sp];
        const float childSize = e.s / 2.f;
        const uint2 ch = __ldg(&bchildren[base + e.n]);
        for (int i = 0; i < 4; ++i) {
            float cox = e.ox, coy = e.oy;
            if (i & 1) cox += childSize;
            if (i & 2) coy += childSize;
            const float lx = fmaxf(fminf(origin.x + size, cox + childSize) - fmaxf(origin.x, cox), 0.0f);
            const float ly = fmaxf(fminf(origin.y + size, coy + childSize) - fmaxf(origin.y, coy), 0.0f);
            const float w = lx * ly;
            if (w > 0.0f) {
                const uint32_t next = child16(ch, i);
                if (next == 0u) red_add(reinterpret_cast<float *>(&bsums[base + e.n]) + i, value * w);
                else if (sp < 48) st[sp++] = E{next, cox, coy, childSize};
            }
        }
    }
}
// DTree::recordIrradiance -- GP:395-413 (the statistical-weight add is done by the caller, warp-aggregated)
__device__ __forceinline__ void dtree_record_irradiance(const uint2 *__restrict__ bchildren, float4 *bsums, uint32_t base, float2 p,
                                                        float irradiance, float statisticalWeight, int directionalFilter) {
    if (isfinite(irradiance) && irradiance > 0.f) {
        if (directionalFilter == 0) dtree_record_nearest(bchildren, bsums, base, p, irradiance * statisticalWeight);
        else {
            const int depth = dtree_depth_at(bchildren, base, p);
            const float size = ldexpf(1.0f, -depth);          // std::pow(0.5f, depth), exact
            float2 origin = p;
            origin.x -= size / 2.f; origin.y -= size / 2.f;
            dtree_record_box(bchildren, bsums, base, origin, size, irradiance * statisticalWeight / (size * size));
        }
    }
}

__device__ __forceinline__ float logistic(float x) { return 1.f / (1.f + expf(-x)); }   // GP:64-66

// ------------------------------------------------------------------ next event estimation (GP:1964-2021)
#define PPG_SHADOW_EPSILON 1e-3f
__device__ __forceinline__ float mi_weight(float pdfA, float pdfB) { pdfA *= pdfA; pdfB *= pdfB; return pdfA / (pdfA + pdfB); }   // GP:2247-2250

// DiscreteDistribution::sample (include/mitsuba/core/pmf.h:124-137): lower_bound on the cdf, clamp, skip empty entries
__device__ __forceinline__ uint32_t cdf_sample(const float *__restrict__ cdf, uint32_t size /* entries incl. leading 0 */, float v) {
    uint32_t lo = 0, hi = size;                       // first index with cdf[idx] >= v
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (cdf[mid] < v) lo = mid + 1; else hi = mid; }
    int index = (int) lo - 1; if (index < 0) index = 0; if ((uint32_t) index > size - 2) index = (int) size - 2;
    while (cdf[index + 1] - cdf[index] == 0.f && (uint32_t) index < size - 1) ++index;
    return (uint32_t) index;
}

// The normal ShapeKDTree::rayIntersect(ray, t, shape, n, uv) reports (skdtree.cpp:165-175: plain face normal; spheres: geoFrame.n)
template <class Acc>
__device__ __forceinline__ float3 hit_geo_normal(const Acc &A_, const Hit &h, float3 ro, float3 rd) {
    if (h.prim & PPG_SPHERE_BIT) {
        const uint32_t k = h.prim & ~PPG_SPHERE_BIT;
        const float4 cr = __ldg(&A_.g.spheres[2 * k]), mt = __ldg(&A_.g.spheres[2 * k + 1]);
        const float3 c = f3(cr.x, cr.y, cr.z);
        float3 p = ro + rd * h.t; p = c + normalize(p - c) * cr.w;
        float3 n = normalize(p - c); if (__float_as_uint(mt.z)) n = n * -1.0f;
        return n;
    }
    const float4 g0 = A_.geom(6 * h.tri), g1 = A_.geom(6 * h.tri + 1), g2 = A_.geom(6 * h.tri + 2);
    const float3 p0 = f3(g0.x, g0.y, g0.z), p1 = f3(g1.x, g1.y, g1.z), p2 = f3(g2.x, g2.y, g2.z);
    return normalize(cross(p1 - p0, p2 - p0));
}
template <class Acc> __device__ __forceinline__ int hit_bsdf(const Acc &A_, const Hit &h) {
    return (h.prim & PPG_SPHERE_BIT) ? __float_as_int(__ldg(&A_.g.spheres[2 * (h.prim & ~PPG_SPHERE_BIT) + 1]).x) : A_.meta(h.tri).x;
}
// Scene::evalTransmittance with index-matched surfaces (scene.cpp:619-679, both end points on surfaces): a null surface multiplies its
// straight-through transmittance (evaluated in the GEOMETRIC frame, :650-655) and the ray continues behind it, at most maxInteractions
// times (negative = unlimited); anything else blocks.  Full-feature variants only; not inlined (rare path, keeps the callers' registers).
template <class Acc>
__device__ __noinline__ float3 eval_transmittance(const Acc &A_, float3 p1, float3 d, float remaining, int maxInteractions) {
    const float lengthFactor = 1.f - PPG_SHADOW_EPSILON;
    float3 ro = p1, transmittance = f3(1, 1, 1);
    int interactions = 0;
    float maxt = remaining * lengthFactor;
    while (remaining > 0.f) {
        const float mint = PPG_EPSILON * fmaxf(fmaxf(fabsf(ro.x), fabsf(ro.y)), fabsf(ro.z));
        Hit h;
        if (!bvh_intersect<true>(A_, ro, d, mint, maxt, h)) break;
        const Bsdf b = load_bsdf<true>(A_, hit_bsdf(A_, h));
        if (interactions == maxInteractions || !bsdf_has_null(b)) return f3(0, 0, 0);
        const float3 n = hit_geo_normal(A_, h, ro, d);
        transmittance = transmittance * bsdf_eval_null(b, -dot(n, d));
        if (is_zero(transmittance)) break;
        if (++interactions > 100) break;
        ro = ro + d * h.t; remaining -= h.t; maxt = remaining * lengthFactor;
    }
    return transmittance;
}
// rayIntersectAndLookForEmitter (GP:2184-2245) behind a first hit on an index-matched, non-emitting surface: follow the ray through up to
// maxInteractions null surfaces; returns transmittance * Le of the emitter found (0 if none / blocked) and the query the light-sampling
// pdf needs (emitter, shading normal, distance of the LAST segment -- dRec.setQuery after ray.o has moved, a reference quirk kept).
template <class Acc>
__device__ __noinline__ float3 look_through(const Acc &A_, float3 o, float3 d, const Its &first, float firstT, int maxInteractions,
                                            int &qEmitter, float3 &qN, float &qDist) {
    qEmitter = -1; qN = f3(0, 0, 0); qDist = 0.f;
    float3 ro = o, transmittance = f3(1, 1, 1);
    Its cur = first; float curT = firstT; bool surface = true;
    int interactions = 0;
    for (;;) {
        if (surface) {
            const Bsdf b = load_bsdf<true>(A_, cur.bsdf);
            if (interactions == maxInteractions || !bsdf_has_null(b) || cur.emitter >= 0) break;
            if (is_zero(transmittance)) return f3(0, 0, 0);
            transmittance = transmittance * bsdf_eval_null(b, -dot(d, cur.shN));            // bRec(its, -wo, wo) in the shading frame
        } else break;
        ro = ro + d * curT;
        const float mint = PPG_EPSILON * fmaxf(fmaxf(fmaxf(fabsf(ro.x), fabsf(ro.y)), fabsf(ro.z)), PPG_EPSILON);
        Hit h;
        surface = bvh_intersect<true>(A_, ro, d, mint, __int_as_float(0x7f800000), h);
        if (surface) { fill_its<true>(A_, h, ro, d, cur); curT = h.t; }
        if (++interactions > 100) return f3(0, 0, 0);
    }
    if (!surface) {                                                                         // "perhaps there is an environment map?" (GP:2228-2243)
        if (!A_.g.envW) return f3(0, 0, 0);
        qEmitter = PPG_ENV_EMITTER;                                                         // fillDirectSamplingRecord: dRec.object = the environment emitter
        return transmittance * env_eval(A_.g, d);
    }
    if (cur.emitter < 0) return f3(0, 0, 0);
    qEmitter = cur.emitter; qN = cur.shN; qDist = curT;
    if (!(dot(cur.shN, -d) > 0.f)) return f3(0, 0, 0);
    const float4 r = A_.radiance(cur.emitter);
    return transmittance * f3(r.x, r.y, r.z);
}

struct DirectSample { float3 value, d; float pdf; };
// coordinateSystem(a, b, c), src/libcore/util.cpp:592-601
__device__ __forceinline__ void coordinate_system(float3 a, float3 &b, float3 &c) {
    if (fabsf(a.x) > fabsf(a.y)) { const float invLen = 1.0f / sqrtf(a.x * a.x + a.z * a.z); c = f3(a.z * invLen, 0.0f, -a.x * invLen); }
    else { const float invLen = 1.0f / sqrtf(a.y * a.y + a.z * a.z); c = f3(0.0f, a.z * invLen, -a.y * invLen); }
    b = cross(c, a);
}
// Scene::sampleAttenuatedEmitterDirect (scene.cpp:876-897) -> AreaLight::sampleDirect (area.cpp:158-173) -> Shape::sampleDirect
// (shape.cpp:102-115) -> TriMesh::samplePosition (trimesh.cpp:412-423) -> Triangle::sample (libcore/triangle.cpp:24-59);
// visibility (Scene::evalTransmittance, scene.cpp:619-679) is tested by the caller.  Returns false when the sample carries nothing.
template <bool SPHERES, class Acc>
__device__ __forceinline__ bool sample_emitter_direct(const Acc &A_, float3 ref, float3 refN, float sx, float sy, DirectSample &out, float &dist) {
    const SceneView &sc = A_.g;        // the emitter tables stay in HBM (read-only path)
    const uint32_t ei = cdf_sample(sc.emitterCdf, sc.nLights + 1, sx);
    const float c0 = sc.emitterCdf[ei], c1 = sc.emitterCdf[ei + 1];
    const float emPdf = c1 - c0;
    sx = (sx - c0) / (c1 - c0);
    if (SPHERES && ei == sc.envLight) {                 // EnvironmentMap::sampleDirect, src/emitters/envmap.cpp:516-543 (no dRec.refN test there)
        float3 dl, value; float pdf;
        env_sample_direction(sc, sx, sy, dl, value, pdf);
        const float *m = sc.env->toWorld;
        const float3 d = f3(m[0] * dl.x + m[1] * dl.y + m[2] * dl.z, m[3] * dl.x + m[4] * dl.y + m[5] * dl.z, m[6] * dl.x + m[7] * dl.y + m[8] * dl.z);
        out.d = d;
        // m_sceneBSphere.rayIntersect (bsphere.h:88-95) -> solveQuadratic (util.cpp:447-485): the far intersection carries the sample
        const float3 o = ref - f3(sc.env->center[0], sc.env->center[1], sc.env->center[2]);
        const float A = dot(d, d), B = 2.f * dot(o, d), C = dot(o, o) - sc.env->radius * sc.env->radius;
        if (A == 0.f) return false;
        const float discrim = B * B - 4.0f * A * C;
        if (discrim < 0.f) return false;
        const float sq = sqrtf(discrim), temp = B < 0.f ? -0.5f * (B - sq) : -0.5f * (B + sq);
        float nearT = temp / A, farT = C / temp;
        if (nearT > farT) { const float s_ = nearT; nearT = farT; farT = s_; }
        if (is_zero(value) || pdf == 0.f || nearT >= 0.f || farT <= 0.f) return false;
        dist = farT;
        out.value = (value * (1.0f / pdf)) * (1.0f / emPdf);
        out.pdf = pdf * emPdf;
        return true;
    }
    const float4 info = sc.emitterInfo[ei];
    const uint32_t first = __float_as_uint(info.x), nTris = __float_as_uint(info.y), cdfOff = __float_as_uint(info.w);
    if (SPHERES && (first & PPG_SPHERE_BIT)) {          // Sphere::sampleDirect, src/shapes/sphere.cpp:286-355
        const uint32_t k = first & ~PPG_SPHERE_BIT;
        const float4 cr = __ldg(&sc.spheres[2 * k]), mt = __ldg(&sc.spheres[2 * k + 1]);
        const float3 c = f3(cr.x, cr.y, cr.z);
        const float3 refToCenter = c - ref;
        const float refDist2 = dot(refToCenter, refToCenter);
        const float invRefDist = 1.0f / sqrtf(refDist2);
        const float sinAlpha = cr.w * invRefDist;
        float3 d, n; float pdf;
        if (sinAlpha < 1.f - PPG_EPSILON) {   // outside: uniform cone
            const float cosAlpha = sqrtf(fmaxf(0.0f, 1.0f - sinAlpha * sinAlpha));
            const float3 fn = refToCenter * invRefDist; float3 fs, ft; coordinate_system(fn, fs, ft);
            const float cosTheta = (1.f - sx) + sx * cosAlpha, sinTheta = sqrtf(fmaxf(0.0f, 1.0f - cosTheta * cosTheta));
            float sinPhi, cosPhi; sincosf(2.0f * PPG_PI * sy, &sinPhi, &cosPhi);
            const float3 lv = f3(cosPhi * sinTheta, sinPhi * sinTheta, cosTheta);
            d = fs * lv.x + ft * lv.y + fn * lv.z;
            pdf = (0.5f * PPG_INV_PI) / (1.f - cosAlpha);
            const float projDist = dot(refToCenter, d);
            const float baseT = refDist2 / projDist;
            const float3 query = ref + d * baseT;
            const float3 queryToCenter = c - query;
            const float queryDist2 = dot(queryToCenter, queryToCenter), queryProjDist = dot(queryToCenter, d);
            const float A = 1.0f, B = -2.f * queryProjDist, C = queryDist2 - cr.w * cr.w;
            float nearT;
            { const float discrim = B * B - 4.0f * A * C;                                       // solveQuadratic, util.cpp:447-485
              if (discrim < 0.f) nearT = queryProjDist;
              else { const float sq = sqrtf(discrim); const float temp = B < 0.f ? -0.5f * (B - sq) : -0.5f * (B + sq); float x0 = temp / A, x1 = C / temp; if (x0 > x1) { const float s_ = x0; x0 = x1; x1 = s_; } nearT = x0; } }
            dist = baseT + nearT;
            n = normalize(d * nearT - queryToCenter);
        } else {                             // inside: uniform sphere
            const float z = 1.0f - 2.0f * sy, r = sqrtf(fmaxf(0.0f, 1.0f - z * z));
            float sinPhi, cosPhi; sincosf(2.0f * PPG_PI * sx, &sinPhi, &cosPhi);
            const float3 v = f3(r * cosPhi, r * sinPhi, z);
            const float3 p = c + v * cr.w;
            n = v; d = p - ref;
            const float dist2 = dot(d, d);
            dist = sqrtf(dist2);
            d = d * (1.0f / dist);
            pdf = info.z * dist2 / fabsf(dot(d, n));
        }
        if (__float_as_uint(mt.z)) n = n * -1.0f;
        out.d = d;
        if (!(dot(d, refN) >= 0.f && dot(d, n) < 0.f && pdf != 0.f)) return false;
        const float4 r = A_.radiance(ei);
        out.value = (f3(r.x, r.y, r.z) * (1.0f / pdf)) * (1.0f / emPdf);
        out.pdf = pdf * emPdf;
        return true;
    }
    if (nTris == 0u) return false;
    const float *tcdf = sc.emitterTriCdf + cdfOff;
    const uint32_t ti = cdf_sample(tcdf, nTris + 1, sy);
    sy = (sy - tcdf[ti]) / (tcdf[ti + 1] - tcdf[ti]);
    const uint32_t t = first + ti;
    const float4 g0 = sc.emitterGeom[6 * t], g1 = sc.emitterGeom[6 * t + 1], g2 = sc.emitterGeom[6 * t + 2];
    const float3 p0 = f3(g0.x, g0.y, g0.z), p1 = f3(g1.x, g1.y, g1.z), p2 = f3(g2.x, g2.y, g2.z);
    const float a = sqrtf(fmaxf(0.0f, 1.0f - sx));                                             // warp::squareToUniformTriangle
    const float bx = 1.f - a, by = a * sy;
    const float3 sideA = p1 - p0, sideB = p2 - p0;
    const float3 p = p0 + (sideA * bx) + (sideB * by);
    float3 n;
    if (sc.emitterFlags[ei] & 1u) {
        const float4 h0 = sc.emitterGeom[6 * t + 3], h1 = sc.emitterGeom[6 * t + 4], h2 = sc.emitterGeom[6 * t + 5];
        n = normalize(f3(g0.w, h0.x, h0.y) * (1.0f - bx - by) + f3(g1.w, h1.x, h1.y) * bx + f3(g2.w, h2.x, h2.y) * by);
    } else n = normalize(cross(sideA, sideB));
    float pdf = info.z;
    float3 d = p - ref;
    const float distSquared = dot(d, d);
    dist = sqrtf(distSquared);
    d = d * (1.0f / dist);
    const float dp = fabsf(dot(d, n));
    pdf *= dp != 0.f ? (distSquared / dp) : 0.0f;
    out.d = d;
    if (!(dot(d, refN) >= 0.f && dot(d, n) < 0.f && pdf != 0.f)) return false;
    const float4 r = A_.radiance(ei);
    out.value = (f3(r.x, r.y, r.z) * (1.0f / pdf)) * (1.0f / emPdf);
    out.pdf = pdf * emPdf;
    return true;
}
// Scene::pdfEmitterDirect (scene.cpp:949-952) for an emitter hit found by BSDF / guiding sampling
template <bool SPHERES>
__device__ __forceinline__ float pdf_emitter_direct(const SceneView &sc, int emitter, float3 ref, float3 refN, float3 d, float3 n, float dist) {
    if (SPHERES && emitter == PPG_ENV_EMITTER) return env_pdf_direction(sc, d) * (1.0f * sc.emitterNormalization);   // EnvironmentMap::pdfDirect, ESolidAngle (envmap.cpp:371, 545-548)
    if (!(dot(d, refN) >= 0.f && dot(d, n) < 0.f)) return 0.0f;
    const float4 info = sc.emitterInfo[emitter];
    if (SPHERES && (__float_as_uint(info.x) & PPG_SPHERE_BIT)) {                                            // Sphere::pdfDirect, sphere.cpp:357-392
        const float4 cr = __ldg(&sc.spheres[2 * (__float_as_uint(info.x) & ~PPG_SPHERE_BIT)]);
        const float3 refToCenter = f3(cr.x, cr.y, cr.z) - ref;
        const float invRefDist = 1.0f / sqrtf(dot(refToCenter, refToCenter));
        const float sinAlpha = cr.w * invRefDist;
        float pdfSA;
        if (sinAlpha < 1.f - PPG_EPSILON) { const float cosAlpha = sqrtf(fmaxf(0.0f, 1.f - sinAlpha * sinAlpha)); pdfSA = (0.5f * PPG_INV_PI) / (1.f - cosAlpha); }
        else pdfSA = info.z * dist * dist / fabsf(dot(d, n));
        return pdfSA * (1.0f * sc.emitterNormalization);
    }
    return sc.emitterInfo[emitter].z * (dist * dist) / fabsf(dot(d, n)) * (1.0f * sc.emitterNormalization);
}

}  // namespace ppg
