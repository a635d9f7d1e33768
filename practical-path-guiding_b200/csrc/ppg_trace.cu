// ppg_trace.cu -- nearest-hit pass for scenes that are walked through the BVH (everything that does not fit shared memory).
//
// Inside the fused bounce kernel a warp's 32 rays walk the BVH together and the warp waits for its longest walk: ncu on KITCHEN
// (profiles/r02_kitchen_bounce.md) shows 3.7 of 32 lanes active in the box test and 1.5 in the triangle test -- walk lengths inside a
// warp differ by ~8x.  This kernel does the walks alone, with persistent warps in the manner of Aila & Laine ("Understanding the
// efficiency of ray traversal on GPUs"): a lane whose ray is finished takes the NEXT unclaimed ray of the launch instead of waiting, and
// the walk is while-while (all lanes descend to a leaf, then all test triangles).  It writes {t, u, v, slot} per input path; the bounce
// kernel that follows reads the hit instead of walking (RenderParams::hits).  Rays, tests and the tie rule (lower original triangle index)
// are the ones of bvh_walk / bvh_intersect in ppg_device.cuh, so the hit set is identical whichever kernel finds it
// (tests/test_gpu_parity.py renders both ways).
//
// Reference: ShapeKDTree::rayIntersect skdtree.cpp:112-142 (nearest hit, adaptive epsilon), renderBlock's camera ray GP:1613-1632.
#include "ppg_wavefront.cuh"
#include <cstdlib>

namespace ppg {

constexpr int PPG_TRACE_BLOCK = 256;
constexpr int PPG_TRACE_MIN_BLOCKS = 4;
constexpr unsigned PPG_TRACE_REFILL = 8u;    // idle lanes that trigger a refill (one atomic per refill and warp)
constexpr int PPG_TRACE_STEPS = 16;          // inner-node steps a lane may take before the warp looks at leaves / refills again

template <bool FIRST, bool SPHERES>
__global__ void __launch_bounds__(PPG_TRACE_BLOCK, PPG_TRACE_MIN_BLOCKS) trace_kernel(const __grid_constant__ RenderParams P) {
    const SceneAccess<false> A_(P.scene);
    const SceneView &sc = P.scene;
    const uint32_t nIn = FIRST ? P.nPaths : *P.liveIn;
    const uint32_t nFront = FIRST ? 0u : (uint32_t) *P.splitIn;
    const uint32_t lane = threadIdx.x & 31u, lt = (1u << lane) - 1u;
    bool active = false, done = false, exhausted = false;
    uint32_t my = 0, left = 0, count = 0;
    float3 o = f3(0, 0, 0), d = f3(0, 0, 1), inv = f3(0, 0, 0); float mint = 0.f, maxt = 0.f;
    Hit hit; hit.t = 0.f; hit.u = hit.v = 0.f; hit.tri = 0; hit.prim = 0xFFFFFFFFu;
    uint32_t stackN[PPG_BVH_STACK]; float stackT[PPG_BVH_STACK]; int sp = 0;
    auto pop = [&]() -> bool {
        while (sp > 0) {
            --sp;
            if (stackT[sp] <= hit.t) { left = stackN[sp] & 0x0fffffffu; count = stackN[sp] >> 28; return true; }
        }
        return false;
    };
    for (;;) {
        // ---- refill: idle lanes take the next rays of the launch
        const unsigned idle = __ballot_sync(0xffffffffu, !active);
        const uint32_t nIdle = (uint32_t) __popc(idle);
        if (!exhausted && nIdle >= PPG_TRACE_REFILL) {
            uint32_t base = 0;
            if (lane == 0) base = atomicAdd(P.traceWork, nIdle);
            base = __shfl_sync(0xffffffffu, base, 0);
            if (base + nIdle >= nIn) exhausted = true;
            const uint32_t take = base + (uint32_t) __popc(idle & lt);
            if (!active && take < nIn) {
                my = take;
                if (FIRST) { Pcg32 rng; uint64_t sampleIndex; camera_ray(P, my, rng, sampleIndex, o, d, mint, maxt); }
                else {
                    const uint32_t s = state_slot(my, nFront, P.pathCapacity);       // hits and bins are indexed by `my`, the compact index
                    const float4 a = P.in.s0[s], b = P.in.s1[s];
                    o = f3(a.x, a.y, a.z); d = f3(a.w, b.x, b.y);
                    mint = surface_ray_mint(o); maxt = __int_as_float(0x7f800000);
                }
                hit.t = __int_as_float(0x7f800000); hit.u = hit.v = 0.f; hit.prim = 0xFFFFFFFFu; hit.tri = 0;
                sp = 0; count = 0; left = 0; active = true; done = true;
                // a ray with a non-finite origin or direction is a miss (see the bounce kernel, which also counts it)
                const bool rayOk = isfinite(o.x + o.y + o.z) && isfinite(d.x + d.y + d.z);
                if (!rayOk) { maxt = -1.f; }                      // nothing can be hit: spheres are skipped below as well
                else if (sc.nTris != 0u) {
                    inv = f3(1.0f / d.x, 1.0f / d.y, 1.0f / d.z);
                    const float4 r0 = A_.bvh(0), r1 = A_.bvh(1);
                    float te;
                    if (bvh_slab(o, inv, mint, maxt, r0, r1, te)) { left = __float_as_uint(r0.w); count = __float_as_uint(r1.w); done = false; }
                }
            }
        }
        if (!__any_sync(0xffffffffu, active)) { if (exhausted) break; continue; }

        // ---- inner nodes: every lane descends until it holds a leaf, is done, or has used its budget
        {
            int steps = 0;
            while (active && !done && count == 0u && steps < PPG_TRACE_STEPS) {
                ++steps;
                const float4 a0 = A_.bvh(2 * left), a1 = A_.bvh(2 * left + 1), b0 = A_.bvh(2 * left + 2), b1 = A_.bvh(2 * left + 3);
                float ta, tb;
                const float tmax = fminf(maxt, hit.t);
                const bool ha = bvh_slab(o, inv, mint, tmax, a0, a1, ta), hb = bvh_slab(o, inv, mint, tmax, b0, b1, tb);
                if (ha && hb) {
                    const bool aFirst = ta <= tb;
                    const float4 f0 = aFirst ? b0 : a0, f1 = aFirst ? b1 : a1, n0 = aFirst ? a0 : b0, n1 = aFirst ? a1 : b1;
                    stackN[sp] = __float_as_uint(f0.w) | (__float_as_uint(f1.w) << 28); stackT[sp] = aFirst ? tb : ta; ++sp;
                    left = __float_as_uint(n0.w); count = __float_as_uint(n1.w);
                } else if (ha) { left = __float_as_uint(a0.w); count = __float_as_uint(a1.w); }
                else if (hb) { left = __float_as_uint(b0.w); count = __float_as_uint(b1.w); }
                else done = !pop();
            }
        }
        // ---- leaves: the lanes that hold one test its triangles together
        if (active && !done && count != 0u) {
            for (uint32_t i = left; i < left + count; ++i) {
                const float4 A = A_.accel(3 * i), B = A_.accel(3 * i + 1), C = A_.accel(3 * i + 2);
                float u, v, t;
                if (tri_intersect(A, B, C, o, d, mint, maxt, u, v, t)) {
                    const uint32_t prim = __float_as_uint(C.z);
                    if (t < hit.t || (t == hit.t && prim < hit.prim)) { hit.t = t; hit.u = u; hit.v = v; hit.prim = prim; hit.tri = i; }
                }
            }
            done = !pop();
        }
        // ---- finished rays: spheres (tested after the triangles, bvh_intersect), then the hit record
        if (active && done) {
            uint32_t w = hit.prim == 0xFFFFFFFFu ? 0xFFFFFFFFu : hit.tri;
            if (SPHERES && maxt >= 0.f) {
                for (uint32_t k = 0; k < sc.nSpheres; ++k) {
                    float t;
                    if (sphere_intersect(__ldg(&sc.spheres[2 * k]), o, d, mint, maxt, t) && t < hit.t) { hit.t = t; hit.u = hit.v = 0.f; w = PPG_SPHERE_BIT | k; }
                }
            }
            __stcs(&P.hits[my], make_float4(hit.t, hit.u, hit.v, __uint_as_float(w)));
            if (P.order) {
                // bin of the material class that will shade this path (the BSDF's type id; the last bin takes the misses)
                uint32_t key = PPG_BINS - 1u;
                if (w != 0xFFFFFFFFu) {
                    const int bs = (w & PPG_SPHERE_BIT) ? __float_as_int(__ldg(&sc.spheres[2 * (w & ~PPG_SPHERE_BIT) + 1]).x) : A_.meta(w).x;
                    key = min(__float_as_uint(A_.bsdf(PPG_BSDF_F4 * bs).w) & 0xffu, PPG_BINS - 2u);
                }
                const unsigned here = __activemask();
                const unsigned peers = __match_any_sync(here, key);
                const int leader = __ffs(peers) - 1;
                uint32_t base = 0;
                if ((int) lane == leader) base = atomicAdd(&P.binCount[key], (uint32_t) __popc(peers));
                base = __shfl_sync(peers, base, leader);
                P.order[(size_t) key * P.binStride + base + (uint32_t) __popc(peers & lt)] = my;
            }
            active = false; done = false;
        }
    }
}

void ppg_launch_trace(const RenderParams &P, cudaStream_t stream, int grid, bool first, bool spheres) {
    if (first) { if (spheres) trace_kernel<true, true><<<grid, PPG_TRACE_BLOCK, 0, stream>>>(P); else trace_kernel<true, false><<<grid, PPG_TRACE_BLOCK, 0, stream>>>(P); }
    else { if (spheres) trace_kernel<false, true><<<grid, PPG_TRACE_BLOCK, 0, stream>>>(P); else trace_kernel<false, false><<<grid, PPG_TRACE_BLOCK, 0, stream>>>(P); }
}
int ppg_trace_occupancy() {
    int occ = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, trace_kernel<false, true>, PPG_TRACE_BLOCK, 0);
    return occ;
}

}  // namespace ppg
