// ppg_wavefront.cuh -- structures shared by the wavefront kernels of the guided path tracer (sm_90a).
//
// One pass-batch of N paths is processed as
//     bounce<FIRST>  (ray generation + bounce 1)          GP:1613-1637 + one turn of the Li loop
//     bounce         (one launch per further path depth)  GP:1798-2146
//     commit         (all recorded vertices -> building trees)   GP:2150-2154 -> 1730-1768 -> 575-584
//     film           (per-pixel sum and sum of squares)   GP:1633-1634, imageblock.h:127-186
// Live paths are compacted between bounces (warp ballot + prefix popcount + one atomic per warp, ordered by the next vertex's sampling technique),
// path state is SoA float4 (5 x 16 B per path, coalesced), the scene (CBOX: ~9 KB) is staged in
// shared memory, the read-only sampling trees go through the read-only/L1 path.
#pragma once
#include "ppg_device.cuh"

namespace ppg {

constexpr int PPG_BLOCK = 256;
constexpr int PPG_BOUNCE_BLOCK = 1024;       // threads per block of the bounce kernel: one block per SM stages the scene once (measured 256x4 -> 5589, 512x2 -> 5643,
                                             // 1024x1 -> 5676 Msamples/s on CBOX 1024^2)
constexpr int PPG_BOUNCE_BLOCK_HBM = 256;    // scenes that do not fit shared memory (nothing to stage) keep 256 x 4: SPACESHIP 485 vs 450 Msamples/s of bounce-kernel time,
                                             // 269 vs 232 with the kl loss; the staged CBOX variants gain 1-4 % from 1024 x 1
constexpr int PPG_MIN_BLOCKS = 1;            // resident blocks per SM the bounce kernel is compiled for: 1024 threads x 64 registers = the whole register file
constexpr unsigned PPG_CLAIM = 1u;           // groups of 32 paths a warp claims per atomic (measured on CBOX 1024^2: 1 -> 5585, 4 -> 5385, 16 -> 4819 Msamples/s:
                                             // running warps then sweep ONE contiguous window of the SoA path state)
constexpr int PPG_MIN_BLOCKS_HBM = 4;        // 64 registers as well (beat 80 and 128 on the rough CBOX variants)
#define PPG_MAX_VERTICES 32         // MAX_NUM_VERTICES, GP:1771
#define PPG_INVALID 0xFFFFFFFFu

// ------------------------------------------------------------------ SoA buffers
struct PathState {      // 5 x float4 per path
    float4 *s0;         // o.xyz, d.x
    float4 *s1;         // d.yz, throughput.xy
    float4 *s2;         // throughput.z, eta, Li.xy
    float4 *s3;         // Li.z, bits(pathId), bits(rng.lo), bits(rng.hi)
    float4 *s4;         // bits(sampleIndex.lo), bits(sampleIndex.hi), bits(nVertices | flags<<8), rrRecip
    float4 *s5;         // NEE only: woPdf of the last sampled direction, refN.xyz of the vertex it left (GP:2084-2087)
    float4 *s6;         // NEE only: bits(slab slot of the last vertex | isDelta<<31 | hasVertex<<30), 0, 0, 0
};
#define PPG_FLAG_NULL 2u             // the ray arrived through an index-matched (ENull) transition: plain intersection, no emitter lookup / MIS (GP:2070-2074)
#define PPG_FLAG_UNSCATTERED 4u      // `scattered` is still false (camera ray that has only crossed null surfaces so far)
#define PPG_FLAG_DYING 1u            // lost Russian roulette: trace one more ray for the emitter lookup, then stop (GP:2078-2091 precede GP:2123-2142)

struct VertexSlab {     // one slab per path depth; entry i belongs to the i-th live path of that bounce
    float4 *v0;         // d.xyz, woPdf
    float4 *v1;         // throughput.xyz, bits(leafNode)
    float4 *v2;         // LiPrefix.xyz, bits(pathId | isDelta<<31)   (pathId == PPG_INVALID: no vertex)
    float4 *v3;         // bsdfVal.xyz, bsdfPdf                       (full mode only)
    float4 *v4;         // o.xyz, dTreePdf                            (full mode only)
    float4 *v5;         // bits(sampleIndex.lo), bits(sampleIndex.hi), bits(streeLevels | ordinal<<8), 0   (full mode only)
};

struct RenderParams {
    SceneView scene; Camera cam; TreeView tree;
    PathState in, out;
    VertexSlab slab;               // slab of the CURRENT depth (already offset by the host)
    float4 *liFinal;               // per path: Li.rgb, 1
    const uint32_t *pixelMap;      // local pixel -> x | y<<16
    const uint32_t *liveIn; uint32_t *liveOut;      // device counters
    // Survivors are stored by the sampling technique their next vertex is predicted to take (see warp_compact_split): nFront | nBack << 32
    // of the input / output wavefront.  The input's compact index j lives at state_slot(j, nFront, pathCapacity).
    const unsigned long long *splitIn; unsigned long long *splitOut;
    uint32_t pathCapacity;                          // entries of each PathState array
    uint32_t *work;                                 // dynamic scheduling: next unclaimed input index of this launch (zeroed by the host), or nullptr
    unsigned long long *counters;  // [0]: rays traced, [1]: vertices recorded, [2]: sum of S-tree levels over recorded vertices, [3]: truncated paths,
                                   // [4]: dropped sampling-fraction records, [5]: rays with a non-finite origin / direction
    uint32_t nPaths;               // paths of this batch (FIRST kernel)
    uint32_t nLocalPixels, spp;
    uint64_t passBase;             // global index of the first pass in the batch
    uint64_t seed;
    int depth;                     // rRec.depth of this bounce (1 = primary hit)
    int maxDepth, rrDepth;
    int strictNormals, hideEmitters;
    int isBuilt;                   // m_isBuilt: guide with the sampling trees
    int lossMode;                  // bsdfSamplingFractionLoss
    float fixedFraction;           // bsdfSamplingFraction
    uint32_t sceneSmemBytes;       // >0: stage the scene into shared memory
    int neeMode, doNee;            // m_nee, m_doNee (GP:1331-1340)
    int training;                  // vertex records are being written in this iteration (the last bounce kernel itself runs with RECORD == 0)
    VertexSlab neeSlab;            // half-weight vertices of the sampled light directions (GP:1999-2016), slab of the current depth
    VertexSlab prevSlab;           // slab of depth-1 (nee == always: the vertex's radiance excludes the emitter hit that follows it, GP:2101)
    float4 *hits;                  // nullptr: the bounce kernel intersects its own ray.  Otherwise trace_kernel (ppg_trace.cu) has left the nearest hit of
                                   // input path i here: {t, u, v, bits(w)}, w = 0xFFFFFFFF miss | PPG_SPHERE_BIT + sphere | triangle slot
    uint32_t *traceWork;           // trace_kernel: next unclaimed ray (zeroed by the host)
    // Material binning (with `hits`): trace_kernel appends every finished ray to the bin of the BSDF class it hit (PPG_BINS - 1: miss);
    // the bounce kernel walks the bins one after the other, so that the 32 paths of a warp shade the same kind of material.
    uint32_t *order;               // [PPG_BINS x binStride] input path indices, or nullptr
    uint32_t *binCount;            // [PPG_BINS] fill of each bin (zeroed by the host)
    uint32_t binStride;
};
#define PPG_BINS 16u

// renderBlock's ray (GP:1613-1632): pixel of path i of the batch, the path's random stream, the jittered film position, the camera ray.
// Shared by the bounce kernel and the trace kernel, which must generate bit-identical rays.
__device__ __forceinline__ void camera_ray(const RenderParams &P, uint32_t i, Pcg32 &rng, uint64_t &sampleIndex, float3 &o, float3 &d, float &mint, float &maxt) {
    const uint32_t perPass = P.nLocalPixels * P.spp;
    const uint32_t passInBatch = i / perPass, rem = i - passInBatch * perPass;
    const uint32_t lp = rem / P.spp, s = rem - lp * P.spp;
    const uint32_t xy = __ldg(&P.pixelMap[lp]);
    const uint32_t x = xy & 0xffffu, y = xy >> 16;
    sampleIndex = (((P.passBase + passInBatch) * (uint64_t) P.cam.H + y) * (uint64_t) P.cam.W + x) * P.spp + s;
    seed_path_rng(rng, P.seed, sampleIndex);
    const float jx = rng.next1D(), jy = rng.next1D();                 // samplePos = pixel + next2D (GP:1620)
    const float sx = ((float) x + jx) * (1.0f / (float) P.cam.W), sy = ((float) y + jy) * (1.0f / (float) P.cam.H);
    const float3 nearP = f3((1.0f - 2.0f * sx) * P.cam.tanX, (1.0f - 2.0f * sy) * P.cam.tanY, 1.0f);
    const float3 dl = normalize(nearP);
    const float invZ = 1.0f / dl.z;
    mint = P.cam.nearClip * invZ; maxt = P.cam.farClip * invZ;
    o = P.cam.o;
    d = P.cam.left * dl.x + P.cam.up * dl.y + P.cam.dir * dl.z;
}
// adaptive ray epsilon of rays leaving a surface (skdtree.cpp:125-128)
__device__ __forceinline__ float surface_ray_mint(float3 o) { return PPG_EPSILON * fmaxf(fmaxf(fmaxf(fabsf(o.x), fabsf(o.y)), fabsf(o.z)), PPG_EPSILON); }

// warp-wide compaction: returns the output slot of this lane (valid when `alive`); no block barrier, so warps of a block never wait for
// each other inside the path loop.  The survivors are split by `back` (the next vertex is predicted to sample the D-tree): front paths fill
// the PathState from slot 0 upward, back paths from slot cap - 1 downward, so that a guided warp of the next bounce holds lanes of one
// technique and issues one branch of sampleMat (only the warp that straddles the boundary holds both).  One returning 64-bit atomic per
// warp on split = nFront | nBack << 32 claims both ranges; the total (liveOut: commit's slab counts, the host's read-back) is added
// without waiting for its result.
__device__ __forceinline__ uint32_t warp_compact_split(bool alive, bool back, unsigned long long *split, uint32_t *total, uint32_t cap) {
    const unsigned live = __ballot_sync(0xffffffffu, alive), backs = __ballot_sync(0xffffffffu, alive && back);
    const int lane = threadIdx.x & 31;
    unsigned long long base = 0;
    if (lane == 0 && live) {
        const uint32_t nAlive = __popc(live), nBack = __popc(backs);
        base = atomicAdd(split, (unsigned long long) (nAlive - nBack) | ((unsigned long long) nBack << 32));
        atomicAdd(total, nAlive);
    }
    base = __shfl_sync(0xffffffffu, base, 0);
    const unsigned below = (1u << lane) - 1u;
    return back ? cap - 1u - ((uint32_t) (base >> 32) + __popc(backs & below)) : (uint32_t) base + __popc(live & ~backs & below);
}
// PathState slot of compact index j of a wavefront written by warp_compact_split (nFront: the low half of its split counter): compact indices
// enumerate the front range, then the back range from its first-written slot.  Slabs, hit records and material bins keep using j.
__device__ __forceinline__ uint32_t state_slot(uint32_t j, uint32_t nFront, uint32_t cap) {
    return j < nFront ? j : cap - 1u - (j - nFront);
}

// The bounce kernel itself lives in ppg_bounce.cuh; it is compiled in four translation units (ppg_bounce_inst.cu with
// -DPPG_INST_SMEM / -DPPG_INST_FULL) so that the 40 instantiations build in parallel.  Host-callable launchers:
struct BounceLaunch { cudaStream_t stream; int grid; int record; int nee; int first; };
void ppg_launch_bounce_00(const RenderParams &P, const BounceLaunch &L); void ppg_launch_bounce_01(const RenderParams &P, const BounceLaunch &L);   // <SMEM, FULL>
void ppg_launch_bounce_10(const RenderParams &P, const BounceLaunch &L); void ppg_launch_bounce_11(const RenderParams &P, const BounceLaunch &L);
// Separate nearest-hit pass for scenes that are walked through the BVH (ppg_trace.cu): persistent warps that refill idle lanes with new rays.
void ppg_launch_trace(const RenderParams &P, cudaStream_t stream, int grid, bool first, bool spheres);
int ppg_trace_occupancy();
int ppg_bounce_occupancy_00(size_t smem); int ppg_bounce_occupancy_01(size_t smem); int ppg_bounce_occupancy_10(size_t smem); int ppg_bounce_occupancy_11(size_t smem);

}  // namespace ppg
