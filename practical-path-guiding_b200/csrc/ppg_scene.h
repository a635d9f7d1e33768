// ppg_scene.h -- host-only scene packing: a ppg_scene_desc validated and turned into the arrays of ppg_scene_layout.h (BVH, coplanar groups,
// Wald rows, vertex slabs, material records, emitter and environment CDFs, repacked texels, camera).  No CUDA runtime calls: the library
// uploads what pack_scene returns, and the CPU tests run the device code on the very same arrays.
#pragma once
#include "../../include/ppg.h"
#include "ppg_scene_layout.h"

#include <cstddef>
#include <string>
#include <vector>

namespace ppg {

// Threads of the host-side loops (PPG_HOST_THREADS, default: the cores this process may run on, at most 16).
int host_threads();

struct HostBvh {
    std::vector<float> nodes;        // 8 floats per node
    std::vector<uint32_t> order;     // leaf order -> original triangle
    int maxDepth = 0;                // the device walk keeps one stack entry per level (PPG_BVH_STACK)
};
// Binned-SAH BVH over the triangles; the result does not depend on `threads`.
HostBvh build_bvh(const float *positions, const uint32_t *indices, uint32_t nTriangles, int threads);

// DiscreteDistribution::normalize on a cumulative table c[0..n]: scales c[1..n-1] by 1 / c[n] and sets c[n] = 1.  Returns 1 / c[n].
// The caller decides what a zero sum means.
float normalize_cdf(float *c, size_t n);

// The device arrays of a scene, in upload order.
enum SceneArray {
    kAccel, kGeom, kMeta, kBvh, kBsdf, kBsdfTables, kRadiance, kGroups, kEmitterCdf, kEmitterInfo, kEmitterTriCdf, kEmitterGeom, kEmitterFlags,
    kSpheres, kTexMeta, kTexels, kEnvTexels, kEnvCdfRows, kEnvCdfCols, kEnvRowWeights, kSceneArrays
};

struct PackedScene {
    std::vector<float> accel, geom, bvh, bsdf, bsdfTables, radiance, groups, emitterCdf, emitterInfo, emitterTriCdf, emitterGeom, spheres, texMeta,
        envCdfRows, envCdfCols, envRowWeights;
    std::vector<int32_t> meta;
    std::vector<uint32_t> emitterFlags;
    std::vector<uint2> texels, envTexels;   // the environment arrays are empty without an environment emitter
    SceneView view{};      // counts and scalars; bind_scene sets the array pointers
    EnvLight env{};        // scalars of the environment emitter (view.envW != 0); bind_scene sets the table pointers
    Camera cam{};
    float aabbMin[3] = {}, aabbMax[3] = {}, extent[3] = {};   // extent: the S-tree's cube (STree::STree, GP:850-860)
    int W = 0, H = 0;
    uint32_t nRealEmitters = 0, sceneSmemBytes = 0;          // sceneSmemBytes: 0 = the kernels read the scene from HBM
    bool fullFeature = false;                                // the scene needs the full-feature kernel variants

    struct Span { const void *data; size_t bytes; };
    Span array(int i) const;                                 // data == nullptr when the array is empty
};

// Validates `s` and packs it.  Returns PPG_OK, or a ppg_status with the reason in `error` (then `out` is unspecified).
int pack_scene(const ppg_scene_desc &s, PackedScene &out, std::string &error);

// Sets the array pointers of `v` and `env` to addr(i), the address array i of `p` has where the kernels read it (nullptr for an empty array),
// and v.env to `envAt` when the scene has an environment emitter.  Everything else comes from p.view and p.env.
template <class Addr> void bind_scene(const PackedScene &p, Addr addr, const EnvLight *envAt, SceneView &v, EnvLight &env) {
    v = p.view; env = p.env;
    v.accel = (const float4 *) addr(kAccel); v.geom = (const float4 *) addr(kGeom); v.meta = (const int4 *) addr(kMeta); v.bvh = (const float4 *) addr(kBvh);
    v.bsdf = (const float4 *) addr(kBsdf); v.bsdfTables = (const float *) addr(kBsdfTables); v.radiance = (const float4 *) addr(kRadiance);
    v.groups = (const float4 *) addr(kGroups);
    v.emitterCdf = (const float *) addr(kEmitterCdf); v.emitterInfo = (const float4 *) addr(kEmitterInfo); v.emitterTriCdf = (const float *) addr(kEmitterTriCdf);
    v.emitterGeom = (const float4 *) addr(kEmitterGeom); v.emitterFlags = (const uint32_t *) addr(kEmitterFlags);
    v.spheres = (const float4 *) addr(kSpheres); v.texMeta = (const float4 *) addr(kTexMeta); v.texels = (const uint2 *) addr(kTexels);
    v.envTexels = (const uint2 *) addr(kEnvTexels);
    env.cdfRows = (const float *) addr(kEnvCdfRows); env.cdfCols = (const float *) addr(kEnvCdfCols); env.rowWeights = (const float *) addr(kEnvRowWeights);
    v.env = p.view.envW ? envAt : nullptr;
}

}  // namespace ppg
