// ppg_scene_layout.h -- the scene as the kernels read it: the arrays ppg_scene.cpp packs on the host and ppg_device.cuh reads on the device.
// Plain structs over CUDA's vector types, so that both host-only code and device code include it.
#pragma once
#include <vector_types.h>
#include <stdint.h>

namespace ppg {

#define PPG_BRUTE_FORCE_TRIS 64u  // scenes with at most this many triangles may take the coplanar-group test instead of the BVH walk
#define PPG_SPHERE_BIT 0x80000000u
#define PPG_BVH_STACK 64          // the host builder refuses deeper trees

// ------------------------------------------------------------------ scene in HBM / shared memory
// Triangles are stored in BVH-leaf order.  Per triangle:
//   accel[3t+0] = {n_u, n_v, n_d, bits(k)}            Wald projection test constants
//   accel[3t+1] = {a_u, a_v, b_nu, b_nv}              (restated from render/triaccel.h:60-158)
//   accel[3t+2] = {c_nu, c_nv, bits(origPrim), bits(meta index == t)}
//   geom[6t+0..2] = {p_i.xyz, n_i.x}, geom[6t+3..5] = {n_i.yz, uv_i}   (i = 0,1,2)
//   meta[t] = {bsdf, emitter (-1 none), flags (bit0 has_normals), shape}
// BVH node: 2 x float4 = {bmin.xyz, bits(left)}, {bmax.xyz, bits(count)}; count>0 -> leaf [left, left+count)
// Material: 7 float4 = {reflectance.rgb, bits(type | flags<<8)}, {specularTransmittance.rgb, eta}, {eta.rgb, 1/eta}, {k.rgb, alpha (negative: Beckmann,
// else GGX)}, {specularReflectance.rgb, fdrInt}, {specularSamplingWeight, bits(table), bits(reflectanceTexture), bits(bumpTexture)},
// {opacity.rgb, luminance(opacity)} (mask flag)
#define PPG_BSDF_F4 7      // float4 per material, see load_bsdf
#define PPG_BSDF_LUT 100   // PPG_BSDF_TABLE_SIZE
struct SceneView {
    const float4 *accel;
    const float4 *geom;
    const int4 *meta;
    const float4 *bvh;
    const float4 *bsdf;       // PPG_BSDF_F4 per material, see load_bsdf
    const float4 *spheres;    // analytic spheres (sphere.cpp): [2k] = {center.xyz, radius}, [2k+1] = {bits(bsdf), bits(emitter), bits(flipNormals), -}
    uint32_t nSpheres;
    const float *bsdfTables;  // roughplastic: PPG_BSDF_LUT floats per table (external rough transmittance), read through L1/L2
    const float4 *radiance;   // per emitter: rgb
    uint32_t nTris, nBvhNodes, nBsdfs, nEmitters;
    // brute-force layout (nTris <= PPG_BRUTE_FORCE_TRIS): coplanar triangle groups ordered by projection axis k.
    //   groups[2q+0] = {n_u, n_v, n_d, bits(firstTri | count<<16)}   plane of the group's first triangle
    //   groups[2q+1] = {umin, vmin, umax, vmax}                      padded bounds of the group in the projection plane
    const float4 *groups;
    uint32_t nGroups;
    // next event estimation (nee != never): discrete emitter choice + per-emitter triangle area distribution
    //   emitterCdf[nEmitters+1]; emitterInfo[e] = {bits(firstTri into emitterGeom), bits(nTris), invArea, bits(cdfOffset into emitterTriCdf)}
    //   emitterGeom: 6 float4 per emitter triangle in ORIGINAL order (same packing as geom); emitterFlags[e] bit0: has vertex normals
    const float *emitterCdf; const float4 *emitterInfo; const float *emitterTriCdf; const float4 *emitterGeom; const uint32_t *emitterFlags;
    float emitterNormalization;
    uint32_t kBegin[4];       // group ranges per k (k == 3: degenerate triangles, never tested)
    // bitmap textures (level 0; src/textures/bitmap.cpp) and the lat-long environment map (src/emitters/envmap.cpp), half precision like the
    // reference's storage, one uint2 = {r|g<<16, b} per texel (luminance textures are replicated)
    //   texMeta[2i+0] = {bits(width), bits(height), bits(wrapU | wrapV<<8), bits(first texel)}, texMeta[2i+1] = {uScale, vScale, uOffset, vOffset}
    const float4 *texMeta; const uint2 *texels; uint32_t nTextures;
    const uint2 *envTexels; uint32_t envW, envH; float envScale; float worldToEnv[9];
    // light sampling of the environment emitter (nee != never; EnvironmentMap::configure, src/emitters/envmap.cpp:260-329): marginal row CDF [envH + 1],
    // conditional column CDFs [envH x (envW + 1)], sin(theta) row weights [envH]; the scene's bounding sphere x 1.5 (createShape, :330-335).
    // nLights = entries of emitterCdf - 1 (area emitters, then the environment emitter as the LAST light when there is one: envLight, else 0xFFFFFFFF)
    // The tables live behind one pointer (device memory): only the light-sampling code of the NEE variants reads them, and the kernels that keep a
    // local copy of this struct (noinline callees take it by reference) stay small.
    const struct EnvLight *env;
    uint32_t nLights, envLight;
};
struct EnvLight { const float *cdfRows, *cdfCols, *rowWeights; float normalization, pixelX, pixelY, radius; float center[3]; float toWorld[9]; };
struct Camera {             // src/sensors/perspective.cpp:271-298 for a lookAt camera
    float3 o, left, up, dir;
    float tanX, tanY, nearClip, farClip;
    int W, H;
};

}  // namespace ppg
