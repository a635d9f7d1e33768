// TEST INFRASTRUCTURE -- C entry points over the product's CUDA device functions compiled for the host (see cuda_host_shim.h); same shape as oracle/microfacet_ref/wrapper.h.
// Scenes are packed by the product's own pack_scene (ppg_scene.cpp, compiled into the same library) and the device code reads the packed arrays in place.
#include "cuda_host_shim.h"
#include "../../practical-path-guiding_b200/csrc/ppg_kernels.cuh"      // (includes ppg_device.cuh; the __global__ functions run here as plain loops of one thread)
#include "../../practical-path-guiding_b200/csrc/ppg_scene.h"
#include "../../include/ppg.h"
#include <cstddef>
#include <string>
#include <vector>
using namespace ppg;
static inline float3 v3(const float *p, size_t i) { return make_float3(p[3 * i], p[3 * i + 1], p[3 * i + 2]); }
// a packed scene with its SceneView bound to the packed arrays themselves
struct HostScene { PackedScene p; SceneView v; EnvLight env; std::string error; };
static int open_scene(const ppg_scene_desc &d, HostScene &hs) {
    const int rc = pack_scene(d, hs.p, hs.error);
    if (rc == PPG_OK) bind_scene(hs.p, [&](int i) { return hs.p.array(i).data; }, &hs.env, hs.v, hs.env);
    return rc;
}
// the Bsdf load_bsdf reads from the record pack_scene writes for material `m`, in a one-triangle scene with the rough-transmittance tables `tables`
static int packed_bsdf(const ppg_bsdf &m, const float *tables, uint32_t nTables, HostScene &hs, Bsdf &b) {
    static const float pos[9] = {0, 0, 0, 1, 0, 0, 0, 1, 0};
    static const uint32_t idx[3] = {0, 1, 2}, triShape[1] = {0};
    ppg_shape sh{}; sh.n_triangles = 1; sh.bsdf = 0; sh.emitter = -1;
    ppg_scene_desc d{}; d.n_vertices = 3; d.n_triangles = 1; d.n_shapes = 1; d.n_bsdfs = 1;
    d.positions = pos; d.indices = idx; d.triangle_shape = triShape; d.shapes = &sh; d.bsdfs = &m; d.bsdf_tables = tables; d.n_bsdf_tables = nTables;
    d.camera.film_width = d.camera.film_height = 1;
    const int rc = open_scene(d, hs);
    if (rc == PPG_OK) b = load_bsdf<true>(SceneAccess<false>(hs.v), 0);
    return rc;
}
extern "C" {
// pack_scene alone: its status, and its message in `error`
int dev_pack_scene(const ppg_scene_desc *d, char *error, size_t error_len) {
    HostScene hs; const int rc = pack_scene(*d, hs.p, hs.error);
    snprintf(error, error_len, "%s", hs.error.c_str());
    return rc;
}
void *dev_scene_open(const ppg_scene_desc *d) { HostScene *hs = new HostScene(); if (open_scene(*d, *hs) == PPG_OK) return hs; delete hs; return nullptr; }
void dev_scene_close(void *hs) { delete (HostScene *) hs; }
int dev_mf_eval(int type, float alpha, size_t n, const float *m, float *out) { for (size_t i = 0; i < n; ++i) out[i] = mf_eval(type, alpha, v3(m, i)); return 0; }
int dev_mf_smith_g1(int type, float alpha, size_t n, const float *v, const float *m, float *out) { for (size_t i = 0; i < n; ++i) out[i] = mf_smithG1(type, alpha, v3(v, i), v3(m, i)); return 0; }
int dev_mf_pdf(int type, float alpha, size_t n, const float *wi, const float *m, float *out) { for (size_t i = 0; i < n; ++i) out[i] = mf_pdfVisible(type, alpha, v3(wi, i), v3(m, i)); return 0; }
int dev_mf_sample(int type, float alpha, size_t n, const float *wi, const float *sample, float *m_out, float *pdf_out) {
    for (size_t i = 0; i < n; ++i) {
        const float3 m = mf_sampleVisible(type, alpha, v3(wi, i), sample[2 * i], sample[2 * i + 1]);
        m_out[3 * i] = m.x; m_out[3 * i + 1] = m.y; m_out[3 * i + 2] = m.z; pdf_out[i] = mf_pdfVisible(type, alpha, v3(wi, i), m);
    }
    return 0;
}
int dev_erf(size_t n, const float *x, float *erf_out, float *erfinv_out) { for (size_t i = 0; i < n; ++i) { erf_out[i] = mts_erf(x[i]); erfinv_out[i] = mts_erfinv(x[i]); } return 0; }
int dev_fresnel_dielectric_ext(size_t n, const float *c, float eta, float *f_out, float *ct_out) { for (size_t i = 0; i < n; ++i) { float ct = 0; f_out[i] = fresnel_dielectric_ext(c[i], ct, eta); ct_out[i] = ct; } return 0; }
int dev_fresnel_conductor_exact(size_t n, const float *c, const float eta[3], const float k[3], float *out) {
    for (size_t i = 0; i < n; ++i) for (int ch = 0; ch < 3; ++ch) out[3 * i + ch] = fresnel_conductor_exact(c[i], eta[ch], k[ch]);
    return 0;
}
int dev_coordinate_system(size_t n, const float *a, float *b_out, float *c_out) {
    for (size_t i = 0; i < n; ++i) { float3 b, c; coordinate_system(v3(a, i), b, c); b_out[3 * i] = b.x; b_out[3 * i + 1] = b.y; b_out[3 * i + 2] = b.z; c_out[3 * i] = c.x; c_out[3 * i + 1] = c.y; c_out[3 * i + 2] = c.z; }
    return 0;
}
int dev_square_to_cosine_hemisphere(size_t n, const float *s, float *out) { for (size_t i = 0; i < n; ++i) { const float3 v = square_to_cosine_hemisphere(s[2 * i], s[2 * i + 1]); out[3 * i] = v.x; out[3 * i + 1] = v.y; out[3 * i + 2] = v.z; } return 0; }
// the kernels' triangle test on the accel rows pack_scene writes: {n_u, n_v, n_d, bits(k)}, {a_u, a_v, b_nu, b_nv}, {c_nu, c_nv, -, -}
int dev_tri_intersect(size_t n, const int *k, const float *consts /* 9n, TriAccel order */, const float *o, const float *d, const float *mint, const float *maxt, unsigned char *hit_out, float *tuv_out) {
    for (size_t i = 0; i < n; ++i) {
        const float *c = consts + 9 * i;
        const float4 A = make_float4(c[0], c[1], c[2], __int_as_float(k[i])), B = make_float4(c[3], c[4], c[5], c[6]), C = make_float4(c[7], c[8], 0.f, 0.f);
        float u = 0, v = 0, t = 0;
        hit_out[i] = tri_intersect(A, B, C, v3(o, i), v3(d, i), mint[i], maxt[i], u, v, t) ? 1 : 0;
        tuv_out[3 * i] = t; tuv_out[3 * i + 1] = u; tuv_out[3 * i + 2] = v;
    }
    return 0;
}
// ---- whole BSDF models, as load_bsdf() reads them from the packed material record
int dev_bsdf_eval_pdf(const ppg_bsdf *m, size_t n, const float *wi, const float *wo, float *eval_out, float *pdf_out, const float *tables, uint32_t n_tables) {
    HostScene hs; Bsdf b;
    if (const int rc = packed_bsdf(*m, tables, n_tables, hs, b)) return rc;
    for (size_t i = 0; i < n; ++i) { const float3 e = bsdf_eval(b, v3(wi, i), v3(wo, i)); eval_out[3 * i] = e.x; eval_out[3 * i + 1] = e.y; eval_out[3 * i + 2] = e.z; pdf_out[i] = bsdf_pdf(b, v3(wi, i), v3(wo, i)); }
    return 0;
}
int dev_bsdf_sample(const ppg_bsdf *m, size_t n, const float *wi, const float *sample, float *wo_out, float *weight_out, float *pdf_out, unsigned char *delta_out,
                    const float *tables, uint32_t n_tables) {
    HostScene hs; Bsdf b;
    if (const int rc = packed_bsdf(*m, tables, n_tables, hs, b)) return rc;
    for (size_t i = 0; i < n; ++i) {
        float3 wo = make_float3(0, 0, 0); float eta = 1.f, pdf = 0.f; bool delta = false, isNull = false;
        Pcg32 extra; extra.seed(splitmix64(i), i);                      // like ppgo_bsdf_sample: the model's own draws from the path sampler (roughdielectric)
        const float3 w = bsdf_sample(b, v3(wi, i), sample[2 * i], sample[2 * i + 1], wo, eta, delta, pdf, extra, isNull);
        wo_out[3 * i] = wo.x; wo_out[3 * i + 1] = wo.y; wo_out[3 * i + 2] = wo.z; weight_out[3 * i] = w.x; weight_out[3 * i + 1] = w.y; weight_out[3 * i + 2] = w.z;
        pdf_out[i] = pdf; if (delta_out) delta_out[i] = delta ? 1 : 0;
    }
    return 0;
}
// bitmap textures: tex_eval / tex_gradient_lum of texture `k` of a packed scene
int dev_texture_eval(const void *scene, uint32_t k, size_t n, const float *uv, float *rgb_out, float *grad_out) {
    const SceneView &sc = ((const HostScene *) scene)->v;
    for (size_t i = 0; i < n; ++i) {
        const float2 q = make_float2(uv[2 * i], uv[2 * i + 1]);
        const float3 c = tex_eval(sc, k, q); const float2 g = tex_gradient_lum(sc, k, q);
        rgb_out[3 * i] = c.x; rgb_out[3 * i + 1] = c.y; rgb_out[3 * i + 2] = c.z; grad_out[2 * i] = g.x; grad_out[2 * i + 1] = g.y;
    }
    return 0;
}
// the emitter-list table the host builds from `n_entries` weights: running float sum, then normalize_cdf (n_entries + 1 values)
int dev_emitter_cdf(size_t n_entries, const float *weights, float *cdf_out) {
    cdf_out[0] = 0.f;
    for (size_t i = 0; i < n_entries; ++i) cdf_out[i + 1] = cdf_out[i] + weights[i];
    normalize_cdf(cdf_out, n_entries);
    return 0;
}
// cdf_sample + the sample reuse of the device's sample_emitter_direct, on a normalised cdf (n_entries + 1 values) the host built
int dev_discrete(size_t n_entries, const float *cdf, size_t n, const float *sample, unsigned *index_out, float *reused_out) {
    for (size_t i = 0; i < n; ++i) {
        const uint32_t k = cdf_sample(cdf, (uint32_t) n_entries + 1u, sample[i]);
        const float c0 = cdf[k], c1 = cdf[k + 1];
        index_out[i] = k; reused_out[i] = (sample[i] - c0) / (c1 - c0);
    }
    return 0;
}
// ---- SD-tree: S-tree descent through the prefix table stree_table_kernel builds, D-tree pdf / sample on a sampling pool laid out like the device's (SampNode)
int dev_stree_lookup(const uint32_t *node_children /* 2 per node */, size_t n_nodes, const float aabb_min[3], const float extent[3], const float *points, size_t n, uint32_t *leaf_out, float *size_out) {
    std::vector<uint2> sn(n_nodes);
    for (size_t i = 0; i < n_nodes; ++i) sn[i] = make_uint2(node_children[2 * i], node_children[2 * i + 1]);
    std::vector<uint32_t> table;                     // under the render's rule: no table past 0xFFFFFF nodes
    if (stree_table_usable(n_nodes)) { table.resize((size_t) 1 << (3 * PPG_STREE_TABLE_BITS)); stree_table_kernel(sn.data(), table.data()); }
    const float3 mn = make_float3(aabb_min[0], aabb_min[1], aabb_min[2]), ex = make_float3(extent[0], extent[1], extent[2]);
    for (size_t i = 0; i < n; ++i) {
        int lv = 0; leaf_out[i] = stree_lookup(sn.data(), table.empty() ? nullptr : table.data(), mn, ex, v3(points, i), lv);
        const float3 v = voxel_size(ex, lv); size_out[3 * i] = v.x; size_out[3 * i + 1] = v.y; size_out[3 * i + 2] = v.z;
    }
    return 0;
}
struct ReplayRng { const float *v; uint32_t n, i; float next1D() { return i < n ? v[i++] : 0.5f; } };
int dev_dtree(const float *sums, const uint16_t *children, size_t n_nodes, const uint32_t *tree_first, const float *tree_sum, const float *tree_weight,
              const uint32_t *query_tree, const float *query_dir, const float *rnd, size_t rnd_stride, size_t n, float *pdf_out, float *dir_out,
              float *canonical_out /* 2n or NULL: the point dtree_sample returns, before canonical_to_dir */) {
    std::vector<SampNode> pool(n_nodes);
    for (size_t i = 0; i < n_nodes; ++i) {
        pool[i].sums = make_float4(sums[4 * i], sums[4 * i + 1], sums[4 * i + 2], sums[4 * i + 3]);
        pool[i].children = make_uint2((uint32_t) children[4 * i] | ((uint32_t) children[4 * i + 1] << 16), (uint32_t) children[4 * i + 2] | ((uint32_t) children[4 * i + 3] << 16));
        pool[i].pad = make_uint2(0u, 0u);
    }
    for (size_t i = 0; i < n; ++i) {
        const uint32_t t = query_tree[i];
        float mean = 0.f; if (tree_weight[t] != 0.f) mean = (1.f / (PPG_PI * 4.f * tree_weight[t])) * tree_sum[t];       // DTree::mean, GP:386-394
        pdf_out[i] = dtree_pdf(pool.data() + tree_first[t], mean > 0.f, dir_to_canonical(v3(query_dir, i)));
        ReplayRng r{rnd + rnd_stride * i, (uint32_t) rnd_stride, 0u};
        const float2 c = dtree_sample(pool.data() + tree_first[t], mean > 0.f, r);
        const float3 d = canonical_to_dir(c);
        dir_out[3 * i] = d.x; dir_out[3 * i + 1] = d.y; dir_out[3 * i + 2] = d.z;
        if (canonical_out) { canonical_out[2 * i] = c.x; canonical_out[2 * i + 1] = c.y; }
    }
    return 0;
}
// the stochastic spatial filter's jitter of commit_kernel: the three uniforms of the vertex stream seed_vertex_rng(seed, sampleIndex, ordinal)
int dev_vertex_jitter(uint64_t seed, size_t n, const uint64_t *sample_index, const uint32_t *ordinal, float *out) {
    for (size_t i = 0; i < n; ++i) {
        Pcg32 r; seed_vertex_rng(r, seed, sample_index[i], ordinal[i]);
        out[3 * i] = r.next1D(); out[3 * i + 1] = r.next1D(); out[3 * i + 2] = r.next1D();
    }
    return 0;
}
// ---- packed scenes: nearest hit, light sampling, environment emitter
// bvh_intersect (coplanar groups or BVH walk, whichever the packing chose), and the brute-force minimum of tri_intersect over every packed accel row
// (ties to the lower original triangle index).  t_out / prim_out: 2 per ray {bvh_intersect, brute force}; prim 0xFFFFFFFF = miss.
int dev_closest_hit(const void *scene, size_t n, const float *o, const float *d, float mint, float maxt, float *t_out, uint32_t *prim_out) {
    const SceneView &sc = ((const HostScene *) scene)->v;
    const SceneAccess<false> acc(sc);
    for (size_t i = 0; i < n; ++i) {
        Hit h; h.t = 0.f;
        const bool found = bvh_intersect<true>(acc, v3(o, i), v3(d, i), mint, maxt, h);
        t_out[2 * i] = found ? h.t : 0.f; prim_out[2 * i] = found ? h.prim : 0xFFFFFFFFu;
        float bt = __int_as_float(0x7f800000); uint32_t bp = 0xFFFFFFFFu;
        for (uint32_t s = 0; s < sc.nTris; ++s) {
            float u, v, t;
            const float4 A = sc.accel[3 * s], B = sc.accel[3 * s + 1], C = sc.accel[3 * s + 2];
            if (!tri_intersect(A, B, C, v3(o, i), v3(d, i), mint, maxt, u, v, t)) continue;
            const uint32_t prim = __float_as_uint(C.z);
            if (t < bt || (t == bt && prim < bp)) { bt = t; bp = prim; }
        }
        t_out[2 * i + 1] = bp != 0xFFFFFFFFu ? bt : 0.f; prim_out[2 * i + 1] = bp;
    }
    return 0;
}
// the body of op_emitter_sample_kernel (ppg_host.cu): Scene::sampleAttenuatedEmitterDirect at caller-supplied reference points
int dev_emitter_sample_direct(const void *scene, size_t n, const float *ref, const float *refN, const float *smp, int maxInteractions,
                              float *dOut, float *valueOut, float *pdfOut, float *distOut) {
    const SceneAccess<false> sc(((const HostScene *) scene)->v);
    for (size_t i = 0; i < n; ++i) {
        const float3 p = v3(ref, i), rn = v3(refN, i);
        DirectSample ds; ds.value = make_float3(0, 0, 0); ds.d = make_float3(0, 0, 0); ds.pdf = 0.f; float dist = 0.f;
        const bool ok = sample_emitter_direct<true>(sc, p, rn, smp[2 * i], smp[2 * i + 1], ds, dist);
        if (ok) ds.value = ds.value * eval_transmittance(sc, p, ds.d, dist, maxInteractions);
        else { ds.value = make_float3(0, 0, 0); ds.pdf = 0.f; dist = 0.f; }
        dOut[3 * i] = ds.d.x; dOut[3 * i + 1] = ds.d.y; dOut[3 * i + 2] = ds.d.z;
        valueOut[3 * i] = ds.value.x; valueOut[3 * i + 1] = ds.value.y; valueOut[3 * i + 2] = ds.value.z;
        pdfOut[i] = ds.pdf; distOut[i] = dist;
    }
    return 0;
}
// the body of op_env_pdf_kernel (ppg_host.cu): the environment emitter's pdfEmitterDirect and radiance for world directions
int dev_env_pdf(const void *scene, size_t n, const float *dir, float *pdfOut, float *valueOut) {
    const SceneView &sc = ((const HostScene *) scene)->v;
    for (size_t i = 0; i < n; ++i) {
        const float3 d = v3(dir, i);
        pdfOut[i] = pdf_emitter_direct<true>(sc, PPG_ENV_EMITTER, make_float3(0, 0, 0), make_float3(0, 0, 0), d, make_float3(0, 0, 0), 0.f);
        const float3 v = env_eval(sc, d); valueOut[3 * i] = v.x; valueOut[3 * i + 1] = v.y; valueOut[3 * i + 2] = v.z;
    }
    return 0;
}
int dev_rough_transmittance(size_t n, const float *c, const float *values, float *out) { for (size_t i = 0; i < n; ++i) out[i] = rough_transmittance(values, c[i]); return 0; }
}
