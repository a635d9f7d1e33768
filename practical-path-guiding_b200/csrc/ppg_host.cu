// ppg_host.cu -- host side of libppg_b200.so: the C ABI of include/ppg.h, the iteration schedule of the
// reference integrator (GP = mitsuba/src/integrators/path/guided_path.cpp), the scene upload and the
// launch sequence of the wavefront kernels (scene packing and the BVH: ppg_scene.cpp).  C++ host, CUDA kernels, no torch, no CPU fallback.
#include "../../include/ppg.h"
#include "ppg_kernels.cuh"
#include "ppg_scene.h"

#include <dlfcn.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <new>
#include <numeric>
#include <string>
#include <vector>

using namespace ppg;

// ------------------------------------------------------------------ errors
static thread_local std::string g_lastError;
static int fail(int code, const std::string &msg) { g_lastError = msg; return code; }
// "no exceptions cross this boundary" (ppg.h): the entry points that allocate host memory in proportion to their input run under this guard
template <class F> static int guarded(const char *what, F body) {
    try { return body(); }
    catch (const std::bad_alloc &) { return fail(PPG_ERR_INVALID_ARGUMENT, std::string(what) + ": out of host memory"); }
    catch (const std::exception &e) { return fail(PPG_ERR_INVALID_ARGUMENT, std::string(what) + ": " + e.what()); }
}
#define CK(call)                                                                                         \
    do {                                                                                                 \
        cudaError_t e_ = (call);                                                                         \
        if (e_ != cudaSuccess) {                                                                         \
            g_lastError = std::string(#call) + ": " + cudaGetErrorString(e_) + " (" + __FILE__ + ":" + std::to_string(__LINE__) + ")"; \
            return PPG_ERR_CUDA;                                                                         \
        }                                                                                                \
    } while (0)

template <class T> struct DevBuf {
    T *p = nullptr; size_t n = 0;
    ~DevBuf() { release(); }
    void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
    cudaError_t alloc(size_t count) {
        if (count <= n && p) return cudaSuccess;
        release();
        cudaError_t e = cudaMalloc(&p, std::max<size_t>(count, 1) * sizeof(T));
        if (e == cudaSuccess) n = count;
        return e;
    }
    // grow preserving contents
    cudaError_t grow(size_t count, cudaStream_t s) {
        if (count <= n && p) return cudaSuccess;
        T *q = nullptr; cudaError_t e = cudaMalloc(&q, count * sizeof(T));
        if (e != cudaSuccess) return e;
        if (p && n) cudaMemcpyAsync(q, p, n * sizeof(T), cudaMemcpyDeviceToDevice, s);
        cudaStreamSynchronize(s);
        if (p) cudaFree(p);
        p = q; n = count; return cudaSuccess;
    }
};

// ------------------------------------------------------------------ parameters (GP:1014-1085, integrator.cpp:190-225)
extern "C" void ppg_params_default(ppg_params *p) {
    p->nee = PPG_NEE_NEVER; p->sample_combination = PPG_COMB_AUTOMATIC; p->spatial_filter = PPG_SFILTER_NEAREST;
    p->directional_filter = PPG_DFILTER_NEAREST; p->bsdf_sampling_fraction_loss = PPG_LOSS_NONE;
    p->sd_tree_max_memory = -1; p->s_tree_threshold = 12000; p->d_tree_threshold = 0.01f; p->bsdf_sampling_fraction = 0.5f;
    p->spp_per_pass = 4; p->budget_type = PPG_BUDGET_SECONDS; p->budget = 300.0f; p->dump_sd_tree = 0;
    p->max_depth = -1; p->rr_depth = 5; p->strict_normals = 0; p->hide_emitters = 0; p->seed = 1234;
}

static bool parse_enum(const char *v, const char *const *names, int n, int32_t *out) {
    for (int i = 0; i < n; ++i) if (!strcmp(v, names[i])) { *out = i; return true; }
    return false;
}
static bool parse_bool(const char *v, int32_t *out) {
    if (!strcmp(v, "true")) { *out = 1; return true; }
    if (!strcmp(v, "false")) { *out = 0; return true; }
    return false;
}
static bool parse_int(const char *v, long long *out) { char *e = nullptr; *out = strtoll(v, &e, 10); return e && *e == '\0' && e != v; }
static bool parse_float(const char *v, float *out) { char *e = nullptr; *out = strtof(v, &e); return e && *e == '\0' && e != v; }

extern "C" int ppg_params_set(ppg_params *p, const char *name, const char *value) {
    if (!p || !name || !value) return fail(PPG_ERR_INVALID_ARGUMENT, "null argument");
    static const char *const nee[] = {"never", "kickstart", "always"};
    static const char *const comb[] = {"discard", "automatic", "inversevar"};
    static const char *const sf[] = {"nearest", "stochastic", "box"};
    static const char *const df[] = {"nearest", "box"};
    static const char *const loss[] = {"none", "kl", "var"};
    static const char *const bt[] = {"spp", "seconds"};
    bool ok; long long iv;
    std::string n(name);
    if (n == "nee") ok = parse_enum(value, nee, 3, &p->nee);
    else if (n == "sampleCombination") ok = parse_enum(value, comb, 3, &p->sample_combination);
    else if (n == "spatialFilter") ok = parse_enum(value, sf, 3, &p->spatial_filter);
    else if (n == "directionalFilter") ok = parse_enum(value, df, 2, &p->directional_filter);
    else if (n == "bsdfSamplingFractionLoss") ok = parse_enum(value, loss, 3, &p->bsdf_sampling_fraction_loss);
    else if (n == "budgetType") ok = parse_enum(value, bt, 2, &p->budget_type);
    else if (n == "sdTreeMaxMemory") { ok = parse_int(value, &iv); if (ok) p->sd_tree_max_memory = (int32_t) iv; }
    else if (n == "sTreeThreshold") { ok = parse_int(value, &iv); if (ok) p->s_tree_threshold = (int32_t) iv; }
    else if (n == "sppPerPass") { ok = parse_int(value, &iv); if (ok) p->spp_per_pass = (int32_t) iv; }
    else if (n == "maxDepth") { ok = parse_int(value, &iv); if (ok) p->max_depth = (int32_t) iv; }
    else if (n == "rrDepth") { ok = parse_int(value, &iv); if (ok) p->rr_depth = (int32_t) iv; }
    else if (n == "seed") { ok = parse_int(value, &iv); if (ok) p->seed = (uint64_t) iv; }
    else if (n == "dTreeThreshold") ok = parse_float(value, &p->d_tree_threshold);
    else if (n == "bsdfSamplingFraction") ok = parse_float(value, &p->bsdf_sampling_fraction);
    else if (n == "budget") ok = parse_float(value, &p->budget);
    else if (n == "dumpSDTree") ok = parse_bool(value, &p->dump_sd_tree);
    else if (n == "strictNormals") ok = parse_bool(value, &p->strict_normals);
    else if (n == "hideEmitters") ok = parse_bool(value, &p->hide_emitters);
    else return fail(PPG_ERR_INVALID_ARGUMENT, "unknown integrator parameter '" + n + "'");
    if (!ok) return fail(PPG_ERR_INVALID_ARGUMENT, "invalid value '" + std::string(value) + "' for parameter '" + n + "'");
    return PPG_OK;
}

extern "C" int ppg_params_validate(const ppg_params *p) {
    if (!p) return fail(PPG_ERR_INVALID_ARGUMENT, "null params");
    auto in = [](int v, int lo, int hi) { return v >= lo && v <= hi; };
    if (!in(p->nee, 0, 2) || !in(p->sample_combination, 0, 2) || !in(p->spatial_filter, 0, 2) || !in(p->directional_filter, 0, 1) ||
        !in(p->bsdf_sampling_fraction_loss, 0, 2) || !in(p->budget_type, 0, 1))
        return fail(PPG_ERR_INVALID_ARGUMENT, "enum parameter out of range (the reference Assert(false)s, GP:1023-1080)");
    if (p->rr_depth <= 0) return fail(PPG_ERR_INVALID_ARGUMENT, "'rrDepth' must be set to a value greater than zero!");
    if (p->max_depth <= 0 && p->max_depth != -1) return fail(PPG_ERR_INVALID_ARGUMENT, "'maxDepth' must be set to -1 (infinite) or a value greater than zero!");
    if (p->spp_per_pass < 1) return fail(PPG_ERR_INVALID_ARGUMENT, "'sppPerPass' must be at least 1");
    if (!(p->budget > 0)) return fail(PPG_ERR_INVALID_ARGUMENT, "'budget' must be positive");
    if (!(p->bsdf_sampling_fraction >= 0.f && p->bsdf_sampling_fraction <= 1.f)) return fail(PPG_ERR_INVALID_ARGUMENT, "'bsdfSamplingFraction' must lie in [0,1]");
    return PPG_OK;
}

extern "C" const char *ppg_description(void) { return "Guided path tracer"; }
extern "C" int ppg_abi_version(void) { return PPG_ABI_VERSION; }
extern "C" const char *ppg_last_error(void) { return g_lastError.c_str(); }

// ------------------------------------------------------------------ flat scene files (python -m ppg_b200.convert)
struct ppg_scene_file { std::vector<std::vector<char>> blobs; std::string props; };
extern "C" int ppg_scene_file_load(const char *path, ppg_scene_desc *d, ppg_scene_file **file, const char **integrator_props) {
    if (!path || !d || !file) return fail(PPG_ERR_INVALID_ARGUMENT, "null argument");
    FILE *f = fopen(path, "rb");
    if (!f) return fail(PPG_ERR_IO, std::string("cannot open ") + path);
    char magic[8];
    if (fread(magic, 1, 8, f) != 8 || memcmp(magic, "PPGSCN02", 8) != 0) { fclose(f); return fail(PPG_ERR_IO, "not a PPGSCN02 scene file"); }
    long fileBytes = 0;                                   // no array can be larger than the file: a corrupt header must not turn into a huge allocation
    if (fseek(f, 0, SEEK_END) != 0 || (fileBytes = ftell(f)) < 8 || fseek(f, 8, SEEK_SET) != 0) { fclose(f); return fail(PPG_ERR_IO, "cannot size the scene file"); }
    ppg_scene_file *sf = new (std::nothrow) ppg_scene_file();
    if (!sf) { fclose(f); return fail(PPG_ERR_IO, "out of memory"); }
    memset(d, 0, sizeof(*d));
    struct Arr { const char *p; size_t bytes; uint64_t dims[4]; uint32_t ndim; };
    auto fail_io = [&](const char *m) { fclose(f); delete sf; return fail(PPG_ERR_IO, m); };
    static const size_t esz[6] = {4, 4, 4, 2, 1, 8};
    std::vector<std::pair<std::string, Arr>> arrs;
    for (;;) {
        uint32_t nl;
        if (fread(&nl, 4, 1, f) != 1) break;
        if (nl > 64) return fail_io("corrupt scene file (name)");
        std::string name(nl, 0); uint32_t hdr[2];
        if (fread(&name[0], 1, nl, f) != nl || fread(hdr, 4, 2, f) != 2 || hdr[0] > 5 || hdr[1] > 4) return fail_io("corrupt scene file (header)");
        Arr a; a.ndim = hdr[1]; size_t count = 1;
        for (uint32_t k = 0; k < a.ndim; ++k) {
            if (fread(&a.dims[k], 8, 1, f) != 1) return fail_io("corrupt scene file (dims)");
            if (a.dims[k] > (uint64_t) fileBytes || (a.dims[k] && count > (size_t) fileBytes / (size_t) a.dims[k])) return fail_io("corrupt scene file (array larger than the file)");
            count *= (size_t) a.dims[k];
        }
        a.bytes = count * esz[hdr[0]];
        if (a.bytes > (size_t) fileBytes) return fail_io("corrupt scene file (array larger than the file)");
        try { sf->blobs.emplace_back(a.bytes + 8); } catch (const std::bad_alloc &) { return fail_io("out of memory"); }
        if (a.bytes && fread(sf->blobs.back().data(), 1, a.bytes, f) != a.bytes) return fail_io("truncated scene file");
        a.p = sf->blobs.back().data();
        arrs.emplace_back(name, a);
    }
    fclose(f);
    auto get = [&](const char *n) -> const Arr * { for (auto &kv : arrs) if (kv.first == n) return &kv.second; return nullptr; };
    const Arr *P = get("positions"), *N = get("normals"), *UV = get("uvs"), *I = get("indices"), *TS = get("triangle_shape"), *SH = get("shapes"), *B = get("bsdfs"),
              *R = get("area_radiance"), *T = get("bsdf_tables"), *SP = get("spheres"), *CW = get("cam_to_world"), *CAM = get("cam"), *BB = get("aabb"),
              *TX = get("textures"), *TL = get("texels"), *ET = get("env_texels"), *EM = get("env_meta"), *IP = get("integrator");
    if (!P || !N || !UV || !I || !TS || !SH || !B || !R || !CW || !CAM || !BB || CW->bytes != 64 || CAM->bytes != 40 || BB->bytes != 24 || B->bytes % sizeof(ppg_bsdf) || SH->bytes % sizeof(ppg_shape))
        { delete sf; return fail(PPG_ERR_IO, "scene file lacks a required array"); }
    // per-vertex / per-triangle arrays must cover what the counts promise (ppg_set_scene indexes them without further checks)
    if (P->bytes % 12 || I->bytes % 12 || R->bytes % 12 || N->bytes != P->bytes || UV->bytes != P->bytes / 12 * 8 || TS->bytes != I->bytes / 12 * 4 ||
        (T && T->bytes % (4 * PPG_BSDF_TABLE_SIZE)) || (SP && SP->bytes % sizeof(ppg_sphere)) || (TX && TX->bytes % sizeof(ppg_texture)) ||
        (ET && ET->bytes && (ET->ndim != 3 || ET->dims[2] != 3 || ET->bytes != ET->dims[0] * ET->dims[1] * 6)))
        { delete sf; return fail(PPG_ERR_IO, "scene file: array sizes do not match each other"); }
    d->n_vertices = (uint32_t) (P->bytes / 12); d->n_triangles = (uint32_t) (I->bytes / 12); d->n_shapes = (uint32_t) (SH->bytes / sizeof(ppg_shape));
    d->n_bsdfs = (uint32_t) (B->bytes / sizeof(ppg_bsdf)); d->n_emitters = (uint32_t) (R->bytes / 12);
    d->positions = (const float *) P->p; d->normals = (const float *) N->p; d->uvs = (const float *) UV->p; d->indices = (const uint32_t *) I->p;
    d->triangle_shape = (const uint32_t *) TS->p; d->shapes = (const ppg_shape *) SH->p; d->bsdfs = (const ppg_bsdf *) B->p; d->area_radiance = (const float *) R->p;
    if (T && T->bytes) { d->bsdf_tables = (const float *) T->p; d->n_bsdf_tables = (uint32_t) (T->bytes / (4 * PPG_BSDF_TABLE_SIZE)); }
    if (SP && SP->bytes) { d->spheres = (const ppg_sphere *) SP->p; d->n_spheres = (uint32_t) (SP->bytes / sizeof(ppg_sphere)); }
    memcpy(d->camera.to_world, CW->p, 64);
    const double *cam = (const double *) CAM->p;
    d->camera.x_fov_deg = (float) cam[0]; d->camera.near_clip = (float) cam[1]; d->camera.far_clip = (float) cam[2]; d->camera.film_width = (int32_t) cam[3]; d->camera.film_height = (int32_t) cam[4];
    memcpy(d->aabb_min, BB->p, 12); memcpy(d->aabb_max, BB->p + 12, 12);
    if (TX && TX->bytes && TL) { d->textures = (const ppg_texture *) TX->p; d->n_textures = (uint32_t) (TX->bytes / sizeof(ppg_texture)); d->texels = (const uint16_t *) TL->p; d->n_texels = TL->bytes / 2; }
    if (ET && ET->bytes && EM && EM->bytes == 40 && ET->ndim == 3) {
        d->envmap.height = (uint32_t) ET->dims[0]; d->envmap.width = (uint32_t) ET->dims[1]; d->envmap.texels = (const uint16_t *) ET->p;
        const float *em = (const float *) EM->p; d->envmap.scale = em[0]; memcpy(d->envmap.world_to_env, em + 1, 36);
    }
    if (IP) sf->props.assign(IP->p, IP->bytes);
    if (integrator_props) *integrator_props = sf->props.c_str();
    *file = sf;
    return PPG_OK;
}
extern "C" void ppg_scene_file_free(ppg_scene_file *file) { delete file; }

// ------------------------------------------------------------------ SD-tree storage and its launch sequences
static float bits_f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static uint32_t f_bits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
// the ABI's quadtree nodes (NULL: zeros) as sampling-pool nodes: children keep their bytes, uint2 {c0 | c1 << 16, c2 | c3 << 16} == 4 x uint16
static std::vector<SampNode> to_pool(const float *sums, const uint16_t *children, size_t n) {
    std::vector<SampNode> pool(n);
    for (size_t i = 0; i < n; ++i) {
        if (sums) memcpy(&pool[i].sums, sums + 4 * i, 16);
        if (children) memcpy(&pool[i].children, children + 4 * i, 8);
    }
    return pool;
}
// the 6-float sampling-fraction record of the ABI <-> the float4 + float2 pair the device keeps it in
static void records_split(const float *r, size_t n, std::vector<float4> &a, std::vector<float2> &b) {
    a.resize(n); b.resize(n);
    for (size_t i = 0; i < n; ++i) { memcpy(&a[i], r + 6 * i, 16); memcpy(&b[i], r + 6 * i + 4, 8); }
}
static int records_join(const float4 *dA, const float2 *dB, size_t n, float *r) {
    std::vector<float4> a(n); std::vector<float2> b(n);
    CK(cudaMemcpy(a.data(), dA, 16 * n, cudaMemcpyDeviceToHost)); CK(cudaMemcpy(b.data(), dB, 8 * n, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < n; ++i) { memcpy(r + 6 * i, &a[i], 16); memcpy(r + 6 * i + 4, &b[i], 8); }
    return PPG_OK;
}

// The SD-tree on the device and its launch sequences, shared by the render and the ppg_op_* entry points.  Launch members return their launch count.
struct TreeStore {
    cudaStream_t stream = nullptr; int numSMs = 132, commitGrid = 0;
    uint32_t capNodes = 0; size_t capPool = 0;
    DevBuf<uint2> dSnodes; DevBuf<float4> dLeafA; DevBuf<float> dBweight, dSampSum, dSampWeight, dAdam, dAdamBefore /* 4 x capNodes: iter, batchAcc, batchGrad, theta before a replay */;
    DevBuf<uint32_t> dAdamCount, dAdamCursor, dAdamOffset; DevBuf<float4> dAdamRecA, dAdamSortA; DevBuf<float2> dAdamRecB, dAdamSortB; size_t adamCap = 0;
    DevBuf<int> dSampDepth, dBuildDepth; DevBuf<uint32_t> dSampCount, dBuildCount, dBuildBase, dScalars /* [0]=nNodes [1]=totalBuild */;
    DevBuf<uint32_t> dStable; DevBuf<TreeStats> dTreeStats;
    DevBuf<SampNode> dSamp; DevBuf<uint2> dBchildren; DevBuf<float> dTrain /* bsums | packed tail */;
    uint32_t hNodes = 1; uint32_t hTotalBuild = 1;
    static constexpr size_t kTableEntries = (size_t) 1 << (3 * PPG_STREE_TABLE_BITS);

    // the whole buffer zeroed, then its first n elements copied from the host (host may be null: zeros)
    template <class T> cudaError_t put(DevBuf<T> &b, const void *host = nullptr, size_t n = 0) {
        cudaError_t e = cudaMemsetAsync(b.p, 0, b.n * sizeof(T), stream); if (e != cudaSuccess) return e;
        return (host && n) ? cudaMemcpyAsync(b.p, host, n * sizeof(T), cudaMemcpyHostToDevice, stream) : cudaSuccess;
    }

    // room for `nodes` S-tree nodes and `pool` quadtree nodes: grown by doubling (the render), or to exactly that size
    int reserve(uint32_t nodes, size_t pool, bool exact = false) {
        CK(dScalars.alloc(8)); CK(dTreeStats.alloc(1));
        if (nodes > capNodes) {
            const uint32_t cap = exact ? nodes : std::max<uint32_t>(nodes, std::max<uint32_t>(2 * capNodes, 1u << 16));
            CK(dSnodes.grow(cap, stream)); CK(dLeafA.grow(cap, stream)); CK(dBweight.grow(cap, stream));
            CK(dSampSum.grow(cap, stream)); CK(dSampWeight.grow(cap, stream)); CK(dAdam.grow(6 * (size_t) cap, stream));
            CK(dAdamBefore.grow(4 * (size_t) cap, stream)); CK(dSampDepth.grow(cap, stream));
            {   // record-bucket bookkeeping must stay zero between commit launches: reallocate zeroed
                dAdamCount.release(); dAdamCursor.release(); dAdamOffset.release();
                CK(dAdamCount.alloc(cap)); CK(dAdamCursor.alloc(cap)); CK(dAdamOffset.alloc(cap));
                CK(cudaMemsetAsync(dAdamCount.p, 0, 4 * (size_t) cap, stream)); CK(cudaMemsetAsync(dAdamCursor.p, 0, 4 * (size_t) cap, stream));
            }
            CK(dBuildDepth.grow(cap, stream)); CK(dSampCount.grow(cap, stream)); CK(dBuildCount.grow(cap, stream));
            CK(dBuildBase.grow(cap, stream));
            capNodes = cap;
        }
        if (pool > capPool) {
            const size_t cap = exact ? pool : std::max<size_t>(pool, std::max<size_t>(2 * capPool, (size_t) 1 << 20));
            CK(dSamp.grow(cap, stream)); CK(dBchildren.grow(cap, stream));
            capPool = cap;
        }
        // bsums (4 floats per pool node) followed by the packed exchange tail (building weights, or 6 Adam arrays; + scalars)
        CK(dTrain.grow(4 * capPool + 6 * (size_t) capNodes + 64, stream));
        return PPG_OK;
    }

    MaintParams maint() const {
        MaintParams M;
        M.snodes = dSnodes.p; M.leafA = dLeafA.p; M.bweight = dBweight.p; M.sampSum = dSampSum.p; M.sampWeight = dSampWeight.p;
        M.sampDepth = dSampDepth.p; M.sampCount = dSampCount.p; M.adam = dAdam.p; M.buildCount = dBuildCount.p; M.buildDepth = dBuildDepth.p;
        M.nNodes = dScalars.p; M.capNodes = capNodes; M.samp = dSamp.p; M.bchildren = dBchildren.p; M.bsums = reinterpret_cast<float4 *>(dTrain.p);
        return M;
    }
    TreeView view(const float *aabbMin, const float *extent) const {
        TreeView T;
        T.snodes = dSnodes.p; T.stable = stree_table_usable(hNodes) ? dStable.p : nullptr; T.leafA = dLeafA.p; T.samp = dSamp.p; T.bchildren = dBchildren.p;
        T.bsums = reinterpret_cast<float4 *>(dTrain.p); T.bweight = dBweight.p;
        T.aabbMin = make_float3(aabbMin[0], aabbMin[1], aabbMin[2]); T.extent = make_float3(extent[0], extent[1], extent[2]);
        return T;
    }

    // new STree (GP:1519): one leaf whose sampling tree is a single empty quadtree node
    int init() {
        // buffers persist across renders (cudaMalloc/cudaFree are synchronous and slow): only their contents are reset
        int rc = reserve(std::max<uint32_t>(capNodes, 1u << 16), std::max<size_t>(capPool, (size_t) 1 << 20));
        if (rc) return rc;
        const uint32_t one[2] = {1u, 1u};
        CK(put(dScalars, one, 2));
        CK(put(dSnodes)); CK(put(dLeafA)); CK(put(dBweight)); CK(put(dSampSum)); CK(put(dSampWeight));
        CK(put(dAdam)); CK(put(dAdamCount)); CK(put(dAdamCursor)); CK(put(dSampDepth));
        CK(cudaMemsetAsync(dSamp.p, 0, sizeof(SampNode), stream));          // one empty quadtree node at pool offset 0
        CK(cudaMemcpyAsync(dSampCount.p, one, 4, cudaMemcpyHostToDevice, stream));
        hNodes = 1; hTotalBuild = 1;
        CK(cudaStreamSynchronize(stream));
        return PPG_OK;
    }

    // A caller's ppg_sdtree on the default stream, in exactly max(nodeCap, n_nodes) S-tree and n_pool quadtree nodes: the sampling trees
    // (which == 0), with the leafA flag dtree_build_kernel writes, or the building trees (which == 1)
    int load(int which, const ppg_sdtree &in, uint32_t nodeCap = 0) {
        const size_t n = in.n_nodes;
        if (n >= 0xFFFFFFFFull) return fail(PPG_ERR_INVALID_ARGUMENT, "more S-tree nodes than 32-bit node numbers hold");
        std::vector<uint32_t> first(n, 0u); std::vector<float4> la(n);
        for (size_t i = 0; i < n; ++i) {
            if (in.tree_first && in.tree_first[i] > 0xFFFFFFFFull) return fail(PPG_ERR_INVALID_ARGUMENT, "tree_first past the 32 bits of the leaf record");
            if (in.tree_first) first[i] = (uint32_t) in.tree_first[i];
            const bool valid = !which && dtree_mean(in.tree_sum ? in.tree_sum[i] : 0.f, in.tree_weight ? in.tree_weight[i] : 0.f) > 0.f;
            la[i] = make_float4(bits_f(first[i]), which ? bits_f(first[i]) : 0.f, in.adam ? in.adam[6 * i + 3] : 0.f, bits_f(valid ? 1u : 0u));
        }
        int dev = 0;
        CK(cudaGetDevice(&dev)); CK(cudaDeviceGetAttribute(&numSMs, cudaDevAttrMultiProcessorCount, dev)); CK(dStable.alloc(kTableEntries));
        int rc = reserve(std::max<uint32_t>(std::max<uint32_t>((uint32_t) n, nodeCap), 1), std::max<size_t>(in.n_pool, 1), true); if (rc) return rc;
        CK(put(dSnodes, in.node_children, n)); CK(put(dLeafA, la.data(), n)); CK(put(dAdam, in.adam, 6 * n)); CK(put(dSampSum, which ? nullptr : in.tree_sum, n));
        CK(put(dSampWeight, which ? nullptr : in.tree_weight, n)); CK(put(dSampCount, which ? nullptr : in.tree_count, n)); CK(put(dSampDepth, which ? nullptr : in.tree_depth, n));
        CK(put(dBweight, which ? in.tree_weight : nullptr, n)); CK(put(dBuildCount, which ? in.tree_count : nullptr, n)); CK(put(dBuildDepth, which ? in.tree_depth : nullptr, n));
        CK(put(dBuildBase, which ? first.data() : nullptr, n));
        const std::vector<SampNode> pool = which ? std::vector<SampNode>() : to_pool(in.sums, in.children, in.n_pool);
        CK(put(dSamp, pool.data(), pool.size())); CK(put(dBchildren, which ? in.children : nullptr, in.n_pool)); CK(put(dTrain, which ? in.sums : nullptr, 4 * in.n_pool));
        const uint32_t sc[8] = {(uint32_t) n, 0, 0, 0, 0, 0, 0, 0};
        CK(put(dScalars, sc, 8));
        hNodes = (uint32_t) n; hTotalBuild = 0;
        return PPG_OK;
    }

    // STree::refine at `threshold`; a refine that runs out of node capacity raises the flag sync_counts reports
    int refine(float threshold) { stree_refine_kernel<<<1, 1024, 0, stream>>>(maint(), threshold, dScalars.p + 5); return 1; }
    // DTree::reset of every leaf, first half: node count of every new building tree, and their offsets in the pool
    int reset_count(int maxDepth, float threshold) {
        dtree_reset_kernel<false><<<numSMs * 4, 128, 0, stream>>>(maint(), nullptr, maxDepth, threshold);
        exclusive_scan_kernel<<<1, 1024, 0, stream>>>(dBuildCount.p, dBuildBase.p, dScalars.p, dScalars.p + 1);
        return 2;
    }
    // between the halves: read back the S-tree node count and the building pool total (waits for the stream), and make room for them and the table
    int sync_counts(bool exact = false) {
        uint32_t sc[8];
        CK(cudaMemcpyAsync(sc, dScalars.p, 32, cudaMemcpyDeviceToHost, stream));
        CK(cudaStreamSynchronize(stream));
        if (sc[5]) return fail(PPG_ERR_CUDA, "S-tree refinement ran out of node capacity");
        hNodes = sc[0]; hTotalBuild = sc[1];
        CK(dStable.alloc(kTableEntries));
        return reserve(hNodes, std::max<size_t>(hTotalBuild, 1), exact);
    }
    // second half: write the building trees, point every leaf at its own
    int reset_fill(int maxDepth, float threshold) {
        const MaintParams M = maint();
        dtree_reset_kernel<true><<<numSMs * 4, 128, 0, stream>>>(M, dBuildBase.p, maxDepth, threshold);
        leaf_after_reset_kernel<<<numSMs * 4, 256, 0, stream>>>(M, dBuildBase.p);
        return 2;
    }
    // prefix table of the S-tree (stree_lookup): the first 3 * PPG_STREE_TABLE_BITS levels of every descent become one load.
    // Past 0xFFFFFF nodes its entries cannot hold the node numbers: view() then hands out no table and the kernels walk from the root.
    int stree_table() {
        if (!stree_table_usable(hNodes)) return 0;
        stree_table_kernel<<<numSMs * 8, 256, 0, stream>>>(dSnodes.p, dStable.p);
        return 1;
    }
    // DTree::build of every leaf; then the distribution statistics (tree_stats_kernel writes the whole record)
    int build() { dtree_build_kernel<<<numSMs * 4, 128, 0, stream>>>(maint(), dBuildBase.p); return 1; }
    int tree_stats() { tree_stats_kernel<<<1, 1024, 0, stream>>>(maint(), dTreeStats.p); return 1; }
    // Vertex::commit into the building trees, gridY rows of blocks (one per slab); sampling-fraction records to dAdamRecA / B, their count to dScalars[3]
    int commit(CommitParams C, int record, uint32_t nPaths, uint32_t gridY) {
        if (!commitGrid) {      // resident blocks per SM from the occupancy calculator
            int occ = 0;
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, commit_kernel<1>, PPG_BLOCK, 0);
            commitGrid = numSMs * std::max(occ, 1);
        }
        C.snodes = dSnodes.p;
        C.adamRecA = dAdamRecA.p; C.adamRecB = dAdamRecB.p; C.adamTotal = dScalars.p + 3; C.adamCap = (uint32_t) std::min<size_t>(adamCap, 0xFFFFFFFFu);
        const dim3 g(std::min<int>(commitGrid, (int) ((nPaths + PPG_BLOCK - 1) / PPG_BLOCK)), gridY);
        if (record == 1) commit_kernel<1><<<g, PPG_BLOCK, 0, stream>>>(C); else commit_kernel<2><<<g, PPG_BLOCK, 0, stream>>>(C);
        return 1;
    }
    // the dScalars[3] records of dAdamRecA / B into per-leaf buckets in dAdamSortA / B (histogram, scan, scatter)
    int adam_bucket() {
        adam_hist_kernel<<<numSMs * 4, 256, 0, stream>>>(dAdamRecA.p, dScalars.p + 3, (uint32_t) adamCap, dAdamCount.p);
        exclusive_scan_kernel<<<1, 1024, 0, stream>>>(dAdamCount.p, dAdamOffset.p, dScalars.p, dScalars.p + 4);
        adam_scatter_kernel<<<numSMs * 4, 256, 0, stream>>>(dAdamRecA.p, dAdamRecB.p, dScalars.p + 3, (uint32_t) adamCap, dAdamOffset.p,
                                                            dAdamCursor.p, dAdamSortA.p, dAdamSortB.p);
        return 3;
    }
    int adam_replay(int loss) {
        adam_seq_kernel<<<numSMs * 16, 128, 0, stream>>>(maint(), dAdamSortA.p, dAdamSortB.p, dAdamOffset.p, dAdamCount.p, dAdamCursor.p,
                                                         loss == PPG_LOSS_KL ? 1.0f : 2.0f);
        return 1;
    }

    // The sampling (which == 0) or building trees into a caller's ppg_sdtree.  compact: the leaves' quadtrees concatenated in node order and
    // tree_first counted along them (ppg_export_sdtree: between the reset and the build of an iteration the sampling trees still sit where the
    // previous build put them, and a leaf the refine made shares its parent's).  Otherwise tree_first is the offset in the device pool, which
    // is copied from 0 to the end of the last leaf's quadtree: the ops' results keep the offsets the caller loaded.
    int store(int which, ppg_sdtree &out, bool compact = true) const {
        if (capNodes == 0) return fail(PPG_ERR_NO_SCENE, "no SD-tree yet");
        const uint32_t n = hNodes;
        std::vector<uint2> sn(n); std::vector<float4> la(n); std::vector<float> sum(n, 0.f), weight(n), adam(6 * (size_t) n); std::vector<int> depth(n); std::vector<uint32_t> count(n);
        CK(cudaMemcpy(sn.data(), dSnodes.p, sizeof(uint2) * n, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(la.data(), dLeafA.p, sizeof(float4) * n, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(adam.data(), dAdam.p, 24 * (size_t) n, cudaMemcpyDeviceToHost));
        if (which == 0) CK(cudaMemcpy(sum.data(), dSampSum.p, 4 * (size_t) n, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(weight.data(), which ? dBweight.p : dSampWeight.p, 4 * (size_t) n, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(depth.data(), which ? dBuildDepth.p : dSampDepth.p, 4 * (size_t) n, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(count.data(), which ? dBuildCount.p : dSampCount.p, 4 * (size_t) n, cudaMemcpyDeviceToHost));
        const auto first = [&](uint32_t i) { return f_bits(which ? la[i].y : la[i].x); };
        size_t total = 0, end = 0;
        for (uint32_t i = 0; i < n; ++i) if (sn[i].x == 0u) { total += count[i]; end = std::max<size_t>(end, (size_t) first(i) + count[i]); }
        if (end > capPool) return fail(PPG_ERR_CUDA, "SD-tree leaf points past the quadtree pool");
        out.n_nodes = n; out.n_pool = compact ? total : end;
        if (out.n_nodes > out.node_capacity || out.n_pool > out.pool_capacity)
            return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_sdtree output arrays too small (n_nodes and n_pool hold the sizes needed)");
        std::vector<SampNode> pool(end);                // building pool: bsums and bchildren, strided into the sampling pool's layout
        if (end && (out.sums || out.children)) {
            if (which) {
                CK(cudaMemcpy2D(&pool[0].sums, sizeof(SampNode), dTrain.p, sizeof(float4), sizeof(float4), end, cudaMemcpyDeviceToHost));
                CK(cudaMemcpy2D(&pool[0].children, sizeof(SampNode), dBchildren.p, sizeof(uint2), sizeof(uint2), end, cudaMemcpyDeviceToHost));
            } else CK(cudaMemcpy(pool.data(), dSamp.p, sizeof(SampNode) * end, cudaMemcpyDeviceToHost));
        }
        const auto row = [&](size_t k, const SampNode &q) {      // children keep their bytes (see to_pool)
            if (out.sums) memcpy(out.sums + 4 * k, &q.sums, 16);
            if (out.children) memcpy(out.children + 4 * k, &q.children, 8);
        };
        uint64_t off = 0;
        for (uint32_t i = 0; i < n; ++i) {          // inner nodes carry no tree and no optimiser state (STree::subdivide, GP:876-895)
            const bool leaf = sn[i].x == 0u;
            if (out.node_children) memcpy(out.node_children + 2 * (size_t) i, &sn[i], 8);
            if (out.tree_first) out.tree_first[i] = compact ? off : first(i);
            if (out.tree_count) out.tree_count[i] = leaf ? count[i] : 0u;
            if (out.tree_depth) out.tree_depth[i] = leaf ? depth[i] : 0;
            if (out.tree_sum) out.tree_sum[i] = leaf ? sum[i] : 0.f;
            if (out.tree_weight) out.tree_weight[i] = leaf ? weight[i] : 0.f;
            if (out.adam)                           // theta as the bounce kernel reads it
                for (int j = 0; j < 6; ++j) out.adam[6 * (size_t) i + j] = !leaf ? 0.f : j == 3 ? la[i].z : adam[6 * (size_t) i + j];
            if (!leaf || !compact) continue;
            for (uint32_t k = 0; k < count[i]; ++k) row(off + k, pool[first(i) + k]);
            off += count[i];
        }
        if (!compact) for (size_t k = 0; k < end; ++k) row(k, pool[k]);
        return PPG_OK;
    }
    // the building sums and weights a record or commit added to, back into the caller's tree
    int copy_back(const ppg_sdtree &b) const {
        if (b.sums) CK(cudaMemcpy(b.sums, dTrain.p, 16 * b.n_pool, cudaMemcpyDeviceToHost));
        if (b.tree_weight) CK(cudaMemcpy(b.tree_weight, dBweight.p, 4 * b.n_nodes, cudaMemcpyDeviceToHost));
        return PPG_OK;
    }
};

// ------------------------------------------------------------------ the integrator object
struct ppg_integrator {
    ppg_params prm;
    int device = 0, numSMs = 132;
    cudaStream_t stream = nullptr;
    cudaEvent_t evA = nullptr, evB = nullptr;
    TreeStats *hTreeStats = nullptr; bool treeStatsPending[PPG_MAX_ITERATIONS] = {};       // pinned; see build_sd_tree
    cudaEvent_t evLive[2] = {nullptr, nullptr}; uint32_t *liveHost = nullptr;   // pinned read-backs of the live counts, looked at one check point late
    std::atomic<bool> cancelled{false};
    std::string destination;
    int rank = 0, world = 1;
    ppg_allreduce_fn allreduce = nullptr; void *allreduceUser = nullptr;
    void *ncclComm = nullptr;                              // ncclComm_t when ppg_nccl_init was called: collectives are enqueued on `stream`, no host sync
    bool multi() const { return world > 1 && (ncclComm || allreduce); }
    ppg_clock_fn clockFn = nullptr; void *clockUser = nullptr; ppg_film_fn filmFn = nullptr; void *filmUser = nullptr;
    float clock_s() const { return clockFn ? (float) clockFn(clockUser) : (float) std::chrono::duration_cast<std::chrono::milliseconds>(std::chrono::steady_clock::now() - startTime).count() / 1000; }
    unsigned long long adamProgress[2] = {0, 0};          // [sum steps * |df| * 2^20, sum steps] of the last Adam replay
    uint64_t lastRecorded = 0;                             // guiding records of the last performRenderPasses (all ranks): bounds the growth of the S-tree

    // scene
    bool haveScene = false;
    DevBuf<unsigned char> dScene[kSceneArrays]; DevBuf<EnvLight> dEnvLight;     // one buffer per SceneArray (ppg_scene.h)
    SceneView sceneView; Camera cam; uint32_t sceneSmemBytes = 0;
    float aabbMin[3], aabbMax[3], extent[3];
    int W = 0, H = 0;
    DevBuf<uint32_t> dPixelMap, dPixelMapPerm; uint32_t nLocalPixels = 0, minLocalPixels = 0, maxLocalPixels = 0;

    // film
    DevBuf<float4> dImage, dSqImage, dFilm; DevBuf<float> dRgb; DevBuf<double> dVar;
    std::vector<DevBuf<float4> *> images; std::vector<float> variances;

    TreeStore tree;

    // wavefront
    size_t pathCapacity = 0; int maxBounces = 0, nSlabs = 0; int recordMode = 0; int stateVecs = 5, slabSets = 1;
    DevBuf<float4> dStateA, dStateB, dSlabs, dLiFinal; DevBuf<uint32_t> dLive, dWork; DevBuf<unsigned long long> dSplit, dCounters;
    DevBuf<float4> dHits; DevBuf<uint32_t> dTraceWork; int gridTrace = 0; uint32_t traceMinPaths = 0;   // separate nearest-hit pass (ppg_trace.cu), BVH scenes only
    DevBuf<uint32_t> dOrder, dBinCount;                                                                   // ... which also bins the paths by the BSDF class they hit
    int gridBounce = 0;

    // per-kernel-class CUDA-event timing on the launching stream
    struct Timed { cudaEvent_t a, b; int cls; uint32_t launches; };
    std::vector<Timed> evPool; size_t evUsed = 0; cudaEvent_t evRender0 = nullptr, evRender1 = nullptr;
    void tic(int cls) {
        if (evUsed == evPool.size()) { Timed t; cudaEventCreate(&t.a); cudaEventCreate(&t.b); t.cls = cls; t.launches = 1; evPool.push_back(t); }
        evPool[evUsed].cls = cls; evPool[evUsed].launches = 1; cudaEventRecord(evPool[evUsed].a, stream);
    }
    void toc(uint32_t nLaunches = 1) { evPool[evUsed].launches = nLaunches; cudaEventRecord(evPool[evUsed].b, stream); ++evUsed; }   // one bracket may hold several launches of a class
    void resolve_timers() {   // call after a stream synchronize
        for (size_t i = 0; i < evUsed; ++i) {
            float ms = 0; if (cudaEventElapsedTime(&ms, evPool[i].a, evPool[i].b) == cudaSuccess) { stats.kernel_ms[evPool[i].cls] += ms; stats.kernel_count[evPool[i].cls] += evPool[i].launches; }
        }
        evUsed = 0;
    }

    // run state (GP:2313-2323)
    bool isBuilt = false, isFinalIter = false, doNee = false; int iter = 0, passesRendered = 0; uint32_t nRealEmitters = 0; bool fullFeature = false;
    bool useNee() const { return prm.nee != PPG_NEE_NEVER && nRealEmitters > 0; }
    std::chrono::steady_clock::time_point startTime;
    ppg_stats stats; uint64_t launches = 0; double deviceMs = 0;

    ~ppg_integrator();
    void destroy_body() {
        for (auto *b : images) delete b;
        for (auto &t : evPool) { cudaEventDestroy(t.a); cudaEventDestroy(t.b); }
        if (evRender0) cudaEventDestroy(evRender0);
        if (evRender1) cudaEventDestroy(evRender1);
        if (evA) cudaEventDestroy(evA);
        if (evB) cudaEventDestroy(evB);
        for (auto &e : evLive) if (e) cudaEventDestroy(e);
        if (liveHost) cudaFreeHost(liveHost);
        if (hTreeStats) cudaFreeHost(hTreeStats);
        if (stream) cudaStreamDestroy(stream);
    }
};

ppg_integrator::~ppg_integrator() { destroy_body(); }
static double elapsed_ms(std::chrono::steady_clock::time_point s) { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - s).count(); }
static float elapsed_s(std::chrono::steady_clock::time_point s) {
    return (float) std::chrono::duration_cast<std::chrono::milliseconds>(std::chrono::steady_clock::now() - s).count() / 1000;
}

extern "C" int ppg_create(const ppg_params *params, int device, ppg_integrator **out) {
    if (!params || !out) return fail(PPG_ERR_INVALID_ARGUMENT, "null argument");
    int rc = ppg_params_validate(params);
    if (rc != PPG_OK) return rc;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return fail(PPG_ERR_NO_DEVICE, "no CUDA device available (this library has no CPU fallback)");
    }
    if (device < 0) { if (cudaGetDevice(&device) != cudaSuccess) device = 0; }
    if (device >= ndev) return fail(PPG_ERR_NO_DEVICE, "CUDA device index out of range");
    CK(cudaSetDevice(device));
    ppg_integrator *h = new ppg_integrator();
    h->prm = *params; h->device = device;
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, device));
    h->numSMs = prop.multiProcessorCount;
    CK(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    h->tree.stream = h->stream; h->tree.numSMs = h->numSMs;
    CK(cudaEventCreate(&h->evA)); CK(cudaEventCreate(&h->evB)); CK(cudaEventCreate(&h->evRender0)); CK(cudaEventCreate(&h->evRender1));
    for (auto &e : h->evLive) CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    CK(cudaHostAlloc((void **) &h->liveHost, 128 * sizeof(uint32_t), cudaHostAllocDefault));
    CK(cudaHostAlloc((void **) &h->hTreeStats, PPG_MAX_ITERATIONS * sizeof(TreeStats), cudaHostAllocDefault));
    memset(&h->stats, 0, sizeof(h->stats));
    *out = h;
    return PPG_OK;
}
static void release_comm(ppg_integrator *h);
extern "C" void ppg_destroy(ppg_integrator *h) {
    if (!h) return;
    cudaSetDevice(h->device);
    cudaStreamSynchronize(h->stream);
    release_comm(h);
    delete h;
}
extern "C" int ppg_set_destination(ppg_integrator *h, const char *destination) {
    if (!h) return PPG_ERR_INVALID_ARGUMENT; h->destination = destination ? destination : ""; return PPG_OK;
}
extern "C" int ppg_cancel(ppg_integrator *h) { if (!h) return PPG_ERR_INVALID_ARGUMENT; h->cancelled.store(true); return PPG_OK; }
extern "C" int ppg_set_allreduce(ppg_integrator *h, ppg_allreduce_fn cb, void *user) {
    if (!h) return PPG_ERR_INVALID_ARGUMENT; h->allreduce = cb; h->allreduceUser = user; return PPG_OK;
}

// ------------------------------------------------------------------ NCCL, resolved at run time (no link-time dependency: single-GPU hosts need no NCCL)
namespace {
struct NcclId { char internal[PPG_NCCL_UNIQUE_ID_BYTES]; };                // ncclUniqueId (nccl.h:37-38), passed by value
struct NcclApi {
    void *lib = nullptr;
    int (*getUniqueId)(NcclId *) = nullptr;
    int (*commInitRank)(void **, int, NcclId, int) = nullptr;
    int (*allReduce)(const void *, void *, size_t, int, int, void *, cudaStream_t) = nullptr;
    int (*commDestroy)(void *) = nullptr;
    const char *(*getErrorString)(int) = nullptr;
};
static NcclApi *nccl_api() {
    static NcclApi api; static bool tried = false;
    if (!tried) {
        tried = true;
        // a process that already holds NCCL (e.g. PyTorch's bundled copy) gets that one: same soname
        for (const char *name : {"libnccl.so.2", "libnccl.so"}) { api.lib = dlopen(name, RTLD_NOW | RTLD_GLOBAL); if (api.lib) break; }
        if (api.lib) {
            api.getUniqueId = (int (*)(NcclId *)) dlsym(api.lib, "ncclGetUniqueId");
            api.commInitRank = (int (*)(void **, int, NcclId, int)) dlsym(api.lib, "ncclCommInitRank");
            api.allReduce = (int (*)(const void *, void *, size_t, int, int, void *, cudaStream_t)) dlsym(api.lib, "ncclAllReduce");
            api.commDestroy = (int (*)(void *)) dlsym(api.lib, "ncclCommDestroy");
            api.getErrorString = (const char *(*)(int)) dlsym(api.lib, "ncclGetErrorString");
            if (!api.getUniqueId || !api.commInitRank || !api.allReduce) api.lib = nullptr;
        }
    }
    return api.lib ? &api : nullptr;
}
}  // namespace

static void release_comm(ppg_integrator *h) {
    if (h->ncclComm) { NcclApi *a = nccl_api(); if (a && a->commDestroy) a->commDestroy(h->ncclComm); h->ncclComm = nullptr; }
}
extern "C" int ppg_nccl_unique_id(void *id_out) {
    NcclApi *a = nccl_api();
    if (!a || !id_out) return fail(PPG_ERR_COMM, "libnccl.so.2 could not be loaded");
    NcclId id; const int rc = a->getUniqueId(&id);
    if (rc != 0) return fail(PPG_ERR_COMM, std::string("ncclGetUniqueId: ") + (a->getErrorString ? a->getErrorString(rc) : "error"));
    memcpy(id_out, &id, sizeof(id));
    return PPG_OK;
}
extern "C" int ppg_nccl_init(ppg_integrator *h, const void *id, int rank, int world_size) {
    if (!h || !id || world_size < 1 || rank < 0 || rank >= world_size) return fail(PPG_ERR_INVALID_ARGUMENT, "bad communicator arguments");
    NcclApi *a = nccl_api();
    if (!a) return fail(PPG_ERR_COMM, "libnccl.so.2 could not be loaded");
    CK(cudaSetDevice(h->device));
    release_comm(h);
    NcclId nid; memcpy(&nid, id, sizeof(nid));
    void *comm = nullptr;
    const int rc = a->commInitRank(&comm, world_size, nid, rank);
    if (rc != 0) return fail(PPG_ERR_COMM, std::string("ncclCommInitRank: ") + (a->getErrorString ? a->getErrorString(rc) : "error"));
    h->ncclComm = comm;
    return ppg_set_shard(h, rank, world_size);
}
extern "C" int ppg_set_clock(ppg_integrator *h, ppg_clock_fn fn, void *user) { if (!h) return PPG_ERR_INVALID_ARGUMENT; h->clockFn = fn; h->clockUser = user; return PPG_OK; }
extern "C" int ppg_set_film_callback(ppg_integrator *h, ppg_film_fn fn, void *user) { if (!h) return PPG_ERR_INVALID_ARGUMENT; h->filmFn = fn; h->filmUser = user; return PPG_OK; }

// sum `n` floats in place over all ranks.  NCCL: enqueued on the render stream, nothing waits on the host.  Callback: the stream is drained
// first and the callback returns once the result is visible in device memory.
static int allreduce_sum(ppg_integrator *h, float *dev, size_t n) {
    if (h->world <= 1) return PPG_OK;
    if (h->ncclComm) {
        const int rc = nccl_api()->allReduce(dev, dev, n, /* ncclFloat32 */ 7, /* ncclSum */ 0, h->ncclComm, h->stream);
        if (rc != 0) return fail(PPG_ERR_COMM, "ncclAllReduce failed");
        return PPG_OK;
    }
    if (!h->allreduce) return PPG_OK;
    CK(cudaStreamSynchronize(h->stream));
    if (h->allreduce(h->allreduceUser, dev, n) != 0) return fail(PPG_ERR_COMM, "allreduce callback failed");
    return PPG_OK;
}

// a stride near 0.618 n (golden ratio) that is coprime to n: j -> j * stride % n visits 0 .. n-1 once each, scattered over the whole range
static uint64_t golden_stride(uint64_t n) {
    uint64_t stride = std::max<uint64_t>(1, (uint64_t) ((double) n * 0.6180339887498949));
    while (std::gcd(stride, n) != 1) ++stride;
    return stride;
}

static int build_pixel_map(ppg_integrator *h) {
    // 32x32 image blocks (scene.cpp:24), dealt to the ranks round-robin along a scattered order of the blocks (golden_stride over the blocks):
    // every rank's blocks are spread over the whole image whatever the image width (plain `block % world` gives each rank
    // whole COLUMNS of blocks when the blocks per row are a multiple of the world size, and the columns of an image do not cost the same).
    // A rank visits its blocks row-major; row-major inside a block.
    const int bs = 32, bx = (h->W + bs - 1) / bs, by = (h->H + bs - 1) / bs, nb = bx * by;
    std::vector<int> owner((size_t) nb, 0);
    if (h->world > 1) {
        const uint64_t stride = golden_stride((uint64_t) nb);
        for (uint64_t j = 0; j < (uint64_t) nb; ++j) owner[(j * stride) % nb] = (int) (j % h->world);
    }
    std::vector<uint32_t> map; map.reserve((size_t) h->W * h->H / h->world + 1024);
    for (int b = 0; b < nb; ++b) {
        if (owner[b] != h->rank) continue;
        const int x0 = (b % bx) * bs, y0 = (b / bx) * bs;
        for (int y = y0; y < std::min(y0 + bs, h->H); ++y)
            for (int x = x0; x < std::min(x0 + bs, h->W); ++x) map.push_back((uint32_t) x | ((uint32_t) y << 16));
    }
    h->nLocalPixels = (uint32_t) map.size();
    h->minLocalPixels = 0xffffffffu; h->maxLocalPixels = 0;   // smallest / largest share of any rank: decisions every rank must take alike
    for (int r = 0; r < h->world; ++r) {
        uint64_t c = 0;
        for (int b = 0; b < nb; ++b) { if (owner[b] != r) continue; const int x0 = (b % bx) * bs, y0 = (b / bx) * bs; c += (uint64_t) (std::min(x0 + bs, h->W) - x0) * (std::min(y0 + bs, h->H) - y0); }
        h->minLocalPixels = std::min<uint32_t>(h->minLocalPixels, (uint32_t) c); h->maxLocalPixels = std::max<uint32_t>(h->maxLocalPixels, (uint32_t) c);
    }
    CK(h->dPixelMap.alloc(std::max<size_t>(map.size(), 1)));
    if (!map.empty()) CK(cudaMemcpy(h->dPixelMap.p, map.data(), map.size() * 4, cudaMemcpyHostToDevice));
    // A second, scattered order of the same pixels (golden_stride over runs of 8 pixels): any contiguous range of it is spread evenly over
    // the image.  The sub-batches of a learning iteration (perform_render_passes) take their pixels from it, so that every S-tree leaf receives its
    // share of every sub-batch -- like the reference, whose worker threads interleave image blocks while the sampling fractions adapt.
    std::vector<uint32_t> perm(map.size());
    if (!map.empty()) {
        const uint64_t n = map.size();
        // ... in runs of 8 consecutive map entries (8 neighbouring pixels of one block row): a quarter of a warp starts coherent,
        // which the BVH walk of the first bounce -- the largest launch of a sub-batch -- feels; a slice of 10^4 paths still holds
        // > 10^3 runs spread over the whole image
        const uint64_t run = 8, nr = (n + run - 1) / run, rs = golden_stride(nr);
        uint64_t w = 0;
        for (uint64_t r = 0; r < nr; ++r) { const uint64_t src = (r * rs) % nr; for (uint64_t k = src * run; k < std::min(n, (src + 1) * run); ++k) perm[w++] = map[k]; }
    }
    CK(h->dPixelMapPerm.alloc(std::max<size_t>(perm.size(), 1)));
    if (!perm.empty()) CK(cudaMemcpy(h->dPixelMapPerm.p, perm.data(), perm.size() * 4, cudaMemcpyHostToDevice));
    return PPG_OK;
}

extern "C" int ppg_set_shard(ppg_integrator *h, int rank, int world_size) {
    if (!h || world_size < 1 || rank < 0 || rank >= world_size) return fail(PPG_ERR_INVALID_ARGUMENT, "bad shard");
    CK(cudaSetDevice(h->device));
    h->rank = rank; h->world = world_size;
    if (h->haveScene) return build_pixel_map(h);
    return PPG_OK;
}

static int ppg_set_scene_impl(ppg_integrator *h, const ppg_scene_desc *s);
extern "C" int ppg_set_scene(ppg_integrator *h, const ppg_scene_desc *s) { return guarded("ppg_set_scene", [&] { return ppg_set_scene_impl(h, s); }); }
static int ppg_set_scene_impl(ppg_integrator *h, const ppg_scene_desc *s) {
    if (!h || !s) return fail(PPG_ERR_INVALID_ARGUMENT, "null argument");
    PackedScene p; std::string err;
    if (const int rc = pack_scene(*s, p, err)) return fail(rc, err);
    CK(cudaSetDevice(h->device));
    // From here on the old scene is being overwritten: until the new one is complete there is none (ppg_render: PPG_ERR_NO_SCENE).
    h->haveScene = false;
    for (int i = 0; i < kSceneArrays; ++i) {          // the buffers are kept across calls and grow only: a repeated set_scene allocates nothing
        const PackedScene::Span a = p.array(i);
        if (!a.bytes) continue;
        CK(h->dScene[i].alloc(a.bytes));
        CK(cudaMemcpy(h->dScene[i].p, a.data, a.bytes, cudaMemcpyHostToDevice));
    }
    if (p.view.envW) CK(h->dEnvLight.alloc(1));
    EnvLight env;
    bind_scene(p, [&](int i) -> const void * { return p.array(i).bytes ? h->dScene[i].p : nullptr; }, h->dEnvLight.p, h->sceneView, env);
    if (p.view.envW) CK(cudaMemcpy(h->dEnvLight.p, &env, sizeof(env), cudaMemcpyHostToDevice));
    h->cam = p.cam; h->W = p.W; h->H = p.H;
    h->sceneSmemBytes = p.sceneSmemBytes; h->nRealEmitters = p.nRealEmitters; h->fullFeature = p.fullFeature;
    for (int i = 0; i < 3; ++i) { h->aabbMin[i] = p.aabbMin[i]; h->aabbMax[i] = p.aabbMax[i]; h->extent[i] = p.extent[i]; }
    const size_t npx = (size_t) h->W * h->H;
    CK(h->dImage.alloc(npx)); CK(h->dSqImage.alloc(npx)); CK(h->dFilm.alloc(npx)); CK(h->dRgb.alloc(3 * npx)); CK(h->dVar.alloc(1));
    h->haveScene = true;
    return build_pixel_map(h);
}

// S-tree node capacity for a refine: a leaf splits only while its weight exceeds the threshold, so the refinement creates at most
// 4 nodes per threshold worth of building weight
static double refine_capacity(size_t nodes, double totalWeight, float threshold) { return (double) nodes + 4.0 * totalWeight / std::max(1.0f, threshold) + 1024; }

// resetSDTree, GP:1108-1113
static int reset_sd_tree(ppg_integrator *h) {
    const double thr = std::sqrt(std::pow(2.0, h->iter) * h->prm.spp_per_pass / 4) * h->prm.s_tree_threshold;
    const float threshold = (float) (size_t) thr;                   // (size_t) cast then Float comparison, GP:1111 + 953-955
    // upper bound of the node count after refinement: every leaf can at most double per halving of its weight;
    // the total weight of the last iteration bounds the number of new leaves by 2*W/threshold
    bool memCapped = false;
    if (h->prm.sd_tree_max_memory >= 0) {   // GP:958-967 (footprint approximated by node counts: 2 trees x 24 B per node + per-tree overhead)
        const size_t fp = (size_t) h->tree.hTotalBuild * 2 * 24 + (size_t) h->tree.hNodes * 96;
        memCapped = fp / 1000000 >= (size_t) h->prm.sd_tree_max_memory;
    }
    if (!memCapped) {
        // capacity: the refinement creates at most 2 nodes per threshold worth of recorded weight.  The total weight of the iteration is at most
        // its number of guiding records (weights <= 1), summed over the ranks whose weights are reduced.
        const double totalW = 1.25 * (double) h->lastRecorded + 4096;
        const double est = refine_capacity(h->tree.hNodes, totalW, threshold);
        int rc = h->tree.reserve((uint32_t) std::min<double>(est, 4.0e9), h->tree.capPool);
        if (rc) return rc;
        h->tic(PPG_K_REFINE); h->launches += h->tree.refine(threshold); h->toc();
    }
    h->tic(PPG_K_RESET); h->launches += h->tree.reset_count(20, h->prm.d_tree_threshold); h->toc();
    int rc = h->tree.sync_counts(); if (rc) return rc;
    h->tic(PPG_K_RESET); h->launches += h->tree.reset_fill(20, h->prm.d_tree_threshold); h->toc();
    if (stree_table_usable(h->tree.hNodes)) { h->tic(PPG_K_REFINE); h->launches += h->tree.stree_table(); h->toc(); }
    CK(cudaGetLastError());
    return PPG_OK;      // no synchronize: the passes queue behind the reset
}

// the one exchange step (SURVEY 8e): sum the building statistics over all ranks
__global__ void pack_tail_kernel(float *tail, float *bweight, uint32_t n, int dir) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        if (dir == 0) tail[i] = bweight[i]; else bweight[i] = tail[i];
    }
}
static int exchange_training_statistics(ppg_integrator *h) {
    if (!h->multi()) return PPG_OK;
    float *tail = h->tree.dTrain.p + 4 * (size_t) h->tree.hTotalBuild;
    pack_tail_kernel<<<h->numSMs, 256, 0, h->stream>>>(tail, h->tree.dBweight.p, h->tree.hNodes, 0); h->launches++;
    int rc = allreduce_sum(h, h->tree.dTrain.p, 4 * (size_t) h->tree.hTotalBuild + (size_t) h->tree.hNodes); if (rc) return rc;
    pack_tail_kernel<<<h->numSMs, 256, 0, h->stream>>>(tail, h->tree.dBweight.p, h->tree.hNodes, 1); h->launches++;
    return PPG_OK;
}
// a host scalar made identical on all ranks (rank 0's value wins): time-based decisions must not diverge
static int sync_scalar(ppg_integrator *h, float *v) {
    if (!h->multi()) return PPG_OK;
    float *slot = h->tree.dTrain.p + h->tree.dTrain.n - 16;
    const float mine = h->rank == 0 ? *v : 0.f;
    CK(cudaMemcpyAsync(slot, &mine, 4, cudaMemcpyHostToDevice, h->stream));
    int rc = allreduce_sum(h, slot, 1); if (rc) return rc;
    CK(cudaMemcpyAsync(v, slot, 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return PPG_OK;
}

// buildSDTree, GP:1115-1189, with its "Distribution statistics" (GP:1121-1186) reduced on the device: 64 bytes come back
static int build_sd_tree(ppg_integrator *h, ppg_iteration_stats &st) {
    int rc = exchange_training_statistics(h);
    if (rc) return rc;
    h->tic(PPG_K_BUILD); h->launches += h->tree.build(); h->toc();
    CK(cudaGetLastError());
    h->launches += h->tree.tree_stats();
    // the statistics are only reported: they go to pinned memory and are folded into ppg_stats after the render's last synchronize
    const int slot = std::min(h->iter, PPG_MAX_ITERATIONS - 1);
    CK(cudaMemcpyAsync(h->hTreeStats + slot, h->tree.dTreeStats.p, sizeof(TreeStats), cudaMemcpyDeviceToHost, h->stream));
    h->treeStatsPending[slot] = true;
    st.s_tree_nodes = h->tree.hNodes;
    h->isBuilt = true;
    return PPG_OK;
}
static void finish_tree_stats(ppg_integrator *h) {      // after a stream synchronize
    for (int i = 0; i < PPG_MAX_ITERATIONS; ++i) {
        if (!h->treeStatsPending[i]) continue;
        h->treeStatsPending[i] = false;
        const TreeStats &ts = h->hTreeStats[i]; ppg_iteration_stats &st = h->stats.iterations[i];
        const int nPoints = (int) ts.leaves, nPointsNodes = (int) ts.leavesWithNodes;
        float avgDepth = (float) ts.depthSum, avgR = (float) ts.meanSum, avgN = (float) ts.nodesSum, avgW = (float) ts.weightSum;
        if (nPoints > 0) { avgDepth /= nPoints; avgR /= nPoints; if (nPointsNodes > 0) avgN /= nPointsNodes; avgW /= nPoints; }
        st.depth_min = nPoints ? ts.depthMin : std::numeric_limits<int>::max(); st.depth_max = ts.depthMax; st.depth_avg = avgDepth;
        st.mean_radiance_min = nPoints ? ts.meanMin : std::numeric_limits<float>::max(); st.mean_radiance_avg = avgR; st.mean_radiance_max = ts.meanMax;
        st.nodes_min = nPointsNodes ? ts.nodesMin : std::numeric_limits<size_t>::max(); st.nodes_max = ts.nodesMax; st.nodes_avg = avgN;
        st.weight_min = nPoints ? ts.weightMin : std::numeric_limits<float>::max(); st.weight_avg = avgW; st.weight_max = ts.weightMax;
        st.s_tree_leaves = ts.leaves;
    }
}

// ------------------------------------------------------------------ wavefront buffers
static int ensure_wavefront(ppg_integrator *h) {
    const size_t perPass = (size_t) h->maxLocalPixels * h->prm.spp_per_pass;       // the largest share of any rank: every rank splits an iteration into the same batches
    h->maxBounces = h->prm.max_depth > 0 ? h->prm.max_depth : 64;
    h->nSlabs = std::max(1, h->maxBounces - 1);
    const bool nee = h->useNee();
    const bool full = nee || h->prm.spatial_filter != PPG_SFILTER_NEAREST || h->prm.bsdf_sampling_fraction_loss != PPG_LOSS_NONE;
    h->recordMode = full ? 2 : 1;
    const int stateVecs = nee ? 7 : 5, slabSets = nee ? 2 : 1;
    const size_t perPath = 2 * 16 * (size_t) stateVecs + 16 + (size_t) h->nSlabs * (full ? 96 : 48) * slabSets;
    size_t cap = std::min((size_t) 1 << 23, ((size_t) 24 << 30) / perPath);   // at most 2^23 paths and 24 GiB of path state and slabs
    cap = std::max(cap, perPass);                          // one pass must fit
    cap = (cap / std::max<size_t>(perPass, 1)) * std::max<size_t>(perPass, 1);   // whole passes only
    cap = std::max(cap, perPass);
    if (cap >= (1ull << 30)) return fail(PPG_ERR_INVALID_ARGUMENT, "pass too large for 30-bit path ids");
    if (cap != h->pathCapacity || stateVecs != h->stateVecs || slabSets != h->slabSets) {
        h->dStateA.release(); h->dStateB.release(); h->dSlabs.release(); h->dLiFinal.release();
        CK(h->dStateA.alloc(stateVecs * cap)); CK(h->dStateB.alloc(stateVecs * cap)); CK(h->dLiFinal.alloc(cap));
        CK(h->dSlabs.alloc((size_t) h->nSlabs * (full ? 6 : 3) * cap * slabSets));
        h->pathCapacity = cap; h->stateVecs = stateVecs; h->slabSets = slabSets;
    }
    CK(h->dLive.alloc(h->maxBounces + 2)); CK(h->dSplit.alloc(h->maxBounces + 2)); CK(h->dWork.alloc(h->maxBounces + 2)); CK(h->dCounters.alloc(8));
    if (h->prm.bsdf_sampling_fraction_loss != PPG_LOSS_NONE) {
        // sampling-fraction records: one per (recorded vertex, leaf) pair.  Sized once for the largest wavefront with 16 records per path (mean path
        // lengths of the bundled scenes: 4 - 9 vertices; the spatial box filter touches ~2 leaves per vertex); a record beyond it is dropped and
        // counted in ppg_stats.dropped_records.  Allocating per batch (cudaMalloc / cudaFree are synchronous) cost 11 ms per sub-batch.
        const size_t want = cap * 16 * (h->prm.spatial_filter == PPG_SFILTER_BOX ? 2 : 1);
        if (want > h->tree.adamCap) {
            h->tree.dAdamRecA.release(); h->tree.dAdamRecB.release(); h->tree.dAdamSortA.release(); h->tree.dAdamSortB.release();
            CK(h->tree.dAdamRecA.alloc(want)); CK(h->tree.dAdamRecB.alloc(want)); CK(h->tree.dAdamSortA.alloc(want)); CK(h->tree.dAdamSortB.alloc(want));
            h->tree.adamCap = want;
        }
    }
    // persistent grids: resident blocks per SM from the occupancy calculator
    int occ = 0;
    if (h->sceneSmemBytes) occ = h->fullFeature ? ppg_bounce_occupancy_11(h->sceneSmemBytes) : ppg_bounce_occupancy_10(h->sceneSmemBytes);
    else occ = h->fullFeature ? ppg_bounce_occupancy_01(0) : ppg_bounce_occupancy_00(0);
    CK(cudaGetLastError());
    // one block per resident slot; warps claim their work dynamically (bounce_kernel)
    h->gridBounce = h->numSMs * std::max(occ, 1);
    // Scenes walked through the BVH find their hits in a separate pass of persistent warps (ppg_trace.cu) whenever the wavefront is large enough
    // to pay for the second launch per depth; tiny learning sub-batches keep the fused kernel.  PPG_TRACE_MIN_PATHS=0 turns the pass off
    // (the tests use it to compare the pass with the fused kernel).
    h->gridTrace = 0;
    const char *minPaths = getenv("PPG_TRACE_MIN_PATHS");
    h->traceMinPaths = (uint32_t) std::max(minPaths && *minPaths ? atoi(minPaths) : 32768, 0);
    if (!h->sceneSmemBytes && h->sceneView.nGroups == 0u && h->sceneView.nTris != 0u && h->traceMinPaths != 0u) {
        CK(h->dHits.alloc(h->pathCapacity)); CK(h->dTraceWork.alloc(h->maxBounces + 2));
        // ... and the trace pass bins the paths by the BSDF class they hit (render_batch); a lean scene has one kind of BSDF only: nothing to sort
        if (h->fullFeature) { CK(h->dOrder.alloc((size_t) PPG_BINS * h->pathCapacity)); CK(h->dBinCount.alloc((size_t) PPG_BINS * (h->maxBounces + 2))); }
        h->gridTrace = h->numSMs * std::max(ppg_trace_occupancy(), 1);
        CK(cudaGetLastError());
    }
    return PPG_OK;
}

static PathState path_state(float4 *base, size_t cap, bool nee) {
    PathState s; s.s0 = base; s.s1 = base + cap; s.s2 = base + 2 * cap; s.s3 = base + 3 * cap; s.s4 = base + 4 * cap;
    s.s5 = nee ? base + 5 * cap : nullptr; s.s6 = nee ? base + 6 * cap : nullptr; return s;
}
static VertexSlab slab_at(ppg_integrator *h, int k, int set = 0) {
    const size_t cap = h->pathCapacity; const int per = h->recordMode == 2 ? 6 : 3;
    float4 *b = h->dSlabs.p + (size_t) set * h->nSlabs * per * cap;
    VertexSlab s;
    // field-major layout: field f of slab k at ((f * nSlabs) + k) * cap, so that slab k+1 of a field is +cap (commit's slabStride)
    s.v0 = b + ((size_t) 0 * h->nSlabs + k) * cap; s.v1 = b + ((size_t) 1 * h->nSlabs + k) * cap; s.v2 = b + ((size_t) 2 * h->nSlabs + k) * cap;
    if (per == 6) { s.v3 = b + ((size_t) 3 * h->nSlabs + k) * cap; s.v4 = b + ((size_t) 4 * h->nSlabs + k) * cap; s.v5 = b + ((size_t) 5 * h->nSlabs + k) * cap; }
    else { s.v3 = s.v4 = s.v5 = nullptr; }
    return s;
}

static void launch_bounce(ppg_integrator *h, const RenderParams &P, bool first, int record, int grid, bool nee) {
    // scene staged in shared memory or read from HBM; lean instantiations for diffuse-only triangle scenes
    const BounceLaunch L{h->stream, grid, record, nee ? 1 : 0, first ? 1 : 0};
    if (P.sceneSmemBytes) { if (h->fullFeature) ppg_launch_bounce_11(P, L); else ppg_launch_bounce_10(P, L); }
    else { if (h->fullFeature) ppg_launch_bounce_01(P, L); else ppg_launch_bounce_00(P, L); }
    h->launches++;
}

// one batch of `nPasses` passes as a single wavefront, over `pixelCount` of this rank's pixels taken from `pixelMap` (a range of the block-ordered
// map or of its scattered permutation).  A rank without pixels in the batch still takes part in the collective of the Adam replay.
static int render_batch(ppg_integrator *h, int nPasses, const uint32_t *pixelMap, uint32_t pixelCount) {
    const uint32_t nPaths = (uint32_t) ((size_t) nPasses * pixelCount * h->prm.spp_per_pass);
    const int record = h->isFinalIter ? 0 : h->recordMode;
    const bool nee = h->useNee();                      // the NEE kernels also carry the MIS state when doNee is off (kickstart after 128 spp)
    const int lossMode = (record && h->isBuilt) ? h->prm.bsdf_sampling_fraction_loss : PPG_LOSS_NONE;       // GP:2152
    const bool useAdam = lossMode != PPG_LOSS_NONE;
    const bool neeSlabs = nee && h->doNee && h->prm.nee != PPG_NEE_ALWAYS;
    if (useAdam) CK(cudaMemsetAsync(h->tree.dScalars.p + 3, 0, 4, h->stream));      // record cursor (buffers: ensure_wavefront)
    if (nPaths) {
        CK(cudaMemsetAsync(h->dLive.p, 0, 4 * (size_t) (h->maxBounces + 2), h->stream));
        CK(cudaMemsetAsync(h->dWork.p, 0, 4 * (size_t) (h->maxBounces + 2), h->stream));
        CK(cudaMemsetAsync(h->dSplit.p, 0, 8 * (size_t) (h->maxBounces + 2), h->stream));
        CK(cudaMemcpyAsync(h->dLive.p, &nPaths, 4, cudaMemcpyHostToDevice, h->stream));
        RenderParams P;
        P.scene = h->sceneView; P.cam = h->cam; P.tree = h->tree.view(h->aabbMin, h->extent);
        P.pathCapacity = (uint32_t) h->pathCapacity;
        P.liFinal = h->dLiFinal.p; P.pixelMap = pixelMap; P.counters = h->dCounters.p;
        P.nPaths = nPaths; P.nLocalPixels = pixelCount; P.spp = (uint32_t) h->prm.spp_per_pass;
        P.passBase = (uint64_t) h->passesRendered; P.seed = h->prm.seed;
        P.maxDepth = h->prm.max_depth; P.rrDepth = h->prm.rr_depth; P.strictNormals = h->prm.strict_normals; P.hideEmitters = h->prm.hide_emitters;
        P.isBuilt = h->isBuilt ? 1 : 0; P.lossMode = h->prm.bsdf_sampling_fraction_loss; P.fixedFraction = h->prm.bsdf_sampling_fraction;
        P.sceneSmemBytes = h->sceneSmemBytes;
        P.neeMode = h->prm.nee; P.doNee = (nee && h->doNee) ? 1 : 0; P.training = record != 0 ? 1 : 0;
        PathState A = path_state(h->dStateA.p, h->pathCapacity, nee), B = path_state(h->dStateB.p, h->pathCapacity, nee);
        const int bb = h->sceneSmemBytes ? PPG_BOUNCE_BLOCK : PPG_BOUNCE_BLOCK_HBM;
        const int grid = std::min<int>(h->gridBounce, (int) ((nPaths + bb - 1) / bb));
        const bool useTrace = h->gridTrace > 0 && nPaths >= h->traceMinPaths;
        P.hits = useTrace ? h->dHits.p : nullptr; P.traceWork = nullptr;
        const bool bins = useTrace && h->fullFeature;              // material bins (buffers: ensure_wavefront)
        P.order = bins ? h->dOrder.p : nullptr; P.binCount = nullptr; P.binStride = (uint32_t) h->pathCapacity;
        if (useTrace) CK(cudaMemsetAsync(h->dTraceWork.p, 0, 4 * (size_t) (h->maxBounces + 2), h->stream));
        if (bins) CK(cudaMemsetAsync(h->dBinCount.p, 0, 4 * (size_t) PPG_BINS * (h->maxBounces + 2), h->stream));
        int lastDepth = 0, pendingDepth = 0; uint32_t bracket = 0;
        for (int depth = 1; depth <= h->maxBounces; ++depth) {
            P.depth = depth; P.in = (depth & 1) ? B : A; P.out = (depth & 1) ? A : B;
            P.liveIn = h->dLive.p + (depth - 1); P.liveOut = h->dLive.p + depth; P.work = h->dWork.p + depth;
            P.splitIn = h->dSplit.p + (depth - 1); P.splitOut = h->dSplit.p + depth;
            const int k = std::min(depth - 1, h->nSlabs - 1);
            P.slab = slab_at(h, k);
            if (nee) { P.neeSlab = slab_at(h, k, 1); P.prevSlab = slab_at(h, std::max(k - 1, 0)); if (depth - 1 >= h->nSlabs) P.prevSlab = slab_at(h, h->nSlabs - 1); }
            const int rec = (depth - 1 < h->nSlabs) ? record : 0;
            if (h->cancelled.load()) { if (bracket) h->toc(bracket); return PPG_ERR_CANCELLED; }   // Integrator::cancel() (GP:1643-1648): the batch in flight is dropped
            if (!bracket) h->tic(PPG_K_BOUNCE);                                // one event pair around the consecutive bounce launches (2 records per launch were
            if (useTrace) {                                                    // nearest hits of this depth's rays, then the bounce kernel shades them
                P.traceWork = h->dTraceWork.p + depth;
                if (bins) P.binCount = h->dBinCount.p + (size_t) PPG_BINS * depth;
                ppg_launch_trace(P, h->stream, std::min<int>(h->gridTrace, (int) ((nPaths + 255) / 256)), depth == 1, h->sceneView.nSpheres != 0u); h->launches++;
            }
            launch_bounce(h, P, depth == 1, rec, grid, nee);                   // (host time per launch adds up when a step is short: several GPUs split one step)
            ++bracket;
            lastDepth = depth;
            // unbounded path length (maxDepth == -1 runs up to the 64-bounce cap): stop launching once the wavefront is empty.  The live count is
            // copied to pinned memory at every check point and LOOKED AT one check point later, after the next launches are queued: the host
            // never drains the stream (a blocking read-back cost ~25 us of idle GPU per check: 3-5 ms per CBOX step), and a dead wavefront costs
            // at most two check intervals of empty launches (~2 us each).
            const bool small = nPaths <= 65536u;          // small wavefronts are launch bound: look every 4 bounces from the start
            if ((h->prm.max_depth <= 0 || small) && depth < h->maxBounces && depth % 4 == 0 && (small || depth >= 8)) {
                CK(cudaMemcpyAsync(h->liveHost + depth, h->dLive.p + depth, 4, cudaMemcpyDeviceToHost, h->stream));
                CK(cudaEventRecord(h->evLive[(depth >> 2) & 1], h->stream));
                if (pendingDepth) {
                    CK(cudaEventSynchronize(h->evLive[(pendingDepth >> 2) & 1]));
                    if (h->liveHost[pendingDepth] == 0) break;
                }
                pendingDepth = depth;
            }
        }
        if (bracket) h->toc(bracket);
        {   // survivors of the bounce cap (maxDepth == -1 only) keep the radiance they have; they are counted (ppg_stats.truncated_paths)
            const PathState last = (lastDepth & 1) ? A : B;
            flush_kernel<<<std::max(grid / 4, 1), PPG_BLOCK, 0, h->stream>>>(last, h->dLive.p + lastDepth, h->dSplit.p + lastDepth, (uint32_t) h->pathCapacity, h->dLiFinal.p, h->dCounters.p + 3); h->launches++;
        }
        if (record) {
            CommitParams C;
            C.tree = h->tree.view(h->aabbMin, h->extent); C.slab0 = slab_at(h, 0); C.slabStride = h->pathCapacity; C.liveCounts = h->dLive.p; C.liFinal = h->dLiFinal.p;
            C.spatialFilter = h->prm.spatial_filter; C.directionalFilter = h->prm.directional_filter;
            C.lossMode = lossMode;
            C.statisticalWeight = (h->prm.nee == PPG_NEE_KICKSTART && h->doNee && nee) ? 0.5f : 1.0f;   // GP:2152
            C.seed = h->prm.seed; C.nSlabs = (uint32_t) std::min(h->nSlabs, lastDepth);
            C.nee0 = neeSlabs ? slab_at(h, 0, 1) : C.slab0;
            C.dropped = h->dCounters.p + 4;
            h->tic(PPG_K_COMMIT); h->launches += h->tree.commit(C, record, nPaths, C.nSlabs * (neeSlabs ? 2 : 1)); h->toc();
        }
        h->tic(PPG_K_FILM);
        film_kernel<<<std::min<int>(h->numSMs * 8, (int) ((pixelCount + PPG_BLOCK - 1) / PPG_BLOCK)), PPG_BLOCK, 0, h->stream>>>(
            h->dLiFinal.p, pixelMap, pixelCount, (uint32_t) h->prm.spp_per_pass, (uint32_t) nPasses, h->W, h->dImage.p, h->dSqImage.p);
        h->toc(); h->launches++;
    }
    if (useAdam) {
        // replay the sampling-fraction records leaf by leaf (see adam_seq_kernel)
        const MaintParams M = h->tree.maint();
        const bool multi = h->multi();
        float *tail = h->tree.dTrain.p + 4 * (size_t) h->tree.hTotalBuild;       // [6 x nNodes] exchange area (the building weights are packed there only at iteration end)
        adam_pack_kernel<<<h->numSMs, 256, 0, h->stream>>>(M, tail, h->tree.dAdamBefore.p, nullptr, 0); h->launches++;
        h->tic(PPG_K_OTHER); h->launches += h->tree.adam_bucket(); h->toc();      // bucket the records by leaf (histogram, scan, scatter): "other"
        h->tic(PPG_K_ADAM); h->launches += h->tree.adam_replay(lossMode); h->toc();      // the sequential replay itself: "adam"
        if (multi) {
            // replicas replayed their own records from the common state: merge them (steps and moves of the variable add up, moments are
            // weighted by the steps, batch accumulators add up relative to the common start) so that all ranks continue identically
            adam_pack_kernel<<<h->numSMs, 256, 0, h->stream>>>(M, tail, h->tree.dAdamBefore.p, nullptr, 1); h->launches++;
            int rc = allreduce_sum(h, tail, 6 * (size_t) h->tree.hNodes); if (rc) return rc;
            adam_merge_kernel<<<h->numSMs, 256, 0, h->stream>>>(M, tail, h->tree.dAdamBefore.p, (float) (h->world - 1)); h->launches++;
        }
        // movement of the fractions in this replay (identical on all ranks after the merge): steers the size of the next sub-batch
        CK(cudaMemsetAsync(h->dCounters.p + 6, 0, 16, h->stream));
        adam_progress_kernel<<<h->numSMs, 256, 0, h->stream>>>(M, h->tree.dAdamBefore.p, h->dCounters.p + 6); h->launches++;
        CK(cudaMemcpyAsync(h->adamProgress, h->dCounters.p + 6, 16, cudaMemcpyDeviceToHost, h->stream));
    }
    CK(cudaGetLastError());
    return PPG_OK;
}

// performRenderPasses, GP:1210-1329
static int perform_render_passes(ppg_integrator *h, float &variance, int numPasses, ppg_iteration_stats &st) {
    const size_t npx = (size_t) h->W * h->H;
    CK(cudaMemsetAsync(h->dImage.p, 0, sizeof(float4) * npx, h->stream));
    CK(cudaMemsetAsync(h->dSqImage.p, 0, sizeof(float4) * npx, h->stream));
    CK(cudaMemsetAsync(h->dCounters.p, 0, 64, h->stream));
    const auto t0 = std::chrono::steady_clock::now();
    CK(cudaEventRecord(h->evA, h->stream));
    const size_t perPass = (size_t) h->nLocalPixels * h->prm.spp_per_pass;
    const size_t perPassMax = (size_t) h->maxLocalPixels * h->prm.spp_per_pass;                 // rank independent
    const int maxBatch = (int) std::max<size_t>(1, perPassMax ? h->pathCapacity / perPassMax : 1);
    // Sampling-fraction learning (GP:672-697).  The reference takes an optimiser step after every ~2 records WHILE the passes run, so the
    // fractions that guide the paths follow the optimiser with a lag of a few paths.  A wavefront samples all its paths with the fractions
    // it starts with; the Adam replay after it (adam_seq_kernel) then takes every step the reference would.  To bound that staleness a
    // learning iteration is rendered as a sequence of sub-batches (first fractions of a pass in the scattered pixel order, later whole passes)
    // whose size follows a step-size control: see `target` below.  All quantities that shape the sequence are identical on every rank.
    const bool learning = h->isBuilt && !h->isFinalIter && h->prm.bsdf_sampling_fraction_loss != PPG_LOSS_NONE;
    // Step-size control: after every replay the device reports how far the fractions moved (steps-weighted mean |df|).  The next sub-batch is sized
    // so that the fractions move by about `target` during it: that movement IS the staleness of the fractions a wavefront samples with.
    // Measured on SPACESHIP 640x360 (recorded vertices of iterations 1-4 against the CPU restatement of the reference, which learns online like it; its
    // own run-to-run spread is ~0.5 %): target 0.005 -> +0.2 % (2200 sub-batches), 0.01 -> +0.4 % (1130), 0.02 -> +1.2 % (223), 0.04 -> +4 % (58).
    constexpr double target = 0.02;
    constexpr double growthMax = 1.0;      // a sub-batch holds at most as many passes as the iteration has rendered before it
    constexpr double leafPaths = 4.0;      // paths per S-tree leaf in the first sub-batch
    const double pathsPerPass = (double) npx * h->prm.spp_per_pass;                                  // whole image
    const double minFrac = std::min(1.0, std::max(256.0, leafPaths * 0.5 * (h->tree.hNodes + 1)) / std::max(pathsPerPass, 1.0));
    double done = 0.0, frac = 0.0;          // passes rendered in this call (real number), fraction of the pass in progress
    double want = learning ? minFrac : (double) maxBatch, lastSize = 0.0;
    int local = 0; int rcode = PPG_OK;
    while (local < numPasses) {
        int rc = PPG_OK; int nb = 0;
        if (learning && lastSize > 0.0) {
            CK(cudaStreamSynchronize(h->stream));                       // the progress read-back of the batch just issued
            const double moved = h->adamProgress[1] ? (double) h->adamProgress[0] / 1048576.0 / (double) h->adamProgress[1] : 0.0;
            const double ratio = moved > 0.0 ? target / moved : 2.0;
            want = lastSize * std::min(2.0, std::max(0.5, ratio));
            want = std::max(minFrac, std::min(want, std::max(minFrac, growthMax * done)));
            ++h->stats.sub_batches;
        }
        if (frac > 0.0 || want < 1.0) {
            // a slice [frac, f1) of one pass, in the scattered pixel order
            double f1 = std::min(1.0, frac + want);
            if (1.0 - f1 < 0.5 * want) f1 = 1.0;                       // no tiny remainder
            const uint32_t p0 = (uint32_t) std::llround(frac * h->nLocalPixels), p1 = f1 >= 1.0 ? h->nLocalPixels : (uint32_t) std::llround(f1 * h->nLocalPixels);
            rc = render_batch(h, 1, h->dPixelMapPerm.p + p0, p1 - p0);
            lastSize = f1 - frac; done += f1 - frac; frac = f1;
            if (frac >= 1.0) { frac = 0.0; nb = 1; }
        } else {
            nb = std::min(std::min(maxBatch, numPasses - local), std::max(1, (int) want));
            rc = render_batch(h, nb, h->dPixelMap.p, h->nLocalPixels);
            lastSize = nb; done += nb;
        }
        if (rc == PPG_ERR_CANCELLED) { rcode = rc; break; }
        if (rc) return rc;
        h->passesRendered += nb; local += nb;
        if (h->cancelled.load()) { rcode = PPG_ERR_CANCELLED; break; }
        if (nb == 0) continue;
        bool shouldAbort = false;
        if (h->prm.budget_type == PPG_BUDGET_SECONDS) {              // GP:1259-1262, checked per batch
            CK(cudaStreamSynchronize(h->stream));
            float el = h->clock_s();
            rc = sync_scalar(h, &el); if (rc) return rc;
            shouldAbort = (int) el > h->prm.budget;
        }
        if (shouldAbort) break;
    }
    add_image_kernel<<<h->numSMs * 4, 256, 0, h->stream>>>(h->dFilm.p, h->dImage.p, npx); h->launches++;   // film->put(block), renderproc.cpp:143-151
    if (h->prm.sample_combination == PPG_COMB_INVERSEVAR) {            // GP:1292-1296: keep the iteration's image (ring of the last four)
        if (h->images.size() < 4) { DevBuf<float4> *img = new DevBuf<float4>(); CK(img->alloc(npx)); h->images.push_back(img); }
        else std::rotate(h->images.begin(), h->images.begin() + 1, h->images.end());
        CK(cudaMemcpyAsync(h->images.back()->p, h->dImage.p, sizeof(float4) * npx, cudaMemcpyDeviceToDevice, h->stream));
    }
    // variance, GP:1298-1319: the numerator is reduced on the device (double), summed over ranks as a float together with the guiding records
    // (the next refine's capacity), and read back with the counters
    const int N = local * h->prm.spp_per_pass;
    CK(cudaMemsetAsync(h->dVar.p, 0, 8, h->stream));
    if (h->nLocalPixels)
        variance_kernel<<<std::min<int>(h->numSMs * 4, (int) ((h->nLocalPixels + PPG_BLOCK - 1) / PPG_BLOCK)), PPG_BLOCK, 0, h->stream>>>(
            h->dImage.p, h->dSqImage.p, h->dPixelMap.p, h->nLocalPixels, h->W, (float) N, h->dVar.p);
    h->launches++;
    float *slot = h->tree.dTrain.p + h->tree.dTrain.n - 16;
    iteration_scalars_kernel<<<1, 1, 0, h->stream>>>(h->dVar.p, h->dCounters.p, slot); h->launches++;
    if (h->multi()) { int rc = allreduce_sum(h, slot, 2); if (rc) return rc; }
    float reduced[2] = {0, 0}; unsigned long long cnt[8];
    CK(cudaMemcpyAsync(reduced, slot, 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(cnt, h->dCounters.p, 64, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaEventRecord(h->evB, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    float ms = 0; cudaEventElapsedTime(&ms, h->evA, h->evB); h->deviceMs += ms;
    h->resolve_timers();
    const float numF = reduced[0];
    variance = (float) ((double) numF / ((double) h->W * h->H * (N - 1)));
    if (h->prm.sample_combination == PPG_COMB_INVERSEVAR) { h->variances.push_back(variance); if (h->variances.size() > 4) h->variances.erase(h->variances.begin()); }
    st.seconds += elapsed_s(t0); st.passes += local; st.variance = variance; st.total_passes = h->passesRendered;
    st.vertices += cnt[0]; st.paths += (uint64_t) local * perPass; st.recorded_vertices += cnt[1];
    if (cnt[1]) st.s_tree_depth_avg = (double) cnt[2] / (double) cnt[1];
    h->stats.total_vertices += cnt[0]; h->stats.total_paths += (uint64_t) local * perPass;
    h->stats.truncated_paths += cnt[3]; h->stats.dropped_records += cnt[4]; h->stats.invalid_rays += cnt[5];
    // every rank sizes the next refine from the same count: the records of all ranks (a rank that owns few pixels would size too small a tree)
    h->lastRecorded = h->multi() ? (uint64_t) reduced[1] : cnt[1] * (uint64_t) h->world;
    return rcode;
}

static ppg_iteration_stats &iter_stats(ppg_integrator *h) {
    ppg_iteration_stats &st = h->stats.iterations[std::min(h->iter, PPG_MAX_ITERATIONS - 1)];
    memset(&st, 0, sizeof(st)); st.iteration = h->iter;
    return st;
}
// progressive film (renderproc.cpp:143-151 puts finished blocks into the film while rendering): hand the current film to the host's callback
static int flush_film(ppg_integrator *h) {
    if (!h->filmFn) return PPG_OK;
    const size_t npx = (size_t) h->W * h->H;
    develop_kernel<<<h->numSMs * 4, 256, 0, h->stream>>>(h->dFilm.p, h->dRgb.p, npx, 1.0f, 0); h->launches++;
    CK(cudaStreamSynchronize(h->stream));
    h->filmFn(h->filmUser, h->dRgb.p, h->W, h->H, h->passesRendered);
    return PPG_OK;
}
static int clear_film(ppg_integrator *h) { CK(cudaMemsetAsync(h->dFilm.p, 0, sizeof(float4) * (size_t) h->W * h->H, h->stream)); return PPG_OK; }

static int dump_iteration(ppg_integrator *h) {      // dumpSDTree: "<dest>-NN.sdt", GP:1191-1195
    if (h->destination.empty() || h->rank != 0) return PPG_OK;
    char ext[32]; snprintf(ext, sizeof(ext), "-%02d.sdt", h->iter);
    return ppg_dump_sdtree(h, (h->destination + ext).c_str());
}

// renderSPP, GP:1342-1426
static int render_spp(ppg_integrator *h) {
    const int nPasses = (int) std::ceil((size_t) h->prm.budget / (float) h->prm.spp_per_pass);
    float currentVarAtEnd = std::numeric_limits<float>::infinity();
    while (h->passesRendered < nPasses) {
        const int sppRendered = h->passesRendered * h->prm.spp_per_pass;
        h->doNee = h->prm.nee == PPG_NEE_NEVER ? false : (h->prm.nee == PPG_NEE_KICKSTART ? sppRendered < 128 : true);   // doNeeWithSpp, GP:1331-1340, 1362
        int remainingPasses = nPasses - h->passesRendered;
        int passesThisIteration = std::min(remainingPasses, 1 << std::min(h->iter, 30));
        if (remainingPasses - passesThisIteration < 2 * passesThisIteration) passesThisIteration = remainingPasses;
        h->isFinalIter = passesThisIteration >= remainingPasses;
        ppg_iteration_stats &st = iter_stats(h);
        int rc = clear_film(h); if (rc) return rc;
        auto t0 = std::chrono::steady_clock::now();
        rc = reset_sd_tree(h); if (rc) return rc;
        st.reset_seconds = elapsed_s(t0);                               // host time up to the node-count read-back inside the reset
        float variance = 0;
        rc = perform_render_passes(h, variance, passesThisIteration, st); if (rc) return rc;
        rc = flush_film(h); if (rc) return rc;
        const float lastVarAtEnd = currentVarAtEnd;
        currentVarAtEnd = passesThisIteration * variance / remainingPasses;
        remainingPasses -= passesThisIteration;
        if (h->prm.sample_combination == PPG_COMB_AUTOMATIC && remainingPasses > 0 &&
            (remainingPasses < passesThisIteration || (sppRendered > 256 && currentVarAtEnd > lastVarAtEnd))) {
            h->isFinalIter = true;
            rc = perform_render_passes(h, variance, remainingPasses, st); if (rc) return rc;
            rc = flush_film(h); if (rc) return rc;
        }
        st.is_final = h->isFinalIter;
        t0 = std::chrono::steady_clock::now();
        rc = build_sd_tree(h, st); if (rc) return rc;
        st.build_seconds = elapsed_s(t0);
        if (h->prm.dump_sd_tree && !h->isFinalIter) { rc = dump_iteration(h); if (rc) return rc; }     // GP:1417-1419
        ++h->iter; h->stats.n_iterations = std::min(h->iter, PPG_MAX_ITERATIONS);
    }
    return PPG_OK;
}

// renderTime, GP:1434-1514
static int render_time(ppg_integrator *h) {
    const float nSeconds = h->prm.budget;
    float currentVarAtEnd = std::numeric_limits<float>::infinity(), elapsedSeconds = 0;
    while (elapsedSeconds < nSeconds) {
        const int sppRendered = h->passesRendered * h->prm.spp_per_pass;
        h->doNee = h->prm.nee == PPG_NEE_NEVER ? false : (h->prm.nee == PPG_NEE_KICKSTART ? sppRendered < 128 : true);   // GP:1452
        float remainingTime = nSeconds - elapsedSeconds;
        const int passesThisIteration = 1 << std::min(h->iter, 30);
        ppg_iteration_stats &st = iter_stats(h);
        const auto startIter = std::chrono::steady_clock::now(); const float startIterClock = h->clock_s();
        int rc = clear_film(h); if (rc) return rc;
        rc = reset_sd_tree(h); if (rc) return rc;
        st.reset_seconds = elapsed_s(startIter);
        float variance = 0;
        rc = perform_render_passes(h, variance, passesThisIteration, st); if (rc) return rc;
        rc = flush_film(h); if (rc) return rc;
        float secondsIter = h->clock_s() - startIterClock;
        rc = sync_scalar(h, &secondsIter); if (rc) return rc;
        const float lastVarAtEnd = currentVarAtEnd;
        currentVarAtEnd = secondsIter * variance / remainingTime;
        remainingTime -= secondsIter;
        if (h->prm.sample_combination == PPG_COMB_AUTOMATIC && remainingTime > 0 &&
            (remainingTime < secondsIter || (sppRendered > 256 && currentVarAtEnd > lastVarAtEnd))) {
            h->isFinalIter = true;
            do {
                rc = perform_render_passes(h, variance, passesThisIteration, st); if (rc) return rc;
                rc = flush_film(h); if (rc) return rc;
                elapsedSeconds = h->clock_s();
                rc = sync_scalar(h, &elapsedSeconds); if (rc) return rc;
            } while (elapsedSeconds < nSeconds);
        }
        st.is_final = h->isFinalIter;
        const auto t0 = std::chrono::steady_clock::now();
        rc = build_sd_tree(h, st); if (rc) return rc;
        st.build_seconds = elapsed_s(t0);
        if (h->prm.dump_sd_tree && !h->isFinalIter) { rc = dump_iteration(h); if (rc) return rc; }     // GP:1504-1506
        ++h->iter; h->stats.n_iterations = std::min(h->iter, PPG_MAX_ITERATIONS);
        elapsedSeconds = h->clock_s();
        rc = sync_scalar(h, &elapsedSeconds); if (rc) return rc;
    }
    return PPG_OK;
}

// render, GP:1516-1585
static int ppg_render_device_impl(ppg_integrator *h, float **rgb_dev, ppg_stats *stats);
extern "C" int ppg_render_device(ppg_integrator *h, float **rgb_dev, ppg_stats *stats) { return guarded("ppg_render_device", [&] { return ppg_render_device_impl(h, rgb_dev, stats); }); }
static int ppg_render_device_impl(ppg_integrator *h, float **rgb_dev, ppg_stats *stats) {
    if (!h) return fail(PPG_ERR_INVALID_ARGUMENT, "null handle");
    if (!h->haveScene) return fail(PPG_ERR_NO_SCENE, "ppg_render called before ppg_set_scene");
    CK(cudaSetDevice(h->device));
    h->cancelled.store(false);
    const auto wall0 = std::chrono::steady_clock::now();
    memset(&h->stats, 0, sizeof(h->stats)); h->launches = 0; h->deviceMs = 0; h->evUsed = 0;
    memset(h->treeStatsPending, 0, sizeof(h->treeStatsPending));
    CK(cudaEventRecord(h->evRender0, h->stream));
    int rc = h->tree.init(); if (rc) return rc;                                   // m_sdTree = new STree(scene->getAABB()), GP:1519
    rc = ensure_wavefront(h); if (rc) return rc;
    h->iter = 0; h->isFinalIter = false; h->isBuilt = false; h->passesRendered = 0;
    for (auto *b : h->images) delete b;
    h->images.clear(); h->variances.clear();
    rc = clear_film(h); if (rc) return rc;
    h->startTime = std::chrono::steady_clock::now();
    rc = h->prm.budget_type == PPG_BUDGET_SPP ? render_spp(h) : render_time(h);
    if (rc != PPG_OK && rc != PPG_ERR_CANCELLED) return rc;
    const size_t npx = (size_t) h->W * h->H;
    const int blocks = h->numSMs * 4;
    if (h->prm.sample_combination == PPG_COMB_INVERSEVAR && !h->images.empty()) {   // GP:1567-1582
        float totalWeight = 0;
        for (float v : h->variances) totalWeight += 1.0f / v;
        CK(cudaMemsetAsync(h->dRgb.p, 0, 12 * npx, h->stream));
        for (size_t i = 0; i < h->images.size(); ++i) {
            develop_kernel<<<blocks, 256, 0, h->stream>>>(h->images[i]->p, h->dRgb.p, npx, 1.0f / h->variances[i] / totalWeight, 1); h->launches++;
        }
    } else {
        develop_kernel<<<blocks, 256, 0, h->stream>>>(h->dFilm.p, h->dRgb.p, npx, 1.0f, 0); h->launches++;
    }
    if (h->ncclComm && h->world > 1) {     // disjoint tiles: summing the zero-padded frames assembles the film on every rank; on the render stream
        int rc2 = allreduce_sum(h, h->dRgb.p, 3 * npx); if (rc2) return rc2;
    }
    CK(cudaEventRecord(h->evRender1, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    h->resolve_timers(); finish_tree_stats(h);
    { float ms = 0; cudaEventElapsedTime(&ms, h->evRender0, h->evRender1); h->stats.render_device_ms = ms; }
    if (!h->ncclComm && h->multi()) {      // callback path: the collective runs outside the library's stream, after the timed region
        int rc2 = allreduce_sum(h, h->dRgb.p, 3 * npx); if (rc2) return rc2;
    }
    CK(cudaGetLastError());
    h->stats.total_passes = h->passesRendered;
    h->stats.render_seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - wall0).count();
    h->stats.device_seconds = h->deviceMs / 1000.0;
    h->stats.final_variance = h->stats.n_iterations ? h->stats.iterations[h->stats.n_iterations - 1].variance : 0;
    h->stats.kernel_launches = h->launches;
    if (stats) *stats = h->stats;
    if (rgb_dev) *rgb_dev = h->dRgb.p;
    return rc;
}

extern "C" int ppg_render(ppg_integrator *h, float *rgb_out, ppg_stats *stats) {
    float *dev = nullptr;
    const int rc = ppg_render_device(h, &dev, stats);
    if (rc != PPG_OK && rc != PPG_ERR_CANCELLED) return rc;
    if (rgb_out) CK(cudaMemcpy(rgb_out, dev, 12 * (size_t) h->W * h->H, cudaMemcpyDeviceToHost));
    return rc;
}

extern "C" int ppg_copy_from_device(void *host_dst, const void *device_src, size_t bytes) {
    if (!host_dst || !device_src) return fail(PPG_ERR_INVALID_ARGUMENT, "null argument");
    CK(cudaMemcpy(host_dst, device_src, bytes, cudaMemcpyDeviceToHost));
    return PPG_OK;
}

extern "C" int ppg_get_moment_images(ppg_integrator *h, float *sum_rgbw, float *sumsq_rgbw) {
    if (!h || !h->haveScene) return fail(PPG_ERR_NO_SCENE, "no scene");
    CK(cudaSetDevice(h->device));
    const size_t npx = (size_t) h->W * h->H;
    if (sum_rgbw) CK(cudaMemcpy(sum_rgbw, h->dImage.p, 16 * npx, cudaMemcpyDeviceToHost));
    if (sumsq_rgbw) CK(cudaMemcpy(sumsq_rgbw, h->dSqImage.p, 16 * npx, cudaMemcpyDeviceToHost));
    return PPG_OK;
}

static int store_tree(ppg_integrator *h, int which, ppg_sdtree &out) {
    if (!h->haveScene) return fail(PPG_ERR_NO_SCENE, "no SD-tree yet");
    CK(cudaSetDevice(h->device));
    return h->tree.store(which, out);
}

extern "C" int ppg_export_sdtree(ppg_integrator *h, int which, ppg_sdtree *out, float *aabb_min_max) {
  return guarded("ppg_export_sdtree", [&]() -> int {
    if (!h || !out || (which != 0 && which != 1)) return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_export_sdtree: null argument or `which` not 0 / 1");
    int rc = store_tree(h, which, *out); if (rc) return rc;
    if (aabb_min_max) {                           // the cubified box of the S-tree (STree::STree, GP:850-860; pack_scene)
        const float m = std::max(std::max(h->aabbMax[0] - h->aabbMin[0], h->aabbMax[1] - h->aabbMin[1]), h->aabbMax[2] - h->aabbMin[2]);
        for (int a = 0; a < 3; ++a) { aabb_min_max[a] = h->aabbMin[a]; aabb_min_max[3 + a] = h->aabbMin[a] + m; }
    }
    return PPG_OK;
  });
}

// dumpSDTree wire format (GP:1191-1208, 699-711, 945-951): 16 floats camera matrix, then for every leaf with
// sampling weight > 0, in forEachLeaf order (child 0 before child 1): pos, size, mean, u64 weight, u64 nNodes,
// nNodes x 4 x (f32 sum, u16 child)
static int ppg_dump_sdtree_impl(ppg_integrator *h, const char *path);
extern "C" int ppg_dump_sdtree(ppg_integrator *h, const char *path) { return guarded("ppg_dump_sdtree", [&] { return ppg_dump_sdtree_impl(h, path); }); }
static int ppg_dump_sdtree_impl(ppg_integrator *h, const char *path) {
    if (!h || !path) return fail(PPG_ERR_INVALID_ARGUMENT, "null argument");
    ppg_sdtree t = {};
    int rc = store_tree(h, 0, t);                 // no room (an S-tree has a node): only the sizes
    if (rc != PPG_ERR_INVALID_ARGUMENT) return rc;
    std::vector<uint32_t> sn(2 * t.n_nodes), count(t.n_nodes); std::vector<uint64_t> first(t.n_nodes); std::vector<float> sum(t.n_nodes), weight(t.n_nodes);
    std::vector<float> sums(4 * t.n_pool); std::vector<uint16_t> children(4 * t.n_pool);
    t.node_capacity = t.n_nodes; t.pool_capacity = t.n_pool;
    t.node_children = sn.data(); t.tree_first = first.data(); t.tree_count = count.data(); t.tree_sum = sum.data(); t.tree_weight = weight.data();
    t.sums = sums.data(); t.children = children.data();
    rc = store_tree(h, 0, t); if (rc) return rc;
    FILE *f = fopen(path, "wb");
    if (!f) return fail(PPG_ERR_IO, std::string("cannot open ") + path);
    float cm[16];
    const Camera &c = h->cam;   // camera-to-world matrix, row-major (GP:1197-1205)
    cm[0] = c.left.x; cm[1] = c.up.x; cm[2] = c.dir.x; cm[3] = c.o.x; cm[4] = c.left.y; cm[5] = c.up.y; cm[6] = c.dir.y; cm[7] = c.o.y;
    cm[8] = c.left.z; cm[9] = c.up.z; cm[10] = c.dir.z; cm[11] = c.o.z; cm[12] = 0; cm[13] = 0; cm[14] = 0; cm[15] = 1;
    fwrite(cm, 4, 16, f);
    struct E { uint32_t n; float p[3], s[3]; int axis; };
    std::vector<E> st; E root; root.n = 0; root.axis = 0;
    for (int i = 0; i < 3; ++i) { root.p[i] = h->aabbMin[i]; root.s[i] = h->extent[i]; }
    st.push_back(root);
    while (!st.empty()) {
        E e = st.back(); st.pop_back();
        if (sn[2 * e.n] == 0u) {
            if (!(weight[e.n] > 0)) continue;
            const float mean = (1 / (3.14159265358979323846f * 4 * weight[e.n])) * sum[e.n];
            fwrite(e.p, 4, 3, f); fwrite(e.s, 4, 3, f); fwrite(&mean, 4, 1, f);
            const uint64_t w64 = (uint64_t) weight[e.n], nn = count[e.n];
            fwrite(&w64, 8, 1, f); fwrite(&nn, 8, 1, f);
            for (uint64_t k = 4 * first[e.n]; k < 4 * (first[e.n] + nn); ++k) { fwrite(&sums[k], 4, 1, f); fwrite(&children[k], 2, 1, f); }
        } else {
            E a = e, b = e;
            a.s[e.axis] = b.s[e.axis] = e.s[e.axis] / 2; b.p[e.axis] += b.s[e.axis];
            a.axis = b.axis = (e.axis + 1) % 3; a.n = sn[2 * e.n]; b.n = sn[2 * e.n + 1];
            st.push_back(b); st.push_back(a);
        }
    }
    fclose(f);
    return PPG_OK;
}

// ------------------------------------------------------------------ kernel-level entry points on caller-supplied tree arrays
namespace {
struct ReplayRng { const float *v; uint32_t n, i; __device__ float next1D() { return i < n ? v[i++] : 0.5f; } };

// the sampling tree of node t as the bounce kernel reads it
__device__ __forceinline__ const SampNode *op_tree(const TreeView &T, uint32_t t, bool &valid) {
    const float4 la = T.leafA[t];
    valid = __float_as_uint(la.w) & 1u;
    return T.samp + __float_as_uint(la.x);
}
__global__ void op_pdf_kernel(const __grid_constant__ TreeView T, const uint32_t *qt, const float *qd, size_t n, float *out) {
    for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t) gridDim.x * blockDim.x) {
        bool valid; const SampNode *tree = op_tree(T, qt[i], valid);
        out[i] = dtree_pdf(tree, valid, dir_to_canonical(f3(qd[3 * i], qd[3 * i + 1], qd[3 * i + 2])));
    }
}
__global__ void op_sample_kernel(const __grid_constant__ TreeView T, const uint32_t *qt, const float *rnd, size_t stride, size_t n, float *out, float *canon) {
    for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t) gridDim.x * blockDim.x) {
        bool valid; const SampNode *tree = op_tree(T, qt[i], valid);
        ReplayRng r{rnd + stride * i, (uint32_t) stride, 0u};
        const float2 c = dtree_sample(tree, valid, r);
        const float3 d = canonical_to_dir(c);
        out[3 * i] = d.x; out[3 * i + 1] = d.y; out[3 * i + 2] = d.z;
        if (canon) { canon[2 * i] = c.x; canon[2 * i + 1] = c.y; }
    }
}
__global__ void op_record_kernel(const __grid_constant__ TreeView T, const uint32_t *rt, const float *rd, const float *rrad, const float *rpdf, const float *rw, size_t n, int filter) {
    const size_t nPad = (n + 31) / 32 * 32;
    for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < nPad; i += (size_t) gridDim.x * blockDim.x) {
        const bool ok = i < n;
        const uint32_t t = ok ? rt[i] : 0u; const float w = ok ? rw[i] : 0.f;
        const bool wOk = ok && isfinite(w) && w > 0.f;
        warp_aggregated_add(T.bweight, t, w, wOk);
        if (wOk) {
            const float4 la = T.leafA[t];
            dtree_record_irradiance(T.bchildren, T.bsums, __float_as_uint(la.y), dir_to_canonical(f3(rd[3 * i], rd[3 * i + 1], rd[3 * i + 2])), rrad[i] / rpdf[i], w, filter);
        }
    }
}
__global__ void op_lookup_kernel(const uint2 *snodes, const uint32_t *table, float3 mn, float3 ext, const float *pts, size_t n, uint32_t *leaf, float *size) {
    for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t) gridDim.x * blockDim.x) {
        int lv; const uint32_t l = stree_lookup(snodes, table, mn, ext, f3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]), lv);
        leaf[i] = l;
        const float3 v = voxel_size(ext, lv);
        size[3 * i] = v.x; size[3 * i + 1] = v.y; size[3 * i + 2] = v.z;
    }
}
// Scene::sampleAttenuatedEmitterDirect at caller-supplied reference points, exactly as the bounce kernel's light-sampling block calls it
__global__ void op_emitter_sample_kernel(const __grid_constant__ SceneView scene, const float *ref, const float *refN, const float *smp, int maxInteractions, size_t n,
                                         float *dOut, float *valueOut, float *pdfOut, float *distOut) {
    const SceneAccess<false> sc(scene);
    for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t) gridDim.x * blockDim.x) {
        const float3 p = f3(ref[3 * i], ref[3 * i + 1], ref[3 * i + 2]), rn = f3(refN[3 * i], refN[3 * i + 1], refN[3 * i + 2]);
        DirectSample ds; ds.value = f3(0, 0, 0); ds.d = f3(0, 0, 0); ds.pdf = 0.f; float dist = 0.f;
        const bool ok = sample_emitter_direct<true>(sc, p, rn, smp[2 * i], smp[2 * i + 1], ds, dist);
        if (ok) ds.value = ds.value * eval_transmittance(sc, p, ds.d, dist, maxInteractions);
        else { ds.value = f3(0, 0, 0); ds.pdf = 0.f; dist = 0.f; }
        dOut[3 * i] = ds.d.x; dOut[3 * i + 1] = ds.d.y; dOut[3 * i + 2] = ds.d.z;
        valueOut[3 * i] = ds.value.x; valueOut[3 * i + 1] = ds.value.y; valueOut[3 * i + 2] = ds.value.z;
        pdfOut[i] = ds.pdf; distOut[i] = dist;
    }
}
__global__ void op_env_pdf_kernel(const __grid_constant__ SceneView scene, const float *dir, size_t n, float *pdfOut, float *valueOut) {
    for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t) gridDim.x * blockDim.x) {
        const float3 d = f3(dir[3 * i], dir[3 * i + 1], dir[3 * i + 2]);
        pdfOut[i] = pdf_emitter_direct<true>(scene, PPG_ENV_EMITTER, f3(0, 0, 0), f3(0, 0, 0), d, f3(0, 0, 0), 0.f);
        if (valueOut) { const float3 v = env_eval(scene, d); valueOut[3 * i] = v.x; valueOut[3 * i + 1] = v.y; valueOut[3 * i + 2] = v.z; }
    }
}
template <class T> struct Up {
    DevBuf<T> b;
    int up(const T *host, size_t n) { if (b.alloc(std::max<size_t>(n, 1)) != cudaSuccess) return 1; return n ? cudaMemcpy(b.p, host, n * sizeof(T), cudaMemcpyHostToDevice) != cudaSuccess : 0; }
};
static int op_device(int device) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return fail(PPG_ERR_NO_DEVICE, "no CUDA device available (no CPU fallback)"); }
    if (device < 0) device = 0;
    if (device >= ndev) return fail(PPG_ERR_NO_DEVICE, "device index out of range");
    CK(cudaSetDevice(device));
    return PPG_OK;
}
}  // namespace

static const float kNoBox[3] = {0.f, 0.f, 0.f};     // the D-tree ops look up no point

extern "C" int ppg_op_dtree_pdf(int device, const ppg_sdtree *tree, const uint32_t *query_tree, const float *query_dir, size_t n, float *pdf_out) {
  return guarded("ppg_op_dtree_pdf", [&]() -> int {
    int rc = op_device(device); if (rc) return rc;
    if (!tree) return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_op_dtree_pdf: null tree");
    TreeStore t; rc = t.load(0, *tree); if (rc) return rc;
    Up<uint32_t> dq; Up<float> dd; DevBuf<float> out;
    if (dq.up(query_tree, n) || dd.up(query_dir, 3 * n)) return fail(PPG_ERR_CUDA, "upload failed");
    CK(out.alloc(std::max<size_t>(n, 1)));
    if (n) op_pdf_kernel<<<296, 256>>>(t.view(kNoBox, kNoBox), dq.b.p, dd.b.p, n, out.p);
    CK(cudaGetLastError());
    CK(cudaMemcpy(pdf_out, out.p, 4 * n, cudaMemcpyDeviceToHost));
    return PPG_OK;
  });
}
extern "C" int ppg_op_dtree_sample(int device, const ppg_sdtree *tree, const uint32_t *query_tree, const float *rnd, size_t rnd_stride, size_t n,
                                   float *dir_out, float *canonical_out) {
  return guarded("ppg_op_dtree_sample", [&]() -> int {
    int rc = op_device(device); if (rc) return rc;
    if (!tree) return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_op_dtree_sample: null tree");
    TreeStore t; rc = t.load(0, *tree); if (rc) return rc;
    Up<uint32_t> dq; Up<float> dr; DevBuf<float> out, canon;
    if (dq.up(query_tree, n) || dr.up(rnd, rnd_stride * n)) return fail(PPG_ERR_CUDA, "upload failed");
    CK(out.alloc(std::max<size_t>(3 * n, 1)));
    if (canonical_out) CK(canon.alloc(std::max<size_t>(2 * n, 1)));
    if (n) op_sample_kernel<<<296, 256>>>(t.view(kNoBox, kNoBox), dq.b.p, dr.b.p, rnd_stride, n, out.p, canon.p);
    CK(cudaGetLastError());
    CK(cudaMemcpy(dir_out, out.p, 12 * n, cudaMemcpyDeviceToHost));
    if (canonical_out) CK(cudaMemcpy(canonical_out, canon.p, 8 * n, cudaMemcpyDeviceToHost));
    return PPG_OK;
  });
}
extern "C" int ppg_op_dtree_record(int device, const ppg_sdtree *tree, const uint32_t *rec_tree, const float *rec_dir, const float *rec_radiance,
                                   const float *rec_wo_pdf, const float *rec_weight, size_t n, int filter) {
  return guarded("ppg_op_dtree_record", [&]() -> int {
    int rc = op_device(device); if (rc) return rc;
    if (!tree) return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_op_dtree_record: null tree");
    TreeStore t; rc = t.load(1, *tree); if (rc) return rc;
    Up<float> dd, drad, dpdf, dw; Up<uint32_t> drt;
    if (drt.up(rec_tree, n) || dd.up(rec_dir, 3 * n) || drad.up(rec_radiance, n) || dpdf.up(rec_wo_pdf, n) || dw.up(rec_weight, n))
        return fail(PPG_ERR_CUDA, "upload failed");
    if (n) op_record_kernel<<<296, 256>>>(t.view(kNoBox, kNoBox), drt.b.p, dd.b.p, drad.b.p, dpdf.b.p, dw.b.p, n, filter);
    CK(cudaGetLastError());
    return t.copy_back(*tree);
  });
}
// The acceleration structure ppg_set_scene builds, on the host alone (no CUDA device needed): for tests of the builder and for timing it.
extern "C" int ppg_op_bvh_build(const float *positions, const uint32_t *indices, size_t n_triangles, int threads, float *nodes_out, size_t nodes_capacity,
                                uint32_t *order_out, size_t *n_nodes_out, int *max_depth_out, double *ms_out) {
  return guarded("ppg_op_bvh_build", [&]() -> int {
    if (!positions || !indices || !n_triangles || n_triangles >= 0xFFFFFFFFull) return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_op_bvh_build: empty or oversized input");
    const uint32_t nt = (uint32_t) n_triangles;
    const auto t0 = std::chrono::steady_clock::now();
    const int T = threads > 0 ? threads : host_threads();
    const HostBvh bvh = build_bvh(positions, indices, nt, T);
    if (ms_out) *ms_out = elapsed_ms(t0);
    if (n_nodes_out) *n_nodes_out = bvh.nodes.size() / 8;
    if (max_depth_out) *max_depth_out = bvh.maxDepth;
    if (nodes_out) { if (nodes_capacity < bvh.nodes.size() / 8) return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_op_bvh_build: nodes_out too small (2 * n_triangles + 1 always suffices)"); memcpy(nodes_out, bvh.nodes.data(), bvh.nodes.size() * 4); }
    if (order_out) memcpy(order_out, bvh.order.data(), (size_t) nt * 4);
    return PPG_OK;
  });
}
extern "C" int ppg_op_emitter_sample_direct(ppg_integrator *h, size_t n, const float *ref, const float *ref_n, const float *sample, int max_interactions,
                                            float *d_out, float *value_out, float *pdf_out, float *dist_out) {
    if (!h || !h->haveScene) return fail(PPG_ERR_NO_SCENE, "ppg_op_emitter_sample_direct needs a handle with a scene");
    if (!ref || !ref_n || !sample || !d_out || !value_out || !pdf_out || !dist_out) return fail(PPG_ERR_INVALID_ARGUMENT, "null argument");
    if (!h->fullFeature) return fail(PPG_ERR_UNSUPPORTED, "emitter-level ops run the full-feature code path (scene with spheres, textures, non-diffuse BSDFs or an environment emitter)");
    CK(cudaSetDevice(h->device));
    Up<float> dr, dn, ds; DevBuf<float> od, ov, op, ot;
    if (dr.up(ref, 3 * n) || dn.up(ref_n, 3 * n) || ds.up(sample, 2 * n)) return fail(PPG_ERR_CUDA, "upload failed");
    CK(od.alloc(std::max<size_t>(3 * n, 1))); CK(ov.alloc(std::max<size_t>(3 * n, 1))); CK(op.alloc(std::max<size_t>(n, 1))); CK(ot.alloc(std::max<size_t>(n, 1)));
    if (n) op_emitter_sample_kernel<<<296, 128>>>(h->sceneView, dr.b.p, dn.b.p, ds.b.p, max_interactions, n, od.p, ov.p, op.p, ot.p);
    CK(cudaGetLastError());
    CK(cudaMemcpy(d_out, od.p, 12 * n, cudaMemcpyDeviceToHost)); CK(cudaMemcpy(value_out, ov.p, 12 * n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(pdf_out, op.p, 4 * n, cudaMemcpyDeviceToHost)); CK(cudaMemcpy(dist_out, ot.p, 4 * n, cudaMemcpyDeviceToHost));
    return PPG_OK;
}
extern "C" int ppg_op_env_pdf(ppg_integrator *h, size_t n, const float *d, float *pdf_out, float *value_out) {
    if (!h || !h->haveScene) return fail(PPG_ERR_NO_SCENE, "ppg_op_env_pdf needs a handle with a scene");
    if (!h->sceneView.envW) return fail(PPG_ERR_NO_SCENE, "the scene has no environment emitter");
    if (!d || !pdf_out) return fail(PPG_ERR_INVALID_ARGUMENT, "null argument");
    CK(cudaSetDevice(h->device));
    Up<float> dd; DevBuf<float> op, ov;
    if (dd.up(d, 3 * n)) return fail(PPG_ERR_CUDA, "upload failed");
    CK(op.alloc(std::max<size_t>(n, 1))); CK(ov.alloc(std::max<size_t>(3 * n, 1)));
    if (n) op_env_pdf_kernel<<<296, 128>>>(h->sceneView, dd.b.p, n, op.p, value_out ? ov.p : nullptr);
    CK(cudaGetLastError());
    CK(cudaMemcpy(pdf_out, op.p, 4 * n, cudaMemcpyDeviceToHost));
    if (value_out) CK(cudaMemcpy(value_out, ov.p, 12 * n, cudaMemcpyDeviceToHost));
    return PPG_OK;
}
extern "C" int ppg_op_stree_lookup(int device, const ppg_sdtree *tree, const float aabb_min[3], const float aabb_extent[3],
                                   const float *points, size_t n, uint32_t *leaf_out, float *size_out) {
  return guarded("ppg_op_stree_lookup", [&]() -> int {
    int rc = op_device(device); if (rc) return rc;
    if (!tree) return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_op_stree_lookup: null tree");
    TreeStore t; rc = t.load(0, *tree); if (rc) return rc;
    Up<float> dp; DevBuf<uint32_t> dl; DevBuf<float> dsz;
    if (dp.up(points, 3 * n)) return fail(PPG_ERR_CUDA, "upload failed");
    CK(dl.alloc(std::max<size_t>(n, 1))); CK(dsz.alloc(std::max<size_t>(3 * n, 1)));
    t.stree_table();
    const TreeView T = t.view(aabb_min, aabb_extent);
    if (n) op_lookup_kernel<<<t.numSMs * 2, 256>>>(T.snodes, T.stable, T.aabbMin, T.extent, dp.b.p, n, dl.p, dsz.p);
    CK(cudaGetLastError());
    CK(cudaMemcpy(leaf_out, dl.p, 4 * n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(size_out, dsz.p, 12 * n, cudaMemcpyDeviceToHost));
    return PPG_OK;
  });
}

// ------------------------------------------------------------------ the learning half: the render's own maintenance, commit and Adam launches (TreeStore)

extern "C" int ppg_op_sdtree_refine_reset(int device, int stages, float threshold, int new_max_depth, float dtree_threshold, size_t node_capacity,
                                          const ppg_sdtree *in, const float *building_weight, ppg_sdtree *sampling_out, ppg_sdtree *building_out) {
  return guarded("ppg_op_sdtree_refine_reset", [&]() -> int {
    int rc = op_device(device); if (rc) return rc;
    if (!in || !in->n_nodes || !building_weight || !sampling_out || !building_out) return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_op_sdtree_refine_reset: empty or null input");
    const size_t n_nodes = in->n_nodes;
    double totalW = 0; for (size_t i = 0; i < n_nodes; ++i) totalW += building_weight[i];
    const uint32_t cap = node_capacity ? (uint32_t) std::min<size_t>(node_capacity, 0xFFFFFFFFull)
                                       : std::max<uint32_t>((uint32_t) std::min<double>(refine_capacity(n_nodes, 1.25 * totalW + 4096, threshold), 4.0e9), 1u << 16);
    if (cap < n_nodes) return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_op_sdtree_refine_reset: node_capacity below n_nodes");
    TreeStore t; rc = t.load(0, *in, cap); if (rc) return rc;
    CK(t.put(t.dBweight, building_weight, n_nodes));
    if (stages & 1) t.refine(threshold);
    if (stages & 2) t.reset_count(new_max_depth, dtree_threshold);
    CK(cudaGetLastError());
    rc = t.sync_counts(true); if (rc) return rc;
    building_out->n_nodes = t.hNodes; building_out->n_pool = t.hTotalBuild;
    rc = t.store(0, *sampling_out, false);        // the refine's result: the reset changes no sampling tree
    if (rc || t.hNodes > building_out->node_capacity || t.hTotalBuild > building_out->pool_capacity)
        return rc ? rc : fail(PPG_ERR_INVALID_ARGUMENT, "ppg_op_sdtree_refine_reset: building_out too small (its n_nodes and n_pool hold the sizes needed)");
    if (building_out->tree_weight) CK(cudaMemcpy(building_out->tree_weight, t.dBweight.p, 4 * (size_t) t.hNodes, cudaMemcpyDeviceToHost));     // reset_fill clears it
    if (stages & 2) t.reset_fill(new_max_depth, dtree_threshold);
    CK(cudaGetLastError());
    ppg_sdtree b = *building_out; b.tree_weight = nullptr;
    return t.store(1, b, false);
  });
}

extern "C" int ppg_op_sdtree_build(int device, const ppg_sdtree *building, ppg_sdtree *sampling_out, uint8_t *mean_positive_out, double *stats_out) {
  return guarded("ppg_op_sdtree_build", [&]() -> int {
    int rc = op_device(device); if (rc) return rc;
    if (!building || !building->n_nodes || !sampling_out) return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_op_sdtree_build: empty or null input");
    TreeStore t; rc = t.load(1, *building); if (rc) return rc;
    t.build(); t.tree_stats();
    CK(cudaGetLastError());
    rc = t.store(0, *sampling_out, false); if (rc) return rc;
    if (mean_positive_out) {
        std::vector<float4> la(t.hNodes); CK(cudaMemcpy(la.data(), t.dLeafA.p, sizeof(float4) * la.size(), cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < la.size(); ++i) mean_positive_out[i] = f_bits(la[i].w) != 0u;
    }
    if (stats_out) {
        TreeStats s; CK(cudaMemcpy(&s, t.dTreeStats.p, sizeof(s), cudaMemcpyDeviceToHost));
        const double v[14] = {(double) s.leaves, (double) s.leavesWithNodes, (double) s.depthMin, (double) s.depthMax, s.meanMin, s.meanMax, s.weightMin, s.weightMax,
                              (double) s.nodesMin, (double) s.nodesMax, s.depthSum, s.meanSum, s.nodesSum, s.weightSum};
        memcpy(stats_out, v, sizeof(v));
    }
    return PPG_OK;
  });
}

extern "C" int ppg_op_commit(int device, int record_mode, const ppg_sdtree *building, const float aabb_min[3], const float aabb_extent[3],
                             const float *vertices, size_t n, const float *li_final, size_t n_li, int spatial_filter, int directional_filter, int loss,
                             uint64_t seed, float statistical_weight, float *adam_records_out, size_t adam_capacity, size_t *n_adam_out) {
  return guarded("ppg_op_commit", [&]() -> int {
    int rc = op_device(device); if (rc) return rc;
    if (record_mode != 1 && record_mode != 2) return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_op_commit: record_mode is 1 (nearest, 3 vertex fields) or 2 (6 fields)");
    if (!building || !building->n_nodes || !building->n_pool || !aabb_min || !aabb_extent || (n && (!vertices || !li_final)) || n >= 0x40000000ull || !n_adam_out)
        return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_op_commit: empty or null input");
    TreeStore t; rc = t.load(1, *building); if (rc) return rc;
    t.adamCap = std::min<size_t>(adam_capacity, 0xFFFFFFFFull); CK(t.dAdamRecA.alloc(t.adamCap)); CK(t.dAdamRecB.alloc(t.adamCap));
    // the bounce kernel's slab layout: field f of vertex i at f * n + i
    std::vector<float4> slab(6 * std::max<size_t>(n, 1));
    for (size_t i = 0; i < n; ++i)
        for (int f = 0; f < 6; ++f) memcpy(&slab[(size_t) f * n + i], vertices + 24 * i + 4 * f, 16);
    const uint32_t live = (uint32_t) n; const unsigned long long dropped = 0;
    Up<float4> dSlab, dLi; Up<uint32_t> dLive; Up<unsigned long long> dDrop;
    if (dSlab.up(slab.data(), slab.size()) || dLi.up(reinterpret_cast<const float4 *>(li_final), n_li) || dLive.up(&live, 1) || dDrop.up(&dropped, 1))
        return fail(PPG_ERR_CUDA, "upload failed");
    t.stree_table();
    CommitParams C; memset(&C, 0, sizeof(C));
    C.tree = t.view(aabb_min, aabb_extent);
    VertexSlab S; float4 *b = dSlab.b.p;
    S.v0 = b; S.v1 = b + n; S.v2 = b + 2 * n; S.v3 = b + 3 * n; S.v4 = b + 4 * n; S.v5 = b + 5 * n;
    C.slab0 = S; C.slabStride = n; C.liveCounts = dLive.b.p; C.liFinal = dLi.b.p;
    C.spatialFilter = spatial_filter; C.directionalFilter = directional_filter; C.lossMode = loss; C.statisticalWeight = statistical_weight;
    C.nee0 = S; C.nSlabs = 1; C.seed = seed; C.dropped = dDrop.b.p;
    if (n) t.commit(C, record_mode, live, 1);
    CK(cudaGetLastError());
    rc = t.copy_back(*building); if (rc) return rc;
    uint32_t tot = 0; CK(cudaMemcpy(&tot, t.dScalars.p + 3, 4, cudaMemcpyDeviceToHost));
    *n_adam_out = tot;
    const size_t kept = std::min<size_t>(tot, t.adamCap);
    return adam_records_out && kept ? records_join(t.dAdamRecA.p, t.dAdamRecB.p, kept, adam_records_out) : PPG_OK;
  });
}

extern "C" int ppg_op_adam_replay(int device, int loss, int bucket, float *state_inout, size_t n_nodes, const float *records, size_t n_records,
                                  const uint32_t *leaf_offset, const uint32_t *leaf_count, float *theta_out, float *bucketed_out, uint32_t *leaf_offset_out,
                                  uint32_t *count_out, uint32_t *cursor_out) {
  return guarded("ppg_op_adam_replay", [&]() -> int {
    int rc = op_device(device); if (rc) return rc;
    if (loss != PPG_LOSS_KL && loss != PPG_LOSS_VAR) return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_op_adam_replay: loss is kl or var");
    if (!state_inout || !n_nodes || n_nodes >= 0xFFFFFFFFull || n_records >= 0xFFFFFFFFull || (n_records && !records) || (!bucket && (!leaf_offset || !leaf_count)))
        return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_op_adam_replay: empty or null input");
    if (!bucket)
        for (size_t i = 0; i < n_nodes; ++i)
            if ((size_t) leaf_offset[i] + leaf_count[i] > n_records) return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_op_adam_replay: a leaf's records run past n_records");
    ppg_sdtree s = {}; s.n_nodes = s.node_capacity = n_nodes; s.adam = state_inout;
    TreeStore t; rc = t.load(0, s); if (rc) return rc;
    t.adamCap = n_records; CK(t.dAdamRecA.alloc(n_records)); CK(t.dAdamRecB.alloc(n_records)); CK(t.dAdamSortA.alloc(n_records)); CK(t.dAdamSortB.alloc(n_records));
    std::vector<float4> ra; std::vector<float2> rb; records_split(records, n_records, ra, rb);
    // records to bucket go where commit appends them; records already grouped go straight into the buckets
    const uint32_t nRec = (uint32_t) n_records;
    CK(cudaMemcpy(t.dScalars.p + 3, &nRec, 4, cudaMemcpyHostToDevice));
    CK(t.put(bucket ? t.dAdamRecA : t.dAdamSortA, ra.data(), n_records));
    CK(t.put(bucket ? t.dAdamRecB : t.dAdamSortB, rb.data(), n_records));
    if (bucket) {
        t.adam_bucket();
        CK(cudaGetLastError());
        if (bucketed_out && n_records) { rc = records_join(t.dAdamSortA.p, t.dAdamSortB.p, n_records, bucketed_out); if (rc) return rc; }
        if (leaf_offset_out) CK(cudaMemcpy(leaf_offset_out, t.dAdamOffset.p, 4 * n_nodes, cudaMemcpyDeviceToHost));
    } else {            // the cursors hold the counts, as after adam_scatter_kernel
        CK(cudaMemcpy(t.dAdamCount.p, leaf_count, 4 * n_nodes, cudaMemcpyHostToDevice)); CK(cudaMemcpy(t.dAdamCursor.p, leaf_count, 4 * n_nodes, cudaMemcpyHostToDevice));
        CK(cudaMemcpy(t.dAdamOffset.p, leaf_offset, 4 * n_nodes, cudaMemcpyHostToDevice));
        if (leaf_offset_out) memcpy(leaf_offset_out, leaf_offset, 4 * n_nodes);
    }
    t.adam_replay(loss);
    CK(cudaGetLastError());
    rc = t.store(0, s); if (rc) return rc;
    if (theta_out) for (size_t i = 0; i < n_nodes; ++i) theta_out[i] = state_inout[6 * i + 3];
    if (count_out) CK(cudaMemcpy(count_out, t.dAdamCount.p, 4 * n_nodes, cudaMemcpyDeviceToHost));
    if (cursor_out) CK(cudaMemcpy(cursor_out, t.dAdamCursor.p, 4 * n_nodes, cudaMemcpyDeviceToHost));
    return PPG_OK;
  });
}
