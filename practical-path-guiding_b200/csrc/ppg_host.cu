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
    float aabbMin[3], aabbMax[3];
    int W = 0, H = 0;
    DevBuf<uint32_t> dPixelMap, dPixelMapPerm; uint32_t nLocalPixels = 0, minLocalPixels = 0, maxLocalPixels = 0;

    // film
    DevBuf<float4> dImage, dSqImage, dFilm; DevBuf<float> dRgb; DevBuf<double> dVar;
    std::vector<DevBuf<float4> *> images; std::vector<float> variances;

    // SD-tree
    uint32_t capNodes = 0; size_t capPool = 0;
    DevBuf<uint2> dSnodes; DevBuf<float4> dLeafA; DevBuf<float> dBweight, dSampSum, dSampWeight, dAdam, dAdamBefore /* 4 x capNodes: iter, batchAcc, batchGrad, theta before a replay */;
    DevBuf<uint32_t> dAdamCount, dAdamCursor, dAdamOffset; DevBuf<float4> dAdamRecA, dAdamSortA; DevBuf<float2> dAdamRecB, dAdamSortB; size_t adamCap = 0;
    DevBuf<int> dSampDepth, dBuildDepth; DevBuf<uint32_t> dSampCount, dBuildCount, dBuildBase, dScalars /* [0]=nNodes [1]=totalBuild */;
    DevBuf<uint32_t> dStable; DevBuf<TreeStats> dTreeStats;
    DevBuf<SampNode> dSamp; DevBuf<uint2> dBchildren; DevBuf<float> dTrain /* bsums | packed tail */;
    uint32_t hNodes = 1; uint32_t hTotalBuild = 1;
    float extent[3];

    // wavefront
    size_t pathCapacity = 0; int maxBounces = 0, nSlabs = 0; int recordMode = 0; int stateVecs = 5, slabSets = 1;
    DevBuf<float4> dStateA, dStateB, dSlabs, dLiFinal; DevBuf<uint32_t> dLive, dWork; DevBuf<unsigned long long> dCounters;
    DevBuf<float4> dHits; DevBuf<uint32_t> dTraceWork; int gridTrace = 0; uint32_t traceMinPaths = 0;   // separate nearest-hit pass (ppg_trace.cu), BVH scenes only
    DevBuf<uint32_t> dOrder, dBinCount; bool binMaterials = false;                                        // ... which also bins the paths by the BSDF class they hit
    int gridBounce = 0, gridCommit = 0;

    // per-kernel-class CUDA-event timing on the launching stream
    struct Timed { cudaEvent_t a, b; int cls; uint32_t launches; };
    std::vector<Timed> evPool; size_t evUsed = 0; cudaEvent_t evRender0 = nullptr, evRender1 = nullptr;
    bool kernelTiming = true;
    void tic(int cls) {
        if (!kernelTiming) return;
        if (evUsed == evPool.size()) { Timed t; cudaEventCreate(&t.a); cudaEventCreate(&t.b); t.cls = cls; t.launches = 1; evPool.push_back(t); }
        evPool[evUsed].cls = cls; evPool[evUsed].launches = 1; cudaEventRecord(evPool[evUsed].a, stream);
    }
    void toc(uint32_t nLaunches = 1) { if (!kernelTiming) return; evPool[evUsed].launches = nLaunches; cudaEventRecord(evPool[evUsed].b, stream); ++evUsed; }   // one bracket may hold several launches of a class
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
    CK(cudaEventCreate(&h->evA)); CK(cudaEventCreate(&h->evB)); CK(cudaEventCreate(&h->evRender0)); CK(cudaEventCreate(&h->evRender1));
    for (auto &e : h->evLive) CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    CK(cudaHostAlloc((void **) &h->liveHost, 128 * sizeof(uint32_t), cudaHostAllocDefault));
    CK(cudaHostAlloc((void **) &h->hTreeStats, PPG_MAX_ITERATIONS * sizeof(TreeStats), cudaHostAllocDefault));
    if (const char *e = getenv("PPG_KERNEL_TIMING")) h->kernelTiming = atoi(e) != 0;
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

static int env_int(const char *name, int dflt) { const char *v = getenv(name); return v && *v ? atoi(v) : dflt; }   // tuning experiments only

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

static int build_pixel_map(ppg_integrator *h) {
    // 32x32 image blocks (scene.cpp:24), dealt to the ranks round-robin along a scattered order of the blocks (golden-ratio stride, coprime to
    // the block count): every rank's blocks are spread over the whole image whatever the image width (plain `block % world` gives each rank
    // whole COLUMNS of blocks when the blocks per row are a multiple of the world size, and the columns of an image do not cost the same).
    // A rank visits its blocks row-major; row-major inside a block.
    const int bs = 32, bx = (h->W + bs - 1) / bs, by = (h->H + bs - 1) / bs, nb = bx * by;
    std::vector<int> owner((size_t) nb, 0);
    if (h->world > 1) {
        auto gcd = [](uint64_t a, uint64_t b) { while (b) { const uint64_t t = a % b; a = b; b = t; } return a; };
        uint64_t stride = std::max<uint64_t>(1, (uint64_t) ((double) nb * 0.6180339887498949));
        while (gcd(stride, (uint64_t) nb) != 1) ++stride;
        for (uint64_t j = 0; j < (uint64_t) nb; ++j) owner[(j * stride) % nb] = (int) (j % h->world);
    }
    std::vector<uint32_t> map; map.reserve((size_t) h->W * h->H / h->world + 1024);
    for (int b = 0; b < nb; ++b) {
        if (owner[b] != h->rank) continue;
        const int x0 = (b % bx) * bs, y0 = (b / bx) * bs;
        if (env_int("PPG_PIXEL_ORDER", 0) == 1) {      // experiment: Morton order inside the block (results do not depend on the order)
            for (uint32_t m = 0; m < (uint32_t) (bs * bs); ++m) {
                uint32_t x = 0, y = 0;
                for (int bit = 0; bit < 5; ++bit) { x |= ((m >> (2 * bit)) & 1u) << bit; y |= ((m >> (2 * bit + 1)) & 1u) << bit; }
                if (x0 + (int) x < h->W && y0 + (int) y < h->H) map.push_back((uint32_t) (x0 + x) | ((uint32_t) (y0 + y) << 16));
            }
            continue;
        }
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
    // A second, scattered order of the same pixels (golden-ratio stride over runs of 8 pixels, coprime to the run count): any contiguous range of it is spread evenly over
    // the image.  The sub-batches of a learning iteration (perform_render_passes) take their pixels from it, so that every S-tree leaf receives its
    // share of every sub-batch -- like the reference, whose worker threads interleave image blocks while the sampling fractions adapt.
    std::vector<uint32_t> perm(map.size());
    if (!map.empty()) {
        const uint64_t n = map.size();
        auto gcd = [](uint64_t a, uint64_t b) { while (b) { const uint64_t t = a % b; a = b; b = t; } return a; };
        // ... in runs of 8 consecutive map entries (8 neighbouring pixels of one block row): a quarter of a warp starts coherent,
        // which the BVH walk of the first bounce -- the largest launch of a sub-batch -- feels; a slice of 10^4 paths still holds
        // > 10^3 runs spread over the whole image
        const uint64_t run = (uint64_t) std::max(env_int("PPG_PERM_RUN", 8), 1), nr = (n + run - 1) / run;
        uint64_t rs = std::max<uint64_t>(1, (uint64_t) ((double) nr * 0.6180339887498949));
        while (gcd(rs, nr) != 1) ++rs;
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

// ------------------------------------------------------------------ SD-tree storage
static int ensure_tree_capacity(ppg_integrator *h, uint32_t nodes, size_t pool) {
    if (nodes > h->capNodes) {
        const uint32_t cap = std::max<uint32_t>(nodes, std::max<uint32_t>(2 * h->capNodes, 1u << 16));
        CK(h->dSnodes.grow(cap, h->stream)); CK(h->dLeafA.grow(cap, h->stream)); CK(h->dBweight.grow(cap, h->stream));
        CK(h->dSampSum.grow(cap, h->stream)); CK(h->dSampWeight.grow(cap, h->stream)); CK(h->dAdam.grow(6 * (size_t) cap, h->stream));
        CK(h->dAdamBefore.grow(4 * (size_t) cap, h->stream)); CK(h->dSampDepth.grow(cap, h->stream));
        {   // record-bucket bookkeeping must stay zero between commit launches: reallocate zeroed
            h->dAdamCount.release(); h->dAdamCursor.release(); h->dAdamOffset.release();
            CK(h->dAdamCount.alloc(cap)); CK(h->dAdamCursor.alloc(cap)); CK(h->dAdamOffset.alloc(cap));
            CK(cudaMemsetAsync(h->dAdamCount.p, 0, 4 * (size_t) cap, h->stream)); CK(cudaMemsetAsync(h->dAdamCursor.p, 0, 4 * (size_t) cap, h->stream));
        }
        CK(h->dBuildDepth.grow(cap, h->stream)); CK(h->dSampCount.grow(cap, h->stream)); CK(h->dBuildCount.grow(cap, h->stream));
        CK(h->dBuildBase.grow(cap, h->stream));
        h->capNodes = cap;
    }
    if (pool > h->capPool) {
        const size_t cap = std::max<size_t>(pool, std::max<size_t>(2 * h->capPool, (size_t) 1 << 20));
        CK(h->dSamp.grow(cap, h->stream)); CK(h->dBchildren.grow(cap, h->stream));
        h->capPool = cap;
    }
    // bsums (4 floats per pool node) followed by the packed exchange tail (building weights, or 6 Adam arrays; + scalars)
    CK(h->dTrain.grow(4 * h->capPool + 6 * (size_t) h->capNodes + 64, h->stream));
    return PPG_OK;
}

static MaintParams maint(ppg_integrator *h) {
    MaintParams M;
    M.snodes = h->dSnodes.p; M.leafA = h->dLeafA.p; M.bweight = h->dBweight.p; M.sampSum = h->dSampSum.p; M.sampWeight = h->dSampWeight.p;
    M.sampDepth = h->dSampDepth.p; M.sampCount = h->dSampCount.p; M.adam = h->dAdam.p; M.buildCount = h->dBuildCount.p; M.buildDepth = h->dBuildDepth.p;
    M.nNodes = h->dScalars.p; M.capNodes = h->capNodes; M.samp = h->dSamp.p; M.bchildren = h->dBchildren.p; M.bsums = reinterpret_cast<float4 *>(h->dTrain.p);
    return M;
}

// new STree (GP:1519): one leaf whose sampling tree is a single empty quadtree node
static int init_tree(ppg_integrator *h) {
    CK(h->dScalars.alloc(8)); CK(h->dTreeStats.alloc(1));
    CK(cudaMemsetAsync(h->dScalars.p, 0, 32, h->stream));
    // buffers persist across renders (cudaMalloc/cudaFree are synchronous and slow): only their contents are reset
    int rc = ensure_tree_capacity(h, std::max<uint32_t>(h->capNodes, 1u << 16), std::max<size_t>(h->capPool, (size_t) 1 << 20));
    if (rc) return rc;
    CK(cudaMemsetAsync(h->dSnodes.p, 0, sizeof(uint2) * h->capNodes, h->stream));
    CK(cudaMemsetAsync(h->dLeafA.p, 0, sizeof(float4) * h->capNodes, h->stream));
    CK(cudaMemsetAsync(h->dBweight.p, 0, 4 * (size_t) h->capNodes, h->stream));
    CK(cudaMemsetAsync(h->dSampSum.p, 0, 4 * (size_t) h->capNodes, h->stream));
    CK(cudaMemsetAsync(h->dSampWeight.p, 0, 4 * (size_t) h->capNodes, h->stream));
    CK(cudaMemsetAsync(h->dAdam.p, 0, 24 * (size_t) h->capNodes, h->stream));
    CK(cudaMemsetAsync(h->dAdamCount.p, 0, 4 * (size_t) h->capNodes, h->stream));
    CK(cudaMemsetAsync(h->dAdamCursor.p, 0, 4 * (size_t) h->capNodes, h->stream));
    CK(cudaMemsetAsync(h->dSampDepth.p, 0, 4 * (size_t) h->capNodes, h->stream));
    CK(cudaMemsetAsync(h->dSamp.p, 0, sizeof(SampNode), h->stream));          // one empty quadtree node at pool offset 0
    const uint32_t one[2] = {1u, 1u};
    CK(cudaMemcpyAsync(h->dScalars.p, one, 8, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->dSampCount.p, one, 4, cudaMemcpyHostToDevice, h->stream));
    h->hNodes = 1; h->hTotalBuild = 1;
    CK(cudaStreamSynchronize(h->stream));
    return PPG_OK;
}

static TreeView tree_view(ppg_integrator *h) {
    TreeView T;
    T.snodes = h->dSnodes.p; T.stable = stree_table_usable(h->hNodes) ? h->dStable.p : nullptr; T.leafA = h->dLeafA.p; T.samp = h->dSamp.p; T.bchildren = h->dBchildren.p;
    T.bsums = reinterpret_cast<float4 *>(h->dTrain.p); T.bweight = h->dBweight.p;
    T.aabbMin = make_float3(h->aabbMin[0], h->aabbMin[1], h->aabbMin[2]); T.extent = make_float3(h->extent[0], h->extent[1], h->extent[2]);
    return T;
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
        const size_t fp = (size_t) h->hTotalBuild * 2 * 24 + (size_t) h->hNodes * 96;
        memCapped = fp / 1000000 >= (size_t) h->prm.sd_tree_max_memory;
    }
    if (!memCapped) {
        // capacity: the refinement creates at most 2 nodes per threshold worth of recorded weight.  The total weight of the iteration is at most
        // its number of guiding records (weights <= 1), summed over the ranks whose weights are reduced.
        const double totalW = 1.25 * (double) h->lastRecorded + 4096;
        const double est = refine_capacity(h->hNodes, totalW, threshold);
        int rc = ensure_tree_capacity(h, (uint32_t) std::min<double>(est, 4.0e9), h->capPool);
        if (rc) return rc;
        MaintParams M = maint(h);
        h->tic(PPG_K_REFINE); stree_refine_kernel<<<1, 1024, 0, h->stream>>>(M, threshold, h->dScalars.p + 5); h->toc(); h->launches++;
    }
    MaintParams M = maint(h);
    const int blocks = h->numSMs * 4;
    h->tic(PPG_K_RESET);
    dtree_reset_kernel<false><<<blocks, 128, 0, h->stream>>>(M, nullptr, 20, h->prm.d_tree_threshold); h->launches++;
    exclusive_scan_kernel<<<1, 1024, 0, h->stream>>>(h->dBuildCount.p, h->dBuildBase.p, h->dScalars.p, h->dScalars.p + 1); h->launches++;
    h->toc();
    uint32_t sc[8];
    CK(cudaMemcpyAsync(sc, h->dScalars.p, 32, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (sc[5]) return fail(PPG_ERR_CUDA, "S-tree refinement ran out of node capacity");
    h->hNodes = sc[0]; h->hTotalBuild = sc[1];
    int rc = ensure_tree_capacity(h, h->hNodes, std::max<size_t>(h->hTotalBuild, 1));
    if (rc) return rc;
    M = maint(h);
    h->tic(PPG_K_RESET);
    dtree_reset_kernel<true><<<blocks, 128, 0, h->stream>>>(M, h->dBuildBase.p, 20, h->prm.d_tree_threshold); h->launches++;
    leaf_after_reset_kernel<<<blocks, 256, 0, h->stream>>>(M, h->dBuildBase.p); h->launches++;
    h->toc();
    // prefix table of the refined S-tree (stree_lookup): the first 3 * PPG_STREE_TABLE_BITS levels of every descent become one load.
    // Past 0xFFFFFF nodes its entries cannot hold the node numbers: tree_view then hands out no table and the kernels walk from the root.
    if (stree_table_usable(h->hNodes)) {
        CK(h->dStable.alloc((size_t) 1 << (3 * PPG_STREE_TABLE_BITS)));
        h->tic(PPG_K_REFINE); stree_table_kernel<<<h->numSMs * 8, 256, 0, h->stream>>>(h->dSnodes.p, h->dStable.p); h->toc(); h->launches++;
    }
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
    float *tail = h->dTrain.p + 4 * (size_t) h->hTotalBuild;
    pack_tail_kernel<<<h->numSMs, 256, 0, h->stream>>>(tail, h->dBweight.p, h->hNodes, 0); h->launches++;
    int rc = allreduce_sum(h, h->dTrain.p, 4 * (size_t) h->hTotalBuild + (size_t) h->hNodes); if (rc) return rc;
    pack_tail_kernel<<<h->numSMs, 256, 0, h->stream>>>(tail, h->dBweight.p, h->hNodes, 1); h->launches++;
    return PPG_OK;
}
// a host scalar made identical on all ranks (rank 0's value wins): time-based decisions must not diverge
static int sync_scalar(ppg_integrator *h, float *v) {
    if (!h->multi()) return PPG_OK;
    float *slot = h->dTrain.p + h->dTrain.n - 16;
    const float mine = h->rank == 0 ? *v : 0.f;
    CK(cudaMemcpyAsync(slot, &mine, 4, cudaMemcpyHostToDevice, h->stream));
    int rc = allreduce_sum(h, slot, 1); if (rc) return rc;
    CK(cudaMemcpyAsync(v, slot, 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return PPG_OK;
}

// buildSDTree, GP:1115-1189
static int build_sd_tree(ppg_integrator *h, ppg_iteration_stats &st) {
    int rc = exchange_training_statistics(h);
    if (rc) return rc;
    MaintParams M = maint(h);
    h->tic(PPG_K_BUILD); dtree_build_kernel<<<h->numSMs * 4, 128, 0, h->stream>>>(M, h->dBuildBase.p); h->toc(); h->launches++;
    CK(cudaGetLastError());
    // "Distribution statistics" (GP:1121-1186): reduced on the device, 64 bytes come back
    CK(cudaMemsetAsync(h->dTreeStats.p, 0, sizeof(TreeStats), h->stream));
    tree_stats_kernel<<<1, 1024, 0, h->stream>>>(M, h->dTreeStats.p); h->launches++;
    // the statistics are only reported: they go to pinned memory and are folded into ppg_stats after the render's last synchronize
    const int slot = std::min(h->iter, PPG_MAX_ITERATIONS - 1);
    CK(cudaMemcpyAsync(h->hTreeStats + slot, h->dTreeStats.p, sizeof(TreeStats), cudaMemcpyDeviceToHost, h->stream));
    h->treeStatsPending[slot] = true;
    st.s_tree_nodes = h->hNodes;
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
    size_t cap = (size_t) 1 << 23;
    if (const char *e = getenv("PPG_PATH_CAPACITY")) cap = std::max<size_t>(strtoull(e, nullptr, 10), 1024);
    size_t budget = (size_t) 24 << 30;
    if (const char *e = getenv("PPG_WAVEFRONT_BYTES")) budget = strtoull(e, nullptr, 10);
    cap = std::min(cap, budget / perPath);
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
    CK(h->dLive.alloc(h->maxBounces + 2)); CK(h->dWork.alloc(h->maxBounces + 2)); CK(h->dCounters.alloc(8));
    if (h->prm.bsdf_sampling_fraction_loss != PPG_LOSS_NONE) {
        // sampling-fraction records: one per (recorded vertex, leaf) pair.  Sized once for the largest wavefront with 16 records per path (mean path
        // lengths of the bundled scenes: 4 - 9 vertices; the spatial box filter touches ~2 leaves per vertex); a record beyond it is dropped and
        // counted in ppg_stats.dropped_records.  Allocating per batch (cudaMalloc / cudaFree are synchronous) cost 11 ms per sub-batch.
        const size_t want = cap * 16 * (h->prm.spatial_filter == PPG_SFILTER_BOX ? 2 : 1);
        if (want > h->adamCap) {
            h->dAdamRecA.release(); h->dAdamRecB.release(); h->dAdamSortA.release(); h->dAdamSortB.release();
            CK(h->dAdamRecA.alloc(want)); CK(h->dAdamRecB.alloc(want)); CK(h->dAdamSortA.alloc(want)); CK(h->dAdamSortB.alloc(want));
            h->adamCap = want;
        }
    }
    // persistent grids: resident blocks per SM from the occupancy calculator
    int occ = 0;
    if (h->sceneSmemBytes) occ = h->fullFeature ? ppg_bounce_occupancy_11(h->sceneSmemBytes) : ppg_bounce_occupancy_10(h->sceneSmemBytes);
    else occ = h->fullFeature ? ppg_bounce_occupancy_01(0) : ppg_bounce_occupancy_00(0);
    CK(cudaGetLastError());
    // one block per resident slot; warps claim their work dynamically (bounce_kernel)
    h->gridBounce = h->numSMs * std::max(occ, 1) * std::max(env_int("PPG_GRID_MULT", 1), 1);
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, commit_kernel<1>, PPG_BLOCK, 0));
    h->gridCommit = h->numSMs * std::max(occ, 1);
    // Scenes walked through the BVH find their hits in a separate pass of persistent warps (ppg_trace.cu) whenever the wavefront is large enough
    // to pay for the second launch per depth; tiny learning sub-batches keep the fused kernel.  PPG_TRACE_MIN_PATHS=0 turns the pass off.
    h->gridTrace = 0;
    h->traceMinPaths = (uint32_t) std::max(env_int("PPG_TRACE_MIN_PATHS", 32768), 0);
    if (!h->sceneSmemBytes && h->sceneView.nGroups == 0u && h->sceneView.nTris != 0u && h->traceMinPaths != 0u) {
        CK(h->dHits.alloc(h->pathCapacity)); CK(h->dTraceWork.alloc(h->maxBounces + 2));
        h->binMaterials = h->fullFeature && env_int("PPG_BIN_MATERIALS", 1) != 0;       // one kind of BSDF only: nothing to sort
        if (h->binMaterials) { CK(h->dOrder.alloc((size_t) PPG_BINS * h->pathCapacity)); CK(h->dBinCount.alloc((size_t) PPG_BINS * (h->maxBounces + 2))); }
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
    if (useAdam) CK(cudaMemsetAsync(h->dScalars.p + 3, 0, 4, h->stream));      // record cursor (buffers: ensure_wavefront)
    if (nPaths) {
        CK(cudaMemsetAsync(h->dLive.p, 0, 4 * (size_t) (h->maxBounces + 2), h->stream));
        CK(cudaMemsetAsync(h->dWork.p, 0, 4 * (size_t) (h->maxBounces + 2), h->stream));
        CK(cudaMemcpyAsync(h->dLive.p, &nPaths, 4, cudaMemcpyHostToDevice, h->stream));
        RenderParams P;
        P.scene = h->sceneView; P.cam = h->cam; P.tree = tree_view(h);
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
        const bool bins = useTrace && h->binMaterials;
        P.order = bins ? h->dOrder.p : nullptr; P.binCount = nullptr; P.binStride = (uint32_t) h->pathCapacity;
        if (useTrace) CK(cudaMemsetAsync(h->dTraceWork.p, 0, 4 * (size_t) (h->maxBounces + 2), h->stream));
        if (bins) CK(cudaMemsetAsync(h->dBinCount.p, 0, 4 * (size_t) PPG_BINS * (h->maxBounces + 2), h->stream));
        int lastDepth = 0, pendingDepth = 0; uint32_t bracket = 0;
        for (int depth = 1; depth <= h->maxBounces; ++depth) {
            P.depth = depth; P.in = (depth & 1) ? B : A; P.out = (depth & 1) ? A : B;
            P.liveIn = h->dLive.p + (depth - 1); P.liveOut = h->dLive.p + depth; P.work = h->dWork.p + depth;
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
            flush_kernel<<<std::max(grid / 4, 1), PPG_BLOCK, 0, h->stream>>>(last, h->dLive.p + lastDepth, h->dLiFinal.p, h->dCounters.p + 3); h->launches++;
        }
        if (record) {
            CommitParams C;
            C.tree = tree_view(h); C.slab0 = slab_at(h, 0); C.slabStride = h->pathCapacity; C.liveCounts = h->dLive.p; C.liFinal = h->dLiFinal.p;
            C.spatialFilter = h->prm.spatial_filter; C.directionalFilter = h->prm.directional_filter;
            C.lossMode = lossMode;
            C.statisticalWeight = (h->prm.nee == PPG_NEE_KICKSTART && h->doNee && nee) ? 0.5f : 1.0f;   // GP:2152
            C.seed = h->prm.seed; C.snodes = h->dSnodes.p; C.nSlabs = (uint32_t) std::min(h->nSlabs, lastDepth);
            C.nee0 = neeSlabs ? slab_at(h, 0, 1) : C.slab0;
            C.adamRecA = h->dAdamRecA.p; C.adamRecB = h->dAdamRecB.p; C.adamTotal = h->dScalars.p + 3; C.adamCap = (uint32_t) std::min<size_t>(h->adamCap, 0xFFFFFFFFu);
            C.dropped = h->dCounters.p + 4;
            dim3 g(std::min<int>(h->gridCommit, (int) ((nPaths + PPG_BLOCK - 1) / PPG_BLOCK)), C.nSlabs * (neeSlabs ? 2 : 1));
            h->tic(PPG_K_COMMIT);
            if (record == 1) commit_kernel<1><<<g, PPG_BLOCK, 0, h->stream>>>(C); else commit_kernel<2><<<g, PPG_BLOCK, 0, h->stream>>>(C);
            h->toc(); h->launches++;
        }
        h->tic(PPG_K_FILM);
        film_kernel<<<std::min<int>(h->numSMs * 8, (int) ((pixelCount + PPG_BLOCK - 1) / PPG_BLOCK)), PPG_BLOCK, 0, h->stream>>>(
            h->dLiFinal.p, pixelMap, pixelCount, (uint32_t) h->prm.spp_per_pass, (uint32_t) nPasses, h->W, h->dImage.p, h->dSqImage.p);
        h->toc(); h->launches++;
    }
    if (useAdam) {
        // replay the sampling-fraction records leaf by leaf (see adam_seq_kernel)
        MaintParams M = maint(h);
        const bool multi = h->multi();
        float *tail = h->dTrain.p + 4 * (size_t) h->hTotalBuild;       // [6 x nNodes] exchange area (the building weights are packed there only at iteration end)
        adam_pack_kernel<<<h->numSMs, 256, 0, h->stream>>>(M, tail, h->dAdamBefore.p, nullptr, 0); h->launches++;
        h->tic(PPG_K_OTHER);      // bucket the records by leaf (histogram, scan, scatter): "other"; the sequential replay itself: "adam"
        adam_hist_kernel<<<h->numSMs * 4, 256, 0, h->stream>>>(h->dAdamRecA.p, h->dScalars.p + 3, (uint32_t) h->adamCap, h->dAdamCount.p); h->launches++;
        exclusive_scan_kernel<<<1, 1024, 0, h->stream>>>(h->dAdamCount.p, h->dAdamOffset.p, h->dScalars.p, h->dScalars.p + 4); h->launches++;
        adam_scatter_kernel<<<h->numSMs * 4, 256, 0, h->stream>>>(h->dAdamRecA.p, h->dAdamRecB.p, h->dScalars.p + 3, (uint32_t) h->adamCap, h->dAdamOffset.p,
                                                                  h->dAdamCursor.p, h->dAdamSortA.p, h->dAdamSortB.p); h->launches++;
        h->toc();
        h->tic(PPG_K_ADAM);
        adam_seq_kernel<<<h->numSMs * 16, 128, 0, h->stream>>>(M, h->dAdamSortA.p, h->dAdamSortB.p, h->dAdamOffset.p, h->dAdamCount.p, h->dAdamCursor.p,
                                                              lossMode == PPG_LOSS_KL ? 1.0f : 2.0f); h->launches++;
        h->toc();
        if (multi) {
            // replicas replayed their own records from the common state: merge them (steps and moves of the variable add up, moments are
            // weighted by the steps, batch accumulators add up relative to the common start) so that all ranks continue identically
            adam_pack_kernel<<<h->numSMs, 256, 0, h->stream>>>(M, tail, h->dAdamBefore.p, nullptr, 1); h->launches++;
            int rc = allreduce_sum(h, tail, 6 * (size_t) h->hNodes); if (rc) return rc;
            adam_merge_kernel<<<h->numSMs, 256, 0, h->stream>>>(M, tail, h->dAdamBefore.p, (float) (h->world - 1)); h->launches++;
        }
        // movement of the fractions in this replay (identical on all ranks after the merge): steers the size of the next sub-batch
        CK(cudaMemsetAsync(h->dCounters.p + 6, 0, 16, h->stream));
        adam_progress_kernel<<<h->numSMs, 256, 0, h->stream>>>(M, h->dAdamBefore.p, h->dCounters.p + 6); h->launches++;
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
    static const double target = std::max(env_int("PPG_LOSS_TARGET_X1000", 20), 1) * 1e-3;
    static const double growthMax = std::max(env_int("PPG_LOSS_GROWTH_MAX_PCT", 100), 1) * 0.01;
    static const double leafPaths = std::max(env_int("PPG_LOSS_LEAF_PATHS_X10", 40), 1) * 0.1;   // paths per S-tree leaf in the first sub-batch
    const double pathsPerPass = (double) npx * h->prm.spp_per_pass;                                  // whole image
    const double minFrac = std::min(1.0, std::max(256.0, leafPaths * 0.5 * (h->hNodes + 1)) / std::max(pathsPerPass, 1.0));
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
            static const int trace2 = env_int("PPG_TRACE", 0);
            if (trace2 > 1) fprintf(stderr, "[ppg trace]   sub-batch %.5f passes moved %.4f next %.5f at %.2f ms\n", lastSize, moved, want, elapsed_ms(t0));
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
    float *slot = h->dTrain.p + h->dTrain.n - 16;
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
    static const int trace = env_int("PPG_TRACE", 0);
    if (trace)    // cumulative kernel times after every iteration's passes (stderr): where a render's time goes, iteration by iteration
        fprintf(stderr, "[ppg trace] iter %d final %d passes %d sub_batches %llu vertices %llu entered at %.1f ms wall %.1f ms | cumulative ms: bounce %.1f commit %.1f adam %.1f other %.1f film %.1f launches %llu\n",
                h->iter, (int) h->isFinalIter, local, (unsigned long long) h->stats.sub_batches, (unsigned long long) cnt[0], elapsed_ms(h->startTime) - elapsed_ms(t0), elapsed_ms(t0),
                h->stats.kernel_ms[PPG_K_BOUNCE], h->stats.kernel_ms[PPG_K_COMMIT], h->stats.kernel_ms[PPG_K_ADAM], h->stats.kernel_ms[PPG_K_OTHER], h->stats.kernel_ms[PPG_K_FILM],
                (unsigned long long) h->launches);
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
    int rc = init_tree(h); if (rc) return rc;                                   // m_sdTree = new STree(scene->getAABB()), GP:1519
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

// The integrator's SD-tree on the host: the S-tree and, per node, either the sampling trees (which == 0: the trees the passes guide with) or the
// building trees (which == 1: the trees the passes record into).  Between the reset and the build of an iteration (the film callback) the sampling
// trees still sit where the previous build put them, past the new building total: the copy of the quadtree pool is sized from the leaves.
struct TreeGather {
    uint32_t n = 0;
    std::vector<uint2> sn; std::vector<float4> la; std::vector<float> sum, weight, adam; std::vector<int> depth; std::vector<uint32_t> count;
    std::vector<uint2> children; std::vector<float4> sums;      // the quadtree pool from offset 0 (building: bchildren / bsums; sampling: dSamp)
    uint32_t first(uint32_t i, int which) const { uint32_t u; memcpy(&u, which ? &la[i].y : &la[i].x, 4); return u; }
};
static int gather_tree(ppg_integrator *h, int which, TreeGather &g) {
    if (!h->haveScene || h->capNodes == 0) return fail(PPG_ERR_NO_SCENE, "no SD-tree yet");
    CK(cudaSetDevice(h->device));
    const uint32_t n = g.n = h->hNodes;
    g.sn.resize(n); g.la.resize(n); g.sum.assign(n, 0.f); g.weight.resize(n); g.adam.resize(6 * (size_t) n); g.depth.resize(n); g.count.resize(n);
    CK(cudaMemcpy(g.sn.data(), h->dSnodes.p, sizeof(uint2) * n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(g.la.data(), h->dLeafA.p, sizeof(float4) * n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(g.adam.data(), h->dAdam.p, 24 * (size_t) n, cudaMemcpyDeviceToHost));
    if (which == 0) CK(cudaMemcpy(g.sum.data(), h->dSampSum.p, 4 * (size_t) n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(g.weight.data(), which ? h->dBweight.p : h->dSampWeight.p, 4 * (size_t) n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(g.depth.data(), which ? h->dBuildDepth.p : h->dSampDepth.p, 4 * (size_t) n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(g.count.data(), which ? h->dBuildCount.p : h->dSampCount.p, 4 * (size_t) n, cudaMemcpyDeviceToHost));
    size_t end = 1;
    for (uint32_t i = 0; i < n; ++i) if (g.sn[i].x == 0u) end = std::max<size_t>(end, (size_t) g.first(i, which) + g.count[i]);
    if (end > h->capPool) return fail(PPG_ERR_CUDA, "SD-tree leaf points past the quadtree pool");
    g.children.resize(end); g.sums.resize(end);
    if (which) {
        CK(cudaMemcpy(g.children.data(), h->dBchildren.p, sizeof(uint2) * end, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(g.sums.data(), h->dTrain.p, sizeof(float4) * end, cudaMemcpyDeviceToHost));
    } else {
        std::vector<SampNode> pool(end);
        CK(cudaMemcpy(pool.data(), h->dSamp.p, sizeof(SampNode) * end, cudaMemcpyDeviceToHost));
        for (size_t k = 0; k < end; ++k) { g.children[k] = pool[k].children; g.sums[k] = pool[k].sums; }
    }
    return PPG_OK;
}

extern "C" int ppg_export_sdtree(ppg_integrator *h, int which, size_t node_capacity, size_t *n_nodes_out, uint32_t *node_children, uint64_t *tree_first,
                                 uint32_t *tree_count, int32_t *tree_depth, float *tree_sum, float *tree_weight, float *adam,
                                 size_t pool_capacity, size_t *n_pool_out, float *sums, uint16_t *children, float *aabb_min_max) {
  return guarded("ppg_export_sdtree", [&]() -> int {
    if (!h || !n_nodes_out || !n_pool_out || (which != 0 && which != 1)) return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_export_sdtree: null argument or `which` not 0 / 1");
    TreeGather g; int rc = gather_tree(h, which, g); if (rc) return rc;
    size_t total = 0;
    for (uint32_t i = 0; i < g.n; ++i) if (g.sn[i].x == 0u) total += g.count[i];
    *n_nodes_out = g.n; *n_pool_out = total;
    if (g.n > node_capacity || total > pool_capacity)
        return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_export_sdtree: output arrays too small (*n_nodes_out and *n_pool_out hold the sizes needed)");
    uint64_t off = 0;
    for (uint32_t i = 0; i < g.n; ++i) {          // inner nodes carry no tree and no optimiser state (STree::subdivide, GP:876-895)
        const bool leaf = g.sn[i].x == 0u;
        if (node_children) { node_children[2 * i] = g.sn[i].x; node_children[2 * i + 1] = g.sn[i].y; }
        if (tree_first) tree_first[i] = off;
        if (tree_count) tree_count[i] = leaf ? g.count[i] : 0u;
        if (tree_depth) tree_depth[i] = leaf ? g.depth[i] : 0;
        if (tree_sum) tree_sum[i] = leaf ? g.sum[i] : 0.f;
        if (tree_weight) tree_weight[i] = leaf ? g.weight[i] : 0.f;
        if (adam) {
            for (int j = 0; j < 6; ++j) adam[6 * (size_t) i + j] = leaf ? g.adam[6 * (size_t) i + j] : 0.f;
            if (leaf) adam[6 * (size_t) i + 3] = g.la[i].z;           // theta as the bounce kernel reads it
        }
        if (!leaf) continue;
        const uint32_t base = g.first(i, which);
        for (uint32_t k = 0; k < g.count[i]; ++k) {
            const float4 s = g.sums[base + k]; const uint2 c = g.children[base + k];
            if (sums) { float *o = sums + 4 * (off + k); o[0] = s.x; o[1] = s.y; o[2] = s.z; o[3] = s.w; }
            if (children) { uint16_t *o = children + 4 * (off + k); o[0] = (uint16_t) (c.x & 0xffff); o[1] = (uint16_t) (c.x >> 16); o[2] = (uint16_t) (c.y & 0xffff); o[3] = (uint16_t) (c.y >> 16); }
        }
        off += g.count[i];
    }
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
    TreeGather g; int rc = gather_tree(h, 0, g); if (rc) return rc;
    const std::vector<uint2> &sn = g.sn; const std::vector<float> &ssum = g.sum, &sw = g.weight; const std::vector<uint32_t> &scnt = g.count;
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
        if (sn[e.n].x == 0u) {
            if (!(sw[e.n] > 0)) continue;
            const float mean = (1 / (3.14159265358979323846f * 4 * sw[e.n])) * ssum[e.n];
            fwrite(e.p, 4, 3, f); fwrite(e.s, 4, 3, f); fwrite(&mean, 4, 1, f);
            const uint64_t w64 = (uint64_t) sw[e.n], nn = scnt[e.n];
            fwrite(&w64, 8, 1, f); fwrite(&nn, 8, 1, f);
            const uint32_t base = g.first(e.n, 0);
            for (uint32_t k = 0; k < scnt[e.n]; ++k) {
                const float4 &s = g.sums[base + k]; const uint2 &c = g.children[base + k];
                const float s4[4] = {s.x, s.y, s.z, s.w};
                const uint16_t c4[4] = {(uint16_t) (c.x & 0xffff), (uint16_t) (c.x >> 16), (uint16_t) (c.y & 0xffff), (uint16_t) (c.y >> 16)};
                for (int j = 0; j < 4; ++j) { fwrite(&s4[j], 4, 1, f); fwrite(&c4[j], 2, 1, f); }
            }
        } else {
            E a = e, b = e;
            a.s[e.axis] = b.s[e.axis] = e.s[e.axis] / 2; b.p[e.axis] += b.s[e.axis];
            a.axis = b.axis = (e.axis + 1) % 3; a.n = sn[e.n].x; b.n = sn[e.n].y;
            st.push_back(b); st.push_back(a);
        }
    }
    fclose(f);
    return PPG_OK;
}

// ------------------------------------------------------------------ kernel-level entry points on caller-supplied tree arrays
namespace {
struct ReplayRng { const float *v; uint32_t n, i; __device__ float next1D() { return i < n ? v[i++] : 0.5f; } };

__global__ void op_pdf_kernel(const SampNode *pool, const uint32_t *first, const float *tsum, const float *tweight, const uint32_t *qt, const float *qd, size_t n, float *out) {
    for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t) gridDim.x * blockDim.x) {
        const uint32_t t = qt[i];
        float mean = 0.f; if (tweight[t] != 0.f) mean = (1.f / (PPG_PI * 4.f * tweight[t])) * tsum[t];
        out[i] = dtree_pdf(pool + first[t], mean > 0.f, dir_to_canonical(f3(qd[3 * i], qd[3 * i + 1], qd[3 * i + 2])));
    }
}
__global__ void op_sample_kernel(const SampNode *pool, const uint32_t *first, const float *tsum, const float *tweight, const uint32_t *qt, const float *rnd, size_t stride, size_t n, float *out,
                                 float *canon) {
    for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t) gridDim.x * blockDim.x) {
        const uint32_t t = qt[i];
        float mean = 0.f; if (tweight[t] != 0.f) mean = (1.f / (PPG_PI * 4.f * tweight[t])) * tsum[t];
        ReplayRng r{rnd + stride * i, (uint32_t) stride, 0u};
        const float2 c = dtree_sample(pool + first[t], mean > 0.f, r);
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
static std::vector<SampNode> to_pool(const float *sums, const uint16_t *children, size_t n) {
    std::vector<SampNode> pool(n);
    for (size_t i = 0; i < n; ++i) {
        pool[i].sums = make_float4(sums[4 * i], sums[4 * i + 1], sums[4 * i + 2], sums[4 * i + 3]);
        pool[i].children = make_uint2((uint32_t) children[4 * i] | ((uint32_t) children[4 * i + 1] << 16), (uint32_t) children[4 * i + 2] | ((uint32_t) children[4 * i + 3] << 16));
        pool[i].pad = make_uint2(0u, 0u);
    }
    return pool;
}
}  // namespace

extern "C" int ppg_op_dtree_pdf(int device, const float *sums, const uint16_t *children, size_t n_nodes, const uint32_t *tree_first_node,
                                const float *tree_sum, const float *tree_weight, size_t n_trees, const uint32_t *query_tree, const float *query_dir,
                                size_t n, float *pdf_out) {
    int rc = op_device(device); if (rc) return rc;
    std::vector<SampNode> pool = to_pool(sums, children, n_nodes);
    Up<SampNode> dp; Up<uint32_t> df, dq; Up<float> ds, dw, dd; DevBuf<float> out;
    if (dp.up(pool.data(), n_nodes) || df.up(tree_first_node, n_trees) || ds.up(tree_sum, n_trees) || dw.up(tree_weight, n_trees) || dq.up(query_tree, n) || dd.up(query_dir, 3 * n))
        return fail(PPG_ERR_CUDA, "upload failed");
    CK(out.alloc(std::max<size_t>(n, 1)));
    if (n) op_pdf_kernel<<<296, 256>>>(dp.b.p, df.b.p, ds.b.p, dw.b.p, dq.b.p, dd.b.p, n, out.p);
    CK(cudaGetLastError());
    CK(cudaMemcpy(pdf_out, out.p, 4 * n, cudaMemcpyDeviceToHost));
    return PPG_OK;
}
extern "C" int ppg_op_dtree_sample(int device, const float *sums, const uint16_t *children, size_t n_nodes, const uint32_t *tree_first_node,
                                   const float *tree_sum, const float *tree_weight, size_t n_trees, const uint32_t *query_tree, const float *rnd,
                                   size_t rnd_stride, size_t n, float *dir_out, float *canonical_out) {
    int rc = op_device(device); if (rc) return rc;
    std::vector<SampNode> pool = to_pool(sums, children, n_nodes);
    Up<SampNode> dp; Up<uint32_t> df, dq; Up<float> ds, dw, dr; DevBuf<float> out, canon;
    if (dp.up(pool.data(), n_nodes) || df.up(tree_first_node, n_trees) || ds.up(tree_sum, n_trees) || dw.up(tree_weight, n_trees) || dq.up(query_tree, n) || dr.up(rnd, rnd_stride * n))
        return fail(PPG_ERR_CUDA, "upload failed");
    CK(out.alloc(std::max<size_t>(3 * n, 1)));
    if (canonical_out) CK(canon.alloc(std::max<size_t>(2 * n, 1)));
    if (n) op_sample_kernel<<<296, 256>>>(dp.b.p, df.b.p, ds.b.p, dw.b.p, dq.b.p, dr.b.p, rnd_stride, n, out.p, canon.p);
    CK(cudaGetLastError());
    CK(cudaMemcpy(dir_out, out.p, 12 * n, cudaMemcpyDeviceToHost));
    if (canonical_out) CK(cudaMemcpy(canonical_out, canon.p, 8 * n, cudaMemcpyDeviceToHost));
    return PPG_OK;
}
extern "C" int ppg_op_dtree_record(int device, float *sums_inout, const uint16_t *children, size_t n_nodes, const uint32_t *tree_first_node,
                                   float *tree_weight_inout, size_t n_trees, const uint32_t *rec_tree, const float *rec_dir, const float *rec_radiance,
                                   const float *rec_wo_pdf, const float *rec_weight, size_t n, int filter) {
    int rc = op_device(device); if (rc) return rc;
    std::vector<uint2> bch(n_nodes);
    for (size_t i = 0; i < n_nodes; ++i)
        bch[i] = make_uint2((uint32_t) children[4 * i] | ((uint32_t) children[4 * i + 1] << 16), (uint32_t) children[4 * i + 2] | ((uint32_t) children[4 * i + 3] << 16));
    std::vector<float4> la(n_trees);
    for (size_t t = 0; t < n_trees; ++t) { uint32_t b = tree_first_node[t]; float fb; memcpy(&fb, &b, 4); la[t] = make_float4(fb, fb, 0.f, 0.f); }
    Up<uint2> dch; Up<float4> dla; Up<float> dsums, dwt, dd, drad, dpdf, dw; Up<uint32_t> drt;
    if (dch.up(bch.data(), n_nodes) || dla.up(la.data(), n_trees) || dsums.up(sums_inout, 4 * n_nodes) || dwt.up(tree_weight_inout, n_trees) || drt.up(rec_tree, n) ||
        dd.up(rec_dir, 3 * n) || drad.up(rec_radiance, n) || dpdf.up(rec_wo_pdf, n) || dw.up(rec_weight, n))
        return fail(PPG_ERR_CUDA, "upload failed");
    TreeView T; memset(&T, 0, sizeof(T));
    T.leafA = dla.b.p; T.bchildren = dch.b.p; T.bsums = reinterpret_cast<float4 *>(dsums.b.p); T.bweight = dwt.b.p;
    if (n) op_record_kernel<<<296, 256>>>(T, drt.b.p, dd.b.p, drad.b.p, dpdf.b.p, dw.b.p, n, filter);
    CK(cudaGetLastError());
    CK(cudaMemcpy(sums_inout, dsums.b.p, 16 * n_nodes, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(tree_weight_inout, dwt.b.p, 4 * n_trees, cudaMemcpyDeviceToHost));
    return PPG_OK;
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
extern "C" int ppg_op_stree_lookup(int device, const uint32_t *node_children, size_t n_nodes, const float aabb_min[3], const float aabb_extent[3],
                                   const float *points, size_t n, uint32_t *leaf_out, float *size_out) {
    int rc = op_device(device); if (rc) return rc;
    Up<uint2> dn; Up<float> dp; DevBuf<uint32_t> dl; DevBuf<float> dsz;
    if (dn.up(reinterpret_cast<const uint2 *>(node_children), n_nodes) || dp.up(points, 3 * n)) return fail(PPG_ERR_CUDA, "upload failed");
    CK(dl.alloc(std::max<size_t>(n, 1))); CK(dsz.alloc(std::max<size_t>(3 * n, 1)));
    DevBuf<uint32_t> dt;
    if (stree_table_usable(n_nodes)) {                    // the same prefix table the render kernels use, under the same rule
        CK(dt.alloc((size_t) 1 << (3 * PPG_STREE_TABLE_BITS)));
        stree_table_kernel<<<296, 256>>>(dn.b.p, dt.p);
    }
    if (n) op_lookup_kernel<<<296, 256>>>(dn.b.p, dt.p,make_float3(aabb_min[0], aabb_min[1], aabb_min[2]), make_float3(aabb_extent[0], aabb_extent[1], aabb_extent[2]), dp.b.p, n, dl.p, dsz.p);
    CK(cudaGetLastError());
    CK(cudaMemcpy(leaf_out, dl.p, 4 * n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(size_out, dsz.p, 12 * n, cudaMemcpyDeviceToHost));
    return PPG_OK;
}

// ------------------------------------------------------------------ the learning half: the render's own maintenance, commit and Adam kernels
namespace {
static float bits_f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static uint32_t f_bits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static int op_sm_count() { int d = 0, n = 0; if (cudaGetDevice(&d) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, d) != cudaSuccess) n = 132; return n; }
// a zero-filled device array of `cap` elements whose first n are copied from the host (host may be null: zeros)
template <class T> static cudaError_t dev_array(DevBuf<T> &b, size_t cap, const T *host = nullptr, size_t n = 0) {
    cudaError_t e = b.alloc(std::max<size_t>(cap, 1)); if (e != cudaSuccess) return e;
    e = cudaMemset(b.p, 0, std::max<size_t>(cap, 1) * sizeof(T)); if (e != cudaSuccess) return e;
    return (host && n) ? cudaMemcpy(b.p, host, n * sizeof(T), cudaMemcpyHostToDevice) : cudaSuccess;
}
}  // namespace

extern "C" int ppg_op_sdtree_refine_reset(int device, int stages, float threshold, int new_max_depth, float dtree_threshold, size_t node_capacity,
                                          const uint32_t *node_children, size_t n_nodes, const uint32_t *tree_first, const uint32_t *tree_count, const int32_t *tree_depth,
                                          const float *tree_sum, const float *tree_weight, const float *adam, const float *building_weight,
                                          const float *sums, const uint16_t *children, size_t n_pool,
                                          size_t out_capacity, size_t *n_nodes_out, uint32_t *node_children_out, uint32_t *tree_first_out, uint32_t *tree_count_out,
                                          int32_t *tree_depth_out, float *tree_sum_out, float *tree_weight_out, float *adam_out, float *building_weight_out,
                                          uint32_t *build_first_out, uint32_t *build_count_out, int32_t *build_depth_out,
                                          size_t build_capacity, size_t *n_build_out, uint16_t *build_children_out, float *build_sums_out) {
  return guarded("ppg_op_sdtree_refine_reset", [&]() -> int {
    int rc = op_device(device); if (rc) return rc;
    if (!n_nodes || n_nodes >= 0xFFFFFFFFull || !node_children || !tree_first || !tree_count || !tree_depth || !tree_sum || !tree_weight || !adam || !building_weight ||
        !sums || !children || !n_pool || !n_nodes_out || !n_build_out)
        return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_op_sdtree_refine_reset: empty or null input");
    double totalW = 0; for (size_t i = 0; i < n_nodes; ++i) totalW += building_weight[i];
    const uint32_t cap = node_capacity ? (uint32_t) std::min<size_t>(node_capacity, 0xFFFFFFFFull)
                                       : std::max<uint32_t>((uint32_t) std::min<double>(refine_capacity(n_nodes, 1.25 * totalW + 4096, threshold), 4.0e9), 1u << 16);
    if (cap < n_nodes) return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_op_sdtree_refine_reset: node_capacity below n_nodes");
    std::vector<float4> la(n_nodes);
    for (size_t i = 0; i < n_nodes; ++i) la[i] = make_float4(bits_f(tree_first[i]), 0.f, adam[6 * i + 3], 0.f);
    std::vector<SampNode> pool = to_pool(sums, children, n_pool);
    DevBuf<uint2> dS, dBch; DevBuf<float4> dLA, dBs; DevBuf<float> dBW, dSS, dSW, dAd; DevBuf<int> dSD, dBD; DevBuf<uint32_t> dSC, dBC, dBB, dSc; DevBuf<SampNode> dSamp;
    CK(dev_array(dS, cap, reinterpret_cast<const uint2 *>(node_children), n_nodes)); CK(dev_array(dLA, cap, la.data(), n_nodes));
    CK(dev_array(dBW, cap, building_weight, n_nodes)); CK(dev_array(dSS, cap, tree_sum, n_nodes)); CK(dev_array(dSW, cap, tree_weight, n_nodes));
    CK(dev_array(dSD, cap, tree_depth, n_nodes)); CK(dev_array(dSC, cap, tree_count, n_nodes)); CK(dev_array(dAd, 6 * (size_t) cap, adam, 6 * n_nodes));
    CK(dev_array(dBC, cap)); CK(dev_array(dBD, cap)); CK(dev_array(dBB, cap)); CK(dev_array(dSamp, n_pool, pool.data(), n_pool));
    const uint32_t sc0[8] = {(uint32_t) n_nodes, 0, 0, 0, 0, 0, 0, 0};
    CK(dev_array(dSc, 8, sc0, 8));
    MaintParams M;
    M.snodes = dS.p; M.leafA = dLA.p; M.bweight = dBW.p; M.sampSum = dSS.p; M.sampWeight = dSW.p; M.sampDepth = dSD.p; M.sampCount = dSC.p; M.adam = dAd.p;
    M.buildCount = dBC.p; M.buildDepth = dBD.p; M.nNodes = dSc.p; M.capNodes = cap; M.samp = dSamp.p; M.bchildren = nullptr; M.bsums = nullptr;
    if (stages & 1) stree_refine_kernel<<<1, 1024>>>(M, threshold, dSc.p + 5);        // launch shapes of reset_sd_tree
    CK(cudaGetLastError());
    uint32_t hs[8]; CK(cudaMemcpy(hs, dSc.p, 32, cudaMemcpyDeviceToHost));
    if (hs[5]) return fail(PPG_ERR_CUDA, "S-tree refinement ran out of node capacity");
    const size_t N = hs[0];
    std::vector<float> bwRefined(N); CK(cudaMemcpy(bwRefined.data(), dBW.p, 4 * N, cudaMemcpyDeviceToHost));      // leaf_after_reset_kernel zeroes it
    size_t total = 0;
    if (stages & 2) {
        const int blocks = op_sm_count() * 4;
        dtree_reset_kernel<false><<<blocks, 128>>>(M, nullptr, new_max_depth, dtree_threshold);
        exclusive_scan_kernel<<<1, 1024>>>(dBC.p, dBB.p, dSc.p, dSc.p + 1);
        CK(cudaGetLastError());
        CK(cudaMemcpy(hs, dSc.p, 32, cudaMemcpyDeviceToHost)); total = hs[1];
        CK(dev_array(dBch, total)); CK(dev_array(dBs, total));
        M.bchildren = dBch.p; M.bsums = dBs.p;
        dtree_reset_kernel<true><<<blocks, 128>>>(M, dBB.p, new_max_depth, dtree_threshold);
        leaf_after_reset_kernel<<<blocks, 256>>>(M, dBB.p);
        CK(cudaGetLastError());
    }
    *n_nodes_out = N; *n_build_out = total;
    if (N > out_capacity || total > build_capacity)
        return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_op_sdtree_refine_reset: output arrays too small (*n_nodes_out and *n_build_out hold the sizes needed)");
    std::vector<float4> laOut(N); CK(cudaMemcpy(laOut.data(), dLA.p, 16 * N, cudaMemcpyDeviceToHost));
    if (tree_first_out) for (size_t i = 0; i < N; ++i) tree_first_out[i] = f_bits(laOut[i].x);
    if (node_children_out) CK(cudaMemcpy(node_children_out, dS.p, 8 * N, cudaMemcpyDeviceToHost));
    if (tree_count_out) CK(cudaMemcpy(tree_count_out, dSC.p, 4 * N, cudaMemcpyDeviceToHost));
    if (tree_depth_out) CK(cudaMemcpy(tree_depth_out, dSD.p, 4 * N, cudaMemcpyDeviceToHost));
    if (tree_sum_out) CK(cudaMemcpy(tree_sum_out, dSS.p, 4 * N, cudaMemcpyDeviceToHost));
    if (tree_weight_out) CK(cudaMemcpy(tree_weight_out, dSW.p, 4 * N, cudaMemcpyDeviceToHost));
    if (adam_out) CK(cudaMemcpy(adam_out, dAd.p, 24 * N, cudaMemcpyDeviceToHost));
    if (building_weight_out) memcpy(building_weight_out, bwRefined.data(), 4 * N);
    if (build_first_out) CK(cudaMemcpy(build_first_out, dBB.p, 4 * N, cudaMemcpyDeviceToHost));
    if (build_count_out) CK(cudaMemcpy(build_count_out, dBC.p, 4 * N, cudaMemcpyDeviceToHost));
    if (build_depth_out) CK(cudaMemcpy(build_depth_out, dBD.p, 4 * N, cudaMemcpyDeviceToHost));
    if (build_children_out && total) CK(cudaMemcpy(build_children_out, dBch.p, 8 * total, cudaMemcpyDeviceToHost));     // uint2 {c0 | c1 << 16, c2 | c3 << 16} == 4 x uint16
    if (build_sums_out && total) CK(cudaMemcpy(build_sums_out, dBs.p, 16 * total, cudaMemcpyDeviceToHost));
    return PPG_OK;
  });
}

extern "C" int ppg_op_sdtree_build(int device, const uint32_t *node_children, size_t n_nodes, const uint32_t *build_first, const uint32_t *build_count,
                                   const int32_t *build_depth, const float *building_weight, const float *sums, const uint16_t *children, size_t n_pool,
                                   float *sampling_sums_out, uint16_t *sampling_children_out, float *tree_sum_out, float *tree_weight_out,
                                   int32_t *tree_depth_out, uint32_t *tree_count_out, uint8_t *mean_positive_out, double *stats_out) {
  return guarded("ppg_op_sdtree_build", [&]() -> int {
    int rc = op_device(device); if (rc) return rc;
    if (!n_nodes || n_nodes >= 0xFFFFFFFFull || !node_children || !build_first || !build_count || !build_depth || !building_weight || !sums || !children || !n_pool)
        return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_op_sdtree_build: empty or null input");
    std::vector<float4> la(n_nodes);
    for (size_t i = 0; i < n_nodes; ++i) la[i] = make_float4(bits_f(build_first[i]), bits_f(build_first[i]), 0.f, 0.f);
    DevBuf<uint2> dS, dBch; DevBuf<float4> dLA, dBs; DevBuf<float> dBW, dSS, dSW; DevBuf<int> dSD, dBD; DevBuf<uint32_t> dSC, dBC, dBB, dSc; DevBuf<SampNode> dSamp;
    DevBuf<TreeStats> dTS;
    CK(dev_array(dS, n_nodes, reinterpret_cast<const uint2 *>(node_children), n_nodes)); CK(dev_array(dLA, n_nodes, la.data(), n_nodes));
    CK(dev_array(dBW, n_nodes, building_weight, n_nodes)); CK(dev_array(dSS, n_nodes)); CK(dev_array(dSW, n_nodes)); CK(dev_array(dSD, n_nodes)); CK(dev_array(dSC, n_nodes));
    CK(dev_array(dBC, n_nodes, build_count, n_nodes)); CK(dev_array(dBD, n_nodes, build_depth, n_nodes)); CK(dev_array(dBB, n_nodes, build_first, n_nodes));
    CK(dev_array(dBch, n_pool, reinterpret_cast<const uint2 *>(children), n_pool)); CK(dev_array(dBs, n_pool, reinterpret_cast<const float4 *>(sums), n_pool));
    CK(dev_array(dSamp, n_pool)); CK(dev_array(dTS, 1));
    const uint32_t sc0[8] = {(uint32_t) n_nodes, 0, 0, 0, 0, 0, 0, 0};
    CK(dev_array(dSc, 8, sc0, 8));
    MaintParams M;
    M.snodes = dS.p; M.leafA = dLA.p; M.bweight = dBW.p; M.sampSum = dSS.p; M.sampWeight = dSW.p; M.sampDepth = dSD.p; M.sampCount = dSC.p; M.adam = nullptr;
    M.buildCount = dBC.p; M.buildDepth = dBD.p; M.nNodes = dSc.p; M.capNodes = (uint32_t) n_nodes; M.samp = dSamp.p; M.bchildren = dBch.p; M.bsums = dBs.p;
    dtree_build_kernel<<<op_sm_count() * 4, 128>>>(M, dBB.p);        // launch shapes of build_sd_tree
    tree_stats_kernel<<<1, 1024>>>(M, dTS.p);
    CK(cudaGetLastError());
    std::vector<SampNode> pool(n_pool); CK(cudaMemcpy(pool.data(), dSamp.p, sizeof(SampNode) * n_pool, cudaMemcpyDeviceToHost));
    for (size_t k = 0; k < n_pool; ++k) {
        if (sampling_sums_out) memcpy(sampling_sums_out + 4 * k, &pool[k].sums, 16);
        if (sampling_children_out) memcpy(sampling_children_out + 4 * k, &pool[k].children, 8);
    }
    if (tree_sum_out) CK(cudaMemcpy(tree_sum_out, dSS.p, 4 * n_nodes, cudaMemcpyDeviceToHost));
    if (tree_weight_out) CK(cudaMemcpy(tree_weight_out, dSW.p, 4 * n_nodes, cudaMemcpyDeviceToHost));
    if (tree_depth_out) CK(cudaMemcpy(tree_depth_out, dSD.p, 4 * n_nodes, cudaMemcpyDeviceToHost));
    if (tree_count_out) CK(cudaMemcpy(tree_count_out, dSC.p, 4 * n_nodes, cudaMemcpyDeviceToHost));
    if (mean_positive_out) {
        std::vector<float4> laOut(n_nodes); CK(cudaMemcpy(laOut.data(), dLA.p, 16 * n_nodes, cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < n_nodes; ++i) mean_positive_out[i] = f_bits(laOut[i].w) != 0u;
    }
    if (stats_out) {
        TreeStats t; CK(cudaMemcpy(&t, dTS.p, sizeof(t), cudaMemcpyDeviceToHost));
        const double v[14] = {(double) t.leaves, (double) t.leavesWithNodes, (double) t.depthMin, (double) t.depthMax, t.meanMin, t.meanMax, t.weightMin, t.weightMax,
                              (double) t.nodesMin, (double) t.nodesMax, t.depthSum, t.meanSum, t.nodesSum, t.weightSum};
        memcpy(stats_out, v, sizeof(v));
    }
    return PPG_OK;
  });
}

extern "C" int ppg_op_commit(int device, int record_mode, const uint32_t *node_children, size_t n_nodes, const float aabb_min[3], const float aabb_extent[3],
                             const uint32_t *build_first, float *building_weight_inout, float *sums_inout, const uint16_t *children, size_t n_pool,
                             const float *vertices, size_t n, const float *li_final, size_t n_li, int spatial_filter, int directional_filter, int loss,
                             uint64_t seed, float statistical_weight, float *adam_records_out, size_t adam_capacity, size_t *n_adam_out) {
  return guarded("ppg_op_commit", [&]() -> int {
    int rc = op_device(device); if (rc) return rc;
    if (record_mode != 1 && record_mode != 2) return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_op_commit: record_mode is 1 (nearest, 3 vertex fields) or 2 (6 fields)");
    if (!n_nodes || !node_children || !aabb_min || !aabb_extent || !build_first || !building_weight_inout || !sums_inout || !children || !n_pool ||
        (n && (!vertices || !li_final)) || n >= 0x40000000ull || !n_adam_out)
        return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_op_commit: empty or null input");
    std::vector<float4> la(n_nodes);
    for (size_t i = 0; i < n_nodes; ++i) la[i] = make_float4(bits_f(build_first[i]), bits_f(build_first[i]), 0.f, 0.f);
    // the bounce kernel's slab layout: field f of vertex i at f * n + i
    std::vector<float4> slab(6 * std::max<size_t>(n, 1));
    for (size_t i = 0; i < n; ++i)
        for (int f = 0; f < 6; ++f) memcpy(&slab[(size_t) f * n + i], vertices + 24 * i + 4 * f, 16);
    const uint32_t live = (uint32_t) n, cap = (uint32_t) std::min<size_t>(adam_capacity, 0xFFFFFFFFull);
    DevBuf<uint2> dS, dBch; DevBuf<uint32_t> dTab, dLive, dTot; DevBuf<float4> dLA, dBs, dSlab, dLi, dRA; DevBuf<float> dBW; DevBuf<float2> dRB; DevBuf<unsigned long long> dDrop;
    CK(dev_array(dS, n_nodes, reinterpret_cast<const uint2 *>(node_children), n_nodes)); CK(dev_array(dLA, n_nodes, la.data(), n_nodes));
    CK(dev_array(dBW, n_nodes, building_weight_inout, n_nodes));
    CK(dev_array(dBch, n_pool, reinterpret_cast<const uint2 *>(children), n_pool)); CK(dev_array(dBs, n_pool, reinterpret_cast<const float4 *>(sums_inout), n_pool));
    CK(dev_array(dSlab, slab.size(), slab.data(), slab.size())); CK(dev_array(dLi, n_li, reinterpret_cast<const float4 *>(li_final), n_li));
    CK(dev_array(dLive, 1, &live, 1)); CK(dev_array(dTot, 1)); CK(dev_array(dDrop, 1)); CK(dev_array(dRA, cap)); CK(dev_array(dRB, cap));
    if (stree_table_usable(n_nodes)) {                      // as after every refine (reset_sd_tree)
        CK(dev_array(dTab, (size_t) 1 << (3 * PPG_STREE_TABLE_BITS)));
        stree_table_kernel<<<296, 256>>>(dS.p, dTab.p);
    }
    CommitParams C; memset(&C, 0, sizeof(C));
    C.tree.snodes = dS.p; C.tree.stable = dTab.p; C.tree.leafA = dLA.p; C.tree.samp = nullptr; C.tree.bchildren = dBch.p; C.tree.bsums = dBs.p; C.tree.bweight = dBW.p;
    C.tree.aabbMin = make_float3(aabb_min[0], aabb_min[1], aabb_min[2]); C.tree.extent = make_float3(aabb_extent[0], aabb_extent[1], aabb_extent[2]);
    VertexSlab S; float4 *b = dSlab.p;
    S.v0 = b; S.v1 = b + n; S.v2 = b + 2 * n; S.v3 = b + 3 * n; S.v4 = b + 4 * n; S.v5 = b + 5 * n;
    C.slab0 = S; C.slabStride = n; C.liveCounts = dLive.p; C.liFinal = dLi.p;
    C.spatialFilter = spatial_filter; C.directionalFilter = directional_filter; C.lossMode = loss; C.statisticalWeight = statistical_weight;
    C.nee0 = S; C.nSlabs = 1; C.seed = seed; C.snodes = dS.p;
    C.adamRecA = dRA.p; C.adamRecB = dRB.p; C.adamTotal = dTot.p; C.adamCap = cap; C.dropped = dDrop.p;
    if (n) {
        int occ = 0;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, commit_kernel<1>, PPG_BLOCK, 0));       // grid of render_batch
        const dim3 g(std::min<int>(op_sm_count() * std::max(occ, 1), (int) ((n + PPG_BLOCK - 1) / PPG_BLOCK)), 1);
        if (record_mode == 1) commit_kernel<1><<<g, PPG_BLOCK>>>(C); else commit_kernel<2><<<g, PPG_BLOCK>>>(C);
    }
    CK(cudaGetLastError());
    CK(cudaMemcpy(sums_inout, dBs.p, 16 * n_pool, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(building_weight_inout, dBW.p, 4 * n_nodes, cudaMemcpyDeviceToHost));
    uint32_t tot = 0; CK(cudaMemcpy(&tot, dTot.p, 4, cudaMemcpyDeviceToHost));
    *n_adam_out = tot;
    const size_t kept = std::min<size_t>(tot, cap);
    if (adam_records_out && kept) {
        std::vector<float4> ra(kept); std::vector<float2> rb(kept);
        CK(cudaMemcpy(ra.data(), dRA.p, 16 * kept, cudaMemcpyDeviceToHost)); CK(cudaMemcpy(rb.data(), dRB.p, 8 * kept, cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < kept; ++i) { memcpy(adam_records_out + 6 * i, &ra[i], 16); memcpy(adam_records_out + 6 * i + 4, &rb[i], 8); }
    }
    return PPG_OK;
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
    std::vector<float4> ra(std::max<size_t>(n_records, 1)); std::vector<float2> rb(std::max<size_t>(n_records, 1));
    for (size_t i = 0; i < n_records; ++i) { memcpy(&ra[i], records + 6 * i, 16); memcpy(&rb[i], records + 6 * i + 4, 8); }
    std::vector<float4> la(n_nodes);
    for (size_t i = 0; i < n_nodes; ++i) la[i] = make_float4(0.f, 0.f, state_inout[6 * i + 3], 0.f);
    const uint32_t sc0[8] = {(uint32_t) n_nodes, 0, 0, (uint32_t) n_records, 0, 0, 0, 0};
    DevBuf<float4> dLA, dRA, dSA; DevBuf<float2> dRB, dSB; DevBuf<float> dAd; DevBuf<uint32_t> dCount, dCursor, dOff, dSc;
    CK(dev_array(dLA, n_nodes, la.data(), n_nodes)); CK(dev_array(dAd, 6 * n_nodes, state_inout, 6 * n_nodes)); CK(dev_array(dSc, 8, sc0, 8));
    CK(dev_array(dRA, n_records, ra.data(), n_records)); CK(dev_array(dRB, n_records, rb.data(), n_records));
    MaintParams M; memset(&M, 0, sizeof(M));
    M.leafA = dLA.p; M.adam = dAd.p; M.nNodes = dSc.p; M.capNodes = (uint32_t) n_nodes;
    const int sms = op_sm_count();
    if (bucket) {       // render_batch: histogram -> scan -> scatter into per-leaf buckets
        CK(dev_array(dCount, n_nodes)); CK(dev_array(dCursor, n_nodes)); CK(dev_array(dOff, n_nodes)); CK(dev_array(dSA, n_records)); CK(dev_array(dSB, n_records));
        adam_hist_kernel<<<sms * 4, 256>>>(dRA.p, dSc.p + 3, (uint32_t) n_records, dCount.p);
        exclusive_scan_kernel<<<1, 1024>>>(dCount.p, dOff.p, dSc.p, dSc.p + 4);
        adam_scatter_kernel<<<sms * 4, 256>>>(dRA.p, dRB.p, dSc.p + 3, (uint32_t) n_records, dOff.p, dCursor.p, dSA.p, dSB.p);
        CK(cudaGetLastError());
        if (bucketed_out && n_records) {
            CK(cudaMemcpy(ra.data(), dSA.p, 16 * n_records, cudaMemcpyDeviceToHost)); CK(cudaMemcpy(rb.data(), dSB.p, 8 * n_records, cudaMemcpyDeviceToHost));
            for (size_t i = 0; i < n_records; ++i) { memcpy(bucketed_out + 6 * i, &ra[i], 16); memcpy(bucketed_out + 6 * i + 4, &rb[i], 8); }
        }
        if (leaf_offset_out) CK(cudaMemcpy(leaf_offset_out, dOff.p, 4 * n_nodes, cudaMemcpyDeviceToHost));
    } else {            // records already grouped; the cursors hold the counts, as after adam_scatter_kernel
        for (size_t i = 0; i < n_nodes; ++i)
            if ((size_t) leaf_offset[i] + leaf_count[i] > n_records) return fail(PPG_ERR_INVALID_ARGUMENT, "ppg_op_adam_replay: a leaf's records run past n_records");
        CK(dev_array(dCount, n_nodes, leaf_count, n_nodes)); CK(dev_array(dCursor, n_nodes, leaf_count, n_nodes)); CK(dev_array(dOff, n_nodes, leaf_offset, n_nodes));
        if (leaf_offset_out) memcpy(leaf_offset_out, leaf_offset, 4 * n_nodes);
    }
    adam_seq_kernel<<<sms * 16, 128>>>(M, bucket ? dSA.p : dRA.p, bucket ? dSB.p : dRB.p, dOff.p, dCount.p, dCursor.p, loss == PPG_LOSS_KL ? 1.0f : 2.0f);
    CK(cudaGetLastError());
    CK(cudaMemcpy(state_inout, dAd.p, 24 * n_nodes, cudaMemcpyDeviceToHost));
    if (theta_out) {
        CK(cudaMemcpy(la.data(), dLA.p, 16 * n_nodes, cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < n_nodes; ++i) theta_out[i] = la[i].z;
    }
    if (count_out) CK(cudaMemcpy(count_out, dCount.p, 4 * n_nodes, cudaMemcpyDeviceToHost));
    if (cursor_out) CK(cudaMemcpy(cursor_out, dCursor.p, 4 * n_nodes, cudaMemcpyDeviceToHost));
    return PPG_OK;
  });
}
