// ppg_scene.cpp -- host-only scene packing (see ppg_scene.h): validation, BVH construction and the tables the kernels read.
#include "ppg_scene.h"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <system_error>
#include <thread>
#ifdef __linux__
#include <sched.h>
#endif

namespace ppg {
namespace {
struct H3 { float x, y, z; };
static inline float half_to_float(uint16_t h) {                                  // IEEE binary16 -> binary32 (host side of the texel tables)
    const uint32_t sgn = (uint32_t) (h >> 15) << 31, e = (h >> 10) & 31u, m = h & 1023u;
    uint32_t bits;
    if (e == 0) {
        if (m == 0) bits = sgn;
        else { int sh = 0; uint32_t mm = m; while (!(mm & 1024u)) { mm <<= 1; ++sh; } bits = sgn | ((uint32_t) (113 - sh) << 23) | ((mm & 1023u) << 13); }
    } else if (e == 31) bits = sgn | 0x7f800000u | (m << 13);
    else bits = sgn | ((e + 112u) << 23) | (m << 13);
    float f; memcpy(&f, &bits, 4); return f;
}
static inline H3 h3(float x, float y, float z) { return H3{x, y, z}; }
static inline H3 operator-(H3 a, H3 b) { return h3(a.x - b.x, a.y - b.y, a.z - b.z); }
static inline H3 hcross(H3 a, H3 b) { return h3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
static inline float hdot(H3 a, H3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
static inline float hcomp(H3 a, int i) { return i == 0 ? a.x : (i == 1 ? a.y : a.z); }

// restated from include/mitsuba/render/triaccel.h:60-93 (Wald's projection-plane precomputation)
static void wald_constants(H3 A, H3 B, H3 C, float out[9], int &k) {
    static const int mod3[4] = {1, 2, 0, 1};
    const H3 b = C - A, c = B - A, N = hcross(c, b);
    k = 0;
    for (int j = 0; j < 3; ++j) if (std::fabs(hcomp(N, j)) > std::fabs(hcomp(N, k))) k = j;
    const int u = mod3[k], v = mod3[k + 1];
    const float n_k = hcomp(N, k), denom = hcomp(b, u) * hcomp(c, v) - hcomp(b, v) * hcomp(c, u);
    if (denom == 0) { k = 3; for (int i = 0; i < 9; ++i) out[i] = 0; return; }
    out[0] = hcomp(N, u) / n_k; out[1] = hcomp(N, v) / n_k; out[2] = hdot(A, N) / n_k;   // n_u n_v n_d
    out[3] = hcomp(A, u); out[4] = hcomp(A, v);                                           // a_u a_v
    out[5] = hcomp(b, u) / denom; out[6] = -hcomp(b, v) / denom;                          // b_nu b_nv
    out[7] = hcomp(c, v) / denom; out[8] = -hcomp(c, u) / denom;                          // c_nu c_nv
}

static int env_int(const char *name, int dflt) { const char *v = getenv(name); return v && *v ? atoi(v) : dflt; }   // tuning experiments only

// Host-side parallelism of the packing (per-triangle tables, BVH build, texel repacking): plain std::thread fork / join over index ranges.
// Every parallel loop below computes exactly what its serial form computes (min / max / integer counts / independent elements), so the
// scene tables do not depend on the thread count.
template <class F> static void parallel_for(size_t n, int threads, size_t minChunk, F fn) {   // fn(begin, end, chunk index)
    const int T = (int) std::max<size_t>(1, std::min<size_t>((size_t) threads, n / std::max<size_t>(minChunk, 1)));
    if (T <= 1) { fn((size_t) 0, n, 0); return; }
    std::vector<std::thread> pool; pool.reserve(T - 1);
    int started = 1;
    for (int k = 1; k < T; ++k) {
        try { pool.emplace_back([&, k] { fn(n * k / T, n * (k + 1) / T, k); }); ++started; }
        catch (const std::system_error &) { break; }                 // no more threads to be had: the remaining chunks run here
    }
    fn((size_t) 0, n / T, 0);
    for (int k = started; k < T; ++k) fn(n * k / T, n * (k + 1) / T, k);
    for (auto &th : pool) th.join();
}

// Binned-SAH BVH (16 bins per axis, leaves of at most PPG_BVH_LEAF triangles, a traversal-cost term decides the last splits).
// The tree is a function of the triangle bounds alone: a node's split depends only on the triangles of its range, children work on disjoint
// ranges of `order`.  It is therefore built in any order -- big nodes one after the other with their O(n) loops spread over the threads, the
// subtrees below them concurrently -- into an arena, and numbered afterwards in the order a depth-first stack visits it (right child first),
// which is the numbering the device layout (siblings adjacent, `left` = index of the first child) has always had.
static void build_bvh_from_bounds(const std::vector<H3> &tminV, const std::vector<H3> &tmaxV, HostBvh &out, int threads) {
    const uint32_t nt = (uint32_t) tminV.size();
    out.order.resize(nt);
    std::vector<H3> cenV(nt);
    const H3 *const tmin = tminV.data(), *const tmax = tmaxV.data(); H3 *const cen = cenV.data();
    parallel_for(nt, threads, 1 << 15, [&](size_t b, size_t e, int) {
        for (size_t t = b; t < e; ++t) { out.order[t] = (uint32_t) t; cen[t] = h3(0.5f * (tmin[t].x + tmax[t].x), 0.5f * (tmin[t].y + tmax[t].y), 0.5f * (tmin[t].z + tmax[t].z)); }
    });
    const int maxLeaf = std::min(std::max(env_int("PPG_BVH_LEAF", 4), 1), 15);   // <= 15: the device stack packs the count in 4 bits
    const float Ct = (float) env_int("PPG_BVH_CT_X10", 10) * 0.1f;
    constexpr int NB = 16;
    struct Node { H3 mn, mx; uint32_t left, count; };                                 // count == 0: inner node, `left` = arena index of its first child
    struct Job { uint32_t node, first, count; int depth; };
    struct Bounds { H3 mn, mx, cmn, cmx; };
    struct Bins { H3 mn[3][NB], mx[3][NB]; uint32_t c[3][NB]; };
    const H3 big = h3(1e30f, 1e30f, 1e30f), small = h3(-1e30f, -1e30f, -1e30f);
    auto hmin = [](H3 a, H3 b) { return h3(std::min(a.x, b.x), std::min(a.y, b.y), std::min(a.z, b.z)); };
    auto hmax = [](H3 a, H3 b) { return h3(std::max(a.x, b.x), std::max(a.y, b.y), std::max(a.z, b.z)); };
    auto area = [](H3 mn, H3 mx) { const float dx = mx.x - mn.x, dy = mx.y - mn.y, dz = mx.z - mn.z; return 2.f * (dx * dy + dy * dz + dz * dx); };
    auto binOf = [&](uint32_t t, int ax, float lo, float hi) { int b = (int) (NB * (hcomp(cen[t], ax) - lo) / (hi - lo)); return std::min(std::max(b, 0), NB - 1); };

    std::vector<Node> arena(2 * (size_t) nt + 1);
    std::atomic<uint32_t> arenaUsed{1};
    std::atomic<int> deepest{0};
    const uint32_t *order = out.order.data();

    // one node: bounds, best binned split, partition of its range.  Returns true and the left count when the node was split.
    auto process = [&](const Job &j, int loopThreads, uint32_t &nlOut) -> bool {
        Bounds bd{big, small, big, small};
        if (loopThreads > 1) {
            std::vector<Bounds> part((size_t) loopThreads, Bounds{big, small, big, small});
            parallel_for(j.count, loopThreads, 1 << 14, [&](size_t b, size_t e, int k) {
                Bounds l{big, small, big, small};
                for (size_t i = j.first + b; i < j.first + e; ++i) { const uint32_t t = order[i]; l.mn = hmin(l.mn, tmin[t]); l.mx = hmax(l.mx, tmax[t]); l.cmn = hmin(l.cmn, cen[t]); l.cmx = hmax(l.cmx, cen[t]); }
                part[k] = l;
            });
            for (const Bounds &l : part) { bd.mn = hmin(bd.mn, l.mn); bd.mx = hmax(bd.mx, l.mx); bd.cmn = hmin(bd.cmn, l.cmn); bd.cmx = hmax(bd.cmx, l.cmx); }
        } else
            for (uint32_t i = j.first; i < j.first + j.count; ++i) { const uint32_t t = order[i]; bd.mn = hmin(bd.mn, tmin[t]); bd.mx = hmax(bd.mx, tmax[t]); bd.cmn = hmin(bd.cmn, cen[t]); bd.cmx = hmax(bd.cmx, cen[t]); }
        Node nd; nd.mn = bd.mn; nd.mx = bd.mx; nd.left = j.first; nd.count = j.count;
        arena[j.node] = nd;
        if (j.count <= 1) return false;
        // binned SAH over the three axes (one pass fills the bins of all axes with a centroid extent)
        bool axisOk[3]; float lo[3], hi[3];
        for (int ax = 0; ax < 3; ++ax) { lo[ax] = hcomp(bd.cmn, ax); hi[ax] = hcomp(bd.cmx, ax); axisOk[ax] = hi[ax] > lo[ax]; }
        auto clearBins = [&](Bins &B) { for (int ax = 0; ax < 3; ++ax) if (axisOk[ax]) for (int b = 0; b < NB; ++b) { B.mn[ax][b] = big; B.mx[ax][b] = small; B.c[ax][b] = 0; } };
        auto fillBins = [&](Bins &B, size_t b0, size_t e0) {
            for (size_t i = j.first + b0; i < j.first + e0; ++i) {
                const uint32_t t = order[i];
                for (int ax = 0; ax < 3; ++ax) {
                    if (!axisOk[ax]) continue;
                    const int b = binOf(t, ax, lo[ax], hi[ax]);
                    B.c[ax][b]++; B.mn[ax][b] = hmin(B.mn[ax][b], tmin[t]); B.mx[ax][b] = hmax(B.mx[ax][b], tmax[t]);
                }
            }
        };
        Bins bins; clearBins(bins);
        if (loopThreads > 1) {
            std::vector<Bins> part((size_t) loopThreads);
            for (Bins &B : part) clearBins(B);
            parallel_for(j.count, loopThreads, 1 << 14, [&](size_t b, size_t e, int k) { fillBins(part[k], b, e); });
            for (const Bins &B : part)
                for (int ax = 0; ax < 3; ++ax) if (axisOk[ax]) for (int b = 0; b < NB; ++b) { bins.c[ax][b] += B.c[ax][b]; bins.mn[ax][b] = hmin(bins.mn[ax][b], B.mn[ax][b]); bins.mx[ax][b] = hmax(bins.mx[ax][b], B.mx[ax][b]); }
        } else fillBins(bins, 0, j.count);
        float bestCost = std::numeric_limits<float>::infinity(); int bestAxis = -1, bestBin = -1;
        for (int ax = 0; ax < 3; ++ax) {
            if (!axisOk[ax]) continue;
            const H3 *bmn = bins.mn[ax], *bmx = bins.mx[ax]; const uint32_t *bc = bins.c[ax];
            float rightArea[NB]; uint32_t rightCount[NB];
            H3 rmn = big, rmx = small; uint32_t rc = 0;
            for (int b = NB - 1; b > 0; --b) { rmn = hmin(rmn, bmn[b]); rmx = hmax(rmx, bmx[b]); rc += bc[b]; rightArea[b] = rc ? area(rmn, rmx) : 0.f; rightCount[b] = rc; }
            H3 lmn = big, lmx = small; uint32_t lc = 0;
            for (int b = 0; b < NB - 1; ++b) {
                lmn = hmin(lmn, bmn[b]); lmx = hmax(lmx, bmx[b]); lc += bc[b];
                if (lc == 0 || rightCount[b + 1] == 0) continue;
                const float cost = area(lmn, lmx) * lc + rightArea[b + 1] * rightCount[b + 1];
                if (cost < bestCost) { bestCost = cost; bestAxis = ax; bestBin = b; }
            }
        }
        // SAH with a traversal term: splitting pays when Ct * A + A_L N_L + A_R N_R < A * N (intersection cost 1)
        const float leafCost = area(bd.mn, bd.mx) * ((float) j.count - Ct);
        if (bestAxis >= 0 && (j.count > (uint32_t) maxLeaf || bestCost < leafCost)) {
            uint32_t *first = out.order.data() + j.first;
            uint32_t *mid = std::partition(first, first + j.count, [&](uint32_t t) { return binOf(t, bestAxis, lo[bestAxis], hi[bestAxis]) <= bestBin; });
            const uint32_t nl = (uint32_t) (mid - first);
            if (nl > 0 && nl < j.count) { nlOut = nl; return true; }
        }
        if (j.count > (uint32_t) maxLeaf) { nlOut = j.count / 2; return true; }     // degenerate centroids: split in the middle
        return false;
    };
    auto split = [&](const Job &j, uint32_t nl, Job &l, Job &r) {
        const uint32_t c0 = arenaUsed.fetch_add(2u);
        arena[j.node].left = c0; arena[j.node].count = 0;
        l = Job{c0, j.first, nl, j.depth + 1}; r = Job{c0 + 1, j.first + nl, j.count - nl, j.depth + 1};
    };
    auto noteDepth = [&](int d) { int cur = deepest.load(std::memory_order_relaxed); while (d > cur && !deepest.compare_exchange_weak(cur, d, std::memory_order_relaxed)) {} };

    // phase 1: the big nodes, one at a time, loops spread over the threads; everything smaller is queued
    const uint32_t bigCount = threads > 1 ? std::max<uint32_t>(1u << 16, nt / (4u * (uint32_t) threads)) : 0xFFFFFFFFu;
    std::vector<Job> top, queued; top.push_back(Job{0, 0, nt, 0});
    if (threads <= 1) { queued.swap(top); }
    while (!top.empty()) {
        const Job j = top.back(); top.pop_back();
        if (j.count < bigCount) { queued.push_back(j); continue; }
        noteDepth(j.depth);
        uint32_t nl = 0;
        if (process(j, threads, nl)) { Job l, r; split(j, nl, l, r); top.push_back(l); top.push_back(r); }
    }
    // phase 2: the subtrees below, each by one thread, largest first
    std::sort(queued.begin(), queued.end(), [](const Job &a, const Job &b) { return a.count > b.count; });
    std::atomic<size_t> nextJob{0};
    auto worker = [&] {
        std::vector<Job> stack;
        for (;;) {
            const size_t q = nextJob.fetch_add(1);
            if (q >= queued.size()) break;
            stack.push_back(queued[q]);
            int localDeepest = 0;
            while (!stack.empty()) {
                const Job j = stack.back(); stack.pop_back();
                localDeepest = std::max(localDeepest, j.depth);
                uint32_t nl = 0;
                if (process(j, 1, nl)) { Job l, r; split(j, nl, l, r); stack.push_back(l); stack.push_back(r); }
            }
            noteDepth(localDeepest);
        }
    };
    {
        const int T = (int) std::min<size_t>((size_t) std::max(threads, 1), queued.size());
        std::vector<std::thread> pool;
        for (int k = 1; k < T; ++k) { try { pool.emplace_back(worker); } catch (const std::system_error &) { break; } }   // the queue is dynamic: fewer threads, same result
        worker();
        for (auto &th : pool) th.join();
    }
    out.maxDepth = deepest.load();
    // phase 3: number the nodes as the depth-first stack of a serial build allocates them: a split node takes the next two indices when it is
    // popped, its right child is popped before its left one
    const uint32_t nNodes = arenaUsed.load();
    out.nodes.resize((size_t) nNodes * 8);
    struct Visit { uint32_t finalIndex, arenaIndex; };
    std::vector<Visit> st; st.push_back(Visit{0, 0});
    uint32_t finalUsed = 1;
    while (!st.empty()) {
        const Visit v = st.back(); st.pop_back();
        const Node &nd = arena[v.arenaIndex];
        uint32_t left = nd.left;
        if (nd.count == 0) { left = finalUsed; finalUsed += 2; st.push_back(Visit{left, nd.left}); st.push_back(Visit{left + 1, nd.left + 1}); }
        float *f = &out.nodes[8 * (size_t) v.finalIndex];
        f[0] = nd.mn.x; f[1] = nd.mn.y; f[2] = nd.mn.z; memcpy(&f[3], &left, 4);
        f[4] = nd.mx.x; f[5] = nd.mx.y; f[6] = nd.mx.z; memcpy(&f[7], &nd.count, 4);
    }
}

// one triangle's 6 float4 of vertex data {p_i.xyz, n_i.x} x 3, {n_i.yz, uv_i} x 3; missing normals or uvs are zero
static void geom_row(const ppg_scene_desc &s, uint32_t t, bool withUvs, float g[24]) {
    for (int k = 0; k < 3; ++k) {
        const uint32_t vi = s.indices[3 * t + k];
        const float *p = &s.positions[3 * vi];
        const float nz[3] = {0, 0, 0}; const float *n = s.normals ? &s.normals[3 * vi] : nz;
        const float uz[2] = {0, 0}; const float *uv = withUvs && s.uvs ? &s.uvs[2 * vi] : uz;
        g[4 * k] = p[0]; g[4 * k + 1] = p[1]; g[4 * k + 2] = p[2]; g[4 * k + 3] = n[0];
        g[12 + 4 * k] = n[1]; g[12 + 4 * k + 1] = n[2]; g[12 + 4 * k + 2] = uv[0]; g[12 + 4 * k + 3] = uv[1];
    }
}

// half texels repacked to one uint2 {r | g << 16, b} per texel; one-channel texels are replicated
static void repack_texels(const uint16_t *src, size_t nTexels, uint32_t channels, uint2 *dst) {
    parallel_for(nTexels, host_threads(), 1 << 18, [&](size_t i0, size_t i1, int) {
        for (size_t i = i0; i < i1; ++i) {
            const uint16_t r = src[i * channels], g = channels == 3 ? src[i * channels + 1] : r, b = channels == 3 ? src[i * channels + 2] : r;
            dst[i] = uint2{(uint32_t) r | ((uint32_t) g << 16), (uint32_t) b};
        }
    });
}

static int validate(const ppg_scene_desc &s, std::string &error) {
    auto fail = [&](int code, const char *msg) { error = msg; return code; };
    if (!s.n_triangles || !s.positions || !s.indices || !s.triangle_shape || !s.shapes || !s.bsdfs)
        return fail(PPG_ERR_INVALID_ARGUMENT, "scene needs triangles, shapes and bsdfs");
    if ((s.n_emitters && !s.area_radiance) || (s.n_spheres && !s.spheres)) return fail(PPG_ERR_INVALID_ARGUMENT, "emitter / sphere count without its array");
    if (s.camera.film_width <= 0 || s.camera.film_height <= 0 || s.camera.film_width > 65535 || s.camera.film_height > 65535)
        return fail(PPG_ERR_INVALID_ARGUMENT, "film size out of range");
    for (uint32_t t = 0; t < s.n_triangles; ++t) {
        if (s.triangle_shape[t] >= s.n_shapes) return fail(PPG_ERR_INVALID_ARGUMENT, "triangle_shape out of range");
        for (int k = 0; k < 3; ++k) if (s.indices[3 * t + k] >= s.n_vertices) return fail(PPG_ERR_INVALID_ARGUMENT, "vertex index out of range");
    }
    for (uint32_t i = 0; i < s.n_shapes; ++i) {
        if (s.shapes[i].bsdf < 0 || (uint32_t) s.shapes[i].bsdf >= s.n_bsdfs) return fail(PPG_ERR_INVALID_ARGUMENT, "shape bsdf out of range");
        if (s.shapes[i].emitter >= (int) s.n_emitters) return fail(PPG_ERR_INVALID_ARGUMENT, "shape emitter out of range");
    }
    for (uint32_t i = 0; i < s.n_bsdfs; ++i) {
        const ppg_bsdf &b = s.bsdfs[i];
        const int t = b.type;
        const bool transmissive = t == PPG_BSDF_DIELECTRIC || t == PPG_BSDF_ROUGHDIELECTRIC || t == PPG_BSDF_THINDIELECTRIC;
        if (t != PPG_BSDF_DIFFUSE && t != PPG_BSDF_NULL_BLACK && t != PPG_BSDF_DIELECTRIC && t != PPG_BSDF_CONDUCTOR && t != PPG_BSDF_ROUGHCONDUCTOR && t != PPG_BSDF_ROUGHPLASTIC && t != PPG_BSDF_ROUGHDIELECTRIC && t != PPG_BSDF_PLASTIC && t != PPG_BSDF_THINDIELECTRIC)
            return fail(PPG_ERR_UNSUPPORTED, "BSDF type outside the implemented hot-path scope");
        if ((b.flags & PPG_BSDF_FLAG_MASK) && t == PPG_BSDF_THINDIELECTRIC) return fail(PPG_ERR_UNSUPPORTED, "mask around another null-type BSDF");
        if (t == PPG_BSDF_ROUGHPLASTIC && (!s.bsdf_tables || b.table < 0 || (uint32_t) b.table >= s.n_bsdf_tables))
            return fail(PPG_ERR_INVALID_ARGUMENT, "roughplastic needs its rough-transmittance table (ppg_scene_desc.bsdf_tables)");
        if (transmissive && !(b.eta[0] > 0)) return fail(PPG_ERR_INVALID_ARGUMENT, "dielectric needs eta > 0");
        if (transmissive && (b.flags & PPG_BSDF_FLAG_TWOSIDED)) return fail(PPG_ERR_INVALID_ARGUMENT, "twosided cannot wrap a transmissive BSDF (twosided.cpp)");
        if (b.reflectance_texture > s.n_textures || b.bump_texture > s.n_textures) return fail(PPG_ERR_INVALID_ARGUMENT, "BSDF texture index out of range");
        if (b.reflectance_texture && t != PPG_BSDF_DIFFUSE && t != PPG_BSDF_ROUGHPLASTIC && t != PPG_BSDF_PLASTIC)
            return fail(PPG_ERR_UNSUPPORTED, "reflectance_texture: only the diffuse reflectance of diffuse / roughplastic / plastic can be textured");
        if ((b.flags & PPG_BSDF_FLAG_BUMPMAP) && !b.bump_texture) return fail(PPG_ERR_INVALID_ARGUMENT, "bumpmap: A displacement texture must be specified");
    }
    if (s.n_textures && (!s.textures || !s.texels)) return fail(PPG_ERR_INVALID_ARGUMENT, "textures without texel data");
    for (uint32_t i = 0; i < s.n_textures; ++i) {
        const ppg_texture &t = s.textures[i];
        if (!t.width || !t.height || (t.channels != 1 && t.channels != 3) || t.wrap_u > 2 || t.wrap_v > 2) return fail(PPG_ERR_INVALID_ARGUMENT, "texture: bad size, channel count or wrap mode");
        if (t.first_texel + (uint64_t) t.width * t.height * t.channels > s.n_texels) return fail(PPG_ERR_INVALID_ARGUMENT, "texture: texel range out of bounds");
    }
    for (uint32_t k = 0; k < s.n_spheres; ++k)       // spheres carry no texture coordinates here
        if (s.spheres[k].shape >= 0 && (uint32_t) s.spheres[k].shape < s.n_shapes) {
            const ppg_bsdf &b = s.bsdfs[s.shapes[s.spheres[k].shape].bsdf];
            if (b.reflectance_texture || (b.flags & PPG_BSDF_FLAG_BUMPMAP)) return fail(PPG_ERR_UNSUPPORTED, "textured / bump-mapped BSDF on an analytic sphere");
        }
    if (s.envmap.width && s.envmap.height && !s.envmap.texels) return fail(PPG_ERR_INVALID_ARGUMENT, "envmap without texel data");
    return PPG_OK;
}
}  // namespace

int host_threads() {
    static const int n = [] {
        int t = env_int("PPG_HOST_THREADS", 0);
        if (t <= 0) {
            t = (int) std::thread::hardware_concurrency();
#ifdef __linux__
            cpu_set_t set; CPU_ZERO(&set);
            if (sched_getaffinity(0, sizeof(set), &set) == 0) t = CPU_COUNT(&set);
#endif
            t = std::min(t, 16);
        }
        return std::max(t, 1);
    }();
    return n;
}

HostBvh build_bvh(const float *positions, const uint32_t *indices, uint32_t nt, int threads) {
    std::vector<H3> tmin(nt), tmax(nt);
    auto P = [&](uint32_t i) { return h3(positions[3 * i], positions[3 * i + 1], positions[3 * i + 2]); };
    parallel_for(nt, threads, 1 << 15, [&](size_t b0, size_t e0, int) {
        for (size_t t = b0; t < e0; ++t) {
            const H3 a = P(indices[3 * t]), b = P(indices[3 * t + 1]), c = P(indices[3 * t + 2]);
            tmin[t] = h3(std::min(a.x, std::min(b.x, c.x)), std::min(a.y, std::min(b.y, c.y)), std::min(a.z, std::min(b.z, c.z)));
            tmax[t] = h3(std::max(a.x, std::max(b.x, c.x)), std::max(a.y, std::max(b.y, c.y)), std::max(a.z, std::max(b.z, c.z)));
        }
    });
    HostBvh bvh; build_bvh_from_bounds(tmin, tmax, bvh, threads);
    return bvh;
}

float normalize_cdf(float *c, size_t n) {
    const float nrm = 1.0f / c[n];
    for (size_t i = 1; i < n; ++i) c[i] *= nrm;
    c[n] = 1.0f;
    return nrm;
}

PackedScene::Span PackedScene::array(int i) const {
    auto span = [](const auto &v) { return Span{v.empty() ? nullptr : (const void *) v.data(), v.size() * sizeof(v[0])}; };
    switch (i) {
    case kAccel: return span(accel);             case kGeom: return span(geom);                   case kMeta: return span(meta);
    case kBvh: return span(bvh);                 case kBsdf: return span(bsdf);                   case kBsdfTables: return span(bsdfTables);
    case kRadiance: return span(radiance);       case kGroups: return span(groups);               case kEmitterCdf: return span(emitterCdf);
    case kEmitterInfo: return span(emitterInfo); case kEmitterTriCdf: return span(emitterTriCdf); case kEmitterGeom: return span(emitterGeom);
    case kEmitterFlags: return span(emitterFlags); case kSpheres: return span(spheres);          case kTexMeta: return span(texMeta);
    case kTexels: return span(texels);           case kEnvTexels: return span(envTexels);         case kEnvCdfRows: return span(envCdfRows);
    case kEnvCdfCols: return span(envCdfCols);   case kEnvRowWeights: return span(envRowWeights);
    }
    return Span{nullptr, 0};
}

int pack_scene(const ppg_scene_desc &desc, PackedScene &p, std::string &error) {
    auto fail = [&](int code, const char *msg) { error = msg; return code; };
    if (const int rc = validate(desc, error)) return rc;
    const ppg_scene_desc *const s = &desc;
    SceneView &v = p.view;
    v = SceneView{}; p.env = EnvLight{};
    const uint32_t nt = s->n_triangles;
    const bool haveEnv = s->envmap.width && s->envmap.height;
    auto P = [&](uint32_t i) { return h3(s->positions[3 * i], s->positions[3 * i + 1], s->positions[3 * i + 2]); };
    HostBvh bvh = build_bvh(s->positions, s->indices, nt, host_threads());
    if (bvh.maxDepth >= PPG_BVH_STACK) return fail(PPG_ERR_UNSUPPORTED, "BVH deeper than the device traversal stack");
    // brute-force layout for tiny scenes: coplanar groups ordered by projection axis (see bvh_intersect)
    uint32_t kBegin[4] = {0, 0, 0, 0};
    std::vector<float> &groups = p.groups;
    groups.clear();
    if (nt <= PPG_BRUTE_FORCE_TRIS) {
        struct Tri { int k; float w[9]; uint32_t t; };
        std::vector<Tri> tris(nt);
        for (uint32_t t = 0; t < nt; ++t) { tris[t].t = t; wald_constants(P(s->indices[3 * t]), P(s->indices[3 * t + 1]), P(s->indices[3 * t + 2]), tris[t].w, tris[t].k); }
        static const int mod3[4] = {1, 2, 0, 1};
        std::vector<uint32_t> order; std::vector<char> used(nt, 0);
        for (int k = 0; k < 3; ++k) {
            kBegin[k] = (uint32_t) (groups.size() / 8);
            for (uint32_t a = 0; a < nt; ++a) {
                if (used[a] || tris[a].k != k) continue;
                // gather the triangles lying in (numerically) the same plane as `a`
                std::vector<uint32_t> members;
                for (uint32_t b = a; b < nt; ++b) {
                    if (used[b] || tris[b].k != k) continue;
                    const float *wa = tris[a].w, *wb = tris[b].w;
                    const float scale = 1.0f + std::fabs(wa[2]);
                    if (std::fabs(wa[0] - wb[0]) <= 1e-6f && std::fabs(wa[1] - wb[1]) <= 1e-6f && std::fabs(wa[2] - wb[2]) <= 1e-6f * scale) { members.push_back(b); used[b] = 1; }
                }
                float umin = 1e30f, vmin = 1e30f, umax = -1e30f, vmax = -1e30f;
                for (uint32_t b : members)
                    for (int c = 0; c < 3; ++c) {
                        const H3 vtx = P(s->indices[3 * b + c]);
                        umin = std::min(umin, hcomp(vtx, mod3[k])); umax = std::max(umax, hcomp(vtx, mod3[k]));
                        vmin = std::min(vmin, hcomp(vtx, mod3[k + 1])); vmax = std::max(vmax, hcomp(vtx, mod3[k + 1]));
                    }
                const float pad = 0.01f * std::max(umax - umin, vmax - vmin) + 1e-3f * (1.0f + std::max(std::max(std::fabs(umin), std::fabs(umax)), std::max(std::fabs(vmin), std::fabs(vmax))));
                const uint32_t fc = (uint32_t) order.size() | ((uint32_t) members.size() << 16);
                float g[8] = {tris[a].w[0], tris[a].w[1], tris[a].w[2], 0.f, umin - pad, vmin - pad, umax + pad, vmax + pad};
                memcpy(&g[3], &fc, 4);
                groups.insert(groups.end(), g, g + 8);
                for (uint32_t b : members) order.push_back(tris[b].t);
            }
        }
        kBegin[3] = (uint32_t) (groups.size() / 8);
        for (uint32_t t = 0; t < nt; ++t) if (tris[t].k == 3) order.push_back(t);
        if (groups.size() / 8 <= 32) bvh.order = order;       // the candidate mask of the lock-step test has 32 bits
        else { groups.clear(); kBegin[0] = kBegin[1] = kBegin[2] = kBegin[3] = 0; }
    }
    const bool bruteForce = !groups.empty();
    if (groups.empty()) groups.assign(8, 0.f);
    v.nGroups = bruteForce ? (uint32_t) (groups.size() / 8) : 0u;
    for (int k = 0; k < 4; ++k) v.kBegin[k] = kBegin[k];
    p.accel.assign(12 * (size_t) nt, 0.f); p.geom.assign(24 * (size_t) nt, 0.f); p.meta.assign(4 * (size_t) nt, 0);
    parallel_for(nt, host_threads(), 1 << 14, [&](size_t slot0, size_t slot1, int) {
    for (uint32_t slot = (uint32_t) slot0; slot < (uint32_t) slot1; ++slot) {
        const uint32_t t = bvh.order[slot];
        float w[9]; int k; wald_constants(P(s->indices[3 * t]), P(s->indices[3 * t + 1]), P(s->indices[3 * t + 2]), w, k);
        float *a = &p.accel[12 * (size_t) slot];
        a[0] = w[0]; a[1] = w[1]; a[2] = w[2]; memcpy(&a[3], &k, 4);
        a[4] = w[3]; a[5] = w[4]; a[6] = w[5]; a[7] = w[6];
        a[8] = w[7]; a[9] = w[8]; memcpy(&a[10], &t, 4); memcpy(&a[11], &slot, 4);
        geom_row(*s, t, true, &p.geom[24 * (size_t) slot]);
        const ppg_shape &sh = s->shapes[s->triangle_shape[t]];
        int32_t *m = &p.meta[4 * (size_t) slot];
        m[0] = sh.bsdf; m[1] = sh.emitter; m[2] = ((sh.has_normals && s->normals) ? 1 : 0) | ((sh.has_uvs && s->uvs) ? 2 : 0); m[3] = (int32_t) s->triangle_shape[t];
    }
    });
    p.bvh = std::move(bvh.nodes);
    p.fullFeature = false;
    for (uint32_t i = 0; i < s->n_bsdfs; ++i) if ((s->bsdfs[i].type != PPG_BSDF_DIFFUSE && s->bsdfs[i].type != PPG_BSDF_NULL_BLACK) || (s->bsdfs[i].flags & ~PPG_BSDF_FLAG_TWOSIDED)) p.fullFeature = true;   // any non-diffuse model or wrapper other than twosided
    if (s->n_spheres) p.fullFeature = true;                                            // ... or analytic spheres: the full-feature kernel variants
    if (s->n_textures || haveEnv) p.fullFeature = true;                                // ... or textures / an environment emitter
    p.bsdf.assign(4 * PPG_BSDF_F4 * (size_t) s->n_bsdfs, 0.f);
    for (uint32_t i = 0; i < s->n_bsdfs; ++i) {
        float *b = &p.bsdf[4 * PPG_BSDF_F4 * (size_t) i]; const ppg_bsdf &m = s->bsdfs[i];
        b[0] = m.reflectance[0]; b[1] = m.reflectance[1]; b[2] = m.reflectance[2];
        uint32_t type = (uint32_t) m.type;
        if (m.type == PPG_BSDF_NULL_BLACK) { b[0] = b[1] = b[2] = 0.f; type = PPG_BSDF_DIFFUSE; }
        const uint32_t tf = type | ((m.flags & 0xffffffu) << 8); memcpy(&b[3], &tf, 4);
        b[4] = m.specular_transmittance[0]; b[5] = m.specular_transmittance[1]; b[6] = m.specular_transmittance[2]; b[7] = m.eta[0];
        b[8] = m.eta[0]; b[9] = m.eta[1]; b[10] = m.eta[2]; b[11] = m.eta[0] != 0.f ? 1.0f / m.eta[0] : 0.f;
        b[12] = m.k[0]; b[13] = m.k[1]; b[14] = m.k[2];
        b[15] = std::max(m.alpha, 1e-4f) * (m.distribution == PPG_MICROFACET_BECKMANN ? -1.0f : 1.0f);   // microfacet.h:63 clamp; sign encodes the distribution
        b[16] = m.specular_reflectance[0]; b[17] = m.specular_reflectance[1]; b[18] = m.specular_reflectance[2]; b[19] = m.fdr_int;
        b[20] = m.specular_sampling_weight; const uint32_t tab = (uint32_t) std::max(m.table, 0); memcpy(&b[21], &tab, 4);
        memcpy(&b[22], &m.reflectance_texture, 4); memcpy(&b[23], &m.bump_texture, 4);
        b[24] = m.opacity[0]; b[25] = m.opacity[1]; b[26] = m.opacity[2];
        b[27] = m.opacity[0] * 0.212671f + m.opacity[1] * 0.715160f + m.opacity[2] * 0.072169f;                // getLuminance (spectrum.h:725-727)
    }
    // (one zero float without tables: the plastic models still form their table pointer from it)
    p.bsdfTables.assign(s->bsdf_tables, s->bsdf_tables + (s->bsdf_tables ? (size_t) s->n_bsdf_tables * PPG_BSDF_TABLE_SIZE : 0));
    if (p.bsdfTables.empty()) p.bsdfTables.assign(1, 0.f);
    p.radiance.assign(4 * (size_t) std::max<uint32_t>(s->n_emitters, 1), 0.f);
    for (uint32_t i = 0; i < s->n_emitters; ++i) { p.radiance[4 * i] = s->area_radiance[3 * i]; p.radiance[4 * i + 1] = s->area_radiance[3 * i + 1]; p.radiance[4 * i + 2] = s->area_radiance[3 * i + 2]; }
    {   // emitter sampling tables for next event estimation (TriMesh::prepareSamplingTable trimesh.cpp:388-403; Scene::configure scene.cpp:357-381)
        const uint32_t ne = std::max<uint32_t>(s->n_emitters, 1);
        std::vector<float> &ecdf = p.emitterCdf, &tcdf = p.emitterTriCdf, &egeom = p.emitterGeom, &einfo = p.emitterInfo;
        ecdf.assign(1, 0.f); tcdf.clear(); egeom.clear(); einfo.assign(4 * (size_t) ne, 0.f); p.emitterFlags.assign(ne, 0u);
        for (uint32_t e = 0; e < s->n_emitters; ++e) {
            int shape = -1;
            for (uint32_t si = 0; si < s->n_shapes; ++si) if (s->shapes[si].emitter == (int) e) shape = (int) si;
            const uint32_t first = (uint32_t) (egeom.size() / 24), cdfOff = (uint32_t) tcdf.size();
            uint32_t ntri = 0; float invArea = 0.f;
            int sphere = -1;
            for (uint32_t k = 0; k < s->n_spheres; ++k) if (shape >= 0 && s->spheres[k].shape == shape) sphere = (int) k;
            if (sphere >= 0) {                                                                      // sphere.cpp:128: m_invSurfaceArea
                const uint32_t tag = PPG_SPHERE_BIT | (uint32_t) sphere; const float r = s->spheres[sphere].radius;
                invArea = 1 / (4 * 3.14159265358979323846f * r * r);
                memcpy(&einfo[4 * e], &tag, 4); memcpy(&einfo[4 * e + 1], &ntri, 4); einfo[4 * e + 2] = invArea; memcpy(&einfo[4 * e + 3], &cdfOff, 4);
                ecdf.push_back(ecdf.back() + 1.0f);
                continue;
            }
            if (shape >= 0) {
                const ppg_shape &sh = s->shapes[shape];
                if ((uint64_t) sh.first_triangle + sh.n_triangles > nt) return fail(PPG_ERR_INVALID_ARGUMENT, "shape triangle range out of bounds");
                ntri = sh.n_triangles; p.emitterFlags[e] = (sh.has_normals && s->normals) ? 1u : 0u;
                std::vector<float> c(1, 0.f);
                for (uint32_t t = sh.first_triangle; t < sh.first_triangle + sh.n_triangles; ++t) {
                    const H3 p0 = P(s->indices[3 * t]), p1 = P(s->indices[3 * t + 1]), p2 = P(s->indices[3 * t + 2]);
                    const H3 cr = hcross(p1 - p0, p2 - p0);
                    c.push_back(c.back() + 0.5f * std::sqrt(hdot(cr, cr)));                       // Triangle::surfaceArea
                    egeom.resize(egeom.size() + 24);
                    geom_row(*s, t, false, &egeom[egeom.size() - 24]);
                }
                if (c.back() > 0) invArea = normalize_cdf(c.data(), c.size() - 1);
                tcdf.insert(tcdf.end(), c.begin(), c.end());
            }
            memcpy(&einfo[4 * e], &first, 4); memcpy(&einfo[4 * e + 1], &ntri, 4); einfo[4 * e + 2] = invArea; memcpy(&einfo[4 * e + 3], &cdfOff, 4);
            ecdf.push_back(ecdf.back() + 1.0f);                                                    // getSamplingWeight() == 1
        }
        v.envLight = 0xFFFFFFFFu;
        if (haveEnv) { v.envLight = s->n_emitters; ecdf.push_back(ecdf.back() + 1.0f); }          // the environment emitter: last entry of the light list
        v.nLights = (uint32_t) ecdf.size() - 1u;
        float norm = 0.f;
        if (ecdf.back() > 0) norm = normalize_cdf(ecdf.data(), ecdf.size() - 1);
        if (ecdf.size() < 2) { ecdf.push_back(1.0f); v.nLights = 1u; }                             // no light at all: one empty entry (never sampled, useNee() is false)
        if (tcdf.empty()) tcdf.assign(2, 0.f);
        if (egeom.empty()) egeom.assign(24, 0.f);
        v.emitterNormalization = norm; p.nRealEmitters = s->n_emitters + (haveEnv ? 1u : 0u);
    }
    p.spheres.assign(8 * (size_t) std::max<uint32_t>(s->n_spheres, 1), 0.f);                      // analytic spheres
    for (uint32_t k = 0; k < s->n_spheres; ++k) {
        const ppg_sphere &sp = s->spheres[k];
        if (sp.shape < 0 || (uint32_t) sp.shape >= s->n_shapes || !(sp.radius > 0)) return fail(PPG_ERR_INVALID_ARGUMENT, "sphere: bad shape index or radius");
        float *o = &p.spheres[8 * (size_t) k];
        o[0] = sp.center[0]; o[1] = sp.center[1]; o[2] = sp.center[2]; o[3] = sp.radius;
        const int32_t bs = s->shapes[sp.shape].bsdf, em = s->shapes[sp.shape].emitter; const uint32_t fl = sp.flip_normals ? 1u : 0u;
        memcpy(&o[4], &bs, 4); memcpy(&o[5], &em, 4); memcpy(&o[6], &fl, 4);
    }
    v.nSpheres = s->n_spheres;
    {   // bitmap textures
        size_t total = 0;
        for (uint32_t i = 0; i < s->n_textures; ++i) total += (size_t) s->textures[i].width * s->textures[i].height;
        if (total >= (1ull << 32)) return fail(PPG_ERR_UNSUPPORTED, "more than 2^32 texels");
        p.texels.assign(std::max<size_t>(total, 1), uint2{0u, 0u}); p.texMeta.assign(8 * (size_t) std::max<uint32_t>(s->n_textures, 1), 0.f);
        size_t off = 0;
        for (uint32_t i = 0; i < s->n_textures; ++i) {
            const ppg_texture &t = s->textures[i];
            repack_texels(s->texels + t.first_texel, (size_t) t.width * t.height, t.channels, p.texels.data() + off);
            float *m = &p.texMeta[8 * (size_t) i];
            const uint32_t wr = t.wrap_u | (t.wrap_v << 8), o32 = (uint32_t) off;
            memcpy(&m[0], &t.width, 4); memcpy(&m[1], &t.height, 4); memcpy(&m[2], &wr, 4); memcpy(&m[3], &o32, 4);
            m[4] = t.uv_scale[0]; m[5] = t.uv_scale[1]; m[6] = t.uv_offset[0]; m[7] = t.uv_offset[1];
            off += (size_t) t.width * t.height;
        }
        v.nTextures = s->n_textures;
    }
    v.envW = v.envH = 0; v.envScale = 1.f;
    for (int i = 0; i < 9; ++i) v.worldToEnv[i] = (i % 4 == 0) ? 1.f : 0.f;
    p.envTexels.clear(); p.envCdfRows.clear(); p.envCdfCols.clear(); p.envRowWeights.clear();
    if (haveEnv) {
        // the lat-long map, then the light-sampling tables of EnvironmentMap::configure (src/emitters/envmap.cpp:260-329), in the reference's float / double mix
        p.envTexels.resize((size_t) s->envmap.width * s->envmap.height);
        repack_texels(s->envmap.texels, p.envTexels.size(), 3, p.envTexels.data());
        v.envW = s->envmap.width; v.envH = s->envmap.height; v.envScale = s->envmap.scale;
        for (int i = 0; i < 9; ++i) v.worldToEnv[i] = s->envmap.world_to_env[i];
        EnvLight &el = p.env;
        const uint32_t Wd = s->envmap.width, Hd = s->envmap.height;
        const double kPi = 3.14159265358979323846;
        auto lum = [&](uint32_t x, uint32_t y) {                                               // Color3::getLuminance of texel (x, y)
            const uint16_t *px = s->envmap.texels + ((size_t) y * Wd + x) * 3;
            return half_to_float(px[0]) * 0.212671f + half_to_float(px[1]) * 0.715160f + half_to_float(px[2]) * 0.072169f;
        };
        std::vector<float> &cols = p.envCdfCols, &rows = p.envCdfRows, &weights = p.envRowWeights;
        cols.assign((size_t) (Wd + 1) * Hd, 0.f); rows.assign((size_t) Hd + 1, 0.f); weights.assign(Hd, 0.f);
        float rowSum = 0.0f;
        for (uint32_t y = 0; y < Hd; ++y) {
            float *col = &cols[(size_t) y * (Wd + 1)];
            float colSum = 0;
            for (uint32_t x = 0; x < Wd; ++x) { colSum += lum(x, y); col[x + 1] = colSum; }
            normalize_cdf(col, Wd);                                                                // a black row keeps its NaNs, as in the reference
            const float weight = (float) std::sin((double) ((float) y + 0.5f) * kPi / (double) Hd);
            weights[y] = weight;
            rowSum += colSum * weight;
            rows[y + 1] = rowSum;
        }
        if (rowSum == 0) return fail(PPG_ERR_INVALID_ARGUMENT, "The environment map is completely black -- this is not allowed.");
        if (!std::isfinite(rowSum)) return fail(PPG_ERR_INVALID_ARGUMENT, "The environment map contains an invalid floating point value (nan/inf) -- giving up.");
        normalize_cdf(rows.data(), Hd);
        el.normalization = (float) (1.0 / ((double) rowSum * (2 * kPi / (double) Wd) * (kPi / (double) Hd)));
        el.pixelX = (float) (2 * kPi / (double) Wd); el.pixelY = (float) (kPi / (double) Hd);
        float ctr[3], dd = 0.f;                                                                // AABB::getBSphere (libcore/aabb.cpp:44-47), radius x 1.5 (envmap.cpp:333)
        for (int i = 0; i < 3; ++i) { ctr[i] = (s->aabb_max[i] + s->aabb_min[i]) * 0.5f; el.center[i] = ctr[i]; }
        { const float ex = ctr[0] - s->aabb_max[0], ey = ctr[1] - s->aabb_max[1], ez = ctr[2] - s->aabb_max[2]; dd = std::sqrt(ex * ex + ey * ey + ez * ez); }
        el.radius = std::max(1e-4f, dd * 1.5f);
        const float *m = s->envmap.world_to_env;                                               // the emitter-to-world rotation back from its inverse
        const double a = m[0], b = m[1], c = m[2], d = m[3], e = m[4], f = m[5], g = m[6], hh = m[7], ii = m[8];
        const double det = a * (e * ii - f * hh) - b * (d * ii - f * g) + c * (d * hh - e * g);
        if (!(std::fabs(det) > 0)) return fail(PPG_ERR_INVALID_ARGUMENT, "envmap: singular world_to_env");
        const double id = 1.0 / det;
        const double inv[9] = {(e * ii - f * hh) * id, (c * hh - b * ii) * id, (b * f - c * e) * id, (f * g - d * ii) * id, (a * ii - c * g) * id, (c * d - a * f) * id,
                               (d * hh - e * g) * id, (b * g - a * hh) * id, (a * e - b * d) * id};
        for (int k = 0; k < 9; ++k) el.toWorld[k] = (float) inv[k];
    }
    v.nTris = nt; v.nBvhNodes = (uint32_t) (p.bvh.size() / 8); v.nBsdfs = s->n_bsdfs; v.nEmitters = std::max<uint32_t>(s->n_emitters, 1);
    const size_t sceneBytes = 16 * ((size_t) 3 * nt + 6 * nt + nt + 2 * (size_t) v.nBvhNodes + PPG_BSDF_F4 * s->n_bsdfs + v.nEmitters + 2 * std::max<uint32_t>(v.nGroups, 1));
    // tiny scenes (CBOX: ~9 KB) live in shared memory.  Only those with coplanar groups: the staged bounce kernels test the groups and have no
    // BVH walk, whose 512-byte stack would put every thread's frame in local memory.
    p.sceneSmemBytes = sceneBytes <= 48 * 1024 && v.nGroups != 0u ? (uint32_t) sceneBytes : 0u;
    // camera (src/sensors/perspective.cpp:120-298; lookAt columns: left, up, dir, origin -- transform.cpp:191-214)
    const float *m = s->camera.to_world;
    Camera &c = p.cam;
    c.left = float3{m[0], m[4], m[8]}; c.up = float3{m[1], m[5], m[9]}; c.dir = float3{m[2], m[6], m[10]}; c.o = float3{m[3], m[7], m[11]};
    const float aspect = (float) s->camera.film_width / (float) s->camera.film_height;
    c.tanX = std::tan(0.5f * s->camera.x_fov_deg * (3.14159265358979323846f / 180.0f)); c.tanY = c.tanX / aspect;
    c.nearClip = s->camera.near_clip; c.farClip = s->camera.far_clip; c.W = s->camera.film_width; c.H = s->camera.film_height;
    p.W = c.W; p.H = c.H;
    for (int i = 0; i < 3; ++i) { p.aabbMin[i] = s->aabb_min[i]; p.aabbMax[i] = s->aabb_max[i]; }
    // STree::STree (GP:850-860): cubify from the min corner
    const float sx = p.aabbMax[0] - p.aabbMin[0], sy = p.aabbMax[1] - p.aabbMin[1], sz = p.aabbMax[2] - p.aabbMin[2];
    const float mxs = std::max(std::max(sx, sy), sz);
    for (int i = 0; i < 3; ++i) { const float mx = p.aabbMin[i] + mxs; p.extent[i] = mx - p.aabbMin[i]; }
    return PPG_OK;
}

}  // namespace ppg
