// ppg_bounce.cuh -- the fused bounce kernel (ray generation / intersect / shade / guide / compaction), see ppg_kernels.cuh for the pipeline.
#pragma once
#include "ppg_wavefront.cuh"

namespace ppg {

// ------------------------------------------------------------------ the bounce kernel
// FIRST: generate the camera ray (renderBlock, GP:1613-1632) instead of loading a path state.
// RECORD: 0 = no vertex records (final iteration), 1 = basic record (nearest spatial filter, no loss),
//         2 = full record (stochastic/box spatial filter or a sampling-fraction loss).
template <bool FIRST, int RECORD, bool NEE, bool SMEM, bool FULL>
__global__ void __launch_bounds__(SMEM ? PPG_BOUNCE_BLOCK : PPG_BOUNCE_BLOCK_HBM, SMEM ? PPG_MIN_BLOCKS : PPG_MIN_BLOCKS_HBM) bounce_kernel(const __grid_constant__ RenderParams P) {
    const SceneAccess<SMEM> sc(P.scene);
    sc.stage();
    const uint32_t nIn = FIRST ? P.nPaths : *P.liveIn;
    uint32_t raysLocal = 0, recLocal = 0, levelsLocal = 0;          // per thread: 32 bits hold a launch's worth; widened for the warp sum
    // material bins left by trace_kernel: position j of the launch is the (j - start)-th entry of the bin that contains it
    __shared__ uint32_t binStart[PPG_BINS + 1];
    const bool binned = !SMEM && P.order != nullptr;
    if (binned) {
        if (threadIdx.x == 0) { uint32_t acc = 0; for (uint32_t b = 0; b < PPG_BINS; ++b) { binStart[b] = acc; acc += P.binCount[b]; } binStart[PPG_BINS] = acc; }
        __syncthreads();
    }

    // Work distribution: every warp claims PPG_CLAIM consecutive groups of 32 paths at a time from a launch-wide counter, so exactly one
    // block per resident slot is launched (the scene is staged once per slot) and the tail still balances.  No block barrier in the loop.
    const uint32_t lane = threadIdx.x & 31u;
    uint32_t claimBase = 0, claimLeft = 0;
    for (;;) {
        if (claimLeft == 0) {
            if (lane == 0) claimBase = atomicAdd(P.work, 32u * PPG_CLAIM);
            claimBase = __shfl_sync(0xffffffffu, claimBase, 0);
            claimLeft = PPG_CLAIM;
        }
        if (claimBase >= nIn) break;
        uint32_t i = claimBase + lane;
        claimBase += 32u; --claimLeft;
        bool alive = i < nIn;
        if (binned && alive) {
            uint32_t b = 0;
            while (b + 1 < PPG_BINS && i >= binStart[b + 1]) ++b;
            i = __ldg(&P.order[(size_t) b * P.binStride + (i - binStart[b])]);
        }
        float3 o, d, thr, Li; float eta = 1.f, rrRecip = 1.f, mint, maxt;
        float prevWoPdf = 0.f; float3 prevRefN = f3(0, 0, 0); uint32_t prevSlot = 0;      // NEE only
        uint32_t pathId = 0, nVertices = 0, flags = 0;
        Pcg32 rng; rng.state = 0; rng.inc = 1;        // the path's stream is keyed by its sample index: rng.inc == 2 * sampleIndex + 1
        if (alive) {
            if (FIRST) {
                pathId = i;
                uint64_t sampleIndex;
                camera_ray(P, i, rng, sampleIndex, o, d, mint, maxt);
                thr = f3(1, 1, 1); Li = f3(0, 0, 0);
            } else {
                const uint32_t s = state_slot(i, (uint32_t) __ldg(P.splitIn), P.pathCapacity);     // reloaded (L1) rather than held across the loop
                const float4 a = __ldcs(&P.in.s0[s]), b = __ldcs(&P.in.s1[s]), c = __ldcs(&P.in.s2[s]), e = __ldcs(&P.in.s3[s]), f = __ldcs(&P.in.s4[s]);   // streamed once: evict-first keeps the L2 for the trees
                o = f3(a.x, a.y, a.z); d = f3(a.w, b.x, b.y); thr = f3(b.z, b.w, c.x); eta = c.y; Li = f3(c.z, c.w, e.x);
                pathId = __float_as_uint(e.y);
                rng.state = ((uint64_t) __float_as_uint(e.w) << 32) | __float_as_uint(e.z);
                const uint64_t sampleIndex = ((uint64_t) __float_as_uint(f.y) << 32) | __float_as_uint(f.x);
                rng.inc = (sampleIndex << 1) | 1u;
                const uint32_t nf = __float_as_uint(f.z); nVertices = nf & 0xffu; flags = nf >> 8;
                rrRecip = f.w;
                if (NEE) { const float4 g5 = __ldcs(&P.in.s5[s]), g6 = __ldcs(&P.in.s6[s]); prevWoPdf = g5.x; prevRefN = f3(g5.y, g5.z, g5.w); prevSlot = __float_as_uint(g6.x); }
                mint = surface_ray_mint(o);
                maxt = __int_as_float(0x7f800000);
            }
        }
        bool wroteVertex = false, wroteNee = false, unscattered = FIRST, dtreeNext = false;
        Hit hit; bool rayOk = false, found = false;
        if (alive) {
            ++raysLocal;
            // a ray with a non-finite origin or direction (a BSDF sample gone wrong) would pass every node's slab test and walk the whole
            // tree; the reference's kd-tree clips such a ray away (AABB::rayIntersect fails on NaN comparisons): a miss.  Counted in counters[5].
            rayOk = isfinite(o.x + o.y + o.z) && isfinite(d.x + d.y + d.z);
            if (!rayOk) atomicAdd(&P.counters[5], 1ull);
            if (!SMEM && P.hits) {          // the nearest hit was found by trace_kernel (same rays, same tests, same tie rule)
                const float4 hv = __ldcs(&P.hits[i]);
                const uint32_t w = __float_as_uint(hv.w);
                hit.t = hv.x; hit.u = hv.y; hit.v = hv.z; hit.tri = 0; hit.prim = w;
                found = rayOk && w != 0xFFFFFFFFu;
                if (found && !(w & PPG_SPHERE_BIT)) { hit.tri = w; hit.prim = __float_as_uint(sc.accel(3 * w + 2).z); }
                if (!found) { hit.t = __int_as_float(0x7f800000); hit.prim = 0xFFFFFFFFu; }
            } else
                found = rayOk && bvh_intersect<FULL>(sc, o, d, mint, maxt, hit);
        }
        // the lanes leave the walk at different times: make them wait for each other HERE, so that shading runs with the whole warp (without
        // the barrier the scheduler may carry the early leavers through the shading code on their own)
        __syncwarp();
        if (alive) {
            bool cont = found;
            if (FULL && !found && rayOk && P.scene.envW) {
                // the ray left the scene: radiance of the environment emitter.  Camera rays and rays that have only crossed index-matched surfaces
                // take it through the EEmittedRadiance branch (GP:1902-1914: only while unscattered, and not with hideEmitters); after a real
                // bounce it is the `value` of rayIntersectAndLookForEmitter (GP:2228-2243), always added -- MIS-weighted against the light
                // sampling of the environment emitter when that runs (GP:2084-2088)
                const bool viaNull = !FIRST && (flags & PPG_FLAG_NULL);
                const bool add = (FIRST || viaNull) ? ((FIRST || (flags & PPG_FLAG_UNSCATTERED)) && !P.hideEmitters) : true;
                if (add) {
                    float3 Lenv = thr * env_eval(P.scene, d);
                    if (NEE && !FIRST && !viaNull && P.doNee && !(prevSlot >> 31))
                        Lenv = Lenv * mi_weight(prevWoPdf, pdf_emitter_direct<FULL>(P.scene, PPG_ENV_EMITTER, o, prevRefN, d, f3(0, 0, 0), 0.f));
                    Li = Li + Lenv;
                }
                if (NEE && !FIRST && !viaNull && P.training && P.neeMode == 2 && ((prevSlot >> 30) & 1u)) {
                    // nee == always: the vertex created at the previous bounce starts with radiance 0 instead of L (GP:2101), also when L came from the environment
                    const uint32_t ps = prevSlot & 0x3fffffffu;
                    float4 pv = P.prevSlab.v2[ps]; pv.x = Li.x; pv.y = Li.y; pv.z = Li.z; P.prevSlab.v2[ps] = pv;
                }
            }
            Its its;
            if (cont) {
                fill_its<FULL>(sc, hit, o, d, its);
                // emitted radiance: primary hit via EEmittedRadiance (GP:1917-1919), later hits via the `value`
                // returned by rayIntersectAndLookForEmitter (GP:2078-2091; miWeight(woPdf, 0) == 1)
                float3 Lhit = f3(0, 0, 0);
                const bool viaNull = FULL && !FIRST && (flags & PPG_FLAG_NULL);
                unscattered = FIRST || (FULL && (flags & PPG_FLAG_UNSCATTERED));
                if (FULL && viaNull) {
                    // after a null transition the hit is an ordinary path vertex: emitted radiance only while ERadiance is still
                    // requested, i.e. the path has not scattered yet (GP:2070-2071, 1917-1919)
                    if (its.emitter >= 0 && unscattered && !P.hideEmitters && dot(its.shN, -d) > 0.f) {
                        const float4 r = sc.radiance(its.emitter);
                        Li = Li + thr * f3(r.x, r.y, r.z);
                    }
                } else if (FULL && !FIRST && its.emitter < 0 && bsdf_has_null(load_bsdf<FULL>(sc, its.bsdf))) {
                    // first hit on an index-matched surface: the emitter lookup continues behind it (GP:2184-2245)
                    int qEmitter; float3 qN; float qDist;
                    const float3 value = look_through(sc, o, d, its, hit.t, P.maxDepth - P.depth, qEmitter, qN, qDist);
                    if (!is_zero(value)) {
                        Lhit = thr * value;
                        if (NEE && P.doNee && !(prevSlot >> 31)) Lhit = Lhit * mi_weight(prevWoPdf, pdf_emitter_direct<FULL>(sc.g, qEmitter, o, prevRefN, d, qN, qDist));
                        Li = Li + Lhit;
                    }
                } else if (its.emitter >= 0 && (!FIRST || !P.hideEmitters)) {
                    if (dot(its.shN, -d) > 0.f) {                                    // area.cpp:104-109
                        const float4 r = sc.radiance(its.emitter);
                        Lhit = thr * f3(r.x, r.y, r.z);
                        if (NEE && !FIRST && P.doNee && !(prevSlot >> 31)) {            // MIS against light sampling, GP:2084-2088
                            const float emitterPdf = pdf_emitter_direct<FULL>(sc.g, its.emitter, o, prevRefN, d, its.shN, hit.t);
                            Lhit = Lhit * mi_weight(prevWoPdf, emitterPdf);
                        }
                        Li = Li + Lhit;
                    }
                }
                if (NEE && !FIRST && P.training && P.neeMode == 2 && ((prevSlot >> 30) & 1u)) {
                    // nee == always: the vertex created at the previous bounce starts with radiance 0 instead of L (GP:2101):
                    // move its radiance prefix past this emitter hit
                    const uint32_t ps = prevSlot & 0x3fffffffu;
                    float4 pv = P.prevSlab.v2[ps]; pv.x = Li.x; pv.y = Li.y; pv.z = Li.z; P.prevSlab.v2[ps] = pv;
                }
                thr = thr * rrRecip;                                                // throughput /= successProb happens after L was recorded (GP:2141)
                if (flags & PPG_FLAG_DYING) cont = false;
                if (P.depth >= P.maxDepth && P.maxDepth != -1) cont = false;        // GP:1925
            }
            if (cont) {
                const float wiDotGeoN = -dot(its.geoN, d);
                if (wiDotGeoN * its.wi.z < 0.f && P.strictNormals) cont = false;     // GP:1929-1932
            }
            if (cont) {
                Bsdf bsdf = load_bsdf<FULL>(sc, its.bsdf);
                const float3 n0 = its.shN;                                           // normal of the interpolated shading frame (see apply_textures)
                const bool bump = FULL && bsdf.bumpTex && !(hit.prim & PPG_SPHERE_BIT);
                if (FULL && (bsdf.reflTex | bsdf.bumpTex) && !(hit.prim & PPG_SPHERE_BIT)) apply_textures(sc, hit, d, its, bsdf);   // its.getBSDF() without ray differentials (GP:1934)
                const bool smooth = bsdf_has_smooth(bsdf);                           // only smooth BSDFs are guided (GP:1942-1944)
                int levels = 0; uint32_t leaf = 0; float4 la = make_float4(0, 0, 0, 0);
                if (smooth) {
                    leaf = stree_lookup(P.tree.snodes, P.tree.stable, P.tree.aabbMin, P.tree.extent, its.p, levels);
                    la = __ldg(&P.tree.leafA[leaf]);
                }
                float frac = P.fixedFraction;
                if (smooth && P.lossMode != 0) frac = logistic(la.z);                 // GP:1946-1949
                // ---- sampleMat, GP:1650-1691
                float woPdf, bsdfPdf, dTreePdf, bsEta = 1.f; float3 wo, bsdfWeight; bool isDelta = false, isNull = false;
                float sx = rng.next1D(); const float sy = rng.next1D();
                if (!P.isBuilt || !smooth) {                                         // not built / no dTree / all-delta BSDF (GP:1654)
                    bsdfWeight = bsdf_sample(bsdf, its.wi, sx, sy, wo, bsEta, isDelta, bsdfPdf, rng, isNull);
                    if (bump && !is_zero(bsdfWeight) && dot(its.toWorld(wo), n0) * wo.z <= 0.f) bsdfWeight = f3(0, 0, 0);   // bumpmap.cpp:229-231
                    woPdf = bsdfPdf; dTreePdf = 0.f;
                } else {
                    const SampNode *tree = P.tree.samp + __float_as_uint(la.x);
                    const bool valid = __float_as_uint(la.w) & 1u;
                    float3 result; bool zero = false, deltaEarly = false;
                    if (sx < frac) {
                        sx /= frac;
                        result = bsdf_sample(bsdf, its.wi, sx, sy, wo, bsEta, isDelta, bsdfPdf, rng, isNull);
                        if (bump && !is_zero(result) && dot(its.toWorld(wo), n0) * wo.z <= 0.f) result = f3(0, 0, 0);
                        if (is_zero(result)) { woPdf = bsdfPdf = dTreePdf = 0.f; zero = true; }
                        else if (FULL && isDelta) { dTreePdf = 0.f; woPdf = bsdfPdf * frac; result = result * (1.0f / frac); deltaEarly = true; }   // GP:1670-1676
                        else result = result * bsdfPdf;
                    } else {
                        const float2 c2 = dtree_sample(tree, valid, rng);
                        const float3 dw = canonical_to_dir(c2);
                        wo = its.toLocal(dw);
                        result = (bump && dot(dw, n0) * wo.z <= 0.f) ? f3(0, 0, 0) : bsdf_eval(bsdf, its.wi, wo);   // bumpmap.cpp:169-170
                    }
                    if (zero) bsdfWeight = f3(0, 0, 0);
                    else if (deltaEarly) bsdfWeight = result;
                    else {   // pdfMat, GP:1693-1710
                        bsdfPdf = (bump && dot(its.toWorld(wo), n0) * wo.z <= 0.f) ? 0.0f : bsdf_pdf(bsdf, its.wi, wo);          // bumpmap.cpp:185-186
                        if (!isfinite(bsdfPdf)) { woPdf = 0.f; dTreePdf = 0.f; }
                        else {
                            dTreePdf = dtree_pdf(tree, valid, dir_to_canonical(its.toWorld(wo)));
                            woPdf = frac * bsdfPdf + (1.f - frac) * dTreePdf;
                        }
                        bsdfWeight = (woPdf == 0.f) ? f3(0, 0, 0) : result * (1.0f / woPdf);
                    }
                }
                const float3 refN = bsdf_has_transmission_or_backside(bsdf) ? f3(0, 0, 0) : n0;   // DirectSamplingRecord(its), records.inl:160-164
                if (NEE && P.doNee && smooth) {                                       // GP:1967-1969
                    // ---- luminaire sampling, GP:1964-2021
                    const float ex = rng.next1D(), ey = rng.next1D();
                    DirectSample ds; float dist;
                    if (sample_emitter_direct<FULL>(sc, its.p, refN, ex, ey, ds, dist)) {
                        // Scene::evalTransmittance: shadow ray, epsilon scaled without the clamp (skdtree.cpp:154-158)
                        const float smint = PPG_EPSILON * fmaxf(fmaxf(fabsf(its.p.x), fabsf(its.p.y)), fabsf(its.p.z));
                        Hit sh;      // (shadow rays are not path vertices: not counted in the samples metric)
                        bool visible;
                        if (FULL) {  // index-matched surfaces attenuate instead of blocking (Scene::evalTransmittance, interactions = maxDepth - depth - 1, GP:1970)
                            const float3 T = eval_transmittance(sc, its.p, ds.d, dist, P.maxDepth - P.depth - 1);
                            ds.value = ds.value * T; visible = !is_zero(ds.value);
                        } else visible = !bvh_intersect<FULL>(sc, its.p, ds.d, smint, dist * (1.f - PPG_SHADOW_EPSILON), sh);
                        if (visible) {
                            const float3 dl = its.toLocal(ds.d);
                            const float dlZ0 = bump ? dot(ds.d, n0) : dl.z;              // cos(theta) in the un-perturbed frame
                            if (!P.strictNormals || dot(its.geoN, ds.d) * dlZ0 > 0.f) {
                                const bool bumpReject = bump && dlZ0 * dl.z <= 0.f;
                                const float3 bsdfVal = bumpReject ? f3(0, 0, 0) : bsdf_eval(bsdf, its.wi, dl);
                                float nWoPdf = 0.f, nBsdfPdf = bumpReject ? 0.0f : bsdf_pdf(bsdf, its.wi, dl), nDTreePdf = 0.f;
                                if (!P.isBuilt) nWoPdf = nBsdfPdf;
                                else if (isfinite(nBsdfPdf)) {
                                    nDTreePdf = dtree_pdf(P.tree.samp + __float_as_uint(la.x), __float_as_uint(la.w) & 1u, dir_to_canonical(ds.d));
                                    nWoPdf = frac * nBsdfPdf + (1.f - frac) * nDTreePdf;
                                }
                                const float3 L = thr * (ds.value * bsdfVal) * mi_weight(ds.pdf, nWoPdf);
                                if (RECORD && P.neeMode != 2) {                          // GP:1999-2016: half-weight vertex with a fixed radiance
                                    const float3 tv = thr * bsdfVal * (1.0f / ds.pdf);
                                    __stcs(&P.neeSlab.v0[i], make_float4(ds.d.x, ds.d.y, ds.d.z, ds.pdf));
                                    __stcs(&P.neeSlab.v1[i], make_float4(tv.x, tv.y, tv.z, __uint_as_float(leaf)));
                                    __stcs(&P.neeSlab.v2[i], make_float4(L.x, L.y, L.z, __uint_as_float(pathId | 0x40000000u)));   // bit 30: absolute radiance
                                    __stcs(&P.neeSlab.v3[i], make_float4(bsdfVal.x, bsdfVal.y, bsdfVal.z, nBsdfPdf));
                                    __stcs(&P.neeSlab.v4[i], make_float4(its.p.x, its.p.y, its.p.z, nDTreePdf));
                                    __stcs(&P.neeSlab.v5[i], make_float4(__uint_as_float((uint32_t) (rng.inc >> 1)), __uint_as_float((uint32_t) (rng.inc >> 33)),
                                                                  __uint_as_float((uint32_t) levels | ((32u + (uint32_t) P.depth) << 8)), 0.f));
                                    wroteNee = true;
                                }
                                Li = Li + L;                                             // recordRadiance(L)
                            }
                        }
                    }
                }
                if (P.isBuilt && !binned) {
                    // the next vertex's technique (its sampleMat: sx = the draw after this vertex's Russian roulette, D-tree when sx >= frac),
                    // predicted here where frac is last needed -- exact for a fixed fraction; with a learned one the next leaf's fraction
                    // decides, and a wrong guess only costs divergence.  It places the path in the output wavefront (warp_compact_split) and
                    // changes nothing the path computes.  Material-binned launches take their warps from the bins instead: there the split
                    // would only spread the rays of a trace_kernel warp over twice the pixels (TORUS: 3.6 % slower), so every path stays in front.
                    Pcg32 peek = rng;
                    if (!(FULL && isNull) && P.depth >= P.rrDepth) peek.nextU32();
                    dtreeNext = !(peek.next1D() < frac);
                }
                if (is_zero(bsdfWeight)) cont = false;                               // GP:2024-2025
                float3 woW = f3(0, 0, 0);
                if (cont) {
                    woW = its.toWorld(wo);
                    if (dot(its.geoN, woW) * (bump ? dot(woW, n0) : wo.z) <= 0.f && P.strictNormals) cont = false;   // GP:2028-2032
                }
                if (cont) {
                    o = its.p; d = woW;
                    thr = thr * bsdfWeight; eta *= bsEta;
                    // ---- vertex record (GP:2093-2110); its radiance is Li_final - Li_prefix (SURVEY 3.2)
                    if (RECORD && smooth && (!isDelta || P.lossMode != 0) && nVertices < PPG_MAX_VERTICES && (1.f / woPdf > 0.f)) {
                        __stcs(&P.slab.v0[i], make_float4(d.x, d.y, d.z, woPdf));
                        __stcs(&P.slab.v1[i], make_float4(thr.x, thr.y, thr.z, __uint_as_float(leaf)));
                        __stcs(&P.slab.v2[i], make_float4(Li.x, Li.y, Li.z, __uint_as_float(pathId | (isDelta ? 0x80000000u : 0u))));
                        if (RECORD == 2) {
                            const float3 bv = bsdfWeight * woPdf;
                            __stcs(&P.slab.v3[i], make_float4(bv.x, bv.y, bv.z, bsdfPdf));
                            __stcs(&P.slab.v4[i], make_float4(o.x, o.y, o.z, dTreePdf));
                            __stcs(&P.slab.v5[i], make_float4(__uint_as_float((uint32_t) (rng.inc >> 1)), __uint_as_float((uint32_t) (rng.inc >> 33)),
                                                       __uint_as_float((uint32_t) levels | (nVertices << 8)), 0.f));
                        }
                        wroteVertex = true; ++nVertices; ++recLocal; levelsLocal += levels;
                    }
                    if (NEE) { prevWoPdf = woPdf; prevRefN = refN; prevSlot = i | (isDelta ? 0x80000000u : 0u) | ((wroteVertex && !(FULL && isNull)) ? 0x40000000u : 0u); }   // a null vertex starts at radiance 0: nothing to move (GP:2058)
                    // ---- Russian roulette (GP:2123-2142); the decision takes effect after the next emitter lookup
                    rrRecip = 1.f; flags = 0;
                    if (FULL && isNull) flags = PPG_FLAG_NULL | (unscattered ? PPG_FLAG_UNSCATTERED : 0u);   // GP:2044-2075: no roulette, `scattered` unchanged
                    else if (P.depth >= P.rrDepth) {
                        float successProb = 1.0f;
                        if (smooth && !isDelta) {
                            if (!P.isBuilt) successProb = max3(thr) * eta * eta;
                            successProb = fmaxf(0.1f, fminf(successProb, 0.99f));
                        }
                        if (rng.next1D() >= successProb) flags |= PPG_FLAG_DYING;
                        else rrRecip = 1.0f / successProb;
                    }
                }
            }
            if (!cont) {
                __stcs(&P.liFinal[pathId], make_float4(Li.x, Li.y, Li.z, 1.f));
                alive = false;
            }
        }
        if (RECORD && i < nIn && !wroteVertex) __stcs(&P.slab.v2[i], make_float4(0.f, 0.f, 0.f, __uint_as_float(PPG_INVALID)));
        if (NEE && RECORD && P.neeMode != 2 && i < nIn && !wroteNee) __stcs(&P.neeSlab.v2[i], make_float4(0.f, 0.f, 0.f, __uint_as_float(PPG_INVALID)));
        const uint32_t slot = warp_compact_split(alive, dtreeNext, P.splitOut, P.liveOut, P.pathCapacity);
        if (alive) {
            __stcs(&P.out.s0[slot], make_float4(o.x, o.y, o.z, d.x));
            __stcs(&P.out.s1[slot], make_float4(d.y, d.z, thr.x, thr.y));
            __stcs(&P.out.s2[slot], make_float4(thr.z, eta, Li.x, Li.y));
            __stcs(&P.out.s3[slot], make_float4(Li.z, __uint_as_float(pathId), __uint_as_float((uint32_t) rng.state), __uint_as_float((uint32_t) (rng.state >> 32))));
            __stcs(&P.out.s4[slot], make_float4(__uint_as_float((uint32_t) (rng.inc >> 1)), __uint_as_float((uint32_t) (rng.inc >> 33)),
                                         __uint_as_float(nVertices | (flags << 8)), rrRecip));
            if (NEE) {
                __stcs(&P.out.s5[slot], make_float4(prevWoPdf, prevRefN.x, prevRefN.y, prevRefN.z));
                __stcs(&P.out.s6[slot], make_float4(__uint_as_float(prevSlot), 0.f, 0.f, 0.f));
            }
        }
    }
    // per-warp reduction of the statistics counters
    unsigned long long rays = raysLocal, rec = recLocal, lev = levelsLocal;
    for (int off = 16; off; off >>= 1) {
        rays += __shfl_xor_sync(0xffffffffu, rays, off);
        rec += __shfl_xor_sync(0xffffffffu, rec, off);
        lev += __shfl_xor_sync(0xffffffffu, lev, off);
    }
    if ((threadIdx.x & 31) == 0) {
        if (rays) atomicAdd(&P.counters[0], rays);
        if (rec) { atomicAdd(&P.counters[1], rec); atomicAdd(&P.counters[2], lev); }
    }
}

}  // namespace ppg
