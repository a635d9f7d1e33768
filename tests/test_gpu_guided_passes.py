"""The render's guided passes against the CPU oracle pixel by pixel, on the SD-tree the GPU built.

From iteration 1 on, the GPU and the oracle guide with different trees: both add the recorded statistics with float atomics, in different orders,
so their trees part after the first build and the renders then share only their statistics.  Here the oracle is handed the GPU's own tree instead.
In the film callback of an iteration (after its passes, before its build) the test reads the GPU's moment images, its sampling trees (the trees
those passes guided with, on the refined S-tree) and its building trees (what those passes recorded) through ppg_export_sdtree.  A port oracle on
the same scene and parameters imports the sampling trees and the pass count (ppgo_tree_import), resets its building trees as resetSDTree does
after the refine (ppgo_tree_reset), and renders the same passes with the same per-path PCG streams.  The guided passes -- sampleMat / pdfMat
(GP:1650-1710) at the leaf's fraction, the guided NEE MIS weight, the guided Russian roulette, the vertex records -- then become as deterministic a
comparison as the unguided first pass (common.assert_render_parity), and are held to the same bar:
  * the per-pixel sample counts are equal;
  * the RGB sums agree to rtol 1e-3 / atol 1e-5 on >= 99.8 % of the pixels, with relMSE <= 1e-9 over those pixels (libm ulps in
    dir_to_canonical / canonical_to_dir / logistic / the microfacet code may flip a discrete decision of a few paths);
  * building trees of a training iteration: the post-reset topology equals the oracle's reset bit for bit; per-leaf statistical weights (sums of
    1 and 1/2, exact in float; with the spatial box filter sums of volume fractions, to 1e-5) are equal except on the few leaves that a flipped
    path reached (at most max(4, 0.1 %) of them, each within max(40, 2e-4 x weight): one path records at most 10 + 10 x 1/2 on each side), and
    their total is within max(4, 2e-4 x total); quadtree sums within 1e-4 of their leaf's total (the scale of the dTreeThreshold = 0.01 decision they feed).  The GPU's vertex radiance is the prefix difference
    Li_final - Li_prefix added by atomics, the oracle's is accumulated per vertex.
Measured once on one H100 80GB HBM3 (700 W): pixel shares 1.0 everywhere except the NEE configuration (0.99994) and cbox-textured (0.99951 /
0.99957, relMSE over the close pixels 1.2e-10 / 1.9e-10; elsewhere <= 1.4e-12); at most two leaves per configuration with unequal weights, by
0.5 - 5 records; largest sum deviation 6.7e-5 of the leaf's total on cbox-textured, <= 2.3e-6 elsewhere.

Iteration 1 of a render that learns the sampling fractions (loss kl) is not compared: the GPU learns them in sub-batches (the Adam replay after
each wavefront), the oracle online, so the two end that iteration with different fractions.  Its final iteration 2 learns nothing and guides every
vertex with logistic(theta) of the GPU's learned theta, which the oracle imports."""
import numpy as np
import pytest

import oracle_lib as O
from common import cbox_with_sphere, load_cbox, load_fixture_scene, relmse

pytestmark = pytest.mark.gpu

BASE = dict(budget="28", sppPerPass="4", rrDepth="5")           # passes 1 + 2 + 4; roulette from depth 5 (CBOX's own rrDepth equals its maxDepth)


def _scene(name):
    from ppg_b200 import builtin_scenes as B
    if name == "cbox":
        return load_cbox(128)
    if name == "sphere":
        return cbox_with_sphere(128, subdiv=2)
    if name == "rough-metal-sphere":
        return B.cbox_rough_metal(cbox_with_sphere(128, subdiv=2))
    if name == "smooth-plastic":
        return B.cbox_smooth_plastic(load_cbox(128))
    return load_fixture_scene(name, 128)


# (scene, parameters, iterations compared) -- each reaches a different part of the bounce kernel
CONFIGS = {
    # staged scene, FULL = false, RECORD 1; the mixture at a fraction other than 1/2
    "cbox-frac0.3": ("cbox", dict(bsdfSamplingFractionLoss="none", bsdfSamplingFraction="0.3"), (1, 2)),
    # light sampling: guided MIS weight, NEE vertex slabs (weight 1/2), RECORD 2
    "cbox-nee-stochastic-box": ("cbox", dict(bsdfSamplingFractionLoss="none", bsdfSamplingFraction="0.3", nee="kickstart", spatialFilter="stochastic",
                                             directionalFilter="box"), (1, 2)),
    # HBM scene: BVH walk and trace_kernel (65 536 paths per pass >= 32 768), spatial box filter
    "sphere-box": ("sphere", dict(bsdfSamplingFractionLoss="none", spatialFilter="box"), (1, 2)),
    # FULL on the HBM path: paths shaded in material-bin order
    "rough-metal-sphere": ("rough-metal-sphere", dict(bsdfSamplingFractionLoss="none", bsdfSamplingFraction="0.3"), (1, 2)),
    # FULL: bump-map rejections in sampleMat / pdfMat, bitmap textures, environment emitter (the stored scene of builtin_scenes.cbox_textured)
    "textured": ("cbox-textured", dict(bsdfSamplingFractionLoss="none", bsdfSamplingFraction="0.3"), (1, 2)),
    # FULL: the delta early-out of sampleMat (GP:1670-1676)
    "smooth-plastic": ("smooth-plastic", dict(bsdfSamplingFractionLoss="none", bsdfSamplingFraction="0.3"), (1, 2)),
    # learned fractions: per-leaf frac = logistic(theta) in the final iteration
    "cbox-kl": ("cbox", dict(bsdfSamplingFractionLoss="kl"), (2,)),
    "plastic-kl": ("cbox-plastic", dict(bsdfSamplingFractionLoss="kl"), (2,)),
}


def _render_with_snapshots(sc, props, iterations):
    """GPU render; in the film callback of each listed iteration: passes rendered, moment images, sampling and building export."""
    from ppg_b200.integrator import GuidedPathTracer
    g = GuidedPathTracer(props); g.set_scene(sc)
    snaps, calls, errors = {}, [0], []

    def cb(ptr, w, h, passes_rendered):
        k = calls[0]; calls[0] += 1
        if k in iterations:
            try:
                snaps[k] = dict(passes_rendered=passes_rendered, moments=g.moment_images(), sampling=g.export_sdtree(0), building=g.export_sdtree(1))
            except Exception as e:      # noqa: BLE001 - an exception cannot cross the C callback; reported below
                errors.append(repr(e))
    g.set_film_callback(cb)
    _, st = g.render()
    try:        # the emitter-level op runs only for scenes that take the full-feature (FULL) instantiations of the bounce kernel
        g.op_emitter_sample_direct(np.full((1, 3), 200.0, np.float32), np.zeros((1, 3), np.float32), np.full((1, 2), 0.5, np.float32))
        st["full_feature"] = True
    except RuntimeError as e:
        assert getattr(e, "code", None) == -6, e
        st["full_feature"] = False
    g.close()
    assert not errors, errors
    assert calls[0] == 3 and [i["passes"] for i in st["iterations"]] == [1, 2, 4], (calls[0], [i["passes"] for i in st["iterations"]])
    return snaps, st


def _leaf_ranges(e):
    leaves = np.nonzero(e["s_children"][:, 0] == 0)[0]
    return leaves, e["tree_first"][leaves].astype(np.int64), e["tree_count"][leaves].astype(np.int64)


def _check_images(gpu, ora, what):
    (gs, _), (os_, _) = gpu, ora
    assert np.array_equal(gs[..., 3], os_[..., 3]), what
    close = np.isclose(gs[..., :3], os_[..., :3], rtol=1e-3, atol=1e-5).all(axis=2)
    r = relmse(gs[..., :3][close], os_[..., :3][close])
    print(f"{what}: pixels close {close.mean():.6f}, relMSE over them {r:.3e}, overall {relmse(gs[..., :3], os_[..., :3]):.3e}")
    assert close.mean() >= 0.998 and r <= 1e-9, (what, close.mean(), r)


def _check_building(gpu, ora, what, box):
    leaves, first, count = _leaf_ranges(ora)
    wg, wo = gpu["tree_weight"][leaves], ora["tree_weight"][leaves]
    # nearest / stochastic: every record adds 1 or 1/2 to one leaf, exact in float.  The spatial box filter spreads a record over the leaves
    # it overlaps by volume: fractional weights, added in a different order (1e-5, as for the commit kernel in test_gpu_sdtree_learning.py)
    same = np.isclose(wg, wo, rtol=1e-5, atol=0) if box else wg == wo
    tot = float(wo.sum())
    assert tot > 0
    # A path whose discrete decision flipped on a libm ulp records its vertices (at most maxDepth = 10, plus as many NEE vertices of weight 1/2)
    # on one side only: a few leaves may differ by that much, none by more
    diff = np.abs(wg.astype(np.float64) - wo)
    assert (~same).sum() <= max(4, 1e-3 * len(leaves)) and (diff <= np.maximum(40.0, 2e-4 * wo)).all(), (what, len(leaves), diff[~same], wo[~same])
    assert abs(float(wg.sum()) - tot) <= max(4.0, 2e-4 * tot), (what, float(wg.sum()), tot)
    worst = 0.0
    for l, f, c in zip(range(len(leaves)), first, count):
        if not same[l]:
            continue
        a, b = gpu["sums"][f:f + c].astype(np.float64), ora["sums"][f:f + c].astype(np.float64)
        scale = max(a.sum(), b.sum())
        if scale > 0:
            worst = max(worst, float(np.abs(a - b).max() / scale))
    print(f"{what}: leaves {len(leaves)}, unequal weights {diff[~same].tolist()} of {wo[~same].tolist()}, total weight {float(wg.sum())} / {tot}, largest sum deviation {worst:.3e} of the leaf total")
    assert worst <= 1e-4, (what, worst)


@pytest.mark.parametrize("config", list(CONFIGS))
def test_guided_passes_match_oracle_on_the_gpu_tree(config):
    name, extra, iterations = CONFIGS[config]
    sc = _scene(name)
    props = dict(dict(sc.integrator, **BASE), **extra)
    snaps, st = _render_with_snapshots(sc, props, iterations)
    assert st["full_feature"] == (name not in ("cbox", "sphere"))
    if name in ("sphere", "rough-metal-sphere"):
        # HBM scenes (> 64 triangles: BVH walk) whose passes of 128^2 x 4 = 65 536 paths reach trace_kernel (from 32 768 paths); with a
        # full-feature scene the trace pass also bins the paths by material and the bounce kernel shades them in bin order (ensure_wavefront)
        assert len(sc.indices) > 64 and 128 * 128 * 4 >= 32768
    p = O.params_from_xml(props)
    for k in iterations:
        s = snaps[k]
        n = st["iterations"][k]["passes"]
        final = bool(st["iterations"][k]["is_final"])
        assert final == (k == 2)
        o = O.Oracle(p, sc, kind="port")
        assert o.import_tree(s["sampling"], iter=k, passes_rendered=s["passes_rendered"] - n) == 0
        e = o.export(0)
        for key in ("s_children", "tree_first", "tree_count", "tree_depth", "tree_sum", "tree_weight", "sums", "children", "adam"):
            assert np.array_equal(e[key], s["sampling"][key]), key
        assert np.array_equal(e["aabb"], s["sampling"]["aabb"])             # the same cubified S-tree box
        leaves = e["s_is_leaf"] == 1
        assert leaves.sum() > 1                                               # a refined S-tree
        if p.bsdf_sampling_fraction_loss != 0:
            theta = e["adam"][leaves, 3]
            print(f"{config} iteration {k}: theta in [{theta.min():.4f}, {theta.max():.4f}]")
            assert np.abs(theta).max() > 0.05                                 # the learned fractions differ from 1/2
        o.reset(20, p.d_tree_threshold)
        if not final:
            reset = o.export(1)                                               # the GPU's building topology is the oracle's reset of the imported tree
            for key in ("s_children", "tree_first", "tree_count", "tree_depth", "children"):
                assert np.array_equal(reset[key], s["building"][key]), key
        o.step_passes(n, is_final=final)
        _check_images(s["moments"], o.moment_images(), f"{config} iteration {k}")
        if not final:
            _check_building(s["building"], o.export(1), f"{config} iteration {k}", box=p.spatial_filter == 2)
        o.close()

