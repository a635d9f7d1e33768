"""GPU parity tests: the CUDA path (through the C ABI of libppg_b200.so) against the CPU oracle on the same
seeded inputs.  Tolerances are stated per test.  Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

import oracle_lib as O
from common import assert_render_parity, load_cbox, relmse

pytestmark = pytest.mark.gpu


def _gpu(props, scene):
    from ppg_b200.integrator import GuidedPathTracer
    g = GuidedPathTracer(props)
    g.set_scene(scene)
    return g


def test_unguided_single_pass_matches_oracle_per_pixel():
    """budget = sppPerPass -> one final, unguided iteration; both sides use the same PCG32 streams, so the
    per-pixel sums agree up to libm ulps (a few paths may flip a discrete decision).
    Tolerance: >= 99.5 % of pixels within 1e-3 relative (+1e-4 abs); image mean within 1e-3 relative."""
    sc = load_cbox(128)
    props = dict(sc.integrator, budget="4")
    g = _gpu(props, sc)
    img, st = g.render()
    o = O.Oracle(O.params_from_xml(props), sc, kind="port")
    ref, ost = o.render()
    assert st["total_paths"] == ost["total_paths"] == 128 * 128 * 4
    assert abs(st["total_vertices"] - ost["total_vertices"]) <= 2e-4 * ost["total_vertices"]
    close = np.isclose(img, ref, rtol=1e-3, atol=1e-4).all(axis=2)
    assert close.mean() >= 0.995, close.mean()
    assert abs(img.mean() - ref.mean()) <= 1e-3 * ref.mean()


def test_iteration_statistics_match_oracle():
    """CBOX 256^2, sppPerPass 4, budget 28 spp (passes 1+2+4), maxDepth 4 -- BASELINE.json configs[0].
    Iteration 0 is unguided: same paths on both sides, so the recorded statistical weight agrees to 1e-4 and the
    D-tree topology (85 nodes, depth 4) exactly.  Later iterations diverge through float-atomic ordering, so they are
    compared statistically (weight 1 %, variance 10 %)."""
    sc = load_cbox(256)
    props = dict(sc.integrator, budget="28", maxDepth="4", rrDepth="10")
    g = _gpu(props, sc)
    img, st = g.render()
    o = O.Oracle(O.params_from_xml(props), sc, kind="port")
    ref, ost = o.render()
    assert st["n_iterations"] == ost["n_iterations"] == 3
    gi, oi = st["iterations"], ost["iterations"]
    assert [i["passes"] for i in gi] == [i["passes"] for i in oi] == [1, 2, 4]
    assert gi[0]["nodes_min"] == gi[0]["nodes_max"] == 85 and gi[0]["depth_max"] == 4
    assert abs(gi[0]["weight_avg"] - oi[0]["weight_avg"]) <= 1e-4 * oi[0]["weight_avg"]
    assert abs(gi[0]["mean_radiance_avg"] - oi[0]["mean_radiance_avg"]) <= 2e-3 * oi[0]["mean_radiance_avg"]
    assert abs(gi[0]["variance"] - oi[0]["variance"]) <= 1e-3 * oi[0]["variance"]
    assert gi[1]["s_tree_leaves"] == oi[1]["s_tree_leaves"]
    for k in (1, 2):
        assert abs(gi[k]["weight_avg"] * gi[k]["s_tree_leaves"] - oi[k]["weight_avg"] * oi[k]["s_tree_leaves"]) <= 0.01 * oi[k]["weight_avg"] * oi[k]["s_tree_leaves"]
        assert abs(gi[k]["variance"] - oi[k]["variance"]) <= 0.10 * oi[k]["variance"]
    assert abs(img.mean() - ref.mean()) <= 0.02 * ref.mean()


def test_known_answers_of_the_reference_log():
    """The authors' render log embedded in scenes/cbox/cbox.exr pins iteration 0 of CBOX 512^2 / 4 spp per pass:
    one D-tree of 85 nodes, stat. weight 4 349 763, mean radiance 0.135707 (tests/golden/cbox_log_stats.json).
    Seeded Monte Carlo: weight within 0.3 %, mean radiance within 3 %, Var within 4 % (spread measured over oracle seeds)."""
    import json, os
    from common import ROOT
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "cbox_log_stats.json")))["cbox"]["iterations"]
    sc = load_cbox(512)
    props = dict(sc.integrator, budget="12")        # passes 1 + 2 (final)
    g = _gpu(props, sc)
    _, st = g.render()
    it0 = st["iterations"][0]
    assert it0["nodes_min"] == it0["nodes_max"] == int(gold[0]["node_count"][0]) == 85
    assert abs(it0["weight_avg"] - gold[0]["stat_weight"][1]) <= 0.003 * gold[0]["stat_weight"][1]
    assert abs(it0["mean_radiance_avg"] - gold[0]["mean_radiance"][1]) <= 0.03 * gold[0]["mean_radiance"][1]
    assert abs(it0["variance"] - gold[0]["var"]) <= 0.04 * gold[0]["var"]
    assert st["iterations"][1]["s_tree_leaves"] == 512    # 4.35 M / 2^9 < 12000: uniform refinement to 512 leaves


def test_full_render_equal_spp_relmse_vs_oracle():
    """Equal-spp image parity (BASELINE north_star: relMSE within 5 % of the reference algorithm's image):
    both the CUDA render and the oracle render of CBOX 128^2 at 252 spp are compared with a converged 4032-spp-equivalent
    reference built from oracle renders with other seeds; the two relMSEs must agree within 15 % (MC noise of the relMSE
    itself at this size; the 5 % claim is made at bench size in bench.py)."""
    sc = load_cbox(128)
    props = dict(sc.integrator, budget="252")
    refs = []
    for seed in range(8):
        o = O.Oracle(O.params_from_xml(props, seed=100 + seed), sc, kind="port")
        refs.append(o.render()[0]); o.close()
    ref = np.mean(refs, axis=0)
    o = O.Oracle(O.params_from_xml(props), sc, kind="port")
    oimg, _ = o.render()
    g = _gpu(props, sc)
    gimg, _ = g.render()
    ro, rg = relmse(oimg, ref), relmse(gimg, ref)
    assert abs(rg - ro) <= 0.15 * ro, (rg, ro)


def _trained_oracle():
    sc = load_cbox(128)
    props = dict(sc.integrator, budget="60")
    o = O.Oracle(O.params_from_xml(props), sc, kind="ref" if O.have_ref() else "port")
    o.render()
    return o


def test_op_dtree_pdf_and_sample_match_reference_trees():
    """D-tree pdf / sample kernels on the oracle's trained CBOX trees (verbatim reference SD-tree code when
    oracle/_ref is present).  pdf: relative 2e-6 (top-down product vs the reference's bottom-up product);
    sample: replayed uniforms, direction within 2e-6 absolute."""
    from ppg_b200 import integrator as I
    o = _trained_oracle()
    e = o.export(0)
    leaves = np.nonzero(e["s_is_leaf"])[0].astype(np.uint32)
    rng = np.random.default_rng(7)
    n = 200000
    ql = rng.choice(leaves, n).astype(np.uint32)
    d = rng.normal(size=(n, 3)).astype(np.float32); d /= np.linalg.norm(d, axis=1, keepdims=True)
    first = e["tree_first"].astype(np.uint32)
    ref = o.pdf(ql, d)
    got = I.op_dtree_pdf(e["sums"], e["children"], first, e["tree_sum"], e["tree_weight"], ql, d)
    assert np.allclose(got, ref, rtol=2e-6, atol=1e-12), np.abs(got - ref).max()
    rnd = rng.random((n, 24), dtype=np.float32)
    refd = o.sample(ql, rnd)
    gotd = I.op_dtree_sample(e["sums"], e["children"], first, e["tree_sum"], e["tree_weight"], ql, rnd)
    assert np.abs(gotd - refd).max() <= 2e-6


def test_op_stree_lookup_bit_exact():
    """S-tree descent: leaf index and voxel size are integer / power-of-two work -> bit exact."""
    from ppg_b200 import integrator as I
    o = _trained_oracle()
    e = o.export(0)
    rng = np.random.default_rng(3)
    mn, mx = e["aabb"]
    pts = (mn + rng.random((100000, 3)) * (mx - mn)).astype(np.float32)
    leaf, size = o.lookup(pts)
    gl, gs = I.op_stree_lookup(e["s_children"], mn, mx - mn, pts)
    assert np.array_equal(gl, leaf)
    assert np.array_equal(gs, size)


@pytest.mark.parametrize("dfilter", [0, 1])
def test_op_dtree_record_matches_reference(dfilter):
    """Splat kernels (nearest and box directional filter) into the building trees: atomics reorder the float
    adds, so sums agree to 1e-5 relative of the per-tree total; statistical weights are integers -> exact."""
    from ppg_b200 import integrator as I
    o = _trained_oracle()
    o.refine(2000); o.reset(20, 0.01)
    e = o.export(1)
    leaves = np.nonzero(e["s_is_leaf"])[0].astype(np.uint32)
    rng = np.random.default_rng(11)
    n = 100000
    mn, mx = e["aabb"]
    # positions inside the cornell box proper so that many leaves are hit
    pos = (np.array([0, 0, 0]) + rng.random((n, 3)) * np.array([556, 548.8, 559.2])).astype(np.float32)
    d = rng.normal(size=(n, 3)).astype(np.float32); d /= np.linalg.norm(d, axis=1, keepdims=True)
    rad = rng.lognormal(0, 1, n).astype(np.float32); pdf = (0.05 + rng.random(n)).astype(np.float32); w = np.ones(n, np.float32)
    leaf, _ = o.lookup(pos)
    sums, tw = I.op_dtree_record(e["sums"], e["children"], e["tree_first"].astype(np.uint32), e["tree_weight"], leaf, d, rad, pdf, w, dfilter)
    o.record(pos, d, rad, pdf, weight=w, dfilter=dfilter)
    e2 = o.export(1)
    assert np.array_equal(tw, e2["tree_weight"])
    scale = np.abs(e2["sums"]).sum() / max(1, len(leaves))
    assert np.abs(sums - e2["sums"]).max() <= 1e-5 * scale + 1e-3 * np.abs(e2["sums"]).max() * 1e-3


@pytest.mark.parametrize("extra", [dict(directionalFilter="box"), dict(spatialFilter="stochastic"), dict(spatialFilter="box"), dict(sampleCombination="inversevar"),
                                   dict(sppPerPass="1"), dict(sTreeThreshold="4000"), dict(nee="kickstart"), dict(nee="always"),
                                   dict(nee="kickstart", spatialFilter="stochastic", directionalFilter="box", budget="300")])
def test_each_improvement_matches_oracle_image(extra):
    """Every non-learning option (filters, inverse-variance combination, sppPerPass, sTreeThreshold, light sampling) follows the same paths as
    the oracle (same PCG32 streams, IEEE arithmetic without FMA contraction): see common.assert_render_parity for the claim (typically the
    images agree to relMSE 1e-13 .. 1e-7 through all training iterations)."""
    sc = load_cbox(128)
    props = dict(dict(sc.integrator, budget="60"), **extra)
    g = _gpu(props, sc); img, st = g.render()
    o = O.Oracle(O.params_from_xml(props), sc, kind="port"); ref, ost = o.render()
    assert_render_parity(img, ref, st, ost, sc, props)
    for a, b in zip(st["iterations"], ost["iterations"]):
        if np.isfinite(b["variance"]):
            assert np.isclose(a["variance"], b["variance"], rtol=2e-2)


@pytest.mark.parametrize("loss", ["kl", "var"])
def test_sampling_fraction_learning_tracks_oracle(loss):
    """bsdfSamplingFractionLoss: the reference learns theta online (one Adam step per ~2 records, under a spin lock, while the pass runs).
    The CUDA path replays each leaf's records sequentially with the same arithmetic after every wavefront, and sizes the wavefronts of a
    learning iteration so that the fractions move by ~0.02 per wavefront (step-size control, perform_render_passes).  Measured against the
    oracle (which learns online like the reference; its own run-to-run spread is ~0.5 - 1 %): recorded vertices of every learning iteration
    within 1.8 % on SPACESHIP, 3.2 % here.  Tolerances: recorded vertex count 4 %, leaf count 5 %, per-iteration variance 10 %."""
    from common import load_fixture_scene
    sc = load_fixture_scene("cbox-improved")          # the reference's own cbox-improved.xml (512^2; inversevar / stochastic / box / kl, threshold 4000, sppPerPass 1)
    props = dict(sc.integrator, budget="15", bsdfSamplingFractionLoss=loss)
    g = _gpu(props, sc); img, st = g.render()
    o = O.Oracle(O.params_from_xml(props), sc, kind="port"); ref, ost = o.render()
    assert st["sub_batches"] > 10 and st["dropped_records"] == 0
    for k in (1, 2, 3):
        a, b = st["iterations"][k], ost["iterations"][k]
        assert abs(a["s_tree_leaves"] - b["s_tree_leaves"]) <= max(2, 0.05 * b["s_tree_leaves"]), (k, a["s_tree_leaves"], b["s_tree_leaves"])
        assert abs(a["variance"] - b["variance"]) <= 0.10 * b["variance"], (k, a["variance"], b["variance"])
        wa, wb = a["weight_avg"] * a["s_tree_leaves"], b["weight_avg"] * b["s_tree_leaves"]
        if wb > 0:
            assert abs(wa - wb) <= 0.04 * wb, (k, wa, wb)
    if loss == "kl":      # ... and the authors' own log of this configuration (tests/golden/cbox_log_stats.json): per-leaf averages 2220.9 / 4557.1 / 5863.9
        import json, os
        from common import ROOT
        gold = json.load(open(os.path.join(ROOT, "tests", "golden", "cbox_log_stats.json")))["cbox-improved"]["iterations"]
        for k in (1, 2):          # (iteration 3 is the final one at this budget: nothing is recorded)
            assert abs(st["iterations"][k]["weight_avg"] - gold[k]["stat_weight"][1]) <= 0.04 * gold[k]["stat_weight"][1], (k, st["iterations"][k]["weight_avg"])
    # learning must have moved the run away from the fixed-fraction one (iteration 1 records more vertices than without a loss)
    g0 = _gpu(dict(props, bsdfSamplingFractionLoss="none"), sc); _, st0 = g0.render()
    assert abs(st["iterations"][2]["weight_avg"] * st["iterations"][2]["s_tree_leaves"] - st0["iterations"][2]["weight_avg"] * st0["iterations"][2]["s_tree_leaves"]) > 0.05 * st0["iterations"][2]["weight_avg"] * st0["iterations"][2]["s_tree_leaves"]


def test_dump_sdtree_wire_format(tmp_path):
    """dumpSDTree (GP:1191-1208, 699-711, 945-951), read back with the layout of the reference's visualizer (visualizer/src/main.cpp:142-173)."""
    import struct
    sc = load_cbox(64)
    g = _gpu(dict(sc.integrator, budget="28", dumpSDTree="true"), sc)
    g.set_destination(str(tmp_path / "cbox"))
    _, st = g.render()
    import os
    assert sorted(os.listdir(tmp_path)) == ["cbox-00.sdt", "cbox-01.sdt"]          # iterations 0 and 1 train, iteration 2 is final (GP:1417)
    for k in (0, 1):
        b = open(str(tmp_path / f"cbox-{k:02d}.sdt"), "rb").read()
        cam = struct.unpack("<16f", b[:64])
        assert np.allclose(np.array(cam).reshape(4, 4), sc.cam_to_world, atol=1e-6)
        p = 64; leaves = 0; total_w = 0; nodes = []
        while p < len(b):
            size = struct.unpack("<3f", b[p + 12:p + 24]); mean, = struct.unpack("<f", b[p + 24:p + 28])
            w, n = struct.unpack("<QQ", b[p + 28:p + 44]); p += 44
            assert w > 0 and 1 <= n <= 65535 and all(s > 0 for s in size) and mean >= 0
            rec = np.frombuffer(b[p:p + 24 * n], dtype=np.dtype([("s", "<f4"), ("c", "<u2")])).reshape(n, 4); p += 24 * n
            assert (rec["c"] < n).all() and (rec["s"] >= 0).all()
            leaves += 1; total_w += w; nodes.append(n)
        assert p == len(b)
        it = st["iterations"][k]
        assert 0 < leaves <= it["s_tree_leaves"]
        assert abs(total_w - it["weight_avg"] * it["s_tree_leaves"]) <= max(leaves, 1e-6 * total_w)     # u64 truncation per leaf
        assert max(nodes) == it["nodes_max"]


@pytest.mark.parametrize("subdiv,smooth", [(2, True), (3, False)])
def test_bvh_path_matches_oracle(subdiv, smooth):
    """Scenes with more than 64 triangles intersect through the BVH walk (the tiny-scene lock-step test is off): CBOX plus a
    tessellated sphere (320 / 1280 triangles, interpolated or face normals).  Hit sets are traversal-order independent
    (ties on t go to the lower triangle index on both sides): a single unguided pass is bit-identical to the oracle, the trained
    render follows it to relMSE <= 1e-5 (measured 3e-13 .. 2e-6: at most one pixel differs)."""
    from common import cbox_with_sphere
    sc = cbox_with_sphere(128, subdiv=subdiv, smooth=smooth)
    props = dict(sc.integrator, budget="60")
    g = _gpu(props, sc); img, st = g.render()
    o = O.Oracle(O.params_from_xml(props), sc, kind="port"); ref, ost = o.render()
    assert st["total_vertices"] > 0 and abs(st["total_vertices"] - ost["total_vertices"]) <= 1e-4 * ost["total_vertices"]
    assert_render_parity(img, ref, st, ost, sc, props)
    for a, b in zip(st["iterations"], ost["iterations"]):
        assert a["s_tree_leaves"] == b["s_tree_leaves"]
        assert np.isclose(a["weight_avg"], b["weight_avg"], rtol=1e-4)


@pytest.mark.parametrize("nee", ["never", "kickstart"])
def test_delta_bsdfs_match_oracle(nee):
    """CBOX with a glass box (dielectric.cpp) and a mirror box (conductor.cpp): delta lobes are sampled with their discrete
    probabilities, are never guided, never recorded and skip NEE (GP:1654, 1942, 1969, 2093).  Same paths as the oracle: relMSE <= 1e-5."""
    from ppg_b200.builtin_scenes import cbox_glass_mirror
    sc = cbox_glass_mirror(load_cbox(128))
    props = dict(sc.integrator, budget="60", nee=nee)
    g = _gpu(props, sc); img, st = g.render()
    o = O.Oracle(O.params_from_xml(props), sc, kind="port"); ref, ost = o.render()
    assert abs(st["total_vertices"] - ost["total_vertices"]) <= 1e-4 * ost["total_vertices"]
    assert_render_parity(img, ref, st, ost, sc, props)
    for a, b in zip(st["iterations"], ost["iterations"]):
        assert a["s_tree_leaves"] == b["s_tree_leaves"] and np.isclose(a["weight_avg"], b["weight_avg"], rtol=1e-4)


def test_torus_standin_scene_matches_oracle():
    """TORUS stand-in (ppg_b200.builtin_scenes.torus_scene: diffuse torus in a glass cube, SDS paths only; the original asset is
    not bundled with the reference): BVH walk + dielectric + guiding.  A single unguided pass is bit-identical to the oracle;
    the trained 63-spp render agrees to relMSE <= 1e-4 and reproduces the oracle's per-iteration statistics."""
    from ppg_b200.builtin_scenes import torus_scene
    sc = torus_scene(128)
    for budget, tol in (("1", 0.0), ("63", 1e-4)):
        props = dict(sc.integrator, budget=budget)
        g = _gpu(props, sc); img, st = g.render()
        o = O.Oracle(O.params_from_xml(props), sc, kind="port"); ref, ost = o.render()
        assert st["total_vertices"] == ost["total_vertices"] or budget != "1"
        assert relmse(img, ref) <= tol, (budget, relmse(img, ref))
    for a, b in zip(st["iterations"], ost["iterations"]):
        assert abs(a["s_tree_leaves"] - b["s_tree_leaves"]) <= 1 and np.isclose(a["weight_avg"] * a["s_tree_leaves"], b["weight_avg"] * b["s_tree_leaves"], rtol=1e-3)


@pytest.mark.parametrize("extra", [dict(), dict(nee="kickstart", bsdfSamplingFractionLoss="none"), dict(spatialFilter="stochastic", directionalFilter="box")])
def test_rough_conductor_matches_oracle(extra):
    """CBOX with GGX and Beckmann rough-conductor boxes (roughconductor.cpp + microfacet.h: D, Smith G1, visible-normal
    sampling, exact conductor Fresnel).  Glossy lobes are ESmooth: guided, recorded and light-sampled like the diffuse ones.
    The device libm (tanf/acosf/atan2f/erf polynomials) differs from glibc by ulps, so a few paths flip: relMSE <= 1e-4,
    per-iteration statistics within 1e-3."""
    from ppg_b200.builtin_scenes import cbox_rough_metal
    sc = cbox_rough_metal(load_cbox(128))
    props = dict(dict(sc.integrator, budget="60"), **extra)
    g = _gpu(props, sc); img, st = g.render()
    o = O.Oracle(O.params_from_xml(props), sc, kind="port"); ref, ost = o.render()
    assert_render_parity(img, ref, st, ost, sc, props)
    assert abs(st["total_vertices"] - ost["total_vertices"]) <= 1e-3 * ost["total_vertices"]
    for a, b in zip(st["iterations"], ost["iterations"]):
        assert abs(a["s_tree_leaves"] - b["s_tree_leaves"]) <= 1
        assert np.isclose(a["weight_avg"] * a["s_tree_leaves"], b["weight_avg"] * b["s_tree_leaves"], rtol=1e-3)
        assert np.isclose(a["variance"], b["variance"], rtol=2e-2)


@pytest.mark.gpu
@pytest.mark.parametrize("extra", [dict(), dict(nee="always"), dict(spatialFilter="stochastic", directionalFilter="box", sampleCombination="inversevar")])
def test_rough_plastic_matches_oracle(extra):
    """CBOX with rough-plastic boxes (roughplastic.cpp: microfacet coat with dielectric Fresnel over a diffuse base attenuated by the
    tabulated rough transmittance, linear and nonlinear variants; Beckmann 0.4 like spaceship.xml's leather and GGX 0.2).
    Same tolerance as the other microfacet model (device libm differs from glibc by ulps)."""
    from common import load_fixture_scene
    sc = load_fixture_scene("cbox-plastic", 128)
    props = dict(dict(sc.integrator, budget="60"), **extra)
    g = _gpu(props, sc); img, st = g.render()
    o = O.Oracle(O.params_from_xml(props), sc, kind="port"); ref, ost = o.render()
    assert_render_parity(img, ref, st, ost, sc, props)
    assert abs(st["total_vertices"] - ost["total_vertices"]) <= 1e-3 * ost["total_vertices"]
    for a, b in zip(st["iterations"], ost["iterations"]):
        assert abs(a["s_tree_leaves"] - b["s_tree_leaves"]) <= 1
        assert np.isclose(a["weight_avg"] * a["s_tree_leaves"], b["weight_avg"] * b["s_tree_leaves"], rtol=1e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("extra", [dict(), dict(nee="always"), dict(bsdfSamplingFractionLoss="none", spatialFilter="box")])
def test_rough_dielectric_matches_oracle(extra):
    """CBOX with rough-glass boxes (roughdielectric.cpp: glossy reflection + glossy transmission, one extra path-sampler draw per
    sample for the lobe choice, eta tracking for Russian roulette)."""
    from ppg_b200.builtin_scenes import cbox_rough_glass
    sc = cbox_rough_glass(load_cbox(128))
    props = dict(dict(sc.integrator, budget="60"), **extra)
    g = _gpu(props, sc); img, st = g.render()
    o = O.Oracle(O.params_from_xml(props), sc, kind="port"); ref, ost = o.render()
    assert_render_parity(img, ref, st, ost, sc, props)
    assert abs(st["total_vertices"] - ost["total_vertices"]) <= 1e-3 * ost["total_vertices"]
    for a, b in zip(st["iterations"], ost["iterations"]):
        assert abs(a["s_tree_leaves"] - b["s_tree_leaves"]) <= 1
        assert np.isclose(a["weight_avg"] * a["s_tree_leaves"], b["weight_avg"] * b["s_tree_leaves"], rtol=1e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("extra", [dict(), dict(nee="always"), dict(nee="kickstart", spatialFilter="stochastic", directionalFilter="box")])
def test_analytic_spheres_match_oracle(extra):
    """CBOX + analytic spheres (sphere.cpp): double-precision ray/sphere quadratic, re-projected hit point, frame from dpdu;
    emitting spheres sampled by uniform cone (reference point outside) and uniform sphere (inside the inward-facing shell)."""
    from ppg_b200.builtin_scenes import cbox_with_analytic_spheres
    sc = cbox_with_analytic_spheres(load_cbox(128))
    props = dict(dict(sc.integrator, budget="60"), **extra)
    g = _gpu(props, sc); img, st = g.render()
    o = O.Oracle(O.params_from_xml(props), sc, kind="port"); ref, ost = o.render()
    assert_render_parity(img, ref, st, ost, sc, props)
    assert abs(st["total_vertices"] - ost["total_vertices"]) <= 1e-3 * ost["total_vertices"]
    for a, b in zip(st["iterations"], ost["iterations"]):
        assert abs(a["s_tree_leaves"] - b["s_tree_leaves"]) <= 1
        assert np.isclose(a["weight_avg"] * a["s_tree_leaves"], b["weight_avg"] * b["s_tree_leaves"], rtol=1e-3)


@pytest.mark.gpu
def test_spaceship_matches_oracle():
    """BASELINE config 4's scene (spaceship-improved.xml: 457 560 triangles through the BVH walk, twosided rough plastics / conductors,
    GGX glass with alpha 0.01, rectangle emitters, the radius-100 emitting shell), at 160x90 and 31 spp.  Deterministic options
    (no sampling-fraction loss, nearest filters) so that the comparison with the multi-threaded oracle is sample by sample."""
    from common import load_fixture_scene
    sc = load_fixture_scene("spaceship-improved").with_film(160, 90)
    props = dict(sc.integrator, budget="31", bsdfSamplingFractionLoss="none", spatialFilter="nearest", directionalFilter="nearest")
    g = _gpu(props, sc); img, st = g.render()
    o = O.Oracle(O.params_from_xml(props), sc, kind="port"); ref, ost = o.render()
    assert np.isfinite(img).all()
    # trained render: an S-tree split or a quadtree subdivision that sits on its threshold flips with the last ulp of an atomic float sum, and the
    # region it covers then decorrelates to noise level (leaf counts differ by up to 2 here): a majority of identical pixels is the robust claim
    assert_render_parity(img, ref, st, ost, sc, props, counts=2e-3, leaves=2, pixels=0.6)
    assert abs(st["total_vertices"] - ost["total_vertices"]) <= 2e-3 * ost["total_vertices"]
    for a, b in zip(st["iterations"], ost["iterations"]):
        assert abs(a["s_tree_leaves"] - b["s_tree_leaves"]) <= 2
        assert np.isclose(a["weight_avg"] * a["s_tree_leaves"], b["weight_avg"] * b["s_tree_leaves"], rtol=2e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["spaceship-improved", "kitchen-improved"])
def test_trace_pass_finds_the_same_hits(name, monkeypatch):
    """Large wavefronts of BVH scenes find their nearest hits in a separate pass of persistent warps that refill idle lanes
    (csrc/ppg_trace.cu) instead of inside the fused bounce kernel.  Same rays, same tests, same tie rule: the unguided render must be
    the SAME image bit for bit whichever kernel finds the hits, and a trained render must agree like two runs of one configuration
    (PPG_TRACE_MIN_PATHS: 0 = pass off, 1 = pass on for every wavefront; the default engages it from 32 768 paths)."""
    from common import load_fixture_scene
    sc = load_fixture_scene(name).with_film(160, 90)
    base = dict(sc.integrator, sampleCombination="automatic", bsdfSamplingFractionLoss="none", spatialFilter="nearest", directionalFilter="nearest")
    out = {}
    for mode in ("0", "1"):
        monkeypatch.setenv("PPG_TRACE_MIN_PATHS", mode)
        out[mode, 1] = _gpu(dict(base, budget="1"), sc).render()
        out[mode, 15] = _gpu(dict(base, budget="15"), sc).render()
    (img0, st0), (img1, st1) = out["0", 1], out["1", 1]
    assert st0["total_vertices"] == st1["total_vertices"]
    assert st1["kernel_launches"] > st0["kernel_launches"]          # the pass really ran
    assert np.array_equal(img0, img1)
    (img0, st0), (img1, st1) = out["0", 15], out["1", 15]
    assert_render_parity(img1, img0, st1, st0, counts=2e-3, leaves=2, pixels=0.6)


@pytest.mark.gpu
def test_spaceship_improved_settings_statistics():
    """Same scene with the XML's own settings (inversevar / stochastic / box / kl): the Adam replay order differs from the
    multi-threaded oracle's, so the comparison is statistical -- image mean, per-iteration tree statistics."""
    from common import load_fixture_scene
    sc = load_fixture_scene("spaceship-improved").with_film(160, 90)
    props = dict(sc.integrator, budget="63")
    g = _gpu(props, sc); img, st = g.render()
    o = O.Oracle(O.params_from_xml(props), sc, kind="port"); ref, ost = o.render()
    assert np.isfinite(img).all()
    assert abs(img.mean() - ref.mean()) <= 0.03 * ref.mean(), (img.mean(), ref.mean())
    assert abs(st["total_vertices"] - ost["total_vertices"]) <= 0.02 * ost["total_vertices"]
    for a, b in list(zip(st["iterations"], ost["iterations"]))[:-1]:
        assert abs(a["s_tree_leaves"] - b["s_tree_leaves"]) <= max(4, 0.15 * b["s_tree_leaves"])   # splits near the threshold flip


@pytest.mark.parametrize("extra", [dict(), dict(nee="always"), dict(bsdfSamplingFractionLoss="none", bsdfSamplingFraction="0.3")])
def test_smooth_plastic_matches_oracle(extra):
    """CBOX with smooth-plastic boxes and floor (plastic.cpp): a delta coat reflection mixed with a diffuse base.  A guided vertex
    whose BSDF sample lands on the delta lobe returns early with woPdf = bsdfPdf * fraction and weight / fraction (GP:1670-1676)."""
    from ppg_b200.builtin_scenes import cbox_smooth_plastic
    sc = cbox_smooth_plastic(load_cbox(128))
    props = dict(dict(sc.integrator, budget="60"), **extra)
    g = _gpu(props, sc); img, st = g.render()
    o = O.Oracle(O.params_from_xml(props), sc, kind="port"); ref, ost = o.render()
    assert_render_parity(img, ref, st, ost, sc, props)
    assert abs(st["total_vertices"] - ost["total_vertices"]) <= 1e-4 * ost["total_vertices"]
    for a, b in zip(st["iterations"], ost["iterations"]):
        assert abs(a["s_tree_leaves"] - b["s_tree_leaves"]) <= 1
        assert np.isclose(a["weight_avg"] * a["s_tree_leaves"], b["weight_avg"] * b["s_tree_leaves"], rtol=1e-4)


@pytest.mark.parametrize("extra", [dict(), dict(nee="always"), dict(hideEmitters="true", nee="kickstart"), dict(maxDepth="4", nee="always")])
def test_thin_dielectric_null_transitions_match_oracle(extra):
    """CBOX with thin-dielectric panes (thindielectric.cpp): index-matched (ENull) transitions.  Covers the null branch of Li
    (GP:2044-2075: no roulette, `scattered` unchanged, emitted radiance only while unscattered), the emitter lookup THROUGH null
    surfaces (rayIntersectAndLookForEmitter GP:2184-2245, incl. its last-segment distance quirk in the MIS pdf) and the attenuated
    shadow rays of light sampling (Scene::evalTransmittance scene.cpp:619-679) with their interaction budget (maxDepth 4)."""
    from ppg_b200.builtin_scenes import cbox_thin_glass
    sc = cbox_thin_glass(load_cbox(128))
    props = dict(dict(sc.integrator, budget="60"), **extra)
    g = _gpu(props, sc); img, st = g.render()
    o = O.Oracle(O.params_from_xml(props), sc, kind="port"); ref, ost = o.render()
    assert_render_parity(img, ref, st, ost, sc, props)
    assert abs(st["total_vertices"] - ost["total_vertices"]) <= 1e-4 * ost["total_vertices"]
    for a, b in zip(st["iterations"], ost["iterations"]):
        assert abs(a["s_tree_leaves"] - b["s_tree_leaves"]) <= 1
        assert np.isclose(a["weight_avg"] * a["s_tree_leaves"], b["weight_avg"] * b["s_tree_leaves"], rtol=1e-4)


@pytest.mark.parametrize("extra", [dict(), dict(nee="always"), dict(nee="kickstart", spatialFilter="box")])
def test_mask_smooth_null_hybrid_matches_oracle(extra):
    """CBOX with `mask` panes (mask.cpp, kitchen.xml's "Blinds"): nested diffuse lobe scaled by the opacity, else a null transition;
    guided vertices can return the null sample (delta early-out of sampleMat), light sampling and the emitter lookup see 1 - opacity."""
    from ppg_b200.builtin_scenes import cbox_blinds
    sc = cbox_blinds(load_cbox(128))
    props = dict(dict(sc.integrator, budget="60"), **extra)
    g = _gpu(props, sc); img, st = g.render()
    o = O.Oracle(O.params_from_xml(props), sc, kind="port"); ref, ost = o.render()
    assert_render_parity(img, ref, st, ost, sc, props)
    assert abs(st["total_vertices"] - ost["total_vertices"]) <= 1e-4 * ost["total_vertices"]
    for a, b in zip(st["iterations"], ost["iterations"]):
        assert abs(a["s_tree_leaves"] - b["s_tree_leaves"]) <= 1
        assert np.isclose(a["weight_avg"] * a["s_tree_leaves"], b["weight_avg"] * b["s_tree_leaves"], rtol=1e-4)


def test_mask_null_transitions_feed_the_sampling_fraction_optimiser():
    """With a loss, null transitions of a smooth/null hybrid are recorded as delta vertices (GP:2049-2066).  Adam replay order differs
    from the multi-threaded oracle's, so the check is statistical: image mean, vertex count and per-iteration variance track the oracle."""
    from ppg_b200.builtin_scenes import cbox_blinds
    sc = cbox_blinds(load_cbox(128))
    props = dict(sc.integrator, budget="124", bsdfSamplingFractionLoss="kl")
    g = _gpu(props, sc); img, st = g.render()
    o = O.Oracle(O.params_from_xml(props), sc, kind="port"); ref, ost = o.render()
    assert abs(img.mean() - ref.mean()) <= 0.02 * ref.mean(), (img.mean(), ref.mean())
    assert abs(st["total_vertices"] - ost["total_vertices"]) <= 0.025 * ost["total_vertices"]      # measured +1.2 % (step-size control of the fractions)
    for k in (2, 3, 4):
        a, b = st["iterations"][k], ost["iterations"][k]
        assert abs(a["variance"] - b["variance"]) <= 0.15 * b["variance"], (k, a["variance"], b["variance"])


def test_spaceship_known_answers_of_the_reference_log():
    """The CUDA path against the authors' own render log of spaceship-improved.xml (640x360, embedded in spaceship-improved.exr;
    tests/golden/spaceship_log_stats.json): the same known answers as the oracle's pin (tests/test_oracle_golden.py).  Measured with the
    step-size control of the sampling fractions: recorded vertices of iterations 1-3 +3.4 / +2.9 / +3.2 % against the log (the oracle itself:
    +2.6 / +2.5 / +1.3 %), leaf counts 480 / 803 (log: 480 / 802), variances within 4 %.  Tolerances: totals and per-leaf averages 5 %, leaf
    counts 5 %, the heavy-tailed variance estimate of 2-8 samples per pixel 15 % (plus one clamped firefly pixel, see below)."""
    import json, os
    from common import ROOT, load_fixture_scene
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "spaceship_log_stats.json")))["spaceship-improved"]["iterations"]
    sc = load_fixture_scene("spaceship-improved")
    g = _gpu(dict(sc.integrator, budget="31"), sc); img, st = g.render()
    it = st["iterations"]
    assert np.isfinite(img).all() and [i["passes"] for i in it] == [1, 2, 4, 8, 16]
    assert it[0]["nodes_min"] == it[0]["nodes_max"] == 85 and it[0]["depth_max"] == 4
    assert abs(it[0]["weight_avg"] - gold[0]["stat_weight"][1]) <= 0.006 * gold[0]["stat_weight"][1]
    assert abs(it[0]["mean_radiance_avg"] - gold[0]["mean_radiance"][1]) <= 0.02 * gold[0]["mean_radiance"][1]
    report = [(k, it[k]["variance"], gold[k]["var"], it[k]["weight_avg"], gold[k]["stat_weight"][1], it[k]["nodes_avg"], it[k]["depth_avg"], it[k]["s_tree_leaves"]) for k in (1, 2, 3)]
    for k in (1, 2, 3):
        # The estimate sums min(luminance variance, 1e4) over the pixels (GP:1298-1319): ONE firefly pixel that reaches the clamp adds
        # 1e4 / (W H (N - 1)) = 0.043 / 0.014 / 0.006 at N = 2 / 4 / 8 samples, 44 % of the logged value of iteration 1.  Eight seeds
        # gave 0.091 - 0.106 against the log's 0.0976; a run with such a pixel gave 0.123.  Hence 15 % plus one clamped pixel.
        firefly = 1e4 / (640 * 360 * (it[k]["passes"] - 1))
        assert -0.15 * gold[k]["var"] <= it[k]["variance"] - gold[k]["var"] <= 0.15 * gold[k]["var"] + firefly, report
        assert abs(it[k]["weight_avg"] - gold[k]["stat_weight"][1]) <= 0.06 * gold[k]["stat_weight"][1], report
        assert abs(it[k]["nodes_avg"] - gold[k]["node_count"][1]) <= 6 and abs(it[k]["depth_avg"] - gold[k]["depth"][1]) <= 0.3, report
    assert abs(it[2]["s_tree_leaves"] - 480) <= 24 and abs(it[3]["s_tree_leaves"] - 802) <= 40, report
    # total recorded weight = number of recorded vertices; it depends on the learned fractions through the D-tree samples that fall below
    # the surface and end their path
    total = [it[k]["weight_avg"] * it[k]["s_tree_leaves"] for k in (1, 2, 3)]
    assert abs(total[0] - 2866.964844 * 256) <= 0.05 * 2866.964844 * 256 and abs(total[1] - 3042.777344 * 480) <= 0.05 * 3042.777344 * 480, (total, report)


def test_spaceship_render_matches_the_reference_image():
    """Image-level known answer: the authors' spaceship-improved.exr (640x360, 1023 spp), box-downsampled 4x4 (tests/golden/
    spaceship_improved_160x90.npy), against the CUDA render of the same XML at 255 spp downsampled the same way: channel means within
    2 %, relMSE of the downsampled images (remaining Monte Carlo noise of both) below 0.02."""
    import os
    from common import ROOT, load_fixture_scene
    gold = np.load(os.path.join(ROOT, "tests", "golden", "spaceship_improved_160x90.npy")).astype(np.float64)
    sc = load_fixture_scene("spaceship-improved")
    g = _gpu(dict(sc.integrator, budget="255"), sc); img, st = g.render()
    small = img.astype(np.float64).reshape(90, 4, 160, 4, 3).mean(axis=(1, 3))
    assert np.isfinite(img).all()
    assert np.allclose(small.mean(axis=(0, 1)), gold.mean(axis=(0, 1)), rtol=0.02), (small.mean(axis=(0, 1)), gold.mean(axis=(0, 1)))
    assert relmse(small, gold) <= 0.02, relmse(small, gold)
