"""The sharded render (world > 1) and the image end of performRenderPasses / render, pixel by pixel.

Every rank is a process of sharded_snapshot_worker.py on cuda:0; the library's collectives go through gloo.  In the film callback of every
performRenderPasses (after the passes, before build_sd_tree) each rank saves its moment images, its sampling trees and its building trees,
which then hold only this rank's records.  From these the tests check:
  (a) the partition: whole 32x32 blocks, one owner per pixel for the whole render, block counts within 1 of each other, and exactly
      passes x sppPerPass samples in every owned pixel (also in the sub-batches of a learning iteration);
  (b) iteration 0 (one unguided pass, paths keyed by seed, pass, pixel and sample) against one GPU: summed moments bit for bit, summed
      building trees to the order of the float atomics;
  (c) the exchange: from iteration 1 on every rank holds the same sampling trees, Adam state included, and the first refine gives the
      single-GPU S-tree;
  (d) the guided iterations of every rank against the port oracle rendering on rank 0's tree (test_gpu_guided_passes.py's bar);
  (e) the variance (GP:1298-1319, the getPixel quirk of SURVEY A.6) restated on the summed moments, the discard / inversevar / automatic
      images restated from the iterations' moments;
  (f) learning iterations: the sub-batch slices cover every pixel once per pass, and the merged sampling-fraction optimiser moves as far
      as one optimiser that saw every record;
  (g) a rank that owns no pixels, and (h) the refine capacity of such a rank.
Measured once on one H100 80GB HBM3 (700 W): see the printed lines (-s)."""
import os
import shutil
import socket
import subprocess
import sys
import tempfile
import time

import numpy as np
import pytest

import oracle_lib as O
import sharded_snapshot_worker as SW
from common import ROOT
from test_gpu_guided_passes import _check_building, _check_images, _leaf_ranges

pytestmark = pytest.mark.gpu

WORKER = os.path.join(ROOT, "tests", "sharded_snapshot_worker.py")
SPAWN_TIMEOUT_S = 600
BASE = dict(budget="28", sppPerPass="4", rrDepth="5", sampleCombination="discard")      # passes 1 + 2 + 4 (test_gpu_guided_passes.py)

# (scene, width, height, world, parameters, iterations compared with the oracle) -- each reaches something different
CONFIGS = {
    # staged scene, lean bounce kernel, mixture at a fraction other than 1/2
    "cbox-frac0.3": ("cbox", 128, 128, 2, dict(bsdfSamplingFractionLoss="none", bsdfSamplingFraction="0.3"), (1, 2)),
    # 4 x 4 blocks over 3 ranks (ragged last row and column): uneven shares; NEE slabs; fractional box-filter weights
    "cbox100-nee-box": ("cbox", 100, 100, 3, dict(bsdfSamplingFractionLoss="none", bsdfSamplingFraction="0.3", nee="kickstart", spatialFilter="box",
                                                  directionalFilter="box"), (1, 2)),
    # HBM scene (BVH walk) whose passes per rank still reach trace_kernel
    "sphere-stochastic": ("sphere", 128, 128, 2, dict(bsdfSamplingFractionLoss="none", spatialFilter="stochastic"), (1, 2)),
    # one block, two ranks: rank 1 owns no pixel and joins every collective (a lower sTreeThreshold refines the S-tree of so small a film)
    "cbox32-idle-rank": ("cbox", 32, 32, 2, dict(bsdfSamplingFractionLoss="none", sTreeThreshold="200"), (1, 2)),
    # learned fractions: iteration 1 in sub-batches with an optimiser merge after each; its final iteration guides with the merged theta.
    # (more S-tree leaves than the default threshold gives, so that the per-leaf theta moves of (f) and (g) are a sample)
    "cbox-kl": ("cbox", 128, 128, 2, dict(bsdfSamplingFractionLoss="kl", sTreeThreshold="1000"), (2,)),
    # (the default threshold: one S-tree leaf, whose ~10^4 records move theta far)
    "cbox32-idle-rank-kl": ("cbox", 32, 32, 2, dict(bsdfSamplingFractionLoss="kl"), (2,)),
}
_cache = {}


def _free_port():
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _spawn(name, width, height, world, props):
    """Runs `world` ranks; returns (exit codes, {rank: error text}, {rank: snapshots}).  Every worker is gone when this returns."""
    d = tempfile.mkdtemp(prefix="ppg_sharded_")
    args = [f"{k}={v}" for k, v in props.items()]
    procs = []
    try:
        port = _free_port()
        for r in range(world):
            procs.append(subprocess.Popen([sys.executable, WORKER, str(r), str(world), str(port), d, name, str(width), str(height), *args]))
        deadline = time.monotonic() + SPAWN_TIMEOUT_S
        for p in procs:
            p.wait(timeout=max(1.0, deadline - time.monotonic()))
        codes = [p.returncode for p in procs]
        errs = {r: open(os.path.join(d, f"rank{r}.err")).read() for r in range(world) if os.path.exists(os.path.join(d, f"rank{r}.err"))}
        res = {r: SW.load(os.path.join(d, f"rank{r}.npz")) for r in range(world) if codes[r] == 0}
        return codes, errs, res
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
            p.wait()
        shutil.rmtree(d, ignore_errors=True)


def _props(sc, extra):
    return dict(dict(sc.integrator, **BASE), **extra)


def _sharded(config):
    if ("sharded", config) not in _cache:
        name, w, h, world, extra, _ = CONFIGS[config]
        codes, errs, res = _spawn(name, w, h, world, dict(BASE, **extra))
        assert codes == [0] * world, (codes, errs)
        _cache[("sharded", config)] = [res[r] for r in range(world)]
    return _cache[("sharded", config)]


def _single(config, run=0):
    if ("single", config, run) not in _cache:
        name, w, h, _, extra, _ = CONFIGS[config]
        sc = SW.scene(name, w, h)
        _cache[("single", config, run)] = SW.render_snapshots(sc, _props(sc, extra))
    return _cache[("single", config, run)]


def _calls_passes(r):
    pr = [c["passes_rendered"] for c in r["calls"]]
    return [b - a for a, b in zip([0] + pr[:-1], pr)]


def _summed_moments(rs, k):
    return (np.sum([r["calls"][k]["moments"][0] for r in rs], axis=0, dtype=np.float32),
            np.sum([r["calls"][k]["moments"][1] for r in rs], axis=0, dtype=np.float32))


def _variance_numerator(s1, s2, n):
    """variance_kernel restated (GP:1298-1319 with the getPixel quirk): per pixel in float32 in the kernel's order, summed in float64."""
    A = s1.reshape(-1, 4).astype(np.float32); Q = s2.reshape(-1, 4).astype(np.float32)
    one, N = np.float32(1), np.float32(n)
    with np.errstate(divide="ignore"):
        iw = np.where(A[:, 3] != 0, one / A[:, 3], np.float32(0)).astype(np.float32)
        isw = np.where(Q[:, 3] != 0, one / Q[:, 3], np.float32(0)).astype(np.float32)
    p = A[:, :3] * iw[:, None]
    l = Q[:, :3] * isw[:, None] - p * p / N
    lum = l[:, 0] * np.float32(0.212671) + l[:, 1] * np.float32(0.715160) + l[:, 2] * np.float32(0.072169)
    return float(np.fmin(lum, np.float32(10000.0)).astype(np.float64).sum())


def _check_variances(rs, what, spp):
    """Every iteration's variance is the same on all ranks and equals the restatement on the summed moments of its last call (the final
    iteration of `automatic` makes two calls)."""
    st = rs[0]["stats"]
    H, W = rs[0]["img"].shape[:2]
    for r in rs[1:]:
        assert np.array_equal([i["variance"] for i in r["stats"]["iterations"]], [i["variance"] for i in st["iterations"]], equal_nan=True), what
    passes = _calls_passes(rs[0])
    k = 0
    for it in st["iterations"]:
        n_it = 0
        while n_it < it["passes"]:
            n_it += passes[k]; k += 1
        assert n_it == it["passes"], (what, it["iteration"], passes)
        s1, s2 = _summed_moments(rs, k - 1)
        N = passes[k - 1] * spp
        if N == 1:
            assert np.isnan(it["variance"]), (what, it["variance"])       # N - 1 = 0: the reference divides 0 by 0
            continue
        v = _variance_numerator(s1, s2, N) / (W * H * (N - 1))
        assert np.isclose(it["variance"], v, rtol=1e-6, atol=0), (what, it["iteration"], it["variance"], v)
    assert k == len(rs[0]["calls"]), what


def _owners(rs, k):
    w = np.stack([r["calls"][k]["moments"][0][..., 3] for r in rs])
    return w > 0


# ---------------------------------------------------------------------------------------------------------- (a) partition
@pytest.mark.parametrize("config", list(CONFIGS))
def test_partition_in_whole_blocks_with_every_sample(config):
    name, W, H, world, extra, _ = CONFIGS[config]
    rs = _sharded(config)
    spp = int(BASE["sppPerPass"])
    passes = _calls_passes(rs[0])
    owner0 = None
    for k, n in enumerate(passes):
        own = _owners(rs, k)
        assert (own.sum(axis=0) == 1).all(), (config, k)                      # every pixel owned by exactly one rank
        owner = np.argmax(own, axis=0)
        if owner0 is None:
            owner0 = owner
        assert np.array_equal(owner, owner0), (config, k)                   # ... for the whole render
        for r, res in enumerate(rs):
            s1, s2 = res["calls"][k]["moments"]
            assert (s1[..., 3][own[r]] == n * spp).all() and (s2[..., 3][own[r]] == n * spp).all(), (config, k, r)
            assert not s1[~own[r]].any() and not s2[~own[r]].any(), (config, k, r)   # nothing outside this rank's pixels
    blocks = [[owner0[y:y + 32, x:x + 32] for x in range(0, W, 32)] for y in range(0, H, 32)]
    counts = np.zeros(world, np.int64)
    for row in blocks:
        for b in row:
            assert (b == b.flat[0]).all(), config                           # whole (ragged at the edges) 32x32 blocks
            counts[b.flat[0]] += 1
    shares = [float((owner0 == r).mean()) for r in range(world)]
    print(f"{config}: blocks per rank {counts.tolist()}, pixel shares {[round(s, 4) for s in shares]}")
    assert counts.max() - counts.min() <= 1, (config, counts)
    assert sum(int(r["stats"]["total_paths"]) for r in rs) == W * H * int(BASE["budget"])
    if name == "sphere":
        # BVH scene whose passes reach trace_kernel (from 32 768 paths): 8 blocks x 1024 pixels x 4 spp per rank and pass
        assert counts.tolist() == [8, 8] and 8 * 1024 * spp >= 32768
    if config.startswith("cbox32-idle-rank"):
        assert counts.tolist() == [1, 0]


# ---------------------------------------------------------------------------------------------------------- (b) iteration 0
@pytest.mark.parametrize("config", list(CONFIGS))
def test_iteration0_sums_to_the_single_gpu_render(config):
    extra = CONFIGS[config][4]
    box = extra.get("spatialFilter") == "box"
    rs, one = _sharded(config), _single(config)
    s1, s2 = _summed_moments(rs, 0)
    o1, o2 = one["calls"][0]["moments"]
    assert np.array_equal(s1, o1) and np.array_equal(s2, o2), config
    b = [r["calls"][0]["building"] for r in rs]
    ob = one["calls"][0]["building"]
    for key in ("s_children", "tree_first", "tree_count", "children"):
        for e in b:
            assert np.array_equal(e[key], ob[key]), (config, key)
    wsum = np.sum([e["tree_weight"] for e in b], axis=0, dtype=np.float64)
    leaves, first, count = _leaf_ranges(ob)
    if box:
        # fractional weights: one leaf's float accumulator of ~10^5 of them rounds by ~1e-5 of its total on either side
        dev = float(np.max(np.abs(wsum[leaves] - ob["tree_weight"][leaves]) / ob["tree_weight"][leaves]))
        print(f"{config}: iteration 0 box-filter weights within {dev:.2e} of one GPU's")
        assert dev <= 1e-4, (config, dev)
    else:
        assert np.array_equal(wsum[leaves], ob["tree_weight"][leaves].astype(np.float64)), config
    sums = np.sum([e["sums"].astype(np.float64) for e in b], axis=0)
    worst = 0.0
    for f, c in zip(first, count):
        a, o = sums[f:f + c], ob["sums"][f:f + c].astype(np.float64)
        scale = max(a.sum(), o.sum())
        if scale > 0:
            worst = max(worst, float(np.abs(a - o).max() / scale))
    print(f"{config}: iteration 0 total weight {wsum[leaves].sum()}, largest sum deviation {worst:.2e} of the leaf total")
    assert worst <= 1e-5, (config, worst)


# ---------------------------------------------------------------------------------------------------------- (c) exchange
@pytest.mark.parametrize("config", list(CONFIGS))
def test_ranks_hold_identical_sampling_trees_after_the_exchange(config):
    extra = CONFIGS[config][4]
    rs, one = _sharded(config), _single(config)
    for k in range(1, len(rs[0]["calls"])):
        e0 = rs[0]["calls"][k]["sampling"]
        for r in rs[1:]:
            for key, v in r["calls"][k]["sampling"].items():
                assert np.array_equal(v, e0[key]), (config, k, key)
    for r in rs[1:]:
        for key, v in r["final"].items():
            assert np.array_equal(v, rs[0]["final"][key]), (config, key)
        assert np.array_equal(r["img"], rs[0]["img"]), config
    if extra.get("spatialFilter") != "box":
        # the first refine reads the reduced iteration-0 weights: sums of 1 and 1/2, exact in any order
        assert np.array_equal(rs[0]["calls"][1]["sampling"]["s_children"], one["calls"][1]["sampling"]["s_children"]), config
        assert (rs[0]["calls"][1]["sampling"]["s_children"][:, 0] == 0).sum() > (0 if config == "cbox32-idle-rank-kl" else 1)


# ---------------------------------------------------------------------------------------------------------- (d) guided iterations
@pytest.mark.parametrize("config", list(CONFIGS))
def test_guided_iterations_of_every_rank_match_the_oracle(config):
    name, W, H, world, extra, iterations = CONFIGS[config]
    rs = _sharded(config)
    sc = SW.scene(name, W, H)
    p = O.params_from_xml(_props(sc, extra))
    st = rs[0]["stats"]
    own = _owners(rs, 0)
    for k in iterations:
        n = st["iterations"][k]["passes"]
        final = bool(st["iterations"][k]["is_final"])
        assert final == (k == 2) and len(rs[0]["calls"]) == 3
        s = rs[0]["calls"][k]
        o = O.Oracle(p, sc, kind="port")
        assert o.import_tree(s["sampling"], iter=k, passes_rendered=s["passes_rendered"] - n) == 0
        o.reset(20, p.d_tree_threshold)
        if not final:
            reset = o.export(1)
            for r in rs:
                for key in ("s_children", "tree_first", "tree_count", "tree_depth", "children"):
                    assert np.array_equal(reset[key], r["calls"][k]["building"][key]), (config, k, key)
        o.step_passes(n, is_final=final)
        o1, o2 = o.moment_images()
        for r, res in enumerate(rs):
            if not own[r].any():
                continue
            g1, g2 = res["calls"][k]["moments"]
            m = own[r]
            _check_images((g1[m][:, None], g2[m][:, None]), (o1[m][:, None], o2[m][:, None]), f"{config} iteration {k} rank {r}")
        if not final:
            b = dict(rs[0]["calls"][k]["building"])
            b["tree_weight"] = np.sum([r["calls"][k]["building"]["tree_weight"] for r in rs], axis=0, dtype=np.float32)
            b["sums"] = np.sum([r["calls"][k]["building"]["sums"] for r in rs], axis=0, dtype=np.float32)
            _check_building(b, o.export(1), f"{config} iteration {k} (sum over ranks)", box=p.spatial_filter == 2)
        o.close()


# ---------------------------------------------------------------------------------------------------------- (e) variance and film
@pytest.mark.parametrize("config", list(CONFIGS))
def test_variance_and_discard_image_from_the_summed_moments(config):
    rs, one = _sharded(config), _single(config)
    _check_variances(rs, config, int(BASE["sppPerPass"]))
    _check_variances([one], config + " (one GPU)", int(BASE["sppPerPass"]))
    s1, _ = _summed_moments(rs, len(rs[0]["calls"]) - 1)
    expect = s1[..., :3] * (np.float32(1) / s1[..., 3:4])
    assert np.array_equal(rs[0]["img"], expect), config                    # discard: the final iteration's film, developed


@pytest.mark.parametrize("world", [1, 2])
def test_inversevar_combines_the_last_four_iterations(world):
    """sppPerPass 1, budget 31: iterations of 1, 2, 4, 8, 16 passes, so the ring of four images rotates once.  Iteration 0 has N = 1 and a NaN
    variance (a reference quirk): it has to leave the ring, or the image would be NaN."""
    props = dict(sppPerPass="1", budget="31", sampleCombination="inversevar", bsdfSamplingFractionLoss="none")
    if world == 1:
        sc = SW.scene("cbox", 64, 64)
        rs = [SW.render_snapshots(sc, dict(sc.integrator, **props))]
    else:
        codes, errs, res = _spawn("cbox", 64, 64, 2, props)
        assert codes == [0, 0], (codes, errs)
        rs = [res[0], res[1]]
        assert np.array_equal(rs[0]["img"], rs[1]["img"])
    st = rs[0]["stats"]
    assert [i["passes"] for i in st["iterations"]] == [1, 2, 4, 8, 16]
    _check_variances(rs, f"inversevar world {world}", 1)
    v = [i["variance"] for i in st["iterations"]]
    assert np.isnan(v[0]) and np.isfinite(v[1:]).all()
    num = np.zeros(rs[0]["img"].shape, np.float64)
    for k in range(1, 5):
        s1, _ = _summed_moments(rs, k)
        num += s1[..., :3].astype(np.float64) / s1[..., 3:4].astype(np.float64) / v[k]
    expect = num / sum(1.0 / x for x in v[1:])
    img = rs[0]["img"]
    print(f"inversevar world {world}: variances {v}, largest relative deviation {float(np.max(np.abs(img - expect) / np.maximum(np.abs(expect), 1e-6))):.2e}")
    assert np.isfinite(img).all() and np.allclose(img, expect, rtol=1e-5, atol=1e-7)


def test_automatic_final_iteration_renders_into_one_film():
    """budgetType=seconds with test_gpu_schedule.py's injected clock (0.05 s per pass): iteration 5 becomes final after its 32 passes and renders
    32 more into the same film, so it makes two performRenderPasses calls (two film callbacks).  The image is the film of both calls; the
    iteration reports the second call's variance."""
    sc = SW.scene("cbox", 48, 48)
    props = dict(sc.integrator, budgetType="seconds", budget="4", sampleCombination="automatic")

    def clock(state):
        state["reads"] += 1
        return 0.05 * state["passes"] + 1e-5 * state["reads"]
    r = SW.render_snapshots(sc, props, clock=clock)
    st = r["stats"]
    assert [i["passes"] for i in st["iterations"]] == [1, 2, 4, 8, 16, 64] and st["iterations"][-1]["is_final"]
    assert _calls_passes(r) == [1, 2, 4, 8, 16, 32, 32]
    spp = int(O.params_from_xml(props).spp_per_pass)
    _check_variances([r], "automatic", spp)
    (a1, _), (b1, _) = r["calls"][5]["moments"], r["calls"][6]["moments"]
    film = a1 + b1
    expect = film[..., :3] * (np.float32(1) / film[..., 3:4])
    assert (film[..., 3] == 64 * spp).all()
    print(f"automatic: image equals the two calls' film bit for bit: {np.array_equal(r['img'], expect)}")
    assert np.allclose(r["img"], expect, rtol=1e-6, atol=0)


# ---------------------------------------------------------------------------------------------------------- (f) learning iterations
@pytest.mark.parametrize("config", ["cbox-kl", "cbox32-idle-rank-kl"])
def test_learning_iteration_slices_cover_every_pixel_and_ranks_agree(config):
    rs, one = _sharded(config), _single(config)
    for runs in (rs, [one]):
        st = runs[0]["stats"]
        assert st["sub_batches"] > 0 and st["iterations"][1]["passes"] == 2
        s1, _ = _summed_moments(runs, 1)
        assert (s1[..., 3] == 2 * int(BASE["sppPerPass"])).all(), config   # every pixel sampled once per pass by the sub-batch slices
        assert sum(int(r["stats"]["total_paths"]) for r in runs) == s1.shape[0] * s1.shape[1] * int(BASE["budget"])
    for k in range(len(rs[0]["calls"])):
        for r in rs[1:]:
            assert np.array_equal(r["calls"][k]["sampling"]["adam"], rs[0]["calls"][k]["sampling"]["adam"]), (config, k)


def _theta_moves(r):
    """theta of every S-tree leaf after the learning iteration 1 (it starts at 0 everywhere: the iteration-0 tree learns nothing)."""
    assert not r["calls"][0]["sampling"]["adam"].any()
    e = r["calls"][1]["sampling"]
    return e["s_children"], e["adam"][e["s_children"][:, 0] == 0, 3].astype(np.float64)


def _median_move_ratio(r, ref, what, min_leaves=16):
    """Median over the S-tree leaves of theta(r) / theta(ref) after the learning iteration (same S-tree: the first refine is exact)."""
    c, t = _theta_moves(r)
    cr, tr = _theta_moves(ref)
    assert np.array_equal(c, cr), what
    sel = np.abs(tr) > 0.05
    ratio = float(np.median(t[sel] / tr[sel]))
    print(f"{what}: median per-leaf theta move ratio {ratio:.3f} over {int(sel.sum())} of {len(t)} leaves (|theta| up to {np.abs(tr).max():.3f})")
    assert sel.sum() >= min_leaves, what
    return ratio


def test_merged_optimiser_moves_theta_as_far_as_one_optimiser():
    """Every replica replays only its own records from the common start.  Merged by the sum of their moves, the ranks' theta moves as far as one
    optimiser that saw all records.  Measured once on one H100 80GB HBM3 (700 W): median ratio 1.06 over 28 leaves; 0.47 when the replicas were
    averaged."""
    ratio = _median_move_ratio(_sharded("cbox-kl")[0], _single("cbox-kl"), "cbox-kl world 2 / world 1")
    assert 0.75 <= ratio <= 1.35, ratio


# ---------------------------------------------------------------------------------------------------------- (g) an idle rank
def test_idle_rank_leaves_the_learned_fractions_of_the_single_gpu_render():
    """CBOX 32x32 is one block: with two ranks rank 0 renders everything and rank 1 nothing, so the merged optimiser has to end where a single
    GPU's does; averaging with the idle replica halves every move.  The learning iteration is not reproducible from run to run (records reach the
    replay in atomic order and the sub-batch sizes follow the fractions' movement).  Measured on one H100 80GB HBM3 (700 W), theta of the one leaf
    ~0.9: two single-GPU runs 0.6 % to 21 % apart, the sharded run 10 % from a single-GPU run, the averaging merge 45 % short of it."""
    rs = _sharded("cbox32-idle-rank-kl")
    spread = abs(_median_move_ratio(_single("cbox32-idle-rank-kl", 1), _single("cbox32-idle-rank-kl", 0), "idle rank, kl: one GPU, run 2 / run 1", 1) - 1)
    ratio = _median_move_ratio(rs[0], _single("cbox32-idle-rank-kl", 0), "idle rank, kl: world 2 / world 1", 1)
    assert spread <= 0.35 and abs(ratio - 1) <= 0.3, (spread, ratio)


# ---------------------------------------------------------------------------------------------------------- (h) refine capacity
def test_refine_capacity_is_sized_from_the_records_of_all_ranks():
    """CBOX 64x32 is two blocks over three ranks: rank 2 owns nothing and records nothing.  The first refine (threshold 2 at sTreeThreshold 1 and
    16 spp per pass) meets ~10^5 records and needs more S-tree nodes than the minimum capacity of 65 536, so a rank that sized the capacity from
    its own records would run out of nodes alone.  Every rank sizes it from the records of all ranks and ends with the same tree."""
    props = dict(sTreeThreshold="1", sppPerPass="16", budget="48", bsdfSamplingFractionLoss="none", sampleCombination="discard")
    codes, errs, res = _spawn("cbox", 64, 32, 3, props)
    assert codes == [0, 0, 0], (codes, errs)
    rs = [res[r] for r in range(3)]
    assert not rs[2]["calls"][0]["moments"][0].any() and rs[2]["stats"]["total_paths"] == 0
    st = rs[0]["stats"]
    assert [i["passes"] for i in st["iterations"]] == [1, 2]
    nodes = st["iterations"][1]["s_tree_nodes"]
    print(f"refine capacity: iteration 0 records {[r['stats']['iterations'][0]['recorded_vertices'] for r in rs]}, S-tree nodes after the first refine {nodes}")
    assert nodes > 65536
    for r in rs[1:]:
        assert r["stats"]["iterations"][1]["s_tree_nodes"] == nodes
        for key, v in r["final"].items():
            assert np.array_equal(v, rs[0]["final"][key]), key
