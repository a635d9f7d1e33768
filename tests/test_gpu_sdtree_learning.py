"""The learning half of the SD-tree, one launch at a time: the render's own refine, reset, build, commit and Adam kernels (ppg_op_sdtree_refine_reset,
ppg_op_sdtree_build, ppg_op_commit, ppg_op_adam_replay) on trees the oracle built, against the oracle's restated SD-tree (kind "port") and, where
oracle/_ref was built, the reference's own SD-tree code (kind "ref"; port == ref bit for bit is pinned on the CPU by tests/test_oracle_sdtree.py).

The GPU refine numbers S-tree nodes by rounds (breadth first), the reference depth first: nodes are paired by a depth-first walk of both trees
(child 0 first) and compared along it."""
import numpy as np
import pytest

import oracle_lib as O
from common import CUDA_INC, compile_device_on_host

pytestmark = pytest.mark.gpu
KINDS = ["port"] + (["ref"] if O.have_ref() else [])
BOX = (np.zeros(3, np.float32), np.ones(3, np.float32))


def _I():
    from ppg_b200 import integrator as I
    return I


def _dfs(sch):
    sch = np.asarray(sch)
    order, st = [], [0]
    while st:
        n = st.pop(); order.append(n)
        if sch[n, 0] != 0:
            st.append(int(sch[n, 1])); st.append(int(sch[n, 0]))
    return np.array(order, np.int64)


def _rows(first, count):
    """Pool rows of the trees (first, count), concatenated in the given order."""
    first = np.asarray(first, np.int64); count = np.asarray(count, np.int64)
    starts = np.repeat(first - np.concatenate([[0], np.cumsum(count)[:-1]]), count)
    return starts + np.arange(int(count.sum()))


def _same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def _dirs(rng, n):
    d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    return d.astype(np.float32)


def _record(o, rng, n, pos=None, weight=1.0, loss=1, dfilter=0, d=None):
    pos = rng.beta(2, 3, (n, 3)).astype(np.float32) if pos is None else pos
    o.record(pos, _dirs(rng, n) if d is None else d, rng.lognormal(0, 1, n).astype(np.float32), (0.05 + rng.random(n)).astype(np.float32),
             product=rng.lognormal(0, 1, n).astype(np.float32), bsdf_pdf=rng.random(n).astype(np.float32), dtree_pdf=rng.random(n).astype(np.float32),
             weight=np.broadcast_to(np.float32(weight), (n,)), dfilter=dfilter, loss=loss)


def _sampling_half(o):
    e = o.export(0)
    return e, dict(s_children=e["s_children"], tree_first=e["tree_first"].astype(np.uint32), tree_count=e["tree_count"], tree_depth=e["tree_depth"],
                   tree_sum=e["tree_sum"], tree_weight=e["tree_weight"], adam=e["adam"], sums=e["sums"], children=e["children"])


def _trained(kind, rounds=2, thr=2000, n=20000, half_last=False, dfilter=0, seed=5):
    """reset -> record -> build rounds (the render's iteration), S-tree refined at `thr` before every reset; with half_last the last round records
    only in x < 0.5, so the leaves of the other half keep untrained (total == 0) sampling trees next to trained ones."""
    rng = np.random.default_rng(seed)
    o = O.Oracle(O.default_params(), aabb=BOX, kind=kind)
    for r in range(rounds):
        o.refine(thr); o.reset(20, 0.01)
        pos = rng.beta(2, 3, (n, 3)).astype(np.float32)
        if half_last and r == rounds - 1:
            pos[:, 0] *= 0.5
        _record(o, rng, n, pos=pos, dfilter=dfilter)
        o.build()
    return o, rng


def _refine_reset(o, thr, refine, reset, dthr):
    """GPU op on the oracle's current tree (twice: must be identical), then the oracle's own refine / reset; returns (gpu, sampling export and
    building weights after the refine, building export after the reset, DFS pairs of leaves)."""
    I = _I()
    _, tree = _sampling_half(o)
    bw = o.export(1)["tree_weight"]
    g = I.op_sdtree_refine_reset(tree, bw, thr, refine=refine, reset=reset, dtree_threshold=dthr)
    g2 = I.op_sdtree_refine_reset(tree, bw, thr, refine=refine, reset=reset, dtree_threshold=dthr)
    assert g.keys() == g2.keys() and all(_same(g[k], g2[k]) for k in g), "two launches on the same input differ"
    if refine:
        o.refine(thr)
    r0, bwo = o.export(0), o.export(1)["tree_weight"]
    r1 = None
    if reset:
        o.reset(20, dthr); r1 = o.export(1)
    pg, po = _dfs(g["s_children"]), _dfs(r0["s_children"])
    assert len(g["s_children"]) == len(r0["s_children"]) == len(pg) == len(po)
    lg, lo = g["s_children"][pg, 0] == 0, r0["s_children"][po, 0] == 0
    assert np.array_equal(lg, lo), "S-tree topology differs"
    lg, lo = pg[lg], po[lo]
    assert _same(g["building_weight"][lg], bwo[lo])
    for k in ("tree_sum", "tree_weight", "tree_depth", "tree_count", "adam"):
        assert _same(g[k][lg], r0[k][lo]), k
    # the inherited sampling trees themselves: the GPU children point at their ancestor's tree in the input pool
    assert _same(tree["sums"][_rows(g["tree_first"][lg], g["tree_count"][lg])], r0["sums"][_rows(r0["tree_first"][lo], r0["tree_count"][lo])])
    assert _same(tree["children"][_rows(g["tree_first"][lg], g["tree_count"][lg])], r0["children"][_rows(r0["tree_first"][lo], r0["tree_count"][lo])])
    if reset:
        assert _same(g["build_count"][lg], r1["tree_count"][lo]) and _same(g["build_depth"][lg], r1["tree_depth"][lo])
        rows_g, rows_o = _rows(g["build_first"][lg], g["build_count"][lg]), _rows(r1["tree_first"][lo], r1["tree_count"][lo])
        assert _same(g["build_children"][rows_g], r1["children"][rows_o])
        assert not g["build_sums"].any() and not r1["sums"][rows_o].any() and int(g["build_count"].sum()) == len(g["build_sums"])
    return g, r0, r1, lg, lo


@pytest.mark.parametrize("kind", KINDS)
def test_refine_with_a_frontier_of_many_chunks(kind):
    """~4e6 of building weight at threshold 200 over a trained S-tree: > 2e4 leaves, refine rounds whose frontier spans many 1024-node chunks of the
    block scan.  Bit-exact: topology, halved building weights, inherited sampling sum / weight / depth / count, sampling trees and Adam state; then the
    reset of every new leaf (dTreeThreshold 0.01): per-leaf building topology, node counts and depths, zeroed sums."""
    o, rng = _trained(kind)
    _record(o, rng, 40000, pos=rng.random((40000, 3)).astype(np.float32), weight=100.0)
    g, _, _, lg, _ = _refine_reset(o, 200, True, True, 0.01)
    assert len(lg) >= 20000, len(lg)


@pytest.mark.parametrize("kind", KINDS)
def test_refine_edges(kind):
    """Eight leaves; one holds 2^5 * thr * (1 + 2^-10) and splits on six levels in one call, one holds exactly thr (no split: the test is `>`), one
    thr - 1.  Then a refine with nothing to split.  Bit-exact as above.  A node capacity too small for the refine is reported, not ignored."""
    I = _I()
    rng = np.random.default_rng(9)
    o = O.Oracle(O.default_params(), aabb=BOX, kind=kind)
    o.reset(20, 0.01); _record(o, rng, 1, pos=np.full((1, 3), 0.5, np.float32), weight=8000.0); o.build()
    o.refine(1000); o.reset(20, 0.01)
    _record(o, rng, 4000, pos=rng.random((4000, 3)).astype(np.float32), weight=0.25)      # sampling trees and Adam states per leaf
    o.build(); o.reset(20, 0.01)
    centers = np.array([[0.25 + 0.5 * (k & 1), 0.25 + 0.5 * ((k >> 1) & 1), 0.25 + 0.5 * (k >> 2)] for k in range(8)], np.float32)
    for c, w in zip(centers[:3], (32000.0 * (1 + 2.0 ** -10), 1000.0, 999.0)):
        _record(o, rng, 1, pos=c[None], weight=w)
    _, tree = _sampling_half(o)
    with pytest.raises(I.PpgError) as e:
        I.op_sdtree_refine_reset(tree, o.export(1)["tree_weight"], 1000, reset=False, node_capacity=len(tree["s_children"]) + 8)
    assert e.value.code == -3
    g, _, _, lg, _ = _refine_reset(o, 1000, True, False, 0.01)
    assert len(lg) == 7 + 64
    n0 = len(g["s_children"])
    g, _, _, _, _ = _refine_reset(o, 1000, True, True, 0.01)
    assert len(g["s_children"]) == n0


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("dthr", [0.0625, 1e-5])
def test_reset_trained_and_untrained_leaves(kind, dthr):
    """DTree::reset of trained leaves next to untrained ones (total == 0: the fraction is 0.25^depth).  dTreeThreshold 0.0625 == 0.25^2: an untrained
    leaf stops at depth 2 (the test is `>`).  1e-5: untrained leaves would reach depth 9 (87 381 nodes) and stop at the 65 535-node cap with 65 536 nodes.
    Bit-exact: children arrays, node counts, depths, zeroed sums."""
    o, _ = _trained(kind, rounds=2, half_last=True)
    _, _, r1, _, lo = _refine_reset(o, 1 << 30, False, True, dthr)
    e0 = o.export(0)
    assert (e0["tree_sum"][lo] == 0).any() and (e0["tree_sum"][lo] > 0).any()
    if dthr == 0.0625:
        assert (r1["tree_count"][lo] == 5).any()
    else:
        assert (r1["tree_count"][lo] == 65536).any()


@pytest.mark.parametrize("kind", KINDS)
def test_reset_reaches_the_depth_cap(kind):
    """Records concentrated on one direction over seven reset / record / build rounds: every reset deepens the tree around it until depth 20.  Bit-exact."""
    rng = np.random.default_rng(4)
    o = O.Oracle(O.default_params(), aabb=BOX, kind=kind)
    d = np.tile(np.array([[0.3, 0.4, 0.866]], np.float32) / np.float32(np.linalg.norm([0.3, 0.4, 0.866])), (2000, 1))
    for _ in range(7):
        o.reset(20, 0.01); _record(o, rng, 2000, pos=np.full((2000, 3), 0.5, np.float32), d=d); o.build()
    g, _, r1, lg, lo = _refine_reset(o, 1 << 30, False, True, 0.01)
    assert r1["tree_depth"][lo].max() == g["build_depth"][lg].max() == 20


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("dfilter", [0, 1])
def test_build_and_tree_statistics(kind, dfilter):
    """DTree::build of building trees the oracle recorded (nearest and box directional filter): every sampling sum and child, tree sum / weight /
    depth / count and the mean > 0 flag bit-exact.  The distribution statistics against GP:1121-1186 evaluated in float64 on the oracle's export:
    counts, minima and maxima exact, the sums of depths and node counts exact, the sums of means and weights to 1e-6 relative."""
    I = _I()
    o, rng = _trained(kind, rounds=3, dfilter=dfilter)
    o.refine(2000); o.reset(20, 0.01)
    _record(o, rng, 20000, dfilter=dfilter)
    e1 = o.export(1)
    ss, sc, per, st = I.op_sdtree_build(e1["s_children"], e1["tree_first"].astype(np.uint32), e1["tree_count"], e1["tree_depth"], e1["tree_weight"],
                                        e1["sums"], e1["children"])
    o.build()
    e0 = o.export(0)
    assert _same(ss, e0["sums"]) and _same(sc, e0["children"])
    leaf = e0["s_is_leaf"] != 0
    for k in ("tree_sum", "tree_weight", "tree_depth", "tree_count"):
        assert _same(per[k][leaf], e0[k][leaf]), k
    w, s = e0["tree_weight"][leaf], e0["tree_sum"][leaf]
    with np.errstate(divide="ignore", invalid="ignore"):
        mean = np.where(w != 0, (np.float32(1) / (np.float32(np.pi) * np.float32(4) * w)) * s, np.float32(0)).astype(np.float32)
    assert np.array_equal(per["mean_positive"][leaf] != 0, mean > 0) and (mean > 0).any()
    depth, cnt = e0["tree_depth"][leaf], e0["tree_count"][leaf]
    big = cnt > 1
    assert st["leaves"] == leaf.sum() and st["leaves_with_nodes"] == big.sum()
    assert (st["depth_min"], st["depth_max"]) == (depth.min(), depth.max())
    assert (st["mean_min"], st["mean_max"], st["weight_min"], st["weight_max"]) == (mean.min(), mean.max(), w.min(), w.max())
    assert (st["nodes_min"], st["nodes_max"]) == (cnt[big].min(), cnt[big].max())
    assert st["depth_sum"] == depth.astype(np.float64).sum() and st["nodes_sum"] == cnt[big].astype(np.float64).sum()
    assert st["mean_sum"] == pytest.approx(mean.astype(np.float64).sum(), rel=1e-6) and st["weight_sum"] == pytest.approx(w.astype(np.float64).sum(), rel=1e-6)


@pytest.fixture(scope="module")
def jitter(tmp_path_factory):
    if CUDA_INC is None:
        pytest.skip("needs the CUDA headers")
    import ctypes as C
    dev = compile_device_on_host(tmp_path_factory.mktemp("hostdev") / "libdevice_on_host.so")
    dev.dev_vertex_jitter.argtypes = [C.c_uint64, C.c_size_t, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.POINTER(C.c_float)]

    def f(seed, si, od):
        si = np.ascontiguousarray(si, np.uint64); od = np.ascontiguousarray(od, np.uint32); out = np.zeros((len(si), 3), np.float32)
        assert dev.dev_vertex_jitter(seed, len(si), si.ctypes.data_as(C.POINTER(C.c_uint64)), od.ctypes.data_as(C.POINTER(C.c_uint32)),
                                     out.ctypes.data_as(C.POINTER(C.c_float))) == 0
        return out
    return f


def _vertices(o, rng, n):
    """Vertices as the bounce kernel writes them, with the invalid and edge cases of Vertex::commit mixed in."""
    f = np.float32
    pos = rng.random((n, 3)).astype(f)
    k = n // 20
    pos[:k, 0] = 0.0; pos[k:2 * k, 1] = 1.0; pos[2 * k:3 * k, 2] = f(1 + 1e-3); pos[3 * k:4 * k, 0] = f(-1e-3)      # on and just outside the faces
    d = _dirs(rng, n)
    wo = (0.05 + rng.random(n)).astype(f); wo[4 * k:4 * k + 50] = 0; wo[4 * k + 50:4 * k + 100] = -0.5
    thr = (0.1 + rng.random((n, 3))).astype(f)
    thr[5 * k:5 * k + 200, 1] = 1e-5                                        # below epsilon
    thr[6 * k:6 * k + 200, 0] = 5e-4; wo[6 * k:6 * k + 200] = 0.1           # above epsilon, but thr * woPdf = 5e-5 is not
    rad = rng.lognormal(0, 1, (n, 3)).astype(f)
    rad[7 * k:7 * k + 50, 1] = np.nan; rad[7 * k + 50:7 * k + 100, 2] = -1.0
    bv = rng.random((n, 3)).astype(f); bv[8 * k:8 * k + 50, 0] = np.inf
    bp, dp = rng.random(n).astype(f), rng.random(n).astype(f)
    delta = np.zeros(n, bool); delta[9 * k:9 * k + 300] = True
    leaf, size = o.lookup(pos)
    level = np.rint(-np.log2(size.astype(np.float64))).sum(axis=1).astype(np.uint32)
    si = rng.integers(0, 1 << 62, n, dtype=np.uint64); od = rng.integers(0, 1 << 20, n, dtype=np.uint32)
    v = np.zeros((n, 6, 4), f)
    v[:, 0, :3] = d; v[:, 0, 3] = wo
    v[:, 1, :3] = thr; v[:, 1, 3] = leaf.view(f)
    v[:, 2, 3] = (np.arange(n, dtype=np.uint32) | (delta.astype(np.uint32) << 31)).view(f)
    v[:, 3, :3] = bv; v[:, 3, 3] = bp
    v[:, 4, :3] = pos; v[:, 4, 3] = dp
    v[:, 5, 0] = (si & 0xFFFFFFFF).astype(np.uint32).view(f); v[:, 5, 1] = (si >> 32).astype(np.uint32).view(f)
    v[:, 5, 2] = (level | (od << 8)).view(f)
    li = np.concatenate([rad, np.ones((n, 1), f)], axis=1)
    return dict(v=v, li=li, pos=pos, d=d, wo=wo, thr=thr, rad=rad, bv=bv, bp=bp, dp=dp, delta=delta, leaf=leaf, size=size, si=si, od=od)


def _adam_records(o, V, rnd, sfilter, weight):
    """The sampling-fraction records of Vertex::commit (GP:1735-1741) restated in float32 numpy: one per valid vertex with product > 0, into the
    vertex's own leaf (nearest) or the leaf of its jittered, clipped position (stochastic)."""
    f = np.float32
    ok = (V["wo"] > 0) & np.isfinite(V["rad"]).all(1) & (V["rad"] >= 0).all(1) & np.isfinite(V["bv"]).all(1) & (V["bv"] >= 0).all(1)
    with np.errstate(all="ignore"):
        local = np.where(V["thr"] * V["wo"][:, None] > f(1e-4), V["rad"] / V["thr"], f(0)).astype(f)
        p = (local * V["bv"]).astype(f)
        prod = ((p[:, 0] + p[:, 1]) + p[:, 2]) * (f(1) / f(3))
    keep = ok & (prod > 0)
    if sfilter == 0:
        leaf = V["leaf"]
    else:
        q = np.clip(V["pos"] + V["size"] * (rnd - f(0.5)), f(0), f(1)).astype(f)
        leaf, _ = o.lookup(q)
    rec = np.stack([leaf.view(f), prod, V["wo"], V["bp"], V["dp"], np.full(len(leaf), weight, f)], axis=1)[keep]
    return rec


def _sorted_rows(r):
    u = np.ascontiguousarray(r, np.float32).view(np.uint32)
    return u[np.lexsort(u.T[::-1])]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("sfilter", [0, 1, 2])
@pytest.mark.parametrize("dfilter", [0, 1])
@pytest.mark.parametrize("loss", [0, 1])
def test_commit_kernel_matches_vertex_commit(kind, sfilter, dfilter, loss, jitter):
    """commit_kernel on vertices written in the bounce kernel's layout -- NaN and negative radiance, an inf BSDF value, woPdf 0 and < 0, throughput
    channels below epsilon, channels above it whose product with woPdf is not, delta vertices, positions on and just outside the faces of the box --
    against Vertex::commit of the oracle with the same jitter numbers (seed_vertex_rng, evaluated on the host).  Statistical weight 1 without a loss,
    0.5 with it.  Weights: exact for nearest and stochastic (dyadic adds); 1e-5 relative for the box filter, whose weights are sums of hundreds of
    fractional overlaps added in atomic order (measured on one H100: up to 3e-6).  Sums: the float atomics reorder the adds
    (the tolerance of test_op_dtree_record_matches_reference).  Sampling-fraction records (nearest, stochastic): as a multiset, bit for bit, the
    float32 restatement of GP:1735-1741."""
    I = _I()
    o, rng = _trained(kind, rounds=3, dfilter=dfilter)
    o.refine(2000); o.reset(20, 0.01)
    e1 = o.export(1)
    n, seed, weight = 20000, 77, (0.5 if loss else 1.0)
    V = _vertices(o, rng, n)
    rnd = jitter(seed, V["si"], V["od"])
    mn, mx = e1["aabb"]
    sums, bw, rec = I.op_commit(e1["s_children"], mn, mx - mn, e1["tree_first"].astype(np.uint32), e1["tree_weight"], e1["sums"], e1["children"], V["v"], V["li"],
                                record_mode=2, spatial_filter=sfilter, directional_filter=dfilter, loss=loss, seed=seed, statistical_weight=weight)
    o.commit(V["pos"], V["d"], V["thr"], V["bv"], V["rad"], V["wo"], V["bp"], V["dp"], np.full(n, weight, np.float32), V["delta"], rnd,
             sfilter=sfilter, dfilter=dfilter, loss=loss)
    e2 = o.export(1)
    leaf = e2["s_is_leaf"] != 0
    if sfilter == 2:
        assert np.allclose(bw, e2["tree_weight"], rtol=1e-5, atol=1e-6 * np.abs(e2["tree_weight"]).max())
    else:
        assert _same(bw, e2["tree_weight"])
    assert (e2["tree_weight"][leaf] > 0).sum() > 8
    scale = np.abs(e2["sums"]).sum() / max(1, leaf.sum())
    assert np.abs(sums - e2["sums"]).max() <= 1e-5 * scale + 1e-6 * np.abs(e2["sums"]).max()
    if loss == 0:
        assert len(rec) == 0
    elif sfilter in (0, 1):
        want = _adam_records(o, V, rnd, sfilter, weight)
        assert len(rec) == len(want) > n // 2
        assert np.array_equal(_sorted_rows(rec), _sorted_rows(want))


# Adam replay against the reference optimizer, measured on one H100 80GB HBM3 (700 W) with this file's chains: |dtheta| <= 5.8e-8 (KL) and 4.5e-8 (var);
# m1, m2 and batchGrad within 8e-8 of each column's largest magnitude.  adam_seq_kernel's __fdividef / __expf and float learning rate stay far inside
# the 1e-4 ceiling on theta.  Bounds: theta 1e-6, the others 1e-6 of the column's largest magnitude (the var loss squares ratios up to 1e15).
_ADAM_BOUND = dict(theta=1e-6, m=1e-6, grad=1e-6)


def _octant_oracle(kind, rng):
    o = O.Oracle(O.default_params(), aabb=BOX, kind=kind)
    o.reset(20, 0.01); _record(o, rng, 1, pos=np.full((1, 3), 0.5, np.float32), weight=8000.0, loss=0); o.build()
    o.refine(1000); o.reset(20, 0.01); o.build()
    centers = np.array([[0.25 + 0.5 * (k & 1), 0.25 + 0.5 * ((k >> 1) & 1), 0.25 + 0.5 * (k >> 2)] for k in range(8)], np.float32)
    leaf, _ = o.lookup(centers)
    return o, centers, leaf


def _chain(rng, n, kind):
    f = np.float32
    prod = rng.lognormal(0, 1, n).astype(f); wo = (0.05 + rng.random(n)).astype(f)
    bp, dp = (0.05 + rng.random(n)).astype(f), (0.05 + rng.random(n)).astype(f)
    w = np.ones(n, f)
    if kind == "half":
        w[:] = 0.5
    elif kind == "frac":
        w = (0.05 + 0.9 * rng.random(n)).astype(f)
    elif kind == "zeros":
        dp[::3] = 0; bp[1::3] = 0
    elif kind == "clamp":                        # bsdfPdf 0 and a gradient that outweighs the L2 term down to theta = -20: theta runs into the clamp
        prod[:] = 1e8; wo[:] = 0.05; bp[:] = 0.0; dp[:] = 2.0
    return np.stack([prod, wo, bp, dp, w], axis=1)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("loss", [1, 2])
def test_adam_replay_matches_the_reference_optimizer(kind, loss):
    """adam_seq_kernel on chains of 1, 31, 32, 33, 64 and 10^5 records (the warp fetches 32 records per chunk), eight leaves in one launch, each starting
    from a carried state (iter > 0, batchAcc > 0) left by a prefix of records; weights 1, 0.5 and fractional, dTreePdf = 0 and bsdfPdf = 0, and a
    one-sided chain that drives theta into the -20 clamp.  Reference: DTreeWrapper::record of the oracle with the same records in the same order.
    iter and batchAcc bit-exact (the step decisions add the same floats in the same order); theta, m1, m2 and batchGrad within _ADAM_BOUND."""
    I = _I()
    rng = np.random.default_rng(31 + loss)
    o, centers, leaf = _octant_oracle(kind, rng)
    plan = [(1, "one"), (31, "half"), (32, "frac"), (33, "zeros"), (64, "one"), (100000, "clamp"), (257, "frac"), (0, "one")]
    f = np.float32
    # carried start state: a prefix of 7 records of weight 0.3 per leaf (one step, batchAcc 0.9 left over)
    for k in range(8):
        pre = _chain(rng, 7, "one"); pre[:, 4] = 0.3
        o.record(np.tile(centers[k], (7, 1)), _dirs(rng, 7), np.ones(7, f), pre[:, 1], product=pre[:, 0], bsdf_pdf=pre[:, 2], dtree_pdf=pre[:, 3], weight=pre[:, 4], loss=loss)
    start = o.export(0)["adam"].copy()
    assert (start[leaf, 0] > 0).all() and (start[leaf, 4] > 0).all()
    recs, offs, cnts = [], np.zeros(len(start), np.uint32), np.zeros(len(start), np.uint32)
    pos = 0
    for k, (n, how) in enumerate(plan):
        c = _chain(rng, n, how)
        if n:
            o.record(np.tile(centers[k], (n, 1)), _dirs(rng, n), np.ones(n, f), c[:, 1], product=c[:, 0], bsdf_pdf=c[:, 2], dtree_pdf=c[:, 3], weight=c[:, 4], loss=loss)
        r = np.zeros((n, 6), f); r[:, 0] = np.full(n, leaf[k], np.uint32).view(f); r[:, 1:] = c[:, [0, 1, 2, 3, 4]]
        recs.append(r); offs[leaf[k]] = pos; cnts[leaf[k]] = n; pos += n
    g = I.op_adam_replay(start, np.concatenate(recs), loss, leaf_offset=offs, leaf_count=cnts)
    want = o.export(0)["adam"]
    gs = g["state"]
    assert not g["count"].any() and not g["cursor"].any()
    assert _same(gs[:, 0], want[:, 0]) and _same(gs[:, 4], want[:, 4])
    assert want[leaf, 0].max() > 40000 and want[leaf, 3].min() == -20.0
    assert _same(g["theta"][leaf], gs[leaf, 3])
    dt, dm1, dm2, dg = (np.abs(gs[:, j] - want[:, j]).max() for j in (3, 1, 2, 5))
    rel = [np.abs(gs[:, j] - want[:, j]).max() / max(np.abs(want[:, j]).max(), 1e-30) for j in (1, 2, 5)]
    print(f"adam replay loss={loss} kind={kind}: max |dtheta| {dt:.3g}, |dm1| {dm1:.3g}, |dm2| {dm2:.3g}, |dbatchGrad| {dg:.3g}, relative to the column max {rel}")
    assert dt <= _ADAM_BOUND["theta"]
    assert np.allclose(gs[:, 1], want[:, 1], rtol=_ADAM_BOUND["m"], atol=_ADAM_BOUND["m"] * np.abs(want[:, 1]).max())
    assert np.allclose(gs[:, 2], want[:, 2], rtol=_ADAM_BOUND["m"], atol=_ADAM_BOUND["m"] * np.abs(want[:, 2]).max())
    assert np.allclose(gs[:, 5], want[:, 5], rtol=_ADAM_BOUND["grad"], atol=_ADAM_BOUND["grad"] * np.abs(want[:, 5]).max())


def test_adam_buckets_are_permutations_of_each_leafs_records():
    """histogram -> scan -> scatter on records of 5000 leaves in random order: every bucket is, bit for bit, a permutation of its leaf's records, the
    offsets are the exclusive prefix sum of the counts, count and cursor are zero after adam_seq_kernel, and the bucketed replay equals a replay of the
    buckets in the order the scatter left them."""
    I = _I()
    rng = np.random.default_rng(2)
    nl, n = 5000, 300000
    leaf = np.minimum(rng.zipf(1.5, n) - 1, nl - 1).astype(np.uint32)
    rec = np.zeros((n, 6), np.float32)
    rec[:, 0] = leaf.view(np.float32); rec[:, 1] = rng.lognormal(0, 1, n); rec[:, 2] = 0.05 + rng.random(n); rec[:, 3:5] = rng.random((n, 2)); rec[:, 5] = rng.random(n)
    state = np.zeros((nl, 6), np.float32)
    g = I.op_adam_replay(state, rec, 1, bucket=True)
    cnt = np.bincount(leaf, minlength=nl).astype(np.uint32)
    assert np.array_equal(g["leaf_offset"], np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.uint32))
    assert not g["count"].any() and not g["cursor"].any()
    order = np.argsort(leaf, kind="stable"); by_leaf = rec[order]; first = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.int64)
    for l in np.nonzero(cnt)[0]:
        got = g["records"][g["leaf_offset"][l]:g["leaf_offset"][l] + cnt[l]]
        assert np.array_equal(_sorted_rows(got), _sorted_rows(by_leaf[first[l]:first[l] + cnt[l]])), l
    h = I.op_adam_replay(state, g["records"], 1, leaf_offset=g["leaf_offset"], leaf_count=cnt)
    assert _same(h["state"], g["state"]) and (g["state"][:, 0] > 0).sum() > 100
