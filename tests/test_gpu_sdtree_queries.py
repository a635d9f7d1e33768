"""The query half of the SD-tree on the GPU, at the depths the render reaches: ppg_op_stree_lookup (stree_lookup through the prefix table, then the
walk past its 21 levels), ppg_op_dtree_pdf and ppg_op_dtree_sample (dtree_pdf, dtree_sample and the cylindrical maps), against the numpy restatements
of tests/sdtree_queries.py and the oracle's trees: kind "port" (restated SD-tree) and, where oracle/_ref was built, "ref" (the reference's own code).
The same cases run through the host build of the device source in tests/test_device_source_on_host.py."""
import numpy as np
import pytest

import oracle_lib as O
import sdtree_queries as Q
from common import load_cbox

pytestmark = pytest.mark.gpu
KINDS = ["port"] + (["ref"] if O.have_ref() else [])
f32 = np.float32


def _I():
    from ppg_b200 import integrator as I
    return I


def _box(name):
    if name == "dyadic":
        return Q.DYADIC_BOX
    o = O.Oracle(O.default_params(), load_cbox(16), kind="port")        # the cubified CBOX box: not dyadic
    mn, mx = o.export(0)["aabb"]; o.close()
    return mn.astype(f32), mx.astype(f32)


def _same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("box", ["dyadic", "cbox"])
def test_stree_lookup_deep_trained_tree(kind, box):
    """An S-tree the oracle refines for eight rounds around one point (~7 levels per round over ~5000 uniform leaves): leaves at depth >= 45.
    Uniform points, points exactly on the split planes of every inner node from depth 15 down and of up to 24 levels per axis around the deep point,
    on the faces and one ulp inside / outside them, far outside.  Leaf and voxel size bit for bit against the oracle's lookup and the numpy walk."""
    mn, mx = _box(box)
    q = np.array([0.3137, 0.6271, 0.4519])
    o = Q.deep_trained_stree(O, kind, (mn, mx), q)
    e = o.export(0)
    mn, mx = e["aabb"]; ext = (mx - mn).astype(f32)
    sch = e["s_children"]
    rng = np.random.default_rng(41)
    pts = np.concatenate([Q.stree_points(rng, mn, ext, [q, (0, 0, 0), (1, 1, 1)], 10000), Q.split_plane_points(sch, mn, ext, 15)])
    wl, ws, wd = Q.stree_walk(sch, mn, ext, pts)
    assert wd.max() >= 45 and (wd > Q.TABLE_LEVELS).sum() > 500, (wd.max(), (wd > Q.TABLE_LEVELS).sum())
    ol, os_ = o.lookup(pts)
    assert np.array_equal(ol, wl) and _same_bits(os_, ws)
    gl, gs = _I().op_stree_lookup(sch, mn, ext, pts)
    assert np.array_equal(gl, wl) and _same_bits(gs, ws)


@pytest.mark.parametrize("box", ["dyadic", "cbox"])
def test_stree_lookup_at_the_prefix_table_boundary(box):
    """A synthetic S-tree with leaves at exactly 20, 21 and 22 levels (the table resolves 21), some in corners of the box: the points above; leaf and
    voxel size bit for bit against the numpy walk."""
    mn, mx = _box(box); ext = (mx - mn).astype(f32)
    sch = Q.synthetic_stree(Q.SYNTHETIC_ANCHORS)
    rng = np.random.default_rng(42)
    pts = np.concatenate([Q.stree_points(rng, mn, ext, [a for a, _ in Q.SYNTHETIC_ANCHORS]), Q.split_plane_points(sch, mn, ext, 15)])
    wl, ws, wd = Q.stree_walk(sch, mn, ext, pts)
    assert {20, 21, 22} <= set(wd.tolist())
    gl, gs = _I().op_stree_lookup(sch, mn, ext, pts)
    assert np.array_equal(gl, wl) and _same_bits(gs, ws)


def test_stree_lookup_past_2to24_nodes():
    """The synthetic tree renumbered so that every node but the root is >= 2^24 (2^24 + 5 unreachable leaves in between, ~134 MB): the prefix
    table's 24-bit node field cannot hold those numbers, so the lookup walks from the root.  Leaves and voxel sizes bit for bit."""
    mn, mx = Q.DYADIC_BOX; ext = (mx - mn).astype(f32)
    sch = Q.synthetic_stree(Q.SYNTHETIC_ANCHORS, offset=(1 << 24) + 5)
    rng = np.random.default_rng(43)
    pts = np.concatenate([Q.stree_points(rng, mn, ext, [a for a, _ in Q.SYNTHETIC_ANCHORS], 20000), Q.split_plane_points(sch, mn, ext, 15)])
    wl, ws, wd = Q.stree_walk(sch, mn, ext, pts)
    assert len(sch) > 1 << 24 and (wl >= 1 << 24).all() and {20, 21, 22} <= set(wd.tolist())
    gl, gs = _I().op_stree_lookup(sch, mn, ext, pts)
    assert np.array_equal(gl, wl), f"{int((gl != wl).sum())} of {len(wl)} leaves differ, e.g. {gl[gl != wl][:4]} for {wl[gl != wl][:4]}"
    assert _same_bits(gs, ws)


@pytest.fixture(scope="module", params=KINDS)
def dtrees(request):
    return Q.dtree_trees(O, request.param)


def test_dtree_trees_reach_their_edges(dtrees):
    """The trees of tests/sdtree_queries.dtree_trees are what the cases below claim: six at depth 20 with zero-sum quadrants, inner ones included;
    one of 65 536 nodes; one untrained."""
    _, e, leaves, _ = dtrees
    first = e["tree_first"].astype(np.int64)
    valid = Q.valid_flags(e["tree_sum"], e["tree_weight"])
    assert (e["tree_depth"][leaves[:6]] == 20).all() and e["tree_count"][leaves[6]] == 65536 and valid[leaves[:7]].all() and not valid[leaves[7]]
    rng = np.random.default_rng(0)
    assert any(Q.zero_sum_cells(e["sums"], e["children"], int(first[leaf]), rng)[1].any() for leaf in leaves[:6])


@pytest.mark.parametrize("op", ["pdf", "sample"])
def test_dtree_queries_at_the_depth_cap(dtrees, op):
    """pdf: random directions, both poles, the phi seam (y = +0 / -0 with x < 0 and x > 0), canonical x on quadrant boundaries of levels 1-22 near each
    cone (with exact phi 0, pi/2, pi and with the cone's phi), canonical y = 0.25 / 0.5, centres of zero-sum cells.  Zeros exact, 1 / 4 pi exact for the
    untrained tree, elsewhere the kernel and the reference trees within (5 * depth + 2) * 2^-24 of the float64 product of the exact per-level ratios
    (3 adds, 1 divide, 1 multiply per level).  Where phi comes from a general atan2f, the canonical y of the host's atan2f +- 2 ulps is allowed.
    sample: random uniforms, rows of 0 and of 1 - 2^-24, single extreme entries, and uniforms equal to a node's float32 partial / total boundary or
    re-stretching exactly onto its topLeft / partial or topRight / partial boundary.  The canonical point bit-equal to the reference's DTree::sample
    point and to the float32 restatement; directions within 2e-6 (sincosf)."""
    o, e, leaves, cones = dtrees
    I = _I()
    rng = np.random.default_rng(44)
    first = e["tree_first"].astype(np.int64); valid = Q.valid_flags(e["tree_sum"], e["tree_weight"]); ft = e["tree_first"].astype(np.uint32)
    if op == "pdf":
        ql, d, ex = [], [], []
        for k, leaf in enumerate(leaves):
            dk, exk = Q.pdf_directions(rng, e["sums"], e["children"], int(first[leaf]), cones[k], n_random=20000)
            ql.append(np.full(len(dk), leaf, np.uint32)); d.append(dk); ex.append(exk)
        ql, d, ex = np.concatenate(ql), np.concatenate(d), np.concatenate(ex)
        got = I.op_dtree_pdf(e["sums"], e["children"], ft, e["tree_sum"], e["tree_weight"], ql, d)
        ok, depth = Q.pdf_matches(got, e["sums"], e["children"], first[ql], valid[ql], d, exact_phi=ex)
        assert ok.all(), (np.nonzero(~ok)[0][:8], got[~ok][:8])
        ok_o, _ = Q.pdf_matches(o.pdf(ql, d), e["sums"], e["children"], first[ql], valid[ql], d, exact_phi=ex)
        assert ok_o.all()
        assert depth.max() == 20 and (got == 0).any() and (got[~valid[ql]] == f32(1) / (f32(4) * Q.PI32)).all()
    else:
        ql = np.repeat(leaves, 25000).astype(np.uint32)
        rnd = Q.sample_uniforms(rng, e["sums"], e["children"], first[ql], valid[ql], len(ql))
        dirs, canon = I.op_dtree_sample(e["sums"], e["children"], ft, e["tree_sum"], e["tree_weight"], ql, rnd, canonical=True)
        want, levels = Q.sample_reference(e["sums"], e["children"], first[ql], valid[ql], rnd)
        assert levels.max() == 20
        assert _same_bits(canon, want), int((canon != want).any(axis=1).sum())
        # the restated oracle is built from this tree and always returns the point; a prebuilt reference library may predate the entry
        assert o.has_sample_canonical() or o.kind == "ref"
        if o.has_sample_canonical():
            assert _same_bits(canon, o.sample_canonical(ql, rnd))
        assert np.abs(dirs - o.sample(ql, rnd)).max() <= 2e-6


def _cells(sums, children, root, max_depth):
    """Cells of one tree: every quadrant whose child is a leaf or which lies at max_depth, keyed (node * 4 + quadrant), with its float64
    probability (the product of s_c / total down to it)."""
    prob = {}
    st = [(0, 1.0, 1)]
    while st:
        nd, p, d = st.pop()
        s = sums[root + nd].astype(np.float64); tot = s.sum()
        for c in range(4):
            pc = p * s[c] / tot if tot > 0 else 0.0
            ch = int(children[root + nd, c])
            if ch and d < max_depth:
                st.append((ch, pc, d + 1))
            else:
                prob[nd * 4 + c] = pc
    return prob


def _cell_of(sums, children, root, p, max_depth):
    px, py = p[:, 0].copy(), p[:, 1].copy(); node = np.zeros(len(p), np.int64); key = np.full(len(p), -1, np.int64)
    act = np.arange(len(p))
    for d in range(1, max_depth + 1):
        lx, ly = px[act] < f32(0.5), py[act] < f32(0.5)
        px[act] = np.where(lx, px[act] * f32(2), (px[act] - f32(0.5)) * f32(2)); py[act] = np.where(ly, py[act] * f32(2), (py[act] - f32(0.5)) * f32(2))
        c = (~lx).astype(np.int64) | ((~ly).astype(np.int64) << 1)
        ch = children[root + node[act], c].astype(np.int64)
        stop = (ch == 0) | (d == max_depth)
        key[act[stop]] = node[act[stop]] * 4 + c[stop]
        node[act] = ch
        act = act[~stop]
    return key


def test_dtree_sample_chi_square_at_depth_20():
    """2^20 GPU samples of one depth-20 cone tree, binned by the cells of its first 12 levels (deeper cells merged into their level-12 ancestor), against
    the probabilities of those cells in float64 from the sums; cells expecting < 5 samples pooled.  chi^2 p-value >= 1e-4.  Zero-probability cells
    receive at most 1e-5 of the samples: the float32 fold of a sample at the far edge of a cell can round onto the next cell's boundary."""
    from scipy import stats
    _, e, leaves, _ = Q.dtree_trees(O, "port")
    leaf = int(leaves[4]); root = int(e["tree_first"][leaf])        # its cone did not move in the last round: the mass lies in depth-20 cells
    assert e["tree_depth"][leaf] == 20
    n = 1 << 20
    rng = np.random.default_rng(45)
    rnd = rng.random((n, Q.RND_STRIDE), dtype=np.float32)
    _, canon = _I().op_dtree_sample(e["sums"], e["children"], e["tree_first"].astype(np.uint32), e["tree_sum"], e["tree_weight"],
                                    np.full(n, leaf, np.uint32), rnd, canonical=True)
    prob = _cells(e["sums"], e["children"], root, 12)
    keys = np.array(sorted(prob)); p = np.array([prob[k] for k in keys])
    assert abs(p.sum() - 1) < 1e-9
    got = _cell_of(e["sums"], e["children"], root, canon, 12)
    count = np.bincount(np.searchsorted(keys, got), minlength=len(keys))
    assert np.array_equal(keys[np.searchsorted(keys, got)], got)
    zero = p == 0
    assert count[zero].sum() <= 1e-5 * n, count[zero].sum()
    exp = n * p[~zero]; obs = count[~zero]
    small = exp < 5
    exp = np.append(exp[~small], exp[small].sum()); obs = np.append(obs[~small], obs[small].sum())
    if exp[-1] == 0:
        exp, obs = exp[:-1], obs[:-1]
    exp *= obs.sum() / exp.sum()
    chi2 = float(((obs - exp) ** 2 / exp).sum())
    pval = stats.chi2.sf(chi2, len(exp) - 1)
    assert len(exp) > 20 and pval >= 1e-4, (chi2, len(exp), pval)
