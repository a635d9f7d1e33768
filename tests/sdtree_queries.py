"""The query half of the SD-tree -- S-tree lookup, D-tree pdf and sample -- restated in numpy, and the trees and inputs that drive it to its edges.
Shared by the GPU tests (tests/test_gpu_sdtree_queries.py: ppg_op_stree_lookup, ppg_op_dtree_pdf, ppg_op_dtree_sample) and the host build of the
same device source (tests/test_device_source_on_host.py: dev_stree_lookup, dev_dtree).

* S-tree: STree::dTreeWrapper (GP:897-905, 761-769): the point normalised in float32 exactly as stree_lookup does, then midpoint splits with the axes
  cycling x, y, z and `p < 0.5`.  Every step is exact in float32, so leaf and voxel size are compared bit for bit.
* D-tree pdf (GP:415-421, 232-245): a float64 product of the exact per-level ratios 4 s_c / (s_0 + s_1 + s_2 + s_3).  A float32 implementation rounds
  3 adds, 1 divide and 1 multiply per level (relative error <= 2^-24 each), and once more in the final division by 4 pi: PDF_ULPS_PER_LEVEL * depth + 2
  units of 2^-24 bound both the kernel's top-down product and the reference's bottom-up one.
* D-tree sample (GP:431-442, 257-301): restated in float32 (every operation is IEEE +, -, *, /): the canonical point is bit-exact."""
import numpy as np

f32 = np.float32
PI32 = f32(3.14159265358979323846)          # PPG_PI, M_PI as Float
U = 2.0 ** -24
PDF_ULPS_PER_LEVEL = 5                      # 3 adds, 1 divide, 1 multiply
TABLE_LEVELS = 21                           # 3 * PPG_STREE_TABLE_BITS
RND_STRIDE = 24                             # uniforms per sample query: 20 levels + 2 at the leaf + spare
ONE_MINUS = f32(1 - 2.0 ** -24)             # the largest uniform below 1


# ------------------------------------------------------------------ S-tree
def stree_walk(sch, mn, ext, pts):
    """(leaf node, voxel size float32 (n, 3), depth) of every point."""
    sch = np.asarray(sch)
    p = ((np.asarray(pts, f32) - np.asarray(mn, f32)) / np.asarray(ext, f32)).astype(f32)
    n = np.zeros(len(p), np.int64); depth = np.zeros(len(p), np.int64)
    size = np.tile(np.asarray(ext, f32), (len(p), 1))
    act = np.nonzero(sch[n, 0] != 0)[0]
    level = 0
    while len(act):
        a = level % 3
        v = p[act, a]
        lo = v < f32(0.5)
        p[act, a] = np.where(lo, v * f32(2), (v - f32(0.5)) * f32(2))
        n[act] = np.where(lo, sch[n[act], 0], sch[n[act], 1])
        size[act, a] = size[act, a] / f32(2)
        depth[act] += 1
        level += 1
        act = act[sch[n[act], 0] != 0]
    return n.astype(np.uint32), size, depth


def synthetic_stree(anchors, base=9, offset=0):
    """An S-tree (node_children, uint32 (N, 2)) refined uniformly to `base` levels and, around every (unit point, depth) anchor, down to exactly that
    depth: every cell whose closed box holds the point splits while shallower.  With `offset`, every node but the root is renumbered n + offset and the
    rows in between are unreachable leaves -- the layout later refines produce, where children of shallow leaves follow every existing node."""
    pts = np.array([a for a, _ in anchors], np.float64).reshape(-1, 3); tgt = np.array([d for _, d in anchors], np.int64)
    kids = [[0, 0]]
    st = [(0, 0, np.zeros(3), np.ones(3))]
    while st:
        node, d, lo, sz = st.pop()
        inside = np.all((pts >= lo) & (pts <= lo + sz), axis=1)
        if not (d < base or (inside & (tgt > d)).any()):
            continue
        a = d % 3
        c0, c1 = len(kids), len(kids) + 1
        kids += [[0, 0], [0, 0]]; kids[node] = [c0, c1]
        h = sz.copy(); h[a] /= 2
        lo1 = lo.copy(); lo1[a] += h[a]
        st += [(c1, d + 1, lo1, h), (c0, d + 1, lo.copy(), h)]
    k = np.array(kids, np.uint32)
    if not offset:
        return k
    out = np.zeros((len(k) + offset, 2), np.uint32)
    out[0] = np.where(k[0] != 0, k[0] + offset, 0)
    out[offset + 1:] = np.where(k[1:] != 0, k[1:] + offset, 0)
    return out


# leaves at exactly 20, 21 and 22 levels (the prefix table covers 21), some in corners of the box so that face points reach them
SYNTHETIC_ANCHORS = [((0.3, 0.7, 0.2), 20), ((0.55, 0.1, 0.9), 20), ((0.0, 1.0, 0.0), 20),
                     ((0.8, 0.4, 0.6), 21), ((0.123, 0.456, 0.789), 21), ((1.0, 1.0, 1.0), 21),
                     ((0.61, 0.27, 0.33), 22), ((0.05, 0.93, 0.48), 22), ((0.0, 0.0, 0.0), 22), ((1.0, 0.0, 1.0), 22)]

DYADIC_BOX = (np.full(3, -8, np.float32), np.full(3, 8, np.float32))    # extent 16: p - min and the division are exact for dyadic points


def stree_points(rng, mn, ext, anchors_unit, n_uniform=20000):
    """World points: uniform; on the split planes of up to 24 levels per axis around every anchor (one axis or all three snapped to a multiple of
    2^-L); on the min and max faces, one ulp inside and one ulp outside them; far outside the box.  float32 (n, 3)."""
    mn = np.asarray(mn, f32); ext = np.asarray(ext, f32); mx = (mn + ext).astype(f32)
    world = lambda u: (mn + np.asarray(u, np.float64).astype(f32) * ext).astype(f32)
    out = [world(rng.random((n_uniform, 3)))]
    A = np.asarray(anchors_unit, np.float64).reshape(-1, 3)
    for a in A:
        jit = np.clip(a + rng.normal(scale=1e-6, size=(24, 3)), 0, 1)
        for L in range(1, 25):
            q = np.round(jit[L - 1] * 2.0 ** L) / 2.0 ** L
            rows = np.tile(jit[L - 1], (4, 1))
            for ax in range(3):
                rows[ax, ax] = q[ax]
            rows[3] = q
            out.append(world(rows))
    # faces: the other two coordinates near the anchors and random
    base = np.concatenate([np.clip(A + rng.normal(scale=1e-7, size=A.shape), 0, 1), rng.random((64, 3))])
    for ax in range(3):
        for v in (mn[ax], mx[ax]):
            for w in (v, np.nextafter(v, f32(-np.inf)), np.nextafter(v, f32(np.inf))):
                p = world(base); p[:, ax] = w
                out.append(p)
    far = world(rng.random((64, 3)))
    for k, s in enumerate((-1.0, -100.0, 2.0, 1e6)):        # below the min face, far below, above the max face, far above
        p = far[16 * k:16 * k + 16].copy(); ax = k % 3
        p[:, ax] = (mn[ax] + f32(s) * ext[ax]).astype(f32)
        out.append(p)
    out.append(np.array([mn - ext, mx + ext, mn - f32(1e-3), mx + f32(1e-3)], f32))
    return np.concatenate(out).astype(f32)


def split_plane_points(sch, mn, ext, min_depth, max_depth=69):
    """World points exactly on the split plane of every inner node at depth min_depth..max_depth (the other coordinates at the cell's centre).
    In a box whose min and extent are powers of two these are exact float32 points (at most 24 bits per axis)."""
    mn = np.asarray(mn, f32); ext = np.asarray(ext, f32)
    out = []
    st = [(0, 0, np.zeros(3), np.ones(3))]
    while st:
        n, d, lo, sz = st.pop()
        if sch[n, 0] == 0 or d > max_depth:
            continue
        a = d % 3
        h = sz.copy(); h[a] /= 2
        if d >= min_depth:
            c = lo + sz / 2
            out.append(c)
        lo1 = lo.copy(); lo1[a] += h[a]
        st += [(int(sch[n, 0]), d + 1, lo.copy(), h), (int(sch[n, 1]), d + 1, lo1, h)]
    u = np.array(out, np.float64).reshape(-1, 3)
    return (mn + u.astype(f32) * ext).astype(f32)


def deep_trained_stree(O, kind, box, q_unit, rounds=8, thr=1000):
    """An S-tree the oracle refines over `rounds` record / build / refine / reset rounds: ~5000 leaves of uniform background, then each round one
    record of 65 * thr at the point q (~7 more levels around it per round)."""
    mn, mx = (np.asarray(b, f32) for b in box)
    rng = np.random.default_rng(21)
    o = O.Oracle(O.default_params(), aabb=box, kind=kind)
    o.reset(20, 0.01)
    q = (mn + np.asarray(q_unit, f32) * (mx - mn)).astype(f32)[None]
    pos = (mn + rng.random((50000, 3)).astype(f32) * (mx - mn)).astype(f32)
    one = lambda k: np.ones(k, f32)
    d = np.tile(np.array([[0, 0, 1]], f32), (len(pos), 1))
    o.record(pos, d, one(len(pos)), one(len(pos)), weight=np.full(len(pos), 100, f32))
    for _ in range(rounds):
        o.record(q, d[:1], one(1), one(1), weight=np.full(1, 65 * thr, f32))
        o.build(); o.refine(thr); o.reset(20, 0.01)
    return o


# ------------------------------------------------------------------ D-tree
def canonical(d, dphi=0):
    """dir_to_canonical in float32; dphi moves atan2's result by that many ulps (atan2f of the host and of the GPU may differ by an ulp or two)."""
    d = np.asarray(d, f32)
    x = ((np.clip(d[:, 2], f32(-1), f32(1)) + f32(1)) / f32(2)).astype(f32)
    phi = np.arctan2(d[:, 1], d[:, 0]).astype(f32)
    for _ in range(abs(dphi)):
        phi = np.nextafter(phi, f32(np.inf if dphi > 0 else -np.inf)).astype(f32)
    phi = np.where(phi < f32(0), (phi + f32(2) * PI32).astype(f32), phi)
    return np.stack([x, (phi / (f32(2) * PI32)).astype(f32)], axis=1).astype(f32)


def to_dir(c):
    """canonical point(s) -> float32 direction (float64 arithmetic, for choosing query directions)"""
    c = np.asarray(c, np.float64)
    z = 2 * c[:, 0] - 1; s = np.sqrt(np.maximum(0, 1 - z * z)); phi = 2 * np.pi * c[:, 1]
    return np.stack([s * np.cos(phi), s * np.sin(phi), z], axis=1).astype(f32)


def valid_flags(tree_sum, tree_weight):
    """DTree::mean() > 0 as the op kernels compute it (GP:386-394)"""
    w = np.asarray(tree_weight, f32); s = np.asarray(tree_sum, f32)
    with np.errstate(divide="ignore", invalid="ignore"):
        mean = np.where(w != 0, (f32(1) / (PI32 * f32(4) * w)) * s, f32(0)).astype(f32)
    return mean > 0


def pdf_reference(sums, children, root, valid, p):
    """(float64 pdf, levels walked, zero) of canonical points p (n, 2) in the trees rooted at `root`; invalid trees: 1 / 4 pi in float32."""
    sums = np.asarray(sums, f32); children = np.asarray(children, np.int64)
    n = len(p); px = np.asarray(p, f32)[:, 0].copy(); py = np.asarray(p, f32)[:, 1].copy()
    res = np.ones(n); depth = np.zeros(n, np.int64); zero = np.zeros(n, bool); node = np.asarray(root, np.int64).copy()
    act = np.nonzero(valid)[0]
    while len(act):
        lx, ly = px[act] < f32(0.5), py[act] < f32(0.5)
        px[act] = np.where(lx, px[act] * f32(2), (px[act] - f32(0.5)) * f32(2)); py[act] = np.where(ly, py[act] * f32(2), (py[act] - f32(0.5)) * f32(2))
        c = (~lx).astype(np.int64) | ((~ly).astype(np.int64) << 1)
        s = sums[node[act]]; sc = s[np.arange(len(act)), c]
        z = ~(sc > 0)
        res[act] *= np.where(z, 1.0, 4.0 * sc.astype(np.float64) / s.astype(np.float64).sum(1))
        depth[act] += 1; zero[act[z]] = True
        nxt = children[node[act], c]
        done = z | (nxt == 0)
        node[act] = np.where(done, node[act], np.asarray(root, np.int64)[act] + nxt)
        act = act[~done]
    pdf = np.where(zero, 0.0, res / np.float64(f32(4) * PI32))
    pdf = np.where(valid, pdf, np.float64(f32(1) / (f32(4) * PI32)))
    return pdf, depth, zero


def pdf_within_bound(got, ref, depth, zero, valid):
    """Zeros and the untrained 1 / 4 pi exact; elsewhere within (PDF_ULPS_PER_LEVEL * depth + 2) * 2^-24 of the float64 product."""
    got = np.asarray(got, np.float64)
    ok_zero = zero & (got == 0)
    ok_val = ~zero & (np.abs(got - ref) <= (PDF_ULPS_PER_LEVEL * depth + 2) * U * ref)
    return np.where(valid, ok_zero | ok_val, got == ref)


def pdf_matches(got, sums, children, root, valid, d, exact_phi=None, dphis=(0, -1, 1, -2, 2)):
    """Per query: `got` is within the bound of the reference pdf of one of the canonical points atan2f may produce (exact_phi rows: only the
    correctly rounded one -- their atan2 is exact in every libm).  Returns (ok, depth of the dphi = 0 walk)."""
    ok = np.zeros(len(d), bool); depth0 = None
    for k in dphis:
        ref, depth, zero = pdf_reference(sums, children, root, valid, canonical(d, k))
        m = pdf_within_bound(got, ref, depth, zero, valid)
        if k == 0:
            depth0 = depth; ok |= m
        elif exact_phi is not None:
            ok |= m & ~exact_phi
        else:
            ok |= m
    return ok, depth0


def sample_reference(sums, children, root, valid, rnd, craft=None, rng=None):
    """DTree::sample with replayed uniforms (one per level, two at the leaf; 0.5 past the end), float32 -> (canonical (n, 2), levels).
    craft = (level, kind) per query (level -1: none) rewrites that level's uniform before it is drawn, in place in `rnd`: kind 0 = the float32
    partial / total boundary itself; kind 1 / 2 = a uniform whose re-stretched value equals the topLeft / partial (lower branch) or topRight / partial
    (upper branch) boundary, when one exists within a few ulps (otherwise kind 0)."""
    sums = np.asarray(sums, f32); children = np.asarray(children, np.int64)
    n, stride = rnd.shape
    cur = np.zeros(n, np.int64); node = np.asarray(root, np.int64).copy(); levels = np.zeros(n, np.int64)
    bx = np.zeros(n, np.uint64); by = np.zeros(n, np.uint64); res = np.zeros((n, 2), f32)

    def next1(ix):
        v = np.where(cur[ix] < stride, rnd[ix, np.minimum(cur[ix], stride - 1)], f32(0.5)).astype(f32); cur[ix] += 1
        return v
    inv = np.nonzero(~np.asarray(valid))[0]
    res[inv, 0] = next1(inv); res[inv, 1] = next1(inv)
    act = np.nonzero(valid)[0]
    with np.errstate(all="ignore"):
        while len(act):
            s = sums[node[act]]
            tl, tr = s[:, 0], s[:, 1]
            partial = (tl + s[:, 2]).astype(f32); total = (partial + tr + s[:, 3]).astype(f32)
            bad = ~(total > f32(0))
            ib = act[bad]
            res[ib, 0] = next1(ib); res[ib, 1] = next1(ib)
            act, s, tl, tr, partial, total = act[~bad], s[~bad], tl[~bad], tr[~bad], partial[~bad], total[~bad]
            b1 = (partial / total).astype(f32)
            if craft is not None:
                lv, kind = craft
                hit = np.nonzero(lv[act] == levels[act])[0]
                for j in hit:
                    i = act[j]; u = b1[j]
                    if kind[i] == 1 and b1[j] > 0 and partial[j] > 0:
                        u = _solve(lambda v: v < b1[j] and f32(v / b1[j]) == f32(tl[j] / partial[j]), f32(f32(tl[j] / partial[j]) * b1[j]), b1[j])
                    elif kind[i] == 2 and b1[j] < 1 and total[j] - partial[j] > 0:
                        b2 = f32(tr[j] / f32(total[j] - partial[j]))
                        u = _solve(lambda v: v >= b1[j] and f32(f32(v - b1[j]) / f32(f32(1) - b1[j])) == b2, f32(b1[j] + f32(b2 * f32(f32(1) - b1[j]))), b1[j])
                    if cur[i] < stride and u < f32(1):
                        rnd[i, cur[i]] = u
            smp = next1(act)
            lo1 = smp < b1
            smp = np.where(lo1, smp / b1, (smp - b1) / (f32(1) - b1)).astype(f32)
            part2 = np.where(lo1, partial, (total - partial).astype(f32))
            b2 = (np.where(lo1, tl, tr) / part2).astype(f32)
            lo2 = smp < b2
            idx = (~lo1).astype(np.int64) | ((~lo2).astype(np.int64) << 1)
            bx[act] |= (~lo1).astype(np.uint64) << levels[act].astype(np.uint64)
            by[act] |= (~lo2).astype(np.uint64) << levels[act].astype(np.uint64)
            levels[act] += 1
            nxt = children[node[act], idx]
            leaf = nxt == 0
            il = act[leaf]
            res[il, 0] = next1(il); res[il, 1] = next1(il)
            node[act] = np.where(leaf, node[act], np.asarray(root, np.int64)[act] + nxt)
            act = act[~leaf]
    for L in range(int(levels.max(initial=0)) - 1, -1, -1):
        m = levels > L
        hx = np.where((bx >> np.uint64(L)) & np.uint64(1), f32(0.5), f32(0)).astype(f32)
        hy = np.where((by >> np.uint64(L)) & np.uint64(1), f32(0.5), f32(0)).astype(f32)
        res[m, 0] = (hx[m] + f32(0.5) * res[m, 0]).astype(f32); res[m, 1] = (hy[m] + f32(0.5) * res[m, 1]).astype(f32)
    return np.clip(res, f32(0), f32(1)).astype(f32), levels


def _solve(pred, guess, fallback):
    v = f32(guess)
    for k in range(8):
        for c in (v, ) if k == 0 else (_ulps(v, k), _ulps(v, -k)):
            if 0 <= c < 1 and pred(c):
                return f32(c)
    return f32(fallback)


def _ulps(v, k):
    for _ in range(abs(k)):
        v = np.nextafter(v, f32(np.inf if k > 0 else -np.inf))
    return f32(v)


def sample_uniforms(rng, sums, children, root, valid, n):
    """Replayed uniforms (n, RND_STRIDE): random rows; rows of 0 and of 1 - 2^-24; random rows with single 0 / 1 - 2^-24 entries; and rows whose
    uniform at one level of the path sits exactly on that node's partial / total boundary or re-stretches exactly onto its second boundary."""
    rnd = rng.random((n, RND_STRIDE), dtype=np.float32)
    k = n // 8
    rnd[:k] = 0; rnd[k:2 * k] = ONE_MINUS
    e = rng.integers(0, RND_STRIDE, (2 * k, 2))
    rnd[2 * k + np.arange(k), e[:k, 0]] = 0; rnd[3 * k + np.arange(k), e[k:, 0]] = ONE_MINUS
    _, levels = sample_reference(sums, children, root, valid, rnd.copy())
    lv = np.full(n, -1, np.int64); kind = np.zeros(n, np.int64)
    c = np.arange(4 * k, n)
    lv[c] = (rng.random(len(c)) * np.maximum(levels[c], 1)).astype(np.int64)
    kind[c] = rng.integers(0, 3, len(c))
    sample_reference(sums, children, root, valid, rnd, craft=(lv, kind))
    return rnd


def dtree_trees(O, kind):
    """Sampling D-trees the oracle trains in eight S-tree leaves of the unit box (pool export of the oracle handle, and the leaf of each tree):
      0-5  records in narrow cones (one per leaf; sigma 1e-5 rad) over nine rounds at dTreeThreshold 1e-3, 1e-5 in the last: trees at the depth cap
           of 20 with zero-sum quadrants on every level beside the path; the cones of leaves 0-2 move in the last round, so subdivided quadrants
           of the previous cone are left with zero sums;
      6    untrained before the last reset: the 1e-5 reset subdivides it to the 65 535-node limit (65 536 nodes), then 3000 uniform records
      7    no records in the last round: mean 0, uniform sampling and pdf 1 / 4 pi."""
    f = np.float32
    rng = np.random.default_rng(17)
    o = O.Oracle(O.default_params(), aabb=(np.zeros(3, f), np.ones(3, f)), kind=kind)
    o.reset(20, 0.01)
    o.record(np.full((1, 3), 0.5, f), np.array([[0, 0, 1]], f), np.ones(1, f), np.ones(1, f), weight=np.full(1, 8000, f))
    o.build(); o.refine(1000); o.reset(20, 0.01)
    centers = np.array([[0.25 + 0.5 * (k & 1), 0.25 + 0.5 * ((k >> 1) & 1), 0.25 + 0.5 * (k >> 2)] for k in range(8)], f)
    cone = np.array([[(a + 0.5) / 4096, (b + 0.5) / 4096] for a, b in ((1000, 3000), (2500, 2049), (3333, 100), (17, 1111), (2048, 2047), (4000, 3999))])
    moved = cone.copy(); moved[:3] += 3.0 / 4096

    def rec(leaf, d, rad):
        m = len(d)
        o.record(np.tile(centers[leaf], (m, 1)), d, rad.astype(f), np.ones(m, f), weight=np.ones(m, f))
    rounds = 9
    for r in range(rounds):
        last = r == rounds - 1
        if r:
            o.reset(20, 1e-5 if last else 1e-3)
        for leaf in range(6):
            c = to_dir((moved if last else cone)[leaf:leaf + 1]).astype(np.float64)
            d = c + 1e-5 * rng.normal(size=(4000, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
            bg = rng.normal(size=(400, 3)); bg /= np.linalg.norm(bg, axis=1, keepdims=True)
            rec(leaf, np.concatenate([d, bg]).astype(f), np.concatenate([np.full(4000, 10.0), rng.random(400)]))
        if last:
            u = rng.normal(size=(3000, 3)); u /= np.linalg.norm(u, axis=1, keepdims=True)
            rec(6, u.astype(f), rng.lognormal(0, 1, 3000))
        else:
            rec(7, to_dir(rng.random((500, 2))), rng.lognormal(0, 1, 500))
        o.build()
    e = o.export(0)
    leaves = np.nonzero(e["s_is_leaf"])[0].astype(np.uint32)
    assert len(leaves) == 8
    order = o.lookup(centers)[0]          # the S-tree node of each of the eight leaves
    return o, e, order, np.concatenate([moved, [[0.3, 0.7], [0.6, 0.2]]])


def zero_sum_cells(sums, children, root, rng, per_tree=200):
    """Canonical points at the centres of quadrants with zero sum (with and without children below them) in the tree rooted at `root`."""
    out, internal = [], []
    st = [(0, 0.0, 0.0, 1.0)]
    while st:
        nd, ox, oy, s = st.pop()
        for c in range(4):
            cx, cy = ox + (c & 1) * s / 2, oy + (c >> 1) * s / 2
            ch = int(children[root + nd, c])
            if not sums[root + nd, c] > 0:
                out.append((cx + s / 4, cy + s / 4)); internal.append(ch != 0)
            if ch:
                st.append((ch, cx, cy, s / 2))
    out = np.array(out); internal = np.array(internal)
    if len(out) > per_tree:
        keep = np.concatenate([np.nonzero(internal)[0][:per_tree // 2], rng.choice(len(out), per_tree // 2, replace=False)])
        out, internal = out[keep], internal[keep]
    return out, internal


def pdf_directions(rng, sums, children, root, cone_canon, n_random=2000):
    """Query directions for one tree and which of them have an exact atan2: random; both poles; the phi seam (y = +0 / -0, x < 0 / x > 0);
    canonical x on quadrant boundaries of every level 1..22 near the tree's cone (phi exact: 0, pi/2, pi; and phi of the cone); canonical y = 0.25,
    0.5; centres of zero-sum cells."""
    f = np.float32
    r = rng.normal(size=(n_random, 3)); r /= np.linalg.norm(r, axis=1, keepdims=True)
    d = [r.astype(f)]; ex = [np.zeros(n_random, bool)]
    seam = np.array([[0, 0, 1], [0, 0, -1], [-1, 0, 0.3], [-1, -0.0, 0.3], [1, 0, -0.2], [1, -0.0, -0.2], [-0.5, 0.0, -0.9], [0.5, -0.0, 0.9],
                     [0, 1, 0.1], [0, 1, -0.7]], f)
    d.append(seam); ex.append(np.ones(len(seam), bool))
    cx, cy = cone_canon
    for L in range(1, 23):
        x = f(np.round(cx * 2.0 ** L) / 2.0 ** L)
        z = f(2 * x - 1)
        s = f(np.sqrt(max(0.0, 1 - float(z) ** 2)))
        rows = np.array([[s, 0, z], [-s, 0, z], [-s, -0.0, z], [0, s, z]], f)
        d.append(rows); ex.append(np.ones(len(rows), bool))
        dc = to_dir(np.array([[float(x), cy]])); dc[0, 2] = z
        d.append(dc); ex.append(np.zeros(1, bool))
    zc, _ = zero_sum_cells(sums, children, root, rng)
    if len(zc):
        d.append(to_dir(zc)); ex.append(np.zeros(len(zc), bool))
    return np.concatenate(d).astype(f), np.concatenate(ex)
