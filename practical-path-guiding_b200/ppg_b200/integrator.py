"""Host-side mirror of the reference's integrator plugin surface.

``GuidedPathTracer(props)`` takes the same XML parameter names and string values as
``<integrator type="guided_path">`` (reference: mitsuba/src/integrators/path/guided_path.cpp:1014-1085
plus MonteCarloIntegrator, src/librender/integrator.cpp:190-225), validates them the same way (an unknown
enum string raises, like the reference's ``Assert(false)``) and renders through the C ABI of
libppg_b200.so (include/ppg.h).  All compute happens in the CUDA library; there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import capi
from .scene import SceneDesc


class PpgError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"ppg error {code}: {msg}")
        self.code = code


def _check(lib, rc, allow=()):
    if rc != 0 and rc not in allow:
        raise PpgError(rc, lib.ppg_last_error().decode(errors="replace"))
    return rc


def make_params(props: dict | None = None, **kw) -> capi.PpgParams:
    """Properties -> ppg_params through ppg_params_default / ppg_params_set (values as XML strings)."""
    lib = capi.load_library()
    p = capi.PpgParams()
    lib.ppg_params_default(C.byref(p))
    allp = dict(props or {})
    allp.update(kw)
    for name, value in allp.items():
        if isinstance(value, bool):
            value = "true" if value else "false"
        _check(lib, lib.ppg_params_set(C.byref(p), name.encode(), str(value).encode()))
    _check(lib, lib.ppg_params_validate(C.byref(p)))
    return p


class GuidedPathTracer:
    """CreateInstance(props) + Integrator::render() of the reference plugin, on one GPU."""

    description = "Guided path tracer"

    def __init__(self, props: dict | None = None, device: int = -1, **kw):
        self.lib = capi.load_library()
        self.params = make_params(props, **kw)
        self._h = C.c_void_p()
        _check(self.lib, self.lib.ppg_create(C.byref(self.params), device, C.byref(self._h)))
        self._scene_arrays = None
        self._cb = None
        self.W = self.H = 0

    def close(self):
        if self._h:
            self.lib.ppg_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_scene(self, scene: SceneDesc):
        arrays = capi.SceneArrays(scene)
        _check(self.lib, self.lib.ppg_set_scene(self._h, C.byref(arrays.desc)))
        self._scene_arrays = arrays
        self.W, self.H = scene.film_width, scene.film_height
        return self

    def set_shard(self, rank: int, world_size: int):
        _check(self.lib, self.lib.ppg_set_shard(self._h, rank, world_size))
        return self

    def set_allreduce(self, fn):
        """fn(device_ptr: int, n_floats: int) -> None must sum the fp32 buffer in place over all ranks."""
        def _cb(user, ptr, n):
            try:
                fn(ptr, n)
                return 0
            except Exception as e:  # noqa: BLE001 - must not propagate through C
                print("allreduce callback failed:", e, flush=True)
                return 1
        self._cb = capi.ALLREDUCE_FN(_cb)
        _check(self.lib, self.lib.ppg_set_allreduce(self._h, self._cb, None))
        return self

    def init_nccl(self, rank: int | None = None, world_size: int | None = None, broadcast=None):
        """Create the library's own NCCL communicator (ppg_nccl_unique_id / ppg_nccl_init): collectives then run on the render stream
        without a host round trip.  The 128-byte unique id of rank 0 reaches the other ranks through `broadcast(bytes_or_None) -> bytes`
        (default: torch.distributed.broadcast_object_list on the default process group -- bootstrap plumbing only)."""
        if broadcast is None:
            import torch.distributed as dist
            rank = dist.get_rank() if rank is None else rank
            world_size = dist.get_world_size() if world_size is None else world_size

            def broadcast(b):
                box = [b]
                dist.broadcast_object_list(box, src=0)
                return box[0]
        buf = C.create_string_buffer(128)
        if rank == 0:
            _check(self.lib, self.lib.ppg_nccl_unique_id(buf))
        ident = broadcast(bytes(buf.raw) if rank == 0 else None)
        buf = C.create_string_buffer(ident, 128)
        _check(self.lib, self.lib.ppg_nccl_init(self._h, buf, rank, world_size))
        return self

    def set_clock(self, fn):
        """budgetType=seconds reads fn() -> seconds since the render started (None: the steady clock)."""
        self._clock = capi.CLOCK_FN(lambda user: float(fn())) if fn is not None else C.cast(None, capi.CLOCK_FN)
        _check(self.lib, self.lib.ppg_set_clock(self._h, self._clock, None))
        return self

    def set_film_callback(self, fn):
        """fn(rgb_device_ptr, width, height, passes_rendered) after every performRenderPasses (progressive film)."""
        self._film = capi.FILM_FN(lambda user, ptr, w, h, n: fn(ptr, w, h, n)) if fn is not None else C.cast(None, capi.FILM_FN)
        _check(self.lib, self.lib.ppg_set_film_callback(self._h, self._film, None))
        return self

    def render(self):
        """Integrator::render(): returns (rgb HxWx3 float32 on the host, stats dict)."""
        img = np.empty((self.H, self.W, 3), np.float32)
        st = capi.PpgStats()
        self.last_status = _check(self.lib, self.lib.ppg_render(self._h, img.ctypes.data_as(C.POINTER(C.c_float)), C.byref(st)), allow=(-5,))   # -5: cancelled, partial film
        return img, st.as_dict()

    def render_device(self):
        """Same, film left in HBM: returns (device pointer of W*H*3 floats, stats dict)."""
        ptr = C.c_void_p()
        st = capi.PpgStats()
        self.last_status = _check(self.lib, self.lib.ppg_render_device(self._h, C.byref(ptr), C.byref(st)), allow=(-5,))
        return ptr.value, st.as_dict()

    def cancel(self):
        self.lib.ppg_cancel(self._h)

    def set_destination(self, destination: str):
        """scene->getDestinationFile(): with dumpSDTree=true every non-final iteration writes <destination>-NN.sdt."""
        _check(self.lib, self.lib.ppg_set_destination(self._h, destination.encode()))
        return self

    def dump_sdtree(self, path: str):
        _check(self.lib, self.lib.ppg_dump_sdtree(self._h, path.encode()))

    def export_sdtree(self, which: int = 0):
        """The SD-tree as flat arrays (ppg_export_sdtree), after render() or from inside the film callback; which: 0 = sampling trees,
        1 = building trees.  Returns a dict: s_children (N, 2), tree_first / tree_count / tree_depth /
        tree_sum / tree_weight (N,), adam (N, 6), sums (M, 4), children (M, 4) uint16, aabb (2, 3)."""
        aabb = np.zeros((2, 3), np.float32)
        e, = _sized(self.lib, lambda t: self.lib.ppg_export_sdtree(self._h, which, t, _p(aabb, C.c_float)), [(0, 0)])
        e["aabb"] = aabb
        return e

    def op_emitter_sample_direct(self, ref, ref_n, sample, max_interactions=-1):
        """Scene::sampleAttenuatedEmitterDirect at the points `ref` of this handle's scene (ppg_op_emitter_sample_direct): (d, value, pdf, dist)."""
        f = C.POINTER(C.c_float)
        ref = np.ascontiguousarray(ref, np.float32); ref_n = np.ascontiguousarray(ref_n, np.float32); smp = np.ascontiguousarray(sample, np.float32)
        n = len(ref); d = np.zeros((n, 3), np.float32); val = np.zeros((n, 3), np.float32); pdf = np.zeros(n, np.float32); dist = np.zeros(n, np.float32)
        _check(self.lib, self.lib.ppg_op_emitter_sample_direct(self._h, n, ref.ctypes.data_as(f), ref_n.ctypes.data_as(f), smp.ctypes.data_as(f), max_interactions,
                                                               d.ctypes.data_as(f), val.ctypes.data_as(f), pdf.ctypes.data_as(f), dist.ctypes.data_as(f)))
        return d, val, pdf, dist

    def op_env_pdf(self, d):
        """(light-sampling density incl. the emitter choice, radiance) of the environment emitter for world directions `d` (ppg_op_env_pdf)."""
        f = C.POINTER(C.c_float)
        d = np.ascontiguousarray(d, np.float32); pdf = np.zeros(len(d), np.float32); val = np.zeros((len(d), 3), np.float32)
        _check(self.lib, self.lib.ppg_op_env_pdf(self._h, len(d), d.ctypes.data_as(f), pdf.ctypes.data_as(f), val.ctypes.data_as(f)))
        return pdf, val

    def moment_images(self):
        a = np.empty((self.H, self.W, 4), np.float32)
        b = np.empty_like(a)
        _check(self.lib, self.lib.ppg_get_moment_images(self._h, a.ctypes.data_as(C.POINTER(C.c_float)), b.ctypes.data_as(C.POINTER(C.c_float))))
        return a, b


def torch_allreduce(stream_sync=True):
    """Returns an allreduce callback for ``GuidedPathTracer.set_allreduce`` that runs
    ``torch.distributed.all_reduce`` (NCCL over NVLink/NVSwitch) on the library's device buffer in place."""
    import torch
    import torch.distributed as dist

    class _Ptr:
        def __init__(self, ptr, n):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (ptr, False), "version": 3, "strides": None}

    def fn(ptr, n):
        t = torch.as_tensor(_Ptr(ptr, n), device=torch.device("cuda", torch.cuda.current_device()))
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
        if stream_sync:
            torch.cuda.current_stream().synchronize()
    return fn


# ---- kernel-level operators on caller-supplied tree arrays (ppg_op_*) --------------------------------------

def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


# ppg_sdtree (include/ppg.h) as a dict of arrays, keyed as GuidedPathTracer.export_sdtree returns them: key -> (field, C type, columns)
_SDTREE = dict(s_children=("node_children", C.c_uint32, 2), tree_first=("tree_first", C.c_uint64, 1), tree_count=("tree_count", C.c_uint32, 1),
               tree_depth=("tree_depth", C.c_int32, 1), tree_sum=("tree_sum", C.c_float, 1), tree_weight=("tree_weight", C.c_float, 1),
               adam=("adam", C.c_float, 6), sums=("sums", C.c_float, 4), children=("children", C.c_uint16, 4))
_POOL = ("sums", "children")


def _sdtree(arrays):
    """A ppg_sdtree over `arrays` (keys of _SDTREE; absent or None: NULL), sized and with room for their lengths.  The arrays are converted to
    the C types in the dict, which the struct keeps alive as `.arrays`."""
    t = capi.PpgSdtree()
    for k, (field, ct, w) in _SDTREE.items():
        if arrays.get(k) is None:
            continue
        a = arrays[k] = np.ascontiguousarray(arrays[k], ct).reshape((-1, w) if w > 1 else -1)
        setattr(t, field, _p(a, ct))
        if k in _POOL:
            t.n_pool = t.pool_capacity = len(a)
        else:
            t.n_nodes = t.node_capacity = len(a)
    t.arrays = arrays
    return t


def _sdtree_out(n_nodes, n_pool):
    return _sdtree({k: np.zeros(((n_pool if k in _POOL else n_nodes), w) if w > 1 else n_nodes, ct) for k, (_, ct, w) in _SDTREE.items()})


def _sized(lib, call, caps):
    """call(*trees) with output trees of the capacities caps [(nodes, pool), ...], repeated once at the sizes it reports if they were too small.
    Returns the trees' arrays, trimmed to their sizes."""
    for _ in range(2):
        outs = [_sdtree_out(n, m) for n, m in caps]
        rc = call(*outs)
        if rc != -1 or all(t.n_nodes <= n and t.n_pool <= m for t, (n, m) in zip(outs, caps)):
            break
        caps = [(max(n, t.n_nodes), max(m, t.n_pool)) for t, (n, m) in zip(outs, caps)]
    _check(lib, rc)
    return [{k: v[:t.n_pool] if k in _POOL else v[:t.n_nodes] for k, v in t.arrays.items()} for t in outs]


def op_dtree_pdf(sums, children, tree_first, tree_sum, tree_weight, query_tree, query_dir, device=0):
    lib = capi.load_library()
    t = _sdtree(dict(tree_first=tree_first, tree_sum=tree_sum, tree_weight=tree_weight, sums=sums, children=children))
    qt = np.ascontiguousarray(query_tree, np.uint32); qd = np.ascontiguousarray(query_dir, np.float32)
    out = np.zeros(len(qt), np.float32)
    _check(lib, lib.ppg_op_dtree_pdf(device, t, _p(qt, C.c_uint32), _p(qd, C.c_float), len(qt), _p(out, C.c_float)))
    return out


def op_dtree_sample(sums, children, tree_first, tree_sum, tree_weight, query_tree, rnd, device=0, canonical=False):
    """Sampled directions (n, 3); with canonical=True also the points DTree::sample returns before canonicalToDir, (n, 2)."""
    lib = capi.load_library()
    t = _sdtree(dict(tree_first=tree_first, tree_sum=tree_sum, tree_weight=tree_weight, sums=sums, children=children))
    qt = np.ascontiguousarray(query_tree, np.uint32); rnd = np.ascontiguousarray(rnd, np.float32)
    out = np.zeros((len(qt), 3), np.float32)
    canon = np.zeros((len(qt), 2), np.float32) if canonical else None
    _check(lib, lib.ppg_op_dtree_sample(device, t, _p(qt, C.c_uint32), _p(rnd, C.c_float), rnd.shape[1], len(qt), _p(out, C.c_float),
                                        None if canon is None else _p(canon, C.c_float)))
    return (out, canon) if canonical else out


def op_dtree_record(sums, children, tree_first, tree_weight, rec_tree, rec_dir, rec_radiance, rec_wo_pdf, rec_weight, directional_filter=0, device=0):
    lib = capi.load_library()
    t = _sdtree(dict(tree_first=tree_first, tree_weight=np.array(tree_weight, np.float32), sums=np.array(sums, np.float32), children=children))
    rt = np.ascontiguousarray(rec_tree, np.uint32); rd = np.ascontiguousarray(rec_dir, np.float32)
    rr = np.ascontiguousarray(rec_radiance, np.float32); rp = np.ascontiguousarray(rec_wo_pdf, np.float32); rw = np.ascontiguousarray(rec_weight, np.float32)
    _check(lib, lib.ppg_op_dtree_record(device, t, _p(rt, C.c_uint32), _p(rd, C.c_float), _p(rr, C.c_float), _p(rp, C.c_float), _p(rw, C.c_float), len(rt),
                                        directional_filter))
    return t.arrays["sums"], t.arrays["tree_weight"]


def _c(a, dt):
    return np.ascontiguousarray(a, dt)


TREE_STATS = ("leaves", "leaves_with_nodes", "depth_min", "depth_max", "mean_min", "mean_max", "weight_min", "weight_max",
              "nodes_min", "nodes_max", "depth_sum", "mean_sum", "nodes_sum", "weight_sum")


def op_sdtree_refine_reset(tree, building_weight, threshold, refine=True, reset=True, new_max_depth=20, dtree_threshold=0.01, node_capacity=0, device=0):
    """STree::refine and/or DTree::reset of every leaf through the render's kernels (ppg_op_sdtree_refine_reset).  `tree`: the sampling half of an
    S-tree as a dict of flat arrays (s_children, tree_first/count/depth/sum/weight, adam, sums, children); `building_weight` per node.
    Returns a dict of the new S-tree: s_children, tree_first/count/depth/sum/weight, adam, building_weight (after the refine) and the new
    building trees: build_first/count/depth, build_children, build_sums."""
    lib = capi.load_library()
    t = _sdtree({k: tree.get(k) for k in _SDTREE})
    bw = _c(building_weight, np.float32)
    cap = max(2 * t.n_nodes, 1024)
    s, b = _sized(lib, lambda s, b: lib.ppg_op_sdtree_refine_reset(device, (1 if refine else 0) | (2 if reset else 0), threshold, new_max_depth, dtree_threshold,
                                                                   node_capacity, t, _p(bw, C.c_float), s, b),
                  [(cap, t.n_pool), (cap, max(4 * t.n_pool, 1024))])
    o = {k: s[k] for k in ("s_children", "tree_first", "tree_count", "tree_depth", "tree_sum", "tree_weight", "adam")}
    o["tree_first"] = o["tree_first"].astype(np.uint32)
    o.update(building_weight=b["tree_weight"], build_first=b["tree_first"].astype(np.uint32), build_count=b["tree_count"], build_depth=b["tree_depth"],
             build_children=b["children"], build_sums=b["sums"])
    return o


def op_sdtree_build(s_children, build_first, build_count, build_depth, building_weight, sums, children, device=0):
    """DTree::build of every leaf + "sampling = building" + the distribution statistics through the render's kernels (ppg_op_sdtree_build).
    Returns (sampling sums, sampling children, dict of per-node tree_sum / tree_weight / tree_depth / tree_count / mean_positive, stats dict)."""
    lib = capi.load_library()
    b = _sdtree(dict(s_children=s_children, tree_first=build_first, tree_count=build_count, tree_depth=build_depth, tree_weight=building_weight, sums=sums,
                     children=children))
    s = _sdtree_out(b.n_nodes, b.n_pool)
    mp = np.zeros(b.n_nodes, np.uint8); st = np.zeros(14, np.float64)
    _check(lib, lib.ppg_op_sdtree_build(device, b, s, _p(mp, C.c_uint8), _p(st, C.c_double)))
    e = s.arrays
    per = dict(tree_sum=e["tree_sum"], tree_weight=e["tree_weight"], tree_depth=e["tree_depth"], tree_count=e["tree_count"], mean_positive=mp)
    return e["sums"], e["children"], per, dict(zip(TREE_STATS, st.tolist()))


def op_commit(s_children, aabb_min, aabb_extent, build_first, building_weight, sums, children, vertices, li_final, record_mode=2, spatial_filter=0,
              directional_filter=0, loss=0, seed=0, statistical_weight=1.0, adam_capacity=None, device=0):
    """Vertex::commit of the vertices (n, 6, 4) float32 -- the six float4 the bounce kernel writes -- through the render's commit kernel
    (ppg_op_commit).  Returns (building sums, building weights, sampling-fraction records (m, 6) float32 with the leaf's bits in column 0)."""
    lib = capi.load_library()
    t = _sdtree(dict(s_children=s_children, tree_first=build_first, tree_weight=np.array(building_weight, np.float32), sums=np.array(sums, np.float32),
                     children=children))
    mn = _c(aabb_min, np.float32); ex = _c(aabb_extent, np.float32)
    v = _c(vertices, np.float32).reshape(-1, 24); li = _c(li_final, np.float32).reshape(-1, 4)
    cap = len(v) * 64 if adam_capacity is None else adam_capacity
    rec = np.zeros((max(cap, 1), 6), np.float32); na = C.c_size_t()
    _check(lib, lib.ppg_op_commit(device, record_mode, t, _p(mn, C.c_float), _p(ex, C.c_float), _p(v, C.c_float), len(v), _p(li, C.c_float), len(li),
                                  spatial_filter, directional_filter, loss, seed, statistical_weight, _p(rec, C.c_float), cap, C.byref(na)))
    return t.arrays["sums"], t.arrays["tree_weight"], rec[:min(na.value, cap)]


def op_adam_replay(state, records, loss, leaf_offset=None, leaf_count=None, bucket=False, device=0):
    """The sampling-fraction replay (adam_seq_kernel) of records (m, 6) float32 into the per-node states (n, 6) (ppg_op_adam_replay).  Without
    `bucket` the records of node i are records[leaf_offset[i]:leaf_offset[i] + leaf_count[i]]; with it they are bucketed by leaf first, as the render
    does.  Returns a dict: state, theta, count, cursor, and with `bucket` the buckets (records) and their offsets (leaf_offset)."""
    lib = capi.load_library()
    st = np.array(state, np.float32, copy=True, order="C").reshape(-1, 6); n = len(st)
    rec = _c(records, np.float32).reshape(-1, 6)
    off = None if leaf_offset is None else _c(leaf_offset, np.uint32); cnt = None if leaf_count is None else _c(leaf_count, np.uint32)
    o = dict(theta=np.zeros(n, np.float32), records=np.zeros_like(rec), leaf_offset=np.zeros(n, np.uint32), count=np.zeros(n, np.uint32), cursor=np.zeros(n, np.uint32))
    _check(lib, lib.ppg_op_adam_replay(device, loss, 1 if bucket else 0, _p(st, C.c_float), n, _p(rec, C.c_float), len(rec),
                                       None if off is None else _p(off, C.c_uint32), None if cnt is None else _p(cnt, C.c_uint32), _p(o["theta"], C.c_float),
                                       _p(o["records"], C.c_float), _p(o["leaf_offset"], C.c_uint32), _p(o["count"], C.c_uint32), _p(o["cursor"], C.c_uint32)))
    o["state"] = st
    return o


def op_bvh_build(positions, indices, threads=0):
    """The BVH ppg_set_scene builds, on the host (no device): (nodes (N,8) float32, order (T,) uint32, max depth, milliseconds)."""
    lib = capi.load_library()
    pos = np.ascontiguousarray(positions, np.float32); idx = np.ascontiguousarray(indices, np.uint32)
    nt = len(idx); nodes = np.zeros((2 * nt + 1, 8), np.float32); order = np.zeros(nt, np.uint32)
    n = C.c_size_t(); depth = C.c_int(); ms = C.c_double()
    _check(lib, lib.ppg_op_bvh_build(_p(pos, C.c_float), _p(idx, C.c_uint32), nt, threads, _p(nodes, C.c_float), len(nodes), _p(order, C.c_uint32),
                                     C.byref(n), C.byref(depth), C.byref(ms)))
    return nodes[:n.value], order, depth.value, ms.value


def op_stree_lookup(node_children, aabb_min, aabb_extent, points, device=0):
    lib = capi.load_library()
    t = _sdtree(dict(s_children=node_children))
    pts = np.ascontiguousarray(points, np.float32); mn = np.ascontiguousarray(aabb_min, np.float32); ex = np.ascontiguousarray(aabb_extent, np.float32)
    leaf = np.zeros(len(pts), np.uint32); size = np.zeros((len(pts), 3), np.float32)
    _check(lib, lib.ppg_op_stree_lookup(device, t, _p(mn, C.c_float), _p(ex, C.c_float), _p(pts, C.c_float), len(pts), _p(leaf, C.c_uint32), _p(size, C.c_float)))
    return leaf, size
