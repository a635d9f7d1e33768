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
        nn, nq = C.c_size_t(), C.c_size_t()
        rc = self.lib.ppg_export_sdtree(self._h, which, 0, C.byref(nn), None, None, None, None, None, None, None, 0, C.byref(nq), None, None, None)
        _check(self.lib, rc, allow=(-1,) if nn.value or nq.value else ())      # -1 with the sizes filled in: the arrays were too small
        N, M = nn.value, nq.value
        e = dict(s_children=np.zeros((N, 2), np.uint32), tree_first=np.zeros(N, np.uint64), tree_count=np.zeros(N, np.uint32), tree_depth=np.zeros(N, np.int32),
                 tree_sum=np.zeros(N, np.float32), tree_weight=np.zeros(N, np.float32), adam=np.zeros((N, 6), np.float32), sums=np.zeros((M, 4), np.float32),
                 children=np.zeros((M, 4), np.uint16), aabb=np.zeros((2, 3), np.float32))
        P = lambda k, t: e[k].ctypes.data_as(C.POINTER(t))
        _check(self.lib, self.lib.ppg_export_sdtree(self._h, which, N, C.byref(nn), P("s_children", C.c_uint32), P("tree_first", C.c_uint64), P("tree_count", C.c_uint32),
                                                    P("tree_depth", C.c_int32), P("tree_sum", C.c_float), P("tree_weight", C.c_float), P("adam", C.c_float),
                                                    M, C.byref(nq), P("sums", C.c_float), P("children", C.c_uint16), P("aabb", C.c_float)))
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


def op_dtree_pdf(sums, children, tree_first, tree_sum, tree_weight, query_tree, query_dir, device=0):
    lib = capi.load_library()
    sums = np.ascontiguousarray(sums, np.float32); children = np.ascontiguousarray(children, np.uint16)
    tf = np.ascontiguousarray(tree_first, np.uint32); ts = np.ascontiguousarray(tree_sum, np.float32); tw = np.ascontiguousarray(tree_weight, np.float32)
    qt = np.ascontiguousarray(query_tree, np.uint32); qd = np.ascontiguousarray(query_dir, np.float32)
    out = np.zeros(len(qt), np.float32)
    _check(lib, lib.ppg_op_dtree_pdf(device, _p(sums, C.c_float), _p(children, C.c_uint16), len(sums), _p(tf, C.c_uint32), _p(ts, C.c_float),
                                     _p(tw, C.c_float), len(tf), _p(qt, C.c_uint32), _p(qd, C.c_float), len(qt), _p(out, C.c_float)))
    return out


def op_dtree_sample(sums, children, tree_first, tree_sum, tree_weight, query_tree, rnd, device=0, canonical=False):
    """Sampled directions (n, 3); with canonical=True also the points DTree::sample returns before canonicalToDir, (n, 2)."""
    lib = capi.load_library()
    sums = np.ascontiguousarray(sums, np.float32); children = np.ascontiguousarray(children, np.uint16)
    tf = np.ascontiguousarray(tree_first, np.uint32); ts = np.ascontiguousarray(tree_sum, np.float32); tw = np.ascontiguousarray(tree_weight, np.float32)
    qt = np.ascontiguousarray(query_tree, np.uint32); rnd = np.ascontiguousarray(rnd, np.float32)
    out = np.zeros((len(qt), 3), np.float32)
    canon = np.zeros((len(qt), 2), np.float32) if canonical else None
    _check(lib, lib.ppg_op_dtree_sample(device, _p(sums, C.c_float), _p(children, C.c_uint16), len(sums), _p(tf, C.c_uint32), _p(ts, C.c_float),
                                        _p(tw, C.c_float), len(tf), _p(qt, C.c_uint32), _p(rnd, C.c_float), rnd.shape[1], len(qt), _p(out, C.c_float),
                                        None if canon is None else _p(canon, C.c_float)))
    return (out, canon) if canonical else out


def op_dtree_record(sums, children, tree_first, tree_weight, rec_tree, rec_dir, rec_radiance, rec_wo_pdf, rec_weight, directional_filter=0, device=0):
    lib = capi.load_library()
    sums = np.array(sums, np.float32, copy=True, order="C"); children = np.ascontiguousarray(children, np.uint16)
    tf = np.ascontiguousarray(tree_first, np.uint32); tw = np.array(tree_weight, np.float32, copy=True, order="C")
    rt = np.ascontiguousarray(rec_tree, np.uint32); rd = np.ascontiguousarray(rec_dir, np.float32)
    rr = np.ascontiguousarray(rec_radiance, np.float32); rp = np.ascontiguousarray(rec_wo_pdf, np.float32); rw = np.ascontiguousarray(rec_weight, np.float32)
    _check(lib, lib.ppg_op_dtree_record(device, _p(sums, C.c_float), _p(children, C.c_uint16), len(sums), _p(tf, C.c_uint32), _p(tw, C.c_float), len(tf),
                                        _p(rt, C.c_uint32), _p(rd, C.c_float), _p(rr, C.c_float), _p(rp, C.c_float), _p(rw, C.c_float), len(rt), directional_filter))
    return sums, tw


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
    sch = _c(tree["s_children"], np.uint32); n = len(sch)
    ins = [_c(tree["tree_first"], np.uint32), _c(tree["tree_count"], np.uint32), _c(tree["tree_depth"], np.int32), _c(tree["tree_sum"], np.float32),
           _c(tree["tree_weight"], np.float32), _c(tree["adam"], np.float32), _c(building_weight, np.float32)]
    sums = _c(tree["sums"], np.float32); ch = _c(tree["children"], np.uint16)
    cap, bcap = max(2 * n, 1024), max(4 * len(sums), 1024)
    nn, nb = C.c_size_t(), C.c_size_t()
    for _ in range(2):
        o = dict(s_children=np.zeros((cap, 2), np.uint32), tree_first=np.zeros(cap, np.uint32), tree_count=np.zeros(cap, np.uint32), tree_depth=np.zeros(cap, np.int32),
                 tree_sum=np.zeros(cap, np.float32), tree_weight=np.zeros(cap, np.float32), adam=np.zeros((cap, 6), np.float32), building_weight=np.zeros(cap, np.float32),
                 build_first=np.zeros(cap, np.uint32), build_count=np.zeros(cap, np.uint32), build_depth=np.zeros(cap, np.int32),
                 build_children=np.zeros((bcap, 4), np.uint16), build_sums=np.zeros((bcap, 4), np.float32))
        T = (C.c_uint32, C.c_uint32, C.c_uint32, C.c_int32, C.c_float, C.c_float, C.c_float, C.c_float, C.c_uint32, C.c_uint32, C.c_int32)
        keys = ("s_children", "tree_first", "tree_count", "tree_depth", "tree_sum", "tree_weight", "adam", "building_weight", "build_first", "build_count", "build_depth")
        rc = lib.ppg_op_sdtree_refine_reset(device, (1 if refine else 0) | (2 if reset else 0), threshold, new_max_depth, dtree_threshold, node_capacity,
                                            _p(sch, C.c_uint32), n, *[_p(a, t) for a, t in zip(ins, (C.c_uint32, C.c_uint32, C.c_int32) + (C.c_float,) * 4)],
                                            _p(sums, C.c_float), _p(ch, C.c_uint16), len(sums), cap, C.byref(nn), *[_p(o[k], t) for k, t in zip(keys, T)],
                                            bcap, C.byref(nb), _p(o["build_children"], C.c_uint16), _p(o["build_sums"], C.c_float))
        if rc == -1 and (nn.value > cap or nb.value > bcap):
            cap, bcap = max(cap, nn.value), max(bcap, nb.value)
            continue
        _check(lib, rc)
        break
    o = {k: (v[:nb.value] if k in ("build_children", "build_sums") else v[:nn.value]) for k, v in o.items()}
    return o


def op_sdtree_build(s_children, build_first, build_count, build_depth, building_weight, sums, children, device=0):
    """DTree::build of every leaf + "sampling = building" + the distribution statistics through the render's kernels (ppg_op_sdtree_build).
    Returns (sampling sums, sampling children, dict of per-node tree_sum / tree_weight / tree_depth / tree_count / mean_positive, stats dict)."""
    lib = capi.load_library()
    sch = _c(s_children, np.uint32); n = len(sch)
    bf, bc, bd, bw = _c(build_first, np.uint32), _c(build_count, np.uint32), _c(build_depth, np.int32), _c(building_weight, np.float32)
    sums = _c(sums, np.float32); ch = _c(children, np.uint16)
    ss, sc = np.zeros_like(sums), np.zeros_like(ch)
    per = dict(tree_sum=np.zeros(n, np.float32), tree_weight=np.zeros(n, np.float32), tree_depth=np.zeros(n, np.int32), tree_count=np.zeros(n, np.uint32),
               mean_positive=np.zeros(n, np.uint8))
    st = np.zeros(14, np.float64)
    _check(lib, lib.ppg_op_sdtree_build(device, _p(sch, C.c_uint32), n, _p(bf, C.c_uint32), _p(bc, C.c_uint32), _p(bd, C.c_int32), _p(bw, C.c_float),
                                        _p(sums, C.c_float), _p(ch, C.c_uint16), len(sums), _p(ss, C.c_float), _p(sc, C.c_uint16),
                                        _p(per["tree_sum"], C.c_float), _p(per["tree_weight"], C.c_float), _p(per["tree_depth"], C.c_int32),
                                        _p(per["tree_count"], C.c_uint32), _p(per["mean_positive"], C.c_uint8), _p(st, C.c_double)))
    return ss, sc, per, dict(zip(TREE_STATS, st.tolist()))


def op_commit(s_children, aabb_min, aabb_extent, build_first, building_weight, sums, children, vertices, li_final, record_mode=2, spatial_filter=0,
              directional_filter=0, loss=0, seed=0, statistical_weight=1.0, adam_capacity=None, device=0):
    """Vertex::commit of the vertices (n, 6, 4) float32 -- the six float4 the bounce kernel writes -- through the render's commit kernel
    (ppg_op_commit).  Returns (building sums, building weights, sampling-fraction records (m, 6) float32 with the leaf's bits in column 0)."""
    lib = capi.load_library()
    sch = _c(s_children, np.uint32); mn = _c(aabb_min, np.float32); ex = _c(aabb_extent, np.float32); bf = _c(build_first, np.uint32)
    bw = np.array(building_weight, np.float32, copy=True, order="C"); sums = np.array(sums, np.float32, copy=True, order="C"); ch = _c(children, np.uint16)
    v = _c(vertices, np.float32).reshape(-1, 24); li = _c(li_final, np.float32).reshape(-1, 4)
    cap = len(v) * 64 if adam_capacity is None else adam_capacity
    rec = np.zeros((max(cap, 1), 6), np.float32); na = C.c_size_t()
    _check(lib, lib.ppg_op_commit(device, record_mode, _p(sch, C.c_uint32), len(sch), _p(mn, C.c_float), _p(ex, C.c_float), _p(bf, C.c_uint32), _p(bw, C.c_float),
                                  _p(sums, C.c_float), _p(ch, C.c_uint16), len(sums), _p(v, C.c_float), len(v), _p(li, C.c_float), len(li), spatial_filter,
                                  directional_filter, loss, seed, statistical_weight, _p(rec, C.c_float), cap, C.byref(na)))
    return sums, bw, rec[:min(na.value, cap)]


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
    nc = np.ascontiguousarray(node_children, np.uint32); pts = np.ascontiguousarray(points, np.float32)
    mn = np.ascontiguousarray(aabb_min, np.float32); ex = np.ascontiguousarray(aabb_extent, np.float32)
    leaf = np.zeros(len(pts), np.uint32); size = np.zeros((len(pts), 3), np.float32)
    _check(lib, lib.ppg_op_stree_lookup(device, _p(nc, C.c_uint32), len(nc), _p(mn, C.c_float), _p(ex, C.c_float), _p(pts, C.c_float), len(pts),
                                        _p(leaf, C.c_uint32), _p(size, C.c_float)))
    return leaf, size
