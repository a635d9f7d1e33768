"""One rank of a sharded GPU render that records what every performRenderPasses left behind (spawned by test_gpu_sharded_passes.py).

All ranks share cuda:0; the library's collectives (ppg_set_shard / ppg_set_allreduce) are staged through the host for gloo, as in
dist_worker.py.  In the film callback of every performRenderPasses -- after the passes, before build_sd_tree, so the building trees hold this
rank's records only -- it saves the passes rendered, the moment images, the sampling export and the building export.  After the render it saves
the image, the stats and the final sampling export.  `render_snapshots` with world = 1 is the same render without a shard: the single-GPU
reference of the tests comes from the same code.

    python sharded_snapshot_worker.py RANK WORLD PORT OUTDIR SCENE WIDTH HEIGHT [key=value ...]

A rank that fails writes its traceback to rank<R>.err and exits at once: it never waits at a barrier, so its peers fail in gloo (the process
group is created with a timeout) instead of waiting for it."""
import json
import os
import sys
import traceback

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "practical-path-guiding_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

COLLECTIVE_TIMEOUT_S = 120


def scene(name, width, height):
    from common import cbox_with_sphere, load_cbox
    if name == "cbox":
        return load_cbox().with_film(width, height)
    if name == "sphere":
        return cbox_with_sphere(subdiv=2).with_film(width, height)
    raise ValueError(name)


def render_snapshots(sc, props, rank=0, world=1, allreduce=None, clock=None):
    """GPU render of this rank's share; returns dict(calls=[{passes_rendered, moments, sampling, building}, ...], img, stats, final)."""
    from ppg_b200.integrator import GuidedPathTracer
    g = GuidedPathTracer(props, device=0)
    g.set_scene(sc)
    if world > 1:
        g.set_shard(rank, world); g.set_allreduce(allreduce)
    calls, errors, state = [], [], {"passes": 0, "reads": 0}

    def film(ptr, w, h, passes_rendered):
        state["passes"] = passes_rendered
        try:
            calls.append(dict(passes_rendered=passes_rendered, moments=g.moment_images(), sampling=g.export_sdtree(0), building=g.export_sdtree(1)))
        except Exception as e:      # noqa: BLE001 - an exception cannot cross the C callback; reported below
            errors.append(repr(e))
    g.set_film_callback(film)
    if clock is not None:
        g.set_clock(lambda: clock(state))
    img, st = g.render()
    final = g.export_sdtree(0)
    g.close()
    if errors:
        raise RuntimeError(f"film callback failed: {errors}")
    return dict(calls=calls, img=img, stats=st, final=final)


def save(path, r):
    a = dict(img=r["img"], stats=np.frombuffer(json.dumps(r["stats"]).encode(), np.uint8), ncalls=len(r["calls"]))
    for k, v in r["final"].items():
        a[f"final.{k}"] = v
    for i, c in enumerate(r["calls"]):
        a[f"c{i}.passes_rendered"] = c["passes_rendered"]
        a[f"c{i}.s1"], a[f"c{i}.s2"] = c["moments"]
        for which in ("sampling", "building"):
            for k, v in c[which].items():
                a[f"c{i}.{which}.{k}"] = v
    np.savez(path, **a)


def load(path):
    z = np.load(path)
    calls = []
    for i in range(int(z["ncalls"])):
        c = dict(passes_rendered=int(z[f"c{i}.passes_rendered"]), moments=(z[f"c{i}.s1"], z[f"c{i}.s2"]), sampling={}, building={})
        for which in ("sampling", "building"):
            pre = f"c{i}.{which}."
            c[which] = {k[len(pre):]: z[k] for k in z.files if k.startswith(pre)}
        calls.append(c)
    return dict(calls=calls, img=z["img"], stats=json.loads(bytes(z["stats"]).decode()), final={k[6:]: z[k] for k in z.files if k.startswith("final.")})


def main():
    rank, world, port, outdir, name, width, height = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3], sys.argv[4], sys.argv[5], int(sys.argv[6]), int(sys.argv[7])
    props = dict(kv.split("=", 1) for kv in sys.argv[8:])
    try:
        import datetime
        import torch
        import torch.distributed as dist
        dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world,
                                timeout=datetime.timedelta(seconds=COLLECTIVE_TIMEOUT_S))

        class _Ptr:
            def __init__(self, ptr, n):
                self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (ptr, False), "version": 3, "strides": None}

        def red(ptr, n):
            t = torch.as_tensor(_Ptr(ptr, n), device="cuda:0")
            c = t.cpu()
            dist.all_reduce(c)
            t.copy_(c)
            torch.cuda.synchronize()
        sc = scene(name, width, height)
        r = render_snapshots(sc, dict(sc.integrator, **props), rank, world, red)
        save(os.path.join(outdir, f"rank{rank}.npz"), r)
    except BaseException:           # noqa: BLE001 - report and leave at once, without a barrier
        with open(os.path.join(outdir, f"rank{rank}.err"), "w") as f:
            f.write(traceback.format_exc())
        sys.stderr.write(traceback.format_exc())
        sys.stderr.flush()
        os._exit(1)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
