"""Edge cases of the hot path's inputs on the GPU, each against the oracle on the same seeds: ragged film sizes (image blocks that
are not 32x32), unbounded depth, tiny budgets, single-sample passes, the memory cap of the S-tree, lenient normals."""
import numpy as np
import pytest

import oracle_lib as O
from common import assert_render_parity, load_cbox, relmse

pytestmark = pytest.mark.gpu


def _both(sc, props):
    from ppg_b200.integrator import GuidedPathTracer
    g = GuidedPathTracer(props); g.set_scene(sc); img, st = g.render()
    o = O.Oracle(O.params_from_xml(props), sc, kind="port"); ref, ost = o.render()
    return img, st, ref, ost


@pytest.mark.parametrize("w,h", [(100, 70), (33, 65), (31, 17), (1, 1)])
def test_ragged_film_sizes(w, h):
    sc = load_cbox().with_film(w, h)
    props = dict(sc.integrator, budget="28")
    img, st, ref, ost = _both(sc, props)
    assert img.shape == (h, w, 3) and np.isfinite(img).all()
    assert st["total_paths"] == ost["total_paths"] == w * h * 28
    assert abs(st["total_vertices"] - ost["total_vertices"]) <= max(2, 1e-4 * ost["total_vertices"])
    assert_render_parity(img, ref, st, ost, sc, props)


@pytest.mark.parametrize("extra", [dict(maxDepth="-1", rrDepth="3"), dict(maxDepth="2"), dict(maxDepth="1"), dict(rrDepth="1"), dict(strictNormals="false"),
                                   dict(sppPerPass="1", budget="7"), dict(sppPerPass="8", budget="24"), dict(budget="3"), dict(sdTreeMaxMemory="1"),
                                   dict(sTreeThreshold="200", budget="60"), dict(dTreeThreshold="0.1", budget="60"), dict(bsdfSamplingFraction="0.0", budget="60"),
                                   dict(bsdfSamplingFraction="1.0", budget="60")])
def test_parameter_extremes(extra):
    sc = load_cbox(64)
    props = dict(dict(sc.integrator, budget="28"), **extra)
    img, st, ref, ost = _both(sc, props)
    assert np.isfinite(img).all()
    assert st["n_iterations"] == ost["n_iterations"] and [i["passes"] for i in st["iterations"]] == [i["passes"] for i in ost["iterations"]]
    assert abs(st["total_vertices"] - ost["total_vertices"]) <= max(2, 1e-4 * ost["total_vertices"])
    assert_render_parity(img, ref, st, ost, sc, props)
    for a, b in zip(st["iterations"], ost["iterations"]):
        assert abs(a["s_tree_leaves"] - b["s_tree_leaves"]) <= 1


def test_rejected_scene_leaves_the_previous_scene_intact():
    """set_scene(CBOX), then a set_scene that is rejected only after the BVH and the tables are built (a sphere of radius 0; smaller film): it reports
    the error, and the integrator still holds CBOX -- film size and all -- so the next render is bit for bit the render of a fresh integrator (unguided
    single pass, CBOX 128^2, budget = 4).  At these settings renders are deterministic: four fresh integrators on an H100 gave bit-identical films."""
    from ppg_b200 import builtin_scenes as B
    from ppg_b200.integrator import GuidedPathTracer, PpgError
    sc = load_cbox(128)
    props = dict(sc.integrator, budget="4")
    bad = B.cbox_with_analytic_spheres(load_cbox(64))
    bad.spheres = np.array(bad.spheres, np.float32); bad.spheres[0, 3] = 0.0
    g = GuidedPathTracer(props); g.set_scene(sc)
    with pytest.raises(PpgError, match="sphere: bad shape index or radius") as e:
        g.set_scene(bad)
    assert e.value.code == -1 and (g.W, g.H) == (128, 128)
    img, st = g.render()
    ref, sref = GuidedPathTracer(props).set_scene(sc).render()
    assert st["total_paths"] == sref["total_paths"] == 128 * 128 * 4 and st["total_vertices"] == sref["total_vertices"]
    assert img.shape == ref.shape and np.array_equal(img.view(np.uint32), ref.view(np.uint32))
