"""The product's CUDA device functions (practical-path-guiding_b200/csrc/ppg_device.cuh) compiled for the HOST with g++ (tests/hostdev/: CUDA's own headers supply
float3 / float4, the intrinsics get host meanings) and compared, function by function and bit for bit, with the reference's own code compiled verbatim
(oracle/_ref/libmicrofacet_ref.so) -- or with the oracle's restatement where the reference tree was absent at build time.  The kernels are built with -fmad=false
-prec-div=true -prec-sqrt=true, this harness with -ffp-contract=off: +, -, *, / and sqrt round identically; only the libm calls are the host's here and the
device's on the GPU (their ulps are what the `-m gpu` parity tests allow for).  So: reference source == oracle == the source the kernels are compiled from.
The scenes the device code reads here are packed by the library's own host module (csrc/ppg_scene.cpp, compiled into the harness): the same bytes
ppg_set_scene uploads, so the packing is part of the chain."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import oracle_lib as O
from common import CUDA_INC, ROOT, compile_device_on_host

pytestmark = pytest.mark.skipif(CUDA_INC is None or shutil.which("g++") is None, reason="needs g++ and the CUDA headers")
f32p = C.POINTER(C.c_float)


@pytest.fixture(scope="module")
def dev(tmp_path_factory):
    lib = compile_device_on_host(tmp_path_factory.mktemp("hostdev") / "libdevice_on_host.so")
    lib.dev_scene_open.restype = C.c_void_p; lib.dev_scene_open.argtypes = [C.c_void_p]
    lib.dev_scene_close.restype = None; lib.dev_scene_close.argtypes = [C.c_void_p]
    return lib


class _Packed:
    """A scene packed by pack_scene inside the harness, its SceneView bound to the packed arrays (a context manager)."""

    def __init__(self, dev, scene):
        from ppg_b200 import capi
        self.dev, self.arrays = dev, capi.SceneArrays(scene)
        self.h = dev.dev_scene_open(C.addressof(self.arrays.desc))
        assert self.h, "pack_scene rejected the scene"

    def __enter__(self):
        return self.h

    def __exit__(self, *exc):
        self.dev.dev_scene_close(self.h)


def _truth():
    """The reference's own functions when they were compiled here, the oracle's restatement (bit-equal to them, tests/test_oracle_bsdf.py) otherwise."""
    return O.microfacet("ref" if os.path.exists(O.MFREF_SO) else "port")


def _dirs(rng, n, upper):
    d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    if upper:
        d[:, 2] = np.abs(d[:, 2])
    return np.ascontiguousarray(d, np.float32)


@pytest.mark.parametrize("type_", [0, 1])
@pytest.mark.parametrize("alpha", [0.01, 0.1, 0.6])
def test_device_microfacet_source_equals_the_reference(dev, type_, alpha):
    ref = _truth(); rng = np.random.default_rng(7 + 10 * type_ + int(100 * alpha)); n = 100000
    m, v, wi = _dirs(rng, n, False), _dirs(rng, n, False), _dirs(rng, n, True)
    wi[:500] = [0, 0, 1]; wi[500:1000, 2] = 1e-3 * rng.random(500); wi[500:1000] /= np.linalg.norm(wi[500:1000], axis=1, keepdims=True)
    smp = rng.random((n, 2), dtype=np.float32)
    out = np.zeros(n, np.float32)
    dev.dev_mf_eval.argtypes = [C.c_int, C.c_float, C.c_size_t, f32p, f32p]
    dev.dev_mf_eval(type_, alpha, n, m.ctypes.data_as(f32p), out.ctypes.data_as(f32p)); assert np.array_equal(out, ref.eval(type_, alpha, m))
    dev.dev_mf_smith_g1.argtypes = [C.c_int, C.c_float, C.c_size_t, f32p, f32p, f32p]
    dev.dev_mf_smith_g1(type_, alpha, n, v.ctypes.data_as(f32p), m.ctypes.data_as(f32p), out.ctypes.data_as(f32p)); assert np.array_equal(out, ref.smith_g1(type_, alpha, v, m))
    ma = np.ascontiguousarray(np.abs(m))
    dev.dev_mf_pdf.argtypes = [C.c_int, C.c_float, C.c_size_t, f32p, f32p, f32p]
    dev.dev_mf_pdf(type_, alpha, n, wi.ctypes.data_as(f32p), ma.ctypes.data_as(f32p), out.ctypes.data_as(f32p)); assert np.array_equal(out, ref.pdf(type_, alpha, wi, ma))
    mo = np.zeros((n, 3), np.float32); po = np.zeros(n, np.float32)
    dev.dev_mf_sample.argtypes = [C.c_int, C.c_float, C.c_size_t, f32p, f32p, f32p, f32p]
    dev.dev_mf_sample(type_, alpha, n, wi.ctypes.data_as(f32p), smp.ctypes.data_as(f32p), mo.ctypes.data_as(f32p), po.ctypes.data_as(f32p))
    mr, pr = ref.sample(type_, alpha, wi, smp)
    ok = np.isfinite(mr).all(axis=1)
    assert ok.mean() > 0.999 and np.array_equal(mo[ok], mr[ok]) and np.array_equal(po[ok], pr[ok])


def test_device_helper_sources_equal_the_reference(dev):
    ref = _truth(); rng = np.random.default_rng(3); n = 100000
    x = np.concatenate([rng.uniform(-0.999999, 0.999999, n), rng.uniform(-6, 6, 1000)]).astype(np.float32)
    a = np.zeros_like(x); b = np.zeros_like(x)
    dev.dev_erf.argtypes = [C.c_size_t, f32p, f32p, f32p]
    dev.dev_erf(len(x), x.ctypes.data_as(f32p), a.ctypes.data_as(f32p), b.ctypes.data_as(f32p))
    er, eir = ref.erf(x)
    assert np.array_equal(a, er) and np.array_equal(b[np.abs(x) < 1], eir[np.abs(x) < 1])
    c = np.concatenate([rng.uniform(-1, 1, n), [0.0, 1.0, -1.0, 1e-6]]).astype(np.float32)
    f = np.zeros_like(c); ct = np.zeros_like(c)
    dev.dev_fresnel_dielectric_ext.argtypes = [C.c_size_t, f32p, C.c_float, f32p, f32p]
    for eta in (1.0, 1.5046 / 1.000277, 1 / 1.5, 1.33):
        dev.dev_fresnel_dielectric_ext(len(c), c.ctypes.data_as(f32p), eta, f.ctypes.data_as(f32p), ct.ctypes.data_as(f32p))
        fr, tr = ref.fresnel_dielectric_ext(c, eta)
        assert np.array_equal(f, fr) and np.array_equal(ct, tr)
    ca = np.ascontiguousarray(np.abs(c)); out3 = np.zeros((len(c), 3), np.float32)
    dev.dev_fresnel_conductor_exact.argtypes = [C.c_size_t, f32p, f32p, f32p, f32p]
    for eta, k in (((0.2, 0.9, 1.1), (3.9, 2.4, 2.2)), ((1.65746, 0.880369, 0.521229), (9.22387, 6.26952, 4.837)), ((0, 0, 0), (1, 1, 1))):
        e = np.float32(eta); kk = np.float32(k)
        dev.dev_fresnel_conductor_exact(len(c), ca.ctypes.data_as(f32p), e.ctypes.data_as(f32p), kk.ctypes.data_as(f32p), out3.ctypes.data_as(f32p))
        assert np.array_equal(out3, ref.fresnel_conductor_exact(ca, eta, k))
    d = _dirs(rng, n, False); d[:3] = np.eye(3)
    bo = np.zeros_like(d); co = np.zeros_like(d)
    dev.dev_coordinate_system.argtypes = [C.c_size_t, f32p, f32p, f32p]
    dev.dev_coordinate_system(n, d.ctypes.data_as(f32p), bo.ctypes.data_as(f32p), co.ctypes.data_as(f32p))
    br, cr = ref.coordinate_system(d)
    assert np.array_equal(bo, br) and np.array_equal(co, cr)
    smp = rng.random((n, 2), dtype=np.float32); smp[:3] = [[0.5, 0.5], [0, 0], [0.99999994, 0.5]]
    vo = np.zeros((n, 3), np.float32)
    dev.dev_square_to_cosine_hemisphere.argtypes = [C.c_size_t, f32p, f32p]
    dev.dev_square_to_cosine_hemisphere(n, smp.ctypes.data_as(f32p), vo.ctypes.data_as(f32p))
    assert np.array_equal(vo, ref.square_to_cosine_hemisphere(smp))


def test_device_triangle_test_and_transmittance_sources_equal_the_reference(dev):
    """tri_intersect on the accel rows pack_scene writes, fed with the reference's own TriAccel constants: same hit decision, same (t, u, v) as TriAccel::rayIntersect."""
    truth = C.CDLL(O.MFREF_SO) if os.path.exists(O.MFREF_SO) else O.load("port"); name = "mfref_triaccel" if os.path.exists(O.MFREF_SO) else "ppgo_triaccel"
    rng = np.random.default_rng(5); n = 200000
    A = rng.normal(size=(n, 3)).astype(np.float32) * 10; B = A + rng.normal(size=(n, 3)).astype(np.float32); Cc = A + rng.normal(size=(n, 3)).astype(np.float32)
    B[:100] = A[:100]
    w = rng.random((n, 2)); tgt = A + (B - A) * (w[:, :1] * 1.4 - 0.2) + (Cc - A) * (w[:, 1:] * 1.4 - 0.2)
    o = (tgt + rng.normal(size=(n, 3)) * 5).astype(np.float32); d = tgt - o; d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    mint = np.full(n, 1e-4, np.float32); maxt = np.where(rng.random(n) < 0.1, 3.0, np.inf).astype(np.float32)
    k = np.zeros(n, np.int32); c9 = np.zeros((n, 9), np.float32); hit = np.zeros(n, np.uint8); tuv = np.zeros((n, 3), np.float32)
    fn = getattr(truth, name); fn.argtypes = [C.c_size_t] + [f32p] * 7 + [C.POINTER(C.c_int), f32p, C.POINTER(C.c_ubyte), f32p]
    arrs = [np.ascontiguousarray(a, np.float32) for a in (A, B, Cc, o, d, mint, maxt)]
    fn(n, *[a.ctypes.data_as(f32p) for a in arrs], k.ctypes.data_as(C.POINTER(C.c_int)), c9.ctypes.data_as(f32p), hit.ctypes.data_as(C.POINTER(C.c_ubyte)), tuv.ctypes.data_as(f32p))
    hit2 = np.zeros(n, np.uint8); tuv2 = np.zeros((n, 3), np.float32)
    dev.dev_tri_intersect.argtypes = [C.c_size_t, C.POINTER(C.c_int), f32p, f32p, f32p, f32p, f32p, C.POINTER(C.c_ubyte), f32p]
    dev.dev_tri_intersect(n, k.ctypes.data_as(C.POINTER(C.c_int)), c9.ctypes.data_as(f32p), arrs[3].ctypes.data_as(f32p), arrs[4].ctypes.data_as(f32p), mint.ctypes.data_as(f32p),
                          maxt.ctypes.data_as(f32p), hit2.ctypes.data_as(C.POINTER(C.c_ubyte)), tuv2.ctypes.data_as(f32p))
    assert 0.1 < hit.mean() < 0.5 and np.array_equal(hit, hit2) and np.array_equal(tuv[hit == 1], tuv2[hit == 1])
    lut = np.ascontiguousarray(ROUGH_TABLES["beckmann 1.49 0.1"], np.float32)
    cs = np.concatenate([rng.uniform(-0.2, 1, 100000), [0.0, 1.0]]).astype(np.float32)
    a = np.zeros_like(cs); b = np.zeros_like(cs)
    dev.dev_rough_transmittance.argtypes = [C.c_size_t, f32p, f32p, f32p]
    dev.dev_rough_transmittance(len(cs), cs.ctypes.data_as(f32p), lut.ctypes.data_as(f32p), a.ctypes.data_as(f32p))
    port = O.load("port"); port.ppgo_rough_transmittance.argtypes = [C.c_size_t, f32p, f32p, f32p]
    port.ppgo_rough_transmittance(len(cs), cs.ctypes.data_as(f32p), lut.ctypes.data_as(f32p), b.ctypes.data_as(f32p))
    assert np.array_equal(a, b)                                                     # (the oracle's lookup is itself checked against evalCubicInterp1D, tests/test_oracle_bsdf.py)


def _material(name):
    """One BSDF configuration of the hot path (DESIGN.md 1.1) with the wrappers that change its arithmetic: (ppg_bsdf, tables).  The rough-plastic rows and
    tables are what ppg_b200.scene.make_roughplastic reduces from the reference's data files, stored in tests/golden/reference_rough_transmittance.npz."""
    from ppg_b200 import scene as S
    mk = lambda **kw: O.make_bsdf(**kw)
    if name in ROUGHPLASTICS:
        row, tables = ROUGH_TABLES[name + " row"], np.ascontiguousarray(ROUGH_TABLES[name + " tables"], np.float32)
        from ppg_b200 import rtrans
        if os.path.exists(os.path.join(rtrans._DATA_DIR, "ggx.dat")):                    # the reference's tables: recompute and compare
            t = []
            assert np.array_equal(S.make_roughplastic(*ROUGHPLASTICS[name], t), row) and np.array_equal(np.asarray(t, np.float32), tables)
        return O.bsdf_from_row(row), tables
    if name == "plastic nonlinear":
        return O.bsdf_from_row(S.make_plastic(0, (0.6, 0.3, 0.2), (1, 1, 1), 1.49, True)), None
    if name == "plastic twosided":
        return O.bsdf_from_row(S.make_plastic(1, (0.2, 0.3, 0.6), (0.8, 0.8, 0.8), 1.9, False)), None
    if name.startswith("mask"):
        m = mk(type=0, flags=1 | 4, reflectance=(0.6, 0.5, 0.4)) if "diffuse" in name else mk(type=4, flags=4, reflectance=(1, 1, 1), eta=(0.2, 0.9, 1.1), k=(3.9, 2.4, 2.2), alpha=0.2, distribution=1)
        op = (0.6, 0.5, 0.7) if "diffuse" in name else (0.3, 0.3, 0.3)
        m.opacity[0], m.opacity[1], m.opacity[2] = op
        return m, None
    return mk(**SIMPLE[name]), None


SIMPLE = {
    "diffuse": dict(type=0, reflectance=(0.6, 0.5, 0.4)),
    "diffuse twosided": dict(type=0, flags=1, reflectance=(0.6, 0.5, 0.4)),
    "black (emitter without a BSDF)": dict(type=1, reflectance=(0, 0, 0)),                 # (the loaders hand NULL_BLACK over with zero reflectance)
    "dielectric bk7": dict(type=2, reflectance=(1, 1, 1), transmittance=(1, 1, 1), eta=(1.5046 / 1.000277,) * 3),
    "conductor": dict(type=3, reflectance=(1, 1, 1), eta=(0.2, 0.9, 1.1), k=(3.9, 2.4, 2.2)),
    "roughconductor ggx 0.1 twosided": dict(type=4, flags=1, reflectance=(1, 1, 1), eta=(1.65746, 0.880369, 0.521229), k=(9.22387, 6.26952, 4.837), alpha=0.1, distribution=1),
    "roughconductor beckmann 0.3": dict(type=4, reflectance=(0.9, 0.9, 0.9), eta=(0.2, 0.9, 1.1), k=(3.9, 2.4, 2.2), alpha=0.3, distribution=0),
    "roughdielectric ggx 0.1": dict(type=6, reflectance=(1, 1, 1), transmittance=(1, 1, 1), eta=(1.5,) * 3, alpha=0.1, distribution=1),
    "roughdielectric beckmann 0.3 tinted": dict(type=6, reflectance=(0.9, 0.8, 1), transmittance=(0.7, 0.9, 1), eta=(1.33,) * 3, alpha=0.3, distribution=0),
    "thindielectric": dict(type=8, reflectance=(1, 1, 1), transmittance=(0.9, 0.95, 1), eta=(1.5,) * 3),
}
ROUGHPLASTICS = {"roughplastic ggx 0.2": (0, (0.256, 0.013, 0.08), (1, 1, 1), 1.5 / 1.000277, 0.2, 1, False),
                 "roughplastic beckmann 0.4 nonlinear twosided": (1, (0.5, 0.4, 0.3), (0.9, 0.9, 0.9), 1.49, 0.4, 0, True)}
ROUGH_TABLES = dict(np.load(os.path.join(ROOT, "tests", "golden", "reference_rough_transmittance.npz")))
MATERIALS = list(SIMPLE) + list(ROUGHPLASTICS) + ["plastic nonlinear", "plastic twosided", "mask over twosided diffuse", "mask over roughconductor"]


@pytest.mark.parametrize("name", MATERIALS)
def test_device_bsdf_sources_equal_the_oracle(dev, name):
    """bsdf_eval / bsdf_pdf / bsdf_sample of csrc/ppg_device.cuh (host-compiled) against the oracle's restatement of the same Mitsuba models, on the same directions and
    random numbers: every value bit for bit -- eval and pdf on 10^5 direction pairs over the whole sphere (both sides of the surface), sampling on 10^5 (wi, u) pairs
    incl. the model's own extra draw (roughdielectric) and the delta / null lobes.  The device side is the material as load_bsdf reads it from the record
    pack_scene writes for it (a one-triangle scene with the material's tables)."""
    b, tables = _material(name)
    nt = tables.size // 100 if tables is not None else 0
    rng = np.random.default_rng(MATERIALS.index(name)); n = 100000
    wi, wo = _dirs(rng, n, False), _dirs(rng, n, False)
    wi[:200, 2] = np.abs(wi[:200, 2]) * 1e-3; wi[:200] /= np.linalg.norm(wi[:200], axis=1, keepdims=True)         # grazing incidence
    wo[200:1200] = wi[200:1200] * [-1, -1, 1]                                                                    # the mirror direction (delta lobes evaluate to 0 without the discrete measure)
    tp = tables.ctypes.data_as(f32p) if tables is not None else None
    ev = np.zeros((n, 3), np.float32); pd = np.zeros(n, np.float32)
    dev.dev_bsdf_eval_pdf.argtypes = [C.POINTER(type(b)), C.c_size_t, f32p, f32p, f32p, f32p, f32p, C.c_uint32]
    assert dev.dev_bsdf_eval_pdf(C.byref(b), n, wi.ctypes.data_as(f32p), wo.ctypes.data_as(f32p), ev.ctypes.data_as(f32p), pd.ctypes.data_as(f32p), tp, nt) == 0
    ev0, pd0 = O.bsdf_eval_pdf(b, wi, wo, tables=tables)
    assert np.array_equal(ev.view(np.uint32), ev0.view(np.uint32)) and np.array_equal(pd.view(np.uint32), pd0.view(np.uint32))
    smp = rng.random((n, 2), dtype=np.float32)
    so = np.zeros((n, 3), np.float32); sw = np.zeros((n, 3), np.float32); sp = np.zeros(n, np.float32); sd = np.zeros(n, np.uint8)
    dev.dev_bsdf_sample.argtypes = [C.POINTER(type(b)), C.c_size_t, f32p, f32p, f32p, f32p, f32p, C.POINTER(C.c_ubyte), f32p, C.c_uint32]
    assert dev.dev_bsdf_sample(C.byref(b), n, wi.ctypes.data_as(f32p), smp.ctypes.data_as(f32p), so.ctypes.data_as(f32p), sw.ctypes.data_as(f32p), sp.ctypes.data_as(f32p),
                               sd.ctypes.data_as(C.POINTER(C.c_ubyte)), tp, nt) == 0
    so0, sw0, sp0, sd0 = O.bsdf_sample(b, wi, smp, tables=tables)
    lit = (sw0 != 0).any(axis=1)                                                    # a failed sample carries weight 0; its wo is unspecified on both sides
    assert np.array_equal(lit, (sw != 0).any(axis=1)) and (lit.mean() > 0.2 or b.type == 1)
    assert np.array_equal(sw[lit].view(np.uint32), sw0[lit].view(np.uint32)) and np.array_equal(so[lit].view(np.uint32), so0[lit].view(np.uint32))
    assert np.array_equal(sp[lit].view(np.uint32), sp0[lit].view(np.uint32)) and np.array_equal(sd[lit], sd0[lit])


def test_device_texture_source_equals_the_oracle(dev):
    """tex_eval (BitmapTexture::eval -> TMIPMap::evalBilinear, level 0) and tex_gradient_lum (evalGradientBilinear -> the luminances BumpMap::getFrame uses) of the
    device source on the textures of the cbox-textured fixture (RGB and one-channel, repeat / clamp / mirror wrapping, uv scale and offset), read from the
    whole scene as pack_scene packs it, against the oracle's texture code at 10^5 texture coordinates reaching far outside [0, 1]^2: bit for bit."""
    from common import load_fixture_scene
    sc = load_fixture_scene("cbox-textured")
    o = O.Oracle(O.params_from_xml(sc.integrator), sc, kind="port")
    lib = O.load("port"); lib.ppgo_texture_eval.argtypes = [C.c_void_p, C.c_uint32, C.c_size_t, f32p, f32p, f32p]
    arrays = o.scene_arrays
    rng = np.random.default_rng(17); n = 100000
    uv = (rng.random((n, 2)) * 6 - 2.5).astype(np.float32); uv[:4] = [[0, 0], [1, 1], [0.5, 0.5], [np.nan, 0.3]]
    dev.dev_texture_eval.argtypes = [C.c_void_p, C.c_uint32, C.c_size_t, f32p, f32p, f32p]
    assert len(sc.textures) == 3
    with _Packed(dev, sc) as h:
        for k in range(len(sc.textures)):
            a = np.zeros((n, 3), np.float32); ga = np.zeros((n, 2), np.float32); b = np.zeros((n, 3), np.float32); gb = np.zeros((n, 2), np.float32)
            assert lib.ppgo_texture_eval(o.h, k, n, uv.ctypes.data_as(f32p), a.ctypes.data_as(f32p), ga.ctypes.data_as(f32p)) == 0
            assert dev.dev_texture_eval(h, k, n, uv.ctypes.data_as(f32p), b.ctypes.data_as(f32p), gb.ctypes.data_as(f32p)) == 0
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)) and np.array_equal(ga.view(np.uint32), gb.view(np.uint32)), k
            assert np.abs(a[4:]).max() > 0.1 and np.abs(ga[4:]).max() > 0


def test_device_discrete_sampling_source_equals_the_reference(dev):
    """cdf_sample + the sample reuse of the device's sample_emitter_direct on the normalised table pack_scene builds (running sum, normalize_cdf), against
    DiscreteDistribution::sampleReuse of the reference compiled verbatim (or the oracle's, bit-equal to it): table, index and reused sample bit for bit,
    zero-weight entries skipped the same way."""
    have_ref = os.path.exists(O.MFREF_SO)
    truth = C.CDLL(O.MFREF_SO) if have_ref else O.load("port"); name = "mfref_discrete" if have_ref else "ppgo_discrete"
    u32p = C.POINTER(C.c_uint32)
    rng = np.random.default_rng(44)
    for ne in (1, 3, 40, 1000):
        w = rng.lognormal(0, 2, ne).astype(np.float32)
        if ne > 2:
            w[rng.integers(0, ne, max(1, ne // 5))] = 0; w[0] = 0; w[-1] = 0
            w[ne // 2] = max(w[ne // 2], 1e-3)
        n = 100000
        smp = rng.random(n, dtype=np.float32); smp[0] = 0.0
        pdf = np.zeros(ne, np.float32); s = C.c_float(); idx = np.zeros(n, np.uint32); reuse = np.zeros(n, np.float32)
        fn = getattr(truth, name); fn.argtypes = [C.c_size_t, f32p, C.c_size_t, f32p, f32p, C.POINTER(C.c_float), u32p, f32p]
        fn(ne, w.ctypes.data_as(f32p), n, smp.ctypes.data_as(f32p), pdf.ctypes.data_as(f32p), C.byref(s), idx.ctypes.data_as(u32p), reuse.ctypes.data_as(f32p))
        cdf = np.zeros(ne + 1, np.float32)
        dev.dev_emitter_cdf.argtypes = [C.c_size_t, f32p, f32p]
        dev.dev_emitter_cdf(ne, w.ctypes.data_as(f32p), cdf.ctypes.data_as(f32p))
        assert np.array_equal(np.diff(cdf), pdf) or np.allclose(np.diff(cdf), pdf, rtol=0, atol=0)
        idx2 = np.zeros(n, np.uint32); reuse2 = np.zeros(n, np.float32)
        dev.dev_discrete.argtypes = [C.c_size_t, f32p, C.c_size_t, f32p, u32p, f32p]
        dev.dev_discrete(ne, cdf.ctypes.data_as(f32p), n, smp.ctypes.data_as(f32p), idx2.ctypes.data_as(u32p), reuse2.ctypes.data_as(f32p))
        assert np.array_equal(idx, idx2) and np.array_equal(reuse.view(np.uint32), reuse2.view(np.uint32)), ne


def test_device_sdtree_sources_against_the_reference_trees(dev):
    """stree_lookup (through the prefix table stree_table_kernel builds -- the __global__ function runs here as a plain loop), dtree_pdf, dtree_sample and the
    cylindrical maps of the device source on trees trained by the oracle (the reference's own SD-tree code where oracle/_ref exists): leaf index and voxel size bit
    for bit; sampled directions within 2e-6 (the fold of the per-level origins is the reference's, the two leaf numbers enter in its order); pdf to 2e-6 relative
    (top-down product here, bottom-up recursion there) -- the tolerances of the same comparison on the GPU (tests/test_gpu_parity.py::test_op_*)."""
    from common import load_cbox
    sc = load_cbox(96)
    o = O.Oracle(O.params_from_xml(dict(sc.integrator, budget="60")), sc, kind="ref" if O.have_ref() else "port"); o.render()
    e = o.export(0)
    rng = np.random.default_rng(8); n = 100000
    mn, mx = e["aabb"]; ext = (mx - mn).astype(np.float32)
    pts = (mn + rng.random((n, 3)) * (mx - mn)).astype(np.float32); pts[:8] = [mn, mx, (mn + mx) / 2, mn - 1, mx + 1, [mn[0], mx[1], mn[2]], [mx[0], mn[1], mx[2]], (mn + mx) / 2 + 1e-3]
    leaf, size = o.lookup(pts)
    u32p = C.POINTER(C.c_uint32)
    sch = np.ascontiguousarray(e["s_children"], np.uint32); gl = np.zeros(n, np.uint32); gs = np.zeros((n, 3), np.float32)
    dev.dev_stree_lookup.argtypes = [u32p, C.c_size_t, f32p, f32p, f32p, C.c_size_t, u32p, f32p]
    dev.dev_stree_lookup(sch.ctypes.data_as(u32p), len(sch), np.float32(mn).ctypes.data_as(f32p), ext.ctypes.data_as(f32p), pts.ctypes.data_as(f32p), n, gl.ctypes.data_as(u32p), gs.ctypes.data_as(f32p))
    assert np.array_equal(gl, leaf) and np.array_equal(gs, size) and len(np.unique(leaf)) > 10
    leaves = np.nonzero(e["s_is_leaf"])[0].astype(np.uint32)
    ql = rng.choice(leaves, n).astype(np.uint32)
    d = rng.normal(size=(n, 3)).astype(np.float32); d /= np.linalg.norm(d, axis=1, keepdims=True)
    rnd = rng.random((n, 24), dtype=np.float32)
    pdf = np.zeros(n, np.float32); dirs = np.zeros((n, 3), np.float32)
    sums = np.ascontiguousarray(e["sums"], np.float32); ch = np.ascontiguousarray(e["children"], np.uint16); first = e["tree_first"].astype(np.uint32)
    dev.dev_dtree.argtypes = [f32p, C.POINTER(C.c_uint16), C.c_size_t, u32p, f32p, f32p, u32p, f32p, f32p, C.c_size_t, C.c_size_t, f32p, f32p, f32p]
    dev.dev_dtree(sums.ctypes.data_as(f32p), ch.ctypes.data_as(C.POINTER(C.c_uint16)), len(sums), first.ctypes.data_as(u32p), e["tree_sum"].ctypes.data_as(f32p),
                  e["tree_weight"].ctypes.data_as(f32p), ql.ctypes.data_as(u32p), d.ctypes.data_as(f32p), rnd.ctypes.data_as(f32p), 24, n, pdf.ctypes.data_as(f32p), dirs.ctypes.data_as(f32p), None)
    ref_pdf = o.pdf(ql, d); ref_dir = o.sample(ql, rnd)
    assert np.allclose(pdf, ref_pdf, rtol=2e-6, atol=1e-12) and np.abs(dirs - ref_dir).max() <= 2e-6
    assert (dirs == ref_dir).all(axis=1).mean() > 0.9                              # (mostly bit-equal: same libm here)


def _bsdf_ints(a):
    return a.bsdfs.view(np.int32)          # ppg_bsdf as 28 int32: type 0, flags 1, eta 8-10, table 21, reflectance_texture 25, bump_texture 26


def _shape_of_textured_bsdf(a):
    return int(np.nonzero(_bsdf_ints(a)[a.shapes[:, 2], 25] != 0)[0][0])


def _sphere_on(a, shape, radius=1.0):
    a.extra = np.zeros((1, 6), np.float32); a.extra[0, 3] = radius; a.extra.view(np.int32)[0, 4] = shape
    a.desc.n_spheres = 1; a.desc.spheres = C.cast(a.extra.ctypes.data, type(a.desc.spheres))


def _emitter_shape(a):
    return int(np.nonzero(a.shapes[:, 3] >= 0)[0][0])


INVALID, UNSUPPORTED = -1, -6
# (fixture, change to the description, expected status, part of the message); every validation path of pack_scene
REJECTIONS = {
    "no triangles": ("cbox", lambda a: setattr(a.desc, "n_triangles", 0), INVALID, "needs triangles"),
    "emitters without radiance": ("cbox", lambda a: setattr(a.desc, "area_radiance", None), INVALID, "without its array"),
    "film size 0": ("cbox", lambda a: setattr(a.desc.camera, "film_width", 0), INVALID, "film size"),
    "film size 65536": ("cbox", lambda a: setattr(a.desc.camera, "film_height", 65536), INVALID, "film size"),
    "triangle_shape out of range": ("cbox", lambda a: a.triangle_shape.__setitem__(3, len(a.shapes)), INVALID, "triangle_shape out of range"),
    "vertex index out of range": ("cbox", lambda a: a.indices.__setitem__((5, 1), len(a.positions)), INVALID, "vertex index out of range"),
    "shape bsdf out of range": ("cbox", lambda a: a.shapes.__setitem__((0, 2), len(a.bsdfs)), INVALID, "shape bsdf out of range"),
    "shape emitter out of range": ("cbox", lambda a: a.shapes.__setitem__((0, 3), len(a.radiance)), INVALID, "shape emitter out of range"),
    "unsupported bsdf": ("cbox", lambda a: _bsdf_ints(a).__setitem__((0, 0), 9), UNSUPPORTED, "hot-path scope"),
    "mask around thindielectric": ("cbox", lambda a: _bsdf_ints(a).__setitem__((0, slice(0, 2)), (8, 4)), UNSUPPORTED, "mask around"),
    "roughplastic without a table": ("cbox", lambda a: _bsdf_ints(a).__setitem__((0, 0), 5), INVALID, "rough-transmittance table"),
    "roughplastic table out of range": ("cbox-plastic", lambda a: setattr(a.desc, "n_bsdf_tables", 0), INVALID, "rough-transmittance table"),
    "dielectric without eta": ("cbox", lambda a: _bsdf_ints(a).__setitem__((0, 0), 2), INVALID, "eta > 0"),
    "twosided dielectric": ("cbox", lambda a: (_bsdf_ints(a).__setitem__((0, slice(0, 2)), (2, 1)), a.bsdfs.__setitem__((0, 8), 1.5)), INVALID, "twosided cannot wrap"),
    "texture index out of range": ("cbox", lambda a: _bsdf_ints(a).__setitem__((0, 25), 1), INVALID, "texture index out of range"),
    "texture on a conductor": ("cbox-textured", lambda a: _bsdf_ints(a).__setitem__((int(a.shapes[_shape_of_textured_bsdf(a), 2]), 0), 3), UNSUPPORTED, "only the diffuse reflectance"),
    "bumpmap without texture": ("cbox", lambda a: _bsdf_ints(a).__setitem__((0, 1), 8), INVALID, "displacement texture"),
    "textures without texels": ("cbox-textured", lambda a: setattr(a.desc, "texels", None), INVALID, "without texel data"),
    "texture of width 0": ("cbox-textured", lambda a: a.textures["width"].__setitem__(0, 0), INVALID, "bad size"),
    "texture with 2 channels": ("cbox-textured", lambda a: a.textures["channels"].__setitem__(1, 2), INVALID, "bad size"),
    "texture wrap mode 3": ("cbox-textured", lambda a: a.textures["wrap_v"].__setitem__(2, 3), INVALID, "bad size"),
    "texel range out of bounds": ("cbox-textured", lambda a: setattr(a.desc, "n_texels", len(a.texels) - 1), INVALID, "texel range"),
    "texture on a sphere": ("cbox-textured", lambda a: _sphere_on(a, _shape_of_textured_bsdf(a)), UNSUPPORTED, "analytic sphere"),
    "envmap without texels": ("env", lambda a: setattr(a.desc.envmap, "texels", None), INVALID, "envmap without texel data"),
    "black envmap": ("env", lambda a: a.env_texels.fill(0), INVALID, "completely black"),
    "NaN in the envmap": ("env", lambda a: a.env_texels.__setitem__((3, 5, 1), 0x7E00), INVALID, "nan/inf"),
    "singular world_to_env": ("env", lambda a: [a.desc.envmap.world_to_env.__setitem__(i, 0.0) for i in range(3)], INVALID, "singular world_to_env"),
    "sphere of radius 0": ("spheres", lambda a: a.spheres.__setitem__((0, 3), 0.0), INVALID, "bad shape index or radius"),
    "sphere without a shape": ("spheres", lambda a: a.spheres.view(np.int32).__setitem__((1, 4), -1), INVALID, "bad shape index or radius"),
    "emitter triangle range out of bounds": ("cbox", lambda a: a.shapes.__setitem__((_emitter_shape(a), 1), len(a.indices) + 1), INVALID, "triangle range out of bounds"),
    "2^32 texels": ("cbox-textured", lambda a: (a.textures["width"].__setitem__(0, 65536), a.textures["height"].__setitem__(0, 65536), a.textures["channels"].__setitem__(0, 1),
                                                a.textures["first_texel"].__setitem__(0, 0), setattr(a.desc, "n_texels", 1 << 32)), UNSUPPORTED, "2^32 texels"),
}


def _fixture(name):
    from common import load_cbox, load_fixture_scene
    from ppg_b200 import builtin_scenes as B
    if name == "cbox":
        return load_cbox(32)
    if name == "env":
        return B.env_lit_scene(32)
    if name == "spheres":
        return B.cbox_with_analytic_spheres(load_cbox(32))
    return load_fixture_scene(name, 32)


@pytest.mark.parametrize("case", list(REJECTIONS))
def test_pack_scene_rejects_malformed_scenes(dev, case):
    """pack_scene validates the whole description before anything is uploaded: each malformed variant of a fixture scene gets its documented status and
    message, and the unmodified fixture packs."""
    from ppg_b200 import capi
    fixture, change, code, message = REJECTIONS[case]
    err = C.create_string_buffer(256)
    dev.dev_pack_scene.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
    a = capi.SceneArrays(_fixture(fixture))
    assert dev.dev_pack_scene(C.addressof(a.desc), err, len(err)) == 0, err.value
    change(a)
    assert dev.dev_pack_scene(C.addressof(a.desc), err, len(err)) == code, err.value
    assert message in err.value.decode(), err.value


@pytest.mark.parametrize("scene", ["cbox", "torus"])
def test_closest_hit_on_packed_scenes_equals_brute_force(dev, scene):
    """bvh_intersect on the packed scene -- CBOX: the coplanar-group test, torus: the BVH walk -- against the minimum of the exact triangle test over every
    packed triangle, ties to the lower original index (DESIGN.md 2): the same triangle and the same t for every ray.  On the host __fdividef is an exact
    division, so this checks the packing and the traversal, not the device's approximate pre-filter."""
    from ppg_b200 import builtin_scenes as B
    sc = _fixture("cbox") if scene == "cbox" else B.torus_scene(32)
    rng = np.random.default_rng(21 if scene == "cbox" else 22); n = 20000
    lo, hi = np.asarray(sc.aabb_min, np.float64), np.asarray(sc.aabb_max, np.float64)
    o = (lo + (hi - lo) * (0.02 + 0.96 * rng.random((n, 3)))).astype(np.float32)
    d = rng.normal(size=(n, 3)); d[: n // 10, 1] = 0; d /= np.linalg.norm(d, axis=1, keepdims=True); d = d.astype(np.float32)
    t = np.zeros((n, 2), np.float32); prim = np.zeros((n, 2), np.uint32)
    dev.dev_closest_hit.argtypes = [C.c_void_p, C.c_size_t, f32p, f32p, C.c_float, C.c_float, f32p, C.POINTER(C.c_uint32)]
    with _Packed(dev, sc) as h:
        assert dev.dev_closest_hit(h, n, o.ctypes.data_as(f32p), d.ctypes.data_as(f32p), 1e-4, np.inf, t.ctypes.data_as(f32p), prim.ctypes.data_as(C.POINTER(C.c_uint32))) == 0
    hit = prim[:, 1] != 0xFFFFFFFF
    assert hit.mean() > (0.3 if scene == "cbox" else 0.05)                          # (the box is open towards the camera)
    assert np.array_equal(prim[:, 0], prim[:, 1]) and np.array_equal(t[:, 0].view(np.uint32), t[:, 1].view(np.uint32))


def test_emitter_sampling_and_environment_pdf_on_packed_scenes_match_oracle(dev):
    """sample_emitter_direct (+ eval_transmittance) and the environment emitter's pdf / radiance of the device source, on the packed scenes of
    tests/test_gpu_z_envnee.py (env_lit_scene(32); cbox-textured-flat: area + environment light), against the oracle with the same inputs and at that file's
    tolerances.  Observed on x86-64 with glibc: every direction, value, pdf and distance is bit-equal to the oracle's (the same libm on both sides)."""
    from ppg_b200 import builtin_scenes as B
    from common import load_fixture_scene
    for name, sc in (("env-only", B.env_lit_scene(32)), ("area+env", load_fixture_scene("cbox-textured-flat", 32))):
        props = dict(sc.integrator, nee="always")
        o = O.Oracle(O.params_from_xml(props), sc, kind="port")
        rng = np.random.default_rng(11); n = 100000
        lo, hi = np.asarray(sc.aabb_min, np.float64), np.asarray(sc.aabb_max, np.float64)
        ref = (lo + (hi - lo) * (0.1 + 0.8 * rng.random((n, 3)))).astype(np.float32)
        nrm = rng.normal(size=(n, 3)); nrm /= np.linalg.norm(nrm, axis=1, keepdims=True); nrm[n // 2:] = 0; nrm = nrm.astype(np.float32)
        smp = rng.random((n, 2), dtype=np.float32)
        d = np.zeros((n, 3), np.float32); val = np.zeros((n, 3), np.float32); pdf = np.zeros(n, np.float32); dist = np.zeros(n, np.float32)
        dev.dev_emitter_sample_direct.argtypes = [C.c_void_p, C.c_size_t, f32p, f32p, f32p, C.c_int, f32p, f32p, f32p, f32p]
        with _Packed(dev, sc) as h:
            assert dev.dev_emitter_sample_direct(h, n, ref.ctypes.data_as(f32p), nrm.ctypes.data_as(f32p), smp.ctypes.data_as(f32p), 3,
                                                 d.ctypes.data_as(f32p), val.ctypes.data_as(f32p), pdf.ctypes.data_as(f32p), dist.ctypes.data_as(f32p)) == 0
            d0, val0, pdf0, dist0 = o.emitter_sample_direct(ref, nrm, smp, 3)
            assert np.isfinite(val).all() and np.isfinite(pdf).all() and (pdf0 > 0).mean() > 0.05
            same = (np.isclose(pdf, pdf0, rtol=1e-4, atol=1e-7) & np.isclose(val, val0, rtol=1e-4, atol=1e-6).all(axis=1) & np.isclose(dist, dist0, rtol=1e-4, atol=1e-5)
                    & ((np.abs(d - d0).max(axis=1) < 1e-5) | (pdf0 == 0)))
            assert same.mean() >= 0.998, (name, same.mean())
            assert abs(float(val.sum()) - float(val0.sum())) <= 2e-3 * float(val0.sum())
            if name == "env-only":
                rng = np.random.default_rng(12)
                q = rng.normal(size=(200000, 3)); q = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
                epdf = np.zeros(len(q), np.float32); eval_ = np.zeros((len(q), 3), np.float32)
                dev.dev_env_pdf.argtypes = [C.c_void_p, C.c_size_t, f32p, f32p, f32p]
                assert dev.dev_env_pdf(h, len(q), q.ctypes.data_as(f32p), epdf.ctypes.data_as(f32p), eval_.ctypes.data_as(f32p)) == 0
                epdf0, eval0 = o.env_pdf(q)
                assert np.isclose(epdf, epdf0, rtol=2e-3, atol=1e-5).mean() >= 0.999
                assert np.isclose(eval_, eval0, rtol=2e-3, atol=1e-4).all(axis=1).mean() >= 0.999
                assert abs(float(epdf.sum()) - float(epdf0.sum())) <= 1e-4 * float(epdf0.sum())


def _pcg_vertex_jitter(seed, sample_index, ordinal):
    """PCG32 (O'Neill's pcg32_random_r with the splitmix64 keying of seed_vertex_rng), restated on Python integers: three next1D()."""
    M = (1 << 64) - 1

    def splitmix(x):
        x = (x + 0x9E3779B97F4A7C15) & M
        x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M
        x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M
        return x ^ (x >> 31)

    key = (sample_index * 64 + ordinal) & M
    state, inc = 0, ((key << 1) | 1) & M

    def nxt():
        nonlocal state
        old = state
        state = (old * 6364136223846793005 + inc) & M
        xs = (((old >> 18) ^ old) >> 27) & 0xFFFFFFFF
        rot = old >> 59
        return ((xs >> rot) | (xs << ((32 - rot) & 31))) & 0xFFFFFFFF

    nxt(); state = (state + splitmix(((seed + 0x5851F42D4C957F2D) & M) ^ splitmix(key))) & M; nxt()
    return [np.float32(nxt() >> 8) * np.float32(1.0 / 16777216.0) for _ in range(3)]


def test_vertex_jitter_source_is_pcg32_of_the_vertex_stream(dev):
    """dev_vertex_jitter -- the uniforms commit_kernel's stochastic spatial filter draws from seed_vertex_rng(seed, sampleIndex, ordinal), which the GPU
    commit tests hand to the oracle -- equals PCG32 restated on Python integers, bit for bit, including 64-bit sample indices and ordinals up to 2^24."""
    rng = np.random.default_rng(21); n = 300
    si = rng.integers(0, 1 << 63, n, dtype=np.uint64); si[:4] = [0, 1, (1 << 32) - 1, (1 << 64) - 1]
    od = rng.integers(0, 1 << 24, n, dtype=np.uint32); od[:4] = [0, 31, 1 << 23, (1 << 24) - 1]
    for seed in (0, 1234, (1 << 64) - 1):
        out = np.zeros((n, 3), np.float32)
        dev.dev_vertex_jitter.argtypes = [C.c_uint64, C.c_size_t, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), f32p]
        assert dev.dev_vertex_jitter(seed, n, si.ctypes.data_as(C.POINTER(C.c_uint64)), od.ctypes.data_as(C.POINTER(C.c_uint32)), out.ctypes.data_as(f32p)) == 0
        want = np.array([_pcg_vertex_jitter(seed, int(s), int(o)) for s, o in zip(si, od)], np.float32)
        assert np.array_equal(out.view(np.uint32), want.view(np.uint32)), seed
        assert ((out >= 0) & (out < 1)).all() and len(np.unique(out)) > 2 * n


# ---- the query half of the SD-tree at the depths the render reaches (tests/sdtree_queries.py; the same cases run on the GPU in tests/test_gpu_sdtree_queries.py)
def _dev_lookup(dev, sch, mn, ext, pts):
    u32p = C.POINTER(C.c_uint32)
    sch = np.ascontiguousarray(sch, np.uint32); pts = np.ascontiguousarray(pts, np.float32)
    mn = np.ascontiguousarray(mn, np.float32); ext = np.ascontiguousarray(ext, np.float32)
    leaf = np.zeros(len(pts), np.uint32); size = np.zeros((len(pts), 3), np.float32)
    dev.dev_stree_lookup.argtypes = [u32p, C.c_size_t, f32p, f32p, f32p, C.c_size_t, u32p, f32p]
    assert dev.dev_stree_lookup(sch.ctypes.data_as(u32p), len(sch), mn.ctypes.data_as(f32p), ext.ctypes.data_as(f32p), pts.ctypes.data_as(f32p), len(pts),
                                leaf.ctypes.data_as(u32p), size.ctypes.data_as(f32p)) == 0
    return leaf, size


def _cbox_box():
    from common import load_cbox
    o = O.Oracle(O.default_params(), load_cbox(16), kind="port")
    mn, mx = o.export(0)["aabb"]; o.close()
    return mn.astype(np.float32), mx.astype(np.float32)


@pytest.mark.parametrize("box", ["dyadic", "cbox"])
def test_device_stree_lookup_at_the_prefix_table_boundary(dev, box):
    """stree_lookup on a synthetic S-tree with leaves at exactly 20, 21 and 22 levels (the prefix table resolves 21), in a power-of-two box and in
    the cubified CBOX box: uniform points, points exactly on the split planes of every inner node from depth 15 down and of up to 24 levels per axis
    around the deep leaves, points on the faces and one ulp inside / outside them, points far outside.  Leaf and voxel size equal the float32 walk of
    the reference bit for bit."""
    import sdtree_queries as Q
    mn, mx = Q.DYADIC_BOX if box == "dyadic" else _cbox_box()
    ext = (mx - mn).astype(np.float32)
    sch = Q.synthetic_stree(Q.SYNTHETIC_ANCHORS)
    rng = np.random.default_rng(31)
    pts = np.concatenate([Q.stree_points(rng, mn, ext, [a for a, _ in Q.SYNTHETIC_ANCHORS]), Q.split_plane_points(sch, mn, ext, 15)])
    wl, ws, wd = Q.stree_walk(sch, mn, ext, pts)
    assert {20, 21, 22} <= set(wd.tolist())
    gl, gs = _dev_lookup(dev, sch, mn, ext, pts)
    assert np.array_equal(gl, wl) and np.array_equal(gs.view(np.uint32), ws.view(np.uint32))


def test_device_stree_lookup_past_2to24_nodes(dev):
    """The synthetic tree above renumbered so that every node but the root carries a number >= 2^24 (2^24 + 5 unreachable leaves in between, the
    layout later refines produce): the table's 24-bit node field cannot hold them, so the lookup walks from the root -- leaves bit for bit."""
    import sdtree_queries as Q
    mn, mx = Q.DYADIC_BOX; ext = (mx - mn).astype(np.float32)
    sch = Q.synthetic_stree(Q.SYNTHETIC_ANCHORS, offset=(1 << 24) + 5)
    rng = np.random.default_rng(32)
    pts = np.concatenate([Q.stree_points(rng, mn, ext, [a for a, _ in Q.SYNTHETIC_ANCHORS], 5000), Q.split_plane_points(sch, mn, ext, 15)])
    wl, ws, wd = Q.stree_walk(sch, mn, ext, pts)
    assert len(sch) > 1 << 24 and (wl >= 1 << 24).all() and {20, 21, 22} <= set(wd.tolist())
    gl, gs = _dev_lookup(dev, sch, mn, ext, pts)
    assert np.array_equal(gl, wl), f"{int((gl != wl).sum())} of {len(wl)} leaves differ, e.g. {gl[gl != wl][:4]} for {wl[gl != wl][:4]}"
    assert np.array_equal(gs.view(np.uint32), ws.view(np.uint32))


@pytest.fixture(scope="module")
def dtrees():
    import sdtree_queries as Q
    return Q.dtree_trees(O, "ref" if O.have_ref() else "port")


def _dev_dtree(dev, e, ql, d, rnd):
    u32p = C.POINTER(C.c_uint32)
    n = len(ql); pdf = np.zeros(n, np.float32); dirs = np.zeros((n, 3), np.float32); canon = np.zeros((n, 2), np.float32)
    sums = np.ascontiguousarray(e["sums"], np.float32); ch = np.ascontiguousarray(e["children"], np.uint16); first = e["tree_first"].astype(np.uint32)
    ql = np.ascontiguousarray(ql, np.uint32); d = np.ascontiguousarray(d, np.float32); rnd = np.ascontiguousarray(rnd, np.float32)
    dev.dev_dtree.argtypes = [f32p, C.POINTER(C.c_uint16), C.c_size_t, u32p, f32p, f32p, u32p, f32p, f32p, C.c_size_t, C.c_size_t, f32p, f32p, f32p]
    dev.dev_dtree(sums.ctypes.data_as(f32p), ch.ctypes.data_as(C.POINTER(C.c_uint16)), len(sums), first.ctypes.data_as(u32p), e["tree_sum"].ctypes.data_as(f32p),
                  e["tree_weight"].ctypes.data_as(f32p), ql.ctypes.data_as(u32p), d.ctypes.data_as(f32p), rnd.ctypes.data_as(f32p), rnd.shape[1], n,
                  pdf.ctypes.data_as(f32p), dirs.ctypes.data_as(f32p), canon.ctypes.data_as(f32p))
    return pdf, dirs, canon


def test_device_dtree_queries_at_the_depth_cap(dev, dtrees):
    """dtree_pdf and dtree_sample on the oracle's depth-20 cone trees, the 65 536-node tree and an untrained tree (tests/sdtree_queries.dtree_trees).
    pdf at random directions, the poles, the phi seam, canonical points on quadrant boundaries of every level and inside zero-sum cells: zeros exact,
    elsewhere within (5 * depth + 2) * 2^-24 of the float64 product of the exact ratios (the oracle's pdf too).  Samples with random, extreme and
    boundary uniforms: the canonical point bit-equal to the float32 restatement and to the reference's DTree::sample point; directions within 2e-6."""
    import sdtree_queries as Q
    o, e, leaves, cones = dtrees
    rng = np.random.default_rng(33)
    first = e["tree_first"].astype(np.int64); valid = Q.valid_flags(e["tree_sum"], e["tree_weight"])
    ql, d, ex = [], [], []
    for k, leaf in enumerate(leaves):
        dk, exk = Q.pdf_directions(rng, e["sums"], e["children"], int(first[leaf]), cones[k])
        ql.append(np.full(len(dk), leaf, np.uint32)); d.append(dk); ex.append(exk)
    ql, d, ex = np.concatenate(ql), np.concatenate(d), np.concatenate(ex)
    rnd = Q.sample_uniforms(rng, e["sums"], e["children"], first[ql], valid[ql], len(ql))
    pdf, dirs, canon = _dev_dtree(dev, e, ql, d, rnd)
    ok, depth = Q.pdf_matches(pdf, e["sums"], e["children"], first[ql], valid[ql], d, exact_phi=ex)
    assert ok.all(), (np.nonzero(~ok)[0][:8], pdf[~ok][:8])
    ok_o, _ = Q.pdf_matches(o.pdf(ql, d), e["sums"], e["children"], first[ql], valid[ql], d, exact_phi=ex)
    assert ok_o.all()
    assert depth.max() == 20 and (pdf == 0).any() and (pdf[~valid[ql]] == np.float32(1) / (np.float32(4) * Q.PI32)).all()
    want, levels = Q.sample_reference(e["sums"], e["children"], first[ql], valid[ql], rnd)
    assert np.array_equal(canon.view(np.uint32), want.view(np.uint32)), int((canon != want).any(axis=1).sum())
    assert o.has_sample_canonical() or o.kind == "ref"          # (a prebuilt reference library may predate the entry)
    if o.has_sample_canonical():
        assert np.array_equal(canon.view(np.uint32), o.sample_canonical(ql, rnd).view(np.uint32))
    assert np.abs(dirs - o.sample(ql, rnd)).max() <= 2e-6 and levels.max() == 20
