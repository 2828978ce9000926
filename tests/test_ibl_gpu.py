"""IBL cube-map precomputation on the GPU: dfx_pass_irradiance_cube and dfx_pass_prefilter_env_map against oracle_ibl_py (the oracle
tests/test_ibl_reference.py pins to the reference's own shaders), their properties, Hydrogent's flow into the environment-map
background, and the C++ PBR_Renderer.

Every sample is computed alike on both sides; only the summation order differs, so every value is held to ibl_cases.bound (DESIGN.md
§2) and the largest error relative to that bound is printed. With 1 or 2 samples no reordering is possible and the cube outputs are
compared bit for bit."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import gpu_frame
import ibl_cases as IC
from diligentfx_b200 import capi, ibl, synth
from diligentfx_b200.chain import ChainConfig, PostProcessChain
from helpers import psnr
from oracle import oracle_env_map_py as oe
from oracle import oracle_ibl_py as oi
from oracle import oracle_py as op

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CUBE, SPHERE = capi.ENV_MAP_TYPE_CUBE, capi.ENV_MAP_TYPE_SPHERE


def _src(pl, levels, src16):
    return [pl.native(l.astype(np.float16)) if src16 else pl.up(l) for l in levels]


def _host_levels(levels, src16):
    """What the kernels read: the fp16 source's values widened to fp32."""
    return [l.astype(np.float16).astype(np.float32) if src16 else l for l in levels]


def _arr(bufs):
    return (capi.Plane * len(bufs))(*[b.p for b in bufs])


def irradiance(pl, env_type, levels, size, n, opt, src16=False, out16=False):
    src = _src(pl, levels, src16)
    out = pl.new(6 * size, size, 4, dtype=torch.float16 if out16 else torch.float32)
    capi.check(capi.load().dfx_pass_irradiance_cube(None, env_type, _arr(src), len(src), C.c_uint32(n), int(opt), out.ref), "dfx_pass_irradiance_cube")
    return out


def prefilter(pl, env_type, levels, size, n_out, n, opt, src16=False, out16=False):
    src = _src(pl, levels, src16)
    outs = [pl.new(6 * max(size >> m, 1), max(size >> m, 1), 4, dtype=torch.float16 if out16 else torch.float32) for m in range(n_out)]
    capi.check(capi.load().dfx_pass_prefilter_env_map(None, env_type, _arr(src), len(src), C.c_uint32(n), int(opt), _arr(outs), n_out),
               "dfx_pass_prefilter_env_map")
    return outs


def _check(got, want, n, prefilter_, out16, what):
    """got (6s, s, 4) vs want (faces, rows, s, 4) flattened alike; returns the largest error / bound."""
    got, want = got.reshape(want.shape), want
    b = IC.bound(want, n, prefilter_, out16)
    err = np.abs(got.astype(np.float64) - want.astype(np.float64))
    assert np.isfinite(got).all(), what
    worst = float((err / np.maximum(b, 1e-300)).max())
    assert (err <= b).all(), f"{what}: {(err > b).sum()} values beyond the bound, worst {worst:.3g} x bound"
    return worst


MAPS = {CUBE: IC.cube_chain(16, 3), SPHERE: IC.sphere_chain(64, 32, 4)}


@pytest.mark.parametrize("layout", gpu_frame.LAYOUTS)
@pytest.mark.parametrize("env_type", [CUBE, SPHERE])
@pytest.mark.parametrize("opt", [0, 1])
@pytest.mark.parametrize("fmt", ["32/32", "16/16", "16/32", "32/16"])
def test_both_passes_against_the_oracle(built, layout, env_type, opt, fmt):
    src16, out16 = fmt.startswith("16"), fmt.endswith("16")
    pl = gpu_frame.Planes(layout)
    lv = MAPS[env_type]
    host = _host_levels(lv, src16)
    worst = []
    for n in (64, 100):
        got = irradiance(pl, env_type, lv, 8, n, opt, src16, out16).host()
        worst.append(_check(got, oi.irradiance(env_type, host, 8, n, bool(opt)), n, False, out16, f"irradiance n={n}"))
    outs = prefilter(pl, env_type, lv, 8, 4, 37, opt, src16, out16)
    for m, o in enumerate(outs):
        want = oi.prefilter(env_type, host, max(8 >> m, 1), oi.roughness(m, 4), 37, bool(opt))
        worst.append(_check(o.host(), want, 37, True, out16, f"prefilter level {m}"))
    torch.cuda.synchronize()
    assert pl.padding_damage() == 0
    print(f"largest error / bound: {max(worst):.3g}")


@pytest.mark.parametrize("n", [1, 2])
@pytest.mark.parametrize("opt", [0, 1])
def test_one_and_two_samples_are_bit_identical_on_a_cube(built, n, opt):
    pl = gpu_frame.Planes("padded")
    lv = MAPS[CUBE]
    got = irradiance(pl, CUBE, lv, 8, n, opt).host()
    assert got.tobytes() == oi.as_cube(oi.irradiance(CUBE, lv, 8, n, bool(opt))).tobytes()
    for m, o in enumerate(prefilter(pl, CUBE, lv, 8, 3, n, opt)):
        want = oi.as_cube(oi.prefilter(CUBE, lv, max(8 >> m, 1), oi.roughness(m, 3), n, bool(opt)))
        assert o.host().tobytes() == want.tobytes(), m


def test_sun_and_level_clamp(built):
    """A sun 10^4 times brighter than the rest; a 2-level source, so the LOD clamp to g_EnvMipCount - 1 is hit."""
    pl = gpu_frame.Planes("tight")
    lv = IC.sun_sphere(64, 32, 2)
    got = irradiance(pl, SPHERE, lv, 8, 300, 1).host()
    w = _check(got, oi.irradiance(SPHERE, lv, 8, 300), 300, False, False, "irradiance")
    for m, o in enumerate(prefilter(pl, SPHERE, lv, 8, 3, 64, 1)):
        w = max(w, _check(o.host(), oi.prefilter(SPHERE, lv, max(8 >> m, 1), oi.roughness(m, 3), 64), 64, True, False, f"level {m}"))
    print(f"largest error / bound: {w:.3g}")


@pytest.mark.parametrize("env_type", [CUBE, SPHERE])
def test_hydrogent_defaults_at_full_size(built, env_type):
    """A 1024^2 cube with 11 levels or a 2048 x 1024 sphere with 12; 64^2 irradiance with 8192 samples and the 256^2 prefilter with 9
    levels and 256 samples, each checked against the oracle on two drawn rows of every face and level."""
    lv = IC.cube_chain(1024, 11) if env_type == CUBE else IC.sphere_chain(2048, 1024, 12)
    dev = [torch.from_numpy(l).cuda().half() for l in lv]
    irr, pre = ibl.precompute_cubemaps(env_type, dev, dtype=torch.float32)
    torch.cuda.synchronize()
    host = _host_levels(lv, True)
    rng = np.random.default_rng(env_type)
    worst = 0.0
    for f in range(6):
        r = int(rng.integers(0, 63))
        want = oi.irradiance(env_type, host, 64, 0, faces=[f], rows=(r, r + 2))
        got = irr.cpu().numpy().reshape(6, 64, 64, 4)[f:f + 1, r:r + 2]
        worst = max(worst, _check(got, want, 8192, False, False, f"irradiance face {f}"))
        for m, p in enumerate(pre):
            s = max(256 >> m, 1)
            r = int(rng.integers(0, max(s - 1, 1)))
            rows = (r, min(r + 2, s))
            want = oi.prefilter(env_type, host, s, oi.roughness(m, len(pre)), 0, faces=[f], rows=rows)
            got = p.cpu().numpy().reshape(6, s, s, 4)[f:f + 1, rows[0]:rows[1]]
            worst = max(worst, _check(got, want, 256, True, False, f"prefilter face {f} level {m}"))
    assert len(pre) == 9 and irr.shape == (384, 64, 4)
    print(f"largest error / bound: {worst:.3g}")


def test_round_trip_gives_back_the_source(built):
    """A cube whose level 0 is the output size, prefiltered at roughness 0 (level 0 of the chain) with the LOD at 0: every texel reads
    its own texel centre back, which pins the face order, the face matrices, the flips and the texel-centre rule."""
    pl = gpu_frame.Planes("aligned")
    for s in (8, 16):
        src = IC.face_gradient_cube(s)
        for opt in (0, 1):
            outs = prefilter(pl, CUBE, [src], s, 2, 16, opt)
            got = outs[0].host()
            assert np.abs(got[..., :3] - src[..., :3]).max() <= 4e-6 * np.abs(src[..., :3]).max(), (s, opt)


def test_constant_map_gives_the_constant(built):
    pl = gpu_frame.Planes("tight")
    c = 2.75
    for env_type, lv in ((CUBE, [np.full((6 * 8, 8, 4), c, np.float32), np.full((24, 4, 4), c, np.float32)]),
                         (SPHERE, [np.full((16, 32, 4), c, np.float32)])):
        got = irradiance(pl, env_type, lv, 8, 8192, 1).host()
        assert np.abs(got[..., :3] - c).max() <= c * (IC.gamma(8192 // 32 + 4) + 16 * IC.U) and (got[..., 3] == 1).all()
        for o in prefilter(pl, env_type, lv, 8, 4, 256, 1):
            g = o.host()
            assert np.abs(g[..., :3] - c).max() <= c * (2 * IC.gamma(256 // 32 + 4) + 16 * IC.U) and (g[..., 3] == 0).all()


def test_hydrogent_white_default_dome(built):
    dome = [torch.from_numpy(IC.white_dome()[0]).cuda()]
    irr, pre = ibl.precompute_cubemaps(SPHERE, dome)
    torch.cuda.synchronize()
    assert irr.dtype == torch.float16 and (irr[..., :3].float() == 1.0).all() and (irr[..., 3] == 1).all()
    for p in pre:
        assert (p[..., :3].float() == 1.0).all() and (p[..., 3] == 0).all()


def test_repeatable(built):
    dev = [torch.from_numpy(l).cuda() for l in MAPS[SPHERE]]
    a = ibl.precompute_cubemaps(SPHERE, dev, 16, 16, num_diffuse_samples=500, num_specular_samples=70)
    b = ibl.precompute_cubemaps(SPHERE, dev, 16, 16, num_diffuse_samples=500, num_specular_samples=70)
    torch.cuda.synchronize()
    assert torch.equal(a[0].view(torch.int16), b[0].view(torch.int16))
    assert all(torch.equal(x.view(torch.int16), y.view(torch.int16)) for x, y in zip(a[1], b[1]))


def test_hydrogent_flow_into_the_environment_map_background(built):
    """Precompute from a sphere sky, hand prefiltered[:8] to set_environment_map with HnRenderEnvMapTask's attribs (MipLevel 1), run
    chain frames: they equal oracle_env_map_py.frame fed the same prefiltered planes, within E's bounds."""
    W, H = 96, 54
    sky = [torch.from_numpy(l).cuda() for l in IC.sphere_chain(256, 128, 8)]
    _, pre = ibl.precompute_cubemaps(SPHERE, sky, num_diffuse_samples=64)
    chain = PostProcessChain(W, H, ChainConfig(enable_taa=True))
    chain.set_environment_map(CUBE, pre[:8])
    planes = [p.float().cpu().numpy() for p in pre[:8]]
    o = op.Oracle(W, H)
    for k, fr in enumerate(synth.generate_sequence(W, H, 3)):
        got = chain.run_frame(fr).cpu().numpy()
        want = oe.frame(o, fr, CUBE, planes)
        p = psnr(np.clip(got[..., :3], 0, 1), np.clip(want[..., :3], 0, 1))
        print(f"frame {k}: LDR PSNR {p:.2f} dB")
        assert p >= 49.0, (k, p)
    chain.close()


def test_refusals(built):
    lib = capi.load()
    pl = gpu_frame.Planes("tight")
    cube = _src(pl, MAPS[CUBE], False)
    out = pl.new(48, 8, 4)
    ok = lambda st: st == capi.DFX_ERR_INVALID_ARG  # noqa: E731

    def irr(env_type=CUBE, src=cube, n=None, o=out):
        return lib.dfx_pass_irradiance_cube(None, env_type, _arr(src), len(src) if n is None else n, C.c_uint32(16), 1, o.ref)

    def pre(src=cube, outs=None, n_out=None, env_type=CUBE):
        outs = outs or [pl.new(48, 8, 4), pl.new(24, 4, 4)]
        return lib.dfx_pass_prefilter_env_map(None, env_type, _arr(src), len(src), C.c_uint32(16), 1, _arr(outs), len(outs) if n_out is None else n_out)

    assert irr() == capi.DFX_OK and pre() == capi.DFX_OK
    assert ok(irr(env_type=2)) and ok(pre(env_type=-1))                                     # unknown type
    assert ok(irr(src=[pl.new(40, 8, 4)]))                                                   # cube level not s x 6s
    assert ok(irr(src=[cube[0], cube[2]]))                                                   # a chain that does not halve
    assert ok(irr(src=[cube[0], pl.native(np.zeros((24, 4, 4), np.float16))]))              # mixed formats
    assert ok(irr(n=0)) and ok(irr(src=[cube[0]] * 17, n=17))                                # 0 or more than 16 levels
    assert ok(irr(o=pl.new(48, 8, 2)))                                                       # output format
    assert ok(irr(o=pl.new(40, 8, 4)))                                                       # output not a cube
    assert ok(pre(outs=[pl.new(48, 8, 4)]))                                                  # one prefiltered level: 0 / 0
    assert ok(pre(outs=[pl.new(48, 8, 4), pl.new(48, 8, 4)]))                                # an output chain that does not halve
    assert ok(pre(outs=[pl.new(48, 8, 4), pl.new(24, 4, 2)]))                                # output format
    assert ok(pre(outs=[pl.new(48, 8, 4), pl.native(np.zeros((24, 4, 4), np.float16))]))   # mixed output formats
    assert ok(pre(outs=[pl.new(6 * max(8 >> m, 1), max(8 >> m, 1), 4) for m in range(17)]))  # more than 16 levels
    assert ok(lib.dfx_pass_irradiance_cube(None, CUBE, None, 1, C.c_uint32(16), 1, out.ref))
    assert ok(lib.dfx_pass_irradiance_cube(None, CUBE, _arr(cube), len(cube), C.c_uint32(16), 1, None))


def test_cpp_pbr_renderer(built, tmp_path):
    """tests/cpp/ibl_driver.cpp drives include/dfx/PBR_Renderer.hpp: PrecomputeCubemaps with default attribs on a white sphere map (the
    outputs are 1), the same with 16 source and 16 prefiltered levels, and PrecomputeBRDF, whose 512 x 512 table must be the oracle's
    (512 samples) byte for byte."""
    exe = str(tmp_path / "ibl_driver")
    libdir = os.path.dirname(capi.LIB_PATH)
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", os.path.join(HERE, "cpp", "ibl_driver.cpp"), "-I", os.path.join(ROOT, "include"),
                        "-L", libdir, "-ldfx_b200", f"-Wl,-rpath,{libdir}", "-Wl,--allow-shlib-undefined", "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    table = str(tmp_path / "brdf_lut.bin")
    r = subprocess.run([exe, table], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "ok" in r.stdout
    o = op.Oracle(8, 8)
    o.brdf_lut(512, 512)
    assert open(table, "rb").read() == o.get("brdf_lut").tobytes(), "PBR_Renderer::PrecomputeBRDF's table is not the oracle's"
