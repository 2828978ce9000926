"""The full compose step (SURVEY.md §8f rank 1): Hydrogent/shaders/HnPostProcess.psh:145-185 and the pre-integrated GGX table it
samples (Shaders/PBR/private/PrecomputeBRDF.psh:10-48).

CPU: known answers of the oracle — limits of the split-sum table, the compose identities. GPU: table and pass against
the oracle through the C-ABI."""
import ctypes as C

import numpy as np
import pytest

from diligentfx_b200 import capi, synth
from gpu_frame import Planes
from helpers import assert_close

W, H = 96, 54


def _oracle(w=W, h=H, threads=4):
    from oracle import oracle_py as op
    return op.Oracle(w, h, threads=threads)


def _inputs(seed=5):
    """One synthetic frame plus the planes only the full compose reads: base colour, metallic in material.y, a specular-IBL
    plane, SSR (rgb radiance, a = confidence), AO and a partly transparent colour alpha."""
    fr = synth.generate_sequence(W, H, 1)[0]
    rng = np.random.default_rng(seed)
    color = fr["color"].copy()
    color[..., 3] = rng.choice([0.0, 0.35, 1.0], (H, W), p=[0.1, 0.2, 0.7])          # opacity 0 must leave the pixel untouched
    mat = fr["material"].copy()
    mat[..., 1] = rng.choice([0.0, 0.5, 1.0], (H, W))
    mat[..., 0] = np.where(rng.random((H, W)) < 0.05, 1.5, mat[..., 0])               # out-of-range roughness is saturated
    base = np.concatenate([rng.uniform(0.02, 1.0, (H, W, 3)), np.ones((H, W, 1))], -1).astype(np.float32)
    ibl = np.concatenate([np.exp2(rng.uniform(-4, 2, (H, W, 3))), np.ones((H, W, 1))], -1).astype(np.float32)
    ssr = np.concatenate([np.exp2(rng.uniform(-4, 3, (H, W, 3))), rng.uniform(0, 1, (H, W, 1))], -1).astype(np.float32)
    ao = rng.uniform(0.2, 1.0, (H, W)).astype(np.float32)
    return fr, dict(color=color, material=mat, base_color=base, specular_ibl=ibl, ssr_out=ssr, ssao_out=ao, normal=fr["normal"])


def test_oracle_brdf_table_limits(built):
    o = _oracle()
    o.brdf_lut(64, 512)
    lut = o.get("brdf_lut")
    assert lut.shape == (64, 64, 2) and np.isfinite(lut).all() and lut.min() >= 0.0 and lut.max() <= 1.0 + 1e-6
    # mirror-like, facing the viewer: scale -> 1, bias -> 0 (no Fresnel boost, no energy loss)
    assert abs(lut[0, -1, 0] - 1.0) < 2e-2 and lut[0, -1, 1] < 1e-3
    # grazing view of a smooth surface: everything moves into the Fresnel bias
    assert lut[0, 0, 1] > 0.9 and lut[0, 0, 0] < 0.1
    # a white furnace stays <= 1 and loses energy with roughness (single scattering)
    total = lut[..., 0] + lut[..., 1]
    assert total.max() <= 1.0 + 1e-3 and total[-1, 32] < total[0, 32]


def test_oracle_compose_identities(built):
    fr, p = _inputs()
    o = _oracle()
    o.set_inputs(fr)
    o.brdf_lut(32, 128)
    for k, v in p.items():
        o.set(k, v)
    o.set_compose_scales(1.0, 1.0)
    o.run("compose_ibl")
    full = o.get("composed")
    assert np.isfinite(full).all() and np.array_equal(full[..., 3], p["color"][..., 3])             # alpha passes through
    clear = p["color"][..., 3] == 0.0
    assert clear.any() and np.array_equal(full[clear], p["color"][clear])                           # opacity 0: nothing applied
    # SSR confidence 0 everywhere: only the occlusion term remains
    o.set("ssr_out", np.concatenate([p["ssr_out"][..., :3], np.zeros((H, W, 1), np.float32)], -1))
    o.run("compose_ibl")
    want = p["color"][..., :3] * (1.0 + p["color"][..., 3:4] * (p["ssao_out"][..., None] - 1.0))
    assert np.allclose(o.get("composed")[..., :3], want, rtol=1e-5, atol=1e-6)
    # both scales 0: identity
    o.set_compose_scales(0.0, 0.0)
    o.run("compose_ibl")
    assert np.array_equal(o.get("composed"), p["color"])


@pytest.mark.gpu
def test_cuda_brdf_table_and_compose(built):
    fr, p = _inputs()
    o = _oracle()
    o.set_inputs(fr)
    o.brdf_lut(64, 512)
    for k, v in p.items():
        o.set(k, v)
    o.set_compose_scales(0.8, 0.6)
    o.run("compose_ibl")
    L, Pl = capi.load(), Planes("tight")
    lut = Pl.new(64, 64, 2, fill=-1.0)
    capi.check(L.dfx_pass_precompute_brdf_lut(None, 512, lut.ref), "brdf lut")
    # 512 sequential fp32 additions of sin / cos / pow terms: libm (oracle) and CUDA differ in the last bits of each term
    assert_close("BRDF table", lut.host(), o.get("brdf_lut"), tol=3e-4, min_psnr=100.0)
    cams = Pl.cameras(fr["curr_camera"], fr["prev_camera"])
    out = Pl.new(H, W, 4, fill=-1.0)
    P = lambda a: Pl.up(a).ref  # noqa: E731
    rows = capi.Rows(0, H)
    capi.check(L.dfx_pass_compose_ibl(None, cams, P(p["color"]), P(p["ssr_out"]), P(p["ssao_out"]), P(p["specular_ibl"]), P(p["normal"]),
                                      P(p["base_color"]), P(p["material"]), P(o.get("brdf_lut")), C.c_float(0.8), C.c_float(0.6), out.ref, rows), "compose_ibl")
    assert_close("composed (IBL form)", out.host(), o.get("composed"), tol=1e-4, max_outliers=1e-4, min_psnr=90.0, hdr=True)
    # without SSR the five extra planes may be null; without AO too -> copy
    capi.check(L.dfx_pass_compose_ibl(None, cams, P(p["color"]), None, None, None, None, None, None, None, C.c_float(1.0), C.c_float(1.0), out.ref, rows),
               "compose_ibl (no SSR, no AO)")
    assert np.array_equal(out.host(), p["color"])
    # SSR given but a plane it needs missing: refused
    assert L.dfx_pass_compose_ibl(None, cams, P(p["color"]), P(p["ssr_out"]), None, None, P(p["normal"]), P(p["base_color"]), P(p["material"]),
                                  P(o.get("brdf_lut")), C.c_float(1.0), C.c_float(1.0), out.ref, rows) == capi.DFX_ERR_INVALID_ARG
