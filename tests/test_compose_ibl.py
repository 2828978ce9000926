"""The full compose step (SURVEY.md §8f rank 1): Hydrogent/shaders/HnPostProcess.psh:145-185 and the pre-integrated GGX table it
samples (Shaders/PBR/private/PrecomputeBRDF.psh:10-48).

Both passes follow DESIGN.md §2's rule on both sides: every operation rounded once in the oracle's order, cos / sin correctly rounded,
pow(x, 5) as ((x * x) * (x * x)) * x in double. Each texel of the table adds its samples in order on both sides, so the CUDA table and
compose are the oracle's bit for bit, at every size, sample count and plane layout. Where NaN is expected, its position is compared and
not its payload (CUDA's canonical NaN and x86's differ).

CPU: known answers of the oracle (limits of the split-sum table, the compose identities) and the oracle against a float64 numpy
restatement of the same discrete sums and the same compose, within bounds measured and stated below. GPU: table and pass against the
oracle through the C-ABI."""
import ctypes as C

import numpy as np
import pytest
import torch

import gpu_frame
from diligentfx_b200 import capi, synth
from gpu_frame import LAYOUTS, Planes

W, H = 96, 54


def _oracle(w=W, h=H, threads=0):
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


_CAMS = {}


def cameras(w: int, h: int) -> dict:
    """The cameras of test_view_mode_gpu.py's cases: the synthetic frame's (forward depth), the same with reversed depth and with
    reversed depth and an infinite far plane (its ViewProj and inverse recomputed from that projection), with the viewport of w x h."""
    if not _CAMS:
        fr = synth.generate_sequence(W, H, 1)[0]
        rv = synth.reverse_depth_frame({"depth": fr["depth"], "prev_depth": fr["prev_depth"], "curr_camera": fr["curr_camera"],
                                        "prev_camera": fr["prev_camera"]})["curr_camera"]
        inf = capi.CameraAttribs.from_buffer_copy(bytes(rv))
        inf.mProj.m[2][2], inf.mProj.m[3][2], inf.fFarPlaneZ = 0.0, rv.fNearPlaneZ, float("inf")
        m = lambda f: np.array([[f.m[r][c] for c in range(4)] for r in range(4)], np.float64)  # noqa: E731
        vp = m(inf.mView) @ m(inf.mProj)
        for name, a in (("mViewProj", vp), ("mViewProjInv", np.linalg.inv(vp))):
            for r in range(4):
                for c in range(4):
                    getattr(inf, name).m[r][c] = float(np.float32(a[r, c]))
        _CAMS.update(forward=fr["curr_camera"], reversed=rv, reversed_infinite=inf)
    out = {}
    for name, cam in _CAMS.items():
        c = capi.CameraAttribs.from_buffer_copy(bytes(cam))
        c.f4ViewportSize[0], c.f4ViewportSize[1] = float(w), float(h)
        c.f4ViewportSize[2], c.f4ViewportSize[3] = float(np.float32(1.0) / np.float32(w)), float(np.float32(1.0) / np.float32(h))
        out[name] = c
    return out


def drawn_inputs(w: int, h: int, seed: int) -> dict:
    """Planes where the compose goes wrong: opacity 0, -0, negative, above 1, +inf and NaN; roughness and metallic below 0, above 1 and
    NaN; zero and unnormalised normals; HDR SSR up to 6e4 and specular IBL larger than the SSR (a negative exchange)."""
    rng = np.random.default_rng(seed)
    u = lambda lo, hi, *s: rng.uniform(lo, hi, (h, w, *s)).astype(np.float32)  # noqa: E731
    color = np.concatenate([u(0.0, 4.0, 3), rng.choice(np.array([0.0, -0.0, -0.4, 0.35, 1.0, 1.0, 1.0, 1.6, np.inf, np.nan], np.float32), (h, w, 1))], -1)
    mat = u(0.0, 1.0, 4)
    for k in (0, 1):
        edge = rng.random((h, w)) < 0.25
        mat[..., k] = np.where(edge, rng.choice(np.array([-0.3, -0.0, 0.0, 1.0, 1.4, np.nan], np.float32), (h, w)), mat[..., k])
    n = rng.normal(size=(h, w, 3))
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    n *= rng.choice([1.0, 1.0, 1.0, 0.0, 0.3, 2.5], (h, w, 1))                       # zero and unnormalised normals
    normal = np.concatenate([n, np.zeros((h, w, 1))], -1).astype(np.float32)
    ssr = np.concatenate([np.exp2(u(-6.0, 15.87, 3)), u(0.0, 1.0, 1)], -1)            # up to 6e4
    ibl = np.concatenate([np.exp2(u(-6.0, 12.0, 3)), np.ones((h, w, 1), np.float32)], -1)
    return dict(color=color, material=mat, base_color=np.concatenate([u(0.0, 1.0, 3), np.ones((h, w, 1), np.float32)], -1),
                specular_ibl=ibl, ssr_out=ssr, ssao_out=u(0.0, 1.0), normal=normal)


def oracle_compose(cam, p: dict, lut: np.ndarray, ssr_scale: float, ssao_scale: float, use_ssr=True, use_ao=True) -> np.ndarray:
    """oracle_compose_ibl.cpp's compose; without SSR (or AO) the pass is the oracle's with that scale 0, which skips the step."""
    h, w = p["color"].shape[:2]
    o = _oracle(w, h)
    o.set_cameras(cam, cam)
    for k, v in p.items():
        o.set(k, v)
    o.set("brdf_lut", lut)
    o.set_compose_scales(ssr_scale if use_ssr else 0.0, ssao_scale if use_ao else 0.0)
    o.run("compose_ibl")
    return o.get("composed")


def oracle_lut(w: int, h: int, n: int) -> np.ndarray:
    o = _oracle(8, 8)
    o.brdf_lut((w, h), n)
    return o.get("brdf_lut")


def same_bits(got: np.ndarray, want: np.ndarray) -> str | None:
    """None when every value has the same bits, NaN where the other side has NaN (any payload)."""
    if got.shape != want.shape:
        return f"shape {got.shape} vs {want.shape}"
    gn, wn = np.isnan(got), np.isnan(want)
    if (gn != wn).any():
        return f"NaN at {int((gn != wn).sum())} values where the other side has none, first at {tuple(np.argwhere(gn != wn)[0])}"
    diff = (np.ascontiguousarray(got, np.float32).view(np.uint32) != np.ascontiguousarray(want, np.float32).view(np.uint32)) & ~gn
    if diff.any():
        i = tuple(int(k) for k in np.argwhere(diff)[0])
        return f"{int(diff.sum())} values differ, first at {i}: {got[i]!r} vs {want[i]!r}"
    return None


# ---------------------------------------------------------------------------------------------------------------------------------
# float64 restatements (CPU)
# ---------------------------------------------------------------------------------------------------------------------------------
def lut_f64(w: int, h: int, n: int, rows=None) -> np.ndarray:
    """PrecomputeBRDF.psh's discrete sum in float64 from the texel-centre UV the oracle uses (float): rows `rows` (default all) of a
    w x h table with n samples, (len(rows), w, 2)."""
    rows = np.arange(h) if rows is None else np.asarray(rows)
    nov = ((np.arange(w, dtype=np.float32) + np.float32(0.5)) / np.float32(w)).astype(np.float64)[None, :, None]
    rough = ((rows.astype(np.float32) + np.float32(0.5)) / np.float32(h)).astype(np.float64)[:, None, None]
    # the sample points are the shader's float Hammersley points and float Phi = (2 PI) Xi.x; the rest is float64
    f32 = np.float32
    rev = np.array([int(f"{k:032b}"[::-1], 2) for k in range(n)], np.float64).astype(f32)
    xi_x = np.arange(n, dtype=f32) / f32(n)
    xi_y = (rev * f32(2.0 ** -32)).astype(np.float64)[None, None, :]
    phi = ((f32(2.0) * f32(np.pi)) * xi_x).astype(np.float64)[None, None, :]
    a2 = rough ** 4
    ct = np.sqrt(np.clip((1.0 - xi_y) / (1.0 + (a2 - 1.0) * xi_y), 0.0, 1.0))
    st = np.sqrt(np.clip(1.0 - ct * ct, 0.0, 1.0))
    hx, hz = st * np.sin(phi), ct                                     # TangentX = -y, TangentY = x: H = (st sin phi, -st cos phi, ct)
    vx = np.sqrt(1.0 - nov * nov)
    vh = vx * hx + nov * hz
    nol, noh, voh = np.clip(2.0 * vh * hz - nov, 0.0, 1.0), np.clip(hz, 0.0, 1.0), np.clip(vh, 0.0, 1.0)
    ggxv = nol * np.sqrt(np.maximum(nov * nov * (1.0 - a2) + a2, 1e-7))
    ggxl = nov * np.sqrt(np.maximum(nol * nol * (1.0 - a2) + a2, 1e-7))
    with np.errstate(divide="ignore", invalid="ignore"):
        gvis = np.where(nol > 0.0, 4.0 * (0.5 / (ggxv + ggxl)) * voh * nol / noh, 0.0)
    fc = (1.0 - voh) ** 5
    return np.stack([((1.0 - fc) * gvis).sum(-1) / n, (fc * gvis).sum(-1) / n], -1)


def compose_f64(cam, p: dict, lut: np.ndarray, ssr_scale: float, ssao_scale: float) -> np.ndarray:
    """HnPostProcess.psh:145-185 in float64 from the same float32 planes and table (the 1/256-texel snap of the table lookup included)."""
    h, w = p["color"].shape[:2]
    d = {k: np.asarray(v, np.float64) for k, v in p.items()}
    c, op_ = d["color"][..., :3].copy(), d["color"][..., 3]
    s_ssr = ssr_scale * op_
    sat = lambda x: np.fmin(np.fmax(x, 0.0), 1.0)  # noqa: E731
    rough, metal = sat(d["material"][..., 0]), sat(d["material"][..., 1])
    r0 = 0.04 + metal[..., None] * (d["base_color"][..., :3] - 0.04)
    m = np.array([[cam.mViewProjInv.m[r][k] for k in range(4)] for r in range(4)], np.float64)
    u = (np.arange(w) + 0.5) * float(cam.f4ViewportSize[2])
    v = (np.arange(h) + 0.5) * float(cam.f4ViewportSize[3])
    ndc = np.stack(np.broadcast_arrays((u[None, :] - 0.5) * 2.0, (v[:, None] - 0.5) * -2.0, np.full((h, w), 0.5), np.ones((h, w))), -1)
    wp = ndc @ m
    view = np.array([cam.f4Position[0], cam.f4Position[1], cam.f4Position[2]]) - wp[..., :3] / wp[..., 3:]
    view /= np.linalg.norm(view, axis=-1, keepdims=True)
    ndv = sat((d["normal"][..., :3] * view).sum(-1))
    lh, lw = lut.shape[:2]
    snap = lambda q: np.floor(q * 256.0 + 0.5) / 256.0  # noqa: E731
    px, py = snap(ndv * lw - 0.5), snap(rough * lh - 0.5)
    x0, y0 = np.floor(px), np.floor(py)
    fx, fy = (px - x0)[..., None], (py - y0)[..., None]
    tap = lambda xx, yy: lut[np.clip(yy, 0, lh - 1).astype(int), np.clip(xx, 0, lw - 1).astype(int)].astype(np.float64)  # noqa: E731
    pre = (tap(x0, y0) * (1 - fx) * (1 - fy) + tap(x0 + 1, y0) * fx * (1 - fy) + tap(x0, y0 + 1) * (1 - fx) * fy + tap(x0 + 1, y0 + 1) * fx * fy)
    r90 = np.fmax((1.0 - rough)[..., None], r0)
    ks = r0 + (r90 - r0) * (np.clip(1.0 - ndv, 0.0, 1.0) ** 5)[..., None]
    spec = d["ssr_out"][..., :3] * (ks * pre[..., :1] + pre[..., 1:])
    on = (s_ssr > 0.0)[..., None]
    with np.errstate(invalid="ignore", over="ignore"):
        c = np.where(on, c + (spec - d["specular_ibl"][..., :3]) * d["ssr_out"][..., 3:] * s_ssr[..., None], c)
        s_ao = ssao_scale * op_
        c = np.where((s_ao > 0.0)[..., None], c * (1.0 + s_ao * (d["ssao_out"] - 1.0))[..., None], c)
    return np.concatenate([c, op_[..., None]], -1)


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


def test_oracle_brdf_table_non_square(built):
    """A w x h table holds NdotV = (x + 0.5) / w across and roughness = (y + 0.5) / h down: texels at the same (NdotV, roughness) of
    tables of other shapes are the same bits (column 1 of 3 and row 2 of 5 are at 0.5, as the one texel of a 1 x 1 table is)."""
    one, t35 = oracle_lut(1, 1, 33), oracle_lut(3, 5, 33)
    assert t35.shape == (5, 3, 2)
    assert np.array_equal(t35[2, 1].view(np.uint32), one[0, 0].view(np.uint32))
    assert np.array_equal(oracle_lut(1, 5, 33)[:, 0].view(np.uint32), t35[:, 1].view(np.uint32))
    assert np.array_equal(oracle_lut(3, 1, 33)[0].view(np.uint32), t35[2].view(np.uint32))


# Bounds of the oracle's table against the float64 sum, measured here (float32 oracle against float64 on the same float sample points),
# relative to the texel's value plus 1e-3. A term (1 - Fc) G_Vis or Fc G_Vis takes about 30 roundings, and NoL = 2 VoH H.z - NoV cancels
# near the horizon, where G_Vis ~ NoL / (NoV alpha NoH) magnifies that error by 1 / alpha at small roughness; the n terms are added in
# order. Largest seen: 3.7e-7 (N = 1), 4.8e-7 (N = 2), 5.9e-4 (N = 3, roughness 1/32: a sample just above the horizon), 7.4e-5 (512 x 512,
# 512 samples, the drawn rows). Held to 4x that.
LUT_REL = {1: 1.5e-6, 2: 2e-6, 3: 2.4e-3, 512: 3e-4}


@pytest.mark.parametrize("n", [1, 2, 3])
def test_oracle_brdf_table_against_float64_small(built, n):
    """Small tables (16 x 16 and 7 x 5) at N = 1, 2, 3: no summation order can hide a wrong term."""
    for w, h in ((16, 16), (7, 5)):
        got, want = oracle_lut(w, h, n).astype(np.float64), lut_f64(w, h, n)
        err = np.abs(got - want) / (np.abs(want) + 1e-3)
        assert err.max() <= LUT_REL[n], (w, h, n, err.max())


def test_oracle_brdf_table_against_float64_512(built):
    """The renderer's 512 x 512 table with 512 samples on drawn rows (the first, the last and six drawn between)."""
    rows = np.r_[0, np.sort(np.random.default_rng(11).choice(np.arange(1, 511), 6, replace=False)), 511]
    got, want = oracle_lut(512, 512, 512)[rows].astype(np.float64), lut_f64(512, 512, 512, rows)
    err = np.abs(got - want) / (np.abs(want) + 1e-3)
    assert err.max() <= LUT_REL[512], err.max()


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


# Bound of the oracle's compose against the float64 restatement, measured here (2026-10): the exchange adds a product of about 12
# roundings of magnitude |SSR| (up to 6e4) to the colour, so the error is relative to E = |c| + |SSR| |ks pre.x + pre.y| + |IBL| (times
# the confidence and scale); a lookup whose float and float64 NdotV snap to different 1/256 texel positions moves pre by at most the
# table's step over 1/256 of a texel, which stays inside it. The largest seen was 1.3e-7 E; held to 1e-6 E.
COMPOSE_REL = 1e-6


@pytest.mark.parametrize("cam_name", ["forward", "reversed", "reversed_infinite"])
def test_oracle_compose_against_float64(built, cam_name):
    w, h = 61, 37
    p = drawn_inputs(w, h, 3)
    finite = np.isfinite(p["color"][..., 3])
    p["color"][..., 3] = np.where(finite, p["color"][..., 3], 0.5)                   # inf / NaN opacity: checked bit for bit on the GPU
    cam = cameras(w, h)[cam_name]
    lut = oracle_lut(64, 64, 64)
    for ssr_scale, ssao_scale in ((1.0, 1.0), (0.7, 0.0), (1.6, -0.5)):
        got = oracle_compose(cam, p, lut, ssr_scale, ssao_scale).astype(np.float64)
        want = compose_f64(cam, p, lut, ssr_scale, ssao_scale)
        assert np.isfinite(got).all() and np.array_equal(got[..., 3], want[..., 3])
        e = (np.abs(p["color"][..., :3]) + np.abs(p["ssr_out"][..., :3]) * 2.0 + np.abs(p["specular_ibl"][..., :3])) * \
            np.maximum(1.0, abs(ssr_scale) * np.abs(p["color"][..., 3:4]))
        err = np.abs(got[..., :3] - want[..., :3]) / e
        assert err.max() <= COMPOSE_REL, (cam_name, ssr_scale, ssao_scale, err.max(), np.unravel_index(err.argmax(), err.shape))


# ---------------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------------
TABLE_SIZES = [(1, 1), (7, 5), (32, 8), (64, 64), (513, 257)]
SAMPLE_COUNTS = [1, 2, 3, 31, 32, 33, 100, 1000, 4096]


def cuda_lut(pl: Planes, w: int, h: int, n: int):
    lut = pl.new(h, w, 2, fill=-1.0)
    capi.check(capi.load().dfx_pass_precompute_brdf_lut(None, C.c_uint32(n), lut.ref), "dfx_pass_precompute_brdf_lut")
    return lut


@pytest.mark.gpu
def test_cuda_brdf_table_512(built):
    """The table PBR_Renderer::PrecomputeBRDF builds (512 x 512, 512 samples), bit for bit."""
    bad = same_bits(cuda_lut(Planes("aligned"), 512, 512, 512).host(), oracle_lut(512, 512, 512))
    assert bad is None, bad


@pytest.mark.gpu
@pytest.mark.parametrize("layout", LAYOUTS)
def test_cuda_brdf_table_sizes(built, layout):
    """1 x 1 up to 513 x 257 (not a multiple of the 32 x 8 CTA on either axis) with 64 samples; the row padding stays untouched."""
    pl, bad = Planes(layout), []
    for w, h in TABLE_SIZES:
        err = same_bits(cuda_lut(pl, w, h, 64).host(), oracle_lut(w, h, 64))
        if err:
            bad.append(f"{w} x {h}: {err}")
    assert not pl.padding_damage(), "a table store wrote into the row padding"
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
def test_cuda_brdf_table_sample_counts(built):
    pl, bad = Planes("padded"), []
    for w, h in ((7, 5), (32, 8)):
        for n in SAMPLE_COUNTS:
            err = same_bits(cuda_lut(pl, w, h, n).host(), oracle_lut(w, h, n))
            if err:
                bad.append(f"{w} x {h}, {n} samples: {err}")
    assert not pl.padding_damage()
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
def test_cuda_brdf_table_refusals(built):
    L, pl = capi.load(), Planes("tight")
    lut = pl.new(8, 8, 2, fill=-1.0)
    assert L.dfx_pass_precompute_brdf_lut(None, C.c_uint32(0), lut.ref) == capi.DFX_ERR_INVALID_ARG          # 0 samples
    assert L.dfx_pass_precompute_brdf_lut(None, C.c_uint32(16), pl.new(8, 8, 4).ref) == capi.DFX_ERR_INVALID_ARG  # RGBA32F
    assert L.dfx_pass_precompute_brdf_lut(None, C.c_uint32(16), pl.new(8, 8, 1).ref) == capi.DFX_ERR_INVALID_ARG  # R32F
    assert L.dfx_pass_precompute_brdf_lut(None, C.c_uint32(16), None) == capi.DFX_ERR_INVALID_ARG
    torch.cuda.synchronize()
    assert np.all(lut.host() == -1.0)


PLANES = ("color", "ssr_out", "ssao_out", "specular_ibl", "normal", "base_color", "material")


def cuda_compose(pl: Planes, cam, p: dict, lut, ssr_scale: float, ssao_scale: float, use_ssr=True, use_ao=True, rows=None, fill=-7.0,
                 lut_ref=None):
    """dfx_pass_compose_ibl on planes of `pl`; `lut` a host table (uploaded into `pl`) unless `lut_ref` is a device plane."""
    h, w = p["color"].shape[:2]
    up = {k: pl.up(p[k]).ref for k in PLANES}
    lr = lut_ref if lut_ref is not None else pl.up(lut).ref
    out = pl.new(h, w, 4, fill=fill)
    st = capi.load().dfx_pass_compose_ibl(None, pl.cameras(cam, cam), up["color"], up["ssr_out"] if use_ssr else None, up["ssao_out"] if use_ao else None,
                                          up["specular_ibl"], up["normal"], up["base_color"], up["material"], lr, C.c_float(ssr_scale),
                                          C.c_float(ssao_scale), out.ref, rows or capi.Rows(0, h))
    return st, out


SIZES = [(1, 1), (7, 3), (33, 17), (61, 37)]
SCALES = [(1.0, 1.0), (0.0, 0.0), (-0.5, 1.7), (1.7, -0.5), (0.6, 0.0), (0.0, 0.8)]
MODES = [(True, True), (False, True), (True, False), (False, False)]      # SSR, AO planes given


@pytest.mark.gpu
@pytest.mark.parametrize("layout", LAYOUTS)
def test_cuda_compose_matches_oracle(built, layout):
    """Drawn sizes x the three cameras x tables of 64^2, 1 x 1 and 40 x 24 x scales 0, negative, 1 and above 1 x the no-SSR / no-AO /
    neither combinations, on every plane layout, bit for bit (NaN positions for NaN)."""
    pl, bad, checked = Planes(layout), [], 0
    luts = {"64x64": oracle_lut(64, 64, 64), "1x1": oracle_lut(1, 1, 16), "40x24": oracle_lut(40, 24, 32)}
    for si, (w, h) in enumerate(SIZES):
        p = drawn_inputs(w, h, 100 + si)
        for cname, cam in cameras(w, h).items():
            for lname, lut in luts.items():
                for k, (ss, sa) in enumerate(SCALES):
                    use_ssr, use_ao = MODES[(k + si) % len(MODES)] if lname != "64x64" else (True, True)
                    st, out = cuda_compose(pl, cam, p, lut, ss, sa, use_ssr, use_ao)
                    capi.check(st, "dfx_pass_compose_ibl")
                    err = same_bits(out.host(), oracle_compose(cam, p, lut, ss, sa, use_ssr, use_ao))
                    checked += 1
                    if err:
                        bad.append(f"{w} x {h} {cname} lut {lname} scales ({ss}, {sa}) ssr {use_ssr} ao {use_ao}: {err}")
        for use_ssr, use_ao in MODES:                                                   # every combination at the default table
            st, out = cuda_compose(pl, cameras(w, h)["forward"], p, luts["64x64"], 1.0, 1.0, use_ssr, use_ao)
            capi.check(st, "dfx_pass_compose_ibl")
            err = same_bits(out.host(), oracle_compose(cameras(w, h)["forward"], p, luts["64x64"], 1.0, 1.0, use_ssr, use_ao))
            if err:
                bad.append(f"{w} x {h} ssr {use_ssr} ao {use_ao}: {err}")
    assert not pl.padding_damage(), "the compose wrote into the row padding"
    assert checked and not bad, f"{len(bad)} of {checked} cases:\n" + "\n".join(bad[:20])


@pytest.mark.gpu
def test_cuda_compose_full_hd_and_tables(built):
    """One 1920 x 1080 frame with the renderer's 512^2 table, and the 64^2 and a non-square table, on the reversed-infinite camera."""
    w, h = 1920, 1080
    p = drawn_inputs(w, h, 7)
    cam = cameras(w, h)["reversed_infinite"]
    pl, bad = Planes("aligned"), []
    for lut in (oracle_lut(512, 512, 512), oracle_lut(37, 300, 8)):
        st, out = cuda_compose(pl, cam, p, lut, 0.9, 0.7)
        capi.check(st, "dfx_pass_compose_ibl")
        err = same_bits(out.host(), oracle_compose(cam, p, lut, 0.9, 0.7))
        if err:
            bad.append(f"table {lut.shape[1]} x {lut.shape[0]}: {err}")
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
def test_cuda_table_feeds_compose(built):
    """Hydrogent's flow: dfx_pass_precompute_brdf_lut at 512^2 (512 samples) feeds dfx_pass_compose_ibl at 1920 x 1080; the output is
    the oracle's table fed to the oracle's compose."""
    w, h = 1920, 1080
    p = drawn_inputs(w, h, 8)
    cam = cameras(w, h)["forward"]
    pl = Planes("aligned")
    lut = cuda_lut(pl, 512, 512, 512)
    st, out = cuda_compose(pl, cam, p, None, 1.0, 1.0, lut_ref=lut.ref)
    capi.check(st, "dfx_pass_compose_ibl")
    err = same_bits(out.host(), oracle_compose(cam, p, oracle_lut(512, 512, 512), 1.0, 1.0))
    assert err is None, err


@pytest.mark.gpu
@pytest.mark.parametrize("layout", LAYOUTS)
def test_cuda_compose_row_ranges(built, layout):
    """Odd, empty and single-row ranges compute exactly those rows of the whole call; the other rows keep the sentinel."""
    w, h = 45, 29
    p = drawn_inputs(w, h, 9)
    cam = cameras(w, h)["reversed"]
    lut = oracle_lut(64, 64, 64)
    pl = Planes(layout)

    def launch(r, outs):
        up = {k: pl.up(p[k]).ref for k in PLANES}
        return capi.load().dfx_pass_compose_ibl(None, pl.cameras(cam, cam), up["color"], up["ssr_out"], up["ssao_out"], up["specular_ibl"],
                                                up["normal"], up["base_color"], up["material"], pl.up(lut).ref, C.c_float(0.8), C.c_float(0.6),
                                                outs[0], r)
    bad = gpu_frame.row_range_failures(pl, [("compose_ibl", [(h, w, 4, torch.float32)], launch)], np.random.default_rng(3))
    for y0, y1 in ((h - 1, h), (0, 1), (13, 14)):                                      # single rows, at both ends and inside
        st, out = cuda_compose(pl, cam, p, lut, 0.8, 0.6, rows=capi.Rows(y0, y1), fill=gpu_frame.SENTINEL)
        capi.check(st, f"rows [{y0}, {y1})")
        got, want = out.host(), oracle_compose(cam, p, lut, 0.8, 0.6)
        err = same_bits(got[y0:y1], want[y0:y1])
        if err or not (np.all(got[:y0] == gpu_frame.SENTINEL) and np.all(got[y1:] == gpu_frame.SENTINEL)):
            bad.append(f"rows [{y0}, {y1}): {err or 'rows outside the range were written'}")
    assert not pl.padding_damage()
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
def test_cuda_compose_refusals(built):
    """A missing plane the SSR term needs, a null camera, a bad row range, a wrong-format table and a size mismatch of every plane are
    refused, and nothing is written."""
    w, h = 16, 8
    p = drawn_inputs(w, h, 10)
    cam = cameras(w, h)["forward"]
    lut = oracle_lut(8, 8, 8)
    L, pl = capi.load(), Planes("tight")
    out = pl.new(h, w, 4, fill=-7.0)
    rows = capi.Rows(0, h)

    def call(planes, lut_ref, cams="ok", out_ref=None, r=rows):
        c = pl.cameras(cam, cam) if cams == "ok" else None
        return L.dfx_pass_compose_ibl(None, c, *[planes[k] for k in PLANES], lut_ref, C.c_float(1.0), C.c_float(1.0), out_ref or out.ref, r)

    good = {k: pl.up(p[k]).ref for k in PLANES}
    lref = pl.up(lut).ref
    assert call(good, lref) == capi.DFX_OK
    torch.cuda.synchronize()
    out.t.fill_(-7.0)
    refused = []
    for k in ("specular_ibl", "normal", "base_color", "material"):                       # the SSR term without a plane it needs
        refused.append((f"no {k}", call({**good, k: None}, lref)))
    refused.append(("no table", call(good, None)))
    refused.append(("RGBA32F table", call(good, pl.new(8, 8, 4, fill=0.5).ref)))
    refused.append(("R32F table", call(good, pl.new(8, 8, 1, fill=0.5).ref)))
    refused.append(("null cameras", call(good, lref, cams=None)))
    refused.append(("rows past the end", call(good, lref, r=capi.Rows(0, h + 1))))
    for k in PLANES[1:]:                                                                   # one row or column too many
        a = p[k]
        for shape in ((h + 1, w), (h, w - 1)):
            b = np.zeros(shape + a.shape[2:], np.float32)
            refused.append((f"{k} {shape[1]} x {shape[0]}", call({**good, k: pl.up(b).ref}, lref)))
    big = pl.new(h, w + 1, 4)
    refused.append(("out one column wider", call(good, lref, out_ref=big.ref)))
    refused.append(("colour one row taller", call({**good, "color": pl.up(np.zeros((h + 1, w, 4), np.float32)).ref}, lref)))
    wrong = [name for name, st in refused if st != capi.DFX_ERR_INVALID_ARG]
    assert not wrong, wrong
    torch.cuda.synchronize()
    assert np.all(out.host() == -7.0)
