"""DepthOfField (SURVEY.md §8f rank 2): the eleven passes of PostProcess/DepthOfField/src/DepthOfField.cpp:292-331
(Shaders/PostProcess/DepthOfField/private/DOF_*.fx), between TAA and Bloom in the reference chain.

CPU: known answers of the oracle (thin-lens CoC formula, kernel point counts, pass-through of an in-focus frame, energy of the
Gaussian). GPU: every pass against the oracle through the C-ABI on the oracle's own inputs, then the effect object inside
the chain."""
import ctypes as C

import numpy as np
import pytest

from diligentfx_b200 import capi, synth
from gpu_frame import Planes, assert_default, run_sequence
from helpers import psnr, reinhard
from oracle.refshader.driver import Variant

W, H, FRAMES = 160, 96, 3
FLAGS = capi.DOF_FLAG_TEMPORAL_SMOOTHING | capi.DOF_FLAG_KARIS_INVERSE


def _oracle(w=W, h=H, threads=4):
    from oracle import oracle_py as op
    return op.Oracle(w, h, threads=threads)


def _lens(fr, focus=6.0, fstop=1.4):
    for k in ("curr_camera", "prev_camera"):
        fr[k].fFocusDistance, fr[k].fFStop, fr[k].fFocalLength, fr[k].fSensorWidth = focus, fstop, 50.0, 36.0
    return fr


def _attribs():
    a = capi.DOFAttribs.default()
    a.MaxCircleOfConfusion = 0.02
    return a


def test_oracle_coc_formula(built):
    """CoC = clamp(1000 * K * (z - F) / z / (sensor * MaxCoC), -1, 1), K = f^2 / (N * (F - f)), f in metres (…CircleOfConfusion.fx:24-39)."""
    from oracle import oracle_py as op
    fr = _lens(synth.generate_sequence(32, 16, 1)[0], focus=5.0, fstop=2.0)
    o = _oracle(32, 16, 1)
    a = _attribs()
    o.set_dof(a, 0)
    o.set_inputs(fr)
    o.frame(op.STAGE_POSTFX | op.STAGE_DOF)
    got, depth = o.get("dof_coc"), fr["depth"]
    proj = fr["curr_camera"].mProj
    z = np.array([[o.L.orc_depth_to_camera_z(C.c_float(float(d)), C.byref(proj)) for d in row] for row in depth], np.float64)
    f, N, F = 0.05, 2.0, 5.0
    want = np.clip(1000.0 * (f * f / (N * (F - f))) * (z - F) / np.maximum(z, 1e-4) / (36.0 * a.MaxCircleOfConfusion), -1, 1)
    assert np.allclose(got, want, atol=2e-5)
    assert got.min() < 0 < got.max()                          # the scene straddles the focus plane


def test_kernel_point_counts():
    # ComputeSampleCount (DOF_Common.fx:4-7) == points generated (DepthOfField.cpp:49-73): 1 + density * rings * (rings - 1) / 2
    for rings in range(2, 6):
        for density in range(2, 8):
            gen = sum(max(density * i, 1) for i in range(rings))
            assert gen == 1 + density * ((rings - 1) * rings >> 1) <= 71


def test_oracle_in_focus_frame_passes_through(built):
    """With the whole scene at the focus distance every CoC is 0: both layer alphas are 0 and D11 returns the source."""
    from oracle import oracle_py as op
    fr = synth.generate_sequence(64, 40, 1)[0]
    fr["depth"][:] = fr["depth"][20, 32]                      # a flat wall
    z = _oracle(64, 40).L.orc_depth_to_camera_z(C.c_float(float(fr["depth"][0, 0])), C.byref(fr["curr_camera"].mProj))
    _lens(fr, focus=float(z))
    o = _oracle(64, 40)
    o.set_dof(_attribs(), 0)
    o.set_inputs(fr)
    o.frame(op.STAGE_POSTFX | op.STAGE_DOF)
    assert np.abs(o.get("dof_coc")).max() < 1e-3
    assert np.allclose(o.get("dof_out"), o.get("dof_in"), atol=1e-6)


@pytest.fixture(scope="module")
def ref(built):
    from oracle import oracle_py as op
    seq = [_lens(f) for f in synth.generate_sequence(W, H, FRAMES)]
    o = _oracle()
    o.set_dof(_attribs(), FLAGS)
    for fr in seq:
        o.set_inputs(fr)
        o.frame(op.STAGE_ALL | op.STAGE_DOF)
    return seq, o


def test_oracle_frame_structure(ref):
    _, o = ref
    assert o.get("dof_dilation3").shape == (H >> 3, W >> 3) and o.get("dof_pre0").shape == (H // 2, W // 2, 4)
    src, out = o.get("dof_in"), o.get("dof_out")
    assert np.isfinite(out).all() and np.array_equal(out[..., 3], src[..., 3])
    # defocus removes high frequencies: the Laplacian energy of the blurred frame is lower
    lap = lambda x: np.abs(4 * x[1:-1, 1:-1] - x[:-2, 1:-1] - x[2:, 1:-1] - x[1:-1, :-2] - x[1:-1, 2:]).mean()  # noqa: E731
    assert lap(reinhard(out[..., :3])) < 0.8 * lap(reinhard(src[..., :3]))
    assert np.isfinite(o.get("ldr")).all()


@pytest.mark.gpu
def test_cuda_dof_passes(built):
    """D1 .. D11 against the oracle on its own inputs (gpu_frame.run_frame), then D4 (level 3) -> D5 -> D6 and D7 -> D8 -> D9 -> D10
    -> D11 on the GPU's own planes against the planes the oracle holds at the end of its frame, all to the default bounds of
    gpu_frame.tolerance; the D6 blur in place is refused."""
    v = Variant(dof=True, dof_flags=FLAGS, dof_attribs=_attribs())
    seq = [_lens(f) for f in synth.generate_sequence(W, H, FRAMES)]
    fr = seq[-1]
    o, res = run_sequence(seq, v)
    assert_default(res, v, "D")
    L, P, g, a = capi.load(), Planes("tight"), o.get, v.dof_attribs
    cams = P.cameras(fr["curr_camera"], fr["prev_camera"])
    src, coc = P.up(g("dof_in")), P.up(g(f"dof_coc_temporal{fr['frame'] & 1}"))
    l3, tmp = P.like(g("dof_dilation3")), P.like(g("dof_dilation3"))
    fg, bg, b0, b1 = (P.like(g("dof_pre0")) for _ in range(4))
    out = P.like(g("dof_out"))
    r3, rh = capi.Rows(0, H >> 3), capi.Rows(0, H // 2)
    capi.check(L.dfx_pass_dof_dilation(None, P.up(g("dof_dilation2")).ref, l3.ref, r3), "D4.3")
    capi.check(L.dfx_pass_dof_blur_coc(None, l3.ref, 0, tmp.ref, r3), "D5")
    capi.check(L.dfx_pass_dof_blur_coc(None, tmp.ref, 1, l3.ref, r3), "D6")
    assert L.dfx_pass_dof_blur_coc(None, l3.ref, 1, l3.ref, r3) == capi.DFX_ERR_INVALID_ARG  # not in-place
    capi.check(L.dfx_pass_dof_prefilter(None, src.ref, coc.ref, P.up(g("dof_dilation3")).ref, fg.ref, bg.ref, rh), "D7")
    capi.check(L.dfx_pass_dof_bokeh(None, cams, C.byref(a), FLAGS, 0, fg.ref, bg.ref, src.ref, b0.ref, b1.ref, rh), "D8")
    capi.check(L.dfx_pass_dof_bokeh(None, cams, C.byref(a), FLAGS, 1, b0.ref, b1.ref, None, fg.ref, bg.ref, rh), "D9")
    chained = {"D6 chained": (l3.host(), g("dof_dilation3")), "D9 chained.near": (fg.host(), g("dof_pre0")), "D9 chained.far": (bg.host(), g("dof_pre1"))}
    capi.check(L.dfx_pass_dof_postfilter(None, fg.ref, bg.ref, b0.ref, b1.ref, rh), "D10")
    capi.check(L.dfx_pass_dof_combine(None, C.byref(a), src.ref, b0.ref, b1.ref, out.ref, capi.Rows(0, H)), "D11")
    chained.update({"D10 chained.near": (b0.host(), g("dof_bokeh0")), "D10 chained.far": (b1.host(), g("dof_bokeh1")), "D11 chained": (out.host(), g("dof_out"))})
    assert_default(chained, v, "D")


@pytest.mark.gpu
def test_cuda_dof_in_the_chain(ref):
    from diligentfx_b200.chain import ChainConfig, PostProcessChain
    seq, o = ref
    chain = PostProcessChain(W, H, ChainConfig(dof=_attribs(), dof_flags=FLAGS))
    for fr in seq:
        ldr = chain.run_frame(fr).cpu().numpy()
    assert psnr(chain.fetch("dof", 1), o.get("dof_coc")) >= 80.0
    assert psnr(reinhard(chain.fetch("dof", 0)), reinhard(o.get("dof_out"))) >= 45.0
    assert psnr(np.clip(ldr[..., :3], 0, 1), np.clip(o.get("ldr")[..., :3], 0, 1)) >= 45.0
    # and it is a different picture from the chain without it
    plain = PostProcessChain(W, H)
    for fr in seq:
        ldr0 = plain.run_frame(fr).cpu().numpy()
    assert psnr(np.clip(ldr[..., :3], 0, 1), np.clip(ldr0[..., :3], 0, 1)) < 40.0
    chain.close(), plain.close()
