"""ScreenSpaceAmbientOcclusion::FEATURE_FLAG_HALF_RESOLUTION (ScreenSpaceAmbientOcclusion.hpp:59-82): A0 checkerboard depth
(SSAO_ComputeDownsampledDepth.fx:8-29), A1-A3 at width/2 x height/2 (GetInvViewportSize() doubled, SSAO_ComputeAmbientOcclusion.fx:
68-75), A4 joint-bilateral upsampling (SSAO_ComputeBilateralUpsampling.fx:62-139), A5-A8 at full resolution.

CPU: hand-computed known answers for the oracle's A0 / A4 and the structure of a half-resolution frame. GPU: every new
pass against the oracle through the C-ABI, then the whole chain with the flag."""
import numpy as np
import pytest

from diligentfx_b200 import capi, synth
from gpu_frame import Planes, assert_default, run_sequence
from helpers import psnr
from oracle.refshader.driver import Variant

W, H, FRAMES = 160, 96, 3


def _oracle(w=W, h=H, threads=4):
    from oracle import oracle_py as op
    return op.Oracle(w, h, threads=threads)


def test_oracle_checkerboard_known_answer(built):
    o = _oracle(4, 4, 1)
    d = np.array([[0.1, 0.2, 0.5, 0.6], [0.3, 0.4, 0.7, 0.8], [0.9, 0.8, 0.2, 0.1], [0.7, 0.6, 0.4, 0.3]], np.float32)
    o.set("depth", d)
    o.run("ssao_downsample")
    got = o.get("ssao_checker")
    # (x + y) even -> min of the 2x2 block, odd -> max (ComputeCheckerboardPattern :8-11)
    want = np.array([[0.1, 0.8], [0.9, 0.1]], np.float32)
    assert got.shape == (2, 2) and np.allclose(got, want, atol=1e-7), got


def test_oracle_upsampling_properties(built):
    fr = synth.generate_sequence(64, 40, 1)[0]
    o = _oracle(64, 40, 2)
    o.set_inputs(fr)
    o.set("ssao_occ", np.full((20, 32), 0.37, np.float32))
    o.run("ssao_upsample")
    up = o.get("ssao_occ_up")
    bg = fr["depth"] >= 1.0 - 1e-6
    assert up.shape == (40, 64) and bg.any() and (~bg).any()
    assert np.all(up[bg] == 1.0)                                  # background pixels: 1.0 (:71-73)
    # a normalised filter reproduces a constant signal — except where every depth weight exp(-alpha^2 / 1.1e-4) is denormal
    # (silhouette pixels whose 9 half-res neighbours are all at another depth): the quotient of two denormals is coarse
    dev = np.abs(up[~bg] - 0.37)
    assert np.median(dev) < 1e-7 and (dev > 1e-6).mean() < 2e-3 and dev.max() < 0.05


def test_oracle_half_resolution_frame_structure(built):
    seq = synth.generate_sequence(W, H, FRAMES)
    o = _oracle()
    o.set_ssao_flags(capi.SSAO_FLAG_HALF_RESOLUTION)
    for fr in seq:
        o.set_inputs(fr)
        o.frame()
    assert o.get("ssao_checker").shape == (H // 2, W // 2) and o.get("ssao_occ").shape == (H // 2, W // 2)
    assert o.get("ssao_occ_up").shape == (H, W) and o.get("ssao_out").shape == (H, W)
    out = o.get("ssao_out")
    assert np.isfinite(out).all() and 0.0 <= out.min() and out.max() <= 1.0 + 1e-6 and out.std() > 0.01


@pytest.mark.gpu
def test_cuda_half_resolution_passes(built):
    """A0 (bit-exact), A2 at half resolution and A4 against the oracle on its own inputs, to the default bounds of
    gpu_frame.tolerance; an A0 output that is not half the depth plane is refused instead of written out of bounds."""
    v = Variant(ssao_flags=capi.SSAO_FLAG_HALF_RESOLUTION)
    _, res = run_sequence(synth.generate_sequence(W, H, 2), v)
    assert_default(res, v, "A0", "A2", "A4")
    P = Planes("tight")
    assert capi.load().dfx_pass_ssao_downsample_depth(None, P.new(H, W, fill=0.5).ref, P.new(H // 2 + 1, W // 2).ref, capi.Rows(0, H // 2)) == \
        capi.DFX_ERR_INVALID_ARG


@pytest.mark.gpu
def test_cuda_half_resolution_chain(built):
    from diligentfx_b200.chain import ChainConfig, PostProcessChain
    seq = synth.generate_sequence(W, H, FRAMES)
    o = _oracle()
    o.set_ssao_flags(capi.SSAO_FLAG_HALF_RESOLUTION)
    chain = PostProcessChain(W, H, ChainConfig(ssao_flags=capi.SSAO_FLAG_HALF_RESOLUTION))
    for fr in seq:
        o.set_inputs(fr)
        o.frame()
        ldr = chain.run_frame(fr).cpu().numpy()
    assert chain.fetch("ssao", 1).shape == (H // 2, W // 2)       # raw occlusion is half size
    assert psnr(chain.fetch("ssao", 5), o.get("ssao_occ_up")) >= 50.0
    assert psnr(chain.fetch("ssao", 0), o.get("ssao_out")) >= 50.0
    assert psnr(np.clip(ldr[..., :3], 0, 1), np.clip(o.get("ldr")[..., :3], 0, 1)) >= 49.0
    # switching the mode on a live chain re-allocates and resets the temporal state instead of mixing sizes
    chain.cfg.ssao_flags = 0
    full = chain.run_frame({**seq[-1], "frame": seq[-1]["frame"] + 1}).cpu().numpy()
    assert chain.fetch("ssao", 1).shape == (H, W) and np.isfinite(full).all()
    chain.close()


def test_oracle_half_precision_depth_offset(built):
    """FEATURE_FLAG_HALF_PRECISION_DEPTH: what the shaders see of it is the self-occlusion offset 0.005 instead of 0.00001
    (SSAO_ComputeAmbientOcclusion.fx:145-150): the centre point is pushed further off the surface, so the raw AO can only
    get brighter on average; storage stays fp32."""
    seq = synth.generate_sequence(W, H, 1)
    outs = []
    for flags in (0, 1):
        o = _oracle()
        o.set_ssao_flags(flags)
        o.set_inputs(seq[0])
        o.frame()
        outs.append(o.get("ssao_occ"))
    assert not np.array_equal(outs[0], outs[1]) and outs[1].mean() > outs[0].mean()


@pytest.mark.gpu
def test_cuda_half_precision_depth_flag(built):
    from diligentfx_b200.chain import ChainConfig, PostProcessChain
    seq = synth.generate_sequence(W, H, FRAMES)
    o = _oracle()
    o.set_ssao_flags(1)
    chain = PostProcessChain(W, H, ChainConfig(ssao_flags=1, postfx_flags=2))  # SSAO + PostFX HALF_PRECISION_DEPTH
    for fr in seq:
        o.set_inputs(fr)
        o.frame()
        ldr = chain.run_frame(fr).cpu().numpy()
    assert psnr(chain.fetch("ssao", 1), o.get("ssao_occ")) >= 50.0
    assert psnr(chain.fetch("ssao", 0), o.get("ssao_out")) >= 50.0
    assert psnr(np.clip(ldr[..., :3], 0, 1), np.clip(o.get("ldr")[..., :3], 0, 1)) >= 49.0
    chain.close()
