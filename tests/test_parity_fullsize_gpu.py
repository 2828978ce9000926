"""GPU parity at the sizes BASELINE.json's configurations are quoted on (test_parity_gpu.py runs at <= 333x187):

  config 2  1920x1080  SSAO A1-A8, every pass isolated on the oracle's own input planes (4th frame of a sequence);
  config 3  3840x2160  the whole chain, four consecutive frames, LDR >= 49 dB + per-stage PSNR floors; TAA and Bloom isolated;
  config 4  7680x4320  PostFX and SSR S1-S7, every pass isolated on the oracle's planes (3rd frame, PostFX + SSR stages only).

Size-dependent paths these reach and the small tests do not: the 8-level Bloom pyramid with its five exact-2:1 levels, AO taps
at prefiltered-depth mips 3-4 (the pixel radius scales with the resolution), the 16-bit packing of Hi-Z level sizes, 32-bit texel
indexing of 530 MB planes, the 1/512-texel margin of the TAA Catmull-Rom taps at 3840 / 7680 columns.
The isolated passes run through gpu_frame.run_frame, limited to the stages each size checks, to the default bounds; each test
checks the labels of the passes it names.
"""
import numpy as np
import pytest

import test_parity_gpu as P
from diligentfx_b200 import synth
from gpu_frame import assert_default, run_sequence
from oracle import oracle_py as op
from oracle.refshader.driver import Variant

pytestmark = pytest.mark.gpu


def _ctx(w, h, frames, history, before, stages):
    """The oracle runs `history` on every frame but the last and `before` on the last; run_frame then steps it through `stages`,
    comparing the CUDA passes of those stages."""
    seq = synth.generate_sequence(w, h, frames)
    v = Variant()
    o, res = run_sequence(seq, v, history, before, stages)
    return dict(w=w, h=h, seq=seq, fr=seq[-1], o=o, f=seq[-1]["frame"], v=v, res=res)


def _check(ctx, *labels):
    assert_default(ctx["res"], ctx["v"], *labels)


@pytest.fixture(scope="module")
def ctx1080(built):
    return _ctx(1920, 1080, 4, op.STAGE_POSTFX | op.STAGE_SSAO, op.STAGE_POSTFX, op.STAGE_SSAO)


@pytest.fixture(scope="module")
def ctx4k(built):
    # the chain tests compare every stage of the 4th frame: the oracle runs the stages before TAA first, run_frame the rest
    return _ctx(3840, 2160, 4, op.STAGE_ALL, op.STAGE_POSTFX | op.STAGE_SSR | op.STAGE_SSAO | op.STAGE_COMPOSE,
                op.STAGE_TAA | op.STAGE_BLOOM | op.STAGE_TONEMAP)


@pytest.fixture(scope="module")
def ctx8k(built):
    return _ctx(7680, 4320, 3, op.STAGE_POSTFX | op.STAGE_SSR, 0, op.STAGE_POSTFX | op.STAGE_SSR)


# ---- config 2: SSAO + bilateral blur at 1920x1080 ---------------------------------------------------------------------
def test_config2_ssao_prefilter_1080p(ctx1080):
    _check(ctx1080, "A1")


def test_config2_ssao_ambient_occlusion_1080p(ctx1080):
    _check(ctx1080, "A2")


def test_config2_ssao_temporal_1080p(ctx1080):
    _check(ctx1080, "A5")


def test_config2_ssao_convolute_resample_spatial_1080p(ctx1080):
    _check(ctx1080, "A6", "A7", "A8")


def test_config2_ssao_effect_1080p(ctx1080):
    """The effect object (all of A1-A8 in sequence, four frames) against the oracle's final AO plane."""
    from diligentfx_b200.chain import STAGE_POSTFX, STAGE_SSAO, ChainConfig, PostProcessChain
    from helpers import assert_close
    o, seq, h, w = ctx1080["o"], ctx1080["seq"], ctx1080["h"], ctx1080["w"]
    chain = PostProcessChain(w, h, ChainConfig(stages=STAGE_POSTFX | STAGE_SSAO))
    for fr in seq:
        chain.run_frame(fr)
    print(assert_close("ssao output 1080p", chain.fetch("ssao", 0), o.get("ssao_out"), tol=1e-2, max_outliers=2e-2, min_psnr=50.0))
    chain.close()


# ---- config 3: the whole chain at 3840x2160 ------------------------------------------------------------------------------
def test_config3_full_chain_4k(ctx4k):
    P.test_full_chain_four_frames(ctx4k)


def test_config3_bloom_passes_4k(ctx4k):
    _check(ctx4k, "B1", "B2", "B3", "B4")


def test_config3_taa_4k(ctx4k):
    _check(ctx4k, "T1")


def test_config3_fused_chain_4k(ctx4k):
    """The benchmarked configuration (fused compose + TAA, fused composite + tone map, async compute) at 4K: LDR PSNR."""
    from diligentfx_b200.chain import PostProcessChain
    from helpers import psnr
    o, seq, h, w = ctx4k["o"], ctx4k["seq"], ctx4k["h"], ctx4k["w"]
    chain = PostProcessChain(w, h)
    for fr in seq:
        ldr = chain.run_frame(fr)
    got, want = ldr.cpu().numpy(), o.get("ldr")
    p = psnr(np.clip(got[..., :3], 0, 1), np.clip(want[..., :3], 0, 1))
    print(f"benchmarked chain, LDR PSNR after 4 frames at {w}x{h}: {p:.2f} dB")
    assert p >= 49.0
    chain.close()


# ---- config 4: SSR at 7680x4320 ----------------------------------------------------------------------------------------
def test_config4_ssr_hiz_and_mask_8k(ctx8k):
    _check(ctx8k, "S1", "S2")


def test_config4_ssr_intersect_8k(ctx8k):
    _check(ctx8k, "S4")


def test_config4_ssr_spatial_temporal_bilateral_8k(ctx8k):
    _check(ctx8k, "S5", "S6", "S7")


def test_config4_postfx_prepare_8k(ctx8k):
    _check(ctx8k, "P1", "P2", "P3")
