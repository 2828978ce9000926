"""ScreenSpaceReflection::FEATURE_FLAG_HALF_RESOLUTION (ScreenSpaceReflection.hpp:64-76): S3 downsampled mask
(SSR_ComputeDownsampledStencilMask.fx:13-61), S4 one ray per 2x2 block into width/2 x height/2 targets
(SSR_ComputeIntersection.fx:283-288, pattern PostFX_Common.fxh:45-55), S5 gathering from the half-size targets
(SSR_ComputeSpatialReconstruction.fx:153-157); S6 / S7 unchanged.

CPU: known answers of the oracle for the 4x4 offset pattern and the mask rule. GPU: S3 bit-exact, S4 / S5 and the whole chain
against the oracle through the C-ABI."""
import ctypes as C

import numpy as np
import pytest

from diligentfx_b200 import capi, synth
from gpu_frame import Planes, assert_default, run_sequence
from helpers import psnr, reinhard
from oracle.refshader.driver import Variant

W, H, FRAMES = 160, 96, 3


def _oracle(w=W, h=H, threads=4):
    from oracle import oracle_py as op
    return op.Oracle(w, h, threads=threads)


def test_half_resolution_offset_pattern():
    # PostFX_Common.fxh:47-51 prints the matrix the packed constant encodes; index = ((x & 3) << 3) + ((y & 3) << 1)
    packed = 1320229860
    got = [[(packed >> (((x & 3) << 3) + ((y & 3) << 1))) & 3 for y in range(4)] for x in range(4)]
    assert got == [[0, 1, 2, 3], [3, 2, 1, 0], [1, 0, 3, 2], [2, 3, 0, 1]]
    assert all(sorted(r) == [0, 1, 2, 3] for r in got) and all(sorted(c) == [0, 1, 2, 3] for c in zip(*got))  # a Latin square


def test_oracle_downsampled_mask_rule(built):
    o = _oracle(4, 4, 1)
    depth = np.full((4, 4), 0.5, np.float32)
    depth[0:2, 0:2] = 1.0                       # block (0,0): all background -> fails
    depth[0, 2] = 1.0                           # block (1,0): one background texel, closest depth 0.5 -> passes
    rough = np.zeros((4, 4), np.float32)
    rough[2, 0] = 0.9                           # block (0,1): max roughness above the 0.2 threshold -> fails
    o.set("depth", depth), o.set("ssr_roughness", rough)
    o.run("ssr_downsample_mask")
    assert o.get("ssr_mask_half").tolist() == [[0.0, 1.0], [0.0, 1.0]]


@pytest.fixture(scope="module")
def half(built):
    seq = synth.generate_sequence(W, H, FRAMES)
    o = _oracle()
    o.set_ssr(capi.SSRAttribs.default(), capi.SSR_FLAG_HALF_RESOLUTION)
    for fr in seq:
        o.set_inputs(fr)
        o.frame()
    return seq, o


def test_oracle_half_resolution_frame_structure(half):
    _, o = half
    assert o.get("ssr_mask_half").shape == (H // 2, W // 2) and o.get("ssr_radiance").shape == (H // 2, W // 2, 4)
    assert o.get("ssr_resolved_rad").shape == (H, W, 4) and o.get("ssr_out").shape == (H, W, 4)
    out = o.get("ssr_out")
    assert np.isfinite(out).all() and out[..., 3].max() > 0.1      # some confident reflections survive


@pytest.mark.gpu
def test_cuda_half_resolution_passes(built):
    """S3 (bit-exact), S4 (one ray per 2x2 block) and S5 (gathering from the half-size targets) against the oracle on its own
    inputs, to the default bounds of gpu_frame.tolerance; ray planes neither full nor half size are refused."""
    import torch
    v = Variant(ssr_flags=capi.SSR_FLAG_HALF_RESOLUTION)
    _, res = run_sequence(synth.generate_sequence(W, H, FRAMES), v)
    assert_default(res, v, "S3", "S4", "S5")
    L, P = capi.load(), Planes("tight")
    cams = P.cameras(capi.CameraAttribs(), capi.CameraAttribs())
    depth, rough, normal, mask = P.new(H, W, fill=0.5), P.new(H, W, fill=0.0), P.new(H, W, 4, fill=0.0), P.new(H, W, fill=1, dtype=torch.uint8)
    bad = P.new(H // 2, W // 2 + 1, 4, fill=0.0)
    outs = [P.new(H, W, 4, fill=0.0), P.new(H, W, fill=0.0), P.new(H, W, fill=0.0)]
    assert L.dfx_pass_ssr_spatial(None, cams, C.byref(capi.SSRAttribs.default()), rough.ref, mask.ref, normal.ref, depth.ref, bad.ref, bad.ref,
                                  *[b.ref for b in outs], capi.Rows(0, H)) == capi.DFX_ERR_INVALID_ARG


@pytest.mark.gpu
def test_cuda_half_resolution_chain(half):
    from diligentfx_b200.chain import ChainConfig, PostProcessChain
    seq, o = half
    chain = PostProcessChain(W, H, ChainConfig(ssr_flags=capi.SSR_FLAG_HALF_RESOLUTION))
    for fr in seq:
        ldr = chain.run_frame(fr).cpu().numpy()
    assert chain.fetch("ssr", 3).shape == (H // 2, W // 2, 4)
    assert np.array_equal(chain.fetch("ssr", 20), o.get("ssr_mask_half"))
    assert psnr(reinhard(chain.fetch("ssr", 0)), reinhard(o.get("ssr_out"))) >= 38.0
    assert psnr(np.clip(ldr[..., :3], 0, 1), np.clip(o.get("ldr")[..., :3], 0, 1)) >= 49.0
    chain.close()
