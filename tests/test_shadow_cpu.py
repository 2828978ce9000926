"""Filterable shadow maps without a GPU: the constant blocks' layout, the filter radii, the PCF no-op and every refusal of
dfx_shadow_convert_to_filterable (all decided before any device work), the new formats refused by the other passes, ShadowMapManager.hpp
on its own, and properties of the oracle that do not depend on the reference."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import shadow_cases as SC
from diligentfx_b200 import capi, shadow, synth
from oracle import oracle_shadow_py as osh

ROOT = capi.REPO_ROOT
# device addresses that are never dereferenced: every call below is refused on the host, before any launch. Each role has its own
# range so that no two planes of a call overlap unless a test makes them.
FAKE, FAKE_OUT, FAKE_INTER = 0x10000, 0x10000 + (1 << 32), 0x10000 + (1 << 33)
OK, BAD = capi.DFX_OK, capi.DFX_ERR_INVALID_ARG
VSM, EVSM2, EVSM4 = SC.VSM, SC.EVSM2, SC.EVSM4


@pytest.fixture(scope="module", autouse=True)
def _built(built):
    osh.build()


# BasicStructures.fxh:6-14 and :28-67 (C++ form): name -> byte offset
OFFSETS = {"mWorldToLightView": 0, "Cascades": 64, "mWorldToShadowMapUVDepth": 576, "fCascadeCamSpaceZEnd": 1088, "f4ShadowMapDim": 1120,
           "iNumCascades": 1136, "fNumCascades": 1140, "bVisualizeCascades": 1144, "bVisualizeShadowing": 1148,
           "fReceiverPlaneDepthBiasClamp": 1152, "fFixedDepthBias": 1156, "fCascadeTransitionRegion": 1160, "iMaxAnisotropy": 1164,
           "fVSMBias": 1168, "fVSMLightBleedingReduction": 1172, "fEVSMPositiveExponent": 1176, "fEVSMNegativeExponent": 1180,
           "bIs32BitEVSM": 1184, "iFixedFilterSize": 1188, "fFilterWorldSize": 1192, "fDummy": 1196}


def test_struct_layouts_and_defaults():
    assert C.sizeof(capi.CascadeAttribs) == 64 and C.sizeof(capi.ShadowMapAttribs) == 1200
    assert [capi.CascadeAttribs.f4LightSpaceScale.offset, capi.CascadeAttribs.f4LightSpaceScaledBias.offset,
            capi.CascadeAttribs.f4StartEndZ.offset, capi.CascadeAttribs.f4MarginProjSpace.offset] == [0, 16, 32, 48]
    for name, off in OFFSETS.items():
        assert getattr(capi.ShadowMapAttribs, name).offset == off, name
    d = capi.ShadowMapAttribs.default()
    f32 = lambda v: float(np.float32(v))  # noqa: E731
    assert (d.iNumCascades, d.fNumCascades, d.bVisualizeCascades, d.bVisualizeShadowing) == (0, 0.0, 0, 0)
    assert (d.fReceiverPlaneDepthBiasClamp, d.fFixedDepthBias, d.fCascadeTransitionRegion, d.iMaxAnisotropy) == (10.0, f32(1e-5), f32(0.1), 4)
    assert (d.fVSMBias, d.fVSMLightBleedingReduction, d.fEVSMPositiveExponent, d.fEVSMNegativeExponent) == (f32(1e-4), 0.0, 40.0, 5.0)
    assert (d.bIs32BitEVSM, d.iFixedFilterSize, d.fFilterWorldSize) == (1, 3, 0.0)
    # the C header and the C++ class agree with these offsets
    checks = "".join(f"static_assert(offsetof(dfx_shadow_map_attribs, {k}) == {v}, \"{k}\");\n" for k, v in OFFSETS.items())
    src = ('#include <cstddef>\n#include "dfx/ShadowMapManager.hpp"\n' + checks +
           "static_assert(sizeof(dfx_cascade_attribs) == 64 && sizeof(dfx_shadow_map_attribs) == 1200, \"sizes\");\n"
           "int main() { Diligent::HLSL::ShadowMapAttribs a; return a.iFixedFilterSize == 3 && a.bIs32BitEVSM == 1 ? 0 : 1; }\n")
    r = subprocess.run(["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-x", "c++", "-", "-I", os.path.join(ROOT, "include")],
                       input=src.encode(), capture_output=True)
    assert r.returncode == 0, r.stderr.decode()


def test_shadow_map_manager_header_is_self_contained():
    src = '#include "dfx/ShadowMapManager.hpp"\nint main() { return 0; }\n'
    r = subprocess.run(["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-x", "c++", "-", "-I", os.path.join(ROOT, "include")],
                       input=src.encode(), capture_output=True)
    assert r.returncode == 0, r.stderr.decode()


@pytest.mark.parametrize("fixed", [1, 2, 3, 4, 5, 8, 65536])
def test_fixed_filter_radius(fixed):
    a = SC.attribs(1, fixed=fixed, world=3.0, scales=[(0.5, 0.25)])
    want = float((fixed - 1) // 2)
    assert shadow.filter_radii(a, 0, 2048, 1024) == (want, want) == osh.filter_radii(a, 0, 2048, 1024)


def test_varying_radius_is_the_float_order_formula():
    rng = np.random.default_rng(0)
    f32 = np.float32
    for _ in range(300):
        world, sx, sy = (f32(v) for v in rng.uniform(0.0, 3.0, 3) * 10.0 ** rng.integers(-3, 2, 3))
        w, h = (int(v) for v in rng.integers(1, 4097, 2))
        a = SC.attribs(1, fixed=int(rng.integers(-3, 1)), world=float(world), scales=[(float(sx), float(sy))])
        want = (float(f32(f32(f32(world * sx) * f32(0.5)) / f32(2.0)) * f32(w)), float(f32(f32(f32(world * sy) * f32(0.5)) / f32(2.0)) * f32(h)))
        assert shadow.filter_radii(a, 0, w, h) == want == osh.filter_radii(a, 0, w, h)
    a = SC.attribs(8, fixed=0, world=1.0, scales=[(0.1 * (i + 1), 0.05 * (i + 1)) for i in range(8)])
    assert len({shadow.filter_radii(a, i, 64, 64) for i in range(8)}) == 8


def test_fixed_size_two_skips_the_vertical_pass():
    """iFixedFilterSize 2 has radius 0 and writes the horizontal result, each texel its own moments; size 1 runs both passes with one
    tap each, and one tap of weight 1 changes nothing."""
    depth = synth.shadow_cascades(1, 9, 7, seed=1)
    two = osh.convert(VSM, SC.attribs(1, True, fixed=2), depth, True)
    one = osh.convert(VSM, SC.attribs(1, True, fixed=1), depth, True)
    assert np.array_equal(two[0, ..., 0], depth[0]) and np.array_equal(two[0, ..., 1], depth[0] * depth[0])
    assert np.array_equal(one, two)


def test_oracle_constant_map_and_warp():
    """A constant depth gives its own moments wherever the filter stays inside the map; the warp is exp(+-c (2d - 1)) with the clamps."""
    depth = np.full((1, 16, 16), 0.25, np.float32)
    v = osh.convert(VSM, SC.attribs(1, True, fixed=5), depth, True)
    assert np.array_equal(v[0, 2:-2, 2:-2, 0], np.full((12, 12), 0.25, np.float32))
    assert np.array_equal(v[0, 2:-2, 2:-2, 1], np.full((12, 12), 0.0625, np.float32))
    d = np.linspace(0, 1, 101, dtype=np.float32)
    for pos, neg, is32, cp, cn in [(40.0, 5.0, True, 40.0, 5.0), (100.0, 100.0, True, 42.0, 42.0), (100.0, 3.0, False, 5.54, 3.0)]:
        w = osh.warp(d, pos, neg, is32)
        dd = (np.float32(2) * d - np.float32(1)).astype(np.float64)
        assert np.array_equal(w[:, 0], np.exp(np.float64(np.float32(cp) * dd.astype(np.float32))).astype(np.float32))
        assert np.array_equal(w[:, 1], -np.exp(np.float64(-np.float32(cn) * dd.astype(np.float32))).astype(np.float32))


# ------------------------------------------------------------------------------------------------------------------------------------
# the C-ABI's decisions, made before any device work


def _planes(n, w, h, fmt, base=FAKE):
    bpt = {capi.FORMAT_R8U: 1, capi.FORMAT_R16U: 2, capi.FORMAT_R32F: 4, capi.FORMAT_RG16U: 4, capi.FORMAT_RG16F: 4, capi.FORMAT_RG32F: 8,
           capi.FORMAT_RGBA16F: 8, capi.FORMAT_RGBA32F: 16}[fmt]
    return (capi.Plane * n)(*[capi.Plane(base + i * (1 << 24), w * bpt, w, h, fmt, 0) for i in range(n)])


def call(mode, a, n=None, w=64, h=64, in_fmt=capi.FORMAT_R16U, out_fmt=None, inter=None, src=None, dst=None):
    n = a.iNumCascades if n is None else n
    out_fmt = out_fmt or shadow.filterable_format(mode if mode in (VSM, EVSM2, EVSM4) else VSM, bool(a.bIs32BitEVSM))[0]
    src = _planes(max(n, 1), w, h, in_fmt) if src is None else src
    dst = _planes(max(n, 1), w, h, out_fmt, FAKE_OUT) if dst is None else dst
    return capi.load().dfx_shadow_convert_to_filterable(None, mode, C.byref(a), src, n, dst, C.byref(inter) if inter else None)


def _error() -> str:
    return capi.load().dfx_last_error().decode()


def test_pcf_is_a_no_op():
    assert capi.load().dfx_shadow_convert_to_filterable(None, capi.SHADOW_MODE_PCF, None, None, 0, None, None) == OK


@pytest.mark.parametrize("mode", [0, 5, -1])
def test_refuses_unknown_mode(mode):
    assert call(mode, SC.attribs(1)) == BAD and "unknown shadow mode" in _error()


@pytest.mark.parametrize("n", [0, 9])
def test_refuses_cascade_count_out_of_range(n):
    a = SC.attribs(1)
    a.iNumCascades = n
    assert call(VSM, a, n=n) == BAD and "cascades" in _error()


def test_refuses_cascade_count_other_than_attribs():
    assert call(EVSM4, SC.attribs(3), n=2) == BAD and "iNumCascades" in _error()


@pytest.mark.parametrize("mode", [VSM, EVSM2, EVSM4])
def test_refuses_32bit_flag_disagreeing_with_format(mode):
    a = SC.attribs(1, is32=False)
    assert call(mode, a, out_fmt=shadow.filterable_format(mode, True)[0]) == BAD and "bIs32BitEVSM" in _error()
    a = SC.attribs(1, is32=True)
    assert call(mode, a, out_fmt=shadow.filterable_format(mode, False)[0]) == BAD and "bIs32BitEVSM" in _error()


@pytest.mark.parametrize("in_fmt", [capi.FORMAT_RG32F, capi.FORMAT_R8U, capi.FORMAT_RG16U, capi.FORMAT_RGBA16F])
def test_refuses_wrong_input_format(in_fmt):
    assert call(VSM, SC.attribs(1), in_fmt=in_fmt) == BAD


@pytest.mark.parametrize("mode,out_fmt", [(VSM, capi.FORMAT_RG16F), (VSM, capi.FORMAT_RGBA32F), (EVSM2, capi.FORMAT_RG16U),
                                          (EVSM2, capi.FORMAT_RGBA16F), (EVSM4, capi.FORMAT_RG32F), (EVSM4, capi.FORMAT_R32F)])
def test_refuses_wrong_output_format(mode, out_fmt):
    assert call(mode, SC.attribs(1), out_fmt=out_fmt) == BAD


def test_refuses_mixed_formats_and_sizes():
    a = SC.attribs(2)
    src = _planes(2, 64, 64, capi.FORMAT_R16U)
    src[1].format, src[1].pitch_bytes = capi.FORMAT_R32F, 256
    assert call(VSM, a, src=src) == BAD and "slice 1" in _error()
    src = _planes(2, 64, 64, capi.FORMAT_R16U)
    src[1].width = 63
    assert call(VSM, a, src=src) == BAD and "slice 1" in _error()
    dst = _planes(2, 64, 64, capi.FORMAT_RG32F, FAKE_OUT)
    dst[0].height = 65
    assert call(VSM, a, dst=dst) == BAD and "filterable slice 0" in _error()
    dst = _planes(2, 64, 64, capi.FORMAT_RG32F, FAKE_OUT)
    dst[1].format = capi.FORMAT_RGBA32F
    assert call(VSM, a, dst=dst) == BAD
    assert call(VSM, SC.attribs(1), w=16385, h=4) == BAD and "16384" in _error()


def test_two_pass_hook_always_needs_the_intermediate():
    a = SC.attribs(1)
    src, dst = _planes(1, 64, 64, capi.FORMAT_R16U), _planes(1, 64, 64, capi.FORMAT_RG32F, FAKE_OUT)
    assert capi.load().dfx_testing_shadow_convert_two_pass(None, VSM, C.byref(a), src, 1, dst, None) == BAD and "intermediate" in _error()


def test_refuses_missing_or_mismatched_intermediate():
    a = SC.attribs(2, fixed=0, world=1.0, scales=SC.radius_scales([(1.0, 1.0), (17.0, 2.0)], 64, 64))
    assert call(EVSM4, a) == BAD and "intermediate" in _error()
    inter = capi.Plane(FAKE_INTER, 64 * 8, 64, 64, capi.FORMAT_RG32F, 0)
    assert call(EVSM4, a, inter=inter) == BAD and "intermediate" in _error()
    inter = capi.Plane(FAKE_INTER, 64 * 16, 64, 32, capi.FORMAT_RGBA32F, 0)
    assert call(EVSM4, a, inter=inter) == BAD and "intermediate" in _error()


@pytest.mark.parametrize("r", [-0.5, float("nan"), float("inf"), -float("inf"), 32767.5, 1e9])
def test_refuses_bad_radius(r):
    a = SC.attribs(1, fixed=0, world=1.0, scales=SC.radius_scales([(1.0, 1.0)], 64, 64))
    a.Cascades[0].f4LightSpaceScale[1] = r if not np.isfinite(r) else 4.0 * r / 64
    assert call(VSM, a) == BAD and "radius" in _error()


def test_largest_range_passes_the_radius_checks():
    """Range 32767 (iFixedFilterSize 65536) passes the radius checks and is refused only for its wrong intermediate, which is checked
    after them; range 32768 (65537) is refused for its radius. Nothing is launched."""
    wrong = capi.Plane(FAKE_INTER, 64 * 16, 64, 64, capi.FORMAT_RGBA32F, 0)   # VSM 32-bit needs RG32F
    a = SC.attribs(1, fixed=65536)
    assert shadow.filter_radii(a, 0, 64, 64) == (32767.0, 32767.0)
    assert call(VSM, a, inter=wrong) == BAD and "intermediate" in _error() and "radius" not in _error()
    a = SC.attribs(1, fixed=65537)
    assert call(VSM, a, inter=wrong) == BAD and "radius" in _error()


def test_refuses_overlapping_planes():
    lib = capi.load()
    a = SC.attribs(2)
    src, dst = _planes(2, 64, 64, capi.FORMAT_R16U), _planes(2, 64, 64, capi.FORMAT_RG32F, FAKE_OUT)
    dst[1].ptr = src[0].ptr + 64 * 2 * 63   # its first row is the shadow map's last
    assert call(VSM, a, dst=dst) == BAD and "filterable slice 1 overlaps shadow-map slice 0" in _error()
    dst = _planes(2, 64, 64, capi.FORMAT_RG32F, FAKE_OUT)
    dst[1].ptr = dst[0].ptr + 8 * 63        # the last texel of slice 0's first row
    assert call(VSM, a, dst=dst) == BAD and "filterable slices" in _error()
    big = SC.attribs(2, fixed=40)              # range 19: the two-pass path, which uses the intermediate
    dst = _planes(2, 64, 64, capi.FORMAT_RG32F, FAKE_OUT)
    inter = capi.Plane(dst[1].ptr + 64 * 8 * 10, 64 * 8, 64, 64, capi.FORMAT_RG32F, 0)
    assert call(VSM, big, dst=dst, inter=inter) == BAD and "the intermediate overlaps slice 1" in _error()
    inter = capi.Plane(src[0].ptr, 64 * 8, 64, 64, capi.FORMAT_RG32F, 0)
    assert lib.dfx_testing_shadow_convert_two_pass(None, VSM, C.byref(a), src, 2, dst, C.byref(inter)) == BAD
    assert "the intermediate overlaps slice 0" in _error()


@pytest.mark.parametrize("fmt", [capi.FORMAT_R16U, capi.FORMAT_RG16U])
def test_other_passes_refuse_the_shadow_formats(fmt):
    """dfx_pass_ssao_downsample_depth stands for the passes that take an fp32 plane: a UNORM16 plane is refused as input and output."""
    lib = capi.load()
    good = capi.Plane(FAKE, 256, 64, 64, capi.FORMAT_R32F, 0)
    bad = capi.Plane(FAKE, 256, 64, 64, fmt, 0)
    half = capi.Plane(FAKE, 128, 32, 32, capi.FORMAT_R32F, 0)
    bad_half = capi.Plane(FAKE, 128, 32, 32, fmt, 0)
    assert lib.dfx_pass_ssao_downsample_depth(None, C.byref(bad), C.byref(half), capi.rows_all(64)) == BAD
    assert lib.dfx_pass_ssao_downsample_depth(None, C.byref(good), C.byref(bad_half), capi.rows_all(64)) == BAD


def test_c_abi_and_python_interface():
    syms = capi.declared_symbols()
    assert "dfx_shadow_convert_to_filterable" in syms and "dfx_shadow_filter_radii" in syms
    assert not [s for s in syms if "two_pass" in s or "testing" in s]      # the path is the library's choice, not the application's
    assert hasattr(capi.load(), "dfx_testing_shadow_convert_two_pass")      # the tests' and cost tool's hook (csrc/dfx_testing.h)
    header = open(capi.HEADER_PATH).read()
    for k, v in [("DFX_SHADOW_MODE_PCF", 1), ("DFX_SHADOW_MODE_VSM", 2), ("DFX_SHADOW_MODE_EVSM2", 3), ("DFX_SHADOW_MODE_EVSM4", 4),
                 ("DFX_MAX_CASCADES", 8)]:
        assert f"#define {k}" in header and header.split(f"#define {k}")[1].split()[0] == str(v)
    assert (capi.FORMAT_R16U, capi.FORMAT_RG16U) == (9, 10) and "DFX_FORMAT_R16U    = 9" in header and "DFX_FORMAT_RG16U   = 10" in header
