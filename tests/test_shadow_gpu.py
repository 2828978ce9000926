"""Filterable shadow maps on the GPU (dfx_shadow_convert_to_filterable), held to the oracle bit for bit: every mode, output width and
input format on the three plane layouts with the row padding checked, 1 to 8 cascades with their own radii, ranges on both sides of the
fused / two-pass switch, the edges, hostile depth, the reference's defaults at 4 x 2048^2, the warp of every D16 code at both clamps,
repeatability, the Python wrapper and the C++ class."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import shadow_cases as SC
from diligentfx_b200 import capi, shadow, synth
from gpu_frame import LAYOUTS, MASK_FILL, Planes
from oracle import oracle_shadow_py as osh

pytestmark = pytest.mark.gpu
VSM, EVSM2, EVSM4 = SC.VSM, SC.EVSM2, SC.EVSM4
_TORCH = {np.dtype(np.float32): torch.float32, np.dtype(np.float16): torch.float16, np.dtype(np.uint16): torch.int16}


class Plane:
    """One device plane of (h, w, ch) `dtype` texels in a layout of gpu_frame, its row padding filled with MASK_FILL bytes."""

    def __init__(self, layout: str, h: int, w: int, ch: int, dtype, fmt: int, data: np.ndarray | None = None):
        dtype = np.dtype(dtype)
        self.h, self.w, self.bpt = h, w, ch * dtype.itemsize
        self.pitch = Planes(layout).pitch(w, self.bpt)
        self.storage = torch.full((h * self.pitch,), MASK_FILL, dtype=torch.uint8, device="cuda")
        tt = _TORCH[dtype]
        esz = dtype.itemsize
        self.t = self.storage.view(tt).as_strided((h, w, ch), (self.pitch // esz, ch, 1))
        self.dtype, self.ch = dtype, ch
        if data is not None:
            a = np.ascontiguousarray(np.asarray(data, dtype).reshape(h, w, ch))
            self.t.copy_(torch.from_numpy(a.view(np.int16) if dtype == np.uint16 else a).cuda())
        self.p = capi.Plane(self.storage.data_ptr(), self.pitch, w, h, fmt, 0)

    def host(self) -> np.ndarray:
        a = self.t.cpu().numpy()
        return a.view(np.uint16) if self.dtype == np.uint16 else a

    def padding_untouched(self) -> bool:
        raw = self.storage.cpu().numpy().reshape(self.h, self.pitch)[:, self.w * self.bpt:]
        return bool((raw == MASK_FILL).all())


def convert(mode, attribs, depth: np.ndarray, is32: bool, layout: str = "tight", intermediate: bool = True, two_pass: bool = False,
            shared_input: bool = False):
    """Runs the C-ABI entry (two_pass: the tests' two-pass hook); returns (status, (n, h, w, ch) stored texels, planes), the
    intermediate last when there is one. shared_input: every cascade reads one plane holding depth[0]."""
    n, h, w = depth.shape
    fmt, ch, tdt = shadow.filterable_format(mode, is32)
    odt = {torch.uint16: np.uint16, torch.float16: np.float16, torch.float32: np.float32}[tdt]
    in_fmt = capi.FORMAT_R16U if depth.dtype == np.uint16 else capi.FORMAT_R32F
    ins = [Plane(layout, h, w, 1, depth.dtype, in_fmt, depth[i]) for i in range(1 if shared_input else n)]
    ins = ins * n if shared_input else ins
    outs = [Plane(layout, h, w, ch, odt, fmt) for _ in range(n)]
    inter = Plane(layout, h, w, ch, odt, fmt) if intermediate else None
    fn = capi.load().dfx_testing_shadow_convert_two_pass if two_pass else capi.load().dfx_shadow_convert_to_filterable
    st = fn(None, mode, C.byref(attribs), (capi.Plane * n)(*[p.p for p in ins]), n,
                                                      (capi.Plane * n)(*[p.p for p in outs]), C.byref(inter.p) if inter else None)
    torch.cuda.synchronize()
    got = np.stack([p.host() for p in outs]) if st == capi.DFX_OK else None
    return st, got, ins + outs + ([inter] if inter else [])


def check(mode, attribs, depth, is32, layout="tight", what="", two_pass=False):
    st, got, planes = convert(mode, attribs, depth, is32, layout, two_pass=two_pass)
    assert st == capi.DFX_OK, capi.load().dfx_last_error()
    want = osh.stored(mode, is32, osh.convert(mode, attribs, depth, is32))
    SC.assert_same(got, want, what or f"mode {mode} is32 {is32} {depth.dtype} {layout}")
    assert all(p.padding_untouched() for p in planes), "a store reached the row padding"
    return got


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("d16", [False, True])
@pytest.mark.parametrize("is32", [False, True])
@pytest.mark.parametrize("mode", SC.MODES)
def test_modes_formats_layouts(mode, is32, d16, layout):
    depth = synth.shadow_cascades(2, 67, 45, seed=3, d16=d16)
    check(mode, SC.attribs(2, is32), depth, is32, layout)
    # exponents above both clamps
    check(mode, SC.attribs(2, is32, fixed=5, pos=60.0, neg=47.0), depth, is32, layout)


@pytest.mark.parametrize("n", range(1, 9))
def test_cascades_with_their_own_radii(n):
    w, h = 96, 80
    radii = [(0.3 + 1.1 * i, 4.6 - 0.55 * i) for i in range(n)]
    a = SC.attribs(n, True, fixed=0, world=1.0, scales=SC.radius_scales(radii, w, h))
    got = [osh.filter_radii(a, i, w, h) for i in range(n)]
    assert len(set(got)) == n and all(rh != rv for rh, rv in got)
    for mode in SC.MODES:
        check(mode, a, synth.shadow_cascades(n, w, h, seed=n, d16=(n % 2 == 0)), True)


@pytest.mark.parametrize("r", [0.0, 0.3, 0.5, 1.0, 1.2, 1.5, 4.5, 7.9])
def test_radii(r):
    w, h = 53, 41
    a = SC.attribs(2, False, fixed=0, world=1.0, scales=SC.radius_scales([(r, r), (r, 0.5 * r)], w, h))
    depth = synth.shadow_cascades(2, w, h, seed=11, d16=True)
    for mode in SC.MODES:
        check(mode, a, depth, False)


@pytest.mark.parametrize("fixed", [1, 2, 3, 5, 8, -4])
def test_fixed_filter_sizes(fixed):
    depth = synth.shadow_cascades(3, 40, 33, seed=5)
    for mode in SC.MODES:
        for is32 in (False, True):
            check(mode, SC.attribs(3, is32, fixed=fixed, world=0.0 if fixed > 0 else 0.7, scales=[(0.2, 0.3)] * 3), depth, is32)


@pytest.mark.parametrize("mode", SC.MODES)
def test_fused_and_two_pass_paths_agree(mode):
    """A range of 16 runs fused, 17 and 40 run the two passes. A cascade filtered alone (fused) and beside a cascade of range 17 (which
    sends the whole call down the two-pass path) gives the same bits, and both equal the oracle."""
    w, h = 150, 97
    depth = synth.shadow_cascades(2, w, h, seed=21, d16=True)
    for r0, r1 in [(16.0, 16.4), (16.0, 17.0), (3.3, 40.0)]:
        a = SC.attribs(2, True, fixed=0, world=1.0, scales=SC.radius_scales([(r0, r0 - 0.7), (r1, r1)], w, h))
        both = check(mode, a, depth, True, what=f"ranges {r0} / {r1}")
        a1 = SC.attribs(1, True, fixed=0, world=1.0, scales=SC.radius_scales([(r0, r0 - 0.7)], w, h))
        alone = check(mode, a1, depth[:1], True)
        SC.assert_same(alone[0], both[0], "the fused and the two-pass path")
    st, _, _ = convert(mode, a, depth, True, intermediate=False)
    assert st == capi.DFX_ERR_INVALID_ARG   # the two-pass path needs an intermediate


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("is32", [False, True])
@pytest.mark.parametrize("mode", SC.MODES)
def test_two_pass_hook_equals_the_fused_path(mode, is32, layout):
    """At ranges the fused path takes (0 to 16, and the iFixedFilterSize 2 skip), the public entry leaves the intermediate untouched,
    and the two-pass hook gives the same bits."""
    w, h = 131, 70
    depth = synth.shadow_cascades(4, w, h, seed=31, d16=not is32)
    for a in (SC.attribs(4, is32, fixed=0, world=1.0, scales=SC.radius_scales([(0.0, 16.0), (1.2, 0.3), (7.9, 4.5), (16.4, 15.6)], w, h)),
              SC.attribs(4, is32, fixed=2), SC.attribs(4, is32)):
        st, _, planes = convert(mode, a, depth, is32, layout)
        assert st == capi.DFX_OK and (planes[-1].storage.cpu().numpy() == MASK_FILL).all(), "the fused path wrote the intermediate"
        fused = check(mode, a, depth, is32, layout)
        two = check(mode, a, depth, is32, layout, two_pass=True)
        SC.assert_same(two, fused, "the two-pass entry and the fused path")


def test_largest_range():
    """Range 32767 (iFixedFilterSize 65536), the largest admitted, on a small map: every tap beyond the map reads 0."""
    depth = synth.shadow_cascades(2, 45, 23, seed=12, d16=True)
    for mode in SC.MODES:
        check(mode, SC.attribs(2, mode != VSM, fixed=65536), depth, mode != VSM)


@pytest.mark.parametrize("mode", SC.MODES)
def test_cascades_may_share_the_shadow_map(mode):
    """Shadow-map slices are only read, so several cascades may read one plane."""
    depth = synth.shadow_cascades(1, 70, 50, seed=14)
    depth3 = np.repeat(depth, 3, axis=0)
    a = SC.attribs(3, True, fixed=0, world=1.0, scales=SC.radius_scales([(1.0, 2.0), (5.0, 0.5), (20.0, 3.0)], 70, 50))
    st, got, _ = convert(mode, a, depth3, True, shared_input=True)
    assert st == capi.DFX_OK
    SC.assert_same(got, osh.stored(mode, True, osh.convert(mode, a, depth3, True)), "shared shadow-map plane")


@pytest.mark.parametrize("size", [(1, 1), (3, 2), (2, 3), (1, 37), (37, 1), (130, 7)])
def test_edges(size):
    w, h = size
    for r in (0.0, 1.0, 4.5, 20.0):
        a = SC.attribs(2, True, fixed=0, world=1.0, scales=SC.radius_scales([(r, r), (r * 0.5, r)], w, h))
        for mode in SC.MODES:
            for d16 in (False, True):
                check(mode, a, synth.shadow_cascades(2, w, h, seed=w * h, d16=d16), True)


@pytest.mark.parametrize("mode", SC.MODES)
def test_hostile_depth(mode):
    """Depth outside [0, 1], +-inf and NaN in D32 maps, at 16 and 32 bits."""
    depth = synth.shadow_cascades(3, 71, 38, seed=9, hostile=True)
    for is32 in (False, True):
        check(mode, SC.attribs(3, is32, fixed=0, world=1.0, scales=SC.radius_scales([(1.2, 2.5), (0.0, 6.0), (17.5, 1.0)], 71, 38)), depth, is32)


def test_reference_defaults_at_full_size():
    """ShadowMapAttribs' defaults (3 x 3 filter, EVSM exponents 40 / 5, 32-bit) on 4 x 2048^2 D16 cascades, EVSM4 and VSM."""
    depth = synth.shadow_cascades(4, 2048, 2048, seed=1, d16=True)
    for mode in (EVSM4, VSM):
        check(mode, SC.attribs(4, True), depth, True, "aligned")


def test_warp_of_every_d16_code_at_both_clamps():
    """EVSM4 with iFixedFilterSize 2 stores each texel's warp: all 65,536 D16 codes, against the oracle's warp."""
    codes = np.arange(65536, dtype=np.uint16).reshape(1, 256, 256)
    d = codes[0].astype(np.float32) / np.float32(65535)
    for pos, neg in [(100.0, 100.0), (5.54, 5.54), (40.0, 5.0)]:
        st, got, _ = convert(EVSM4, SC.attribs(1, True, fixed=2, pos=pos, neg=neg), codes, True)
        assert st == capi.DFX_OK
        want = osh.warp(d, pos, neg, True)
        SC.assert_same(got[0][..., 0], want[..., 0], f"positive warp at {pos}")
        SC.assert_same(got[0][..., 2], want[..., 1], f"negative warp at {neg}")
        SC.assert_same(got[0][..., 1], want[..., 0] * want[..., 0], f"positive moment at {pos}")
    check(EVSM4, SC.attribs(1, False, fixed=2, pos=100.0, neg=100.0), codes, False, what="16-bit clamp")


def test_repeatable():
    depth = synth.shadow_cascades(4, 300, 200, seed=2, d16=True)
    a = SC.attribs(4, True, fixed=0, world=1.0, scales=SC.radius_scales([(1, 2), (5, 5), (16, 9), (30, 2)], 300, 200))
    runs = [convert(EVSM4, a, depth, True)[1] for _ in range(3)]
    assert all(np.array_equal(runs[0].view(np.uint32), r.view(np.uint32)) for r in runs[1:])


def test_python_wrapper():
    depth = synth.shadow_cascades(3, 90, 64, seed=4, d16=True)
    t = torch.from_numpy(depth.view(np.int16)).cuda().view(torch.uint16)
    for mode, is32 in [(VSM, False), (EVSM2, False), (EVSM4, True)]:
        for a in (SC.attribs(3, is32), SC.attribs(3, is32, fixed=0, world=1.0, scales=SC.radius_scales([(1, 1), (18, 3), (2, 25)], 90, 64))):
            out = shadow.convert_to_filterable(t, mode, a, is32)
            torch.cuda.synchronize()
            got = out.cpu().view(torch.int16).numpy().view(np.uint16) if out.dtype == torch.uint16 else out.cpu().numpy()
            SC.assert_same(got, osh.stored(mode, is32, osh.convert(mode, a, depth, is32)), f"wrapper mode {mode}")
    assert shadow.convert_to_filterable(t, capi.SHADOW_MODE_PCF, SC.attribs(3), True) is None
    d32 = torch.from_numpy(synth.shadow_cascades(2, 33, 20, seed=6)).cuda()
    out = shadow.convert_to_filterable(d32, EVSM4, SC.attribs(2), True)
    torch.cuda.synchronize()
    SC.assert_same(out.cpu().numpy(), osh.convert(EVSM4, SC.attribs(2), d32.cpu().numpy(), True), "wrapper D32")


def test_cpp_shadow_map_manager(built, tmp_path):
    """tests/cpp/shadow_map_driver.cpp: ShadowMapManager::Initialize, the cascades written through GetCascadeDSV, ConvertToFilterable,
    and the filterable slices read back, against the oracle."""
    root = capi.REPO_ROOT
    exe = str(tmp_path / "shadow_map_driver")
    libdir = os.path.dirname(capi.LIB_PATH)
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", os.path.join(root, "tests", "cpp", "shadow_map_driver.cpp"), "-I",
                        os.path.join(root, "include"), "-L", libdir, "-ldfx_b200", f"-Wl,-rpath,{libdir}", "-Wl,--allow-shlib-undefined", "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    n, s = 3, 200
    for mode, is32, d16, fixed in [(VSM, False, True, 3), (EVSM2, True, False, 0), (EVSM4, False, True, 2), (EVSM4, True, True, 0)]:
        depth = synth.shadow_cascades(n, s, s, seed=mode, d16=d16)
        depth.tofile(tmp_path / "depth.bin")
        a = SC.attribs(n, is32, fixed=fixed, world=1.0, scales=SC.radius_scales([(1.5, 2.5), (20.0, 3.0), (0.4, 0.4)], s, s))
        (tmp_path / "attribs.bin").write_bytes(bytes(a))
        r = subprocess.run([exe, str(tmp_path), str(s), str(n), str(mode), str(int(is32)), str(int(d16))], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        want = osh.stored(mode, is32, osh.convert(mode, a, depth, is32))
        got = np.fromfile(tmp_path / "filterable.bin", want.dtype).reshape(want.shape)
        SC.assert_same(got, want, f"C++ mode {mode}")
