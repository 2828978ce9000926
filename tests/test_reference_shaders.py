"""Pins the oracle against the reference ITSELF: every pass of the oracle is compared with the reference's own HLSL pixel
shader for that pass, compiled for the CPU by oracle/refshader (sources read in place from a DiligentFX tree, never copied) and
run on the same inputs.

Bar: BIT-EXACT. The shader runner and the oracle state the HLSL intrinsics and the fixed-function sampler the same way
(fp32, no contraction, 1/256-texel bilinear snap), so any difference is a difference between the oracle's restatement and
the reference's shader text. The one tolerated pass is the first bokeh gather of DepthOfField, whose 142 bilinear taps per
pixel are aimed with a texture coordinate the shader derives from the interpolated NDC position (0.5 + 0.5 * ndc) while
the oracle uses (x + 0.5) / W: the last-bit difference moves a few taps across a 1/256-texel snap boundary. The second bokeh
gather (the 3 x 5 flood fill) aims its taps the same way; at the default settings it happens to stay bit-exact, at random
frame sizes and circles of confusion a few taps cross a boundary there too.

Where oracle/_ref/librefshaders.so exists (build() makes it where the DiligentFX tree is present) the shaders run live.
Everywhere else the reference's side of every comparison comes from tests/golden/reference_shader_checks.npz, which holds what
the shaders produced for each case: a 128-bit digest of the bits of every output compared bit for bit, the output itself where
a tolerance applies. A live run checks that file against the shaders; DFX_RECORD_REFERENCE_SHADERS=1 rewrites it.
"""
import hashlib
import os

import numpy as np
import pytest

from diligentfx_b200 import capi, synth
from oracle.refshader import refsh

from oracle.refshader.driver import EDGE_SIZES, Variant, compare_frame, make_oracle, random_trial, random_variant, variant_sequence

W, H = 157, 89                                   # odd on both axes: the odd-size branches of every mip chain run
TOLERATED = {f"{p}.{layer}": (1e-3, 0.02) for p in ("D8 dof_bokeh_first", "D9 dof_bokeh_second") for layer in ("near", "far")}   # (max abs, max fraction of texels that differ)
STORED = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_shader_checks.npz")


def _bits(a: np.ndarray) -> np.ndarray:
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _digest(a: np.ndarray) -> np.ndarray:
    a = _bits(a)
    return np.frombuffer(hashlib.sha256(repr(a.shape).encode() + a.tobytes()).digest()[:16], np.uint8)


class Reference:
    """The reference shaders' side of the comparisons, per output `name` ("<test id>/<pass label>"): the live shader output where
    librefshaders.so exists (checked against, or with DFX_RECORD_REFERENCE_SHADERS=1 recorded into, STORED), else what STORED holds."""

    def __init__(self):
        self.live = refsh.available()
        self.stored = dict(np.load(STORED)) if os.path.exists(STORED) else {}
        self.record = {} if self.live and os.environ.get("DFX_RECORD_REFERENCE_SHADERS") else None

    def _keep(self, name: str, value: np.ndarray):
        if self.record is not None:
            self.record[name] = value
        elif name in self.stored:
            assert np.array_equal(self.stored[name], value), f"{name}: the reference shaders no longer produce what {STORED} holds"

    def exact_mismatch(self, name: str, got, want) -> str | None:
        """None when the oracle's `want` has the bits of the shader's output."""
        if not self.live:
            if name not in self.stored:
                return f"{name}: no stored reference output"
            return None if np.array_equal(self.stored[name], _digest(want)) else f"{name}: NOT bit-exact (digest of the stored reference output differs)"
        self._keep(name, _digest(got))
        if np.array_equal(_bits(got), _bits(want)):                                   # bit patterns: NaN == NaN
            return None
        d = np.abs(got.astype(np.float64) - want)
        return f"{name}: NOT bit-exact (max abs {d.max():.3e}, {(d > 0).mean():.3%} of values differ)"

    def array(self, name: str, got) -> np.ndarray:
        """The shader's output itself, for comparisons with a tolerance."""
        if not self.live:
            assert name in self.stored, f"{name}: no stored reference output"
            return self.stored[name]
        got = np.ascontiguousarray(got, np.float32)
        self._keep(name, got)
        return got

    def save(self):
        if self.record:
            np.savez_compressed(STORED, **{**self.stored, **self.record})


@pytest.fixture(scope="module")
def shaders(built):
    try:
        refsh.build()
    except Exception as e:                       # pragma: no cover - only where the reference is present but does not compile
        pytest.fail(f"the reference shaders no longer compile for the CPU: {e}")
    ref = Reference()
    yield ref
    ref.save()


@pytest.fixture
def case(request):
    return request.node.name


def _run(v: Variant, frames=None, warm: int = 2, live: bool = True):
    seq = frames if frames is not None else synth.generate_sequence(W, H, warm + 1)
    h, w = seq[0]["depth"].shape
    o = make_oracle(w, h, v)
    o.set_reversed_depth(v.reversed_depth)
    try:
        for fr in seq[:warm]:
            o.set_inputs(fr)
            o.frame(v.stages())
        return compare_frame(o, seq[warm], v, with_reference=live)
    finally:
        o.set_reversed_depth(False)


def _check(ref: Reference, key: str, res):
    """res: {label: (shader output, oracle output)}; the shader output is only read where the shaders run live."""
    bad = []
    for label, (got, want) in res.items():
        assert got.shape == want.shape, label
        name = f"{key}/{label}"
        if label in TOLERATED:
            tol, frac = TOLERATED[label]
            d = np.abs(ref.array(name, got).astype(np.float64) - want)
            if d.max() > tol or (d > 0).mean() > frac:
                bad.append(f"{label}: max abs {d.max():.3e}, differing texels {(d > 0).mean():.3%}")
        else:
            msg = ref.exact_mismatch(name, got, want)
            if msg:
                bad.append(msg)
    assert not bad, "oracle differs from the reference's shaders:\n  " + "\n  ".join(bad)
    return len(res)


def test_default_chain_bit_exact(shaders, case):
    """The benchmarked configuration: every pass of PostFX, SSR, SSAO, TAA, Bloom and ToneMap, third frame of a sequence."""
    n = _check(shaders, case, _run(Variant(), live=shaders.live))
    assert n >= 45


def test_reversed_depth_bit_exact(shaders, case):
    seq = [synth.reverse_depth_frame(f) for f in synth.generate_sequence(W, H, 3)]
    _check(shaders, case, _run(Variant(reversed_depth=True), seq, live=shaders.live))


def test_half_resolution_bit_exact(shaders, case):
    _check(shaders, case, _run(Variant(ssr_flags=capi.SSR_FLAG_HALF_RESOLUTION, ssao_flags=capi.SSAO_FLAG_HALF_RESOLUTION), live=shaders.live))


def test_ssr_previous_frame_and_half_precision_depth_bit_exact(shaders, case):
    _check(shaders, case, _run(Variant(ssr_flags=1, ssao_flags=1), live=shaders.live))


@pytest.mark.parametrize("algorithm", [1, 2], ids=["hbao", "vbao"])
def test_ssao_algorithms_bit_exact(shaders, case, algorithm):
    res = _run(Variant(ssao_algorithm=algorithm), live=shaders.live)
    _check(shaders, case, {k: v for k, v in res.items() if k.startswith("A")})


@pytest.mark.parametrize("flags", [0, 1, 4, 5, 6, 7], ids=lambda f: f"taa_flags_{f}")
def test_taa_variants_bit_exact(shaders, case, flags):
    res = _run(Variant(taa_flags=flags), live=shaders.live)
    _check(shaders, case, {k: v for k, v in res.items() if k.startswith("T")})


@pytest.mark.parametrize("mode", [1, 2, 3, 5, 6, 7, 8, 9, 10, 11])
def test_tone_map_operators_bit_exact(shaders, case, mode):
    res = _run(Variant(tonemap_mode=mode, to_srgb=bool(mode & 1)), warm=0, live=shaders.live)
    _check(shaders, case, {k: v for k, v in res.items() if k.startswith("M")})


def test_depth_of_field_bit_exact(shaders, case):
    a = capi.DOFAttribs.default()
    a.MaxCircleOfConfusion = 0.02
    frames = []
    for f in synth.generate_sequence(W, H, 3):
        g = dict(f)
        for k in ("curr_camera", "prev_camera"):
            c = capi.CameraAttribs.from_buffer_copy(bytes(f[k]))
            c.fFocusDistance, c.fFStop = 6.0, 1.4
            g[k] = c
        frames.append(g)
    for flags in (capi.DOF_FLAG_TEMPORAL_SMOOTHING | capi.DOF_FLAG_KARIS_INVERSE, 0):
        res = _run(Variant(dof=True, dof_flags=flags, dof_attribs=a), frames, live=shaders.live)
        assert any(k.startswith("D11") for k in res)
        _check(shaders, f"{case}[dof_flags={flags}]", {k: v for k, v in res.items() if k[0] in "DB"})


@pytest.mark.parametrize("size", [(34, 18), (33, 17)], ids=["even", "odd"])
def test_bilateral_quad_derivatives_everywhere(shaders, case, size):
    """SSR_ComputeBilateralCleanup.fx takes ddx / ddy of the camera-space depth. With the filter branch live on EVERY pixel
    (the sequence tests reach it only where the variance is high) the oracle's 2x2 differences equal the shader's quad
    derivatives bit for bit - including, on odd-sized targets, the last column / row, whose quad partner lies outside the
    target: Direct3D runs it as a helper lane whose Load returns 0. (The oracle and dfx_ssr.cu used to clamp that partner onto
    the pixel itself; this comparison is what showed the difference, and both were changed to the Load-returns-0 rule.)"""
    from oracle import oracle_py as op
    w, h = size
    fr = synth.generate_sequence(w, h, 1)[0]
    rng = np.random.default_rng(1)
    ssr = capi.SSRAttribs.default()
    o = op.Oracle(w, h)
    o.set_ssr(ssr, 0)
    o.set_inputs(fr)
    depth = rng.uniform(0.3, 0.9, (h, w)).astype(np.float32)
    normal = np.zeros((h, w, 4), np.float32)
    normal[..., 2] = 1.0
    o.set("depth", depth), o.set("normal", normal), o.set("material", np.full((h, w, 4), 0.2, np.float32))
    o.run("ssr_mask")
    rough, mask = o.get("ssr_roughness"), o.get("ssr_mask")
    assert mask.all() and rough.min() >= 0.125                            # every pixel traced, full filter radius
    ci = fr["frame"] & 1
    rad, var = rng.uniform(0, 4, (h, w, 4)).astype(np.float32), np.ones((h, w), np.float32)
    o.set(f"ssr_radhist{ci}", rad), o.set(f"ssr_varhist{ci}", var)
    o.run("ssr_bilateral")
    want = o.get("ssr_out")
    assert np.abs(want - rad).max() > 0.1                                  # the filter really ran
    got = np.zeros_like(want)
    if shaders.live:
        refsh.run("ssr_bilateral", [depth, normal, rough, rad, var], [got], cbs=[fr["curr_camera"], ssr], mask=np.ones((h, w), np.uint8))
    _check(shaders, case, {"S7 ssr_bilateral": (got, want)})


@pytest.mark.parametrize("trial", list(range(6)) + [f"{w}x{h}" for w, h in EDGE_SIZES])
def test_random_configurations_bit_exact(shaders, case, trial):
    """driver.random_variant (seeded): random frame size - or one of the edge sizes where every pyramid reaches 1 x 1 -, scene seed,
    feature flags, tone-map operator and every attribute field the passes read. Every pass of the third frame must still equal
    its shader bit for bit. The CUDA kernels are compared with the oracle at the same draws (test_random_configurations_gpu.py)."""
    w, h, seed, v = random_variant(*random_trial(trial))
    assert _check(shaders, case, _run(v, variant_sequence(w, h, seed, v, 3), live=shaders.live)) >= 40


def test_oracle_refuses_a_bloom_pyramid_of_one_level(built):
    """At 7 x 3 the Bloom pyramid of the default radius has one level (3 x 1): the composite would sample an up-sampled level nobody
    wrote. The oracle refuses the pass and the frame, as the CUDA effect does, instead of reading an empty texture."""
    from oracle import oracle_py as op
    fr = synth.generate_sequence(7, 3, 1)[0]
    o = op.Oracle(7, 3)
    o.set_inputs(fr)
    with pytest.raises(RuntimeError, match="fewer than two pyramid levels"):
        o.frame()
    o.set("bloom_in", fr["color"])
    with pytest.raises(RuntimeError, match="fewer than two pyramid levels"):
        o.run("bloom")


@pytest.mark.parametrize("size", [(128, 64), (157, 89)], ids=["128x64", "157x89"])
def test_full_compose(shaders, case, size):
    """Hydrogent's HnPostProcess.psh (SSR re-weighted by the split-sum BRDF and exchanged for the specular IBL, then SSAO)
    against the oracle's compose_ibl, on planes that exercise opacity 0, out-of-range roughness and metals.

    The shader builds the view direction from the interpolated NDC position of the pixel; the runner interpolates it as
    -1 + 2 (x + 0.5) / W, the oracle as ((x + 0.5) / W - 0.5) / 0.5. For power-of-two sizes both are exact and the pass is
    bit-exact; for other sizes the last bit of the NDC position differs and the result agrees to 1e-5 (relative to 1 + |c|)."""
    from oracle import oracle_py as op
    w, h = size
    fr = synth.generate_sequence(w, h, 1)[0]
    rng = np.random.default_rng(5)
    color = fr["color"].copy()
    color[..., 3] = rng.choice([0.0, 0.35, 1.0], (h, w), p=[0.1, 0.2, 0.7])
    mat = fr["material"].copy()
    mat[..., 1] = rng.choice([0.0, 0.5, 1.0], (h, w))
    mat[..., 0] = np.where(rng.random((h, w)) < 0.05, 1.5, mat[..., 0])
    base = np.concatenate([rng.uniform(0.02, 1.0, (h, w, 3)), np.ones((h, w, 1))], -1).astype(np.float32)
    ibl = np.concatenate([np.exp2(rng.uniform(-4, 2, (h, w, 3))), np.ones((h, w, 1))], -1).astype(np.float32)
    ssr = np.concatenate([np.exp2(rng.uniform(-4, 3, (h, w, 3))), rng.uniform(0, 1, (h, w, 1))], -1).astype(np.float32)
    ao = rng.uniform(0.2, 1.0, (h, w)).astype(np.float32)
    o = op.Oracle(w, h)
    o.set_inputs(fr)
    o.brdf_lut(64, 512)
    lut = o.get("brdf_lut")
    for k, v in dict(color=color, material=mat, base_color=base, specular_ibl=ibl, ssr_out=ssr, ssao_out=ao).items():
        o.set(k, v)
    bits = lambda f: int(np.float32(f).view(np.uint32))  # noqa: E731
    for ssr_scale, ssao_scale in ((0.8, 0.6), (1.0, 0.0), (0.0, 1.0)):
        o.set_compose_scales(ssr_scale, ssao_scale)
        o.run("compose_ibl")
        want = o.get("composed")
        got = np.zeros_like(want)
        if shaders.live:
            refsh.run("compose_ibl", [color, ssr, ao, fr["normal"], ibl, mat, base, lut], [got], cbs=[fr["curr_camera"]], iparams=[bits(ssr_scale), bits(ssao_scale)])
        label = f"compose (SSRScale {ssr_scale}, SSAOScale {ssao_scale})"
        if w & (w - 1) == 0 and h & (h - 1) == 0:
            _check(shaders, case, {label: (got, want)})
        else:
            rel = np.abs(shaders.array(f"{case}/{label}", got).astype(np.float64) - want) / (1.0 + np.abs(want))
            assert rel.max() < 1e-5, rel.max()


def test_constant_buffer_layouts_match_the_reference_structures(shaders):
    """Each harness memcpy's the C struct of include/dfx_b200.h into the structure the reference's .fxh declares and refuses
    (error 2) when the sizes differ; feeding a short struct must therefore fail."""
    import ctypes as C
    if not shaders.live:
        pytest.skip("checks the shader harness of librefshaders.so, which is not built here")

    class Short(C.Structure):
        _fields_ = [("x", C.c_float * 3)]

    d = np.zeros((8, 8), np.float32)
    with pytest.raises(RuntimeError, match="failed with 2"):
        refsh.run("postfx_reprojected_depth", [d], [d.copy()], cbs=[Short(), Short()])
