"""The vector field overlay on the GPU: dfx_pass_vector_field against oracle_vector_field_py.vector_field (the oracle that
tests/test_vector_field_reference.py pins to the reference's own VectorField.vsh and default PS main), the C++ VectorFieldRenderer, and
the motion-vector view of the chain against oracle_vector_field_py.frame.

Coverage is integer arithmetic and every floating-point operation is rounded once on both sides, so with sRGB off the pass is compared
bit for bit: the stored bytes and the set of pixels written. sRGB's pow is held to the bound the environment map's sRGB cases use."""
import ctypes as C
import importlib.util
import os
import subprocess

import numpy as np
import pytest
import torch

import gpu_frame
from diligentfx_b200 import capi, synth
from diligentfx_b200.chain import STAGE_COMPOSE, STAGE_TAA, STAGE_TONEMAP, ChainConfig, PostProcessChain
from oracle import oracle_py as op
from oracle import oracle_vector_field_py as ov

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _gen():
    spec = importlib.util.spec_from_file_location("make_vector_field_reference", os.path.join(HERE, "golden", "make_vector_field_reference.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


M = _gen()


def _cuda(pl, a, options, field, color, rows=None, field16=False, color16=False, scratch=None):
    """The pass on device copies; returns (target, scratch) on the host."""
    h, w = color.shape[:2]
    f = pl.native(field.astype(np.float16)) if field16 else pl.up(field)
    c = pl.native(color.astype(np.float16)) if color16 else pl.up(color)
    s = scratch if scratch is not None else pl.up(np.zeros((h, w), np.float32))
    capi.check(capi.load().dfx_pass_vector_field(None, C.byref(a), C.c_uint32(options), f.ref, c.ref, s.ref, rows or capi.Rows(0, h)),
               "dfx_pass_vector_field")
    return c.host(), s.host()


def _same(a, b) -> bool:
    """Bit-identical, except that any NaN equals any NaN (the GPU's NaN payloads are not x86's)."""
    na, nb = np.isnan(a), np.isnan(b)
    return bool((na == nb).all() and a[~na].tobytes() == b[~nb].tobytes())


def _within_srgb_bound(got, want, sentinel) -> tuple[bool, str]:
    """The same pixels written; at most 0.5 % of the written values beyond 1e-5 relative (test_env_map_gpu's sRGB bound)."""
    wg = ~(got.view(np.uint32) == sentinel.view(np.uint32)).all(-1)
    ww = ~(want.view(np.uint32) == sentinel.view(np.uint32)).all(-1)
    if not (wg == ww).all():
        return False, f"written pixels differ at {int((wg != ww).sum())}"
    g, o = got[ww], want[ww]
    if g.size == 0:
        return True, ""
    rel = np.abs(g - o) / np.maximum(np.abs(o), 1e-3)
    frac = float((rel > 1e-5).mean())
    return frac <= 0.005, f"{frac:.3%} beyond 1e-5, largest {rel.max():.3e}"


def _synthetic(w, h):
    """(name, attribs, field) of the synth fields at the Hydrogent scale over a w x h target, with two grids each."""
    out = []
    for name, f in (("pan", synth.motion_pan(w, h)), ("rotation", synth.motion_rotation(w, h)), ("vortex", synth.motion_vortex(w, h, 0.4, 0.6)),
                    ("random", synth.motion_random(w, h, 1, 0.05)), ("extreme", synth.motion_extreme(w, h, 2))):
        for g in ((w // 20, h // 20), (w // 3, h // 4)):
            out.append((f"{name}/{g[0]}x{g[1]}", capi.VectorFieldAttribs.make(grid=g, scale=(-1.2, -1.2), end_color=(0.5, 0.5, 0.5, 1.0)), f))
    return out


@pytest.mark.parametrize("layout", gpu_frame.LAYOUTS)
def test_every_fixture_case_and_synthetic_field_is_bit_identical(built, layout):
    pl = gpu_frame.Planes(layout)
    bad, drawn = [], 0
    for (w, h) in M.SIZES:
        c0 = M.initial(w, h)
        for name, a, f in M.cases(w, h):
            got, scratch = _cuda(pl, a, 0, f, c0)
            want = ov.vector_field(a, 0, f, c0)
            if not _same(got, want):
                bad.append(f"{w}x{h} {name}: differs at {int((got != want).any(-1).sum())} px")
            if scratch.any():
                bad.append(f"{w}x{h} {name}: scratch not zero after the call")
            drawn += int((want.view(np.uint32) != c0.view(np.uint32)).any(-1).sum())
    w, h = 160, 90
    c0 = np.full((h, w, 4), np.float32(0.25))
    for name, a, f in _synthetic(w, h):
        got, scratch = _cuda(pl, a, 0, f, c0)
        if not _same(got, ov.vector_field(a, 0, f, c0)) or scratch.any():
            bad.append(f"{w}x{h} {name}")
    torch.cuda.synchronize()
    assert pl.padding_damage() == 0
    assert drawn > 10000 and not bad, "\n".join(bad[:20])


def test_srgb_within_the_environment_maps_bound(built):
    pl = gpu_frame.Planes("padded")
    bad = []
    for (w, h) in M.SIZES:
        c0 = M.initial(w, h)
        for name, a, f in M.cases(w, h):
            got, scratch = _cuda(pl, a, capi.VECTOR_FIELD_OPTION_CONVERT_OUTPUT_TO_SRGB, f, c0)
            ok, why = _within_srgb_bound(got, ov.vector_field(a, ov.OPTION_SRGB, f, c0), c0)
            if not ok or scratch.any():
                bad.append(f"{w}x{h} {name}: {why}")
    assert not bad, "\n".join(bad[:20])


def test_untouched_pixels_keep_a_sentinel(built):
    w, h = 97, 61
    rng = np.random.default_rng(3)
    sentinel = rng.uniform(-5, 5, (h, w, 4)).astype(np.float32)
    sentinel.view(np.uint32)[::3, ::2, 1] = 0x7FC01234
    pl = gpu_frame.Planes("padded")
    for name, a, f in M.cases(w, h):
        got, _ = _cuda(pl, a, 0, f, sentinel)
        want = ov.vector_field(a, 0, f, sentinel)
        kept = (want.view(np.uint32) == sentinel.view(np.uint32)).all(-1)
        assert got[kept].tobytes() == sentinel[kept].tobytes(), name
        assert _same(got, want), name


def test_row_ranges_are_the_rows_of_a_full_call(built):
    w, h = 97, 61
    pl = gpu_frame.Planes("aligned")
    c0 = M.initial(w, h)
    for name, a, f in [c for c in M.cases(w, h) if c[0] in ("vortex/dense/same", "rotation/non_divisor/other", "pan/dense/other")]:
        full, _ = _cuda(pl, a, 0, f, c0)
        union = c0.copy()
        for y0, y1 in ((0, 7), (7, 40), (40, 41), (41, 61), (10, 10)):
            got, scratch = _cuda(pl, a, 0, f, c0, rows=capi.Rows(y0, y1))
            assert got[y0:y1].tobytes() == full[y0:y1].tobytes(), (name, y0, y1)
            assert got[:y0].tobytes() == c0[:y0].tobytes() and got[y1:].tobytes() == c0[y1:].tobytes(), (name, y0, y1)
            assert not scratch.any()
            union[y0:y1] = got[y0:y1]
        assert union.tobytes() == full.tobytes(), name


def test_two_calls_give_identical_bytes_and_leave_the_scratch_zero(built):
    """The overlap rule does not depend on scheduling: the heaviest overlap (the vortex, the dense grid) twice on one scratch plane."""
    w, h = 320, 180
    pl = gpu_frame.Planes("tight")
    c0 = np.zeros((h, w, 4), np.float32)
    a = capi.VectorFieldAttribs.make(grid=(w // 2, h // 2), scale=(-1.5, -1.5), start_color=(1, 0, 0, 1), end_color=(0, 0, 1, 0))
    f = synth.motion_vortex(w, h, 0.5, 0.8)
    s = pl.up(np.zeros((h, w), np.float32))
    first, _ = _cuda(pl, a, 0, f, c0, scratch=s)
    second, scratch = _cuda(pl, a, 0, f, c0, scratch=s)
    assert first.tobytes() == second.tobytes() and not scratch.any()
    assert first.tobytes() == ov.vector_field(a, 0, f, c0).tobytes()


def test_half_precision_field_and_target(built):
    """An RG16F field reads the same values as its fp32 widening; an RGBA16F target holds the oracle's result rounded to nearest even."""
    w, h = 97, 61
    pl = gpu_frame.Planes("padded")
    c0 = M.initial(w, h).astype(np.float16).astype(np.float32)
    for name, a, f in M.cases(w, h)[::3]:
        fh = f.astype(np.float16).astype(np.float32)
        want = ov.vector_field(a, 0, fh, c0)
        got, _ = _cuda(pl, a, 0, fh, c0, field16=True)
        assert _same(got, want), name
        got, _ = _cuda(pl, a, 0, fh, c0, field16=True, color16=True)
        assert _same(got, want.astype(np.float16).astype(np.float32)), name


def test_hydrogent_grid_at_4k(built):
    w, h = 3840, 2160
    pl = gpu_frame.Planes("tight")
    a = capi.VectorFieldAttribs()
    capi.load().dfx_vector_field_attribs_hydrogent(w, h, C.c_float(1 / 60), C.byref(a))
    assert tuple(a.GridSize) == (192, 108)
    c0 = np.zeros((h, w, 4), np.float32)
    for f in (synth.motion_pan(w, h, 0.01, 0.005), synth.motion_vortex(w, h, 0.05, 0.5)):
        got, scratch = _cuda(pl, a, 0, f, c0)
        assert got.tobytes() == ov.vector_field(a, 0, f, c0).tobytes() and not scratch.any()


def test_refusals(built):
    lib = capi.load()
    w, h = 33, 17
    pl = gpu_frame.Planes("tight")
    f, c, s = pl.up(np.zeros((5, 4, 2), np.float32)), pl.up(np.zeros((h, w, 4), np.float32)), pl.up(np.zeros((h, w), np.float32))
    small = pl.up(np.zeros((h - 1, w), np.float32))
    wrong = pl.up(np.zeros((h, w, 4), np.float32))
    a = capi.VectorFieldAttribs.make(grid=(3, 2))
    call = lambda opts, field=f, col=c, scr=s, attribs=a: lib.dfx_pass_vector_field(None, C.byref(attribs), C.c_uint32(opts), field.ref, col.ref,  # noqa: E731
                                                                                      scr.ref, capi.Rows(0, h))
    assert call(2) == capi.DFX_ERR_UNSUPPORTED
    assert call(0, scr=small) == capi.DFX_ERR_INVALID_ARG
    assert call(0, field=wrong) == capi.DFX_ERR_INVALID_ARG
    assert call(0, col=s) == capi.DFX_ERR_INVALID_ARG
    for g in ((65536, 32768), (0xFFFFFFFF, 1), (0xFFFFFFFF, 0xFFFFFFFF)):  # 2 * gx * gy >= 2^32: the draw's vertex count overflows
        assert call(0, attribs=capi.VectorFieldAttribs.make(grid=g)) == capi.DFX_ERR_INVALID_ARG, g
    torch.cuda.synchronize()
    assert lib.dfx_pass_vector_field(None, C.byref(a), 0, f.ref, c.ref, s.ref, capi.Rows(3, 2)) == capi.DFX_ERR_INVALID_ARG
    nan = capi.VectorFieldAttribs.make(grid=(3, 2), scale=(float("nan"), 1.0), bias=(float("inf"), 0.0))
    assert call(0, attribs=nan) == capi.DFX_OK and call(1) == capi.DFX_OK and call(0, attribs=capi.VectorFieldAttribs.make(grid=(0, 5))) == capi.DFX_OK
    torch.cuda.synchronize()
    assert not s.host().any()


def test_cpp_vector_field_renderer(built, tmp_path):
    w, h, fw, fh = 97, 61, 40, 30
    exe = str(tmp_path / "vector_field_driver")
    libdir = os.path.dirname(capi.LIB_PATH)
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", os.path.join(ROOT, "tests", "cpp", "vector_field_driver.cpp"), "-I",
                        os.path.join(ROOT, "include"), "-L", libdir, "-ldfx_b200", f"-Wl,-rpath,{libdir}", "-Wl,--allow-shlib-undefined", "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    c0 = M.initial(w, h)
    f = synth.motion_vortex(fw, fh, 0.3, 0.5)
    f.tofile(tmp_path / "field.bin"), c0.tofile(tmp_path / "color.bin")
    for srgb in (0, 1):
        r = subprocess.run([exe, str(tmp_path), str(w), str(h), str(fw), str(fh), "24", "15", "-1.2", str(srgb)], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        a = capi.VectorFieldAttribs.make(grid=(24, 15), scale=(-1.2, -1.2), end_color=(0.5, 0.5, 0.5, 1.0))
        want = ov.vector_field(a, srgb, f, c0)
        got = np.fromfile(tmp_path / "out_color.bin", np.float32).reshape(h, w, 4)
        assert np.fromfile(tmp_path / "out_color2.bin", np.float32).tobytes() == got.tobytes()
        if srgb:
            ok, why = _within_srgb_bound(got, want, c0)
            assert ok, why
        else:
            assert got.tobytes() == want.tobytes()


# ---- chain level --------------------------------------------------------------------------------------------------------------------
W, H = 160, 90
SPHERES = [3, 11]


def _seq(n=4):
    """The synthetic sequence with a vortex added to its motion: the camera's own motion is a pixel or less at this size, too short for
    the Hydrogent scale to draw lines."""
    return [dict(fr, motion=np.asarray(fr["motion"], np.float32) + synth.motion_vortex(W, H, 0.05, 0.5)) for fr in synth.generate_sequence(W, H, n)]


def _sel_attribs():
    a = capi.SelectionAttribs.default()
    a.NonselectionDesaturationFactor, a.selection_id = 0.5, 7
    return a


def _psnr(got, want) -> float:
    mse = float(np.mean((np.clip(np.nan_to_num(got[..., :3]), 0, 1).astype(np.float64) - np.clip(np.nan_to_num(want[..., :3]), 0, 1)) ** 2))
    return 200.0 if mse == 0 else 10 * np.log10(1.0 / mse)


class _Extras:
    """E, B, the selection and the grid on a chain, and the same on the oracle's frame."""

    def __init__(self, on: bool):
        self.on = on
        self.cube = synth.env_map_cube(16, 3)
        self.box = synth.sphere_bound_box(SPHERES[0])
        self.sel_t = None

    def setup(self, chain):
        if not self.on:
            return
        chain.set_environment_map(capi.ENV_MAP_TYPE_CUBE, [torch.from_numpy(l).cuda() for l in self.cube])
        chain.set_bound_box(self.box, color=(1.0, 0.8, 0.2, 1.0))
        self.sel_t = torch.empty((H, W), dtype=torch.float32, device="cuda")
        chain.set_selection(_sel_attribs(), self.sel_t)
        chain.set_coordinate_grid(capi.GRID_FLAG_PLANES | capi.GRID_FLAG_AXES)

    def before(self, fr):
        if self.on:
            self.sel_t.copy_(torch.from_numpy(synth.selection_depth(W, H, fr["frame"], SPHERES)))

    def gbuffer(self, fr):
        from oracle import oracle_bound_box_py as ob
        from oracle import oracle_env_map_py as oe
        if not self.on:
            return fr
        return ob.apply(oe.apply(fr, 0, self.cube), ob.chain_attribs(self.box, (1.0, 0.8, 0.2, 1.0)))

    def oracle_mv(self, o, fr, elapsed):
        g = self.gbuffer(fr)
        if not self.on:
            return ov.frame(o, g, elapsed)
        return ov.frame(o, g, elapsed, synth.selection_depth(W, H, fr["frame"], SPHERES), _sel_attribs(), capi.GRID_FLAG_PLANES | capi.GRID_FLAG_AXES)


def _check_mv(got, want, fr_elapsed_field, tag):
    """The chain's motion-vector frame against the oracle's: the frame at the chain-level floor (49 dB), and the field's lines, which
    overwrite the compose's pixels, on the same pixels within the sRGB bound."""
    p = _psnr(got, want)
    assert p >= 49.0, (tag, p)
    motion, elapsed = fr_elapsed_field
    sentinel = np.full(got.shape, np.float32(-3.0))
    lines = ov.vector_field(ov.hydrogent_attribs(W, H, elapsed), ov.OPTION_SRGB, motion, sentinel)
    drawn = ~(lines == sentinel).all(-1)
    assert drawn.sum() > 20, tag
    ok, why = _within_srgb_bound(np.where(drawn[..., None], got, sentinel), lines, sentinel)
    assert ok, (tag, why)


@pytest.mark.parametrize("taa", [True, False])
@pytest.mark.parametrize("extras", [False, True])
def test_chain_motion_vector_frames_match_the_oracle(built, taa, extras):
    seq = _seq()
    chain = PostProcessChain(W, H, ChainConfig(enable_taa=taa))
    x = _Extras(extras)
    x.setup(chain)
    o = op.Oracle(W, H)
    for k, fr in enumerate(seq):
        elapsed = [1 / 60, 1 / 30, 0.0, 1 / 144][k]
        chain.set_motion_vector_view(elapsed)
        x.before(fr)
        got = chain.run_frame(fr).cpu().numpy().copy()
        gbuf = chain.inputs["motion"].cpu().numpy().copy()
        want = x.oracle_mv(o, fr, elapsed)
        assert gbuf.tobytes() == x.gbuffer(fr)["motion"].tobytes(), k
        _check_mv(got, want, (gbuf, elapsed), (taa, extras, k))
    chain.close()


def test_schedule_shaded_motion_vectors_shaded_resets_taa(built):
    """SHADED x3 -> MOTION_VECTORS x2 (two elapsed times) -> SHADED x3, each frame against the oracle's. The view's frames advance no TAA
    history on either side, so the first SHADED frame after them resets TAA (the frame indices are not consecutive), as after TAA-off
    frames."""
    seq = _seq(8)
    chain = PostProcessChain(W, H)
    o = op.Oracle(W, H)
    elapsed = [None, None, None, 1 / 60, 1 / 24, None, None, None]
    for k, fr in enumerate(seq):
        chain.set_motion_vector_view(elapsed[k])
        got = chain.run_frame(fr).cpu().numpy().copy()
        if elapsed[k] is None:
            o.set_inputs(fr)
            o.frame()
            want = o.get("ldr")
            assert _psnr(got, want) >= 49.0, (k, _psnr(got, want))
        else:
            _check_mv(got, ov.frame(o, fr, elapsed[k]), (np.asarray(fr["motion"], np.float32), elapsed[k]), k)
    chain.close()


def _launches(chain, seq, elapsed):
    lib = capi.load()
    out = []
    for fr in seq:
        if elapsed is not None:
            chain.set_motion_vector_view(elapsed)
        n0 = lib.dfx_launch_count()
        chain.run_frame(fr)
        out.append(lib.dfx_launch_count() - n0)
    return out


def test_launches(built):
    """A motion-vector frame issues F and the field's two launches, whatever the TAA setting (E, B and J when on, with the camera upload
    E and B read); a chain that switched the view on and off before its first frame issues the kernels of one that never had it."""
    seq = _seq()
    lib = capi.load()
    plain = _launches(PostProcessChain(W, H), seq, None)
    c = PostProcessChain(W, H)
    n0 = lib.dfx_launch_count()
    c.set_motion_vector_view(1 / 60)
    c.set_motion_vector_view(None)
    assert lib.dfx_launch_count() == n0
    assert _launches(c, seq, None) == plain
    for taa in (True, False):
        assert _launches(PostProcessChain(W, H, ChainConfig(enable_taa=taa)), seq, 1 / 60) == [3] * len(seq), taa
    e = PostProcessChain(W, H)
    e.set_environment_map(capi.ENV_MAP_TYPE_CUBE, [torch.from_numpy(l).cuda() for l in synth.env_map_cube(16, 3)])
    e.set_bound_box(synth.sphere_bound_box(SPHERES[0]))
    assert _launches(e, seq, 1 / 60) == [3 + 3] * len(seq)  # + camera upload, E, B
    s = PostProcessChain(W, H)
    sel = torch.from_numpy(synth.selection_depth(W, H, 0, SPHERES)).cuda()
    s.set_selection(_sel_attribs(), sel)
    n_sel = _launches(s, seq, 1 / 60)
    assert all(n > 3 for n in n_sel) and len(set(n_sel)) == 1


def test_graph_replay_with_a_new_elapsed_time_every_frame_equals_eager(built):
    seq = _seq(6)
    res, built_counts = [], []
    for graph in (True, False):
        ch = PostProcessChain(W, H, ChainConfig(graph=graph))
        out, counts = [], []
        for k, fr in enumerate(seq):
            ch.set_motion_vector_view(1 / (30 + 7 * k))
            out.append(ch.run_frame(fr).cpu().numpy().copy())
            counts.append(ch.stats())
        res.append(out)
        if graph:
            built_counts = counts
        ch.close()
    for k in range(len(seq)):
        assert res[0][k].tobytes() == res[1][k].tobytes(), k
    # one graph per frame parity (the ping-pong planes), recorded on the first replayed frame of each; none after that
    first = next(i for i, s in enumerate(built_counts) if s["frames_replayed"] > 0)
    assert all(s["graphs_built"] == built_counts[first + 1]["graphs_built"] <= 2 for s in built_counts[first + 1:])
    assert built_counts[-1]["frames_replayed"] >= len(seq) - 2


def test_chain_refusals(built):
    ch = PostProcessChain(W, H)
    for bad in (float("nan"), float("inf"), -float("inf")):
        with pytest.raises(capi.DfxError):
            ch.set_motion_vector_view(bad)
    with pytest.raises(capi.DfxError) as e:
        ch.set_view_mode(capi.VIEW_MODE_MOTION_VECTORS)
    assert "set_motion_vector_view" in str(e.value)
    ch.set_motion_vector_view(-1.0)  # clamps to 0.001, as Hydrogent's max does
    cfg = capi.ChainConfigC()
    capi.check(ch.lib.dfx_chain_get_config(ch.chain, C.byref(cfg)))
    for drop in (STAGE_COMPOSE, STAGE_TONEMAP):
        bad = capi.ChainConfigC.from_buffer_copy(bytes(cfg))
        bad.stages &= ~drop
        assert ch.lib.dfx_chain_set_config(ch.chain, C.byref(bad)) == capi.DFX_ERR_INVALID_ARG
    no_taa = capi.ChainConfigC.from_buffer_copy(bytes(cfg))
    no_taa.stages &= ~STAGE_TAA
    assert ch.lib.dfx_chain_set_config(ch.chain, C.byref(no_taa)) == capi.DFX_OK  # the view needs no TAA
    ch.set_motion_vector_view(None)
    capi.check(ch.lib.dfx_chain_set_config(ch.chain, C.byref(cfg)))
    lacking = capi.ChainConfigC.from_buffer_copy(bytes(cfg))
    lacking.stages &= ~STAGE_TONEMAP
    capi.check(ch.lib.dfx_chain_set_config(ch.chain, C.byref(lacking)))
    with pytest.raises(capi.DfxError):
        ch.set_motion_vector_view(1 / 60)
    ch.close()
