"""B, the selected prim's bounding box, on the GPU: dfx_pass_bound_box against oracle_bound_box_py.bound_box (the oracle that
tests/test_bound_box_reference.py pins to the reference's own BoundBox.vsh / BoundBox.psh), the C++ BoundBoxRenderer, and B in the chain
against oracle_bound_box_py.frame.

The rasteriser's coverage is integer arithmetic and every floating-point operation is rounded once on both sides, so the pass is
compared bit for bit: colour, motion and the set of pixels written."""
import ctypes as C
import importlib.util
import os
import subprocess

import numpy as np
import pytest
import torch

import gpu_frame
from diligentfx_b200 import capi, synth
from diligentfx_b200.chain import ChainConfig, PostProcessChain, pack_frame
from helpers import psnr
from oracle import oracle_bound_box_py as ob
from oracle import oracle_py as op

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _gen():
    spec = importlib.util.spec_from_file_location("make_bound_box_reference", os.path.join(HERE, "golden", "make_bound_box_reference.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


M = _gen()


def _cuda(pl, case, w, h, options, color=None, motion=None, rows=None, color16=False, motion16=False, attribs=None):
    name, cam, prev, depth, rev, a = case
    c0, m0 = M.initial(w, h)
    color = c0 if color is None else color
    motion = m0 if motion is None else motion
    d = pl.up(depth)
    c = pl.native(color.astype(np.float16)) if color16 else pl.up(color)
    mo = pl.native(motion.astype(np.float16)) if motion16 else pl.up(motion)
    opts = options | (4 if rev else 0)
    capi.check(capi.load().dfx_pass_bound_box(None, pl.cameras(cam, prev), C.byref(attribs or a), C.c_uint32(opts), d.ref, c.ref, mo.ref,
                                              rows or capi.Rows(0, h)), "dfx_pass_bound_box")
    return c.host(), mo.host()


def _oracle(case, w, h, options, color=None, motion=None, attribs=None, rows=None):
    name, cam, prev, depth, rev, a = case
    c0, m0 = M.initial(w, h)
    return ob.bound_box(cam, prev, attribs or a, options | (4 if rev else 0), depth, c0 if color is None else color, m0 if motion is None else motion,
                        rows=rows)


def _same(a, b) -> bool:
    """Bit-identical, except that any NaN equals any NaN (the GPU's NaN payloads are not x86's)."""
    na, nb = np.isnan(a), np.isnan(b)
    return bool((na == nb).all() and a[~na].tobytes() == b[~nb].tobytes())


@pytest.mark.parametrize("layout", gpu_frame.LAYOUTS)
def test_every_fixture_case_is_bit_identical(built, layout):
    pl = gpu_frame.Planes(layout)
    bad, drawn = [], 0
    for (w, h) in M.SIZES:
        for case in M.cases(w, h):
            for s, v in M.variants():
                opts = s | (2 if v else 0)
                got, want = _cuda(pl, case, w, h, opts), _oracle(case, w, h, opts)
                for k in (0, 1):
                    if not _same(got[k], want[k]):
                        bad.append(f"{w}x{h} {case[0]} {opts}: {'colour motion'.split()[k]} differs at {int((got[k] != want[k]).any(-1).sum())} px")
                drawn += int((want[0][..., 3] == 0).sum())
    torch.cuda.synchronize()
    assert pl.padding_damage() == 0
    assert drawn > 1000 and not bad, "\n".join(bad[:20])


def test_untouched_pixels_keep_a_sentinel(built):
    """Uncovered, occluded and discarded pixels keep every byte (NaN payloads included); drawn ones carry the box colour."""
    w, h = 97, 61
    rng = np.random.default_rng(3)
    sentinel = rng.uniform(-5, 5, (h, w, 4)).astype(np.float32)
    sentinel.view(np.uint32)[::3, ::2, 1] = 0x7FC01234
    msent = np.full((h, w, 2), np.float32(-0.0))
    pl = gpu_frame.Planes("padded")
    for case in M.cases(w, h):
        c, m = _cuda(pl, case, w, h, 2, color=sentinel, motion=msent)
        wc, wm = _oracle(case, w, h, 2, color=sentinel, motion=msent)
        written = ~((wc.view(np.uint32) == sentinel.view(np.uint32)).all(-1))
        assert c[~written].tobytes() == sentinel[~written].tobytes() and m[~written].tobytes() == msent[~written].tobytes(), case[0]
        assert (c[written] == np.float32([0.9, 0.35, 0.125, 0.0])).all(), case[0]


def test_row_ranges_are_the_rows_of_a_full_call(built):
    w, h = 97, 61
    pl = gpu_frame.Planes("aligned")
    c0, m0 = M.initial(w, h)
    for case in [c for c in M.cases(w, h) if c[0] in ("standard/in_view", "standard/crosses_near", "ortho/camera_inside")]:
        full = _cuda(pl, case, w, h, 2)
        for y0, y1 in ((0, 61), (7, 40), (23, 24), (60, 61), (10, 10)):
            c, m = _cuda(pl, case, w, h, 2, rows=capi.Rows(y0, y1))
            assert c[y0:y1].tobytes() == full[0][y0:y1].tobytes() and m[y0:y1].tobytes() == full[1][y0:y1].tobytes(), (case[0], y0, y1)
            for a, b in ((c, c0), (m, m0)):
                assert a[:y0].tobytes() == b[:y0].tobytes() and a[y1:].tobytes() == b[y1:].tobytes(), (case[0], y0, y1)


def test_crossing_edges_keep_the_last_lines_motion(built):
    """A box seen along a diagonal: its projected edges cross and share corner pixels, where lines of different motion meet. The pass
    equals the oracle (which stores the lines in primitive order) on those pixels, and they exist."""
    w, h = 64, 48
    cam = synth.look_at_camera([2.5, 2.0, -2.5], [0.5, 0.5, 0.5], w, h)
    prev = synth.look_at_camera([2.6, 1.9, -2.3], [0.5, 0.5, 0.5], w, h)
    a = ob.chain_attribs(np.eye(4, dtype=np.float32))
    depth = np.ones((h, w), np.float32)
    case = ("diagonal", cam, prev, depth, False, a)
    pl = gpu_frame.Planes("tight")
    got, want = _cuda(pl, case, w, h, 2), _oracle(case, w, h, 2)
    assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes()
    # pixels drawn by more than one line: the rasteriser on the 12 lines' clip positions
    verts = ob.vertices(cam, prev, a)
    count = np.zeros((h, w), np.int32)
    for l in range(12):
        r = ob.raster(verts[2 * l, 0], verts[2 * l + 1, 0], w, h)
        if r is not None:
            np.add.at(count, (r[0][:, 1], r[0][:, 0]), 1)
    assert (count > 1).sum() >= 4, int((count > 1).sum())


def test_half_precision_targets(built):
    """RGBA16F / RG16F targets hold the oracle's fp32 result rounded to nearest even (numpy's float16 conversion)."""
    w, h = 97, 61
    pl = gpu_frame.Planes("padded")
    c0, m0 = M.initial(w, h)
    c0h, m0h = c0.astype(np.float16).astype(np.float32), m0.astype(np.float16).astype(np.float32)
    for case in M.cases(w, h)[:12]:
        want = _oracle(case, w, h, 2, color=c0h, motion=m0h)
        got = _cuda(pl, case, w, h, 2, color=c0h, motion=m0h, color16=True, motion16=True)
        assert _same(got[0], want[0].astype(np.float16).astype(np.float32)), case[0]
        assert _same(got[1], want[1].astype(np.float16).astype(np.float32)), case[0]


def test_srgb_option_changes_nothing(built):
    w, h = 97, 61
    pl = gpu_frame.Planes("tight")
    for case in M.cases(w, h):
        a, b = _cuda(pl, case, w, h, 2), _cuda(pl, case, w, h, 3)
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes(), case[0]


def test_refusals_on_the_device_path(built):
    lib = capi.load()
    w, h = 33, 17
    pl = gpu_frame.Planes("tight")
    case = M.cases(w, h)[0]
    d, c, m = pl.up(case[3]), pl.like(np.zeros((h, w, 4)), fill=0.0), pl.like(np.zeros((h, w, 2)), fill=0.0)
    small = pl.like(np.zeros((h - 1, w, 4)), fill=0.0)
    cams = pl.cameras(case[1], case[2])
    a = capi.BoundBoxAttribs.default()
    call = lambda opts, col, mot, attribs=a: lib.dfx_pass_bound_box(None, cams, C.byref(attribs), C.c_uint32(opts), d.ref, col.ref, mot.ref if mot else None,  # noqa: E731
                                                                     capi.Rows(0, h))
    assert call(8, c, m) == capi.DFX_ERR_UNSUPPORTED
    assert call(0, small, None) == capi.DFX_ERR_INVALID_ARG
    assert call(2, c, None) == capi.DFX_ERR_INVALID_ARG
    for bad in (0.0, -1.0, float("nan"), float("inf")):
        b = capi.BoundBoxAttribs.make(pattern_length=bad)
        assert call(0, c, None, b) == capi.DFX_ERR_INVALID_ARG, bad
    assert call(0, c, None) == capi.DFX_OK and call(7, c, m) == capi.DFX_OK
    torch.cuda.synchronize()


def test_cpp_bound_box_renderer(built, tmp_path):
    w, h = 97, 61
    case = M.cases(w, h)[0]
    exe = str(tmp_path / "bound_box_driver")
    libdir = os.path.dirname(capi.LIB_PATH)
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", os.path.join(ROOT, "tests", "cpp", "bound_box_driver.cpp"), "-I",
                        os.path.join(ROOT, "include"), "-L", libdir, "-ldfx_b200", f"-Wl,-rpath,{libdir}", "-Wl,--allow-shlib-undefined", "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    c0, m0 = M.initial(w, h)
    np.ascontiguousarray(case[3], np.float32).tofile(tmp_path / "depth.bin")
    c0.tofile(tmp_path / "color.bin"), m0.tofile(tmp_path / "motion.bin")
    (tmp_path / "cameras.bin").write_bytes(bytes(case[1]) + bytes(case[2]))
    (tmp_path / "transform.bin").write_bytes(bytes(case[5].Transform))
    np.float32([0.25, 0.5, 1.0, 0.75]).tofile(tmp_path / "rgba.bin")
    r = subprocess.run([exe, str(tmp_path), str(w), str(h), "2", "7.5", "0x0000FFFF"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    a = capi.BoundBoxAttribs.make(np.array(case[5].Transform.m, np.float32), (0.25, 0.5, 1.0, 0.75), 7.5, 0x0000FFFF)
    want = ob.bound_box(case[1], case[2], a, 2, case[3], c0, m0)
    assert (want[0][..., 3] == np.float32(0.75)).any()
    assert np.fromfile(tmp_path / "out_color.bin", np.float32).tobytes() == want[0].tobytes()
    assert np.fromfile(tmp_path / "out_motion.bin", np.float32).tobytes() == want[1].tobytes()


# ---- chain level --------------------------------------------------------------------------------------------------------------------
W, H, FRAMES = 96, 54, 4
SPHERE = 3   # a sphere of the synthetic scene in view in every frame of _seq()


def _seq():
    return synth.generate_sequence(W, H, FRAMES)                # the camera translates and turns from frame to frame


def _box():
    return synth.sphere_bound_box(SPHERE)


def _run_chain(chain, seq, gbuf=False):
    lib = capi.load()
    out, launches, planes = [], [], []
    for fr in seq:
        n0 = lib.dfx_launch_count()
        out.append(chain.run_frame(fr).cpu().numpy().copy())
        launches.append(lib.dfx_launch_count() - n0)
        if gbuf:
            planes.append((chain.inputs["color"].cpu().numpy().copy(), chain.inputs["motion"].cpu().numpy().copy()))
    return out, launches, planes


@pytest.mark.parametrize("taa", [True, False])
@pytest.mark.parametrize("with_env", [False, True])
def test_chain_matches_the_oracle_frame(built, taa, with_env):
    from oracle import oracle_env_map_py as oe
    seq = _seq()
    chain = PostProcessChain(W, H, ChainConfig(enable_taa=taa))
    cube = synth.env_map_cube(16, 3)
    if with_env:
        chain.set_environment_map(capi.ENV_MAP_TYPE_CUBE, [torch.from_numpy(l).cuda() for l in cube])
    chain.set_bound_box(_box(), color=(1.0, 0.8, 0.2, 1.0))
    got, _, planes = _run_chain(chain, seq, gbuf=True)
    o = op.Oracle(W, H)
    a = ob.chain_attribs(_box(), (1.0, 0.8, 0.2, 1.0))
    drawn = 0
    for k, fr in enumerate(seq):
        g = oe.apply(fr, 0, cube) if with_env else fr
        g = ob.apply(g, a)
        drawn += int((g["color"] != np.asarray(fr["color"], np.float32)).any(-1).sum())
        assert planes[k][0].tobytes() == g["color"].tobytes() and planes[k][1].tobytes() == g["motion"].tobytes(), k
        if taa:
            o.set_inputs(g)
            o.frame(op.STAGE_ALL)
            want = o.get("ldr")
        else:
            from oracle import oracle_compose_final_py as ocf
            want = ocf.frame(o, g)
        p = psnr(np.clip(got[k][..., :3], 0, 1), np.clip(want[..., :3], 0, 1))
        print(f"frame {k}: LDR PSNR {p:.2f} dB")
        assert p >= 49.0, (k, p)
    assert drawn > 100
    chain.close()


def test_chain_with_the_selection_outline_of_the_same_sphere(built):
    """The chain with the box and the selection outline of the sphere it bounds equals, byte for byte, the chain without the box run on
    the oracle's G-buffer with the box drawn."""
    seq = _seq()
    ch = PostProcessChain(W, H)
    ch.set_bound_box(_box())
    outs = []
    for k, fr in enumerate(seq):
        sd = torch.from_numpy(synth.selection_depth(W, H, k, [SPHERE])).cuda()
        ch.set_selection(capi.SelectionAttribs.default(), sd)
        outs.append(ch.run_frame(fr).cpu().numpy().copy())
    ref = PostProcessChain(W, H)
    a = ob.chain_attribs(_box())
    for k, fr in enumerate(seq):
        g = ob.apply(fr, a)
        sd = torch.from_numpy(synth.selection_depth(W, H, k, [SPHERE])).cuda()
        ref.set_selection(capi.SelectionAttribs.default(), sd)
        want = ref.run_frame(g).cpu().numpy()
        assert outs[k].tobytes() == want.tobytes(), k
    ch.close(), ref.close()


def test_off_issues_the_kernels_of_today_and_on_adds_one(built):
    seq = _seq()
    a = PostProcessChain(W, H)
    _, plain, _ = _run_chain(a, seq)
    b = PostProcessChain(W, H)
    b.set_bound_box(_box())
    b.set_bound_box(None)
    _, off, _ = _run_chain(b, seq)
    c = PostProcessChain(W, H)
    c.set_bound_box(_box())
    _, on, _ = _run_chain(c, seq)
    assert off == plain and on == [n + 1 for n in plain], (plain, off, on)
    for ch in (a, b, c):
        ch.close()


def test_graph_replay_equals_eager_frames(built):
    seq = _seq()
    res = []
    for graph in (True, False):
        ch = PostProcessChain(W, H, ChainConfig(graph=graph))
        ch.set_bound_box(_box(), pattern_length=7.5, pattern_mask=0x0000FFFF)
        res.append(_run_chain(ch, seq, gbuf=True))
        if graph:
            assert ch.stats()["frames_replayed"] > 0
        ch.close()
    for k in range(FRAMES):
        assert res[0][0][k].tobytes() == res[1][0][k].tobytes(), k
        assert res[0][2][k][0].tobytes() == res[1][2][k][0].tobytes() and res[0][2][k][1].tobytes() == res[1][2][k][1].tobytes(), k


def test_a_change_of_attribs_is_replayed_from_the_next_frame(built):
    seq = _seq()
    res = []
    for graph in (True, False):
        ch = PostProcessChain(W, H, ChainConfig(graph=graph))
        out = []
        for k, fr in enumerate(seq):
            ch.set_bound_box(_box(), color=(1.0, 0.0, 0.0, 1.0) if k % 2 else (0.0, 1.0, 0.0, 1.0))
            out.append(ch.run_frame(fr).cpu().numpy().copy())
        res.append(out)
        ch.close()
    for k in range(FRAMES):
        assert res[0][k].tobytes() == res[1][k].tobytes(), k


def test_packed_streaming_equals_frame_by_frame(built):
    seq = _seq()
    packed = [pack_frame(fr) for fr in seq]
    a = PostProcessChain(W, H)
    a.set_bound_box(_box())
    host = [torch.empty((H, W, 4), dtype=torch.uint8).pin_memory() for _ in range(FRAMES)]
    assert a.stream_frames(packed, ldr_host=host, packed=True) == FRAMES
    torch.cuda.synchronize()
    b = PostProcessChain(W, H)
    b.set_bound_box(_box())
    lib = capi.load()
    for k, fr in enumerate(packed):
        ins = {n: torch.from_numpy(np.ascontiguousarray(fr[n], np.float32)).cuda() for n in ("depth", "prev_depth")}
        ins["color"], ins["motion"], ins["normal"], ins["material"] = fr["color16"].cuda(), fr["motion16"].cuda(), fr["normal16"].cuda(), fr["material8"].cuda()
        ldr = b.execute(fr["frame"], fr["curr_camera"], fr["prev_camera"], ins)
        ldr8 = torch.empty((H, W, 4), dtype=torch.uint8, device="cuda")
        capi.check(lib.dfx_pass_pack_ldr8(C.c_void_p(torch.cuda.current_stream().cuda_stream), C.byref(capi.plane_of(ldr)), C.byref(capi.plane_of(ldr8)),
                                          capi.Rows(0, H)))
        assert ldr8.cpu().numpy().tobytes() == host[k].numpy().tobytes(), k
    a.close(), b.close()


@pytest.mark.parametrize("mode", [capi.VIEW_MODE_SCENE_DEPTH, capi.VIEW_MODE_EDGE_MAP, capi.VIEW_MODE_MESH_ID])
def test_box_is_drawn_in_the_debug_views(built, mode):
    seq = _seq()
    mesh = torch.from_numpy(synth.mesh_id(W, H, 0)).cuda() if mode == capi.VIEW_MODE_MESH_ID else None
    a = PostProcessChain(W, H)
    a.set_view_mode(mode, mesh)
    _, plain, _ = _run_chain(a, seq)
    b = PostProcessChain(W, H)
    b.set_view_mode(mode, mesh)
    b.set_bound_box(_box())
    _, on, planes = _run_chain(b, seq, gbuf=True)
    assert on == [n + 1 for n in plain]
    box = ob.chain_attribs(_box())
    for k, fr in enumerate(seq):
        g = ob.apply(fr, box)
        assert planes[k][0].tobytes() == g["color"].tobytes() and planes[k][1].tobytes() == g["motion"].tobytes(), k
    a.close(), b.close()


def test_box_pixels_carry_the_box_motion(built):
    """Where the box is drawn, the motion is the box's own (the oracle's GetMotionVector of its interpolated clip positions), not the
    surface's behind it; elsewhere the frame's motion is untouched."""
    seq = _seq()
    ch = PostProcessChain(W, H)
    ch.set_bound_box(_box())
    _, _, planes = _run_chain(ch, seq, gbuf=True)
    fr = seq[-1]
    mot = np.asarray(fr["motion"], np.float32)
    drawn = (planes[-1][0] != np.asarray(fr["color"], np.float32)).any(-1)
    want = ob.apply(fr, ob.chain_attribs(_box()))["motion"]
    assert drawn.sum() > 20
    assert planes[-1][1][drawn].tobytes() == want[drawn].tobytes() and planes[-1][1][~drawn].tobytes() == mot[~drawn].tobytes()
    assert (np.abs(planes[-1][1][drawn] - mot[drawn]).max(-1) > 1e-6).mean() > 0.5
    ch.close()


def test_chain_refusals(built):
    ch = PostProcessChain(W, H)
    for bad in (0.0, float("nan"), float("inf"), -3.0):
        with pytest.raises(capi.DfxError):
            ch.set_bound_box(_box(), pattern_length=bad)
    ch.close()
