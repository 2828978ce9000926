"""CPU checks of B, the selected prim's bounding box: the aliased-line rule of DESIGN.md §2 through the oracle's bare rasteriser (one pixel
per major-axis step, no gaps or doubles, the box's corners, zero-length and in-diamond segments, the diamond's ties, near-plane
clipping), GetBoxCorner's table, the oracle against a numpy restatement of BoundBox.vsh / BoundBox.psh, the constant block against
BoundBoxStructures.fxh's layout, the defaults, the exported entries and their host-side refusals, and the synthetic boxes."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from diligentfx_b200 import capi, synth
from oracle import oracle_bound_box_py as ob

ENTRIES = ["dfx_bound_box_attribs_default", "dfx_pass_bound_box", "dfx_chain_set_bound_box"]
F = np.float32


def _in_diamond(px, py, x, y):
    """numpy statement of the half-open diamond, 1/256 units."""
    du, dv = px - (256 * x + 128), py - (256 * y + 128)
    s = abs(du) + abs(dv)
    return s < 128 or (s == 128 and du >= 0 and dv >= 0)


def _segments(n, seed):
    rng = np.random.default_rng(seed)
    return [tuple(int(v) for v in rng.integers(-3000, 3000, 4)) for _ in range(n)]


def test_one_pixel_per_major_step_without_gaps_or_doubles():
    for ax, ay, bx, by in _segments(400, 1):
        px = ob.raster_fixed(ax, ay, bx, by)
        xmajor = abs(bx - ax) >= abs(by - ay)
        major, minor = (px[:, 0], px[:, 1]) if xmajor else (px[:, 1], px[:, 0])
        assert len(set(major.tolist())) == len(major), (ax, ay, bx, by)                   # no doubles
        if len(major) > 1:
            assert (np.abs(np.diff(major)) == 1).all() and (np.abs(np.diff(minor)) <= 1).all(), (ax, ay, bx, by)  # no gaps


def test_diamond_exit_on_every_pixel():
    """A pixel is drawn iff the segment meets its diamond and its end is outside it (a convex diamond is left iff the end is outside).
    Checked on a fine sampling of each segment: every diamond a sample lies well inside (by 1/256 pixel) is drawn unless the end lies in
    it, and no drawn diamond holds the end."""
    for ax, ay, bx, by in _segments(150, 2):
        got = {tuple(p) for p in ob.raster_fixed(ax, ay, bx, by).tolist()}
        ts = np.linspace(0.0, 1.0, 20001)
        xs, ys = ax + (bx - ax) * ts, ay + (by - ay) * ts
        ix, iy = np.floor(xs / 256.0).astype(np.int64), np.floor(ys / 256.0).astype(np.int64)
        met = set()
        for dx in (0, 1, -1):
            for dy in (0, 1, -1):
                cx, cy = ix + dx, iy + dy
                inside = np.abs(xs - (256 * cx + 128)) + np.abs(ys - (256 * cy + 128)) <= 127.0
                met |= set(zip(cx[inside].tolist(), cy[inside].tolist()))
        want = {p for p in met if not _in_diamond(bx, by, *p)}
        assert want <= got, (ax, ay, bx, by, want - got)
        assert all(not _in_diamond(bx, by, *p) for p in got), (ax, ay, bx, by)


def test_zero_length_and_in_diamond_segments_draw_nothing():
    for p in [(128, 128), (0, 0), (300, 77), (-5, 1000)]:
        assert len(ob.raster_fixed(*p, *p)) == 0
    assert len(ob.raster_fixed(128 - 60, 128 + 10, 128 + 50, 128 - 40)) == 0
    assert len(ob.raster_fixed(128, 128, 128 + 127, 128)) == 0


def test_ties_on_the_diamond_corners_and_edges():
    c = 256 * 3 + 128
    # the bottom and right corners belong to the diamond, the top and left ones do not: a segment that ends there is not drawn there
    # (the left corner of (3, 3) is the right corner of (2, 3), the top corner of (3, 3) the bottom corner of (3, 2))
    drawn = lambda *s: {tuple(p) for p in ob.raster_fixed(*s).tolist()}  # noqa: E731
    assert (3, 3) not in drawn(0, c, c + 128, c) and (2, 3) in drawn(0, c, c + 128, c)       # ends on the right corner: inside
    assert (3, 3) in drawn(2000, c, c - 128, c) and (2, 3) not in drawn(2000, c, c - 128, c)  # ends on the left corner: outside
    assert (3, 3) not in drawn(c, 0, c, c + 128) and (3, 2) in drawn(c, 0, c, c + 128)       # ends on the bottom corner: inside
    assert (3, 3) in drawn(c, 2000, c, c - 128) and (3, 2) not in drawn(c, 2000, c, c - 128)  # ends on the top corner: outside
    # a horizontal line exactly between two rows passes through the bottom corners of the upper row: that row is drawn, once per column
    px = ob.raster_fixed(0, 256 * 4, 256 * 8, 256 * 4)
    assert px[:, 1].tolist() == [3] * len(px) and px[:, 0].tolist() == list(range(len(px)))
    # a vertical line exactly between two columns: the right corners of the left column
    px = ob.raster_fixed(256 * 4, 0, 256 * 4, 256 * 8)
    assert px[:, 0].tolist() == [3] * len(px)
    # the open bottom-right edge is inside, the other three edges are not
    assert _in_diamond(c + 64, c + 64, 3, 3) and not _in_diamond(c - 64, c + 64, 3, 3) and not _in_diamond(c + 64, c - 64, 3, 3)


def test_last_pixel_rule_and_start_inside_a_diamond():
    c = 256 * 2 + 128
    px = [tuple(p) for p in ob.raster_fixed(c, c, c + 5 * 256, c).tolist()]
    assert px == [(2, 2), (3, 2), (4, 2), (5, 2), (6, 2)]                    # from centre to centre: the start drawn, the end not
    px = [tuple(p) for p in ob.raster_fixed(c + 60, c, c + 5 * 256 - 60, c).tolist()]
    assert px[0] == (2, 2) and px[-1] == (6, 2)                               # a start past the centre inside a diamond is drawn


def test_box_edges_joined_at_corners_leave_no_corner_pixel_undrawn():
    """Every corner of a projected box that lies inside a pixel's diamond is drawn by one of the edges that start there."""
    w, h = 64, 48
    for eye in ([2.5, 2.0, -2.5], [0.4, 0.6, -3.0], [-1.7, -0.8, -2.2]):
        cam = synth.look_at_camera(eye, [0.5, 0.5, 0.5], w, h)
        a = ob.chain_attribs(np.eye(4, dtype=np.float32))
        verts = ob.vertices(cam, cam, a)
        drawn = set()
        for l in range(12):
            r = ob.raster(verts[2 * l, 0], verts[2 * l + 1, 0], w, h)
            drawn |= {tuple(p) for p in r[0].tolist()}
        for v in verts[:, 0]:
            X = np.rint(F(F(F(F(v[0] / v[3]) * F(0.5)) + F(0.5)) * F(w)) * F(256.0))
            Y = np.rint(F(F(F(0.5) - F(F(v[1] / v[3]) * F(0.5))) * F(h)) * F(256.0))
            x, y = (int(X) - 1) // 256, (int(Y) - 1) // 256
            for ix in (x, x + 1):
                for iy in (y, y + 1):
                    if _in_diamond(int(X), int(Y), ix, iy) and 0 <= ix < w and 0 <= iy < h:
                        assert (ix, iy) in drawn, (eye, ix, iy)


def test_near_plane_clipping_equals_a_numpy_clip():
    rng = np.random.default_rng(4)
    for _ in range(200):
        p0 = rng.uniform(-2, 2, 4).astype(F)
        p1 = rng.uniform(-2, 2, 4).astype(F)
        p0[3], p1[3] = abs(p0[3]) + F(0.5), abs(p1[3]) + F(0.5)
        p0[2] = F(-abs(p0[2]))
        p1[2] = F(abs(p1[2])) * F(0.2)                     # p0 in front of the near plane, p1 behind it and before the far plane
        q = ob.clip(p0, p1)
        t = F(p0[2] / F(p0[2] - p1[2]))
        want = (p0 + (p1 - p0) * t).astype(F)
        assert q is not None and q[0].tobytes() == want.tobytes() and q[1].tobytes() == p1.tobytes()
    assert ob.clip([0, 0, -1, 1], [0.5, 0.5, -0.1, 1]) is None                  # entirely behind the near plane
    assert ob.raster([0.1, 0.2, -1, 1], [0.5, 0.5, -0.1, 1], 16, 16) is None
    assert ob.raster([0.1, 0.2, 2, 1], [0.5, 0.5, 3, 1], 16, 16) is None        # beyond the far plane


def test_box_corner_table_makes_the_twelve_edges():
    a = capi.BoundBoxAttribs.default()
    cam = capi.CameraAttribs()
    for k in range(4):
        cam.mViewProj.m[k][k] = 1.0
    v = ob.vertices(cam, cam, a)[:, 0, :3]
    edges = {tuple(sorted((tuple(v[2 * l]), tuple(v[2 * l + 1])))) for l in range(12)}
    cube = {(float(x), float(y), float(z)) for x in (0, 1) for y in (0, 1) for z in (0, 1)}
    want = {tuple(sorted((p, q))) for p in cube for q in cube if sum(abs(a_ - b_) for a_, b_ in zip(p, q)) == 1}
    assert edges == want and len(edges) == 12
    es = ob.vertices(cam, cam, a)[:, 2, :3]
    for i in range(24):
        assert tuple(es[i]) == tuple(v[i & ~1])                             # EDGE_START_CLIP_POS is the corner of id & ~1


def _np_vs(cam, prev, T, id_):
    def corner(i):
        if i < 8:
            i = ((i + 1) >> 1) & 3
        elif i < 16:
            i = 4 + (((i + 1) >> 1) & 3)
        else:
            i = ((i - 16) >> 1) + (i & 1) * 4
        return np.array([1.0 if i & 2 else 0.0, 1.0 if (i + 1) & 2 else 0.0, 1.0 if i & 4 else 0.0, 1.0], F)

    def mul(v, m):
        m = np.array(m.m if hasattr(m, "m") else m, F)
        out = np.zeros(4, F)
        for c in range(4):
            s = F(m[0, c] * v[0])
            for r in range(1, 4):
                s = F(s + F(m[r, c] * v[r]))
            out[c] = s
        return out

    bc = mul(corner(id_), T)
    return mul(bc, cam.mViewProj), mul(bc, prev.mViewProj), mul(mul(corner(id_ & ~1), T), cam.mViewProj)


def _np_ps(attr, cam, prev, length, mask):
    cx, cy, ex, ey = F(attr[0] / attr[3]), F(attr[1] / attr[3]), F(attr[8] / attr[11]), F(attr[9] / attr[11])
    vx, vy = F(F(cx - ex) * F(cam.f4ViewportSize[0])), F(F(cy - ey) * F(cam.f4ViewportSize[1]))
    dist = np.sqrt(F(F(vx * vx) + F(vy * vy)))
    q = F(dist / F(length))
    bit = min(int(F(F(q - np.floor(q)) * F(length))), 31)
    if not (mask >> bit) & 1:
        return None
    px, py = F(attr[4] / attr[7]), F(attr[5] / attr[7])
    return (F(F(cx - F(cam.f2Jitter[0])) - F(px - F(prev.f2Jitter[0]))), F(F(cy - F(cam.f2Jitter[1])) - F(py - F(prev.f2Jitter[1]))))


@pytest.mark.parametrize("length,mask", [(32.0, 0xFFFFFFFF), (7.5, 0x0000FFFF), (1.0, 0xAAAAAAAA), (5.25, 0x5A5A0F0F)])
def test_oracle_against_a_numpy_restatement_of_the_shaders(length, mask):
    """The vertex shader bit for bit; then, on one in-view edge at a time (depth test always passing), every drawn pixel's pattern bit and
    motion from the oracle's interpolated attributes, and the sRGB option changing nothing."""
    w, h = 61, 43
    cam = synth.look_at_camera([0.4, 0.9, -3.0], [0.2, 0.3, 0.4], w, h)
    prev = synth.look_at_camera([0.5, 0.85, -2.9], [0.2, 0.3, 0.4], w, h)
    cam.f2Jitter[0], cam.f2Jitter[1], prev.f2Jitter[0], prev.f2Jitter[1] = 0.004, -0.002, -0.001, 0.003
    T = synth.bound_box_transform([-0.5, -0.4, -0.3], [0.8, 0.7, 0.9])
    a = capi.BoundBoxAttribs.make(T, (0.3, 0.6, 0.9, 0.5), length, mask)
    verts = ob.vertices(cam, prev, a)
    for i in range(24):
        want = _np_vs(cam, prev, T, i)
        assert all(verts[i, k].tobytes() == want[k].tobytes() for k in range(3)), i
    depth = np.ones((h, w), F)
    c0, m0 = np.full((h, w, 4), -1.0, F), np.full((h, w, 2), -9.0, F)
    c, m = ob.bound_box(cam, prev, a, 2, depth, c0, m0)
    cs, ms = ob.bound_box(cam, prev, a, 3, depth, c0, m0)
    assert c.tobytes() == cs.tobytes() and m.tobytes() == ms.tobytes()
    # the last line drawing a pixel decides it: replay the lines in order with the numpy pixel shader
    want_m = m0.copy()
    for l in range(12):
        v0, v1 = verts[2 * l], verts[2 * l + 1]
        r = ob.raster(v0[0], v1[0], w, h)
        if r is None:
            continue
        for (x, y), t in zip(r[0].tolist(), r[1].tolist()):
            iw0, iw1 = F(F(1.0) / v0[0, 3]), F(F(1.0) / v1[0, 3])
            t = F(t)
            tp = F(F(t * iw1) / F(F(F(F(1.0) - t) * iw0) + F(t * iw1)))
            attr = np.array([F(v0[k // 4, k % 4] + F(F(v1[k // 4, k % 4] - v0[k // 4, k % 4]) * tp)) for k in range(12)], F)
            mv = _np_ps(attr, cam, prev, length, mask)
            if mv is not None:
                want_m[y, x] = mv
    assert m.tobytes() == want_m.tobytes()
    assert ((c == F([0.3, 0.6, 0.9, 0.5])).all(-1) == (want_m != m0).any(-1)).all()


def test_constant_block_layout_and_defaults():
    """dfx_bound_box_attribs is BoundBoxStructures.fxh's BoundBoxAttribs: float4x4 Transform, float4 Color, PatternLength, PatternMask and
    two paddings, 96 bytes; the defaults are BoundBoxRenderer::RenderAttribs'."""
    A = capi.BoundBoxAttribs
    assert C.sizeof(A) == 96
    assert [(f, getattr(A, f).offset) for f, _ in A._fields_] == [("Transform", 0), ("Color", 64), ("PatternLength", 80), ("PatternMask", 84),
                                                                  ("Padding0", 88), ("Padding1", 92)]
    lib = capi.load()
    a = A()
    lib.dfx_bound_box_attribs_default(C.byref(a))
    assert bytes(a) == bytes(A.default())
    assert np.array(a.Transform.m).tolist() == np.eye(4).tolist() and list(a.Color) == [1.0] * 4
    assert a.PatternLength == 32.0 and a.PatternMask == 0xFFFFFFFF
    assert (capi.BOUND_BOX_OPTION_CONVERT_OUTPUT_TO_SRGB, capi.BOUND_BOX_OPTION_COMPUTE_MOTION_VECTORS, capi.BOUND_BOX_OPTION_USE_REVERSE_DEPTH) == (1, 2, 4)


def test_entries_are_exported():
    out = subprocess.run(["nm", "-D", "--defined-only", capi.LIB_PATH], capture_output=True, text=True).stdout
    for e in ENTRIES:
        assert f" T {e}" in out, e
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "dfx_b200.h")).read()
    for e in ENTRIES + ["DFX_BOUND_BOX_OPTION_CONVERT_OUTPUT_TO_SRGB (1u << 0)", "DFX_BOUND_BOX_OPTION_COMPUTE_MOTION_VECTORS (1u << 1)",
                        "DFX_BOUND_BOX_OPTION_USE_REVERSE_DEPTH      (1u << 2)"]:
        assert e in header, e


def test_host_side_refusals():
    """What dfx_pass_bound_box and dfx_chain_set_bound_box refuse before touching a device: a null argument, a PatternLength that is not
    finite and > 0 (uint() of a NaN is undefined in HLSL), unknown option bits."""
    lib = capi.load()
    cams = C.c_void_p(16)
    plane = capi.Plane()
    for bad in (0.0, -1.0, float("nan"), float("inf"), float("-inf")):
        a = capi.BoundBoxAttribs.make(pattern_length=bad)
        assert lib.dfx_pass_bound_box(None, cams, C.byref(a), 0, C.byref(plane), C.byref(plane), None, capi.Rows(0, 1)) == capi.DFX_ERR_INVALID_ARG
        assert b"PatternLength" in lib.dfx_last_error()
        assert lib.dfx_chain_set_bound_box(None, C.byref(a)) == capi.DFX_ERR_INVALID_ARG
    a = capi.BoundBoxAttribs.default()
    assert lib.dfx_pass_bound_box(None, cams, C.byref(a), 8, C.byref(plane), C.byref(plane), None, capi.Rows(0, 1)) == capi.DFX_ERR_UNSUPPORTED
    assert lib.dfx_pass_bound_box(None, None, C.byref(a), 0, C.byref(plane), C.byref(plane), None, capi.Rows(0, 1)) == capi.DFX_ERR_INVALID_ARG
    assert lib.dfx_pass_bound_box(None, cams, None, 0, C.byref(plane), C.byref(plane), None, capi.Rows(0, 1)) == capi.DFX_ERR_INVALID_ARG


def test_synthetic_boxes():
    """bound_box_transform is HnRenderBoundBoxTask's Scale(max - min) * Translation(min) * PrimTransform: the unit cube's corners land on
    the extent's corners, then go through the prim transform; sphere k's box is its centre -+ radius."""
    lo, hi = np.array([-1.0, 0.5, 2.0]), np.array([1.5, 2.0, 2.25])
    m = synth.bound_box_transform(lo, hi)
    assert m.dtype == np.float32
    for c in [(0, 0, 0), (1, 0, 1), (1, 1, 1)]:
        p = np.array([*c, 1.0], np.float32) @ m
        assert np.allclose(p[:3], lo + (hi - lo) * np.array(c)) and p[3] == 1.0
    prim = np.eye(4, dtype=np.float32)
    prim[3, :3] = [10.0, 0.0, -1.0]
    assert np.allclose(synth.bound_box_transform(lo, hi, prim)[3, :3], lo + prim[3, :3])
    scene = synth.make_scene()
    b = synth.sphere_bound_box(3)
    assert np.allclose(np.array([0, 0, 0, 1.0], np.float32) @ b, [*(scene.centers[3] - scene.radii[3]), 1.0], atol=1e-5)
    assert np.allclose(np.array([1, 1, 1, 1.0], np.float32) @ b, [*(scene.centers[3] + scene.radii[3]), 1.0], atol=1e-5)
