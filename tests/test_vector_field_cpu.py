"""The vector field overlay on the CPU: the C-ABI's constant block, defaults, HnPostProcessTask's attribs, export and header text, the
host-side refusals, the synthetic motion fields, and the oracle (oracle_vector_field_py) against a scalar numpy restatement of
VectorField.vsh, the default PS main and the line rule of DESIGN.md §2 on hand-made fields."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from diligentfx_b200 import capi, synth
from oracle import oracle_vector_field_py as ov

ENTRIES = ["dfx_vector_field_attribs_default", "dfx_vector_field_attribs_hydrogent", "dfx_pass_vector_field", "dfx_chain_set_motion_vector_view"]
f32 = np.float32


def test_constant_block_layout_and_defaults(built):
    A = capi.VectorFieldAttribs
    assert C.sizeof(A) == 56
    assert [(f, getattr(A, f).offset) for f, _ in A._fields_] == [("Bias", 0), ("Scale", 8), ("StartColor", 16), ("EndColor", 32), ("GridSize", 48)]
    a = A()
    capi.load().dfx_vector_field_attribs_default(C.byref(a))
    assert bytes(a) == bytes(A.default())
    assert list(a.Bias) == [0, 0] and list(a.Scale) == [1, 1] and list(a.StartColor) == [1] * 4 and list(a.EndColor) == [1] * 4
    assert list(a.GridSize) == [0, 0] and capi.VECTOR_FIELD_OPTION_CONVERT_OUTPUT_TO_SRGB == 1


@pytest.mark.parametrize("elapsed", [1 / 60, 1 / 24, 0.5, 0.001, 0.0005, 0.0, -1.0, float("inf")])
def test_hydrogent_attribs(built, elapsed):
    """HnPostProcessTask.cpp:932-938: a line per 20 x 20 pixels, Scale -0.02 / max(ElapsedTime, 0.001) (0 and negative clamp), white to
    grey; the oracle's restatement agrees byte for byte."""
    a = capi.VectorFieldAttribs()
    capi.load().dfx_vector_field_attribs_hydrogent(3840, 2161, C.c_float(elapsed), C.byref(a))
    assert list(a.GridSize) == [192, 108] and list(a.Bias) == [0, 0]
    t = max(f32(elapsed), f32(0.001))
    assert a.Scale[0] == a.Scale[1] == f32(-0.02) / t
    assert list(a.StartColor) == [1, 1, 1, 1] and list(a.EndColor) == [0.5, 0.5, 0.5, 1]
    assert bytes(a) == bytes(ov.hydrogent_attribs(3840, 2161, elapsed))
    if elapsed <= 0.001:
        assert a.Scale[0] == f32(-0.02) / f32(0.001)


def test_entries_are_exported():
    out = subprocess.run(["nm", "-D", "--defined-only", capi.LIB_PATH], capture_output=True, text=True).stdout
    for e in ENTRIES:
        assert f" T {e}" in out, e
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "dfx_b200.h")).read()
    for e in ENTRIES + ["DFX_VECTOR_FIELD_OPTION_CONVERT_OUTPUT_TO_SRGB (1u << 0)", "typedef struct dfx_vector_field_attribs"]:
        assert e in header, e


def test_host_side_refusals(built):
    """What dfx_pass_vector_field and dfx_chain_set_motion_vector_view refuse before touching a device."""
    lib = capi.load()
    a = capi.VectorFieldAttribs.make(grid=(2, 2))
    empty = capi.Plane()
    call = lambda attribs, opts, f, c, s: lib.dfx_pass_vector_field(None, attribs, C.c_uint32(opts), f, c, s, capi.Rows(0, 1))  # noqa: E731
    assert call(None, 0, C.byref(empty), C.byref(empty), C.byref(empty)) == capi.DFX_ERR_INVALID_ARG
    assert call(C.byref(a), 2, C.byref(empty), C.byref(empty), C.byref(empty)) == capi.DFX_ERR_UNSUPPORTED
    assert call(C.byref(a), 0, None, C.byref(empty), C.byref(empty)) == capi.DFX_ERR_INVALID_ARG
    fake = lambda w, h, fmt, bpt: capi.Plane(C.c_void_p(1 << 20), w * bpt, w, h, fmt, 0)  # noqa: E731  (never dereferenced: refused first)
    field, color, scratch = fake(4, 4, capi.FORMAT_RG32F, 8), fake(8, 6, capi.FORMAT_RGBA32F, 16), fake(8, 6, capi.FORMAT_R32F, 4)
    assert call(C.byref(a), 0, C.byref(color), C.byref(color), C.byref(scratch)) == capi.DFX_ERR_INVALID_ARG       # field not RG
    assert call(C.byref(a), 0, C.byref(field), C.byref(scratch), C.byref(scratch)) == capi.DFX_ERR_INVALID_ARG     # target not RGBA
    assert call(C.byref(a), 0, C.byref(field), C.byref(color), C.byref(fake(8, 5, capi.FORMAT_R32F, 4))) == capi.DFX_ERR_INVALID_ARG
    assert call(C.byref(a), 0, C.byref(field), C.byref(color), C.byref(color)) == capi.DFX_ERR_INVALID_ARG        # scratch not R32F
    big = capi.VectorFieldAttribs.make(grid=(1 << 16, 1 << 15))
    assert call(C.byref(big), 0, C.byref(field), C.byref(color), C.byref(scratch)) == capi.DFX_ERR_INVALID_ARG
    assert b"32 bits" in lib.dfx_last_error()
    assert lib.dfx_pass_vector_field(None, C.byref(a), 0, C.byref(field), C.byref(color), C.byref(scratch), capi.Rows(4, 7)) == capi.DFX_ERR_INVALID_ARG
    # a GridSize of 0 or an empty row range draws nothing, after every check
    zero = capi.VectorFieldAttribs.make(grid=(0, 3))
    assert call(C.byref(zero), 1, C.byref(field), C.byref(color), C.byref(scratch)) == capi.DFX_OK
    assert lib.dfx_chain_set_motion_vector_view(None, 1, C.c_float(0.01)) == capi.DFX_ERR_INVALID_ARG


def test_synthetic_motion_fields():
    w, h = 40, 30
    for f in (synth.motion_pan(w, h), synth.motion_rotation(w, h), synth.motion_vortex(w, h), synth.motion_random(w, h), synth.motion_extreme(w, h)):
        assert f.shape == (h, w, 2) and f.dtype == np.float32
    assert (synth.motion_pan(w, h) == synth.motion_pan(w, h)[0, 0]).all()
    r = synth.motion_rotation(w, h, 0.1)
    assert np.abs(r[h // 2 - 1: h // 2 + 1, w // 2 - 1: w // 2 + 1]).max() < np.abs(r[0, 0]).max()
    v = synth.motion_vortex(w, h, 0.5, 0.0)
    X = (np.arange(w) + 0.5) / w * 2 - 1
    assert np.allclose(v[0, :, 0], 0.5 * X)  # points away from the centre; drawn at a negative scale, towards and past it
    e = synth.motion_extreme(w, h)
    assert np.isnan(e).any() and np.isinf(e).any() and (np.abs(e[np.isfinite(e)]) > 1e3).any()


# ---- a scalar restatement: numpy float32 scalars (one rounding per operation), python integers for the rule --------------------------

def _sample(field, u, v):
    fh, fw = field.shape[:2]
    px, py = f32(u * f32(fw)) - f32(0.5), f32(v * f32(fh)) - f32(0.5)
    px, py = f32(np.floor(f32(px * f32(256)) + f32(0.5)) * f32(1 / 256)), f32(np.floor(f32(py * f32(256)) + f32(0.5)) * f32(1 / 256))
    fx0, fy0 = np.floor(px), np.floor(py)
    x0, y0 = int(fx0), int(fy0)
    fx, fy = f32(px - fx0), f32(py - fy0)
    tap = lambda x, y: field[min(max(y, 0), fh - 1), min(max(x, 0), fw - 1)]  # noqa: E731
    w = [f32((f32(1) - fx) * (f32(1) - fy)), f32(fx * (f32(1) - fy)), f32((f32(1) - fx) * fy), f32(fx * fy)]
    t = [tap(x0, y0), tap(x0 + 1, y0), tap(x0, y0 + 1), tap(x0 + 1, y0 + 1)]
    out = []
    for c in range(2):
        s = f32(t[0][c] * w[0])
        for k in range(1, 4):
            s = f32(s + f32(t[k][c] * w[k]))
        out.append(s)
    return out


def _snap(x, y, W, H):
    sx = f32(f32(f32(f32(x * f32(0.5)) + f32(0.5)) * f32(W)) * f32(256))
    sy = f32(f32(f32(f32(0.5) - f32(y * f32(0.5))) * f32(H)) * f32(256))
    if not (abs(sx) < 2.0 ** 28 and abs(sy) < 2.0 ** 28):
        return None
    return int(np.rint(sx)), int(np.rint(sy))


def _in_diamond(pu, pv, cu, cv):
    du, dv = pu - cu, pv - cv
    s = abs(du) + abs(dv)
    return s < 128 or (s == 128 and du >= 0 and dv >= 0)


def _step(au, av, bu, bv, i):
    cu = 256 * i + 128
    if au != bu and min(au, bu) <= cu <= max(au, bu):
        num, den = av * (bu - au) + (cu - au) * (bv - av), bu - au
        if den < 0:
            num, den = -num, -den
        j = (num - 1) // (256 * den)
    else:
        j = (av - 1) // 256
        if not _in_diamond(au, av, cu, 256 * j + 128):
            return None
    return None if _in_diamond(bu, bv, cu, 256 * j + 128) else j


def _numpy_vector_field(a, srgb, field, color):
    out = color.copy()
    H, W = out.shape[:2]
    gx, gy = int(a.GridSize[0]), int(a.GridSize[1])
    with np.errstate(all="ignore"):
        for k in range(gx * gy):
            col, row = k % gx, k // gx
            u, v = f32(f32(f32(col) + f32(0.5)) / f32(gx)), f32(f32(f32(row) + f32(0.5)) / f32(gy))
            sx, sy = _sample(field, u, v)
            mx, my = f32(f32(sx + f32(a.Bias[0])) * f32(a.Scale[0])), f32(f32(sy + f32(a.Bias[1])) * f32(a.Scale[1]))
            nx, ny = f32(f32(u - f32(0.5)) / f32(0.5)), f32(f32(v - f32(0.5)) / f32(-0.5))
            A, B = _snap(nx, ny, W, H), _snap(f32(nx + mx), f32(ny + my), W, H)
            if A is None or B is None:
                continue
            xmajor = abs(B[0] - A[0]) >= abs(B[1] - A[1])
            (au, av), (bu, bv) = (A, B) if xmajor else ((A[1], A[0]), (B[1], B[0]))
            for i in range((min(au, bu) - 256) // 256, (max(au, bu) + 256) // 256 + 1):
                j = _step(au, av, bu, bv, i)
                if j is None:
                    continue
                x, y = (i, j) if xmajor else (j, i)
                if not (0 <= x < W and 0 <= y < H):
                    continue
                dx, dy = B[0] - A[0], B[1] - A[1]
                t = f32(f32((256 * x + 128 - A[0]) * dx + (256 * y + 128 - A[1]) * dy) / f32(dx * dx + dy * dy))
                t = min(max(t, f32(0)), f32(1))
                tp = f32(f32(t * f32(1)) / f32(f32(f32(f32(1) - t) * f32(1)) + f32(t * f32(1))))
                c = [f32(f32(a.StartColor[i]) + f32(f32(f32(a.EndColor[i]) - f32(a.StartColor[i])) * tp)) for i in range(4)]
                if srgb:
                    c[:3] = [f32(np.power(v, f32(1) / f32(2.2), dtype=np.float32)) for v in c[:3]]
                out[y, x] = c
    return out


FIELDS = {
    "zero": np.zeros((4, 5, 2), np.float32),
    "pan": synth.motion_pan(5, 4, 0.3, -0.2),
    "vortex": synth.motion_vortex(7, 6, 0.8, 0.6),
    "texel_ties": np.arange(2 * 3 * 2, dtype=np.float32).reshape(3, 2, 2) * np.float32(0.125) - np.float32(0.5),
    "extreme": synth.motion_extreme(6, 5, 4),
}


@pytest.mark.parametrize("srgb", [0, 1])
@pytest.mark.parametrize("name", list(FIELDS))
def test_oracle_against_a_numpy_restatement(built, name, srgb):
    W, H = 23, 17
    rng = np.random.default_rng(2)
    c0 = rng.uniform(-1, 2, (H, W, 4)).astype(np.float32)
    for grid, bias, scale in (((4, 3), (0.0, 0.0), (-1.2, -1.2)), ((1, 1), (0.05, -0.1), (2.0, 0.5)), ((9, 7), (0.0, 0.02), (-0.8, 1.3))):
        a = capi.VectorFieldAttribs.make(grid=grid, bias=bias, scale=scale, start_color=(1, 0.75, 0.5, 1), end_color=(0.25, 0.5, 0.125, 0.5))
        got, want = ov.vector_field(a, srgb, FIELDS[name], c0), _numpy_vector_field(a, srgb, FIELDS[name], c0)
        if srgb:
            np.testing.assert_allclose(got, want, rtol=2e-7, atol=0)
        else:
            assert got.tobytes() == want.tobytes(), (name, grid)


def test_overlap_keeps_the_last_line(built):
    """Two lines over the same pixels of one row: where both draw, the pixel holds the later line's (higher k) fragment, whose colour
    differs from the earlier line's there; each line alone draws exactly its own pixels."""
    W, H = 16, 5
    field = np.zeros((1, 2, 2), np.float32)   # the taps of a 2 x 1 grid land on the texel centres: no blending
    field[0, 0] = (0.75, 0.0)                 # line 0: NDC x -0.5 -> 0.25 on the centre row
    field[0, 1] = (-0.9, 0.0)                 # line 1: 0.5 -> -0.4
    a = capi.VectorFieldAttribs.make(grid=(2, 1), start_color=(1, 0, 0, 1), end_color=(0, 0, 1, 1))
    c0 = np.zeros((H, W, 4), np.float32)
    both = ov.vector_field(a, 0, field, c0)
    only = []
    for k in (0, 1):
        f = field.copy()
        f[0, 1 - k] = 0.0
        only.append(ov.vector_field(a, 0, f, c0))
    d0, d1 = (only[0] != 0).any(-1), (only[1] != 0).any(-1)
    shared = d0 & d1
    assert shared.sum() >= 4 and not (d0 | d1)[[0, 1, 3, 4]].any()
    assert both[shared].tobytes() == only[1][shared].tobytes() and (both[shared] != only[0][shared]).any()
    assert both[d0 & ~d1].tobytes() == only[0][d0 & ~d1].tobytes()
    assert both.tobytes() == _numpy_vector_field(a, 0, field, c0).tobytes()
    v = ov.vertices(a, field)
    assert np.allclose(v[:, 0, :2], [[-0.5, 0.0], [0.5, 0.0]]) and np.allclose(v[:, 1, :2], [[0.25, 0.0], [-0.4, 0.0]])
