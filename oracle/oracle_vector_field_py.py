"""ORACLE — TEST INFRASTRUCTURE ONLY. ctypes wrapper over oracle/_build/liboracle_vector_field.so: the vector field overlay of
oracle_vector_field.cpp (pinned against the reference's own VectorField.vsh and VectorFieldRenderer's default PS main,
tests/test_vector_field_reference.py).

`vector_field` is the pass (VectorFieldRenderer::Render); `frame` is what HnPostProcessTask draws in the motion-vector view: the TAA-off
compose with zero SSR and SSAO scales straight into the final target, then the field of the frame's motion plane over it. Importers:
tests/, tests/golden/ and tools/. Never the product path.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(_HERE, "_build", "liboracle_vector_field.so")
SOURCES = [os.path.join(_HERE, "oracle_vector_field.cpp")]
HEADERS = [os.path.join(_HERE, f) for f in ("oracle.h", "oracle_common.h", "oracle_math.h", "oracle_tex.h")] + [
    os.path.join(os.path.dirname(_HERE), "include", "dfx_b200.h")]
# the flags of oracle/Makefile: scalar C++, no FMA contraction
CXXFLAGS = ["-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fvisibility=hidden", "-pthread", "-shared"]

OPTION_SRGB = 1


def build(force: bool = False) -> str:
    newest = max(os.path.getmtime(p) for p in SOURCES + HEADERS)
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < newest:
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call([os.environ.get("CXX", "g++"), *CXXFLAGS, "-o", LIB, *SOURCES])
    return LIB


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB)
        L.orcv_vector_field.restype = C.c_uint64
        L.orcv_vertices.restype = None
        L.orcv_vertices.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_uint64, C.c_void_p]
        _lib = L
    return _lib


def _f32(a) -> np.ndarray:
    return np.ascontiguousarray(a, np.float32)


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def vector_field(attribs, options: int, field: np.ndarray, color: np.ndarray, rows: tuple[int, int] | None = None,
                 count: bool = False):
    """The field `field` (fh x fw x 2) drawn over a copy of `color` (H x W x 4) with `attribs` (capi.VectorFieldAttribs) and `options`
    (OPTION_SRGB). Pixels no line draws keep their bytes. With `count`: (target, fragments drawn, each line's pixels counted)."""
    f, c = _f32(field), _f32(color).copy()
    fh, fw = f.shape[:2]
    assert f.shape == (fh, fw, 2)
    h, w = c.shape[:2]
    assert c.shape == (h, w, 4)
    y0, y1 = rows or (0, h)
    n = lib().orcv_vector_field(C.byref(attribs), C.c_uint32(options), _ptr(f), fw, fh, _ptr(c), w, h, y0, y1)
    return (c, int(n)) if count else c


def vertices(attribs, field: np.ndarray) -> np.ndarray:
    """VectorField.vsh's positions for every line: (GridSize.y * GridSize.x, 2, 4), start then end."""
    f = _f32(field)
    n = int(attribs.GridSize[0]) * int(attribs.GridSize[1])
    out = np.zeros((n, 2, 4), np.float32)
    lib().orcv_vertices(C.addressof(attribs), f.ctypes.data, f.shape[1], f.shape[0], n, out.ctypes.data)
    return out


def hydrogent_attribs(width: int, height: int, elapsed: float):
    """HnPostProcessTask's attribs (HnPostProcessTask.cpp:932-938), restated here: GridSize (W / 20, H / 20), Scale -0.02 / max(elapsed,
    0.001) in fp32, StartColor 1, EndColor (0.5, 0.5, 0.5, 1)."""
    from diligentfx_b200 import capi
    t = np.float32(elapsed)
    t = np.float32(0.001) if t < np.float32(0.001) else t
    s = float(np.float32(-0.02) / t)
    return capi.VectorFieldAttribs.make(grid=(width // 20, height // 20), scale=(s, s), end_color=(0.5, 0.5, 0.5, 1.0))


def frame(o, fr: dict, elapsed: float, selection_depth: np.ndarray | None = None, attribs=None, grid_flags: int = 0, grid_attribs=None,
          tonemap=None, ave_log_lum: float = 0.3, to_srgb: bool = True) -> np.ndarray:
    """One frame of the oracle chain in the motion-vector view, with TAA off whatever the chain is configured with
    (HnPostProcessTask.cpp:625-654, :788, :928-943): no PostFX, SSR, SSAO, TAA, Bloom or DepthOfField. `fr` is the frame as the post-process
    task reads it (after E and B: oracle_env_map_py.apply / oracle_bound_box_py.apply). The compose (compose_final with zero SSR and AO
    contributions) writes the LDR frame with the tone map, the selection of `attribs` on `selection_depth` with its colours as given, the
    grid and sRGB; then the field of fr["motion"] with hydrogent_attribs(W, H, elapsed) and sRGB = `to_srgb` over it. `o` gets the
    frame's inputs (its TAA history is not advanced, so its next TAA frame resets). Returns the LDR frame."""
    from diligentfx_b200 import capi
    from oracle import oracle_compose_final_py as ocf
    from oracle import oracle_selection_py as osp
    o.set_inputs(fr)
    sel = loc = None
    if selection_depth is not None:
        sel = attribs or capi.SelectionAttribs.default()
        loc = osp.closest_selected_location(selection_depth, sel.ClearDepth, sel.SelectionOutlineWidth)
    ldr = ocf.compose_final(fr["curr_camera"], tonemap or capi.ToneMapAttribs.default(), ave_log_lum, to_srgb, fr["color"], fr["depth"], sel,
                            selection_depth, loc, grid_flags, grid_attribs)
    h, w = ldr.shape[:2]
    return vector_field(hydrogent_attribs(w, h, elapsed), OPTION_SRGB if to_srgb else 0, fr["motion"], ldr)
