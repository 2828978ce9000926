"""ORACLE — TEST INFRASTRUCTURE ONLY. ctypes wrapper over oracle/_build/liboracle_bound_box.so: B, the selected prim's bounding box of
oracle_bound_box.cpp (pinned against the reference's own BoundBox.vsh / BoundBox.psh, tests/test_bound_box_reference.py).

`bound_box` is the pass (BoundBoxRenderer); `apply` / `frame` are what HnRenderBoundBoxTask does to a frame's G-buffer before the
post-process task reads it: B in place on the frame's colour and motion with motion vectors on, alpha 0 and the reverse-depth option of
the frame, then the oracle's chain frame on the result. `raster`, `raster_fixed`, `clip` and `vertices` expose the line rasteriser of
DESIGN.md §2 and the vertex shader on their own. Importers: tests/ and tests/golden/. Never the product path.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(_HERE, "_build", "liboracle_bound_box.so")
SOURCES = [os.path.join(_HERE, "oracle_bound_box.cpp")]
HEADERS = [os.path.join(_HERE, f) for f in ("oracle.h", "oracle_common.h", "oracle_math.h", "oracle_tex.h")] + [
    os.path.join(os.path.dirname(_HERE), "include", "dfx_b200.h")]
# the flags of oracle/Makefile: scalar C++, no FMA contraction
CXXFLAGS = ["-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fvisibility=hidden", "-pthread", "-shared"]

OPTION_SRGB, OPTION_MOTION, OPTION_REVERSE_DEPTH = 1, 2, 4


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
        L.orcb_bound_box.restype = None
        L.orcb_vertices.restype = None
        L.orcb_raster.restype = C.c_int
        L.orcb_raster_fixed.restype = C.c_int
        L.orcb_raster_fixed.argtypes = [C.c_int64] * 4 + [C.c_void_p, C.c_int]
        L.orcb_clip.restype = C.c_int
        _lib = L
    return _lib


def _f32(a) -> np.ndarray:
    return np.ascontiguousarray(a, np.float32)


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def bound_box(curr_camera, prev_camera, attribs, options: int, depth: np.ndarray, color: np.ndarray, motion: np.ndarray | None = None,
              rows: tuple[int, int] | None = None) -> tuple[np.ndarray, np.ndarray | None]:
    """B on copies of `color` (H x W x 4) and `motion` (H x W x 2, required with OPTION_MOTION) over `depth` (H x W). Returns (colour,
    motion); pixels B does not draw keep their bytes."""
    d, c = _f32(depth), _f32(color).copy()
    h, w = d.shape
    assert c.shape == (h, w, 4)
    m = _f32(motion).copy() if motion is not None else None
    if options & OPTION_MOTION:
        assert m is not None and m.shape == (h, w, 2)
    y0, y1 = rows or (0, h)
    cams = (type(curr_camera) * 2)(curr_camera, prev_camera)
    lib().orcb_bound_box(cams, C.c_uint32(options), C.byref(attribs), _ptr(d), _ptr(c), _ptr(m) if m is not None else None, w, h, y0, y1)
    return c, m


def vertices(curr_camera, prev_camera, attribs, motion: bool = True) -> np.ndarray:
    """BoundBoxVS for the vertex IDs 0..23: (24, 3, 4) = CLIP_POS, PREV_CLIP_POS, EDGE_START_CLIP_POS."""
    out = np.zeros((24, 3, 4), np.float32)
    cams = (type(curr_camera) * 2)(curr_camera, prev_camera)
    lib().orcb_vertices(cams, C.byref(attribs), int(motion), _ptr(out))
    return out


def raster(p0, p1, w: int, h: int):
    """The rule on one segment of clip-space positions in a w x h viewport: (pixels (n, 2) as (x, y), t (n,), z / w (n,)) in major-axis
    order, or None when nothing is left after clipping and the guard band."""
    p0, p1 = _f32(p0), _f32(p1)
    cap = 4 * (w + h) + 16
    xy, t, z = np.zeros((cap, 2), np.int32), np.zeros(cap, np.float32), np.zeros(cap, np.float32)
    n = lib().orcb_raster(_ptr(p0), _ptr(p1), w, h, xy.ctypes.data_as(C.POINTER(C.c_int)), _ptr(t), _ptr(z), cap)
    return None if n < 0 else (xy[:n], t[:n], z[:n])


def raster_fixed(ax: int, ay: int, bx: int, by: int, cap: int = 4096) -> np.ndarray:
    """The coverage rule on snapped endpoints in 1/256 pixel, no viewport: the pixels drawn, (n, 2) as (x, y), in major-axis order."""
    xy = np.zeros((cap, 2), np.int32)
    n = lib().orcb_raster_fixed(ax, ay, bx, by, xy.ctypes.data, cap)
    return xy[:n]


def clip(p0, p1):
    """The near / far clip of a segment of clip-space positions: (q0, q1), or None when nothing is left."""
    p0, p1 = _f32(p0), _f32(p1)
    q0, q1 = np.zeros(4, np.float32), np.zeros(4, np.float32)
    return (q0, q1) if lib().orcb_clip(_ptr(p0), _ptr(p1), _ptr(q0), _ptr(q1)) else None


def chain_attribs(transform, color=(1.0, 1.0, 1.0, 1.0), pattern_length: float = 32.0, pattern_mask: int = 0xFFFFFFFF):
    """HnRenderBoundBoxTask's attribs for a box transform: its parameters' defaults (HnRenderBoundBoxTask.hpp:47-55), with alpha 0 as
    its PS main stores it (HnRenderBoundBoxTask.cpp:90-93)."""
    from diligentfx_b200 import capi
    a = capi.BoundBoxAttribs.make(transform, (color[0], color[1], color[2], 0.0), pattern_length, pattern_mask)
    return a


def apply(fr: dict, attribs, reversed_depth: bool = False) -> dict:
    """The frame `fr` after HnRenderBoundBoxTask: B with motion vectors on (and the reverse-depth option with `reversed_depth`) on
    copies of its colour and motion. `attribs` as chain_attribs() makes them (alpha 0)."""
    opts = OPTION_MOTION | (OPTION_REVERSE_DEPTH if reversed_depth else 0)
    color, motion = bound_box(fr["curr_camera"], fr["prev_camera"], attribs, opts, fr["depth"], fr["color"], fr["motion"])
    out = dict(fr)
    out["color"], out["motion"] = color, motion
    return out


def frame(o, fr: dict, attribs, stages: int | None = None, reversed_depth: bool = False) -> np.ndarray:
    """One frame of the oracle chain with the box: `apply`, then `o.set_inputs` and the oracle's frame of `stages`. Returns the LDR frame
    (None without the tone-map stage)."""
    from oracle import oracle_py as op
    stages = op.STAGE_ALL if stages is None else stages
    o.set_inputs(apply(fr, attribs, reversed_depth))
    o.frame(stages)
    return o.get("ldr") if stages & op.STAGE_TONEMAP else None
