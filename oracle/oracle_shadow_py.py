"""ORACLE — TEST INFRASTRUCTURE ONLY. ctypes wrapper over oracle/_build/liboracle_shadow.so: ShadowMapManager::ConvertToFilterable of
oracle_shadow.cpp (pinned against the reference's own ShadowConversions.fx, tests/test_shadow_reference.py).

`convert` gives the filterable map of chosen cascades as the values the filterable format stores; `stored` turns them into that
format's texels (uint16 codes, float16 or float32), which is what the GPU's planes hold. Importers: tests/ and tests/golden/. Never the
product path.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(_HERE, "_build", "liboracle_shadow.so")
SOURCES = [os.path.join(_HERE, "oracle_shadow.cpp")]
HEADERS = [os.path.join(_HERE, "oracle_quant.h")]
# the flags of oracle/Makefile: scalar C++, no FMA contraction
CXXFLAGS = ["-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fvisibility=hidden", "-pthread", "-shared"]

PCF, VSM, EVSM2, EVSM4 = 1, 2, 3, 4
ATTRIBS_BYTES = 1200


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
        L.ors_convert.restype = C.c_int
        L.ors_filter_radii.restype = None
        L.ors_warp.restype = None
        _lib = L
    return _lib


def _bytes(attribs) -> C.Array:
    b = bytes(attribs)
    assert len(b) == ATTRIBS_BYTES
    return (C.c_ubyte * ATTRIBS_BYTES).from_buffer_copy(b)


def channels(mode: int) -> int:
    return 4 if mode == EVSM4 else 2


def filter_radii(attribs, cascade: int, width: int, height: int) -> tuple[float, float]:
    rh, rv = C.c_float(), C.c_float()
    lib().ors_filter_radii(_bytes(attribs), cascade, width, height, C.byref(rh), C.byref(rv))
    return rh.value, rv.value


def warp(depth: np.ndarray, pos: float, neg: float, is32: bool) -> np.ndarray:
    """WarpDepthEVSM of every depth with GetEVSMExponents(pos, neg, is32): (..., 2) float32."""
    d = np.ascontiguousarray(depth, np.float32).ravel()
    out = np.zeros((d.size, 2), np.float32)
    lib().ors_warp(d.ctypes.data_as(C.POINTER(C.c_float)), d.size, C.c_float(pos), C.c_float(neg), int(is32),
                   out.ctypes.data_as(C.POINTER(C.c_float)))
    return out.reshape(np.shape(depth) + (2,))


def convert(mode: int, attribs, depth: np.ndarray, is32: bool, cascades=None, threads: int = 0) -> np.ndarray:
    """The filterable map of `depth` (n x h x w, float32 = D32_FLOAT or uint16 = D16_UNORM codes): (len(cascades), h, w, channels)
    float32 values as the filterable format stores them. `cascades` default: all n."""
    assert mode in (VSM, EVSM2, EVSM4)
    assert depth.ndim == 3 and depth.dtype in (np.float32, np.uint16)
    n, h, w = depth.shape
    cascades = list(range(n)) if cascades is None else list(cascades)
    ab = _bytes(attribs)
    out = np.zeros((len(cascades), h, w, channels(mode)), np.float32)
    for k, i in enumerate(cascades):
        src = np.ascontiguousarray(depth[i])
        lib().ors_convert(mode, ab, i, src.ctypes.data_as(C.c_void_p), int(depth.dtype == np.uint16), w, h, int(is32),
                          out[k].ctypes.data_as(C.POINTER(C.c_float)), threads or (os.cpu_count() or 1))
    return out


def stored(mode: int, is32: bool, values: np.ndarray) -> np.ndarray:
    """The filterable format's texels of `values` (already quantised): RG16_UNORM codes as uint16, RG16F / RGBA16F as float16, the 32-bit
    formats as float32."""
    if is32:
        return values.astype(np.float32)
    if mode == VSM:
        return np.rint(values.astype(np.float64) * 65535.0).astype(np.uint16)
    return values.astype(np.float16)
