"""ORACLE — TEST INFRASTRUCTURE ONLY. ctypes wrapper over oracle/_build/liboracle_depth_range.so: DepthRangeCalculator's two compute
shaders as oracle_depth_range.cpp restates them, group by group. Importers: tests/ and tools/. Never the product path.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(_HERE, "_build", "liboracle_depth_range.so")
SOURCES = [os.path.join(_HERE, "oracle_depth_range.cpp")]
HEADERS = [os.path.join(os.path.dirname(_HERE), "include", "dfx_b200.h")]
# the flags of oracle/Makefile: scalar C++, no FMA contraction
CXXFLAGS = ["-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fvisibility=hidden", "-shared"]


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
        L.ordr_depth_range.restype = None
        _lib = L
    return _lib


def depth_range(camera, depth: np.ndarray) -> np.ndarray:
    """ClearDepthRange.csh, then ComputeDepthRange.csh on `depth` (H x W) with `camera` (capi.CameraAttribs). Returns the four floats
    fSceneNearZ, fSceneFarZ, fSceneNearDepth, fSceneFarDepth (float32)."""
    d = np.ascontiguousarray(depth, np.float32)
    h, w = d.shape
    out = np.zeros(4, np.float32)
    f = C.POINTER(C.c_float)
    lib().ordr_depth_range(C.byref(camera), d.ctypes.data_as(f), w, h, out.ctypes.data_as(f))
    return out
