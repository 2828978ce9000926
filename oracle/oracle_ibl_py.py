"""ORACLE — TEST INFRASTRUCTURE ONLY. ctypes wrapper over oracle/_build/liboracle_ibl.so: the IBL cube-map precomputation of
oracle_ibl.cpp (pinned against the reference's own CubemapFace.vsh, ComputeIrradianceMap.psh and PrefilterEnvMap.psh,
tests/test_ibl_reference.py).

`irradiance` and `prefilter` compute a row range of chosen faces of one output level, so that a full-size GPU run can be checked on a
drawn subset. Importers: tests/ and tests/golden/. Never the product path.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(_HERE, "_build", "liboracle_ibl.so")
SOURCES = [os.path.join(_HERE, "oracle_ibl.cpp")]
HEADERS = [os.path.join(_HERE, "oracle_math.h"), os.path.join(_HERE, "oracle_ibl_math.h")]
# the flags of oracle/Makefile: scalar C++, no FMA contraction
CXXFLAGS = ["-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fvisibility=hidden", "-pthread", "-shared"]

TYPE_CUBE, TYPE_SPHERE = 0, 1
DEFAULT_DIFFUSE_SAMPLES, DEFAULT_SPECULAR_SAMPLES = 8192, 256


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
        L.orci_ibl.restype = None
        _lib = L
    return _lib


def roughness(level: int, levels: int) -> float:
    """PBR_Renderer.cpp:951: static_cast<float>(mip) / static_cast<float>(levels - 1), in float."""
    return float(np.float32(level) / np.float32(levels - 1))


def _run(pass_: int, env_type: int, levels, num_samples: int, optimize: bool, rough: float, size: int, faces, rows, threads: int) -> np.ndarray:
    lv = [np.ascontiguousarray(a, np.float32) for a in levels]
    assert 1 <= len(lv) <= 16 and all(a.ndim == 3 and a.shape[2] == 4 for a in lv)
    ptrs = (C.POINTER(C.c_float) * len(lv))(*[a.ctypes.data_as(C.POINTER(C.c_float)) for a in lv])
    lw = (C.c_int * len(lv))(*[a.shape[1] for a in lv])
    lh = (C.c_int * len(lv))(*[a.shape[0] for a in lv])
    faces = list(range(6)) if faces is None else list(faces)
    r0, r1 = (0, size) if rows is None else rows
    out = np.zeros((len(faces), r1 - r0, size, 4), np.float32)
    for k, f in enumerate(faces):
        lib().orci_ibl(pass_, env_type, ptrs, lw, lh, len(lv), C.c_uint32(num_samples), int(optimize), C.c_float(rough), size, f, r0, r1,
                       out[k].ctypes.data_as(C.POINTER(C.c_float)), threads or (os.cpu_count() or 1))
    return out


def irradiance(env_type: int, levels, size: int, num_samples: int = 0, optimize: bool = True, faces=None, rows=None, threads: int = 0) -> np.ndarray:
    """The irradiance cube's faces `faces` (default all six), rows [rows[0], rows[1]) (default all) of an s = `size` face:
    (len(faces), rows, s, 4) fp32, alpha 1. `levels`: the source's mip levels, (6s, s, 4) for a cube, (h, w, 4) for a sphere.
    num_samples 0 = 8192."""
    return _run(0, env_type, levels, num_samples or DEFAULT_DIFFUSE_SAMPLES, optimize, 0.0, size, faces, rows, threads)


def prefilter(env_type: int, levels, size: int, rough: float, num_samples: int = 0, optimize: bool = True, faces=None, rows=None,
              threads: int = 0) -> np.ndarray:
    """One level of the prefiltered environment map (face size `size`, PerceptualRoughness `rough`, see roughness()), as irradiance();
    alpha 0. num_samples 0 = 256."""
    return _run(1, env_type, levels, num_samples or DEFAULT_SPECULAR_SAMPLES, optimize, rough, size, faces, rows, threads)


def as_cube(faces: np.ndarray) -> np.ndarray:
    """(6, s, s, 4) -> the (6s, s, 4) plane layout (faces stacked top to bottom)."""
    return faces.reshape(-1, faces.shape[2], faces.shape[3])
