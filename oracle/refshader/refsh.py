"""REFERENCE-SHADER RUNNER — TEST INFRASTRUCTURE ONLY. ctypes wrapper over oracle/_ref/librefshaders.so.

The library holds the reference's own pixel shaders compiled for the CPU (build_ref.py). Importers: tests/,
tests/golden/make_reference_shader_golden.py and bench.py's `--impl reference` arm (the CPU baseline: it times these shaders).
Never the product path.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(os.path.dirname(_HERE), "_ref", "librefshaders.so")


class Plane(C.Structure):
    _fields_ = [("data", C.c_void_p), ("w", C.c_int), ("h", C.c_int), ("ch", C.c_int)]


class Args(C.Structure):
    _fields_ = [("inp", C.POINTER(Plane)), ("n_in", C.c_int), ("out", C.POINTER(Plane)), ("n_out", C.c_int),
                ("cb", C.POINTER(C.c_void_p)), ("cb_size", C.POINTER(C.c_int)), ("n_cb", C.c_int),
                ("iparam", C.POINTER(C.c_int)), ("n_iparam", C.c_int), ("mask", C.c_void_p), ("threads", C.c_int)]


def available() -> bool:
    return os.path.exists(LIB)


def build(force: bool = False) -> str:
    """(Re)build where /root/reference is mounted; elsewhere the prebuilt library under oracle/_ref/ is used as is."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("dfx_refshader_build", os.path.join(_HERE, "build_ref.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    if os.path.isdir(mod.REF_SHADERS):
        mod.build(force)
    return LIB


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        _lib = C.CDLL(LIB)
    return _lib


def _plane(a: np.ndarray) -> Plane:
    assert a.flags["C_CONTIGUOUS"] and a.dtype in (np.float32, np.uint32), (a.dtype, a.flags)
    return Plane(a.ctypes.data, a.shape[1], a.shape[0], 1 if a.ndim == 2 else a.shape[2])


def run(name: str, ins, outs, cbs=(), iparams=(), mask: np.ndarray | None = None, threads: int = 0, library: C.CDLL | None = None) -> None:
    """One full-screen pass of the reference shader `name`: `outs` (fp32 arrays, H x W [x C]) are written in place. `library`: another
    library built with the same harness protocol (default librefshaders.so)."""
    ins = [np.ascontiguousarray(a) if a.dtype == np.uint32 else np.ascontiguousarray(a, np.float32) for a in ins]
    for o in outs:
        assert o.dtype == np.float32 and o.flags["C_CONTIGUOUS"]
    pin = (Plane * max(len(ins), 1))(*[_plane(a) for a in ins])
    pout = (Plane * max(len(outs), 1))(*[_plane(a) for a in outs])
    cb_ptr = (C.c_void_p * max(len(cbs), 1))(*[C.cast(C.byref(c), C.c_void_p) for c in cbs])
    cb_size = (C.c_int * max(len(cbs), 1))(*[C.sizeof(c) for c in cbs])
    ip = (C.c_int * max(len(iparams), 1))(*[int(v) for v in iparams])
    m = None
    if mask is not None:
        m = np.ascontiguousarray(mask, np.uint8)
        assert m.shape == outs[0].shape[:2]
    a = Args(pin, len(ins), pout, len(outs), cb_ptr, cb_size, len(cbs), ip, len(iparams), m.ctypes.data if m is not None else None,
             threads or (os.cpu_count() or 1))
    fn = getattr(library or lib(), "refsh_" + name)
    fn.restype = C.c_int
    r = fn(C.byref(a))
    if r != 0:
        raise RuntimeError(f"refsh_{name} failed with {r} (1: wrong resource count, 2: a constant buffer's size differs from the reference structure)")
