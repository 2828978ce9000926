"""REFERENCE-SHADER RUNNER — TEST INFRASTRUCTURE ONLY. DepthRangeCalculator's two compute shaders, compiled for the CPU like every pass
of build_ref.py (same include flattening, text rewrites and harness protocol, read in place from the reference's tree) with the group
runner of compute_defs.inc, into a library of its own, oracle/_ref/librefshaders_depth_range.so:

  clear_depth_range      ClearDepthRange.csh                                   harness/depth_range.inc with REFSH_CLEAR
  compute_depth_range    ComputeDepthRange.csh, THREAD_GROUP_SIZE 8            harness/depth_range.inc
                         (DepthRangeCalculator.cpp:37, :125)

`depth_range(camera, depth)` runs both in order on one buffer, as ComputeRange does. Beyond build_ref.py's rewrites, the
`[numthreads(...)]` attribute is removed, FullScreenTriangleVSOutput.fxh goes in first (harness/common.inc, shared by every pass,
names it), and the unit is compiled as C++20 (std::barrier, std::atomic_ref).

Usage: python oracle/refshader/build_depth_range_ref.py [--force]
"""
from __future__ import annotations

import argparse
import hashlib
import importlib.util
import os
import re
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
OUT_DIR = os.path.join(os.path.dirname(HERE), "_ref")
LIB = os.path.join(OUT_DIR, "librefshaders_depth_range.so")
PASSES = [{"name": "clear_depth_range", "shader": ["FullScreenTriangleVSOutput.fxh", "ClearDepthRange.csh"], "harness": "depth_range.inc", "macros": {"REFSH_CLEAR": 1}},
          {"name": "compute_depth_range", "shader": ["FullScreenTriangleVSOutput.fxh", "ComputeDepthRange.csh"], "harness": "depth_range.inc", "macros": {"THREAD_GROUP_SIZE": 8}}]


def _build_ref():
    spec = importlib.util.spec_from_file_location("dfx_refshader_build_ref", os.path.join(HERE, "build_ref.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def translation_unit(br, p: dict, idx: dict) -> str:
    core = open(os.path.join(HERE, "core_defs.inc")).read()
    tu = br.translation_unit(p, idx)
    assert tu.count(core) == 1
    tu = tu.replace(core, core + open(os.path.join(HERE, "compute_defs.inc")).read())
    tu = re.sub(r"\[numthreads\s*\([^)]*\)\s*\]", "", tu)
    return "#include <atomic>\n#include <barrier>\n#include <cstring>\n#include <thread>\n#include <vector>\n" + tu


def available() -> bool:
    return os.path.exists(LIB)


def build(force: bool = False) -> str:
    """(Re)build where the reference's shaders are mounted; elsewhere a prebuilt library under oracle/_ref/ is used as is."""
    br = _build_ref()
    if not os.path.isdir(br.REF_SHADERS):
        return LIB
    os.makedirs(os.path.join(OUT_DIR, "obj"), exist_ok=True)
    idx = br._index()
    extra = "".join(open(os.path.join(HERE, f)).read() for f in ("hlsl.hpp", "prelude.hpp"))
    objs = []
    for p in PASSES:
        tu = translation_unit(br, p, idx)
        obj = os.path.join(OUT_DIR, "obj", p["name"] + ".o")
        digest = hashlib.sha256((tu + extra).encode()).hexdigest()
        stamp = obj + ".sha"
        if force or not os.path.exists(obj) or not os.path.exists(stamp) or open(stamp).read() != digest:
            r = subprocess.run(["g++", *br.CXXFLAGS, "-std=c++20", "-x", "c++", "-c", "-", "-o", obj], input=tu, text=True, capture_output=True)
            if r.returncode != 0:
                raise RuntimeError(f"==== {p['name']}: compile failed\n{r.stderr[:6000]}")
            open(stamp, "w").write(digest)
        objs.append(obj)
    subprocess.check_call(["g++", "-shared", "-pthread", "-o", LIB, *objs])
    return LIB


_lib = None


def _run(name: str, camera, ins, out) -> None:
    global _lib
    import ctypes as C

    import numpy as np

    from oracle.refshader import refsh
    if _lib is None:
        _lib = C.CDLL(LIB)
    ins = [np.ascontiguousarray(a, np.float32) for a in ins]
    pin = (refsh.Plane * max(len(ins), 1))(*[refsh._plane(a) for a in ins])
    pout = (refsh.Plane * 1)(refsh._plane(out))
    cb_ptr = (C.c_void_p * 1)(C.cast(C.byref(camera), C.c_void_p))
    cb_size = (C.c_int * 1)(C.sizeof(camera))
    ip = (C.c_int * 1)(0)
    a = refsh.Args(pin, len(ins), pout, 1, cb_ptr, cb_size, 1, ip, 0, None, 1)
    fn = getattr(_lib, "refsh_" + name)
    fn.restype = C.c_int
    r = fn(C.byref(a))
    if r != 0:
        raise RuntimeError(f"refsh_{name} failed with {r} (1: wrong resource count, 2: a constant buffer's size differs from the reference structure)")


def depth_range(camera, depth):
    """ClearDepthRange.csh, then ComputeDepthRange.csh on `depth` (H x W) with `camera` (capi.CameraAttribs), on one DepthRangeI buffer.
    Returns it as four float32: fSceneNearZ, fSceneFarZ, fSceneNearDepth, fSceneFarDepth."""
    import numpy as np
    out = np.zeros((1, 4), np.float32)
    _run("clear_depth_range", camera, [], out)
    _run("compute_depth_range", camera, [depth], out)
    return out.reshape(4)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    print(build(ap.parse_args().force))
