"""REFERENCE-SHADER RUNNER — TEST INFRASTRUCTURE ONLY. ShadowMapManager's conversion shaders (Shaders/Shadows/private/
ShadowConversions.fx: VSMHorzPS, EVSMHorzPS, VertBlurPS), compiled for the CPU like every pass of build_ref.py (same include flattening,
text rewrites and harness protocol, read in place from the reference's tree) into a library of their own,
oracle/_ref/librefshaders_shadow.so, with one entry, refsh_shadow_conversions, that draws any of the three (harness/shadow_conversions.inc).

What the build supplies, in this library only: shadow_defs.inc, a Texture2DArray whose Load(int4) reads 0 outside the array, and the
correctly rounded exp of DESIGN.md §2. `convert` replays ShadowMapManager::ConvertToFilterable's draws (ShadowMapManager.cpp:533-600):
per cascade the horizontal entry into the one-slice intermediate, then VertBlurPS into the filterable slice, or the horizontal entry
straight into the filterable slice when iFixedFilterSize == 2.

Usage: python oracle/refshader/build_shadow_ref.py [--force]
"""
from __future__ import annotations

import argparse
import ctypes as C
import hashlib
import importlib.util
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT_DIR = os.path.join(os.path.dirname(HERE), "_ref")
LIB = os.path.join(OUT_DIR, "librefshaders_shadow.so")
NAME = "shadow_conversions"
ARRAY_DECL = "Texture2DArray g_tex2DShadowMap;"
PASS = {"name": NAME, "shader": "ShadowConversions.fx", "harness": "shadow_conversions.inc"}
ENTRY_VSM_HORZ, ENTRY_EVSM_HORZ, ENTRY_VERT_BLUR = 0, 1, 2
FMT_RG32F, FMT_RGBA32F, FMT_RGBA16F, FMT_RG16F, FMT_RG16U = 2, 3, 5, 6, 10


def _build_ref():
    spec = importlib.util.spec_from_file_location("dfx_refshader_build", os.path.join(HERE, "build_ref.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def translation_unit(br, idx: dict) -> str:
    core = open(os.path.join(HERE, "core_defs.inc")).read()
    tu = br.translation_unit(PASS, idx)
    assert tu.count(core) == 1 and tu.count(ARRAY_DECL) == 1
    tu = tu.replace(ARRAY_DECL, "Texture2DArray<float4> g_tex2DShadowMap;")
    return tu.replace(core, core + open(os.path.join(HERE, "shadow_defs.inc")).read())


def available() -> bool:
    return os.path.exists(LIB)


def build(force: bool = False) -> str:
    """(Re)build where the reference's shaders are mounted; elsewhere a prebuilt library under oracle/_ref/ is used as is."""
    br = _build_ref()
    if not os.path.isdir(br.REF_SHADERS):
        return LIB
    os.makedirs(os.path.join(OUT_DIR, "obj"), exist_ok=True)
    tu = translation_unit(br, br._index())
    extra = "".join(open(os.path.join(HERE, f)).read() for f in ("hlsl.hpp", "prelude.hpp"))
    obj = os.path.join(OUT_DIR, "obj", NAME + ".o")
    digest = hashlib.sha256((tu + extra).encode()).hexdigest()
    stamp = obj + ".sha"
    if force or not (os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == digest and os.path.exists(LIB)):
        r = subprocess.run(["g++", *br.CXXFLAGS, "-x", "c++", "-c", "-", "-o", obj], input=tu, text=True, capture_output=True)
        if r.returncode != 0:
            raise RuntimeError(f"==== {NAME}: compile failed\n{r.stderr[:6000]}")
        open(stamp, "w").write(digest)
        subprocess.check_call(["g++", "-shared", "-pthread", "-o", LIB, obj])
    return LIB


_lib = None


class _CB(C.Structure):
    """The constant block as ShadowMapManager.cpp:553-582 writes it."""
    _fields_ = [("iCascade", C.c_int32), ("fHorzFilterRadius", C.c_float), ("fVertFilterRadius", C.c_float),
                ("fEVSMPositiveExponent", C.c_float), ("fEVSMNegativeExponent", C.c_float), ("Is32BitEVSM", C.c_int32)]


def draw(entry: int, slices, out: np.ndarray, cb: _CB, fmt: int) -> None:
    """One full-screen draw of `entry` with `slices` (h x w [x c] float32 arrays) bound as g_tex2DShadowMap into `out` (in place)."""
    global _lib
    from oracle.refshader import refsh
    if _lib is None:
        _lib = C.CDLL(LIB)
    refsh.run(NAME, list(slices), [out], cbs=[cb], iparams=[len(slices), entry, fmt], library=_lib)


def radii(attribs, cascade: int, width: int, height: int) -> tuple[float, float]:
    """ShadowMapManager.cpp:563-579 in float32, in its order."""
    if attribs.iFixedFilterSize > 0:
        r = float(np.float32(int((attribs.iFixedFilterSize - 1) / 2)))
        return r, r
    f32 = np.float32
    s = attribs.Cascades[cascade].f4LightSpaceScale
    fw = f32(f32(attribs.fFilterWorldSize) * f32(s[0])) * f32(0.5)
    fh = f32(f32(attribs.fFilterWorldSize) * f32(s[1])) * f32(0.5)
    return float(f32(fw / f32(2.0)) * f32(width)), float(f32(fh / f32(2.0)) * f32(height))


def convert(mode: int, attribs, depth: np.ndarray, is32: bool, cascades=None) -> np.ndarray:
    """ConvertToFilterable of `depth` (n x h x w float32 = D32, or uint16 D16 codes, read as k / 65535) as the reference draws it:
    (len(cascades), h, w, channels) float32, the values the filterable format stores."""
    n, h, w = depth.shape
    d = depth.astype(np.float32) / np.float32(65535) if depth.dtype == np.uint16 else depth.astype(np.float32)
    ch = 4 if mode == 4 else 2
    fmt = {2: FMT_RG32F if is32 else FMT_RG16U, 3: FMT_RG32F if is32 else FMT_RG16F, 4: FMT_RGBA32F if is32 else FMT_RGBA16F}[mode]
    horz = ENTRY_VSM_HORZ if mode == 2 else ENTRY_EVSM_HORZ
    slices = [np.ascontiguousarray(d[i]) for i in range(n)]
    out = []
    for i in (range(n) if cascades is None else cascades):
        rh, rv = radii(attribs, i, w, h)
        cb = _CB(i, rh, rv, attribs.fEVSMPositiveExponent, attribs.fEVSMNegativeExponent, attribs.bIs32BitEVSM)
        target = np.zeros((h, w, ch), np.float32)
        if attribs.iFixedFilterSize == 2:
            draw(horz, slices, target, cb, fmt)
        else:
            inter = np.zeros((h, w, ch), np.float32)
            draw(horz, slices, inter, cb, fmt)
            draw(ENTRY_VERT_BLUR, [inter], target, cb, fmt)
        out.append(target)
    return np.stack(out)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    print(build(ap.parse_args().force))
