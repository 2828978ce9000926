"""REFERENCE-SHADER RUNNER — TEST INFRASTRUCTURE ONLY. VectorFieldRenderer's shaders, compiled for the CPU like every pass of
build_ref.py (same include flattening, text rewrites and harness protocol, read in place from the reference's tree) into a library of
their own, oracle/_ref/librefshaders_vector_field.so:

  vector_field__<s>    Shaders/Common/private/VectorField.vsh and the default PS main with CONVERT_OUTPUT_TO_SRGB s, the one macro
                       VectorFieldRenderer::GetPSO derives from its key (VectorFieldRenderer.cpp:108-110); harness/vector_field.inc
                       (the vertices, the lines rasterised by line_defs.inc, the PS output stored over the target).

What the shaders expect from their environment is supplied here, in this library only:
  * the pixel shader is VectorFieldRenderer.cpp's `DefaultPSMain` string, read out of that file at build time (the
    "PSMainGenerated.generated" file the renderer compiles when no PSMainSource is given);
  * both shaders define `main`; each goes into a namespace of its own (vfvs, vfps);
  * the COLOR semantic of both is removed as build_ref.py removes SV_*;
  * line_defs.inc (pasted after core_defs.inc) is the rasteriser of DESIGN.md §2 the graphics API would provide.

Usage: python oracle/refshader/build_vector_field_ref.py [--force]
"""
from __future__ import annotations

import argparse
import concurrent.futures as cf
import ctypes as C
import hashlib
import importlib.util
import os
import re
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
OUT_DIR = os.path.join(os.path.dirname(HERE), "_ref")
LIB = os.path.join(OUT_DIR, "librefshaders_vector_field.so")
SEMANTICS = r"COLOR"


def _build_ref():
    spec = importlib.util.spec_from_file_location("dfx_refshader_build", os.path.join(HERE, "build_ref.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def name(s: int) -> str:
    return f"vector_field__{s}"


PASSES = [{"name": name(s), "harness": "vector_field.inc", "macros": {"CONVERT_OUTPUT_TO_SRGB": s}} for s in (0, 1)]


def default_ps_main(br) -> str:
    """DefaultPSMain of Components/src/VectorFieldRenderer.cpp, as the renderer hands it to the shader compiler."""
    path = os.path.join(os.path.dirname(br.REF_SHADERS), "Components", "src", "VectorFieldRenderer.cpp")
    m = re.search(r'static\s+constexpr\s+char\s+DefaultPSMain\[\]\s*=\s*R"\((.*?)\)"\s*;', open(path, encoding="utf-8").read(), flags=re.S)
    assert m, f"DefaultPSMain not found in {path}"
    return m.group(1)


def translation_unit(br, p: dict, idx: dict) -> str:
    """build_ref.translation_unit's layout, with the vertex and the pixel shader in namespaces of their own."""
    ns = "refsh_ns_" + p["name"]
    seen: set[str] = set()
    fst = br.flatten("FullScreenTriangleVSOutput.fxh", idx, seen)  # what harness/common.inc's full-screen rasteriser is written against
    vs = re.sub(r":\s*(?:" + SEMANTICS + r")\b", "", br.flatten("VectorField.vsh", idx, seen))
    ps = re.sub(r":\s*(?:" + SEMANTICS + r")\b", "", br.rewrite(default_ps_main(br)))
    parts = ['#include "prelude.hpp"\n']
    parts += [f"#define {k} {v}\n" for k, v in p["macros"].items()]
    parts.append(f"namespace {ns} {{\nusing namespace hlsl;\n")
    parts.append(open(os.path.join(HERE, "core_defs.inc")).read())
    parts.append(open(os.path.join(HERE, "line_defs.inc")).read())
    parts.append(fst)
    parts.append("namespace vfvs {\n" + vs + "} // namespace vfvs\n")
    parts.append("namespace vfps {\n" + ps + "} // namespace vfps\n")
    parts.append(open(os.path.join(HERE, "harness", "common.inc")).read())
    parts.append(open(os.path.join(HERE, "harness", p["harness"])).read())
    parts.append(f"\n}} // namespace {ns}\n")
    parts.append(f'extern "C" __attribute__((visibility("default"))) int refsh_{p["name"]}(const refsh_args* a) {{ return {ns}::entry(a); }}\n')
    return "".join(parts)


def available() -> bool:
    return os.path.exists(LIB)


def build(force: bool = False) -> str:
    """(Re)build where the reference's shaders are mounted; elsewhere a prebuilt library under oracle/_ref/ is used as is."""
    br = _build_ref()
    if not os.path.isdir(br.REF_SHADERS):
        return LIB
    os.makedirs(os.path.join(OUT_DIR, "obj"), exist_ok=True)
    idx = br._index()
    extra = "".join(open(os.path.join(HERE, f)).read() for f in ("hlsl.hpp", "prelude.hpp", "core_defs.inc", "line_defs.inc", os.path.join("harness", "common.inc"),
                                                                 os.path.join("harness", "vector_field.inc")))

    def compile_one(p: dict) -> tuple[str, str]:
        tu = translation_unit(br, p, idx)
        obj = os.path.join(OUT_DIR, "obj", p["name"] + ".o")
        digest = hashlib.sha256((tu + extra).encode()).hexdigest()
        stamp = obj + ".sha"
        if not force and os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == digest:
            return obj, ""
        r = subprocess.run(["g++", *br.CXXFLAGS, "-x", "c++", "-c", "-", "-o", obj], input=tu, text=True, capture_output=True)
        if r.returncode != 0:
            return "", f"==== {p['name']}: compile failed\n{r.stderr[:6000]}"
        open(stamp, "w").write(digest)
        return obj, ""

    with cf.ThreadPoolExecutor(max_workers=2) as ex:
        results = list(ex.map(compile_one, PASSES))
    errors = [e for _, e in results if e]
    if errors:
        raise RuntimeError("\n".join(errors))
    subprocess.check_call(["g++", "-shared", "-pthread", "-o", LIB, *[o for o, _ in results]])
    return LIB


class Attribs(C.Structure):
    """VectorField.vsh's VectorFieldRenderAttribs (64 bytes): what VectorFieldRenderer::Render writes (VectorFieldRenderer.cpp:209-216)."""
    _fields_ = [("ScaleAndBias", C.c_float * 4), ("fGridWidth", C.c_float), ("fGridHeight", C.c_float), ("uGridWidth", C.c_uint32),
                ("uGridHeight", C.c_uint32), ("Colors", C.c_float * 8)]


def shader_attribs(a) -> Attribs:
    """dfx_vector_field_attribs (capi.VectorFieldAttribs) -> the constant block, as Render fills it."""
    import numpy as np
    cb = Attribs()
    cb.ScaleAndBias[:] = [a.Scale[0], a.Scale[1], a.Bias[0], a.Bias[1]]
    cb.fGridWidth, cb.fGridHeight = float(np.float32(a.GridSize[0])), float(np.float32(a.GridSize[1]))
    cb.uGridWidth, cb.uGridHeight = a.GridSize[0], a.GridSize[1]
    cb.Colors[:] = list(a.StartColor) + list(a.EndColor)
    return cb


_lib = None


def run(attribs, srgb: bool, field, color):
    """The shaders on `field` (fh x fw x 2) over a copy of `color` (H x W x 4): returns the drawn target."""
    global _lib
    from oracle.refshader import refsh
    import numpy as np
    if _lib is None:
        _lib = C.CDLL(LIB)
    f = np.ascontiguousarray(field, np.float32)
    out = np.ascontiguousarray(color, np.float32).copy()
    cb = shader_attribs(attribs)
    pin = (refsh.Plane * 1)(refsh._plane(f))
    pout = (refsh.Plane * 1)(refsh._plane(out))
    cb_ptr = (C.c_void_p * 1)(C.cast(C.byref(cb), C.c_void_p))
    cb_size = (C.c_int * 1)(C.sizeof(cb))
    ip = (C.c_int * 1)(0)
    a = refsh.Args(pin, 1, pout, 1, cb_ptr, cb_size, 1, ip, 0, None, 1)
    fn = getattr(_lib, "refsh_" + name(int(bool(srgb))))
    fn.restype = C.c_int
    r = fn(C.byref(a))
    if r != 0:
        raise RuntimeError(f"refsh_{name(int(bool(srgb)))} failed with {r} (1: wrong resource count, 2: a constant buffer's size differs from the reference structure)")
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    print(build(ap.parse_args().force))
