"""REFERENCE-SHADER RUNNER — TEST INFRASTRUCTURE ONLY. BoundBoxRenderer's shaders (Shaders/Common/private/BoundBox.vsh / BoundBox.psh),
compiled for the CPU like every pass of build_ref.py (same include flattening, text rewrites and harness protocol, read in place from
the reference's tree) into a library of their own, oracle/_ref/librefshaders_bound_box.so:

  bound_box__<s>_<v>   BoundBox.vsh and BoundBox.psh with the macros BoundBoxRenderer::GetPSO derives from its key
                       (BoundBoxRenderer.cpp:117-120): CONVERT_OUTPUT_TO_SRGB s, COMPUTE_MOTION_VECTORS v; harness/bound_box.inc
                       (the 24 vertices, the lines rasterised by line_defs.inc, the depth test, GetBoundBoxOutput per fragment).

What the shaders expect from their environment is supplied here, in this library only:
  * both shaders declare the cbuffers cbCameraAttribs and cbBoundBoxAttribs; each is flattened into a namespace of its own (bbvs,
    bbps) so that both sets of globals exist, and the harness fills both;
  * `#include "PSMainGenerated.generated"` (the PS main BoundBoxRenderer or HnRenderBoundBoxTask generates) reads an empty file: the
    harness stores GetBoundBoxOutput's result as HnRenderBoundBoxTask's PS main does;
  * the pattern bit's `uint(PatternPos * g_Attribs.PatternLength)` becomes `refsh_ftou(...)`, D3D's conversion (NaN -> 0,
    saturating), where C++'s conversion of a NaN is undefined;
  * BoundBoxVSOutput's semantics (CLIP_POS, PREV_CLIP_POS, EDGE_START_CLIP_POS) are removed as build_ref.py removes SV_*;
  * line_defs.inc (pasted after core_defs.inc) is the rasteriser of DESIGN.md §2 the graphics API would provide.

Usage: python oracle/refshader/build_bound_box_ref.py [--force]
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
LIB = os.path.join(OUT_DIR, "librefshaders_bound_box.so")


def _build_ref():
    spec = importlib.util.spec_from_file_location("dfx_refshader_build", os.path.join(HERE, "build_ref.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


# (CONVERT_OUTPUT_TO_SRGB, COMPUTE_MOTION_VECTORS): all four
VARIANTS = [(s, v) for s in (0, 1) for v in (0, 1)]
SEMANTICS = r"CLIP_POS|PREV_CLIP_POS|EDGE_START_CLIP_POS"  # BoundBoxVSOutput's, which build_ref.rewrite does not know
PATTERN_BIT = "uint(PatternPos * g_Attribs.PatternLength)"


def name(s: int, v: int) -> str:
    return f"bound_box__{s}_{v}"


PASSES = [{"name": name(*k), "harness": "bound_box.inc", "macros": {"CONVERT_OUTPUT_TO_SRGB": k[0], "COMPUTE_MOTION_VECTORS": k[1]}}
          for k in VARIANTS]


def translation_unit(br, p: dict, idx: dict) -> str:
    """build_ref.translation_unit's layout, with the vertex and the pixel shader in namespaces of their own."""
    idx = dict(idx, **{"PSMainGenerated.generated": os.devnull})
    ns = "refsh_ns_" + p["name"]
    seen: set[str] = set()
    fst = br.flatten("FullScreenTriangleVSOutput.fxh", idx, seen)  # what harness/common.inc's full-screen rasteriser is written against
    vs = re.sub(r":\s*(?:" + SEMANTICS + r")\b", "", br.flatten("BoundBox.vsh", idx, seen))
    ps = re.sub(r":\s*(?:" + SEMANTICS + r")\b", "", br.flatten("BoundBox.psh", idx, seen))
    assert ps.count(PATTERN_BIT) == 1
    ps = ps.replace(PATTERN_BIT, "refsh_ftou(PatternPos * g_Attribs.PatternLength)")
    parts = ['#include "prelude.hpp"\n']
    parts += [f"#define {k} {v}\n" for k, v in p["macros"].items()]
    parts.append(f"namespace {ns} {{\nusing namespace hlsl;\n")
    parts.append(open(os.path.join(HERE, "core_defs.inc")).read())
    parts.append(open(os.path.join(HERE, "line_defs.inc")).read())
    parts.append(fst)
    parts.append("namespace bbvs {\n" + vs + "} // namespace bbvs\n")
    parts.append("namespace bbps {\nusing namespace bbvs;\n" + ps + "} // namespace bbps\nusing namespace bbvs;\n")
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
    extra = "".join(open(os.path.join(HERE, f)).read() for f in ("hlsl.hpp", "prelude.hpp", "core_defs.inc", "line_defs.inc", os.path.join("harness", "common.inc"), os.path.join("harness", "bound_box.inc")))

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

    with cf.ThreadPoolExecutor(max_workers=min(16, os.cpu_count() or 4)) as ex:
        results = list(ex.map(compile_one, PASSES))
    errors = [e for _, e in results if e]
    if errors:
        raise RuntimeError("\n".join(errors))
    subprocess.check_call(["g++", "-shared", "-pthread", "-o", LIB, *[o for o, _ in results]])
    return LIB


_lib = None


def run(name: str, ins, outs, cbs=(), iparams=(), threads: int = 0) -> None:
    """refsh.run for the passes of this library: `outs` (fp32 H x W x C arrays) are written in place."""
    global _lib
    from oracle.refshader import refsh
    import numpy as np
    if _lib is None:
        _lib = C.CDLL(LIB)
    ins = [np.ascontiguousarray(a, np.float32) for a in ins]
    for o in outs:
        assert o.dtype == np.float32 and o.flags["C_CONTIGUOUS"]
    pin = (refsh.Plane * len(ins))(*[refsh._plane(a) for a in ins])
    pout = (refsh.Plane * len(outs))(*[refsh._plane(a) for a in outs])
    cb_ptr = (C.c_void_p * max(len(cbs), 1))(*[C.cast(C.byref(c), C.c_void_p) for c in cbs])
    cb_size = (C.c_int * max(len(cbs), 1))(*[C.sizeof(c) for c in cbs])
    ip = (C.c_int * max(len(iparams), 1))(*[int(v) for v in iparams])
    a = refsh.Args(pin, len(ins), pout, len(outs), cb_ptr, cb_size, len(cbs), ip, len(iparams), None, threads or (os.cpu_count() or 1))
    fn = getattr(_lib, "refsh_" + name)
    fn.restype = C.c_int
    r = fn(C.byref(a))
    if r != 0:
        raise RuntimeError(f"refsh_{name} failed with {r} (1: wrong resource count, 2: a constant buffer's size differs from the reference structure)")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    print(build(ap.parse_args().force))
