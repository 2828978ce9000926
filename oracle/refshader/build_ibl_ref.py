"""REFERENCE-SHADER RUNNER — TEST INFRASTRUCTURE ONLY. PBR_Renderer's IBL precomputation shaders (Shaders/PBR/private/CubemapFace.vsh,
ComputeIrradianceMap.psh, PrefilterEnvMap.psh), compiled for the CPU like every pass of build_ref.py (same include flattening, text
rewrites and harness protocol, read in place from the reference's tree) into a library of their own, oracle/_ref/librefshaders_ibl.so:

  ibl_irradiance__<type>_<opt>   ComputeIrradianceMap.psh with harness/irradiance_cube.inc
  ibl_prefilter__<type>_<opt>    PrefilterEnvMap.psh with harness/prefilter_env_map.inc
  with the macros PBR_Renderer::PrecomputeCubemaps sets (PBR_Renderer.cpp:794-798): ENV_MAP_TYPE (0 cube, 1 sphere), OPTIMIZE_SAMPLES.
  brdf_lut__<n>                  PrecomputeBRDF.psh with harness/brdf_lut.inc and NUM_SAMPLES n (PBR_Renderer::PrecomputeBRDF uses 512),
                                 built as build_ref.py builds a full-screen pass

What the build supplies, in this library only:
  * the vertex and the pixel shader both declare cbConstants; each is flattened into a namespace of its own (ibvs, ibps), and the
    harness fills both;
  * CubemapFace.vsh's `PosXY[VertexId]` becomes the harness's pixel-centre NDC (`g_RefshPosXY`, one per host thread), so the vertex
    shader is evaluated at the pixel centre; the `WORLD_POS` semantic is dropped like the SV_ ones;
  * `TextureCube<float4> g_EnvironmentMap` becomes `EnvCube<float4> g_EnvironmentMap`, the cube sampler of env_map_defs.inc with the
    seamless rule of DESIGN.md §2, as build_env_map_ref.py does for EnvMap.psh;
  * ibl_defs.inc states the shaders' transcendentals and PrecomputeBRDF.psh's pow(x, 5.0) as correctly rounded (DESIGN.md §2); hlsl.hpp
    is left as it is.

Usage: python oracle/refshader/build_ibl_ref.py [--force]
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
LIB = os.path.join(OUT_DIR, "librefshaders_ibl.so")
VS_POS = "PosXY[VertexId]"
CUBE_DECL = "TextureCube<float4> g_EnvironmentMap;"


def _build_ref():
    spec = importlib.util.spec_from_file_location("dfx_refshader_build", os.path.join(HERE, "build_ref.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


VARIANTS = [(p, t, o) for p in ("irradiance", "prefilter") for t in (0, 1) for o in (0, 1)]


def name(p: str, t: int, o: int) -> str:
    return f"ibl_{p}__{t}_{o}"


PASSES = [{"name": name(*k), "shader": "ComputeIrradianceMap.psh" if k[0] == "irradiance" else "PrefilterEnvMap.psh",
           "harness": "irradiance_cube.inc" if k[0] == "irradiance" else "prefilter_env_map.inc",
           "macros": {"ENV_MAP_TYPE_CUBE": 0, "ENV_MAP_TYPE_SPHERE": 1, "ENV_MAP_TYPE": k[1], "OPTIMIZE_SAMPLES": k[2]}} for k in VARIANTS]


BRDF_SAMPLES = (1, 2, 64, 512)


def brdf_name(n: int) -> str:
    return f"brdf_lut__{n}"


BRDF_PASSES = [{"name": brdf_name(n), "shader": "PrecomputeBRDF.psh", "harness": "brdf_lut.inc", "macros": {"NUM_SAMPLES": f"{n}u"}, "brdf": True}
               for n in BRDF_SAMPLES]


def translation_unit(br, p: dict, idx: dict) -> str:
    if p.get("brdf"):
        core = open(os.path.join(HERE, "core_defs.inc")).read()
        tu = br.translation_unit(p, idx)
        assert tu.count(core) == 1
        return tu.replace(core, core + open(os.path.join(HERE, "ibl_defs.inc")).read())
    ns = "refsh_ns_" + p["name"]
    drop = lambda t: re.sub(r":\s*(?:" + br.SEMANTICS + r"|WORLD_POS)\b", "", t)  # noqa: E731
    fst = br.flatten("FullScreenTriangleVSOutput.fxh", idx, set())  # what harness/common.inc's full-screen rasteriser is written against
    vs = drop(br.flatten("CubemapFace.vsh", idx, set()))
    ps = drop(br.flatten(p["shader"], idx, set()))
    assert vs.count(VS_POS) == 1 and ps.count(CUBE_DECL) == 1
    vs = vs.replace(VS_POS, "g_RefshPosXY")
    ps = ps.replace(CUBE_DECL, "EnvCube<float4> g_EnvironmentMap;")
    parts = ['#include "prelude.hpp"\n']
    parts += [f"#define {k} {v}\n" for k, v in p["macros"].items()]
    parts.append(f"namespace {ns} {{\nusing namespace hlsl;\n")
    for f in ("core_defs.inc", "env_map_defs.inc", "ibl_defs.inc"):
        parts.append(open(os.path.join(HERE, f)).read())
    parts.append(fst)
    parts.append("namespace ibvs {\nthread_local float2 g_RefshPosXY;\n" + vs + "} // namespace ibvs\n")
    parts.append("namespace ibps {\n" + ps + "} // namespace ibps\n")
    parts.append(open(os.path.join(HERE, "harness", "common.inc")).read())
    parts.append(f'#include "harness/{p["harness"]}"\n')
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
    extra = "".join(open(os.path.join(HERE, f)).read() for f in ("hlsl.hpp", "prelude.hpp", "env_map_defs.inc", "ibl_defs.inc",
                                                                  os.path.join("harness", "ibl_common.inc"),
                                                                  os.path.join("harness", "irradiance_cube.inc"),
                                                                  os.path.join("harness", "prefilter_env_map.inc")))

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
        results = list(ex.map(compile_one, PASSES + BRDF_PASSES))
    errors = [e for _, e in results if e]
    if errors:
        raise RuntimeError("\n".join(errors))
    subprocess.check_call(["g++", "-shared", "-pthread", "-o", LIB, *[o for o, _ in results]])
    return LIB


_lib = None


def run(name_: str, levels, out, num_samples: int, face: int, roughness: float = 0.0, threads: int = 0) -> None:
    """One face of one output level: `out` (s x s x 4 fp32) is written in place. `levels`: the source's levels."""
    global _lib
    from oracle.refshader import refsh
    import numpy as np
    if _lib is None:
        _lib = C.CDLL(LIB)
    ins = [np.ascontiguousarray(a, np.float32) for a in levels]
    assert out.dtype == np.float32 and out.flags["C_CONTIGUOUS"]
    pin = (refsh.Plane * len(ins))(*[refsh._plane(a) for a in ins])
    pout = (refsh.Plane * 1)(refsh._plane(out))
    cb = C.c_float(roughness)
    cb_ptr = (C.c_void_p * 1)(C.cast(C.byref(cb), C.c_void_p))
    cb_size = (C.c_int * 1)(4)
    ip = (C.c_int * 3)(len(ins), face, num_samples)
    a = refsh.Args(pin, len(ins), pout, 1, cb_ptr, cb_size, 1, ip, 3, None, threads or (os.cpu_count() or 1))
    fn = getattr(_lib, "refsh_" + name_)
    fn.restype = C.c_int
    r = fn(C.byref(a))
    if r != 0:
        raise RuntimeError(f"refsh_{name_} failed with {r} (1: wrong resource count, 2: wrong constant buffer)")


def run_brdf(num_samples: int, out) -> None:
    """PrecomputeBRDF.psh with NUM_SAMPLES `num_samples` (one of BRDF_SAMPLES) into `out` (h x w x 2 fp32), in place."""
    global _lib
    from oracle.refshader import refsh
    if _lib is None:
        _lib = C.CDLL(LIB)
    refsh.run(brdf_name(num_samples), [], [out], library=_lib)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    print(build(ap.parse_args().force))
