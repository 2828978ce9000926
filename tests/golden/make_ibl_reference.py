#!/usr/bin/env python3
"""Regenerates tests/golden/ibl_reference.npz: the outputs of the REFERENCE'S OWN CubemapFace.vsh with ComputeIrradianceMap.psh and
PrefilterEnvMap.psh (compiled for the CPU by oracle/refshader/build_ibl_ref.py, which needs the reference's shaders mounted) in all
eight variants (pass x cube / sphere x OPTIMIZE_SAMPLES 0 / 1) on the cases below. tests/test_ibl_reference.py holds the oracle
(oracle/oracle_ibl.cpp) to them bit for bit. The source maps are regenerated from synth's seeds, not stored.

Each case is a source map and a sample count; every case runs the 4^2 irradiance cube and a 3-level 4^2 prefiltered chain (roughness
0, 0.5 and 1), both with OPTIMIZE_SAMPLES 0 and 1:
  * cube sources: 16^2 with 3 levels, 8^2 with one level, 4^2 with 2 levels (the LOD clamp to g_EnvMipCount - 1 is hit);
  * sphere sources: 64 x 32 with 4 levels, 32 x 16 with one level, a sky with a sun 10^4 times brighter than the rest (64 x 32, 3
    levels), and Hydrogent's default dome (32 x 32 white, one level; HnLight.cpp:667-685);
  * sample counts 1, 2, 37 (not a power of two) and 64.
Beside them, PrecomputeBRDF.psh's pre-integrated GGX table (the same library, the same statement of the transcendentals) against
oracle_compose_ibl.cpp's brdf_lut at 64 x 64 and 32 x 8 with 1, 2, 64 and 512 samples: power-of-two sizes, where the shader runner's
interpolated texture coordinate is the oracle's (x + 0.5) / w exactly.
Every output plane (the six faces of one level, fp32, or one table) is stored as the SHA-256 of its bytes.

    python tests/golden/make_ibl_reference.py
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
import ibl_cases as IC  # noqa: E402

OUT = os.path.join(HERE, "ibl_reference.npz")
SIZE, LEVELS = 4, 3
SAMPLES = (1, 2, 37, 64)
BRDF_SIZES = ((64, 64), (32, 8))
BRDF_SAMPLES = (1, 2, 64, 512)


def sources() -> dict:
    """name -> (type, levels)."""
    return {"cube16x3": (0, IC.cube_chain(16, 3)), "cube8x1": (0, IC.cube_chain(8, 1, seed=3)), "cube4x2_clamp": (0, IC.cube_chain(4, 2, seed=7)),
            "sphere64x32x4": (1, IC.sphere_chain(64, 32, 4)), "sphere32x16x1": (1, IC.sphere_chain(32, 16, 1, seed=3)),
            "sun64x32x3": (1, IC.sun_sphere(64, 32, 3)), "white_dome": (1, IC.white_dome())}


def planes(with_reference: bool):
    """Yields (key, (6, s, s, 4) fp32) for every case, pass, OPTIMIZE_SAMPLES and level: the reference shaders or the oracle."""
    from oracle import oracle_ibl_py as oi
    from oracle.refshader import build_ibl_ref as br

    def ref(p, t, o, lv, s, n, rough):
        out = np.zeros((6, s, s, 4), np.float32)
        for f in range(6):
            br.run(br.name(p, t, o), lv, out[f], n, f, rough)
        return out

    for src, (t, lv) in sources().items():
        for n in SAMPLES:
            for o in (0, 1):
                key = f"{src}/n{n}/opt{o}"
                yield f"{key}/irradiance", (ref("irradiance", t, o, lv, SIZE, n, 0.0) if with_reference else oi.irradiance(t, lv, SIZE, n, bool(o)))
                for m in range(LEVELS):
                    s, r = max(SIZE >> m, 1), oi.roughness(m, LEVELS)
                    yield f"{key}/prefilter{m}", (ref("prefilter", t, o, lv, s, n, r) if with_reference else oi.prefilter(t, lv, s, r, n, bool(o)))
    yield from brdf_tables(with_reference)


def brdf_tables(with_reference: bool):
    """Yields (key, (h, w, 2) fp32) for every BRDF table case: the reference shader or the oracle."""
    from oracle import oracle_py as op
    from oracle.refshader import build_ibl_ref as br
    o = None if with_reference else op.Oracle(8, 8)
    for w, h in BRDF_SIZES:
        for n in BRDF_SAMPLES:
            if with_reference:
                lut = np.zeros((h, w, 2), np.float32)
                br.run_brdf(n, lut)
            else:
                o.brdf_lut((w, h), n)
                lut = o.get("brdf_lut")
            yield f"brdf/{w}x{h}/n{n}", lut


def run(with_reference: bool) -> dict:
    return {k: np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8) for k, a in planes(with_reference)}


def main():
    from oracle.refshader import build_ibl_ref
    build_ibl_ref.build()
    if not build_ibl_ref.available():
        raise SystemExit("librefshaders_ibl.so is not available: the reference's shaders must be mounted")
    np.savez_compressed(OUT, **run(with_reference=True))
    print(OUT)


if __name__ == "__main__":
    main()
