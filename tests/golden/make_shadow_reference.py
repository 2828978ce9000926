#!/usr/bin/env python3
"""Regenerates tests/golden/shadow_reference.npz: the filterable maps the REFERENCE'S OWN ShadowConversions.fx draws (VSMHorzPS /
EVSMHorzPS, then VertBlurPS, through ShadowMapManager::ConvertToFilterable's sequence; compiled for the CPU by
oracle/refshader/build_shadow_ref.py, which needs the reference's shaders mounted) on the cases below. tests/test_shadow_reference.py
holds the oracle (oracle/oracle_shadow.cpp) to them bit for bit. The depth is regenerated from synth's seeds, not stored; every case's
output (all cascades, the stored texels of the filterable format) is stored as the SHA-256 of its bytes.

The cases cover every mode x 16 / 32 bits x D16 / D32; radii 0, 0.3, 0.5, 1, 1.2, 1.5, 4.5 and 7.9; fixed filter sizes 1, 2, 3, 5 and
8 and the varying filter with other radii per cascade and per axis; 1 x 1, 3 x 2 and non-square maps; exponents above both clamps; and
depth outside [0, 1], inf and NaN.

    python tests/golden/make_shadow_reference.py
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
import shadow_cases as SC  # noqa: E402
from diligentfx_b200 import synth  # noqa: E402

OUT = os.path.join(HERE, "shadow_reference.npz")
RADII = (0.0, 0.3, 0.5, 1.0, 1.2, 1.5, 4.5, 7.9)
FIXED = (1, 2, 3, 5, 8)


def cases() -> dict:
    """name -> (mode, is32, d16, hostile, n, w, h, seed, attribs kwargs)."""
    c = {}
    for mode in SC.MODES:
        for is32 in (False, True):
            for d16 in (False, True):
                c[f"m{mode}_{32 if is32 else 16}_{'d16' if d16 else 'd32'}"] = (mode, is32, d16, False, 2, 29, 21, 1, {})
                c[f"m{mode}_{32 if is32 else 16}_{'d16' if d16 else 'd32'}_clamped"] = (mode, is32, d16, False, 1, 17, 13, 2,
                                                                                          {"fixed": 5, "pos": 61.0, "neg": 44.0})
            c[f"m{mode}_{32 if is32 else 16}_hostile"] = (mode, is32, False, True, 2, 26, 19, 3,
                                                          {"fixed": 0, "world": 1.0, "radii": [(1.2, 2.5), (4.5, 0.3)]})
        for r in RADII:
            c[f"m{mode}_r{r}"] = (mode, mode != 2, True, False, 1, 24, 18, 4, {"fixed": 0, "world": 1.0, "radii": [(r, r)]})
        for f in FIXED:
            c[f"m{mode}_fixed{f}"] = (mode, mode == 3, False, False, 2, 20, 15, 5, {"fixed": f})
        c[f"m{mode}_varying"] = (mode, True, True, False, 4, 32, 24, 6,
                                 {"fixed": 0, "world": 1.0, "radii": [(0.3, 1.5), (1.2, 0.5), (4.5, 1.0), (7.9, 2.6)]})
        for w, h in ((1, 1), (3, 2), (2, 3), (37, 5)):
            c[f"m{mode}_{w}x{h}"] = (mode, mode == 4, True, False, 2, w, h, 7, {"fixed": 0, "world": 1.0, "radii": [(1.5, 1.5), (4.5, 0.5)]})
    return c


def inputs(case):
    mode, is32, d16, hostile, n, w, h, seed, kw = case
    kw = dict(kw)
    radii = kw.pop("radii", None)
    if radii:
        kw["scales"] = SC.radius_scales(radii, w, h)
    return SC.attribs(n, is32, **kw), synth.shadow_cascades(n, w, h, seed=seed, d16=d16, hostile=hostile)


def digest(a: np.ndarray) -> np.ndarray:
    """SHA-256 of the texels with every NaN made the one quiet NaN: a NaN's payload is not part of the rule."""
    if a.dtype != np.uint16:
        a = np.where(np.isnan(a), np.array(np.nan, a.dtype), a)
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def run(with_reference: bool) -> dict:
    """name -> the SHA-256 of the stored texels, from the reference's shaders (with_reference) or the oracle."""
    from oracle import oracle_shadow_py as osh
    if with_reference:
        from oracle.refshader import build_shadow_ref as ref
        ref.build()
    out = {}
    for name, case in cases().items():
        a, depth = inputs(case)
        mode, is32 = case[0], case[1]
        vals = ref.convert(mode, a, depth, is32) if with_reference else osh.convert(mode, a, depth, is32)
        out[name] = digest(osh.stored(mode, is32, vals))
    return out


if __name__ == "__main__":
    got = run(with_reference=True)
    np.savez_compressed(OUT, **got)
    print(f"wrote {OUT}: {len(got)} cases")
