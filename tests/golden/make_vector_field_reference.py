#!/usr/bin/env python3
"""Regenerates tests/golden/vector_field_reference.npz: the outputs of the REFERENCE'S OWN VectorField.vsh and VectorFieldRenderer's
default PS main (compiled for the CPU by oracle/refshader/build_vector_field_ref.py, which needs the reference's sources mounted, with the
line rasteriser of DESIGN.md §2), with sRGB off and on, on the cases below. tests/test_vector_field_reference.py holds the oracle
(oracle/oracle_vector_field.cpp) to them bit for bit.

Cases, at 1 x 1, 33 x 17 and 97 x 61: the fields zero, a pan, a rotation, a converging vortex, NaN / Inf / huge texels, and vectors whose
ends lie beyond the guard band; each on a field plane of the target's size and on one of another size; with grids of 0 x n, 1 x 1,
a width that does not divide the target's (taps between texels) and more lines than the field has texels; with and without a bias.
Every output plane is stored as the SHA-256 of its bytes (bit-exact all the same, and the fixture stays small).

    python tests/golden/make_vector_field_reference.py
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from diligentfx_b200 import capi, synth  # noqa: E402

OUT = os.path.join(HERE, "vector_field_reference.npz")
SIZES = [(1, 1), (33, 17), (97, 61)]
FIELDS = ["zero", "pan", "rotation", "vortex", "nonfinite", "beyond_guard"]
GRIDS = ["0xn", "1x1", "non_divisor", "dense"]
SRGB = [0, 1]


def field(kind: str, fw: int, fh: int) -> np.ndarray:
    if kind == "zero":
        return np.zeros((fh, fw, 2), np.float32)
    if kind == "pan":
        return synth.motion_pan(fw, fh, 0.05, -0.03)
    if kind == "rotation":
        return synth.motion_rotation(fw, fh, 0.2)
    if kind == "vortex":
        return synth.motion_vortex(fw, fh, 0.4, 0.7)
    if kind == "nonfinite":
        return synth.motion_extreme(fw, fh, seed=fw * 131 + fh)
    f = synth.motion_random(fw, fh, seed=fw + fh, sigma=0.1)  # beyond_guard: every third texel 1e6 (2^20 pixels is ~4e3 NDC here)
    f.reshape(-1, 2)[::3] = np.float32(1e6)
    return f


def grid(kind: str, w: int, h: int, fw: int, fh: int) -> tuple[int, int]:
    return {"0xn": (0, max(h // 4, 1)), "1x1": (1, 1), "non_divisor": (max(w // 3 + 1, 2), max(h // 5 + 1, 2)), "dense": (2 * fw + 1, 2 * fh + 1)}[kind]


def cases(w: int, h: int) -> list:
    """(name, attribs, field) for a w x h target: every field kind x grid x field size (the target's, and another), the bias on in
    every other case."""
    out, n = [], 0
    for fk in FIELDS:
        for gk in GRIDS:
            for other in (False, True):
                fw, fh = (max(w // 2 + 3, 2), max(h // 3 + 2, 2)) if other else (w, h)
                bias = (0.01, -0.02) if n % 2 else (0.0, 0.0)
                a = capi.VectorFieldAttribs.make(grid=grid(gk, w, h, fw, fh), bias=bias, scale=(-1.2, -1.2 if n % 3 else 0.8),
                                                 start_color=(1.0, 0.9, 0.25, 1.0), end_color=(0.5, 0.125, 0.75, 0.5))
                out.append((f"{fk}/{gk}/{'other' if other else 'same'}", a, field(fk, fw, fh)))
                n += 1
    return out


def initial(w: int, h: int) -> np.ndarray:
    """What the target holds before the field: a pattern with a NaN and a -0 (kept byte for byte where no line draws)."""
    rng = np.random.default_rng(5)
    color = rng.uniform(-1, 2, (h, w, 4)).astype(np.float32)
    color[0, 0, 1], color[h - 1, w - 1, 2] = np.float32("nan"), np.float32(-0.0)
    return color


def run_one(srgb: int, case, w: int, h: int, with_reference: bool) -> np.ndarray:
    """The target after one case: the reference shaders (with_reference) or the oracle."""
    name, a, f = case
    if not with_reference:
        from oracle import oracle_vector_field_py as ov
        return ov.vector_field(a, srgb, f, initial(w, h))
    from oracle.refshader import build_vector_field_ref as br
    return br.run(a, srgb, f, initial(w, h))


def run(with_reference: bool) -> dict:
    out = {}
    for (w, h) in SIZES:
        for case in cases(w, h):
            for s in SRGB:
                c = run_one(s, case, w, h, with_reference)
                out[f"{w}x{h}/{case[0]}/{s}"] = np.frombuffer(hashlib.sha256(c.tobytes()).digest(), np.uint8)
    return out


def main():
    from oracle.refshader import build_vector_field_ref
    build_vector_field_ref.build()
    if not build_vector_field_ref.available():
        raise SystemExit("librefshaders_vector_field.so is not available: the reference's sources must be mounted")
    np.savez_compressed(OUT, **run(with_reference=True))
    print(OUT)


if __name__ == "__main__":
    main()
