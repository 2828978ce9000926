#!/usr/bin/env python3
"""Regenerates tests/golden/bound_box_reference.npz: the outputs of the REFERENCE'S OWN BoundBox.vsh / BoundBox.psh (compiled for the CPU by
oracle/refshader/build_bound_box_ref.py, which needs the reference's shaders mounted, with the line rasteriser of DESIGN.md §2) in all
four sRGB x motion variants, on the cases below. tests/test_bound_box_reference.py holds the oracle (oracle/oracle_bound_box.cpp) to
them bit for bit.

Cases, at 1 x 1, 33 x 17 and 97 x 61: a standard, a reversed, a reversed-infinite and an orthographic camera, each with a box fully in
view, one crossing the near plane, one around the camera, one behind it, one partly off screen and a flat (zero-thickness) one. Every
other case has jittered cameras. The scene depth hides part of the edges in half of the cases and none in the rest. The pattern cycles
through the masks 0xFFFFFFFF, 0x0000FFFF, 0xAAAAAAAA and 0 and the lengths 32, 7.5 and 1. Every output plane is stored as the SHA-256 of
its bytes (bit-exact all the same, and the fixture stays small).

    python tests/golden/make_bound_box_reference.py
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from diligentfx_b200 import capi, synth  # noqa: E402

OUT = os.path.join(HERE, "bound_box_reference.npz")
SIZES = [(1, 1), (33, 17), (97, 61)]
MASKS = [0xFFFFFFFF, 0x0000FFFF, 0xAAAAAAAA, 0]
LENGTHS = [32.0, 7.5, 1.0]
EYE, TARGET = np.array([0.3, 0.5, -4.0]), np.array([0.0, 0.0, 0.0])


def _rot_y(deg: float) -> np.ndarray:
    c, s = np.cos(np.radians(deg)), np.sin(np.radians(deg))
    m = np.eye(4)
    m[0, 0], m[0, 2], m[2, 0], m[2, 2] = c, -s, s, c
    return m.astype(np.float32)


# (name, extent min, extent max, prim transform): world-space boxes around the cameras at EYE looking at TARGET
BOXES = [
    ("in_view", (-1.0, -0.7, -0.8), (1.2, 0.9, 1.0), _rot_y(20.0)),
    ("crosses_near", (-0.8, -0.5, -6.0), (0.9, 0.6, 0.0), None),
    ("camera_inside", (-1.0, -0.5, -5.0), (1.5, 1.5, -3.0), _rot_y(-10.0)),
    ("behind", (-1.0, -1.0, -9.0), (1.0, 1.0, -6.0), None),
    ("off_screen", (1.5, -0.5, -1.0), (6.0, 0.5, 1.0), None),
    ("flat", (-1.0, -1.0, 0.0), (1.0, 1.0, 0.0), _rot_y(35.0)),
]
CAMERAS = ["standard", "reversed", "reversed_infinite", "ortho"]


def variants() -> list:
    from oracle.refshader import build_bound_box_ref
    return build_bound_box_ref.VARIANTS


def camera(kind: str, w: int, h: int, prev: bool, jitter: bool):
    eye = EYE + (np.array([0.08, -0.05, 0.1]) if prev else 0.0)
    rev, inf, ortho = kind.startswith("reversed"), kind == "reversed_infinite", kind == "ortho"
    c = synth.look_at_camera(eye, TARGET, w, h, ortho=ortho, reversed_depth=rev, infinite=inf)
    if jitter:
        c.f2Jitter[0], c.f2Jitter[1] = (-0.0021, 0.0037) if prev else (0.0043, -0.0017)
    return c


def attribs(c: int, b: int, box) -> capi.BoundBoxAttribs:
    """Camera c, box b: the pattern cycles so that every box meets every mask and length; alpha 0, as HnRenderBoundBoxTask's PS main
    stores it (the reference harness stores that main)."""
    return capi.BoundBoxAttribs.make(synth.bound_box_transform(box[1], box[2], box[3]), (0.9, 0.35, 0.125, 0.0), LENGTHS[(b + 2 * c) % 3],
                                     MASKS[(b + c) % 4])


def cases(w: int, h: int) -> list:
    """[(name, curr camera, prev camera, depth, reversed, attribs)]."""
    out = []
    k = 0
    xs = (np.arange(w, dtype=np.float32) + 0.5) / np.float32(w)
    for ci, cam in enumerate(CAMERAS):
        rev = cam.startswith("reversed")
        for bi, box in enumerate(BOXES):
            jit = k % 2 == 1
            c, p = camera(cam, w, h, False, jit), camera(cam, w, h, True, jit)
            far = np.float32(c.fFarPlaneDepth)
            if (k // 2) % 2:
                # a slope of scene depth across the frame that hides the boxes' edges on one side
                lo = np.float32(0.025) if cam == "ortho" else np.float32(0.96)
                d = lo + np.float32(0.03) * xs
                depth = np.broadcast_to((np.float32(1.0) - d) if rev else d, (h, w)).astype(np.float32)
            else:
                depth = np.full((h, w), far, np.float32)
            out.append((f"{cam}/{box[0]}", c, p, depth, rev, attribs(ci, bi, box)))
            k += 1
    return out


def initial(w: int, h: int) -> tuple[np.ndarray, np.ndarray]:
    """What the targets hold before B: a pattern with a NaN and a -0 (kept byte for byte where B does not draw), motion -7."""
    rng = np.random.default_rng(5)
    color = rng.uniform(-1, 2, (h, w, 4)).astype(np.float32)
    color[0, 0, 1], color[h - 1, w - 1, 2] = np.float32("nan"), np.float32(-0.0)
    return color, np.full((h, w, 2), -7.0, np.float32)


def run_one(variant, case, w: int, h: int, with_reference: bool) -> tuple[np.ndarray, np.ndarray]:
    """(colour, motion) of one variant on one case: the reference shaders (with_reference) or the oracle."""
    s, v = variant
    name, cam, prev, depth, rev, a = case
    color, motion = initial(w, h)
    if not with_reference:
        from oracle import oracle_bound_box_py as ob
        return ob.bound_box(cam, prev, a, s | (2 if v else 0) | (4 if rev else 0), depth, color, motion)
    from oracle.refshader import build_bound_box_ref as br
    br.run(br.name(*variant), [depth], [color, motion], cbs=[cam, prev, a], iparams=[int(rev)])
    return color, motion


def run(with_reference: bool) -> dict:
    out = {}
    for (w, h) in SIZES:
        for case in cases(w, h):
            for var in variants():
                c, m = run_one(var, case, w, h, with_reference)
                key = f"{w}x{h}/{case[0]}/{'_'.join(map(str, var))}"
                for k, a in (("color", c), ("motion", m)):
                    out[f"{key}/{k}"] = np.frombuffer(hashlib.sha256(a.tobytes()).digest(), np.uint8)
    return out


def main():
    from oracle.refshader import build_bound_box_ref
    build_bound_box_ref.build()
    if not build_bound_box_ref.available():
        raise SystemExit("librefshaders_bound_box.so is not available: the reference's shaders must be mounted")
    np.savez_compressed(OUT, **run(with_reference=True))
    print(OUT)


if __name__ == "__main__":
    main()
