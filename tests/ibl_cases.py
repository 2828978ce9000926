"""Shared by the IBL tests: synthetic source maps and the GPU-vs-oracle error bound of DESIGN.md §2 (IBL precomputation).

The kernels and the oracle compute every sample bit for bit alike; they sum a texel's N samples in different orders. The oracle adds
them in order (error at most gamma(N - 1) times the sum of the terms); the GPU adds samples k, k + 32, ... in lane k and then the 32
partial sums in a 5-level tree (error at most gamma(ceil(N / 32) + 4) times the same sum). gamma(k) = k u / (1 - k u), u = 2^-24. The
terms are non-negative (radiance, and radiance times NoL), so the sum of their magnitudes is the sum itself.
"""
from __future__ import annotations

import numpy as np

from diligentfx_b200 import synth

U = 2.0 ** -24


def gamma(k: int) -> float:
    return k * U / (1.0 - k * U)


def bound(want: np.ndarray, n: int, prefilter: bool, out16: bool) -> np.ndarray:
    """The largest |GPU - oracle| per value, `want` the oracle's fp32 result of N = n samples. Irradiance: mean = sum / N, the two sums
    within gamma(N - 1) and gamma(ceil(N / 32) + 4) of the exact sum, each quotient rounded once. Prefilter: sum(L NoL) / sum(NoL), each
    quotient within (2 gamma + u) / (1 - gamma) of the exact ratio. RGBA16F outputs add half an fp16 ulp (the GPU's store rounds, the
    oracle's value is fp32)."""
    go, gg = gamma(n - 1), gamma(-(-n // 32) + 4)
    a = np.abs(want.astype(np.float64))
    if prefilter:
        ro, rg = (2 * go + U) / (1 - go), (2 * gg + U) / (1 - gg)
        b = a / (1 - ro) * (ro + rg)
    else:
        b = a / (1 - go - U) * (go + gg + 2 * U)
    if out16:
        e = np.floor(np.log2(np.maximum(a * (1 + 1e-3), 2.0 ** -14)))
        b = b + 0.5 * 2.0 ** (e - 10) * (1 + 1e-3)
    return b


def face_gradient_cube(s: int) -> np.ndarray:
    """A (6s, s, 4) cube level whose faces differ in colour and run a gradient along both face axes, so a swapped or mirrored face,
    or a texel-centre error, changes the texels read back."""
    i = (np.arange(s) + 0.5) / s
    jj, ii = np.meshgrid(i, i, indexing="ij")                      # rows j, columns i
    faces = [np.stack([np.full_like(ii, 0.25 + 0.5 * f), 1.0 + 3.0 * ii, 2.0 + 5.0 * jj + f, np.ones_like(ii)], -1) for f in range(6)]
    return np.concatenate(faces, 0).astype(np.float32)


def sun_sphere(w: int, h: int, levels: int) -> list[np.ndarray]:
    """A sky with a sun 10^4 times brighter than the rest (one 2 x 2 texel spot), as a sphere map with a box chain."""
    a = synth.env_map_sphere(w, h, 1, seed=5)[0].copy()
    a[h // 4:h // 4 + 2, w // 3:w // 3 + 2, :3] = 1.0e4 * a[..., :3].mean()
    return synth._box_chain(a, levels, cube=False)


def cube_chain(size: int, levels: int, seed: int = 11) -> list[np.ndarray]:
    """synth's procedural sky as a cube of `levels` levels (up to 16)."""
    return synth._box_chain(synth.env_map_cube(size, 1, seed)[0], levels, cube=True)


def sphere_chain(w: int, h: int, levels: int, seed: int = 11) -> list[np.ndarray]:
    return synth._box_chain(synth.env_map_sphere(w, h, 1, seed)[0], levels, cube=False)


def white_dome() -> list[np.ndarray]:
    """Hydrogent's default dome light texture (HnLight.cpp:667-685): 32 x 32 white, one level, a sphere map."""
    return [np.ones((32, 32, 4), np.float32)]
