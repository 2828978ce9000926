"""Shared helpers for the parity tests: error metrics (device planes: gpu_frame.Planes)."""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def psnr(a: np.ndarray, b: np.ndarray, peak: float = 1.0) -> float:
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    mse = float(np.mean((a - b) ** 2))
    return 200.0 if mse == 0.0 else 10.0 * np.log10(peak * peak / mse)


def reinhard(x: np.ndarray) -> np.ndarray:
    x = np.maximum(np.asarray(x, np.float64), 0.0)
    return x / (1.0 + x)


def outlier_fraction(a: np.ndarray, b: np.ndarray, tol: float) -> float:
    d = np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64))
    if d.ndim == 3:
        d = d.max(axis=2)
    return float((d > tol).mean())


def assert_close(name: str, got: np.ndarray, want: np.ndarray, *, tol: float, max_outliers: float = 0.0, min_psnr: float | None = None,
                 hdr: bool = False, mask: np.ndarray | None = None):
    """|got-want| <= tol everywhere except at most `max_outliers` fraction of pixels (branch flips at discontinuities);
    optional PSNR floor (peak 1; HDR planes are compared after Reinhard c/(1+c), SURVEY.md §8d)."""
    assert got.shape == want.shape, f"{name}: shape {got.shape} vs {want.shape}"
    g, w = (reinhard(got), reinhard(want)) if hdr else (np.asarray(got, np.float64), np.asarray(want, np.float64))
    g = np.nan_to_num(g, nan=0.0, posinf=1e30, neginf=-1e30)
    w = np.nan_to_num(w, nan=0.0, posinf=1e30, neginf=-1e30)
    if mask is not None:
        m = mask if g.ndim == 2 else mask[..., None]
        g, w = g * m, w * m
    frac = outlier_fraction(g, w, tol)
    p = psnr(g, w)
    msg = f"{name}: outliers(>{tol:g})={frac:.5%} (allowed {max_outliers:.5%}), max_abs={np.abs(g - w).max():.3e}, psnr={p:.1f} dB"
    assert frac <= max_outliers, msg
    if min_psnr is not None:
        assert p >= min_psnr, msg
    return msg
