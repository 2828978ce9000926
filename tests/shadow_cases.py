"""Shared pieces of the filterable-shadow-map tests: attribs builders and the bit comparison of filterable texels."""
from __future__ import annotations

import numpy as np

from diligentfx_b200 import capi

VSM, EVSM2, EVSM4 = capi.SHADOW_MODE_VSM, capi.SHADOW_MODE_EVSM2, capi.SHADOW_MODE_EVSM4
MODES = (VSM, EVSM2, EVSM4)


def attribs(n: int, is32: bool = True, fixed: int = 3, world: float = 0.0, scales=None, pos: float = 40.0, neg: float = 5.0) -> capi.ShadowMapAttribs:
    """ShadowMapAttribs with its defaults but for these fields; `scales`: per cascade (f4LightSpaceScale.x, .y)."""
    a = capi.ShadowMapAttribs.default()
    a.iNumCascades, a.fNumCascades = n, float(n)
    a.bIs32BitEVSM, a.iFixedFilterSize, a.fFilterWorldSize = int(is32), fixed, world
    a.fEVSMPositiveExponent, a.fEVSMNegativeExponent = pos, neg
    for i, (sx, sy) in enumerate(scales or []):
        a.Cascades[i].f4LightSpaceScale[0], a.Cascades[i].f4LightSpaceScale[1] = sx, sy
    return a


def radius_scales(radii, width: int, height: int) -> list[tuple[float, float]]:
    """Light-space scales that make the varying filter's radius about (rh, rv) per cascade with fFilterWorldSize 1: r = s * 0.5 / 2 * size."""
    return [(4.0 * rh / width, 4.0 * rv / height) for rh, rv in radii]


def same_bits(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """Element-wise: identical bits, or both NaN (a NaN's payload is not part of the rule)."""
    assert a.dtype == b.dtype and a.shape == b.shape, (a.dtype, b.dtype, a.shape, b.shape)
    if a.dtype == np.uint16:
        return a == b
    u = np.uint16 if a.dtype == np.float16 else np.uint32
    return (a.view(u) == b.view(u)) | (np.isnan(a) & np.isnan(b))


def assert_same(got: np.ndarray, want: np.ndarray, what: str = "") -> None:
    ok = same_bits(got, want)
    if not ok.all():
        idx = np.argwhere(~ok)
        k = tuple(idx[0])
        raise AssertionError(f"{what}: {int((~ok).sum())} of {ok.size} texels differ; first at {k}: got {got[k]!r}, want {want[k]!r}")
