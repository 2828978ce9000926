"""Filterable shadow maps (ShadowMapManager::ConvertToFilterable): the variance shadow maps of every cascade, converted on the GPU by
dfx_shadow_convert_to_filterable from the depth an application rendered into its cascades.

    attribs = capi.ShadowMapAttribs.default()          # a 3 x 3 filter, EVSM exponents 40 / 5, 32-bit
    attribs.iNumCascades = 4
    evsm = shadow.convert_to_filterable(depth, capi.SHADOW_MODE_EVSM4, attribs, is_32bit=True)   # (4, H, W, 4) float32
"""
from __future__ import annotations

import ctypes as C

import torch

from . import capi

# the filterable format of (mode, is_32bit): (dfx_format, channels, torch dtype of a channel)
_FORMATS = {
    (capi.SHADOW_MODE_VSM, False): (capi.FORMAT_RG16U, 2, torch.uint16), (capi.SHADOW_MODE_VSM, True): (capi.FORMAT_RG32F, 2, torch.float32),
    (capi.SHADOW_MODE_EVSM2, False): (capi.FORMAT_RG16F, 2, torch.float16), (capi.SHADOW_MODE_EVSM2, True): (capi.FORMAT_RG32F, 2, torch.float32),
    (capi.SHADOW_MODE_EVSM4, False): (capi.FORMAT_RGBA16F, 4, torch.float16), (capi.SHADOW_MODE_EVSM4, True): (capi.FORMAT_RGBA32F, 4, torch.float32),
}


def _plane(t: torch.Tensor, fmt: int) -> capi.Plane:
    """A contiguous (H, W[, C]) CUDA tensor as a plane of `fmt`."""
    assert t.is_cuda and t.is_contiguous()
    h, w = int(t.shape[0]), int(t.shape[1])
    return capi.Plane(t.data_ptr(), t.stride(0) * t.element_size(), w, h, fmt, 0)


def filterable_format(mode: int, is_32bit: bool) -> tuple[int, int, torch.dtype]:
    """(dfx_format, channels, element dtype) of the mode's filterable map: VSM RG16_UNORM / RG32F, EVSM2 RG16F / RG32F, EVSM4 RGBA16F /
    RGBA32F."""
    return _FORMATS[(int(mode), bool(is_32bit))]


def convert_to_filterable(depth: torch.Tensor, mode: int, attribs: capi.ShadowMapAttribs, is_32bit: bool,
                          out: torch.Tensor | None = None) -> torch.Tensor | None:
    """The filterable map of `depth`, an N x H x W CUDA tensor of the cascades' depth: float32 (D32_FLOAT) or uint16 (D16_UNORM codes).
    Returns an (N, H, W, C) tensor in the filterable format (uint16 RG16_UNORM codes for 16-bit VSM, float16, or float32; C = 4 for EVSM4,
    2 otherwise), or `out` filled. attribs.iNumCascades must be N and attribs.bIs32BitEVSM must agree with is_32bit. PCF returns None: it
    filters the depth itself. The reference's one-slice intermediate is allocated with the map; the conversion uses it only for ranges
    above 16. Enqueued on the current torch stream; nothing is synchronised."""
    if int(mode) == capi.SHADOW_MODE_PCF:
        return None
    assert depth.dim() == 3 and depth.dtype in (torch.float32, torch.uint16) and depth.is_cuda
    depth = depth.contiguous()
    n, h, w = (int(v) for v in depth.shape)
    fmt, ch, dtype = filterable_format(mode, is_32bit)
    if out is None:
        out = torch.empty((n, h, w, ch), dtype=dtype, device=depth.device)
    assert out.shape == (n, h, w, ch) and out.dtype == dtype and out.is_contiguous()
    in_fmt = capi.FORMAT_R16U if depth.dtype == torch.uint16 else capi.FORMAT_R32F
    src = (capi.Plane * n)(*[_plane(depth[i], in_fmt) for i in range(n)])
    dst = (capi.Plane * n)(*[_plane(out[i], fmt) for i in range(n)])
    # allocated on the stream the conversion runs on, so the caching allocator reuses it only after the conversion
    inter = torch.empty((h, w, ch), dtype=dtype, device=depth.device)
    s = C.c_void_p(torch.cuda.current_stream(depth.device).cuda_stream)
    capi.check(capi.load().dfx_shadow_convert_to_filterable(s, int(mode), C.byref(attribs), src, n, dst, C.byref(_plane(inter, fmt))),
               "dfx_shadow_convert_to_filterable")
    return out


def filter_radii(attribs: capi.ShadowMapAttribs, cascade: int, width: int, height: int) -> tuple[float, float]:
    """dfx_shadow_filter_radii: the (horizontal, vertical) radius ConvertToFilterable uses for a cascade of a width x height map."""
    rh, rv = C.c_float(), C.c_float()
    capi.check(capi.load().dfx_shadow_filter_radii(C.byref(attribs), int(cascade), int(width), int(height), C.byref(rh), C.byref(rv)),
               "dfx_shadow_filter_radii")
    return rh.value, rv.value
