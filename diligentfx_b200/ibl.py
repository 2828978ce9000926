"""IBL cube-map precomputation (PBR_Renderer::PrecomputeCubemaps): the irradiance cube and the prefiltered environment map a PBR renderer
samples, convolved on the GPU from an environment map by dfx_pass_irradiance_cube and dfx_pass_prefilter_env_map.

Hydrogent runs this once per dome-light texture, not per frame. Its environment-map background draws the prefiltered map at MipLevel 1:

    irradiance, prefiltered = ibl.precompute_cubemaps(capi.ENV_MAP_TYPE_SPHERE, sky_levels)
    chain.set_environment_map(capi.ENV_MAP_TYPE_CUBE, prefiltered[:8])   # the chain takes up to 8 levels; level 8 is never read
"""
from __future__ import annotations

import ctypes as C

import torch

from . import capi


def _planes(levels) -> "C.Array":
    return (capi.Plane * len(levels))(*[capi.plane_of(t) for t in levels])


def precompute_cubemaps(env_type: int, levels, irradiance_dim: int = capi.IRRADIANCE_CUBE_DIM,
                        prefiltered_dim: int = capi.PREFILTERED_ENV_MAP_DIM, prefiltered_levels: int = 0, num_diffuse_samples: int = 0,
                        num_specular_samples: int = 0, optimize_samples: bool = True, dtype: torch.dtype = torch.float16,
                        stream: int | None = None) -> tuple[torch.Tensor, list[torch.Tensor]]:
    """Both passes over the source map `levels` (its mip chain as contiguous CUDA tensors, float32 or float16 RGBA: (6s, s, 4) per level
    for a cube with faces +X, -X, +Y, -Y, +Z, -Z stacked, (h, w, 4) for a sphere; up to capi.MAX_ENV_LEVELS). Returns (irradiance,
    prefiltered): the irradiance cube as one (6d, d, 4) tensor and the prefiltered map's levels as (6 s_m, s_m, 4) tensors, in `dtype`
    (float16, the reference's RGBA16_FLOAT, or float32), the layout PostProcessChain.set_environment_map takes. `prefiltered_levels` 0 =
    the full chain down to 1 x 1 (9 levels at 256). Sample counts 0 = the reference's 8192 and 256. Enqueued on `stream` (default: the
    current torch stream); nothing is synchronised."""
    assert dtype in (torch.float16, torch.float32)
    n_pre = prefiltered_levels or prefiltered_dim.bit_length()
    dev = levels[0].device
    irr = torch.empty((6 * irradiance_dim, irradiance_dim, 4), dtype=dtype, device=dev)
    pre = [torch.empty((6 * max(prefiltered_dim >> m, 1), max(prefiltered_dim >> m, 1), 4), dtype=dtype, device=dev) for m in range(n_pre)]
    lib = capi.load()
    s = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream if stream is None else stream)
    src = _planes(levels)
    capi.check(lib.dfx_pass_irradiance_cube(s, int(env_type), src, len(levels), C.c_uint32(num_diffuse_samples), int(optimize_samples),
                                            C.byref(capi.plane_of(irr))), "dfx_pass_irradiance_cube")
    capi.check(lib.dfx_pass_prefilter_env_map(s, int(env_type), src, len(levels), C.c_uint32(num_specular_samples), int(optimize_samples),
                                              _planes(pre), n_pre), "dfx_pass_prefilter_env_map")
    return irr, pre
