"""IBL cube-map precomputation without a GPU: properties of oracle_ibl_py (round trip, constant and linear maps), and the
interface (the face matrices the kernels hard-code, the C-ABI export, the Python constants)."""
import os
import re

import numpy as np
import pytest

import ibl_cases as IC
from diligentfx_b200 import capi
from oracle import oracle_ibl_py as oi

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CUBE, SPHERE = capi.ENV_MAP_TYPE_CUBE, capi.ENV_MAP_TYPE_SPHERE


@pytest.fixture(scope="module", autouse=True)
def _oracle():
    oi.build()


@pytest.mark.parametrize("s", [4, 16])
@pytest.mark.parametrize("opt", [False, True])
def test_round_trip_gives_back_the_source(s, opt):
    """Prefiltered at roughness 0 into a face of the source's size, every texel reads back its own texel: this pins the face order, the
    face matrices (a mirrored or swapped face changes colour or gradient direction) and the texel-centre rule."""
    src = IC.face_gradient_cube(s)
    got = oi.as_cube(oi.prefilter(CUBE, [src], s, 0.0, 16, opt))
    assert np.abs(got[..., :3] - src[..., :3]).max() <= 4e-6 * np.abs(src[..., :3]).max()


@pytest.mark.parametrize("env_type", [CUBE, SPHERE])
def test_constant_map_gives_the_constant(env_type):
    c = 3.5
    lv = [np.full((48, 8, 4), c, np.float32), np.full((24, 4, 4), c, np.float32)] if env_type == CUBE else [np.full((16, 32, 4), c, np.float32)]
    irr = oi.irradiance(env_type, lv, 4, 1000)
    assert np.abs(irr[..., :3] - c).max() <= c * (IC.gamma(999) + 16 * IC.U) and (irr[..., 3] == 1).all()
    for m in range(3):
        p = oi.prefilter(env_type, lv, max(4 >> m, 1), oi.roughness(m, 3), 256)
        assert np.abs(p[..., :3] - c).max() <= c * (2 * IC.gamma(255) + 16 * IC.U) and (p[..., 3] == 0).all()


def _linear_cube(s: int, c: np.ndarray, a: np.ndarray) -> np.ndarray:
    """L(w) = c + a . w at every texel centre's direction of a (6s, s, 4) cube (the D3D face table)."""
    t = (np.arange(s) + 0.5) / s * 2.0 - 1.0
    tc, sc = np.meshgrid(t, t, indexing="ij")
    axes_s, axes_t = [(2, -1), (2, 1), (0, 1), (0, 1), (0, 1), (0, -1)], [(1, -1), (1, -1), (2, 1), (2, -1), (1, -1), (1, -1)]
    faces = []
    for f in range(6):
        d = np.zeros((s, s, 3))
        d[..., f // 2] = -1.0 if f % 2 else 1.0
        d[..., axes_s[f][0]] = axes_s[f][1] * sc
        d[..., axes_t[f][0]] = axes_t[f][1] * tc
        d /= np.linalg.norm(d, axis=-1, keepdims=True)
        faces.append(np.concatenate([c + d @ np.diag(a), np.ones((s, s, 1))], -1))
    return np.concatenate(faces, 0).astype(np.float32)


def test_linear_map_irradiance_is_c_plus_two_thirds_a_dot_n():
    """For L(w) = c + a . w the cosine-weighted mean over the hemisphere around N is c + (2/3) a . N. With OPTIMIZE_SAMPLES 0 the
    oracle reads level 0 only; the Hammersley estimate of the mean of a linear function converges as O(log N / N) and the bilinear
    texels differ from the linear function by O(1/s^2), so at N = 4096 and s = 64 every texel is within 0.004 |a| of the exact value."""
    c, a = np.array([1.0, 1.0, 1.0]), np.array([0.6, -0.4, 0.8])
    src = _linear_cube(64, c, a)
    got = oi.irradiance(CUBE, [src], 8, 4096, optimize=False)
    lin = _linear_cube(8, c, a)[..., :3] - c                      # a . N at the output's texel directions
    err = np.abs(oi.as_cube(got)[..., :3] - (c + 2.0 / 3.0 * lin))
    print(f"largest error / |a|: {err.max() / np.linalg.norm(a):.3g}")
    assert err.max() <= 0.004 * np.linalg.norm(a)


def test_face_matrices_are_diligent_cores_float_rotations():
    """dfx_ibl.cu hard-codes cos(-pi/2) and sin(-pi) of DiligentCore's float angles (PI_F / 2, PI_F); they must be those values."""
    src = open(os.path.join(ROOT, "diligentfx_b200", "csrc", "dfx_ibl.cu")).read()
    m = re.search(r"kC90 = ([-\d.e+]+)f, kS180 = ([-\d.e+]+)f", src)
    pi = np.float32(np.pi)
    assert np.float32(m.group(1)) == np.float32(np.cos(np.float64(-pi / np.float32(2))))
    assert np.float32(m.group(2)) == np.float32(np.sin(np.float64(-pi)))
    assert np.float32(np.sin(np.float64(-pi / np.float32(2)))) == -1.0 and np.float32(np.cos(np.float64(-pi))) == -1.0


def test_c_abi_and_python_interface():
    syms = capi.declared_symbols()
    assert "dfx_pass_irradiance_cube" in syms and "dfx_pass_prefilter_env_map" in syms
    header = open(capi.HEADER_PATH).read()
    assert re.search(r"#define DFX_MAX_ENV_LEVELS 16\b", header)
    assert capi.MAX_ENV_LEVELS == 16 and (capi.IRRADIANCE_CUBE_DIM, capi.PREFILTERED_ENV_MAP_DIM) == (64, 256)
    assert (capi.DEFAULT_DIFFUSE_SAMPLES, capi.DEFAULT_SPECULAR_SAMPLES) == (8192, 256)
    cpp = open(os.path.join(ROOT, "include", "dfx", "PBR_Renderer.hpp")).read()
    for k in ("IrradianceCubeDim    = 64", "PrefilteredEnvMapDim = 256", "IrradianceCubeFmt    = TEX_FORMAT_RGBA16_FLOAT"):
        assert k in cpp
    assert [oi.roughness(m, 9) for m in (0, 4, 8)] == [0.0, 0.5, 1.0]
