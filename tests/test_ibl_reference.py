"""The oracle's IBL precomputation (oracle/oracle_ibl.cpp) against the reference's own CubemapFace.vsh, ComputeIrradianceMap.psh and
PrefilterEnvMap.psh, bit for bit (the bytes of every output level are compared through their SHA-256), in all eight variants of
oracle/refshader/build_ibl_ref.py on the cases of tests/golden/make_ibl_reference.py: cube and sphere sources with one and several
levels and the LOD clamp, a sun 10^4 times brighter than the rest, Hydrogent's white default dome, 1, 2, 37 and 64 samples,
OPTIMIZE_SAMPLES 0 and 1, the irradiance cube and three prefiltered levels (roughness 0, 0.5, 1); and PrecomputeBRDF.psh's GGX table
against oracle_compose_ibl.cpp's at 64 x 64 and 32 x 8 with 1, 2, 64 and 512 samples. The recorded shader outputs are
tests/golden/ibl_reference.npz; where the shader can be run, the fixture must be what it produces now."""
import hashlib
import importlib.util
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


def _gen():
    spec = importlib.util.spec_from_file_location("make_ibl_reference", os.path.join(HERE, "golden", "make_ibl_reference.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_oracle_matches_committed_reference_outputs(built):
    m = _gen()
    want = np.load(m.OUT)
    got = m.run(with_reference=False)
    cubes = len(m.sources()) * len(m.SAMPLES) * 2 * (1 + m.LEVELS)
    assert set(got) == set(want.files) and len(got) == cubes + len(m.BRDF_SIZES) * len(m.BRDF_SAMPLES)
    bad = [k for k in want.files if got[k].tobytes() != want[k].tobytes()]
    assert not bad, f"the oracle's IBL passes no longer reproduce the reference shaders on {len(bad)} planes:\n  " + "\n  ".join(bad[:20])


def test_brdf_table_matches_the_reference_shader(built):
    """PrecomputeBRDF.psh against oracle_compose_ibl.cpp's brdf_lut() under DESIGN.md §2's rule (one rounding per operation, cos / sin
    correctly rounded, pow(x, 5) as ((x * x) * (x * x)) * x in double), bit for bit, at 64 x 64 and 32 x 8 with 1, 2, 64 and 512
    samples: every table case of the committed reference outputs is present and reproduced."""
    m = _gen()
    want = np.load(m.OUT)
    keys = [f"brdf/{w}x{h}/n{n}" for w, h in m.BRDF_SIZES for n in m.BRDF_SAMPLES]
    assert set(keys) <= set(want.files)
    got = {k: np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8) for k, a in m.brdf_tables(False)}
    bad = [k for k in keys if got[k].tobytes() != want[k].tobytes()]
    assert not bad, f"the oracle's BRDF table no longer reproduces PrecomputeBRDF.psh on {bad}"


def test_cases_reach_the_lod_clamp_and_a_sun(built):
    """The sun is 10^4 times the sky's mean; the 2-level cube and the 1-level sources make g_EnvMipCount - 1 the clamp."""
    m = _gen()
    src = m.sources()
    sun = src["sun64x32x3"][1][0][..., :3]
    assert sun.max() >= 1e3 * np.median(sun)
    assert len(src["cube4x2_clamp"][1]) == 2 and len(src["white_dome"][1]) == 1 and src["white_dome"][1][0].shape == (32, 32, 4)


def test_fixture_is_current_where_the_shader_is_present(built):
    from oracle.refshader import build_ibl_ref
    build_ibl_ref.build()
    if not build_ibl_ref.available():
        pytest.skip("librefshaders_ibl.so not available")
    m = _gen()
    want, got = np.load(m.OUT), m.run(with_reference=True)
    assert set(got) == set(want.files)
    for k in want.files:
        assert got[k].tobytes() == want[k].tobytes(), f"{k}: regenerate tests/golden/ibl_reference.npz deliberately"
