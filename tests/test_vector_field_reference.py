"""The oracle's vector field overlay (VectorField.vsh and VectorFieldRenderer's default PS main under its pipeline state, rasterised by
the line rule of DESIGN.md §2) against the reference's own shaders, bit for bit (NaN payloads included: the bytes of every output plane
are compared through their SHA-256), with sRGB off and on: at 1 x 1, 33 x 17 and 97 x 61, for zero, pan, rotation, converging-vortex,
non-finite and beyond-the-guard-band fields on field planes of the target's size and of another, with grids of 0 x n, 1 x 1, a width
that does not divide the target's and more lines than field texels, with and without a bias. The recorded shader outputs are
tests/golden/vector_field_reference.npz; where the shaders can be run, the fixture must be what they produce now."""
import importlib.util
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


def _gen():
    spec = importlib.util.spec_from_file_location("make_vector_field_reference", os.path.join(HERE, "golden", "make_vector_field_reference.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_oracle_matches_committed_reference_outputs(built):
    m = _gen()
    want = np.load(m.OUT)
    got = m.run(with_reference=False)
    assert set(got) == set(want.files) and len(got) == len(m.SIZES) * len(m.cases(33, 17)) * len(m.SRGB)
    bad = [k for k in want.files if got[k].tobytes() != want[k].tobytes()]
    assert not bad, f"the oracle's vector field no longer reproduces the reference shaders on {len(bad)} planes:\n  " + "\n  ".join(bad[:20])


def test_cases_cover_the_fields_grids_and_sizes(built):
    """Every field kind and grid, both field sizes, bias on and off; lines are drawn in most cases, none with a 0 x n grid, and the
    non-finite and far fields leave some lines out."""
    m = _gen()
    cs = m.cases(97, 61)
    assert len(cs) == len(m.FIELDS) * len(m.GRIDS) * 2
    assert any(c[1].Bias[0] != 0 for c in cs) and any(c[1].Bias[0] == 0 for c in cs)
    assert any(c[2].shape[:2] != (61, 97) for c in cs) and any(c[2].shape[:2] == (61, 97) for c in cs)
    assert any(int(c[1].GridSize[0]) * int(c[1].GridSize[1]) > c[2].shape[0] * c[2].shape[1] for c in cs)
    assert any(97 % int(c[1].GridSize[0]) != 0 for c in cs if c[1].GridSize[0] > 1)
    assert np.isnan(next(c[2] for c in cs if c[0].startswith("nonfinite"))).any()
    c0 = m.initial(97, 61)
    drawn = {c[0]: int((m.run_one(0, c, 97, 61, False).view(np.uint32) != c0.view(np.uint32)).any(-1).sum()) for c in cs}
    assert all(v == 0 for k, v in drawn.items() if "/0xn/" in k)
    for fk in m.FIELDS:
        assert any(v > 0 for k, v in drawn.items() if k.startswith(fk + "/")), fk


def test_fixture_is_current_where_the_shader_is_present(built):
    from oracle.refshader import build_vector_field_ref
    build_vector_field_ref.build()
    if not build_vector_field_ref.available():
        pytest.skip("librefshaders_vector_field.so not available")
    m = _gen()
    want, got = np.load(m.OUT), m.run(with_reference=True)
    assert set(got) == set(want.files)
    for k in want.files:
        assert got[k].tobytes() == want[k].tobytes(), f"{k}: regenerate tests/golden/vector_field_reference.npz deliberately"
