"""The oracle's ConvertToFilterable (oracle/oracle_shadow.cpp) against the reference's own ShadowConversions.fx, bit for bit (the stored
texels of every case are compared through their SHA-256, NaN payloads aside), on the cases of tests/golden/make_shadow_reference.py:
every mode x 16 / 32 bits x D16 / D32, radii 0 to 7.9, fixed filter sizes 1, 2, 3, 5 and 8, the varying filter per cascade and axis,
1 x 1, 3 x 2 and non-square maps, exponents above both clamps, and depth outside [0, 1], inf and NaN. The recorded shader outputs are
tests/golden/shadow_reference.npz; where the shader can be run, the fixture must be what it produces now."""
import importlib.util
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


def _gen():
    spec = importlib.util.spec_from_file_location("make_shadow_reference", os.path.join(HERE, "golden", "make_shadow_reference.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_oracle_matches_committed_reference_outputs(built):
    m = _gen()
    want = np.load(m.OUT)
    got = m.run(with_reference=False)
    assert set(got) == set(want.files) and len(got) == len(m.cases())
    bad = [k for k in got if not np.array_equal(got[k], want[k])]
    assert not bad, f"the oracle differs from the reference's shader on {bad}"


def test_fixture_is_what_the_reference_shader_draws_now(built):
    from oracle.refshader import build_shadow_ref
    if not build_shadow_ref.available():
        pytest.skip("the reference's shaders are not built here")
    m = _gen()
    want = np.load(m.OUT)
    got = m.run(with_reference=True)
    assert all(np.array_equal(got[k], want[k]) for k in got)
