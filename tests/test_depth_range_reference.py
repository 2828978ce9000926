"""The depth range oracle (oracle/oracle_depth_range.cpp) against the reference's own ClearDepthRange.csh and ComputeDepthRange.csh, bit
for bit, on every case of tests/test_depth_range_cpu.cases(): standard, reversed and reversed-infinite depth, all-background planes,
1x1 and odd sizes, and planes of negative values, +-0, NaN and +-inf. The shaders run on the CPU with a group runner
(oracle/refshader/build_depth_range_ref.py): groupshared as a static array, the 64 invocations of a group as host threads meeting at
a std::barrier, the Interlocked* through std::atomic_ref. So the oracle's reading of which invocation holds which partial, and of how
min / max treat +-0 and NaN, is the shader's. The recorded outputs are tests/golden/depth_range_reference.npz; where the shaders can be
run, the fixture must be what they produce now."""
import importlib.util
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


def _gen():
    spec = importlib.util.spec_from_file_location("make_depth_range_reference", os.path.join(HERE, "golden", "make_depth_range_reference.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_oracle_matches_committed_reference_outputs():
    m = _gen()
    want = np.load(m.OUT)
    got = m.run(with_reference=False)
    assert set(got) == set(want.files)
    bad = [f"{k}: {got[k].tolist()} != {want[k].tolist()}" for k in want.files if got[k].tobytes() != want[k].tobytes()]
    assert not bad, "the depth range oracle no longer reproduces the reference shaders:\n  " + "\n  ".join(bad)


def test_fixture_is_current_where_the_shaders_are_present():
    from oracle.refshader import build_depth_range_ref
    build_depth_range_ref.build()
    if not build_depth_range_ref.available():
        pytest.skip("librefshaders_depth_range.so not available")
    m = _gen()
    want, got = np.load(m.OUT), m.run(with_reference=True)
    assert set(got) == set(want.files)
    for k in want.files:
        assert got[k].tobytes() == want[k].tobytes(), f"{k}: regenerate tests/golden/depth_range_reference.npz deliberately"
