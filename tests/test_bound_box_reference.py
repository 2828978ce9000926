"""The oracle's bounding box (B: BoundBox.vsh / BoundBox.psh under BoundBoxRenderer's pipeline state, rasterised by the line rule of
DESIGN.md §2) against the reference's own shaders, bit for bit (NaN payloads included: the bytes of every output plane are compared
through their SHA-256), in all four sRGB x motion variants of oracle/refshader/build_bound_box_ref.py: at 1 x 1, 33 x 17 and 97 x 61,
for a standard, a reversed, a reversed-infinite and an orthographic camera, with boxes in view, crossing the near plane, around the
camera, behind it, partly off screen and flat, jittered and not, partly hidden by scene depth, with four pattern masks and three
pattern lengths. The recorded shader outputs are tests/golden/bound_box_reference.npz; where the shaders can be run, the fixture must
be what they produce now."""
import importlib.util
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


def _gen():
    spec = importlib.util.spec_from_file_location("make_bound_box_reference", os.path.join(HERE, "golden", "make_bound_box_reference.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_oracle_matches_committed_reference_outputs(built):
    m = _gen()
    want = np.load(m.OUT)
    got = m.run(with_reference=False)
    assert set(got) == set(want.files) and len(got) == 2 * len(m.SIZES) * len(m.cases(33, 17)) * len(m.variants())
    bad = [k for k in want.files if got[k].tobytes() != want[k].tobytes()]
    assert not bad, f"the oracle's bounding box no longer reproduces the reference shaders on {len(bad)} planes:\n  " + "\n  ".join(bad[:20])


def test_cases_cover_the_cameras_boxes_and_patterns(built):
    """Every box position and camera, every mask and length, jittered and hidden cases; the box is drawn in most cases and not at all
    behind the camera; the flat box has zero thickness."""
    m = _gen()
    cs = m.cases(97, 61)
    assert len(cs) == len(m.CAMERAS) * len(m.BOXES)
    assert {c[5].PatternMask for c in cs} == set(m.MASKS) and {c[5].PatternLength for c in cs} == set(m.LENGTHS)
    assert any(c[1].f2Jitter[0] != 0 for c in cs) and any(c[1].f2Jitter[0] == 0 for c in cs)
    assert any(c[3].min() != c[3].max() for c in cs) and any(c[3].min() == c[3].max() for c in cs)
    drawn = {}
    for c in cs:
        col, _ = m.run_one((0, 1), c, 97, 61, False)
        c0, _ = m.initial(97, 61)
        drawn[c[0]] = int((col.view(np.uint32) != c0.view(np.uint32)).any(-1).sum())
    assert all(v == 0 for k, v in drawn.items() if k.endswith("/behind"))
    for box in ("in_view", "crosses_near", "camera_inside", "off_screen", "flat"):
        assert any(v > 0 for k, v in drawn.items() if k.endswith("/" + box)), box
    flat = next(b for b in m.BOXES if b[0] == "flat")
    assert flat[1][2] == flat[2][2]


def test_fixture_is_current_where_the_shader_is_present(built):
    from oracle.refshader import build_bound_box_ref
    build_bound_box_ref.build()
    if not build_bound_box_ref.available():
        pytest.skip("librefshaders_bound_box.so not available")
    m = _gen()
    want, got = np.load(m.OUT), m.run(with_reference=True)
    assert set(got) == set(want.files)
    for k in want.files:
        assert got[k].tobytes() == want[k].tobytes(), f"{k}: regenerate tests/golden/bound_box_reference.npz deliberately"
