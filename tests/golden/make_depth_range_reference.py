#!/usr/bin/env python3
"""Regenerates tests/golden/depth_range_reference.npz: what the REFERENCE'S OWN ClearDepthRange.csh and ComputeDepthRange.csh produce
(compiled for the CPU with a group runner by oracle/refshader/build_depth_range_ref.py; the reference's shaders must be mounted) on
every case of tests/test_depth_range_cpu.cases(). tests/test_depth_range_reference.py holds the oracle (oracle_depth_range.cpp) to
them bit for bit. Every entry is the DepthRangeI buffer as four uint32: iSceneNearZ, iSceneFarZ, iSceneNearDepth, iSceneFarDepth.

    python tests/golden/make_depth_range_reference.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
OUT = os.path.join(HERE, "depth_range_reference.npz")


def run(with_reference: bool) -> dict[str, np.ndarray]:
    """{case name: four uint32} from the reference's shaders (with_reference) or from the oracle."""
    from test_depth_range_cpu import cases
    if with_reference:
        from oracle.refshader import build_depth_range_ref as R
        fn = R.depth_range
    else:
        from oracle import oracle_depth_range_py as odr
        fn = odr.depth_range
    return {name: np.asarray(fn(cam, depth), np.float32).view(np.uint32) for name, cam, depth in cases()}


if __name__ == "__main__":
    from oracle.refshader import build_depth_range_ref
    build_depth_range_ref.build()
    assert build_depth_range_ref.available(), "the reference's shaders are not mounted"
    np.savez_compressed(OUT, **run(with_reference=True))
    print(OUT)
