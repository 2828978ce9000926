"""The depth range R without a device: the C-ABI struct against the camera's layout, the C++ drop-in header, and the oracle
(oracle/oracle_depth_range.cpp, the two compute shaders restated group by group) against a second, vectorised restatement here on
every case the GPU test runs, plus the properties the grouping implies: plain min / max for non-negative depths, and a different
answer for negative depths.

`cases()` is shared with tests/test_depth_range_gpu.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from diligentfx_b200 import capi, synth
from oracle import oracle_depth_range_py as odr

ROOT = capi.REPO_ROOT
INC = os.path.join(ROOT, "include")


def cameras():
    """(standard, reversed, reversed with an infinite far plane: depth = near / z, DepthToCameraZ(0) = +inf)."""
    std = synth.generate_sequence(64, 36, 1)[0]["curr_camera"]
    rev = synth._reversed_camera(std)
    inf = capi.CameraAttribs.from_buffer_copy(bytes(rev))
    inf.mProj.m[2][2], inf.mProj.m[3][2], inf.fFarPlaneZ = 0.0, std.fNearPlaneZ, float("inf")
    return std, rev, inf


def _specials(rng, h, w):
    """Negative depths, -0, +0, NaN, +-inf, values above 1 and exact background among ordinary depths."""
    d = rng.uniform(-1.0, 1.5, (h, w)).astype(np.float32)
    pick = rng.integers(0, 10, (h, w))
    for k, v in enumerate((-0.0, 0.0, np.nan, np.inf, -np.inf, 1.0, -1e-30)):
        d[pick == k] = v
    return d


def cases():
    """[(name, camera, depth)]: standard and reversed depth from the synthetic scene, the reversed infinite far plane, all-background
    planes, 1x1 and sizes that are not multiples of 16, and planes of special values where the grouping decides."""
    std, rev, inf = cameras()
    fr = synth.generate_sequence(75, 41, 1)[0]
    d = np.asarray(fr["depth"], np.float32)
    rd = (np.float32(1.0) - d).astype(np.float32)
    rng = np.random.default_rng(11)
    out = [("standard", std, d), ("reversed", rev, rd), ("reversed_infinite", inf, rd),
           ("background_standard", std, np.ones((37, 21), np.float32)), ("background_reversed", rev, np.zeros((16, 16), np.float32)),
           ("1x1", std, np.full((1, 1), 0.25, np.float32)), ("1x1_background", rev, np.zeros((1, 1), np.float32)),
           ("column", std, d[:, 40:41].copy()), ("row", rev, rd[17:18].copy()), ("16x16", std, d[:16, :16].copy())]
    for k, (h, w) in enumerate(((9, 17), (47, 33), (16, 48), (1, 5))):
        out.append((f"specials_{h}x{w}_standard", std, _specials(rng, h, w)))
        out.append((f"specials_{h}x{w}_reversed", rev, _specials(rng, h, w)))
    neg = rng.uniform(-2.0, -0.5, (40, 40)).astype(np.float32)
    out.append(("negative", std, neg))
    return out


# ---- a second restatement, vectorised over the whole dispatch -------------------------------------------------------------------
def _fmin(a, b):
    # the C library's fminf, which the reference's shader runner evaluates HLSL's min with: NaN b -> a, equal (+0 / -0) -> b
    return np.where((a < b) | np.isnan(b), a, b)


def _fmax(a, b):
    return np.where((a > b) | np.isnan(b), a, b)


def _z(d, cam):
    P = cam.mProj.m
    with np.errstate(all="ignore"):
        return (np.float32(P[3][2]) - d * np.float32(P[3][3])) / (d * np.float32(P[2][3]) - np.float32(P[2][2]))


def numpy_depth_range(cam, depth) -> np.ndarray:
    d = np.asarray(depth, np.float32)
    h, w = d.shape
    gx, gy = -(-w // 16), -(-h // 16)
    X, Y = np.arange(gx * 8) * 2, np.arange(gy * 8) * 2
    mn = np.full((gy * 8, gx * 8), 1.0, np.float32)
    mx = np.zeros_like(mn)
    far = np.float32(cam.fFarPlaneDepth)
    for ox, oy in ((0, 0), (0, 1), (1, 0), (1, 1)):
        D = d[np.minimum(Y + oy, h - 1)[:, None], np.minimum(X + ox, w - 1)[None, :]]
        keep = D != far
        mn, mx = np.where(keep, _fmin(mn, D), mn), np.where(keep, _fmax(mx, D), mx)
    own = [a.reshape(gy, 8, gx, 8) for a in (mn, mx)]             # [group y, thread y, group x, thread x]
    held = [a.copy() for a in own]
    for k, f in ((0, _fmin), (1, _fmax)):
        row = own[k][..., 0]
        for i in range(1, 8):
            row = f(row, own[k][..., i])
        grp = row[:, 0]
        for j in range(1, 8):
            grp = f(grp, row[:, j])
        held[k][..., 0] = row
        held[k][:, 0, :, 0] = grp
    lo, hi = held
    zlo, zhi = _z(lo, cam), _z(hi, cam)
    bits = lambda a: np.asarray(a, np.float32).view(np.int32)           # noqa: E731
    seed = np.array([cam.fFarPlaneZ, cam.fNearPlaneZ, cam.fFarPlaneDepth, cam.fNearPlaneDepth], np.float32).view(np.int32)
    r = seed.copy()
    if cam.fNearPlaneDepth <= cam.fFarPlaneDepth:
        r[0], r[1] = min(r[0], bits(zlo).min()), max(r[1], bits(zhi).max())
        r[2], r[3] = min(r[2], bits(lo).min()), max(r[3], bits(hi).max())
    else:
        r[0], r[1] = min(r[0], bits(zhi).min()), max(r[1], bits(zlo).max())
        r[3], r[2] = min(r[3], bits(lo).min()), max(r[2], bits(hi).max())
    return r.view(np.float32)


@pytest.mark.parametrize("case", range(len(cases())))
def test_oracle_matches_the_vectorised_restatement(case):
    name, cam, depth = cases()[case]
    got, want = odr.depth_range(cam, depth), numpy_depth_range(cam, depth)
    assert got.view(np.uint32).tolist() == want.view(np.uint32).tolist(), (name, got, want)


def test_non_negative_depths_give_the_plain_min_and_max():
    std, rev, _ = cameras()
    rng = np.random.default_rng(5)
    d = rng.uniform(0.3, 1.0, (53, 70)).astype(np.float32)
    d[rng.random(d.shape) < 0.2] = 1.0                                   # background
    r = odr.depth_range(std, d)
    fg = d[d != 1.0]
    assert r[2] == fg.min() and r[3] == fg.max()
    assert r[0] == _z(fg.min(), std) and r[1] == _z(fg.max(), std)
    rd = (np.float32(1.0) - d).astype(np.float32)
    r = odr.depth_range(rev, rd)
    fg = rd[rd != 0.0]
    assert r[3] == fg.min() and r[2] == fg.max()                         # reversed: the near depth is the largest
    assert r[0] == _z(fg.max(), rev) and r[1] == _z(fg.min(), rev)


def test_background_only_leaves_the_cleared_range():
    for cam, bg in zip(cameras()[:2], (1.0, 0.0)):
        r = odr.depth_range(cam, np.full((20, 35), bg, np.float32))
        assert r[2:].tolist() == [cam.fFarPlaneDepth, cam.fNearPlaneDepth]


def test_negative_depths_depend_on_the_grouping():
    """Integer min of negative floats picks the one closest to -0, while each partial is the float minimum of its pixels: in one
    2x2 block holding -1 and -2, the partial is -2 and no thread issues -1 or -2 alone."""
    std = cameras()[0]
    d = np.full((2, 2), 0.5, np.float32)
    d[0, 0], d[1, 1] = -1.0, -2.0
    assert odr.depth_range(std, d)[2] == -2.0
    d = np.full((16, 32), 0.5, np.float32)
    d[0, 0], d[0, 16] = -1.0, -2.0                                       # two groups: each issues its own partial
    assert odr.depth_range(std, d)[2] == -1.0


def test_scene_depth_range_struct_is_the_camera_slice():
    assert ctypes.sizeof(capi.SceneDepthRange) == 16
    cam = capi.CameraAttribs
    names = ("fSceneNearZ", "fSceneFarZ", "fSceneNearDepth", "fSceneFarDepth")
    base = getattr(cam, names[0]).offset
    for k, n in enumerate(names):
        assert getattr(cam, n).offset == base + 4 * k and getattr(capi.SceneDepthRange, n).offset == 4 * k
    assert not capi.SceneDepthRange() and capi.SceneDepthRange(1.0, 2.0, 0.5, 0.9)


def test_header_is_self_contained():
    src = '#include "dfx/DepthRangeCalculator.hpp"\nint main() { return 0; }\n'
    r = subprocess.run(["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-x", "c++", "-", "-I", INC], input=src.encode(), capture_output=True)
    assert r.returncode == 0, r.stderr.decode()


def build_driver(out_dir) -> str:
    """Compiles tests/cpp/depth_range_driver.cpp into `out_dir` (the repository tree may be read-only)."""
    exe = os.path.join(str(out_dir), "depth_range_driver")
    libdir = os.path.dirname(capi.LIB_PATH)
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", os.path.join(ROOT, "tests", "cpp", "depth_range_driver.cpp"), "-I", INC, "-L", libdir,
                        "-ldfx_b200", f"-Wl,-rpath,{libdir}", "-Wl,--allow-shlib-undefined", "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_driver_links_against_the_c_abi_only(built, tmp_path):
    exe = build_driver(tmp_path)
    needed = subprocess.check_output(["objdump", "-p", exe]).decode()
    assert "libdfx_b200.so" in needed
    assert "libcudart" not in "".join(l for l in needed.splitlines() if "NEEDED" in l)
