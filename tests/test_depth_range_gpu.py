"""The depth range R on the GPU (dfx_pass_depth_range, the dfx_depth_range effect and the C++ DepthRangeCalculator) against the oracle
(oracle/oracle_depth_range.cpp, itself bit-exact against the reference's shaders, tests/test_depth_range_reference.py), bit for bit: on every case of test_depth_range_cpu.cases() in the tight, padded and 128-byte-pitched
layouts, at 3840x2160, written into a device camera, and through the read-back slots."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from diligentfx_b200 import capi
from oracle import oracle_depth_range_py as odr

import gpu_frame
from test_depth_range_cpu import build_driver, cameras, cases

pytestmark = pytest.mark.gpu


def _bits(a) -> list[int]:
    return np.asarray(a, np.float32).view(np.uint32).tolist()


def _pass(pl: gpu_frame.Planes, cam, depth) -> np.ndarray:
    lib = capi.load()
    d = pl.up(depth)
    out = torch.full((4,), float("nan"), dtype=torch.float32, device="cuda")
    capi.check(lib.dfx_pass_depth_range(None, pl.cameras(cam, cam), d.ref, C.c_void_p(out.data_ptr())), "dfx_pass_depth_range")
    return out.cpu().numpy()


def _download(ptr: int) -> np.ndarray:
    lib = capi.load()
    out = np.zeros(4, np.float32)
    p = capi.Plane(ptr, 16, 4, 1, capi.FORMAT_R32F, 0)
    capi.check(lib.dfx_plane_download(None, C.byref(p), out.ctypes.data_as(C.c_void_p), C.c_size_t(0)), "dfx_plane_download")
    capi.check(lib.dfx_stream_synchronize(None), "dfx_stream_synchronize")
    return out


@pytest.mark.parametrize("layout", gpu_frame.LAYOUTS)
def test_pass_matches_oracle(built, layout):
    pl = gpu_frame.Planes(layout)
    lib = capi.load()
    bad = []
    for name, cam, depth in cases():
        n0 = lib.dfx_launch_count()
        got = _pass(pl, cam, depth)
        assert lib.dfx_launch_count() - n0 == 2, name
        want = odr.depth_range(cam, depth)
        if _bits(got) != _bits(want):
            bad.append(f"{name} {depth.shape}: {got} != {want}")
    torch.cuda.synchronize()
    assert pl.padding_damage() == 0
    assert not bad, "\n".join(bad)


def test_pass_matches_oracle_at_4k(built):
    rng = np.random.default_rng(3)
    h, w = 2160, 3840
    d = rng.uniform(0.4, 0.999, (h, w)).astype(np.float32)
    d[rng.random((h, w)) < 0.3] = 1.0
    std, rev, inf = cameras()
    rd = (np.float32(1.0) - d).astype(np.float32)
    spec = d.copy()
    spec[rng.random((h, w)) < 1e-3] = -0.5
    spec[rng.random((h, w)) < 1e-3] = -0.0
    spec[rng.random((h, w)) < 1e-3] = np.nan
    pl = gpu_frame.Planes("aligned")
    for name, cam, depth in (("standard", std, d), ("reversed", rev, rd), ("reversed_infinite", inf, rd), ("specials", std, spec)):
        assert _bits(_pass(pl, cam, depth)) == _bits(odr.depth_range(cam, depth)), name


def test_range_written_into_the_camera(built):
    """out_dev = &cameras_dev[0].fSceneNearZ (HnComputeDepthBoundsTask's CopyBuffer into the frame constants): those 16 bytes hold the
    range and no other byte of either camera changes."""
    lib = capi.load()
    name, cam, depth = cases()[0]
    pl = gpu_frame.Planes("tight")
    cams = pl.cameras(cam, cam)
    off = capi.CameraAttribs.fSceneNearZ.offset
    capi.check(lib.dfx_pass_depth_range(None, cams, pl.up(depth).ref, C.c_void_p(cams.value + off)), "dfx_pass_depth_range")
    got = pl.keep[-1].cpu().numpy().tobytes()
    want = bytearray(bytes(cam) * 2)
    want[off:off + 16] = odr.depth_range(cam, depth).tobytes()
    assert got == bytes(want)


def test_effect_read_back(built):
    lib = capi.load()
    pl = gpu_frame.Planes("padded")
    cs = cases()
    for read_back in (1, 0):
        fx = C.c_void_p()
        capi.check(lib.dfx_depth_range_create(read_back, C.byref(fx)), "dfx_depth_range_create")
        r = capi.SceneDepthRange()
        capi.check(lib.dfx_depth_range_get_range(fx, 1, C.byref(r)), "dfx_depth_range_get_range")
        assert _bits([r.fSceneNearZ, r.fSceneFarZ, r.fSceneNearDepth, r.fSceneFarDepth]) == [0] * 4 and not r
        buf = lib.dfx_depth_range_get_buffer(fx)
        assert _bits(_download(buf)) == [0] * 4
        # nine computes before one synchronise, more than the four initial slots: each compute is read back (a new slot when every
        # slot is in flight), and the range returned is the last one's, whatever order the copies complete in
        for name, cam, depth in cs[:9]:
            capi.check(lib.dfx_depth_range_compute(fx, None, pl.cameras(cam, cam), pl.up(depth).ref), "dfx_depth_range_compute")
        torch.cuda.synchronize()
        device = _download(buf)
        assert _bits(device) == _bits(odr.depth_range(cs[8][1], cs[8][2]))
        capi.check(lib.dfx_depth_range_get_range(fx, 1, C.byref(r)), "dfx_depth_range_get_range")
        host = [r.fSceneNearZ, r.fSceneFarZ, r.fSceneNearDepth, r.fSceneFarDepth]
        assert _bits(host) == (_bits(device) if read_back else [0] * 4), read_back
        if read_back:
            assert bool(r)
        lib.dfx_depth_range_destroy(fx)


def test_cpp_class_matches_the_pass(built, tmp_path):
    exe = build_driver(tmp_path)
    for name, cam, depth in (cases()[1], cases()[11]):
        h, w = depth.shape
        np.ascontiguousarray(depth, np.float32).tofile(tmp_path / "depth.bin")
        (tmp_path / "camera.bin").write_bytes(bytes(cam))
        r = subprocess.run([exe, str(tmp_path), str(w), str(h)], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        want = odr.depth_range(cam, depth)
        assert _bits(np.fromfile(tmp_path / "out_buffer.bin", np.float32)) == _bits(want), name
        assert _bits(np.fromfile(tmp_path / "out_readback.bin", np.float32)) == _bits(want), name


def test_refusals(built):
    lib = capi.load()
    std = cameras()[0]
    pl = gpu_frame.Planes("tight")
    cams = pl.cameras(std, std)
    d = pl.up(np.full((8, 8), 0.5, np.float32))
    rgba = pl.up(np.zeros((8, 8, 4), np.float32))
    out = torch.zeros(8, dtype=torch.float32, device="cuda")
    o = C.c_void_p(out.data_ptr())
    n0 = lib.dfx_launch_count()
    assert lib.dfx_pass_depth_range(None, None, d.ref, o) == capi.DFX_ERR_INVALID_ARG
    assert lib.dfx_pass_depth_range(None, cams, d.ref, None) == capi.DFX_ERR_INVALID_ARG
    assert lib.dfx_pass_depth_range(None, cams, None, o) == capi.DFX_ERR_INVALID_ARG
    assert lib.dfx_pass_depth_range(None, cams, rgba.ref, o) == capi.DFX_ERR_INVALID_ARG
    assert lib.dfx_pass_depth_range(None, cams, d.ref, C.c_void_p(out.data_ptr() + 2)) == capi.DFX_ERR_INVALID_ARG
    assert lib.dfx_depth_range_compute(None, None, cams, d.ref) == capi.DFX_ERR_INVALID_ARG
    assert lib.dfx_launch_count() == n0
    assert (out.cpu().numpy() == 0).all()
