"""The C++ drop-in layer (include/dfx/*.hpp): header self-containment like the reference's Tests/IncludeTest (one TU per public
header, compile only — CPU), and an end-to-end run of tests/cpp/chain_driver.cpp against the oracle (GPU)."""
import os
import subprocess

import numpy as np
import pytest

from diligentfx_b200 import capi, synth

ROOT = capi.REPO_ROOT
INC = os.path.join(ROOT, "include")


@pytest.mark.parametrize("header", ["dfx/DiligentShim.hpp", "dfx/GBuffer.hpp", "dfx/PostFXContext.hpp", "dfx/PostProcessEffects.hpp", "dfx_b200.h"])
def test_header_is_self_contained(header):
    src = f'#include "{header}"\nint main() {{ return 0; }}\n'
    r = subprocess.run(["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-x", "c++", "-", "-I", INC], input=src.encode(), capture_output=True)
    assert r.returncode == 0, r.stderr.decode()


def build_driver(built, out_dir) -> str:
    """Compiles tests/cpp/chain_driver.cpp into `out_dir` (a per-test temporary directory: the repository tree may be read-only)."""
    exe = os.path.join(str(out_dir), "chain_driver")
    libdir = os.path.dirname(capi.LIB_PATH)
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", os.path.join(ROOT, "tests", "cpp", "chain_driver.cpp"), "-I", INC, "-L", libdir, "-ldfx_b200",
           f"-Wl,-rpath,{libdir}", "-Wl,--allow-shlib-undefined", "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_driver_links_against_the_c_abi_only(built, tmp_path):
    exe = build_driver(built, tmp_path)
    needed = subprocess.check_output(["objdump", "-p", exe]).decode()
    assert "libdfx_b200.so" in needed
    assert "libcudart" not in "".join(l for l in needed.splitlines() if "NEEDED" in l), "user code must not need CUDA itself"


@pytest.mark.gpu
def test_cpp_chain_matches_oracle(built, tmp_path):
    from oracle import oracle_py as op
    exe = build_driver(built, tmp_path)
    w, h, n = 288, 162, 3
    seq = synth.generate_sequence(w, h, n)
    o = op.Oracle(w, h)
    for k, fr in enumerate(seq):
        for name in ("depth", "prev_depth", "motion", "normal", "color", "material"):
            np.ascontiguousarray(fr[name], np.float32).tofile(tmp_path / f"f{k}_{name}.bin")
        with open(tmp_path / f"f{k}_cameras.bin", "wb") as f:
            f.write(bytes(fr["curr_camera"]) + bytes(fr["prev_camera"]))
        o.set_inputs(fr)
        o.frame()
    r = subprocess.run([exe, str(tmp_path), str(w), str(h), str(n)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    print(r.stdout.strip())
    ldr = np.fromfile(tmp_path / "out_ldr.bin", np.float32).reshape(h, w, 4)
    ao = np.fromfile(tmp_path / "out_ao.bin", np.float32).reshape(h, w)
    want = o.get("ldr")
    mse = float(np.mean((np.clip(ldr[..., :3], 0, 1).astype(np.float64) - np.clip(want[..., :3], 0, 1)) ** 2))
    p = 200.0 if mse == 0 else 10 * np.log10(1.0 / mse)
    print(f"C++ drop-in chain vs oracle: LDR PSNR {p:.2f} dB")
    assert p >= 49.0
    assert float(np.mean((ao - o.get("ssao_out")) ** 2)) < 1e-5
