"""Cost of the IBL cube-map precomputation on the GPU at Hydrogent's defaults: the 64^2 irradiance cube with 8192 samples and the 256^2
prefiltered map with 9 levels and 256 samples, RGBA16F outputs, from an RGBA16F 1024^2 cube with 11 levels and from an RGBA16F 2048 x 1024
sphere with 12 levels. Each pass is timed with CUDA events over repeated launches after a warm-up, and reported with its samples per
second (output texels x samples, each sample one trilinear read of up to 8 bilinear taps). The card's name, power limit and SM clock are
read in the same run.

    python tools/ibl_cost.py [--out profiles/h100_ibl_cost.json] [--reps 10]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import ibl_cases as IC  # noqa: E402
from diligentfx_b200 import capi  # noqa: E402


def _card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, sm, sm_max = [v.strip() for v in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def _time(fn, reps: int) -> float:
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_ibl_cost.json"))
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    lib = capi.load()
    irr = torch.empty((384, 64, 4), dtype=torch.float16, device="cuda")
    pre = [torch.empty((6 * (256 >> m), 256 >> m, 4), dtype=torch.float16, device="cuda") for m in range(9)]
    irr_p = capi.plane_of(irr)
    pre_p = (capi.Plane * 9)(*[capi.plane_of(t) for t in pre])
    irr_samples = 6 * 64 * 64 * 8192
    pre_samples = sum(6 * (256 >> m) ** 2 for m in range(9)) * 256
    res = {"card": _card(), "outputs": "RGBA16F", "irradiance": "64^2 x 6, 8192 samples", "prefiltered": "256^2 x 6, 9 levels, 256 samples", "sources": {}}
    for name, env_type, lv in (("cube 1024^2, 11 levels", 0, IC.cube_chain(1024, 11)), ("sphere 2048x1024, 12 levels", 1, IC.sphere_chain(2048, 1024, 12))):
        dev = [torch.from_numpy(l).cuda().half() for l in lv]
        src = (capi.Plane * len(dev))(*[capi.plane_of(t) for t in dev])
        t_irr = _time(lambda: capi.check(lib.dfx_pass_irradiance_cube(None, env_type, src, len(dev), C.c_uint32(0), 1, C.byref(irr_p))), args.reps)
        t_pre = _time(lambda: capi.check(lib.dfx_pass_prefilter_env_map(None, env_type, src, len(dev), C.c_uint32(0), 1, pre_p, 9)), args.reps)
        res["sources"][name] = {"irradiance_ms": round(t_irr, 3), "irradiance_gsamples_per_s": round(irr_samples / t_irr / 1e6, 2),
                                "prefilter_ms": round(t_pre, 3), "prefilter_gsamples_per_s": round(pre_samples / t_pre / 1e6, 2)}
    res["card_after"] = _card()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    line = json.dumps(res)
    with open(args.out, "w") as f:
        f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
