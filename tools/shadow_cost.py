"""Cost of ConvertToFilterable on the GPU: 4 cascades of 2048^2 D16 depth to VSM 16-bit, EVSM2 32-bit and EVSM4 32-bit, at the reference's
3 x 3 default and at a varying filter of range 5. Each case is timed with CUDA events over repeated launches after a warm-up, on the
fused path (what dfx_shadow_convert_to_filterable runs at these ranges) and on the two-pass path (reached through the tests' hook of
csrc/dfx_testing.h), alternated in rounds on the same inputs; the median round is reported. Compulsory bytes are the depth read once
and the filterable map written once; their share of the HBM bound is against the H100 SXM's 3.35 TB/s. The card's name, power limit
and SM clock are read in the same run.

    python tools/shadow_cost.py [--out profiles/h100_shadow_cost.json] [--reps 200] [--rounds 5]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from diligentfx_b200 import capi, shadow, synth  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
N, S = 4, 2048


def _attribs(is32: bool, fixed: int, radius: float = 0.0) -> capi.ShadowMapAttribs:
    """ShadowMapAttribs' defaults for N cascades; fixed 0 = the varying filter at `radius` on both axes (fFilterWorldSize 1:
    r = scale * 0.5 / 2 * S)."""
    a = capi.ShadowMapAttribs.default()
    a.iNumCascades, a.fNumCascades, a.bIs32BitEVSM, a.iFixedFilterSize = N, float(N), int(is32), fixed
    if fixed <= 0:
        a.fFilterWorldSize = 1.0
        for i in range(N):
            a.Cascades[i].f4LightSpaceScale[0] = a.Cascades[i].f4LightSpaceScale[1] = 4.0 * radius / S
    return a


def _card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, sm, sm_max = [v.strip() for v in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def _time(fn, reps: int) -> float:
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_shadow_cost.json"))
    ap.add_argument("--reps", type=int, default=200)   # 50-160 ms per timed window
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    lib = capi.load()
    depth = torch.from_numpy(synth.shadow_cascades(N, S, S, seed=1, d16=True).view(np.int16)).cuda()
    src = (capi.Plane * N)(*[capi.Plane(depth[i].data_ptr(), 2 * S, S, S, capi.FORMAT_R16U, 0) for i in range(N)])
    filters = {"3x3 default": dict(fixed=3), "varying, range 5": dict(fixed=0, radius=5.0)}
    res = {"card": _card(), "workload": f"{N} cascades of {S}^2, D16 depth", "hbm_bytes_per_s": HBM_BYTES_PER_S, "cases": {}}
    for mode, is32, label in [(capi.SHADOW_MODE_VSM, False, "VSM 16-bit"), (capi.SHADOW_MODE_EVSM2, True, "EVSM2 32-bit"),
                              (capi.SHADOW_MODE_EVSM4, True, "EVSM4 32-bit")]:
        fmt, ch, dt = shadow.filterable_format(mode, is32)
        esz = torch.tensor([], dtype=dt).element_size()
        out = torch.empty((N, S, S, ch), dtype=dt, device="cuda")
        inter = torch.empty((S, S, ch), dtype=dt, device="cuda")
        dst = (capi.Plane * N)(*[capi.Plane(out[i].data_ptr(), S * ch * esz, S, S, fmt, 0) for i in range(N)])
        ip = capi.Plane(inter.data_ptr(), S * ch * esz, S, S, fmt, 0)
        for fname, kw in filters.items():
            a = _attribs(is32, **kw)
            assert {int(np.floor(np.float32(r) + np.float32(0.5))) for i in range(N) for r in shadow.filter_radii(a, i, S, S)} <= {1, 5}
            fused = lambda: capi.check(lib.dfx_shadow_convert_to_filterable(None, mode, C.byref(a), src, N, dst, None))  # noqa: E731
            two = lambda: capi.check(lib.dfx_testing_shadow_convert_two_pass(None, mode, C.byref(a), src, N, dst, C.byref(ip)))  # noqa: E731
            fused(), two()
            torch.cuda.synchronize()
            tf, tt = [], []
            for _ in range(args.rounds):
                tf.append(_time(fused, args.reps))
                tt.append(_time(two, args.reps))
            t_f, t_t = statistics.median(tf), statistics.median(tt)
            compulsory = N * S * S * (2 + ch * esz)
            res["cases"][f"{label}, {fname}"] = {
                "fused_ms": round(t_f, 4), "two_pass_ms": round(t_t, 4), "fused_rounds_ms": [round(t, 4) for t in tf],
                "two_pass_rounds_ms": [round(t, 4) for t in tt], "compulsory_mb": round(compulsory / 1e6, 1),
                "fused_share_of_hbm_bound": round(compulsory / HBM_BYTES_PER_S / (t_f * 1e-3), 3),
                "two_pass_share_of_hbm_bound": round(compulsory / HBM_BYTES_PER_S / (t_t * 1e-3), 3)}
    res["card_after"] = _card()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    line = json.dumps(res)
    with open(args.out, "w") as f:
        f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
