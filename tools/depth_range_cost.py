#!/usr/bin/env python3
"""What R (dfx_pass_depth_range, both launches) costs on the GPU: one JSON line with the time per call, CUDA events around `--iters`
calls after a warm-up, on a depth plane of the synthetic scene's depth range with 30 % background, and the bound its 4 B/px imply at
3.35 TB/s (the H100 SXM data-sheet figure), with the card's name, power limit and maximum SM clock read in the same run. Repeated
`--runs` times; the median and the spread are printed.

    python tools/depth_range_cost.py [--width 3840 --height 2160 --runs 5 --iters 200]
"""
import argparse
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from diligentfx_b200 import capi, synth  # noqa: E402
from tools.grid_cost import HBM_BYTES_PER_S, gpu_info, time_ms  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--iters", type=int, default=200)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device: there is no CPU path"
    lib = capi.load()
    w, h = a.width, a.height
    cam = synth.generate_sequence(64, 36, 1)[0]["curr_camera"]
    rng = np.random.default_rng(1)
    d = rng.uniform(0.4, 0.999, (h, w)).astype(np.float32)
    d[rng.random((h, w)) < 0.3] = 1.0
    depth = torch.from_numpy(d).cuda()
    cams = torch.frombuffer(bytearray(bytes(cam) * 2), dtype=torch.uint8).cuda()
    out = torch.zeros(4, dtype=torch.float32, device="cuda")
    plane = capi.plane_of(depth)
    cp, op = C.c_void_p(cams.data_ptr()), C.c_void_p(out.data_ptr())

    def call():
        capi.check(lib.dfx_pass_depth_range(None, cp, C.byref(plane), op), "dfx_pass_depth_range")

    time_ms(call, 20)
    runs = sorted(time_ms(call, a.iters) for _ in range(a.runs))
    ms = runs[len(runs) // 2]
    bound_ms = 4.0 * w * h / HBM_BYTES_PER_S * 1e3
    print(json.dumps({"what": "R, dfx_pass_depth_range (clear + reduction)", "width": w, "height": h, "ms": round(ms, 5),
                      "runs_ms": [round(r, 5) for r in runs], "alg_bytes_per_px": 4, "hbm_bound_ms": round(bound_ms, 5),
                      "frac_of_hbm_bound": round(bound_ms / ms, 4), **gpu_info()}))


if __name__ == "__main__":
    main()
