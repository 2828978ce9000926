#!/usr/bin/env python3
"""What the selected prim's bounding box (B) costs on the GPU: one JSON line.

  * B (dfx_pass_bound_box, motion vectors on) at 4K on the benchmark scene's frame, for a box that fills the screen (3 to 6 units
    ahead of the camera, its front face nearly the frame: its edges run across the whole screen) and for a small one (sphere 3 of the
    scene);
  * the 4K chain frame with B off and on (the small box), timed in the same process on alternating runs (CUDA events around
    `--frames` steady-state frames per run, after a warm-up that records both sets of graphs).

Each pass time is printed next to its algorithmic bytes (per covered pixel: 4 B of depth read, 16 B of colour and 8 B of motion
written; the covered pixels are counted by the oracle's rasteriser) and the HBM bound those bytes imply at 3.35 TB/s (the H100 SXM
data-sheet figure), with the card's name, power limit and maximum SM clock read in the same run.

    python tools/bound_box_cost.py [--width 3840 --height 2160 --runs 6 --frames 30 --iters 200]
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
from diligentfx_b200.chain import PostProcessChain  # noqa: E402
from tools.grid_cost import HBM_BYTES_PER_S, gpu_info, time_ms  # noqa: E402

SPHERE = 3


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--runs", type=int, default=6, help="runs per setting, alternating")
    ap.add_argument("--frames", type=int, default=30, help="timed frames per run")
    ap.add_argument("--iters", type=int, default=200, help="timed calls per pass")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bound_box_cost.py measures on the GPU: no CUDA device")
    from oracle import oracle_bound_box_py as ob
    w, h = a.width, a.height
    fr = synth.generate_sequence(w, h, 1)[0]
    cam = fr["curr_camera"]
    small = synth.sphere_bound_box(SPHERE)
    # a box 3..6 units ahead whose front face nearly fills the frame (view space, taken to the world by the camera's mViewInv as
    # Hydrogent's prim transform): its edges run across the whole screen
    view_inv = np.array([[cam.mViewInv.m[r][k] for k in range(4)] for r in range(4)], np.float32)
    full = synth.bound_box_transform([-2.9, -1.6, 3.0], [2.9, 1.6, 6.0], view_inv)

    chain = PostProcessChain(w, h)
    chain.upload(fr, non_blocking=False)
    idx = [0]

    def frame():
        chain.execute(idx[0], cam, cam)
        idx[0] += 1

    times = {"off": [], "on": []}
    for on in (False, True, False, True):  # warm-up: both graph sets recorded
        chain.set_bound_box(small if on else None)
        for _ in range(3):
            frame()
    for r in range(2 * a.runs):
        on = r % 2 == 1
        chain.set_bound_box(small if on else None)
        for _ in range(2):
            frame()
        times["on" if on else "off"].append(time_ms(frame, a.frames))
    chain.close()

    lib = capi.load()
    cams = torch.frombuffer(bytearray(bytes(cam) * 2), dtype=torch.uint8).cuda()
    cp = C.c_void_p(cams.data_ptr())
    depth = torch.from_numpy(np.ascontiguousarray(fr["depth"])).cuda()
    color = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
    motion = torch.zeros((h, w, 2), dtype=torch.float32, device="cuda")
    pd, pc, pm = capi.plane_of(depth), capi.plane_of(color), capi.plane_of(motion)
    rows = capi.Rows(0, h)
    passes = {}
    for name, transform in (("B_full_screen_box", full), ("B_small_box", small)):
        attribs = ob.chain_attribs(transform)
        covered = sum(len(r[0]) for r in (ob.raster(v0, v1, w, h) for v0, v1 in _lines(ob.vertices(cam, cam, attribs))) if r is not None)
        fn = lambda: capi.check(lib.dfx_pass_bound_box(None, cp, C.byref(attribs), C.c_uint32(capi.BOUND_BOX_OPTION_COMPUTE_MOTION_VECTORS),  # noqa: E731
                                                       C.byref(pd), C.byref(pc), C.byref(pm), rows))
        for _ in range(5):
            fn()
        ms = min(time_ms(fn, a.iters) for _ in range(3))
        nbytes = covered * (4 + 16 + 8)
        bound_ms = nbytes / HBM_BYTES_PER_S * 1e3
        passes[name] = {"ms": round(ms, 5), "covered_pixels": int(covered), "bytes": int(nbytes), "hbm_bound_ms": round(bound_ms, 6)}
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    print(json.dumps({"size": f"{w}x{h}", **gpu_info(), "chain_ms_box_off": round(med(times["off"]), 4), "chain_ms_box_on": round(med(times["on"]), 4),
                      "chain_ms_box_off_runs": [round(t, 4) for t in times["off"]], "chain_ms_box_on_runs": [round(t, 4) for t in times["on"]],
                      "passes": passes}))


def _lines(verts):
    return [(verts[2 * l, 0], verts[2 * l + 1, 0]) for l in range(12)]


if __name__ == "__main__":
    main()
