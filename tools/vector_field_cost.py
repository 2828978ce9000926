#!/usr/bin/env python3
"""What the vector field overlay (the motion-vector view) costs on the GPU: one JSON line, written to
profiles/h100_vector_field_cost.json with --out.

  * dfx_pass_vector_field at 4K with HnPostProcessTask's attribs (a 192 x 108 grid, elapsed 1/60 s) over an RGBA32F target, for the
    Hydrogent-typical field (a camera pan at 60 fps: every vector a few pixels long) and a pathological one (every vector points through
    the frame's centre to the other side: every line crosses the frame, and they all cross each other);
  * the chain's motion-vector frame against its SHADED frame with TAA off, timed in the same process on alternating runs (CUDA events
    around `--frames` steady-state frames per run, after a warm-up that records both graphs).

Each pass time is printed next to the fragments drawn (counted by the oracle's rasteriser), the pixels written, the algorithmic bytes
(every fragment reads and updates its owner word in the mark launch and reads it in the resolve launch, 12 B; every written pixel
clears it and stores 16 B of colour) and the HBM bound those bytes imply at 3.35 TB/s (the H100 SXM data-sheet figure), with the
card's name, power limit and maximum SM clock read in the same run.

    python tools/vector_field_cost.py [--width 3840 --height 2160 --runs 6 --frames 30 --iters 100] [--out FILE]
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
from diligentfx_b200.chain import ChainConfig, PostProcessChain  # noqa: E402
from tools.grid_cost import HBM_BYTES_PER_S, gpu_info, time_ms  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--runs", type=int, default=6, help="runs per setting, alternating")
    ap.add_argument("--frames", type=int, default=30, help="timed frames per run")
    ap.add_argument("--iters", type=int, default=100, help="timed calls per pass")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vector_field_cost.py measures on the GPU: no CUDA device")
    from oracle import oracle_vector_field_py as ov
    w, h, elapsed = a.width, a.height, 1.0 / 60.0
    fr = synth.generate_sequence(w, h, 1)[0]
    cam = fr["curr_camera"]

    chain = PostProcessChain(w, h, ChainConfig(enable_taa=False))
    chain.upload(fr, non_blocking=False)
    idx = [0]

    def frame():
        chain.execute(idx[0], cam, cam)
        idx[0] += 1

    times = {"shaded": [], "motion_vectors": []}
    for on in (False, True, False, True):  # warm-up: both graphs recorded
        chain.set_motion_vector_view(elapsed if on else None)
        for _ in range(3):
            frame()
    for r in range(2 * a.runs):
        on = r % 2 == 1
        chain.set_motion_vector_view(elapsed if on else None)
        for _ in range(2):
            frame()
        times["motion_vectors" if on else "shaded"].append(time_ms(frame, a.frames))
    chain.close()

    lib = capi.load()
    attribs = ov.hydrogent_attribs(w, h, elapsed)
    color = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
    scratch = torch.zeros((h, w), dtype=torch.float32, device="cuda")
    pc, ps = capi.plane_of(color), capi.plane_of(scratch)
    rows = capi.Rows(0, h)
    passes = {}
    X, Y = np.meshgrid((np.arange(w) + 0.5) / w * 2 - 1, 1 - (np.arange(h) + 0.5) / h * 2)
    crossing = np.stack([1.4 * X, 1.4 * Y], -1).astype(np.float32)  # scaled by -1.2: each end at -0.68 x its start, past the centre
    for name, field in (("pan_60fps", synth.motion_pan(w, h)), ("every_line_crosses_the_frame", crossing)):
        f = torch.from_numpy(field).cuda()
        pf = capi.plane_of(f)
        blank = np.zeros((h, w, 4), np.float32)
        drawn, fragments = ov.vector_field(attribs, 0, field, blank, count=True)
        written = int((drawn != 0).any(-1).sum())
        color.zero_()
        fn = lambda: capi.check(lib.dfx_pass_vector_field(None, C.byref(attribs), C.c_uint32(0), C.byref(pf), C.byref(pc), C.byref(ps), rows))  # noqa: E731
        for _ in range(5):
            fn()
        ms = min(time_ms(fn, a.iters) for _ in range(3))
        torch.cuda.synchronize()
        assert not scratch.any().item() and color.cpu().numpy().tobytes() == drawn.tobytes(), name
        nbytes = fragments * 12 + written * (4 + 16)
        passes[name] = {"ms": round(ms, 5), "lines": int(attribs.GridSize[0] * attribs.GridSize[1]), "fragments": int(fragments),
                        "written_pixels": written, "bytes": int(nbytes), "hbm_bound_ms": round(nbytes / HBM_BYTES_PER_S * 1e3, 6)}
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    line = json.dumps({"size": f"{w}x{h}", **gpu_info(), "elapsed": elapsed,
                       "chain_ms_shaded_taa_off": round(med(times["shaded"]), 4), "chain_ms_motion_vectors": round(med(times["motion_vectors"]), 4),
                       "chain_ms_shaded_taa_off_runs": [round(t, 4) for t in times["shaded"]],
                       "chain_ms_motion_vectors_runs": [round(t, 4) for t in times["motion_vectors"]], "passes": passes})
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
