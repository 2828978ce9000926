"""Seeded synthetic G-buffer generator (SURVEY.md §8d "Synthetic G-buffer").

Produces, for a sequence of frames, the inputs the reference chain consumes
(Hydrogent/src/Tasks/HnPostProcessTask.cpp:776-832): depth, normal, colour, material, motion vectors, previous depth
and the curr/prev `CameraAttribs`. The scene is an analytic ray-cast (ground plane + K seeded spheres + sky), so any
resolution can be generated and depth / normals / motion are mutually consistent with the cameras:

* camera: LH perspective, fovY 60 deg, near 0.1, far 100 (D3D convention, row-vector matrices), translated a little
  every frame; the projection is jittered exactly like the reference does it
  (TemporalAntiAliasing::GetJitteredProjMatrix, TemporalAntiAliasing.hpp:138-156; Hydrogent/src/HnCamera.cpp:124-139;
  camera block filled like Hydrogent/src/Tasks/HnBeginFrameTask.cpp:490-515: mProj/mViewProj are the jittered ones).
* motion = (NDC_curr - jitter_curr) - (NDC_prev - jitter_prev)  (Shaders/Common/public/ShaderUtilities.fxh:88-91).
* depth 1.0 = background (sky); colour is HDR with log-uniform highlights so the Bloom threshold and the TAA
  clipping are exercised; material.x = roughness from {0, 0.05, 0.15, 0.3, 0.6} so about half the pixels pass
  the SSR roughness threshold.

Everything is numpy on the host (it feeds both the CUDA path and the CPU oracle with identical bits).
"""
from __future__ import annotations

import ctypes
import math
import os
from dataclasses import dataclass, field

import numpy as np

from .capi import CameraAttribs

NEAR, FAR, FOVY = 0.1, 100.0, math.radians(60.0)
PITCH = math.radians(18.0)


def halton(base: int, index: int) -> float:
    """TemporalAntiAliasing.cpp:43-54 (host-side float32 arithmetic)."""
    result = np.float32(0.0)
    f = np.float32(1.0)
    while index > 0:
        f = np.float32(f / np.float32(base))
        result = np.float32(result + f * np.float32(index % base))
        index = int(math.floor(np.float32(index) / np.float32(base)))
    return float(result)


def taa_jitter(frame: int, width: int, height: int) -> tuple[float, float]:
    """TemporalAntiAliasing::GetJitterOffset, TemporalAntiAliasing.cpp:63-78."""
    jx = np.float32(np.float32(halton(2, (frame % 16) + 1)) - np.float32(0.5)) / np.float32(np.float32(0.5) * np.float32(width))
    jy = np.float32(np.float32(halton(3, (frame % 16) + 1)) - np.float32(0.5)) / np.float32(np.float32(0.5) * np.float32(height))
    return float(jx), float(jy)


def _proj(width: int, height: int, jitter: tuple[float, float]) -> np.ndarray:
    aspect = width / height
    t = math.tan(FOVY / 2)
    m = np.zeros((4, 4), np.float64)
    m[0, 0] = 1.0 / (aspect * t)
    m[1, 1] = 1.0 / t
    m[2, 2] = FAR / (FAR - NEAR)
    m[2, 3] = 1.0
    m[3, 2] = -NEAR * FAR / (FAR - NEAR)
    # GetJitteredProjMatrix: perspective -> m20 += jx, m21 += jy
    m[2, 0] += jitter[0]
    m[2, 1] += jitter[1]
    return m


def _view(pos: np.ndarray, yaw: float) -> tuple[np.ndarray, np.ndarray]:
    """Returns (view, world) row-vector matrices for a camera at `pos` rotated by `yaw` about +y."""
    c, s = math.cos(yaw), math.sin(yaw)
    cp, sp = math.cos(PITCH), math.sin(PITCH)
    yaw_m = np.array([[c, 0, -s, 0], [0, 1, 0, 0], [s, 0, c, 0], [0, 0, 0, 1]], np.float64)
    pitch_m = np.array([[1, 0, 0, 0], [0, cp, sp, 0], [0, -sp, cp, 0], [0, 0, 0, 1]], np.float64)  # look down by PITCH
    rot = pitch_m @ yaw_m                                                                        # camera->world rotation rows
    world = rot.copy()
    world[3, :3] = pos
    view = np.linalg.inv(world)
    return view, world


@dataclass
class CameraState:
    view: np.ndarray
    world: np.ndarray
    proj: np.ndarray
    jitter: tuple[float, float]
    pos: np.ndarray
    attribs: CameraAttribs = field(default=None)


def make_camera(frame: int, width: int, height: int, use_jitter: bool = True) -> CameraState:
    pos = np.array([0.004 * frame, 0.15 + 0.001 * frame, -0.002 * frame], np.float64)
    yaw = 0.0004 * frame
    jitter = taa_jitter(frame, width, height) if use_jitter else (0.0, 0.0)
    view, world = _view(pos, yaw)
    proj = _proj(width, height, jitter)
    vp = view @ proj
    cam = CameraAttribs()
    cam.f4Position[:] = [pos[0], pos[1], pos[2], 1.0]
    cam.f4ViewportSize[:] = [float(width), float(height), float(np.float32(1.0) / np.float32(width)), float(np.float32(1.0) / np.float32(height))]
    # SetClipPlanes(0.1, 100) — BasicStructures.fxh:134-147
    cam.fNearPlaneZ, cam.fFarPlaneZ, cam.fNearPlaneDepth, cam.fFarPlaneDepth = NEAR, FAR, 0.0, 1.0
    cam.fSceneNearZ, cam.fSceneFarZ, cam.fSceneNearDepth, cam.fSceneFarDepth = NEAR, FAR, 0.0, 1.0
    cam.fHandness = 1.0 if np.linalg.det(view) > 0 else -1.0
    cam.uiFrameIndex = frame
    cam.fFocusDistance, cam.fFStop, cam.fFocalLength, cam.fSensorWidth = 10.0, 5.6, 50.0, 36.0
    cam.fSensorHeight, cam.fExposure = 24.0, 0.0
    cam.f2Jitter[:] = [jitter[0], jitter[1]]

    def put(dst, m):
        m32 = np.asarray(m, np.float32)
        for r in range(4):
            for c in range(4):
                dst.m[r][c] = float(m32[r, c])

    put(cam.mView, view), put(cam.mProj, proj), put(cam.mViewProj, vp)
    put(cam.mViewInv, world), put(cam.mProjInv, np.linalg.inv(proj)), put(cam.mViewProjInv, np.linalg.inv(vp))
    return CameraState(view, world, proj, jitter, pos, cam)


@dataclass
class Scene:
    centers: np.ndarray    # (K,3)
    radii: np.ndarray      # (K,)
    albedo: np.ndarray     # (K+1,3)   last = ground
    rough: np.ndarray      # (K+1,)
    emissive: np.ndarray   # (K+1,)


def make_scene(seed: int = 7, k: int = 24) -> Scene:
    rng = np.random.default_rng(seed)
    z = rng.uniform(3.0, 28.0, k)
    x = rng.uniform(-0.55, 0.55, k) * z * 1.6
    r = rng.uniform(0.35, 1.4, k)
    y = -1.0 + r * rng.uniform(0.6, 1.3, k)
    centers = np.stack([x, y, z], 1)
    albedo = rng.uniform(0.15, 0.95, (k + 1, 3))
    albedo[-1] = [0.55, 0.55, 0.6]
    rough_set = np.array([0.0, 0.05, 0.15, 0.3, 0.6])
    rough = rough_set[rng.integers(0, 5, k + 1)]
    rough[-1] = 0.12
    emissive = np.where(rng.uniform(size=k + 1) < 0.2, np.exp2(rng.uniform(2.0, 6.0, k + 1)), 0.0)
    emissive[-1] = 0.0
    return Scene(centers, r, albedo, rough, emissive)


def _raycast(scene: Scene, cam: CameraState, width: int, height: int, rows: slice):
    """Ray-cast rows `rows` of the frame. Returns dict of per-pixel arrays (float64)."""
    ys = np.arange(rows.start, rows.stop, dtype=np.float64)
    xs = np.arange(width, dtype=np.float64)
    ndc_x = (2.0 * (xs + 0.5) / width - 1.0)[None, :]
    ndc_y = (1.0 - 2.0 * (ys + 0.5) / height)[:, None]
    p = cam.proj
    # clip = v * P (row vector): ndc.x = (x*m00 + z*m20)/z  ->  x/z = (ndc.x - m20)/m00
    dx = np.broadcast_to((ndc_x - p[2, 0]) / p[0, 0], (len(ys), width))
    dy = np.broadcast_to((ndc_y - p[2, 1]) / p[1, 1], (len(ys), width))
    dv = np.stack([dx, dy, np.ones_like(dx)], -1)           # view-space direction with dz == 1  => t == view z
    rot = cam.world[:3, :3]
    dw = dv @ rot                                            # world direction (row-vector)
    o = cam.pos

    t_best = np.full(dx.shape, np.inf)
    obj = np.full(dx.shape, -1, np.int32)
    # ground plane y = -1
    with np.errstate(divide="ignore", invalid="ignore"):
        tg = (-1.0 - o[1]) / dw[..., 1]
    hit = (tg > NEAR) & (tg < FAR * 0.6) & np.isfinite(tg)
    t_best = np.where(hit, tg, t_best)
    obj = np.where(hit, len(scene.radii), obj)
    a = np.sum(dw * dw, -1)
    for k in range(len(scene.radii)):
        oc = o - scene.centers[k]
        b = 2.0 * (dw @ oc)
        c = float(oc @ oc) - scene.radii[k] ** 2
        disc = b * b - 4 * a * c
        ok = disc > 0
        sq = np.sqrt(np.where(ok, disc, 0.0))
        t0 = (-b - sq) / (2 * a)
        hit = ok & (t0 > NEAR) & (t0 < t_best)
        t_best = np.where(hit, t0, t_best)
        obj = np.where(hit, k, obj)

    is_bg = obj < 0
    t = np.where(is_bg, FAR, t_best)
    pw = o + dw * t[..., None]
    normal = np.zeros_like(pw)
    ground = obj == len(scene.radii)
    normal[ground] = [0.0, 1.0, 0.0]
    sph = (~is_bg) & (~ground)
    idx = np.clip(obj, 0, len(scene.radii) - 1)
    nrm = (pw - scene.centers[idx]) / scene.radii[idx][..., None]
    normal = np.where(sph[..., None], nrm, normal)
    normal[is_bg] = -dw[is_bg] / np.linalg.norm(dw[is_bg], axis=-1, keepdims=True) if is_bg.any() else normal[is_bg]
    return dict(t=t, pw=pw, normal=normal, obj=obj, is_bg=is_bg, ndc_x=np.broadcast_to(ndc_x, dx.shape), ndc_y=np.broadcast_to(ndc_y, dx.shape))


def _hash01(a: np.ndarray, b: np.ndarray, seed: int) -> np.ndarray:
    h = (a.astype(np.uint64) * np.uint64(73856093)) ^ (b.astype(np.uint64) * np.uint64(19349663)) ^ np.uint64(seed * 83492791)
    h = (h ^ (h >> np.uint64(13))) * np.uint64(1274126177)
    h = h ^ (h >> np.uint64(16))
    return (h & np.uint64(0xFFFFFF)).astype(np.float64) / float(0x1000000)


def generate_frame(scene: Scene, frame: int, width: int, height: int, prev_depth: np.ndarray | None = None,
                   use_jitter: bool = True, chunk_rows: int = 256) -> dict:
    """Returns dict(depth (H,W) f32, normal (H,W,4), color (H,W,4), material (H,W,4), motion (H,W,2), prev_depth (H,W),
    curr_camera, prev_camera (CameraAttribs))."""
    return generate_rows(scene, frame, width, height, 0, height, prev_depth, use_jitter, chunk_rows)


def _map_chunks(fn, starts) -> None:
    starts = list(starts)
    workers = min(len(starts), max(1, min(16, (os.cpu_count() or 1) // max(1, int(os.environ.get("LOCAL_WORLD_SIZE", "1"))))))
    if workers <= 1:
        for g0 in starts:
            fn(g0)
        return
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max_workers=workers) as pool:
        list(pool.map(fn, starts))


def generate_rows(scene: Scene, frame: int, width: int, height: int, row0: int, row1: int, prev_depth: np.ndarray | None = None,
                  use_jitter: bool = True, chunk_rows: int = 256) -> dict:
    """Rows [row0, row1) of frame `frame` of the full width x height image (arrays have row1 - row0 rows). When `prev_depth`
    is None the previous frame's depth of the same rows is ray-cast too (frame 0: a copy of the current depth)."""
    cam = make_camera(frame, width, height, use_jitter)
    prev = make_camera(max(frame - 1, 0), width, height, use_jitter)
    nrows = row1 - row0
    depth = np.empty((nrows, width), np.float32)
    normal = np.zeros((nrows, width, 4), np.float32)
    color = np.zeros((nrows, width, 4), np.float32)
    material = np.zeros((nrows, width, 4), np.float32)
    motion = np.empty((nrows, width, 2), np.float32)
    light = np.array([0.4, 0.8, -0.45])
    light = light / np.linalg.norm(light)
    nobj = len(scene.radii)
    pvp = prev.view @ prev.proj

    def chunk(g0: int) -> None:
        grows = slice(g0, min(g0 + chunk_rows, row1))
        rows = slice(g0 - row0, grows.stop - row0)
        rc = _raycast(scene, cam, width, height, grows)
        z = rc["t"]
        p = cam.proj
        d = (z * p[2, 2] + p[3, 2]) / z
        d = np.where(rc["is_bg"], 1.0, d)
        depth[rows] = d.astype(np.float32)
        normal[rows, :, :3] = rc["normal"].astype(np.float32)
        # motion: curr NDC of the pixel centre is (ndc_x, ndc_y) by construction
        pw1 = np.concatenate([rc["pw"], np.ones_like(z)[..., None]], -1)
        clip_prev = pw1 @ pvp
        ndc_prev = clip_prev[..., :2] / clip_prev[..., 3:4]
        mx = (rc["ndc_x"] - cam.jitter[0]) - (ndc_prev[..., 0] - prev.jitter[0])
        my = (rc["ndc_y"] - cam.jitter[1]) - (ndc_prev[..., 1] - prev.jitter[1])
        motion[rows, :, 0] = mx.astype(np.float32)
        motion[rows, :, 1] = my.astype(np.float32)
        # shading
        obj = np.where(rc["is_bg"], nobj, rc["obj"])
        oid = np.clip(obj, 0, nobj)
        alb = scene.albedo[oid]
        ndl = np.clip(rc["normal"] @ light, 0.0, 1.0)
        # checker on the ground, stripes on spheres: gives TAA / bloom some texture
        gx = np.floor(rc["pw"][..., 0] * 1.5).astype(np.int64)
        gz = np.floor(rc["pw"][..., 2] * 1.5).astype(np.int64)
        checker = np.where(((gx + gz) & 1) == 0, 1.0, 0.55)
        tex = np.where(obj == nobj, checker, 0.8 + 0.2 * np.sin(rc["pw"][..., 1] * 9.0))
        col = alb * (0.08 + 1.6 * ndl[..., None]) * tex[..., None]
        col = col + alb * scene.emissive[oid][..., None]
        # sparse log-uniform highlights (5 % of pixels in [4, 64]) keyed on world cell so they are temporally stable
        hx = np.floor(rc["pw"][..., 0] * 40.0).astype(np.int64)
        hz = np.floor((rc["pw"][..., 2] + rc["pw"][..., 1]) * 40.0).astype(np.int64)
        h = _hash01(hx, hz, 11)
        spark = np.where(h < 0.05, np.exp2(2.0 + 4.0 * _hash01(hx, hz, 29)), 0.0)
        col = col + spark[..., None] * alb
        sky = np.stack([0.35 + 0.3 * rc["ndc_y"], 0.5 + 0.3 * rc["ndc_y"], 0.9 + 0.0 * rc["ndc_y"]], -1) * 1.2
        col = np.where(rc["is_bg"][..., None], sky, col)
        color[rows, :, :3] = np.maximum(col, 0.0).astype(np.float32)
        color[rows, :, 3] = 1.0
        material[rows, :, 0] = np.where(rc["is_bg"], 1.0, scene.rough[oid]).astype(np.float32)
        material[rows, :, 1] = np.where(obj == nobj, 0.0, 0.5).astype(np.float32)

    # Chunks are independent (every value is a per-pixel function) and numpy releases the GIL inside its kernels, so they are
    # ray-cast on a thread pool: same chunk size, same arithmetic, same bits as the sequential loop — only the wall time of
    # a 4K frame changes (bench.py generates its inputs at start-up, also under torchrun where OMP_NUM_THREADS is 1).
    _map_chunks(chunk, range(row0, row1, chunk_rows))
    if prev_depth is None:
        if frame == 0:
            prev_depth = depth.copy()
        else:
            prev_depth = np.empty_like(depth)

            def prev_chunk(g0: int) -> None:
                grows = slice(g0, min(g0 + chunk_rows, row1))
                rc = _raycast(scene, prev, width, height, grows)
                z = rc["t"]
                prev_depth[g0 - row0:grows.stop - row0] = np.where(rc["is_bg"], 1.0, (z * prev.proj[2, 2] + prev.proj[3, 2]) / z).astype(np.float32)

            _map_chunks(prev_chunk, range(row0, row1, chunk_rows))
    return dict(depth=depth, normal=normal, color=color, material=material, motion=motion, prev_depth=prev_depth,
                curr_camera=cam.attribs, prev_camera=prev.attribs, frame=frame)


def generate_sequence(width: int, height: int, frames: int, seed: int = 7, k: int = 24, use_jitter: bool = True, first_frame: int = 0) -> list[dict]:
    scene = make_scene(seed, k)
    out = []
    prev_depth = None
    if first_frame > 0:
        prev_depth = generate_frame(scene, first_frame - 1, width, height, None, use_jitter)["depth"]
    for f in range(first_frame, first_frame + frames):
        fr = generate_frame(scene, f, width, height, prev_depth, use_jitter)
        prev_depth = fr["depth"]
        out.append(fr)
    return out


def selection_depth(width: int, height: int, frame: int, selected, seed: int = 7, k: int = 24, use_jitter: bool = True,
                    chunk_rows: int = 256) -> np.ndarray:
    """The selection depth of frame `frame` of `generate_sequence(width, height, ..., seed, k, use_jitter)`: the depth of the spheres
    whose indices are in `selected` alone, ignoring every other sphere and the ground (the selected geometry rendered on its own, as
    a selection pass would), 1 elsewhere. Where a selected sphere is visible the value equals the frame's depth bit for bit: the
    rays, the intersection and the depth are computed by the same expressions, on the same row chunks, as `_raycast`."""
    scene = make_scene(seed, k)
    cam = make_camera(frame, width, height, use_jitter)
    sel = sorted(set(int(i) for i in selected))
    out = np.empty((height, width), np.float32)

    def chunk(g0: int) -> None:
        rows = slice(g0, min(g0 + chunk_rows, height))
        ys = np.arange(rows.start, rows.stop, dtype=np.float64)
        xs = np.arange(width, dtype=np.float64)
        ndc_x = (2.0 * (xs + 0.5) / width - 1.0)[None, :]
        ndc_y = (1.0 - 2.0 * (ys + 0.5) / height)[:, None]
        p = cam.proj
        dx = np.broadcast_to((ndc_x - p[2, 0]) / p[0, 0], (len(ys), width))
        dy = np.broadcast_to((ndc_y - p[2, 1]) / p[1, 1], (len(ys), width))
        dw = np.stack([dx, dy, np.ones_like(dx)], -1) @ cam.world[:3, :3]
        o = cam.pos
        t_best = np.full(dx.shape, np.inf)
        a = np.sum(dw * dw, -1)
        for s in sel:
            oc = o - scene.centers[s]
            b = 2.0 * (dw @ oc)
            c = float(oc @ oc) - scene.radii[s] ** 2
            disc = b * b - 4 * a * c
            ok = disc > 0
            sq = np.sqrt(np.where(ok, disc, 0.0))
            t0 = (-b - sq) / (2 * a)
            hit = ok & (t0 > NEAR) & (t0 < t_best)
            t_best = np.where(hit, t0, t_best)
        z = np.where(np.isfinite(t_best), t_best, FAR)
        d = (z * p[2, 2] + p[3, 2]) / z
        out[rows] = np.where(np.isfinite(t_best), d, 1.0).astype(np.float32)

    _map_chunks(chunk, range(0, height, chunk_rows))
    return out


def mesh_id(width: int, height: int, frame: int, seed: int = 7, k: int = 24, use_jitter: bool = True, chunk_rows: int = 256) -> np.ndarray:
    """The mesh-ID target (R32F) of frame `frame` of `generate_sequence(width, height, ..., seed, k, use_jitter)`: per pixel the index of
    the nearest object, spheres 0 .. k - 1 and the ground k, and -1 on the background. The objects are those of `_raycast`, called on
    the same row chunks as `generate_rows`, so the background is exactly where the frame's depth is 1."""
    scene = make_scene(seed, k)
    cam = make_camera(frame, width, height, use_jitter)
    out = np.empty((height, width), np.float32)

    def chunk(g0: int) -> None:
        rows = slice(g0, min(g0 + chunk_rows, height))
        rc = _raycast(scene, cam, width, height, rows)
        out[rows] = np.where(rc["is_bg"], -1, rc["obj"]).astype(np.float32)

    _map_chunks(chunk, range(0, height, chunk_rows))
    return out


def scene_depth_colour(frame: dict) -> np.ndarray:
    """What the renderer writes in the scene-depth debug view (RenderPBR.psh:602-607) for `frame` (a `generate_sequence` entry, or any
    dict with its "curr_camera" and "depth"): rgb =
    saturate((DepthToCameraZ(depth) - fSceneNearZ) / max(fSceneFarZ - fSceneNearZ, 1e-6)) with the scene range equal to the camera's
    near / far range, as the overlay is drawn; alpha 1. fp32, one rounding per operation."""
    cam = frame["curr_camera"]
    f = np.float32
    d = np.asarray(frame["depth"], f)
    P = cam.mProj.m
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        z = (f(P[3][2]) - d * f(P[3][3])) / (d * f(P[2][3]) - f(P[2][2]))
        rel = (z - f(cam.fNearPlaneZ)) / np.fmax(f(cam.fFarPlaneZ) - f(cam.fNearPlaneZ), f(1e-6))
    rel = np.fmin(np.fmax(rel, f(0.0)), f(1.0)).astype(f)
    out = np.ones(d.shape + (4,), f)
    out[..., 0] = out[..., 1] = out[..., 2] = rel
    return out


def noise_frame(width: int, height: int, seed: int = 3) -> dict:
    """Pure-noise variant (worst case for caches / branch coherence, SURVEY.md §8d): white-noise depth, random normals."""
    rng = np.random.default_rng(seed)
    cam = make_camera(0, width, height, False)
    depth = rng.uniform(0.9, 0.9999, (height, width)).astype(np.float32)
    depth[rng.uniform(size=depth.shape) < 0.1] = 1.0
    n = rng.normal(size=(height, width, 3))
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    normal = np.zeros((height, width, 4), np.float32)
    normal[..., :3] = n
    color = np.zeros((height, width, 4), np.float32)
    color[..., :3] = np.exp2(rng.uniform(-8, 6, (height, width, 3)))
    color[..., 3] = 1
    material = np.zeros((height, width, 4), np.float32)
    material[..., 0] = rng.choice([0.0, 0.05, 0.15, 0.3, 0.6], (height, width))
    motion = (rng.uniform(-1, 1, (height, width, 2)) * 4.0 / np.array([width, height])).astype(np.float32)
    return dict(depth=depth, normal=normal, color=color, material=material, motion=motion, prev_depth=depth.copy(),
                curr_camera=cam.attribs, prev_camera=cam.attribs, frame=0)


def _reversed_camera(a: CameraAttribs) -> CameraAttribs:
    """The same camera with a reversed-depth projection: depth' = 1 - depth, i.e. (row-vector convention, clip.z = z*m22 + m32,
    clip.w = z) m22' = 1 - m22, m32' = -m32; the derived matrices are recomputed in float64 from the stored float32 ones."""
    def get(m):
        return np.array([[m.m[r][c] for c in range(4)] for r in range(4)], np.float64)

    def put(dst, m):
        m32 = np.asarray(m, np.float32)
        for r in range(4):
            for c in range(4):
                dst.m[r][c] = float(m32[r, c])

    out = CameraAttribs.from_buffer_copy(bytes(a))
    view, proj = get(a.mView), get(a.mProj)
    proj[2, 2], proj[3, 2] = 1.0 - proj[2, 2], -proj[3, 2]
    vp = view @ proj
    put(out.mProj, proj), put(out.mViewProj, vp)
    put(out.mProjInv, np.linalg.inv(proj)), put(out.mViewProjInv, np.linalg.inv(vp))
    out.fNearPlaneDepth, out.fFarPlaneDepth, out.fSceneNearDepth, out.fSceneFarDepth = 1.0, 0.0, 1.0, 0.0
    return out


def reverse_depth_frame(frame: dict) -> dict:
    """The same frame as a renderer with a reversed depth buffer would produce it (PostFXContext::FEATURE_FLAG_REVERSED_DEPTH):
    depth' = 1 - depth (exact in fp32 for depth >= 0.5, which is where this scene lives), background = 0, cameras with the
    reversed projection. Everything else is unchanged."""
    out = dict(frame)
    for k in ("depth", "prev_depth"):
        out[k] = (np.float32(1.0) - np.asarray(frame[k], np.float32)).astype(np.float32)
    out["curr_camera"], out["prev_camera"] = _reversed_camera(frame["curr_camera"]), _reversed_camera(frame["prev_camera"])
    return out


# ---- environment maps (E, dfx_pass_env_map) ---------------------------------------------------------------------------------------
# Cube faces +X, -X, +Y, -Y, +Z, -Z: the D3D / Vulkan (sc, tc) axes and signs, direction = ma * e_major + sc * e_s + tc * e_t.
_CUBE_S = [(2, -1), (2, 1), (0, 1), (0, 1), (0, 1), (0, -1)]
_CUBE_T = [(1, -1), (1, -1), (2, 1), (2, -1), (1, -1), (1, -1)]
SUN_DIRECTION = np.array([0.48, 0.36, 0.8]) / np.linalg.norm([0.48, 0.36, 0.8])


def _sky(d: np.ndarray, face: np.ndarray, rng: np.random.Generator) -> np.ndarray:
    """HDR radiance along unit directions d (..., 3): a horizon-to-zenith gradient, a ground below the horizon, a sun disc of peak 40
    with a halo, and a per-face tint times a checker of 8 cells per face edge plus texel noise, so that every face, edge and corner
    is told apart. `face` (...) is the cube face (or the sphere's longitude octant) a texel belongs to."""
    y = d[..., 1]
    t = np.clip(y, 0.0, 1.0)[..., None]
    sky = (1 - t) * np.array([0.9, 0.95, 1.1]) + t * np.array([0.25, 0.45, 1.2])
    ground = np.array([0.35, 0.3, 0.25]) * (0.6 + 0.4 * np.clip(-y, 0, 1))[..., None]
    c = np.where((y >= 0)[..., None], sky, ground)
    cosang = np.clip(d @ SUN_DIRECTION, -1.0, 1.0)
    ang = np.arccos(cosang)
    c = c + (40.0 * (ang < 0.05) + 4.0 * np.exp(-(ang / 0.25) ** 2))[..., None] * np.array([1.0, 0.9, 0.7])
    tint = np.array([[1.2, 0.8, 0.8], [0.8, 1.2, 0.8], [0.8, 0.8, 1.2], [1.2, 1.2, 0.7], [0.7, 1.2, 1.2], [1.2, 0.7, 1.2], [1.0, 1.0, 1.0],
                     [0.9, 0.9, 0.9]])[face]
    rgb = c * tint * (1.0 + 0.05 * rng.standard_normal(c.shape))
    return np.concatenate([rgb, np.ones(rgb.shape[:-1] + (1,))], axis=-1)


def _box_chain(level0: np.ndarray, levels: int, cube: bool) -> list[np.ndarray]:
    """A 2x2 box mip chain (every level the mean of 2x2 texels of the one before, per face for a cube), fp32."""
    out = [np.asarray(level0, np.float32)]
    for _ in range(1, levels):
        a = out[-1].astype(np.float64)
        if cube:
            s = a.shape[1]
            if s == 1:
                break
            f = a.reshape(6, s, s, 4)
            f = 0.25 * (f[:, 0::2, 0::2] + f[:, 1::2, 0::2] + f[:, 0::2, 1::2] + f[:, 1::2, 1::2])
            out.append(f.reshape(6 * (s // 2), s // 2, 4).astype(np.float32))
        else:
            h, w = a.shape[:2]
            if h == 1 and w == 1:
                break
            a = np.pad(a, ((0, h % 2), (0, w % 2), (0, 0)), mode="edge")
            out.append((0.25 * (a[0::2, 0::2] + a[1::2, 0::2] + a[0::2, 1::2] + a[1::2, 1::2])).astype(np.float32))
    return out


def env_map_cube(size: int, levels: int, seed: int = 11) -> list[np.ndarray]:
    """A procedural HDR sky as a cube map for dfx_pass_env_map: `levels` planes (6 s_i, s_i, 4) float32 (s_i = size >> i, faces
    stacked top to bottom), level 0 from the texel-centre directions, the others a 2x2 box chain. `size` a power of two."""
    assert size >= 1 and size & (size - 1) == 0 and 1 <= levels <= 8 and (size >> (levels - 1)) >= 1
    rng = np.random.default_rng(seed)
    c = (np.arange(size) + 0.5) / size * 2.0 - 1.0
    tc, sc = np.meshgrid(c, c, indexing="ij")                     # rows: tc (v), columns: sc (u)
    faces = []
    for f in range(6):
        d = np.zeros((size, size, 3))
        d[..., f // 2] = -1.0 if f % 2 else 1.0
        d[..., _CUBE_S[f][0]] = _CUBE_S[f][1] * sc
        d[..., _CUBE_T[f][0]] = _CUBE_T[f][1] * tc
        d /= np.linalg.norm(d, axis=-1, keepdims=True)
        cell = ((np.floor((sc + 1) * 4) + np.floor((tc + 1) * 4)) % 2)[..., None]
        faces.append(_sky(d, np.full((size, size), f), rng) * np.concatenate([0.75 + 0.5 * cell] * 3 + [np.ones_like(cell)], axis=-1))
    return _box_chain(np.concatenate(faces, axis=0), levels, cube=True)


def env_map_sphere(width: int, height: int, levels: int, seed: int = 11) -> list[np.ndarray]:
    """The same sky as a sphere map (u = atan2(z, x) / 2pi + 0.5, v = asin(y) / pi + 0.5, ShaderUtilities.fxh:98-102): `levels`
    planes (max(height >> i, 1), max(width >> i, 1), 4) float32, a 2x2 box chain."""
    rng = np.random.default_rng(seed)
    u = (np.arange(width) + 0.5) / width
    v = (np.arange(height) + 0.5) / height
    vv, uu = np.meshgrid(v, u, indexing="ij")
    lon, lat = (uu - 0.5) * 2.0 * np.pi, (vv - 0.5) * np.pi
    d = np.stack([np.cos(lat) * np.cos(lon), np.sin(lat), np.cos(lat) * np.sin(lon)], axis=-1)
    octant = np.floor(uu * 8).astype(int) % 8
    cell = ((np.floor(uu * 32) + np.floor(vv * 16)) % 2)[..., None]
    return _box_chain(_sky(d, octant, rng) * np.concatenate([0.75 + 0.5 * cell] * 3 + [np.ones_like(cell)], axis=-1), levels, cube=False)


def look_at_camera(eye, target, width: int, height: int, ortho: bool = False, reversed_depth: bool = False, infinite: bool = False,
                   near: float = NEAR, far: float = FAR) -> CameraAttribs:
    """A camera at `eye` looking at `target` (+y up; +x up when looking along y), row-vector matrices like make_camera. Perspective:
    fovY 60 deg; orthographic: a 6-unit-high view volume. `reversed_depth`: near = 1, far = 0; with `infinite` the far plane is at
    infinity (clip.w = 0 there, so mViewProjInv maps the far plane to a point at infinity)."""
    eye, target = np.asarray(eye, np.float64), np.asarray(target, np.float64)
    fwd = target - eye
    fwd /= np.linalg.norm(fwd)
    up0 = np.array([1.0, 0.0, 0.0]) if abs(fwd[1]) > 0.99 else np.array([0.0, 1.0, 0.0])
    right = np.cross(up0, fwd)
    right /= np.linalg.norm(right)
    up = np.cross(fwd, right)
    world = np.eye(4)
    world[0, :3], world[1, :3], world[2, :3], world[3, :3] = right, up, fwd, eye
    view = np.linalg.inv(world)
    proj = np.zeros((4, 4))
    if ortho:
        hh = 3.0
        proj[0, 0], proj[1, 1] = 1.0 / (hh * width / height), 1.0 / hh
        proj[2, 2], proj[3, 2], proj[3, 3] = 1.0 / (far - near), -near / (far - near), 1.0
    else:
        t = math.tan(math.radians(60.0) / 2)
        proj[0, 0], proj[1, 1], proj[2, 3] = 1.0 / (t * width / height), 1.0 / t, 1.0
        if reversed_depth and infinite:
            proj[2, 2], proj[3, 2] = 0.0, near
        else:
            proj[2, 2], proj[3, 2] = far / (far - near), -near * far / (far - near)
    if reversed_depth and ortho:                                  # depth' = 1 - depth with clip.w = 1
        proj[2, 2], proj[3, 2] = -proj[2, 2], 1.0 - proj[3, 2]
    elif reversed_depth and not infinite:                         # depth' = 1 - depth with clip.w = z
        proj[2, 2], proj[3, 2] = 1.0 - proj[2, 2], -proj[3, 2]
    c = CameraAttribs()
    c.f4Position[:] = [eye[0], eye[1], eye[2], 1.0]
    c.f4ViewportSize[:] = [float(width), float(height), float(np.float32(1.0) / np.float32(width)), float(np.float32(1.0) / np.float32(height))]
    c.fNearPlaneZ, c.fFarPlaneZ = near, far
    c.fNearPlaneDepth, c.fFarPlaneDepth = (1.0, 0.0) if reversed_depth else (0.0, 1.0)
    c.fSceneNearZ, c.fSceneFarZ, c.fSceneNearDepth, c.fSceneFarDepth = near, far, c.fNearPlaneDepth, c.fFarPlaneDepth
    c.fHandness, c.fExposure = 1.0, 0.0

    def put(dst, m):
        m32 = np.asarray(m, np.float32)
        for r in range(4):
            for k in range(4):
                dst.m[r][k] = float(m32[r, k])

    vp = view @ proj
    put(c.mView, view), put(c.mProj, proj), put(c.mViewProj, vp)
    put(c.mViewInv, world), put(c.mProjInv, np.linalg.pinv(proj)), put(c.mViewProjInv, np.linalg.pinv(vp))
    return c


def env_map_cameras(width: int, height: int) -> dict:
    """Cameras for E: looking along each of the six axes (face centres, and face ties at the image corners) and at each of the eight
    cube corners (±1, ±1, ±1) (where three faces meet), from a point off the origin."""
    eye = np.array([0.3, -0.2, 0.1])
    out = {}
    for a in range(3):
        for s in (1.0, -1.0):
            d = np.zeros(3)
            d[a] = s
            out[f"axis{'+-'[s < 0]}{'xyz'[a]}"] = look_at_camera(eye, eye + d, width, height)
    for sx in (1, -1):
        for sy in (1, -1):
            for sz in (1, -1):
                out[f"corner{sx:+d}{sy:+d}{sz:+d}"] = look_at_camera(eye, eye + np.array([sx, sy, sz], np.float64), width, height)
    return out


def bound_box_transform(extent_min, extent_max, prim_transform=None) -> np.ndarray:
    """HnRenderBoundBoxTask's box transform (HnRenderBoundBoxTask.cpp:132-139): Scale(max - min) * Translation(min) * PrimTransform, row
    vectors, in float32 as float4x4's operator* forms it (sum over k of a[i][k] * b[k][j], k in order). `prim_transform` None = the
    identity. The unit cube's corner c goes to float4(c, 1) * result."""
    lo, hi = np.asarray(extent_min, np.float32), np.asarray(extent_max, np.float32)
    scale = np.diag(np.append(hi - lo, np.float32(1.0))).astype(np.float32)
    trans = np.eye(4, dtype=np.float32)
    trans[3, :3] = lo

    def mul(a, b):
        out = np.zeros((4, 4), np.float32)
        for i in range(4):
            for j in range(4):
                s = np.float32(a[i, 0] * b[0, j])
                for k in range(1, 4):
                    s = np.float32(s + np.float32(a[i, k] * b[k, j]))
                out[i, j] = s
        return out

    m = mul(scale, trans)
    return m if prim_transform is None else mul(m, np.asarray(prim_transform, np.float32))


def sphere_bound_box(k: int, seed: int = 7, count: int = 24) -> np.ndarray:
    """The box of sphere `k` of make_scene(seed, count): its extent centre -+ radius, in world space (the identity prim transform)."""
    scene = make_scene(seed, count)
    c, r = scene.centers[k], scene.radii[k]
    return bound_box_transform(c - r, c + r)


# ---- motion fields for the vector field overlay (VectorFieldRenderer): (H, W, 2) float32 in the G-buffer's units, the NDC offset from the
# previous to the current position of a pixel (GetMotionVector); -0.02 / elapsed scales them to the drawn vectors' NDC length

def motion_pan(width: int, height: int, dx: float = 0.004, dy: float = -0.002) -> np.ndarray:
    """A camera pan: the same motion everywhere."""
    out = np.empty((height, width, 2), np.float32)
    out[..., 0], out[..., 1] = np.float32(dx), np.float32(dy)
    return out


def _ndc_grid(width: int, height: int) -> tuple[np.ndarray, np.ndarray]:
    x = (np.arange(width, dtype=np.float64) + 0.5) / width * 2.0 - 1.0
    y = 1.0 - (np.arange(height, dtype=np.float64) + 0.5) / height * 2.0
    return np.meshgrid(x, y)


def motion_rotation(width: int, height: int, angle: float = 0.01) -> np.ndarray:
    """A roll of the camera by `angle` radians about the frame's centre: motion proportional to the distance from it."""
    X, Y = _ndc_grid(width, height)
    c, s = np.cos(angle), np.sin(angle)
    return np.stack([X - (c * X + s * Y), Y - (-s * X + c * Y)], -1).astype(np.float32)


def motion_vortex(width: int, height: int, strength: float = 0.02, swirl: float = 0.5) -> np.ndarray:
    """A converging vortex: every vector points past the centre and turns about it, so many lines cross there (heavy overlap)."""
    X, Y = _ndc_grid(width, height)
    return np.stack([strength * (X - swirl * Y), strength * (Y + swirl * X)], -1).astype(np.float32)


def motion_random(width: int, height: int, seed: int = 0, sigma: float = 0.01) -> np.ndarray:
    """Independent Gaussian motion per pixel."""
    return np.random.default_rng(seed).normal(0.0, sigma, (height, width, 2)).astype(np.float32)


def motion_extreme(width: int, height: int, seed: int = 0) -> np.ndarray:
    """Random motion with the values a renderer must not produce but a field may hold: NaN, +-Inf, the largest floats, denormals, and
    vectors long enough to put a line's end beyond the 2^20-pixel guard band."""
    rng = np.random.default_rng(seed)
    out = rng.normal(0.0, 0.05, (height, width, 2)).astype(np.float32)
    special = np.array([np.nan, np.inf, -np.inf, 3.4e38, -3.4e38, 1e-45, 1e4, -1e4, 0.0], np.float32)
    pick = rng.random((height, width, 2)) < 0.3
    out[pick] = special[rng.integers(0, len(special), int(pick.sum()))]
    return out


def shadow_cascades(n: int, width: int, height: int, seed: int = 0, d16: bool = False, hostile: bool = False) -> np.ndarray:
    """Seeded depth of n shadow-map cascades as a light would render them: cleared to 1, then per cascade a few slanted ground and
    wall planes and sphere occluders, nearer surfaces winning. d16: the D16_UNORM codes (uint16, round(saturate(z) * 65535)); otherwise
    D32_FLOAT (float32). hostile (D32 only): a share of texels replaced by depth outside [0, 1], +-inf and NaN."""
    rng = np.random.default_rng(seed)
    y, x = np.meshgrid((np.arange(height) + 0.5) / height, (np.arange(width) + 0.5) / width, indexing="ij")
    out = np.ones((n, height, width), np.float64)
    for c in range(n):
        z = out[c]
        for _ in range(int(rng.integers(1, 4))):             # slanted planes: z = a + b x + c y, kept where inside [0, 1]
            a, b, cc = rng.uniform(0.3, 0.9), rng.uniform(-0.4, 0.4), rng.uniform(-0.4, 0.4)
            p = a + b * x + cc * y
            z[:] = np.where((p >= 0) & (p < z), p, z)
        for _ in range(int(rng.integers(2, 7))):             # spheres: the near cap of a ball of radius r at (cx, cy, cz)
            cx, cy, r = rng.uniform(0, 1), rng.uniform(0, 1), rng.uniform(0.03, 0.3)
            cz = rng.uniform(r, 1.0)
            d2 = r * r - (x - cx) ** 2 - (y - cy) ** 2
            s = cz - np.sqrt(np.maximum(d2, 0.0))
            z[:] = np.where((d2 > 0) & (s < z), s, z)
    if d16:
        return np.rint(np.clip(out, 0.0, 1.0) * 65535.0).astype(np.uint16)
    out = out.astype(np.float32)
    if hostile:
        special = np.array([np.nan, np.inf, -np.inf, -0.5, 1.5, -3.0, 7.0, -0.0, 3e38], np.float32)
        pick = rng.random(out.shape) < 0.05
        out[pick] = special[rng.integers(0, len(special), int(pick.sum()))]
    return out
