"""ORACLE — TEST INFRASTRUCTURE ONLY. ctypes wrapper over oracle/_build/liboracle.so (pinned against the reference's shaders, see oracle_math.h).

Importers: tests/, __graft_entry__.smoke(), bench.py (cpu_baseline leg and --impl reference). Never the product path.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(_HERE, "_build", "liboracle.so")
TABLES = os.path.join(os.path.dirname(_HERE), "diligentfx_b200", "data", "blue_noise_tables.bin")

STAGE_POSTFX, STAGE_SSR, STAGE_SSAO, STAGE_COMPOSE, STAGE_TAA, STAGE_BLOOM, STAGE_TONEMAP = 1, 2, 4, 8, 16, 32, 64
STAGE_ALL = 127
STAGE_DOF = 128   # DepthOfField between TAA and Bloom (not part of STAGE_ALL: the benchmarked chain of BASELINE.json has no DoF)


def build(force: bool = False) -> str:
    if force or not os.path.exists(LIB):
        subprocess.check_call(["make", "-C", _HERE] + (["-B"] if force else []), stdout=subprocess.DEVNULL)
    return LIB


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB)
        L.orc_create.restype = C.c_void_p
        L.orc_last_error.restype = C.c_char_p
        L.orc_last_ms.restype = C.c_double
        L.orc_bayer4x4.restype = C.c_float
        L.orc_halton.restype = C.c_float
        L.orc_fast_acos.restype = C.c_float
        L.orc_depth_to_camera_z.restype = C.c_float
        L.orc_camera_z_to_depth.restype = C.c_float
        L.orc_pcg_hash.restype = C.c_uint32
        L.orc_quantize.restype = C.c_float
        L.orc_quantize.argtypes = [C.c_int, C.c_float]
        for f in ("orc_destroy", "orc_set_threads", "orc_set_cameras", "orc_set_frame_index", "orc_set_ssao_attribs", "orc_set_ssr_attribs",
                  "orc_set_bloom_attribs", "orc_set_taa_attribs", "orc_set_tonemap_attribs", "orc_set_compose_scales", "orc_tone_map", "orc_taa_jitter", "orc_resize", "orc_last_frames", "orc_force_reset"):
            getattr(L, f).restype = None
        _lib = L
    return _lib


class Oracle:
    """A context of named fp32 planes + the reference pass sequence (see oracle_capi.cpp)."""

    def __init__(self, width: int, height: int, threads: int = 0):
        self.L = lib()
        self.w, self.h = width, height
        self.h_ = C.c_void_p(self.L.orc_create(width, height, threads or (os.cpu_count() or 1)))
        blob = open(TABLES, "rb").read()
        self._chk(self.L.orc_set_tables(self.h_, blob, len(blob)))

    def __del__(self):
        try:
            self.L.orc_destroy(self.h_)
        except Exception:
            pass

    def _chk(self, r: int):
        if r != 0:
            raise RuntimeError(self.L.orc_last_error(self.h_).decode())

    def set(self, name: str, arr: np.ndarray):
        a = np.ascontiguousarray(arr, np.float32)
        ch = 1 if a.ndim == 2 else a.shape[2]
        self._chk(self.L.orc_set_plane(self.h_, name.encode(), a.ctypes.data_as(C.POINTER(C.c_float)), a.shape[1], a.shape[0], ch))

    def get(self, name: str) -> np.ndarray:
        w, h, ch = C.c_int(), C.c_int(), C.c_int()
        self._chk(self.L.orc_get_plane(self.h_, name.encode(), None, C.byref(w), C.byref(h), C.byref(ch)))
        out = np.empty((h.value, w.value) if ch.value == 1 else (h.value, w.value, ch.value), np.float32)
        self._chk(self.L.orc_get_plane(self.h_, name.encode(), out.ctypes.data_as(C.POINTER(C.c_float)), C.byref(w), C.byref(h), C.byref(ch)))
        return out

    def set_cameras(self, curr, prev):
        self.L.orc_set_cameras(self.h_, C.byref(curr), C.byref(prev))

    def set_frame_index(self, idx: int):
        self.L.orc_set_frame_index(self.h_, C.c_uint32(idx))

    def brdf_lut(self, size: int | tuple[int, int] = 512, num_samples: int = 512):
        """Pre-integrated GGX table (PrecomputeBRDF.psh) into the plane "brdf_lut": `size` x `size`, or w x h for size = (w, h); the
        reference uses 512 x 512, 512 samples."""
        w, h = (size, size) if isinstance(size, int) else size
        self.L.orc_brdf_lut(self.h_, int(w), int(h), C.c_uint32(num_samples))

    def set_reversed_depth(self, on: bool):
        """PostFXContext::FEATURE_FLAG_REVERSED_DEPTH (process-wide switch, like the reference's shader macro)."""
        self.L.orc_set_reversed_depth(int(bool(on)))

    def set_storage(self, faithful: bool):
        """False (default): fp32 planes, the parity gate. True: every render target is rounded to the reference's texture format
        (R8_UNORM AO, R16F / RGBA16F SSR and TAA, R11G11B10F Bloom, ...) right after the pass that writes it - SURVEY.md Appendix B.5."""
        self.L.orc_set_storage(self.h_, int(bool(faithful)))

    def set_threads(self, t: int):
        self.L.orc_set_threads(self.h_, t)

    def set_ssao(self, a):
        self.L.orc_set_ssao_attribs(self.h_, C.byref(a))

    def set_ssao_flags(self, flags: int):
        """DFX_SSAO_FEATURE_FLAG_* (bit 0 = HALF_PRECISION_DEPTH, bit 1 = HALF_RESOLUTION). A change of either bit re-creates the
        history and history length at 1.0, like PrepareResources; the last frame index is kept."""
        self.L.orc_set_ssao_flags(self.h_, C.c_uint32(flags))

    def set_ssr(self, a, flags: int = 0):
        """A change of HALF_RESOLUTION (bit 1) re-creates the histories, the roughness and the resolved planes at 0."""
        self.L.orc_set_ssr_attribs(self.h_, C.byref(a), C.c_uint32(flags))

    def set_dof(self, a, flags: int = 0):
        """Any change of the feature flags re-creates the temporal CoC planes at 0."""
        self.L.orc_set_dof_attribs(self.h_, C.byref(a), C.c_uint32(flags))

    def resize(self, width: int, height: int):
        """A new frame size: every frame-sized plane is dropped and comes back at its creation value on the next frame, as the
        effects re-create their targets; the last frame indices of SSAO and TAA are kept."""
        self.L.orc_resize(self.h_, int(width), int(height))
        self.w, self.h = width, height

    def last_frames(self) -> tuple[int, int]:
        """(SSAO, TAA) m_LastFrameIdx: the index of the last frame each ran on, 0xFFFFFFFF before the first."""
        s, t = C.c_uint32(), C.c_uint32()
        self.L.orc_last_frames(self.h_, C.byref(s), C.byref(t))
        return s.value, t.value

    def force_reset(self, ssao: bool | None, taa: bool | None):
        """The reset decisions of the next frame() only: True resets, False does not, None follows the rule (a test's way to take
        the opposite decision, also right after index 0xFFFFFFFF, where the last frame index equals the "no frame yet" value)."""
        m = lambda v: -1 if v is None else int(bool(v))  # noqa: E731
        self.L.orc_force_reset(self.h_, m(ssao), m(taa))

    def set_bloom(self, a):
        self.L.orc_set_bloom_attribs(self.h_, C.byref(a))

    def set_taa(self, a, flags: int = 2):
        self.L.orc_set_taa_attribs(self.h_, C.byref(a), C.c_uint32(flags))

    def set_tonemap(self, a, ave_log_lum: float = 0.3, to_srgb: bool = True):
        self.L.orc_set_tonemap_attribs(self.h_, C.byref(a), C.c_float(ave_log_lum), int(to_srgb))

    def set_compose_scales(self, ssr_scale: float, ssao_scale: float):
        self.L.orc_set_compose_scales(self.h_, C.c_float(ssr_scale), C.c_float(ssao_scale))

    def set_inputs(self, fr: dict):
        """fr: a frame dict from diligentfx_b200.synth.generate_frame."""
        self.set("depth", fr["depth"]), self.set("prev_depth_in", fr["prev_depth"]), self.set("motion", fr["motion"])
        self.set("normal", fr["normal"]), self.set("color", fr["color"]), self.set("material", fr["material"])
        self.set_cameras(fr["curr_camera"], fr["prev_camera"])
        self.set_frame_index(fr["frame"])

    def run(self, pass_name: str) -> float:
        self._chk(self.L.orc_run(self.h_, pass_name.encode()))
        return self.L.orc_last_ms(self.h_)

    def frame(self, stages: int = STAGE_ALL) -> float:
        self._chk(self.L.orc_frame(self.h_, C.c_uint32(stages)))
        return self.L.orc_last_ms(self.h_)


QUANT_UNORM8, QUANT_UNORM16, QUANT_HALF, QUANT_FLOAT11, QUANT_FLOAT10 = range(5)


def quantize(fmt: int, v: float) -> float:
    """One value through a render-target format of the reference (oracle_quant.h)."""
    return float(lib().orc_quantize(fmt, C.c_float(v)))


def tone_map(attribs, ave_log_lum: float, rgb: np.ndarray) -> np.ndarray:
    a = np.ascontiguousarray(rgb, np.float32).reshape(-1, 3)
    out = np.empty_like(a)
    lib().orc_tone_map(C.byref(attribs), C.c_float(ave_log_lum), a.ctypes.data_as(C.POINTER(C.c_float)),
                       out.ctypes.data_as(C.POINTER(C.c_float)), a.shape[0])
    return out.reshape(np.asarray(rgb).shape)
