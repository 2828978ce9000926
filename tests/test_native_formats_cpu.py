"""The passes that read the G-buffer in the renderer's formats (colour and normal RGBA16F, motion RG16F, material RG8U) refuse every
malformed combination with DFX_ERR_INVALID_ARG and a message that names the problem, before any CUDA call: mixed colour / normal
formats, previous-frame motion of the other width, RG8U where only the material may be RG8U, pitches and pointers that do not fit
the texel, and the entries that take fp32 planes only (the peer-sharded ray march, the IBL compose). No device is needed: the
pointers are fake, non-null and aligned, and no kernel is launched."""
import ctypes as C

import pytest

from diligentfx_b200 import capi

W, H = 40, 24
BASE = 1 << 24              # fake device addresses: aligned for every texel size, never dereferenced
RGBA32F, RGBA16F, RG32F, RG16F, RG8U, R32F, R8U = (capi.FORMAT_RGBA32F, capi.FORMAT_RGBA16F, capi.FORMAT_RG32F, capi.FORMAT_RG16F, capi.FORMAT_RG8U,
                                                    capi.FORMAT_R32F, capi.FORMAT_R8U)
BPT = {RGBA32F: 16, RGBA16F: 8, RG32F: 8, RG16F: 4, RG8U: 2, R32F: 4, R8U: 1}


@pytest.fixture(scope="module")
def lib(built):
    return capi.load()


_slot = [0]


def plane(fmt: int, w: int = W, h: int = H, pitch: int | None = None, offset: int = 0) -> C.POINTER(capi.Plane):
    _slot[0] += 1
    p = capi.Plane(BASE * (1 + _slot[0]) + offset, pitch if pitch is not None else w * BPT[fmt], w, h, fmt, 0)
    return C.pointer(p)


def refused(lib, status: int, *words: str) -> None:
    msg = (lib.dfx_last_error() or b"").decode()
    assert status == capi.DFX_ERR_INVALID_ARG, (status, msg)
    for w in words:
        assert w in msg, (w, msg)


CAMS = C.c_void_p(BASE)
ROWS = capi.Rows(0, H)


def _hiz():
    p = capi.Pyramid()
    p.levels = 3
    for i in range(3):
        p.level[i] = plane(R32F, max(W >> i, 1), max(H >> i, 1)).contents
    return C.byref(p), p


def _intersect(lib, color, normal, motion, flags=0):
    hiz, keep = _hiz()
    a = capi.SSRAttribs.default()
    return lib.dfx_pass_ssr_intersect(None, CAMS, C.byref(a), flags, color, normal, plane(R32F), plane(R8U), plane(RG32F, 128, 128), hiz, motion,
                                      plane(RGBA32F), plane(RGBA32F), ROWS)


def test_mixed_colour_and_normal_formats(lib):
    refused(lib, _intersect(lib, plane(RGBA16F), plane(RGBA32F), plane(RG16F)), "colour and normal", "RGBA16F")
    refused(lib, _intersect(lib, plane(RGBA32F), plane(RGBA16F), plane(RG32F)), "colour and normal", "RGBA16F")


def test_previous_frame_motion_must_match_the_gbuffer(lib):
    refused(lib, _intersect(lib, plane(RGBA16F), plane(RGBA16F), plane(RG32F), capi.SSR_FLAG_PREVIOUS_FRAME), "motion must be RG16F")
    refused(lib, _intersect(lib, plane(RGBA32F), plane(RGBA32F), plane(RG16F), capi.SSR_FLAG_PREVIOUS_FRAME), "motion must be RG16F")


def test_rg8u_is_material_only(lib):
    refused(lib, _intersect(lib, plane(RG8U), plane(RGBA16F), plane(RG16F)), "bad plane 'color'")
    refused(lib, _intersect(lib, plane(RGBA16F), plane(RG8U), plane(RG16F)), "bad plane 'normal'")
    refused(lib, lib.dfx_pass_postfx_prepare(None, CAMS, plane(R32F), plane(R32F), plane(RG8U), plane(R32F), plane(RG32F), plane(R32F), ROWS),
            "bad plane 'motion'")
    a = capi.SSRAttribs.default()
    refused(lib, lib.dfx_pass_ssr_spatial(None, CAMS, C.byref(a), plane(R32F), plane(R8U), plane(RG8U), plane(R32F), plane(RGBA32F), plane(RGBA32F),
                                          plane(RGBA32F), plane(R32F), plane(R32F), ROWS), "bad plane 'normal'")


@pytest.mark.parametrize("case", ["rgba16f pitch not a multiple of 8", "rg16f pitch not a multiple of 4", "pitch below the row",
                                  "rgba16f pointer misaligned", "rg16f pointer misaligned"])
def test_pitch_and_alignment_of_narrow_planes(lib, case):
    colour, motion = plane(RGBA16F), plane(RG16F)
    if case == "rgba16f pitch not a multiple of 8":
        colour = plane(RGBA16F, pitch=W * 8 + 4)
    elif case == "rg16f pitch not a multiple of 4":
        motion = plane(RG16F, pitch=W * 4 + 2)
    elif case == "pitch below the row":
        colour = plane(RGBA16F, pitch=W * 8 - 8)
    elif case == "rgba16f pointer misaligned":
        colour = plane(RGBA16F, offset=4)
    else:
        motion = plane(RG16F, offset=2)
    name = "color" if "rg16f" not in case else "motion"
    refused(lib, _intersect(lib, colour, plane(RGBA16F), motion, capi.SSR_FLAG_PREVIOUS_FRAME), f"bad plane '{name}'")
    if name == "color":
        refused(lib, lib.dfx_pass_compose(None, colour, None, None, C.c_float(1.0), C.c_float(1.0), plane(RGBA32F), ROWS), "bad plane 'color'")
    else:
        refused(lib, lib.dfx_pass_postfx_prepare(None, CAMS, plane(R32F), plane(R32F), motion, plane(R32F), plane(RG32F), plane(R32F), ROWS),
                "bad plane 'motion'")


def test_peer_sharded_ray_march_takes_fp32_planes_only(lib):
    hiz, keep = _hiz()
    a = capi.SSRAttribs.default()
    peers = capi.PeerSet()
    peers.count, peers.row_begin[0], peers.row_begin[1] = 1, 0, H
    peers.color[0], peers.normal[0] = BASE * 100, BASE * 101
    for m in range(3):
        peers.hiz[m][0] = BASE * (102 + m)
    st = lib.dfx_pass_ssr_intersect_peer(None, CAMS, C.byref(a), 0, C.byref(peers), plane(RGBA16F), plane(RGBA16F), plane(R32F), plane(R8U),
                                         plane(RG32F, 128, 128), hiz, plane(RGBA32F), plane(RGBA32F), ROWS)
    refused(lib, st, "peer-sharded planes must be RGBA32F")


def test_compose_ibl_takes_fp32_planes_only(lib):
    """dfx_pass_compose_ibl has no narrow-format instantiation: RGBA16F colour, or an RGBA16F normal / material with the SSR term,
    is refused."""
    def call(color=RGBA32F, normal=RGBA32F, material=RGBA32F):
        return lib.dfx_pass_compose_ibl(None, CAMS, plane(color), plane(RGBA32F), plane(R32F), plane(RGBA32F), plane(normal), plane(RGBA32F),
                                        plane(material), plane(RG32F, 32, 32), C.c_float(1.0), C.c_float(1.0), plane(RGBA32F), ROWS)
    refused(lib, call(color=RGBA16F), "bad plane 'color'")
    refused(lib, call(normal=RGBA16F), "bad plane")
    refused(lib, call(material=RGBA16F), "bad plane")
    refused(lib, call(material=RG8U), "bad plane")
