"""The CUDA counterpart of oracle/refshader/driver.compare_frame: steps the oracle through one frame pass by pass and, beside every
oracle pass, runs the CUDA pass through the C-ABI on that pass's oracle input planes. A difference is therefore attributable to
the one pass. Returns {label: (cuda_output, oracle_output)} with compare_frame's labels (P0 ... M1, D1 ... D11) plus the fused
entries and the Bloom pyramid launch shapes, which have labels of their own. `failures()` compares such a result to the bounds
of one table, at a drawn or at the default configuration.

Every device plane is allocated in one of three layouts:
  "tight"   pitch = width * bytes per texel (what capi.plane_of describes);
  "padded"  one or more texels of padding per row, pitch not a multiple of 16 bytes where the texel size allows it (the TMA paths
            need a 16-byte multiple and fall back to plain loads);
  "aligned" pitch rounded up to 128 bytes, like dfx_plane_alloc (the TMA paths run).
The padding is filled with NaN (half NaN for the 16-bit planes, 0xA5 for the 8-bit ones): a kernel that indexes rows with the
width where it should use the pitch, or that reads past the end of a row, turns up as a NaN or a wrong value;
`Planes.padding_damage()` reports writes into it.

`run_frame(..., native=...)` also runs every pass that reads the G-buffer a second time on the same values in the renderer's
formats (colour and normal RGBA16F, motion RG16F, material RG8U or RGBA16F), in the same layout, and records that output as
"<label> [native]". Every half and UNORM8 value is an fp32 value, so `twin_failures()` requires the two outputs to be identical
bit for bit (DESIGN §3).

Test infrastructure only; it never runs the reference's shaders.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from diligentfx_b200 import capi
from helpers import assert_close
from oracle import oracle_py as op
from oracle.refshader.driver import Variant, _count, _levels, make_oracle

LAYOUTS = ("tight", "padded", "aligned")
MASK_FILL = 0xA5
NATIVE = " [native]"
NATIVE_MATERIALS = ("rg8", "rgba16")     # run_frame(native=...): the material plane's format beside RGBA16F colour / normal, RG16F motion
_NP = {torch.float32: np.float32, torch.float16: np.float16, torch.uint8: np.uint8}


class Buf:
    """One device plane: `storage` is the whole allocation (padding included), `t` the (H, W[, C]) view of its texels."""

    def __init__(self, storage, t, plane: capi.Plane, row_elems: int):
        self.storage, self.t, self.p, self.row_elems = storage, t, plane, row_elems

    @property
    def ref(self):
        return C.byref(self.p)

    def host(self) -> np.ndarray:
        return self.t.cpu().numpy().astype(np.float32)


class Planes:
    """Allocates device planes in one layout and keeps them (and their descriptors) alive."""

    _FMT = {(torch.float32, 1): (capi.FORMAT_R32F, 4), (torch.float32, 2): (capi.FORMAT_RG32F, 8), (torch.float32, 4): (capi.FORMAT_RGBA32F, 16),
            (torch.uint8, 1): (capi.FORMAT_R8U, 1), (torch.float16, 4): (capi.FORMAT_RGBA16F, 8), (torch.float16, 2): (capi.FORMAT_RG16F, 4),
            (torch.uint8, 2): (capi.FORMAT_RG8U, 2)}

    def __init__(self, layout: str = "tight"):
        assert layout in LAYOUTS, layout
        self.layout, self.bufs, self.keep = layout, [], []

    def pitch(self, w: int, bpt: int) -> int:
        if self.layout == "tight":
            return w * bpt
        if self.layout == "aligned":
            return -(-w * bpt // 128) * 128
        p = w * bpt + bpt
        while p % 16 == 0 and bpt < 16:                    # RGBA32F texels are 16 bytes: every pitch is a multiple of 16
            p += bpt
        return p

    def new(self, h: int, w: int, ch: int = 1, fill: float | np.ndarray | None = None, flags: int = 0, dtype=torch.float32) -> Buf:
        fmt, bpt = self._FMT[(dtype, ch)]
        pitch = self.pitch(w, bpt)
        esz = torch.tensor([], dtype=dtype).element_size()
        pad_value = MASK_FILL if dtype == torch.uint8 else float("nan")
        storage = torch.full((h * pitch // esz,), pad_value, dtype=dtype, device="cuda")
        row = pitch // esz
        t = storage.as_strided((h, w) if ch == 1 else (h, w, ch), (row, 1) if ch == 1 else (row, ch, 1))
        if isinstance(fill, np.ndarray):
            t.copy_(torch.from_numpy(np.ascontiguousarray(fill, _NP[dtype])).cuda())
        elif fill is not None:
            t.fill_(fill)
        b = Buf(storage, t, capi.Plane(storage.data_ptr(), pitch, w, h, fmt, flags), row)
        self.bufs.append(b)
        return b

    def up(self, a: np.ndarray, flags: int = 0) -> Buf:
        a = np.asarray(a, np.float32)
        return self.new(a.shape[0], a.shape[1], 1 if a.ndim == 2 else a.shape[2], fill=a, flags=flags)

    def native(self, a: np.ndarray) -> Buf:
        """A plane in the format of `a`'s own type: (H, W, 4) / (H, W, 2) float16 -> RGBA16F / RG16F, (H, W, 2) uint8 -> RG8U."""
        dtype = {np.dtype(np.float16): torch.float16, np.dtype(np.uint8): torch.uint8}[a.dtype]
        return self.new(a.shape[0], a.shape[1], a.shape[2], fill=a, dtype=dtype)

    def mask(self, a: np.ndarray) -> Buf:
        return self.new(a.shape[0], a.shape[1], fill=(np.asarray(a) != 0).astype(np.uint8), dtype=torch.uint8)

    def like(self, a: np.ndarray, fill=None, flags: int = 0) -> Buf:
        return self.new(a.shape[0], a.shape[1], 1 if a.ndim == 2 else a.shape[2], fill=fill, flags=flags)

    def pyramid(self, bufs: list[Buf]) -> capi.Pyramid:
        p = capi.Pyramid()
        p.levels = len(bufs)
        for i, b in enumerate(bufs):
            p.level[i] = b.p
        self.keep.append(p)
        return p

    def array(self, bufs: list[Buf]):
        arr = (capi.Plane * len(bufs))(*[b.p for b in bufs])
        self.keep.append(arr)
        return arr

    def cameras(self, curr, prev):
        buf = (capi.CameraAttribs * 2)(curr, prev)
        t = torch.frombuffer(bytearray(bytes(buf)), dtype=torch.uint8).cuda()
        self.keep.append(t)
        return C.c_void_p(t.data_ptr())

    def padding_damage(self) -> int:
        """Number of planes whose row padding no longer holds the fill value."""
        bad = 0
        for b in self.bufs:
            s = b.storage.cpu().numpy().reshape(b.p.height, b.row_elems)
            pad = s[:, b.t.shape[1] * (b.t.shape[2] if b.t.dim() == 3 else 1):]
            if pad.size and not (np.isnan(pad).all() if pad.dtype != np.uint8 else (pad == MASK_FILL).all()):
                bad += 1
        return bad


def rows(h: int) -> capi.Rows:
    return capi.Rows(0, h)


def _exactly(a: np.ndarray, narrow: np.ndarray, what: str) -> np.ndarray:
    """`narrow` if it widens to `a` bit for bit, else a ValueError: a twin of a value the format cannot hold would not be a twin."""
    wide = narrow.astype(np.float32) / np.float32(255.0) if narrow.dtype == np.uint8 else narrow.astype(np.float32)
    if not np.array_equal(wide.view(np.uint32), np.ascontiguousarray(a[..., :narrow.shape[-1]], np.float32).view(np.uint32)):
        raise ValueError(f"the {what} plane is not exactly representable in its native format: quantise the frames first")
    return narrow


def native_gbuffer(P: Planes, g, material: str) -> dict[str, Buf]:
    """The G-buffer planes the oracle holds (`g` = o.get), in the renderer's formats: colour and normal RGBA16F, motion RG16F,
    material RG8U (`material` "rg8": z = w = 0 required) or RGBA16F ("rgba16")."""
    assert material in NATIVE_MATERIALS, material
    out = {n: P.native(_exactly(g(n), g(n).astype(np.float16), n)) for n in ("color", "normal", "motion")}
    m = g("material")
    if material == "rg8":
        if np.any(m[..., 2:].view(np.uint32)):
            raise ValueError("an RG8U material leaves z and w at 0")
        out["material"] = P.native(_exactly(m, np.rint(np.clip(m[..., :2], 0.0, 1.0) * 255.0).astype(np.uint8), "material"))
    else:
        out["material"] = P.native(_exactly(m, m.astype(np.float16), "material"))
    return out


def twin_failures(res: dict) -> list[str]:
    """Every "<label> [native]" output of run_frame(..., native=...) that is not bit-identical to the output of <label>, one message each."""
    bad = []
    for label, (got, _) in res.items():
        if not label.endswith(NATIVE):
            continue
        want = res[label[:-len(NATIVE)]][0]
        if got.shape != want.shape:
            bad.append(f"{label}: shape {got.shape} vs {want.shape}")
            continue
        diff = got.view(np.uint32) != want.view(np.uint32)
        if diff.any():
            i = tuple(int(k) for k in np.argwhere(diff)[0])
            bad.append(f"{label}: {int(diff.sum())} values differ from the fp32 planes' output, first at {i}: {got[i]!r} vs {want[i]!r}")
    return bad


SENTINEL = 1234.5     # row-range outputs are pre-filled with it (77 for the 8-bit ones)


def row_range_failures(P: Planes, cases: list, rng: np.random.Generator) -> list[str]:
    """`cases`: (name, [(h, w, ch, dtype) of the outputs], launch(rows, output refs) -> status) for passes that write one output
    texel per invocation. Each pass is called on the whole frame, on rows [y0, y1) with a random odd y0 (the 2 x 2 quad kernels see
    a range that starts mid-quad) and on the empty range [y0, y0): the partial call must compute exactly those rows of the whole
    call and leave every other row at the sentinel, the empty one must be a no-op returning DFX_OK. The fused Bloom composite +
    tone map must refuse the odd y0 and then runs from y0 - 1. One message per failure."""
    bad = []
    for name, specs, launch in cases:
        def run(r):
            outs = [P.new(h, w, ch, fill=(77 if dt == torch.uint8 else SENTINEL), dtype=dt) for h, w, ch, dt in specs]
            st = launch(r, [b.ref for b in outs])
            torch.cuda.synchronize()
            return st, [b.host() for b in outs]
        st, whole = run(capi.Rows(0, specs[0][0]))
        capi.check(st, name)
        hh = specs[0][0]
        y0 = int(rng.integers(1, hh // 2)) | 1
        y1 = int(rng.integers(y0 + 1, hh))
        if name == "bloom_composite_tonemap":
            assert launch(capi.Rows(y0, y1), [P.new(*specs[0][:3]).ref]) == capi.DFX_ERR_UNSUPPORTED, "odd y0 must be refused"
            y0 -= 1
        st, part = run(capi.Rows(y0, y1))
        capi.check(st, f"{name} rows [{y0}, {y1})")
        for k, (a, b) in enumerate(zip(part, whole)):
            sentinel = 77 if specs[k][3] == torch.uint8 else SENTINEL
            if not np.array_equal(a[y0:y1].view(np.uint32), b[y0:y1].view(np.uint32)):
                bad.append(f"{name} output {k}: rows [{y0}, {y1}) differ from the full-frame call")
            if not (np.all(a[:y0] == sentinel) and np.all(a[y1:] == sentinel)):
                bad.append(f"{name} output {k}: rows outside [{y0}, {y1}) were written")
        st, empty = run(capi.Rows(y0, y0))
        if st != capi.DFX_OK or not all(np.all(e == (77 if s[3] == torch.uint8 else SENTINEL)) for e, s in zip(empty, specs)):
            bad.append(f"{name}: the empty range [{y0}, {y0}) must be a no-op returning DFX_OK (status {st})")
    return bad


def run_frame(o: op.Oracle, fr: dict, v: Variant, layout: str = "tight", planes: Planes | None = None,
              stages: int | None = None, native: str | None = None) -> dict[str, tuple[np.ndarray, np.ndarray]]:
    """`o` holds the history of the frames before `fr` (run with o.frame()); `fr` must be the next frame of the sequence. Outputs
    that a pass leaves untouched where its mask is off (S2 roughness, S5, S6) are pre-filled with the oracle's contents from
    before the pass, so they compare bit for bit there. `planes` (optional) receives the allocations for a padding check.

    `stages` (oracle stage bits) limits the call to the separate passes of those stages, which is what the full-size tests can
    afford: the sections of the other stages are left out on both sides, so the oracle must already hold this frame's planes the
    selected sections read (run those stages with o.frame() first). The fused entries and the Bloom launch shapes run only when
    `stages` is None (the whole frame of `v`).

    `native` ("rg8" / "rgba16", see native_gbuffer): every launch that reads colour, normal, motion or material runs again on the
    native planes, the other inputs unchanged, and its output is recorded as "<label> [native]" (P1-P3, S2, S4-S7, A2, A7, A8,
    C1, the fused compose + TAA), plus TAA on the colour itself: "T1 taa (colour)" (fp32, against the oracle's TAA on that
    colour) and its twin, the RGBA16F TAA a chain runs without COMPOSE in its stage mask. The frame must hold values the native
    formats hold exactly."""
    L = capi.load()
    P = planes if planes is not None else Planes(layout)
    res: dict[str, tuple[np.ndarray, np.ndarray]] = {}
    whole = stages is None
    stages = v.stages() if whole else stages
    rev = capi.PLANE_FLAG_REVERSED_DEPTH if v.reversed_depth else 0
    ci, pi = fr["frame"] & 1, (fr["frame"] + 1) & 1
    o.set_inputs(fr)
    g = o.get
    cams = P.cameras(fr["curr_camera"], fr["prev_camera"])
    H, W = fr["depth"].shape

    def ok(status, what):
        capi.check(status, what)

    # ---------------- PostFXContext ----------------
    depth_np = g("depth")
    depth, motion, normal, color, material = P.up(depth_np, rev), P.up(g("motion")), P.up(g("normal")), P.up(g("color")), P.up(g("material"))
    nat = native_gbuffer(P, g, native) if native is not None else None

    def twins(name: str, wide: Buf) -> list[tuple[str, Buf]]:
        """(label suffix, plane): the fp32 G-buffer plane `name`, and with `native` its native twin."""
        return [("", wide)] + ([(NATIVE, nat[name])] if nat else [])

    if stages & op.STAGE_POSTFX:
        tables = torch.from_numpy(np.fromfile(op.TABLES, np.uint8)).cuda()
        P.keep.append(tables)
        xy, zw = P.new(128, 128, 2), P.new(128, 128, 2)
        ok(L.dfx_pass_blue_noise(None, C.c_void_p(tables.data_ptr()), fr["frame"], xy.ref, zw.ref), "blue noise")
        o.run("blue_noise")
        res["P0 blue_noise.xy"], res["P0 blue_noise.zw"] = (xy.host(), g("bn_xy")), (zw.host(), g("bn_zw"))
        prev_in = P.up(g("prev_depth_in"), rev)
        o.run("reprojected_depth"), o.run("closest_motion"), o.run("previous_depth")
        for sfx, mv in twins("motion", motion):
            rp, cm, pd = P.new(H, W, flags=rev), P.new(H, W, 2), P.new(H, W, flags=rev)
            ok(L.dfx_pass_postfx_prepare(None, cams, depth.ref, prev_in.ref, mv.ref, rp.ref, cm.ref, pd.ref, rows(H)), "postfx prepare" + sfx)
            res["P1 reprojected_depth" + sfx], res["P2 closest_motion" + sfx], res["P3 previous_depth" + sfx] = \
                (rp.host(), g("reproj_depth")), (cm.host(), g("closest_motion")), (pd.host(), g("prev_depth"))
    reproj, closest, prev_depth = P.up(g("reproj_depth"), rev), P.up(g("closest_motion")), P.up(g("prev_depth"), rev)

    # ---------------- ScreenSpaceReflection ----------------
    if stages & op.STAGE_SSR:
        A = v.ssr
        half = bool(v.ssr_flags & capi.SSR_FLAG_HALF_RESOLUTION)
        o.run("ssr_hiz")
        hiz = _levels(o, "ssr_hiz")
        lv = [depth] + [P.like(m) for m in hiz[1:]]
        ok(L.dfx_pass_ssr_hiz(None, C.byref(P.pyramid(lv)), rows(H)), "ssr hiz")
        for i in range(1, len(hiz)):
            res[f"S1 ssr_hiz.{i}"] = (lv[i].host(), hiz[i])
        hiz_pyr = P.pyramid([depth] + [P.up(m) for m in hiz[1:]])
        rough_before = g("ssr_roughness")
        o.run("ssr_mask")
        rough_np, maskf = g("ssr_roughness"), g("ssr_mask")
        for sfx, mat in twins("material", material):
            r_out, m_out = P.up(rough_before), P.new(H, W, fill=7, dtype=torch.uint8)
            ok(L.dfx_pass_ssr_mask_roughness(None, C.byref(A), mat.ref, depth.ref, r_out.ref, m_out.ref, rows(H)), "ssr mask" + sfx)
            res["S2 ssr_roughness" + sfx], res["S2 ssr_stencil" + sfx] = (r_out.host(), rough_np), (m_out.host(), maskf)
        rough, mask = P.up(rough_np), P.mask(maskf)
        trace_mask = mask
        if half:
            o.run("ssr_downsample_mask")
            mh = g("ssr_mask_half")
            out = P.new(mh.shape[0], mh.shape[1], fill=7, dtype=torch.uint8)
            ok(L.dfx_pass_ssr_downsample_mask(None, C.byref(A), rough.ref, depth.ref, out.ref, rows(mh.shape[0])), "ssr downsample mask")
            res["S3 ssr_stencil_half"] = (out.host(), mh)
            trace_mask = P.mask(mh)
        o.run("ssr_intersect")
        rad_np, rdir_np = g("ssr_radiance"), g("ssr_raydir")
        bn_xy = P.up(g("bn_xy"))
        gbuf = [(motion, normal, color)] + ([(nat["motion"], nat["normal"], nat["color"])] if nat else [])
        for sfx, (mv, nrm, col) in zip(("", NATIVE), gbuf):
            rad, rdir = P.like(rad_np, fill=-1.0), P.like(rdir_np, fill=-1.0)
            ok(L.dfx_pass_ssr_intersect(None, cams, C.byref(A), v.ssr_flags, col.ref, nrm.ref, rough.ref, trace_mask.ref, bn_xy.ref, C.byref(hiz_pyr),
                                        mv.ref, rad.ref, rdir.ref, rows(rad_np.shape[0])), "ssr intersect" + sfx)
            res["S4 ssr_intersect.radiance" + sfx], res["S4 ssr_intersect.raydir_pdf" + sfx] = (rad.host(), rad_np), (rdir.host(), rdir_np)
        pre = [g("ssr_resolved_rad"), g("ssr_resolved_var"), g("ssr_resolved_depth")]
        o.run("ssr_spatial")
        want = [g("ssr_resolved_rad"), g("ssr_resolved_var"), g("ssr_resolved_depth")]
        rdir_in, rad_in = P.up(rdir_np), P.up(rad_np)
        for sfx, nrm in twins("normal", normal):
            outs = [P.up(p) for p in pre]
            ok(L.dfx_pass_ssr_spatial(None, cams, C.byref(A), rough.ref, mask.ref, nrm.ref, depth.ref, rdir_in.ref, rad_in.ref,
                                      *[b.ref for b in outs], rows(H)), "ssr spatial" + sfx)
            for n_, b_, w_ in zip(("radiance", "variance", "depth"), outs, want):
                res[f"S5 ssr_spatial.{n_}{sfx}"] = (b_.host(), w_)
        pre = [g(f"ssr_radhist{ci}"), g(f"ssr_varhist{ci}")]
        ins = [P.up(want[2]), reproj, P.up(want[0]), P.up(want[1]), prev_depth, P.up(g(f"ssr_radhist{pi}")), P.up(g(f"ssr_varhist{pi}"))]
        o.run("ssr_temporal")
        acc = [g(f"ssr_radhist{ci}"), g(f"ssr_varhist{ci}")]
        for sfx, mv in twins("motion", motion):
            outs = [P.up(p) for p in pre]
            ok(L.dfx_pass_ssr_temporal(None, cams, C.byref(A), mask.ref, mv.ref, *[b.ref for b in ins], *[b.ref for b in outs], rows(H)), "ssr temporal" + sfx)
            res["S6 ssr_temporal.radiance" + sfx], res["S6 ssr_temporal.variance" + sfx] = (outs[0].host(), acc[0]), (outs[1].host(), acc[1])
        o.run("ssr_bilateral")
        ssr_out_np = g("ssr_out")
        acc_rad, acc_var = P.up(acc[0]), P.up(acc[1])
        for sfx, nrm in twins("normal", normal):
            out = P.like(ssr_out_np, fill=5.0)
            ok(L.dfx_pass_ssr_bilateral(None, cams, C.byref(A), mask.ref, depth.ref, nrm.ref, rough.ref, acc_rad.ref, acc_var.ref, out.ref, rows(H)),
               "ssr bilateral" + sfx)
            res["S7 ssr_bilateral" + sfx] = (out.host(), ssr_out_np)

    # ---------------- ScreenSpaceAmbientOcclusion ----------------
    if stages & op.STAGE_SSAO:
        S = v.ssao
        S.Algorithm = v.ssao_algorithm
        ao_half = bool(v.ssao_flags & capi.SSAO_FLAG_HALF_RESOLUTION)
        src_flags = rev | (2 if v.ssao_flags & 1 else 0)                      # DFX_PLANE_FLAG_HALF_PRECISION_DEPTH
        src = depth_np
        if ao_half:
            o.run("ssao_downsample")
            src = g("ssao_checker")
            out = P.like(src, fill=-3.0)
            ok(L.dfx_pass_ssao_downsample_depth(None, depth.ref, out.ref, rows(src.shape[0])), "ssao downsample")
            res["A0 ssao_downsample"] = (out.host(), src)
        o.run("ssao_prefilter")
        pre = _levels(o, "ssao_pre")
        lv = [P.up(src, src_flags)] + [P.like(m, fill=-3.0) for m in pre[1:]]
        ok(L.dfx_pass_ssao_prefilter_depth(None, cams, C.byref(S), C.byref(P.pyramid(lv)), rows(src.shape[0])), "ssao prefilter")
        for i in range(1, len(pre)):
            res[f"A1 ssao_prefilter.{i}"] = (lv[i].host(), pre[i])
        o.run("ssao_ao")
        occ_np = g("ssao_occ")
        pyr = P.pyramid([P.up(pre[0], src_flags)] + [P.up(m) for m in pre[1:]])
        bn_zw = P.up(g("bn_zw"))
        for sfx, nrm in twins("normal", normal):
            out = P.like(occ_np, fill=-3.0)
            ok(L.dfx_pass_ssao_ambient_occlusion(None, cams, C.byref(S), C.byref(pyr), nrm.ref, bn_zw.ref, out.ref, rows(occ_np.shape[0])), "ssao ao" + sfx)
            res["A2 ssao_ao" + sfx] = (out.host(), occ_np)
        if ao_half:
            o.run("ssao_upsample")
            up_np = g("ssao_occ_up")
            out = P.like(up_np, fill=-3.0)
            ok(L.dfx_pass_ssao_upsample(None, cams, depth.ref, P.up(occ_np).ref, out.ref, rows(H)), "ssao upsample")
            res["A4 ssao_upsample"] = (out.host(), up_np)
            occ_np = up_np
        ins = [P.up(occ_np), P.up(g(f"ssao_hist{pi}")), P.up(g(f"ssao_histlen{pi}")), reproj, prev_depth, closest]
        o.run("ssao_temporal")
        acc_o, hlen = g("ssao_acc"), g(f"ssao_histlen{ci}")
        oo, oh = P.new(H, W, fill=-3.0), P.new(H, W, fill=-3.0)
        ok(L.dfx_pass_ssao_temporal(None, cams, C.byref(S), *[b.ref for b in ins], oo.ref, oh.ref, rows(H)), "ssao temporal")
        res["A5 ssao_temporal.occlusion"], res["A5 ssao_temporal.history"] = (oo.host(), acc_o), (oh.host(), hlen)
        o.run("ssao_convolute")
        co, cd = _levels(o, "ssao_conv_occ"), _levels(o, "ssao_conv_depth")
        lo = [P.up(co[0])] + [P.like(m, fill=-3.0) for m in co[1:]]
        ld = [depth] + [P.like(m, fill=-3.0) for m in cd[1:]]
        ok(L.dfx_pass_ssao_convolute(None, C.byref(P.pyramid(lo)), C.byref(P.pyramid(ld)), rows(H)), "ssao convolute")
        for i in range(1, len(co)):
            res[f"A6 ssao_convolute.occlusion.{i}"], res[f"A6 ssao_convolute.depth.{i}"] = (lo[i].host(), co[i]), (ld[i].host(), cd[i])
        o.run("ssao_resample")
        rs = g("ssao_resampled")
        hl = P.up(hlen)
        po, pdp = P.pyramid([P.up(m) for m in co]), P.pyramid([depth] + [P.up(m) for m in cd[1:]])
        for sfx, nrm in twins("normal", normal):
            out = P.new(H, W, fill=-3.0)
            ok(L.dfx_pass_ssao_resample(None, cams, C.byref(po), C.byref(pdp), hl.ref, nrm.ref, out.ref, rows(H)), "ssao resample" + sfx)
            res["A7 ssao_resample" + sfx] = (out.host(), rs)
        o.run("ssao_spatial")
        ao_np = g("ssao_out")
        rs_in = P.up(rs)
        for sfx, nrm in twins("normal", normal):
            out = P.new(H, W, fill=-3.0)
            ok(L.dfx_pass_ssao_spatial(None, cams, C.byref(S), rs_in.ref, hl.ref, depth.ref, nrm.ref, out.ref, rows(H)), "ssao spatial" + sfx)
            res["A8 ssao_spatial" + sfx] = (out.host(), ao_np)

    # ---------------- compose -> TAA (separate and fused) ----------------
    if stages & op.STAGE_COMPOSE:
        ssr_out, ao = P.up(g("ssr_out")), P.up(g("ssao_out"))
        scales = (C.c_float(1.0), C.c_float(1.0))                             # the oracle's compose scales (orc_create)
        o.run("compose")
        for sfx, col in twins("color", color):
            out = P.like(g("composed"), fill=-3.0)
            ok(L.dfx_pass_compose(None, col.ref, ssr_out.ref, ao.ref, *scales, out.ref, rows(H)), "compose" + sfx)
            res["C1 compose" + sfx] = (out.host(), g("composed"))
    if stages & op.STAGE_TAA:
        composed = g("composed")
        o.set("taa_in", composed)
        v.taa.ResetAccumulation = 0                                           # consecutive frame (TemporalAntiAliasing.cpp:125-128)
        o.set_taa(v.taa, v.taa_flags)
        prev_acc = g(f"taa_accum{pi}")
        o.run("taa")
        acc_t = g(f"taa_accum{ci}")
        taa_ins = [P.up(prev_acc), closest, reproj, prev_depth]
        out = P.like(acc_t, fill=-3.0)
        ok(L.dfx_pass_taa(None, cams, C.byref(v.taa), v.taa_flags, P.up(composed).ref, *[b.ref for b in taa_ins], out.ref, rows(H)), "taa")
        res["T1 taa"] = (out.host(), acc_t)
        if whole:
            for sfx, col in twins("color", color):
                out = P.like(acc_t, fill=-3.0)
                ok(L.dfx_pass_compose_taa(None, cams, C.byref(v.taa), v.taa_flags, col.ref, ssr_out.ref, ao.ref, *scales, *[b.ref for b in taa_ins],
                                          out.ref, rows(H)), "compose + taa" + sfx)
                res["T1 compose_taa (fused)" + sfx] = (out.host(), acc_t)
        if nat:
            # TAA on the G-buffer colour itself (a chain without COMPOSE in its stage mask); the oracle's state is put back afterwards
            o.set("taa_in", g("color"))
            o.run("taa")
            acc_c = g(f"taa_accum{ci}")
            o.set("taa_in", composed), o.set(f"taa_accum{ci}", acc_t)
            for sfx, col in twins("color", color):
                out = P.like(acc_t, fill=-3.0)
                ok(L.dfx_pass_taa(None, cams, C.byref(v.taa), v.taa_flags, col.ref, *[b.ref for b in taa_ins], out.ref, rows(H)), "taa (colour)" + sfx)
                res["T1 taa (colour)" + sfx] = (out.host(), acc_c)
        post_in = acc_t

    # ---------------- DepthOfField ----------------
    if stages & op.STAGE_DOF:
        a, f = v.dof_attribs, v.dof_flags
        o.set("dof_in", post_in)
        pin = P.up(post_in)
        o.run("dof_coc")
        coc = g("dof_coc")
        out = P.like(coc, fill=-3.0)
        ok(L.dfx_pass_dof_coc(None, cams, C.byref(a), depth.ref, out.ref, rows(H)), "dof coc")
        res["D1 dof_coc"] = (out.host(), coc)
        if f & capi.DOF_FLAG_TEMPORAL_SMOOTHING:
            prevc = g(f"dof_coc_temporal{pi}")
            o.run("dof_temporal")
            tc = g(f"dof_coc_temporal{ci}")
            out = P.like(tc, fill=-3.0)
            ok(L.dfx_pass_dof_temporal_coc(None, cams, C.byref(a), P.up(coc).ref, P.up(prevc).ref, closest.ref, out.ref, rows(H)), "dof temporal")
            res["D2 dof_temporal"] = (out.host(), tc)
            coc = tc
        cb = P.up(coc)
        o.run("dof_separated")
        d0 = g("dof_dilation0")
        out = P.like(d0, fill=-3.0)
        ok(L.dfx_pass_dof_separated_coc(None, cb.ref, out.ref, rows(H)), "dof separated")
        res["D3 dof_separated"] = (out.host(), d0)
        o.run("dof_dilation")
        dl = [g(f"dof_dilation{i}") for i in range(4)]
        for i in range(3):
            out = P.like(dl[i + 1], fill=-3.0)
            ok(L.dfx_pass_dof_dilation(None, P.up(dl[i]).ref, out.ref, rows(dl[i + 1].shape[0])), "dof dilation")
            res[f"D4 dof_dilation.{i + 1}"] = (out.host(), dl[i + 1])
        o.run("dof_blur_x")
        bx = g("dof_dilation_tmp")
        out = P.like(bx, fill=-3.0)
        ok(L.dfx_pass_dof_blur_coc(None, P.up(dl[3]).ref, 0, out.ref, rows(bx.shape[0])), "dof blur x")
        res["D5 dof_blur_x"] = (out.host(), bx)
        o.run("dof_blur_y")
        by = g("dof_dilation3")
        out = P.like(by, fill=-3.0)
        ok(L.dfx_pass_dof_blur_coc(None, P.up(bx).ref, 1, out.ref, rows(by.shape[0])), "dof blur y")
        res["D6 dof_blur_y"] = (out.host(), by)
        o.run("dof_prefilter")
        p0, p1 = g("dof_pre0"), g("dof_pre1")
        o0, o1 = P.like(p0, fill=-3.0), P.like(p1, fill=-3.0)
        ok(L.dfx_pass_dof_prefilter(None, pin.ref, cb.ref, P.up(by).ref, o0.ref, o1.ref, rows(p0.shape[0])), "dof prefilter")
        res["D7 dof_prefilter.near"], res["D7 dof_prefilter.far"] = (o0.host(), p0), (o1.host(), p1)
        o.run("dof_bokeh_first")
        b0, b1 = g("dof_bokeh0"), g("dof_bokeh1")
        o0, o1 = P.like(b0, fill=-3.0), P.like(b1, fill=-3.0)
        ok(L.dfx_pass_dof_bokeh(None, cams, C.byref(a), f, 0, P.up(p0).ref, P.up(p1).ref, pin.ref, o0.ref, o1.ref, rows(b0.shape[0])), "dof bokeh 1")
        res["D8 dof_bokeh_first.near"], res["D8 dof_bokeh_first.far"] = (o0.host(), b0), (o1.host(), b1)
        o.run("dof_bokeh_second")
        s0, s1 = g("dof_pre0"), g("dof_pre1")
        o0, o1 = P.like(s0, fill=-3.0), P.like(s1, fill=-3.0)
        ok(L.dfx_pass_dof_bokeh(None, cams, C.byref(a), f, 1, P.up(b0).ref, P.up(b1).ref, None, o0.ref, o1.ref, rows(s0.shape[0])), "dof bokeh 2")
        res["D9 dof_bokeh_second.near"], res["D9 dof_bokeh_second.far"] = (o0.host(), s0), (o1.host(), s1)
        o.run("dof_postfilter")
        f0, f1 = g("dof_bokeh0"), g("dof_bokeh1")
        o0, o1 = P.like(f0, fill=-3.0), P.like(f1, fill=-3.0)
        ok(L.dfx_pass_dof_postfilter(None, P.up(s0).ref, P.up(s1).ref, o0.ref, o1.ref, rows(f0.shape[0])), "dof postfilter")
        res["D10 dof_postfilter.near"], res["D10 dof_postfilter.far"] = (o0.host(), f0), (o1.host(), f1)
        o.run("dof_combine")
        dout = g("dof_out")
        out = P.like(dout, fill=-3.0)
        ok(L.dfx_pass_dof_combine(None, C.byref(a), pin.ref, P.up(f0).ref, P.up(f1).ref, out.ref, rows(H)), "dof combine")
        res["D11 dof_combine"] = (out.host(), dout)
        post_in = dout

    # ---------------- Bloom ----------------
    if stages & op.STAGE_BLOOM:
        B = v.bloom
        o.set("bloom_in", post_in)
        o.run("bloom")
        n = _count(o, "bloom_down")
        dn, up = [g(f"bloom_down{i}") for i in range(n)], [g(f"bloom_up{i}") for i in range(n - 1)]
        pin = P.up(post_in)
        out = P.like(dn[0], fill=-3.0)
        ok(L.dfx_pass_bloom_prefilter(None, C.byref(B), pin.ref, out.ref, rows(dn[0].shape[0])), "bloom prefilter")
        res["B1 bloom_prefilter"] = (out.host(), dn[0])
        dn_dev = [P.up(m) for m in dn]
        for i in range(1, n):
            out = P.like(dn[i], fill=-3.0)
            ok(L.dfx_pass_bloom_downsample(None, dn_dev[i - 1].ref, out.ref, rows(dn[i].shape[0])), "bloom downsample")
            res[f"B2 bloom_downsample.{i}"] = (out.host(), dn[i])
        top = n - 1
        for i in range(top, 0, -1):
            out = P.like(up[i - 1], fill=-3.0)
            coarser = P.up(up[i]) if i != top else dn_dev[i]
            ok(L.dfx_pass_bloom_upsample(None, dn_dev[i - 1].ref, coarser.ref, out.ref, rows(up[i - 1].shape[0])), "bloom upsample")
            res[f"B3 bloom_upsample.{i - 1}"] = (out.host(), up[i - 1])
        # the two pyramid launch shapes: every level after the first in one thread-block cluster (tail) / one cooperative grid (levels)
        for shape in ("tail", "levels") if whole else ():
            dn_o, up_o = [dn_dev[0]] + [P.like(m, fill=-3.0) for m in dn[1:]], [P.like(m, fill=-3.0) for m in dn]
            pd_, pu_ = P.array(dn_o), P.array(up_o)
            if shape == "tail":
                L.dfx_tune_set(b"bloom_tail", 1), L.dfx_tune_set(b"bloom_tail_texels", 1 << 30)
                try:
                    first = L.dfx_bloom_tail_first_level(pd_, n)
                finally:
                    L.dfx_tune_unset(b"bloom_tail"), L.dfx_tune_unset(b"bloom_tail_texels")
                assert first == 1, first
                ok(L.dfx_pass_bloom_tail(None, pd_, pu_, 1, n), "bloom tail")
            else:
                ws = torch.zeros(16, dtype=torch.int32, device="cuda")
                P.keep.append(ws)
                ok(L.dfx_pass_bloom_levels(None, pd_, pu_, 1, n, C.c_void_p(ws.data_ptr())), "bloom levels")
                timed_out = C.c_int32(-1)
                ok(L.dfx_bloom_levels_check(C.c_void_p(ws.data_ptr()), C.byref(timed_out)), "bloom levels check")
                assert timed_out.value == 0
            for i in range(1, n):
                res[f"B2 bloom_{shape}.down.{i}"] = (dn_o[i].host(), dn[i])
            for i in range(n - 1):
                res[f"B3 bloom_{shape}.up.{i}"] = (up_o[i].host(), up[i])
        bout = g("bloom_out")
        up0 = P.up(up[0])
        out = P.like(bout, fill=-3.0)
        ok(L.dfx_pass_bloom_composite(None, C.byref(B), pin.ref, up0.ref, out.ref, rows(H)), "bloom composite")
        res["B4 bloom_composite"] = (out.host(), bout)

    # ---------------- ToneMapping + sRGB (separate and fused with the Bloom composite) ----------------
    if stages & op.STAGE_TONEMAP:
        T = v.tonemap
        T.iToneMappingMode = v.tonemap_mode
        bout = g("bloom_out")
        o.set("tonemap_in", bout)
        o.run("tonemap")
        ldr = g("ldr")
        out = P.like(ldr, fill=-3.0)
        ok(L.dfx_pass_tonemap(None, C.byref(T), C.c_float(v.ave_log_lum), int(v.to_srgb), P.up(bout).ref, out.ref, rows(H)), "tonemap")
        res["M1 tonemap"] = (out.host(), ldr)
        if whole:
            out = P.like(ldr, fill=-3.0)
            st = L.dfx_pass_bloom_composite_tonemap(None, C.byref(B), C.byref(T), C.c_float(v.ave_log_lum), int(v.to_srgb), pin.ref, up0.ref, out.ref,
                                                    rows(H))
            if up[0].shape[0] * 2 == H and up[0].shape[1] * 2 == W:
                ok(st, "bloom composite + tonemap")
                res["M1 bloom_composite_tonemap (fused)"] = (out.host(), ldr)
            else:                                                             # odd frame size: no exact 2:1 level, the caller runs B4 and M1
                assert st == capi.DFX_ERR_UNSUPPORTED, st
    torch.cuda.synchronize()
    return res


# =====================================================================================================================
# comparison of a run_frame result
# =====================================================================================================================
FLOOR_PX = 4          # drawn configurations: every outlier budget allows at least this many pixels (0.5 % of an 8 x 8 frame is less than one)
PSNR_MIN_PX = 4096    # drawn configurations: below this many pixels one permitted outlier dominates the mean square error: PSNR floors apply above it
EXACT = dict(exact=True)


def tolerance(label: str, v: Variant, drawn: bool) -> dict:
    """The comparison of one pass output: keyword arguments of helpers.assert_close, or
      exact    bit for bit;                   wrap     max difference of fractions (0.99999 and 0.0 are neighbours);
      tonemap  max abs RGB difference relative to max(1, peak), alpha bit for bit;
      masked   compared where the SSR mask is set and bit for bit elsewhere (S5 / S6 keep their content there, S7 clears it to 0);
    and in addition
      rgb      alpha left out;                alpha    alpha compared on its own, without Reinhard, to these bounds;
      scale    both sides divided by it;      ones     the fraction of pixels where AO == 1 on one side only stays below it.
    `drawn` = a configuration of driver.random_variant; False = the default attribute values, whose bounds are tighter where a drawn
    setting moves more pixels (the comments give the reason) and have no pixel floor (FLOOR_PX, PSNR_MIN_PX)."""
    ssr_half, ao_half, vbao = bool(v.ssr_flags & capi.SSR_FLAG_HALF_RESOLUTION), bool(v.ssao_flags & capi.SSAO_FLAG_HALF_RESOLUTION), v.ssao_algorithm == 2
    table = {
        "P0": dict(wrap=1e-4),
        "P1": dict(tol=2e-6), "P2": EXACT, "P3": EXACT,
        "S1": EXACT, "S2": EXACT, "S3": EXACT,
        "S5 ssr_spatial.radiance": dict(tol=5e-3, max_outliers=5e-3, hdr=True, masked=True) if ssr_half else
        dict(tol=2e-3, max_outliers=3e-3, min_psnr=55.0, hdr=True, masked=True),
        "S5 ssr_spatial.variance": dict(tol=2e-3, max_outliers=3e-3, hdr=True, masked=True),
        "S5 ssr_spatial.depth": dict(tol=2e-6, max_outliers=3e-3, masked=True),
        "S6 ssr_temporal.radiance": dict(tol=2e-3, max_outliers=5e-3, min_psnr=50.0, hdr=True, masked=True),
        "S6 ssr_temporal.variance": dict(tol=2e-3, max_outliers=5e-3, hdr=True, masked=True),
        "S7": dict(tol=2e-3, max_outliers=3e-3, min_psnr=55.0, hdr=True, masked=True),
        "A0": EXACT,
        "A1": dict(tol=2e-6, max_outliers=1e-3, min_psnr=100.0),
        # GTAO / HBAO: 3 % outliers where the default settings allow 0.5 % (the PSNR floor stays). A tap's mip is
        # log2(radius in texels) - DepthMIPSamplingOffset, rounded: the drawn offsets (down to 1) and radii (up to 3 x 2.5) send most
        # taps to the coarse mips, where a tap on a texel edge that rounds the other way moves by a whole coarse texel. Observed on an
        # H100: 1.9 % at HBAO, offset 1.16, radius 1.84 x 2.32, 153 x 30; the default settings stay within 0.5 %.
        "A2": dict(tol=2e-3, max_outliers=3e-2, min_psnr=40.0) if vbao else dict(tol=2e-3, max_outliers=3e-2, min_psnr=55.0),
        "A4": dict(tol=1e-4, max_outliers=1e-3, min_psnr=60.0),
        "A5 ssao_temporal.occlusion": dict(tol=1e-4, max_outliers=2e-3, min_psnr=60.0),
        # 1 % outliers where the default settings allow 0.2 %: the history length is reset or kept by the 1 % depth-similarity test, a
        # discrete decision per pixel; on the small random frames (4 500 pixels) the few pixels whose decision flips weigh more
        # (observed on an H100: 0.98 % at 153 x 30).
        "A5 ssao_temporal.history": dict(scale=16.0, tol=1e-4, max_outliers=1e-2),
        "A6": dict(tol=1e-6),
        "A7": dict(tol=2e-4, max_outliers=2e-3, min_psnr=60.0),
        "A8": dict(tol=2e-4, max_outliers=2e-3, min_psnr=60.0),
        "C1": dict(tol=1e-5, hdr=True),
        "T1": dict(tol=1e-4, max_outliers=1e-2, min_psnr=70.0, hdr=True),
        "D1": dict(tol=2e-5), "D2": dict(tol=2e-5, max_outliers=1e-3), "D3": EXACT, "D4": EXACT, "D5": dict(tol=1e-6), "D6": dict(tol=1e-6),
        "D7": dict(tol=1e-4, max_outliers=2e-3, hdr=True), "D8": dict(tol=1e-4, max_outliers=2e-3, hdr=True),
        "D9": dict(tol=1e-4, max_outliers=2e-3, hdr=True), "D10": dict(tol=1e-4, max_outliers=2e-3, hdr=True),
        # RGB: the drawn configurations are the ones the oracle is pinned at against the reference, whose R11G11B10 Bloom chain has no alpha
        "D11": dict(tol=1e-4, max_outliers=2e-3, min_psnr=70.0, hdr=True, rgb=True),
        "B1": dict(tol=1e-4, max_outliers=1e-4, min_psnr=90.0, hdr=True, rgb=True),
        "B2": dict(tol=1e-5, min_psnr=95.0, hdr=True, rgb=True), "B3": dict(tol=1e-5, min_psnr=95.0, hdr=True, rgb=True),
        "B4": dict(tol=1e-5, min_psnr=100.0, hdr=True, rgb=True),
        "M1": dict(tonemap=2e-5),
    }
    if not drawn:
        table.update({
            # half resolution: GTAO, on a quarter of the pixels
            "A2": dict(tol=2e-3, max_outliers=2e-3, min_psnr=50.0) if ao_half else
            dict(tol=2e-3, max_outliers=3e-2, min_psnr=40.0, ones=1e-3) if vbao else dict(tol=2e-3, max_outliers=5e-3, min_psnr=55.0, ones=1e-3),
            "A5 ssao_temporal.history": dict(scale=16.0, tol=1e-4, max_outliers=2e-3, min_psnr=50.0),
            "T1": dict(tol=1e-4, max_outliers=1e-2, min_psnr=70.0, hdr=True, alpha=dict(tol=1e-4, max_outliers=1e-2)),
            "D11": dict(tol=1e-4, max_outliers=2e-3, min_psnr=70.0, hdr=True),
            "B1": dict(tol=1e-4, max_outliers=1e-4, min_psnr=90.0, hdr=True),
            "B2": dict(tol=1e-5, min_psnr=95.0, hdr=True), "B3": dict(tol=1e-5, min_psnr=95.0, hdr=True),           # the launch shapes
            "B2 bloom_downsample": dict(tol=1e-5, min_psnr=100.0, hdr=True), "B3 bloom_upsample": dict(tol=1e-5, min_psnr=100.0, hdr=True),
            "B4": dict(tol=1e-5, min_psnr=100.0, hdr=True),
        })
    key = max((k for k in table if label.startswith(k)), key=len)
    return table[key]


def _check(label: str, got: np.ndarray, want: np.ndarray, v: Variant, ssr_mask: np.ndarray | None, drawn: bool) -> str | None:
    """None when `got` passes the comparison `tolerance(label, v, drawn)` prescribes, else the reason."""
    spec = dict(tolerance(label, v, drawn))
    if spec.pop("rgb", False):
        got, want = got[..., :3], want[..., :3]
    if got.shape != want.shape:
        return f"{label}: shape {got.shape} vs {want.shape}"
    fin = np.isfinite(want)
    if not np.isfinite(got)[fin].all():
        return f"{label}: {int((~np.isfinite(got) & fin).sum())} non-finite values where the oracle's are finite"
    if spec.pop("exact", False):
        if np.array_equal(got.view(np.uint32), want.view(np.uint32)):
            return None
        d = np.abs(got.astype(np.float64) - want)
        return f"{label}: not bit-exact ({int((d > 0).sum())} values differ, max abs {np.nanmax(d):.3e})"
    if "wrap" in spec:
        d = np.abs(got - want)
        d = np.minimum(d, 1.0 - d)
        return None if d.max() < spec["wrap"] else f"{label}: max wrapped difference {d.max():.3e}"
    if "tonemap" in spec:
        scale = max(1.0, float(np.abs(want[..., :3]).max()))
        err = np.abs(got[..., :3] - want[..., :3]).max()
        if not np.array_equal(got[..., 3], want[..., 3]) or err > spec["tonemap"] * scale:
            return f"{label}: max abs {err:.3e} (allowed {spec['tonemap'] * scale:.3e}), alpha equal: {np.array_equal(got[..., 3], want[..., 3])}"
        return None
    ones = spec.pop("ones", None)
    if ones is not None and np.mean((got == 1.0) != (want == 1.0)) >= ones:
        return f"{label}: AO == 1 on one side only at {np.mean((got == 1.0) != (want == 1.0)):.4%} of the pixels (allowed < {ones:.4%})"
    mask = None
    if spec.pop("masked", False):
        mask = ssr_mask > 0
        outside = ~mask if got.ndim == 2 else np.broadcast_to(~mask[..., None], got.shape)
        if not np.array_equal(got[outside].view(np.uint32), want[outside].view(np.uint32)):
            return f"{label}: texels outside the SSR mask differ from the oracle's"
    if "scale" in spec:
        s = spec.pop("scale")
        got, want = got / s, want / s
    alpha = spec.pop("alpha", None)
    parts = [(label, got, want, spec)] if alpha is None else [(f"{label} rgb", got[..., :3], want[..., :3], spec),
                                                             (f"{label} alpha", got[..., 3], want[..., 3], dict(alpha))]
    npx = got.shape[0] * got.shape[1]
    for name, g_, w_, kw in parts:
        kw["max_outliers"] = max(kw.get("max_outliers", 0.0), (FLOOR_PX if drawn else 0) / npx)
        if drawn and npx < PSNR_MIN_PX:
            kw.pop("min_psnr", None)
        try:
            assert_close(name, g_, w_, mask=mask, **kw)
        except AssertionError as e:
            return str(e)
    return None


def _check_march(res: dict, trace: np.ndarray, drawn: bool) -> list[str]:
    """S4: the Hi-Z march is a chaotic integer walk (an ulp in the ray set-up can move a hit by a cell), so the hit decision must
    agree on 99 % of the traced rays and the rays that hit on both sides must hit the same point (98 %); pdf and radiance of those
    rays to tolerance."""
    (grad, wrad), (gdir, wdir) = res["S4 ssr_intersect.radiance"], res["S4 ssr_intersect.raydir_pdf"]
    floor_px = FLOOR_PX if drawn else 0
    m = trace > 0
    bad = []
    if not (np.all(grad[~m] == 0.0) and np.all(gdir[~m] == 0.0)):
        bad.append("S4: texels outside the trace mask must hold the clear value 0")
    ghit, whit = grad[..., 3] > 0, wrad[..., 3] > 0
    disagree = int(((ghit != whit) & m).sum())
    if disagree > max(0.01 * m.sum(), floor_px):
        bad.append(f"S4: hit decisions differ on {disagree} of {int(m.sum())} rays")
    both = m & ghit & whit
    norm = lambda a: np.linalg.norm(a[..., :3], axis=-1)  # noqa: E731
    same = both & (np.abs(norm(gdir) - norm(wdir)) < 1e-2 * (1.0 + norm(wdir)))
    if (both & ~same).sum() > max(0.02 * both.sum(), floor_px):
        bad.append(f"S4: {int((both & ~same).sum())} of {int(both.sum())} rays that hit on both sides hit different points")
    for name, g_, w_, kw in (("S4 pdf", gdir[..., 3], wdir[..., 3], dict(tol=1e-3 * max(1.0, float(np.abs(wdir[..., 3]).max())), mask=m)),
                             ("S4 radiance (same hit)", grad, wrad, dict(tol=5e-3, hdr=True, mask=same))):
        try:
            assert_close(name, g_, w_, max_outliers=max(5e-3, floor_px / m.size), **kw)
        except AssertionError as e:
            bad.append(str(e))
    return bad


def failures(res: dict, v: Variant, drawn: bool, labels: tuple[str, ...] = ("",)) -> list[str]:
    """The comparisons of a run_frame result that fail, one message each: every label that starts with one of `labels`, to the bounds
    `tolerance(label, v, drawn)` gives."""
    ssr_mask = res["S2 ssr_stencil"][1] if "S2 ssr_stencil" in res else None
    bad = []
    if "S4 ssr_intersect.radiance" in res and "S4 ssr_intersect".startswith(labels):
        bad += _check_march(res, res["S3 ssr_stencil_half"][1] if "S3 ssr_stencil_half" in res else ssr_mask, drawn)
    for label, (got, want) in res.items():
        if label.startswith(labels) and not label.startswith("S4"):
            msg = _check(label, got, want, v, ssr_mask, drawn)
            if msg:
                bad.append(msg)
    return bad


def run_sequence(seq: list[dict], v: Variant, history: int | None = None, before: int = 0, stages: int | None = None):
    """A fresh oracle for `v` runs `history` (default v.stages()) on every frame of `seq` but the last and `before` on the last;
    then run_frame steps it through the last frame. Returns (oracle, run_frame result)."""
    h, w = seq[0]["depth"].shape
    o = make_oracle(w, h, v)
    for fr in seq[:-1]:
        o.set_inputs(fr)
        o.frame(v.stages() if history is None else history)
    if before:
        o.set_inputs(seq[-1])
        o.frame(before)
    return o, run_frame(o, seq[-1], v, stages=stages)


def assert_default(res: dict, v: Variant, *labels: str) -> None:
    """The outputs whose labels start with one of `labels` (there must be some) hold the default bounds."""
    assert any(k.startswith(labels) for k in res), f"no output labelled {labels}"
    bad = failures(res, v, drawn=False, labels=labels)
    assert not bad, "\n  ".join(bad)
