"""Steps one frame through the oracle pass by pass and, beside every pass, runs the reference's own shader for that pass
(oracle/refshader, the reference HLSL compiled for the CPU) on the SAME inputs. Test infrastructure only: imported by tests/,
tests/golden/make_reference_shader_golden.py and bench.py's `--impl reference` arm (which times the shader calls).

compare_frame() returns an ordered {label: (reference_shader_output, oracle_output)}; the host-side sequencing (which plane
feeds which pass, clears, history ping-pong, per-mip draws) is the oracle's restatement of the reference's .cpp files — what
is pinned here is the per-pixel arithmetic of every pass.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from diligentfx_b200 import capi, synth
from oracle import oracle_py as op
from oracle.refshader import refsh


@dataclass
class Variant:
    reversed_depth: bool = False
    ssr_flags: int = 0             # 1 = PREVIOUS_FRAME, 2 = HALF_RESOLUTION
    ssao_flags: int = 0            # 1 = HALF_PRECISION_DEPTH, 2 = HALF_RESOLUTION
    ssao_algorithm: int = 0        # 0 GTAO, 1 HBAO, 2 VBAO
    taa_flags: int = 2             # 1 gaussian, 2 bicubic, 4 YCoCg
    tonemap_mode: int = 4
    to_srgb: bool = True
    dof: bool = False
    dof_flags: int = 0             # 1 temporal smoothing, 2 Karis inverse
    ssr: capi.SSRAttribs = field(default_factory=capi.SSRAttribs.default)
    ssao: capi.SSAOAttribs = field(default_factory=capi.SSAOAttribs.default)
    taa: capi.TAAAttribs = field(default_factory=capi.TAAAttribs.default)
    bloom: capi.BloomAttribs = field(default_factory=capi.BloomAttribs.default)
    tonemap: capi.ToneMapAttribs = field(default_factory=capi.ToneMapAttribs.default)
    dof_attribs: capi.DOFAttribs = field(default_factory=capi.DOFAttribs.default)
    ave_log_lum: float = 0.3
    lens: tuple[float, float] | None = None   # (fFocusDistance, fFStop) written into both cameras of every frame; None = synth's

    def stages(self) -> int:
        return op.STAGE_ALL | (op.STAGE_DOF if self.dof else 0)


EDGE_SIZES = [(8, 8), (17, 5), (33, 17)]   # every pyramid reaches 1 x 1 and the odd-size branches run; 8 x 8 is DoF's minimum


def _uniform(rng, lo: float, hi: float) -> float:
    return float(rng.uniform(lo, hi))


def _alpha(rng) -> float:
    """AlphaInterpolation in (0, 1]: 1 (a settled effect) half of the time."""
    return 1.0 if rng.random() < 0.5 else float(1.0 - rng.uniform(0.0, 0.95))


def random_variant(rng: np.random.Generator, size: tuple[int, int] | None = None) -> tuple[int, int, int, Variant]:
    """One seeded draw of (width, height, scene seed, Variant): frame size (or `size`), feature flags, tone-map operator and every
    attribute field the passes read. Shared by the oracle-vs-shader test and the CUDA-vs-oracle tests, so both links are checked
    at the same configurations. Combinations the reference builds no shader variant for are folded onto ones it does."""
    w, h = size if size is not None else (int(rng.integers(40, 220)), int(rng.integers(30, 130)))
    v = Variant(reversed_depth=bool(rng.random() < 0.25), ssr_flags=int(rng.integers(0, 3)), ssao_flags=int(rng.integers(0, 3)),
                ssao_algorithm=int(rng.integers(0, 3)), taa_flags=int(rng.integers(0, 8)), tonemap_mode=int(rng.integers(1, 12)),
                to_srgb=bool(rng.integers(0, 2)), dof=bool(rng.integers(0, 2)) and min(w, h) >= 8, dof_flags=int(rng.integers(0, 4)))
    if v.ssao_algorithm:
        v.ssao_flags = 0                                  # HBAO / VBAO are built for the full-resolution, full-precision path
    if v.reversed_depth:                                  # the inverted-depth shaders exist for the default SSR / GTAO path
        v.ssr_flags = v.ssao_flags = v.ssao_algorithm = 0
        v.dof = False
    s = v.ssr
    s.DepthBufferThickness, s.RoughnessThreshold = _uniform(rng, 0.005, 0.1), _uniform(rng, 0.05, 0.6)
    s.MostDetailedMip, s.IsRoughnessPerceptual, s.RoughnessChannel = int(rng.integers(0, 3)), int(rng.integers(0, 2)), int(rng.integers(0, 4))
    s.MaxTraversalIntersections = int(rng.integers(1, 17)) if rng.random() < 0.4 else int(rng.integers(17, 200))
    s.GGXImportanceSampleBias, s.SpatialReconstructionRadius = _uniform(rng, 0, 1), _uniform(rng, 0, 6)
    s.TemporalRadianceStabilityFactor, s.TemporalVarianceStabilityFactor = _uniform(rng, 0, 1), _uniform(rng, 0, 1)
    s.BilateralCleanupSpatialSigmaFactor, s.AlphaInterpolation = _uniform(rng, 0.2, 1.5), _alpha(rng)
    a = v.ssao
    a.EffectRadius, a.EffectFalloffRange, a.RadiusMultiplier = _uniform(rng, 0.2, 3), _uniform(rng, 0.1, 1), _uniform(rng, 0.5, 2.5)
    a.DepthMIPSamplingOffset, a.TemporalStabilityFactor = _uniform(rng, 1, 5), _uniform(rng, 0, 1)
    a.SpatialReconstructionRadius = _uniform(rng, 0.5, 4.0) if rng.random() < 0.5 else _uniform(rng, 4.0, 8.0)   # both sides of the tile kernel's limit
    a.AlphaInterpolation, a.BitmaskThickness = _alpha(rng), _uniform(rng, 0.05, 1)
    b = v.bloom
    b.Threshold, b.SoftTreshold, b.Intensity, b.Radius = _uniform(rng, 0, 2), _uniform(rng, 0, 1), _uniform(rng, 0, 1), _uniform(rng, 0.5, 1.0)
    b.AlphaInterpolation = _alpha(rng)
    levels = lambda: op.lib().orc_bloom_mip_count(max(w // 2, 1), max(h // 2, 1), C.c_float(b.Radius))  # noqa: E731
    while levels() < 2:                                   # Bloom refuses a pyramid of one level
        b.Radius = min(1.0, b.Radius + 0.125)
    v.taa.TemporalStabilityFactor, v.taa.SkipRejection = _uniform(rng, 0, 1), int(rng.integers(0, 2))
    m = v.tonemap
    m.bAutoExposure, m.bLightAdaptation = int(rng.integers(0, 2)), int(rng.integers(0, 2))
    m.fMiddleGray, m.fWhitePoint, m.fLuminanceSaturation = _uniform(rng, 0.05, 0.5), _uniform(rng, 1, 8), _uniform(rng, 0.5, 2)
    m.AgXSaturation, m.AgXSlope, m.AgXPower, m.AgXOffset = _uniform(rng, 0.5, 1.5), _uniform(rng, 0.7, 1.3), _uniform(rng, 0.7, 1.3), _uniform(rng, -0.05, 0.05)
    v.ave_log_lum = _uniform(rng, 0.05, 1.5)
    d = v.dof_attribs
    d.MaxCircleOfConfusion, d.TemporalStabilityFactor = _uniform(rng, 0.005, 0.03), _uniform(rng, 0, 1)
    d.BokehKernelRingCount, d.BokehKernelRingDensity, d.AlphaInterpolation = int(rng.integers(2, 6)), int(rng.integers(2, 8)), _alpha(rng)
    if v.dof:
        v.lens = (_uniform(rng, 2, 12), _uniform(rng, 1.2, 8))
    return w, h, int(rng.integers(1, 1000)), v


def random_trial(trial: int | str) -> tuple[np.random.Generator, tuple[int, int] | None]:
    """The generator and size of a test trial: an integer draws a random size, "WxH" (one of EDGE_SIZES) fixes it."""
    if isinstance(trial, str):
        w, h = (int(x) for x in trial.split("x"))
        return np.random.default_rng(4096 + 1000 * w + h), (w, h)
    return np.random.default_rng(2024 + trial), None


def variant_sequence(w: int, h: int, seed: int, v: Variant, frames: int) -> list[dict]:
    """The synthetic sequence a drawn variant runs on: reversed depth and the lens of `v` applied to every frame."""
    seq = synth.generate_sequence(w, h, frames, seed=seed)
    if v.reversed_depth:
        seq = [synth.reverse_depth_frame(f) for f in seq]
    if v.lens is not None:
        for f in seq:
            for k in ("curr_camera", "prev_camera"):
                c = capi.CameraAttribs.from_buffer_copy(bytes(f[k]))
                c.fFocusDistance, c.fFStop = v.lens
                f[k] = c
    return seq


def make_oracle(width: int, height: int, v: Variant) -> op.Oracle:
    o = op.Oracle(width, height)
    v.ssao.Algorithm = v.ssao_algorithm
    v.tonemap.iToneMappingMode = v.tonemap_mode
    o.set_ssr(v.ssr, v.ssr_flags), o.set_ssao(v.ssao), o.set_ssao_flags(v.ssao_flags), o.set_taa(v.taa, v.taa_flags)
    o.set_bloom(v.bloom), o.set_tonemap(v.tonemap, v.ave_log_lum, v.to_srgb)
    if v.dof:
        o.set_dof(v.dof_attribs, v.dof_flags)
    return o


def _levels(o: op.Oracle, name: str) -> list[np.ndarray]:
    out = []
    while True:
        try:
            out.append(o.get(f"{name}.{len(out)}"))
        except RuntimeError:
            return out


def _count(o: op.Oracle, base: str) -> int:
    n = 0
    while True:
        try:
            o.get(f"{base}{n}")
            n += 1
        except RuntimeError:
            return n


def dof_kernels(a: capi.DOFAttribs):
    L = op.lib()
    L.orc_dof_gauss_kernel.argtypes = [C.c_int, C.c_float, C.POINTER(C.c_float), C.c_int]

    def points(rc, rd):
        buf = (C.c_float * 4096)()
        n = L.orc_dof_kernel_points(rc, rd, buf, 2048)
        return np.array(buf[:2 * n], np.float32).reshape(1, n, 2)

    buf = (C.c_float * 64)()
    n = L.orc_dof_gauss_kernel(6, 5.0, buf, 64)                       # DOF_GAUSS_KERNEL_RADIUS / _SIGMA (DepthOfFieldStructures.fxh:19-22)
    return points(a.BokehKernelRingCount, a.BokehKernelRingDensity), points(3, 5), np.array(buf[:n], np.float32).reshape(1, n)


def compare_frame(o: op.Oracle, fr: dict, v: Variant, with_reference: bool = True) -> dict[str, tuple[np.ndarray, np.ndarray]]:
    """`o` holds the history of the frames before `fr` (run with o.frame()); `fr` must be the next frame of the sequence.
    with_reference=False steps the oracle alone (the first element of every pair is then the untouched target), for
    comparing it with the committed outputs of the reference shaders where librefshaders.so is not available."""
    res: dict[str, tuple[np.ndarray, np.ndarray]] = {}
    rev = "__rev" if v.reversed_depth else ""
    cur, prv = fr["curr_camera"], fr["prev_camera"]
    ci, pi = fr["frame"] & 1, (fr["frame"] + 1) & 1
    z = np.zeros_like
    o.set_inputs(fr)
    g = o.get

    def ref(name, ins, outs, **kw):
        if with_reference:
            refsh.run(name, ins, outs, **kw)
        return outs

    # ---------------- PostFXContext ----------------
    blob = np.frombuffer(open(op.TABLES, "rb").read(), np.uint8)
    sobol, tile = blob[:256].astype(np.uint32).reshape(1, 256), blob[256:].astype(np.uint32).reshape(256, 512)
    o.run("blue_noise")
    xy, zw = g("bn_xy"), g("bn_zw")
    r = ref("postfx_blue_noise", [sobol, tile], [z(xy), z(zw)], iparams=[fr["frame"]])
    res["P0 blue_noise.xy"], res["P0 blue_noise.zw"] = (r[0], xy), (r[1], zw)
    depth, motion, normal, color, material = g("depth"), g("motion"), g("normal"), g("color"), g("material")
    o.run("reprojected_depth")
    reproj = g("reproj_depth")
    res["P1 reprojected_depth"] = (ref("postfx_reprojected_depth", [depth], [z(reproj)], cbs=[cur, prv])[0], reproj)
    o.run("closest_motion")
    closest = g("closest_motion")
    res["P2 closest_motion"] = (ref("postfx_closest_motion" + rev, [depth, motion], [z(closest)])[0], closest)
    o.run("previous_depth")
    prev_depth = g("prev_depth")

    # ---------------- ScreenSpaceReflection ----------------
    half = bool(v.ssr_flags & 2)
    o.run("ssr_hiz")
    hiz = _levels(o, "ssr_hiz")
    for i in range(1, len(hiz)):
        res[f"S1 ssr_hiz.{i}"] = (ref("ssr_hiz" + rev, [hiz[i - 1]], [z(hiz[i])])[0], hiz[i])
    rough_before = g("ssr_roughness")
    o.run("ssr_mask")
    rough, maskf = g("ssr_roughness"), g("ssr_mask")
    r = ref("ssr_mask" + rev, [material, depth], [rough_before.copy(), z(maskf)], cbs=[v.ssr])
    res["S2 ssr_roughness"], res["S2 ssr_stencil"] = (r[0], rough), (r[1], maskf)
    mask = (maskf != 0).astype(np.uint8)
    trace_mask = mask
    if half:
        o.run("ssr_downsample_mask")
        mh = g("ssr_mask_half")
        res["S3 ssr_stencil_half"] = (ref("ssr_downsample_mask", [rough, depth], [z(mh)], cbs=[v.ssr])[0], mh)
        trace_mask = (mh != 0).astype(np.uint8)
    o.run("ssr_intersect")
    rad, rdir = g("ssr_radiance"), g("ssr_raydir")
    name = "ssr_intersect" + ("__prev" if v.ssr_flags & 1 else "__half" if half else rev)
    r = ref(name, [color, normal, rough, motion, xy] + hiz, [z(rad), z(rdir)], cbs=[cur, v.ssr], mask=trace_mask)   # targets cleared to 0
    res["S4 ssr_intersect.radiance"], res["S4 ssr_intersect.raydir_pdf"] = (r[0], rad), (r[1], rdir)
    pre = [g("ssr_resolved_rad"), g("ssr_resolved_var"), g("ssr_resolved_depth")]                                   # not cleared: masked pixels keep old content
    o.run("ssr_spatial")
    want = [g("ssr_resolved_rad"), g("ssr_resolved_var"), g("ssr_resolved_depth")]
    r = ref("ssr_spatial" + ("__half" if half else rev), [rough, normal, depth, rdir, rad], [p.copy() for p in pre], cbs=[cur, v.ssr], mask=mask)
    for n_, a_, b_ in zip(("radiance", "variance", "depth"), r, want):
        res[f"S5 ssr_spatial.{n_}"] = (a_, b_)
    pre = [g(f"ssr_radhist{ci}"), g(f"ssr_varhist{ci}")]
    ins = [motion, want[2], reproj, want[0], want[1], prev_depth, g(f"ssr_radhist{pi}"), g(f"ssr_varhist{pi}")]
    o.run("ssr_temporal")
    acc = [g(f"ssr_radhist{ci}"), g(f"ssr_varhist{ci}")]
    r = ref("ssr_temporal" + rev, ins, [p.copy() for p in pre], cbs=[cur, prv, v.ssr], mask=mask)
    res["S6 ssr_temporal.radiance"], res["S6 ssr_temporal.variance"] = (r[0], acc[0]), (r[1], acc[1])
    o.run("ssr_bilateral")
    ssr_out = g("ssr_out")
    res["S7 ssr_bilateral"] = (ref("ssr_bilateral" + rev, [depth, normal, rough, acc[0], acc[1]], [z(ssr_out)], cbs=[cur, v.ssr], mask=mask)[0], ssr_out)

    # ---------------- ScreenSpaceAmbientOcclusion ----------------
    ao_half = bool(v.ssao_flags & 2)
    src = depth
    if ao_half:
        o.run("ssao_downsample")
        src = g("ssao_checker")
        res["A0 ssao_downsample"] = (ref("ssao_downsample", [depth], [z(src)])[0], src)
    o.run("ssao_prefilter")
    pre = _levels(o, "ssao_pre")
    assert np.array_equal(pre[0], src)                                                                               # mip 0 = copy
    for i in range(1, len(pre)):
        res[f"A1 ssao_prefilter.{i}"] = (ref("ssao_prefilter" + rev, [pre[i - 1]], [z(pre[i])], cbs=[cur, v.ssao])[0], pre[i])
    o.run("ssao_ao")
    occ = g("ssao_occ")
    name = "ssao_ao" + {0: "", 1: "__hbao", 2: "__vbao"}[v.ssao_algorithm]
    if v.ssao_algorithm == 0:
        name += "__half" if ao_half else "__halfprec" if v.ssao_flags & 1 else rev
    res["A2 ssao_ao"] = (ref(name, [normal, zw] + pre, [np.ones_like(occ)], cbs=[cur, v.ssao])[0], occ)                # target cleared to 1
    if ao_half:
        o.run("ssao_upsample")
        up = g("ssao_occ_up")
        res["A4 ssao_upsample"] = (ref("ssao_upsample", [depth, occ], [z(up)], cbs=[cur, v.ssao])[0], up)
        occ = up
    ins = [occ, g(f"ssao_hist{pi}"), g(f"ssao_histlen{pi}"), reproj, prev_depth, closest]
    o.run("ssao_temporal")
    acc_o, hlen = g("ssao_acc"), g(f"ssao_histlen{ci}")
    r = ref("ssao_temporal" + rev, ins, [np.ones_like(acc_o), np.ones_like(hlen)], cbs=[cur, prv, v.ssao])              # both cleared to 1
    res["A5 ssao_temporal.occlusion"], res["A5 ssao_temporal.history"] = (r[0], acc_o), (r[1], hlen)
    o.run("ssao_convolute")
    co, cd = _levels(o, "ssao_conv_occ"), _levels(o, "ssao_conv_depth")
    for i in range(1, len(co)):
        r = ref("ssao_convolute", [co[i - 1], cd[i - 1]], [z(co[i]), z(cd[i])])
        res[f"A6 ssao_convolute.occlusion.{i}"], res[f"A6 ssao_convolute.depth.{i}"] = (r[0], co[i]), (r[1], cd[i])
    o.run("ssao_resample")
    rs = g("ssao_resampled")
    res["A7 ssao_resample"] = (ref("ssao_resample" + rev, [hlen, normal] + co + cd, [z(rs)], cbs=[cur], iparams=[len(co)])[0], rs)
    o.run("ssao_spatial")
    ao = g("ssao_out")
    res["A8 ssao_spatial"] = (ref("ssao_spatial" + rev, [rs, hlen, depth, normal], [z(ao)], cbs=[cur, v.ssao])[0], ao)

    # ---------------- compose (this repository's reduced form; no reference shader) -> TAA ----------------
    o.run("compose")
    o.set("taa_in", g("composed"))
    v.taa.ResetAccumulation = 0                                                                                      # consecutive frame (TemporalAntiAliasing.cpp:125-128)
    o.set_taa(v.taa, v.taa_flags)
    prev_acc = g(f"taa_accum{pi}")
    o.run("taa")
    acc_t = g(f"taa_accum{ci}")
    tname = "taa" + ("__" + "".join(c for c, bit in zip("gby", (1, 2, 4)) if v.taa_flags & bit) if v.taa_flags & 7 else "")
    res["T1 taa"] = (ref(tname, [g("taa_in"), prev_acc, closest, reproj, prev_depth], [z(acc_t)], cbs=[cur, prv, v.taa])[0], acc_t)
    post_in = acc_t

    # ---------------- DepthOfField ----------------
    if v.dof:
        a = v.dof_attribs
        big, small, gauss = dof_kernels(a)
        o.set("dof_in", post_in)
        o.run("dof_coc")
        coc = g("dof_coc")
        res["D1 dof_coc"] = (ref("dof_coc", [depth], [z(coc)], cbs=[cur, a])[0], coc)
        if v.dof_flags & 1:
            prevc = g(f"dof_coc_temporal{pi}")
            o.run("dof_temporal")
            tc = g(f"dof_coc_temporal{ci}")
            res["D2 dof_temporal"] = (ref("dof_temporal", [coc, prevc, closest], [z(tc)], cbs=[cur, a])[0], tc)
            coc = tc
        o.run("dof_separated")
        d0 = g("dof_dilation0")
        res["D3 dof_separated"] = (ref("dof_separated", [coc], [z(d0)])[0], d0)
        o.run("dof_dilation")
        dl = [g(f"dof_dilation{i}") for i in range(4)]
        for i in range(3):
            res[f"D4 dof_dilation.{i + 1}"] = (ref("dof_dilation", [dl[i]], [z(dl[i + 1])])[0], dl[i + 1])
        o.run("dof_blur_x")
        bx = g("dof_dilation_tmp")
        res["D5 dof_blur_x"] = (ref("dof_blur__x", [dl[3], gauss], [z(bx)])[0], bx)
        o.run("dof_blur_y")
        by = g("dof_dilation3")
        res["D6 dof_blur_y"] = (ref("dof_blur__y", [bx, gauss], [z(by)])[0], by)
        o.run("dof_prefilter")
        p0, p1 = g("dof_pre0"), g("dof_pre1")
        r = ref("dof_prefilter", [post_in, coc, by], [z(p0), z(p1)], cbs=[a])
        res["D7 dof_prefilter.near"], res["D7 dof_prefilter.far"] = (r[0], p0), (r[1], p1)
        o.run("dof_bokeh_first")
        b0, b1 = g("dof_bokeh0"), g("dof_bokeh1")
        r = ref("dof_bokeh_first" + ("__karis" if v.dof_flags & 2 else ""), [p0, p1, post_in, big], [z(b0), z(b1)], cbs=[cur, a])
        res["D8 dof_bokeh_first.near"], res["D8 dof_bokeh_first.far"] = (r[0], b0), (r[1], b1)
        o.run("dof_bokeh_second")
        s0, s1 = g("dof_pre0"), g("dof_pre1")
        r = ref("dof_bokeh_second", [b0, b1, small], [z(s0), z(s1)], cbs=[cur, a])
        res["D9 dof_bokeh_second.near"], res["D9 dof_bokeh_second.far"] = (r[0], s0), (r[1], s1)
        o.run("dof_postfilter")
        f0, f1 = g("dof_bokeh0"), g("dof_bokeh1")
        r = ref("dof_postfilter", [s0, s1], [z(f0), z(f1)])
        res["D10 dof_postfilter.near"], res["D10 dof_postfilter.far"] = (r[0], f0), (r[1], f1)
        o.run("dof_combine")
        dout = g("dof_out")
        res["D11 dof_combine"] = (ref("dof_combine", [post_in, coc, f0, f1], [z(dout)], cbs=[cur, a])[0][..., :3], dout[..., :3])
        post_in = dout

    # ---------------- Bloom (RGB targets: alpha is not part of the reference's R11G11B10 chain) ----------------
    o.set("bloom_in", post_in)
    o.run("bloom")
    n = _count(o, "bloom_down")
    dn, up = [g(f"bloom_down{i}") for i in range(n)], [g(f"bloom_up{i}") for i in range(n - 1)]
    res["B1 bloom_prefilter"] = (ref("bloom_prefilter", [post_in], [z(dn[0])], cbs=[v.bloom])[0][..., :3], dn[0][..., :3])
    for i in range(1, n):
        res[f"B2 bloom_downsample.{i}"] = (ref("bloom_downsample", [dn[i - 1]], [z(dn[i])])[0][..., :3], dn[i][..., :3])
    top = n - 1
    for i in range(top, 0, -1):
        r = ref("bloom_upsample", [dn[i - 1], up[i] if i != top else dn[i]], [z(up[i - 1])], cbs=[v.bloom], iparams=[0])
        res[f"B3 bloom_upsample.{i - 1}"] = (r[0][..., :3], up[i - 1][..., :3])
    bout = g("bloom_out")
    res["B4 bloom_composite"] = (ref("bloom_upsample", [post_in, up[0]], [z(bout)], cbs=[v.bloom], iparams=[1])[0][..., :3], bout[..., :3])

    # ---------------- ToneMapping + sRGB ----------------
    o.set("tonemap_in", bout)
    o.run("tonemap")
    ldr = g("ldr")
    bits = int(np.float32(v.ave_log_lum).view(np.uint32))
    res["M1 tonemap"] = (ref(f"tonemap__{v.tonemap_mode}", [bout], [z(ldr)], cbs=[v.tonemap], iparams=[bits, int(v.to_srgb)])[0], ldr)
    return res
