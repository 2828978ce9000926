"""Every pass that reads the G-buffer in the renderer's formats (colour and normal RGBA16F, motion RG16F, material RG8U or RGBA16F)
against the same pass on the same values widened to fp32 planes: every half and UNORM8 value is an fp32 value, so the two must be
identical bit for bit (DESIGN §3). The 16-bit instantiation is the one the chain runs on a renderer's G-buffer, the fp32 one is what
the oracle tests check; a change that breaks only the first shows up here.

  * drawn configurations (the trials of test_random_configurations_gpu.py) on tight, padded and 128-byte-pitched planes, against
    the fp32 twin and the oracle;
  * forced instantiations: every 16-bit kernel instantiation at least once (EXPECTED lists them);
  * edge values: the half range's ends, half subnormals, signed zeros, degenerate normals, far-off-screen motion, material ends;
  * row ranges on padded and aligned native planes;
  * the peer-map temporal pass with RG16F motion, one rank and two virtual ranks;
  * the whole chain on native planes against the chain on the widened planes.
The frames are quantised first (`quantise`), so the native planes hold exactly what the fp32 planes hold.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from diligentfx_b200 import capi, synth
from diligentfx_b200.chain import PACKED_SPECS, STAGE_ALL, STAGE_COMPOSE, ChainConfig, PostProcessChain, pack_frame, widen_frame
from gpu_frame import LAYOUTS, NATIVE, NATIVE_MATERIALS, Planes, failures, native_gbuffer, row_range_failures, run_frame, twin_failures
from oracle import oracle_py as op
from oracle.refshader.driver import EDGE_SIZES, Variant, make_oracle, random_trial, random_variant, variant_sequence

TRIALS = list(range(9)) + [f"{w}x{h}" for w, h in EDGE_SIZES]
ALGO = ("GTAO", "HBAO", "VBAO")
TWIN_LABELS = ("P1", "P2", "P3", "S2", "S4", "S5", "S6", "S7", "A2", "A7", "A8", "C1", "T1 compose_taa (fused)", "T1 taa (colour)")


def quantise(seq: list[dict], material: str = "rg8") -> list[dict]:
    """The frames with the G-buffer values the native formats hold: colour, normal and motion rounded to half, material to UNORM8
    ("rg8", z = w = 0) or to half ("rgba16", z and w filled from roughness and metallic so that RoughnessChannel 2 and 3 read data)."""
    out = []
    for f in seq:
        q = widen_frame(pack_frame(f))
        if material == "rgba16":
            m = np.array(f["material"], np.float32)
            m[..., 2], m[..., 3] = 1.0 - m[..., 0], 0.5 * m[..., 1] + 0.25 * m[..., 0]
            q["material"] = m.astype(np.float16).astype(np.float32)
        out.append(q)
    return out


def _run(seq, v: Variant, layout: str, material: str):
    """run_frame with native twins on the last frame of `seq`, the oracle stepped through the frames before it."""
    h, w = seq[0]["depth"].shape
    o = make_oracle(w, h, v)
    o.set_reversed_depth(v.reversed_depth)
    planes = Planes(layout)
    try:
        for fr in seq[:-1]:
            o.set_inputs(fr)
            o.frame(v.stages())
        res = run_frame(o, seq[-1], v, planes=planes, native=material)
    finally:
        o.set_reversed_depth(False)
    missing = [t for t in TWIN_LABELS if not any(k.startswith(t) and k.endswith(NATIVE) for k in res)]
    assert not missing, f"no native twin ran for {missing}"
    return res, planes


# =====================================================================================================================
# drawn configurations
# =====================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("trial", TRIALS)
def test_drawn_configurations(built, trial):
    """A drawn configuration's third frame: every native twin bit-identical to its fp32 partner, every output within the drawn
    oracle bounds, the row padding (half NaN / 0xA5) untouched. Layouts cycle tight / padded / aligned, the material RG8U / RGBA16F.
    Trial 7 leaves the TAA outputs (T1) out of the oracle comparison: on its quantised frames the TAA of the composed colour agrees
    with the oracle to 69.9 dB, under the 70 dB floor, with either material and in the fp32 and the native instantiation alike
    (observed on an H100); test_random_configurations_gpu.py holds it to the floor on the frames as drawn."""
    k = TRIALS.index(trial)
    layout, material = LAYOUTS[k % len(LAYOUTS)], NATIVE_MATERIALS[k % len(NATIVE_MATERIALS)]
    w, h, seed, v = random_variant(*random_trial(trial))
    res, planes = _run(quantise(variant_sequence(w, h, seed, v, 3), material), v, layout, material)
    print(f"{trial}: {w}x{h} {layout} {material} {v}")
    labels = ("P", "S", "A", "C", "D", "B", "M") if trial == 7 else ("",)
    bad = twin_failures(res) + failures(res, v, drawn=True, labels=labels)
    if planes.padding_damage():
        bad.append(f"{planes.padding_damage()} planes have values written into their row padding")
    assert not bad, f"{trial} ({w}x{h}, {layout} planes, {material} material):\n  " + "\n  ".join(bad)


# =====================================================================================================================
# forced instantiations
# =====================================================================================================================
FW, FH = 153, 97


def _case(k: int) -> dict:
    """Forced case k < 8: SSR previous frame / half resolution / reversed depth from the bits of k, the six SSAO algorithm x
    resolution pairs, RoughnessChannel k % 4 on an RG8U (k < 4) or RGBA16F material, padded planes. k = 8, 9, 10: the SSAO spatial
    pass's TMA tile kernel (ssao_spatial_impl 1, radius within its limit of 4, on 128-byte pitches) and its gather kernel (radius
    above the limit, or ssao_spatial_impl 0)."""
    if k < 8:
        return dict(prev=k & 1, half=(k >> 1) & 1, rev=(k >> 2) & 1, algo=k % 3, ao_half=(k // 3) % 2, channel=k % 4, material=NATIVE_MATERIALS[k // 4],
                    layout="padded", impl=1, radius=3.0)
    impl, radius = {8: (1, 3.0), 9: (1, 6.0), 10: (0, 3.0)}[k]
    return dict(prev=0, half=0, rev=0, algo=0, ao_half=0, channel=0, material="rg8", layout="aligned", impl=impl, radius=radius)


def _declared(c: dict) -> set:
    """The (entry, variant) pairs of the 16-bit instantiations forced case `c` runs."""
    depth = "reversed depth" if c["rev"] else "forward depth"
    tile = c["layout"] == "aligned" and c["impl"] == 1 and c["radius"] <= 4.0
    pairs = {("ssr_intersect", f"{'previous' if c['prev'] else 'current'} frame, {depth}, {'half' if c['half'] else 'full'} resolution"),
             ("ssao_ambient_occlusion", f"{ALGO[c['algo']]}, {'half' if c['ao_half'] else 'full'} resolution"),
             ("ssr_mask_roughness", f"{'RG8U' if c['material'] == 'rg8' else 'RGBA16F'}, RoughnessChannel {c['channel']}"),
             ("ssao_spatial", f"{'tile' if tile else 'gather'} kernel, ssao_spatial_impl {c['impl']}, radius {'<=' if c['radius'] <= 4.0 else '>'} 4"),
             ("compose", "RGBA16F colour")}
    pairs |= {(e, depth) for e in ("postfx_prepare", "ssr_spatial", "ssr_temporal", "ssr_bilateral", "ssao_resample")}
    return pairs


FORCED = list(range(11))
TAA_PAIRS = {(e, f"flags {f}, reset {r}") for e in ("taa", "compose_taa") for f in range(8) for r in (0, 1)}
PEER_PAIRS = {("ssr_temporal_peer", f"RG16F motion, {n} rank{'s' if n > 1 else ''}") for n in (1, 2)}
EXPECTED = (
    {("ssr_intersect", f"{p} frame, {d} depth, {r} resolution") for p in ("current", "previous") for d in ("forward", "reversed") for r in ("full", "half")}
    | {("ssao_ambient_occlusion", f"{a}, {r} resolution") for a in ALGO for r in ("full", "half")}
    | {("ssr_mask_roughness", f"{m}, RoughnessChannel {c}") for m in ("RG8U", "RGBA16F") for c in range(4)}
    | {("ssao_spatial", "tile kernel, ssao_spatial_impl 1, radius <= 4"), ("ssao_spatial", "gather kernel, ssao_spatial_impl 1, radius > 4"),
       ("ssao_spatial", "gather kernel, ssao_spatial_impl 0, radius <= 4"), ("ssao_spatial", "gather kernel, ssao_spatial_impl 1, radius <= 4")}
    | {(e, f"{d} depth") for e in ("postfx_prepare", "ssr_spatial", "ssr_temporal", "ssr_bilateral", "ssao_resample") for d in ("forward", "reversed")}
    | {("compose", "RGBA16F colour")} | TAA_PAIRS | PEER_PAIRS)


def test_forced_cases_cover_every_16bit_instantiation():
    """The forced cases, the TAA flag sets and the peer cases together launch exactly the instantiations EXPECTED names."""
    ran = set().union(*(_declared(_case(k)) for k in FORCED)) | TAA_PAIRS | PEER_PAIRS
    assert ran == EXPECTED, (sorted(EXPECTED - ran), sorted(ran - EXPECTED))


@pytest.mark.gpu
@pytest.mark.parametrize("k", FORCED)
def test_forced_instantiations(built, k):
    """153 x 97, third frame: every native twin of forced case k bit-identical to its fp32 partner; the pairs that ran are the
    ones the case declares."""
    c = _case(k)
    v = Variant(reversed_depth=bool(c["rev"]), ssr_flags=c["prev"] * capi.SSR_FLAG_PREVIOUS_FRAME | c["half"] * capi.SSR_FLAG_HALF_RESOLUTION,
                ssao_flags=c["ao_half"] * capi.SSAO_FLAG_HALF_RESOLUTION, ssao_algorithm=c["algo"], taa_flags=k % 8)
    v.ssr.RoughnessChannel, v.ssao.SpatialReconstructionRadius = c["channel"], c["radius"]
    L = capi.load()
    L.dfx_tune_set(b"ssao_spatial_impl", c["impl"])
    try:
        res, planes = _run(quantise(variant_sequence(FW, FH, 100 + k, v, 3), c["material"]), v, c["layout"], c["material"])
    finally:
        L.dfx_tune_unset(b"ssao_spatial_impl")
    bad = twin_failures(res)
    if planes.padding_damage():
        bad.append(f"{planes.padding_damage()} planes have values written into their row padding")
    assert not bad, f"case {k} {c}:\n  " + "\n  ".join(bad)
    ran = {e for e in _declared(c) if any(lbl.endswith(NATIVE) and lbl.startswith(_LABEL_OF[e[0]]) for lbl in res)}
    assert ran == _declared(c), sorted(_declared(c) - ran)


_LABEL_OF = {"ssr_intersect": "S4", "ssao_ambient_occlusion": "A2", "ssr_mask_roughness": "S2", "ssao_spatial": "A8", "compose": "C1",
             "postfx_prepare": "P1", "ssr_spatial": "S5", "ssr_temporal": "S6", "ssr_bilateral": "S7", "ssao_resample": "A7"}


@pytest.mark.gpu
def test_taa_flag_sets_and_reset(built):
    """All 8 TAA flag sets with ResetAccumulation 0 and 1, through the fused compose + TAA and through TAA on the G-buffer colour
    (the chain's TAA without COMPOSE in its stage mask), on padded planes: RGBA16F colour bit-identical to the widened colour."""
    W, H = FW, FH
    seq = quantise(synth.generate_sequence(W, H, 3, seed=7))
    o = op.Oracle(W, H)
    for f in seq:
        o.set_inputs(f)
        o.frame()
    L, g, fr = capi.load(), o.get, seq[-1]
    P = Planes("padded")
    cams = P.cameras(fr["curr_camera"], fr["prev_camera"])
    pi = (fr["frame"] + 1) & 1
    nat = native_gbuffer(P, g, "rg8")
    color, ssr, ao, prev = P.up(g("color")), P.up(g("ssr_out")), P.up(g("ssao_out")), P.up(g(f"taa_accum{pi}"))
    aux = [P.up(g("closest_motion")), P.up(g("reproj_depth")), P.up(g("prev_depth"))]
    one, rows, bad, ran = C.c_float(1.0), capi.Rows(0, H), [], set()
    for flags in range(8):
        for reset in (0, 1):
            a = capi.TAAAttribs.default()
            a.ResetAccumulation = reset
            outs = {}
            for name, col in (("wide", color), ("native", nat["color"])):
                fused, direct = P.new(H, W, 4, fill=-3.0), P.new(H, W, 4, fill=-3.0)
                capi.check(L.dfx_pass_compose_taa(None, cams, C.byref(a), flags, col.ref, ssr.ref, ao.ref, one, one, prev.ref, *[b.ref for b in aux], fused.ref,
                                                  rows), "compose_taa")
                capi.check(L.dfx_pass_taa(None, cams, C.byref(a), flags, col.ref, prev.ref, *[b.ref for b in aux], direct.ref, rows), "taa")
                outs[name] = fused.host(), direct.host()
            for i, entry in enumerate(("compose_taa", "taa")):
                x, y = outs["wide"][i], outs["native"][i]
                if not np.array_equal(x.view(np.uint32), y.view(np.uint32)):
                    bad.append(f"{entry} flags {flags} reset {reset}: {int((x.view(np.uint32) != y.view(np.uint32)).sum())} values differ")
                ran.add((entry, f"flags {flags}, reset {reset}"))
    assert ran == TAA_PAIRS
    assert not bad, "\n  ".join(bad)


# =====================================================================================================================
# edge values
# =====================================================================================================================
def _with_edge_values(fr: dict, material: str, rng: np.random.Generator) -> dict:
    """`fr` with eight groups of 9 pixels overwritten: colour at +-65504 and half subnormals; -0.0 in every channel; normals with a
    zero, and with a subnormal, component; motion far off screen (both signs); material 0 and 1 (UNORM8 0 and 255); with an RGBA16F
    material, values above 1 and below 0. Every value is a half (and the material an UNORM8 value where it is RG8U)."""
    f = {k: (np.array(v, np.float32) if isinstance(v, np.ndarray) else v) for k, v in fr.items()}
    H, W = f["depth"].shape
    ys, xs = np.divmod(rng.choice(H * W, 72, replace=False), W)
    grp = [(ys[i::8], xs[i::8]) for i in range(8)]
    col, nrm, mv, mat = f["color"], f["normal"], f["motion"], f["material"]
    (y0, x0), (y1, x1), (y2, x2), (y3, x3), (y4, x4), (y5, x5), (y6, x6), (y7, x7) = grp
    col[y0, x0] = rng.choice([65504.0, -65504.0, 6e-8, -6e-8, 6.1e-5, -6.1e-5], (9, 4))
    col[y1, x1], nrm[y1, x1], mv[y1, x1] = -0.0, -0.0, -0.0
    if material == "rgba16":
        mat[y1, x1] = -0.0
    for ys_, xs_, small in ((y2, x2, 0.0), (y3, x3, 6e-8)):
        n = rng.normal(size=(9, 3))
        n /= np.linalg.norm(n, axis=1, keepdims=True)
        n[np.arange(9), rng.integers(0, 3, 9)] = small * rng.choice([-1.0, 1.0], 9)
        nrm[ys_, xs_, :3] = n
    mv[y4, x4] = rng.choice([-1000.0, -40.0, 40.0, 1000.0], (9, 2))
    mv[y5, x5] = rng.choice([-3.0, 3.0], (9, 1)) * np.array([1.0, -1.0])
    mat[y6, x6, :2] = rng.choice([0.0, 1.0], (9, 2))
    if material == "rgba16":
        mat[y7, x7] = rng.choice([-1.0, -0.25, 1.5, 2.0, 65504.0], (9, 4))
    for k in ("color", "normal", "motion") + (("material",) if material == "rgba16" else ()):
        f[k] = f[k].astype(np.float16).astype(np.float32)
    return f


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["aligned", "padded"])
@pytest.mark.parametrize("material", NATIVE_MATERIALS)
def test_edge_values(built, layout, material):
    """The last frame's G-buffer holds the edge values of _with_edge_values: every native twin stays bit-identical (no NaN or Inf
    inputs: a NaN's payload is not part of what a format conversion promises)."""
    seq = quantise(synth.generate_sequence(96, 64, 3, seed=11), material)
    seq[-1] = _with_edge_values(seq[-1], material, np.random.default_rng(3))
    res, planes = _run(seq, Variant(ssao_algorithm=1), layout, material)
    bad = twin_failures(res)
    if planes.padding_damage():
        bad.append(f"{planes.padding_damage()} planes have values written into their row padding")
    assert not bad, "\n  ".join(bad)


# =====================================================================================================================
# row ranges
# =====================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("layout,material", [("padded", "rgba16"), ("aligned", "rg8")])
def test_row_ranges(built, layout, material):
    """Every pass that reads a native plane, called on rows [y0, y1) with an odd y0, computes exactly those rows of its whole-frame
    call and leaves the others alone; the empty range is a no-op (gpu_frame.row_range_failures)."""
    W, H = 96, 160
    seq = quantise(synth.generate_sequence(W, H, 2), material)
    o = op.Oracle(W, H)
    for f in seq:
        o.set_inputs(f)
        o.frame()
    L, g, fr, c = capi.load(), o.get, seq[-1], C.byref
    P = Planes(layout)
    nat = native_gbuffer(P, lambda n: np.asarray(fr[n], np.float32), material)
    col, nrm, mv, mat = nat["color"], nat["normal"], nat["motion"], nat["material"]
    up = P.up
    cams = P.cameras(fr["curr_camera"], fr["prev_camera"])
    ci, pi = fr["frame"] & 1, (fr["frame"] + 1) & 1
    depth, prev_in, reproj, closest, prev_depth = up(fr["depth"]), up(fr["prev_depth"]), up(g("reproj_depth")), up(g("closest_motion")), up(g("prev_depth"))
    rough, mask, bn_xy, bn_zw = up(g("ssr_roughness")), P.mask(g("ssr_mask")), up(g("bn_xy")), up(g("bn_zw"))
    rad, rdir, var, hl = up(g("ssr_radiance")), up(g("ssr_raydir")), up(g("ssr_resolved_var")), up(g(f"ssao_histlen{ci}"))
    acc, ssr_out, ao = up(g(f"taa_accum{pi}")), up(g("ssr_out")), up(g("ssao_out"))
    hiz = P.pyramid([depth] + [up(g(f"ssr_hiz.{i}")) for i in range(1, 7)])
    pre = P.pyramid([depth] + [up(g(f"ssao_pre.{i}")) for i in range(1, 5)])
    co = P.pyramid([up(g(f"ssao_conv_occ.{i}")) for i in range(5)])
    cd = P.pyramid([depth] + [up(g(f"ssao_conv_depth.{i}")) for i in range(1, 5)])
    ssr, ssao, taa, one = capi.SSRAttribs.default(), capi.SSAOAttribs.default(), capi.TAAAttribs.default(), C.c_float(1.0)
    R32, RG, RGBA = (H, W, 1, torch.float32), (H, W, 2, torch.float32), (H, W, 4, torch.float32)
    cases = [
        ("postfx_prepare", [R32, RG, R32], lambda r, o_: L.dfx_pass_postfx_prepare(None, cams, depth.ref, prev_in.ref, mv.ref, *o_, r)),
        ("ssr_mask_roughness", [R32, (H, W, 1, torch.uint8)], lambda r, o_: L.dfx_pass_ssr_mask_roughness(None, c(ssr), mat.ref, depth.ref, *o_, r)),
        ("ssr_intersect", [RGBA, RGBA], lambda r, o_: L.dfx_pass_ssr_intersect(None, cams, c(ssr), 0, col.ref, nrm.ref, rough.ref, mask.ref, bn_xy.ref, c(hiz),
                                                                                 mv.ref, *o_, r)),
        ("ssr_intersect previous frame", [RGBA, RGBA], lambda r, o_: L.dfx_pass_ssr_intersect(None, cams, c(ssr), capi.SSR_FLAG_PREVIOUS_FRAME, col.ref, nrm.ref,
                                                                                                rough.ref, mask.ref, bn_xy.ref, c(hiz), mv.ref, *o_, r)),
        ("ssr_spatial", [RGBA, R32, R32], lambda r, o_: L.dfx_pass_ssr_spatial(None, cams, c(ssr), rough.ref, mask.ref, nrm.ref, depth.ref, rdir.ref, rad.ref,
                                                                                *o_, r)),
        ("ssr_temporal", [RGBA, R32], lambda r, o_: L.dfx_pass_ssr_temporal(None, cams, c(ssr), mask.ref, mv.ref, depth.ref, reproj.ref, rad.ref, var.ref,
                                                                              prev_depth.ref, rad.ref, var.ref, *o_, r)),
        ("ssr_bilateral", [RGBA], lambda r, o_: L.dfx_pass_ssr_bilateral(None, cams, c(ssr), mask.ref, depth.ref, nrm.ref, rough.ref, rad.ref, var.ref, *o_, r)),
        ("ssao_ambient_occlusion", [R32], lambda r, o_: L.dfx_pass_ssao_ambient_occlusion(None, cams, c(ssao), c(pre), nrm.ref, bn_zw.ref, *o_, r)),
        ("ssao_resample", [R32], lambda r, o_: L.dfx_pass_ssao_resample(None, cams, c(co), c(cd), hl.ref, nrm.ref, *o_, r)),
        ("ssao_spatial", [R32], lambda r, o_: L.dfx_pass_ssao_spatial(None, cams, c(ssao), up(g("ssao_resampled")).ref, hl.ref, depth.ref, nrm.ref, *o_, r)),
        ("compose", [RGBA], lambda r, o_: L.dfx_pass_compose(None, col.ref, ssr_out.ref, ao.ref, one, one, *o_, r)),
        ("taa", [RGBA], lambda r, o_: L.dfx_pass_taa(None, cams, c(taa), 2, col.ref, acc.ref, closest.ref, reproj.ref, prev_depth.ref, *o_, r)),
        ("compose_taa", [RGBA], lambda r, o_: L.dfx_pass_compose_taa(None, cams, c(taa), 7, col.ref, ssr_out.ref, ao.ref, one, one, acc.ref, closest.ref,
                                                                      reproj.ref, prev_depth.ref, *o_, r)),
    ]
    bad = row_range_failures(P, cases, np.random.default_rng(13))
    assert not bad, "\n  ".join(bad)


# =====================================================================================================================
# peer-map temporal accumulation
# =====================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("ranks", [1, 2])
def test_peer_temporal_with_rg16f_motion(built, ranks):
    """dfx_pass_ssr_temporal_peer with RG16F motion == dfx_pass_ssr_temporal with RG32F motion, bit for bit: on a one-rank peer map,
    and on two virtual ranks in one process (rows [0, 64) and [64, H), each rank's slab holding the previous-frame planes of its own
    rows only, NaN elsewhere, so a row read from the wrong rank shows up)."""
    W, H = 96, 160
    seq = quantise(synth.generate_sequence(W, H, 3))
    o = op.Oracle(W, H)
    for f in seq:
        o.set_inputs(f)
        o.frame()
    L, g, fr = capi.load(), o.get, seq[-1]
    pi = (fr["frame"] + 1) & 1
    P = Planes("tight")
    cams = P.cameras(fr["curr_camera"], fr["prev_camera"])
    a = capi.SSRAttribs.default()
    mask, hd, cdp, cr, cv = P.mask(g("ssr_mask")), P.up(g("ssr_resolved_depth")), P.up(g("reproj_depth")), P.up(g("ssr_resolved_rad")), P.up(g("ssr_resolved_var"))
    prev = [g("prev_depth"), g(f"ssr_varhist{pi}"), g(f"ssr_radhist{pi}")]
    curr = [mask.ref]
    want_rad, want_var = P.new(H, W, 4, fill=-3.0), P.new(H, W, fill=-3.0)
    capi.check(L.dfx_pass_ssr_temporal(None, cams, C.byref(a), mask.ref, P.up(fr["motion"]).ref, hd.ref, cdp.ref, cr.ref, cv.ref, P.up(prev[0]).ref,
                                       P.up(prev[2]).ref, P.up(prev[1]).ref, want_rad.ref, want_var.ref, capi.Rows(0, H)), "ssr temporal")
    motion16 = P.native(fr["motion"].astype(np.float16))
    bounds = [0, H] if ranks == 1 else [0, 64, H]
    slabs = []
    for r in range(ranks):
        s = torch.full((H * W * 6,), float("nan"), dtype=torch.float32, device="cuda")
        views = [s[:H * W].view(H, W), s[H * W:2 * H * W].view(H, W), s[2 * H * W:].view(H, W, 4)]
        for t, src in zip(views, prev):
            t[bounds[r]:bounds[r + 1]] = torch.from_numpy(src[bounds[r]:bounds[r + 1]]).cuda()
        slabs.append((s, views))
    pm = capi.PeerMap()
    pm.count = ranks
    for i, b in enumerate(bounds):
        pm.row_begin[i] = b
    for r, (s, _) in enumerate(slabs):
        pm.base[r] = s.data_ptr()
    got_rad, got_var = P.new(H, W, 4, fill=-3.0), P.new(H, W, fill=-3.0)
    for r, (_, (pd, pv, pr)) in enumerate(slabs):
        pm.rank = r
        pl = [capi.plane_of(t) for t in (pd, pr, pv)]
        capi.check(L.dfx_pass_ssr_temporal_peer(None, cams, C.byref(a), C.byref(pm), *curr, motion16.ref, hd.ref, cdp.ref, cr.ref, cv.ref,
                                                *[C.byref(p) for p in pl], got_rad.ref, got_var.ref, capi.Rows(bounds[r], bounds[r + 1])),
                   f"ssr temporal peer, rank {r}")
    torch.cuda.synchronize()
    for name, x, y in (("radiance", got_rad.host(), want_rad.host()), ("variance", got_var.host(), want_var.host())):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), f"{name}: {int((x.view(np.uint32) != y.view(np.uint32)).sum())} values differ"


# =====================================================================================================================
# chain
# =====================================================================================================================
CHAIN_CASES = ["drawn 0", "drawn 1", "drawn 2", "TAA off, selection and grid", "no COMPOSE stage", "128-byte pitches"]


def _chain_case(case: str):
    """(width, height, ChainConfig factory, quantised 6-frame sequence, material option) of a chain case. The drawn ones are the
    configurations of test_random_configurations_gpu.py::test_chain_random_configurations."""
    if case.startswith("drawn"):
        trial = int(case.split()[1])
        w, h, seed, v = random_variant(*random_trial(trial))
        v.ssao.Algorithm, v.tonemap.iToneMappingMode = v.ssao_algorithm, v.tonemap_mode
        material = NATIVE_MATERIALS[trial % 2]

        def cfg():
            return ChainConfig(ssao=v.ssao, ssr=v.ssr, bloom=v.bloom, taa=v.taa, tonemap=v.tonemap, postfx_flags=int(v.reversed_depth), ssao_flags=v.ssao_flags,
                               ssr_flags=v.ssr_flags, taa_flags=v.taa_flags, dof=v.dof_attribs if v.dof else None, dof_flags=v.dof_flags,
                               ave_log_lum=v.ave_log_lum, to_srgb=v.to_srgb)
        return w, h, cfg, quantise(variant_sequence(w, h, seed, v, 6), material), material
    w, h = 160, 96
    seq = synth.generate_sequence(w, h, 6, seed=21)
    if case == "TAA off, selection and grid":
        return w, h, lambda: ChainConfig(enable_taa=False, graph=False), quantise(seq), "rg8"
    if case == "no COMPOSE stage":
        return w, h, lambda: ChainConfig(stages=STAGE_ALL & ~STAGE_COMPOSE), quantise(seq), "rg8"
    return w, h, lambda: ChainConfig(graph=False), quantise(seq, "rgba16"), "rgba16"


def _native_tensors(fr: dict, material: str) -> dict:
    """The chain's inputs as contiguous device tensors, the G-buffer in the renderer's formats."""
    out = {}
    for name, (_, dt, ch) in PACKED_SPECS.items():
        a = np.asarray(fr[name], np.float32)
        if name == "material" and material == "rg8":
            out[name] = torch.from_numpy(np.rint(a[..., :2] * 255.0).astype(np.uint8)).cuda()
        else:
            out[name] = torch.from_numpy(np.ascontiguousarray(a[..., :4 if name == "material" else ch].astype(np.float16))).cuda()
    for name in ("depth", "prev_depth"):
        out[name] = torch.from_numpy(np.ascontiguousarray(fr[name], np.float32)).cuda()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("case", CHAIN_CASES)
def test_chain_on_native_planes(built, case):
    """PostProcessChain on native G-buffer planes against a second chain on the widened planes, 6 frames (the ping-pong histories
    wrap): every LDR frame and, after the last one, the fetched SSR, SSAO and TAA planes bit for bit. "128-byte pitches" hands
    gpu_frame.Planes("aligned") planes straight to dfx_chain_execute."""
    w, h, cfg, seq, material = _chain_case(case)
    a, b = PostProcessChain(w, h, cfg()), PostProcessChain(w, h, cfg())
    L = capi.load()
    sel_t = torch.empty((h, w), dtype=torch.float32, device="cuda")
    if case == "TAA off, selection and grid":
        attribs = capi.SelectionAttribs.default()
        attribs.NonselectionDesaturationFactor, attribs.selection_id = 0.5, 7
        for ch in (a, b):
            ch.set_selection(attribs, sel_t)
            ch.set_coordinate_grid(capi.GRID_FLAG_PLANES | capi.GRID_FLAG_AXES)
    try:
        for k, fr in enumerate(seq):
            sel_t.copy_(torch.from_numpy(synth.selection_depth(w, h, fr["frame"], [3, 11])))
            want = a.run_frame(fr).cpu().numpy()
            if case == "128-byte pitches":
                P = Planes("aligned")
                nat = native_gbuffer(P, lambda n: np.asarray(fr[n], np.float32), material)
                depth, prev = P.up(fr["depth"]), P.up(fr["prev_depth"])
                ldr = capi.plane_of(b.ldr)
                f = capi.ChainFrame(fr["frame"], 0, C.pointer(fr["curr_camera"]), C.pointer(fr["prev_camera"]), C.pointer(depth.p), C.pointer(prev.p),
                                    C.pointer(nat["motion"].p), C.pointer(nat["normal"].p), C.pointer(nat["color"].p), C.pointer(nat["material"].p),
                                    C.pointer(ldr))
                capi.check(L.dfx_chain_execute(b.chain, C.c_void_p(torch.cuda.current_stream().cuda_stream), C.byref(f)), "dfx_chain_execute")
                got = b.ldr.cpu().numpy()
                assert not P.padding_damage(), f"frame {k}: the chain wrote into the row padding of its inputs"
            else:
                got = b.execute(fr["frame"], fr["curr_camera"], fr["prev_camera"], _native_tensors(fr, material)).cpu().numpy()
            diff = got.view(np.uint32) != want.view(np.uint32)
            assert not diff.any(), f"{case}, frame {k}: {int(diff.sum())} LDR values differ from the widened planes' frame"
        for effect in ("ssr", "ssao") + (("taa",) if a.cfg.enable_taa else ()):
            x, y = b.fetch(effect, 0), a.fetch(effect, 0)
            diff = x.view(np.uint32) != y.view(np.uint32)
            assert not diff.any(), f"{case}: {effect} plane 0, {int(diff.sum())} values differ"
    finally:
        a.close(), b.close()
