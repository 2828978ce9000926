"""REFERENCE-SHADER RUNNER — TEST INFRASTRUCTURE ONLY. The passes librefshaders.so exports: reference shader file (resolved by
base name under /root/reference/Shaders), the macros the reference's host code compiles it with, and this repository's harness.

Variant suffixes: __rev = *_OPTION_INVERTED_DEPTH (FEATURE_FLAG_REVERSED_DEPTH), __prev = SSR_OPTION_PREVIOUS_FRAME,
__half = *_OPTION_HALF_RESOLUTION. SUPPORTED_SHADER_SRV = 1 everywhere (Direct3D / Vulkan path: one mip bound per draw)."""


def _p(name, shader, harness=None, **macros):
    return {"name": name, "shader": shader, "harness": harness or (name.split("__")[0] + ".inc"), "macros": {"SUPPORTED_SHADER_SRV": 1, **macros}}


_SSAO = dict(SSAO_OPTION_INVERTED_DEPTH=0, SSAO_OPTION_HALF_RESOLUTION=0, SSAO_OPTION_HALF_PRECISION_DEPTH=0)
_SSAO_REV = dict(_SSAO, SSAO_OPTION_INVERTED_DEPTH=1)
_SSAO_HALF = dict(_SSAO, SSAO_OPTION_HALF_RESOLUTION=1)
_SSR = dict(SSR_OPTION_INVERTED_DEPTH=0, SSR_OPTION_PREVIOUS_FRAME=0, SSR_OPTION_HALF_RESOLUTION=0)
_SSR_REV = dict(_SSR, SSR_OPTION_INVERTED_DEPTH=1)

PASSES = [
    # PostFXContext (PostFXContext.cpp:515)
    _p("postfx_blue_noise", "ComputeBlueNoiseTexture.fx"),
    _p("postfx_reprojected_depth", "ComputeReprojectedDepth.fx"),
    _p("postfx_closest_motion", "ComputeClosestMotion.fx", POSTFX_OPTION_INVERTED_DEPTH=0),
    _p("postfx_closest_motion__rev", "ComputeClosestMotion.fx", POSTFX_OPTION_INVERTED_DEPTH=1),
    # ScreenSpaceReflection (ScreenSpaceReflection.cpp:472-475)
    _p("ssr_hiz", "SSR_ComputeHierarchicalDepthBuffer.fx", **_SSR),
    _p("ssr_hiz__rev", "SSR_ComputeHierarchicalDepthBuffer.fx", **_SSR_REV),
    _p("ssr_mask", "SSR_ComputeStencilMaskAndExtractRoughness.fx", **_SSR),
    _p("ssr_mask__rev", "SSR_ComputeStencilMaskAndExtractRoughness.fx", **_SSR_REV),
    _p("ssr_downsample_mask", "SSR_ComputeDownsampledStencilMask.fx", **dict(_SSR, SSR_OPTION_HALF_RESOLUTION=1)),
    _p("ssr_intersect", "SSR_ComputeIntersection.fx", **_SSR),
    _p("ssr_intersect__rev", "SSR_ComputeIntersection.fx", **_SSR_REV),
    _p("ssr_intersect__prev", "SSR_ComputeIntersection.fx", **dict(_SSR, SSR_OPTION_PREVIOUS_FRAME=1)),
    _p("ssr_intersect__half", "SSR_ComputeIntersection.fx", **dict(_SSR, SSR_OPTION_HALF_RESOLUTION=1)),
    _p("ssr_spatial", "SSR_ComputeSpatialReconstruction.fx", **_SSR),
    _p("ssr_spatial__rev", "SSR_ComputeSpatialReconstruction.fx", **_SSR_REV),
    _p("ssr_spatial__half", "SSR_ComputeSpatialReconstruction.fx", **dict(_SSR, SSR_OPTION_HALF_RESOLUTION=1)),
    _p("ssr_temporal", "SSR_ComputeTemporalAccumulation.fx", **_SSR),
    _p("ssr_temporal__rev", "SSR_ComputeTemporalAccumulation.fx", **_SSR_REV),
    _p("ssr_bilateral", "SSR_ComputeBilateralCleanup.fx", **_SSR),
    _p("ssr_bilateral__rev", "SSR_ComputeBilateralCleanup.fx", **_SSR_REV),
    # ScreenSpaceAmbientOcclusion (ScreenSpaceAmbientOcclusion.cpp:471-479); SSAO_ALGORITHM 0 GTAO, 1 HBAO, 2 VBAO
    _p("ssao_downsample", "SSAO_ComputeDownsampledDepth.fx", **_SSAO_HALF),
    _p("ssao_prefilter", "SSAO_ComputePrefilteredDepthBuffer.fx", **_SSAO),
    _p("ssao_prefilter__rev", "SSAO_ComputePrefilteredDepthBuffer.fx", **_SSAO_REV),
    _p("ssao_ao", "SSAO_ComputeAmbientOcclusion.fx", SSAO_ALGORITHM=0, **_SSAO),
    _p("ssao_ao__hbao", "SSAO_ComputeAmbientOcclusion.fx", SSAO_ALGORITHM=1, **_SSAO),
    _p("ssao_ao__vbao", "SSAO_ComputeAmbientOcclusion.fx", SSAO_ALGORITHM=2, **_SSAO),
    _p("ssao_ao__rev", "SSAO_ComputeAmbientOcclusion.fx", SSAO_ALGORITHM=0, **_SSAO_REV),
    _p("ssao_ao__half", "SSAO_ComputeAmbientOcclusion.fx", SSAO_ALGORITHM=0, **_SSAO_HALF),
    _p("ssao_ao__halfprec", "SSAO_ComputeAmbientOcclusion.fx", SSAO_ALGORITHM=0, **dict(_SSAO, SSAO_OPTION_HALF_PRECISION_DEPTH=1)),
    _p("ssao_upsample", "SSAO_ComputeBilateralUpsampling.fx", **_SSAO_HALF),
    _p("ssao_temporal", "SSAO_ComputeTemporalAccumulation.fx", **_SSAO),
    _p("ssao_temporal__rev", "SSAO_ComputeTemporalAccumulation.fx", **_SSAO_REV),
    _p("ssao_convolute", "SSAO_ComputeConvolutedDepthHistory.fx", **_SSAO),
    _p("ssao_resample", "SSAO_ComputeResampledHistory.fx", **_SSAO),
    _p("ssao_resample__rev", "SSAO_ComputeResampledHistory.fx", **_SSAO_REV),
    _p("ssao_spatial", "SSAO_ComputeSpatialReconstruction.fx", **_SSAO),
    _p("ssao_spatial__rev", "SSAO_ComputeSpatialReconstruction.fx", **_SSAO_REV),
    # Bloom
    _p("bloom_prefilter", "Bloom_ComputePrefilteredTexture.fx"),
    _p("bloom_downsample", "Bloom_ComputeDownsampledTexture.fx"),
    _p("bloom_upsample", "Bloom_ComputeUpsampledTexture.fx"),
    # TemporalAntiAliasing (TemporalAntiAliasing.cpp:237-239); variant suffix = g(aussian) b(icubic) y(CoCg) bits
] + [
    _p("taa" + ("__" + "".join(n for n, on in zip("gby", (g, b, y)) if on) if (g or b or y) else ""), "TAA_ComputeTemporalAccumulation.fx", "taa.inc",
       TAA_OPTION_GAUSSIAN_WEIGHTING=g, TAA_OPTION_BICUBIC_FILTER=b, TAA_OPTION_YCOCG_COLOR_SPACE=y)
    for g in (0, 1) for b in (0, 1) for y in (0, 1)
] + [
    # ToneMapping.fxh: the operator is a compile-time choice (TONE_MAPPING_MODE 1..11, ToneMappingStructures.fxh:11-22)
    _p(f"tonemap__{m}", ["ToneMapping.fxh", "SRGBUtilities.fxh", "FullScreenTriangleVSOutput.fxh"], "tonemap.inc", TONE_MAPPING_MODE=m) for m in range(1, 12)
] + [
    # DepthOfField (DepthOfField.cpp:529, :564, :635)
    _p("dof_coc", "DOF_ComputeCircleOfConfusion.fx"),
    _p("dof_temporal", "DOF_ComputeTemporalCircleOfConfusion.fx"),
    _p("dof_separated", "DOF_ComputeSeparatedCircleOfConfusion.fx"),
    _p("dof_dilation", "DOF_ComputeDilationCircleOfConfusion.fx"),
    _p("dof_blur__x", "DOF_ComputeBlurredCircleOfConfusion.fx", "dof_blur.inc", DOF_CIRCLE_OF_CONFUSION_BLUR_TYPE=0),
    _p("dof_blur__y", "DOF_ComputeBlurredCircleOfConfusion.fx", "dof_blur.inc", DOF_CIRCLE_OF_CONFUSION_BLUR_TYPE=1),
    _p("dof_prefilter", "DOF_ComputePrefilteredTexture.fx"),
    _p("dof_bokeh_first", "DOF_ComputeBokehFirstPass.fx", DOF_OPTION_KARIS_INVERSE=0),
    _p("dof_bokeh_first__karis", "DOF_ComputeBokehFirstPass.fx", DOF_OPTION_KARIS_INVERSE=1),
    _p("dof_bokeh_second", "DOF_ComputeBokehSecondPass.fx"),
    _p("dof_postfilter", "DOF_ComputePostfilteredTexture.fx"),
    _p("dof_combine", "DOF_ComputeCombinedTexture.fx"),
] + [
    # the compose step of the application (Hydrogent HnPostProcess.psh); the table it samples (PBR PrecomputeBRDF.psh) is built with the
    # IBL precomputation shaders by build_ibl_ref.py, under their statement of the transcendentals
    # HnPostProcessTask.cpp:219-225: VIEW_MODE = HN_VIEW_MODE_SHADED (0); the three debug modes only need to differ from it
    _p("compose_ibl", "HnPostProcess.psh", VIEW_MODE=0, VIEW_MODE_SCENE_DEPTH=101, VIEW_MODE_EDGE_MAP=102, VIEW_MODE_MESH_ID=103, TONE_MAPPING_MODE=0,
       CONVERT_OUTPUT_TO_SRGB=0),
]
