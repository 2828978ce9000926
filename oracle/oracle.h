// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_math.h). Pinned against the reference's own shaders (oracle/refshader, tests/test_reference_shaders.py).
// Pass-by-pass CPU restatement of the DiligentFX PostProcess chain. One function per reference render pass,
// same plane set and ordering as the reference host code; storage is fp32 (north-star layout).
#pragma once
#include "oracle_common.h"
#include <vector>

namespace orc
{

using TexF  = Tex<float>;
using TexF2 = Tex<float2>;
using TexF4 = Tex<float4>;

// ---------------- PostFXContext ----------------
// ComputeBlueNoiseTexture.fx:81-89. tables = Sobol_256d[256] ++ ScramblingTile[128*128*8]
void postfx_blue_noise(const uint8_t* tables, uint frame_index, TexF2& xy, TexF2& zw);
// ComputeReprojectedDepth.fx:18-30
void postfx_reprojected_depth(const Camera& curr, const Camera& prev, const TexF& depth, TexF& out, int threads);
// ComputeClosestMotion.fx:24-55
void postfx_closest_motion(const TexF& depth, const TexF2& motion, TexF2& out, int threads);

// ---------------- SSAO ----------------
// SSAO_ComputePrefilteredDepthBuffer.fx:79-122 ; mip 0 = copy of depth (ScreenSpaceAmbientOcclusion.cpp:858-865)
void ssao_prefilter_depth(const Camera& cam, const dfx_ssao_attribs& a, const TexF& depth, MipTex<float>& pyr, int threads);
// SSAO_ComputeAmbientOcclusion.fx:132-231 ; target cleared to 1.0 first (…cpp:982-985)
// half_res (FEATURE_FLAG_HALF_RESOLUTION): the pyramid, hence the target, is W/2 x H/2 and GetInvViewportSize() doubles (:68-75)
void ssao_ambient_occlusion(const Camera& cam, const dfx_ssao_attribs& a, const MipTex<float>& prefiltered,
                            const TexF4& normal, const TexF2& blue_noise_zw, TexF& out, int threads, bool half_res = false,
                            bool half_precision_depth = false); // the latter: self-occlusion offset 0.005 (:145-150); storage stays fp32
// A0 SSAO_ComputeDownsampledDepth.fx:8-29 : W/2 x H/2 checkerboard of the 2x2 min / max depth
void ssao_downsample_depth(const TexF& depth, TexF& out, int threads);
// A4 SSAO_ComputeBilateralUpsampling.fx:62-139 : 3x3 joint-bilateral upsampling of the half-res occlusion to W x H
void ssao_bilateral_upsampling(const Camera& cam, const TexF& depth, const TexF& occlusion_half, TexF& out, int threads);
// SSAO_ComputeTemporalAccumulation.fx:151-182 ; both targets cleared to 1.0 first (…cpp:1059-1068)
void ssao_temporal(const Camera& curr, const Camera& prev, const dfx_ssao_attribs& a, const TexF& curr_occlusion,
                   const TexF& prev_occlusion, const TexF& prev_history, const TexF& reprojected_depth,
                   const TexF& previous_depth, const TexF2& closest_motion, TexF& out_occlusion, TexF& out_history,
                   int threads);
// SSAO_ComputeConvolutedDepthHistory.fx:93-109 ; mip 0 = copies (…cpp:1086-1103)
void ssao_convolute(const TexF& accumulated, const TexF& depth, MipTex<float>& occ_pyr, MipTex<float>& depth_pyr, int threads);
// SSAO_ComputeResampledHistory.fx:56-115
void ssao_resample(const Camera& cam, const MipTex<float>& occ_pyr, const MipTex<float>& depth_pyr, const TexF& history,
                   const TexF4& normal, TexF& out, int threads);
// SSAO_ComputeSpatialReconstruction.fx:49-100
void ssao_spatial(const Camera& cam, const dfx_ssao_attribs& a, const TexF& occlusion, const TexF& history,
                  const TexF& depth, const TexF4& normal, TexF& out, int threads);

// ---------------- SSR ----------------
// SSR_ComputeHierarchicalDepthBuffer.fx:30-73 ; mip 0 = copy of depth
void ssr_hiz(const TexF& depth, MipTex<float>& pyr, int threads);
// SSR_ComputeStencilMaskAndExtractRoughness.fx:13-40 ; mask cleared to 0, roughness NOT cleared
void ssr_mask_roughness(const dfx_ssr_attribs& a, const TexF4& material, const TexF& depth, TexF& roughness,
                        Tex<uint8_t>& mask, int threads);
// SSR_ComputeIntersection.fx:281-325 ; both targets cleared to 0; depth-masked
void ssr_intersect(const Camera& cam, const dfx_ssr_attribs& a, uint flags, const TexF4& color, const TexF4& normal,
                   const TexF& roughness, const Tex<uint8_t>& mask, const TexF2& blue_noise_xy, const MipTex<float>& hiz,
                   const TexF2* motion, TexF4& out_radiance, TexF4& out_raydir_pdf, int threads);
// SSR_ComputeSpatialReconstruction.fx:114-172 ; masked, targets not cleared
void ssr_spatial(const Camera& cam, const dfx_ssr_attribs& a, const TexF& roughness, const Tex<uint8_t>& mask,
                 const TexF4& normal, const TexF& depth, const TexF4& raydir_pdf, const TexF4& radiance,
                 TexF4& out_radiance, TexF& out_variance, TexF& out_depth, int threads, bool half_res = false);
// S3 SSR_ComputeDownsampledStencilMask.fx:13-61 (half resolution only): W/2 x H/2 mask of the 2x2 closest depth / max roughness
void ssr_downsample_mask(const dfx_ssr_attribs& a, const TexF& roughness, const TexF& depth, Tex<uint8_t>& mask_half, int threads);
// SSR_ComputeTemporalAccumulation.fx:224-263 ; masked, targets not cleared
void ssr_temporal(const Camera& curr, const Camera& prev, const dfx_ssr_attribs& a, const Tex<uint8_t>& mask,
                  const TexF2& motion, const TexF& hit_depth, const TexF& reprojected_depth, const TexF4& curr_radiance,
                  const TexF& curr_variance, const TexF& previous_depth, const TexF4& prev_radiance,
                  const TexF& prev_variance, TexF4& out_radiance, TexF& out_variance, int threads);
// SSR_ComputeBilateralCleanup.fx:49-97 ; target cleared to 0; masked
void ssr_bilateral(const Camera& cam, const dfx_ssr_attribs& a, const Tex<uint8_t>& mask, const TexF& depth,
                   const TexF4& normal, const TexF& roughness, const TexF4& radiance, const TexF& variance, TexF4& out,
                   int threads);

// ---------------- Bloom ----------------
void bloom_prefilter(const dfx_bloom_attribs& a, const TexF4& color, TexF4& out, int threads);                  // Bloom_ComputePrefilteredTexture.fx:37-83
void bloom_downsample(const TexF4& in, TexF4& out, int threads);                                                 // Bloom_ComputeDownsampledTexture.fx:11-41
void bloom_upsample(const TexF4& same_level_down, const TexF4& coarser, TexF4& out, int threads);                // Bloom_ComputeUpsampledTexture.fx:20-54 (uInstID==0)
void bloom_composite(const dfx_bloom_attribs& a, const TexF4& color, const TexF4& up0, TexF4& out, int threads); // …:45-48 (uInstID!=0)
int  bloom_mip_count(int width, int height, float radius);                                                       // Bloom.cpp:152-156

// ---------------- TAA ----------------
// TAA_ComputeTemporalAccumulation.fx:229-261
void taa_accumulate(const Camera& curr, const Camera& prev, const dfx_taa_attribs& a, uint flags, const TexF4& curr_color,
                    const TexF4& prev_accum, const TexF2& closest_motion, const TexF& reprojected_depth,
                    const TexF& previous_depth, TexF4& out, int threads);
float  halton_sequence(uint base, uint index);                     // TemporalAntiAliasing.cpp:43-54
float2 taa_jitter_offset(uint frame_index, uint width, uint height); // TemporalAntiAliasing.cpp:63-78

// ---------------- compose (reduced form, SURVEY.md §8f) ----------------
void compose(const TexF4& color, const TexF4* ssr, const TexF* ao, float ssr_scale, float ssao_scale, TexF4& out, int threads);
// Full form (Hydrogent/shaders/HnPostProcess.psh:145-185): SSR re-weighted by the split-sum BRDF and exchanged for the specular
// IBL it replaces, both scaled by the pixel's opacity. `lut` = brdf_lut() (PrecomputeBRDF.psh:10-48). oracle_compose_ibl.cpp
void brdf_lut(int w, int h, uint num_samples, TexF2& lut, int threads);
void compose_ibl(const Camera& cam, const TexF4& color, const TexF4* ssr, const TexF* ao, const TexF4& specular_ibl, const TexF4& normal,
                 const TexF4& base_color, const TexF4& material, const TexF2& lut, float ssr_scale, float ssao_scale, TexF4& out, int threads);

// ---------------- DepthOfField (oracle_dof.cpp; DepthOfField.cpp:292-331 gives the order) ----------------
std::vector<float2> dof_kernel_points(int ring_count, int ring_density);  // DepthOfField.cpp:49-73
std::vector<float>  dof_gauss_kernel(int radius, float sigma);            // DepthOfField.cpp:75-91
void dof_circle_of_confusion(const Camera& cam, const dfx_dof_attribs& a, const TexF& depth, TexF& coc, int threads);                       // D1
void dof_temporal_coc(const Camera& cam, const dfx_dof_attribs& a, const TexF& curr, const TexF& prev, const TexF2& closest_motion, TexF& out, int threads); // D2
void dof_separated_coc(const TexF& coc, TexF& out, int threads);                                                                            // D3
void dof_dilation_level(const TexF& last, TexF& out, int threads);                                                                          // D4 (x3)
void dof_blur_coc(const TexF& coc, bool vertical, TexF& out, int threads);                                                                  // D5, D6
void dof_prefilter(const TexF4& color, const TexF& coc, const TexF& dilation, TexF4& out_fg, TexF4& out_bg, int threads);                   // D7
void dof_bokeh_first(const Camera& cam, const dfx_dof_attribs& a, uint flags, const TexF4& fg, const TexF4& bg, const TexF4& radiance, TexF4& out_fg,
                     TexF4& out_bg, int threads);                                                                                           // D8
void dof_bokeh_second(const Camera& cam, const dfx_dof_attribs& a, const TexF4& fg, const TexF4& bg, TexF4& out_fg, TexF4& out_bg, int threads); // D9
void dof_postfilter(const TexF4& fg, const TexF4& bg, TexF4& out_fg, TexF4& out_bg, int threads);                                           // D10
void dof_combine(const dfx_dof_attribs& a, const TexF4& color, const TexF4& dof_near, const TexF4& dof_far, TexF4& out, int threads);       // D11

// ---------------- ToneMapping ----------------
float3 tone_map(float3 color, const dfx_tonemap_attribs& a, float ave_log_lum); // ToneMapping.fxh:87-226
float3 uncharted2_tonemap(float3 x);                                            // ToneMapping.fxh:8-19
void   tonemap_pass(const dfx_tonemap_attribs& a, float ave_log_lum, bool to_srgb, const TexF4& color, TexF4& out, int threads);

} // namespace orc
