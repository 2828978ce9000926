// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_math.h). Pinned against the reference's own shaders (oracle/refshader, tests/test_reference_shaders.py).
// The full compose step of the reference integration (SURVEY.md §8f rank 1): Hydrogent/shaders/HnPostProcess.psh:145-185 with
// the split-sum helpers it calls (Shaders/PBR/public/PBR_Shading.fxh:220-302, :429-451; Shaders/Common/public/PBR_Common.fxh:8-11,
// :86-95) and the pre-integrated GGX look-up table those helpers sample (Shaders/PBR/private/PrecomputeBRDF.psh:10-48,
// PBR_PrecomputeCommon.fxh:10-39; created 512x512 RG16_FLOAT with 512 samples by PBR/src/PBR_Renderer.cpp:548-625).
#include "oracle.h"
#include "oracle_ibl_math.h"

namespace orc
{

// PrecomputeBRDF.psh:10-38 under DESIGN.md §2's rule for PBR_Renderer's precomputations (oracle_ibl_math.h): one rounding per
// operation, cos / sin correctly rounded, pow(1 - VoH, 5.0) as pow5_; the samples are added in order
static float2 IntegrateBRDF(float PerceptualRoughness, float NoV, uint NumSamples)
{
    float3 V(std::sqrt(1.0f - NoV * NoV), 0.0f, NoV);
    const float3 N(0.0f, 0.0f, 1.0f);
    float A = 0.0f, B = 0.0f;
    for (uint i = 0u; i < NumSamples; i++)
    {
        float2 Xi  = iblm::hammersley(i, NumSamples);
        float3 H   = iblm::ImportanceSampleGGX(Xi, PerceptualRoughness, N);
        float3 L   = 2.0f * dot(V, H) * H - V;
        float  NoL = saturate(L.z), NoH = saturate(H.z), VoH = saturate(dot(V, H));
        if (NoL > 0.0f)
        {
            float AlphaRoughness = PerceptualRoughness * PerceptualRoughness;
            float G_Vis = 4.0f * SmithGGXVisibilityCorrelated(NoL, NoV, AlphaRoughness) * VoH * NoL / NoH;
            float Fc    = iblm::pow5_(1.0f - VoH);
            A += (1.0f - Fc) * G_Vis;
            B += Fc * G_Vis;
        }
    }
    return float2(A, B) / float(NumSamples);
}

// PrecomputeBRDF.psh:40-48: texel (x, y) of a w x h table holds IntegrateBRDF(roughness = v, NdotV = u) at its centre
void brdf_lut(int w, int h, uint num_samples, TexF2& lut, int threads)
{
    lut.resize(w, h);
    parallel_rows(0, h, threads, [&](int ya, int yb) {
        for (int y = ya; y < yb; ++y)
            for (int x = 0; x < w; ++x)
            {
                float2 UV((float(x) + 0.5f) / float(w), (float(y) + 0.5f) / float(h));
                lut.at(x, y) = IntegrateBRDF(UV.y, UV.x, num_samples);
            }
    });
}

// PBR_Common.fxh:13-17, :86-95
static inline float  pow5(float x) { float x2 = x * x; return x2 * x2 * x; }
static inline float3 SchlickReflection(float VdotH, float3 R0, float3 R90) { return R0 + (R90 - R0) * pow5(clampf(1.0f - VdotH, 0.0f, 1.0f)); }

// HnPostProcess.psh:145-185 (the ToneMap call that follows in the same shader is the chain's own tone-map pass here)
void compose_ibl(const Camera& cam, const TexF4& color, const TexF4* ssr, const TexF* ao, const TexF4& specular_ibl, const TexF4& normal,
                 const TexF4& base_color, const TexF4& material, const TexF2& lut, float ssr_scale, float ssao_scale, TexF4& out, int threads)
{
    const int W = color.w, H = color.h;
    out.resize(W, H);
    const float3 CamPos = cam.f4Position.xyz();
    parallel_rows(0, H, threads, [&](int ya, int yb) {
        for (int py = ya; py < yb; ++py)
            for (int px = 0; px < W; ++px)
            {
                float4 Color    = color.load(px, py);
                float  Opacity  = Color.w;
                float  SSRScale = ssr_scale * Opacity;
                if (ssr && SSRScale > 0.0f)
                {
                    float4 SpecularIBL = specular_ibl.load(px, py);
                    float4 SSRRadiance = ssr->load(px, py);
                    float3 Normal      = normal.load(px, py).xyz();
                    float4 BaseColor   = base_color.load(px, py);
                    float4 Material    = material.load(px, py);
                    float  Roughness = saturate(Material.x), Metallic = saturate(Material.y);
                    // GetSurfaceReflectanceMR :429-451
                    const float f0 = 0.04f;
                    float3 Reflectance0 = lerp(float3(f0, f0, f0), BaseColor.xyz(), Metallic);
                    // view direction through the pixel centre (:160-161); f2NormalizedXY is the NDC position of the pixel
                    float2 uv((float(px) + 0.5f) * cam.f4ViewportSize.z, (float(py) + 0.5f) * cam.f4ViewportSize.w);
                    float2 ndc      = TexUVToNormalizedDeviceXY(uv);
                    float4 WorldPos = mul(float4(ndc.x, ndc.y, 0.5f, 1.0f), cam.mViewProjInv); // DepthToNormalizedDeviceZ(0.5) = 0.5
                    float3 ViewDir  = normalize(CamPos - WorldPos.xyz() / WorldPos.w);
                    // GetIBLSamplingInfo :232-267 with USE_IBL_MULTIPLE_SCATTERING = 1 (:35-36), no iridescence
                    float  NdotV      = saturate(dot(Normal, ViewDir));
                    float2 PreIntBRDF = sample_linear(lut, float2(NdotV, Roughness), Address::Clamp);
                    float  OneMinusRoughness = 1.0f - Roughness;
                    float3 Reflectance90 = float3(hmax(OneMinusRoughness, Reflectance0.x), hmax(OneMinusRoughness, Reflectance0.y), hmax(OneMinusRoughness, Reflectance0.z));
                    float3 k_S = SchlickReflection(NdotV, Reflectance0, Reflectance90);
                    // GetSpecularIBL_GGX :293-302
                    float3 SSR = SSRRadiance.xyz() * (k_S * PreIntBRDF.x + float3(PreIntBRDF.y, PreIntBRDF.y, PreIntBRDF.y));
                    float3 rgb = Color.xyz() + (SSR - SpecularIBL.xyz()) * SSRRadiance.w * SSRScale; // left to right, as HnPostProcess.psh:170 writes it
                    Color      = float4(rgb, Color.w);
                }
                float SSAOScale = ssao_scale * Opacity;
                if (ao && SSAOScale > 0.0f)
                {
                    float Occlusion = lerp(1.0f, ao->load(px, py), SSAOScale);
                    Color           = float4(Color.xyz() * Occlusion, Color.w);
                }
                out.at(px, py) = Color;
            }
    });
}

} // namespace orc
