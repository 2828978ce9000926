// PBR_Renderer.hpp — the image-based-lighting subset of the reference's PBR/interface/PBR_Renderer.hpp:477-533 and :905 (the cube-map
// formats and sizes, PrecomputeCubemapsAttribs, PrecomputeCubemaps, PrecomputeBRDF), implemented over dfx_pass_irradiance_cube,
// dfx_pass_prefilter_env_map and dfx_pass_precompute_brdf_lut. See DiligentShim.hpp for what the Diligent types stand for here. The rest
// of PBR_Renderer rasterises and is not part of this library.
//
// A texture here is one plane, so a mip-mapped texture is passed as its levels: the source map as views of its levels (a cube's level
// is an s x 6s plane, faces +X, -X, +Y, -Y, +Z, -Z stacked) with IsCube saying which kind it is (the reference asks the texture), and
// the prefiltered map as the textures of its levels (s_m x 6 s_m, s_m = max(s >> m, 1); GetPrefilteredEnvMapDesc's full chain has 9
// levels at 256).
#pragma once
#include "DiligentShim.hpp"

namespace Diligent
{

class PBR_Renderer
{
public:
    static constexpr TEXTURE_FORMAT PrefilteredEnvMapFmt = TEX_FORMAT_RGBA16_FLOAT;
    static constexpr TEXTURE_FORMAT IrradianceCubeFmt    = TEX_FORMAT_RGBA16_FLOAT;
    static constexpr Uint32         IrradianceCubeDim    = 64;
    static constexpr Uint32         PrefilteredEnvMapDim = 256;
    static constexpr Uint32         BRDF_LUT_Dim         = 512; // PBR_Renderer.cpp:548-625

    struct PrecomputeCubemapsAttribs
    {
        /// Source environment map: its mip levels (1..DFX_MAX_ENV_LEVELS), RGBA32_FLOAT or RGBA16_FLOAT.
        ITextureView* const* ppEnvironmentMapLevels  = nullptr;
        Uint32               NumEnvironmentMapLevels = 0;
        bool                 IsCube                  = true;

        /// Output irradiance cube map texture (d x 6d).
        ITexture* pIrradianceCube = nullptr;

        /// Output prefiltered environment map: its levels (2..DFX_MAX_ENV_LEVELS).
        ITexture* const* ppPrefilteredEnvMapLevels  = nullptr;
        Uint32           NumPrefilteredEnvMapLevels = 0;

        /// Number of samples for diffuse irradiance precomputation. If 0, 8192 (the reference's count on a discrete adapter).
        Uint32 NumDiffuseSamples = 0;

        /// Number of samples for specular prefiltering. If 0, 256.
        Uint32 NumSpecularSamples = 0;

        /// Whether to optimize samples (OPTIMIZE_SAMPLES: each sample's LOD from its solid angle).
        bool OptimizeSamples = true;
    };

    PBR_Renderer() : m_BRDF_LUT{BRDF_LUT_Dim, BRDF_LUT_Dim, TEX_FORMAT_RG32_FLOAT} {}
    PBR_Renderer(const PBR_Renderer&)            = delete;
    PBR_Renderer& operator=(const PBR_Renderer&) = delete;

    /// Precompute cubemaps used by IBL (PBR_Renderer.cpp:729-970): the irradiance cube, then every level of the prefiltered map.
    void PrecomputeCubemaps(IDeviceContext* pCtx, const PrecomputeCubemapsAttribs& Attribs)
    {
        if (pCtx == nullptr || Attribs.ppEnvironmentMapLevels == nullptr || Attribs.pIrradianceCube == nullptr || Attribs.ppPrefilteredEnvMapLevels == nullptr)
        {
            DFX_LOG_ERROR_MESSAGE("Device context, environment map SRV, and output cubemaps must not be null");
            return;
        }
        dfx_plane env[DFX_MAX_ENV_LEVELS]{}, pre[DFX_MAX_ENV_LEVELS]{};
        const Uint32 n_env = Attribs.NumEnvironmentMapLevels <= DFX_MAX_ENV_LEVELS ? Attribs.NumEnvironmentMapLevels : DFX_MAX_ENV_LEVELS + 1;
        const Uint32 n_pre = Attribs.NumPrefilteredEnvMapLevels <= DFX_MAX_ENV_LEVELS ? Attribs.NumPrefilteredEnvMapLevels : DFX_MAX_ENV_LEVELS + 1;
        for (Uint32 i = 0; i < n_env && i < DFX_MAX_ENV_LEVELS; ++i)
            if (const dfx_plane* p = Attribs.ppEnvironmentMapLevels[i] ? Attribs.ppEnvironmentMapLevels[i]->GetPlane() : nullptr) env[i] = *p;
        for (Uint32 i = 0; i < n_pre && i < DFX_MAX_ENV_LEVELS; ++i)
            if (Attribs.ppPrefilteredEnvMapLevels[i]) pre[i] = Attribs.ppPrefilteredEnvMapLevels[i]->GetPlane();
        void* const   s    = detail::StreamOf(pCtx);
        const int32_t type = Attribs.IsCube ? DFX_ENV_MAP_TYPE_CUBE : DFX_ENV_MAP_TYPE_SPHERE;
        if (!detail::Check(dfx_pass_irradiance_cube(s, type, env, static_cast<int32_t>(n_env), Attribs.NumDiffuseSamples, Attribs.OptimizeSamples ? 1 : 0,
                                                     &Attribs.pIrradianceCube->GetPlane()),
                           "PBR_Renderer::PrecomputeCubemaps (irradiance cube)"))
            return;
        detail::Check(dfx_pass_prefilter_env_map(s, type, env, static_cast<int32_t>(n_env), Attribs.NumSpecularSamples, Attribs.OptimizeSamples ? 1 : 0, pre,
                                                 static_cast<int32_t>(n_pre)),
                      "PBR_Renderer::PrecomputeCubemaps (prefiltered environment map)");
    }

    /// The pre-integrated GGX table (PrecomputeBRDF.psh) into the renderer's own BRDF_LUT_Dim^2 RG32_FLOAT texture.
    void PrecomputeBRDF(IDeviceContext* pCtx, Uint32 NumBRDFSamples = 512)
    {
        detail::Check(dfx_pass_precompute_brdf_lut(detail::StreamOf(pCtx), NumBRDFSamples, &m_BRDF_LUT.GetPlane()), "PBR_Renderer::PrecomputeBRDF");
    }
    ITextureView* GetPreintegratedGGX_SRV() { return &m_BRDF_LUT_View; }

private:
    ITexture     m_BRDF_LUT;
    ITextureView m_BRDF_LUT_View{&m_BRDF_LUT};
};

} // namespace Diligent
