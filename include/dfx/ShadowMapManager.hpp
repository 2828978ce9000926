// ShadowMapManager.hpp — the filterable-map subset of the reference's Components/interface/ShadowMapManager.hpp (InitInfo, Initialize,
// GetSRV, GetCascadeDSV, GetFilterableSRV, ConvertToFilterable), implemented over dfx_shadow_convert_to_filterable. See DiligentShim.hpp
// for what the Diligent types stand for here. DistributeCascades is not part of this library: the application fills ShadowMapAttribs
// as it does with Diligent.
//
// A texture array here is one plane per slice: the shadow map's slices are the planes the application renders each cascade's depth
// into (GetCascadeDSV(i)), the filterable map's slices the planes its material shaders sample. GetSRV() and GetFilterableSRV() are the
// views of slice 0; GetSRV(i) and GetFilterableSRV(i) give slice i.
#pragma once
#include <vector>

#include "DiligentShim.hpp"

namespace Diligent
{

enum SHADOW_MODE : int
{
    SHADOW_MODE_PCF   = DFX_SHADOW_MODE_PCF,
    SHADOW_MODE_VSM   = DFX_SHADOW_MODE_VSM,
    SHADOW_MODE_EVSM2 = DFX_SHADOW_MODE_EVSM2,
    SHADOW_MODE_EVSM4 = DFX_SHADOW_MODE_EVSM4
};

namespace HLSL
{
// BasicStructures.fxh:6-14 and :28-67 with their DEFAULT_VALUE()s
struct CascadeAttribs : dfx_cascade_attribs
{
    CascadeAttribs() { std::memset(static_cast<dfx_cascade_attribs*>(this), 0, sizeof(dfx_cascade_attribs)); }
};
struct ShadowMapAttribs : dfx_shadow_map_attribs
{
    ShadowMapAttribs()
    {
        std::memset(static_cast<dfx_shadow_map_attribs*>(this), 0, sizeof(dfx_shadow_map_attribs));
        fReceiverPlaneDepthBiasClamp = 10.0f, fFixedDepthBias = 1e-5f, fCascadeTransitionRegion = 0.1f, iMaxAnisotropy = 4;
        fVSMBias = 1e-4f, fVSMLightBleedingReduction = 0.0f, fEVSMPositiveExponent = 40.0f, fEVSMNegativeExponent = 5.0f;
        bIs32BitEVSM = 1, iFixedFilterSize = 3, fFilterWorldSize = 0.0f;
    }
};
static_assert(sizeof(CascadeAttribs) == 64 && sizeof(ShadowMapAttribs) == 1200, "constant blocks must keep the reference layout");
} // namespace HLSL

class ShadowMapManager
{
public:
    struct InitInfo
    {
        /// TEX_FORMAT_D16_UNORM or TEX_FORMAT_D32_FLOAT
        TEXTURE_FORMAT Format               = TEX_FORMAT_UNKNOWN;
        Uint32         Resolution           = 0;
        Uint32         NumCascades          = 0;
        int            ShadowMode           = 0;
        bool           Is32BitFilterableFmt = false;
    };

    ShadowMapManager()                                   = default;
    ShadowMapManager(const ShadowMapManager&)            = delete;
    ShadowMapManager& operator=(const ShadowMapManager&) = delete;

    /// ShadowMapManager.cpp:41-132: the shadow map's slices and, for VSM / EVSM2 / EVSM4, the filterable slices and the one-slice
    /// intermediate in the filterable format (VSM RG16_UNORM / RG32_FLOAT, EVSM2 RG16_FLOAT / RG32_FLOAT, EVSM4 RGBA16_FLOAT /
    /// RGBA32_FLOAT).
    void Initialize(IRenderDevice* /*pDevice*/, IRenderStateCache* /*pStateCache*/, const InitInfo& initInfo)
    {
        if (initInfo.Format == TEX_FORMAT_UNKNOWN || initInfo.NumCascades == 0 || initInfo.Resolution == 0 || initInfo.ShadowMode == 0)
        {
            DFX_LOG_ERROR_MESSAGE("ShadowMapManager::Initialize: format, number of cascades, resolution and shadow mode must be set");
            return;
        }
        m_ShadowMode = initInfo.ShadowMode;
        m_ShadowMap.clear(), m_Filterable.clear(), m_Intermediate.reset();
        for (Uint32 i = 0; i < initInfo.NumCascades; ++i) m_ShadowMap.emplace_back(new Slice{initInfo.Resolution, initInfo.Format});
        if (m_ShadowMode == SHADOW_MODE_VSM || m_ShadowMode == SHADOW_MODE_EVSM2 || m_ShadowMode == SHADOW_MODE_EVSM4)
        {
            TEXTURE_FORMAT Fmt = TEX_FORMAT_UNKNOWN;
            if (m_ShadowMode == SHADOW_MODE_VSM)
                Fmt = initInfo.Is32BitFilterableFmt ? TEX_FORMAT_RG32_FLOAT : TEX_FORMAT_RG16_UNORM;
            else if (m_ShadowMode == SHADOW_MODE_EVSM2)
                Fmt = initInfo.Is32BitFilterableFmt ? TEX_FORMAT_RG32_FLOAT : TEX_FORMAT_RG16_FLOAT;
            else
                Fmt = initInfo.Is32BitFilterableFmt ? TEX_FORMAT_RGBA32_FLOAT : TEX_FORMAT_RGBA16_FLOAT;
            for (Uint32 i = 0; i < initInfo.NumCascades; ++i) m_Filterable.emplace_back(new Slice{initInfo.Resolution, Fmt});
            m_Intermediate.reset(new Slice{initInfo.Resolution, Fmt});
        }
    }

    ITextureView* GetSRV(Uint32 Slice = 0) { return Slice < m_ShadowMap.size() ? &m_ShadowMap[Slice]->View : nullptr; }
    ITextureView* GetCascadeDSV(Uint32 Cascade) { return GetSRV(Cascade); }
    ITextureView* GetFilterableSRV(Uint32 Slice = 0) { return Slice < m_Filterable.size() ? &m_Filterable[Slice]->View : nullptr; }

    /// ShadowMapManager.cpp:533-600: VSMHorzPS / EVSMHorzPS then VertBlurPS for every cascade (one fused launch for most filter sizes);
    /// does nothing for PCF.
    void ConvertToFilterable(IDeviceContext* pCtx, const dfx_shadow_map_attribs& ShadowAttribs)
    {
        if (m_Filterable.empty()) return;
        std::vector<dfx_plane> in, out;
        for (const auto& s : m_ShadowMap) in.push_back(s->Tex.GetPlane());
        for (const auto& s : m_Filterable) out.push_back(s->Tex.GetPlane());
        detail::Check(dfx_shadow_convert_to_filterable(detail::StreamOf(pCtx), m_ShadowMode, &ShadowAttribs, in.data(), static_cast<int32_t>(in.size()),
                                                       out.data(), &m_Intermediate->Tex.GetPlane()),
                      "ShadowMapManager::ConvertToFilterable");
    }

private:
    struct Slice
    {
        Slice(Uint32 Resolution, TEXTURE_FORMAT Fmt) : Tex{Resolution, Resolution, Fmt} {}
        ITexture     Tex;
        ITextureView View{&Tex};
    };
    int                                 m_ShadowMode = 0;
    std::vector<std::unique_ptr<Slice>> m_ShadowMap, m_Filterable;
    std::unique_ptr<Slice>              m_Intermediate;
};

} // namespace Diligent
