// VectorFieldRenderer.hpp — same public surface as the reference's Components/interface/VectorFieldRenderer.hpp:44-160 (CreateInfo,
// RenderAttribs, Render), implemented over dfx_pass_vector_field. See DiligentShim.hpp for what the Diligent types stand for here. There
// are no pipeline states to build: CreateInfo's formats, PSMainSource and PackMatrixRowMajor are accepted and ignored (the target carries
// its format; the default PS main is what the pass computes). The renderer owns the pass's scratch plane, allocated zeroed on the first
// Render into a target of a new size; the pass leaves it zero.
#pragma once
#include "DiligentShim.hpp"

namespace Diligent
{

class VectorFieldRenderer
{
public:
    struct CreateInfo
    {
        IRenderDevice*     pDevice            = nullptr;
        IRenderStateCache* pStateCache        = nullptr; // optional, ignored
        Uint8              NumRenderTargets   = 1;
        TEXTURE_FORMAT     RTVFormats[8]      = {TEX_FORMAT_RGBA32_FLOAT};
        TEXTURE_FORMAT     DSVFormat          = TEX_FORMAT_UNKNOWN;
        const char*        PSMainSource       = nullptr;
        bool               PackMatrixRowMajor = false;
        bool               AsyncShaders       = false;
    };

    struct RenderAttribs
    {
        IDeviceContext* pContext     = nullptr;
        ITextureView*   pVectorField = nullptr; // RG32_FLOAT or RG16_FLOAT, any size
        ITextureView*   pColorRTV    = nullptr; // the render target the reference binds before Render: RGBA32_FLOAT or RGBA16_FLOAT
        float           Bias[2]      = {0, 0};  // applied before the scale
        float           Scale[2]     = {1, 1};
        float           StartColor[4] = {1, 1, 1, 1};
        float           EndColor[4]   = {1, 1, 1, 1};
        Uint32          GridSize[2]   = {0, 0};
        bool            ConvertOutputToSRGB = false;
    };

    explicit VectorFieldRenderer(const CreateInfo& CI) { DFX_DEV_CHECK_ERR(CI.pDevice != nullptr, "Device must not be null"); }
    VectorFieldRenderer(const VectorFieldRenderer&)            = delete;
    VectorFieldRenderer& operator=(const VectorFieldRenderer&) = delete;

    // VectorFieldRenderer.cpp:173-223: GridSize.x * GridSize.y lines over the bound colour target
    void Render(const RenderAttribs& Attribs)
    {
        DFX_DEV_CHECK_ERR(Attribs.pContext != nullptr, "Context must not be null");
        if (Attribs.GridSize[0] == 0 || Attribs.GridSize[1] == 0) return;
        DFX_DEV_CHECK_ERR(Attribs.pVectorField != nullptr && Attribs.pColorRTV != nullptr, "the vector field and the colour target must be given");
        const dfx_plane* color = Attribs.pColorRTV->GetPlane();
        if (color == nullptr) return;
        void* const stream = detail::StreamOf(Attribs.pContext);
        if (!m_Scratch || m_Scratch->GetWidth() != Uint32(color->width) || m_Scratch->GetHeight() != Uint32(color->height))
        {
            m_Scratch.reset(new ITexture{Uint32(color->width), Uint32(color->height), TEX_FORMAT_R32_FLOAT});
            const float zero[4] = {0, 0, 0, 0};
            detail::Check(dfx_plane_fill(stream, &m_Scratch->GetPlane(), zero), "VectorFieldRenderer::Render");
        }
        dfx_vector_field_attribs a;
        dfx_vector_field_attribs_default(&a);
        for (int k = 0; k < 2; ++k) a.Bias[k] = Attribs.Bias[k], a.Scale[k] = Attribs.Scale[k], a.GridSize[k] = Attribs.GridSize[k];
        for (int k = 0; k < 4; ++k) a.StartColor[k] = Attribs.StartColor[k], a.EndColor[k] = Attribs.EndColor[k];
        detail::Check(dfx_pass_vector_field(stream, &a, Attribs.ConvertOutputToSRGB ? DFX_VECTOR_FIELD_OPTION_CONVERT_OUTPUT_TO_SRGB : 0u,
                                            Attribs.pVectorField->GetPlane(), color, &m_Scratch->GetPlane(), dfx_rows{0, color->height}),
                      "VectorFieldRenderer::Render");
    }

private:
    std::unique_ptr<ITexture> m_Scratch;
};

} // namespace Diligent
