// BoundBoxRenderer.hpp — same public surface as the reference's Components/interface/BoundBoxRenderer.hpp:44-160 (CreateInfo,
// OPTION_FLAGS, RenderAttribs, Prepare, Render), implemented over dfx_pass_bound_box. See DiligentShim.hpp for what the Diligent types
// stand for here. There are no pipeline states to build: CreateInfo's formats, render-target mask, PSMainSource and
// PackMatrixRowMajor are accepted and ignored (the colour and motion planes carry their formats; the motion plane is written when
// motion vectors are on; the colour is stored as RenderAttribs::Color gives it, so a caller that wants HnRenderBoundBoxTask's PS main,
// float4(Color.rgb, 0), passes alpha 0; matrices are always row-major, row-vector convention here).
#pragma once
#include "DiligentShim.hpp"

namespace Diligent
{

class BoundBoxRenderer
{
public:
    struct CreateInfo
    {
        IRenderDevice*     pDevice            = nullptr;
        IRenderStateCache* pStateCache        = nullptr; // optional, ignored
        IBuffer*           pCameraAttribsCB   = nullptr; // {current camera, previous camera} in device memory (e.g. PostFXContext's)
        Uint8              NumRenderTargets   = 1;
        TEXTURE_FORMAT     RTVFormats[8]      = {TEX_FORMAT_RGBA32_FLOAT};
        TEXTURE_FORMAT     DSVFormat          = TEX_FORMAT_D32_FLOAT;
        Uint32             RenderTargetMask   = 0x1u;
        const char*        PSMainSource       = nullptr;
        bool               PackMatrixRowMajor = false;
        bool               AsyncShaders       = false;
    };

    enum OPTION_FLAGS : Uint32
    {
        OPTION_FLAG_NONE                   = DFX_BOUND_BOX_OPTION_NONE,
        OPTION_FLAG_CONVERT_OUTPUT_TO_SRGB = DFX_BOUND_BOX_OPTION_CONVERT_OUTPUT_TO_SRGB,
        OPTION_FLAG_COMPUTE_MOTION_VECTORS = DFX_BOUND_BOX_OPTION_COMPUTE_MOTION_VECTORS,
        OPTION_FLAG_USE_REVERSE_DEPTH      = DFX_BOUND_BOX_OPTION_USE_REVERSE_DEPTH,
    };

    struct RenderAttribs
    {
        const dfx_float4x4* BoundBoxTransform = nullptr; // can't be null: the unit cube's corner c goes to float4(c, 1) * M
        const float*        Color             = nullptr; // float4; null = white
        float               PatternLength     = 32;      // pixels
        Uint32              PatternMask       = 0xFFFFFFFFu;
        OPTION_FLAGS        Options           = OPTION_FLAG_NONE;
    };

    // The targets Render() draws into: what the application binds as render targets and depth buffer before the draw.
    struct Targets
    {
        ITextureView* pColorRTV  = nullptr; // RGBA32_FLOAT or RGBA16_FLOAT
        ITextureView* pMotionRTV = nullptr; // RG32_FLOAT or RG16_FLOAT; required with OPTION_FLAG_COMPUTE_MOTION_VECTORS
        ITextureView* pDepthDSV  = nullptr; // D32_FLOAT
    };

    explicit BoundBoxRenderer(const CreateInfo& CI) : m_pCameraAttribsCB{CI.pCameraAttribsCB}
    {
        DFX_DEV_CHECK_ERR(CI.pDevice != nullptr, "Device must not be null");
        DFX_DEV_CHECK_ERR(m_pCameraAttribsCB != nullptr, "Camera Attribs CB must not be null");
    }
    BoundBoxRenderer(const BoundBoxRenderer&)            = delete;
    BoundBoxRenderer& operator=(const BoundBoxRenderer&) = delete;

    // BoundBoxRenderer.cpp:224-255: the key of the draw and BoundBoxAttribs
    void Prepare(IDeviceContext* pContext, const RenderAttribs& Attribs)
    {
        (void)pContext;
        if (Attribs.BoundBoxTransform == nullptr)
        {
            DFX_LOG_ERROR_MESSAGE("Bound box transform must not be null");
            return;
        }
        dfx_bound_box_attribs_default(&m_Attribs);
        m_Attribs.Transform = *Attribs.BoundBoxTransform;
        if (Attribs.Color != nullptr)
            for (int k = 0; k < 4; ++k) m_Attribs.Color[k] = Attribs.Color[k];
        m_Attribs.PatternLength = Attribs.PatternLength;
        m_Attribs.PatternMask   = Attribs.PatternMask;
        m_Options               = Attribs.Options;
        m_Prepared              = true;
    }

    // BoundBoxRenderer.cpp:257-277: the 24-vertex LINE_LIST draw into the bound targets
    void Render(IDeviceContext* pContext, const Targets& T)
    {
        DFX_DEV_CHECK_ERR(pContext != nullptr, "Context must not be null");
        DFX_DEV_CHECK_ERR(m_Prepared, "Prepare() must be called before Render()");
        DFX_DEV_CHECK_ERR(T.pColorRTV != nullptr && T.pDepthDSV != nullptr, "the colour target and the depth buffer must be given");
        const dfx_plane* color = T.pColorRTV->GetPlane();
        detail::Check(dfx_pass_bound_box(detail::StreamOf(pContext), static_cast<const dfx_camera_attribs*>(m_pCameraAttribsCB->GetDevicePtr()), &m_Attribs,
                                         m_Options, T.pDepthDSV->GetPlane(), color, T.pMotionRTV ? T.pMotionRTV->GetPlane() : nullptr,
                                         dfx_rows{0, color ? color->height : 0}),
                      "BoundBoxRenderer::Render");
    }

private:
    IBuffer*              m_pCameraAttribsCB = nullptr;
    dfx_bound_box_attribs m_Attribs{};
    Uint32                m_Options  = 0;
    bool                  m_Prepared = false;
};
DEFINE_FLAG_ENUM_OPERATORS(BoundBoxRenderer::OPTION_FLAGS)

} // namespace Diligent
