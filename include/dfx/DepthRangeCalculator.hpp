// DepthRangeCalculator.hpp — same public surface as the reference's Components/interface/DepthRangeCalculator.hpp:55-176,
// implemented over the C-ABI (dfx_depth_range_*). See DiligentShim.hpp for what the Diligent types stand for here.
// CreateSRB returns the binding object of DiligentShim.hpp; IsReady() is always true (kernels are compiled ahead of time).
#pragma once
#include "DiligentShim.hpp"

namespace Diligent
{

class DepthRangeCalculator
{
public:
    struct CreateInfo
    {
        IRenderDevice*     pDevice            = nullptr;
        IRenderStateCache* pStateCache        = nullptr; // optional, ignored
        bool               PackMatrixRowMajor = false;   // matrices are always row-major, row-vector convention here
        bool               AsyncShaders       = false;   // ignored: nothing to compile
        bool               ReadBackData       = false;   // also read the range back to the host (GetDepthRange)
    };

    explicit DepthRangeCalculator(const CreateInfo& CI)
    {
        detail::Check(dfx_depth_range_create(CI.ReadBackData ? 1 : 0, &m_Fx), "dfx_depth_range_create");
        m_Buffer = IBuffer{m_Fx ? dfx_depth_range_get_buffer(m_Fx) : nullptr};
    }
    ~DepthRangeCalculator() { dfx_depth_range_destroy(m_Fx); }
    DepthRangeCalculator(const DepthRangeCalculator&)            = delete;
    DepthRangeCalculator& operator=(const DepthRangeCalculator&) = delete;

    bool IsReady() const { return m_Fx != nullptr; }

    // pCameraAttribs: the camera (CameraAttribs, device memory) the range is computed for
    std::unique_ptr<IShaderResourceBinding> CreateSRB(ITextureView* pDepthBufferSRV, IBuffer* pCameraAttribs)
    {
        return std::unique_ptr<IShaderResourceBinding>(new IShaderResourceBinding{pDepthBufferSRV, pCameraAttribs});
    }

    struct ComputeRangeAttribs
    {
        IDeviceContext*         pContext = nullptr;
        IShaderResourceBinding* pSRB     = nullptr; // from CreateSRB()
        Uint32                  Width    = 0;       // the depth buffer's size
        Uint32                  Height   = 0;
    };

    // DepthRangeCalculator.cpp:222-272: the range goes to GetDepthRangeBuffer(), and with ReadBackData also to the host.
    void ComputeRange(const ComputeRangeAttribs& Attribs)
    {
        DFX_DEV_CHECK_ERR(Attribs.pContext != nullptr, "Context must not be null");
        DFX_DEV_CHECK_ERR(Attribs.pSRB != nullptr, "SRB must not be null");
        if (Attribs.pContext == nullptr || Attribs.pSRB == nullptr) return;
        const dfx_plane* depth = Attribs.pSRB->GetDepthSRV() ? Attribs.pSRB->GetDepthSRV()->GetPlane() : nullptr;
        DFX_DEV_CHECK_ERR(depth == nullptr || (Uint32(depth->width) == Attribs.Width && Uint32(depth->height) == Attribs.Height),
                          "Width / Height must be the depth buffer's size");
        const IBuffer* cam = Attribs.pSRB->GetCameraAttribs();
        detail::Check(dfx_depth_range_compute(m_Fx, detail::StreamOf(Attribs.pContext),
                                              cam ? static_cast<const dfx_camera_attribs*>(cam->GetDevicePtr()) : nullptr, depth),
                      "DepthRangeCalculator::ComputeRange");
    }

    // four floats in device memory, laid out as CameraAttribs::fSceneNearZ .. fSceneFarDepth
    IBuffer* GetDepthRangeBuffer() const { return &m_Buffer; }

    struct DepthRange
    {
        float fSceneNearZ     = 0;
        float fSceneFarZ      = 0;
        float fSceneNearDepth = 0;
        float fSceneFarDepth  = 0;

        constexpr operator bool() const { return fSceneNearDepth > 0 && fSceneFarDepth > 0; }
    };

    // pCtx != nullptr: poll the read-back copies first (never waits)
    const DepthRange& GetDepthRange(IDeviceContext* pCtx = nullptr)
    {
        dfx_scene_depth_range r{};
        if (detail::Check(dfx_depth_range_get_range(m_Fx, pCtx != nullptr, &r), "DepthRangeCalculator::GetDepthRange"))
            m_DepthRange = DepthRange{r.fSceneNearZ, r.fSceneFarZ, r.fSceneNearDepth, r.fSceneFarDepth};
        return m_DepthRange;
    }

private:
    dfx_depth_range* m_Fx = nullptr;
    mutable IBuffer  m_Buffer; // handed out by the const GetDepthRangeBuffer(), as the reference does
    DepthRange       m_DepthRange;
};

} // namespace Diligent
