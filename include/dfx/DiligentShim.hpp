// DiligentShim.hpp — the minimal slice of DiligentCore's vocabulary that the PostProcess classes expose in their public
// signatures, re-declared over CUDA planes so that code written against the reference's
//     PostProcess/*/interface/*.hpp   (PostFXContext.hpp:51-172, ScreenSpaceAmbientOcclusion.hpp:59-136,
//                                      ScreenSpaceReflection.hpp:64-139, Bloom.hpp:60-114, TemporalAntiAliasing.hpp:62-156)
// compiles against this library instead. Nothing here talks to a graphics API:
//     ITextureView    == a pitched fp32 plane in HBM (dfx_plane)
//     IDeviceContext  == a CUDA stream
//     IRenderDevice   == the current CUDA device (carries no state)
//     IRenderStateCache is accepted and ignored (there are no PSOs to cache: kernels are compiled ahead of time).
// Host code only: no CUDA headers are needed to use these classes, everything goes through the C-ABI (dfx_b200.h).
#pragma once
#include <cassert>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <memory>

#include "../dfx_b200.h"

namespace Diligent
{

using Uint32 = uint32_t;
using Int32  = int32_t;
using Uint8  = uint8_t;
using Bool   = bool;

#define DFX_DEV_CHECK_ERR(expr, msg) assert((expr) && msg)                              /* DEV_CHECK_ERR: debug-build assert only */
#define DFX_LOG_ERROR_MESSAGE(...) (std::fprintf(stderr, "DiligentFX-b200 error: " __VA_ARGS__), std::fputc('\n', stderr)) /* LOG_ERROR_MESSAGE */

#ifndef DEFINE_FLAG_ENUM_OPERATORS
#    define DEFINE_FLAG_ENUM_OPERATORS(ENUMTYPE)                                                                                                   \
        inline ENUMTYPE  operator|(ENUMTYPE a, ENUMTYPE b) { return static_cast<ENUMTYPE>(static_cast<Uint32>(a) | static_cast<Uint32>(b)); }      \
        inline ENUMTYPE  operator&(ENUMTYPE a, ENUMTYPE b) { return static_cast<ENUMTYPE>(static_cast<Uint32>(a) & static_cast<Uint32>(b)); }      \
        inline ENUMTYPE  operator~(ENUMTYPE a) { return static_cast<ENUMTYPE>(~static_cast<Uint32>(a)); }                                          \
        inline ENUMTYPE& operator|=(ENUMTYPE& a, ENUMTYPE b) { return a = a | b; }                                                                 \
        inline ENUMTYPE& operator&=(ENUMTYPE& a, ENUMTYPE b) { return a = a & b; }
#endif

struct float2
{
    float x = 0, y = 0;
    float2() = default;
    float2(float x_, float y_) : x{x_}, y{y_} {}
};

// Row-major 4x4 with the reference's element names (BasicMath.hpp): m<row><col>, row-vector convention.
struct float4x4
{
    float m00 = 1, m01 = 0, m02 = 0, m03 = 0;
    float m10 = 0, m11 = 1, m12 = 0, m13 = 0;
    float m20 = 0, m21 = 0, m22 = 1, m23 = 0;
    float m30 = 0, m31 = 0, m32 = 0, m33 = 1;
};
static_assert(sizeof(float4x4) == sizeof(dfx_float4x4), "float4x4 must alias dfx_float4x4");

enum TEXTURE_FORMAT : Uint32
{
    TEX_FORMAT_UNKNOWN      = DFX_FORMAT_UNKNOWN,
    TEX_FORMAT_R32_FLOAT    = DFX_FORMAT_R32F,
    TEX_FORMAT_RG32_FLOAT   = DFX_FORMAT_RG32F,
    TEX_FORMAT_RGBA32_FLOAT = DFX_FORMAT_RGBA32F,
    TEX_FORMAT_R8_UINT      = DFX_FORMAT_R8U,
    // the G-buffer's own formats (Hydrogent/src/Tasks/HnBeginFrameTask.cpp:63-69): read by the passes as they are
    TEX_FORMAT_RGBA16_FLOAT = DFX_FORMAT_RGBA16F,
    TEX_FORMAT_RG16_FLOAT   = DFX_FORMAT_RG16F,
    TEX_FORMAT_RG8_UNORM    = DFX_FORMAT_RG8U,
    TEX_FORMAT_RGBA8_UNORM  = DFX_FORMAT_RGBA8U,
    TEX_FORMAT_D32_FLOAT    = DFX_FORMAT_R32F, // depth is an R32F plane here
    // the shadow maps' own formats (ShadowMapManager.hpp)
    TEX_FORMAT_D16_UNORM    = DFX_FORMAT_R16U,
    TEX_FORMAT_RG16_UNORM   = DFX_FORMAT_RG16U
};

class IRenderDevice
{
};
class IRenderStateCache
{
};

// A CUDA stream. The stream handle is a cudaStream_t passed as void* (nullptr = the default stream).
class IDeviceContext
{
public:
    explicit IDeviceContext(void* cuda_stream = nullptr) : m_Stream{cuda_stream} {}
    void* GetStream() const { return m_Stream; }
    void  WaitForIdle() const { dfx_stream_synchronize(m_Stream); }

private:
    void* m_Stream;
};

class ITextureView;

// A device plane. Owning instances allocate through the library; non-owning ones wrap an existing dfx_plane
// (effect outputs, or memory the application allocated itself with cudaMalloc / torch).
class ITexture
{
public:
    ITexture() = default;
    ITexture(Uint32 Width, Uint32 Height, TEXTURE_FORMAT Format) : m_Owning{true}
    {
        if (dfx_plane_alloc(static_cast<int32_t>(Width), static_cast<int32_t>(Height), static_cast<int32_t>(Format), &m_Plane) != DFX_OK)
            DFX_LOG_ERROR_MESSAGE("failed to allocate %ux%u plane: %s", Width, Height, dfx_last_error());
    }
    explicit ITexture(const dfx_plane& Plane) : m_Plane{Plane} {}
    ITexture(const ITexture&)            = delete;
    ITexture& operator=(const ITexture&) = delete;
    ~ITexture()
    {
        if (m_Owning) dfx_plane_free(&m_Plane);
    }
    const dfx_plane& GetPlane() const { return m_Plane; }
    void             SetPlane(const dfx_plane& p) { m_Plane = p; }
    Uint32           GetWidth() const { return static_cast<Uint32>(m_Plane.width); }
    Uint32           GetHeight() const { return static_cast<Uint32>(m_Plane.height); }
    bool UpdateData(IDeviceContext* pCtx, const void* pHostData, size_t HostPitchBytes = 0)
    {
        return dfx_plane_upload(pCtx ? pCtx->GetStream() : nullptr, &m_Plane, pHostData, HostPitchBytes) == DFX_OK;
    }
    bool ReadData(IDeviceContext* pCtx, void* pHostData, size_t HostPitchBytes = 0) const
    {
        void* s = pCtx ? pCtx->GetStream() : nullptr;
        return dfx_plane_download(s, &m_Plane, pHostData, HostPitchBytes) == DFX_OK && dfx_stream_synchronize(s) == DFX_OK;
    }

private:
    dfx_plane m_Plane{};
    bool      m_Owning = false;
};

class ITextureView
{
public:
    ITextureView() = default;
    explicit ITextureView(ITexture* pTexture) : m_pTexture{pTexture} {}
    ITexture*        GetTexture() const { return m_pTexture; }
    const dfx_plane* GetPlane() const { return m_pTexture ? &m_pTexture->GetPlane() : nullptr; }

private:
    ITexture* m_pTexture = nullptr;
};

// The camera constant buffer (two CameraAttribs in device memory); only its identity matters to callers.
class IBuffer
{
public:
    explicit IBuffer(const void* pDevice = nullptr) : m_pDevice{pDevice} {}
    const void* GetDevicePtr() const { return m_pDevice; }

private:
    const void* m_pDevice;
};

// What a shader resource binding of the reference holds for a compute pass: the views and buffers it reads. Here it only keeps
// the pointers (DepthRangeCalculator::CreateSRB); the objects must outlive it.
class IShaderResourceBinding
{
public:
    IShaderResourceBinding(ITextureView* pDepthSRV, IBuffer* pCameraAttribs) : m_pDepthSRV{pDepthSRV}, m_pCameraAttribs{pCameraAttribs} {}
    ITextureView* GetDepthSRV() const { return m_pDepthSRV; }
    IBuffer*      GetCameraAttribs() const { return m_pCameraAttribs; }

private:
    ITextureView* m_pDepthSRV;
    IBuffer*      m_pCameraAttribs;
};

// The constant blocks shared by C++ and HLSL in the reference (Shaders/**/public/*Structures.fxh, BasicStructures.fxh) with
// their DEFAULT_VALUE()s; layouts are the byte-identical C structs of dfx_b200.h.
namespace HLSL
{
struct CameraAttribs : dfx_camera_attribs
{
    CameraAttribs()
    {
        std::memset(static_cast<dfx_camera_attribs*>(this), 0, sizeof(dfx_camera_attribs));
        fFocusDistance = 10.0f, fFStop = 5.6f, fFocalLength = 50.0f, fSensorWidth = 36.0f, fSensorHeight = 24.0f, fExposure = 0.0f;
    }
    // BasicStructures.fxh:134-147
    void SetClipPlanes(float fNearZ, float fFarZ)
    {
        const bool UseReverseDepth = fNearZ > fFarZ;
        fNearPlaneZ     = UseReverseDepth ? fFarZ : fNearZ;
        fFarPlaneZ      = UseReverseDepth ? fNearZ : fFarZ;
        fNearPlaneDepth = UseReverseDepth ? 1.f : 0.f;
        fFarPlaneDepth  = UseReverseDepth ? 0.f : 1.f;
        fSceneNearZ = fNearPlaneZ, fSceneFarZ = fFarPlaneZ, fSceneNearDepth = fNearPlaneDepth, fSceneFarDepth = fFarPlaneDepth;
    }
};
struct ScreenSpaceAmbientOcclusionAttribs : dfx_ssao_attribs
{
    ScreenSpaceAmbientOcclusionAttribs() { dfx_ssao_attribs_default(this); }
};
struct ScreenSpaceReflectionAttribs : dfx_ssr_attribs
{
    ScreenSpaceReflectionAttribs() { dfx_ssr_attribs_default(this); }
};
struct DepthOfFieldAttribs : dfx_dof_attribs // DepthOfFieldStructures.fxh:31-56
{
    DepthOfFieldAttribs() : dfx_dof_attribs{0.01f, 0.9375f, 5, 7, 1.0f, 0.0f, 0.0f, 0.0f} {}
};
struct BloomAttribs : dfx_bloom_attribs
{
    BloomAttribs() { dfx_bloom_attribs_default(this); }
};
struct TemporalAntiAliasingAttribs : dfx_taa_attribs
{
    TemporalAntiAliasingAttribs() { dfx_taa_attribs_default(this); }
};
struct ToneMappingAttribs : dfx_tonemap_attribs
{
    ToneMappingAttribs() { dfx_tonemap_attribs_default(this); }
};
static_assert(sizeof(CameraAttribs) == 576 && sizeof(ScreenSpaceAmbientOcclusionAttribs) == 48 && sizeof(ScreenSpaceReflectionAttribs) == 48 &&
                  sizeof(BloomAttribs) == 32 && sizeof(TemporalAntiAliasingAttribs) == 16 && sizeof(ToneMappingAttribs) == 48,
              "constant blocks must keep the reference layout");
} // namespace HLSL

namespace detail
{
// Keeps an ITexture/ITextureView pair alive for a plane that an effect owns (what Get*SRV() hands out).
struct PlaneView
{
    ITexture     Tex;
    ITextureView View{&Tex};
    ITextureView* Update(const dfx_plane& p)
    {
        Tex.SetPlane(p);
        return &View;
    }
};
inline void* StreamOf(IDeviceContext* pCtx) { return pCtx ? pCtx->GetStream() : nullptr; }
inline bool  Check(dfx_status st, const char* what)
{
    if (st != DFX_OK) DFX_LOG_ERROR_MESSAGE("%s failed (%d): %s", what, static_cast<int>(st), dfx_last_error());
    return st == DFX_OK;
}
} // namespace detail

} // namespace Diligent
