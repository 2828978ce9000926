// dfx_common.cuh — device-side vocabulary shared by all kernels of libdfx_b200.so (sm_90a only).
//
// Conventions (SURVEY.md Appendix B; the DiligentCore macros the reference shaders rely on, D3D/Vulkan flavour):
//   pixel centre = (x + 0.5, y + 0.5), y down; UV = pos / size; NDC y up, NDC z == depth in [0,1];
//   matrices are row-major and multiply row vectors: clip = float4(p, 1) * M.
// Planes are pitched fp32 arrays in HBM; all global loads of read-only planes go through the non-coherent path
// (ld.global.nc) and are 64/128-bit wide where the element type allows.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>
#include "../../include/dfx_b200.h"

// Minimum resident CTAs per SM requested from ptxas for the latency-bound gather kernels (register budget = 65536 /
// (256 * N)), from an occupancy sweep of the kernels. Overridable with -D.
#ifndef DFX_OCC_INTERSECT
#    define DFX_OCC_INTERSECT 6
#endif
#ifndef DFX_OCC_SSR_SPATIAL
#    define DFX_OCC_SSR_SPATIAL 6
#endif
#ifndef DFX_OCC_SSR_TEMPORAL
#    define DFX_OCC_SSR_TEMPORAL 6
#endif
#ifndef DFX_OCC_AO
#    define DFX_OCC_AO 5
#endif
#ifndef DFX_OCC_TAA
#    define DFX_OCC_TAA 6
#endif
#ifndef DFX_OCC_FRONT
#    define DFX_OCC_FRONT 6
#endif

namespace dfx
{

// ---------------------------------------------------------------------------------------------------------------------
// host side: status handling and launch accounting
// ---------------------------------------------------------------------------------------------------------------------
dfx_status set_error(dfx_status st, const char* fmt, ...);
dfx_status check_cuda(cudaError_t e, const char* what);
void       count_launch(int n = 1);

#define DFX_REQUIRE(cond, ...)                                       \
    do {                                                             \
        if (!(cond)) return ::dfx::set_error(DFX_ERR_INVALID_ARG, __VA_ARGS__); \
    } while (0)

#define DFX_CUDA(call)                                               \
    do {                                                             \
        cudaError_t e__ = (call);                                    \
        if (e__ != cudaSuccess) return ::dfx::check_cuda(e__, #call); \
    } while (0)

// after a kernel launch
#define DFX_LAUNCHED(name)                                           \
    do {                                                             \
        ::dfx::count_launch();                                       \
        cudaError_t e__ = cudaGetLastError();                        \
        if (e__ != cudaSuccess) return ::dfx::check_cuda(e__, name); \
    } while (0)

// Optional per-pass device timing (dfx_profile_* in the C-ABI): when enabled, every dfx_pass_* call brackets its launches
// with a pair of CUDA events on the launching stream.
struct ProfileScope
{
    cudaStream_t s;
    int          slot;
    ProfileScope(void* stream, const char* name);
    ~ProfileScope();
};
#define DFX_PROFILE(stream, name) ::dfx::ProfileScope profile_scope__(stream, name)
// NVTX range around an effect's Execute(), named like the reference's outer ScopedDebugGroup ("ScreenSpaceAmbientOcclusion", "Bloom", ...)
struct EffectRange
{
    explicit EffectRange(const char* name);
    ~EffectRange();
};

inline cudaStream_t as_stream(void* s) { return static_cast<cudaStream_t>(s); }
inline int          div_up(int a, int b) { return (a + b - 1) / b; }

// ---------------------------------------------------------------------------------------------------------------------
// plane views
// ---------------------------------------------------------------------------------------------------------------------
template <class T>
struct View
{
    T*  p;
    int pitch; // in elements of T
    int w, h;
    __device__ __forceinline__ T&       at(int x, int y) const { return p[(unsigned)(y * pitch + x)]; } // planes hold < 2^31 texels (host-checked): 32-bit index, one IMAD + one IMAD.WIDE
    __device__ __forceinline__ const T* row(int y) const { return p + (unsigned)(y * pitch); }
    __device__ __forceinline__ typename std::remove_const<T>::type ld(int x, int y) const { return __ldg(p + (unsigned)(y * pitch + x)); } // read-only path
};

// A plane of a frame that is split into row strips over several GPUs (dfx_strips.cu): every GPU holds the plane at the same offset of
// an identically laid-out slab, rows are owned in 64-row blocks, and a texel is loaded from the slab of the GPU that owns its row
// (peer memory over NVLink; the own slab for own rows). `delta[g]` = byte distance from this GPU's slab to GPU g's mapping.
constexpr int kPeerBlockShift = 6;
constexpr int kPeerMaxBlocks  = 256; // 64-row blocks: heights up to 16384
struct PeerMap
{
    long long delta[DFX_MAX_PEERS];
    uint8_t   owner[kPeerMaxBlocks];
};
template <class T>
struct PeerView
{
    const T*       p;
    int            pitch, w, h;
    const PeerMap* pm;
    __device__ __forceinline__ T ld(int x, int y) const
    {
        const char* q = reinterpret_cast<const char*>(p + (unsigned)(y * pitch + x)) + pm->delta[pm->owner[y >> kPeerBlockShift]];
        return __ldg(reinterpret_cast<const T*>(q));
    }
};

// G-buffer planes as the renderer stores them (Hydrogent/src/Tasks/HnBeginFrameTask.cpp:63-69: colour and normal RGBA16_FLOAT, motion
// RG16_FLOAT, material RG8_UNORM) or widened to fp32: the kernels that read them take a Tex4 / Tex2, whose storage format is a
// warp-uniform run-time field. Every half and every UNORM8 value is an fp32 value, so a pass computes bit for bit the same from
// either representation; the narrow one halves (or better) the bytes the pass reads.
struct Tex4
{
    const char* p;
    int         pitch; // bytes
    int         w, h, fmt; // DFX_FORMAT_RGBA32F | DFX_FORMAT_RGBA16F | DFX_FORMAT_RG8U (r, g, 0, 0)
    __device__ __forceinline__ float4 ld(int x, int y) const
    {
        const char* row = p + (unsigned)(y * pitch); // planes are < 2^31 bytes (host-checked)
        if (fmt == DFX_FORMAT_RGBA32F) return __ldg(reinterpret_cast<const float4*>(row) + x);
        if (fmt == DFX_FORMAT_RGBA16F)
        {
            const uint2  v = __ldg(reinterpret_cast<const uint2*>(row) + x);
            const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&v.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&v.y));
            return make_float4(a.x, a.y, b.x, b.y);
        }
        const uchar2 v = __ldg(reinterpret_cast<const uchar2*>(row) + x);
        return make_float4(float(v.x) / 255.0f, float(v.y) / 255.0f, 0.0f, 0.0f); // UNORM -> float: c / 255, correctly rounded
    }
};
struct Tex2
{
    const char* p;
    int         pitch; // bytes
    int         w, h, fmt; // DFX_FORMAT_RG32F | DFX_FORMAT_RG16F
    __device__ __forceinline__ float2 ld(int x, int y) const
    {
        const char* row = p + (unsigned)(y * pitch);
        if (fmt == DFX_FORMAT_RG32F) return __ldg(reinterpret_cast<const float2*>(row) + x);
        const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(row) + x);
        return __half22float2(*reinterpret_cast<const __half2*>(&v));
    }
};
// The same with the format as a COMPILE-TIME parameter: what the kernels take. The run-time form above costs the issue-bound kernels
// registers (a fifth field per plane, both load paths live: slower ray march, spills under its 40-register cap);
// the host picks the instantiation from the plane's format (DFX_FMT16 below).
template <int FMT>
struct Tex4T
{
    const char* p;
    int         pitch, w, h;
    __host__ __device__ Tex4T() = default;
    __host__ __device__ Tex4T(const Tex4& t) : p(t.p), pitch(t.pitch), w(t.w), h(t.h) {}
    __device__ __forceinline__ float4 ld(int x, int y) const
    {
        const char* row = p + (unsigned)(y * pitch);
        if constexpr (FMT == DFX_FORMAT_RGBA32F) return __ldg(reinterpret_cast<const float4*>(row) + x);
        else if constexpr (FMT == DFX_FORMAT_RGBA16F)
        {
            const uint2  v = __ldg(reinterpret_cast<const uint2*>(row) + x);
            const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&v.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&v.y));
            return make_float4(a.x, a.y, b.x, b.y);
        }
        else
        {
            const uchar2 v = __ldg(reinterpret_cast<const uchar2*>(row) + x);
            return make_float4(float(v.x) / 255.0f, float(v.y) / 255.0f, 0.0f, 0.0f);
        }
    }
};
template <int FMT>
struct Tex2T
{
    const char* p;
    int         pitch, w, h;
    __host__ __device__ Tex2T() = default;
    __host__ __device__ Tex2T(const Tex2& t) : p(t.p), pitch(t.pitch), w(t.w), h(t.h) {}
    __device__ __forceinline__ float2 ld(int x, int y) const
    {
        const char* row = p + (unsigned)(y * pitch);
        if constexpr (FMT == DFX_FORMAT_RG32F) return __ldg(reinterpret_cast<const float2*>(row) + x);
        else
        {
            const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(row) + x);
            return __half22float2(*reinterpret_cast<const __half2*>(&v));
        }
    }
};
template <bool H16> using TexRGBA = Tex4T<H16 ? DFX_FORMAT_RGBA16F : DFX_FORMAT_RGBA32F>;
template <bool H16> using TexRG   = Tex2T<H16 ? DFX_FORMAT_RG16F : DFX_FORMAT_RG32F>;
inline bool is16(const Tex4& t) { return t.fmt == DFX_FORMAT_RGBA16F; }
inline bool is16(const Tex2& t) { return t.fmt == DFX_FORMAT_RG16F; }
// DFX_FMT16(cond, H, statement): runs `statement` with `constexpr bool H` = cond
#define DFX_FMT16(cond, H, ...)          \
    do {                                 \
        if (cond)                        \
        {                                \
            constexpr bool H = true;     \
            __VA_ARGS__;                 \
        }                                \
        else                             \
        {                                \
            constexpr bool H = false;    \
            __VA_ARGS__;                 \
        }                                \
    } while (0)

inline bool make_tex4(const dfx_plane* pl, Tex4& t, bool allow_rg8 = false)
{
    if (!pl || !pl->ptr || pl->width <= 0 || pl->height <= 0) return false;
    const size_t bpt = pl->format == DFX_FORMAT_RGBA32F ? 16 : pl->format == DFX_FORMAT_RGBA16F ? 8 : (pl->format == DFX_FORMAT_RG8U && allow_rg8) ? 2 : 0;
    if (!bpt || pl->pitch_bytes % bpt != 0 || pl->pitch_bytes < size_t(pl->width) * bpt || reinterpret_cast<uintptr_t>(pl->ptr) % bpt != 0) return false;
    if (pl->pitch_bytes * size_t(pl->height) >= (size_t(1) << 31)) return false;
    t = Tex4{static_cast<const char*>(pl->ptr), int(pl->pitch_bytes), pl->width, pl->height, pl->format};
    return true;
}
inline bool make_tex2(const dfx_plane* pl, Tex2& t)
{
    if (!pl || !pl->ptr || pl->width <= 0 || pl->height <= 0) return false;
    const size_t bpt = pl->format == DFX_FORMAT_RG32F ? 8 : pl->format == DFX_FORMAT_RG16F ? 4 : 0;
    if (!bpt || pl->pitch_bytes % bpt != 0 || pl->pitch_bytes < size_t(pl->width) * bpt || reinterpret_cast<uintptr_t>(pl->ptr) % bpt != 0) return false;
    if (pl->pitch_bytes * size_t(pl->height) >= (size_t(1) << 31)) return false;
    t = Tex2{static_cast<const char*>(pl->ptr), int(pl->pitch_bytes), pl->width, pl->height, pl->format};
    return true;
}
#define DFX_TEX4(name, plane)                                                                                                      \
    ::dfx::Tex4 name;                                                                                                              \
    if (!::dfx::make_tex4(plane, name)) return ::dfx::set_error(DFX_ERR_INVALID_ARG, "bad plane '%s' (RGBA32F or RGBA16F expected; null, pitch or alignment)", #plane)
#define DFX_TEX2(name, plane)                                                                                                      \
    ::dfx::Tex2 name;                                                                                                              \
    if (!::dfx::make_tex2(plane, name)) return ::dfx::set_error(DFX_ERR_INVALID_ARG, "bad plane '%s' (RG32F or RG16F expected; null, pitch or alignment)", #plane)

// host: dfx_peer_map (C-ABI) -> the table the kernels index
inline bool make_peer_map(const dfx_peer_map* m, int height, PeerMap& out)
{
    if (!m || m->count < 1 || m->count > DFX_MAX_PEERS || m->rank < 0 || m->rank >= m->count) return false;
    if (m->row_begin[0] != 0 || m->row_begin[m->count] != height || ((height + 63) >> kPeerBlockShift) > kPeerMaxBlocks) return false;
    for (int r = 0; r < m->count; ++r)
    {
        if (!m->base[r] || m->row_begin[r + 1] < m->row_begin[r] || (r > 0 && m->row_begin[r] % 64 != 0)) return false;
        out.delta[r] = static_cast<long long>(reinterpret_cast<intptr_t>(m->base[r]) - reinterpret_cast<intptr_t>(m->base[m->rank]));
    }
    for (int r = m->count; r < DFX_MAX_PEERS; ++r) out.delta[r] = 0;
    for (int b = 0, r = 0; b < kPeerMaxBlocks; ++b)
    {
        while (r + 1 < m->count && (b << kPeerBlockShift) >= m->row_begin[r + 1]) ++r;
        out.owner[b] = (uint8_t)r;
    }
    return true;
}

template <class T> __device__ __forceinline__ T ldg(const T* p) { return __ldg(p); }

// Texture.Load semantics: out of bounds -> 0. V = View<const T> or PeerView<T>.
template <class T> __device__ __forceinline__ T zero_of();
template <> __device__ __forceinline__ float  zero_of<float>() { return 0.0f; }
template <> __device__ __forceinline__ float2 zero_of<float2>() { return make_float2(0.f, 0.f); }
template <> __device__ __forceinline__ float4 zero_of<float4>() { return make_float4(0.f, 0.f, 0.f, 0.f); }
template <class V>
__device__ __forceinline__ auto load0(const V& v, int x, int y) -> decltype(v.ld(0, 0))
{
    using T = decltype(v.ld(0, 0));
    return ((unsigned)x < (unsigned)v.w && (unsigned)y < (unsigned)v.h) ? v.ld(x, y) : zero_of<T>();
}
template <class V>
__device__ __forceinline__ auto loadc(const V& v, int x, int y) -> decltype(v.ld(0, 0)) // clamp addressing
{
    x = min(max(x, 0), v.w - 1);
    y = min(max(y, 0), v.h - 1);
    return v.ld(x, y);
}

template <class T>
inline bool make_view(const dfx_plane* pl, int fmt, View<T>& v)
{
    if (!pl || !pl->ptr || pl->format != fmt || pl->width <= 0 || pl->height <= 0) return false;
    if (pl->pitch_bytes % sizeof(T) != 0 || pl->pitch_bytes < (size_t)pl->width * sizeof(T)) return false;
    if (reinterpret_cast<uintptr_t>(pl->ptr) % sizeof(T) != 0) return false;
    if ((pl->pitch_bytes / sizeof(T)) * (size_t)pl->height >= (size_t(1) << 31)) return false; // kernels index texels with 32 bits
    v.p     = static_cast<T*>(pl->ptr);
    v.pitch = int(pl->pitch_bytes / sizeof(T));
    v.w     = pl->width;
    v.h     = pl->height;
    return true;
}
#define DFX_VIEW(T, name, plane, fmt)                                                                   \
    ::dfx::View<T> name;                                                                                \
    if (!::dfx::make_view<T>(plane, fmt, name)) return ::dfx::set_error(DFX_ERR_INVALID_ARG, "bad plane '%s' (null, wrong format, pitch or alignment)", #plane)

#define DFX_SAME_SIZE(a, b) DFX_REQUIRE((a).w == (b).w && (a).h == (b).h, "plane size mismatch: %s vs %s", #a, #b)

inline bool rows_ok(dfx_rows r, int h) { return r.y0 >= 0 && r.y1 <= h && r.y0 <= r.y1; }
// A G-buffer plane a pass writes in place in one of two formats (bytes per texel bpt32 / bpt16): its pointer, pitch and whether it is
// the 16-bit one; false on a null, mis-pitched, misaligned or >= 2 GiB plane.
inline bool writable(const dfx_plane* pl, int f32, int f16, int bpt32, int bpt16, char*& p, int& pitch, int& is16)
{
    if (!pl || !pl->ptr || pl->width <= 0 || pl->height <= 0 || (pl->format != f32 && pl->format != f16)) return false;
    const size_t bpt = pl->format == f32 ? bpt32 : bpt16;
    if (pl->pitch_bytes % bpt != 0 || pl->pitch_bytes < size_t(pl->width) * bpt || reinterpret_cast<uintptr_t>(pl->ptr) % bpt != 0) return false;
    if (pl->pitch_bytes * size_t(pl->height) >= (size_t(1) << 31)) return false;
    p = static_cast<char*>(pl->ptr), pitch = int(pl->pitch_bytes), is16 = pl->format == f16;
    return true;
}

struct PyrView
{
    View<const float> lv[DFX_MAX_MIPS];
    int               levels;
};
struct PyrViewRW
{
    View<float> lv[DFX_MAX_MIPS];
    int         levels;
};

// ---------------------------------------------------------------------------------------------------------------------
// small vector helpers (CUDA has the types but no operators)
// ---------------------------------------------------------------------------------------------------------------------
#define DFX_HD __device__ __forceinline__
DFX_HD float2 operator+(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
DFX_HD float2 operator-(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
DFX_HD float2 operator*(float2 a, float2 b) { return make_float2(a.x * b.x, a.y * b.y); }
DFX_HD float2 operator*(float2 a, float b) { return make_float2(a.x * b, a.y * b); }
DFX_HD float2 operator*(float a, float2 b) { return make_float2(a * b.x, a * b.y); }
DFX_HD float3 operator+(float3 a, float3 b) { return make_float3(a.x + b.x, a.y + b.y, a.z + b.z); }
DFX_HD float3 operator-(float3 a, float3 b) { return make_float3(a.x - b.x, a.y - b.y, a.z - b.z); }
DFX_HD float3 operator*(float3 a, float3 b) { return make_float3(a.x * b.x, a.y * b.y, a.z * b.z); }
DFX_HD float3 operator*(float3 a, float b) { return make_float3(a.x * b, a.y * b, a.z * b); }
DFX_HD float3 operator*(float a, float3 b) { return make_float3(a * b.x, a * b.y, a * b.z); }
DFX_HD float3 operator/(float3 a, float b) { return make_float3(a.x / b, a.y / b, a.z / b); }
DFX_HD float3 operator-(float3 a) { return make_float3(-a.x, -a.y, -a.z); }
DFX_HD float4 operator+(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
DFX_HD float4 operator-(float4 a, float4 b) { return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w); }
DFX_HD float4 operator*(float4 a, float4 b) { return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }
DFX_HD float4 operator*(float4 a, float b) { return make_float4(a.x * b, a.y * b, a.z * b, a.w * b); }
DFX_HD float4 operator*(float a, float4 b) { return make_float4(a * b.x, a * b.y, a * b.z, a * b.w); }
DFX_HD float4 operator/(float4 a, float b) { return make_float4(a.x / b, a.y / b, a.z / b, a.w / b); }
DFX_HD float  dot(float2 a, float2 b) { return a.x * b.x + a.y * b.y; }
DFX_HD float  dot(float3 a, float3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
DFX_HD float  dot(float4 a, float4 b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }
DFX_HD float3 cross(float3 a, float3 b) { return make_float3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
DFX_HD float  length(float2 a) { return sqrtf(dot(a, a)); }
DFX_HD float  length(float3 a) { return sqrtf(dot(a, a)); }
DFX_HD float3 normalize(float3 a) { return a / length(a); }
DFX_HD float3 xyz(float4 a) { return make_float3(a.x, a.y, a.z); }
DFX_HD float4 f4(float3 a, float w) { return make_float4(a.x, a.y, a.z, w); }
DFX_HD float  saturate(float v) { return __saturatef(v); } // NaN -> 0, same as fmin(fmax(v,0),1)
DFX_HD float  lerpf(float a, float b, float t) { return a + t * (b - a); }
DFX_HD float3 lerp3(float3 a, float3 b, float t) { return a + t * (b - a); }
DFX_HD float4 lerp4(float4 a, float4 b, float t) { return a + t * (b - a); }
DFX_HD float  fracf(float v) { return v - floorf(v); }
DFX_HD float  signf(float v) { return float((v > 0.0f) - (v < 0.0f)); }
DFX_HD float  luminance(float3 c) { return dot(c, make_float3(0.299f, 0.587f, 0.114f)); }
// products and sums rounded separately (never contracted into an FMA): the passes that are bit for bit a shader's arithmetic
DFX_HD float mul_(float a, float b) { return __fmul_rn(a, b); }
DFX_HD float add_(float a, float b) { return __fadd_rn(a, b); }
DFX_HD float sub_(float a, float b) { return __fsub_rn(a, b); }
// HLSL's min / max as the reference's shader runner evaluates them, the C library's fminf / fmaxf: a NaN operand yields the other one;
// of +0 and -0 the second operand wins
DFX_HD float min_(float a, float b) { return (a < b || b != b) ? a : b; }
DFX_HD float max_(float a, float b) { return (a > b || b != b) ? a : b; }
DFX_HD float  smoothstepf(float a, float b, float x)
{
    float t = saturate((x - a) / (b - a));
    return t * t * (3.0f - 2.0f * t);
}

// ---------------------------------------------------------------------------------------------------------------------
// camera block: the fields the kernels use, staged once per CTA into shared memory from dfx_camera_attribs[2] in HBM
// ---------------------------------------------------------------------------------------------------------------------
struct Mat4
{
    float m[4][4];
};
struct CamS
{
    float    vw, vh, ivw, ivh; // f4ViewportSize
    float    px, py, pz;       // f4Position.xyz
    uint32_t frame_index;
    float    jx, jy;
    // projection terms used by depth<->cameraZ and ScreenXYDepthToViewSpace
    float m00, m11, m22, m32, m23, m33;
};

__device__ __forceinline__ void load_cam(CamS& c, const dfx_camera_attribs* a)
{
    c.vw = a->f4ViewportSize[0], c.vh = a->f4ViewportSize[1], c.ivw = a->f4ViewportSize[2], c.ivh = a->f4ViewportSize[3];
    c.px = a->f4Position[0], c.py = a->f4Position[1], c.pz = a->f4Position[2];
    c.frame_index = a->uiFrameIndex;
    c.jx = a->f2Jitter[0], c.jy = a->f2Jitter[1];
    c.m00 = a->mProj.m[0][0], c.m11 = a->mProj.m[1][1], c.m22 = a->mProj.m[2][2], c.m32 = a->mProj.m[3][2];
    c.m23 = a->mProj.m[2][3], c.m33 = a->mProj.m[3][3];
}
__device__ __forceinline__ void load_mat(Mat4& d, const dfx_float4x4& s)
{
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) d.m[r][c] = s.m[r][c];
}

// DepthToCameraZ / CameraZToDepth (ShaderUtilities.fxh:5-39): z = (m32 - d*m33) / (d*m23 - m22)
// (MUFU reciprocal + multiply, <= 2 ulp: every pass is issue-bound, and a correctly-rounded division costs ~8x as much)
DFX_HD float fdiv_(float a, float b) { return __fdividef(a, b); }
DFX_HD float depth_to_camz(float d, const CamS& c) { return fdiv_(c.m32 - d * c.m33, d * c.m23 - c.m22); }
DFX_HD float camz_to_depth(float z, const CamS& c) { return fdiv_(c.m22 * z + c.m32, c.m23 * z + c.m33); }
// ScreenXYDepthToViewSpace (PostFX_Common.fxh:107-111) with TexUVToNormalizedDeviceXY(uv) = (uv - 0.5) * (2, -2)
DFX_HD float3 screen_to_view(float u, float v, float depth, const CamS& c)
{
    float z  = depth_to_camz(depth, c);
    float nx = (u - 0.5f) * 2.0f, ny = (v - 0.5f) * -2.0f;
    return make_float3(fdiv_(z * nx, c.m00), fdiv_(z * ny, c.m11), z);
}
// float4(v,1) * M
DFX_HD float4 mul_point(float3 v, const Mat4& M)
{
    return make_float4(v.x * M.m[0][0] + v.y * M.m[1][0] + v.z * M.m[2][0] + M.m[3][0],
                       v.x * M.m[0][1] + v.y * M.m[1][1] + v.z * M.m[2][1] + M.m[3][1],
                       v.x * M.m[0][2] + v.y * M.m[1][2] + v.z * M.m[2][2] + M.m[3][2],
                       v.x * M.m[0][3] + v.y * M.m[1][3] + v.z * M.m[2][3] + M.m[3][3]);
}
// float4(v,0) * M (xyz)
DFX_HD float3 mul_dir(float3 v, const Mat4& M)
{
    return make_float3(v.x * M.m[0][0] + v.y * M.m[1][0] + v.z * M.m[2][0], v.x * M.m[0][1] + v.y * M.m[1][1] + v.z * M.m[2][1],
                       v.x * M.m[0][2] + v.y * M.m[1][2] + v.z * M.m[2][2]);
}
// ProjectPosition (PostFX_Common.fxh:85-92): world/view -> (u, v, depth)
DFX_HD float3 project_position(float3 p, const Mat4& M)
{
    float4 c = mul_point(p, M);
    float  iw = fdiv_(1.0f, c.w);
    float  x = c.x * iw, y = c.y * iw, z = c.z * iw;
    return make_float3(0.5f + 0.5f * x, 0.5f - 0.5f * y, z);
}
// InvProjectPosition (PostFX_Common.fxh:99-105): (u, v, depth) -> position
DFX_HD float3 inv_project_position(float u, float v, float depth, const Mat4& M)
{
    float4 c = mul_point(make_float3((u - 0.5f) * 2.0f, (v - 0.5f) * -2.0f, depth), M);
    float iw = fdiv_(1.0f, c.w);
    return make_float3(c.x * iw, c.y * iw, c.z * iw);
}

// Bayer4x4 (PostFX_Common.fxh:57-65)
DFX_HD float bayer4x4(uint32_t x, uint32_t y, uint32_t frame)
{
    uint32_t wx = x & 3u, wy = y & 3u;
    uint32_t A  = 2068378560u * (1u - (wx >> 1u)) + 1500172770u * (wx >> 1u);
    uint32_t B  = (wy + ((wx & 1u) << 2u)) << 2u;
    return float(((A >> B) + frame) & 0xFu) * (1.0f / 16.0f);
}

// GetBilinearSamplingInfoUC (ShaderUtilities.fxh:126-142)
struct Bilin
{
    int   x0, y0, x1, y1;
    float w00, w10, w01, w11;
};
DFX_HD Bilin bilinear_uc(float lx, float ly, int w, int h)
{
    lx -= 0.5f, ly -= 0.5f;
    float fx0 = floorf(lx), fy0 = floorf(ly);
    Bilin b;
    int   x0 = (int)fx0, y0 = (int)fy0;
    b.x0 = min(max(x0, 0), w - 1), b.y0 = min(max(y0, 0), h - 1);
    b.x1 = min(max(x0 + 1, 0), w - 1), b.y1 = min(max(y0 + 1, 0), h - 1);
    float x = lx - fx0, y = ly - fy0;
    b.w00 = (1.0f - x) * (1.0f - y), b.w10 = x * (1.0f - y), b.w01 = (1.0f - x) * y, b.w11 = x * y;
    return b;
}

// Fast (approximate, <= 2 ulp) arithmetic for the issue-bound kernels; used only where the parity budget allows.
// The .ftz forms are ONE MUFU instruction each; the non-ftz forms (__fdividef, rsqrtf, sqrt.approx.f32) wrap it in a
// denormal rescue (FSETP + 2-3 FMUL/FSEL) that cost 20 % of the TAA kernel's instructions. Denormal operands do not occur
// in this path (depths, luminances and squared lengths are either 0 or far above 1e-38), and 0 behaves the same.
DFX_HD float frcp(float a)
{
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a));
    return r;
}
DFX_HD float fdiv(float a, float b) { return a * frcp(b); }
DFX_HD float fsqrt(float a)
{
    float r;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a));
    return r;
}
DFX_HD float frsqrt(float a)
{
    float r;
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a));
    return r;
}
DFX_HD float3 fnormalize(float3 a) { return a * frsqrt(dot(a, a)); }

// The fixed-function sampler resolves the sample position to 8 fractional bits: snap to the nearest 1/256 texel.
DFX_HD float snap8(float p) { return floorf(p * 256.0f + 0.5f) * (1.0f / 256.0f); }

// bilinear SampleLevel at normalised uv, clamp addressing
template <class V>
__device__ __forceinline__ auto sample_linear_clamp(const V& t, float u, float v) -> decltype(t.ld(0, 0))
{
    using T = decltype(t.ld(0, 0));
    float px = snap8(u * float(t.w) - 0.5f), py = snap8(v * float(t.h) - 0.5f);
    float fx0 = floorf(px), fy0 = floorf(py);
    int   x0 = (int)fx0, y0 = (int)fy0;
    float fx = px - fx0, fy = py - fy0;
    T     a = loadc(t, x0, y0), b = loadc(t, x0 + 1, y0), c = loadc(t, x0, y0 + 1), d = loadc(t, x0 + 1, y0 + 1);
    return a * ((1.0f - fx) * (1.0f - fy)) + b * (fx * (1.0f - fy)) + c * ((1.0f - fx) * fy) + d * (fx * fy);
}
template <class V>
__device__ __forceinline__ auto sample_linear_border(const V& t, float u, float v) -> decltype(t.ld(0, 0))
{
    using T = decltype(t.ld(0, 0));
    float px = snap8(u * float(t.w) - 0.5f), py = snap8(v * float(t.h) - 0.5f);
    float fx0 = floorf(px), fy0 = floorf(py);
    int   x0 = (int)fx0, y0 = (int)fy0;
    float fx = px - fx0, fy = py - fy0;
    T     a = load0(t, x0, y0), b = load0(t, x0 + 1, y0), c = load0(t, x0, y0 + 1), d = load0(t, x0 + 1, y0 + 1);
    return a * ((1.0f - fx) * (1.0f - fy)) + b * (fx * (1.0f - fy)) + c * ((1.0f - fx) * fy) + d * (fx * fy);
}
// point SampleLevel at normalised uv, clamp addressing
template <class V>
__device__ __forceinline__ auto sample_point_clamp(const V& t, float u, float v) -> decltype(t.ld(0, 0))
{
    return loadc(t, (int)floorf(u * float(t.w)), (int)floorf(v * float(t.h)));
}

// Thread -> pixel mapping of the 32x8 CTAs: one warp = one 32-pixel row segment, so every centre-pixel access of a warp is a
// single fully-coalesced request (128 B for float planes, 512 B for float4 planes).
// Measured alternative: giving each warp an 8x4 pixel tile improves gather locality slightly but splits every centre access of a
// scalar plane into four 32-B sectors on four lines; the chain got slower, so the row mapping stays.
struct PixelXY
{
    int x, y;
};
DFX_HD PixelXY cta_pixel(int row0)
{
    return PixelXY{int(blockIdx.x) * 32 + int(threadIdx.x), row0 + int(blockIdx.y) * 8 + int(threadIdx.y)};
}

// streaming stores for write-once outputs (do not pollute L1)
DFX_HD void st_cs(float* p, float v) { __stcs(p, v); }
DFX_HD void st_cs(float2* p, float2 v) { __stcs(p, v); }
DFX_HD void st_cs(float4* p, float4 v) { __stcs(p, v); }

constexpr float kPi     = 3.14159265358979f;
constexpr float kHalfPi = 1.57079632679490f;
constexpr float kFltEps = 5.960464478e-8f;
constexpr float kFltMax = 3.402823466e+38f;

// a / b correctly rounded, without the slow-path call of div.rn.f32 (the call makes its caller spill). The quotient is formed in
// double from a reciprocal estimate, two Newton steps and one Markstein correction, which gives the correctly rounded double
// quotient; rounding that to float is the correctly rounded float quotient (53 >= 2 * 24 + 2 bits). Zero, infinite and NaN
// operands go through a * (1 / b) with the exact reciprocal of 0 / inf, which gives IEEE's results for them.
DFX_HD float div_(float a, float b)
{
    const double ad = a, bd = b;
    double       y;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(bd));
    if (!(fabsf(a) <= kFltMax) || !(fabsf(b) <= kFltMax) || b == 0.0f) return float(ad * y);
    y              = fma(y, fma(-bd, y, 1.0), y);
    y              = fma(y, fma(-bd, y, 1.0), y);
    const double q = ad * y;
    return float(fma(fma(-bd, q, ad), y, q));
}

// SSAO_Common.fxh:16-23 / SSR_Common.fxh:48-55. `rev` = the depth plane carries DFX_PLANE_FLAG_REVERSED_DEPTH (the reference
// compiles *_OPTION_INVERTED_DEPTH shader variants; here it is a uniform kernel argument: one predicated compare).
DFX_HD bool is_background(float d, int rev) { return rev ? d < 1e-6f : d >= (1.0f - 1e-6f); }
inline int  reversed_depth(const dfx_plane* depth) { return depth && (depth->flags & DFX_PLANE_FLAG_REVERSED_DEPTH) ? 1 : 0; }

} // namespace dfx
