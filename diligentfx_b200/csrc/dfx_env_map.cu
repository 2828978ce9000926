// dfx_env_map.cu — E, the environment-map background, as an sm_90a kernel: the pipeline state of EnvMapRenderer::GetPSO
// (Components/src/EnvMapRenderer.cpp:102-190: a full-screen triangle at the far plane, depth test LESS_EQUAL / GREATER_EQUAL, no depth
// writes) around SampleEnvMap (Shaders/Common/private/EnvMap.psh:45-73), one thread per pixel.
//
// Every operation of the shader is one rounding (mul_ / add_ / div_ / __fsqrt_rn, never contracted), and the sampler is
// dfx_env_sample.cuh's (the project's software bilinear and the seamless cube rule of DESIGN.md §2): so the cube with tone map NONE
// and no sRGB is the oracle's arithmetic bit for bit. pow (sRGB) is evaluated in double and rounded once; the tone map is
// dfx_tonemap.cuh's.
#include "dfx_common.cuh"
#include "dfx_env_sample.cuh"
#include "dfx_tonemap.cuh"

namespace dfx
{
namespace
{
using namespace envs;

// float4(v) * M, the shader's mul(v, M): ((r0 * x + r1 * y) + r2 * z) + r3 * w per column
DFX_HD float4 mul_row(float4 v, const dfx_float4x4& M)
{
    float r[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) r[c] = add_(add_(add_(mul_(M.m[0][c], v.x), mul_(M.m[1][c], v.y)), mul_(M.m[2][c], v.z)), mul_(M.m[3][c], v.w));
    return make_float4(r[0], r[1], r[2], r[3]);
}

template <int TYPE, int MODE, bool T16>
__global__ void __launch_bounds__(256) env_map_kernel(const dfx_camera_attribs* __restrict__ cams, const __grid_constant__ EnvMapLevels M,
                                                      const __grid_constant__ dfx_env_map_attribs A, uint32_t options, View<const float> depth,
                                                      char* color, int color_pitch, int color16, char* motion, int motion_pitch, int motion16, int y0,
                                                      int y1)
{
    const PixelXY q = cta_pixel(y0);
    if (q.x >= depth.w || q.y >= y1) return;
    const dfx_camera_attribs& C  = cams[0];
    const float               zf = C.fFarPlaneDepth; // DepthToNormalizedDeviceZ(fFarPlaneDepth), EnvMap.vsh:20
    const float               d  = depth.ld(q.x, q.y);
    if (!((options & DFX_ENV_MAP_OPTION_USE_REVERSE_DEPTH) ? zf >= d : zf <= d)) return; // the depth test of GetPSO (:175)
    char* const crow = color + size_t(q.y) * size_t(color_pitch) + size_t(q.x) * (color16 ? 8u : 16u);
    char* const mrow = motion + size_t(q.y) * size_t(motion_pitch) + size_t(q.x) * (motion16 ? 4u : 8u);

    // the interpolated CLIP_POS at the pixel centre (DESIGN.md §2)
    const float4 clip = make_float4(sub_(div_(mul_(2.0f, add_(float(q.x), 0.5f)), float(depth.w)), 1.0f),
                                    sub_(1.0f, div_(mul_(2.0f, add_(float(q.y), 0.5f)), float(depth.h))), zf, 1.0f);
    const float4 wp  = mul_row(clip, C.mViewProjInv);
    const float3 dir = make_float3(sub_(div_(wp.x, wp.w), C.f4Position[0]), sub_(div_(wp.y, wp.w), C.f4Position[1]),
                                   sub_(div_(wp.z, wp.w), C.f4Position[2]));
    const float  len = __fsqrt_rn(add_(add_(mul_(dir.x, dir.x), mul_(dir.y, dir.y)), mul_(dir.z, dir.z)));
    const float3 R   = make_float3(div_(dir.x, len), div_(dir.y, len), div_(dir.z, len));
    const float4 s   = sample_env<TYPE, T16>(M, R, A.MipLevel);
    float3       c   = make_float3(mul_(s.x, A.Scale[0]), mul_(s.y, A.Scale[1]), mul_(s.z, A.Scale[2]));
    if constexpr (MODE > DFX_TONE_MAPPING_MODE_NONE) c = tone_map<MODE>(c, A.ToneMapping, A.AverageLogLum);
    if (options & DFX_ENV_MAP_OPTION_CONVERT_OUTPUT_TO_SRGB)
    {
        // pow(c, 1 / 2.2) with the shader's fp32 exponent, as exp2(e * log2(c)) in double rounded once (the same special values as
        // pow for c >= +-0, inf and NaN; a negative c gives NaN); inlined, where double pow() is a call that makes the caller spill
        const double e  = double(div_(1.0f, 2.2f));
        const auto   pw = [e](float v) { return float(exp2(e * log2(double(v)))); };
        c               = make_float3(pw(c.x), pw(c.y), pw(c.z));
    }
    if (color16)
    {
        const __half2 a = __floats2half2_rn(c.x, c.y), b = __floats2half2_rn(c.z, A.Alpha);
        uint2         u;
        u.x = *reinterpret_cast<const uint32_t*>(&a), u.y = *reinterpret_cast<const uint32_t*>(&b);
        *reinterpret_cast<uint2*>(crow) = u;
    }
    else
        *reinterpret_cast<float4*>(crow) = make_float4(c.x, c.y, c.z, A.Alpha);

    if (options & DFX_ENV_MAP_OPTION_COMPUTE_MOTION_VECTORS)
    {
        const dfx_camera_attribs& P  = cams[1];
        const float4              pc = mul_row(make_float4(add_(P.f4Position[0], dir.x), add_(P.f4Position[1], dir.y), add_(P.f4Position[2], dir.z), 1.0f),
                                               P.mViewProj);
        const float px = div_(pc.x, pc.w), py = div_(pc.y, pc.w);
        // GetMotionVector (ShaderUtilities.fxh:88-91): (ClipPos - Jitter) - (PrevClipPos - PrevJitter)
        const float mx = sub_(sub_(clip.x, C.f2Jitter[0]), sub_(px, P.f2Jitter[0]));
        const float my = sub_(sub_(clip.y, C.f2Jitter[1]), sub_(py, P.f2Jitter[1]));
        if (motion16)
        {
            const __half2 h = __floats2half2_rn(mx, my);
            *reinterpret_cast<uint32_t*>(mrow) = *reinterpret_cast<const uint32_t*>(&h);
        }
        else
            *reinterpret_cast<float2*>(mrow) = make_float2(mx, my);
    }
}

// The checks dfx_pass_env_map and dfx_chain_set_environment_map share: the type, the options, the tone-mapping mode and the map
// (a cube's levels s x 6s, every level half the one before, one texel format). Fills `M` and `t16`.
dfx_status check_env_map(int32_t type, const dfx_pyramid* env_map, uint32_t options, const dfx_env_map_attribs* attribs, EnvMapLevels* M, bool* t16)
{
    DFX_REQUIRE(env_map && attribs, "null argument");
    if (type != DFX_ENV_MAP_TYPE_CUBE && type != DFX_ENV_MAP_TYPE_SPHERE) return set_error(DFX_ERR_INVALID_ARG, "unknown environment map type %d", type);
    if (options & ~DFX_ENV_MAP_OPTION_ALL) return set_error(DFX_ERR_UNSUPPORTED, "unknown environment map options 0x%x", options);
    const int mode = attribs->ToneMapping.iToneMappingMode;
    if (mode < DFX_TONE_MAPPING_MODE_NONE || mode > DFX_TONE_MAPPING_MODE_COMMERCE) return set_error(DFX_ERR_INVALID_ARG, "unknown tone mapping mode %d", mode);
    DFX_REQUIRE(env_map->levels >= 1 && env_map->levels <= DFX_MAX_MIPS, "the environment map has %d levels (1..%d)", env_map->levels, DFX_MAX_MIPS);
    EnvMapLevels L{};
    L.levels = env_map->levels;
    int fmt0 = 0;
    for (int i = 0; i < env_map->levels; ++i)
    {
        Tex4 t;
        if (!make_tex4(&env_map->level[i], t)) return set_error(DFX_ERR_INVALID_ARG, "bad environment map level %d (RGBA32F or RGBA16F; null, pitch or alignment)", i);
        if (i == 0) fmt0 = t.fmt;
        DFX_REQUIRE(t.fmt == fmt0, "environment map level %d has another texel format than level 0", i);
        if (type == DFX_ENV_MAP_TYPE_CUBE) DFX_REQUIRE(t.h == 6 * t.w, "cube level %d is %dx%d, not s x 6s (six s x s faces stacked)", i, t.w, t.h);
        const int w = i == 0 ? t.w : std::max(L.w[0] >> i, 1), h = i == 0 ? t.h : (type == DFX_ENV_MAP_TYPE_CUBE ? 6 * w : std::max(L.h[0] >> i, 1));
        DFX_REQUIRE(t.w == w && t.h == h, "environment map level %d is %dx%d, the mip chain needs %dx%d", i, t.w, t.h, w, h);
        L.p[i] = t.p, L.pitch[i] = t.pitch, L.w[i] = t.w, L.h[i] = t.h;
    }
    if (M) *M = L;
    if (t16) *t16 = fmt0 == DFX_FORMAT_RGBA16F;
    return DFX_OK;
}
} // namespace

dfx_status env_map_check(int32_t type, const dfx_pyramid* env_map, uint32_t options, const dfx_env_map_attribs* attribs)
{
    return check_env_map(type, env_map, options, attribs, nullptr, nullptr);
}

} // namespace dfx

using namespace dfx;

extern "C" void dfx_env_map_attribs_default(dfx_env_map_attribs* a)
{
    // EnvMapRenderer.hpp RenderAttribs: AverageLogLum 1, MipLevel 0, Alpha 1, Scale (1, 1, 1) -> float4(Scale, 1) (EnvMapRenderer.cpp:241)
    if (!a) return;
    *a = dfx_env_map_attribs{};
    dfx_tonemap_attribs_default(&a->ToneMapping);
    a->AverageLogLum = 1.0f, a->MipLevel = 0.0f, a->Alpha = 1.0f;
    a->Scale[0] = a->Scale[1] = a->Scale[2] = a->Scale[3] = 1.0f;
}

extern "C" dfx_status dfx_pass_env_map(void* stream, const dfx_camera_attribs* cameras_dev, int32_t type, const dfx_pyramid* env_map, uint32_t options,
                                       const dfx_env_map_attribs* attribs, const dfx_plane* depth_, const dfx_plane* color_inout,
                                       const dfx_plane* motion_inout, dfx_rows rows)
{
    DFX_PROFILE(stream, "env_map");
    DFX_REQUIRE(cameras_dev, "null argument");
    EnvMapLevels M;
    bool         t16 = false;
    dfx_status   st  = check_env_map(type, env_map, options, attribs, &M, &t16);
    if (st != DFX_OK) return st;
    DFX_VIEW(const float, depth, depth_, DFX_FORMAT_R32F);
    char* color = nullptr;
    char* motion = nullptr;
    int   cpitch = 0, c16 = 0, mpitch = 0, m16 = 0;
    DFX_REQUIRE(writable(color_inout, DFX_FORMAT_RGBA32F, DFX_FORMAT_RGBA16F, 16, 8, color, cpitch, c16),
                "bad plane 'color_inout' (RGBA32F or RGBA16F expected; null, pitch or alignment)");
    DFX_REQUIRE(color_inout->width == depth.w && color_inout->height == depth.h, "plane size mismatch: depth vs color_inout");
    if (options & DFX_ENV_MAP_OPTION_COMPUTE_MOTION_VECTORS)
    {
        DFX_REQUIRE(motion_inout, "motion vectors are on: the motion plane must be given");
        DFX_REQUIRE(writable(motion_inout, DFX_FORMAT_RG32F, DFX_FORMAT_RG16F, 8, 4, motion, mpitch, m16),
                    "bad plane 'motion_inout' (RG32F or RG16F expected; null, pitch or alignment)");
        DFX_REQUIRE(motion_inout->width == depth.w && motion_inout->height == depth.h, "plane size mismatch: depth vs motion_inout");
    }
    DFX_REQUIRE(rows_ok(rows, depth.h), "bad row range");
    if (rows.y1 == rows.y0) return DFX_OK;
    const dim3   grid(div_up(depth.w, 32), div_up(rows.y1 - rows.y0, 8));
    const dim3   block(32, 8);
    cudaStream_t s = as_stream(stream);
#define E_LAUNCH(T, M_)                                                                                                                                  \
    DFX_FMT16(t16, H, env_map_kernel<T, M_, H><<<grid, block, 0, s>>>(cameras_dev, M, *attribs, options, depth, color, cpitch, c16, motion, mpitch, m16, \
                                                                      rows.y0, rows.y1))
#define E_MODES(T)                                                                                 \
    switch (attribs->ToneMapping.iToneMappingMode)                                                 \
    {                                                                                              \
        case DFX_TONE_MAPPING_MODE_NONE: E_LAUNCH(T, DFX_TONE_MAPPING_MODE_NONE); break;           \
        case DFX_TONE_MAPPING_MODE_EXP: E_LAUNCH(T, DFX_TONE_MAPPING_MODE_EXP); break;             \
        case DFX_TONE_MAPPING_MODE_REINHARD: E_LAUNCH(T, DFX_TONE_MAPPING_MODE_REINHARD); break;   \
        case DFX_TONE_MAPPING_MODE_REINHARD_MOD: E_LAUNCH(T, DFX_TONE_MAPPING_MODE_REINHARD_MOD); break; \
        case DFX_TONE_MAPPING_MODE_UNCHARTED2: E_LAUNCH(T, DFX_TONE_MAPPING_MODE_UNCHARTED2); break; \
        case DFX_TONE_MAPPING_MODE_FILMIC_ALU: E_LAUNCH(T, DFX_TONE_MAPPING_MODE_FILMIC_ALU); break; \
        case DFX_TONE_MAPPING_MODE_LOGARITHMIC: E_LAUNCH(T, DFX_TONE_MAPPING_MODE_LOGARITHMIC); break; \
        case DFX_TONE_MAPPING_MODE_ADAPTIVE_LOG: E_LAUNCH(T, DFX_TONE_MAPPING_MODE_ADAPTIVE_LOG); break; \
        case DFX_TONE_MAPPING_MODE_AGX: E_LAUNCH(T, DFX_TONE_MAPPING_MODE_AGX); break;             \
        case DFX_TONE_MAPPING_MODE_AGX_CUSTOM: E_LAUNCH(T, DFX_TONE_MAPPING_MODE_AGX_CUSTOM); break; \
        case DFX_TONE_MAPPING_MODE_PBR_NEUTRAL: E_LAUNCH(T, DFX_TONE_MAPPING_MODE_PBR_NEUTRAL); break; \
        default: E_LAUNCH(T, DFX_TONE_MAPPING_MODE_COMMERCE); break;                               \
    }
    if (type == DFX_ENV_MAP_TYPE_CUBE)
        E_MODES(DFX_ENV_MAP_TYPE_CUBE)
    else
        E_MODES(DFX_ENV_MAP_TYPE_SPHERE)
#undef E_MODES
#undef E_LAUNCH
    DFX_LAUNCHED("env_map_kernel");
    return DFX_OK;
}
