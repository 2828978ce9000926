// dfx_env_map.cu — E, the environment-map background, as an sm_90a kernel: the pipeline state of EnvMapRenderer::GetPSO
// (Components/src/EnvMapRenderer.cpp:102-190: a full-screen triangle at the far plane, depth test LESS_EQUAL / GREATER_EQUAL, no depth
// writes) around SampleEnvMap (Shaders/Common/private/EnvMap.psh:45-73), one thread per pixel.
//
// Every operation of the shader is one rounding (mul_ / add_ / div_ / __fsqrt_rn, never contracted), and the sampler is the
// project's software bilinear with 8 fractional bits of position (DESIGN.md §2, as every sampled pass) plus the seamless cube rule
// of DESIGN.md §2: so the cube with tone map NONE and no sRGB is the oracle's arithmetic bit for bit. atan2 / asin (sphere) and pow
// (sRGB) are evaluated in double and rounded once; the tone map is dfx_tonemap.cuh's. No texture objects: the hardware filter's
// weight precision is not documented.
#include "dfx_common.cuh"
#include "dfx_tonemap.cuh"

namespace dfx
{
namespace
{
struct EnvMapLevels
{
    const char* p[DFX_MAX_MIPS];
    int         pitch[DFX_MAX_MIPS]; // bytes
    int         w[DFX_MAX_MIPS], h[DFX_MAX_MIPS];
    int         levels;
};

// D3D / Vulkan cube face table (faces f = +X, -X, +Y, -Y, +Z, -Z; major axis f / 2): the axis and sign of sc, the axis and sign of tc
//   sc: -z, +z, +x, +x, +x, -x    tc: -y, -y, +z, -z, -y, -y
DFX_HD int kSa(int f) { return f < 2 ? 2 : 0; }
DFX_HD int kSs(int f) { return (f == 0 || f == 5) ? -1 : 1; }
DFX_HD int kTa(int f) { return (f == 2 || f == 3) ? 2 : 1; }
DFX_HD int kTs(int f) { return f == 2 ? 1 : -1; }

DFX_HD float  comp(float3 v, int a) { return a == 0 ? v.x : a == 1 ? v.y : v.z; }
DFX_HD float4 add4(float4 a, float4 b) { return make_float4(add_(a.x, b.x), add_(a.y, b.y), add_(a.z, b.z), add_(a.w, b.w)); }
DFX_HD float4 mul4(float4 a, float w) { return make_float4(mul_(a.x, w), mul_(a.y, w), mul_(a.z, w), mul_(a.w, w)); }

template <bool T16>
DFX_HD float4 texel(const EnvMapLevels& M, int m, int x, int y)
{
    TexRGBA<T16> t;
    t.p = M.p[m], t.pitch = M.pitch[m], t.w = M.w[m], t.h = M.h[m];
    return t.ld(x, y);
}

// Bilinear position on a level of `n` texels: px = u * n - 0.5 snapped to 1/256 texel; the first tap clamped to [-1, n - 1] (a NaN
// coordinate gives -1: fmaxf returns the number)
struct Axis
{
    int   i0;
    float f;
};
DFX_HD Axis axis_pos(float u, int n)
{
    float       px  = sub_(mul_(u, float(n)), 0.5f);
    px              = mul_(floorf(add_(mul_(px, 256.0f), 0.5f)), 1.0f / 256.0f);
    const float fx0 = floorf(px);
    return Axis{int(fminf(fmaxf(fx0, -1.0f), float(n - 1))), sub_(px, fx0)};
}
DFX_HD float4 bilerp(float4 t00, float4 t10, float4 t01, float4 t11, float fx, float fy)
{
    const float gx = sub_(1.0f, fx), gy = sub_(1.0f, fy);
    return add4(add4(add4(mul4(t00, mul_(gx, gy)), mul4(t10, mul_(fx, gy))), mul4(t01, mul_(gx, fy))), mul4(t11, mul_(fx, fy)));
}

// the texel (i, j) of face f's s x s grid, i or j one texel outside the face: the adjacent face's edge texel across that edge
// (integer restatement of re-projecting the texel centre's direction; DESIGN.md §2)
DFX_HD void cube_adjacent(int& f, int& i, int& j, int s)
{
    // the texel centre's direction in half-texel units: +-s on the major axis, 2i + 1 - s and 2j + 1 - s along sc and tc
    const int  a = f >> 1, sa = kSa(f), va = (f & 1) ? -s : s, vs = kSs(f) * (2 * i + 1 - s), vt = kTs(f) * (2 * j + 1 - s);
    const auto V = [&](int axis) { return axis == a ? va : axis == sa ? vs : vt; };
    const int  k = (i < 0 || i >= s) ? sa : kTa(f); // the axis it leaves the face on becomes the major axis
    f            = 2 * k + (V(k) < 0 ? 1 : 0);
    const int cs = kSs(f) * V(kSa(f)), ct = kTs(f) * V(kTa(f));
    i = cs >= s ? s - 1 : cs <= -s ? 0 : (cs + s - 1) / 2;
    j = ct >= s ? s - 1 : ct <= -s ? 0 : (ct + s - 1) / 2;
}
template <bool T16>
DFX_HD float4 cube_tap(const EnvMapLevels& M, int m, int f, int i, int j)
{
    const int  s  = M.w[m];
    const bool ox = i < 0 || i >= s, oy = j < 0 || j >= s;
    if (!ox && !oy) return texel<T16>(M, m, i, f * s + j);
    if (ox != oy)
    {
        cube_adjacent(f, i, j, s);
        return texel<T16>(M, m, i, f * s + j);
    }
    // a corner: the three texels that meet there, (this + across x + across y) / 3
    const int ci = min(max(i, 0), s - 1), cj = min(max(j, 0), s - 1);
    int       fa = f, ia = i, ja = cj, fb = f, ib = ci, jb = j;
    cube_adjacent(fa, ia, ja, s);
    cube_adjacent(fb, ib, jb, s);
    const float4 t = add4(add4(texel<T16>(M, m, ci, f * s + cj), texel<T16>(M, m, ia, fa * s + ja)), texel<T16>(M, m, ib, fb * s + jb));
    return make_float4(div_(t.x, 3.0f), div_(t.y, 3.0f), div_(t.z, 3.0f), div_(t.w, 3.0f));
}

template <int TYPE, bool T16>
DFX_HD float4 sample_level(const EnvMapLevels& M, int m, int face, float u, float v)
{
    if constexpr (TYPE == DFX_ENV_MAP_TYPE_CUBE)
    {
        const int  s = M.w[m];
        const Axis a = axis_pos(u, s), b = axis_pos(v, s);
        return bilerp(cube_tap<T16>(M, m, face, a.i0, b.i0), cube_tap<T16>(M, m, face, a.i0 + 1, b.i0), cube_tap<T16>(M, m, face, a.i0, b.i0 + 1),
                      cube_tap<T16>(M, m, face, a.i0 + 1, b.i0 + 1), a.f, b.f);
    }
    else
    {
        const int  w = M.w[m], h = M.h[m];
        const Axis a = axis_pos(u, w), b = axis_pos(v, h);
        const int  x0 = max(a.i0, 0), x1 = min(a.i0 + 1, w - 1), y0 = max(b.i0, 0), y1 = min(b.i0 + 1, h - 1);
        return bilerp(texel<T16>(M, m, x0, y0), texel<T16>(M, m, x1, y0), texel<T16>(M, m, x0, y1), texel<T16>(M, m, x1, y1), a.f, b.f);
    }
}

// Sam_LinearClamp's SampleLevel: trilinear between the two levels around the LOD clamped to [0, levels - 1]
template <int TYPE, bool T16>
DFX_HD float4 sample_env(const EnvMapLevels& M, float3 R, float lod)
{
    int   face = 0;
    float u, v;
    if constexpr (TYPE == DFX_ENV_MAP_TYPE_CUBE)
    {
        const float ax = fabsf(R.x), ay = fabsf(R.y), az = fabsf(R.z);
        const int   a  = (az >= ax && az >= ay) ? 2 : ay >= ax ? 1 : 0;
        const float ma = comp(R, a);
        face           = 2 * a + (ma < 0.0f ? 1 : 0);
        const float am = fabsf(ma);
        u = mul_(0.5f, add_(div_(kSs(face) < 0 ? -comp(R, kSa(face)) : comp(R, kSa(face)), am), 1.0f));
        v = mul_(0.5f, add_(div_(kTs(face) < 0 ? -comp(R, kTa(face)) : comp(R, kTa(face)), am), 1.0f));
    }
    else
    {
        // TransformDirectionToSphereMapUV (ShaderUtilities.fxh:98-102)
        const float kOneOverPi = 0.3183098862f;
        u = add_(mul_(kOneOverPi, mul_(0.5f, float(atan2(double(R.z), double(R.x))))), 0.5f);
        v = add_(mul_(kOneOverPi, float(asin(double(R.y)))), 0.5f);
    }
    if (M.levels == 1) return sample_level<TYPE, T16>(M, 0, face, u, v);
    const float l  = fminf(fmaxf(lod, 0.0f), float(M.levels - 1));
    const int   m0 = int(floorf(l)), m1 = min(m0 + 1, M.levels - 1);
    const float f  = sub_(l, float(m0));
    return add4(mul4(sample_level<TYPE, T16>(M, m0, face, u, v), sub_(1.0f, f)), mul4(sample_level<TYPE, T16>(M, m1, face, u, v), f));
}

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
