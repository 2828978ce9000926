// dfx_ibl.cu — IBL cube-map precomputation (PBR/src/PBR_Renderer.cpp:729-970 PrecomputeCubemaps) as sm_90a kernels: the irradiance cube
// (Shaders/PBR/private/ComputeIrradianceMap.psh) and the prefiltered environment map (PrefilterEnvMap.psh), both drawn through
// CubemapFace.vsh and sampling the source with dfx_env_sample.cuh, E's sampler.
//
// Each sample is the shader's arithmetic with one rounding per operation (mul_ / add_ / div_ / sqrt_, never contracted) and
// every transcendental evaluated in double and rounded once, as the oracle does: only the order in which a texel's samples are summed
// differs from the shader's, within the bound of DESIGN.md §2.
//
// Launch shape. One warp per output texel, eight texels per CTA, all of one face level. The reference's one thread per texel would run
// 8192 dependent iterations on 24576 threads at the irradiance size (under a tenth of an H100), and the prefilter's coarse levels
// have 6 to 96 texels. Lane k sums the samples k, k + 32, ... in order; a shuffle tree adds the 32 partial sums. What depends only
// on the sample index (the Hammersley point, the tangent-space direction, the cosine pdf and, for a cube source, the irradiance
// sample's LOD) is computed once per CTA into shared memory, 256 samples at a time. Every level of the prefiltered chain is one
// launch: a CTA finds its level from the per-level CTA offsets.
#include "dfx_common.cuh"
#include "dfx_env_sample.cuh"
#include "dfx_ibl_math.cuh"

namespace dfx
{
namespace
{
using namespace envs;
using namespace iblm;

constexpr int kWarps = 8, kThreads = 32 * kWarps, kChunk = kThreads; // samples staged per CTA and round

// CubemapFace.vsh's g_Rotation for each face (PBR_Renderer.cpp:913-922), rows r0..r2 (r3 = (0, 0, 0, 1)), as DiligentCore's float
// RotationX / RotationY of -pi/2, +pi/2, -pi with sin / cos evaluated in float (DESIGN.md §2): kC90 = cos(-pi/2), kS180 = sin(-pi)
constexpr float kC90 = -4.37113883e-08f, kS180 = 8.74227766e-08f;
__constant__ float kFaceRot[6][3][4] = {
    {{kC90, 0.0f, 1.0f, 0.0f}, {0.0f, 1.0f, 0.0f, 0.0f}, {-1.0f, 0.0f, kC90, 0.0f}},      // +X RotationY(-pi/2)
    {{kC90, 0.0f, -1.0f, 0.0f}, {0.0f, 1.0f, 0.0f, 0.0f}, {1.0f, 0.0f, kC90, 0.0f}},      // -X RotationY(+pi/2)
    {{1.0f, 0.0f, 0.0f, 0.0f}, {0.0f, kC90, 1.0f, 0.0f}, {0.0f, -1.0f, kC90, 0.0f}},      // +Y RotationX(+pi/2)
    {{1.0f, 0.0f, 0.0f, 0.0f}, {0.0f, kC90, -1.0f, 0.0f}, {0.0f, 1.0f, kC90, 0.0f}},      // -Y RotationX(-pi/2)
    {{1.0f, 0.0f, 0.0f, 0.0f}, {0.0f, 1.0f, 0.0f, 0.0f}, {0.0f, 0.0f, 1.0f, 0.0f}},       // +Z Identity
    {{-1.0f, 0.0f, -kS180, 0.0f}, {0.0f, 1.0f, 0.0f, 0.0f}, {kS180, 0.0f, -1.0f, 0.0f}}, // -Z RotationY(-pi)
};

// acos / log2 correctly rounded (the double result rounded once); cos_, sin_, sqrt_ and the vector helpers are dfx_ibl_math.cuh's
DFX_HD float acos_(float x) { return float(acos(double(x))); }
DFX_HD float log2_(float x) { return float(log2(double(x))); }

// normalize(WorldPos) of CubemapFace.vsh at the centre of texel (i, j) of face f of an s x s face: mul(g_Rotation, (x, y, 1, 1)), xyz / w
DFX_HD float3 texel_dir(int f, int i, int j, int s)
{
    const float x = sub_(div_(mul_(2.0f, add_(float(i), 0.5f)), float(s)), 1.0f), y = sub_(1.0f, div_(mul_(2.0f, add_(float(j), 0.5f)), float(s)));
    float w[3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
        w[r] = add_(add_(add_(mul_(kFaceRot[f][r][0], x), mul_(kFaceRot[f][r][1], y)), mul_(kFaceRot[f][r][2], 1.0f)), mul_(kFaceRot[f][r][3], 1.0f));
    // row 3 is (0, 0, 0, 1): w = ((0 * x + 0 * y) + 0) + 1 = 1 exactly
    return normalize3(make_float3(div_(w[0], 1.0f), div_(w[1], 1.0f), div_(w[2], 1.0f)));
}

// ComputeSphereMapPixelSolidAngle (PBR_PrecomputeCommon.fxh:43-48), the reference's dTheta = PI / Width, dPhi = 2 PI / Height
DFX_HD float sphere_pixel_solid_angle(float w, float h, float theta, float gamma)
{
    const float dtheta = div_(kPi, w), dphi = div_(mul_(2.0f, kPi), h), t = mul_(mul_(0.5f, dtheta), gamma);
    return mul_(dphi, sub_(cos_(sub_(theta, t)), cos_(add_(theta, t))));
}
// clamp(0.5 * log2(OmegaS / max(OmegaP, 1e-10)) + MipBias, 0, g_EnvMipCount - 1), MipBias = 1
DFX_HD float sample_lod(float omega_s, float omega_p, float max_lod)
{
    return fminf(fmaxf(add_(mul_(0.5f, log2_(div_(omega_s, fmaxf(omega_p, 1e-10f)))), 1.0f), 0.0f), max_lod);
}

struct Out
{
    char* p[DFX_MAX_ENV_LEVELS];
    int   pitch[DFX_MAX_ENV_LEVELS], s[DFX_MAX_ENV_LEVELS];
    int   cta0[DFX_MAX_ENV_LEVELS + 1]; // first CTA of each level; cta0[levels] = the grid
    float roughness[DFX_MAX_ENV_LEVELS];
    int   levels;
};

struct IblArgs
{
    uint32_t n;          // g_NumSamples
    float    env_w, env_h, max_lod, omega_p_cube; // g_EnvMapWidth / Height, g_EnvMipCount - 1, ComputeCubeMapPixelSolidAngle
};

template <bool O16>
DFX_HD void store(const Out& O, int m, int x, int y, float4 c)
{
    char* row = O.p[m] + size_t(y) * size_t(O.pitch[m]);
    if constexpr (O16)
    {
        const __half2 a = __floats2half2_rn(c.x, c.y), b = __floats2half2_rn(c.z, c.w);
        uint2         u;
        u.x = *reinterpret_cast<const uint32_t*>(&a), u.y = *reinterpret_cast<const uint32_t*>(&b);
        reinterpret_cast<uint2*>(row)[x] = u;
    }
    else
        reinterpret_cast<float4*>(row)[x] = c;
}

DFX_HD float warp_sum(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = add_(v, __shfl_down_sync(0xffffffffu, v, o));
    return v;
}

// The texel of this warp: level m, face f, (i, j); false past the level's last texel
DFX_HD bool warp_texel(const Out& O, int& m, int& f, int& i, int& j)
{
    m = 0;
    while (m + 1 < O.levels && int(blockIdx.x) >= O.cta0[m + 1]) ++m;
    const int s = O.s[m], t = (int(blockIdx.x) - O.cta0[m]) * kWarps + int(threadIdx.x >> 5);
    if (t >= 6 * s * s) return false;
    f = t / (s * s), j = (t % (s * s)) / s, i = t % s;
    return true;
}

// ComputeIrradianceMap.psh IrradianceMap(N), alpha 1
template <int TYPE, bool T16, bool O16, bool OPT>
__global__ void __launch_bounds__(kThreads, 2) irradiance_kernel(const __grid_constant__ EnvMapLevels M, const __grid_constant__ Out O, IblArgs A)
{
    __shared__ float sx[kChunk], sy[kChunk], sz[kChunk], sw[kChunk]; // tangent-space L and pdf; sw = LOD for a cube source
    int        m, f, i, j;
    const bool live = warp_texel(O, m, f, i, j);
    const int  lane = threadIdx.x & 31;
    float3     N = make_float3(0.0f, 0.0f, 1.0f), T = N, B = N;
    if (live)
    {
        N = texel_dir(f, i, j, O.s[m]);
        // BasisFromNormal (ShaderUtilities.fxh:104-110)
        T = normalize3(cross3(N, fabsf(N.y) > 0.5f ? make_float3(1.0f, 0.0f, 0.0f) : make_float3(0.0f, 1.0f, 0.0f)));
        B = cross3(T, N);
    }
    float3 acc = make_float3(0.0f, 0.0f, 0.0f);
    for (uint64_t c0 = 0; c0 < A.n; c0 += kChunk) // 64-bit: a count near 2^32 must not wrap the chunk index
    {
        const uint64_t k = c0 + threadIdx.x;
        if (k < A.n)
        {
            // SampleDirectionCosineHemisphere(Xi, L, pdf) (PBR_Common.fxh:26-37)
            const float2 xi  = hammersley(uint32_t(k), A.n);
            const float  phi = mul_(mul_(2.0f, kPi), xi.x), r = sqrt_(sub_(1.0f, xi.y)), z = sqrt_(xi.y);
            const float  pdf = div_(fmaxf(z, 1e-6f), kPi);
            sx[threadIdx.x] = mul_(cos_(phi), r), sy[threadIdx.x] = mul_(sin_(phi), r), sz[threadIdx.x] = z;
            float w = pdf;
            if constexpr (OPT && TYPE == DFX_ENV_MAP_TYPE_CUBE) w = sample_lod(div_(1.0f, mul_(float(A.n), pdf)), A.omega_p_cube, A.max_lod);
            sw[threadIdx.x] = w;
        }
        __syncthreads();
        if (live)
        {
            const int nk = int(min(uint64_t(A.n) - c0, uint64_t(kChunk)));
            for (int q = lane; q < nk; q += 32)
            {
                const float3 L = normalize3(combine3(T, sx[q], B, sy[q], N, sz[q]));
                float        lod = 0.0f;
                if constexpr (OPT)
                {
                    if constexpr (TYPE == DFX_ENV_MAP_TYPE_CUBE) lod = sw[q];
                    else
                        lod = sample_lod(div_(1.0f, mul_(float(A.n), sw[q])), sphere_pixel_solid_angle(A.env_w, A.env_h, acos_(L.y), 0.5f), A.max_lod);
                }
                const float4 v = sample_env<TYPE, T16>(M, L, lod);
                acc = make_float3(add_(acc.x, v.x), add_(acc.y, v.y), add_(acc.z, v.z));
            }
        }
        __syncthreads();
    }
    if (!live) return;
    acc = make_float3(warp_sum(acc.x), warp_sum(acc.y), warp_sum(acc.z));
    if (lane == 0)
    {
        const float n = float(A.n);
        store<O16>(O, m, i, f * O.s[m] + j, make_float4(div_(acc.x, n), div_(acc.y, n), div_(acc.z, n), 1.0f));
    }
}

// PrefilterEnvMap.psh PrefilterEnvMap(g_Roughness, R), alpha 0; the level's roughness is O.roughness[m]
template <int TYPE, bool T16, bool O16, bool OPT>
__global__ void __launch_bounds__(kThreads, 2) prefilter_kernel(const __grid_constant__ EnvMapLevels M, const __grid_constant__ Out O, IblArgs A)
{
    __shared__ float sx[kChunk], sy[kChunk], sz[kChunk]; // ImportanceSampleGGX's tangent-space H
    int         m, f, i, j;
    const bool  live = warp_texel(O, m, f, i, j);
    const int   lane = threadIdx.x & 31;
    const float rough = O.roughness[m], alpha = mul_(rough, rough), a2 = mul_(alpha, alpha);
    float3      N = make_float3(0.0f, 0.0f, 1.0f), TX = N, TY = N;
    if (live)
    {
        N = texel_dir(f, i, j, O.s[m]);
        const float3 up = fabsf(N.z) < 0.999f ? make_float3(0.0f, 0.0f, 1.0f) : make_float3(1.0f, 0.0f, 0.0f);
        TX              = normalize3(cross3(up, N));
        TY              = cross3(N, TX);
    }
    float4 acc = make_float4(0.0f, 0.0f, 0.0f, 0.0f); // PrefilteredColor, TotalWeight
    for (uint64_t c0 = 0; c0 < A.n; c0 += kChunk) // 64-bit: a count near 2^32 must not wrap the chunk index
    {
        const uint64_t k = c0 + threadIdx.x;
        if (k < A.n)
        {
            // ImportanceSampleGGX (PBR_PrecomputeCommon.fxh:19-36) up to the tangent-space H
            const float2 xi  = hammersley(uint32_t(k), A.n);
            const float  phi = mul_(mul_(2.0f, kPi), xi.x);
            const float  ct  = sqrt_(sat_(div_(sub_(1.0f, xi.y), add_(1.0f, mul_(sub_(a2, 1.0f), xi.y)))));
            const float  st  = sqrt_(sat_(sub_(1.0f, mul_(ct, ct))));
            sx[threadIdx.x] = mul_(st, cos_(phi)), sy[threadIdx.x] = mul_(st, sin_(phi)), sz[threadIdx.x] = ct;
        }
        __syncthreads();
        if (live)
        {
            const int nk = int(min(uint64_t(A.n) - c0, uint64_t(kChunk)));
            for (int q = lane; q < nk; q += 32)
            {
                const float3 H   = combine3(TX, sx[q], TY, sy[q], N, sz[q]);
                const float  vh  = dot3(N, H), tv = mul_(2.0f, vh); // V = N
                const float3 L   = make_float3(sub_(mul_(tv, H.x), N.x), sub_(mul_(tv, H.y), N.y), sub_(mul_(tv, H.z), N.z));
                const float  NoL = sat_(dot3(N, L)), VoH = sat_(vh);
                if (!(NoL > 0.0f && VoH > 0.0f)) continue;
                float lod = 0.0f;
                if constexpr (OPT)
                {
                    if (alpha != 0.0f)
                    {
                        // SmithGGXSampleDirectionPDF(V, N, L, AlphaRoughness) (PBR_Common.fxh:301-321) with V = N
                        const float3 Hh  = normalize3(make_float3(add_(N.x, L.x), add_(N.y, L.y), add_(N.z, L.z)));
                        const float  ndh = dot3(Hh, N), ndv = dot3(N, N), ndl = dot3(N, L);
                        float        pdf = 0.0f;
                        if (ndh > 0.0f && ndv > 0.0f && ndl > 0.0f)
                        {
                            // NormalDistribution_GGX (:181-194) and SmithGGXMasking (:149-175)
                            const float ar = fmaxf(alpha, 1e-3f), ar2 = mul_(ar, ar), nh2 = mul_(ndh, ndh);
                            const float fx = add_(mul_(nh2, ar2), sub_(1.0f, nh2));
                            const float ndf = div_(ar2, fmaxf(mul_(mul_(kPi, fx), fx), 1e-9f));
                            const float den = add_(ndv, sqrt_(add_(a2, mul_(mul_(sub_(1.0f, a2), ndv), ndv))));
                            const float g1  = div_(mul_(2.0f, fmaxf(ndv, 0.0f)), fmaxf(den, 1e-6f));
                            pdf             = div_(div_(mul_(g1, ndf), ndv), 4.0f);
                        }
                        pdf                  = fmaxf(pdf, 0.0001f);
                        const float omega_s  = div_(1.0f, mul_(float(A.n), pdf));
                        const float omega_p  = TYPE == DFX_ENV_MAP_TYPE_CUBE ? A.omega_p_cube : sphere_pixel_solid_angle(A.env_w, A.env_h, acos_(L.y), 1.0f);
                        lod                  = sample_lod(omega_s, omega_p, A.max_lod);
                    }
                }
                const float4 v = sample_env<TYPE, T16>(M, L, lod);
                acc = make_float4(add_(acc.x, mul_(v.x, NoL)), add_(acc.y, mul_(v.y, NoL)), add_(acc.z, mul_(v.z, NoL)), add_(acc.w, NoL));
            }
        }
        __syncthreads();
    }
    if (!live) return;
    acc = make_float4(warp_sum(acc.x), warp_sum(acc.y), warp_sum(acc.z), warp_sum(acc.w));
    if (lane == 0) store<O16>(O, m, i, f * O.s[m] + j, make_float4(div_(acc.x, acc.w), div_(acc.y, acc.w), div_(acc.z, acc.w), 0.0f));
}

// The source map: the type, 1..16 levels of one RGBA32F / RGBA16F format, a cube's levels s x 6s, every level half the one before
dfx_status check_source(int32_t type, const dfx_plane* levels, int32_t n, EnvMapLevels& L, bool& t16)
{
    if (type != DFX_ENV_MAP_TYPE_CUBE && type != DFX_ENV_MAP_TYPE_SPHERE) return set_error(DFX_ERR_INVALID_ARG, "unknown environment map type %d", type);
    DFX_REQUIRE(levels, "null argument");
    DFX_REQUIRE(n >= 1 && n <= DFX_MAX_ENV_LEVELS, "the environment map has %d levels (1..%d)", n, DFX_MAX_ENV_LEVELS);
    L        = EnvMapLevels{};
    L.levels = n;
    int fmt0 = 0;
    for (int i = 0; i < n; ++i)
    {
        Tex4 t;
        if (!make_tex4(&levels[i], t)) return set_error(DFX_ERR_INVALID_ARG, "bad environment map level %d (RGBA32F or RGBA16F; null, pitch or alignment)", i);
        if (i == 0) fmt0 = t.fmt;
        DFX_REQUIRE(t.fmt == fmt0, "environment map level %d has another texel format than level 0", i);
        if (type == DFX_ENV_MAP_TYPE_CUBE) DFX_REQUIRE(t.h == 6 * t.w, "cube level %d is %dx%d, not s x 6s (six s x s faces stacked)", i, t.w, t.h);
        const int w = i == 0 ? t.w : std::max(L.w[0] >> i, 1), h = i == 0 ? t.h : (type == DFX_ENV_MAP_TYPE_CUBE ? 6 * w : std::max(L.h[0] >> i, 1));
        DFX_REQUIRE(t.w == w && t.h == h, "environment map level %d is %dx%d, the mip chain needs %dx%d", i, t.w, t.h, w, h);
        L.p[i] = t.p, L.pitch[i] = t.pitch, L.w[i] = t.w, L.h[i] = t.h;
    }
    t16 = fmt0 == DFX_FORMAT_RGBA16F;
    return DFX_OK;
}

// An output cube chain: 1..16 levels s_m x 6 s_m, s_m = max(s0 >> m, 1), one RGBA16F / RGBA32F format; fills the per-level CTA offsets
dfx_status check_output(const dfx_plane* levels, int32_t n, Out& O, bool& o16)
{
    DFX_REQUIRE(levels, "null argument");
    O        = Out{};
    O.levels = n;
    int cta  = 0;
    for (int m = 0; m < n; ++m)
    {
        int is16 = 0;
        DFX_REQUIRE(writable(&levels[m], DFX_FORMAT_RGBA32F, DFX_FORMAT_RGBA16F, 16, 8, O.p[m], O.pitch[m], is16),
                    "bad output level %d (RGBA32F or RGBA16F expected; null, pitch or alignment)", m);
        if (m == 0) o16 = is16;
        DFX_REQUIRE(bool(is16) == o16, "output level %d has another texel format than level 0", m);
        const int s = m == 0 ? levels[0].width : std::max(levels[0].width >> m, 1);
        DFX_REQUIRE(levels[m].width == s && levels[m].height == 6 * s, "output level %d is %dx%d, the cube chain needs %dx%d", m, levels[m].width,
                    levels[m].height, s, 6 * s);
        O.s[m] = s, O.cta0[m] = cta;
        cta += div_up(6 * s * s, kWarps);
    }
    O.cta0[n] = cta;
    return DFX_OK;
}

IblArgs make_args(int32_t type, const EnvMapLevels& L, uint32_t n)
{
    IblArgs A;
    A.n     = n;
    A.env_w = float(L.w[0]);
    A.env_h = float(type == DFX_ENV_MAP_TYPE_CUBE ? L.w[0] : L.h[0]); // a cube texture's Desc.Height is the face size
    A.max_lod = float(L.levels) - 1.0f;
    // ComputeCubeMapPixelSolidAngle (PBR_PrecomputeCommon.fxh:38-41): 4 PI / (6 * Width * Height)
    A.omega_p_cube = (4.0f * kPi) / (6.0f * A.env_w * A.env_h);
    return A;
}

template <bool IRR>
dfx_status launch(void* stream, int32_t type, const EnvMapLevels& L, bool t16, const Out& O, bool o16, const IblArgs& A, bool opt)
{
    const dim3   grid(unsigned(O.cta0[O.levels])), block(kThreads);
    cudaStream_t s = as_stream(stream);
#define IBL_LAUNCH(TY)                                                                                                        \
    DFX_FMT16(t16, H, DFX_FMT16(o16, H2, {                                                                                    \
        if (opt)                                                                                                              \
        {                                                                                                                     \
            if constexpr (IRR) irradiance_kernel<TY, H, H2, true><<<grid, block, 0, s>>>(L, O, A);                            \
            else prefilter_kernel<TY, H, H2, true><<<grid, block, 0, s>>>(L, O, A);                                           \
        }                                                                                                                     \
        else                                                                                                                  \
        {                                                                                                                     \
            if constexpr (IRR) irradiance_kernel<TY, H, H2, false><<<grid, block, 0, s>>>(L, O, A);                           \
            else prefilter_kernel<TY, H, H2, false><<<grid, block, 0, s>>>(L, O, A);                                          \
        }                                                                                                                     \
    }))
    if (type == DFX_ENV_MAP_TYPE_CUBE)
        IBL_LAUNCH(DFX_ENV_MAP_TYPE_CUBE);
    else
        IBL_LAUNCH(DFX_ENV_MAP_TYPE_SPHERE);
#undef IBL_LAUNCH
    return DFX_OK;
}
} // namespace
} // namespace dfx

using namespace dfx;

extern "C" dfx_status dfx_pass_irradiance_cube(void* stream, int32_t env_type, const dfx_plane* env_levels, int32_t n_env, uint32_t num_samples,
                                               int32_t optimize_samples, const dfx_plane* out)
{
    DFX_PROFILE(stream, "irradiance_cube");
    EnvMapLevels L;
    bool         t16 = false, o16 = false;
    dfx_status   st = check_source(env_type, env_levels, n_env, L, t16);
    if (st != DFX_OK) return st;
    Out O;
    if ((st = check_output(out, 1, O, o16)) != DFX_OK) return st;
    O.roughness[0] = 0.0f;
    const IblArgs A = make_args(env_type, L, num_samples ? num_samples : 8192u);
    launch<true>(stream, env_type, L, t16, O, o16, A, optimize_samples != 0);
    DFX_LAUNCHED("irradiance_kernel");
    return DFX_OK;
}

extern "C" dfx_status dfx_pass_prefilter_env_map(void* stream, int32_t env_type, const dfx_plane* env_levels, int32_t n_env, uint32_t num_samples,
                                                 int32_t optimize_samples, const dfx_plane* out_levels, int32_t n_out)
{
    DFX_PROFILE(stream, "prefilter_env_map");
    EnvMapLevels L;
    bool         t16 = false, o16 = false;
    dfx_status   st = check_source(env_type, env_levels, n_env, L, t16);
    if (st != DFX_OK) return st;
    DFX_REQUIRE(n_out >= 2 && n_out <= DFX_MAX_ENV_LEVELS, "the prefiltered map has %d levels (2..%d: level m is at roughness m / (levels - 1))", n_out,
                DFX_MAX_ENV_LEVELS);
    Out O;
    if ((st = check_output(out_levels, n_out, O, o16)) != DFX_OK) return st;
    for (int m = 0; m < n_out; ++m) O.roughness[m] = static_cast<float>(m) / static_cast<float>(n_out - 1); // PBR_Renderer.cpp:951
    const IblArgs A = make_args(env_type, L, num_samples ? num_samples : 256u);
    launch<false>(stream, env_type, L, t16, O, o16, A, optimize_samples != 0);
    DFX_LAUNCHED("prefilter_kernel");
    return DFX_OK;
}
