// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_math.h). Pinned against the reference's own CubemapFace.vsh, ComputeIrradianceMap.psh and
// PrefilterEnvMap.psh (oracle/refshader/build_ibl_ref.py, tests/test_ibl_reference.py), and held to properties that do not depend on
// them (tests/test_ibl_cpu.py). Built on its own into oracle/_build/liboracle_ibl.so by oracle/oracle_ibl_py.py.
//
// IBL cube-map precomputation (PBR/src/PBR_Renderer.cpp:729-970 PrecomputeCubemaps): the irradiance cube and one level of the
// prefiltered environment map, for a row range of one face, each texel's samples summed in the shader's order. The texel direction is
// CubemapFace.vsh at the pixel centre through the face matrices of DESIGN.md §2. The source is read with Sam_LinearClamp as DESIGN.md §2
// states it for E: trilinear, bilinear positions snapped to 1/256 texel, the seamless cube rule. Every transcendental (cos, sin, acos,
// log2, and atan2 / asin of the sphere lookup) is the double function rounded once to float: DESIGN.md §2's statement of the HLSL intrinsics for these passes, which
// the reference-shader build follows too (oracle/refshader/ibl_defs.inc).
#include "oracle_ibl_math.h"

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>

namespace orc
{
namespace
{
using namespace iblm; // kPi, cos_, sin_, hammersley, ImportanceSampleGGX

float acos_(float x) { return float(std::acos(double(x))); }
float log2_(float x) { return float(std::log2(double(x))); }

struct Level
{
    const float* p; // RGBA, tightly packed
    int          w, h;
    float4       at(int x, int y) const
    {
        const float* t = p + (size_t(y) * size_t(w) + size_t(x)) * 4;
        return float4(t[0], t[1], t[2], t[3]);
    }
};

// face f (+X, -X, +Y, -Y, +Z, -Z): sc = sign_s(f) * R[axis_s(f)], tc = sign_t(f) * R[axis_t(f)], ma = R[f / 2]
int   axis_s(int f) { return f < 2 ? 2 : 0; }
int   sign_s(int f) { return (f == 0 || f == 5) ? -1 : 1; }
int   axis_t(int f) { return (f == 2 || f == 3) ? 2 : 1; }
int   sign_t(int f) { return f == 2 ? 1 : -1; }
float comp(float3 v, int a) { return a == 0 ? v.x : a == 1 ? v.y : v.z; }

// (f, i, j) one texel beyond an edge of face f -> the adjacent face's edge texel (the texel centre's direction in half-texel units)
void across(int& f, int& i, int& j, int s)
{
    int v[3];
    v[f / 2]       = (f % 2) ? -s : s;
    v[axis_s(f)]   = sign_s(f) * (2 * i + 1 - s);
    v[axis_t(f)]   = sign_t(f) * (2 * j + 1 - s);
    const int k    = (i < 0 || i >= s) ? axis_s(f) : axis_t(f);
    f              = 2 * k + (v[k] < 0 ? 1 : 0);
    const auto idx = [s](int c) { return c >= s ? s - 1 : c <= -s ? 0 : (c + s - 1) / 2; };
    i              = idx(sign_s(f) * v[axis_s(f)]);
    j              = idx(sign_t(f) * v[axis_t(f)]);
}
float4 cube_texel(const Level& L, int f, int i, int j)
{
    const int  s  = L.w;
    const bool oi = i < 0 || i >= s, oj = j < 0 || j >= s;
    if (!oi && !oj) return L.at(i, f * s + j);
    if (oi != oj)
    {
        across(f, i, j, s);
        return L.at(i, f * s + j);
    }
    const int ci = clampi(i, 0, s - 1), cj = clampi(j, 0, s - 1);
    int       fa = f, ia = i, ja = cj, fb = f, ib = ci, jb = j;
    across(fa, ia, ja, s);
    across(fb, ib, jb, s);
    return (L.at(ci, f * s + cj) + L.at(ia, fa * s + ja) + L.at(ib, fb * s + jb)) / 3.0f;
}
void tap(float u, int n, int& i0, float& f)
{
    float px        = u * float(n) - 0.5f;
    px              = std::floor(px * 256.0f + 0.5f) * (1.0f / 256.0f);
    const float fx0 = std::floor(px);
    i0              = int(std::min(float(n - 1), std::max(-1.0f, fx0)));
    f               = px - fx0;
}
float4 bilinear(float4 t00, float4 t10, float4 t01, float4 t11, float fx, float fy)
{
    return t00 * ((1.0f - fx) * (1.0f - fy)) + t10 * (fx * (1.0f - fy)) + t01 * ((1.0f - fx) * fy) + t11 * (fx * fy);
}
float4 sample_level(const Level& L, bool cube, int face, float u, float v)
{
    int   x0, y0;
    float fx, fy;
    if (cube)
    {
        tap(u, L.w, x0, fx), tap(v, L.w, y0, fy);
        return bilinear(cube_texel(L, face, x0, y0), cube_texel(L, face, x0 + 1, y0), cube_texel(L, face, x0, y0 + 1), cube_texel(L, face, x0 + 1, y0 + 1), fx, fy);
    }
    tap(u, L.w, x0, fx), tap(v, L.h, y0, fy);
    const auto c = [&](int x, int y) { return L.at(clampi(x, 0, L.w - 1), clampi(y, 0, L.h - 1)); };
    return bilinear(c(x0, y0), c(x0 + 1, y0), c(x0, y0 + 1), c(x0 + 1, y0 + 1), fx, fy);
}
float3 sample_env(const std::vector<Level>& M, bool cube, float3 R, float lod)
{
    int   face = 0;
    float u, v;
    if (cube)
    {
        const float ax = std::fabs(R.x), ay = std::fabs(R.y), az = std::fabs(R.z);
        const int   a  = (az >= ax && az >= ay) ? 2 : ay >= ax ? 1 : 0;
        const float ma = comp(R, a);
        face           = 2 * a + (ma < 0.0f ? 1 : 0);
        const float sc = sign_s(face) < 0 ? -comp(R, axis_s(face)) : comp(R, axis_s(face));
        const float tc = sign_t(face) < 0 ? -comp(R, axis_t(face)) : comp(R, axis_t(face));
        u = 0.5f * (sc / std::fabs(ma) + 1.0f), v = 0.5f * (tc / std::fabs(ma) + 1.0f);
    }
    else
    {
        // TransformDirectionToSphereMapUV (ShaderUtilities.fxh:98-102)
        const float OneOverPi = 0.3183098862f;
        u = OneOverPi * (0.5f * float(std::atan2(double(R.z), double(R.x)))) + 0.5f;
        v = OneOverPi * float(std::asin(double(R.y))) + 0.5f;
    }
    const int n = int(M.size());
    if (n == 1) return sample_level(M[0], cube, face, u, v).xyz();
    const float l  = std::min(std::max(lod, 0.0f), float(n - 1));
    const int   m0 = int(std::floor(l)), m1 = std::min(m0 + 1, n - 1);
    const float t  = l - float(m0);
    return (sample_level(M[m0], cube, face, u, v) * (1.0f - t) + sample_level(M[m1], cube, face, u, v) * t).xyz();
}

// CubemapFace.vsh's g_Rotation (PBR_Renderer.cpp:913-922) as DiligentCore builds it in float: RotationY(a) rows (c, 0, -s, 0),
// (0, 1, 0, 0), (s, 0, c, 0); RotationX(a) rows (1, 0, 0, 0), (0, c, s, 0), (0, -s, c, 0); row 3 (0, 0, 0, 1); s, c = sin, cos of the
// float angle, correctly rounded.
void face_matrix(int f, float M[4][4])
{
    const float pi = 3.14159265358979323846f;
    const float a  = f == 0 ? -pi / 2.0f : f == 1 ? pi / 2.0f : f == 2 ? pi / 2.0f : f == 3 ? -pi / 2.0f : f == 4 ? 0.0f : -pi;
    const float s = sin_(a), c = cos_(a);
    std::memset(M, 0, 16 * sizeof(float));
    M[3][3] = 1.0f;
    if (f == 4)
        M[0][0] = M[1][1] = M[2][2] = 1.0f;
    else if (f == 2 || f == 3)
        M[0][0] = 1.0f, M[1][1] = c, M[1][2] = s, M[2][1] = -s, M[2][2] = c;
    else
        M[0][0] = c, M[0][2] = -s, M[1][1] = 1.0f, M[2][0] = s, M[2][2] = c;
}

// normalize(WorldPos): mul(g_Rotation, float4(x, y, 1, 1)) at the pixel centre, xyz / w
float3 texel_dir(int f, int i, int j, int s)
{
    float M[4][4];
    face_matrix(f, M);
    const float x = 2.0f * (float(i) + 0.5f) / float(s) - 1.0f, y = 1.0f - 2.0f * (float(j) + 0.5f) / float(s);
    float       w[4];
    for (int r = 0; r < 4; ++r) w[r] = M[r][0] * x + M[r][1] * y + M[r][2] * 1.0f + M[r][3] * 1.0f;
    return normalize(float3(w[0], w[1], w[2]) / w[3]);
}

struct Source
{
    std::vector<Level> M;
    bool               cube;
    float              w, h; // g_EnvMapWidth / Height: level 0's face size (cube) or its width and height (sphere)
};

float pixel_solid_angle(const Source& S, float theta, float gamma)
{
    if (S.cube) return 4.0f * kPi / (6.0f * S.w * S.h); // ComputeCubeMapPixelSolidAngle
    const float dtheta = kPi / S.w, dphi = 2.0f * kPi / S.h; // ComputeSphereMapPixelSolidAngle
    return dphi * (cos_(theta - 0.5f * dtheta * gamma) - cos_(theta + 0.5f * dtheta * gamma));
}
float lod_of(const Source& S, float omega_s, float omega_p)
{
    return clampf(0.5f * log2_(omega_s / std::fmax(omega_p, 1e-10f)) + 1.0f, 0.0f, float(S.M.size()) - 1.0f);
}

// ComputeIrradianceMap.psh IrradianceMap(N)
float3 irradiance(const Source& S, float3 N, uint32_t n, bool opt)
{
    float3 T = normalize(cross(N, std::fabs(N.y) > 0.5f ? float3(1.0f, 0.0f, 0.0f) : float3(0.0f, 1.0f, 0.0f)));
    float3 B = cross(T, N);
    float3 acc(0.0f, 0.0f, 0.0f);
    for (uint32_t i = 0; i < n; ++i)
    {
        const float2 xi = hammersley(i, n);
        const float  phi = 2.0f * kPi * xi.x;
        float3       L(cos_(phi) * std::sqrt(1.0f - xi.y), sin_(phi) * std::sqrt(1.0f - xi.y), std::sqrt(xi.y));
        const float  pdf = std::fmax(L.z, 1e-6f) / kPi;
        L                = normalize(L.x * T + L.y * B + L.z * N);
        float lod        = 0.0f;
        if (opt) lod = lod_of(S, 1.0f / (float(n) * pdf), pixel_solid_angle(S, S.cube ? 0.0f : acos_(L.y), 0.5f));
        acc += sample_env(S.M, S.cube, L, lod);
    }
    return acc / float(n);
}

// PrefilterEnvMap.psh PrefilterEnvMap(PerceptualRoughness, R)
float3 prefilter(const Source& S, float rough, float3 R, uint32_t n, bool opt)
{
    const float3 N = R, V = R;
    const float  alpha = rough * rough, a2 = alpha * alpha;
    float3       acc(0.0f, 0.0f, 0.0f);
    float        total = 0.0f;
    for (uint32_t i = 0; i < n; ++i)
    {
        const float3 H   = ImportanceSampleGGX(hammersley(i, n), rough, N);
        const float3 L   = 2.0f * dot(V, H) * H - V;
        const float  NoL = clampf(dot(N, L), 0.0f, 1.0f), VoH = clampf(dot(V, H), 0.0f, 1.0f);
        if (!(NoL > 0.0f && VoH > 0.0f)) continue;
        float lod = 0.0f;
        if (opt && alpha != 0.0f)
        {
            // SmithGGXSampleDirectionPDF(V, N, L, AlphaRoughness)
            const float3 Hh = normalize(V + L);
            const float  ndh = dot(Hh, N), ndv = dot(N, V), ndl = dot(N, L);
            float        pdf = 0.0f;
            if (ndh > 0.0f && ndv > 0.0f && ndl > 0.0f)
            {
                const float ar = std::fmax(alpha, 1e-3f), ar2 = ar * ar, nh2 = ndh * ndh;
                const float f   = nh2 * ar2 + (1.0f - nh2);
                const float ndf = ar2 / std::fmax(kPi * f * f, 1e-9f); // NormalDistribution_GGX
                const float den = ndv + std::sqrt(a2 + (1.0f - a2) * ndv * ndv);
                const float g1  = 2.0f * std::fmax(ndv, 0.0f) / std::fmax(den, 1e-6f); // SmithGGXMasking
                pdf             = g1 * ndf / ndv / 4.0f;
            }
            pdf = std::fmax(pdf, 0.0001f);
            lod = lod_of(S, 1.0f / (float(n) * pdf), pixel_solid_angle(S, S.cube ? 0.0f : acos_(L.y), 1.0f));
        }
        acc += sample_env(S.M, S.cube, L, lod) * NoL;
        total += NoL;
    }
    return acc / total;
}
} // namespace
} // namespace orc

// C API (ctypes, oracle/oracle_ibl_py.py). Level i of the source is level_w[i] x level_h[i] RGBA fp32, tightly packed (a cube's s x 6s).
// Writes rows [row0, row1) of face `face` of an s_out x s_out output face into `out` ((row1 - row0) x s_out x 4 fp32). `pass` 0 is
// the irradiance (alpha 1), 1 the prefilter at `roughness` (alpha 0).
extern "C" __attribute__((visibility("default"))) void orci_ibl(int pass, int type, const float* const* levels, const int* level_w, const int* level_h,
                                                                int n_levels, uint32_t num_samples, int optimize, float roughness, int s_out, int face,
                                                                int row0, int row1, float* out, int threads)
{
    orc::Source S;
    for (int i = 0; i < n_levels; ++i) S.M.push_back(orc::Level{levels[i], level_w[i], level_h[i]});
    S.cube = type == 0;
    S.w    = float(level_w[0]);
    S.h    = float(S.cube ? level_w[0] : level_h[0]);
    const int rows = row1 - row0;
    threads        = std::max(1, std::min(threads, rows));
    std::vector<std::thread> pool;
    for (int t = 0; t < threads; ++t)
        pool.emplace_back([&, t] {
            for (int r = t; r < rows; r += threads)
                for (int i = 0; i < s_out; ++i)
                {
                    const orc::float3 N = orc::texel_dir(face, i, row0 + r, s_out);
                    const orc::float3 c = pass == 0 ? orc::irradiance(S, N, num_samples, optimize != 0) : orc::prefilter(S, roughness, N, num_samples, optimize != 0);
                    float* o = out + (size_t(r) * size_t(s_out) + size_t(i)) * 4;
                    o[0] = c.x, o[1] = c.y, o[2] = c.z, o[3] = pass == 0 ? 1.0f : 0.0f;
                }
        });
    for (auto& th : pool) th.join();
}
