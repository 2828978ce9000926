// dfx_env_sample.cuh — the project's Sam_LinearClamp over an environment map, shared by E (dfx_env_map.cu) and the IBL precomputation
// (dfx_ibl.cu): the software bilinear with 8 fractional bits of position (DESIGN.md §2, as every sampled pass), the seamless cube rule of
// DESIGN.md §2 and the trilinear LOD clamped to the map's levels. Every operation is one rounding (mul_ / add_ / div_, never contracted);
// atan2 / asin (sphere) are evaluated in double and rounded once. No texture objects: the hardware filter's weight precision is not
// documented.
#pragma once
#include "dfx_common.cuh"

namespace dfx
{
namespace envs
{
// A map's mip chain: a cube's level m is one plane of s_m x 6 s_m texels (faces +X, -X, +Y, -Y, +Z, -Z stacked), a sphere's is w_m x h_m
struct EnvMapLevels
{
    const char* p[DFX_MAX_ENV_LEVELS];
    int         pitch[DFX_MAX_ENV_LEVELS]; // bytes
    int         w[DFX_MAX_ENV_LEVELS], h[DFX_MAX_ENV_LEVELS];
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
} // namespace envs
} // namespace dfx
