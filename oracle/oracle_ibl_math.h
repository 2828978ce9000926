// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_math.h). The arithmetic PBR_Renderer's precomputations share (DESIGN.md §2): the IBL cube
// maps of oracle_ibl.cpp and the pre-integrated GGX table of oracle_compose_ibl.cpp. Built without FMA contraction, every operation is
// rounded once; the transcendentals are the double function rounded once to float; pow(x, 5) is ((x * x) * (x * x)) * x in double,
// rounded once. The kernels state the same in diligentfx_b200/csrc/dfx_ibl_math.cuh, the reference-shader build in
// oracle/refshader/ibl_defs.inc.
#pragma once
#include "oracle_math.h"

#include <cmath>
#include <cstdint>

namespace orc
{
namespace iblm
{
constexpr float kPi = 3.141592653589793f; // PBR_Common.fxh:5, the PI the include order leaves in force

inline float cos_(float x) { return float(std::cos(double(x))); }
inline float sin_(float x) { return float(std::sin(double(x))); }
// x * x is exact in double, so this is the correctly rounded x^5 except within 2^-52 of a float rounding midpoint
inline float pow5_(float x)
{
    const double d = x, d2 = d * d;
    return float((d2 * d2) * d);
}

// Hammersley2D (PBR_PrecomputeCommon.fxh:10-16)
inline float2 hammersley(uint32_t i, uint32_t n)
{
    uint32_t v = i;
    v          = ((v >> 1) & 0x55555555u) | ((v & 0x55555555u) << 1);
    v          = ((v >> 2) & 0x33333333u) | ((v & 0x33333333u) << 2);
    v          = ((v >> 4) & 0x0F0F0F0Fu) | ((v & 0x0F0F0F0Fu) << 4);
    v          = ((v >> 8) & 0x00FF00FFu) | ((v & 0x00FF00FFu) << 8);
    v          = (v >> 16) | (v << 16);
    return float2(float(i) / float(n), float(v) * 2.3283064365386963e-10f);
}

// ImportanceSampleGGX (PBR_PrecomputeCommon.fxh:19-39)
inline float3 ImportanceSampleGGX(float2 Xi, float PerceptualRoughness, float3 N)
{
    const float AlphaRoughness = PerceptualRoughness * PerceptualRoughness;
    const float a2             = AlphaRoughness * AlphaRoughness;
    const float Phi            = 2.0f * kPi * Xi.x;
    const float CosTheta       = std::sqrt(saturate((1.0f - Xi.y) / (1.0f + (a2 - 1.0f) * Xi.y)));
    const float SinTheta       = std::sqrt(saturate(1.0f - CosTheta * CosTheta));
    const float3 H(SinTheta * cos_(Phi), SinTheta * sin_(Phi), CosTheta);
    const float3 UpVector = std::fabs(N.z) < 0.999f ? float3(0.0f, 0.0f, 1.0f) : float3(1.0f, 0.0f, 0.0f);
    const float3 TangentX = normalize(cross(UpVector, N));
    const float3 TangentY = cross(N, TangentX);
    return TangentX * H.x + TangentY * H.y + N * H.z;
}
} // namespace iblm
} // namespace orc
