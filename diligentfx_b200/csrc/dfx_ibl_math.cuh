// dfx_ibl_math.cuh — the arithmetic of PBR_Renderer's precomputations (the IBL cube maps of dfx_ibl.cu and the GGX table of
// dfx_compose.cu) as DESIGN.md §2 states it: every operation rounded once (mul_ / add_ / sub_ / div_ of dfx_common.cuh, never
// contracted) and every transcendental correctly rounded, formed in double. The test oracle states the same arithmetic.
#pragma once
#include "dfx_common.cuh"

namespace dfx
{
namespace iblm
{

// correctly rounded transcendentals: the double result rounded once. cos / sin go through cospi / sinpi of x / pi (a double relative
// error of a few 2^-53 for the arguments here, 2 pi Xi.x in [0, 2 pi) and the sphere's theta -+ dtheta / 2 just outside [0, pi]); double
// cos / sin would pull in the Payne-Hanek slow path's stack frame.
DFX_HD float cos_(float x) { return float(cospi(double(x) * 0.31830988618379067)); }
DFX_HD float sin_(float x) { return float(sinpi(double(x) * 0.31830988618379067)); }
// sqrt(a) correctly rounded without sqrt.rn.f32's slow-path call (the call makes the kernels spill): a double reciprocal square root
// estimate, two Newton steps and one correction give sqrt(a) within a few 2^-53; the square root of a float is never that close to a
// float rounding midpoint, so rounding it to float is the correctly rounded result. Float denormals are normal doubles.
DFX_HD float sqrt_(float a)
{
    if (!(a > 0.0f && a <= kFltMax)) return a == 0.0f || a > kFltMax ? a : __int_as_float(0x7fffffff); // +-0, +inf; NaN for a < 0 or NaN
    const double d = a;
    double       y;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(d));
    const double h = 0.5 * d;
    y              = y * fma(-h * y, y, 1.5);
    y              = y * fma(-h * y, y, 1.5);
    const double r = d * y;
    return float(fma(fma(-r, r, d), 0.5 * y, r));
}
// pow(x, 5.0) as ((x * x) * (x * x)) * x in double, rounded once to float: x * x is exact, so this is the correctly rounded x^5 except
// within 2^-52 of a float rounding midpoint. __dmul_rn keeps the compiler from contracting or reassociating it.
DFX_HD float pow5_(float x)
{
    const double d = x, d2 = __dmul_rn(d, d);
    return float(__dmul_rn(__dmul_rn(d2, d2), d));
}
DFX_HD float sat_(float x) { return fminf(fmaxf(x, 0.0f), 1.0f); } // saturate: NaN -> 0
DFX_HD float dot3(float3 a, float3 b) { return add_(add_(mul_(a.x, b.x), mul_(a.y, b.y)), mul_(a.z, b.z)); }
DFX_HD float3 normalize3(float3 a)
{
    const float l = sqrt_(dot3(a, a));
    return make_float3(div_(a.x, l), div_(a.y, l), div_(a.z, l));
}
DFX_HD float3 cross3(float3 a, float3 b)
{
    return make_float3(sub_(mul_(a.y, b.z), mul_(a.z, b.y)), sub_(mul_(a.z, b.x), mul_(a.x, b.z)), sub_(mul_(a.x, b.y), mul_(a.y, b.x)));
}
// a * x + b * y + c * z per component: ((a.c * x + b.c * y) + c.c * z)
DFX_HD float3 combine3(float3 a, float x, float3 b, float y, float3 c, float z)
{
    return make_float3(add_(add_(mul_(a.x, x), mul_(b.x, y)), mul_(c.x, z)), add_(add_(mul_(a.y, x), mul_(b.y, y)), mul_(c.y, z)),
                       add_(add_(mul_(a.z, x), mul_(b.z, y)), mul_(c.z, z)));
}
// Hammersley2D (PBR_PrecomputeCommon.fxh:10-16)
DFX_HD float2 hammersley(uint32_t i, uint32_t n) { return make_float2(div_(float(i), float(n)), mul_(__uint2float_rn(__brev(i)), 2.3283064365386963e-10f)); }

} // namespace iblm
} // namespace dfx
