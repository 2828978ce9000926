// dfx_line.cuh — the integer part of the aliased-line rule of DESIGN.md §2, shared by the line passes (B, dfx_bound_box.cu; the vector
// field, dfx_vector_field.cu): the viewport transform and 16.8 snap, the half-open diamonds and the pixel a line draws at one major-axis
// step. One statement of the rule, so every line pass covers the pixels the oracle and the reference harness's line_defs.inc cover.
#pragma once
#include "dfx_common.cuh"

namespace dfx
{
constexpr float kGuard = 268435456.0f; // 2^28: the guard band of 2^20 pixels in 1/256 units

// the viewport transform (y down) and the 16.8 snap (round half to even); false beyond the guard band, at w <= 0 or on NaN
DFX_HD bool snap(const float* a, float W, float H, int& X, int& Y, float& nz, float& iw)
{
    if (!(a[3] > 0.0f)) return false;
    const float nx = div_(a[0], a[3]), ny = div_(a[1], a[3]);
    nz = div_(a[2], a[3]), iw = div_(1.0f, a[3]);
    const float sx = mul_(mul_(add_(mul_(nx, 0.5f), 0.5f), W), 256.0f), sy = mul_(mul_(sub_(0.5f, mul_(ny, 0.5f)), H), 256.0f);
    if (!(fabsf(sx) < kGuard) || !(fabsf(sy) < kGuard)) return false;
    X = int(rintf(sx)), Y = int(rintf(sy));
    return true;
}

// floor(n / d) for 0 < d < 2^30, |n| < 2^59, without a 64-bit division: a double estimate from a refined reciprocal is within 2^-15 of
// n / d (|n / d| < 2^30), so the floor is off by at most one, which the remainder corrects
DFX_HD long long floor_div64(long long n, long long d)
{
    double y;
    const double dd = double(d);
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(dd));
    y           = fma(y, fma(-dd, y, 1.0), y);
    y           = fma(y, fma(-dd, y, 1.0), y);
    long long q = (long long)floor(double(n) * y);
    long long r = n - q * d;
    if (r < 0) --q, r += d;
    if (r >= d) ++q, r -= d;
    return q;
}

// the half-open diamond of the pixel centred at (cu, cv): |du| + |dv| < 1/2, plus the right and bottom corners and the edge between them
DFX_HD bool in_diamond(int pu, int pv, int cu, int cv)
{
    const long long du = (long long)pu - cu, dv = (long long)pv - cv, s = llabs(du) + llabs(dv);
    return s < 128 || (s == 128 && du >= 0 && dv >= 0);
}

// major-axis step i, in the frame where the major axis is u: the minor pixel j the line draws there, or false (DESIGN.md §2)
DFX_HD bool step_pixel(int au, int av, int bu, int bv, int i, int& j)
{
    const int cu = 256 * i + 128;
    if (au != bu && min(au, bu) <= cu && cu <= max(au, bu))
    {
        // j = floor((av * den + (cu - au) * (bv - av) - 1) / (256 den)), den = bu - au made positive, through q, r of the product / den
        long long n = (long long)(cu - au) * (long long)(bv - av), d = (long long)bu - au;
        if (d < 0) n = -n, d = -d;
        const long long q = floor_div64(n, d), r = n - q * d;
        j                 = int(((long long)av + q - (r == 0 ? 1 : 0)) >> 8);
    }
    else
    {
        j = (av - 1) >> 8; // the start's diamond, if it lies in one
        if (!in_diamond(au, av, cu, 256 * j + 128)) return false;
    }
    return !in_diamond(bu, bv, cu, 256 * j + 128); // the last-pixel rule: the segment must leave the diamond
}
} // namespace dfx
