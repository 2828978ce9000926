// dfx_shadow.cu — ShadowMapManager::ConvertToFilterable (Components/src/ShadowMapManager.cpp:533-600) as sm_90a kernels: VSMHorzPS or
// EVSMHorzPS, then VertBlurPS (Shaders/Shadows/private/ShadowConversions.fx), for every cascade, bit for bit by the rules of DESIGN.md §2.
//
// Every operation is rounded once in the shader's order (mul_ / add_ / div_, never contracted) and exp is the double function rounded
// once to float. The horizontal result is quantised to the filterable format before the vertical pass reads it, as the reference's
// intermediate texture does.
//
// Two paths, chosen by the range:
//   fused     one launch for all cascades (grid.z). A CTA stages its 64 x 32 tile's depth with both halos in shared memory, warped once
//             per texel; computes the quantised horizontal moments of the tile's rows and the vertical halo rows into shared memory;
//             then sums vertically and stores once. The filterable map is the only plane written. Ranges up to kFusedMaxRange.
//   two-pass  the reference's form through the caller's one-slice intermediate: per cascade a horizontal launch (row segments whose
//             depth is staged and warped in chunks) and a vertical launch. Any admitted range.
// Both compute the same operations on the same values, so they give the same bits.
#include <cmath>
#include "dfx_common.cuh"
#include "dfx_testing.h"

namespace dfx
{
namespace
{
constexpr int kThreads = 256;
constexpr int kTileX = 64, kTileY = 32; // fused tile
constexpr int kFusedMaxRange = 16;      // the fused tile's halo limit: shared memory 114,688 B at EVSM4 with both ranges 16
constexpr int kMaxRange = 1 << 15;      // ranges of 2^15 or more are refused
constexpr int kMaxDim = 16384;          // the largest 2-D texture Direct3D allows

// The weights of one axis. GetSampleWeight(i, r) is 1 for every tap but at most two at each end (DESIGN.md §2: 0.5 - r is exact for
// the admitted radii >= 0.25, and r + 0.5 rounds up to the next integer at most once); lo = the taps -R, -R + 1, hi = the taps R, R - 1.
struct Axis
{
    int   R;
    float lo[2], hi[2], total;
};
struct Cascade
{
    const char* in;
    char*       out;
    int         in_pitch, out_pitch;
    Axis        h, v;
};
struct Args
{
    Cascade c[DFX_MAX_CASCADES];
    int     w, h;
    float   ex, ey; // GetEVSMExponents: the clamped positive and negative exponents
    int     skip;   // iFixedFilterSize == 2: the horizontal result is the filterable map
};

// tap k = i + R of 0..2R
DFX_HD float tap_weight(const Axis& a, int k) { return k < 2 ? a.lo[k] : (k > 2 * a.R - 2 ? a.hi[2 * a.R - k] : 1.0f); }

// What a mode stages per depth texel (B floats) and sums per tap (C moments): VSM d -> (d, d^2); EVSM2 the positive warp p -> (p, p^2)
// (the RG targets keep .xy, so the negative warp is never stored); EVSM4 (p, n) -> (p, p^2, n, n^2).
template <int MODE> struct Mode
{
    static constexpr int B = MODE == DFX_SHADOW_MODE_EVSM4 ? 2 : 1, C = 2 * B;
};

DFX_HD float exp_(float x) { return float(exp(double(x))); } // correctly rounded (DESIGN.md §2)

template <bool D16> DFX_HD float load_depth(const Cascade& c, int x, int y)
{
    const char* row = c.in + size_t(y) * size_t(c.in_pitch);
    if constexpr (D16) return div_(float(__ldg(reinterpret_cast<const uint16_t*>(row) + x)), 65535.0f);
    else return __ldg(reinterpret_cast<const float*>(row) + x);
}

// WarpDepthEVSM (Shadows.fxh:288-295) or the depth itself
template <int MODE> DFX_HD void stage(const Args& A, float d, float* s)
{
    if constexpr (MODE == DFX_SHADOW_MODE_VSM) s[0] = d;
    else
    {
        const float dd = sub_(mul_(2.0f, d), 1.0f);
        s[0]           = exp_(mul_(A.ex, dd));
        if constexpr (MODE == DFX_SHADOW_MODE_EVSM4) s[1] = -exp_(mul_(-A.ey, dd));
    }
}

// m += float{2,4}(s.x, s.x * s.x[, s.y, s.y * s.y]) * w
template <int MODE> DFX_HD void accumulate(float* m, const float* s, float w)
{
#pragma unroll
    for (int b = 0; b < Mode<MODE>::B; ++b)
    {
        m[2 * b]     = add_(m[2 * b], mul_(s[b], w));
        m[2 * b + 1] = add_(m[2 * b + 1], mul_(mul_(s[b], s[b]), w));
    }
}

// The filterable format's store of one value, read back: RG16_UNORM floor(saturate(v) * 65535 + 0.5) (NaN -> 0) as k / 65535; the
// 16-bit floats round to nearest even; the 32-bit formats keep the value
template <int MODE, bool B32> DFX_HD float quantise(float v)
{
    if constexpr (B32) return v;
    else if constexpr (MODE == DFX_SHADOW_MODE_VSM)
    {
        const float c = v != v ? 0.0f : fminf(fmaxf(v, 0.0f), 1.0f);
        return div_(floorf(add_(mul_(c, 65535.0f), 0.5f)), 65535.0f);
    }
    else return __half2float(__float2half_rn(v));
}

// m holds quantised values (so the UNORM code is exact: round(q * 65535))
template <int MODE, bool B32> DFX_HD void store(char* base, int pitch, int x, int y, const float* m)
{
    char* row = base + size_t(y) * size_t(pitch);
    if constexpr (B32)
    {
        if constexpr (Mode<MODE>::C == 4) reinterpret_cast<float4*>(row)[x] = make_float4(m[0], m[1], m[2], m[3]);
        else reinterpret_cast<float2*>(row)[x] = make_float2(m[0], m[1]);
    }
    else if constexpr (MODE == DFX_SHADOW_MODE_VSM)
        reinterpret_cast<ushort2*>(row)[x] = make_ushort2(uint16_t(rintf(m[0] * 65535.0f)), uint16_t(rintf(m[1] * 65535.0f)));
    else if constexpr (Mode<MODE>::C == 4)
    {
        const __half2 a = __floats2half2_rn(m[0], m[1]), b = __floats2half2_rn(m[2], m[3]);
        uint2         u;
        u.x = *reinterpret_cast<const uint32_t*>(&a), u.y = *reinterpret_cast<const uint32_t*>(&b);
        reinterpret_cast<uint2*>(row)[x] = u;
    }
    else reinterpret_cast<__half2*>(row)[x] = __floats2half2_rn(m[0], m[1]);
}

// The intermediate's texel (x, y), read back as the vertical pass's Load does
template <int MODE, bool B32> DFX_HD void load_inter(const char* base, int pitch, int x, int y, float* m)
{
    const char* row = base + size_t(y) * size_t(pitch);
    if constexpr (B32)
    {
        if constexpr (Mode<MODE>::C == 4)
        {
            const float4 v = __ldg(reinterpret_cast<const float4*>(row) + x);
            m[0] = v.x, m[1] = v.y, m[2] = v.z, m[3] = v.w;
        }
        else
        {
            const float2 v = __ldg(reinterpret_cast<const float2*>(row) + x);
            m[0] = v.x, m[1] = v.y;
        }
    }
    else if constexpr (MODE == DFX_SHADOW_MODE_VSM)
    {
        const ushort2 v = __ldg(reinterpret_cast<const ushort2*>(row) + x);
        m[0] = div_(float(v.x), 65535.0f), m[1] = div_(float(v.y), 65535.0f);
    }
    else if constexpr (Mode<MODE>::C == 4)
    {
        const uint2  v = __ldg(reinterpret_cast<const uint2*>(row) + x);
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&v.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&v.y));
        m[0] = a.x, m[1] = a.y, m[2] = b.x, m[3] = b.y;
    }
    else
    {
        const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(row) + x);
        const float2   a = __half22float2(*reinterpret_cast<const __half2*>(&v));
        m[0] = a.x, m[1] = a.y;
    }
}

template <int MODE, bool B32> DFX_HD void finish(float* m, float total)
{
#pragma unroll
    for (int k = 0; k < Mode<MODE>::C; ++k) m[k] = quantise<MODE, B32>(div_(m[k], total));
}

template <int MODE, bool B32, bool D16>
__global__ void __launch_bounds__(kThreads) fused_kernel(const __grid_constant__ Args A)
{
    constexpr int  B = Mode<MODE>::B, C = Mode<MODE>::C;
    extern __shared__ float smem[];
    const Cascade& c = A.c[blockIdx.z];
    const int      Rh = c.h.R, Rv = c.v.R, x0 = int(blockIdx.x) * kTileX, y0 = int(blockIdx.y) * kTileY;
    const int      rows = kTileY + 2 * Rv, cols = kTileX + 2 * Rh;
    float*         s1 = smem;                   // rows x cols staged depth texels, B floats each
    float*         s2 = smem + rows * cols * B; // rows x kTileX quantised horizontal moments, C floats each

    for (int i = threadIdx.x; i < rows * cols; i += kThreads)
    {
        const int r = i / cols, x = x0 - Rh + (i - r * cols), y = y0 - Rv + r;
        if (unsigned(y) >= unsigned(A.h)) continue; // the row's horizontal result reads as 0
        stage<MODE>(A, unsigned(x) < unsigned(A.w) ? load_depth<D16>(c, x, y) : 0.0f, s1 + i * B);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < rows * kTileX; i += kThreads)
    {
        const int r = i / kTileX, q = i - r * kTileX;
        float     m[C] = {};
        if (unsigned(y0 - Rv + r) < unsigned(A.h))
        {
            const float* s = s1 + (r * cols + q) * B;
            for (int k = 0; k <= 2 * Rh; ++k) accumulate<MODE>(m, s + k * B, tap_weight(c.h, k));
            finish<MODE, B32>(m, c.h.total);
        }
#pragma unroll
        for (int k = 0; k < C; ++k) s2[i * C + k] = m[k];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kTileY * kTileX; i += kThreads)
    {
        const int r = i / kTileX, q = i - r * kTileX, x = x0 + q, y = y0 + r;
        if (x >= A.w || y >= A.h) continue;
        float m[C] = {};
        if (A.skip)
        {
#pragma unroll
            for (int k = 0; k < C; ++k) m[k] = s2[((r + Rv) * kTileX + q) * C + k];
        }
        else
        {
            for (int t = 0; t <= 2 * Rv; ++t)
            {
                const float  w = tap_weight(c.v, t);
                const float* s = s2 + ((r + t) * kTileX + q) * C;
#pragma unroll
                for (int k = 0; k < C; ++k) m[k] = add_(m[k], mul_(s[k], w));
            }
            finish<MODE, B32>(m, c.v.total);
        }
        store<MODE, B32>(c.out, c.out_pitch, x, y, m);
    }
}

// Two-pass path, horizontal: one CTA per 256-texel row segment of cascade `ci`; the segment's depth span is staged and warped in
// chunks of 256 texels, and each thread adds the taps of a chunk that are its own, in tap order
template <int MODE, bool B32, bool D16>
__global__ void __launch_bounds__(kThreads) horz_kernel(const __grid_constant__ Args A, int ci, char* dst, int dst_pitch)
{
    constexpr int  B = Mode<MODE>::B, C = Mode<MODE>::C;
    __shared__ float s1[kThreads * B];
    const Cascade&   c = A.c[ci];
    const int        R = c.h.R, x0 = int(blockIdx.x) * kThreads, x = x0 + int(threadIdx.x), y = int(blockIdx.y);
    float            m[C] = {};
    for (int s0 = x0 - R; s0 <= x0 + kThreads - 1 + R; s0 += kThreads)
    {
        const int xs = s0 + int(threadIdx.x);
        stage<MODE>(A, unsigned(xs) < unsigned(A.w) ? load_depth<D16>(c, xs, y) : 0.0f, s1 + threadIdx.x * B);
        __syncthreads();
        const int lo = max(x - R, s0), hi = min(x + R, s0 + kThreads - 1);
        for (int j = lo; j <= hi; ++j) accumulate<MODE>(m, s1 + (j - s0) * B, tap_weight(c.h, j - (x - R)));
        __syncthreads();
    }
    if (x >= A.w) return;
    finish<MODE, B32>(m, c.h.total);
    store<MODE, B32>(dst, dst_pitch, x, y, m);
}

// Two-pass path, vertical: one thread per texel of cascade `ci`, reading the intermediate's column
template <int MODE, bool B32>
__global__ void __launch_bounds__(kThreads) vert_kernel(const __grid_constant__ Args A, int ci, const char* src, int src_pitch)
{
    constexpr int  C = Mode<MODE>::C;
    const Cascade& c = A.c[ci];
    const int      R = c.v.R, x = int(blockIdx.x) * kThreads + int(threadIdx.x), y = int(blockIdx.y);
    if (x >= A.w) return;
    float m[C] = {};
    for (int t = 0; t <= 2 * R; ++t)
    {
        const int yy = y - R + t;
        float     v[C] = {};
        if (unsigned(yy) < unsigned(A.h)) load_inter<MODE, B32>(src, src_pitch, x, yy, v);
        const float w = tap_weight(c.v, t);
#pragma unroll
        for (int k = 0; k < C; ++k) m[k] = add_(m[k], mul_(v[k], w));
    }
    finish<MODE, B32>(m, c.v.total);
    store<MODE, B32>(c.out, c.out_pitch, x, y, m);
}

// ---------------------------------------------------------------------------------------------------------------------------------------
// host

// GetSampleWeight (ShadowConversions.fx:23-28), in float
float sample_weight(int x, float r)
{
    const float lo = std::fmax(float(x), std::fmin(0.5f - r, 0.0f));
    const float hi = std::fmin(float(x) + 1.0f, std::fmax(0.5f + r, 1.0f));
    return hi - lo;
}

dfx_status make_axis(float r, Axis& a, int cascade, const char* axis)
{
    DFX_REQUIRE(std::isfinite(r) && r >= 0.0f, "cascade %d: the %s filter radius %g is negative or not finite", cascade, axis, double(r));
    const float fr = std::floor(r + 0.5f);
    DFX_REQUIRE(fr < float(kMaxRange), "cascade %d: the %s filter radius %g has a range of 2^15 or more", cascade, axis, double(r));
    a.R     = int(fr);
    a.lo[0] = sample_weight(-a.R, r), a.lo[1] = sample_weight(-a.R + 1, r);
    a.hi[0] = sample_weight(a.R, r), a.hi[1] = sample_weight(a.R - 1, r);
    float t = 0.0f; // fTotalWeight, summed in the shader's order
    for (int i = -a.R; i <= a.R; ++i) t += sample_weight(i, r);
    a.total = t;
    return DFX_OK;
}

dfx_status filter_radii(const dfx_shadow_map_attribs& s, int i, int width, int height, float& rh, float& rv)
{
    if (s.iFixedFilterSize > 0)
    {
        rh = rv = static_cast<float>((s.iFixedFilterSize - 1) / 2);
        return DFX_OK;
    }
    const dfx_cascade_attribs& c = s.Cascades[i];
    const float fNDCtoUVScale = 0.5f;
    const float fFilterWidth  = s.fFilterWorldSize * c.f4LightSpaceScale[0] * fNDCtoUVScale;
    const float fFilterHeight = s.fFilterWorldSize * c.f4LightSpaceScale[1] * fNDCtoUVScale;
    rh = fFilterWidth / 2.f * static_cast<float>(width);
    rv = fFilterHeight / 2.f * static_cast<float>(height);
    return DFX_OK;
}

// The filterable format of a mode at 16 / 32 bits
int filterable_format(int mode, bool b32)
{
    if (mode == DFX_SHADOW_MODE_VSM) return b32 ? DFX_FORMAT_RG32F : DFX_FORMAT_RG16U;
    if (mode == DFX_SHADOW_MODE_EVSM2) return b32 ? DFX_FORMAT_RG32F : DFX_FORMAT_RG16F;
    return b32 ? DFX_FORMAT_RGBA32F : DFX_FORMAT_RGBA16F;
}

int format_bytes(int fmt)
{
    switch (fmt)
    {
    case DFX_FORMAT_R16U: return 2;
    case DFX_FORMAT_R32F: case DFX_FORMAT_RG16U: case DFX_FORMAT_RG16F: return 4;
    case DFX_FORMAT_RG32F: case DFX_FORMAT_RGBA16F: return 8;
    case DFX_FORMAT_RGBA32F: return 16;
    default: return 0;
    }
}

// null, size, pitch, alignment and the 2 GiB plane limit; the format is checked by the caller
bool plane_ok(const dfx_plane* p, int w, int h)
{
    const size_t bpt = size_t(format_bytes(p->format));
    return p->ptr && bpt && p->width == w && p->height == h && p->pitch_bytes % bpt == 0 && p->pitch_bytes >= size_t(w) * bpt &&
           reinterpret_cast<uintptr_t>(p->ptr) % bpt == 0 && p->pitch_bytes * size_t(h) < (size_t(1) << 31);
}

// The bytes a plane spans: [first, end)
bool overlap(const dfx_plane& a, const dfx_plane& b)
{
    const uintptr_t a0 = reinterpret_cast<uintptr_t>(a.ptr), b0 = reinterpret_cast<uintptr_t>(b.ptr);
    const uintptr_t a1 = a0 + a.pitch_bytes * size_t(a.height - 1) + size_t(a.width) * size_t(format_bytes(a.format));
    const uintptr_t b1 = b0 + b.pitch_bytes * size_t(b.height - 1) + size_t(b.width) * size_t(format_bytes(b.format));
    return a0 < b1 && b0 < a1;
}

size_t fused_smem(int mode, int Rh, int Rv)
{
    const int b = mode == DFX_SHADOW_MODE_EVSM4 ? 2 : 1;
    return sizeof(float) * size_t(kTileY + 2 * Rv) * size_t((kTileX + 2 * Rh) * b + kTileX * 2 * b);
}

template <int MODE, bool B32, bool D16>
dfx_status launch(cudaStream_t s, const Args& A, int n, bool fused, const dfx_plane* inter)
{
    if (fused)
    {
        int Rh = 0, Rv = 0;
        for (int i = 0; i < n; ++i) Rh = std::max(Rh, A.c[i].h.R), Rv = std::max(Rv, A.c[i].v.R);
        const size_t smem = fused_smem(MODE, Rh, Rv);
        DFX_CUDA(cudaFuncSetAttribute(fused_kernel<MODE, B32, D16>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
        fused_kernel<MODE, B32, D16><<<dim3(unsigned(div_up(A.w, kTileX)), unsigned(div_up(A.h, kTileY)), unsigned(n)), kThreads, smem, s>>>(A);
        DFX_LAUNCHED("shadow_filterable_fused_kernel");
        return DFX_OK;
    }
    const dim3 grid(unsigned(div_up(A.w, kThreads)), unsigned(A.h));
    for (int i = 0; i < n; ++i)
    {
        if (A.skip) // the horizontal pass writes the filterable slice
        {
            horz_kernel<MODE, B32, D16><<<grid, kThreads, 0, s>>>(A, i, A.c[i].out, A.c[i].out_pitch);
            DFX_LAUNCHED("shadow_horz_kernel");
            continue;
        }
        horz_kernel<MODE, B32, D16><<<grid, kThreads, 0, s>>>(A, i, static_cast<char*>(inter->ptr), int(inter->pitch_bytes));
        DFX_LAUNCHED("shadow_horz_kernel");
        vert_kernel<MODE, B32><<<grid, kThreads, 0, s>>>(A, i, static_cast<const char*>(inter->ptr), int(inter->pitch_bytes));
        DFX_LAUNCHED("shadow_vert_kernel");
    }
    return DFX_OK;
}
} // namespace
} // namespace dfx

using namespace dfx;

extern "C" dfx_status dfx_shadow_filter_radii(const dfx_shadow_map_attribs* attribs, int32_t cascade, int32_t width, int32_t height,
                                              float* horz_radius, float* vert_radius)
{
    DFX_REQUIRE(attribs && horz_radius && vert_radius, "null argument");
    DFX_REQUIRE(cascade >= 0 && cascade < DFX_MAX_CASCADES, "cascade %d is outside 0..%d", cascade, DFX_MAX_CASCADES - 1);
    return filter_radii(*attribs, cascade, width, height, *horz_radius, *vert_radius);
}

namespace
{
dfx_status convert(void* stream, int32_t mode, const dfx_shadow_map_attribs* attribs, const dfx_plane* shadow_map, int32_t n,
                   const dfx_plane* filterable, const dfx_plane* intermediate, bool two_pass)
{
    DFX_REQUIRE(mode >= DFX_SHADOW_MODE_PCF && mode <= DFX_SHADOW_MODE_EVSM4, "unknown shadow mode %d", mode);
    if (mode == DFX_SHADOW_MODE_PCF) return DFX_OK; // PCF samples the depth itself: nothing to convert
    DFX_REQUIRE(attribs && shadow_map && filterable, "null argument");
    DFX_REQUIRE(n >= 1 && n <= DFX_MAX_CASCADES, "%d cascades (1..%d)", n, DFX_MAX_CASCADES);
    DFX_REQUIRE(n == attribs->iNumCascades, "%d shadow-map slices but iNumCascades = %d", n, attribs->iNumCascades);
    const int w = shadow_map[0].width, h = shadow_map[0].height, in_fmt = shadow_map[0].format;
    DFX_REQUIRE(in_fmt == DFX_FORMAT_R16U || in_fmt == DFX_FORMAT_R32F, "the shadow map is neither R16U (D16_UNORM) nor R32F (D32_FLOAT)");
    DFX_REQUIRE(w >= 1 && h >= 1 && w <= kMaxDim && h <= kMaxDim, "the shadow map is %dx%d (1..%d each way)", w, h, kMaxDim);
    const int out_fmt = filterable[0].format;
    DFX_REQUIRE(out_fmt == filterable_format(mode, false) || out_fmt == filterable_format(mode, true),
                "the filterable map's format %d is not the mode's 16- or 32-bit format", out_fmt);
    const bool b32 = out_fmt == filterable_format(mode, true);
    DFX_REQUIRE(bool(attribs->bIs32BitEVSM) == b32, "bIs32BitEVSM = %d but the filterable map is %d-bit", attribs->bIs32BitEVSM, b32 ? 32 : 16);

    Args A{};
    A.w = w, A.h = h, A.skip = attribs->iFixedFilterSize == 2;
    const float max_exp = b32 ? 42.0f : 5.54f;
    A.ex = std::fmin(attribs->fEVSMPositiveExponent, max_exp), A.ey = std::fmin(attribs->fEVSMNegativeExponent, max_exp);
    bool fused = !two_pass;
    for (int i = 0; i < n; ++i)
    {
        DFX_REQUIRE(shadow_map[i].format == in_fmt && plane_ok(&shadow_map[i], w, h),
                    "shadow-map slice %d: another format or size than slice 0, or a null, mis-pitched or misaligned plane", i);
        DFX_REQUIRE(filterable[i].format == out_fmt && plane_ok(&filterable[i], w, h),
                    "filterable slice %d: another format or size than the shadow map's slice 0, or a null, mis-pitched or misaligned plane", i);
        float rh, rv;
        filter_radii(*attribs, i, w, h, rh, rv);
        Cascade& c = A.c[i];
        dfx_status st;
        if ((st = make_axis(rh, c.h, i, "horizontal")) != DFX_OK || (st = make_axis(rv, c.v, i, "vertical")) != DFX_OK) return st;
        c.in = static_cast<const char*>(shadow_map[i].ptr), c.in_pitch = int(shadow_map[i].pitch_bytes);
        c.out = static_cast<char*>(filterable[i].ptr), c.out_pitch = int(filterable[i].pitch_bytes);
        fused = fused && c.h.R <= kFusedMaxRange && c.v.R <= kFusedMaxRange;
    }
    if (!fused)
        DFX_REQUIRE(intermediate && intermediate->format == out_fmt && plane_ok(intermediate, w, h),
                    "the two-pass path (a range above %d) needs an intermediate plane of the filterable map's size and format", kFusedMaxRange);
    // a written plane must not share bytes with another plane of the call: the kernels would read what other threads are writing
    for (int i = 0; i < n; ++i)
    {
        for (int j = 0; j < n; ++j)
        {
            DFX_REQUIRE(!overlap(filterable[i], shadow_map[j]), "filterable slice %d overlaps shadow-map slice %d", i, j);
            DFX_REQUIRE(j == i || !overlap(filterable[i], filterable[j]), "filterable slices %d and %d overlap", i, j);
        }
        if (!fused)
            DFX_REQUIRE(!overlap(*intermediate, filterable[i]) && !overlap(*intermediate, shadow_map[i]),
                        "the intermediate overlaps slice %d of the shadow map or the filterable map", i);
    }

    const cudaStream_t s = as_stream(stream);
    const bool         d16 = in_fmt == DFX_FORMAT_R16U;
#define SHADOW_LAUNCH(M) \
    DFX_FMT16(b32, B, DFX_FMT16(d16, D, return launch<M, B, D>(s, A, n, fused, intermediate)))
    if (mode == DFX_SHADOW_MODE_VSM) SHADOW_LAUNCH(DFX_SHADOW_MODE_VSM);
    else if (mode == DFX_SHADOW_MODE_EVSM2) SHADOW_LAUNCH(DFX_SHADOW_MODE_EVSM2);
    else SHADOW_LAUNCH(DFX_SHADOW_MODE_EVSM4);
#undef SHADOW_LAUNCH
    return DFX_OK;
}
} // namespace

extern "C" dfx_status dfx_shadow_convert_to_filterable(void* stream, int32_t mode, const dfx_shadow_map_attribs* attribs,
                                                       const dfx_plane* shadow_map, int32_t n, const dfx_plane* filterable,
                                                       const dfx_plane* intermediate)
{
    DFX_PROFILE(stream, "shadow_convert_to_filterable");
    return convert(stream, mode, attribs, shadow_map, n, filterable, intermediate, false);
}

extern "C" dfx_status dfx_testing_shadow_convert_two_pass(void* stream, int32_t mode, const dfx_shadow_map_attribs* attribs,
                                                          const dfx_plane* shadow_map, int32_t n, const dfx_plane* filterable,
                                                          const dfx_plane* intermediate)
{
    DFX_PROFILE(stream, "shadow_convert_two_pass");
    return convert(stream, mode, attribs, shadow_map, n, filterable, intermediate, true);
}
