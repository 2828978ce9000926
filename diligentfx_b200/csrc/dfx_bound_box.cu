// dfx_bound_box.cu — B, the selected prim's bounding box, as an sm_90a kernel: the pipeline state of BoundBoxRenderer::GetPSO
// (Components/src/BoundBoxRenderer.cpp:150-168: LINE_LIST, depth test LESS_EQUAL / GREATER_EQUAL, no depth writes, no blending) around
// BoundBoxVS (Shaders/Common/private/BoundBox.vsh) and GetBoundBoxOutput (BoundBox.psh:27-48).
//
// The 24 vertices make 12 lines, rasterised by the aliased-line rule of DESIGN.md §2: every coverage decision is integer arithmetic on
// the 16.8 snapped endpoints, so the covered pixels are the oracle's by construction, and every floating-point operation of the rule
// and of the shaders is one rounding (mul_ / add_ / sub_ / div_ / __fsqrt_rn, never contracted), so the fragments are the oracle's
// bit for bit. Each CTA sets the 12 lines up in shared memory; then one thread per major-axis step of one line draws at most one
// pixel. The overlap rule (a pixel keeps the last surviving fragment in primitive order) is resolved without barriers between lines:
// a thread stores its fragment only if no later line covers its pixel with a fragment that survives the depth and pattern tests.
#include "dfx_line.cuh"

namespace dfx
{
namespace
{
constexpr int kBoxThreads = 128;

struct BoxLine
{
    int   ok, xmajor;
    int   ax, ay, bx, by;     // snapped endpoints, 1/256 pixel (|.| < 2^28)
    float nz0, nz1, iw0, iw1; // z / w and 1 / w at the clipped endpoints
    float a0[12], a1[12];     // CLIP_POS, PREV_CLIP_POS, EDGE_START_CLIP_POS at the clipped endpoints
};

// float4(v) * M, the shader's mul(v, M): ((r0 * x + r1 * y) + r2 * z) + r3 * w per column
DFX_HD float4 mul_row(float4 v, const dfx_float4x4& M)
{
    float r[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) r[c] = add_(add_(add_(mul_(M.m[0][c], v.x), mul_(M.m[1][c], v.y)), mul_(M.m[2][c], v.z)), mul_(M.m[3][c], v.w));
    return make_float4(r[0], r[1], r[2], r[3]);
}

// GetBoxCorner (BoundBox.vsh:14-55)
DFX_HD float4 box_corner(uint32_t id, const dfx_float4x4& T)
{
    id = id < 8u ? ((id + 1u) >> 1u) & 3u : id < 16u ? 4u + (((id + 1u) >> 1u) & 3u) : ((id - 16u) >> 1u) + (id & 1u) * 4u;
    return mul_row(make_float4((id & 2u) ? 1.0f : 0.0f, ((id + 1u) & 2u) ? 1.0f : 0.0f, (id & 4u) ? 1.0f : 0.0f, 1.0f), T);
}

DFX_HD void put4(float* a, float4 v) { a[0] = v.x, a[1] = v.y, a[2] = v.z, a[3] = v.w; }

// BoundBoxVS for vertex `id`
DFX_HD void box_vs(uint32_t id, const dfx_camera_attribs* cams, const dfx_float4x4& T, bool motion, float* a)
{
    const float4 corner = box_corner(id, T);
    const float4 p      = mul_row(corner, cams[0].mViewProj);
    put4(a, p);
    put4(a + 4, motion ? mul_row(corner, cams[1].mViewProj) : p);
    put4(a + 8, mul_row(box_corner(id & ~1u, T), cams[0].mViewProj));
}

// Line l: the VS of its two vertices, [near, far] clipping in clip space (d = z, then d = w - z; NaN is outside), the snap
__device__ void setup_line(int l, const dfx_camera_attribs* cams, const dfx_bound_box_attribs& A, bool motion, float W, float H, BoxLine& L)
{
    float v0[12], v1[12];
    box_vs(uint32_t(2 * l), cams, A.Transform, motion, v0);
    box_vs(uint32_t(2 * l + 1), cams, A.Transform, motion, v1);
    L.ok = 0;
    for (int plane = 0; plane < 2; ++plane)
    {
        const float d0 = plane == 0 ? v0[2] : sub_(v0[3], v0[2]), d1 = plane == 0 ? v1[2] : sub_(v1[3], v1[2]);
        const bool  in0 = d0 >= 0.0f, in1 = d1 >= 0.0f;
        if (!in0 && !in1) return;
        if (!in0)
        {
            const float t = div_(d0, sub_(d0, d1));
#pragma unroll
            for (int k = 0; k < 12; ++k) v0[k] = add_(v0[k], mul_(sub_(v1[k], v0[k]), t));
        }
        else if (!in1)
        {
            const float t = div_(d1, sub_(d1, d0));
#pragma unroll
            for (int k = 0; k < 12; ++k) v1[k] = add_(v1[k], mul_(sub_(v0[k], v1[k]), t));
        }
    }
    if (!snap(v0, W, H, L.ax, L.ay, L.nz0, L.iw0) || !snap(v1, W, H, L.bx, L.by, L.nz1, L.iw1)) return;
#pragma unroll
    for (int k = 0; k < 12; ++k) L.a0[k] = v0[k], L.a1[k] = v1[k];
    L.xmajor = abs(L.bx - L.ax) >= abs(L.by - L.ay);
    L.ok     = 1;
}

DFX_HD bool covers(const BoxLine& L, int x, int y)
{
    int j;
    if (!L.ok) return false;
    if (L.xmajor) return step_pixel(L.ax, L.ay, L.bx, L.by, x, j) && j == y;
    return step_pixel(L.ay, L.ax, L.by, L.bx, y, j) && j == x;
}

// the fragment of L at (x, y): the depth test on its z / w, then GetBoundBoxOutput (false = discarded); the motion into mv
DFX_HD bool survives(const BoxLine& L, int x, int y, const dfx_camera_attribs* cams, const dfx_bound_box_attribs& A, bool rev, float d, float2& mv)
{
    const long long cx = 256ll * x + 128, cy = 256ll * y + 128, dx = (long long)L.bx - L.ax, dy = (long long)L.by - L.ay;
    const long long num = (cx - L.ax) * dx + (cy - L.ay) * dy, den = dx * dx + dy * dy;
    const float     t   = fminf(fmaxf(div_(float(num), float(den)), 0.0f), 1.0f);
    const float     z   = add_(L.nz0, mul_(sub_(L.nz1, L.nz0), t));
    if (!(rev ? z >= d : z <= d)) return false;
    const float tp = div_(mul_(t, L.iw1), add_(mul_(sub_(1.0f, t), L.iw0), mul_(t, L.iw1)));
    const auto  at = [&](int k) { return add_(L.a0[k], mul_(sub_(L.a1[k], L.a0[k]), tp)); };
    const float cw = at(3), ew = at(11);
    const float px = div_(at(0), cw), py = div_(at(1), cw), ex = div_(at(8), ew), ey = div_(at(9), ew);
    const dfx_camera_attribs& C = cams[0];
    const float vx = mul_(sub_(px, ex), C.f4ViewportSize[0]), vy = mul_(sub_(py, ey), C.f4ViewportSize[1]);
    const float dist = __fsqrt_rn(add_(mul_(vx, vx), mul_(vy, vy)));
    const float q    = div_(dist, A.PatternLength);
    const uint32_t bit = min(__float2uint_rz(mul_(sub_(q, floorf(q)), A.PatternLength)), 31u); // D3D ftou: NaN -> 0, saturating
    if ((A.PatternMask & (1u << bit)) == 0u) return false;
    const dfx_camera_attribs& P  = cams[1];
    const float               pw = at(7), qx = div_(at(4), pw), qy = div_(at(5), pw);
    // GetMotionVector (ShaderUtilities.fxh:88-91): (ClipPos - Jitter) - (PrevClipPos - PrevJitter)
    mv = make_float2(sub_(sub_(px, C.f2Jitter[0]), sub_(qx, P.f2Jitter[0])), sub_(sub_(py, C.f2Jitter[1]), sub_(qy, P.f2Jitter[1])));
    return true;
}

__global__ void __launch_bounds__(kBoxThreads) bound_box_kernel(const dfx_camera_attribs* __restrict__ cams, const __grid_constant__ dfx_bound_box_attribs A,
                                                                uint32_t options, View<const float> depth, char* color, int color_pitch, int color16,
                                                                char* motion, int motion_pitch, int motion16, int y0, int y1)
{
    __shared__ BoxLine lines[12];
    const bool         mv_on = (options & DFX_BOUND_BOX_OPTION_COMPUTE_MOTION_VECTORS) != 0;
    const bool         rev   = (options & DFX_BOUND_BOX_OPTION_USE_REVERSE_DEPTH) != 0;
    if (threadIdx.x < 12) setup_line(int(threadIdx.x), cams, A, mv_on, float(depth.w), float(depth.h), lines[threadIdx.x]);
    __syncthreads();

    const int      l = int(blockIdx.y);
    const BoxLine& L = lines[l];
    if (!L.ok) return;
    // the line's major-axis steps that can draw inside the scissor (the viewport's columns, or the row range)
    const int a = L.xmajor ? L.ax : L.ay, b = L.xmajor ? L.bx : L.by;
    const int lo = max((min(a, b) - 256) >> 8, L.xmajor ? 0 : y0), hi = min((max(a, b) + 256) >> 8, L.xmajor ? depth.w - 1 : y1 - 1);
    const int i  = lo + int(blockIdx.x) * kBoxThreads + int(threadIdx.x);
    if (i > hi) return;
    int j;
    if (!(L.xmajor ? step_pixel(L.ax, L.ay, L.bx, L.by, i, j) : step_pixel(L.ay, L.ax, L.by, L.bx, i, j))) return;
    const int x = L.xmajor ? i : j, y = L.xmajor ? j : i;
    if (x < 0 || x >= depth.w || y < y0 || y >= y1) return;
    const float d = depth.ld(x, y);
    float2      mv, unused;
    if (!survives(L, x, y, cams, A, rev, d, mv)) return;
    for (int m = l + 1; m < 12; ++m)
        if (covers(lines[m], x, y) && survives(lines[m], x, y, cams, A, rev, d, unused)) return; // a later line's fragment wins

    char* const crow = color + size_t(y) * size_t(color_pitch) + size_t(x) * (color16 ? 8u : 16u);
    if (color16)
    {
        const __half2 c0 = __floats2half2_rn(A.Color[0], A.Color[1]), c1 = __floats2half2_rn(A.Color[2], A.Color[3]);
        uint2         u;
        u.x = *reinterpret_cast<const uint32_t*>(&c0), u.y = *reinterpret_cast<const uint32_t*>(&c1);
        *reinterpret_cast<uint2*>(crow) = u;
    }
    else
        *reinterpret_cast<float4*>(crow) = make_float4(A.Color[0], A.Color[1], A.Color[2], A.Color[3]);
    if (mv_on)
    {
        char* const mrow = motion + size_t(y) * size_t(motion_pitch) + size_t(x) * (motion16 ? 4u : 8u);
        if (motion16)
        {
            const __half2 h = __floats2half2_rn(mv.x, mv.y);
            *reinterpret_cast<uint32_t*>(mrow) = *reinterpret_cast<const uint32_t*>(&h);
        }
        else
            *reinterpret_cast<float2*>(mrow) = mv;
    }
}
} // namespace

dfx_status bound_box_check(const dfx_bound_box_attribs* attribs)
{
    DFX_REQUIRE(attribs, "null argument");
    const float pl = attribs->PatternLength;
    if (!(pl > 0.0f && pl <= kFltMax)) return set_error(DFX_ERR_INVALID_ARG, "PatternLength %g: must be finite and > 0", double(pl));
    return DFX_OK;
}

} // namespace dfx

using namespace dfx;

extern "C" void dfx_bound_box_attribs_default(dfx_bound_box_attribs* a)
{
    // BoundBoxRenderer::RenderAttribs: a null Color is white, PatternLength 32, PatternMask 0xFFFFFFFF (BoundBoxRenderer.hpp)
    if (!a) return;
    *a = dfx_bound_box_attribs{};
    for (int k = 0; k < 4; ++k) a->Transform.m[k][k] = 1.0f, a->Color[k] = 1.0f;
    a->PatternLength = 32.0f, a->PatternMask = 0xFFFFFFFFu;
}

extern "C" dfx_status dfx_pass_bound_box(void* stream, const dfx_camera_attribs* cameras_dev, const dfx_bound_box_attribs* attribs, uint32_t options,
                                         const dfx_plane* depth_, const dfx_plane* color_inout, const dfx_plane* motion_inout, dfx_rows rows)
{
    DFX_PROFILE(stream, "bound_box");
    DFX_REQUIRE(cameras_dev, "null argument");
    dfx_status st = bound_box_check(attribs);
    if (st != DFX_OK) return st;
    if (options & ~DFX_BOUND_BOX_OPTION_ALL) return set_error(DFX_ERR_UNSUPPORTED, "unknown bound box options 0x%x", options);
    DFX_VIEW(const float, depth, depth_, DFX_FORMAT_R32F);
    char* color  = nullptr;
    char* motion = nullptr;
    int   cpitch = 0, c16 = 0, mpitch = 0, m16 = 0;
    DFX_REQUIRE(writable(color_inout, DFX_FORMAT_RGBA32F, DFX_FORMAT_RGBA16F, 16, 8, color, cpitch, c16),
                "bad plane 'color_inout' (RGBA32F or RGBA16F expected; null, pitch or alignment)");
    DFX_REQUIRE(color_inout->width == depth.w && color_inout->height == depth.h, "plane size mismatch: depth vs color_inout");
    if (options & DFX_BOUND_BOX_OPTION_COMPUTE_MOTION_VECTORS)
    {
        DFX_REQUIRE(motion_inout, "motion vectors are on: the motion plane must be given");
        DFX_REQUIRE(writable(motion_inout, DFX_FORMAT_RG32F, DFX_FORMAT_RG16F, 8, 4, motion, mpitch, m16),
                    "bad plane 'motion_inout' (RG32F or RG16F expected; null, pitch or alignment)");
        DFX_REQUIRE(motion_inout->width == depth.w && motion_inout->height == depth.h, "plane size mismatch: depth vs motion_inout");
    }
    DFX_REQUIRE(rows_ok(rows, depth.h), "bad row range");
    if (rows.y1 == rows.y0) return DFX_OK;
    // one thread per major-axis step: at most the viewport's width (x-major) or the row range's height (y-major) per line
    const dim3 grid(div_up(std::max(depth.w, rows.y1 - rows.y0), kBoxThreads), 12);
    bound_box_kernel<<<grid, kBoxThreads, 0, as_stream(stream)>>>(cameras_dev, *attribs, options, depth, color, cpitch, c16, motion, mpitch, m16, rows.y0,
                                                                  rows.y1);
    DFX_LAUNCHED("bound_box_kernel");
    return DFX_OK;
}
