// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_math.h). Pinned against the reference's own BoundBox.vsh / BoundBox.psh (oracle/refshader/
// build_bound_box_ref.py, tests/test_bound_box_reference.py). Built on its own into oracle/_build/liboracle_bound_box.so by
// oracle/oracle_bound_box_py.py.
//
// B, the selected prim's bounding box: the pipeline state of BoundBoxRenderer::GetPSO (Components/src/BoundBoxRenderer.cpp:150-168:
// LINE_LIST, depth test LESS_EQUAL or GREATER_EQUAL, no depth writes, no blending) around BoundBoxVS (BoundBox.vsh) and
// GetBoundBoxOutput (BoundBox.psh:27-48). The 24 vertices make 12 lines, rasterised by the aliased-line rule of DESIGN.md §2 (near / far
// clipping, 16.8 snapping, diamond exit, attributes at the pixel centre's projection onto the snapped segment) in primitive order:
// every surviving fragment is stored, so a pixel keeps the last line's.
#include "oracle.h"

#include <cstdint>

namespace orc
{
namespace
{
// ---- the rasteriser rule of DESIGN.md §2 -------------------------------------------------------------------------------------------

struct Vtx
{
    float a[12]; // CLIP_POS (= SV_Position) xyzw, PREV_CLIP_POS xyzw, EDGE_START_CLIP_POS xyzw
};

struct Line
{
    bool    ok = false;         // something of it is left after clipping and inside the guard band
    int64_t ax, ay, bx, by;     // the snapped endpoints, 1/256 pixel, start A = the line's first vertex
    bool    xmajor;
    float   nz0, nz1, iw0, iw1; // z / w and 1 / w at the clipped endpoints
    Vtx     v0, v1;             // the clipped endpoints' attributes
};

constexpr float kGuard = 268435456.0f; // 2^28 = 2^20 pixels in 1/256 units

// [near, far] clipping in clip space: d = z (0 <= z), then d = w - z (z <= w); a NaN distance is outside
bool clip(Vtx& v0, Vtx& v1)
{
    for (int plane = 0; plane < 2; ++plane)
    {
        const float d0 = plane == 0 ? v0.a[2] : v0.a[3] - v0.a[2];
        const float d1 = plane == 0 ? v1.a[2] : v1.a[3] - v1.a[2];
        const bool  in0 = d0 >= 0.0f, in1 = d1 >= 0.0f;
        if (!in0 && !in1) return false;
        if (!in0)
        {
            const float t = d0 / (d0 - d1);
            for (int k = 0; k < 12; ++k) v0.a[k] = v0.a[k] + (v1.a[k] - v0.a[k]) * t;
        }
        else if (!in1)
        {
            const float t = d1 / (d1 - d0);
            for (int k = 0; k < 12; ++k) v1.a[k] = v1.a[k] + (v0.a[k] - v1.a[k]) * t;
        }
    }
    return true;
}

// the viewport transform (y down) and the 16.8 snap; false beyond the guard band, at w <= 0 or on NaN
bool snap(const Vtx& v, float W, float H, int64_t& X, int64_t& Y, float& nz, float& iw)
{
    if (!(v.a[3] > 0.0f)) return false;
    const float nx = v.a[0] / v.a[3], ny = v.a[1] / v.a[3];
    nz = v.a[2] / v.a[3], iw = 1.0f / v.a[3];
    const float sx = ((nx * 0.5f) + 0.5f) * W * 256.0f, sy = (0.5f - (ny * 0.5f)) * H * 256.0f;
    if (!(std::fabs(sx) < kGuard) || !(std::fabs(sy) < kGuard)) return false;
    X = int64_t(std::nearbyint(sx)), Y = int64_t(std::nearbyint(sy)); // round half to even (the default rounding mode)
    return true;
}

Line setup(Vtx v0, Vtx v1, int W, int H)
{
    Line L;
    if (!clip(v0, v1)) return L;
    if (!snap(v0, float(W), float(H), L.ax, L.ay, L.nz0, L.iw0) || !snap(v1, float(W), float(H), L.bx, L.by, L.nz1, L.iw1)) return L;
    L.ok     = true;
    L.xmajor = std::llabs(L.bx - L.ax) >= std::llabs(L.by - L.ay);
    L.v0 = v0, L.v1 = v1;
    return L;
}

int64_t floor_div(int64_t a, int64_t b) { return a / b - ((a % b != 0) && ((a < 0) != (b < 0))); } // b > 0

// the half-open diamond of the pixel centred at (cu, cv): |du| + |dv| < 1/2, plus the right and bottom corners and the edge between them
bool in_diamond(int64_t pu, int64_t pv, int64_t cu, int64_t cv)
{
    const int64_t du = pu - cu, dv = pv - cv, s = std::llabs(du) + std::llabs(dv);
    return s < 128 || (s == 128 && du >= 0 && dv >= 0);
}

// major-axis step i of a line, in the frame where the major axis is u: the minor pixel j it draws there, or false
bool step_pixel(int64_t au, int64_t av, int64_t bu, int64_t bv, int64_t i, int64_t& j)
{
    const int64_t cu = 256 * i + 128;
    if (au != bu && std::min(au, bu) <= cu && cu <= std::max(au, bu))
    {
        // the crossing with the diamonds' minor diagonals: v(cu) in (cv - 1/2, cv + 1/2]
        int64_t num = av * (bu - au) + (cu - au) * (bv - av), den = bu - au;
        if (den < 0) num = -num, den = -den;
        j = floor_div(num - 1, 256 * den);
    }
    else
    {
        j = floor_div(av - 1, 256); // the start's diamond, if it lies in one
        if (!in_diamond(au, av, cu, 256 * j + 128)) return false;
    }
    return !in_diamond(bu, bv, cu, 256 * j + 128); // the last-pixel rule: the segment must leave the diamond
}

// the major-axis steps of a line, unclamped
void step_range(const Line& L, int64_t& lo, int64_t& hi)
{
    const int64_t a = L.xmajor ? L.ax : L.ay, b = L.xmajor ? L.bx : L.by;
    lo = floor_div(std::min(a, b) - 256, 256), hi = floor_div(std::max(a, b) + 256, 256);
}

// does line L draw pixel (x, y)?
bool covers(const Line& L, int x, int y)
{
    if (!L.ok) return false;
    int64_t j;
    if (L.xmajor) return step_pixel(L.ax, L.ay, L.bx, L.by, x, j) && j == y;
    return step_pixel(L.ay, L.ax, L.by, L.bx, y, j) && j == x;
}

// the fragment of L at pixel (x, y): depth z / w and the interpolated attributes
void interpolate(const Line& L, int x, int y, float& depth, float* attr)
{
    const int64_t cx = 256 * int64_t(x) + 128, cy = 256 * int64_t(y) + 128, dx = L.bx - L.ax, dy = L.by - L.ay;
    const int64_t num = (cx - L.ax) * dx + (cy - L.ay) * dy, den = dx * dx + dy * dy;
    float         t   = float(num) / float(den);
    t                 = std::fmin(std::fmax(t, 0.0f), 1.0f);
    depth             = L.nz0 + (L.nz1 - L.nz0) * t;
    const float tp    = (t * L.iw1) / ((1.0f - t) * L.iw0 + t * L.iw1);
    for (int k = 0; k < 12; ++k) attr[k] = L.v0.a[k] + (L.v1.a[k] - L.v0.a[k]) * tp;
}

// ---- BoundBox.vsh / BoundBox.psh ----------------------------------------------------------------------------------------------------

float4 mul_row(float4 v, const dfx_float4x4& M)
{
    float r[4];
    for (int c = 0; c < 4; ++c) r[c] = M.m[0][c] * v.x + M.m[1][c] * v.y + M.m[2][c] * v.z + M.m[3][c] * v.w;
    return float4(r[0], r[1], r[2], r[3]);
}

// GetBoxCorner (BoundBox.vsh:14-55)
float4 box_corner(uint id, const dfx_bound_box_attribs& A)
{
    if (id < 8u)
        id = ((id + 1u) >> 1u) & 3u;
    else if (id < 16u)
        id = 4u + (((id + 1u) >> 1u) & 3u);
    else
        id = ((id - 16u) >> 1u) + (id & 1u) * 4u;
    const float4 c((id & 2u) ? 1.0f : 0.0f, ((id + 1u) & 2u) ? 1.0f : 0.0f, (id & 4u) ? 1.0f : 0.0f, 1.0f);
    return mul_row(c, A.Transform);
}

Vtx vs(uint id, const dfx_camera_attribs* cams, const dfx_bound_box_attribs& A, bool motion)
{
    const float4 corner = box_corner(id, A), start = box_corner(id & ~1u, A);
    const float4 p = mul_row(corner, cams[0].mViewProj), e = mul_row(start, cams[0].mViewProj);
    const float4 q = motion ? mul_row(corner, cams[1].mViewProj) : p; // BoundBox.vsh:65-69
    Vtx          v;
    const float4 s[3] = {p, q, e};
    for (int k = 0; k < 3; ++k) v.a[4 * k] = s[k].x, v.a[4 * k + 1] = s[k].y, v.a[4 * k + 2] = s[k].z, v.a[4 * k + 3] = s[k].w;
    return v;
}

uint ftou(float v) { return !(v > 0.0f) ? 0u : v >= 4294967296.0f ? 0xFFFFFFFFu : uint(v); } // D3D ftou: NaN -> 0, saturating

// GetBoundBoxOutput (BoundBox.psh:27-48): false = discarded
bool ps(const float* a, const dfx_camera_attribs* cams, const dfx_bound_box_attribs& A, float2& mv)
{
    const dfx_camera_attribs& C = cams[0];
    const float cx = a[0] / a[3], cy = a[1] / a[3], ex = a[8] / a[11], ey = a[9] / a[11];
    const float vx = (cx - ex) * C.f4ViewportSize[0], vy = (cy - ey) * C.f4ViewportSize[1];
    const float dist = std::sqrt(vx * vx + vy * vy);
    const float q    = dist / A.PatternLength;
    const float pos  = q - std::floor(q);
    const uint  bit  = std::min(ftou(pos * A.PatternLength), 31u);
    if ((A.PatternMask & (1u << bit)) == 0u) return false;
    const dfx_camera_attribs& P = cams[1];
    const float               px = a[4] / a[7], py = a[5] / a[7];
    mv = float2((cx - C.f2Jitter[0]) - (px - P.f2Jitter[0]), (cy - C.f2Jitter[1]) - (py - P.f2Jitter[1])); // GetMotionVector
    return true;
}

void setup_lines(const dfx_camera_attribs* cams, const dfx_bound_box_attribs& A, uint options, int W, int H, Line* L)
{
    const bool motion = (options & DFX_BOUND_BOX_OPTION_COMPUTE_MOTION_VECTORS) != 0;
    for (int l = 0; l < 12; ++l) L[l] = setup(vs(2 * l, cams, A, motion), vs(2 * l + 1, cams, A, motion), W, H);
}

// the fragment of line l at (x, y) passes the depth test and is not discarded
bool survives(const Line& L, int x, int y, const dfx_camera_attribs* cams, const dfx_bound_box_attribs& A, uint options, float d, float2& mv)
{
    float z, attr[12];
    interpolate(L, x, y, z, attr);
    if (!((options & DFX_BOUND_BOX_OPTION_USE_REVERSE_DEPTH) ? z >= d : z <= d)) return false;
    return ps(attr, cams, A, mv);
}

void bound_box(const dfx_camera_attribs* cams, uint options, const dfx_bound_box_attribs& A, const float* depth, float* color, float* motion, int W, int H,
               int y0, int y1)
{
    Line L[12];
    setup_lines(cams, A, options, W, H, L);
    // primitive order: each line stores its surviving fragments over what the lines before it stored
    for (int l = 0; l < 12; ++l)
    {
        if (!L[l].ok) continue;
        int64_t lo, hi;
        step_range(L[l], lo, hi);
        for (int64_t i = lo; i <= hi; ++i)
        {
            int64_t j;
            const bool drawn = L[l].xmajor ? step_pixel(L[l].ax, L[l].ay, L[l].bx, L[l].by, i, j) : step_pixel(L[l].ay, L[l].ax, L[l].by, L[l].bx, i, j);
            if (!drawn) continue;
            const int64_t x = L[l].xmajor ? i : j, y = L[l].xmajor ? j : i;
            if (x < 0 || x >= W || y < y0 || y >= y1 || y >= H) continue; // the viewport and the row range are the scissor
            const size_t k = size_t(y) * size_t(W) + size_t(x);
            float2       mv;
            if (!survives(L[l], int(x), int(y), cams, A, options, depth[k], mv)) continue;
            for (int c = 0; c < 4; ++c) color[k * 4 + c] = A.Color[c];
            if (options & DFX_BOUND_BOX_OPTION_COMPUTE_MOTION_VECTORS) motion[k * 2] = mv.x, motion[k * 2 + 1] = mv.y;
        }
    }
}

} // namespace
} // namespace orc

// C API (ctypes, oracle/oracle_bound_box_py.py). Planes are tightly packed fp32: depth w*h, colour w*h*4, motion w*h*2.
extern "C"
{
#define ORCB_API __attribute__((visibility("default")))
ORCB_API void orcb_bound_box(const dfx_camera_attribs* cams, uint32_t options, const dfx_bound_box_attribs* attribs, const float* depth, float* color_inout,
                             float* motion_inout, int w, int h, int y0, int y1)
{
    orc::bound_box(cams, options, *attribs, depth, color_inout, motion_inout, w, h, y0, y1);
}

// The bare rasteriser on one segment given by its two clip-space positions (the attributes are the positions): the pixels it draws
// in a w x h viewport in major-axis order (xy_out pairs, at most max_out), each with its t and interpolated z / w. Returns the count,
// or -1 when nothing is left of it after clipping and the guard band.
ORCB_API int orcb_raster(const float* p0, const float* p1, int w, int h, int* xy_out, float* t_out, float* z_out, int max_out)
{
    orc::Vtx v0{}, v1{};
    for (int k = 0; k < 4; ++k) v0.a[k] = v0.a[4 + k] = v0.a[8 + k] = p0[k], v1.a[k] = v1.a[4 + k] = v1.a[8 + k] = p1[k];
    const orc::Line L = orc::setup(v0, v1, w, h);
    if (!L.ok) return -1;
    int64_t lo, hi;
    orc::step_range(L, lo, hi);
    int n = 0;
    for (int64_t i = lo; i <= hi; ++i)
    {
        int64_t j;
        if (!(L.xmajor ? orc::step_pixel(L.ax, L.ay, L.bx, L.by, i, j) : orc::step_pixel(L.ay, L.ax, L.by, L.bx, i, j))) continue;
        const int64_t x = L.xmajor ? i : j, y = L.xmajor ? j : i;
        if (x < 0 || x >= w || y < 0 || y >= h || n >= max_out) continue;
        float z, attr[12];
        orc::interpolate(L, int(x), int(y), z, attr);
        const int64_t cx = 256 * x + 128, cy = 256 * y + 128, dx = L.bx - L.ax, dy = L.by - L.ay;
        const float   t  = std::fmin(std::fmax(float((cx - L.ax) * dx + (cy - L.ay) * dy) / float(dx * dx + dy * dy), 0.0f), 1.0f);
        xy_out[2 * n] = int(x), xy_out[2 * n + 1] = int(y), t_out[n] = t, z_out[n] = z;
        ++n;
    }
    return n;
}

// The same rule on snapped endpoints given directly (1/256 pixel), unbounded viewport: the pixels drawn in major-axis order.
ORCB_API int orcb_raster_fixed(int64_t ax, int64_t ay, int64_t bx, int64_t by, int* xy_out, int max_out)
{
    orc::Line L;
    L.ok = true, L.ax = ax, L.ay = ay, L.bx = bx, L.by = by, L.xmajor = std::llabs(bx - ax) >= std::llabs(by - ay);
    int64_t lo, hi;
    orc::step_range(L, lo, hi);
    int n = 0;
    for (int64_t i = lo; i <= hi && n < max_out; ++i)
    {
        int64_t j;
        if (!(L.xmajor ? orc::step_pixel(ax, ay, bx, by, i, j) : orc::step_pixel(ay, ax, by, bx, i, j))) continue;
        xy_out[2 * n] = int(L.xmajor ? i : j), xy_out[2 * n + 1] = int(L.xmajor ? j : i);
        ++n;
    }
    return n;
}

// The near / far clip of one segment of clip-space positions; false when nothing is left.
ORCB_API int orcb_clip(const float* p0, const float* p1, float* q0, float* q1)
{
    orc::Vtx v0{}, v1{};
    for (int k = 0; k < 4; ++k) v0.a[k] = p0[k], v1.a[k] = p1[k];
    if (!orc::clip(v0, v1)) return 0;
    for (int k = 0; k < 4; ++k) q0[k] = v0.a[k], q1[k] = v1.a[k];
    return 1;
}

// The 24 vertices of BoundBoxVS: out 24 x 12 floats (CLIP_POS, PREV_CLIP_POS, EDGE_START_CLIP_POS).
ORCB_API void orcb_vertices(const dfx_camera_attribs* cams, const dfx_bound_box_attribs* attribs, int motion, float* out)
{
    for (uint id = 0; id < 24; ++id)
    {
        const orc::Vtx v = orc::vs(id, cams, *attribs, motion != 0);
        for (int k = 0; k < 12; ++k) out[id * 12 + k] = v.a[k];
    }
}
}
