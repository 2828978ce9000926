// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_math.h). Pinned against the reference's own VectorField.vsh and VectorFieldRenderer's
// default PS main (oracle/refshader/build_vector_field_ref.py, tests/test_vector_field_reference.py). Built on its own into
// oracle/_build/liboracle_vector_field.so by oracle/oracle_vector_field_py.py.
//
// The vector field overlay: the pipeline state of VectorFieldRenderer::GetPSO (Components/src/VectorFieldRenderer.cpp:142-157:
// LINE_LIST, DSS_DisableDepth, no blending) around VectorField.vsh and DefaultPSMain (:76-86), as Render (:173-223) draws it:
// GridSize.x * GridSize.y lines in primitive order, each rasterised by the aliased-line rule of DESIGN.md §2 (never clipped at z = 0,
// w = 1; the 16.8 snap and its guard band; diamond exit; the colour at the pixel centre's projection onto the snapped segment) and
// stored over whatever is there, so a pixel keeps the last line's fragment.
#include "oracle.h"

#include <cstdint>

namespace orc
{
namespace
{
// ---- the rasteriser rule of DESIGN.md §2 on a line with z = 0, w = 1 at both ends --------------------------------------------------

constexpr float kGuard = 268435456.0f; // 2^28 = 2^20 pixels in 1/256 units

struct Line
{
    bool    ok = false;
    int64_t ax, ay, bx, by; // the snapped endpoints, 1/256 pixel
    bool    xmajor;
    float   iw0, iw1;       // 1 / w at the ends
};

// the viewport transform (y down) and the 16.8 snap; false beyond the guard band, at w <= 0 or on NaN
bool snap(const float* a, float W, float H, int64_t& X, int64_t& Y, float& iw)
{
    if (!(a[3] > 0.0f)) return false;
    const float nx = a[0] / a[3], ny = a[1] / a[3];
    iw = 1.0f / a[3];
    const float sx = ((nx * 0.5f) + 0.5f) * W * 256.0f, sy = (0.5f - (ny * 0.5f)) * H * 256.0f;
    if (!(std::fabs(sx) < kGuard) || !(std::fabs(sy) < kGuard)) return false;
    X = int64_t(std::nearbyint(sx)), Y = int64_t(std::nearbyint(sy)); // round half to even (the default rounding mode)
    return true;
}

int64_t floor_div(int64_t a, int64_t b) { return a / b - ((a % b != 0) && ((a < 0) != (b < 0))); } // b > 0

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
        int64_t num = av * (bu - au) + (cu - au) * (bv - av), den = bu - au;
        if (den < 0) num = -num, den = -den;
        j = floor_div(num - 1, 256 * den);
    }
    else
    {
        j = floor_div(av - 1, 256);
        if (!in_diamond(au, av, cu, 256 * j + 128)) return false;
    }
    return !in_diamond(bu, bv, cu, 256 * j + 128);
}

// ---- VectorField.vsh ----------------------------------------------------------------------------------------------------------------

// SampleLevel(Sam_LinearClamp, uv, 0) of a one-level RG field (fw x fh texels): the 1/256 snap of §2, clamped taps, hlsl's sample_mip order
void sample(const float* field, int fw, int fh, float u, float v, float& sx, float& sy)
{
    float px = u * float(fw) - 0.5f, py = v * float(fh) - 0.5f;
    px = std::floor(px * 256.0f + 0.5f) * (1.0f / 256.0f);
    py = std::floor(py * 256.0f + 0.5f) * (1.0f / 256.0f);
    const float fx0 = std::floor(px), fy0 = std::floor(py);
    const int   x0 = int(fx0), y0 = int(fy0);
    const float fx = px - fx0, fy = py - fy0;
    const auto  tap = [&](int x, int y, int c) {
        x = std::min(std::max(x, 0), fw - 1), y = std::min(std::max(y, 0), fh - 1);
        return field[(size_t(y) * size_t(fw) + size_t(x)) * 2 + size_t(c)];
    };
    const float w00 = (1.0f - fx) * (1.0f - fy), w10 = fx * (1.0f - fy), w01 = (1.0f - fx) * fy, w11 = fx * fy;
    sx = tap(x0, y0, 0) * w00 + tap(x0 + 1, y0, 0) * w10 + tap(x0, y0 + 1, 0) * w01 + tap(x0 + 1, y0 + 1, 0) * w11;
    sy = tap(x0, y0, 1) * w00 + tap(x0 + 1, y0, 1) * w10 + tap(x0, y0 + 1, 1) * w01 + tap(x0 + 1, y0 + 1, 1) * w11;
}

// the two vertices of line k: Pos (x, y, 0, 1) each
void vertices(uint64_t k, const dfx_vector_field_attribs& A, const float* field, int fw, int fh, float* p0, float* p1)
{
    const uint32_t col = uint32_t(k % A.GridSize[0]), row = uint32_t(k / A.GridSize[0]);
    const float    u = (float(col) + 0.5f) / float(A.GridSize[0]), v = (float(row) + 0.5f) / float(A.GridSize[1]);
    float          sx, sy;
    sample(field, fw, fh, u, v, sx, sy);
    const float mx = (sx + A.Bias[0]) * A.Scale[0], my = (sy + A.Bias[1]) * A.Scale[1];
    const float nx = (u - 0.5f) / 0.5f, ny = (v - 0.5f) / -0.5f; // TexUVToNormalizedDeviceXY
    p0[0] = nx, p0[1] = ny, p0[2] = 0.0f, p0[3] = 1.0f;
    p1[0] = nx + mx, p1[1] = ny + my, p1[2] = 0.0f, p1[3] = 1.0f;
}

Line setup(const float* p0, const float* p1, int W, int H)
{
    Line L;
    if (!snap(p0, float(W), float(H), L.ax, L.ay, L.iw0) || !snap(p1, float(W), float(H), L.bx, L.by, L.iw1)) return L; // z = 0, w = 1: never clipped
    L.ok     = true;
    L.xmajor = std::llabs(L.bx - L.ax) >= std::llabs(L.by - L.ay);
    return L;
}

// DefaultPSMain (VectorFieldRenderer.cpp:76-86) on the colour interpolated at pixel (x, y)
void fragment(const Line& L, int64_t x, int64_t y, const dfx_vector_field_attribs& A, bool srgb, float* out)
{
    const int64_t cx = 256 * x + 128, cy = 256 * y + 128, dx = L.bx - L.ax, dy = L.by - L.ay;
    float         t  = float((cx - L.ax) * dx + (cy - L.ay) * dy) / float(dx * dx + dy * dy);
    t                = std::fmin(std::fmax(t, 0.0f), 1.0f);
    const float tp   = (t * L.iw1) / ((1.0f - t) * L.iw0 + t * L.iw1);
    for (int c = 0; c < 4; ++c) out[c] = A.StartColor[c] + (A.EndColor[c] - A.StartColor[c]) * tp;
    if (srgb)
        for (int c = 0; c < 3; ++c) out[c] = std::pow(out[c], 1.0f / 2.2f);
}

// returns the number of fragments drawn (pixels stored, counted once per line that covers them)
uint64_t vector_field(const dfx_vector_field_attribs& A, uint32_t options, const float* field, int fw, int fh, float* color, int W, int H, int y0, int y1)
{
    uint64_t       fragments = 0;
    const uint64_t lines = uint64_t(A.GridSize[0]) * uint64_t(A.GridSize[1]);
    const bool     srgb  = (options & DFX_VECTOR_FIELD_OPTION_CONVERT_OUTPUT_TO_SRGB) != 0;
    for (uint64_t k = 0; k < lines; ++k)
    {
        float p0[4], p1[4];
        vertices(k, A, field, fw, fh, p0, p1);
        const Line L = setup(p0, p1, W, H);
        if (!L.ok) continue;
        const int64_t a = L.xmajor ? L.ax : L.ay, b = L.xmajor ? L.bx : L.by;
        for (int64_t i = floor_div(std::min(a, b) - 256, 256); i <= floor_div(std::max(a, b) + 256, 256); ++i)
        {
            int64_t j;
            if (!(L.xmajor ? step_pixel(L.ax, L.ay, L.bx, L.by, i, j) : step_pixel(L.ay, L.ax, L.by, L.bx, i, j))) continue;
            const int64_t x = L.xmajor ? i : j, y = L.xmajor ? j : i;
            if (x < 0 || x >= W || y < y0 || y >= y1 || y >= H) continue; // the viewport and the row range are the scissor
            fragment(L, x, y, A, srgb, color + (size_t(y) * size_t(W) + size_t(x)) * 4);
            ++fragments;
        }
    }
    return fragments;
}

} // namespace
} // namespace orc

// C API (ctypes, oracle/oracle_vector_field_py.py). Planes are tightly packed fp32: field fw*fh*2, colour w*h*4.
extern "C"
{
#define ORCV_API __attribute__((visibility("default")))
ORCV_API uint64_t orcv_vector_field(const dfx_vector_field_attribs* attribs, uint32_t options, const float* field, int fw, int fh, float* color_inout, int w,
                                    int h, int y0, int y1)
{
    return orc::vector_field(*attribs, options, field, fw, fh, color_inout, w, h, y0, y1);
}

// The two vertex positions of lines [0, n): out n x 2 x 4 floats.
ORCV_API void orcv_vertices(const dfx_vector_field_attribs* attribs, const float* field, int fw, int fh, uint64_t n, float* out)
{
    for (uint64_t k = 0; k < n; ++k) orc::vertices(k, *attribs, field, fw, fh, out + k * 8, out + k * 8 + 4);
}
}
