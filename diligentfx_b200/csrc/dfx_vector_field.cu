// dfx_vector_field.cu — the vector field overlay as sm_90a kernels: the pipeline state of VectorFieldRenderer::GetPSO
// (Components/src/VectorFieldRenderer.cpp:142-157: LINE_LIST, DSS_DisableDepth, no blending) around VectorField.vsh and the default PS
// main (:76-86), drawn over a colour target the way Render (:173-223) draws GridSize.x * GridSize.y * 2 vertices.
//
// Line k (k = row * gx + col) runs from the cell's centre to the centre plus the field's vector there, rasterised by the aliased-line
// rule of DESIGN.md §2 through the shared integer functions of dfx_line.cuh; every float operation of the vertex shader, the bilinear
// tap and the rule is one rounding (mul_ / add_ / sub_ / div_, never contracted), so the covered pixels and the stored colours are the
// oracle's bit for bit. A pixel keeps the fragment of the last line in primitive order, the highest k. That is resolved without a
// frame-sized clear and without ordering between lines, in two launches over a 32-bit owner plane that is zero on entry:
//   mark:    each fragment does atomicMax(owner[p], k + 1);
//   resolve: each fragment whose owner[p] is k + 1 stores its colour and writes 0 back.
// A line draws a pixel at most once (one pixel per major-axis step), and a lower line reads k + 1 or 0 at p, never its own k' + 1, so
// exactly the owner stores, and the plane is zero again afterwards. One warp per line, its lanes striding over the major-axis steps.
#include "dfx_line.cuh"

namespace dfx
{
namespace
{
constexpr int kFieldThreads = 256; // 8 lines per CTA; two CTAs per SM give ptxas room for the sRGB resolve without spills

struct FieldLine
{
    bool  ok, xmajor;
    int   ax, ay, bx, by; // snapped endpoints, 1/256 pixel
    float iw0, iw1;       // 1 / w at the ends (1)
};

// VectorField.vsh for line k: the two vertices' positions; the tap follows hlsl's sample_mip (Sam_LinearClamp on a one-level field)
DFX_HD void field_line(uint32_t k, const dfx_vector_field_attribs& A, const Tex2& F, float W, float H, FieldLine& L)
{
    const uint32_t gx = A.GridSize[0], col = k % gx, row = k / gx;
    const float    u = div_(add_(float(col), 0.5f), float(gx)), v = div_(add_(float(row), 0.5f), float(A.GridSize[1]));
    float          px = sub_(mul_(u, float(F.w)), 0.5f), py = sub_(mul_(v, float(F.h)), 0.5f);
    px             = mul_(floorf(add_(mul_(px, 256.0f), 0.5f)), 1.0f / 256.0f); // 8 fractional bits of the fixed-function sampler
    py             = mul_(floorf(add_(mul_(py, 256.0f), 0.5f)), 1.0f / 256.0f);
    const float fx0 = floorf(px), fy0 = floorf(py);
    const int   x0 = int(fx0), y0 = int(fy0);
    const float fx = sub_(px, fx0), fy = sub_(py, fy0), gx_ = sub_(1.0f, fx), gy_ = sub_(1.0f, fy);
    const float w00 = mul_(gx_, gy_), w10 = mul_(fx, gy_), w01 = mul_(gx_, fy), w11 = mul_(fx, fy);
    const float2 t00 = loadc(F, x0, y0), t10 = loadc(F, x0 + 1, y0), t01 = loadc(F, x0, y0 + 1), t11 = loadc(F, x0 + 1, y0 + 1);
    const float  sx = add_(add_(add_(mul_(t00.x, w00), mul_(t10.x, w10)), mul_(t01.x, w01)), mul_(t11.x, w11));
    const float  sy = add_(add_(add_(mul_(t00.y, w00), mul_(t10.y, w10)), mul_(t01.y, w01)), mul_(t11.y, w11));
    // (MotionVec + Bias) * Scale; TexUVToNormalizedDeviceXY: (UV - 0.5) / (0.5, -0.5), which is (UV - 0.5) * (2, -2) exactly
    const float mx = mul_(add_(sx, A.Bias[0]), A.Scale[0]), my = mul_(add_(sy, A.Bias[1]), A.Scale[1]);
    const float nx = mul_(sub_(u, 0.5f), 2.0f), ny = mul_(sub_(v, 0.5f), -2.0f);
    const float a0[4] = {nx, ny, 0.0f, 1.0f}, a1[4] = {add_(nx, mx), add_(ny, my), 0.0f, 1.0f};
    float       nz;
    // z = 0, w = 1: never clipped; a non-finite or far end fails the guard band and draws nothing
    L.ok = snap(a0, W, H, L.ax, L.ay, nz, L.iw0) && snap(a1, W, H, L.bx, L.by, nz, L.iw1);
    L.xmajor = abs(L.bx - L.ax) >= abs(L.by - L.ay);
}

// the default PS main's output at pixel (x, y) of L: the colour interpolated through the rule's tp, then pow(rgb, 1 / 2.2) with sRGB
DFX_HD float4 fragment_color(const FieldLine& L, int x, int y, const dfx_vector_field_attribs& A, bool srgb)
{
    const long long cx = 256ll * x + 128, cy = 256ll * y + 128, dx = (long long)L.bx - L.ax, dy = (long long)L.by - L.ay;
    const long long num = (cx - L.ax) * dx + (cy - L.ay) * dy, den = dx * dx + dy * dy;
    const float     t   = fminf(fmaxf(div_(float(num), float(den)), 0.0f), 1.0f);
    const float     tp  = div_(mul_(t, L.iw1), add_(mul_(sub_(1.0f, t), L.iw0), mul_(t, L.iw1)));
    float           c[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) c[i] = add_(A.StartColor[i], mul_(sub_(A.EndColor[i], A.StartColor[i]), tp));
    if (srgb)
    {
        // dfx_env_map.cu's pow(c, 1 / 2.2): exp2(e * log2(c)) in double with the shader's fp32 exponent, rounded once
        const double e = double(div_(1.0f, 2.2f));
#pragma unroll
        for (int i = 0; i < 3; ++i) c[i] = float(exp2(e * log2(double(c[i]))));
    }
    return make_float4(c[0], c[1], c[2], c[3]);
}

// PASS 0 marks owners, PASS 1 stores the owners' colours and clears the marks (SRGB: pow(rgb, 1 / 2.2) before the store)
template <int PASS, bool C16, bool SRGB>
__global__ void __launch_bounds__(kFieldThreads, 2) vector_field_kernel(const __grid_constant__ dfx_vector_field_attribs A, Tex2 field, char* color,
                                                                      int color_pitch, uint32_t* owner, int owner_pitch, int W, int H, int y0, int y1,
                                                                      uint32_t lines)
{
    const uint32_t k = blockIdx.x * (kFieldThreads / 32) + (threadIdx.x >> 5);
    if (k >= lines) return;
    FieldLine L;
    field_line(k, A, field, float(W), float(H), L);
    if (!L.ok) return;
    // the line's major-axis steps that can draw inside the scissor (the target's columns, or the row range)
    const int a = L.xmajor ? L.ax : L.ay, b = L.xmajor ? L.bx : L.by;
    const int lo = max((min(a, b) - 256) >> 8, L.xmajor ? 0 : y0), hi = min((max(a, b) + 256) >> 8, L.xmajor ? W - 1 : y1 - 1);
    const uint32_t mark = k + 1u;
    for (int i = lo + int(threadIdx.x & 31u); i <= hi; i += 32)
    {
        int j;
        if (!(L.xmajor ? step_pixel(L.ax, L.ay, L.bx, L.by, i, j) : step_pixel(L.ay, L.ax, L.by, L.bx, i, j))) continue;
        const int x = L.xmajor ? i : j, y = L.xmajor ? j : i;
        if (x < 0 || x >= W || y < y0 || y >= y1) continue;
        uint32_t* const o = owner + size_t(y) * size_t(owner_pitch) + size_t(x);
        if constexpr (PASS == 0)
            atomicMax(o, mark);
        else
        {
            if (*o != mark) continue;
            *o = 0u;
            const float4 c   = fragment_color(L, x, y, A, SRGB);
            char* const  row = color + size_t(y) * size_t(color_pitch);
            if constexpr (C16)
            {
                const __half2 h0 = __floats2half2_rn(c.x, c.y), h1 = __floats2half2_rn(c.z, c.w);
                uint2         u;
                u.x = *reinterpret_cast<const uint32_t*>(&h0), u.y = *reinterpret_cast<const uint32_t*>(&h1);
                reinterpret_cast<uint2*>(row)[x] = u;
            }
            else
                reinterpret_cast<float4*>(row)[x] = c;
        }
    }
}

template <bool C16>
dfx_status launch_field(cudaStream_t s, const dfx_vector_field_attribs& A, const Tex2& F, char* color, int cpitch, uint32_t* owner, int opitch, int W, int H,
                        dfx_rows rows, uint32_t lines, int srgb)
{
    const unsigned grid = unsigned((uint64_t(lines) + kFieldThreads / 32 - 1) / (kFieldThreads / 32));
    vector_field_kernel<0, false, false><<<grid, kFieldThreads, 0, s>>>(A, F, color, cpitch, owner, opitch, W, H, rows.y0, rows.y1, lines);
    DFX_LAUNCHED("vector_field_kernel<mark>");
    if (srgb)
        vector_field_kernel<1, C16, true><<<grid, kFieldThreads, 0, s>>>(A, F, color, cpitch, owner, opitch, W, H, rows.y0, rows.y1, lines);
    else
        vector_field_kernel<1, C16, false><<<grid, kFieldThreads, 0, s>>>(A, F, color, cpitch, owner, opitch, W, H, rows.y0, rows.y1, lines);
    DFX_LAUNCHED("vector_field_kernel<resolve>");
    return DFX_OK;
}
} // namespace
} // namespace dfx

using namespace dfx;

extern "C" void dfx_vector_field_attribs_default(dfx_vector_field_attribs* a)
{
    // VectorFieldRenderer::RenderAttribs (VectorFieldRenderer.hpp): Bias 0, Scale 1, both colours 1, GridSize 0
    if (!a) return;
    *a = dfx_vector_field_attribs{};
    for (int k = 0; k < 2; ++k) a->Scale[k] = 1.0f;
    for (int k = 0; k < 4; ++k) a->StartColor[k] = a->EndColor[k] = 1.0f;
}

extern "C" void dfx_vector_field_attribs_hydrogent(uint32_t width, uint32_t height, float elapsed_time, dfx_vector_field_attribs* a)
{
    // HnPostProcessTask.cpp:932-938: a vector per 20 x 20 pixels, drawn against the motion (-0.02 / max(ElapsedTime, 0.001)), from white to
    // grey; std::max keeps its first operand when the second is not greater, so a NaN elapsed time stays NaN (the chain refuses it)
    if (!a) return;
    dfx_vector_field_attribs_default(a);
    a->GridSize[0] = width / 20u, a->GridSize[1] = height / 20u;
    const float t = elapsed_time < 0.001f ? 0.001f : elapsed_time;
    a->Scale[0] = a->Scale[1] = -0.02f / t;
    for (int k = 0; k < 3; ++k) a->EndColor[k] = 0.5f;
}

extern "C" dfx_status dfx_pass_vector_field(void* stream, const dfx_vector_field_attribs* attribs, uint32_t options, const dfx_plane* vector_field,
                                            const dfx_plane* color_inout, const dfx_plane* scratch, dfx_rows rows)
{
    DFX_PROFILE(stream, "vector_field");
    DFX_REQUIRE(attribs, "null argument");
    if (options & ~DFX_VECTOR_FIELD_OPTION_ALL) return set_error(DFX_ERR_UNSUPPORTED, "unknown vector field options 0x%x", options);
    DFX_TEX2(field, vector_field);
    char* color  = nullptr;
    int   cpitch = 0, c16 = 0;
    DFX_REQUIRE(writable(color_inout, DFX_FORMAT_RGBA32F, DFX_FORMAT_RGBA16F, 16, 8, color, cpitch, c16),
                "bad plane 'color_inout' (RGBA32F or RGBA16F expected; null, pitch or alignment)");
    DFX_VIEW(float, owner, scratch, DFX_FORMAT_R32F);
    DFX_REQUIRE(owner.w == color_inout->width && owner.h == color_inout->height, "plane size mismatch: scratch vs color_inout");
    const uint64_t lines = uint64_t(attribs->GridSize[0]) * uint64_t(attribs->GridSize[1]);
    DFX_REQUIRE(2u * lines <= 0xFFFFFFFFull, "GridSize %u x %u: the draw's vertex count 2 * %llu does not fit in 32 bits", attribs->GridSize[0],
                attribs->GridSize[1], (unsigned long long)lines);
    DFX_REQUIRE(rows_ok(rows, owner.h), "bad row range");
    if (lines == 0 || rows.y1 == rows.y0) return DFX_OK; // VectorFieldRenderer.cpp:181-182: GridSize 0 in either axis draws nothing
    const int srgb = (options & DFX_VECTOR_FIELD_OPTION_CONVERT_OUTPUT_TO_SRGB) ? 1 : 0;
    uint32_t* const o = reinterpret_cast<uint32_t*>(owner.p);
    DFX_FMT16(c16, C16,
              return launch_field<C16>(as_stream(stream), *attribs, field, color, cpitch, o, owner.pitch, owner.w, owner.h, rows, uint32_t(lines), srgb));
}
