// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_math.h). Pinned against the reference's own ShadowConversions.fx
// (oracle/refshader/build_shadow_ref.py, tests/test_shadow_reference.py). Built on its own into oracle/_build/liboracle_shadow.so by
// oracle/oracle_shadow_py.py.
//
// ShadowMapManager::ConvertToFilterable (Components/src/ShadowMapManager.cpp:533-600): for each cascade, VSMHorzPS or EVSMHorzPS into
// the one-slice intermediate, then VertBlurPS into the filterable slice, as the reference draws them, by the rules of DESIGN.md §2:
// scalar float arithmetic without contraction (one rounding per operation, in the shader's order); exp is the double function rounded
// once; a Load outside the texture reads 0; the intermediate and the output are stored in the filterable format (oracle_quant.h's
// UNORM and half rules) and read back from it; iFixedFilterSize == 2 writes the horizontal result straight into the filterable map.
#include "oracle_quant.h"

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>

namespace
{
enum
{
    PCF = 1,
    VSM = 2,
    EVSM2 = 3,
    EVSM4 = 4
};

// the fields of ShadowMapAttribs ConvertToFilterable reads (offsets of BasicStructures.fxh, C++ form)
struct Attribs
{
    int   num_cascades, fixed_filter_size, is32;
    float pos_exp, neg_exp, filter_world_size, scale_x[8], scale_y[8];
};
Attribs parse(const unsigned char* b)
{
    Attribs a;
    auto f = [&](size_t off) { float v; std::memcpy(&v, b + off, 4); return v; };
    auto i = [&](size_t off) { int32_t v; std::memcpy(&v, b + off, 4); return int(v); };
    for (int c = 0; c < 8; ++c) a.scale_x[c] = f(64 + 64 * c), a.scale_y[c] = f(64 + 64 * c + 4);
    a.num_cascades      = i(1136);
    a.pos_exp           = f(1176);
    a.neg_exp           = f(1180);
    a.is32              = i(1184);
    a.fixed_filter_size = i(1188);
    a.filter_world_size = f(1192);
    return a;
}

// ShadowMapManager.cpp:560-579
void radii(const Attribs& s, int i, int width, int height, float& rh, float& rv)
{
    if (s.fixed_filter_size > 0)
    {
        rh = rv = static_cast<float>((s.fixed_filter_size - 1) / 2);
        return;
    }
    const float fNDCtoUVScale = 0.5f;
    const float fFilterWidth  = s.filter_world_size * s.scale_x[i] * fNDCtoUVScale;
    const float fFilterHeight = s.filter_world_size * s.scale_y[i] * fNDCtoUVScale;
    rh = fFilterWidth / 2.f * static_cast<float>(width);
    rv = fFilterHeight / 2.f * static_cast<float>(height);
}

// GetSampleWeight (ShadowConversions.fx:23-28)
float sample_weight(int x, float r)
{
    const float lo = std::fmax(float(x), std::fmin(0.5f - r, 0.0f));
    const float hi = std::fmin(float(x) + 1.0f, std::fmax(0.5f + r, 1.0f));
    return hi - lo;
}

float exp_(float x) { return float(std::exp(double(x))); }

struct Conv
{
    int          mode, is32, d16, w, h;
    float        ex, ey;
    const void*  in;
    float depth(int x, int y) const
    {
        if (x < 0 || y < 0 || x >= w || y >= h) return 0.0f;
        const size_t k = size_t(y) * size_t(w) + size_t(x);
        return d16 ? float(static_cast<const uint16_t*>(in)[k]) / 65535.0f : static_cast<const float*>(in)[k];
    }
    // the filterable format's store, read back
    float q(float v) const
    {
        if (is32) return v;
        return mode == VSM ? orc::q_unorm(v, 16) : orc::q_half(v);
    }
};

// the horizontal pass's float4 at (x, y)
void horz(const Conv& c, float r, int x, int y, float m[4])
{
    m[0] = m[1] = m[2] = m[3] = 0.0f;
    const int range = int(std::floor(r + 0.5f));
    float     total = 0.0f;
    for (int i = -range; i <= +range; ++i)
    {
        const float wt = sample_weight(i, r);
        const float d  = c.depth(x + i, y);
        if (c.mode == VSM)
        {
            m[0] = m[0] + d * wt;
            m[1] = m[1] + (d * d) * wt;
        }
        else
        {
            // WarpDepthEVSM (Shadows.fxh:288-295)
            const float dd = 2.0f * d - 1.0f, p = exp_(c.ex * dd), n = -exp_(-c.ey * dd);
            m[0] = m[0] + p * wt;
            m[1] = m[1] + (p * p) * wt;
            m[2] = m[2] + n * wt;
            m[3] = m[3] + (n * n) * wt;
        }
        total = total + wt;
    }
    if (c.mode == VSM)
        m[0] = m[0] / total, m[1] = m[1] / total, m[2] = m[3] = 0.0f;
    else
        for (int k = 0; k < 4; ++k) m[k] = m[k] / total;
}
} // namespace

// The filter radii of cascade i of a width x height map.
extern "C" __attribute__((visibility("default"))) void ors_filter_radii(const unsigned char* attribs, int i, int width, int height, float* rh, float* rv)
{
    radii(parse(attribs), i, width, height, *rh, *rv);
}

// WarpDepthEVSM of n depths with the clamped exponents of (pos, neg, is32): out[2k], out[2k + 1].
extern "C" __attribute__((visibility("default"))) void ors_warp(const float* depth, int n, float pos, float neg, int is32, float* out)
{
    const float mx = is32 ? 42.0f : 5.54f, ex = std::fmin(pos, mx), ey = std::fmin(neg, mx);
    for (int k = 0; k < n; ++k)
    {
        const float dd = 2.0f * depth[k] - 1.0f;
        out[2 * k] = exp_(ex * dd), out[2 * k + 1] = -exp_(-ey * dd);
    }
}

// ConvertToFilterable of cascade `cascade` of a w x h map (`in`: float or uint16 texels, tightly packed) into out (h x w x ch floats,
// the filterable map's values as stored: ch = 2 for VSM / EVSM2, 4 for EVSM4). Returns the channel count; 0 for PCF.
extern "C" __attribute__((visibility("default"))) int ors_convert(int mode, const unsigned char* attribs, int cascade, const void* in, int d16, int w,
                                                                   int h, int is32, float* out, int threads)
{
    if (mode == PCF) return 0;
    const Attribs a  = parse(attribs);
    const float   mx = a.is32 ? 42.0f : 5.54f; // GetEVSMExponents takes the flag of the constant block
    Conv          c{mode, is32, d16, w, h, std::fmin(a.pos_exp, mx), std::fmin(a.neg_exp, mx), in};
    const int     ch = mode == EVSM4 ? 4 : 2;
    float         rh, rv;
    radii(a, cascade, w, h, rh, rv);
    const bool         skip = a.fixed_filter_size == 2;
    std::vector<float> inter(size_t(w) * size_t(h) * size_t(ch));
    auto               rows = [&](auto&& body) {
        const int                nt = std::max(1, std::min(threads, h));
        std::vector<std::thread> pool;
        for (int t = 0; t < nt; ++t)
            pool.emplace_back([&, t] {
                for (int y = t * h / nt; y < (t + 1) * h / nt; ++y) body(y);
            });
        for (auto& th : pool) th.join();
    };
    float* hdst = skip ? out : inter.data();
    rows([&](int y) {
        for (int x = 0; x < w; ++x)
        {
            float m[4];
            horz(c, rh, x, y, m);
            for (int k = 0; k < ch; ++k) hdst[(size_t(y) * size_t(w) + size_t(x)) * ch + k] = c.q(m[k]);
        }
    });
    if (skip) return ch;
    rows([&](int y) {
        const int range = int(std::floor(rv + 0.5f));
        for (int x = 0; x < w; ++x)
        {
            float m[4] = {0.0f, 0.0f, 0.0f, 0.0f}, total = 0.0f;
            for (int i = -range; i <= +range; ++i)
            {
                const float wt = sample_weight(i, rv);
                const int   yy = y + i;
                // the intermediate's Load: (r, g, 0, 1) of an RG texel, 0 outside; only the stored channels reach the output
                for (int k = 0; k < ch; ++k)
                {
                    const float v = (yy < 0 || yy >= h) ? 0.0f : inter[(size_t(yy) * size_t(w) + size_t(x)) * ch + k];
                    m[k]          = m[k] + v * wt;
                }
                total = total + wt;
            }
            for (int k = 0; k < ch; ++k) out[(size_t(y) * size_t(w) + size_t(x)) * ch + k] = c.q(m[k] / total);
        }
    });
    return ch;
}
