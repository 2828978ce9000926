// ibl_driver.cpp — drives Diligent::PBR_Renderer (include/dfx/PBR_Renderer.hpp) the way an application does: PrecomputeCubemaps with
// default attribs into RGBA16_FLOAT textures of the default sizes, from Hydrogent's default dome (32 x 32 white, one level, a sphere
// map; HnLight.cpp:667-685), then PrecomputeBRDF. Host-only translation unit: everything goes through the C++ header and the C-ABI.
// Then the same with DFX_MAX_ENV_LEVELS levels on both sides: a white 4^2 cube with 16 levels into a 16-level prefiltered chain from 2^2.
// Every irradiance and prefiltered texel of a white map is white; prints "ok" when they are and the BRDF table is finite. With a path
// argument, PrecomputeBRDF's table (BRDF_LUT_Dim^2 texels, RG fp32, rows top to bottom) is written there.
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <memory>
#include <vector>

#include "dfx/PBR_Renderer.hpp"

using namespace Diligent;

static float half_to_float(uint16_t h)
{
    const int e = (h >> 10) & 31, m = h & 1023;
    const float v = e == 0 ? std::ldexp(float(m), -24) : e == 31 ? (m ? NAN : INFINITY) : std::ldexp(float(m | 1024), e - 25);
    return (h & 0x8000) ? -v : v;
}

static bool all_rgb_one(ITexture& t, float alpha)
{
    std::vector<uint16_t> b(size_t(t.GetWidth()) * t.GetHeight() * 4);
    IDeviceContext        ctx;
    if (!t.ReadData(&ctx, b.data())) return false;
    for (size_t i = 0; i < b.size(); ++i)
        if (half_to_float(b[i]) != ((i % 4 == 3) ? alpha : 1.0f)) return false;
    return true;
}

int main(int argc, char** argv)
{
    IDeviceContext ctx;
    ITexture       dome{32, 32, TEX_FORMAT_RGBA32_FLOAT};
    std::vector<float> white(32 * 32 * 4, 1.0f);
    if (!dome.UpdateData(&ctx, white.data())) return 1;
    ITextureView   dome_srv{&dome};
    ITextureView*  levels[] = {&dome_srv};

    const Uint32 d = PBR_Renderer::IrradianceCubeDim, p = PBR_Renderer::PrefilteredEnvMapDim;
    ITexture     irradiance{d, 6 * d, PBR_Renderer::IrradianceCubeFmt};
    std::vector<std::unique_ptr<ITexture>> pre;
    std::vector<ITexture*>                 pre_ptrs;
    for (Uint32 s = p;; s /= 2)
    {
        pre.emplace_back(new ITexture{s, 6 * s, PBR_Renderer::PrefilteredEnvMapFmt});
        pre_ptrs.push_back(pre.back().get());
        if (s == 1) break;
    }

    PBR_Renderer                                 renderer;
    PBR_Renderer::PrecomputeCubemapsAttribs      A;
    A.ppEnvironmentMapLevels = levels, A.NumEnvironmentMapLevels = 1, A.IsCube = false;
    A.pIrradianceCube = &irradiance;
    A.ppPrefilteredEnvMapLevels = pre_ptrs.data(), A.NumPrefilteredEnvMapLevels = static_cast<Uint32>(pre_ptrs.size());
    renderer.PrecomputeCubemaps(&ctx, A);
    renderer.PrecomputeBRDF(&ctx);
    ctx.WaitForIdle();

    if (pre_ptrs.size() != 9 || !all_rgb_one(irradiance, 1.0f)) return std::printf("irradiance\n"), 3;
    for (auto* t : pre_ptrs)
        if (!all_rgb_one(*t, 0.0f)) return std::printf("prefiltered %u\n", t->GetWidth()), 4;
    std::vector<float> lut(size_t(PBR_Renderer::BRDF_LUT_Dim) * PBR_Renderer::BRDF_LUT_Dim * 2);
    if (!renderer.GetPreintegratedGGX_SRV()->GetTexture()->ReadData(&ctx, lut.data())) return 5;
    for (float v : lut)
        if (!std::isfinite(v) || v < 0.0f || v > 1.5f) return std::printf("brdf %g\n", v), 6;
    if (argc > 1)
    {
        std::FILE* f = std::fopen(argv[1], "wb");
        if (!f || std::fwrite(lut.data(), sizeof(float), lut.size(), f) != lut.size() || std::fclose(f) != 0) return std::printf("cannot write %s\n", argv[1]), 10;
    }

    // DFX_MAX_ENV_LEVELS levels: the source s_i = max(4 >> i, 1), the prefiltered chain s_m = max(2 >> m, 1)
    std::vector<std::unique_ptr<ITexture>>     src16;
    std::vector<std::unique_ptr<ITextureView>> src16_views;
    std::vector<ITextureView*>                 src16_ptrs;
    std::vector<std::unique_ptr<ITexture>>     pre16;
    std::vector<ITexture*>                     pre16_ptrs;
    for (Uint32 i = 0; i < DFX_MAX_ENV_LEVELS; ++i)
    {
        const Uint32 s = (4u >> i) > 1u ? (4u >> i) : 1u, o = (2u >> i) > 1u ? (2u >> i) : 1u;
        src16.emplace_back(new ITexture{s, 6 * s, TEX_FORMAT_RGBA32_FLOAT});
        std::vector<float> w(size_t(s) * 6 * s * 4, 1.0f);
        if (!src16.back()->UpdateData(&ctx, w.data())) return 7;
        src16_views.emplace_back(new ITextureView{src16.back().get()});
        src16_ptrs.push_back(src16_views.back().get());
        pre16.emplace_back(new ITexture{o, 6 * o, PBR_Renderer::PrefilteredEnvMapFmt});
        pre16_ptrs.push_back(pre16.back().get());
    }
    ITexture irradiance16{2, 12, PBR_Renderer::IrradianceCubeFmt};
    PBR_Renderer::PrecomputeCubemapsAttribs B;
    B.ppEnvironmentMapLevels = src16_ptrs.data(), B.NumEnvironmentMapLevels = DFX_MAX_ENV_LEVELS, B.IsCube = true;
    B.pIrradianceCube = &irradiance16, B.NumDiffuseSamples = 64, B.NumSpecularSamples = 16;
    B.ppPrefilteredEnvMapLevels = pre16_ptrs.data(), B.NumPrefilteredEnvMapLevels = DFX_MAX_ENV_LEVELS;
    renderer.PrecomputeCubemaps(&ctx, B);
    ctx.WaitForIdle();
    if (!all_rgb_one(irradiance16, 1.0f)) return std::printf("irradiance, %d levels\n", DFX_MAX_ENV_LEVELS), 8;
    for (auto* t : pre16_ptrs)
        if (!all_rgb_one(*t, 0.0f)) return std::printf("prefiltered, %d levels\n", DFX_MAX_ENV_LEVELS), 9;
    std::printf("ok\n");
    return 0;
}
