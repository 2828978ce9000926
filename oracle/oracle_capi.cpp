// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_math.h). Pinned against the reference's own shaders (oracle/refshader, tests/test_reference_shaders.py).
// C API (ctypes) over the oracle passes: a context of named fp32 planes + one "run" entry per reference pass and a
// whole-frame driver that sequences them exactly as the reference's host code does
// (Hydrogent/src/Tasks/HnPostProcessTask.cpp:743-947; per-effect Execute() methods).
#include "oracle.h"
#include "oracle_quant.h"
#include <initializer_list>
#include <iterator>
#include <map>
#include <string>
#include <chrono>
#include <cstdio>
#include <atomic>

using namespace orc;

namespace
{
struct Ctx
{
    int W = 0, H = 0, threads = 1;
    std::map<std::string, TexF>          f1;
    std::map<std::string, TexF2>         f2;
    std::map<std::string, TexF4>         f4;
    std::map<std::string, Tex<uint8_t>>  u8;
    std::map<std::string, MipTex<float>> pyr;

    std::vector<uint8_t> tables;
    Camera               curr, prev;
    dfx_dof_attribs      dof{0.01f, 0.9375f, 5, 7, 1.0f, 0.0f, 0.0f, 0.0f};
    uint                 dof_flags = 0; // DFX_DOF_FEATURE_FLAG_*
    dfx_ssao_attribs     ssao{};
    uint                 ssao_flags = 0; // DFX_SSAO_FEATURE_FLAG_*
    dfx_ssr_attribs      ssr{};
    dfx_bloom_attribs    bloom{};
    dfx_taa_attribs      taa{};
    dfx_tonemap_attribs  tm{};
    float                ave_log_lum = 0.3f;
    int                  to_srgb     = 1;
    uint                 ssr_flags = 0, taa_flags = DFX_TAA_FEATURE_FLAG_BICUBIC_FILTER;
    uint                 frame_index = 0;
    float                ssr_scale = 1.0f, ssao_scale = 1.0f;
    // reset logic of the effect classes (m_LastFrameIdx), ScreenSpaceAmbientOcclusion.cpp:797-800, TemporalAntiAliasing.cpp:125-128
    uint   ssao_last = ~0u, taa_last = ~0u;
    // which inputs the compose step takes: orc_frame leaves out the output of an effect its stage mask does not run, the way
    // HnPostProcess.psh skips the term of an effect whose scale is 0 (HnPostProcess.psh:147-180, HnPostProcessTask.cpp:632-651)
    bool   compose_ssr = true, compose_ssao = true;
    // the next orc_frame's reset decisions: -1 = the rule above, 0 = no reset, 1 = reset (orc_force_reset: a test takes the opposite
    // decision with it, also where the rule cannot be steered through the last frame index, e.g. right after index 0xFFFFFFFF)
    int    ssao_force = -1, taa_force = -1;
    double last_ms = 0.0;
    std::string err;
    // 0 = fp32 planes (the gate); 1 = "faithful": every render target is rounded to the reference's texture format after the pass that
    // writes it (oracle_quant.h, SURVEY.md Appendix B.5) - a sensitivity figure, never the parity target
    int faithful = 0;
};

std::string slot(const char* base, uint idx) { return std::string(base) + char('0' + (idx & 1u)); }

void ensure_persistent(Ctx& c)
{
    const int W = c.W, H = c.H;
    auto mk1 = [&](const std::string& n, float v) { if (!c.f1.count(n)) c.f1[n] = TexF(W, H, v); };
    auto mk4 = [&](const std::string& n) { if (!c.f4.count(n)) c.f4[n] = TexF4(W, H, float4()); };
    // SSAO history: cleared to 1.0 at creation (…SSAO.cpp:304-305, :320-321)
    mk1("ssao_hist0", 1.0f), mk1("ssao_hist1", 1.0f), mk1("ssao_histlen0", 1.0f), mk1("ssao_histlen1", 1.0f);
    // SSR: history cleared to 0 at creation (ScreenSpaceReflection.cpp:263-264, :279-280); other targets start as zero memory
    mk4("ssr_radhist0"), mk4("ssr_radhist1"), mk1("ssr_varhist0", 0.0f), mk1("ssr_varhist1", 0.0f);
    mk1("ssr_roughness", 0.0f), mk4("ssr_resolved_rad"), mk1("ssr_resolved_var", 0.0f), mk1("ssr_resolved_depth", 0.0f);
    // TAA accumulation: cleared to 0 at creation (TemporalAntiAliasing.cpp:101-119)
    mk4("taa_accum0"), mk4("taa_accum1");
}

enum Fmt { F_UNORM8, F_UNORM16, F_HALF, F_R11G11B10 };
void quant(TexF& t, Fmt f)
{
    for (float& v : t.d) v = f == F_UNORM8 ? q_unorm(v, 8) : f == F_UNORM16 ? q_unorm(v, 16) : q_half(v);
}
void quant(TexF2& t, Fmt f)
{
    for (auto& v : t.d) v.x = f == F_UNORM8 ? q_unorm(v.x, 8) : q_half(v.x), v.y = f == F_UNORM8 ? q_unorm(v.y, 8) : q_half(v.y);
}
void quant(TexF4& t, Fmt f)
{
    for (auto& v : t.d)
    {
        if (f == F_R11G11B10) v.x = q_float11(v.x), v.y = q_float11(v.y), v.z = q_float10(v.z); // no alpha channel: .w is never read
        else v.x = q_half(v.x), v.y = q_half(v.y), v.z = q_half(v.z), v.w = q_half(v.w);
    }
}
// the render targets pass `p` has just written, rounded to the formats the reference allocates them in
void quantize_outputs(Ctx& c, const std::string& p)
{
    const uint cur = c.frame_index & 1u;
    auto pyr = [&](const char* name, Fmt f, int from) {
        auto it = c.pyr.find(name);
        if (it != c.pyr.end())
            for (int i = from; i < it->second.levels(); ++i) quant(it->second.mip[i], f);
    };
    if (p == "blue_noise") quant(c.f2["bn_xy"], F_UNORM8), quant(c.f2["bn_zw"], F_UNORM8);
    else if (p == "closest_motion") quant(c.f2["closest_motion"], F_HALF);
    else if (p == "ssao_prefilter") { if (c.ssao_flags & 1u) pyr("ssao_pre", F_UNORM16, 1); }
    else if (p == "ssao_ao") quant(c.f1["ssao_occ"], F_UNORM8);
    else if (p == "ssao_upsample") quant(c.f1["ssao_occ_up"], F_UNORM8);
    else if (p == "ssao_temporal") quant(c.f1["ssao_acc"], F_UNORM8), quant(c.f1[slot("ssao_histlen", cur)], F_HALF);
    else if (p == "ssao_convolute") { pyr("ssao_conv_occ", F_UNORM8, 0); if (c.ssao_flags & 1u) pyr("ssao_conv_depth", F_UNORM16, 1); }
    else if (p == "ssao_resample") quant(c.f1["ssao_resampled"], F_UNORM8);
    else if (p == "ssao_spatial") quant(c.f1["ssao_out"], F_UNORM8), quant(c.f1[slot("ssao_hist", cur)], F_UNORM8);
    else if (p == "ssr_mask") quant(c.f1["ssr_roughness"], F_UNORM8);
    else if (p == "ssr_intersect") quant(c.f4["ssr_radiance"], F_HALF), quant(c.f4["ssr_raydir"], F_HALF);
    else if (p == "ssr_spatial") quant(c.f4["ssr_resolved_rad"], F_HALF), quant(c.f1["ssr_resolved_var"], F_HALF), quant(c.f1["ssr_resolved_depth"], F_HALF);
    else if (p == "ssr_temporal") quant(c.f4[slot("ssr_radhist", cur)], F_HALF), quant(c.f1[slot("ssr_varhist", cur)], F_HALF);
    else if (p == "ssr_bilateral") quant(c.f4["ssr_out"], F_HALF);
    else if (p == "compose") quant(c.f4["composed"], F_HALF);
    else if (p == "taa") quant(c.f4[slot("taa_accum", cur)], F_HALF);
    // "bloom" rounds each level as soon as it is written (the next level reads the stored texels): see run_pass_impl
}

int run_pass_impl(Ctx& c, const std::string& p);
int run_pass(Ctx& c, const std::string& p)
{
    const int r = run_pass_impl(c, p);
    if (r == 0 && c.faithful) quantize_outputs(c, p);
    return r;
}
int run_pass_impl(Ctx& c, const std::string& p)
{
    const int  T   = c.threads;
    const uint cur = c.frame_index & 1u, prv = (c.frame_index + 1u) & 1u;
    ensure_persistent(c);
    if (p == "blue_noise")
    {
        if (c.tables.size() != 256 + 128 * 128 * 8) return c.err = "blue-noise tables not set", 1;
        postfx_blue_noise(c.tables.data(), c.frame_index, c.f2["bn_xy"], c.f2["bn_zw"]);
    }
    else if (p == "reprojected_depth") postfx_reprojected_depth(c.curr, c.prev, c.f1["depth"], c.f1["reproj_depth"], T);
    else if (p == "closest_motion") postfx_closest_motion(c.f1["depth"], c.f2["motion"], c.f2["closest_motion"], T);
    else if (p == "previous_depth") c.f1["prev_depth"] = c.f1["prev_depth_in"];
    // FEATURE_FLAG_HALF_RESOLUTION (bit 1 of the SSAO flags): A0, then A1-A3 on W/2 x H/2, then A4 (…SSAO.cpp:818-857, :992-1049)
    else if (p == "ssao_downsample") ssao_downsample_depth(c.f1["depth"], c.f1["ssao_checker"], T);
    else if (p == "ssao_prefilter") ssao_prefilter_depth(c.curr, c.ssao, c.f1[(c.ssao_flags & 2u) ? "ssao_checker" : "depth"], c.pyr["ssao_pre"], T);
    else if (p == "ssao_ao")
        ssao_ambient_occlusion(c.curr, c.ssao, c.pyr["ssao_pre"], c.f4["normal"], c.f2["bn_zw"], c.f1["ssao_occ"], T, (c.ssao_flags & 2u) != 0, (c.ssao_flags & 1u) != 0);
    else if (p == "ssao_upsample") ssao_bilateral_upsampling(c.curr, c.f1["depth"], c.f1["ssao_occ"], c.f1["ssao_occ_up"], T);
    else if (p == "ssao_temporal")
        ssao_temporal(c.curr, c.prev, c.ssao, c.f1[(c.ssao_flags & 2u) ? "ssao_occ_up" : "ssao_occ"], c.f1[slot("ssao_hist", prv)], c.f1[slot("ssao_histlen", prv)], c.f1["reproj_depth"],
                      c.f1["prev_depth"], c.f2["closest_motion"], c.f1["ssao_acc"], c.f1[slot("ssao_histlen", cur)], T);
    else if (p == "ssao_convolute") ssao_convolute(c.f1["ssao_acc"], c.f1["depth"], c.pyr["ssao_conv_occ"], c.pyr["ssao_conv_depth"], T);
    else if (p == "ssao_resample")
        ssao_resample(c.curr, c.pyr["ssao_conv_occ"], c.pyr["ssao_conv_depth"], c.f1[slot("ssao_histlen", cur)], c.f4["normal"], c.f1["ssao_resampled"], T);
    else if (p == "ssao_spatial")
    {
        // resolved output, then CopyTexture(resolved -> history[curr]) (…SSAO.cpp:1319-1328)
        ssao_spatial(c.curr, c.ssao, c.f1["ssao_resampled"], c.f1[slot("ssao_histlen", cur)], c.f1["depth"], c.f4["normal"], c.f1["ssao_out"], T);
        c.f1[slot("ssao_hist", cur)] = c.f1["ssao_out"];
    }
    else if (p == "ssr_hiz") ssr_hiz(c.f1["depth"], c.pyr["ssr_hiz"], T);
    else if (p == "ssr_mask") ssr_mask_roughness(c.ssr, c.f4["material"], c.f1["depth"], c.f1["ssr_roughness"], c.u8["ssr_mask"], T);
    // FEATURE_FLAG_HALF_RESOLUTION (bit 1 of the SSR flags): S3, S4 on W/2 x H/2 with the downsampled mask, S5 gathers from the half-size targets
    else if (p == "ssr_downsample_mask") ssr_downsample_mask(c.ssr, c.f1["ssr_roughness"], c.f1["depth"], c.u8["ssr_mask_half"], T);
    else if (p == "ssr_intersect")
        ssr_intersect(c.curr, c.ssr, c.ssr_flags, c.f4["color"], c.f4["normal"], c.f1["ssr_roughness"], c.u8[(c.ssr_flags & 2u) ? "ssr_mask_half" : "ssr_mask"], c.f2["bn_xy"], c.pyr["ssr_hiz"],
                      &c.f2["motion"], c.f4["ssr_radiance"], c.f4["ssr_raydir"], T);
    else if (p == "ssr_spatial")
        ssr_spatial(c.curr, c.ssr, c.f1["ssr_roughness"], c.u8["ssr_mask"], c.f4["normal"], c.f1["depth"], c.f4["ssr_raydir"], c.f4["ssr_radiance"],
                    c.f4["ssr_resolved_rad"], c.f1["ssr_resolved_var"], c.f1["ssr_resolved_depth"], T, (c.ssr_flags & 2u) != 0);
    else if (p == "ssr_temporal")
        ssr_temporal(c.curr, c.prev, c.ssr, c.u8["ssr_mask"], c.f2["motion"], c.f1["ssr_resolved_depth"], c.f1["reproj_depth"], c.f4["ssr_resolved_rad"],
                     c.f1["ssr_resolved_var"], c.f1["prev_depth"], c.f4[slot("ssr_radhist", prv)], c.f1[slot("ssr_varhist", prv)],
                     c.f4[slot("ssr_radhist", cur)], c.f1[slot("ssr_varhist", cur)], T);
    else if (p == "ssr_bilateral")
        ssr_bilateral(c.curr, c.ssr, c.u8["ssr_mask"], c.f1["depth"], c.f4["normal"], c.f1["ssr_roughness"], c.f4[slot("ssr_radhist", cur)],
                      c.f1[slot("ssr_varhist", cur)], c.f4["ssr_out"], T);
    // DepthOfField, D1-D11 in the order of DepthOfField::Execute (DepthOfField.cpp:292-331). "dof_in" = the colour it blurs.
    // Each step is also a pass of its own, so that tests can look at one at a time.
    else if (p == "dof")
    {
        static const char* steps[] = {"dof_coc", "dof_temporal", "dof_separated", "dof_dilation", "dof_blur_x", "dof_blur_y", "dof_prefilter",
                                      "dof_bokeh_first", "dof_bokeh_second", "dof_postfilter", "dof_combine"};
        for (const char* st : steps)
            if (int r = run_pass(c, st)) return r;
    }
    else if (p.rfind("dof_", 0) == 0)
    {
        const bool  temporal = (c.dof_flags & 1u) != 0;
        const TexF& coc      = temporal ? c.f1[slot("dof_coc_temporal", cur)] : c.f1["dof_coc"];
        if (p == "dof_coc") dof_circle_of_confusion(c.curr, c.dof, c.f1["depth"], c.f1["dof_coc"], T);
        else if (p == "dof_temporal")
        {
            if (temporal)
            {
                TexF& prevc = c.f1[slot("dof_coc_temporal", prv)];
                if (prevc.w != c.f1["dof_coc"].w || prevc.h != c.f1["dof_coc"].h) prevc.resize(c.f1["dof_coc"].w, c.f1["dof_coc"].h, 0.0f); // cleared to 0 at creation (:187-189)
                dof_temporal_coc(c.curr, c.dof, c.f1["dof_coc"], prevc, c.f2["closest_motion"], c.f1[slot("dof_coc_temporal", cur)], T);
            }
        }
        else if (p == "dof_separated") dof_separated_coc(coc, c.f1["dof_dilation0"], T);
        else if (p == "dof_dilation")
            for (int i = 0; i < 3; ++i) dof_dilation_level(c.f1["dof_dilation" + std::to_string(i)], c.f1["dof_dilation" + std::to_string(i + 1)], T);
        else if (p == "dof_blur_x") dof_blur_coc(c.f1["dof_dilation3"], false, c.f1["dof_dilation_tmp"], T);
        else if (p == "dof_blur_y") dof_blur_coc(c.f1["dof_dilation_tmp"], true, c.f1["dof_dilation3"], T);
        else if (p == "dof_prefilter") dof_prefilter(c.f4["dof_in"], coc, c.f1["dof_dilation3"], c.f4["dof_pre0"], c.f4["dof_pre1"], T);
        else if (p == "dof_bokeh_first")
            dof_bokeh_first(c.curr, c.dof, c.dof_flags, c.f4["dof_pre0"], c.f4["dof_pre1"], c.f4["dof_in"], c.f4["dof_bokeh0"], c.f4["dof_bokeh1"], T);
        else if (p == "dof_bokeh_second") dof_bokeh_second(c.curr, c.dof, c.f4["dof_bokeh0"], c.f4["dof_bokeh1"], c.f4["dof_pre0"], c.f4["dof_pre1"], T);
        else if (p == "dof_postfilter") dof_postfilter(c.f4["dof_pre0"], c.f4["dof_pre1"], c.f4["dof_bokeh0"], c.f4["dof_bokeh1"], T);
        else if (p == "dof_combine") dof_combine(c.dof, c.f4["dof_in"], c.f4["dof_bokeh0"], c.f4["dof_bokeh1"], c.f4["dof_out"], T);
        else
            return c.err = "unknown pass " + p, 1;
    }
    else if (p == "compose_ibl")
        compose_ibl(c.curr, c.f4["color"], &c.f4["ssr_out"], &c.f1["ssao_out"], c.f4["specular_ibl"], c.f4["normal"], c.f4["base_color"], c.f4["material"],
                    c.f2["brdf_lut"], c.ssr_scale, c.ssao_scale, c.f4["composed"], T);
    else if (p == "compose")
        compose(c.f4["color"], c.compose_ssr ? &c.f4["ssr_out"] : nullptr, c.compose_ssao ? &c.f1["ssao_out"] : nullptr, c.ssr_scale, c.ssao_scale,
                c.f4["composed"], T);
    else if (p == "taa")
        taa_accumulate(c.curr, c.prev, c.taa, c.taa_flags, c.f4["taa_in"], c.f4[slot("taa_accum", prv)], c.f2["closest_motion"], c.f1["reproj_depth"],
                       c.f1["prev_depth"], c.f4[slot("taa_accum", cur)], T);
    else if (p == "bloom")
    {
        // Bloom::Execute (Bloom.cpp:407-436)
        const TexF4& in   = c.f4["bloom_in"];
        const int    mips = bloom_mip_count(std::max(in.w / 2, 1), std::max(in.h / 2, 1), c.bloom.Radius);
        // the composite samples up(0), which only the upsampling of a second level writes: refuse like the CUDA effect does
        if (mips < 2) return c.err = "Bloom radius " + std::to_string(c.bloom.Radius) + " leaves fewer than two pyramid levels at " +
                                     std::to_string(in.w) + "x" + std::to_string(in.h), 1;
        auto dn = [&](int i) -> TexF4& { return c.f4["bloom_down" + std::to_string(i)]; };
        auto up = [&](int i) -> TexF4& { return c.f4["bloom_up" + std::to_string(i)]; };
        auto store = [&](TexF4& t) { if (c.faithful) quant(t, F_R11G11B10); }; // every Bloom target is R11G11B10_FLOAT (Bloom.cpp:111, :125, :137)
        bloom_prefilter(c.bloom, in, dn(0), T), store(dn(0));
        for (int i = 1; i < mips; ++i) bloom_downsample(dn(i - 1), dn(i), T), store(dn(i));
        const int top = mips - 1;
        for (int i = top; i > 0; --i) bloom_upsample(dn(i - 1), i != top ? up(i) : dn(i), up(i - 1), T), store(up(i - 1));
        bloom_composite(c.bloom, in, up(0), c.f4["bloom_out"], T), store(c.f4["bloom_out"]);
    }
    else if (p == "tonemap") tonemap_pass(c.tm, c.ave_log_lum, c.to_srgb != 0, c.f4["tonemap_in"], c.f4["ldr"], T);
    else
        return c.err = "unknown pass " + p, 1;
    return 0;
}
} // namespace

namespace orc
{
float oracle_fast_acos(float v);
extern std::atomic<unsigned long long> g_march_rays, g_march_iterations;
extern unsigned short* g_march_iteration_plane;
extern int             g_march_iteration_pitch;
bool g_reversed_depth = false;
} // namespace orc

extern "C"
{
#define ORC_API __attribute__((visibility("default")))

ORC_API void* orc_create(int w, int h, int threads)
{
    Ctx* c     = new Ctx;
    c->W       = w;
    c->H       = h;
    c->threads = threads < 1 ? 1 : threads;
    dfx_ssao_attribs  s{1.0f, 0.615f, 1.457f, 3.3f, 0.9f, 4.0f, 0, 1.0f, 0.5f, 0u, 0.0f, 0.0f};
    dfx_ssr_attribs   r{0.025f, 0.2f, 0u, 1, 0u, 128u, 0.3f, 4.0f, 1.0f, 0.9f, 0.9f, 1.0f};
    dfx_bloom_attribs b{0.15f, 1.0f, 0.125f, 0.75f, 1.0f, 0, 0, 0};
    dfx_taa_attribs   t{0.9375f, 0, 0, 0.0f};
    dfx_tonemap_attribs m{DFX_TONE_MAPPING_MODE_UNCHARTED2, 1, 0.18f, 1, 3.0f, 1.0f, 0, 0, 1.0f, 1.0f, 1.0f, 0.0f};
    c->ssao = s, c->ssr = r, c->bloom = b, c->taa = t, c->tm = m;
    return c;
}
ORC_API void        orc_destroy(void* h) { delete static_cast<Ctx*>(h); }
ORC_API const char* orc_last_error(void* h) { return static_cast<Ctx*>(h)->err.c_str(); }
ORC_API double      orc_last_ms(void* h) { return static_cast<Ctx*>(h)->last_ms; }
ORC_API void        orc_set_threads(void* h, int t) { static_cast<Ctx*>(h)->threads = t < 1 ? 1 : t; }

ORC_API int orc_set_tables(void* h, const uint8_t* blob, int n)
{
    Ctx& c = *static_cast<Ctx*>(h);
    if (n != 256 + 128 * 128 * 8) return c.err = "bad table size", 1;
    c.tables.assign(blob, blob + n);
    return 0;
}

// ch: 1, 2, 4 (fp32) ; name "x.N" addresses mip N of pyramid x ; u8 masks are exchanged as fp32 0/1 with ch == 1
ORC_API int orc_set_plane(void* h, const char* name, const float* data, int w, int hgt, int ch)
{
    Ctx&        c = *static_cast<Ctx*>(h);
    std::string n(name);
    size_t      cnt = size_t(w) * size_t(hgt);
    if (n == "ssr_mask")
    {
        Tex<uint8_t>& t = c.u8[n];
        t.resize(w, hgt, 0);
        for (size_t i = 0; i < cnt; ++i) t.d[i] = data[i] != 0.0f;
        return 0;
    }
    auto dot_pos = n.find('.');
    if (dot_pos != std::string::npos)
    {
        MipTex<float>& p  = c.pyr[n.substr(0, dot_pos)];
        int            lv = std::stoi(n.substr(dot_pos + 1));
        if (int(p.mip.size()) <= lv) p.mip.resize(lv + 1);
        p.mip[lv].resize(w, hgt);
        std::memcpy(p.mip[lv].d.data(), data, cnt * 4);
        return 0;
    }
    if (ch == 1)
    {
        TexF& t = c.f1[n];
        t.resize(w, hgt);
        std::memcpy(t.d.data(), data, cnt * 4);
    }
    else if (ch == 2)
    {
        TexF2& t = c.f2[n];
        t.resize(w, hgt);
        std::memcpy((void*)t.d.data(), data, cnt * 8);
    }
    else if (ch == 4)
    {
        TexF4& t = c.f4[n];
        t.resize(w, hgt);
        std::memcpy((void*)t.d.data(), data, cnt * 16);
    }
    else
        return c.err = "bad channel count", 1;
    return 0;
}

// out == NULL: query only. Returns 0 and fills w/h/ch; 1 if the plane does not exist.
ORC_API int orc_get_plane(void* h, const char* name, float* out, int* w, int* hgt, int* ch)
{
    Ctx&        c = *static_cast<Ctx*>(h);
    std::string n(name);
    auto        dot_pos = n.find('.');
    if ((n == "ssr_mask" || n == "ssr_mask_half") && c.u8.count(n))
    {
        const Tex<uint8_t>& t = c.u8[n];
        *w = t.w, *hgt = t.h, *ch = 1;
        if (out)
            for (size_t i = 0; i < t.d.size(); ++i) out[i] = float(t.d[i]);
        return 0;
    }
    if (dot_pos != std::string::npos)
    {
        auto it = c.pyr.find(n.substr(0, dot_pos));
        int  lv = std::stoi(n.substr(dot_pos + 1));
        if (it == c.pyr.end() || lv >= it->second.levels()) return c.err = "no such plane " + n, 1;
        const TexF& t = it->second.mip[lv];
        *w = t.w, *hgt = t.h, *ch = 1;
        if (out) std::memcpy(out, t.d.data(), t.d.size() * 4);
        return 0;
    }
    if (c.f1.count(n))
    {
        const TexF& t = c.f1[n];
        *w = t.w, *hgt = t.h, *ch = 1;
        if (out) std::memcpy(out, t.d.data(), t.d.size() * 4);
        return 0;
    }
    if (c.f2.count(n))
    {
        const TexF2& t = c.f2[n];
        *w = t.w, *hgt = t.h, *ch = 2;
        if (out) std::memcpy(out, (const void*)t.d.data(), t.d.size() * 8);
        return 0;
    }
    if (c.f4.count(n))
    {
        const TexF4& t = c.f4[n];
        *w = t.w, *hgt = t.h, *ch = 4;
        if (out) std::memcpy(out, (const void*)t.d.data(), t.d.size() * 16);
        return 0;
    }
    return c.err = "no such plane " + n, 1;
}

ORC_API void orc_set_cameras(void* h, const dfx_camera_attribs* curr, const dfx_camera_attribs* prev)
{
    Ctx& c = *static_cast<Ctx*>(h);
    c.curr = to_camera(*curr);
    c.prev = to_camera(*prev);
}
ORC_API void orc_set_storage(void* h, int faithful) { static_cast<Ctx*>(h)->faithful = faithful; }
ORC_API float orc_quantize(int fmt, float v) { return fmt == 0 ? q_unorm(v, 8) : fmt == 1 ? q_unorm(v, 16) : fmt == 2 ? q_half(v) : fmt == 3 ? q_float11(v) : q_float10(v); }
ORC_API void orc_set_frame_index(void* h, uint32_t idx) { static_cast<Ctx*>(h)->frame_index = idx; }
ORC_API void orc_set_ssao_attribs(void* h, const dfx_ssao_attribs* a) { static_cast<Ctx*>(h)->ssao = *a; }
// The effects' PrepareResources re-create their targets when a feature flag changes the targets' size or format. The planes that
// carry state from frame to frame are set back to their creation value here (a plane that does not exist yet is created at that
// value when first used); the last frame index (m_LastFrameIdx) is kept, so on a consecutive index the next frame does not reset
// and reads the cleared history.
static void clear_planes(Ctx& c, std::initializer_list<const char*> names, float v)
{
    for (const char* n : names)
    {
        if (auto it = c.f1.find(n); it != c.f1.end()) std::fill(it->second.d.begin(), it->second.d.end(), v);
        if (auto it = c.f4.find(n); it != c.f4.end()) std::fill(it->second.d.begin(), it->second.d.end(), float4(v, v, v, v));
    }
}
ORC_API void orc_set_ssao_flags(void* h, uint32_t flags)
{
    // ScreenSpaceAmbientOcclusion.cpp:72-79: HALF_PRECISION_DEPTH or HALF_RESOLUTION changed -> the targets are re-created, the
    // history and history length cleared to 1 (:290-321)
    Ctx& c = *static_cast<Ctx*>(h);
    if ((c.ssao_flags ^ flags) & 3u) clear_planes(c, {"ssao_hist0", "ssao_hist1", "ssao_histlen0", "ssao_histlen1"}, 1.0f);
    c.ssao_flags = flags;
}
ORC_API void orc_set_ssr_attribs(void* h, const dfx_ssr_attribs* a, uint32_t flags)
{
    // HALF_RESOLUTION changed -> the targets are re-created: the histories cleared to 0 (ScreenSpaceReflection.cpp:263-264, :279-280), and
    // the targets the reference leaves uncleared back at the zeroed memory the CUDA effect allocates them with. PREVIOUS_FRAME only
    // selects the colour the rays read.
    Ctx& c = *static_cast<Ctx*>(h);
    if ((c.ssr_flags ^ flags) & 2u)
        clear_planes(c, {"ssr_radhist0", "ssr_radhist1", "ssr_varhist0", "ssr_varhist1", "ssr_roughness", "ssr_resolved_rad", "ssr_resolved_var", "ssr_resolved_depth"},
                     0.0f);
    c.ssr       = *a;
    c.ssr_flags = flags;
}
ORC_API void orc_set_dof_attribs(void* h, const dfx_dof_attribs* a, uint32_t flags)
{
    // DepthOfField.cpp:177-189: any change of the feature flags re-creates the targets, the temporal CoC cleared to 0
    Ctx& c = *static_cast<Ctx*>(h);
    if (c.dof_flags != flags) clear_planes(c, {"dof_coc_temporal0", "dof_coc_temporal1"}, 0.0f);
    c.dof       = *a;
    c.dof_flags = flags;
}
// a new frame size: every frame-sized plane goes, so the next frame creates them at their creation values (the effects re-create
// their targets on a size change and keep m_LastFrameIdx). The BRDF table is not frame-sized and stays.
ORC_API void orc_resize(void* h, int w, int hgt)
{
    Ctx& c = *static_cast<Ctx*>(h);
    c.W = w, c.H = hgt;
    auto keep_lut = [&](auto& planes) {
        for (auto it = planes.begin(); it != planes.end();) it = it->first == "brdf_lut" ? std::next(it) : planes.erase(it);
    };
    keep_lut(c.f1), keep_lut(c.f2), keep_lut(c.f4), keep_lut(c.u8), keep_lut(c.pyr);
}
ORC_API void orc_last_frames(void* h, uint32_t* ssao_last, uint32_t* taa_last)
{
    *ssao_last = static_cast<Ctx*>(h)->ssao_last;
    *taa_last  = static_cast<Ctx*>(h)->taa_last;
}
ORC_API void orc_force_reset(void* h, int ssao, int taa)
{
    static_cast<Ctx*>(h)->ssao_force = ssao;
    static_cast<Ctx*>(h)->taa_force  = taa;
}
ORC_API void orc_set_bloom_attribs(void* h, const dfx_bloom_attribs* a) { static_cast<Ctx*>(h)->bloom = *a; }
ORC_API void orc_set_taa_attribs(void* h, const dfx_taa_attribs* a, uint32_t flags)
{
    static_cast<Ctx*>(h)->taa       = *a;
    static_cast<Ctx*>(h)->taa_flags = flags;
}
ORC_API void orc_set_tonemap_attribs(void* h, const dfx_tonemap_attribs* a, float ave_log_lum, int to_srgb)
{
    Ctx& c        = *static_cast<Ctx*>(h);
    c.tm          = *a;
    c.ave_log_lum = ave_log_lum;
    c.to_srgb     = to_srgb;
}
ORC_API void orc_set_compose_scales(void* h, float ssr_scale, float ssao_scale)
{
    static_cast<Ctx*>(h)->ssr_scale  = ssr_scale;
    static_cast<Ctx*>(h)->ssao_scale = ssao_scale;
}

ORC_API int orc_run(void* h, const char* pass)
{
    Ctx& c  = *static_cast<Ctx*>(h);
    auto t0 = std::chrono::steady_clock::now();
    int  r  = run_pass(c, pass);
    c.last_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return r;
}

// Whole frame in the reference order (HnPostProcessTask.cpp:788-925): PostFX -> SSR -> SSAO -> compose -> TAA -> Bloom -> ToneMap(+sRGB).
// `stages` bit mask: 1 postfx, 2 ssr, 4 ssao, 8 compose, 16 taa, 32 bloom, 64 tonemap.
// Inputs: depth, prev_depth_in, motion, normal, color, material; cameras, frame index and attribs set beforehand.
ORC_API int orc_frame(void* h, uint32_t stages)
{
    Ctx& c  = *static_cast<Ctx*>(h);
    auto t0 = std::chrono::steady_clock::now();
    int  r  = 0;
    auto run = [&](const char* p) { if (!r) r = run_pass(c, p); };
    if (stages & 1u) run("blue_noise"), run("reprojected_depth"), run("closest_motion"), run("previous_depth");
    if (stages & 2u)
    {
        run("ssr_hiz"), run("ssr_mask");
        if (c.ssr_flags & 2u) run("ssr_downsample_mask");
        run("ssr_intersect"), run("ssr_spatial"), run("ssr_temporal"), run("ssr_bilateral");
    }
    if (stages & 4u)
    {
        // UpdateConstantBuffer reset rule (…SSAO.cpp:797-800)
        dfx_ssao_attribs user = c.ssao;
        bool reset = c.ssao_last == ~0u || c.frame_index != c.ssao_last + 1u || user.ResetAccumulation != 0;
        if (c.ssao_force >= 0) reset = c.ssao_force != 0;
        c.ssao.ResetAccumulation = reset ? 1 : 0;
        if (c.ssao_flags & 2u) run("ssao_downsample");
        run("ssao_prefilter"), run("ssao_ao");
        if (c.ssao_flags & 2u) run("ssao_upsample");
        run("ssao_temporal"), run("ssao_convolute"), run("ssao_resample"), run("ssao_spatial");
        c.ssao      = user;
        c.ssao_last = c.frame_index;
    }
    if (stages & 8u)
    {
        c.compose_ssr = (stages & 2u) != 0, c.compose_ssao = (stages & 4u) != 0;
        run("compose");
        c.compose_ssr = c.compose_ssao = true;
    }
    if (stages & 16u)
    {
        dfx_taa_attribs user = c.taa;
        bool reset = c.taa_last == ~0u || c.frame_index != c.taa_last + 1u || user.ResetAccumulation != 0;
        if (c.taa_force >= 0) reset = c.taa_force != 0;
        c.taa.ResetAccumulation = reset ? 1 : 0;
        c.f4["taa_in"] = (stages & 8u) ? c.f4["composed"] : c.f4["color"];
        run("taa");
        c.taa      = user;
        c.taa_last = c.frame_index;
    }
    if (stages & 128u) // DepthOfField sits between TAA and Bloom (HnPostProcessTask.cpp:899-909)
    {
        c.f4["dof_in"] = (stages & 16u) ? c.f4[slot("taa_accum", c.frame_index & 1u)] : ((stages & 8u) ? c.f4["composed"] : c.f4["color"]);
        run("dof");
    }
    if (stages & 32u)
    {
        c.f4["bloom_in"] = (stages & 128u) ? c.f4["dof_out"]
                                           : ((stages & 16u) ? c.f4[slot("taa_accum", c.frame_index & 1u)] : ((stages & 8u) ? c.f4["composed"] : c.f4["color"]));
        run("bloom");
    }
    if (stages & 64u)
    {
        c.f4["tonemap_in"] = (stages & 32u) ? c.f4["bloom_out"] : c.f4["color"];
        run("tonemap");
    }
    c.ssao_force = c.taa_force = -1;
    c.last_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return r;
}

// scalar helpers exposed for the KATs
ORC_API void  orc_tone_map(const dfx_tonemap_attribs* a, float ave_log_lum, const float* rgb_in, float* rgb_out, int n)
{
    for (int i = 0; i < n; ++i)
    {
        float3 o = tone_map(float3(rgb_in[3 * i], rgb_in[3 * i + 1], rgb_in[3 * i + 2]), *a, ave_log_lum);
        rgb_out[3 * i] = o.x, rgb_out[3 * i + 1] = o.y, rgb_out[3 * i + 2] = o.z;
    }
}
ORC_API uint32_t orc_pcg_hash(uint32_t s) { return PCGHash(s); }
ORC_API float    orc_bayer4x4(uint32_t x, uint32_t y, uint32_t f) { return Bayer4x4(x, y, f); }
ORC_API float    orc_halton(uint32_t base, uint32_t idx) { return halton_sequence(base, idx); }
ORC_API void     orc_taa_jitter(uint32_t frame, uint32_t w, uint32_t hgt, float* out)
{
    float2 j = taa_jitter_offset(frame, w, hgt);
    out[0] = j.x, out[1] = j.y;
}
ORC_API void orc_brdf_lut(void* h, int w, int hgt, uint32_t num_samples)
{
    Ctx& c = *static_cast<Ctx*>(h);
    orc::brdf_lut(w, hgt, num_samples, c.f2["brdf_lut"], c.threads);
}
ORC_API void orc_set_reversed_depth(int on) { orc::g_reversed_depth = on != 0; } // process-wide, like a shader macro
ORC_API void orc_march_stats(unsigned long long* rays, unsigned long long* iterations, int reset)
{
    *rays       = orc::g_march_rays.load();
    *iterations = orc::g_march_iterations.load();
    if (reset) orc::g_march_rays = 0, orc::g_march_iterations = 0;
}
// per-pixel trip counts of the next intersection passes into plane[h][pitch] (zero it first; nullptr switches the record off)
ORC_API void orc_march_iteration_plane(unsigned short* plane, int pitch)
{
    orc::g_march_iteration_plane = plane;
    orc::g_march_iteration_pitch = pitch;
}
// kernel textures of DepthOfField (DepthOfField.cpp:49-91): points as x,y pairs; returns the count (writes at most max_count entries)
ORC_API int orc_dof_kernel_points(int ring_count, int ring_density, float* out_xy, int max_count)
{
    const std::vector<float2> k = dof_kernel_points(ring_count, ring_density);
    for (int i = 0; i < int(k.size()) && i < max_count; ++i) out_xy[2 * i] = k[i].x, out_xy[2 * i + 1] = k[i].y;
    return int(k.size());
}
ORC_API int orc_dof_gauss_kernel(int radius, float sigma, float* out, int max_count)
{
    const std::vector<float> k = dof_gauss_kernel(radius, sigma);
    for (int i = 0; i < int(k.size()) && i < max_count; ++i) out[i] = k[i];
    return int(k.size());
}
ORC_API int orc_bloom_mip_count(int w, int hgt, float radius) { return bloom_mip_count(w, hgt, radius); }
ORC_API float orc_fast_acos(float v) { return orc::oracle_fast_acos(v); }
ORC_API float orc_depth_to_camera_z(float d, const dfx_float4x4* proj) { return DepthToCameraZ(d, to_mat(*proj)); }
ORC_API float orc_camera_z_to_depth(float z, const dfx_float4x4* proj) { return CameraZToDepth(z, to_mat(*proj)); }
}
