// dfx_compose.cu — the full compose step of the reference integration (SURVEY.md §8f rank 1) and the table it needs.
//
//   Hydrogent/shaders/HnPostProcess.psh:145-185: with Opacity = Color.a,
//     Color.rgb += (GetSpecularIBL_GGX(SrfInfo, IBLInfo, SSR.rgb) - SpecularIBL.rgb) * SSR.a * SSRScale * Opacity
//     Color.rgb *= lerp(1, AO, SSAOScale * Opacity)
//   i.e. the screen-space reflection is re-weighted by the split-sum BRDF of the surface and EXCHANGED for the image-based
//   specular term the renderer had already added (PBR_Shading.fxh:220-302 with USE_IBL_MULTIPLE_SCATTERING = 1, :429-451).
//   The split sum reads a pre-integrated GGX table: Shaders/PBR/private/PrecomputeBRDF.psh:10-48 (PBR_Renderer.cpp:548-625
//   builds it once, 512 x 512, 512 samples). dfx_pass_compose (dfx_bloom_taa_tonemap.cu) stays as the reduced form for
//   callers without the IBL / base-colour planes.
#include "dfx_ibl_math.cuh"

namespace dfx
{

using namespace iblm;

// ---------------------------------------------------------------------------------------------------------------------
// PrecomputeBRDF.psh:10-48 + PBR_PrecomputeCommon.fxh:10-39 with DESIGN.md §2's rule for PBR_Renderer's precomputations: every
// operation rounded once in the shader's order, cos / sin correctly rounded, pow(1 - VoH, 5) as pow5_. Each texel adds its samples in
// order, as the shader does, so the table is the oracle's bit for bit. N = +z, so ImportanceSampleGGX's UpVector is x and its frame
// is built once per texel, exactly as the shader composes it. What depends only on the sample index (the Hammersley point, Phi's cos
// and sin) is computed once per CTA into shared memory, 256 samples at a time, as dfx_ibl.cu stages its samples; every texel then runs
// the rest of the sample in the shader's order.
// ---------------------------------------------------------------------------------------------------------------------
constexpr unsigned kLutChunk = 256; // the CTA's threads

__global__ void __launch_bounds__(kLutChunk) brdf_lut_kernel(View<float2> lut, unsigned num_samples)
{
    __shared__ float s_xi_y[kLutChunk], s_cos[kLutChunk], s_sin[kLutChunk];
    const int  x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    const int  t    = threadIdx.y * blockDim.x + threadIdx.x;
    const bool live = x < lut.w && y < lut.h;
    // UV of the texel centre: NdotV = u, PerceptualRoughness = v
    const float  NoV = div_(add_(float(x), 0.5f), float(lut.w)), rough = div_(add_(float(y), 0.5f), float(lut.h));
    const float3 V = make_float3(sqrt_(sub_(1.0f, mul_(NoV, NoV))), 0.0f, NoV);
    const float3 N = make_float3(0.0f, 0.0f, 1.0f);
    const float  alpha = mul_(rough, rough), a2 = mul_(alpha, alpha), one_m_a2 = sub_(1.0f, a2);
    const float3 tx = normalize3(cross3(make_float3(1.0f, 0.0f, 0.0f), N)), ty = cross3(N, tx);
    // SmithGGXVisibilityCorrelated's NdotL * sqrt(max(NdotV * NdotV * (1 - a2) + a2, 1e-7)) factor that depends on NdotV only
    const float sv = sqrt_(fmaxf(add_(mul_(mul_(NoV, NoV), one_m_a2), a2), 1e-7f));
    float       A = 0.0f, B = 0.0f;
    for (uint64_t c0 = 0; c0 < num_samples; c0 += kLutChunk) // 64-bit: a count near 2^32 must not wrap the chunk index
    {
        if (c0 + t < num_samples)
        {
            // ImportanceSampleGGX (PBR_PrecomputeCommon.fxh:19-39) up to Phi
            const float2 xi  = hammersley(uint32_t(c0 + t), num_samples);
            const float  phi = mul_(mul_(2.0f, kPi), xi.x);
            s_xi_y[t] = xi.y, s_cos[t] = cos_(phi), s_sin[t] = sin_(phi);
        }
        __syncthreads();
        if (live)
        {
            const unsigned nk = unsigned(min(uint64_t(num_samples) - c0, uint64_t(kLutChunk)));
            for (unsigned q = 0; q < nk; ++q)
            {
                const float  xi_y = s_xi_y[q];
                const float  ct   = sqrt_(sat_(div_(sub_(1.0f, xi_y), add_(1.0f, mul_(sub_(a2, 1.0f), xi_y)))));
                const float  st   = sqrt_(sat_(sub_(1.0f, mul_(ct, ct))));
                const float3 H    = combine3(tx, mul_(st, s_cos[q]), ty, mul_(st, s_sin[q]), N, ct);
                const float  vh   = dot3(V, H), tv = mul_(2.0f, vh);
                const float  NoL = sat_(sub_(mul_(tv, H.z), V.z)), NoH = sat_(H.z), VoH = sat_(vh);
                if (NoL > 0.0f)
                {
                    // SmithGGXVisibilityCorrelated (PBR_Common.fxh:107-124)
                    const float ggxv = mul_(NoL, sv);
                    const float ggxl = mul_(NoV, sqrt_(fmaxf(add_(mul_(mul_(NoL, NoL), one_m_a2), a2), 1e-7f)));
                    const float vis  = div_(0.5f, add_(ggxv, ggxl));
                    const float gvis = div_(mul_(mul_(mul_(4.0f, vis), VoH), NoL), NoH);
                    const float fc   = pow5_(sub_(1.0f, VoH));
                    A = add_(A, mul_(sub_(1.0f, fc), gvis));
                    B = add_(B, mul_(fc, gvis));
                }
            }
        }
        __syncthreads();
    }
    if (live) lut.at(x, y) = make_float2(div_(A, float(num_samples)), div_(B, float(num_samples)));
}

// ---------------------------------------------------------------------------------------------------------------------
// HnPostProcess.psh:145-185, each operation rounded once in the order the test oracle uses: the pass is the oracle's
// bit for bit.
// ---------------------------------------------------------------------------------------------------------------------
struct ComposeCam
{
    CamS c;
    Mat4 vp_inv;
};

// the world position through the pixel centre at NDC depth 0.5: mul(float4(ndc, 0.5, 1), ViewProjInv) left to right, then xyz / w
DFX_HD float3 pixel_world_position(float u, float v, const Mat4& M)
{
    const float nx = mul_(sub_(u, 0.5f), 2.0f), ny = mul_(sub_(v, 0.5f), -2.0f); // TexUVToNormalizedDeviceXY
    float       w[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) w[c] = add_(add_(add_(mul_(nx, M.m[0][c]), mul_(ny, M.m[1][c])), mul_(0.5f, M.m[2][c])), mul_(1.0f, M.m[3][c]));
    return make_float3(div_(w[0], w[3]), div_(w[1], w[3]), div_(w[2], w[3]));
}

// the oracle's bilinear SampleLevel with clamp addressing: 1/256-texel snap, weights ((1 - fx) * (1 - fy), ...), summed t00 .. t11 in order
DFX_HD float2 sample_lut(View<const float2> t, float u, float v)
{
    const auto  snap = [](float p) { return mul_(floorf(add_(mul_(p, 256.0f), 0.5f)), 1.0f / 256.0f); };
    const float px = snap(sub_(mul_(u, float(t.w)), 0.5f)), py = snap(sub_(mul_(v, float(t.h)), 0.5f));
    const float fx0 = floorf(px), fy0 = floorf(py);
    const int   x0 = int(fx0), y0 = int(fy0);
    const float fx = sub_(px, fx0), fy = sub_(py, fy0), gx = sub_(1.0f, fx), gy = sub_(1.0f, fy);
    const float w00 = mul_(gx, gy), w10 = mul_(fx, gy), w01 = mul_(gx, fy), w11 = mul_(fx, fy);
    const float2 a = loadc(t, x0, y0), b = loadc(t, x0 + 1, y0), c = loadc(t, x0, y0 + 1), d = loadc(t, x0 + 1, y0 + 1);
    return make_float2(add_(add_(add_(mul_(a.x, w00), mul_(b.x, w10)), mul_(c.x, w01)), mul_(d.x, w11)),
                       add_(add_(add_(mul_(a.y, w00), mul_(b.y, w10)), mul_(c.y, w01)), mul_(d.y, w11)));
}

__global__ void __launch_bounds__(256) compose_ibl_kernel(const dfx_camera_attribs* __restrict__ cams, View<const float4> color, View<const float4> ssr,
                                                          View<const float> ao, View<const float4> spec_ibl, View<const float4> normal,
                                                          View<const float4> base_color, View<const float4> material, View<const float2> lut,
                                                          float ssr_scale, float ssao_scale, View<float4> out, int y0, int y1)
{
    __shared__ ComposeCam S;
    if (threadIdx.x == 0 && threadIdx.y == 0) load_cam(S.c, &cams[0]), load_mat(S.vp_inv, cams[0].mViewProjInv);
    __syncthreads();
    const CamS&   cam = S.c;
    const PixelXY pix = cta_pixel(y0);
    const int     x = pix.x, y = pix.y;
    if (x >= out.w || y >= y1) return;
    const float4 C = __ldg(&color.at(x, y));
    float        c[3] = {C.x, C.y, C.z};
    const float  opacity = C.w;
    const float  s_ssr = mul_(ssr_scale, opacity);
    if (ssr.p && s_ssr > 0.0f)
    {
        const float4 ibl = __ldg(&spec_ibl.at(x, y)), r = __ldg(&ssr.at(x, y)), bc = __ldg(&base_color.at(x, y)), m = __ldg(&material.at(x, y));
        const float3 n     = xyz(__ldg(&normal.at(x, y)));
        const float  rough = sat_(m.x), metal = sat_(m.y);
        const float3 wp    = pixel_world_position(mul_(add_(float(x), 0.5f), cam.ivw), mul_(add_(float(y), 0.5f), cam.ivh), S.vp_inv);
        const float3 v     = normalize3(make_float3(sub_(cam.px, wp.x), sub_(cam.py, wp.y), sub_(cam.pz, wp.z)));
        const float  ndv   = sat_(dot3(n, v));
        const float2 pre   = sample_lut(lut, ndv, rough);
        const float  omr   = sub_(1.0f, rough);
        const float  t = fminf(fmaxf(sub_(1.0f, ndv), 0.0f), 1.0f), t2 = mul_(t, t), t5 = mul_(mul_(t2, t2), t); // SchlickReflection
        const float  bcv[3] = {bc.x, bc.y, bc.z}, rv[3] = {r.x, r.y, r.z}, iv[3] = {ibl.x, ibl.y, ibl.z};
#pragma unroll
        for (int k = 0; k < 3; ++k)
        {
            const float r0   = add_(0.04f, mul_(metal, sub_(bcv[k], 0.04f))); // lerp(f0, BaseColor, Metallic)
            const float ks   = add_(r0, mul_(sub_(fmaxf(omr, r0), r0), t5));
            const float spec = mul_(rv[k], add_(mul_(ks, pre.x), pre.y));
            c[k]             = add_(c[k], mul_(mul_(sub_(spec, iv[k]), r.w), s_ssr)); // left to right, as HnPostProcess.psh:170 multiplies
        }
    }
    const float s_ao = mul_(ssao_scale, opacity);
    if (ao.p && s_ao > 0.0f)
    {
        const float occ = add_(1.0f, mul_(s_ao, sub_(__ldg(&ao.at(x, y)), 1.0f))); // lerp(1, AO, SSAOScale * Opacity)
#pragma unroll
        for (int k = 0; k < 3; ++k) c[k] = mul_(c[k], occ);
    }
    st_cs(&out.at(x, y), make_float4(c[0], c[1], c[2], C.w));
}

} // namespace dfx

using namespace dfx;

extern "C" dfx_status dfx_pass_precompute_brdf_lut(void* stream, uint32_t num_samples, const dfx_plane* out_lut)
{
    DFX_PROFILE(stream, "precompute_brdf_lut");
    DFX_VIEW(float2, l, out_lut, DFX_FORMAT_RG32F);
    DFX_REQUIRE(num_samples > 0, "num_samples must be positive");
    dim3 block(32, kLutChunk / 32), grid(div_up(l.w, 32), div_up(l.h, int(kLutChunk / 32)));
    brdf_lut_kernel<<<grid, block, 0, as_stream(stream)>>>(l, num_samples);
    DFX_LAUNCHED("brdf_lut_kernel");
    return DFX_OK;
}

extern "C" dfx_status dfx_pass_compose_ibl(void* stream, const dfx_camera_attribs* cameras_dev, const dfx_plane* color, const dfx_plane* ssr,
                                           const dfx_plane* ao, const dfx_plane* specular_ibl, const dfx_plane* normal, const dfx_plane* base_color,
                                           const dfx_plane* material, const dfx_plane* brdf_lut, float ssr_scale, float ssao_scale, const dfx_plane* out,
                                           dfx_rows rows)
{
    DFX_PROFILE(stream, "compose_ibl");
    DFX_REQUIRE(cameras_dev, "null argument");
    DFX_VIEW(const float4, c, color, DFX_FORMAT_RGBA32F);
    DFX_VIEW(float4, o, out, DFX_FORMAT_RGBA32F);
    DFX_SAME_SIZE(c, o);
    View<const float4> s{nullptr, 0, 0, 0}, ibl{nullptr, 0, 0, 0}, n{nullptr, 0, 0, 0}, bc{nullptr, 0, 0, 0}, m{nullptr, 0, 0, 0};
    View<const float>  a{nullptr, 0, 0, 0};
    View<const float2> l{nullptr, 0, 0, 0};
    if (ssr)
    {
        DFX_REQUIRE(specular_ibl && normal && base_color && material && brdf_lut, "the SSR term needs the specular IBL, normal, base colour, material and BRDF table planes");
        DFX_REQUIRE(make_view<const float4>(ssr, DFX_FORMAT_RGBA32F, s) && make_view<const float4>(specular_ibl, DFX_FORMAT_RGBA32F, ibl) &&
                        make_view<const float4>(normal, DFX_FORMAT_RGBA32F, n) && make_view<const float4>(base_color, DFX_FORMAT_RGBA32F, bc) &&
                        make_view<const float4>(material, DFX_FORMAT_RGBA32F, m) && make_view<const float2>(brdf_lut, DFX_FORMAT_RG32F, l),
                    "bad plane (null, wrong format, pitch or alignment)");
        DFX_SAME_SIZE(c, s);
        DFX_SAME_SIZE(c, ibl);
        DFX_SAME_SIZE(c, n);
        DFX_SAME_SIZE(c, bc);
        DFX_SAME_SIZE(c, m);
    }
    if (ao)
    {
        DFX_REQUIRE(make_view<const float>(ao, DFX_FORMAT_R32F, a), "bad plane 'ao'");
        DFX_SAME_SIZE(c, a);
    }
    DFX_REQUIRE(rows_ok(rows, c.h), "bad row range");
    if (rows.y1 == rows.y0) return DFX_OK;
    dim3 block(32, 8), grid(div_up(c.w, 32), div_up(rows.y1 - rows.y0, 8));
    compose_ibl_kernel<<<grid, block, 0, as_stream(stream)>>>(cameras_dev, c, s, a, ibl, n, bc, m, l, ssr_scale, ssao_scale, o, rows.y0, rows.y1);
    DFX_LAUNCHED("compose_ibl_kernel");
    return DFX_OK;
}
