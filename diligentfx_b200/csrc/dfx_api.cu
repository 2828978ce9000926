// dfx_api.cu — status / error plumbing, attribute defaults, host-side helpers and device-plane utilities of the C-ABI.
#include "dfx_common.cuh"
#include "dfx_tma.cuh"
#include <nvtx3/nvToolsExt.h> // header-only: resolves the tool's injection library at run time, no link dependency
#include <tuple>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cmath>
#include <string>
#include <vector>
#include <map>
#include <mutex>
#include <cstdlib>

namespace dfx
{
static thread_local char          g_err[512] = "";
static std::atomic<unsigned long long> g_launches{0};

dfx_status set_error(dfx_status st, const char* fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return st;
}
dfx_status check_cuda(cudaError_t e, const char* what)
{
    if (e == cudaSuccess) return DFX_OK;
    return set_error(DFX_ERR_CUDA, "%s: %s (%s)", what, cudaGetErrorString(e), cudaGetErrorName(e));
}
void count_launch(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

// ---- optional per-pass device timing -------------------------------------------------------------------------------
struct ProfileRecord
{
    const char* name;
    cudaEvent_t a, b;
};
static bool                        g_profile_on = false;
static std::vector<ProfileRecord>  g_records;
static std::vector<cudaEvent_t>    g_event_pool;
struct ProfileEntry
{
    std::string name;
    double      total_ms;
    int         calls;
};
static std::vector<ProfileEntry> g_entries;

static cudaEvent_t take_event()
{
    if (!g_event_pool.empty())
    {
        cudaEvent_t e = g_event_pool.back();
        g_event_pool.pop_back();
        return e;
    }
    cudaEvent_t e = nullptr;
    cudaEventCreate(&e);
    return e;
}

// NVTX range per pass, named like the reference's ScopedDebugGroup of the draw(s) the pass stands for (e.g. Bloom.cpp:298, :320;
// ScreenSpaceAmbientOcclusion.cpp:820 ff.), so that a timeline of this library reads like a capture of the reference.
static const char* reference_group_name(const char* pass)
{
    static const struct { const char *pass, *group; } kNames[] = {
        {"blue_noise", "ComputeBlueNoiseTexture"}, {"postfx_prepare", "ComputeReprojectedDepth+ComputeClosestMotion+ComputePreviousDepth"},
        {"ssao_downsample_depth", "ComputeDownsampledDepth"}, {"ssao_prefilter_depth", "ComputePrefilteredDepth"}, {"ssao_ambient_occlusion", "ComputeAmbientOcclusion"},
        {"ssao_upsample", "ComputeBilateralUpsampling"}, {"ssao_temporal", "ComputeTemporalAccumulation"}, {"ssao_convolute", "ComputeConvolutedDepthHistory"},
        {"ssao_resample", "ComputeResampledHistory"}, {"ssao_spatial", "ComputeSpatialReconstruction"},
        {"front_prepare", "ComputeReprojectedDepth+ComputeClosestMotion+ComputePreviousDepth+ComputeHierarchicalDepthBuffer+ComputeStencilMaskAndExtractRoughness+ComputePrefilteredDepth"},
        {"ssr_hiz", "ComputeHierarchicalDepthBuffer"}, {"ssr_mask_roughness", "ComputeStencilMaskAndExtractRoughness"}, {"ssr_downsample_mask", "ComputeDownsampledStencilMask"},
        {"ssr_intersect", "ComputeIntersection"}, {"ssr_intersect_peer", "ComputeIntersection"}, {"ssr_spatial", "ComputeSpatialReconstruction"},
        {"ssr_temporal", "ComputeTemporalAccumulation"}, {"ssr_temporal_peer", "ComputeTemporalAccumulation"}, {"ssr_bilateral", "ComputeBilateralCleanup"},
        {"bloom_prefilter", "ComputePrefilteredTexture"}, {"bloom_downsample", "ComputeDownsampledTexture"}, {"bloom_tail", "ComputeDownsampledTexture+ComputeUpsampledTexture"},
        {"bloom_upsample", "ComputeUpsampledTexture"}, {"bloom_composite", "ComputeUpsampledTexture"}, {"bloom_composite_tonemap", "ComputeUpsampledTexture+ToneMap"},
        {"taa", "TemporalAccumulation"}, {"compose_taa", "HnPostProcess+TemporalAccumulation"}, {"compose", "HnPostProcess"}, {"tonemap", "ToneMap"},
        {"dof_coc", "ComputeCircleOfConfusion"}, {"dof_temporal_coc", "ComputeTemporalCircleOfConfusion"}, {"dof_separated_coc", "ComputeSeparatedCircleOfConfusion"},
        {"dof_dilation", "ComputeHierarchicalCoC"}, {"dof_blur_coc", "ComputeCircleOfConfusionBlur"}, {"dof_prefilter", "ComputePrefilteredTexture"},
        {"dof_postfilter", "ComputePostFilteredTexture"}, {"dof_combine", "ComputeCombinedTexture"}};
    for (const auto& n : kNames)
        if (strcmp(n.pass, pass) == 0) return n.group;
    return pass;
}

ProfileScope::ProfileScope(void* stream, const char* name) : s(static_cast<cudaStream_t>(stream)), slot(-1)
{
    nvtxRangePushA(reference_group_name(name));
    if (!g_profile_on) return;
    ProfileRecord r{name, take_event(), take_event()};
    cudaEventRecord(r.a, s);
    slot = (int)g_records.size();
    g_records.push_back(r);
}
ProfileScope::~ProfileScope()
{
    if (slot >= 0) cudaEventRecord(g_records[slot].b, s);
    nvtxRangePop();
}

// fill of a plane in one of the renderer's narrow formats: `bpc` bytes per channel (2 = half, 1 = UNORM8), `ch` channels
__global__ void fill_narrow_kernel(unsigned char* p, size_t pitch, int w, int h, int ch, int bpc, float4 v)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= w * ch || y >= h) return;
    const int   c = x % ch;
    const float s = c == 0 ? v.x : c == 1 ? v.y : c == 2 ? v.z : v.w;
    if (bpc == 2)
        reinterpret_cast<__half*>(p + size_t(y) * pitch)[x] = __float2half_rn(s);
    else
        (p + size_t(y) * pitch)[x] = (unsigned char)__fmaf_rn(fminf(fmaxf(s, 0.0f), 1.0f), 255.0f, 0.5f);
}

EffectRange::EffectRange(const char* name) { nvtxRangePushA(name); }
EffectRange::~EffectRange() { nvtxRangePop(); }

__global__ void fill_kernel(float* p, int pitch_f, int wf, int h, int ch, float4 v)
{
    int x = blockIdx.x * blockDim.x + threadIdx.x;
    int y = blockIdx.y;
    if (x >= wf || y >= h) return;
    int   c = x % ch;
    float s = c == 0 ? v.x : c == 1 ? v.y : c == 2 ? v.z : v.w;
    p[(size_t)y * pitch_f + x] = s;
}
} // namespace dfx

using namespace dfx;

extern "C"
{
const char* dfx_last_error(void) { return g_err; }
int         dfx_version(void) { return 100; } // 0.1.0
uint64_t    dfx_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

void dfx_ssao_attribs_default(dfx_ssao_attribs* a)
{
    // ScreenSpaceAmbientOcclusionStructures.fxh:64-98
    *a = dfx_ssao_attribs{1.0f, 0.615f, 1.457f, 3.3f, 0.9f, 4.0f, 0, 1.0f, 0.5f, DFX_SSAO_ALGORITHM_GTAO, 0.0f, 0.0f};
}
void dfx_ssr_attribs_default(dfx_ssr_attribs* a)
{
    // ScreenSpaceReflectionStructures.fxh:43-80
    *a = dfx_ssr_attribs{0.025f, 0.2f, 0u, 1, 0u, 128u, 0.3f, 4.0f, 1.0f, 0.9f, 0.9f, 1.0f};
}
void dfx_bloom_attribs_default(dfx_bloom_attribs* a)
{
    // BloomStructures.fxh:12-34
    *a = dfx_bloom_attribs{0.15f, 1.0f, 0.125f, 0.75f, 1.0f, 0.0f, 0.0f, 0.0f};
}
void dfx_dof_attribs_default(dfx_dof_attribs* a)
{
    // DepthOfFieldStructures.fxh:31-56
    *a = dfx_dof_attribs{0.01f, 0.9375f, 5, 7, 1.0f, 0.0f, 0.0f, 0.0f};
}
void dfx_taa_attribs_default(dfx_taa_attribs* a)
{
    // TemporalAntiAliasingStructures.fxh:35-46
    *a = dfx_taa_attribs{0.9375f, 0, 0, 0.0f};
}
void dfx_tonemap_attribs_default(dfx_tonemap_attribs* a)
{
    // ToneMappingStructures.fxh:24-52
    *a = dfx_tonemap_attribs{DFX_TONE_MAPPING_MODE_UNCHARTED2, 1, 0.18f, 1, 3.0f, 1.0f, 0u, 0u, 1.0f, 1.0f, 1.0f, 0.0f};
}

// TemporalAntiAliasing.cpp:43-54
static float halton_sequence(uint32_t Base, uint32_t Index)
{
    float Result = 0.0f, F = 1.0f;
    while (Index > 0)
    {
        F      = F / static_cast<float>(Base);
        Result = Result + F * static_cast<float>(Index % Base);
        Index  = static_cast<uint32_t>(floorf(static_cast<float>(Index) / static_cast<float>(Base)));
    }
    return Result;
}
// TemporalAntiAliasing.cpp:63-78
void dfx_taa_jitter_offset(uint32_t frame_index, uint32_t width, uint32_t height, float out[2])
{
    const uint32_t SampleCount = 16u;
    out[0] = (halton_sequence(2u, (frame_index % SampleCount) + 1) - 0.5f) / (0.5f * static_cast<float>(width));
    out[1] = (halton_sequence(3u, (frame_index % SampleCount) + 1) - 0.5f) / (0.5f * static_cast<float>(height));
}
// Bloom.cpp:152-156 with DiligentCore's ComputeMipLevelsCount (levels down to 1 of the larger dimension)
int32_t dfx_bloom_mip_count(uint32_t width, uint32_t height, float radius)
{
    uint32_t m = width > height ? width : height, n = 0;
    while (m > 0) ++n, m >>= 1;
    return static_cast<int32_t>(radius * static_cast<float>(n));
}

static size_t bytes_per_texel(int fmt)
{
    switch (fmt)
    {
        case DFX_FORMAT_R32F: return 4;
        case DFX_FORMAT_RG32F: return 8;
        case DFX_FORMAT_RGBA32F: return 16;
        case DFX_FORMAT_R8U: return 1;
        case DFX_FORMAT_RGBA16F: return 8;
        case DFX_FORMAT_RG16F: return 4;
        case DFX_FORMAT_RG8U: return 2;
        case DFX_FORMAT_RGBA8U: return 4;
        case DFX_FORMAT_R16U: return 2;
        case DFX_FORMAT_RG16U: return 4;
        default: return 0;
    }
}

dfx_status dfx_plane_alloc(int32_t width, int32_t height, int32_t format, dfx_plane* out)
{
    DFX_REQUIRE(out != nullptr, "out must not be null");
    size_t bpt = bytes_per_texel(format);
    DFX_REQUIRE(bpt != 0 && width > 0 && height > 0, "bad plane description %dx%d fmt %d", width, height, format);
    // rows padded to 128 B so every row start is a full-line boundary (coalesced 128-bit access, TMA-compatible pitch)
    size_t pitch = ((size_t)width * bpt + 127) / 128 * 128;
    void*  p     = nullptr;
    DFX_CUDA(cudaMalloc(&p, pitch * (size_t)height));
    out->ptr = p, out->pitch_bytes = pitch, out->width = width, out->height = height, out->format = format, out->flags = 0;
    return DFX_OK;
}
void dfx_plane_free(dfx_plane* p)
{
    if (p && p->ptr) cudaFree(p->ptr), p->ptr = nullptr;
}
dfx_status dfx_plane_upload(void* stream, const dfx_plane* dst, const void* host_src, size_t host_pitch)
{
    DFX_REQUIRE(dst && dst->ptr && host_src, "null argument");
    size_t row = (size_t)dst->width * bytes_per_texel(dst->format);
    DFX_CUDA(cudaMemcpy2DAsync(dst->ptr, dst->pitch_bytes, host_src, host_pitch ? host_pitch : row, row, dst->height, cudaMemcpyHostToDevice, as_stream(stream)));
    return DFX_OK;
}
dfx_status dfx_plane_download(void* stream, const dfx_plane* src, void* host_dst, size_t host_pitch)
{
    DFX_REQUIRE(src && src->ptr && host_dst, "null argument");
    size_t row = (size_t)src->width * bytes_per_texel(src->format);
    DFX_CUDA(cudaMemcpy2DAsync(host_dst, host_pitch ? host_pitch : row, src->ptr, src->pitch_bytes, row, src->height, cudaMemcpyDeviceToHost, as_stream(stream)));
    return DFX_OK;
}
dfx_status dfx_plane_fill(void* stream, const dfx_plane* dst, const float value[4])
{
    DFX_REQUIRE(dst && dst->ptr && value, "null argument");
    DFX_REQUIRE(dst->format != DFX_FORMAT_R16U && dst->format != DFX_FORMAT_RG16U, "dfx_plane_fill does not fill the UNORM16 shadow-map formats");
    if (dst->format == DFX_FORMAT_R8U)
    {
        DFX_CUDA(cudaMemset2DAsync(dst->ptr, dst->pitch_bytes, value[0] != 0.0f ? 1 : 0, dst->width, dst->height, as_stream(stream)));
        return DFX_OK;
    }
    if (dst->format == DFX_FORMAT_RGBA16F || dst->format == DFX_FORMAT_RG16F || dst->format == DFX_FORMAT_RG8U || dst->format == DFX_FORMAT_RGBA8U)
    {
        const int nch = (dst->format == DFX_FORMAT_RGBA16F || dst->format == DFX_FORMAT_RGBA8U) ? 4 : 2, bpc = (dst->format == DFX_FORMAT_RGBA16F || dst->format == DFX_FORMAT_RG16F) ? 2 : 1;
        fill_narrow_kernel<<<dim3(div_up(dst->width * nch, 256), dst->height), 256, 0, as_stream(stream)>>>(static_cast<unsigned char*>(dst->ptr), dst->pitch_bytes, dst->width, dst->height,
                                                                                                         nch, bpc, make_float4(value[0], value[1], value[2], value[3]));
        DFX_LAUNCHED("fill_narrow_kernel");
        return DFX_OK;
    }
    int ch = dst->format == DFX_FORMAT_R32F ? 1 : dst->format == DFX_FORMAT_RG32F ? 2 : 4;
    int wf = dst->width * ch;
    dim3 grid(div_up(wf, 256), dst->height);
    fill_kernel<<<grid, 256, 0, as_stream(stream)>>>(static_cast<float*>(dst->ptr), int(dst->pitch_bytes / 4), wf, dst->height, ch,
                                                     make_float4(value[0], value[1], value[2], value[3]));
    DFX_LAUNCHED("fill_kernel");
    return DFX_OK;
}
dfx_status dfx_stream_synchronize(void* stream)
{
    DFX_CUDA(cudaStreamSynchronize(as_stream(stream)));
    return DFX_OK;
}

dfx_status dfx_enable_peer_access(int32_t peer_device)
{
    int dev = -1, can = 0;
    DFX_CUDA(cudaGetDevice(&dev));
    if (dev == peer_device) return DFX_OK;
    DFX_CUDA(cudaDeviceCanAccessPeer(&can, dev, peer_device));
    if (!can) return dfx::set_error(DFX_ERR_UNSUPPORTED, "device %d has no peer path to device %d", dev, peer_device);
    const cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
    if (e == cudaErrorPeerAccessAlreadyEnabled)
    {
        (void)cudaGetLastError();
        return DFX_OK;
    }
    DFX_CUDA(e);
    return DFX_OK;
}

dfx_status dfx_ipc_alloc(size_t bytes, void** out_ptr, uint8_t handle[DFX_IPC_HANDLE_BYTES])
{
    static_assert(sizeof(cudaIpcMemHandle_t) == DFX_IPC_HANDLE_BYTES, "IPC handle size");
    DFX_REQUIRE(out_ptr && handle && bytes > 0, "null argument");
    void* p = nullptr;
    DFX_CUDA(cudaMalloc(&p, bytes));
    cudaIpcMemHandle_t h;
    const cudaError_t  e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess)
    {
        cudaFree(p);
        DFX_CUDA(e);
    }
    memcpy(handle, &h, sizeof(h));
    *out_ptr = p;
    return DFX_OK;
}
dfx_status dfx_ipc_free(void* ptr)
{
    if (ptr) DFX_CUDA(cudaFree(ptr));
    return DFX_OK;
}
dfx_status dfx_ipc_open(const uint8_t handle[DFX_IPC_HANDLE_BYTES], void** out_ptr)
{
    DFX_REQUIRE(out_ptr && handle, "null argument");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof(h));
    // mapped into the CURRENT device's address space; peer access to the owning device is enabled as needed
    DFX_CUDA(cudaIpcOpenMemHandle(out_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return DFX_OK;
}
dfx_status dfx_ipc_close(void* mapped)
{
    if (mapped) DFX_CUDA(cudaIpcCloseMemHandle(mapped));
    return DFX_OK;
}

void dfx_profile_enable(int32_t on) { g_profile_on = on != 0; }

dfx_status dfx_profile_collect(void)
{
    // waits for the recorded events and folds them into per-pass totals (first-seen order)
    for (const ProfileRecord& r : g_records)
    {
        DFX_CUDA(cudaEventSynchronize(r.b));
        float ms = 0.0f;
        DFX_CUDA(cudaEventElapsedTime(&ms, r.a, r.b));
        size_t i = 0;
        for (; i < g_entries.size(); ++i)
            if (g_entries[i].name == r.name) break;
        if (i == g_entries.size()) g_entries.push_back(ProfileEntry{r.name, 0.0, 0});
        g_entries[i].total_ms += ms;
        g_entries[i].calls += 1;
        g_event_pool.push_back(r.a);
        g_event_pool.push_back(r.b);
    }
    g_records.clear();
    return DFX_OK;
}
// ---- implementation switches (A/B measurements) ----------------------------------------------------------------------
static std::mutex                 g_tune_mutex;
static std::map<std::string, int> g_tune;
static bool                       g_tune_env_read = false;
static void tune_read_env()
{
    if (g_tune_env_read) return;
    g_tune_env_read = true;
    const char* e = getenv("DFX_TUNE");
    if (!e) return;
    std::string s(e);
    size_t      pos = 0;
    while (pos < s.size())
    {
        size_t end = s.find(',', pos);
        if (end == std::string::npos) end = s.size();
        const std::string kv = s.substr(pos, end - pos);
        const size_t      eq = kv.find('=');
        if (eq != std::string::npos) g_tune.emplace(kv.substr(0, eq), atoi(kv.c_str() + eq + 1));
        pos = end + 1;
    }
}
void dfx_tune_set(const char* name, int32_t value)
{
    if (!name) return;
    std::lock_guard<std::mutex> lk(g_tune_mutex);
    tune_read_env();
    g_tune[name] = value;
}
void dfx_tune_unset(const char* name)
{
    std::lock_guard<std::mutex> lk(g_tune_mutex);
    tune_read_env();
    if (name)
        g_tune.erase(name);
    else
        g_tune.clear();
}
int32_t dfx_tune_get(const char* name, int32_t fallback)
{
    if (!name) return fallback;
    std::lock_guard<std::mutex> lk(g_tune_mutex);
    tune_read_env();
    auto it = g_tune.find(name);
    return it == g_tune.end() ? fallback : it->second;
}

} // extern "C"
namespace dfx
{
int  tune(const char* name, int fallback) { return dfx_tune_get(name, fallback); }
// Set by the chain executor while it issues (or records) a frame whose SSR and SSAO halves run side by side on two streams.
static thread_local bool t_async_compute = false;
bool async_compute_hint() { return t_async_compute; }
void set_async_compute_hint(bool on) { t_async_compute = on; }
bool profiling_enabled() { return g_profile_on; }

// Tensor maps are encoded once per (plane, box) and cached: a frame touches a dozen planes, and encoding costs a driver call.
const CUtensorMap* tensor_map_r32f(const View<float>& plane, int box_w, int box_h)
{
    static std::mutex                                                                  m;
    static std::map<std::tuple<const void*, int, int, int, int, int>, CUtensorMap>     cache;
    std::lock_guard<std::mutex>                                                        lk(m);
    const auto key = std::make_tuple(static_cast<const void*>(plane.p), plane.w, plane.h, plane.pitch, box_w, box_h);
    auto       it  = cache.find(key);
    if (it != cache.end()) return &it->second;
    CUtensorMap map;
    if (!make_tensor_map_r32f(&map, plane.p, plane.w, plane.h, size_t(plane.pitch) * sizeof(float), box_w, box_h)) return nullptr;
    if (cache.size() > 4096) cache.clear(); // planes come and go with their owners; the cache only ever saves the encode call
    return &cache.emplace(key, map).first->second;
}
} // namespace dfx
extern "C"
{
void    dfx_profile_reset(void) { dfx_profile_collect(), g_entries.clear(); }
int32_t dfx_profile_count(void) { return (int32_t)g_entries.size(); }
dfx_status dfx_profile_entry(int32_t i, char* name, int32_t name_cap, double* total_ms, int32_t* calls)
{
    DFX_REQUIRE(i >= 0 && i < (int32_t)g_entries.size() && name && name_cap > 0 && total_ms && calls, "bad profile entry query");
    snprintf(name, (size_t)name_cap, "%s", g_entries[i].name.c_str());
    *total_ms = g_entries[i].total_ms;
    *calls    = g_entries[i].calls;
    return DFX_OK;
}
} // extern "C"
