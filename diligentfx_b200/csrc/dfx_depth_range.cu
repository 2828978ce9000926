// dfx_depth_range.cu — R, the scene's depth range: DepthRangeCalculator::ComputeRange (Components/src/DepthRangeCalculator.cpp:229-272),
// i.e. ClearDepthRange.csh, then ComputeDepthRange.csh over ceil(W/16) x ceil(H/16) groups of 8x8 threads, and the read-back of
// DepthRangeCalculator's ReadBackData.
//
// What the shader computes. Every thread folds its 2x2 block (coordinates clamped to the plane, background D == fFarPlaneDepth skipped)
// into float min / max seeded with 1 / 0; thread (0, y) then folds the 7 other threads of its row into its own (a 16x2-pixel row
// partial), and thread (0, 0) folds rows 1..7 into row 0's (the 16x16 group partial). Every thread then issues integer
// InterlockedMin / InterlockedMax of asint() of what it holds, and of asint(DepthToCameraZ()) of it. So the result is the integer
// min / max over a fixed set of partials and does not depend on the order the groups run in; for non-negative depths it is the
// plain min / max, while for negative depths and -0 the grouping decides the answer (integer order reverses negative floats).
//
// Here one warp is one group: lane (tx, ty) plays the shader's threads (tx, ty) and (tx, ty + 4). The row and group partials are the
// shader's left folds, evaluated as trees of shuffles. That is exact because the fold operator is associative: min_ / max_ below are
// the C library's fminf / fmaxf as the reference's shader runner evaluates them (a NaN operand yields the other one; of +0 and -0 the
// second operand wins), so a fold picks the last of the extreme values, whatever the bracketing. NaN never reaches a partial (the
// seeds are not NaN). The integer reductions are redux.sync; each CTA keeps its running min / max over the groups it strides through
// and issues one atomic per field.
//
// Two launches: the clear (one thread, the camera's far / near values) and the reduction. R always reduces the whole plane and takes
// no row range, because the shader's groups are anchored at row 0.
#include "dfx_common.cuh"
#include "dfx_grid.cuh"
#include <algorithm>
#include <climits>
#include <cstring>
#include <new>
#include <vector>

namespace dfx
{
namespace
{
constexpr int kWarps = 8; // 256 threads, one group per warp and stride

__device__ __forceinline__ float min_(float a, float b) { return (a < b || b != b) ? a : b; }
__device__ __forceinline__ float max_(float a, float b) { return (a > b || b != b) ? a : b; }

// DepthToCameraZ of a partial. An infinite partial makes it NaN (inf * 0, inf - inf), and asint() of that NaN is what the atomics see.
// The GPU's arithmetic generates 0x7fffffff, x86's (the reference's shader runner, and the oracle) 0xffc00000; the shader itself
// leaves it to the hardware. R returns the x86 NaN, so that its result is one defined value.
__device__ __forceinline__ float camera_z(float d, const dfx_camera_attribs& C)
{
    const float z = depth_to_camz_ieee(d, C);
    return z != z ? __int_as_float(int(0xffc00000u)) : z;
}

// UpdateMinMaxDepth (ComputeDepthRange.csh:15-26)
__device__ __forceinline__ void update(const View<const float>& d, unsigned x, unsigned y, float far_depth, float& mn, float& mx)
{
    x             = min(x, unsigned(d.w) - 1u);
    y             = min(y, unsigned(d.h) - 1u);
    const float D = d.ld(int(x), int(y));
    if (D != far_depth)
    {
        mn = min_(mn, D);
        mx = max_(mx, D);
    }
}

// the ordered fold of the lanes l, l + step, ..., l + (n - 1) * step into lane l
template <int STEP, int N>
__device__ __forceinline__ void fold(float& mn, float& mx)
{
#pragma unroll
    for (int off = STEP; off < STEP * N; off *= 2)
    {
        mn = min_(mn, __shfl_down_sync(0xffffffffu, mn, off));
        mx = max_(mx, __shfl_down_sync(0xffffffffu, mx, off));
    }
}

__global__ void depth_range_clear_kernel(const dfx_camera_attribs* __restrict__ cams, int* __restrict__ out)
{
    // ClearDepthRange.csh: iSceneNearZ, iSceneFarZ, iSceneNearDepth, iSceneFarDepth
    const dfx_camera_attribs& C = cams[0];
    out[0]                      = __float_as_int(C.fFarPlaneZ);
    out[1]                      = __float_as_int(C.fNearPlaneZ);
    out[2]                      = __float_as_int(C.fFarPlaneDepth);
    out[3]                      = __float_as_int(C.fNearPlaneDepth);
}

__global__ void __launch_bounds__(kWarps * 32) depth_range_kernel(const dfx_camera_attribs* __restrict__ cams, View<const float> d, int groups_x, int groups,
                                                                 int* __restrict__ out)
{
    const dfx_camera_attribs& C         = cams[0];
    const float               far_depth = C.fFarPlaneDepth;
    const bool                reversed  = !(C.fNearPlaneDepth <= C.fFarPlaneDepth);
    const int                 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned            tx = lane & 7, ty = lane >> 3;
    // running integer min of asint(min depth) / max of asint(max depth) / min of asint(near Z) / max of asint(far Z)
    int acc0 = INT_MAX, acc1 = INT_MIN, acc2 = INT_MAX, acc3 = INT_MIN;
    for (int g = blockIdx.x * kWarps + warp; g < groups; g += gridDim.x * kWarps)
    {
        const unsigned gx = unsigned(g % groups_x), gy = unsigned(g / groups_x);
        float          v[2][2]; // [shader thread row ty, ty + 4][min, max]
#pragma unroll
        for (int k = 0; k < 2; ++k)
        {
            const unsigned x = (gx * 8u + tx) * 2u, y = (gy * 8u + ty + 4u * k) * 2u;
            float          mn = 1.0f, mx = 0.0f;
            update(d, x, y, far_depth, mn, mx);
            update(d, x, y + 1u, far_depth, mn, mx);
            update(d, x + 1u, y, far_depth, mn, mx);
            update(d, x + 1u, y + 1u, far_depth, mn, mx);
            v[k][0] = mn, v[k][1] = mx;
        }
        float row[2][2], grp[2][2];
#pragma unroll
        for (int k = 0; k < 2; ++k)
        {
            row[k][0] = v[k][0], row[k][1] = v[k][1];
            fold<1, 8>(row[k][0], row[k][1]); // lane 8r: the row partial of shader row r (+ 4k)
            grp[k][0] = row[k][0], grp[k][1] = row[k][1];
            fold<8, 4>(grp[k][0], grp[k][1]); // lane 0: rows 4k .. 4k + 3
        }
        // what each shader thread holds when it issues its atomics
        const float gmn = min_(grp[0][0], grp[1][0]), gmx = max_(grp[0][1], grp[1][1]);
        float       h[2][2];
        h[0][0] = tx ? v[0][0] : ty ? row[0][0] : gmn;
        h[0][1] = tx ? v[0][1] : ty ? row[0][1] : gmx;
        h[1][0] = tx ? v[1][0] : row[1][0];
        h[1][1] = tx ? v[1][1] : row[1][1];
        int i0 = INT_MAX, i1 = INT_MIN, i2 = INT_MAX, i3 = INT_MIN;
#pragma unroll
        for (int k = 0; k < 2; ++k)
        {
            const float min_z = camera_z(h[k][0], C), max_z = camera_z(h[k][1], C);
            i0 = min(i0, __float_as_int(h[k][0]));
            i1 = max(i1, __float_as_int(h[k][1]));
            // reversed depth: the maximum depth is the near plane (ComputeDepthRange.csh:80-88)
            i2 = min(i2, __float_as_int(reversed ? max_z : min_z));
            i3 = max(i3, __float_as_int(reversed ? min_z : max_z));
        }
        acc0 = min(acc0, __reduce_min_sync(0xffffffffu, i0));
        acc1 = max(acc1, __reduce_max_sync(0xffffffffu, i1));
        acc2 = min(acc2, __reduce_min_sync(0xffffffffu, i2));
        acc3 = max(acc3, __reduce_max_sync(0xffffffffu, i3));
    }
    __shared__ int s[kWarps][4];
    if (lane == 0) s[warp][0] = acc0, s[warp][1] = acc1, s[warp][2] = acc2, s[warp][3] = acc3;
    __syncthreads();
    if (threadIdx.x != 0) return;
#pragma unroll
    for (int w = 1; w < kWarps; ++w) acc0 = min(acc0, s[w][0]), acc1 = max(acc1, s[w][1]), acc2 = min(acc2, s[w][2]), acc3 = max(acc3, s[w][3]);
    atomicMin(out + 0, acc2);                // iSceneNearZ
    atomicMax(out + 1, acc3);                // iSceneFarZ
    atomicMin(out + (reversed ? 3 : 2), acc0); // iSceneNearDepth, or iSceneFarDepth with reversed depth
    atomicMax(out + (reversed ? 2 : 3), acc1); // iSceneFarDepth, or iSceneNearDepth with reversed depth
}
} // namespace
} // namespace dfx

using namespace dfx;

extern "C" dfx_status dfx_pass_depth_range(void* stream, const dfx_camera_attribs* cameras_dev, const dfx_plane* depth_, float* out_dev)
{
    DFX_PROFILE(stream, "depth_range");
    DFX_REQUIRE(cameras_dev && out_dev, "null argument");
    DFX_REQUIRE(reinterpret_cast<uintptr_t>(out_dev) % 4 == 0, "out_dev must be 4-byte aligned");
    DFX_VIEW(const float, d, depth_, DFX_FORMAT_R32F);
    const int    groups_x = div_up(d.w, 16), groups = groups_x * div_up(d.h, 16);
    int          dev = 0, sms = 0;
    cudaStream_t s = as_stream(stream);
    DFX_CUDA(cudaGetDevice(&dev));
    DFX_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    int* out = reinterpret_cast<int*>(out_dev);
    depth_range_clear_kernel<<<1, 1, 0, s>>>(cameras_dev, out);
    DFX_LAUNCHED("depth_range_clear_kernel");
    const int blocks = std::min(div_up(groups, kWarps), sms * (2048 / (kWarps * 32)));
    depth_range_kernel<<<blocks, kWarps * 32, 0, s>>>(cameras_dev, d, groups_x, groups, out);
    DFX_LAUNCHED("depth_range_kernel");
    return DFX_OK;
}

// ---- DepthRangeCalculator (DepthRangeCalculator.hpp:62-176) --------------------------------------------------------------------------
// The read-back goes to pinned host slots, each with the event of its copy. get_range polls the events without waiting and keeps the
// range of the latest compute whose copy has completed (an older copy that completes later does not replace it). Like the reference's
// GPUCompletionAwaitQueue, which creates a staging buffer when none is recycled, a compute that finds every slot still in flight adds
// one, so every compute is read back; the number of slots is bounded by the computes in flight at once.
struct ReadBackSlot
{
    float*      host = nullptr; // 4 floats, pinned
    cudaEvent_t ev   = nullptr;
    uint64_t    seq  = 0; // issue number of the copy in flight; 0 = free
};

struct dfx_depth_range
{
    static constexpr int      kInitialSlots = 4;
    float*                    buf_dev       = nullptr; // DepthRangeI: fSceneNearZ, fSceneFarZ, fSceneNearDepth, fSceneFarDepth
    bool                      read_back     = false;
    std::vector<ReadBackSlot> slots;
    uint64_t                  issued = 0, newest = 0;
    dfx_scene_depth_range     range{};
    ~dfx_depth_range()
    {
        for (ReadBackSlot& k : slots)
        {
            if (k.ev) cudaEventDestroy(k.ev);
            cudaFreeHost(k.host);
        }
        cudaFree(buf_dev);
    }
};

static cudaError_t add_slot(dfx_depth_range* fx)
{
    ReadBackSlot k;
    cudaError_t  e = cudaMallocHost((void**)&k.host, sizeof(dfx_scene_depth_range));
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&k.ev, cudaEventDisableTiming);
    if (e != cudaSuccess)
    {
        if (k.host) cudaFreeHost(k.host);
        return e;
    }
    fx->slots.push_back(k);
    return cudaSuccess;
}

static dfx_status poll_read_back(dfx_depth_range* fx)
{
    for (ReadBackSlot& k : fx->slots)
    {
        if (!k.seq) continue;
        const cudaError_t e = cudaEventQuery(k.ev);
        if (e == cudaErrorNotReady) continue;
        if (e != cudaSuccess) return check_cuda(e, "dfx_depth_range: cudaEventQuery");
        if (k.seq > fx->newest)
        {
            fx->newest = k.seq;
            std::memcpy(&fx->range, k.host, sizeof(fx->range));
        }
        k.seq = 0;
    }
    return DFX_OK;
}

extern "C" dfx_status dfx_depth_range_create(int32_t read_back, dfx_depth_range** out)
{
    DFX_REQUIRE(out, "out must not be null");
    dfx_depth_range* fx = new (std::nothrow) dfx_depth_range;
    DFX_REQUIRE(fx, "out of memory");
    fx->read_back = read_back != 0;
    cudaError_t e = cudaMalloc((void**)&fx->buf_dev, sizeof(dfx_scene_depth_range));
    if (e == cudaSuccess) e = cudaMemset(fx->buf_dev, 0, sizeof(dfx_scene_depth_range));
    for (int k = 0; fx->read_back && k < dfx_depth_range::kInitialSlots && e == cudaSuccess; ++k) e = add_slot(fx);
    if (e != cudaSuccess)
    {
        delete fx;
        return check_cuda(e, "dfx_depth_range_create");
    }
    *out = fx;
    return DFX_OK;
}

extern "C" void dfx_depth_range_destroy(dfx_depth_range* fx) { delete fx; }

extern "C" dfx_status dfx_depth_range_compute(dfx_depth_range* fx, void* stream, const dfx_camera_attribs* cameras_dev, const dfx_plane* depth)
{
    DFX_REQUIRE(fx, "null argument");
    EffectRange nvtx_range("DepthRangeCalculator");
    dfx_status  st = dfx_pass_depth_range(stream, cameras_dev, depth, fx->buf_dev);
    if (st != DFX_OK || !fx->read_back) return st;
    if ((st = poll_read_back(fx)) != DFX_OK) return st;
    size_t k = 0;
    while (k < fx->slots.size() && fx->slots[k].seq) ++k;
    if (k == fx->slots.size()) DFX_CUDA(add_slot(fx));
    ReadBackSlot& slot = fx->slots[k];
    cudaStream_t  s    = as_stream(stream);
    DFX_CUDA(cudaMemcpyAsync(slot.host, fx->buf_dev, sizeof(dfx_scene_depth_range), cudaMemcpyDeviceToHost, s));
    DFX_CUDA(cudaEventRecord(slot.ev, s));
    slot.seq = ++fx->issued;
    return DFX_OK;
}

extern "C" float* dfx_depth_range_get_buffer(const dfx_depth_range* fx) { return fx ? fx->buf_dev : nullptr; }

extern "C" dfx_status dfx_depth_range_get_range(dfx_depth_range* fx, int32_t poll, dfx_scene_depth_range* out)
{
    DFX_REQUIRE(fx && out, "null argument");
    if (poll)
    {
        const dfx_status st = poll_read_back(fx);
        if (st != DFX_OK) return st;
    }
    *out = fx->range;
    return DFX_OK;
}
