// ORACLE — TEST INFRASTRUCTURE ONLY. DepthRangeCalculator::ComputeRange (Components/src/DepthRangeCalculator.cpp:229-272) restated
// from its two compute shaders, statement by statement: ClearDepthRange.csh, then ComputeDepthRange.csh run one 8x8 group at a time,
// each phase between two GroupMemoryBarrierWithGroupSync() over all 64 threads of the group, with g_MinMaxDepth as the group's
// shared array and the Interlocked* as integer min / max on the output. min / max are std::fmin / std::fmax, as the reference's
// shader runner evaluates HLSL's min / max (oracle/refshader/hlsl.hpp). Scalar C++, the flags of oracle/Makefile.
#include <cmath>
#include <cstdint>
#include <cstring>

#include "../include/dfx_b200.h"

#define ORACLE_API extern "C" __attribute__((visibility("default")))

namespace
{
constexpr unsigned kThreadGroupSize = 8; // DepthRangeCalculator.cpp:37

int32_t asint(float f)
{
    int32_t i;
    std::memcpy(&i, &f, 4);
    return i;
}

// ShaderUtilities.fxh:24-39 with DepthToNormalizedDeviceZ(d) = d
float depth_to_camera_z(float d, const dfx_float4x4& P) { return (P.m[3][2] - d * P.m[3][3]) / (d * P.m[2][3] - P.m[2][2]); }

struct Group
{
    const dfx_camera_attribs& cam;
    const float*              depth;
    unsigned                  w, h;

    // UpdateMinMaxDepth (ComputeDepthRange.csh:15-26)
    void update(unsigned x, unsigned y, float& mn, float& mx) const
    {
        x             = x < w - 1u ? x : w - 1u; // PixelCoords = min(PixelCoords, DepthDim - 1)
        y             = y < h - 1u ? y : h - 1u;
        const float D = depth[size_t(y) * w + x];
        if (D != cam.fFarPlaneDepth)
        {
            mn = std::fmin(mn, D);
            mx = std::fmax(mx, D);
        }
    }
};
} // namespace

// depth: w x h floats, row-major. out: iSceneNearZ, iSceneFarZ, iSceneNearDepth, iSceneFarDepth as the int bits of floats.
ORACLE_API void ordr_depth_range(const dfx_camera_attribs* cam_, const float* depth, int w, int h, float* out)
{
    const dfx_camera_attribs& C = *cam_;
    // ClearDepthRange.csh
    int32_t R[4] = {asint(C.fFarPlaneZ), asint(C.fNearPlaneZ), asint(C.fFarPlaneDepth), asint(C.fNearPlaneDepth)};
    enum { NEAR_Z, FAR_Z, NEAR_DEPTH, FAR_DEPTH };
    const Group    G{C, depth, unsigned(w), unsigned(h)};
    const unsigned T = kThreadGroupSize, groups_x = (unsigned(w) + 2 * T - 1) / (2 * T), groups_y = (unsigned(h) + 2 * T - 1) / (2 * T);
    for (unsigned gy = 0; gy < groups_y; ++gy)
        for (unsigned gx = 0; gx < groups_x; ++gx)
        {
            float MinDepth[kThreadGroupSize][kThreadGroupSize], MaxDepth[kThreadGroupSize][kThreadGroupSize]; // each thread's locals, [x][y]
            float g_MinMaxDepth[kThreadGroupSize][kThreadGroupSize][2];
            for (unsigned tx = 0; tx < T; ++tx)
                for (unsigned ty = 0; ty < T; ++ty)
                {
                    const unsigned x = (gx * T + tx) * 2u, y = (gy * T + ty) * 2u; // DispatchID.xy * 2
                    float          mn = 1.0f, mx = 0.0f;
                    G.update(x + 0u, y + 0u, mn, mx);
                    G.update(x + 0u, y + 1u, mn, mx);
                    G.update(x + 1u, y + 0u, mn, mx);
                    G.update(x + 1u, y + 1u, mn, mx);
                    MinDepth[tx][ty] = mn, MaxDepth[tx][ty] = mx;
                    g_MinMaxDepth[tx][ty][0] = mn, g_MinMaxDepth[tx][ty][1] = mx;
                }
            // GroupMemoryBarrierWithGroupSync(): the min / max of each row of the group
            for (unsigned ty = 0; ty < T; ++ty)
            {
                for (unsigned i = 1; i < T; ++i)
                {
                    MinDepth[0][ty] = std::fmin(MinDepth[0][ty], g_MinMaxDepth[i][ty][0]);
                    MaxDepth[0][ty] = std::fmax(MaxDepth[0][ty], g_MinMaxDepth[i][ty][1]);
                }
                g_MinMaxDepth[0][ty][0] = MinDepth[0][ty], g_MinMaxDepth[0][ty][1] = MaxDepth[0][ty];
            }
            // GroupMemoryBarrierWithGroupSync(): the min / max of the whole group
            for (unsigned j = 1; j < T; ++j)
            {
                MinDepth[0][0] = std::fmin(MinDepth[0][0], g_MinMaxDepth[0][j][0]);
                MaxDepth[0][0] = std::fmax(MaxDepth[0][0], g_MinMaxDepth[0][j][1]);
            }
            for (unsigned tx = 0; tx < T; ++tx)
                for (unsigned ty = 0; ty < T; ++ty)
                {
                    const float mn = MinDepth[tx][ty], mx = MaxDepth[tx][ty];
                    const float MinZ = depth_to_camera_z(mn, C.mProj), MaxZ = depth_to_camera_z(mx, C.mProj);
                    auto        imin = [&](int f, float v) { R[f] = asint(v) < R[f] ? asint(v) : R[f]; };
                    auto        imax = [&](int f, float v) { R[f] = asint(v) > R[f] ? asint(v) : R[f]; };
                    if (C.fNearPlaneDepth <= C.fFarPlaneDepth)
                    {
                        imin(NEAR_DEPTH, mn), imax(FAR_DEPTH, mx), imin(NEAR_Z, MinZ), imax(FAR_Z, MaxZ);
                    }
                    else
                    {
                        imin(FAR_DEPTH, mn), imax(NEAR_DEPTH, mx), imin(NEAR_Z, MaxZ), imax(FAR_Z, MinZ);
                    }
                }
        }
    std::memcpy(out, R, sizeof(R));
}
