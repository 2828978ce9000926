// depth_range_driver.cpp — drives Diligent::DepthRangeCalculator (include/dfx/DepthRangeCalculator.hpp) the way
// HnComputeDepthBoundsTask does: CreateSRB on the depth buffer and a camera in device memory, ComputeRange, then the device buffer and
// the read-back range. Host-only translation unit (g++, no CUDA headers): everything goes through the C++ header and the C-ABI.
//
//   depth_range_driver <dir> <width> <height>
// reads <dir>/depth.bin (fp32) and camera.bin (576 B); writes <dir>/out_buffer.bin (the device buffer, 16 B) and out_readback.bin
// (GetDepthRange after the context is idle, 16 B). Exits with 7 if the range read back before the first ComputeRange is not all zeros.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "dfx/DepthRangeCalculator.hpp"

using namespace Diligent;

static std::vector<char> read_file(const std::string& path, size_t bytes)
{
    std::vector<char> b(bytes);
    FILE*             f = std::fopen(path.c_str(), "rb");
    if (!f || std::fread(b.data(), 1, bytes, f) != bytes)
    {
        std::fprintf(stderr, "cannot read %zu bytes from %s\n", bytes, path.c_str());
        std::exit(2);
    }
    std::fclose(f);
    return b;
}
static void write_file(const std::string& path, const void* p, size_t n)
{
    FILE* f = std::fopen(path.c_str(), "wb");
    std::fwrite(p, 1, n, f);
    std::fclose(f);
}

int main(int argc, char** argv)
{
    if (argc != 4) return 1;
    const std::string dir = argv[1];
    const Uint32      w = Uint32(std::atoi(argv[2])), h = Uint32(std::atoi(argv[3]));

    std::vector<char> depth = read_file(dir + "/depth.bin", size_t(w) * h * 4);
    std::vector<char> cam   = read_file(dir + "/camera.bin", sizeof(HLSL::CameraAttribs));

    IDeviceContext ctx{nullptr};
    ITexture       depth_tex{w, h, TEX_FORMAT_D32_FLOAT};
    ITextureView   depth_srv{&depth_tex};
    // the camera constant buffer, filled by the application: one CameraAttribs in device memory
    ITexture cb_mem{Uint32(sizeof(dfx_camera_attribs) / 4), 1, TEX_FORMAT_R32_FLOAT};
    if (!depth_tex.UpdateData(&ctx, depth.data()) || !cb_mem.UpdateData(&ctx, cam.data())) return 3;
    IBuffer cb{cb_mem.GetPlane().ptr};

    DepthRangeCalculator::CreateInfo CI;
    CI.ReadBackData = true;
    DepthRangeCalculator calc{CI};
    if (!calc.IsReady()) return 4;
    const DepthRangeCalculator::DepthRange r0 = calc.GetDepthRange(&ctx);
    if (r0 || r0.fSceneNearZ != 0 || r0.fSceneFarZ != 0 || r0.fSceneNearDepth != 0 || r0.fSceneFarDepth != 0) return 7;

    auto                                      srb = calc.CreateSRB(&depth_srv, &cb);
    DepthRangeCalculator::ComputeRangeAttribs a;
    a.pContext = &ctx;
    a.pSRB     = srb.get();
    a.Width    = w;
    a.Height   = h;
    calc.ComputeRange(a);

    // the depth range buffer seen as a 4x1 R32F plane
    dfx_plane buf_plane{};
    const DepthRangeCalculator& const_calc = calc; // GetDepthRangeBuffer() is const, as in the reference
    buf_plane.ptr                          = const_cast<void*>(const_calc.GetDepthRangeBuffer()->GetDevicePtr());
    buf_plane.pitch_bytes = 16;
    buf_plane.width       = 4;
    buf_plane.height      = 1;
    buf_plane.format      = DFX_FORMAT_R32F;
    ITexture buf_tex{buf_plane};
    float    buf[4];
    if (!buf_tex.ReadData(&ctx, buf)) return 5;
    write_file(dir + "/out_buffer.bin", buf, sizeof(buf));

    ctx.WaitForIdle();
    const DepthRangeCalculator::DepthRange& r = calc.GetDepthRange(&ctx);
    const float                             rb[4] = {r.fSceneNearZ, r.fSceneFarZ, r.fSceneNearDepth, r.fSceneFarDepth};
    write_file(dir + "/out_readback.bin", rb, sizeof(rb));
    std::printf("depth_range_driver: %ux%u, range %s\n", w, h, r ? "valid" : "empty");
    return 0;
}
