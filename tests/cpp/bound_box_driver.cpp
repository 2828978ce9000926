// bound_box_driver.cpp — drives Diligent::BoundBoxRenderer (include/dfx/BoundBoxRenderer.hpp) the way an application does: a camera
// buffer in device memory at construction, Prepare with the render attribs, Render into the bound colour / motion targets.
// Host-only translation unit (g++, no CUDA headers): everything goes through the C++ header and the C-ABI.
//
//   bound_box_driver <dir> <width> <height> <options> <pattern length> <pattern mask>
// reads <dir>/depth.bin (fp32), color.bin (fp32 RGBA), motion.bin (fp32 RG), cameras.bin (2 x 576 B), transform.bin (16 fp32) and
// rgba.bin (4 fp32); writes <dir>/out_color.bin and out_motion.bin.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "dfx/BoundBoxRenderer.hpp"

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
    if (argc != 7) return 1;
    const std::string dir = argv[1];
    const Uint32      w = Uint32(std::atoi(argv[2])), h = Uint32(std::atoi(argv[3]));
    const auto        options = static_cast<BoundBoxRenderer::OPTION_FLAGS>(std::atoi(argv[4]));
    const float       length  = float(std::atof(argv[5]));
    const Uint32      mask    = Uint32(std::strtoul(argv[6], nullptr, 0));
    const size_t      px      = size_t(w) * h;

    IRenderDevice  device;
    IDeviceContext ctx{nullptr};
    ITexture       depth_tex{w, h, TEX_FORMAT_D32_FLOAT}, color{w, h, TEX_FORMAT_RGBA32_FLOAT}, motion{w, h, TEX_FORMAT_RG32_FLOAT};
    ITexture       cams{Uint32(2 * sizeof(dfx_camera_attribs) / 4), 1, TEX_FORMAT_R32_FLOAT};
    if (!depth_tex.UpdateData(&ctx, read_file(dir + "/depth.bin", px * 4).data()) || !color.UpdateData(&ctx, read_file(dir + "/color.bin", px * 16).data()) ||
        !motion.UpdateData(&ctx, read_file(dir + "/motion.bin", px * 8).data()) ||
        !cams.UpdateData(&ctx, read_file(dir + "/cameras.bin", 2 * sizeof(dfx_camera_attribs)).data()))
        return 3;
    dfx_float4x4            transform;
    const std::vector<char> t = read_file(dir + "/transform.bin", sizeof(transform)), rgba = read_file(dir + "/rgba.bin", 16);
    std::memcpy(&transform, t.data(), sizeof(transform));
    float col[4];
    std::memcpy(col, rgba.data(), 16);

    IBuffer                      cb{cams.GetPlane().ptr};
    BoundBoxRenderer::CreateInfo ci;
    ci.pDevice          = &device;
    ci.pCameraAttribsCB = &cb;
    ci.RenderTargetMask = 0x3u;
    BoundBoxRenderer renderer{ci};

    BoundBoxRenderer::RenderAttribs ra;
    ra.BoundBoxTransform = &transform;
    ra.Color             = col;
    ra.PatternLength     = length;
    ra.PatternMask       = mask;
    ra.Options           = options;
    renderer.Prepare(&ctx, ra);

    ITextureView rtv{&color}, mv{&motion}, dsv{&depth_tex};
    renderer.Render(&ctx, BoundBoxRenderer::Targets{&rtv, &mv, &dsv});

    std::vector<float> out(px * 4);
    if (!color.ReadData(&ctx, out.data())) return 5;
    write_file(dir + "/out_color.bin", out.data(), px * 16);
    if (!motion.ReadData(&ctx, out.data())) return 6;
    write_file(dir + "/out_motion.bin", out.data(), px * 8);
    std::printf("bound_box_driver: %ux%u, options %u, pattern %g / 0x%08x\n", w, h, unsigned(options), double(length), mask);
    return 0;
}
