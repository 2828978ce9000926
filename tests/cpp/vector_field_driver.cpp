// vector_field_driver.cpp — drives Diligent::VectorFieldRenderer (include/dfx/VectorFieldRenderer.hpp) the way HnPostProcessTask does: a
// renderer per target format, Render with the field, the grid, the scale and the colours over the bound colour target, twice (the
// renderer's scratch plane must come back zero for the second draw to be the first's). Host-only translation unit (g++, no CUDA headers):
// everything goes through the C++ header and the C-ABI.
//
//   vector_field_driver <dir> <width> <height> <field width> <field height> <grid x> <grid y> <scale> <srgb>
// reads <dir>/field.bin (fp32 RG) and color.bin (fp32 RGBA); writes <dir>/out_color.bin and out_color2.bin.
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "dfx/VectorFieldRenderer.hpp"

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
    if (argc != 10) return 1;
    const std::string dir = argv[1];
    const Uint32      w = Uint32(std::atoi(argv[2])), h = Uint32(std::atoi(argv[3])), fw = Uint32(std::atoi(argv[4])), fh = Uint32(std::atoi(argv[5]));
    const Uint32      gx = Uint32(std::atoi(argv[6])), gy = Uint32(std::atoi(argv[7]));
    const float       scale = float(std::atof(argv[8]));
    const bool        srgb  = std::atoi(argv[9]) != 0;

    IRenderDevice  device;
    IDeviceContext ctx{nullptr};
    ITexture       field{fw, fh, TEX_FORMAT_RG32_FLOAT}, color{w, h, TEX_FORMAT_RGBA32_FLOAT};
    const std::vector<char> c0 = read_file(dir + "/color.bin", size_t(w) * h * 16);
    if (!field.UpdateData(&ctx, read_file(dir + "/field.bin", size_t(fw) * fh * 8).data()) || !color.UpdateData(&ctx, c0.data())) return 3;

    VectorFieldRenderer::CreateInfo ci;
    ci.pDevice = &device;
    VectorFieldRenderer renderer{ci};

    ITextureView                       fv{&field}, rtv{&color};
    VectorFieldRenderer::RenderAttribs ra;
    ra.pContext     = &ctx;
    ra.pVectorField = &fv;
    ra.pColorRTV    = &rtv;
    ra.Scale[0] = ra.Scale[1] = scale;
    for (int k = 0; k < 3; ++k) ra.EndColor[k] = 0.5f;
    ra.GridSize[0]         = gx;
    ra.GridSize[1]         = gy;
    ra.ConvertOutputToSRGB = srgb;
    std::vector<float> out(size_t(w) * h * 4);
    for (int pass = 0; pass < 2; ++pass)
    {
        if (pass == 1 && !color.UpdateData(&ctx, c0.data())) return 4;
        renderer.Render(ra);
        if (!color.ReadData(&ctx, out.data())) return 5;
        write_file(dir + (pass ? "/out_color2.bin" : "/out_color.bin"), out.data(), out.size() * 4);
    }
    std::printf("vector_field_driver: %ux%u, field %ux%u, grid %ux%u, scale %g, srgb %d\n", w, h, fw, fh, gx, gy, double(scale), int(srgb));
    return 0;
}
