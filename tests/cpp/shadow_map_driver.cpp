// shadow_map_driver.cpp — drives Diligent::ShadowMapManager (include/dfx/ShadowMapManager.hpp) the way an application does: Initialize
// with an InitInfo, write each cascade's depth through GetCascadeDSV(i) (standing in for the application's depth pass), then
// ConvertToFilterable with the ShadowMapAttribs the application filled, and read the filterable slices back through GetFilterableSRV(i).
// Host-only translation unit: everything goes through the C++ header and the C-ABI.
//
//   shadow_map_driver <dir> <resolution> <cascades> <mode> <is32> <d16>
// reads <dir>/depth.bin (cascades x resolution^2 texels, uint16 D16 codes or float32) and <dir>/attribs.bin (ShadowMapAttribs, 1200
// bytes), writes <dir>/filterable.bin (the filterable slices one after another, tightly packed texels of the filterable format).
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include "dfx/ShadowMapManager.hpp"

using namespace Diligent;

static std::vector<unsigned char> read_file(const std::string& path)
{
    std::vector<unsigned char> b;
    if (FILE* f = std::fopen(path.c_str(), "rb"))
    {
        unsigned char chunk[65536];
        for (size_t k; (k = std::fread(chunk, 1, sizeof(chunk), f)) > 0;) b.insert(b.end(), chunk, chunk + k);
        std::fclose(f);
    }
    return b;
}

int main(int argc, char** argv)
{
    if (argc != 7) return 2;
    const std::string dir = argv[1];
    const Uint32      res = Uint32(std::stoul(argv[2])), n = Uint32(std::stoul(argv[3]));
    const int         mode = std::stoi(argv[4]);
    const bool        is32 = std::stoi(argv[5]) != 0, d16 = std::stoi(argv[6]) != 0;

    HLSL::ShadowMapAttribs attribs;
    const std::vector<unsigned char> ab = read_file(dir + "/attribs.bin"), depth = read_file(dir + "/depth.bin");
    const size_t in_bpt = d16 ? 2 : 4, slice = size_t(res) * res * in_bpt;
    if (ab.size() != sizeof(attribs) || depth.size() != slice * n) return 3;
    std::memcpy(static_cast<dfx_shadow_map_attribs*>(&attribs), ab.data(), sizeof(attribs));

    ShadowMapManager::InitInfo init;
    init.Format               = d16 ? TEX_FORMAT_D16_UNORM : TEX_FORMAT_D32_FLOAT;
    init.Resolution           = res;
    init.NumCascades          = n;
    init.ShadowMode           = mode;
    init.Is32BitFilterableFmt = is32;
    ShadowMapManager smm;
    IRenderDevice    device;
    smm.Initialize(&device, nullptr, init);

    IDeviceContext ctx;
    for (Uint32 i = 0; i < n; ++i)
        if (!smm.GetCascadeDSV(i)->GetTexture()->UpdateData(&ctx, depth.data() + i * slice)) return 4;
    smm.ConvertToFilterable(&ctx, attribs);

    const size_t out_bpt = mode == SHADOW_MODE_EVSM4 ? (is32 ? 16 : 8) : (is32 ? 8 : 4);
    std::vector<unsigned char> out(size_t(res) * res * out_bpt * n);
    for (Uint32 i = 0; i < n; ++i)
        if (!smm.GetFilterableSRV(i)->GetTexture()->ReadData(&ctx, out.data() + i * size_t(res) * res * out_bpt)) return 5;
    FILE* f = std::fopen((dir + "/filterable.bin").c_str(), "wb");
    if (!f || std::fwrite(out.data(), 1, out.size(), f) != out.size()) return 6;
    std::fclose(f);
    std::printf("ok: %u cascades of %u^2, mode %d, %s-bit\n", n, res, mode, is32 ? "32" : "16");
    return 0;
}
