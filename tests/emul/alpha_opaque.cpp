// tests/emul/alpha_opaque.cpp — TEST INFRASTRUCTURE, never shipped: dxb200_is_alpha_all_opaque on the host, with the entry point's
// own signature.  It plans the call with the library's planner (dxb_plan.h) and walks every image with the per-texel rule the
// device scan runs (dxb_alpha_opaque.h) on the same block decoders and pixel loads (dxb_decode.cuh, dxb_pixel.cuh), so that the
// CPU suite can hold the library's answers against the reference without a device.  emul_plan_mipmaps_compress_from_ex reports
// what dxb200_mipmaps_compress_from_ex would return before it touches a device.
#include <cstdint>
#include <cstddef>
#include <cstring>
#include <vector>

#include "dxb_portable.h"
#include "dxb_formats.h"
#include "dxb_plan.h"
#include "dxb_pixel.cuh"
#include "dxb_decode.cuh"
#include "dxb_alpha_opaque.h"

extern "C" int32_t emul_is_alpha_all_opaque(const dxb200_image* images, size_t n, int32_t* opaque)
{
    AlphaOpaquePlan ap;
    const int32_t hr = plan_alpha_opaque(images, n, opaque, &ap);
    if (hr != DXB_S_OK) return hr;
    bool any = false;
    for (size_t i = 0; i < n && ap.scan; ++i)
    {
        const dxb200_image& im = images[i];
        if (ap.blocks)
        {
            const uint32_t bs = dxb_bc_block_bytes(ap.format);
            for (size_t by = 0; by < (im.height + 3) / 4; ++by)
                for (size_t bx = 0; bx < (im.width + 3) / 4; ++bx)
                {
                    alignas(16) uint8_t blk[16];
                    memcpy(blk, im.pixels + by * im.rowPitch + bx * bs, bs);
                    dxb_px px[16];
                    dxb_decode_block(ap.format, blk, px);
                    const uint32_t pw = (uint32_t)std::min<size_t>(4, im.width - bx * 4), ph = (uint32_t)std::min<size_t>(4, im.height - by * 4);
                    any |= dxb_block_not_opaque(px, pw, ph);
                }
        }
        else
        {
            for (size_t y = 0; y < im.height; ++y)
                for (size_t x = 0; x < im.width; ++x)
                    any |= dxb_alpha_not_opaque(dxb_load_pixel(ap.format, im.pixels + y * im.rowPitch, x).w, DXB_OPAQUE_PIXEL);
        }
    }
    *opaque = any ? 0 : 1;
    return DXB_S_OK;
}

// the HRESULT of dxb200_mipmaps_compress_from_ex's planning; *scan = 1 when the call would scan its output (alphaAllOpaque given and
// dstFormat with alpha)
extern "C" int32_t emul_plan_mipmaps_compress_from_ex(const dxb200_image* base, size_t items, const dxb200_chain_source* source, size_t levels,
                                                      uint32_t filter, const dxb200_chain_steps* steps, uint32_t dstFormat, uint32_t flags,
                                                      float threshold, float alphaWeight, const dxb200_image* dst, int32_t* alphaAllOpaque,
                                                      int32_t* scan)
{
    (void)alphaWeight;
    FromPlan fp;
    int32_t hr = plan_mipmaps_compress_from(base, items, source, levels, filter, steps, dstFormat, flags, threshold, dst, &fp);
    AlphaOpaquePlan ap = {};
    if (hr == DXB_S_OK && alphaAllOpaque) hr = plan_alpha_opaque(dst, items * levels, alphaAllOpaque, &ap);
    *scan = ap.scan ? 1 : 0;
    return hr;
}
