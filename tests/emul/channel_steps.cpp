// tests/emul/channel_steps.cpp — TEST INFRASTRUCTURE, never shipped: dxb200_apply_channel_steps on the host, with the entry point's
// own signature.  It plans the call with the library's planner (dxb_plan.h) and runs the per-pixel rule the generic k_convert runs
// (dxb_channel_steps.h) on every pixel, so that the CPU suite can hold the library's steps against the reference's TransformImage
// without a device.  emul_plan_mipmaps_compress_from_channels reports what dxb200_mipmaps_compress_from_channels would return
// before it touches a device, and the plan it would stage.
#include <cstdint>
#include <cstddef>
#include <cstring>
#include <vector>

#include "dxb_portable.h"
#include "dxb_formats.h"
#include "dxb_plan.h"
#include "dxb_pixel.cuh"
#include "dxb_channel_steps.h"

extern "C" int32_t emul_apply_channel_steps(const dxb200_image* src, size_t n, const dxb200_channel_steps* steps, const dxb200_image* dst)
{
    dxb_convert_params P;
    const int32_t hr = plan_channel_steps(src, n, steps, dst, &P);
    if (hr != DXB_S_OK) return hr;
    for (size_t i = 0; i < n; ++i)
        for (size_t y = 0; y < src[i].height; ++y)
            for (size_t x = 0; x < src[i].width; ++x)
                dxb_channel_steps_pixel(P.srcFormat, src[i].pixels + y * src[i].rowPitch, dst[i].pixels + y * dst[i].rowPitch, x, P.steps,
                                        P.key[0], P.key[1], P.key[2]);
    return DXB_S_OK;
}

// out (may be NULL) = { decompress, resize, channel steps, decompress format, level-0 format, level-0 width, level-0 height, step
// word }, filled on S_OK
extern "C" int32_t emul_plan_mipmaps_compress_from_channels(const dxb200_image* base, size_t items, const dxb200_chain_source* source,
                                                           const dxb200_channel_steps* channels, size_t levels, uint32_t filter,
                                                           const dxb200_chain_steps* steps, uint32_t dstFormat, uint32_t flags, float threshold,
                                                           float alphaWeight, const dxb200_image* dst, uint64_t* out)
{
    (void)alphaWeight;
    FromPlan fp;
    const int32_t hr = plan_mipmaps_compress_channels(base, items, source, channels, levels, filter, steps, dstFormat, flags, threshold, dst, &fp);
    if (hr == DXB_S_OK && out)
    {
        const dxb200_image& l0 = fp.chain.chain[0];
        out[0] = fp.decompress; out[1] = fp.resize; out[2] = fp.channels; out[3] = fp.decompress ? fp.dp.dstFormat : 0;
        out[4] = l0.format; out[5] = l0.width; out[6] = l0.height; out[7] = fp.channels ? fp.cp.steps : 0;
    }
    return hr;
}

// the format a BC base decompresses to in dxb200_mipmaps_compress_from_channels with decompressFormat == 0
extern "C" uint32_t emul_channel_decompress_format(uint32_t bcFormat, const dxb200_channel_steps* channels)
{
    return channel_decompress_format(bcFormat, channels);
}

// the UNORM bit reconstruct Z runs with for an implemented format (DXB_CONVF_UNORM of dxb_convert_flags)
extern "C" int emul_channel_unorm(uint32_t fmt)
{
    return (dxb_convert_flags(fmt) & DXB_CONVF_UNORM) ? 1 : 0;
}
