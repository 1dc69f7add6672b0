// tests/emul/from_plan.cpp — TEST INFRASTRUCTURE, never shipped: the planner of dxb200_mipmaps_compress_from (dxb_plan.h) on the
// host, with the entry point's own signature, so that the CPU suite can hold its HRESULTs against the library's without a device.
// It also reports the plan a valid call would stage: which front steps run and the format and size of the chain's level 0.
#include <cstdint>
#include <cstddef>
#include <cstring>
#include <vector>

#include "dxb_portable.h"
#include "dxb_formats.h"
#include "dxb_plan.h"

// out (may be NULL) = { decompress, resize, level-0 format, level-0 width, level-0 height, level-0 row pitch }, filled on S_OK
extern "C" int32_t emul_plan_mipmaps_compress_from(const dxb200_image* base, size_t items, const dxb200_chain_source* source, size_t levels,
                                                   uint32_t filter, const dxb200_chain_steps* steps, uint32_t dstFormat, uint32_t flags,
                                                   float threshold, float alphaWeight, const dxb200_image* dst, uint64_t* out)
{
    (void)alphaWeight;
    FromPlan fp;
    const int32_t hr = plan_mipmaps_compress_from(base, items, source, levels, filter, steps, dstFormat, flags, threshold, dst, &fp);
    if (hr == DXB_S_OK && out)
    {
        const dxb200_image& l0 = fp.chain.chain[0];
        out[0] = fp.decompress; out[1] = fp.resize; out[2] = l0.format; out[3] = l0.width; out[4] = l0.height; out[5] = l0.rowPitch;
    }
    return hr;
}
