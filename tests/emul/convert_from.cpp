// tests/emul/convert_from.cpp — TEST INFRASTRUCTURE, never shipped: the planner of dxb200_mipmaps_convert_from (dxb_plan.h) on the
// host, with the entry point's own signature, so that the CPU suite can hold its HRESULTs against the library's without a device.
// It also reports the plan a valid call would stage: which launches a chunk runs, the Convert's source format and the chain's
// level 0.
#include <cstdint>
#include <cstddef>
#include <cstring>
#include <vector>

#include "dxb_portable.h"
#include "dxb_formats.h"
#include "dxb_plan.h"

// out (may be NULL) = { decompress, resize, channel steps before the Convert (all of them without one), Convert, channel steps after
// it, the Convert's source format (0: none), level-0 format, level-0 width, level-0 height, level-0 row pitch, the first channel
// launch's step word, alpha scan }, filled on S_OK
extern "C" int32_t emul_plan_mipmaps_convert_from(const dxb200_image* base, size_t items, const dxb200_chain_source* source,
                                                  const dxb200_channel_steps* channels, uint32_t dstFormat, uint32_t convertFilter, float threshold,
                                                  size_t levels, uint32_t filter, const dxb200_chain_steps* steps, const dxb200_image* dst,
                                                  int32_t* alphaAllOpaque, uint64_t* out)
{
    FromPlan fp;
    AlphaOpaquePlan ap;
    const int32_t hr = plan_mipmaps_convert_from(base, items, source, channels, dstFormat, convertFilter, threshold, levels, filter, steps, dst,
                                                 alphaAllOpaque, &fp, &ap);
    if (hr == DXB_S_OK && out)
    {
        const dxb200_image& l0 = fp.chain.chain[0];
        out[0] = fp.decompress; out[1] = fp.resize; out[2] = fp.channels; out[3] = fp.convert; out[4] = fp.post;
        out[5] = fp.convert ? fp.cv.srcFormat : 0; out[6] = l0.format; out[7] = l0.width; out[8] = l0.height; out[9] = l0.rowPitch;
        out[10] = fp.channels ? fp.cp.steps : 0; out[11] = ap.scan;
    }
    return hr;
}
