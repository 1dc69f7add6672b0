// tests/emul/levels_from.cpp — TEST INFRASTRUCTURE, never shipped: the planner of dxb200_levels_from (dxb_plan.h) on the host, with
// the entry point's own signature, so that the CPU suite can hold its HRESULTs against the library's without a device.  It also
// reports the plan a valid call would stage, and the same report of the planners of dxb200_mipmaps_compress_from_channels and
// dxb200_mipmaps_convert_from, so that a one-level plan can be held against theirs.
#include <cstdint>
#include <cstddef>
#include <cstring>
#include <vector>

#include "dxb_portable.h"
#include "dxb_formats.h"
#include "dxb_plan.h"

// out = { decompress, resize, channel steps before the Convert (all of them without one), Convert, channel steps after it,
// premultiply, compress, mips, coverage, the decompress format (0: no decompress), the working format (what the front steps leave),
// the first channel launch's step word, pass-through (a BC base that is neither decompressed nor compressed) }
static void report(const FromPlan& fp, const dxb200_image* base, uint64_t* out)
{
    out[0] = fp.decompress; out[1] = fp.resize; out[2] = fp.channels; out[3] = fp.convert; out[4] = fp.post;
    out[5] = fp.chain.premultiply; out[6] = fp.chain.compressed; out[7] = fp.chain.generate; out[8] = fp.chain.coverage;
    out[9] = fp.decompress ? fp.dp.dstFormat : 0; out[10] = fp.level0.empty() ? base[0].format : fp.level0[0].format;
    out[11] = fp.channels ? fp.cp.steps : 0;
    out[12] = is_compressed(base[0].format) && !fp.decompress && !fp.chain.compressed;
}

// out (may be NULL, 14 words) = report(), then the alpha scan; filled on S_OK
extern "C" int32_t emul_plan_levels_from(const dxb200_image* base, size_t items, size_t levels, const dxb200_chain_source* source,
                                         const dxb200_channel_steps* channels, uint32_t dstFormat, uint32_t convertFilter, uint32_t compressFlags,
                                         float threshold, const dxb200_chain_steps* steps, const dxb200_image* dst, int32_t* alphaAllOpaque,
                                         uint64_t* out)
{
    FromPlan fp;
    AlphaOpaquePlan ap;
    const int32_t hr = plan_levels_from(base, items, levels, source, channels, dstFormat, convertFilter, compressFlags, threshold, steps, dst,
                                        alphaAllOpaque, &fp, &ap);
    if (hr == DXB_S_OK && out)
    {
        report(fp, base, out);
        out[13] = ap.scan;
    }
    return hr;
}

// report() of the generating call with the same arguments: dxb200_mipmaps_compress_from_channels for a BC dstFormat (mip filter 0),
// dxb200_mipmaps_convert_from otherwise; base[i] = level 0 of item i, dst[i * levels + l] its chain
extern "C" int32_t emul_plan_generating(const dxb200_image* base, size_t items, size_t levels, const dxb200_chain_source* source,
                                        const dxb200_channel_steps* channels, uint32_t dstFormat, uint32_t convertFilter, uint32_t compressFlags,
                                        float threshold, const dxb200_chain_steps* steps, const dxb200_image* dst, uint64_t* out)
{
    FromPlan fp;
    AlphaOpaquePlan ap;
    const int32_t hr = is_compressed(dstFormat)
        ? plan_mipmaps_compress_channels(base, items, source, channels, levels, 0, steps, dstFormat, compressFlags, threshold, dst, &fp)
        : plan_mipmaps_convert_from(base, items, source, channels, dstFormat, convertFilter, threshold, levels, 0, steps, dst, nullptr, &fp, &ap);
    if (hr == DXB_S_OK && out) report(fp, base, out);
    return hr;
}
