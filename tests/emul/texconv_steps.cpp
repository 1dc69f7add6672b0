// tests/emul/texconv_steps.cpp — TEST INFRASTRUCTURE, never shipped: the planners of dxb200_mipmaps_compress_from_channels_ex,
// dxb200_mipmaps_convert_from_ex and dxb200_levels_from_ex (dxb_plan.h) on the host, with the entry points' own signatures, so that
// the CPU suite can hold their HRESULTs against the library's without a device.  Each also reports the plan a valid call would
// stage, and emul_chunk_plan the planes and steps of its chunks.
#include <cstdint>
#include <cstddef>
#include <cstring>
#include <vector>

#include "dxb_portable.h"
#include "dxb_formats.h"
#include "dxb_plan.h"

// out = { decompress, demultiply, resize, channel steps before the Convert (all of them without one), Convert, channel steps after
// it, generate (mips), coverage, premultiply, BC3 layout, compress, the decompress format (0: no decompress), the working format (what
// the front steps leave), the demultiply's launch flags, the layout's step word, pass-through (a BC base that is neither decompressed
// nor compressed), alpha scan }
constexpr int NOUT = 17;

static void report(const FromPlan& fp, const AlphaOpaquePlan& ap, const dxb200_image* base, uint64_t* out)
{
    const ChainPlan& cp = fp.chain;
    out[0] = fp.decompress; out[1] = fp.demultiply; out[2] = fp.resize; out[3] = fp.channels; out[4] = fp.convert; out[5] = fp.post;
    out[6] = cp.generate; out[7] = cp.coverage; out[8] = cp.premultiply; out[9] = cp.layout; out[10] = cp.compressed;
    out[11] = fp.decompress ? fp.dp.dstFormat : 0; out[12] = fp.level0.empty() ? base[0].format : fp.level0[0].format;
    out[13] = fp.demultiply ? fp.dm.flags : 0; out[14] = cp.layout ? cp.lp.steps : 0;
    out[15] = is_compressed(base[0].format) && !fp.decompress && !cp.compressed;
    out[16] = ap.scan;
}

// the chunk plan of the last valid call (run_chains' planes and steps), for emul_chunk_plan
static ChunkPlan last;

// out = { plane count, step count, per, filter, item 0's weight, then { role, per, first copy, rest copy } of every plane and
// { kind, source role, destination role, cover } of every step }; returns the words written, at most cap
extern "C" size_t emul_chunk_plan(uint64_t* out, size_t cap)
{
    std::vector<uint64_t> w = { last.planes.size(), last.steps.size(), last.per, last.filter, last.weight.empty() ? 0 : last.weight[0] };
    for (const ChunkPlane& p : last.planes) w.insert(w.end(), { (uint64_t)p.role, p.per, (uint64_t)p.first, (uint64_t)p.rest });
    for (const ChunkStep& s : last.steps) w.insert(w.end(), { (uint64_t)s.kind, (uint64_t)s.src, (uint64_t)s.dst, (uint64_t)s.cover });
    const size_t n = std::min(w.size(), cap);
    std::copy(w.begin(), w.begin() + n, out);
    return n;
}

// out (may be NULL, NOUT words) filled on S_OK
extern "C" int32_t emul_plan_compress_from_channels_ex(const dxb200_image* base, size_t items, const dxb200_chain_source* source,
                                                       const dxb200_channel_steps* channels, size_t levels, uint32_t filter,
                                                       const dxb200_chain_steps* steps, uint32_t dstFormat, uint32_t flags, float threshold,
                                                       float alphaWeight, const dxb200_image* dst, int32_t* alphaAllOpaque,
                                                       const dxb200_texconv_steps* ts, uint64_t* out)
{
    (void)alphaWeight;
    FromPlan fp;
    AlphaOpaquePlan ap;
    const int32_t hr = plan_mipmaps_compress_channels(base, items, source, channels, levels, filter, steps, dstFormat, flags, threshold, dst,
                                                      &fp, ts, alphaAllOpaque, &ap);
    if (hr == DXB_S_OK && out) report(fp, ap, base, out);
    if (hr == DXB_S_OK) last = fp.chunk;
    return hr;
}

extern "C" int32_t emul_plan_convert_from_ex(const dxb200_image* base, size_t items, const dxb200_chain_source* source,
                                             const dxb200_channel_steps* channels, uint32_t dstFormat, uint32_t convertFilter, float threshold,
                                             size_t levels, uint32_t filter, const dxb200_chain_steps* steps, const dxb200_image* dst,
                                             int32_t* alphaAllOpaque, const dxb200_texconv_steps* ts, uint64_t* out)
{
    FromPlan fp;
    AlphaOpaquePlan ap;
    const int32_t hr = plan_mipmaps_convert_from(base, items, source, channels, dstFormat, convertFilter, threshold, levels, filter, steps, dst,
                                                 alphaAllOpaque, &fp, &ap, ts);
    if (hr == DXB_S_OK && out) report(fp, ap, base, out);
    if (hr == DXB_S_OK) last = fp.chunk;
    return hr;
}

extern "C" int32_t emul_plan_levels_from_ex(const dxb200_image* base, size_t items, size_t levels, const dxb200_chain_source* source,
                                            const dxb200_channel_steps* channels, uint32_t dstFormat, uint32_t convertFilter, uint32_t compressFlags,
                                            float threshold, const dxb200_chain_steps* steps, const dxb200_image* dst, int32_t* alphaAllOpaque,
                                            const dxb200_texconv_steps* ts, uint64_t* out)
{
    FromPlan fp;
    AlphaOpaquePlan ap;
    const int32_t hr = plan_levels_from(base, items, levels, source, channels, dstFormat, convertFilter, compressFlags, threshold, steps, dst,
                                        alphaAllOpaque, &fp, &ap, ts);
    if (hr == DXB_S_OK && out) report(fp, ap, base, out);
    if (hr == DXB_S_OK) last = fp.chunk;
    return hr;
}
