// dxb_jobs.h — plain job and parameter structs shared by the kernels, the host API and the host emulator (host + device).
// The kernels take the parameter structs and single jobs by value: field order and types are part of their interface.
#pragma once
#include <stdint.h>
#include <stddef.h>

struct dxb_job
{
    const uint8_t* src; uint8_t* dst;
    size_t srcPitch, dstPitch;
    uint32_t width, height;
    uint32_t nbx, nby;
    uint32_t firstUnit;
    uint32_t pad;
};

struct dxb_compress_params
{
    uint32_t srcFormat, dstFormat;
    uint32_t inF, outF, cflags, bcflags;
    float threshold;
    uint32_t totalUnits, njobs;
};

struct dxb_convert_params
{
    uint32_t srcFormat, dstFormat, inF, outF, flags;
    uint32_t totalUnits, njobs;
    float threshold;               // alpha threshold of 1-bit alpha destinations (B5G5R5A1)
};

struct dxb_mip_job
{
    const uint8_t* src; uint8_t* dst;
    size_t srcPitch, dstPitch;
    uint32_t sw, sh, dw, dh;          // source / destination size
    uint32_t firstUnit;               // prefix sum of destination pixels over the batch
    const uint8_t* stale; size_t stalePitch;   // box filter only: see dxb_mip_box
};

// triangle filter gather lists for one axis (CSR): contributions of destination index d are
// entries [off[d], off[d+1]) with ascending source index
struct dxb_tri_axis { const uint32_t* off; const uint32_t* src; const float* w; };

struct dxb_mip_params
{
    uint32_t format, mode /*DXB_FILTER_* mode bits*/, filter, lflags;
    uint32_t totalUnits, njobs;
    dxb_tri_axis triX, triY;       // triangle filter only
};
