// dxb_alpha_opaque.h — the rule of ScratchImage::IsAlphaAllOpaque (DirectXTexImage.cpp:800-852) and of IsAlphaAllOpaqueBC
// (DirectXTexCompress.cpp:539-621), stated once for the host planner (dxb_plan.h, the emulator) and the scan the generic
// k_convert and k_decompress run (dxb_k_rows.cu, dxb_k_decode.cu).
//
// A texel is not opaque when its alpha is below the threshold: 0.997 for a pixel LoadScanline reads (no sRGB step), 0.99 for a
// texel of a decoded BC1 / BC2 / BC3 / BC7 block.  The reference compares with XMVector4Less on the splatted alpha, which is false
// for a NaN, so a NaN alpha counts as opaque, as it does with `<` here.  Only the texels inside the image count: the padding
// texels of a partial block are decoded but never tested.
//
// The scan runs inside the generic k_convert / k_decompress: a destination format of DXGI_FORMAT_UNKNOWN, which no Convert or
// Decompress call can have, selects it.  Each job's dst then points at a 32-bit result word, zero before the launch; a texel
// that is not opaque stores 1 into it (every writer stores the same value, so a plain store is enough) and nothing else is
// written.
#pragma once
#include <stdint.h>
#include "dxb_formats.h"

#ifndef DXB_HD
#if defined(__CUDACC__)
  #define DXB_HD __host__ __device__ __forceinline__
#else
  #define DXB_HD inline
#endif
#endif

#define DXB_SCAN_ALPHA_OPAQUE DXB_FMT_UNKNOWN          // the destination format that selects the scan
#define DXB_OPAQUE_PIXEL 0.997f                        // IsAlphaAllOpaque's threshold (:821)
#define DXB_OPAQUE_BLOCK 0.99f                         // IsAlphaAllOpaqueBC's threshold (:576)

// the BC formats IsAlphaAllOpaqueBC decodes; every other BC format has no alpha (HasAlpha is false for it)
DXB_HD bool dxb_alpha_scan_blocks(uint32_t fmt)
{
    switch (fmt)
    {
    case DXB_FMT_BC1_UNORM: case DXB_FMT_BC1_UNORM_SRGB: case DXB_FMT_BC2_UNORM: case DXB_FMT_BC2_UNORM_SRGB:
    case DXB_FMT_BC3_UNORM: case DXB_FMT_BC3_UNORM_SRGB: case DXB_FMT_BC7_UNORM: case DXB_FMT_BC7_UNORM_SRGB:
        return true;
    default:
        return false;
    }
}

#if defined(__CUDACC__)
// The job's answer is known once its word is set: the scan skips the rest of the job's units, and a texel that is not opaque
// stores only while the word is still clear, so a mostly transparent image does not send one store per texel to the same address.
// The load is volatile so that it sees the other SMs' stores in L2; a stale 0 only costs one redundant store.
__device__ __forceinline__ bool dxb_alpha_word_set(const uint8_t* word) { return *reinterpret_cast<const volatile uint32_t*>(word) != 0u; }
__device__ __forceinline__ void dxb_alpha_word_store(uint8_t* word)
{
    if (!dxb_alpha_word_set(word)) *reinterpret_cast<volatile uint32_t*>(word) = 1u;
}
#endif

// one texel: alpha a against its threshold
DXB_HD bool dxb_alpha_not_opaque(float a, float threshold) { return a < threshold; }

// one decoded 4x4 block (px[y * 4 + x]) of which the pw x ph texels at its top left lie inside the image
#if defined(__CUDACC__)
#pragma nv_exec_check_disable
#endif
template <typename Px>
DXB_HD bool dxb_block_not_opaque(const Px* px, uint32_t pw, uint32_t ph)
{
    bool any = false;
    for (uint32_t y = 0; y < ph; ++y)
        for (uint32_t x = 0; x < pw; ++x) any |= dxb_alpha_not_opaque(px[y * 4u + x].w, DXB_OPAQUE_BLOCK);
    return any;
}
