// dxb_channel_steps.h — texconv's per-pixel channel steps (Texconv/texconv.cpp), each a DirectX::TransformImage (DirectXTexMisc.cpp:
// 606-760, TransformImage_ :215-263) with a texconv lambda, stated once for the host planner (dxb_plan.h, the emulator) and the
// generic k_convert (dxb_k_rows.cu).  In texconv's order:
//   swizzle        -swizzle, :2645-2694   out[c] = in[swizzle[c]]; channels of zeroMask become 0, then channels of oneMask 1
//   colour key     -c,       :3134-3191   |x - kr| <= 0.2 && |y - kg| <= 0.2 && |z - kb| <= 0.2 -> (0, 0, 0, 0), else w = 1
//   invert Y       -inverty, :3193-3240   y = 1 - y
//   reconstruct Z  -reconstructz, :3242-3300   z = sqrt(1 - (a*a + b*b)), with a, b = x, y (SNORM, float) or x*2 - 1, y*2 - 1
//                  and z = z*0.5 + 0.5 (UNORM, sRGB included: FormatDataType(format) == FORMAT_TYPE_UNORM)
// Each step is a LoadScanline (no sRGB step), the op and a StoreScanline at threshold 0 in the image's own format, so between
// two enabled steps the pixel is stored and loaded back: an RGBA8 pixel is quantised between the colour key and invert Y, an
// SNORM -128 becomes -127.  Every multiply-add is a rounded multiply followed by a rounded add (XMVectorMultiplyAdd without FMA3),
// and the dot product is (x*x) + (y*y); x*x + y*y > 1 makes z a NaN, which reaches the store.
//
// The steps run inside the generic k_convert: a launch whose source and destination formats are equal, which Convert never
// builds, selects them.  The enabled steps and their arguments travel in dxb_convert_params::steps (the word below) and
// dxb_convert_params::key (the colour key as floats, computed once on the host by dxb_color_key_vector).
#pragma once
#include <stdint.h>
#include "dxb_portable.h"
#include "dxb_formats.h"
#include "dxb_pixel.cuh"

// the step word: swizzle (2 bits per output channel), the two masks, one bit per enabled step, and the UNORM rule of reconstruct Z
#define DXB_CH_SWIZZLE_SHIFT 0u                 // bits 0-7: source channel of output channel c at bit 2c
#define DXB_CH_ZERO_SHIFT    8u                 // bits 8-11: channels forced to 0
#define DXB_CH_ONE_SHIFT     12u                // bits 12-15: channels forced to 1
#define DXB_CH_SWIZZLE       (1u << 16)
#define DXB_CH_COLOR_KEY     (1u << 17)
#define DXB_CH_INVERT_Y      (1u << 18)
#define DXB_CH_RECONSTRUCT_Z (1u << 19)
#define DXB_CH_UNORM         (1u << 20)         // reconstruct Z maps [0, 1] to [-1, 1] and back
#define DXB_CH_STEPS         (DXB_CH_SWIZZLE | DXB_CH_COLOR_KEY | DXB_CH_INVERT_Y | DXB_CH_RECONSTRUCT_Z)
#define DXB_CH_TOLERANCE     0.2f               // the colour key's s_tolerance (:3150)

// texconv's colour key is a 24-bit 0xRRGGBB value (:1826-1833) loaded as an XMCOLOR (:3145): channel = byte * (1/255).  The same
// rule is the XMLoadColor of the oracle's probe, so the key's floats are computed once, on the host, with this function.
static inline void dxb_color_key_vector(uint32_t colorKey, float key[3])
{
    const uint32_t c = colorKey & 0xFFFFFFu;
    key[0] = (float)((c >> 16) & 0xFFu) * (1.0f / 255.0f);
    key[1] = (float)((c >> 8) & 0xFFu) * (1.0f / 255.0f);
    key[2] = (float)(c & 0xFFu) * (1.0f / 255.0f);
}

// a rounded multiply and a rounded add that no compiler contracts into an FMA; the host build (tests/emul) runs with
// -ffp-contract=off, the device build with -fmad=false, and the device intrinsics say so again
DXB_DEV float dxb_ch_mul(float a, float b)
{
#if DXB_ON_DEVICE
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
DXB_DEV float dxb_ch_add(float a, float b)
{
#if DXB_ON_DEVICE
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
DXB_DEV float dxb_ch_sqrt(float a)
{
#if DXB_ON_DEVICE
    return __fsqrt_rn(a);
#else
    return sqrtf(a);
#endif
}

DXB_DEV float dxb_ch_get(const dxb_px& v, uint32_t c) { return c == 0u ? v.x : c == 1u ? v.y : c == 2u ? v.z : v.w; }

// swizzle: a copy of each source channel's bits, then the two masks (XMVectorSelect with XMVectorSelectControl)
DXB_DEV dxb_px dxb_ch_swizzle(dxb_px v, uint32_t word)
{
    dxb_px o = dxb_make_px(dxb_ch_get(v, word & 3u), dxb_ch_get(v, (word >> 2) & 3u), dxb_ch_get(v, (word >> 4) & 3u), dxb_ch_get(v, (word >> 6) & 3u));
    const uint32_t zero = (word >> DXB_CH_ZERO_SHIFT) & 0xFu, one = (word >> DXB_CH_ONE_SHIFT) & 0xFu;
    if (zero & 1u) o.x = 0.0f;
    if (zero & 2u) o.y = 0.0f;
    if (zero & 4u) o.z = 0.0f;
    if (zero & 8u) o.w = 0.0f;
    if (one & 1u) o.x = 1.0f;
    if (one & 2u) o.y = 1.0f;
    if (one & 4u) o.z = 1.0f;
    if (one & 8u) o.w = 1.0f;
    return o;
}

// colour key: XMVector3NearEqual(v, key, 0.2) is |v - key| <= 0.2 on x, y and z, false for a NaN
DXB_DEV dxb_px dxb_ch_color_key(dxb_px v, float kr, float kg, float kb)
{
    const bool near = fabsf(v.x - kr) <= DXB_CH_TOLERANCE && fabsf(v.y - kg) <= DXB_CH_TOLERANCE && fabsf(v.z - kb) <= DXB_CH_TOLERANCE;
    if (near) return dxb_make_px(0.0f, 0.0f, 0.0f, 0.0f);
    v.w = 1.0f;
    return v;
}

DXB_DEV dxb_px dxb_ch_invert_y(dxb_px v) { v.y = 1.0f - v.y; return v; }

DXB_DEV dxb_px dxb_ch_reconstruct_z(dxb_px v, bool unorm)
{
    if (unorm)
    {
        const float a = dxb_ch_add(dxb_ch_mul(v.x, 2.0f), -1.0f), b = dxb_ch_add(dxb_ch_mul(v.y, 2.0f), -1.0f);
        const float r = dxb_ch_sqrt(1.0f - dxb_ch_add(dxb_ch_mul(a, a), dxb_ch_mul(b, b)));
        v.z = dxb_ch_add(dxb_ch_mul(r, 0.5f), 0.5f);
    }
    else v.z = dxb_ch_sqrt(1.0f - dxb_ch_add(dxb_ch_mul(v.x, v.x), dxb_ch_mul(v.y, v.y)));
    return v;
}

// The enabled steps of `word` on pixel x of a row of format fmt: src row -> dst row (dst may be src: only pixel x is read and
// written).  Between two enabled steps the pixel goes through the format and back, as the reference's stored images do.
DXB_DEV void dxb_channel_steps_pixel(uint32_t fmt, const uint8_t* srow, uint8_t* drow, size_t x, uint32_t word, float kr, float kg, float kb)
{
    dxb_px v = dxb_load_pixel(fmt, srow, x);
    bool stored = false;                        // a step already ran: reload its stored result first
    for (uint32_t step = DXB_CH_SWIZZLE; step <= DXB_CH_RECONSTRUCT_Z; step <<= 1)
    {
        if (!(word & step)) continue;
        if (stored)
        {
            alignas(16) uint8_t px[16];
            dxb_store_pixel(fmt, px, 0, v, 0.0f);
            v = dxb_load_pixel(fmt, px, 0);
        }
        stored = true;
        if (step == DXB_CH_SWIZZLE) v = dxb_ch_swizzle(v, word);
        else if (step == DXB_CH_COLOR_KEY) v = dxb_ch_color_key(v, kr, kg, kb);
        else if (step == DXB_CH_INVERT_Y) v = dxb_ch_invert_y(v);
        else v = dxb_ch_reconstruct_z(v, (word & DXB_CH_UNORM) != 0u);
    }
    dxb_store_pixel(fmt, drow, x, v, 0.0f);
}
