// tests/cpp/channel_steps_probe.cpp — TEST INFRASTRUCTURE.  texconv's swizzle, colour key, invert-Y and reconstruct-Z steps run
// through the reference's own array TransformImage (DirectXTexMisc.cpp:639-760), one call per enabled step, each on the previous
// call's result, as texconv runs them (Texconv/texconv.cpp:2645-3300).  The lambdas are written from the rule the library states
// (directxtex_b200/csrc/dxb_channel_steps.h), on the DirectXMath operations texconv's lambdas use.  Those operations are not in the oracle's
// DirectXMath stand-in (oracle/compat/DirectXMath.h), so they are restated below with its semantics: scalar, IEEE, unfused fp32.
// Compiled against the mirror's header (the reference's Image / TexMetadata / ScratchImage layout, tests/test_cpu_abi.py) and the
// stand-in's XMVECTOR, and linked with the reference build (oracle/_ref/libdxtex_ref.so).
#include "DirectXTexB200.h"
#include "DirectXMath.h"
#include <cmath>
#include <cstdint>
#include <cstring>
#include <functional>
#include <vector>

namespace DirectX
{
    // the reference's array TransformImage (DirectXTex.h), declared here because the mirror leaves it out
    HRESULT TransformImage(const Image* srcImages, size_t nimages, const TexMetadata& metadata,
                           std::function<void(XMVECTOR* outPixels, const XMVECTOR* inPixels, size_t width, size_t y)> pixelFunc,
                           ScratchImage& result);
}

using namespace DirectX;

namespace
{
    // XMVectorSwizzle with run-time indices: a copy of each element's bits
    XMVECTOR swizzle(FXMVECTOR V, uint32_t e0, uint32_t e1, uint32_t e2, uint32_t e3)
    {
        return shim::mku(V.vector4_u32[e0], V.vector4_u32[e1], V.vector4_u32[e2], V.vector4_u32[e3]);
    }
    // XMVectorSelectControl: element i selects the second vector when index i is nonzero
    XMVECTOR select_control(uint32_t i0, uint32_t i1, uint32_t i2, uint32_t i3)
    {
        return shim::mku(i0 ? XM_SELECT_1 : XM_SELECT_0, i1 ? XM_SELECT_1 : XM_SELECT_0, i2 ? XM_SELECT_1 : XM_SELECT_0, i3 ? XM_SELECT_1 : XM_SELECT_0);
    }
    // XMVector3NearEqual: |V1 - V2| <= Epsilon on x, y and z (SSE: max(0 - d, d) <= e; false for a NaN)
    bool near_equal3(FXMVECTOR V1, FXMVECTOR V2, FXMVECTOR E)
    {
        for (int i = 0; i < 3; ++i)
        {
            const float d = V1.vector4_f32[i] - V2.vector4_f32[i];
            const float a = shim::ssemax(0.0f - d, d);
            if (!(a <= E.vector4_f32[i])) return false;
        }
        return true;
    }
    // XMVector2Dot: (x*x') + (y*y'), replicated
    XMVECTOR dot2(FXMVECTOR V1, FXMVECTOR V2)
    {
        const float x = V1.vector4_f32[0] * V2.vector4_f32[0];
        const float y = V1.vector4_f32[1] * V2.vector4_f32[1];
        return XMVectorReplicate(x + y);
    }
    // XMVectorSqrt: correctly rounded per element
    XMVECTOR vsqrt(FXMVECTOR V)
    {
        return shim::mk(sqrtf(V.vector4_f32[0]), sqrtf(V.vector4_f32[1]), sqrtf(V.vector4_f32[2]), sqrtf(V.vector4_f32[3]));
    }
    // XMLoadColor of a packed A8R8G8B8 word: each byte * (1/255)
    XMVECTOR load_color(uint32_t c)
    {
        return shim::mk(static_cast<float>((c >> 16) & 0xFF) * (1.0f / 255.0f), static_cast<float>((c >> 8) & 0xFF) * (1.0f / 255.0f),
                        static_cast<float>(c & 0xFF) * (1.0f / 255.0f), static_cast<float>((c >> 24) & 0xFF) * (1.0f / 255.0f));
    }

    typedef std::function<void(XMVECTOR*, const XMVECTOR*, size_t, size_t)> PixelFn;
}

// The enabled steps on the n images src (an array of src[0]'s size and format, TexMetadata built from src[0]).  swz = 4 swizzle
// elements; zero / one = the masks (bit c = channel c).  Returns the first failing TransformImage's HRESULT; with no step enabled,
// that of a TransformImage with a null function.  On S_OK the result's pixels (GetPixelsSize() bytes) go to out when they fit.
extern "C" int32_t probe_channel_steps(const Image* src, size_t n, const uint8_t* swz, uint32_t zero, uint32_t one, int colorKey,
                                       uint32_t colorKeyValue, int invertY, int reconstructZ, uint8_t* out, size_t outBytes)
{
    TexMetadata md = {};
    if (src && n)
    {
        md.width = src[0].width; md.height = src[0].height; md.format = src[0].format;
    }
    md.depth = 1; md.arraySize = n; md.mipLevels = 1; md.dimension = TEX_DIMENSION_TEXTURE2D;

    std::vector<PixelFn> fns;
    if (swz[0] != 0 || swz[1] != 1 || swz[2] != 2 || swz[3] != 3 || zero || one)
    {
        const XMVECTOR zc = select_control(zero & 1, zero & 2, zero & 4, zero & 8), oc = select_control(one & 1, one & 2, one & 4, one & 8);
        const uint32_t e0 = swz[0], e1 = swz[1], e2 = swz[2], e3 = swz[3];
        fns.push_back([=](XMVECTOR* o, const XMVECTOR* in, size_t w, size_t)
        {
            for (size_t j = 0; j < w; ++j)
            {
                XMVECTOR p = swizzle(in[j], e0, e1, e2, e3);
                p = XMVectorSelect(p, g_XMZero, zc);
                o[j] = XMVectorSelect(p, g_XMOne, oc);
            }
        });
    }
    if (colorKey)
    {
        const XMVECTOR key = load_color(colorKeyValue & 0xFFFFFF);
        fns.push_back([=](XMVECTOR* o, const XMVECTOR* in, size_t w, size_t)
        {
            const XMVECTOR tol = shim::mk(0.2f, 0.2f, 0.2f, 0.0f);
            for (size_t j = 0; j < w; ++j)
                o[j] = near_equal3(in[j], key, tol) ? XMVECTOR(g_XMZero) : XMVectorSelect(g_XMOne, in[j], g_XMSelect1110);
        });
    }
    if (invertY)
    {
        fns.push_back([](XMVECTOR* o, const XMVECTOR* in, size_t w, size_t)
        {
            for (size_t j = 0; j < w; ++j) o[j] = XMVectorSelect(in[j], XMVectorSubtract(g_XMOne, in[j]), g_XMMaskY);
        });
    }
    if (reconstructZ)
    {
        const bool unorm = FormatDataType(static_cast<DXGI_FORMAT>(md.format)) == FORMAT_TYPE_UNORM;
        fns.push_back([=](XMVECTOR* o, const XMVECTOR* in, size_t w, size_t)
        {
            for (size_t j = 0; j < w; ++j)
            {
                XMVECTOR z;
                if (unorm)
                {
                    XMVECTOR a = XMVectorMultiplyAdd(in[j], g_XMTwo, g_XMNegativeOne);
                    a = vsqrt(XMVectorSubtract(g_XMOne, dot2(a, a)));
                    z = XMVectorMultiplyAdd(a, g_XMOneHalf, g_XMOneHalf);
                }
                else z = vsqrt(XMVectorSubtract(g_XMOne, dot2(in[j], in[j])));
                o[j] = XMVectorSelect(in[j], z, g_XMMaskZ);
            }
        });
    }
    if (fns.empty()) fns.push_back(PixelFn());

    ScratchImage cur;
    const Image* images = src;
    for (size_t k = 0; k < fns.size(); ++k)
    {
        ScratchImage next;
        const HRESULT hr = TransformImage(images, n, md, fns[k], next);
        if (FAILED(hr)) return hr;
        cur = std::move(next);
        images = cur.GetImages();
    }
    if (out && cur.GetPixelsSize() <= outBytes) memcpy(out, cur.GetPixels(), cur.GetPixelsSize());
    return S_OK;
}

// FormatDataType(fmt) == FORMAT_TYPE_UNORM: reconstruct Z's rule (:3252)
extern "C" int probe_is_unorm(uint32_t fmt)
{
    return FormatDataType(static_cast<DXGI_FORMAT>(fmt)) == FORMAT_TYPE_UNORM ? 1 : 0;
}
