// tests/cpp/alpha_opaque_probe.cpp — TEST INFRASTRUCTURE.  ScratchImage::IsAlphaAllOpaque of textures a DirectXTex caller builds:
// 2D images, arrays, cube maps and mip chains, whose pixels are copied in from a buffer in the container's own layout.  Compiled
// against the mirror's header (whose ScratchImage has the reference's layout, tests/test_cpu_abi.py) into a shared library, once
// linked with libdxtex_b200.so and once with the reference build (oracle/_ref/libdxtex_ref.so): the same calls answer through the
// mirror and through the reference.
#include "DirectXTexB200.h"
#include <cstdint>
#include <cstring>
using namespace DirectX;

// kind 0: Initialize2D(fmt, w, h, items, levels); kind 1: InitializeCube(fmt, w, h, items, levels).  pixels = GetPixelsSize() bytes
// (nbytes must equal it).  Returns 1 / 0, what IsAlphaAllOpaque() returns, or -1 when the container cannot be built.
extern "C" int probe_is_alpha_all_opaque(int kind, uint32_t fmt, size_t w, size_t h, size_t items, size_t levels, const uint8_t* pixels, size_t nbytes)
{
    ScratchImage s;
    const DXGI_FORMAT f = static_cast<DXGI_FORMAT>(fmt);
    const HRESULT hr = kind ? s.InitializeCube(f, w, h, items, levels) : s.Initialize2D(f, w, h, items, levels);
    if (hr < 0 || s.GetPixelsSize() != nbytes) return -1;
    if (nbytes) memcpy(s.GetPixels(), pixels, nbytes);
    return s.IsAlphaAllOpaque() ? 1 : 0;
}

// an empty container answers false (DirectXTexImage.cpp:802-803)
extern "C" int probe_empty_is_alpha_all_opaque(void)
{
    ScratchImage s;
    return s.IsAlphaAllOpaque() ? 1 : 0;
}

// HasAlpha, which decides whether IsAlphaAllOpaque reads a pixel at all
extern "C" int probe_has_alpha(uint32_t fmt)
{
    return HasAlpha(static_cast<DXGI_FORMAT>(fmt)) ? 1 : 0;
}
