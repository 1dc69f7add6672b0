// dxb_host_tri.h — HOST-side construction of the triangle-filter weights (part of dxb_plan.h's chain records).
#pragma once
#include <vector>
#include <utility>
#include <cstdint>
#include <cstddef>
#include <cmath>

namespace {
// CreateTriangleFilter (filters.h:247-419) restated on the host, then inverted into per-destination
// gather lists that keep ascending source order.  Host fp32 code, no contraction (see build flags).
struct TriLists { std::vector<uint32_t> off, src; std::vector<float> w; };

void build_triangle_axis(size_t source, size_t dest, bool wrap, TriLists& out)
{
    const float scale = float(dest) / float(source);
    const float scaleInv = 0.5f / scale;
    std::vector<std::vector<std::pair<uint32_t, float>>> toLists(dest);
    size_t accumU = 0;
    float accumWeight = 0.f;
    for (size_t u = 0; u < source; ++u)
    {
        auto flush = [&](void)
        {
            if (accumWeight > 0.00001f) toLists[accumU].push_back(std::make_pair((uint32_t)u, accumWeight));
        };
        for (size_t j = 0; j < 2; ++j)
        {
            const float src = float(u + j) - 0.5f;
            float destMin = src * scale;
            float destMax = destMin + scale;
            if (!wrap)
            {
                if (destMin < 0.f) destMin = 0.f;
                if (destMax > float(dest)) destMax = float(dest);
            }
            for (ptrdiff_t k = static_cast<ptrdiff_t>(floorf(destMin)); float(k) < destMax; ++k)
            {
                float d0 = float(k);
                float d1 = d0 + 1.f;
                size_t u0;
                if (k < 0) u0 = size_t(k + ptrdiff_t(dest));
                else if (k >= ptrdiff_t(dest)) u0 = size_t(k - ptrdiff_t(dest));
                else u0 = size_t(k);
                if (u0 != accumU)
                {
                    flush();
                    accumWeight = 0.f;
                    accumU = u0;
                }
                if (d0 < destMin) d0 = destMin;
                if (d1 > destMax) d1 = destMax;
                float weight;
                if (!wrap && src < 0.f) weight = 1.f;
                else if (!wrap && ((src + 1.f) >= float(source))) weight = 0.f;
                else
                {
                    const float sum = d0 + d1;
                    const float prod = sum * scaleInv;
                    weight = prod - src;
                }
                const float span = d1 - d0;
                const float f = j ? (1.f - weight) : weight;
                const float add = span * f;
                accumWeight += add;
            }
        }
        flush();
        accumWeight = 0.f;
    }
    out.off.assign(dest + 1, 0); out.src.clear(); out.w.clear();
    for (size_t d = 0; d < dest; ++d)
    {
        out.off[d] = (uint32_t)out.src.size();
        for (auto& e : toLists[d]) { out.src.push_back(e.first); out.w.push_back(e.second); }
    }
    out.off[dest] = (uint32_t)out.src.size();
}
} // namespace
