// dxb_mips.cuh — one mip level from the previous stored level, one thread per destination pixel.
// Restates, as gathers, the per-level bodies of
//   Generate2DMipsPointFilter   DirectXTexMipmaps.cpp:907-987   (16.16 fixed-point nearest)
//   Generate2DMipsBoxFilter     :991-1083 + AVERAGE4 filters.h:31-37
//   Generate2DMipsLinearFilter  :1087-1197 + CreateLinearFilter / BILINEAR_INTERPOLATE filters.h:56-104
//   Generate2DMipsCubicFilter   :1204-1388 + CreateCubicFilter / bounduvw / CUBIC_INTERPOLATE filters.h:119-207
//   Generate2DMipsTriangleFilter:1392-1602 (weights from CreateTriangleFilter filters.h:247-419 are built on the
//                                host with the same fp32 statements and handed over as per-destination gather lists
//                                that preserve the reference's accumulation order: source row asc., source x asc.)
// Each level reads the PREVIOUS level as stored in the destination format (LoadScanlineLinear) and
// stores through StoreScanlineLinear, exactly like the reference (SURVEY.md fact 9).  All arithmetic
// unfused (-fmad=false), same association order as the macros.
#pragma once
#include "dxb_pixel.cuh"

#include "dxb_jobs.h"

DXB_DEV dxb_px dxb_load_linear(uint32_t fmt, const uint8_t* base, size_t pitch, uint32_t x, uint32_t y, uint32_t lflags)
{
    dxb_px v = dxb_load_pixel(fmt, base + (size_t)y * pitch, x);
    if (lflags & DXB_FILTER_SRGB_IN) v = dxb_srgb_to_linear(v);
    return v;
}
DXB_DEV void dxb_store_linear(uint32_t fmt, uint8_t* base, size_t pitch, uint32_t x, uint32_t y, dxb_px v, uint32_t lflags)
{
    if (lflags & DXB_FILTER_SRGB_OUT) v = dxb_linear_to_srgb(v);
    dxb_store_pixel(fmt, base + (size_t)y * pitch, x, v);
}

DXB_DEV dxb_px dxb_px_add(dxb_px a, dxb_px b) { return dxb_make_px(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
DXB_DEV dxb_px dxb_px_sub(dxb_px a, dxb_px b) { return dxb_make_px(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w); }
DXB_DEV dxb_px dxb_px_scale(dxb_px a, float s) { return dxb_make_px(a.x * s, a.y * s, a.z * s, a.w * s); }
DXB_DEV dxb_px dxb_px_mul(dxb_px a, dxb_px b) { return dxb_make_px(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }

// ---- POINT
DXB_DEV dxb_px dxb_mip_point(uint32_t fmt, const dxb_mip_job& j, uint32_t x, uint32_t y)
{
    const size_t xinc = ((size_t)j.sw << 16) / j.dw;
    const size_t yinc = ((size_t)j.sh << 16) / j.dh;
    const size_t sx = (xinc * x) >> 16, sy = (yinc * y) >> 16;
    return dxb_load_pixel(fmt, j.src + sy * j.srcPitch, sx);     // point uses LoadScanline / StoreScanline (no sRGB step)
}

// ---- BOX: ((p00 + p10) + p01) + p11) * 0.25 with p10 = next row, p01 = next column.
// Degenerate axes follow the reference's pointer aliasing (:1024-1033): height<=1 -> second row = first row,
// width<=1 -> second column = first column.  When height<=1 but width>1 the reference reads the "second row,
// next column" operand from a scanline buffer that is NOT reloaded at this level (urow3 keeps pointing into the
// old urow1 buffer): it still holds row 1 of the last level whose source height was 2.  `stale` points at that
// row (NULL when no such level exists, in which case the reference reads uninitialised memory and no parity is
// defined; we then use the first row).
DXB_DEV dxb_px dxb_mip_box(uint32_t fmt, const dxb_mip_job& j, uint32_t x, uint32_t y, uint32_t lflags)
{
    const uint32_t x2 = (j.sw > 1) ? (x << 1) : 0u;
    const uint32_t xn = (j.sw > 1) ? (x2 + 1u) : x2;
    const uint32_t y0 = (j.sh > 1) ? (y << 1) : 0u;
    const uint32_t y1 = (j.sh > 1) ? (y0 + 1u) : y0;
    const dxb_px p00 = dxb_load_linear(fmt, j.src, j.srcPitch, x2, y0, lflags);
    const dxb_px p10 = dxb_load_linear(fmt, j.src, j.srcPitch, x2, y1, lflags);
    const dxb_px p01 = dxb_load_linear(fmt, j.src, j.srcPitch, xn, y0, lflags);
    dxb_px p11;
    if (j.sh <= 1 && j.sw > 1 && j.stale) p11 = dxb_load_linear(fmt, j.stale, j.stalePitch, xn, 0, lflags);
    else p11 = dxb_load_linear(fmt, j.src, j.srcPitch, xn, y1, lflags);
    dxb_px v = dxb_px_add(p00, p10);
    v = dxb_px_add(v, p01);
    v = dxb_px_add(v, p11);
    return dxb_px_scale(v, 0.25f);
}

// ---- LINEAR (CreateLinearFilter, filters.h:64-104)
struct dxb_lin { uint32_t u0, u1; float w0, w1; };
DXB_DEV dxb_lin dxb_linear_entry(uint32_t source, uint32_t dest, bool wrap, uint32_t u)
{
    const float scale = (float)source / (float)dest;
    const float t = ((float)u + 0.5f) * scale;
    const float srcB = t + 0.5f;
    int64_t isrcB = (int64_t)srcB;
    int64_t isrcA = isrcB - 1;
    const float wsum = 1.0f + (float)isrcB;
    const float weight = wsum - srcB;
    if (isrcA < 0) isrcA = wrap ? ((int64_t)source - 1) : 0;
    if ((uint64_t)isrcB >= source) isrcB = wrap ? 0 : ((int64_t)source - 1);
    dxb_lin e; e.u0 = (uint32_t)isrcA; e.w0 = weight; e.u1 = (uint32_t)isrcB; e.w1 = 1.0f - weight;
    return e;
}
DXB_DEV dxb_px dxb_mip_linear(uint32_t fmt, const dxb_mip_job& j, uint32_t x, uint32_t y, uint32_t filter, uint32_t lflags)
{
    const dxb_lin tx = dxb_linear_entry(j.sw, j.dw, (filter & DXB_FILTER_WRAP_U) != 0, x);
    const dxb_lin ty = dxb_linear_entry(j.sh, j.dh, (filter & DXB_FILTER_WRAP_V) != 0, y);
    const dxb_px a0 = dxb_load_linear(fmt, j.src, j.srcPitch, tx.u0, ty.u0, lflags);
    const dxb_px a1 = dxb_load_linear(fmt, j.src, j.srcPitch, tx.u1, ty.u0, lflags);
    const dxb_px b0 = dxb_load_linear(fmt, j.src, j.srcPitch, tx.u0, ty.u1, lflags);
    const dxb_px b1 = dxb_load_linear(fmt, j.src, j.srcPitch, tx.u1, ty.u1, lflags);
    const dxb_px r0 = dxb_px_scale(dxb_px_add(dxb_px_scale(a0, tx.w0), dxb_px_scale(a1, tx.w1)), ty.w0);
    const dxb_px r1 = dxb_px_scale(dxb_px_add(dxb_px_scale(b0, tx.w0), dxb_px_scale(b1, tx.w1)), ty.w1);
    return dxb_px_add(r0, r1);
}

// ---- CUBIC (bounduvw / CreateCubicFilter / CUBIC_INTERPOLATE, filters.h:123-207)
DXB_DEV int64_t dxb_bounduvw(int64_t u, int64_t maxu, bool wrap, bool mirror)
{
    if (wrap)
    {
        if (u < 0) u = maxu + u + 1;
        else if (u > maxu) u = u - maxu - 1;
    }
    else if (mirror)
    {
        if (u < 0) u = (-u) - 1;
        else if (u > maxu) u = maxu - (u - maxu - 1);
    }
    u = (u < maxu) ? u : maxu;
    u = (u > 0) ? u : 0;
    return u;
}
struct dxb_cub { uint32_t u0, u1, u2, u3; float x; };
DXB_DEV dxb_cub dxb_cubic_entry(uint32_t source, uint32_t dest, bool wrap, bool mirror, uint32_t u)
{
    const float scale = (float)source / (float)dest;
    const float t = ((float)u + 0.5f) * scale;
    const float srcB = t - 0.5f;
    const int64_t maxu = (int64_t)source - 1;
    const int64_t isrcB = dxb_bounduvw((int64_t)srcB, maxu, wrap, mirror);
    const int64_t isrcA = dxb_bounduvw(isrcB - 1, maxu, wrap, mirror);
    const int64_t isrcC = dxb_bounduvw(isrcB + 1, maxu, wrap, mirror);
    const int64_t isrcD = dxb_bounduvw(isrcB + 2, maxu, wrap, mirror);
    dxb_cub e; e.u0 = (uint32_t)isrcA; e.u1 = (uint32_t)isrcB; e.u2 = (uint32_t)isrcC; e.u3 = (uint32_t)isrcD;
    e.x = srcB - (float)isrcB;
    return e;
}
DXB_DEV float dxb_cubic1(float dx, float p0, float p1, float p2, float p3)
{
    const float third = 1.0f / 3.0f, sixth = 1.0f / 6.0f, half = 1.0f / 2.0f;
    const float a0 = p1;
    const float d0 = p0 - a0, d2 = p2 - a0, d3 = p3 - a0;
    float a1 = d2 - third * d0;
    a1 = a1 - sixth * d3;
    const float h0 = half * d0, h2 = half * d2;
    const float a2 = h0 + h2;
    const float s3 = sixth * d3, s0 = sixth * d0;
    float a3 = s3 - s0;
    a3 = a3 - half * d2;
    const float dx2 = dx * dx;
    const float dx3 = dx2 * dx;
    const float t1 = a1 * dx;
    const float r1 = a0 + t1;
    const float t2 = a2 * dx2;
    const float r2 = r1 + t2;
    const float t3 = a3 * dx3;
    return r2 + t3;
}
DXB_DEV dxb_px dxb_cubic4(float dx, dxb_px p0, dxb_px p1, dxb_px p2, dxb_px p3)
{
    return dxb_make_px(dxb_cubic1(dx, p0.x, p1.x, p2.x, p3.x), dxb_cubic1(dx, p0.y, p1.y, p2.y, p3.y),
                       dxb_cubic1(dx, p0.z, p1.z, p2.z, p3.z), dxb_cubic1(dx, p0.w, p1.w, p2.w, p3.w));
}
DXB_DEV dxb_px dxb_mip_cubic(uint32_t fmt, const dxb_mip_job& j, uint32_t x, uint32_t y, uint32_t filter, uint32_t lflags)
{
    const dxb_cub tx = dxb_cubic_entry(j.sw, j.dw, (filter & DXB_FILTER_WRAP_U) != 0, (filter & DXB_FILTER_MIRROR_U) != 0, x);
    const dxb_cub ty = dxb_cubic_entry(j.sh, j.dh, (filter & DXB_FILTER_WRAP_V) != 0, (filter & DXB_FILTER_MIRROR_V) != 0, y);
    const uint32_t rows[4] = { ty.u0, ty.u1, ty.u2, ty.u3 };
    dxb_px C[4];
    for (int r = 0; r < 4; ++r)
    {
        const dxb_px q0 = dxb_load_linear(fmt, j.src, j.srcPitch, tx.u0, rows[r], lflags);
        const dxb_px q1 = dxb_load_linear(fmt, j.src, j.srcPitch, tx.u1, rows[r], lflags);
        const dxb_px q2 = dxb_load_linear(fmt, j.src, j.srcPitch, tx.u2, rows[r], lflags);
        const dxb_px q3 = dxb_load_linear(fmt, j.src, j.srcPitch, tx.u3, rows[r], lflags);
        C[r] = dxb_cubic4(tx.x, q0, q1, q2, q3);
    }
    return dxb_cubic4(ty.x, C[0], C[1], C[2], C[3]);
}

// ---- TRIANGLE: acc = row[x] * (wy*wx) + acc in the reference's order (:1516-1538): source rows ascending, then source x
// ascending, then that row's entries for this destination row, then that column's entries for this destination column.  A row
// (column) has two entries for one destination when wrap brings it back around a short axis; the entries of one source row
// (column) are adjacent in the gather lists.
DXB_DEV dxb_px dxb_mip_triangle(uint32_t fmt, const dxb_mip_job& j, uint32_t x, uint32_t y, uint32_t lflags,
                                const dxb_tri_axis& ax, const dxb_tri_axis& ay)
{
    dxb_px acc = dxb_make_px(0.0f, 0.0f, 0.0f, 0.0f);
    const uint32_t yEnd = ay.off[y + 1], xEnd = ax.off[x + 1];
    for (uint32_t iy = ay.off[y], ny; iy < yEnd; iy = ny)
    {
        const uint32_t sy = ay.src[iy];
        for (ny = iy + 1; ny < yEnd && ay.src[ny] == sy; ++ny) {}
        for (uint32_t ix = ax.off[x], nx; ix < xEnd; ix = nx)
        {
            const uint32_t sx = ax.src[ix];
            for (nx = ix + 1; nx < xEnd && ax.src[nx] == sx; ++nx) {}
            const dxb_px p = dxb_load_linear(fmt, j.src, j.srcPitch, sx, sy, lflags);
            for (uint32_t ey = iy; ey < ny; ++ey)
                for (uint32_t ex = ix; ex < nx; ++ex) acc = dxb_px_add(dxb_px_scale(p, ay.w[ey] * ax.w[ex]), acc);
        }
    }
    if (fmt == DXB_FMT_R10G10B10A2_UNORM) acc.w = acc.w + 0.1f;      // Bias {0,0,0,0.1} (:1560-1575)
    return acc;
}

// ---- one destination pixel of a level in filter `mode`: POINT copies with plain Load / Store, the other filters work in
// linear space and store through StoreScanlineLinear.  Inlined, so a kernel with a compile-time format and mode keeps only
// its own filter.  ax / ay: TRIANGLE's gather lists.
DXB_DEV void dxb_mip_pixel(uint32_t fmt, uint32_t mode, const dxb_mip_job& j, uint32_t x, uint32_t y, uint32_t filter, uint32_t lflags,
                           const dxb_tri_axis& ax, const dxb_tri_axis& ay)
{
    dxb_px v;
    switch (mode)
    {
    case DXB_FILTER_POINT:
        dxb_store_pixel(fmt, j.dst + (size_t)y * j.dstPitch, x, dxb_mip_point(fmt, j, x, y));
        return;
    case DXB_FILTER_BOX: v = dxb_mip_box(fmt, j, x, y, lflags); break;
    case DXB_FILTER_LINEAR: v = dxb_mip_linear(fmt, j, x, y, filter, lflags); break;
    case DXB_FILTER_CUBIC: v = dxb_mip_cubic(fmt, j, x, y, filter, lflags); break;
    default: v = dxb_mip_triangle(fmt, j, x, y, lflags, ax, ay); break;
    }
    dxb_store_linear(fmt, j.dst, j.dstPitch, x, y, v, lflags);
}

// ---------------------------------------------------------------------------------------------
// ScaleMipMapsAlphaForCoverage helpers (DirectXTexMipmaps.cpp:143-356).
// Coverage of one 2x2 cell (CalculateAlphaCoverage :213-308): the four alphas, scaled and saturated, go through the 8x8
// bilinear sub-sample weights IN SEQUENCE: the reference overwrites its vector with the splatted weighted sum, so every
// sub-sample after the first re-weights the previous result (kept: it defines the counts).  VectorSum = XMVectorSum
// (DIRECTX_MATH_VERSION >= 310, :127-128) = (x + y) + (z + w) in the oracle's DirectXMath shim (M).
// a00 = (x, y), a01 = (x, y+1), a10 = (x+1, y), a11 = (x+1, y+1).  Returns how many of the 64 sub-samples exceed `ref`.
DXB_DEV uint32_t dxb_alpha_coverage_cell(float a00, float a01, float a10, float a11, float scale, float ref)
{
    float v0 = dxb_clamp(a00 * scale, 0.0f, 1.0f), v1 = dxb_clamp(a01 * scale, 0.0f, 1.0f);
    float v2 = dxb_clamp(a10 * scale, 0.0f, 1.0f), v3 = dxb_clamp(a11 * scale, 0.0f, 1.0f);
    uint32_t count = 0;
    for (int sy = 0; sy < 8; ++sy)
    {
        const float fy = ((float)sy + 0.5f) / 8.0f, ify = 1.0f - fy;
        for (int sx = 0; sx < 8; ++sx)
        {
            const float fx = ((float)sx + 0.5f) / 8.0f, ifx = 1.0f - fx;
            const float p0 = v0 * (ifx * ify), p1 = v1 * (ifx * fy), p2 = v2 * (fx * ify), p3 = v3 * (fx * fy);
            const float a = p0 + p1, b = p2 + p3;
            const float sum = a + b;
            v0 = v1 = v2 = v3 = sum;
            if (sum > ref) ++count;
        }
    }
    return count;
}
// ScaleAlpha (:143-193): plain Load / Store, alpha * scale
DXB_DEV void dxb_scale_alpha_pixel(uint32_t fmt, const uint8_t* srow, uint8_t* drow, uint32_t x, float scale)
{
    dxb_px v = dxb_load_pixel(fmt, srow, x);
    v.w = v.w * scale;
    dxb_store_pixel(fmt, drow, x, v);
}
