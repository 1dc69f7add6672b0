// dxb_bc6h.cuh — BC6H (UF16 / SF16) block encoder, ONE HALF-WARP PER 4x4 BLOCK, two blocks per warp (single-source SPMD, dxb_warp.cuh).
//
// Replaces D3DXEncodeBC6HU/S -> D3DX_BC6H::Encode (BC6HBC7.cpp:3624-3639, 1817-1859).  Parity contract as for BC7:
// a valid stream for the reference decoder (D3DX_BC6H::Decode, :1658-1813) whose error — in the reference
// encoder's own metric, the squared difference of half-float bit patterns over RGB (Norm / MapColorsQuantized,
// :1167-1173, 2044-2077) — stays within the tolerance stated in DESIGN.md of the reference CPU encoder's error.
//
// Pixel domain = the reference's INTColor domain: F16ToINT(half(rgb)) (:534-552): unsigned -> half bits with
// negatives clamped to 0; signed -> sign-magnitude integer, magnitude clamped to 0x7BFF.
//   stage 1  the 32 two-region shapes ranked by a line-fit residual (two shapes per lane), 7 best kept
//   stage 2  lanes 0..13 = 7 shapes x 2 regions, lane 14 = the one-region fit: PCA axis + least-squares refit
//            of continuous endpoints (3-bit / 4-bit interpolation weights)
//   stage 3  region pairs exchange endpoints (__shfl_xor) and pick the format mode: the highest base precision
//            whose delta fields can hold the endpoint differences (modes 3,4,5 > 1 > 6 > 7,8,9 > 2 > 10 for two
//            regions; 13 > 12 > 11 for one region; BC6HBC7.cpp:1051-1067); endpoints quantised exactly as the
//            reference does (Quantize :1864-1889) and the exact decoder palette (Unquantize / interpolate /
//            FinishUnquantize :1893-1940) gives each lane its region's true error
//   stage 4  winner by integer-key warp min; 16 lanes = 16 pixels choose indices against the exact palette, every
//            lane deposits its header bits / index field into a 128-bit word, warp OR-reduction, one store
#pragma once
#include "dxb_warp.cuh"
#include "dxb_pixel.cuh"
#include "dxb_bc7.cuh"            // moments / estimate helpers, dxb_rne, dxb_u128, dxb_put_bits
#include "dxb_bc6h_tables.h"

#ifndef DXB_BC6H_ROUNDS
#define DXB_BC6H_ROUNDS 2       // endpoint fit rounds: PCA + (ROUNDS - 1) least-squares refits; 3 gives the same error ratios as 2
#endif

// half bits -> INTColor component (F16ToINT, BC6HBC7.cpp:534-552), as float
DXB_DEV float dxb_bc6h_to_int(float v, bool bSigned)
{
    const uint32_t h = dxb_float_to_half(v);
    int32_t out;
    if (bSigned)
    {
        const int32_t m = (int32_t)(h & 0x7FFFu);
        out = (m > 0x7BFF) ? 0x7BFF : m;
        out = (h & 0x8000u) ? -out : out;
    }
    else out = (h & 0x8000u) ? 0 : (int32_t)h;
    return (float)out;
}

// D3DX_BC6H::Quantize (BC6HBC7.cpp:1864-1889)
DXB_DEV int32_t dxb_bc6h_quantize(int32_t v, int32_t prec, bool bSigned)
{
    if (bSigned)
    {
        const int32_t a = v < 0 ? -v : v;
        const int32_t q = (prec >= 16) ? a : ((a << (prec - 1)) / (0x7BFF + 1));
        return v < 0 ? -q : q;
    }
    return (prec >= 15) ? v : ((v << prec) / (0x7BFF + 1));
}
// D3DX_BC6H::Unquantize (BC6HBC7.cpp:1893-1929)
DXB_DEV int32_t dxb_bc6h_unquantize(int32_t comp, int32_t bits, bool bSigned)
{
    if (bSigned)
    {
        if (bits >= 16) return comp;
        const bool neg = comp < 0;
        const int32_t c = neg ? -comp : comp;
        int32_t unq;
        if (c == 0) unq = 0;
        else if (c >= ((1 << (bits - 1)) - 1)) unq = 0x7FFF;
        else unq = ((c << 15) + 0x4000) >> (bits - 1);
        return neg ? -unq : unq;
    }
    if (bits >= 15) return comp;
    if (comp == 0) return 0;
    if (comp == ((1 << bits) - 1)) return 0xFFFF;
    return ((comp << 16) + 0x8000) >> bits;
}
// D3DX_BC6H::FinishUnquantize (BC6HBC7.cpp:1932-1942)
DXB_DEV int32_t dxb_bc6h_finish(int32_t comp, bool bSigned)
{
    if (bSigned) return (comp < 0) ? -(((-comp) * 31) >> 5) : ((comp * 31) >> 5);
    return (comp * 31) >> 6;
}
// decoder palette entry k (3 or 4 index bits) for unquantised endpoints ua, ub (Decode :1771-1779)
DXB_DEV int32_t dxb_bc6h_palette(int32_t ua, int32_t ub, int32_t w, bool bSigned)
{
    return dxb_bc6h_finish((ua * (64 - w) + ub * w + 32) >> 6, bSigned);
}

// does signed delta d fit in n bits (NBits(d, true) <= n, BC6HBC7.cpp:1176-1194)
DXB_DEV bool dxb_fits_signed(int32_t d, int32_t n) { return d >= -(1 << (n - 1)) && d <= ((1 << (n - 1)) - 1); }

// ---------------------------------------------------------------------------------------------------
// stage 2: continuous endpoint fit of one region in the INT domain (3 channels), centred on `ctr`.
//   ib = index bits (3 two-region, 4 one-region); anchor = the region's fix-up pixel
// outputs E0/E1 (absolute INT-domain floats), ordered so that the anchor pixel projects into the first half
// bnd[0..2] / bnd[3..5] = clamp range of the endpoints per channel: the format range [lo, hi], except that for the signed
// format a channel whose values have both signs inside this region is held to the region's own [min, max].  The INT
// domain is the half-float bit pattern, i.e. logarithmic in the value, and runs through zero between the signs: a
// least-squares endpoint that overshoots the data by 10 % of such a span is off by a factor of ten in the decoded float.
DXB_DEV void dxb_bc6h_fit(const dxb_px* px, uint32_t mask, uint32_t ib, int anchor, const float* ctr, float lo, float hi, bool bSigned, float* E0, float* E1, float* bnd)
{
    {
        float mn[3] = { 3.0e38f, 3.0e38f, 3.0e38f }, mx[3] = { -3.0e38f, -3.0e38f, -3.0e38f };
        for (int i = 0; i < 16; ++i)
        {
            const bool in = ((mask >> i) & 1u) != 0u;
            const dxb_px p = px[i];
            mn[0] = in ? fminf(mn[0], p.x) : mn[0]; mx[0] = in ? fmaxf(mx[0], p.x) : mx[0];
            mn[1] = in ? fminf(mn[1], p.y) : mn[1]; mx[1] = in ? fmaxf(mx[1], p.y) : mx[1];
            mn[2] = in ? fminf(mn[2], p.z) : mn[2]; mx[2] = in ? fmaxf(mx[2], p.z) : mx[2];
        }
        for (int c = 0; c < 3; ++c)
        {
            const bool cross = bSigned && (mn[c] < 0.0f) && (mx[c] > 0.0f);
            bnd[c] = cross ? mn[c] : lo; bnd[3 + c] = cross ? mx[c] : hi;
        }
    }
    float n = 0, s0 = 0, s1 = 0, s2 = 0, m00 = 0, m01 = 0, m02 = 0, m11 = 0, m12 = 0, m22 = 0;
    for (int i = 0; i < 16; ++i)
    {
        const float f = dxb_bit_as_float(mask, i);
        const dxb_px p = px[i];
        const float X = p.x - ctr[0], Y = p.y - ctr[1], Z = p.z - ctr[2];
        const float x = X * f, y = Y * f, z = Z * f;
        n += f; s0 += x; s1 += y; s2 += z;
        m00 = dxb_fma(x, X, m00); m01 = dxb_fma(x, Y, m01); m02 = dxb_fma(x, Z, m02);
        m11 = dxb_fma(y, Y, m11); m12 = dxb_fma(y, Z, m12); m22 = dxb_fma(z, Z, m22);
    }
    const float inv = 1.0f / fmaxf(n, 1.0f);
    const float mean[3] = { s0 * inv, s1 * inv, s2 * inv };
    const float c00 = dxb_fma(-mean[0], s0, m00), c01 = dxb_fma(-mean[0], s1, m01), c02 = dxb_fma(-mean[0], s2, m02);
    const float c11 = dxb_fma(-mean[1], s1, m11), c12 = dxb_fma(-mean[1], s2, m12), c22 = dxb_fma(-mean[2], s2, m22);
    float ax[3];
    {
        const bool b0 = (c00 >= c11 && c00 >= c22), b1 = !b0 && (c11 >= c22);
        float v0 = b0 ? c00 : (b1 ? c01 : c02), v1 = b0 ? c01 : (b1 ? c11 : c12), v2 = b0 ? c02 : (b1 ? c12 : c22);
        for (int it = 0; it < 4; ++it)
        {
            const float w0 = dxb_fma(c00, v0, dxb_fma(c01, v1, c02 * v2));
            const float w1 = dxb_fma(c01, v0, dxb_fma(c11, v1, c12 * v2));
            const float w2 = dxb_fma(c02, v0, dxb_fma(c12, v1, c22 * v2));
            const float mx = fmaxf(fabsf(w0), fmaxf(fabsf(w1), fabsf(w2)));
            const float r = (mx > 1e-20f) ? 1.0f / mx : 0.0f;
            v0 = w0 * r; v1 = w1 * r; v2 = w2 * r;
        }
        const float vv = dxb_fma(v0, v0, dxb_fma(v1, v1, v2 * v2));
        const float r = (vv > 1e-20f) ? 1.0f / sqrtf(vv) : 0.0f;
        ax[0] = v0 * r; ax[1] = v1 * r; ax[2] = v2 * r;
    }
    float tmin = 3.0e38f, tmax = -3.0e38f;
    for (int i = 0; i < 16; ++i)
    {
        const dxb_px p = px[i];
        const float t = dxb_fma(p.x - ctr[0] - mean[0], ax[0], dxb_fma(p.y - ctr[1] - mean[1], ax[1], (p.z - ctr[2] - mean[2]) * ax[2]));
        const bool in = ((mask >> i) & 1u) != 0u;
        tmin = in ? fminf(tmin, t) : tmin; tmax = in ? fmaxf(tmax, t) : tmax;
    }
    if (!(tmin <= tmax)) { tmin = 0.0f; tmax = 0.0f; }
    float A[3], B[3];      // centred endpoints
    for (int c = 0; c < 3; ++c) { A[c] = dxb_fma(tmin, ax[c], mean[c]); B[c] = dxb_fma(tmax, ax[c], mean[c]); }

    const float nmax = (float)((1u << ib) - 1u);
    const float c64 = 64.0f / nmax;
    bool live = true;
    for (int round = 0; round + 1 < DXB_BC6H_ROUNDS; ++round)
    {
        dxb_warp_sync();
        const float dx = B[0] - A[0], dy = B[1] - A[1], dz = B[2] - A[2];
        const float dd = dxb_fma(dx, dx, dxb_fma(dy, dy, dz * dz));
        const float idd = (dd > 0.0f) ? nmax / dd : 0.0f;            // index scale folded in
        float la = 0, lb = 0, lc = 0, u0 = 0, u1 = 0, u2 = 0, v0 = 0, v1 = 0, v2 = 0;
#if DXB_ON_DEVICE
        #pragma unroll 4
#endif
        for (int i = 0; i < 16; ++i)
        {
            const float f = dxb_bit_as_float(mask, i);
            const dxb_px p = px[i];
            const float X = p.x - ctr[0], Y = p.y - ctr[1], Z = p.z - ctr[2];
            const float t = dxb_fma(X - A[0], dx, dxb_fma(Y - A[1], dy, (Z - A[2]) * dz)) * idd;
            const float sk = dxb_bc7_weightf(dxb_rne(fminf(fmaxf(t, 0.0f), nmax)), c64);
            const float skf = sk * f, osf = f - skf, os = 1.0f - sk;
            la = dxb_fma(osf, os, la); lb = dxb_fma(osf, sk, lb); lc = dxb_fma(skf, sk, lc);
            u0 = dxb_fma(osf, X, u0); u1 = dxb_fma(osf, Y, u1); u2 = dxb_fma(osf, Z, u2);
            v0 = dxb_fma(skf, X, v0); v1 = dxb_fma(skf, Y, v1); v2 = dxb_fma(skf, Z, v2);
        }
        const float det = dxb_fma(la, lc, -(lb * lb));
        live = live && (det > 1e-4f);
        const float id = live ? 1.0f / det : 0.0f;
        const float uu[3] = { u0, u1, u2 }, vv[3] = { v0, v1, v2 };
        for (int c = 0; c < 3; ++c)
        {
            const float a = dxb_fma(lc, uu[c], -(lb * vv[c])) * id, b = dxb_fma(la, vv[c], -(lb * uu[c])) * id;
            A[c] = live ? a : A[c]; B[c] = live ? b : B[c];
        }
    }
    // order: anchor pixel closer to E0
    {
        const dxb_px p = px[anchor];
        const float dx = B[0] - A[0], dy = B[1] - A[1], dz = B[2] - A[2];
        const float dd = dxb_fma(dx, dx, dxb_fma(dy, dy, dz * dz));
        const float t = dxb_fma(p.x - ctr[0] - A[0], dx, dxb_fma(p.y - ctr[1] - A[1], dy, (p.z - ctr[2] - A[2]) * dz));
        const bool sw = (t * 2.0f > dd);
        for (int c = 0; c < 3; ++c)
        {
            const float a = fminf(fmaxf(A[c] + ctr[c], bnd[c]), bnd[3 + c]), b = fminf(fmaxf(B[c] + ctr[c], bnd[c]), bnd[3 + c]);
            E0[c] = sw ? b : a; E1[c] = sw ? a : b;
        }
    }
}

#if !DXB_ON_DEVICE
// test-infrastructure hooks of the host emulator only (tests/bc67_blocks/record_host.cpp), null / -1 by default.
// Record: per half, the winning mode index and shape (0 for one region), the quantised endpoints A0 B0 A1 B1 before the delta
// transform, the 16 indices and the INT-domain value each pixel's index selects from the exact palette (what the decoder must return).
struct dxb_bc6h_dbg_block { int32_t mode, shape, wq[12], idx[16], texel[16][3]; };
static thread_local dxb_bc6h_dbg_block* dxb_bc6h_dbg_rec = nullptr;                 // [2]: half 0, half 1
// Force, per half: mode (0..13) leaves dxb_bc6h_pick_mode that mode and its always-fitting fallback and drops every candidate of
// another mode from the winner search; shape (0..31) replaces every two-region candidate shape.
struct dxb_bc6h_dbg_forcing { int32_t mode, shape; };
static thread_local const dxb_bc6h_dbg_forcing* dxb_bc6h_dbg_force = nullptr;       // [2]
static thread_local int32_t dxb_bc6h_dbg_pick_only = -1;                             // the forced mode of the lane being picked
#endif

// ---------------------------------------------------------------------------------------------------
// stage 3: pick the mode for a set of endpoints (ep[4][3]: A0 B0 A1 B1, INT domain) and quantise them.
//   two = two regions.  Returns the mode index (0..13); q[4][3] = quantised endpoints (not yet delta-transformed).
DXB_DEV int dxb_bc6h_pick_mode(const int32_t ep[4][3], bool two, bool bSigned, int32_t q[4][3])
{
    // candidates in decreasing base precision; the last of each list has no delta restriction (always fits)
    const int order2[10] = { 2, 3, 4, 0, 5, 6, 7, 8, 1, 9 };
    const int order1[4] = { 13, 12, 11, 10 };          // mode 14 (16-bit endpoints, 4-bit deltas) reproduces near-flat blocks exactly
    const int ncand = two ? 10 : 4;
    const int nep = two ? 4 : 2;
    int chosen = two ? 9 : 10;
    int32_t q12[4][3], amag[4][3]; bool neg[4][3];
    for (int e = 0; e < 4; ++e)
        for (int c = 0; c < 3; ++c)
        {
            const int32_t v = ep[e][c];
            neg[e][c] = bSigned && (v < 0);
            const int32_t a = neg[e][c] ? -v : v;
            amag[e][c] = a;
            q12[e][c] = bSigned ? ((a << 11) / (0x7BFF + 1)) : ((a << 12) / (0x7BFF + 1));
        }
    for (int ci = 0; ci < ncand; ++ci)
    {
        const int m = two ? order2[ci] : order1[ci];
#if !DXB_ON_DEVICE
        if (dxb_bc6h_dbg_pick_only >= 0 && m != dxb_bc6h_dbg_pick_only && ci + 1 < ncand) continue;
#endif
        const uint32_t info = dxb_bc6h_info[m];
        const int32_t prec = (int32_t)((info >> 8) & 31u);
        const bool transformed = ((info >> 6) & 1u) != 0u;
        const int32_t db[3] = { (int32_t)((info >> 16) & 15u), (int32_t)((info >> 20) & 15u), (int32_t)((info >> 24) & 15u) };
        int32_t t[4][3];
        bool ok = true;
        const int32_t qhi = bSigned ? ((1 << (prec - 1)) - 1) : ((1 << prec) - 1);
        // Quantize(v, prec) = floor(|v| 2^prec' / 31744) (:1864-1889) = the 12-bit quantisation shifted down, because
        // nested floor divisions compose; magnitudes and signs are handled apart for the signed format
        for (int e = 0; e < nep; ++e)
            for (int c = 0; c < 3; ++c)
            {
                // prec >= 15 (unsigned) / 16 (signed): the decoder passes the code through Unquantize and scales it by 31/64
                // (31/32 signed) in FinishUnquantize (:1893-1940); the smallest code that decodes to exactly `a` is
                // ceil(a * 64 / 31) (ceil(a * 32 / 31)).  (The reference's own Quantize returns `a` here, :1872, 1885, which
                // decodes to half the value, so its encoder never benefits from mode 14.)
                const bool full = prec >= (bSigned ? 16 : 15);
                const int32_t a = amag[e][c];
                const int32_t wide = bSigned ? ((a * 32 + 30) / 31) : ((a * 64 + 30) / 31);
                const int32_t mag = full ? ((wide > (bSigned ? 0x7FFF : 0xFFFF)) ? (bSigned ? 0x7FFF : 0xFFFF) : wide)
                                         : (q12[e][c] >> (full ? 0 : (12 - prec)));
                t[e][c] = neg[e][c] ? -mag : mag;
            }
        // a region whose two endpoints quantise to the same code wastes its interpolation levels: open the pair by one
        // code so that the 8/16 palette entries subdivide the quantisation step (what the reference's perturbation finds)
        for (int r = 0; r < nep; r += 2)
            for (int c = 0; c < 3; ++c)
                if (t[r][c] == t[r + 1][c])
                {
                    if (t[r + 1][c] < qhi) t[r + 1][c] += 1; else t[r][c] -= 1;
                }
        for (int e = 1; e < nep; ++e)
            for (int c = 0; c < 3; ++c)
                if (transformed) ok = ok && dxb_fits_signed(t[e][c] - t[0][c], db[c]);
        if (ok)
        {
            chosen = m;
            for (int e = 0; e < nep; ++e) for (int c = 0; c < 3; ++c) q[e][c] = t[e][c];
            break;
        }
    }
    return chosen;
}

// decoded endpoint value of code q (weight 0 / 64): FinishUnquantize(Unquantize(q)) = the magnitude scaled by 31/64 (31/32
// signed) and truncated (:1932-1942), as float.  |unq| < 2^16, so the product is exact in fp32 and truncf reproduces the shift.
DXB_DEV float dxb_bc6h_decoded_endpoint(int32_t q, int32_t prec, bool bSigned)
{
    return truncf((float)dxb_bc6h_unquantize(q, prec, bSigned) * (bSigned ? (31.0f / 32.0f) : (31.0f / 64.0f)));
}

// error of one region for quantised endpoints qa/qb at `prec` bits, used to RANK the candidate shapes: indices by
// projection, decoded values modelled in float as in dxb_bc6h_refine_region (within 2 units of the decoder's integers;
// the winner's indices are then chosen exhaustively against the exact palette in stage 4)
template <int NIDX>
DXB_DEV float dxb_bc6h_region_error(const dxb_px* px, uint32_t mask, const float* ctr, const int32_t* qa, const int32_t* qb, int32_t prec, bool bSigned)
{
    const float nmax = (float)(NIDX - 1), c64 = 64.0f / nmax;
    float A[3], D[3];
    for (int c = 0; c < 3; ++c)
    {
        A[c] = dxb_bc6h_decoded_endpoint(qa[c], prec, bSigned) - ctr[c];
        D[c] = (dxb_bc6h_decoded_endpoint(qb[c], prec, bSigned) - ctr[c]) - A[c];
    }
    const float dd = dxb_fma(D[0], D[0], dxb_fma(D[1], D[1], D[2] * D[2]));
    const float idd = (dd > 0.0f) ? nmax / dd : 0.0f;
    float tot = 0.0f;
#if DXB_ON_DEVICE
    #pragma unroll 4
#endif
    for (int i = 0; i < 16; ++i)
    {
        const float f = dxb_bit_as_float(mask, i);
        const dxb_px p = px[i];
        const float X = p.x - ctr[0] - A[0], Y = p.y - ctr[1] - A[1], Z = p.z - ctr[2] - A[2];
        const float t = dxb_fma(X, D[0], dxb_fma(Y, D[1], Z * D[2])) * idd;
        const float sk = dxb_bc7_weightf(dxb_rne(fminf(fmaxf(t, 0.0f), nmax)), c64);
        const float ex = dxb_fma(-sk, D[0], X), ey = dxb_fma(-sk, D[1], Y), ez = dxb_fma(-sk, D[2], Z);
        tot = dxb_fma(f, dxb_fma(ex, ex, dxb_fma(ey, ey, ez * ez)), tot);
    }
    return tot;
}

// +-1 code refinement of one region's quantised endpoints: alternate (1) index assignment by projection onto the current
// decoded segment and (2), with the interpolation weights s_i fixed, the best of the 3x3 neighbouring code pairs per
// channel.  With fixed weights the error of a channel is the quadratic
//     e(A, B) = A^2 sum(1-s)^2 + 2 A B sum s(1-s) + B^2 sum s^2 - 2 A sum (1-s) v - 2 B sum s v  (+ const)
// in the decoded endpoints A, B, so one pass over the pixels gives five sums and every candidate costs a few FMAs.
// Decoded values are modelled in float as unquantize(code) * 31/64 (31/32 signed), i.e. without the decoder's two
// floor operations (< 2 units of 65536); the caller re-measures the result against the exact palette.
// Everything is centred on `ctr` to keep the fp32 sums well conditioned.
template <int NIDX>
DXB_DEV void dxb_bc6h_refine_region(const dxb_px* px, uint32_t mask, const float* ctr, int32_t* qa, int32_t* qb, int32_t prec, bool bSigned, const float* bnd)
{
    const float nmax = (float)(NIDX - 1), c64 = 64.0f / nmax;
    const int32_t qlo = bSigned ? -((1 << (prec - 1)) - 1) : 0, qhi = bSigned ? ((1 << (prec - 1)) - 1) : ((1 << prec) - 1);
    for (int iter = 0; iter < 2; ++iter)
    {
        float A[3], D[3];
        for (int c = 0; c < 3; ++c)
        {
            A[c] = dxb_bc6h_decoded_endpoint(qa[c], prec, bSigned) - ctr[c];
            D[c] = (dxb_bc6h_decoded_endpoint(qb[c], prec, bSigned) - ctr[c]) - A[c];
        }
        const float dd = dxb_fma(D[0], D[0], dxb_fma(D[1], D[1], D[2] * D[2]));
        const float idd = (dd > 0.0f) ? nmax / dd : 0.0f;
        float soo = 0, sos = 0, sss = 0, u0 = 0, u1 = 0, u2 = 0, v0 = 0, v1 = 0, v2 = 0;
#if DXB_ON_DEVICE
        #pragma unroll 4
#endif
        for (int i = 0; i < 16; ++i)
        {
            const float f = dxb_bit_as_float(mask, i);
            const dxb_px p = px[i];
            const float X = p.x - ctr[0], Y = p.y - ctr[1], Z = p.z - ctr[2];
            const float t = dxb_fma(X - A[0], D[0], dxb_fma(Y - A[1], D[1], (Z - A[2]) * D[2])) * idd;
            const float sk = dxb_bc7_weightf(dxb_rne(fminf(fmaxf(t, 0.0f), nmax)), c64);
            const float skf = sk * f, osf = f - skf, os = 1.0f - sk;
            soo = dxb_fma(osf, os, soo); sos = dxb_fma(osf, sk, sos); sss = dxb_fma(skf, sk, sss);
            u0 = dxb_fma(osf, X, u0); u1 = dxb_fma(osf, Y, u1); u2 = dxb_fma(osf, Z, u2);
            v0 = dxb_fma(skf, X, v0); v1 = dxb_fma(skf, Y, v1); v2 = dxb_fma(skf, Z, v2);
        }
        const float U[3] = { u0, u1, u2 }, V[3] = { v0, v1, v2 };
        for (int c = 0; c < 3; ++c)
        {
            float ca[3], cb[3];                                      // decoded, centred values of the 3 neighbouring codes
            for (int k = 0; k < 3; ++k)
            {
                ca[k] = dxb_bc6h_decoded_endpoint(qa[c] + k - 1, prec, bSigned) - ctr[c];
                cb[k] = dxb_bc6h_decoded_endpoint(qb[c] + k - 1, prec, bSigned) - ctr[c];
            }
            float bestE = 3.0e38f; int32_t ba = qa[c], bb = qb[c];
            for (int da = 0; da < 3; ++da)
                for (int dbb = 0; dbb < 3; ++dbb)
                {
                    const int32_t a = qa[c] + da - 1, b = qb[c] + dbb - 1;
                    const float Av = ca[da], Bv = cb[dbb];
                    // a neighbouring code must decode inside the clamp range of its channel (dxb_bc6h_fit); the centre pair always may stay
                    const float blo = bnd[c] - ctr[c] - 0.5f, bhi = bnd[3 + c] - ctr[c] + 0.5f;
                    const bool inb = (da == 1 || (Av >= blo && Av <= bhi)) && (dbb == 1 || (Bv >= blo && Bv <= bhi));
                    const bool ok = !(a < qlo || a > qhi || b < qlo || b > qhi) && inb;
                    // A (A soo + 2 B sos - 2 U) + B (B sss - 2 V)
                    const float e = dxb_fma(Av, dxb_fma(Av, soo, dxb_fma(Bv + Bv, sos, -(U[c] + U[c]))), Bv * dxb_fma(Bv, sss, -(V[c] + V[c])));
                    if (ok && e < bestE) { bestE = e; ba = a; bb = b; }
                }
            qa[c] = ba; qb[c] = bb;
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// The encoder proper, SPMD over the warp: TWO blocks per warp, one per 16-lane half (as dxb_bc7_encode_pair).
//   spx : 32 pixels in the INT domain (x,y,z; w unused): spx[16 h + i] = pixel i of the half-h block
//   out0/out1 : 16 output bytes of the half-0 / half-1 block (nullptr = that half carries no block)
// Per block: stage 1 ranks the 32 two-region shapes (2 per lane) and keeps 7; stage 2/3 lanes 0..13 = 7 shapes x 2
// regions, lane 14 = the one-region fit, lane 15 idles on a copy; stage 4 lanes = pixels.
#define DXB_BC6H_KSHAPES 7

DXB_DEV void dxb_bc6h_encode_pair(const dxb_px* spx, bool bSigned, uint8_t* out0, uint8_t* out1)
{
    const float lo = bSigned ? -31743.0f : 0.0f, hi = 31743.0f;

    // ---- block centre (keeps the fp32 moments well conditioned: values are up to 3e4, squares 1e9) and stage 1
    float cx[DXB_NL], cy[DXB_NL], cz[DXB_NL];
    uint32_t sel[DXB_BC6H_KSHAPES][DXB_NL];
    {
        uint32_t k0[DXB_NL], k1[DXB_NL];
        DXB_LANES_BEGIN
            const dxb_px* px = spx + (lane & 16);
            float ctr[3] = { 0, 0, 0 };
            for (int i = 0; i < 16; ++i) { ctr[0] += px[i].x; ctr[1] += px[i].y; ctr[2] += px[i].z; }
            ctr[0] *= (1.0f / 16.0f); ctr[1] *= (1.0f / 16.0f); ctr[2] *= (1.0f / 16.0f);
            cx[L] = ctr[0]; cy[L] = ctr[1]; cz[L] = ctr[2];
            // centred moments (scaled by 2^-7, exact: dxb_bc7_subset_estimate needs covariance entries below ~5e6) of
            // subset 1 of this lane's two shapes and of the whole block
            const uint32_t maskA = dxb_part2[lane & 15], maskB = dxb_part2[(lane & 15) + 16];
            float sa[3] = { 0, 0, 0 }, ma[6] = { 0, 0, 0, 0, 0, 0 }, sb[3] = { 0, 0, 0 }, mb[6] = { 0, 0, 0, 0, 0, 0 };
            float ts[3] = { 0, 0, 0 }, tm[6] = { 0, 0, 0, 0, 0, 0 };
#if DXB_ON_DEVICE
            #pragma unroll 4
#endif
            for (int i = 0; i < 16; ++i)
            {
                const float fa = dxb_bit_as_float(maskA, i), fb = dxb_bit_as_float(maskB, i);
                const dxb_px p = px[i];
                const float X = (p.x - ctr[0]) * (1.0f / 128.0f), Y = (p.y - ctr[1]) * (1.0f / 128.0f), Z = (p.z - ctr[2]) * (1.0f / 128.0f);
                const float xx = X * X, xy = X * Y, xz = X * Z, yy = Y * Y, yz = Y * Z, zz = Z * Z;
                ts[0] += X; ts[1] += Y; ts[2] += Z;
                tm[0] += xx; tm[1] += xy; tm[2] += xz; tm[3] += yy; tm[4] += yz; tm[5] += zz;
                sa[0] = dxb_fma(fa, X, sa[0]); sa[1] = dxb_fma(fa, Y, sa[1]); sa[2] = dxb_fma(fa, Z, sa[2]);
                ma[0] = dxb_fma(fa, xx, ma[0]); ma[1] = dxb_fma(fa, xy, ma[1]); ma[2] = dxb_fma(fa, xz, ma[2]);
                ma[3] = dxb_fma(fa, yy, ma[3]); ma[4] = dxb_fma(fa, yz, ma[4]); ma[5] = dxb_fma(fa, zz, ma[5]);
                sb[0] = dxb_fma(fb, X, sb[0]); sb[1] = dxb_fma(fb, Y, sb[1]); sb[2] = dxb_fma(fb, Z, sb[2]);
                mb[0] = dxb_fma(fb, xx, mb[0]); mb[1] = dxb_fma(fb, xy, mb[1]); mb[2] = dxb_fma(fb, xz, mb[2]);
                mb[3] = dxb_fma(fb, yy, mb[3]); mb[4] = dxb_fma(fb, yz, mb[4]); mb[5] = dxb_fma(fb, zz, mb[5]);
            }
            uint32_t key[2];
            for (int j = 0; j < 2; ++j)
            {
                const float* s = j ? sb : sa; const float* m = j ? mb : ma;
                const uint32_t mask1 = j ? maskB : maskA;
                const float v1[14] = { s[0], s[1], s[2], 0.0f, m[0], m[1], m[2], 0.0f, m[3], m[4], 0.0f, m[5], 0.0f, 0.0f };
                const float v0[14] = { ts[0] - s[0], ts[1] - s[1], ts[2] - s[2], 0.0f, tm[0] - m[0], tm[1] - m[1], tm[2] - m[2], 0.0f,
                                       tm[3] - m[3], tm[4] - m[4], 0.0f, tm[5] - m[5], 0.0f, 0.0f };
                const uint32_t c1 = dxb_popc16(mask1);
                const float est = dxb_bc7_subset_estimate(16u - c1, v0, 1.0f / 49.0f) + dxb_bc7_subset_estimate(c1, v1, 1.0f / 49.0f);
                key[j] = (dxb_float_as_uint(fmaxf(est, 0.0f)) & 0xFFFFFFE0u) | ((uint32_t)(lane & 15) + 16u * (uint32_t)j);
            }
            k0[L] = (key[0] < key[1]) ? key[0] : key[1];
            k1[L] = (key[0] < key[1]) ? key[1] : key[0];
        DXB_LANES_END
        for (int r = 0; r < DXB_BC6H_KSHAPES; ++r)
        {
            uint32_t win[DXB_NL];
            dxb_half_min_u32(k0, win);
            DXB_LANES_BEGIN
                sel[r][L] = win[L] & 31u;
                if (k0[L] == win[L]) { k0[L] = k1[L]; k1[L] = 0xFFFFFFFFu; }
            DXB_LANES_END
        }
#if !DXB_ON_DEVICE
        DXB_LANES_BEGIN
            if (dxb_bc6h_dbg_force && dxb_bc6h_dbg_force[lane >> 4].shape >= 0)
                for (int r = 0; r < DXB_BC6H_KSHAPES; ++r) sel[r][L] = (uint32_t)dxb_bc6h_dbg_force[lane >> 4].shape;
        DXB_LANES_END
#endif
    }

    // ---- stage 2: continuous fits
    float e0x[DXB_NL], e0y[DXB_NL], e0z[DXB_NL], e1x[DXB_NL], e1y[DXB_NL], e1z[DXB_NL];
    uint32_t tShape[DXB_NL], tMask[DXB_NL];
    float tBnd[6][DXB_NL];
    DXB_LANES_BEGIN
        const int hl = lane & 15;
        const bool one = (hl >= 2 * DXB_BC6H_KSHAPES);
        uint32_t shape = 0;
        for (int r = 0; r < DXB_BC6H_KSHAPES; ++r) shape = ((hl >> 1) == r) ? sel[r][L] : shape;
        const uint32_t m1 = dxb_part2[shape];
        const uint32_t mask = one ? 0xFFFFu : ((hl & 1) ? m1 : (~m1 & 0xFFFFu));
        const int anchor = one ? 0 : ((hl & 1) ? (int)dxb_anchor2[shape] : 0);
        const float ctr[3] = { cx[L], cy[L], cz[L] };
        float E0[3], E1[3];
        float bnd[6];
        dxb_bc6h_fit(spx + (lane & 16), mask, one ? 4u : 3u, anchor, ctr, lo, hi, bSigned, E0, E1, bnd);
        for (int k = 0; k < 6; ++k) tBnd[k][L] = bnd[k];
        e0x[L] = E0[0]; e0y[L] = E0[1]; e0z[L] = E0[2]; e1x[L] = E1[0]; e1y[L] = E1[1]; e1z[L] = E1[2];
        tShape[L] = one ? 0u : shape; tMask[L] = mask;
    DXB_LANES_END

    // ---- stage 3: partner exchange, mode choice, refinement, region error
    float p0x[DXB_NL], p0y[DXB_NL], p0z[DXB_NL], p1x[DXB_NL], p1y[DXB_NL], p1z[DXB_NL];
    dxb_xchg_xor_f32(e0x, p0x, 1); dxb_xchg_xor_f32(e0y, p0y, 1); dxb_xchg_xor_f32(e0z, p0z, 1);
    dxb_xchg_xor_f32(e1x, p1x, 1); dxb_xchg_xor_f32(e1y, p1y, 1); dxb_xchg_xor_f32(e1z, p1z, 1);
    uint32_t rMode[DXB_NL];
    float rErrF[DXB_NL];
    uint32_t rq[12][DXB_NL];            // quantised endpoints A0 B0 A1 B1 (two's complement ints)
    uint32_t mine[6][DXB_NL], theirs[6][DXB_NL];      // refined endpoints of this lane's region / of the partner's
    DXB_LANES_BEGIN
        const int hl = lane & 15;
        const bool one = (hl >= 2 * DXB_BC6H_KSHAPES);
        const bool second = !one && (hl & 1);
        const float ctr[3] = { cx[L], cy[L], cz[L] };
        int32_t ep[4][3];
        // region 0 endpoints come from the even lane, region 1 from the odd lane
        const float mine0[3] = { e0x[L], e0y[L], e0z[L] }, mine1[3] = { e1x[L], e1y[L], e1z[L] };
        const float oth0[3] = { p0x[L], p0y[L], p0z[L] }, oth1[3] = { p1x[L], p1y[L], p1z[L] };
        for (int c = 0; c < 3; ++c)
        {
            const float a0 = second ? oth0[c] : mine0[c], b0 = second ? oth1[c] : mine1[c];
            const float a1 = second ? mine0[c] : oth0[c], b1 = second ? mine1[c] : oth1[c];
            ep[0][c] = dxb_f2i(dxb_rne(a0)); ep[1][c] = dxb_f2i(dxb_rne(b0));
            ep[2][c] = dxb_f2i(dxb_rne(a1)); ep[3][c] = dxb_f2i(dxb_rne(b1));
        }
        int32_t q[4][3];
        for (int e = 0; e < 4; ++e) for (int c = 0; c < 3; ++c) q[e][c] = 0;
#if !DXB_ON_DEVICE
        dxb_bc6h_dbg_pick_only = dxb_bc6h_dbg_force ? dxb_bc6h_dbg_force[lane >> 4].mode : -1;
#endif
        const int mode = dxb_bc6h_pick_mode(ep, !one, bSigned, q);
#if !DXB_ON_DEVICE
        dxb_bc6h_dbg_pick_only = -1;
#endif
        const int32_t prec = (int32_t)((dxb_bc6h_info[mode] >> 8) & 31u);
        // +-1 code refinement of this lane's own region
        int32_t qa[3], qb[3];
        for (int c = 0; c < 3; ++c) { qa[c] = second ? q[2][c] : q[0][c]; qb[c] = second ? q[3][c] : q[1][c]; }
        const float bnd[6] = { tBnd[0][L], tBnd[1][L], tBnd[2][L], tBnd[3][L], tBnd[4][L], tBnd[5][L] };
        if (one) dxb_bc6h_refine_region<16>(spx + (lane & 16), 0xFFFFu, ctr, qa, qb, prec, bSigned, bnd);
        else dxb_bc6h_refine_region<8>(spx + (lane & 16), tMask[L], ctr, qa, qb, prec, bSigned, bnd);
        for (int c = 0; c < 3; ++c) { mine[c][L] = (uint32_t)qa[c]; mine[3 + c][L] = (uint32_t)qb[c]; }
        rMode[L] = (uint32_t)mode;
        for (int e = 0; e < 4; ++e) for (int c = 0; c < 3; ++c) rq[e * 3 + c][L] = (uint32_t)q[e][c];
    DXB_LANES_END
    for (int k = 0; k < 6; ++k) dxb_xchg_xor_u32(mine[k], theirs[k], 1);
    DXB_LANES_BEGIN
        const int hl = lane & 15;
        const bool one = (hl >= 2 * DXB_BC6H_KSHAPES);
        const bool second = !one && (hl & 1);
        const float ctr[3] = { cx[L], cy[L], cz[L] };
        const int mode = (int)rMode[L];
        const uint32_t info = dxb_bc6h_info[mode];
        const int32_t prec = (int32_t)((info >> 8) & 31u);
        const bool transformed = ((info >> 6) & 1u) != 0u;
        const int32_t db[3] = { (int32_t)((info >> 16) & 15u), (int32_t)((info >> 20) & 15u), (int32_t)((info >> 24) & 15u) };
        // refined set of all endpoints (identical on both lanes of a pair): keep it only if the deltas still fit
        int32_t r[4][3];
        for (int c = 0; c < 3; ++c)
        {
            const int32_t ma = (int32_t)mine[c][L], mb = (int32_t)mine[3 + c][L];
            const int32_t ta = one ? 0 : (int32_t)theirs[c][L], tb = one ? 0 : (int32_t)theirs[3 + c][L];
            r[0][c] = second ? ta : ma; r[1][c] = second ? tb : mb;
            r[2][c] = second ? ma : ta; r[3][c] = second ? mb : tb;
        }
        bool ok = true;
        if (transformed)
            for (int e = 1; e < (one ? 2 : 4); ++e)
                for (int c = 0; c < 3; ++c) ok = ok && dxb_fits_signed(r[e][c] - r[0][c], db[c]);
        int32_t q[4][3];
        for (int e = 0; e < 4; ++e) for (int c = 0; c < 3; ++c) q[e][c] = ok ? r[e][c] : (int32_t)rq[e * 3 + c][L];
        float err;
        if (one) err = dxb_bc6h_region_error<16>(spx + (lane & 16), 0xFFFFu, ctr, q[0], q[1], prec, bSigned);
        else err = dxb_bc6h_region_error<8>(spx + (lane & 16), tMask[L], ctr, second ? q[2] : q[0], second ? q[3] : q[1], prec, bSigned);
        rErrF[L] = (hl == 15) ? 3.0e38f : fminf(fmaxf(err, 0.0f), 3.0e37f);
        for (int e = 0; e < 4; ++e) for (int c = 0; c < 3; ++c) rq[e * 3 + c][L] = (uint32_t)q[e][c];
    DXB_LANES_END
    // winner key: the bit pattern of a non-negative float orders like the float itself, so the top 27 bits of the summed
    // error keep a relative resolution of 2^-18 over the whole range (a fixed-point key rounded all small errors to zero and
    // let a coarse two-region candidate beat an exact one-region one on flat blocks)
    float partnerF[DXB_NL];
    dxb_xchg_xor_f32(rErrF, partnerF, 1);
    uint32_t wkeys[DXB_NL], wkey[DXB_NL], src[DXB_NL];
    DXB_LANES_BEGIN
        const int hl = lane & 15;
        float e = rErrF[L];
        if (hl < 2 * DXB_BC6H_KSHAPES) e = e + partnerF[L];
        wkeys[L] = ((dxb_float_as_uint(e) >> 5) << 4) | (uint32_t)hl;
#if !DXB_ON_DEVICE
        if (dxb_bc6h_dbg_force && dxb_bc6h_dbg_force[lane >> 4].mode >= 0 && (int32_t)rMode[L] != dxb_bc6h_dbg_force[lane >> 4].mode)
            wkeys[L] = 0xFFFFFFE0u | (uint32_t)hl;
#endif
        if (hl == 15) wkeys[L] = 0xFFFFFFFFu;
    DXB_LANES_END
    dxb_half_min_u32(wkeys, wkey);
    DXB_LANES_BEGIN
        src[L] = (wkey[L] & 15u) & ~1u;                      // even lane of the winning pair (lane 14 for one region)
    DXB_LANES_END
    uint32_t wMode[DXB_NL], wShape[DXB_NL], wq[12][DXB_NL];
    dxb_half_gather_u32(rMode, src, wMode);
    dxb_half_gather_u32(tShape, src, wShape);
    for (int k = 0; k < 12; ++k) dxb_half_gather_u32(rq[k], src, wq[k]);

    // ---- stage 4: indices against the exact palette (lane = pixel)
    uint32_t idx[DXB_NL];
    DXB_LANES_BEGIN
        const uint32_t hl = (uint32_t)(lane & 15);
        const bool two = (src[L] < 2u * DXB_BC6H_KSHAPES);
        const uint32_t info = dxb_bc6h_info[wMode[L]];
        const int32_t prec = (int32_t)((info >> 8) & 31u);
        const uint32_t ib = two ? 3u : 4u;
        const uint32_t part = two ? dxb_part2[wShape[L]] : 0u;
        const uint32_t anchor1 = two ? dxb_anchor2[wShape[L]] : 0u;
        const int r = (int)((part >> hl) & 1u);
        int32_t ua[3], ub[3];
        for (int c = 0; c < 3; ++c)
        {
            ua[c] = dxb_bc6h_unquantize((int32_t)(r ? wq[6 + c][L] : wq[c][L]), prec, bSigned);
            ub[c] = dxb_bc6h_unquantize((int32_t)(r ? wq[9 + c][L] : wq[3 + c][L]), prec, bSigned);
        }
        const dxb_px p = spx[lane];
        const bool isAnchor = (hl == 0) || (two && hl == anchor1);
        const uint32_t nk = isAnchor ? (1u << (ib - 1u)) : (1u << ib);       // anchors only have ib-1 bits
        float best = 3.0e38f; uint32_t bk = 0;
#if DXB_ON_DEVICE
        #pragma unroll 2
#endif
        for (uint32_t k = 0; k < 16u; ++k)
        {
            const int32_t w = (int32_t)dxb_bc7_weight(ib, k);
            const float dx = p.x - (float)dxb_bc6h_palette(ua[0], ub[0], w, bSigned);
            const float dy = p.y - (float)dxb_bc6h_palette(ua[1], ub[1], w, bSigned);
            const float dz = p.z - (float)dxb_bc6h_palette(ua[2], ub[2], w, bSigned);
            const float e = dxb_fma(dx, dx, dxb_fma(dy, dy, dz * dz));
            if (k < nk && e < best) { best = e; bk = k; }
        }
        idx[L] = bk;
#if !DXB_ON_DEVICE
        if (dxb_bc6h_dbg_rec)
        {
            dxb_bc6h_dbg_block& R = dxb_bc6h_dbg_rec[lane >> 4];
            R.idx[hl] = (int32_t)bk;
            for (int c = 0; c < 3; ++c) R.texel[hl][c] = dxb_bc6h_palette(ua[c], ub[c], (int32_t)dxb_bc7_weight(ib, bk), bSigned);
            if (hl == 0)
            {
                R.mode = (int32_t)wMode[L]; R.shape = two ? (int32_t)wShape[L] : 0;
                for (int k = 0; k < 12; ++k) R.wq[k] = (int32_t)wq[k][L];
            }
        }
#endif
    DXB_LANES_END

    // header fields: endpoint 0 A as is, the others as deltas in transformed modes, masked to their field widths;
    // lane l deposits header bits l, l+16, l+32, ... and its pixel's index field
    uint32_t w0[DXB_NL], w1[DXB_NL], w2[DXB_NL], w3[DXB_NL];
    DXB_LANES_BEGIN
        const uint32_t hl = (uint32_t)(lane & 15);
        const bool two = (src[L] < 2u * DXB_BC6H_KSHAPES);
        const uint32_t mode = wMode[L];
        const uint32_t info = dxb_bc6h_info[mode];
        const int32_t prec = (int32_t)((info >> 8) & 31u);
        const bool transformed = ((info >> 6) & 1u) != 0u;
        const uint32_t ib = two ? 3u : 4u;
        const uint32_t anchor1 = two ? dxb_anchor2[wShape[L]] : 0u;
        const int32_t db[3] = { (int32_t)((info >> 16) & 15u), (int32_t)((info >> 20) & 15u), (int32_t)((info >> 24) & 15u) };
        uint32_t field[15];
        field[0] = 0; field[1] = info & 31u; field[2] = wShape[L];
        for (int c = 0; c < 3; ++c)
        {
            const uint32_t m0 = (prec >= 32) ? 0xFFFFFFFFu : ((1u << prec) - 1u);
            const uint32_t md = transformed ? ((1u << db[c]) - 1u) : m0;
            const int32_t a0 = (int32_t)wq[c][L], b0 = (int32_t)wq[3 + c][L], a1 = (int32_t)wq[6 + c][L], b1 = (int32_t)wq[9 + c][L];
            field[3 + 4 * c + 0] = (uint32_t)a0 & m0;
            field[3 + 4 * c + 1] = (uint32_t)(transformed ? b0 - a0 : b0) & md;
            field[3 + 4 * c + 2] = (uint32_t)(transformed ? a1 - a0 : a1) & md;
            field[3 + 4 * c + 3] = (uint32_t)(transformed ? b1 - a0 : b1) & md;
        }
        const uint32_t hdrBits = two ? 82u : 65u;
        dxb_u128 bits; bits.lo = 0; bits.hi = 0;
        for (uint32_t b = hl; b < hdrBits; b += 16u)
        {
            const uint32_t d = dxb_bc6h_desc[mode][b];
            uint32_t f = 0;
            // field[] is indexed with a lane-varying value: select chain keeps it in registers
            const uint32_t fi = d >> 4;
            for (uint32_t k = 1; k < 15; ++k) f = (fi == k) ? field[k] : f;
            dxb_put_bits(&bits, b, 1, (f >> (d & 15u)) & 1u);
        }
        {
            const uint32_t before = (hl > 0 ? 1u : 0u) + ((two && hl > anchor1) ? 1u : 0u);
            const bool isAnchor = (hl == 0) || (two && hl == anchor1);
            dxb_put_bits(&bits, hdrBits + hl * ib - before, isAnchor ? ib - 1u : ib, idx[L]);
        }
        w0[L] = (uint32_t)bits.lo; w1[L] = (uint32_t)(bits.lo >> 32); w2[L] = (uint32_t)bits.hi; w3[L] = (uint32_t)(bits.hi >> 32);
    DXB_LANES_END
    uint32_t o0[DXB_NL], o1[DXB_NL], o2[DXB_NL], o3[DXB_NL];
    dxb_half_or_u32(w0, o0); dxb_half_or_u32(w1, o1); dxb_half_or_u32(w2, o2); dxb_half_or_u32(w3, o3);
    DXB_LANES_BEGIN
        uint8_t* out = (lane & 16) ? out1 : out0;
        if ((lane & 15) == 0 && out)
        {
            uint32_t* o = (uint32_t*)out;
            o[0] = o0[L]; o[1] = o1[L]; o[2] = o2[L]; o[3] = o3[L];
        }
    DXB_LANES_END
}

#if !DXB_ON_DEVICE
// emulator entry: pxA / pxB = 16 RGBA fp32 pixels each after ConvertScanline; pxB / outB may be null (odd block count)
static inline void dxb_bc6h_encode_pair_emul(const dxb_px* pxA, const dxb_px* pxB, bool bSigned, uint8_t* outA, uint8_t* outB)
{
    dxb_px ip[32];
    for (int i = 0; i < 16; ++i)
    {
        ip[i] = dxb_make_px(dxb_bc6h_to_int(pxA[i].x, bSigned), dxb_bc6h_to_int(pxA[i].y, bSigned), dxb_bc6h_to_int(pxA[i].z, bSigned), 0.0f);
        ip[16 + i] = pxB ? dxb_make_px(dxb_bc6h_to_int(pxB[i].x, bSigned), dxb_bc6h_to_int(pxB[i].y, bSigned), dxb_bc6h_to_int(pxB[i].z, bSigned), 0.0f)
                         : dxb_make_px(0.0f, 0.0f, 0.0f, 0.0f);
    }
    dxb_bc6h_encode_pair(ip, bSigned, outA, pxB ? outB : nullptr);
}
#endif
