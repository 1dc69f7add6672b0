// tests/bc67_blocks/record_host.cpp — TEST INFRASTRUCTURE, never shipped (tests/bc67_blocks_lib.py builds it).
//
// The host emulator (tests/emul/emul.cpp, the same shared sources as the sm_90a kernels) plus one entry point that encodes an image to
// BC6H or BC7 as emul_compress does and records, for every block, what the encoder chose and what the block must decode to, through
// the encoders' host-only hooks dxb_bc7_dbg_rec / dxb_bc6h_dbg_rec; optionally with per-block forcing (dxb_bc7_dbg_force /
// dxb_bc6h_dbg_force).  Built with the emulator's compiler flags (tests/emul/build.sh).
#define DXB_EMUL_BC7
#include "../emul/emul.cpp"

#define REC_WORDS 80

// One block's record, REC_WORDS int32 words:
//   BC7:  mode, shape, rot, idx, q0[3], q1[3], pb[3], err, idxC[16], idxA[16], texel[16] (natural RGBA bytes, R low)
//   BC6H: mode, shape, wq[12], idx[16], texel[16][3] (INT domain)
static void put_bc7(const dxb_bc7_dbg_block& B, int32_t* r)
{
    const dxb_bc7_win& W = B.w;
    r[0] = (int32_t)W.mode; r[1] = (int32_t)W.shape; r[2] = (int32_t)W.rot; r[3] = (int32_t)W.idx;
    for (int s = 0; s < 3; ++s) { r[4 + s] = (int32_t)W.q0[s]; r[7 + s] = (int32_t)W.q1[s]; r[10 + s] = (int32_t)W.pb[s]; }
    r[13] = (int32_t)B.err;
    for (int i = 0; i < 16; ++i) { r[14 + i] = (int32_t)B.idxC[i]; r[30 + i] = (int32_t)B.idxA[i]; r[46 + i] = (int32_t)B.texel[i]; }
}
static void put_bc6h(const dxb_bc6h_dbg_block& B, int32_t* r)
{
    r[0] = B.mode; r[1] = B.shape;
    for (int k = 0; k < 12; ++k) r[2 + k] = B.wq[k];
    for (int i = 0; i < 16; ++i) { r[14 + i] = B.idx[i]; for (int c = 0; c < 3; ++c) r[30 + 3 * i + c] = B.texel[i][c]; }
}

// dst = the blocks, rec[REC_WORDS u ..] = the record of block u.  force = null (free) or per block 5 words (BC7: mode, rot, idx,
// shape, shape3) / 2 words (BC6H: mode, shape), -1 = free.  Returns the planner's HRESULT.
extern "C" int32_t record_compress(const uint8_t* src, size_t w, size_t h, uint32_t srcFmt, uint32_t dstFmt, uint32_t flags,
                                   const int32_t* force, uint8_t* dst, int32_t* rec)
{
    const dxb200_image s = emul_image(src, w, h, srcFmt, 0), d = emul_image(dst, w, h, dstFmt, 0);
    CompressPlan plan;
    const int32_t hr = plan_compress(&s, 1, dstFmt, flags, 0.5f, &d, &plan);
    if (hr != DXB_S_OK) return hr;
    if (!plan.bc7 && !plan.bc6h) return (int32_t)0x80070057;
    const uint32_t inF = plan.P.inF, outF = plan.P.outF, cflags = plan.P.cflags, bcflags = plan.P.bcflags;
    dxb_image_desc img; img.pixels = src; img.rowPitch = s.rowPitch; img.width = (uint32_t)w; img.height = (uint32_t)h; img.format = srcFmt;
    const uint32_t nbx = (uint32_t)((w + 3) / 4), nby = (uint32_t)((h + 3) / 4);
    const long total = (long)nbx * (long)nby;
    const bool bc7 = plan.bc7;
    #pragma omp parallel for schedule(dynamic, 32)
    for (long pair = 0; pair < (total + 1) / 2; ++pair)
    {
        dxb_px px[2][16];
        alignas(16) uint8_t blk[2][16];
        const long u0 = 2 * pair, u1 = u0 + 1;
        const bool has1 = u1 < total;
        dxb_gather_block(img, (uint32_t)(u0 % nbx), (uint32_t)(u0 / nbx), inF, outF, cflags, px[0]);
        if (has1) dxb_gather_block(img, (uint32_t)(u1 % nbx), (uint32_t)(u1 / nbx), inF, outF, cflags, px[1]);
        if (bc7)
        {
            dxb_bc7_dbg_block R[2];
            dxb_bc7_dbg_forcing F[2] = { { -1, -1, -1, -1, -1 }, { -1, -1, -1, -1, -1 } };
            for (long u = u0; force && u <= u1 && u < total; ++u)
            {
                const int32_t* f = force + 5 * u;
                F[u - u0] = { f[0], f[1], f[2], f[3], f[4] };
            }
            dxb_bc7_dbg_rec = R; dxb_bc7_dbg_force = force ? F : nullptr;
            dxb_bc7_encode_pair_emul(px[0], has1 ? px[1] : nullptr, bcflags, blk[0], blk[1]);
            dxb_bc7_dbg_rec = nullptr; dxb_bc7_dbg_force = nullptr;
            for (long u = u0; u <= u1 && u < total; ++u) put_bc7(R[u - u0], rec + REC_WORDS * u);
        }
        else
        {
            dxb_bc6h_dbg_block R[2];
            dxb_bc6h_dbg_forcing F[2] = { { -1, -1 }, { -1, -1 } };
            for (long u = u0; force && u <= u1 && u < total; ++u) F[u - u0] = { force[2 * u], force[2 * u + 1] };
            dxb_bc6h_dbg_rec = R; dxb_bc6h_dbg_force = force ? F : nullptr;
            dxb_bc6h_encode_pair_emul(px[0], has1 ? px[1] : nullptr, dstFmt == DXB_FMT_BC6H_SF16, blk[0], blk[1]);
            dxb_bc6h_dbg_rec = nullptr; dxb_bc6h_dbg_force = nullptr;
            for (long u = u0; u <= u1 && u < total; ++u) put_bc6h(R[u - u0], rec + REC_WORDS * u);
        }
        for (long u = u0; u <= u1 && u < total; ++u) memcpy(dst + (size_t)u * 16u, blk[u - u0], 16);
    }
    return DXB_S_OK;
}
