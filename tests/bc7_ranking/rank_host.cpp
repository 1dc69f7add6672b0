// tests/bc7_ranking/rank_host.cpp — TEST INFRASTRUCTURE, never shipped (tests/test_cpu_bc7_ranking.py builds it).
//
// The host emulator (tests/emul/emul.cpp, the same shared sources as the sm_90a kernels) plus one entry point that encodes an image to
// BC7 as emul_compress does and records BC7 stage 1 for every block through the encoder's host-only hook dxb_bc7_dbg_rank: the
// selected shapes, whether the block is opaque, the dxb_bc7_shape_h1 key of every shape and the part-B rounds of each block pair.
// Built with the emulator's compiler flags (tests/emul/build.sh).
#define DXB_EMUL_BC7
#include "../emul/emul.cpp"

// sel4[4 u ..] = the 3 selected shapes of block u and 1 if it is opaque, key64[64 u ..] = its keys, rounds[u / 2] = the rounds of its
// pair; dst = the BC7 blocks.  Returns the planner's HRESULT.
extern "C" int32_t rank_compress(const uint8_t* src, size_t w, size_t h, uint32_t srcFmt, uint32_t flags, uint8_t* dst,
                                 int32_t* sel4, uint32_t* key64, int32_t* rounds)
{
    const dxb200_image s = emul_image(src, w, h, srcFmt, 0), d = emul_image(dst, w, h, DXB_FMT_BC7_UNORM, 0);
    CompressPlan plan;
    const int32_t hr = plan_compress(&s, 1, DXB_FMT_BC7_UNORM, flags, 0.5f, &d, &plan);
    if (hr != DXB_S_OK) return hr;
    const uint32_t inF = plan.P.inF, outF = plan.P.outF, cflags = plan.P.cflags, bcflags = plan.P.bcflags;
    dxb_image_desc img; img.pixels = src; img.rowPitch = s.rowPitch; img.width = (uint32_t)w; img.height = (uint32_t)h; img.format = srcFmt;
    const uint32_t nbx = (uint32_t)((w + 3) / 4), nby = (uint32_t)((h + 3) / 4);
    const long total = (long)nbx * (long)nby;
    #pragma omp parallel for schedule(dynamic, 32)
    for (long pair = 0; pair < (total + 1) / 2; ++pair)
    {
        dxb_px px[2][16];
        alignas(16) uint8_t blk[2][16];
        const long u0 = 2 * pair, u1 = u0 + 1;
        dxb_gather_block(img, (uint32_t)(u0 % nbx), (uint32_t)(u0 / nbx), inF, outF, cflags, px[0]);
        if (u1 < total) dxb_gather_block(img, (uint32_t)(u1 % nbx), (uint32_t)(u1 / nbx), inF, outF, cflags, px[1]);
        dxb_bc7_dbg_stage1 rec;
        dxb_bc7_dbg_rank = &rec;
        dxb_bc7_encode_pair_emul(px[0], (u1 < total) ? px[1] : nullptr, bcflags, blk[0], blk[1]);
        dxb_bc7_dbg_rank = nullptr;
        rounds[pair] = (int32_t)rec.rounds;
        for (long u = u0; u <= u1 && u < total; ++u)
        {
            for (int r = 0; r < 4; ++r) sel4[4 * u + r] = (int32_t)rec.sel[u - u0][r];
            memcpy(key64 + 64 * u, rec.key[u - u0], 64 * sizeof(uint32_t));
            memcpy(dst + (size_t)u * 16u, blk[u - u0], 16);
        }
    }
    return DXB_S_OK;
}
