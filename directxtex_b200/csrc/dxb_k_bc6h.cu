// dxb_k_bc6h.cu — k_compress_bc6h: one HALF-WARP per 4x4 block (two blocks per warp), BC6H_UF16 / BC6H_SF16 (dxb_bc6h.cuh)
#include "dxb_launch.h"
#include "dxb_bc6h.cuh"

__global__ void __launch_bounds__(DXB_BC6H_WARPS * 32, DXB_BC6H_MINB) k_compress_bc6h(const dxb_job* __restrict__ jobs, dxb_job single, dxb_compress_params P)
{
    __shared__ dxb_px spx[DXB_BC6H_WARPS][32];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u, hl = lane & 15u;
    const uint32_t stride = gridDim.x * DXB_BC6H_WARPS;
    const bool bSigned = (P.dstFormat == DXB_FMT_BC6H_SF16);
    const uint32_t npairs = (P.totalUnits + 1u) >> 1;
    for (uint32_t pair = blockIdx.x * DXB_BC6H_WARPS + warp; pair < npairs; pair += stride)
    {
        // lanes 0-15 stage block 2*pair, lanes 16-31 block 2*pair+1; lane = pixel
        const uint32_t unit = 2u * pair + (lane >> 4);
        uint8_t* out = nullptr;
        dxb_px ip = dxb_make_px(0.0f, 0.0f, 0.0f, 0.0f);
        if (unit < P.totalUnits)
        {
            const dxb_job& j = dxb_find_job(jobs, P.njobs, single, unit);
            const uint32_t local = unit - j.firstUnit;
            const uint32_t by = local / j.nbx, bx = local - by * j.nbx;
            // partial-block replication with source map {0,0,0,1} (DirectXTexCompress.cpp:159-187)
            const uint32_t x0 = bx * 4, y0 = by * 4;
            const uint32_t pw = (j.width - x0 < 4u) ? (j.width - x0) : 4u;
            const uint32_t ph = (j.height - y0 < 4u) ? (j.height - y0) : 4u;
            const uint32_t s = hl & 3u, t = hl >> 2;
            const uint32_t sc = (s < pw) ? s : ((s == 3u && pw > 1u) ? 1u : 0u);
            const uint32_t tr = (t < ph) ? t : ((t == 3u && ph > 1u) ? 1u : 0u);
            dxb_px v = dxb_load_pixel(P.srcFormat, j.src + (size_t)(y0 + tr) * j.srcPitch, x0 + sc);
            v = dxb_convert_pixel(v, P.inF, P.outF, P.cflags);
            ip = dxb_make_px(dxb_bc6h_to_int(v.x, bSigned), dxb_bc6h_to_int(v.y, bSigned), dxb_bc6h_to_int(v.z, bSigned), 0.0f);
            out = j.dst + (size_t)by * j.dstPitch + (size_t)bx * 16u;
        }
        spx[warp][lane] = ip;
        __syncwarp();
        dxb_bc6h_encode_pair(spx[warp], bSigned, out, out);      // every lane passes its own half's pointer in both slots
        __syncwarp();
    }
}

void dxb_launch_bc6h(unsigned grid, cudaStream_t stream, const dxb_job* jobs, const dxb_job* hostJobs, const dxb_compress_params& P)
{
    k_compress_bc6h<<<grid, DXB_BC6H_WARPS * 32, 0, stream>>>(jobs, hostJobs[0], P);
}
int dxb_occupancy_bc6h()
{
    int b = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, k_compress_bc6h, DXB_BC6H_WARPS * 32, 0) != cudaSuccess) { (void)cudaGetLastError(); b = 1; }
    return b > 0 ? b : 1;
}
