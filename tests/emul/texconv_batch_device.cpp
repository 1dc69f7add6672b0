// tests/emul/texconv_batch_device.cpp — TEST INFRASTRUCTURE, never shipped: where dxb200_texconv_batch_device keeps each plane of a
// job's chunks (device_aliases, chunk_end, chunk_bytes and chunk_layout of dxb_plan.h) on the host, so that the CPU suite can check the
// placement and the scratch sizes without a device.  The job is planned by plan_texconv_job, the planner every batch job goes through.
#include <cstdint>
#include <cstddef>
#include <cstring>
#include <vector>

#include "dxb_portable.h"
#include "dxb_formats.h"
#include "dxb_plan.h"

// Plans `job`; on S_OK, out = { plane count, then { role, aliased, first copy, rest copy } of every plane, step count, then { kind,
// source role, destination role, cover } of every step, chunk count, then of every chunk when the items are cut at `budget` bytes
// { first item, end item, staged bytes (chunk_bytes of every plane), scratch bytes (of the planes not aliased), the bytes chunk_layout
// lays out in scratch, 1 when every aliased image keeps the caller's pixels, then each plane's bytes } }, at most cap words, and
// *nout = the words written.  Returns the planner's HRESULT.
extern "C" int32_t emul_device_plan(const dxb200_texconv_job* job, size_t budget, uint64_t* out, size_t cap, size_t* nout)
{
    *nout = 0;
    FromPlan fp;
    AlphaOpaquePlan ap;
    const int32_t hr = plan_texconv_job(*job, &fp, &ap);
    if (hr != DXB_S_OK) return hr;
    const ChunkPlan& ck = fp.chunk;
    // the caller's images of every role, and one result word per item
    uint32_t word = 0;
    std::vector<dxb200_image> roles[PLANE_ROLES];
    roles[(size_t)PlaneRole::Base].assign(job->base, job->base + job->items * ck.per);
    roles[(size_t)PlaneRole::Decompressed] = fp.decompressed;
    roles[(size_t)PlaneRole::Level0] = fp.level0;
    roles[(size_t)PlaneRole::Chain] = fp.chain.chain;
    roles[(size_t)PlaneRole::Dst].assign(job->dst, job->dst + job->items * job->levels);
    roles[(size_t)PlaneRole::Words].assign(job->items, dxb200_image{ 1, 1, DXB_FMT_UNKNOWN, sizeof(uint32_t), sizeof(uint32_t),
                                                                     reinterpret_cast<uint8_t*>(&word) });
    const dxb200_image* host[PLANE_ROLES];
    for (size_t r = 0; r < PLANE_ROLES; ++r) host[r] = roles[r].data();
    const std::vector<Plane> planes = chain_planes(ck, host, 0);
    const std::vector<bool> alias = device_aliases(ck);
    std::vector<uint64_t> w = { planes.size() };
    for (size_t p = 0; p < planes.size(); ++p)
        w.insert(w.end(), { (uint64_t)ck.planes[p].role, alias[p], (uint64_t)planes[p].first, (uint64_t)planes[p].rest });
    w.push_back(ck.steps.size());
    for (const ChunkStep& s : ck.steps) w.insert(w.end(), { (uint64_t)s.kind, (uint64_t)s.src, (uint64_t)s.dst, (uint64_t)s.cover });
    std::vector<uint64_t> chunks;
    size_t count = 0;
    uint8_t* const scratch = reinterpret_cast<uint8_t*>(uintptr_t(1) << 40);
    for (size_t i = 0, k; i < job->items; i = k, ++count)
    {
        k = chunk_end(planes.data(), planes.size(), i, job->items, budget);
        std::vector<dxb200_image> dev[PLANE_ROLES];
        chunk_layout(planes.data(), planes.size(), i, k, &alias, scratch, dev);
        size_t laid = 0;
        bool keeps = true;
        for (size_t p = 0; p < planes.size(); ++p)
            for (size_t m = 0; m < dev[p].size(); ++m)
            {
                if (alias[p]) keeps &= dev[p][m].pixels == planes[p].host[i * planes[p].per + m].pixels;
                else laid = std::max(laid, (size_t)(dev[p][m].pixels - scratch) + padded_bytes(dev[p][m]));
            }
        chunks.insert(chunks.end(), { i, k, chunk_bytes(planes.data(), planes.size(), i, k),
                                      chunk_bytes(planes.data(), planes.size(), i, k, &alias), laid, keeps });
        for (size_t p = 0; p < planes.size(); ++p) chunks.push_back(chunk_bytes(&planes[p], 1, i, k));
    }
    w.push_back(count);
    w.insert(w.end(), chunks.begin(), chunks.end());
    *nout = std::min(w.size(), cap);
    std::copy(w.begin(), w.begin() + *nout, out);
    return DXB_S_OK;
}
