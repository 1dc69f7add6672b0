// tests/emul/texconv_batch.cpp — TEST INFRASTRUCTURE, never shipped: the planner of dxb200_texconv_batch (plan_texconv_batch,
// dxb_plan.h) on the host, so that the CPU suite can hold a batch's HRESULTs, groups, each group's chunk plan and the split of its
// units over the devices against the single calls' planners without a device.  It builds on texconv_steps.cpp, whose entries (the
// three single-call planners and emul_chunk_plan) it exports too.
#include "texconv_steps.cpp"

// ---- dxb200_texconv_batch's plan (plan_texconv_batch) -----------------------------------------------------------------------------
static BatchPlan batch;

// results[i] = job i's HRESULT, group[i] = its group (UINT64_MAX for a job that failed its checks); returns the batch's HRESULT.
// emul_batch_chunk_plan(g) makes group g's chunk plan the one emul_chunk_plan reports.
extern "C" int32_t emul_texconv_batch(const dxb200_texconv_job* jobs, size_t njobs, int32_t* results, uint64_t* group)
{
    const int32_t hr = plan_texconv_batch(jobs, njobs, &batch);
    for (size_t i = 0; i < batch.hr.size(); ++i)
    {
        results[i] = batch.hr[i];
        group[i] = batch.group[i] == SIZE_MAX ? UINT64_MAX : batch.group[i];
    }
    return hr;
}

extern "C" void emul_batch_chunk_plan(size_t g)
{
    last = batch.fp[batch.groups[g][0]].chunk;
}

// out = the unit weights of the last batch (units = group by group, item by item), then cut[0 .. nd] of its split over `devices`
// (nd = min(devices, max(units, 1))); returns the words written, at most cap
extern "C" size_t emul_batch_units(size_t devices, uint64_t* out, size_t cap)
{
    std::vector<uint64_t> w(batch.weight.begin(), batch.weight.end());
    const std::vector<size_t> cut = shard_cuts(batch.weight.size(), devices, [](size_t i) { return batch.weight[i]; });
    w.insert(w.end(), cut.begin(), cut.end());
    const size_t n = std::min(w.size(), cap);
    std::copy(w.begin(), w.begin() + n, out);
    return n;
}
