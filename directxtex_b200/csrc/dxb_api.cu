// dxb_api.cu — the extern "C" boundary of libdxtex_b200.so (see include/dxtex_b200.h) and the host
// logic behind it: each call planned by dxb_plan.h (argument validation with the reference's HRESULTs,
// pitch rules, flags, job records), batching, staging of host images through device memory, kernel launches on sm_90a.
//
// Every host-pointer call stages through one routine, run_staged: whole items (a band and its output, a mip chain, a resize
// pair) are grouped into chunks that pipeline H2D -> kernels -> D2H over the NSLOT (stream, buffer) slots of a lane.  Band calls
// (compress, decompress, convert, premultiply) cut images into ~32 MiB bands and stage 48 MiB per chunk; chain and pair calls
// (generate_mipmaps, resize, mipmaps_compress) stage 80 MiB per chunk.  ScaleMipMapsAlphaForCoverage stages on its own: it
// downloads with a 2D copy into the caller's pitch.  Its search runs on the device for a whole batch (launch_coverage) with no
// host round trip; the per-item call synchronises once, at its end.
//
// Compiled with: nvcc -gencode arch=compute_90a,code=sm_90a -fmad=false (bit-exact fp32 contract
// of the BC1-5 / convert / mip kernels) -lineinfo.  There is no host implementation of any codec in
// this file: if CUDA is unavailable every compute entry point returns E_FAIL.
#include <cuda_runtime.h>
#include <atomic>
#include <mutex>
#include <condition_variable>
#include <memory>
#include <thread>
#include <functional>
#include <unistd.h>
#include <sys/syscall.h>
#include <vector>
#include <map>
#include <string>
#include <cstring>
#include <cstdio>
#include <cmath>
#include <algorithm>

#include "../../include/dxtex_b200.h"
#include "dxb_formats.h"
#include "dxb_launch.h"
#include "dxb_plan.h"

namespace {

constexpr int NSLOT = 3;        // (stream, device buffer) slots of one lane: H2D / kernel / D2H of consecutive chunks overlap
constexpr int NLANE = 2;        // host-staged calls that can be in flight on one device at the same time (each owns a lane)
constexpr size_t BAND_BYTES = size_t(32) << 20;     // source + destination bytes of one band of a band call
constexpr size_t BAND_CHUNK = size_t(48) << 20;     // slot buffer bytes of one chunk of a band call
// slot buffer bytes of one chunk of a chain or pair call; 80 MiB keeps eleven 1024^2 RGBA8 -> BC3 chains of mipmaps_compress in a
// chunk: with 64 MiB (nine) its end-to-end time was about 4 % longer (H100 80GB HBM3 at 400 W, DESIGN.md §4)
constexpr size_t ITEM_CHUNK = size_t(80) << 20;

std::mutex g_mu;                // guards the device table only; calls on different lanes / devices run concurrently
std::atomic<uint64_t> g_launches{0};
std::mutex g_count_mu;                                  // guards g_kernel_launches
std::map<std::string, uint64_t> g_kernel_launches;      // launches per kernel name (dxb200_kernel_launch_count)
std::atomic<int32_t> g_mip_kernels{0};                  // DXB200_OPT_MIP_KERNELS
thread_local std::string t_lastError;

struct Lane
{
    cudaStream_t streams[NSLOT] = { nullptr, nullptr, nullptr };
    void* buf[NSLOT] = { nullptr, nullptr, nullptr }; size_t cap[NSLOT] = { 0, 0, 0 };
    bool busy = false;
};

// one per CUDA device the library was initialised on (dxb200_init / dxb200_init_devices; SURVEY.md 8(b), 8(e))
struct Device
{
    int ordinal = 0;
    int numSMs = 132;
    int numaNode = -1;
    int gridBC15 = 0, gridBC7 = 0, gridBC6H = 0, gridRow = 0;
    std::mutex mu; std::condition_variable cv;
    Lane lanes[NLANE];
};
std::vector<std::unique_ptr<Device>> g_devs;

// the device (and, for host-staged calls, the lane) the calling thread is working on
struct View { Device* dev = nullptr; Lane* lane = nullptr; };
thread_local View t_v;

int32_t cuda_hr(cudaError_t e, const char* what)
{
    if (e == cudaSuccess) return DXB_S_OK;
    char buf[256];
    snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(e));
    t_lastError = buf;
    (void)cudaGetLastError();
    return (e == cudaErrorMemoryAllocation) ? DXB_E_OUTOFMEMORY : DXB_E_FAIL;
}
#define DXB_CUDA(call) do { const int32_t hr__ = cuda_hr((call), #call); if (hr__ != DXB_S_OK) return hr__; } while (0)

// NUMA node of a device's PCI function (sysfs), -1 if unknown
int device_numa_node(int ordinal)
{
    char bus[32] = { 0 };
    if (cudaDeviceGetPCIBusId(bus, sizeof(bus), ordinal) != cudaSuccess) { (void)cudaGetLastError(); return -1; }
    for (char* c = bus; *c; ++c) *c = (char)tolower(*c);
    char path[96];
    snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE* f = fopen(path, "r");
    if (!f) return -1;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    return node;
}

// find or create the Device record of CUDA device `ordinal`; g_mu held.  Leaves `ordinal` current.
int32_t init_device_locked(int ordinal, Device** out)
{
    for (auto& d : g_devs) if (d->ordinal == ordinal) { if (out) *out = d.get(); return DXB_S_OK; }
    int n = 0;
    DXB_CUDA(cudaGetDeviceCount(&n));
    if (n <= 0) { t_lastError = "no CUDA device"; return DXB_E_FAIL; }
    if (ordinal < 0 || ordinal >= n) { t_lastError = "device ordinal out of range"; return DXB_E_INVALIDARG; }
    DXB_CUDA(cudaSetDevice(ordinal));
    std::unique_ptr<Device> d(new Device);
    d->ordinal = ordinal;
    cudaDeviceProp prop;
    DXB_CUDA(cudaGetDeviceProperties(&prop, ordinal));
    d->numSMs = prop.multiProcessorCount;
    d->numaNode = device_numa_node(ordinal);
    for (int l = 0; l < NLANE; ++l)
        for (int i = 0; i < NSLOT; ++i) DXB_CUDA(cudaStreamCreateWithFlags(&d->lanes[l].streams[i], cudaStreamNonBlocking));
    {
        // job arrays use stream-ordered allocation: keep freed blocks in the pool across synchronisation points
        // (the default release threshold of 0 returns them to the OS, which makes the next call's cudaMallocAsync slow)
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, ordinal) == cudaSuccess)
        {
            uint64_t keep = ~uint64_t(0);
            (void)cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
        }
        (void)cudaGetLastError();
    }
    d->gridBC15 = d->numSMs * dxb_occupancy_bc15();
    d->gridBC7 = d->numSMs * dxb_occupancy_bc7();
    d->gridBC6H = d->numSMs * dxb_occupancy_bc6h();
    d->gridRow = d->numSMs * 8;
    if (out) *out = d.get();
    g_devs.push_back(std::move(d));
    return DXB_S_OK;
}

// the devices host-pointer calls are sharded over; a process that never called dxb200_init* gets its current CUDA device
int32_t device_list(std::vector<Device*>* out)
{
    std::lock_guard<std::mutex> lk(g_mu);
    if (g_devs.empty())
    {
        int cur = 0;
        if (cudaGetDevice(&cur) != cudaSuccess) { (void)cudaGetLastError(); cur = 0; }
        const int32_t hr = init_device_locked(cur, nullptr);
        if (hr != DXB_S_OK) return hr;
    }
    out->clear();
    for (auto& d : g_devs) out->push_back(d.get());
    return DXB_S_OK;
}

// host-pointer call on device `d`: waits for one of its lanes, makes device and lane current for the calling thread
struct HostScope
{
    Device* d = nullptr; Lane* l = nullptr; int prev = -1; View saved;
    int32_t enter(Device* dev)
    {
        saved = t_v;
        if (cudaGetDevice(&prev) != cudaSuccess) { (void)cudaGetLastError(); prev = -1; }
        DXB_CUDA(cudaSetDevice(dev->ordinal));
        std::unique_lock<std::mutex> lk(dev->mu);
        for (;;)
        {
            for (int i = 0; i < NLANE && !l; ++i) if (!dev->lanes[i].busy) l = &dev->lanes[i];
            if (l) break;
            dev->cv.wait(lk);
        }
        l->busy = true; d = dev;
        t_v.dev = dev; t_v.lane = l;
        return DXB_S_OK;
    }
    ~HostScope()
    {
        if (l) { { std::lock_guard<std::mutex> lk(d->mu); l->busy = false; } d->cv.notify_one(); }
        t_v = saved;
        if (prev >= 0 && d && prev != d->ordinal) (void)cudaSetDevice(prev);
    }
};

// _device call: the work goes to the device that owns the caller's pointers, on the caller's stream
struct DevScope
{
    int prev = -1, ord = -1; View saved;
    int32_t enter(const void* p)
    {
        saved = t_v;
        if (cudaGetDevice(&prev) != cudaSuccess) { (void)cudaGetLastError(); prev = 0; }
        ord = prev;
        cudaPointerAttributes a;
        if (p && cudaPointerGetAttributes(&a, p) == cudaSuccess && (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged)) ord = a.device;
        (void)cudaGetLastError();
        Device* dev = nullptr;
        {
            std::lock_guard<std::mutex> lk(g_mu);
            const int32_t hr = init_device_locked(ord, &dev);           // leaves `ord` current when it creates the record
            if (hr != DXB_S_OK) return hr;
        }
        DXB_CUDA(cudaSetDevice(ord));
        t_v.dev = dev; t_v.lane = nullptr;
        return DXB_S_OK;
    }
    ~DevScope()
    {
        t_v = saved;
        if (prev >= 0 && ord >= 0 && prev != ord) (void)cudaSetDevice(prev);
    }
};

// Runs fn(lo, hi) over [0, n) split into contiguous ranges of about equal weight, one range per initialised device, each on
// its own host thread (the caller's thread takes the first range).  One device or one unit: runs inline.
template <typename WeightFn, typename Fn>
int32_t run_sharded(size_t n, WeightFn weight, Fn fn)
{
    std::vector<Device*> devs;
    int32_t hr = device_list(&devs);
    if (hr != DXB_S_OK) return hr;
    const size_t nd = std::min(devs.size(), std::max<size_t>(n, 1));
    if (nd <= 1)
    {
        HostScope sc;
        hr = sc.enter(devs[0]);
        return hr != DXB_S_OK ? hr : fn(size_t(0), n);
    }
    const std::vector<size_t> cut = shard_cuts(n, nd, weight);
    std::vector<int32_t> hrs(nd, DXB_S_OK);
    std::vector<std::string> errs(nd);
    auto work = [&](size_t d)
    {
        if (cut[d] == cut[d + 1]) return;
        HostScope sc;
        hrs[d] = sc.enter(devs[d]);
        if (hrs[d] == DXB_S_OK) hrs[d] = fn(cut[d], cut[d + 1]);
        if (hrs[d] != DXB_S_OK) errs[d] = t_lastError;
    };
    std::vector<std::thread> th;
    for (size_t d = 1; d < nd; ++d) th.emplace_back(work, d);
    work(0);
    for (auto& t : th) t.join();
    for (size_t d = 0; d < nd; ++d) if (hrs[d] != DXB_S_OK) { t_lastError = errs[d]; return hrs[d]; }
    return DXB_S_OK;
}

// progress reporting / cancellation of the host-staged calls (the reference's statusCallback, DirectXTexCompress.cpp:115-121, 785-837)
struct Progress
{
    dxb200_status_fn fn = nullptr; void* user = nullptr;
    size_t total = 0; std::atomic<size_t> done{0}; std::atomic<bool> aborted{false};
    std::mutex mu;
    // false = the caller asked to stop
    bool report(size_t add)
    {
        if (!fn) return true;
        if (aborted.load()) return false;
        const size_t d = done.fetch_add(add);                      // units finished before this chunk, as the reference reports (:115-121)
        std::lock_guard<std::mutex> lk(mu);
        if (!fn(std::min(d, total), total, user)) aborted.store(true);
        return !aborted.load();
    }
};

int32_t ensure_buffer(void** p, size_t* cap, size_t need)
{
    if (*cap >= need) return DXB_S_OK;
    if (*p) { cudaFree(*p); *p = nullptr; *cap = 0; }
    const size_t want = (need + (size_t(1) << 20)) & ~((size_t(1) << 20) - 1);
    DXB_CUDA(cudaMalloc(p, want));
    *cap = want;
    return DXB_S_OK;
}

// ---- generic launch helper ------------------------------------------------------------------
template <typename J>
struct DeviceJobs
{
    J* d = nullptr; cudaStream_t s = nullptr;
    int32_t upload(const std::vector<J>& jobs, cudaStream_t stream)
    {
        s = stream;
        if (jobs.size() <= 1) return DXB_S_OK;
        DXB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&d), jobs.size() * sizeof(J), stream));
        DXB_CUDA(cudaMemcpyAsync(d, jobs.data(), jobs.size() * sizeof(J), cudaMemcpyHostToDevice, stream));
        return DXB_S_OK;
    }
    void release() { if (d) { cudaFreeAsync(d, s); d = nullptr; } }
};

// The job table of one launch: one dxb_job per (src[i], dst[i]) whose work units are 4x4 blocks (`blocks`) or pixels, on the
// host and, for more than one job, on the device; the device copy is released on the launch's stream with the table.
struct JobTable
{
    std::vector<dxb_job> host; DeviceJobs<dxb_job> dev; uint32_t total = 0;
    ~JobTable() { dev.release(); }
    int32_t build(const dxb200_image* src, const dxb200_image* dst, size_t n, bool blocks, cudaStream_t stream)
    {
        host.resize(n);
        uint64_t units = 0;
        for (size_t i = 0; i < n; ++i)
        {
            dxb_job& j = host[i];
            j.src = src[i].pixels; j.dst = dst[i].pixels; j.srcPitch = src[i].rowPitch; j.dstPitch = dst[i].rowPitch;
            j.width = (uint32_t)src[i].width; j.height = (uint32_t)src[i].height;
            j.nbx = blocks ? (j.width + 3) / 4 : 0; j.nby = blocks ? (j.height + 3) / 4 : 0;
            j.firstUnit = (uint32_t)units; j.pad = 0;
            units += blocks ? (uint64_t)j.nbx * j.nby : (uint64_t)j.width * j.height;
            if (units > 0x7FFFFFFFull) return DXB_E_INVALIDARG;                // same 2^31-unit limit as CompressBC_Parallel (:258)
        }
        total = (uint32_t)units;
        return dev.upload(host, stream);
    }
};

// CTAs for `units` work units at `perCta` units per CTA: at least one, at most `cap`
uint32_t grid_for(uint32_t units, uint32_t perCta, uint32_t cap)
{
    return std::max(1u, std::min((uint32_t)(((uint64_t)units + perCta - 1) / perCta), cap));
}

int32_t check_launch(const char* name)
{
    g_launches.fetch_add(1, std::memory_order_relaxed);
    {
        std::lock_guard<std::mutex> lk(g_count_mu);
        ++g_kernel_launches[name];
    }
    return cuda_hr(cudaGetLastError(), name);
}

// ---- Compress ---------------------------------------------------------------------------------
// enqueue the kernel for images whose pixels already live on the device
int32_t launch_compress(const CompressPlan& plan, const dxb200_image* src, const dxb200_image* dst, size_t n, cudaStream_t stream)
{
    JobTable jt;
    const int32_t hr = jt.build(src, dst, n, true, stream);
    if (hr != DXB_S_OK) return hr;
    dxb_compress_params P = plan.P;
    P.totalUnits = jt.total; P.njobs = (uint32_t)n;
    const Device& d = *t_v.dev;
    if (plan.bc6h)
    {
        return check_launch(dxb_launch_bc6h(grid_for(jt.total, 2 * DXB_BC6H_WARPS, (uint32_t)d.gridBC6H * 4u), stream, jt.dev.d, jt.host.data(), P));
    }
    if (plan.bc7)
    {
        // RGBA32F sources of full blocks: persistent kernel fed by TMA tile loads; everything else: the direct kernel with one CTA
        // per 2 * DXB_BC7_WARPS blocks (no grid-stride cap): block costs differ (alpha blocks run the separate-alpha tasks), so the
        // hardware CTA scheduler balances better than a static stride
        return check_launch(dxb_launch_bc7(grid_for(jt.total, 2 * DXB_BC7_WARPS, UINT32_MAX), (unsigned)d.gridBC7, stream, jt.dev.d, jt.host.data(), P));
    }
    return check_launch(dxb_launch_bc15(grid_for(jt.total, 128, (uint32_t)d.gridBC15 * 4u), stream, jt.dev.d, jt.host.data(), P));
}

// ---- host staging -------------------------------------------------------------------------------------
// fn(dev, count, stream) of a staged segment: enqueues the kernels of one chunk; dev[p] is plane p's images of the chunk's `count`
// items, with device pointers
using StageFn = std::function<int32_t(const std::vector<dxb200_image>*, size_t, cudaStream_t)>;

// items [0, n) of `nplanes` planes, staged with their own launch function
struct Segment { const Plane* planes; size_t nplanes; size_t n; StageFn fn; };

// Stages the items of every segment, in order, through the calling thread's lane.  Whole items of one segment are grouped into
// chunks of at most `budget` bytes of device memory (chunk_end; a chunk never spans two segments), and chunk c of the call goes
// through slot c % NSLOT, so the H2D copies, kernels and D2H copies of consecutive chunks overlap, from one segment to the next too
// (fully when the caller's memory is pinned, see dxb200_host_alloc).  In the slot's buffer the chunk's images lie as chunk_layout
// lays them out.  prog (optional) is told before each chunk's upload the units[] of the items the chunk completes (units counts the
// items of all segments in order), and stops the call between chunks (E_ABORT).  Every slot is synchronised once, before returning;
// the first error wins.
int32_t run_segments(const Segment* segs, size_t nsegs, size_t budget, Progress* prog = nullptr, const size_t* units = nullptr)
{
    Lane& L = *t_v.lane;
    int slot = 0;
    int32_t hr = DXB_S_OK;
    for (size_t sg = 0; sg < nsegs && hr == DXB_S_OK; units += units ? segs[sg].n : 0, ++sg)
    {
        const Plane* planes = segs[sg].planes;
        const size_t nplanes = segs[sg].nplanes, n = segs[sg].n;
        std::vector<std::vector<dxb200_image>> dev(nplanes);
        size_t i = 0;
        while (i < n && hr == DXB_S_OK)
        {
            const size_t k = chunk_end(planes, nplanes, i, n, budget);
            cudaStream_t st = L.streams[slot];
            hr = cuda_hr(cudaStreamSynchronize(st), "slot sync"); if (hr) break;
            if (prog)
            {
                size_t add = 0;
                for (size_t m = i; m < k; ++m) add += units[m];
                if (!prog->report(add)) { hr = DXB_E_ABORT; break; }
            }
            hr = ensure_buffer(&L.buf[slot], &L.cap[slot], chunk_bytes(planes, nplanes, i, k)); if (hr) break;
            chunk_layout(planes, nplanes, i, k, nullptr, static_cast<uint8_t*>(L.buf[slot]), dev.data());
            for (size_t p = 0; p < nplanes && hr == DXB_S_OK; ++p)
            {
                const Plane& pl = planes[p];
                const dxb200_image* host = pl.host + i * pl.per;
                for (size_t m = 0; m < dev[p].size() && hr == DXB_S_OK; ++m)
                    if ((m % pl.per ? pl.rest : pl.first) == Copy::Up)
                        hr = cuda_hr(cudaMemcpyAsync(dev[p][m].pixels, host[m].pixels, host[m].slicePitch, cudaMemcpyHostToDevice, st), "H2D");
            }
            if (hr) break;
            hr = segs[sg].fn(dev.data(), k - i, st); if (hr) break;
            for (size_t p = 0; p < nplanes && hr == DXB_S_OK; ++p)
            {
                const Plane& pl = planes[p];
                const dxb200_image* host = pl.host + i * pl.per;
                for (size_t m = 0; m < dev[p].size() && hr == DXB_S_OK; ++m)
                    if ((m % pl.per ? pl.rest : pl.first) == Copy::Down)
                        hr = cuda_hr(cudaMemcpyAsync(host[m].pixels, dev[p][m].pixels, host[m].slicePitch, cudaMemcpyDeviceToHost, st), "D2H");
            }
            i = k; slot = (slot + 1) % NSLOT;
        }
    }
    for (int s = 0; s < NSLOT; ++s)
    {
        const int32_t h2 = cuda_hr(cudaStreamSynchronize(L.streams[s]), "final sync");
        if (hr == DXB_S_OK) hr = h2;
    }
    return hr;
}

// run_segments of one segment
int32_t run_staged(const Plane* planes, size_t nplanes, size_t n, size_t budget, StageFn fn, Progress* prog = nullptr, const size_t* units = nullptr)
{
    const Segment seg = { planes, nplanes, n, std::move(fn) };
    return run_segments(&seg, 1, budget, prog, units);
}

// Band calls cut host images into BANDS of whole work rows (4 pixel rows per block row on the BC side) of about BAND_BYTES.
// Band boundaries fall on block rows, so the result is identical to processing the whole image at once.
struct BandSplit { std::vector<dxb200_image> src, dst; std::vector<size_t> units; };      // units = progress units a band completes

// srcRows/dstRows: pixel (or block) rows of the source/destination image consumed/produced per work row
void split_bands(const dxb200_image* src, const dxb200_image* dst, size_t n, size_t srcRows, size_t dstRows, bool srcIsBC, bool dstIsBC, BandSplit& out)
{
    for (size_t m = 0; m < n; ++m)
    {
        const size_t srcTotalRows = srcIsBC ? (src[m].height + 3) / 4 : src[m].height;
        const size_t dstTotalRows = dstIsBC ? (dst[m].height + 3) / 4 : dst[m].height;
        const size_t units = std::max<size_t>(1, (srcTotalRows + srcRows - 1) / srcRows);
        const size_t bytesPerUnit = src[m].rowPitch * srcRows + dst[m].rowPitch * dstRows;
        const size_t per = std::max<size_t>(1, BAND_BYTES / std::max<size_t>(bytesPerUnit, 1));
        for (size_t u0 = 0; u0 < units; u0 += per)
        {
            const size_t u1 = std::min(units, u0 + per);
            dxb200_image s = src[m], d = dst[m];
            const size_t sr0 = u0 * srcRows, sr1 = std::min(srcTotalRows, u1 * srcRows);
            const size_t dr0 = u0 * dstRows, dr1 = std::min(dstTotalRows, u1 * dstRows);
            s.pixels = src[m].pixels + sr0 * src[m].rowPitch; s.slicePitch = (sr1 - sr0) * src[m].rowPitch;
            d.pixels = dst[m].pixels + dr0 * dst[m].rowPitch; d.slicePitch = (dr1 - dr0) * dst[m].rowPitch;
            // pixel heights of the band (the uncompressed side counts pixel rows; the BC side the same pixel rows)
            const size_t pixRows = srcIsBC ? std::min(src[m].height, sr1 * 4) - sr0 * 4 : (sr1 - sr0);
            s.height = pixRows; d.height = pixRows;
            out.src.push_back(s); out.dst.push_back(d);
            // progress as the reference reports it: pixel rows of a single image, images of an array (:115-121, 785-837)
            out.units.push_back(n == 1 ? pixRows : (u1 == units ? 1 : 0));
        }
    }
}

// A band call once its arguments are validated: bands (split_bands) sharded over the devices by bytes and staged BAND_CHUNK
// bytes per chunk; launch(src, dst, count, stream) enqueues the kernel on device images.  status (optional) is called as the
// reference calls it, and with (total, total) at the end.
template <typename LaunchFn>
int32_t run_bands(const dxb200_image* src, const dxb200_image* dst, size_t n, size_t srcRows, size_t dstRows, bool srcIsBC, bool dstIsBC,
                  dxb200_status_fn status, void* user, LaunchFn launch)
{
    BandSplit bands;
    split_bands(src, dst, n, srcRows, dstRows, srcIsBC, dstIsBC, bands);
    Progress prog; prog.fn = status; prog.user = user;
    for (size_t u : bands.units) prog.total += u;
    int32_t hr = run_sharded(bands.src.size(), [&](size_t i) { return bands.src[i].slicePitch + bands.dst[i].slicePitch; },
        [&](size_t lo, size_t hi)
        {
            const Plane planes[2] = { { bands.src.data() + lo, 1, Copy::Up, Copy::Up }, { bands.dst.data() + lo, 1, Copy::Down, Copy::Down } };
            return run_staged(planes, 2, hi - lo, BAND_CHUNK,
                [&](const std::vector<dxb200_image>* dev, size_t cnt, cudaStream_t st) { return launch(dev[0].data(), dev[1].data(), cnt, st); },
                status ? &prog : nullptr, bands.units.data() + lo);
        });
    if (hr == DXB_S_OK && status && !status(prog.total, prog.total, user)) hr = DXB_E_ABORT;
    return hr;
}

// ---- Convert ----------------------------------------------------------------------------------
int32_t launch_convert(dxb_convert_params P, const dxb200_image* src, const dxb200_image* dst, size_t n, cudaStream_t stream)
{
    JobTable jt;
    int32_t hr = jt.build(src, dst, n, false, stream);
    if (hr != DXB_S_OK) return hr;
    P.totalUnits = jt.total; P.njobs = (uint32_t)n;
    if (P.flags & DXB_FILTER_DITHER_DIFFUSION)
    {
        // two error rows of (width + 2) pixels per image
        uint32_t maxw = 0;
        for (const dxb_job& j : jt.host) maxw = std::max(maxw, j.width);
        const uint32_t errStride = 2u * (maxw + 2u);
        void* dErr = nullptr;
        hr = cuda_hr(cudaMallocAsync(&dErr, (size_t)errStride * n * sizeof(float) * 4, stream), "cudaMallocAsync(errors)");
        if (hr != DXB_S_OK) return hr;
        hr = check_launch(dxb_launch_convert_diffuse(stream, (n > 1) ? jt.dev.d : nullptr, jt.host.data(), P, dErr, errStride));
        cudaFreeAsync(dErr, stream);
        return hr;
    }
    return check_launch(dxb_launch_convert(grid_for(jt.total, 256, (uint32_t)t_v.dev->gridRow * 8u), stream, jt.dev.d, jt.host.data(), P));
}

// ---- PremultiplyAlpha ---------------------------------------------------------------------------
int32_t launch_pmalpha(dxb_convert_params P, const dxb200_image* src, const dxb200_image* dst, size_t n, cudaStream_t stream)
{
    JobTable jt;
    const int32_t hr = jt.build(src, dst, n, false, stream);
    if (hr != DXB_S_OK) return hr;
    P.totalUnits = jt.total; P.njobs = (uint32_t)n;
    return check_launch(dxb_launch_pmalpha(grid_for(jt.total, 256, (uint32_t)t_v.dev->gridRow * 8u), stream, jt.dev.d, jt.host.data(), P));
}

// ---- texconv's channel steps (dxb_channel_steps.h) ------------------------------------------------------------------------
int32_t launch_channel_steps(dxb_convert_params P, const dxb200_image* src, const dxb200_image* dst, size_t n, cudaStream_t stream)
{
    JobTable jt;
    const int32_t hr = jt.build(src, dst, n, false, stream);
    if (hr != DXB_S_OK) return hr;
    P.totalUnits = jt.total; P.njobs = (uint32_t)n;
    return check_launch(dxb_launch_channel_steps(grid_for(jt.total, 256, (uint32_t)t_v.dev->gridRow * 8u), stream, jt.dev.d, jt.host.data(), P));
}

// ---- GenerateMipMaps ----------------------------------------------------------------------------
// chain[] holds DEVICE pointers; level 0 of each item is populated
int32_t launch_mips(const dxb200_image* chain, size_t items, size_t levels, uint32_t filter, uint32_t mode, cudaStream_t stream)
{
    const MipPlan mp = build_mip_plan(chain, items, levels, filter, mode);
    const std::vector<dxb_mip_job>& all = mp.jobs;
    const std::vector<TriLists>& tri = mp.tri;
    // the records of every level and then TRIANGLE's gather lists go up with ONE copy (a per-level upload left the GPU idle
    // between the small launches of the tail of the chain)
    size_t bytes = all.size() * sizeof(dxb_mip_job);
    for (const TriLists& t : tri) bytes += (t.off.size() + t.src.size()) * sizeof(uint32_t) + t.w.size() * sizeof(float);
    uint8_t* dev = nullptr;
    std::vector<dxb_tri_axis> axes(tri.size());
    if (all.size() > 1 || !tri.empty())
    {
        DXB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&dev), bytes, stream));
        std::vector<uint8_t> host(bytes);
        size_t at = 0;
        auto put = [&](const void* p, size_t n) { if (n) memcpy(host.data() + at, p, n); at += n; return dev + at - n; };
        put(all.data(), all.size() * sizeof(dxb_mip_job));
        for (size_t i = 0; i < tri.size(); ++i)
        {
            axes[i].off = reinterpret_cast<const uint32_t*>(put(tri[i].off.data(), tri[i].off.size() * sizeof(uint32_t)));
            axes[i].src = reinterpret_cast<const uint32_t*>(put(tri[i].src.data(), tri[i].src.size() * sizeof(uint32_t)));
            axes[i].w = reinterpret_cast<const float*>(put(tri[i].w.data(), tri[i].w.size() * sizeof(float)));
        }
        DXB_CUDA(cudaMemcpyAsync(dev, host.data(), bytes, cudaMemcpyHostToDevice, stream));
    }
    const int32_t hr = dxb_launch_mip_chain(stream, reinterpret_cast<const dxb_mip_job*>(dev), all.data(), (uint32_t)items, (uint32_t)levels, mp.P,
                                            tri.empty() ? nullptr : axes.data(), (unsigned)t_v.dev->gridRow * 8u, g_mip_kernels.load() == 1,
                                            check_launch);
    if (dev) cudaFreeAsync(dev, stream);
    return hr;
}

// ---- Decompress (DirectXTexCompress.cpp:852-979; DecompressBC :425-535) ---------------------------------
int32_t launch_decompress(dxb_compress_params P, const dxb200_image* src, const dxb200_image* dst, size_t n, cudaStream_t stream)
{
    JobTable jt;
    const int32_t hr = jt.build(src, dst, n, true, stream);
    if (hr != DXB_S_OK) return hr;
    P.totalUnits = jt.total; P.njobs = (uint32_t)n;
    return check_launch(dxb_launch_decompress(grid_for(jt.total, 128, (uint32_t)t_v.dev->gridBC15 * 8u), stream, jt.dev.d, jt.host.data(), P));
}

// ---- Resize: a two-"level" chain per item whose second level has an arbitrary size ------------------------------------
int32_t launch_resize(const dxb200_image* src, const dxb200_image* dst, size_t n, uint32_t filter, uint32_t mode, cudaStream_t stream)
{
    std::vector<dxb200_image> pairs(2 * n);
    for (size_t i = 0; i < n; ++i) { pairs[2 * i] = src[i]; pairs[2 * i + 1] = dst[i]; }
    return launch_mips(pairs.data(), n, 2, filter, mode, stream);
}

// ---- ScaleMipMapsAlphaForCoverage -------------------------------------------------------------------------------------
// chains[it * levels + l] (DEVICE pointers) -> out[...]: levels >= 1 of every item scaled so that their alpha-test coverage at `ref`
// matches level 0's; level 0 is not written.  Always DXB_COVERAGE_STEPS k_alpha_coverage launches and one k_scale_alpha, with
// no host round trip in between, whatever the item and level counts.  The job table and the counts are allocated on `stream`.
int32_t launch_coverage(const dxb200_image* chains, const dxb200_image* out, size_t items, size_t levels, float ref, cudaStream_t stream)
{
    CoveragePlan cp;
    int32_t hr = plan_coverage_jobs(chains, out, items, levels, ref, &cp);
    if (hr != DXB_S_OK) return hr;
    const size_t countBytes = cp.jobs.size() * DXB_COVERAGE_STEPS * sizeof(unsigned long long);
    uint8_t* dev = nullptr;
    DXB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&dev), countBytes + cp.jobs.size() * sizeof(dxb_coverage_job), stream));
    unsigned long long* counts = reinterpret_cast<unsigned long long*>(dev);
    const dxb_coverage_job* jobs = reinterpret_cast<const dxb_coverage_job*>(dev + countBytes);
    hr = cuda_hr(cudaMemsetAsync(counts, 0, countBytes, stream), "cudaMemsetAsync(coverage counts)");
    if (hr == DXB_S_OK)
        hr = cuda_hr(cudaMemcpyAsync(dev + countBytes, cp.jobs.data(), cp.jobs.size() * sizeof(dxb_coverage_job), cudaMemcpyHostToDevice, stream), "H2D");
    const uint32_t cap = (uint32_t)t_v.dev->gridRow * 8u;
    for (uint32_t step = 0; step < DXB_COVERAGE_STEPS && hr == DXB_S_OK; ++step)
        hr = check_launch(dxb_launch_alpha_coverage(grid_for(cp.P.totalCells - (step ? cp.P.baseCells : 0u), 256, cap), stream, jobs, cp.P, counts, step));
    if (hr == DXB_S_OK) hr = check_launch(dxb_launch_scale_alpha(grid_for(cp.P.scaledPixels, 256, cap), stream, jobs, cp.P, counts));
    cudaFreeAsync(dev, stream);
    return hr;
}

// ScaleMipMapsAlphaForCoverage of one item (DEVICE pointers): level 0 copied (:3511-3530), the others scaled
int32_t scale_alpha_for_coverage_device(const dxb200_image* src, size_t n, float ref, const dxb200_image* dst, cudaStream_t st)
{
    DXB_CUDA(cudaMemcpy2DAsync(dst[0].pixels, dst[0].rowPitch, src[0].pixels, src[0].rowPitch, std::min(src[0].rowPitch, dst[0].rowPitch),
                               src[0].slicePitch / std::max<size_t>(src[0].rowPitch, 1), cudaMemcpyDeviceToDevice, st));
    return launch_coverage(src, dst, 1, n, ref, st);
}

// ---- IsAlphaAllOpaque (DirectXTexImage.cpp:800-852; IsAlphaAllOpaqueBC, DirectXTexCompress.cpp:539-621) -------------------------
// src (DEVICE pointers) scanned into words[i] (DEVICE, one 32-bit word per job, several jobs may share one; zero before the launch):
// 1 when a texel of src[i] is not opaque, untouched otherwise.  One launch of the generic k_decompress (BC) or k_convert.
int32_t launch_alpha_opaque(const AlphaOpaquePlan& ap, const dxb200_image* src, const dxb200_image* words, size_t n, cudaStream_t stream)
{
    JobTable jt;
    const int32_t hr = jt.build(src, words, n, ap.blocks, stream);
    if (hr != DXB_S_OK) return hr;
    const Device& d = *t_v.dev;
    if (ap.blocks)
        return check_launch(dxb_launch_alpha_opaque_blocks(grid_for(jt.total, 128, (uint32_t)d.gridBC15 * 8u), stream, jt.dev.d, jt.host.data(),
                                                          alpha_opaque_block_params(ap, jt.total, (uint32_t)n)));
    return check_launch(dxb_launch_alpha_opaque_pixels(grid_for(jt.total, 256, (uint32_t)d.gridRow * 8u), stream, jt.dev.d, jt.host.data(),
                                                      alpha_opaque_pixel_params(ap, jt.total, (uint32_t)n)));
}

// the result words of a staged plane: one per item, 256 bytes apart in the chunk's buffer with nothing in between, so one memset
// clears them all
int32_t clear_words(const std::vector<dxb200_image>& words, cudaStream_t stream)
{
    const size_t span = (size_t)(words.back().pixels - words.front().pixels) + sizeof(uint32_t);
    return cuda_hr(cudaMemsetAsync(words.front().pixels, 0, span, stream), "cudaMemsetAsync(alpha words)");
}

// The host side of a scan's staged result plane: one 32-bit word per item, in pinned memory.  A download into pageable memory
// returns only when the copy is done, i.e. when the chunk's kernels are, so it would hold back the uploads of the next chunks
// (64 x 1024^2 BC3 -> BC7 chains through mipmaps_compress_from_ex on an H100: 31.7 ms with pageable words, 28.7 ms pinned).
struct ResultWords
{
    uint32_t* w = nullptr; size_t n = 0;
    ~ResultWords() { if (w) cudaFreeHost(w); }
    int32_t alloc(size_t count)
    {
        DXB_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&w), std::max<size_t>(count, 1) * sizeof(uint32_t), cudaHostAllocPortable));
        n = count;
        memset(w, 0, n * sizeof(uint32_t));
        return DXB_S_OK;
    }
    // the plane's host images: word i as a 1 x 1 image of 4 bytes
    std::vector<dxb200_image> images() const
    {
        std::vector<dxb200_image> out(n);
        for (size_t i = 0; i < n; ++i) out[i] = { 1, 1, DXB_FMT_UNKNOWN, sizeof(uint32_t), sizeof(uint32_t), reinterpret_cast<uint8_t*>(w + i) };
        return out;
    }
    bool all_zero() const { return std::all_of(w, w + n, [](uint32_t v) { return v == 0; }); }
};

// The launches of one chunk of `cnt` items of fp.chunk: dev[p] = plane p's device images
int32_t run_chunk(const FromPlan& fp, const AlphaOpaquePlan& scan, size_t levels, const std::vector<dxb200_image>* dev, size_t cnt, cudaStream_t st)
{
    const ChainPlan& cp = fp.chain;
    const ChunkPlan& ck = fp.chunk;
    size_t at[PLANE_ROLES] = {};                                // the plane of each staged role
    for (size_t p = 0; p < ck.planes.size(); ++p) at[(size_t)ck.planes[p].role] = p;
    const size_t m = cnt * ck.per, all = cnt * levels;
    std::vector<dxb200_image> level(m);
    // the images of a plane a step covers; the Front of a plane of whole chains is gathered into `level`
    const auto images = [&](PlaneRole r, StepCover c) -> const dxb200_image*
    {
        const std::vector<dxb200_image>& d = dev[at[(size_t)r]];
        if (c != StepCover::Front || ck.planes[at[(size_t)r]].per == ck.per) return d.data();
        for (size_t k = 0; k < m; ++k) level[k] = d[k / ck.per * levels + k % ck.per];
        return level.data();
    };
    int32_t h2 = DXB_S_OK;
    for (size_t i = 0; i < ck.steps.size() && h2 == DXB_S_OK; ++i)
    {
        const ChunkStep& s = ck.steps[i];
        const dxb200_image* in = images(s.src, s.cover);
        const dxb200_image* out = images(s.dst, s.cover);
        const size_t n = s.cover == StepCover::Front ? m : all;
        switch (s.kind)
        {
        case StepKind::Decompress: h2 = launch_decompress(fp.dp, in, out, n, st); break;
        case StepKind::Demultiply: h2 = launch_pmalpha(fp.dm, in, out, n, st); break;
        case StepKind::Resize: h2 = launch_resize(in, out, n, fp.resizeFilter, fp.resizeMode, st); break;
        case StepKind::BaseCopy:
            for (size_t k = 0; k < n && h2 == DXB_S_OK; ++k)
            {
                // the planned formats are implemented ones, so compute_pitch succeeds; rows of pixels or of blocks
                size_t row = 0, slice = 0;
                (void)compute_pitch(out[k].format, out[k].width, out[k].height, &row, &slice);
                const size_t rows = is_compressed(out[k].format) ? std::max<size_t>(1, (out[k].height + 3) / 4) : out[k].height;
                h2 = cuda_hr(cudaMemcpy2DAsync(out[k].pixels, out[k].rowPitch, in[k].pixels, in[k].rowPitch, row, rows,
                                               cudaMemcpyDeviceToDevice, st), "base -> level 0");
            }
            break;
        case StepKind::Channels: h2 = launch_channel_steps(fp.cp, in, out, n, st); break;
        case StepKind::Convert: h2 = launch_convert(fp.cv, in, out, n, st); break;
        case StepKind::Post: h2 = launch_channel_steps(fp.pp, in, out, n, st); break;
        case StepKind::Mips: h2 = launch_mips(in, cnt, levels, ck.filter, cp.mode, st); break;
        case StepKind::Coverage: h2 = launch_coverage(in, out, cnt, levels, cp.ref, st); break;
        case StepKind::Premultiply:
            if (s.cover != StepCover::PerLevel) { h2 = launch_pmalpha(cp.pm, in, out, n, st); break; }
            for (size_t l = 0; l < levels && h2 == DXB_S_OK; ++l)
            {
                for (size_t it = 0; it < cnt; ++it) level[it] = in[it * levels + l];
                h2 = launch_pmalpha(cp.pm, level.data(), level.data(), cnt, st);
            }
            break;
        case StepKind::Layout: h2 = launch_channel_steps(cp.lp, in, out, n, st); break;
        case StepKind::Compress: h2 = launch_compress(cp.compress, in, out, n, st); break;
        case StepKind::Scan:
        {
            std::vector<dxb200_image> jobWords(n);      // every level of an item sets the item's word
            for (size_t k = 0; k < n; ++k) jobWords[k] = out[k / levels];
            h2 = clear_words(dev[at[(size_t)PlaneRole::Words]], st);
            if (h2 == DXB_S_OK) h2 = launch_alpha_opaque(scan, in, jobWords.data(), n, st);
            break;
        }
        }
    }
    return h2;
}

// ---- [Decompress] -> [demultiply] -> [Resize] -> [channel steps] -> [Convert] -> [channel steps] -> GenerateMipMaps -> [coverage]
// -> [premultiply] -> [BC3 layout] -> [Compress] -> [IsAlphaAllOpaque], chunk by chunk --------------------------------------------
// texconv runs each step as a separate call, so with the host-pointer calls every intermediate travels device -> host -> device.
// Here each item's base goes up once, the steps of fp.chunk run in device memory and only the results come back: 4 B/texel up +
// 1.33 B/texel down for BC3 from RGBA8 instead of 4 + 5.33 + 5.33 + 1.33.  Chunks of whole items are pipelined over the lane's
// NSLOT (stream, buffer) slots.  Each step is one launch per chunk over all the images it covers: the kernels take mixed-size
// batches through the job tables.  That keeps a Convert or a premultiply of kept levels off its vector kernel, which needs equal
// jobs, yet per-level launches measured no faster (DESIGN.md §4); a generated chain's premultiply is one launch per level, whose
// images are equal as the separate calls' are, so it takes the same kernel they do.  When no step writes the chain's level 0 (no
// front step, no Convert), the uploaded base is copied into it device to device, at the chain's pitch; a BC base that passes
// through is copied the same way, row of blocks by row of blocks.  *alphaAllOpaque (when given) = the answer of the scan, or of
// its plan when nothing has to be scanned.
int32_t run_chains(const dxb200_image* base, size_t items, size_t levels, const FromPlan& fp, const AlphaOpaquePlan& scan,
                   const dxb200_image* dst, int32_t* alphaAllOpaque)
{
    const ChunkPlan& ck = fp.chunk;
    ResultWords words;
    int32_t hr = scan.scan ? words.alloc(items) : DXB_S_OK;
    if (hr != DXB_S_OK) return hr;
    const std::vector<dxb200_image> wimg = words.images();
    const dxb200_image* host[PLANE_ROLES] = { base, fp.decompressed.data(), fp.level0.data(), fp.chain.chain.data(), dst, wimg.data() };
    hr = run_sharded(items, [&](size_t i) { return ck.weight[i]; },
        [&](size_t lo, size_t hi)
        {
            const std::vector<Plane> planes = chain_planes(ck, host, lo);
            return run_staged(planes.data(), planes.size(), hi - lo, ITEM_CHUNK,
                [&](const std::vector<dxb200_image>* dev, size_t cnt, cudaStream_t st) { return run_chunk(fp, scan, levels, dev, cnt, st); });
        });
    if (hr == DXB_S_OK && alphaAllOpaque) *alphaAllOpaque = words.all_zero() ? 1 : 0;
    return hr;
}

// The caller's images of every role of every group of a batch, its jobs' images in job order: host[g * PLANE_ROLES + r] = group g's
// images of role r; the words of group g start at unit bp.firstUnit[g] of wimg.  roles holds the arrays host points into.
void batch_roles(const dxb200_texconv_job* jobs, const BatchPlan& bp, const std::vector<dxb200_image>& wimg,
                 std::vector<std::vector<dxb200_image>>* roles, std::vector<const dxb200_image*>* host)
{
    const size_t ng = bp.groups.size();
    roles->assign(ng * PLANE_ROLES, std::vector<dxb200_image>());
    host->assign(ng * PLANE_ROLES, nullptr);
    for (size_t g = 0; g < ng; ++g)
    {
        std::vector<dxb200_image>* r = &(*roles)[g * PLANE_ROLES];
        for (size_t j : bp.groups[g])
        {
            const FromPlan& fp = bp.fp[j];
            const size_t n = jobs[j].items * fp.chunk.per, all = jobs[j].items * jobs[j].levels;
            r[(size_t)PlaneRole::Base].insert(r[(size_t)PlaneRole::Base].end(), jobs[j].base, jobs[j].base + n);
            r[(size_t)PlaneRole::Decompressed].insert(r[(size_t)PlaneRole::Decompressed].end(), fp.decompressed.begin(), fp.decompressed.end());
            r[(size_t)PlaneRole::Level0].insert(r[(size_t)PlaneRole::Level0].end(), fp.level0.begin(), fp.level0.end());
            r[(size_t)PlaneRole::Chain].insert(r[(size_t)PlaneRole::Chain].end(), fp.chain.chain.begin(), fp.chain.chain.end());
            r[(size_t)PlaneRole::Dst].insert(r[(size_t)PlaneRole::Dst].end(), jobs[j].dst, jobs[j].dst + all);
        }
        for (size_t k = 0; k < PLANE_ROLES; ++k) (*host)[g * PLANE_ROLES + k] = r[k].data();
        if (!wimg.empty()) (*host)[g * PLANE_ROLES + (size_t)PlaneRole::Words] = wimg.data() + bp.firstUnit[g];
    }
}

// whether any group of a batch runs the alpha scan
bool batch_scans(const BatchPlan& bp)
{
    bool scan = false;
    for (const std::vector<size_t>& members : bp.groups) scan |= bp.ap[members[0]].scan;
    return scan;
}

// *alphaAllOpaque of every job that ran: the AND of its items' words (1 when it has no scan)
void batch_answers(const dxb200_texconv_job* jobs, const BatchPlan& bp, const ResultWords& words)
{
    for (size_t g = 0; g < bp.groups.size(); ++g)
    {
        size_t u = bp.firstUnit[g];
        for (size_t j : bp.groups[g])
        {
            const bool opaque = !bp.ap[j].scan || std::all_of(words.w + u, words.w + u + jobs[j].items, [](uint32_t v) { return v == 0; });
            if (jobs[j].alphaAllOpaque) *jobs[j].alphaAllOpaque = opaque ? 1 : 0;
            u += jobs[j].items;
        }
    }
}

// dxb200_texconv_batch once every job is planned: group g's items are units bp.firstUnit[g] .. firstUnit[g + 1], split over the
// devices by run_sharded; each device stages its units of every group as one segment per group, through one lane, with the launches
// of the group's first job's plan (equal to every member's).  The alpha answer of a job is the AND of its items' words.
int32_t run_batch(const dxb200_texconv_job* jobs, const BatchPlan& bp)
{
    const size_t ng = bp.groups.size(), units = bp.firstUnit.back();
    ResultWords words;
    int32_t hr = batch_scans(bp) ? words.alloc(units) : DXB_S_OK;
    if (hr != DXB_S_OK) return hr;
    const std::vector<dxb200_image> wimg = words.images();
    std::vector<std::vector<dxb200_image>> roles;
    std::vector<const dxb200_image*> host;
    batch_roles(jobs, bp, wimg, &roles, &host);
    hr = run_sharded(units, [&](size_t i) { return bp.weight[i]; },
        [&](size_t lo, size_t hi)
        {
            std::vector<std::vector<Plane>> planes(ng);
            std::vector<Segment> segs;
            for (size_t g = 0; g < ng; ++g)
            {
                const size_t a = std::max(lo, bp.firstUnit[g]), b = std::min(hi, bp.firstUnit[g + 1]);
                if (a >= b) continue;
                const size_t j = bp.groups[g][0];
                const FromPlan& fp = bp.fp[j];
                const size_t levels = jobs[j].levels;
                planes[g] = chain_planes(fp.chunk, &host[g * PLANE_ROLES], a - bp.firstUnit[g]);
                segs.push_back({ planes[g].data(), planes[g].size(), b - a,
                                 [&fp, &bp, j, levels](const std::vector<dxb200_image>* dev, size_t cnt, cudaStream_t st)
                                 { return run_chunk(fp, bp.ap[j], levels, dev, cnt, st); } });
            }
            return run_segments(segs.data(), segs.size(), ITEM_CHUNK);
        });
    if (hr != DXB_S_OK) return hr;
    batch_answers(jobs, bp, words);
    return DXB_S_OK;
}

// A job of dxb200_texconv_batch_device may run when every base and dst image lies in device or managed memory of device `ord` and
// every BC image's pixel pointer is a whole number of blocks from 0 (bc_pointers_ok): E_INVALIDARG otherwise, so that a wrong pointer
// is refused before any launch instead of faulting a kernel
int32_t device_job_ok(const dxb200_texconv_job& j, size_t per, int ord)
{
    const dxb200_image* sets[2] = { j.base, j.dst };
    const size_t counts[2] = { j.items * per, j.items * j.levels };
    for (int s = 0; s < 2; ++s)
    {
        if (!bc_pointers_ok(sets[s], counts[s])) return DXB_E_INVALIDARG;
        for (size_t i = 0; i < counts[s]; ++i)
        {
            cudaPointerAttributes a;
            const cudaError_t e = cudaPointerGetAttributes(&a, sets[s][i].pixels);
            (void)cudaGetLastError();
            if (e != cudaSuccess || (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) || a.device != ord)
                return DXB_E_INVALIDARG;
        }
    }
    return DXB_S_OK;
}

// One chunk of a _device batch: items [i, k) of group g, whose planes lie chunk_bytes(..., alias) bytes into scratch memory
struct DeviceChunk { size_t g, i, k; };

// dxb200_texconv_batch_device once every job is planned and checked: every group's units on the calling thread's device and
// `stream`, in chunks cut as run_segments cuts them.  A chunk's aliased planes (device_aliases) are the caller's images; the others lie
// in one scratch allocation, sized for the largest chunk and reused chunk after chunk (stream order makes that safe), as the slot
// buffer lays them out, with their Copy::Up images copied in device to device.  Each chunk's result words are read back into pinned
// memory behind its launches; only when a job asks for the alpha answer is the stream synchronised, at the end.
int32_t run_batch_device(const dxb200_texconv_job* jobs, const BatchPlan& bp, cudaStream_t st)
{
    const size_t ng = bp.groups.size();
    const bool scan = batch_scans(bp);
    ResultWords words;
    int32_t hr = scan ? words.alloc(bp.firstUnit.back()) : DXB_S_OK;
    if (hr != DXB_S_OK) return hr;
    const std::vector<dxb200_image> wimg = words.images();
    std::vector<std::vector<dxb200_image>> roles;
    std::vector<const dxb200_image*> host;
    batch_roles(jobs, bp, wimg, &roles, &host);
    std::vector<std::vector<Plane>> planes(ng);
    std::vector<std::vector<bool>> alias(ng);
    std::vector<DeviceChunk> chunks;
    size_t scratch = 0;
    for (size_t g = 0; g < ng; ++g)
    {
        const ChunkPlan& ck = bp.fp[bp.groups[g][0]].chunk;
        planes[g] = chain_planes(ck, &host[g * PLANE_ROLES], 0);
        alias[g] = device_aliases(ck);
        const size_t n = bp.firstUnit[g + 1] - bp.firstUnit[g];
        for (size_t i = 0, k; i < n; i = k)
        {
            k = chunk_end(planes[g].data(), planes[g].size(), i, n, ITEM_CHUNK);
            chunks.push_back({ g, i, k });
            scratch = std::max(scratch, chunk_bytes(planes[g].data(), planes[g].size(), i, k, &alias[g]));
        }
    }
    uint8_t* buf = nullptr;
    DXB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&buf), std::max<size_t>(scratch, 1), st));
    std::vector<dxb200_image> dev[PLANE_ROLES];
    for (size_t c = 0; c < chunks.size() && hr == DXB_S_OK; ++c)
    {
        const DeviceChunk& ch = chunks[c];
        const std::vector<Plane>& pl = planes[ch.g];
        chunk_layout(pl.data(), pl.size(), ch.i, ch.k, &alias[ch.g], buf, dev);
        for (size_t p = 0; p < pl.size() && hr == DXB_S_OK; ++p)
        {
            const dxb200_image* src = pl[p].host + ch.i * pl[p].per;
            for (size_t m = 0; m < dev[p].size() && hr == DXB_S_OK && !alias[ch.g][p]; ++m)
                if ((m % pl[p].per ? pl[p].rest : pl[p].first) == Copy::Up)
                    hr = cuda_hr(cudaMemcpyAsync(dev[p][m].pixels, src[m].pixels, src[m].slicePitch, cudaMemcpyDeviceToDevice, st), "copy in");
        }
        const size_t j = bp.groups[ch.g][0];
        if (hr == DXB_S_OK) hr = run_chunk(bp.fp[j], bp.ap[j], jobs[j].levels, dev, ch.k - ch.i, st);
        // the words of a chunk lie padded_bytes (256) apart in scratch, one per item, and go to consecutive host words
        for (size_t p = 0; p < pl.size() && hr == DXB_S_OK; ++p)
        {
            if (bp.fp[j].chunk.planes[p].role != PlaneRole::Words) continue;
            const std::vector<dxb200_image>& w = dev[p];
            hr = cuda_hr(cudaMemcpy2DAsync(words.w + bp.firstUnit[ch.g] + ch.i, sizeof(uint32_t), w[0].pixels, padded_bytes(w[0]), sizeof(uint32_t),
                                           w.size(), cudaMemcpyDeviceToHost, st), "alpha words");
        }
    }
    const int32_t hf = cuda_hr(cudaFreeAsync(buf, st), "cudaFreeAsync(scratch)");
    if (hr == DXB_S_OK) hr = hf;
    if (hr == DXB_S_OK && scan) hr = cuda_hr(cudaStreamSynchronize(st), "alpha answer sync");       // the answer is a host value
    if (hr == DXB_S_OK) batch_answers(jobs, bp, words);
    return hr;
}

} // namespace

// =================================================================================================
extern "C" {

const char* dxb200_version(void) { return "dxtex_b200 0.1 (sm_90a)"; }
const char* dxb200_last_error(void) { return t_lastError.c_str(); }
uint64_t dxb200_launch_count(void) { return g_launches.load(); }
uint64_t dxb200_kernel_launch_count(const char* kernel)
{
    if (!kernel) return 0;
    std::lock_guard<std::mutex> lk(g_count_mu);
    const auto it = g_kernel_launches.find(kernel);
    return it == g_kernel_launches.end() ? 0 : it->second;
}
uint64_t dxb200_tma_launch_count(void) { return dxb200_kernel_launch_count("k_compress_bc7_tma"); }
int32_t dxb200_set_option(uint32_t option, int32_t value)
{
    if (option == DXB200_OPT_BC7_FEED) { dxb_bc7_set_feed(value); return DXB_S_OK; }
    if (option == DXB200_OPT_MIP_KERNELS) { g_mip_kernels.store(value == 1 ? 1 : 0); return DXB_S_OK; }
    return DXB_E_INVALIDARG;
}
int32_t dxb200_get_option(uint32_t option)
{
    if (option == DXB200_OPT_BC7_FEED) return dxb_bc7_get_feed();
    if (option == DXB200_OPT_MIP_KERNELS) return g_mip_kernels.load();
    return -1;
}

int32_t dxb200_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { (void)cudaGetLastError(); return 0; }
    return n;
}

int32_t dxb200_init_devices(int ndev, const int* devices)
{
    if (ndev <= 0 || !devices) return DXB_E_INVALIDARG;
    std::lock_guard<std::mutex> lk(g_mu);
    int prev = -1;
    if (cudaGetDevice(&prev) != cudaSuccess) { (void)cudaGetLastError(); prev = -1; }
    int32_t hr = DXB_S_OK;
    for (int i = 0; i < ndev && hr == DXB_S_OK; ++i) hr = init_device_locked(devices[i], nullptr);
    // the calling thread keeps the first listed device current (what dxb200_init(device) always did)
    if (hr == DXB_S_OK) hr = cuda_hr(cudaSetDevice(devices[0]), "cudaSetDevice");
    else if (prev >= 0) (void)cudaSetDevice(prev);
    return hr;
}

int32_t dxb200_init(int device) { return dxb200_init_devices(1, &device); }

int32_t dxb200_initialized_devices(int* devices, int maxDevices)
{
    std::lock_guard<std::mutex> lk(g_mu);
    for (size_t i = 0; i < g_devs.size() && devices && (int)i < maxDevices; ++i) devices[i] = g_devs[i]->ordinal;
    return (int32_t)g_devs.size();
}

void dxb200_shutdown(void)
{
    std::lock_guard<std::mutex> lk(g_mu);
    int prev = -1;
    if (cudaGetDevice(&prev) != cudaSuccess) { (void)cudaGetLastError(); prev = -1; }
    for (auto& d : g_devs)
    {
        if (cudaSetDevice(d->ordinal) != cudaSuccess) { (void)cudaGetLastError(); continue; }
        for (int l = 0; l < NLANE; ++l)
            for (int i = 0; i < NSLOT; ++i)
            {
                Lane& L = d->lanes[l];
                if (L.streams[i]) { cudaStreamSynchronize(L.streams[i]); cudaStreamDestroy(L.streams[i]); L.streams[i] = nullptr; }
                if (L.buf[i]) { cudaFree(L.buf[i]); L.buf[i] = nullptr; L.cap[i] = 0; }
            }
    }
    g_devs.clear();
    if (prev >= 0) (void)cudaSetDevice(prev);
}

// Pinned host memory for full-rate, overlapped H2D / D2H.  The pages are placed on the NUMA node of the calling thread's
// current CUDA device (memory policy MPOL_PREFERRED around the allocation): a rank whose staging buffers sit on the other
// socket pays the inter-socket link on every copy (8 ranks x 51 GB/s measured 0.75 end-to-end efficiency in round 1).
void* dxb200_host_alloc(size_t bytes)
{
    std::vector<Device*> devs;
    if (device_list(&devs) != DXB_S_OK) return nullptr;
    int cur = -1, node = -1;
    if (cudaGetDevice(&cur) != cudaSuccess) { (void)cudaGetLastError(); cur = -1; }
    for (Device* d : devs) if (d->ordinal == cur) node = d->numaNode;
    if (node < 0 && cur >= 0) node = device_numa_node(cur);
    bool policy = false;
#if defined(SYS_set_mempolicy)
    if (node >= 0 && node < 64)
    {
        unsigned long mask = 1ul << node;
        policy = (syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, &mask, sizeof(mask) * 8 + 1) == 0);
    }
#endif
    void* p = nullptr;
    const cudaError_t e = cudaHostAlloc(&p, bytes, cudaHostAllocPortable);
#if defined(SYS_set_mempolicy)
    if (policy) (void)syscall(SYS_set_mempolicy, 0 /* MPOL_DEFAULT */, nullptr, 0);
#endif
    if (e != cudaSuccess) { (void)cudaGetLastError(); return nullptr; }
    return p;
}
void dxb200_host_free(void* p) { if (p) cudaFreeHost(p); }

int32_t dxb200_compute_pitch(uint32_t format, size_t width, size_t height, size_t* rowPitch, size_t* slicePitch)
{
    if (!rowPitch || !slicePitch) return DXB_E_POINTER;
    return compute_pitch(format, width, height, rowPitch, slicePitch);
}

int32_t dxb200_calculate_mip_levels(size_t width, size_t height, size_t* levels)
{
    if (!levels) return DXB_E_POINTER;
    if (*levels > 1) { if (*levels > count_mips(width, height)) return DXB_E_INVALIDARG; }
    else if (*levels == 0) *levels = count_mips(width, height);
    else *levels = 1;
    return DXB_S_OK;
}

// ---- Compress -----------------------------------------------------------------------------------
int32_t dxb200_compress_device(const dxb200_image* src, size_t nimages, uint32_t dstFormat, uint32_t flags, float threshold,
                               float alphaWeight, const dxb200_image* dst, void* stream)
{
    (void)alphaWeight;      // only the reference's DirectCompute path has an alpha weight (DirectXTex.h:919); the CPU encoder we match has none
    CompressPlan plan;
    int32_t hr = plan_compress(src, nimages, dstFormat, flags, threshold, dst, &plan);
    if (hr != DXB_S_OK) return hr;
    if (!bc_pointers_ok(dst, nimages)) return DXB_E_INVALIDARG;
    DevScope scope;
    hr = scope.enter(src[0].pixels);
    if (hr != DXB_S_OK) return hr;
    return launch_compress(plan, src, dst, nimages, static_cast<cudaStream_t>(stream));
}

int32_t dxb200_compress_ex(const dxb200_image* src, size_t nimages, uint32_t dstFormat, uint32_t flags, float threshold,
                           float alphaWeight, const dxb200_image* dst, dxb200_status_fn status, void* user)
{
    (void)alphaWeight;
    CompressPlan plan;
    int32_t hr = plan_compress(src, nimages, dstFormat, flags, threshold, dst, &plan);
    if (hr != DXB_S_OK) return hr;
    return run_bands(src, dst, nimages, 4, 1, false, true, status, user,
        [&](const dxb200_image* ds, const dxb200_image* dd, size_t cnt, cudaStream_t st) { return launch_compress(plan, ds, dd, cnt, st); });
}

int32_t dxb200_compress(const dxb200_image* src, size_t nimages, uint32_t dstFormat, uint32_t flags, float threshold,
                        float alphaWeight, const dxb200_image* dst)
{
    return dxb200_compress_ex(src, nimages, dstFormat, flags, threshold, alphaWeight, dst, nullptr, nullptr);
}

// ---- Decompress (DirectXTexCompress.cpp:852-979; DecompressBC :425-535) ---------------------------------
int32_t dxb200_decompress_device(const dxb200_image* src, size_t nimages, uint32_t dstFormat, const dxb200_image* dst, void* stream)
{
    dxb_compress_params P;
    int32_t hr = plan_decompress(src, nimages, dstFormat, dst, &P);
    if (hr != DXB_S_OK) return hr;
    if (!bc_pointers_ok(src, nimages)) return DXB_E_INVALIDARG;
    DevScope scope;
    hr = scope.enter(src[0].pixels);
    if (hr != DXB_S_OK) return hr;
    return launch_decompress(P, src, dst, nimages, static_cast<cudaStream_t>(stream));
}

int32_t dxb200_decompress(const dxb200_image* src, size_t nimages, uint32_t dstFormat, const dxb200_image* dst)
{
    dxb_compress_params P;
    int32_t hr = plan_decompress(src, nimages, dstFormat, dst, &P);
    if (hr != DXB_S_OK) return hr;
    return run_bands(src, dst, nimages, 1, 4, true, false, nullptr, nullptr,
        [&](const dxb200_image* ds, const dxb200_image* dd, size_t cnt, cudaStream_t st) { return launch_decompress(P, ds, dd, cnt, st); });
}

// ---- Convert ------------------------------------------------------------------------------------
int32_t dxb200_convert_device(const dxb200_image* src, size_t nimages, uint32_t dstFormat, uint32_t filter, float threshold,
                              const dxb200_image* dst, void* stream)
{
    dxb_convert_params P;
    int32_t hr = plan_convert(src, nimages, dstFormat, filter, dst, &P);
    if (hr != DXB_S_OK) return hr;
    P.threshold = threshold;       // alpha threshold of the 1-bit alpha destination (B5G5R5A1)
    DevScope scope;
    hr = scope.enter(src[0].pixels);
    if (hr != DXB_S_OK) return hr;
    return launch_convert(P, src, dst, nimages, static_cast<cudaStream_t>(stream));
}

int32_t dxb200_convert_ex(const dxb200_image* src, size_t nimages, uint32_t dstFormat, uint32_t filter, float threshold, const dxb200_image* dst,
                          dxb200_status_fn status, void* user)
{
    dxb_convert_params P;
    int32_t hr = plan_convert(src, nimages, dstFormat, filter, dst, &P);
    if (hr != DXB_S_OK) return hr;
    P.threshold = threshold;
    // bands start on multiples of 4 rows so that the 4x4 ordered-dither matrix keeps its phase
    // (error diffusion carries state from row to row: whole images only)
    size_t rowsPerUnit = (P.flags & DXB_FILTER_DITHER) ? 4 : 1;
    if (P.flags & DXB_FILTER_DITHER_DIFFUSION) for (size_t i = 0; i < nimages; ++i) rowsPerUnit = std::max(rowsPerUnit, src[i].height);
    return run_bands(src, dst, nimages, rowsPerUnit, rowsPerUnit, false, false, status, user,
        [&](const dxb200_image* ds, const dxb200_image* dd, size_t cnt, cudaStream_t st) { return launch_convert(P, ds, dd, cnt, st); });
}

int32_t dxb200_convert(const dxb200_image* src, size_t nimages, uint32_t dstFormat, uint32_t filter, float threshold, const dxb200_image* dst)
{
    return dxb200_convert_ex(src, nimages, dstFormat, filter, threshold, dst, nullptr, nullptr);
}

// ---- GenerateMipMaps ----------------------------------------------------------------------------
int32_t dxb200_generate_mipmaps_device(const dxb200_image* chain, size_t items, size_t levels, uint32_t filter, void* stream)
{
    uint32_t mode = 0;
    int32_t hr = plan_mips(chain, items, levels, filter, &mode);
    if (hr != DXB_S_OK) return hr;
    DevScope scope;
    hr = scope.enter(chain[0].pixels);
    if (hr != DXB_S_OK) return hr;
    return launch_mips(chain, items, levels, filter, mode, static_cast<cudaStream_t>(stream));
}

int32_t dxb200_generate_mipmaps(const dxb200_image* chain, size_t items, size_t levels, uint32_t filter)
{
    uint32_t mode = 0;
    int32_t hr = plan_mips(chain, items, levels, filter, &mode);
    if (hr != DXB_S_OK) return hr;
    // image-per-GPU sharding: contiguous item ranges per device; a single item's chain stays on one device (SURVEY 8(e))
    return run_sharded(items, [&](size_t i) { return chain[i * levels].slicePitch; },
        [&](size_t lo, size_t hi)
        {
            const Plane chains = { chain + lo * levels, levels, Copy::Up, Copy::Down };
            return run_staged(&chains, 1, hi - lo, ITEM_CHUNK,
                [&](const std::vector<dxb200_image>* dev, size_t cnt, cudaStream_t st) { return launch_mips(dev[0].data(), cnt, levels, filter, mode, st); });
        });
}

// ---- GenerateMipMaps + Compress in one call: the mip chain never leaves HBM (run_chains) --------------------------------
// Per item: base[i] = level 0 (host), dst[i * levels + l] = the BC image of level l (host).  dxb200_mipmaps_compress_ex adds
// texconv's two steps between the mips and the compression (-keepcoverage :3480, -pmalpha :3526), both in place on the chunk's
// chains in device memory; dxb200_mipmaps_compress_from adds Decompress and Resize in front of the mips.
// dxb200_mipmaps_compress_from_ex adds texconv's "set alpha mode" test of the output (:3738-3766): IsAlphaAllOpaque of the blocks,
// scanned where they were made.  dxb200_mipmaps_compress_from_channels adds texconv's channel steps after Resize (:2645-3300).
// dxb200_mipmaps_compress_from_channels_ex adds texconv's -alpha and BC3n / RXGB steps (dxb200_texconv_steps).
int32_t dxb200_mipmaps_compress_from_channels_ex(const dxb200_image* base, size_t items, const dxb200_chain_source* source,
                                                 const dxb200_channel_steps* channels, size_t levels, uint32_t filter, const dxb200_chain_steps* steps,
                                                 uint32_t dstFormat, uint32_t flags, float threshold, float alphaWeight, const dxb200_image* dst,
                                                 int32_t* alphaAllOpaque, const dxb200_texconv_steps* ts)
{
    (void)alphaWeight;
    FromPlan fp;
    AlphaOpaquePlan ap;
    const int32_t hr = plan_mipmaps_compress_channels(base, items, source, channels, levels, filter, steps, dstFormat, flags, threshold, dst,
                                                      &fp, ts, alphaAllOpaque, &ap);
    return hr != DXB_S_OK ? hr : run_chains(base, items, levels, fp, ap, dst, alphaAllOpaque);
}

int32_t dxb200_mipmaps_compress_from_channels(const dxb200_image* base, size_t items, const dxb200_chain_source* source,
                                              const dxb200_channel_steps* channels, size_t levels, uint32_t filter, const dxb200_chain_steps* steps,
                                              uint32_t dstFormat, uint32_t flags, float threshold, float alphaWeight, const dxb200_image* dst,
                                              int32_t* alphaAllOpaque)
{
    return dxb200_mipmaps_compress_from_channels_ex(base, items, source, channels, levels, filter, steps, dstFormat, flags, threshold, alphaWeight,
                                                    dst, alphaAllOpaque, nullptr);
}

int32_t dxb200_mipmaps_compress_from_ex(const dxb200_image* base, size_t items, const dxb200_chain_source* source, size_t levels, uint32_t filter,
                                        const dxb200_chain_steps* steps, uint32_t dstFormat, uint32_t flags, float threshold, float alphaWeight,
                                        const dxb200_image* dst, int32_t* alphaAllOpaque)
{
    return dxb200_mipmaps_compress_from_channels(base, items, source, nullptr, levels, filter, steps, dstFormat, flags, threshold, alphaWeight,
                                                 dst, alphaAllOpaque);
}

int32_t dxb200_mipmaps_compress_from(const dxb200_image* base, size_t items, const dxb200_chain_source* source, size_t levels, uint32_t filter,
                                     const dxb200_chain_steps* steps, uint32_t dstFormat, uint32_t flags, float threshold, float alphaWeight,
                                     const dxb200_image* dst)
{
    return dxb200_mipmaps_compress_from_ex(base, items, source, levels, filter, steps, dstFormat, flags, threshold, alphaWeight, dst, nullptr);
}

int32_t dxb200_mipmaps_compress_ex(const dxb200_image* base, size_t items, size_t levels, uint32_t filter, const dxb200_chain_steps* steps,
                                   uint32_t dstFormat, uint32_t flags, float threshold, float alphaWeight, const dxb200_image* dst)
{
    return dxb200_mipmaps_compress_from(base, items, nullptr, levels, filter, steps, dstFormat, flags, threshold, alphaWeight, dst);
}

int32_t dxb200_mipmaps_compress(const dxb200_image* base, size_t items, size_t levels, uint32_t filter, uint32_t dstFormat,
                                uint32_t flags, float threshold, float alphaWeight, const dxb200_image* dst)
{
    return dxb200_mipmaps_compress_ex(base, items, levels, filter, nullptr, dstFormat, flags, threshold, alphaWeight, dst);
}

// ---- texconv's path to an uncompressed target in one call: the chain never leaves HBM until it is done (run_chains) ------------
int32_t dxb200_mipmaps_convert_from_ex(const dxb200_image* base, size_t items, const dxb200_chain_source* source,
                                       const dxb200_channel_steps* channels, uint32_t dstFormat, uint32_t convertFilter, float threshold,
                                       size_t levels, uint32_t filter, const dxb200_chain_steps* steps, const dxb200_image* dst,
                                       int32_t* alphaAllOpaque, const dxb200_texconv_steps* ts)
{
    FromPlan fp;
    AlphaOpaquePlan ap;
    const int32_t hr = plan_mipmaps_convert_from(base, items, source, channels, dstFormat, convertFilter, threshold, levels, filter, steps, dst,
                                                 alphaAllOpaque, &fp, &ap, ts);
    return hr != DXB_S_OK ? hr : run_chains(base, items, levels, fp, ap, dst, alphaAllOpaque);
}

int32_t dxb200_mipmaps_convert_from(const dxb200_image* base, size_t items, const dxb200_chain_source* source, const dxb200_channel_steps* channels,
                                    uint32_t dstFormat, uint32_t convertFilter, float threshold, size_t levels, uint32_t filter,
                                    const dxb200_chain_steps* steps, const dxb200_image* dst, int32_t* alphaAllOpaque)
{
    return dxb200_mipmaps_convert_from_ex(base, items, source, channels, dstFormat, convertFilter, threshold, levels, filter, steps, dst,
                                          alphaAllOpaque, nullptr);
}

// ---- texconv on items that keep their own levels: every level stays in device memory until it is done (run_chains) -------------
int32_t dxb200_levels_from_ex(const dxb200_image* base, size_t items, size_t levels, const dxb200_chain_source* source,
                              const dxb200_channel_steps* channels, uint32_t dstFormat, uint32_t convertFilter, uint32_t compressFlags,
                              float threshold, const dxb200_chain_steps* steps, const dxb200_image* dst, int32_t* alphaAllOpaque,
                              const dxb200_texconv_steps* ts)
{
    FromPlan fp;
    AlphaOpaquePlan ap;
    const int32_t hr = plan_levels_from(base, items, levels, source, channels, dstFormat, convertFilter, compressFlags, threshold, steps, dst,
                                        alphaAllOpaque, &fp, &ap, ts);
    return hr != DXB_S_OK ? hr : run_chains(base, items, levels, fp, ap, dst, alphaAllOpaque);
}

int32_t dxb200_levels_from(const dxb200_image* base, size_t items, size_t levels, const dxb200_chain_source* source,
                           const dxb200_channel_steps* channels, uint32_t dstFormat, uint32_t convertFilter, uint32_t compressFlags,
                           float threshold, const dxb200_chain_steps* steps, const dxb200_image* dst, int32_t* alphaAllOpaque)
{
    return dxb200_levels_from_ex(base, items, levels, source, channels, dstFormat, convertFilter, compressFlags, threshold, steps, dst,
                                 alphaAllOpaque, nullptr);
}

// ---- texconv over a list of textures: the jobs planned first, then every group's units sharded and staged (run_batch) ----------
int32_t dxb200_texconv_batch(const dxb200_texconv_job* jobs, size_t njobs, int32_t* results)
{
    if (!jobs || !njobs) return DXB_E_INVALIDARG;
    BatchPlan bp;
    (void)plan_texconv_batch(jobs, njobs, &bp);          // each job's HRESULT is in bp.hr
    if (!bp.groups.empty())
        if (const int32_t hr = run_batch(jobs, bp))
            for (size_t i = 0; i < njobs; ++i) if (bp.group[i] != SIZE_MAX) bp.hr[i] = hr;
    if (results) std::copy(bp.hr.begin(), bp.hr.end(), results);
    for (int32_t hr : bp.hr) if (hr != DXB_S_OK) return hr;
    return DXB_S_OK;
}

// ---- the same on textures in device memory, on the caller's stream (run_batch_device) -------------------------------------------
int32_t dxb200_texconv_batch_device(const dxb200_texconv_job* jobs, size_t njobs, int32_t* results, void* stream)
{
    if (!jobs || !njobs) return DXB_E_INVALIDARG;
    // the device is entered when the first job passes its planner, so that a batch of failing jobs needs none
    DevScope scope;
    bool entered = false;
    int32_t hs = DXB_S_OK;
    BatchPlan bp;
    (void)plan_texconv_batch(jobs, njobs, &bp, [&](size_t i)
    {
        if (!entered) { entered = true; hs = scope.enter(jobs[0].base && jobs[0].items ? jobs[0].base[0].pixels : nullptr); }
        return hs != DXB_S_OK ? hs : device_job_ok(jobs[i], bp.fp[i].chunk.per, scope.ord);
    });
    if (!bp.groups.empty())
        if (const int32_t hr = run_batch_device(jobs, bp, static_cast<cudaStream_t>(stream)))
            for (size_t i = 0; i < njobs; ++i) if (bp.group[i] != SIZE_MAX) bp.hr[i] = hr;
    if (results) std::copy(bp.hr.begin(), bp.hr.end(), results);
    for (int32_t hr : bp.hr) if (hr != DXB_S_OK) return hr;
    return DXB_S_OK;
}

int32_t dxb200_premultiply_alpha_device(const dxb200_image* src, size_t nimages, uint32_t flags, const dxb200_image* dst, void* stream)
{
    dxb_convert_params P;
    int32_t hr = plan_pmalpha(src, nimages, flags, dst, &P);
    if (hr != DXB_S_OK) return hr;
    DevScope scope;
    hr = scope.enter(src[0].pixels);
    if (hr != DXB_S_OK) return hr;
    return launch_pmalpha(P, src, dst, nimages, static_cast<cudaStream_t>(stream));
}

int32_t dxb200_premultiply_alpha(const dxb200_image* src, size_t nimages, uint32_t flags, const dxb200_image* dst)
{
    dxb_convert_params P;
    int32_t hr = plan_pmalpha(src, nimages, flags, dst, &P);
    if (hr != DXB_S_OK) return hr;
    return run_bands(src, dst, nimages, 1, 1, false, false, nullptr, nullptr,
        [&](const dxb200_image* ds, const dxb200_image* dd, size_t cnt, cudaStream_t st) { return launch_pmalpha(P, ds, dd, cnt, st); });
}

// ---- texconv's channel steps (TransformImage with texconv's lambdas) --------------------------------------------------------
int32_t dxb200_apply_channel_steps_device(const dxb200_image* src, size_t n, const dxb200_channel_steps* steps, const dxb200_image* dst, void* stream)
{
    dxb_convert_params P;
    int32_t hr = plan_channel_steps(src, n, steps, dst, &P);
    if (hr != DXB_S_OK) return hr;
    DevScope scope;
    hr = scope.enter(src[0].pixels);
    if (hr != DXB_S_OK) return hr;
    return launch_channel_steps(P, src, dst, n, static_cast<cudaStream_t>(stream));
}

int32_t dxb200_apply_channel_steps(const dxb200_image* src, size_t n, const dxb200_channel_steps* steps, const dxb200_image* dst)
{
    dxb_convert_params P;
    int32_t hr = plan_channel_steps(src, n, steps, dst, &P);
    if (hr != DXB_S_OK) return hr;
    return run_bands(src, dst, n, 1, 1, false, false, nullptr, nullptr,
        [&](const dxb200_image* ds, const dxb200_image* dd, size_t cnt, cudaStream_t st) { return launch_channel_steps(P, ds, dd, cnt, st); });
}

// ---- ScaleMipMapsAlphaForCoverage ----------------------------------------------------------------
int32_t dxb200_scale_mipmaps_alpha_for_coverage_device(const dxb200_image* src, size_t nlevels, float alphaReference, const dxb200_image* dst, void* stream)
{
    int32_t hr = plan_alpha_coverage(src, nlevels, dst);
    if (hr != DXB_S_OK) return hr;
    DevScope scope;
    hr = scope.enter(src[0].pixels);
    if (hr != DXB_S_OK) return hr;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    hr = scale_alpha_for_coverage_device(src, nlevels, alphaReference, dst, st);
    const int32_t hs = cuda_hr(cudaStreamSynchronize(st), "alpha coverage sync");       // the documented end of the call
    return hr != DXB_S_OK ? hr : hs;
}

int32_t dxb200_scale_mipmaps_alpha_for_coverage(const dxb200_image* src, size_t nlevels, float alphaReference, const dxb200_image* dst)
{
    int32_t hr = plan_alpha_coverage(src, nlevels, dst);
    if (hr != DXB_S_OK) return hr;
    std::vector<Device*> devs;
    hr = device_list(&devs);
    if (hr != DXB_S_OK) return hr;
    HostScope scope;
    hr = scope.enter(devs[0]);
    if (hr != DXB_S_OK) return hr;
    cudaStream_t st = t_v.lane->streams[0];
    size_t bytes = 0;
    for (size_t l = 0; l < nlevels; ++l) bytes += 2 * ((src[l].slicePitch + 255) & ~size_t(255));
    hr = ensure_buffer(&t_v.lane->buf[0], &t_v.lane->cap[0], bytes);
    if (hr != DXB_S_OK) return hr;
    std::vector<dxb200_image> ds(src, src + nlevels), dd(dst, dst + nlevels);
    size_t off = 0;
    for (size_t l = 0; l < nlevels && hr == DXB_S_OK; ++l)
    {
        ds[l].pixels = static_cast<uint8_t*>(t_v.lane->buf[0]) + off; off += (src[l].slicePitch + 255) & ~size_t(255);
        dd[l].pixels = static_cast<uint8_t*>(t_v.lane->buf[0]) + off; off += (src[l].slicePitch + 255) & ~size_t(255);
        dd[l].rowPitch = src[l].rowPitch; dd[l].slicePitch = src[l].slicePitch;          // device copy uses the source layout
        hr = cuda_hr(cudaMemcpyAsync(ds[l].pixels, src[l].pixels, src[l].slicePitch, cudaMemcpyHostToDevice, st), "H2D");
    }
    if (hr == DXB_S_OK) hr = scale_alpha_for_coverage_device(ds.data(), nlevels, alphaReference, dd.data(), st);
    for (size_t l = 0; l < nlevels && hr == DXB_S_OK; ++l)
        hr = cuda_hr(cudaMemcpy2DAsync(dst[l].pixels, dst[l].rowPitch, dd[l].pixels, dd[l].rowPitch, std::min(dst[l].rowPitch, dd[l].rowPitch),
                                       src[l].slicePitch / std::max<size_t>(src[l].rowPitch, 1), cudaMemcpyDeviceToHost, st), "D2H");
    if (hr == DXB_S_OK) hr = cuda_hr(cudaStreamSynchronize(st), "alpha coverage sync");
    return hr;
}

// ---- IsAlphaAllOpaque ----------------------------------------------------------------------------
int32_t dxb200_is_alpha_all_opaque_device(const dxb200_image* images, size_t nimages, int32_t* opaque, void* stream)
{
    AlphaOpaquePlan ap;
    int32_t hr = plan_alpha_opaque(images, nimages, opaque, &ap);
    if (hr != DXB_S_OK) return hr;
    if (!ap.scan) { *opaque = 1; return DXB_S_OK; }
    if (!bc_pointers_ok(images, nimages)) return DXB_E_INVALIDARG;
    DevScope scope;
    hr = scope.enter(images[0].pixels);
    if (hr != DXB_S_OK) return hr;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    uint8_t* word = nullptr;                            // one word for the whole call: every job may set it
    DXB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&word), sizeof(uint32_t), st));
    const std::vector<dxb200_image> words(nimages, dxb200_image{ 1, 1, DXB_FMT_UNKNOWN, sizeof(uint32_t), sizeof(uint32_t), word });
    uint32_t result = 0;
    hr = cuda_hr(cudaMemsetAsync(word, 0, sizeof(uint32_t), st), "cudaMemsetAsync(alpha word)");
    if (hr == DXB_S_OK) hr = launch_alpha_opaque(ap, images, words.data(), nimages, st);
    if (hr == DXB_S_OK) hr = cuda_hr(cudaMemcpyAsync(&result, word, sizeof(uint32_t), cudaMemcpyDeviceToHost, st), "D2H");
    cudaFreeAsync(word, st);
    const int32_t hs = cuda_hr(cudaStreamSynchronize(st), "alpha opaque sync");        // the answer is a host value
    if (hr == DXB_S_OK && hs == DXB_S_OK) *opaque = result ? 0 : 1;
    return hr != DXB_S_OK ? hr : hs;
}

// Bands of whole (block) rows, as the band calls cut them, sharded over the devices by bytes; the images go up, one result word
// per band comes back, and the answer is the AND of the bands'.
int32_t dxb200_is_alpha_all_opaque(const dxb200_image* images, size_t nimages, int32_t* opaque)
{
    AlphaOpaquePlan ap;
    int32_t hr = plan_alpha_opaque(images, nimages, opaque, &ap);
    if (hr != DXB_S_OK) return hr;
    if (!ap.scan) { *opaque = 1; return DXB_S_OK; }
    std::vector<dxb200_image> none(images, images + nimages);          // no destination: bands count the source's bytes only
    for (dxb200_image& im : none) im.rowPitch = im.slicePitch = 0;
    BandSplit bands;
    split_bands(images, none.data(), nimages, 1, 0, ap.blocks, false, bands);
    ResultWords words;
    if ((hr = words.alloc(bands.src.size())) != DXB_S_OK) return hr;
    const std::vector<dxb200_image> wimg = words.images();
    hr = run_sharded(bands.src.size(), [&](size_t i) { return bands.src[i].slicePitch; },
        [&](size_t lo, size_t hi)
        {
            const Plane planes[2] = { { bands.src.data() + lo, 1, Copy::Up, Copy::Up }, { wimg.data() + lo, 1, Copy::Down, Copy::Down } };
            return run_staged(planes, 2, hi - lo, BAND_CHUNK,
                [&](const std::vector<dxb200_image>* dev, size_t cnt, cudaStream_t st)
                {
                    const int32_t h2 = clear_words(dev[1], st);
                    return h2 != DXB_S_OK ? h2 : launch_alpha_opaque(ap, dev[0].data(), dev[1].data(), cnt, st);
                });
        });
    if (hr == DXB_S_OK) *opaque = words.all_zero() ? 1 : 0;
    return hr;
}

int32_t dxb200_resize_device(const dxb200_image* src, size_t nimages, uint32_t filter, const dxb200_image* dst, void* stream)
{
    uint32_t mode = 0;
    int32_t hr = plan_resize(src, nimages, filter, dst, &mode);
    if (hr != DXB_S_OK) return hr;
    DevScope scope;
    hr = scope.enter(src[0].pixels);
    if (hr != DXB_S_OK) return hr;
    return launch_resize(src, dst, nimages, filter, mode, static_cast<cudaStream_t>(stream));
}

int32_t dxb200_resize(const dxb200_image* src, size_t nimages, uint32_t filter, const dxb200_image* dst)
{
    uint32_t mode = 0;
    int32_t hr = plan_resize(src, nimages, filter, dst, &mode);
    if (hr != DXB_S_OK) return hr;
    return run_sharded(nimages, [&](size_t i) { return src[i].slicePitch + dst[i].slicePitch; },
        [&](size_t lo, size_t hi)
        {
            const Plane planes[2] = { { src + lo, 1, Copy::Up, Copy::Up }, { dst + lo, 1, Copy::Down, Copy::Down } };
            return run_staged(planes, 2, hi - lo, ITEM_CHUNK,
                [&](const std::vector<dxb200_image>* dev, size_t cnt, cudaStream_t st) { return launch_resize(dev[0].data(), dev[1].data(), cnt, filter, mode, st); });
        });
}

} // extern "C"
