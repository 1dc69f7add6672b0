// dxb_api.cu — the extern "C" boundary of libdxtex_b200.so (see include/dxtex_b200.h) and the host
// logic behind it: argument validation with the reference's HRESULTs, pitch rules, batching,
// staging of host images through device memory, kernel launches on sm_90a.
//
// Every host-pointer call stages through one routine, run_staged: whole items (a band and its output, a mip chain, a resize
// pair) are grouped into chunks that pipeline H2D -> kernels -> D2H over the NSLOT (stream, buffer) slots of a lane.  Band calls
// (compress, decompress, convert, premultiply) cut images into ~32 MiB bands and stage 48 MiB per chunk; chain and pair calls
// (generate_mipmaps, resize, mipmaps_compress) stage 80 MiB per chunk.  ScaleMipMapsAlphaForCoverage stages on its own: it
// downloads with a 2D copy into the caller's pitch and its bisection synchronises on the host.
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
#include "dxb_host_tri.h"

namespace {

constexpr int NSLOT = 3;        // (stream, device buffer) slots of one lane: H2D / kernel / D2H of consecutive chunks overlap
constexpr int NLANE = 2;        // host-staged calls that can be in flight on one device at the same time (each owns a lane)
constexpr size_t BAND_BYTES = size_t(32) << 20;     // source + destination bytes of one band of a band call
constexpr size_t BAND_CHUNK = size_t(48) << 20;     // slot buffer bytes of one chunk of a band call
// slot buffer bytes of one chunk of a chain or pair call; 80 MiB keeps eleven 1024^2 RGBA8 -> BC3 chains of mipmaps_compress in a
// chunk: with 64 MiB (nine) its end-to-end time was about 4 % longer (H100 80GB HBM3 at 400 W, DESIGN.md §4)
constexpr size_t ITEM_CHUNK = size_t(80) << 20;

std::mutex g_mu;                // guards the device table only; calls on different lanes / devices run concurrently
std::atomic<uint64_t> g_launches{0}, g_tma_launches{0};
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
    double total = 0;
    for (size_t i = 0; i < n; ++i) total += (double)weight(i);
    std::vector<size_t> cut(nd + 1, n);
    cut[0] = 0;
    {
        double acc = 0; size_t d = 1;
        for (size_t i = 0; i < n && d < nd; ++i)
        {
            acc += (double)weight(i);
            while (d < nd && acc >= total * (double)d / (double)nd) cut[d++] = i + 1;
        }
    }
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

// ---- format predicates (DirectXTex.inl:57-130 / DirectXTexUtil.cpp), implemented subset ----------
bool is_compressed(uint32_t f) { return dxb_bc_block_bytes(f) != 0; }
bool is_supported_pixel_format(uint32_t f) { return dxb_bytes_per_pixel(f) != 0; }

int32_t compute_pitch(uint32_t fmt, size_t w, size_t h, size_t* row, size_t* slice)
{
    if (const uint32_t bs = dxb_bc_block_bytes(fmt))
    {
        const size_t nbw = std::max<size_t>(1, (w + 3) / 4), nbh = std::max<size_t>(1, (h + 3) / 4);
        *row = nbw * bs; *slice = *row * nbh;
        return DXB_S_OK;
    }
    if (const uint32_t bpp = dxb_bytes_per_pixel(fmt))
    {
        *row = w * bpp; *slice = *row * h;
        return DXB_S_OK;
    }
    return DXB_E_NOT_SUPPORTED;
}

size_t count_mips(size_t w, size_t h)
{
    size_t n = 1;
    while (h > 1 || w > 1) { if (h > 1) h >>= 1; if (w > 1) w >>= 1; ++n; }
    return n;
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
struct CompressPlan { dxb_compress_params P; bool bc7, bc6h; };

// validation + flag resolution shared by host and device variants (DirectXTexCompress.cpp:664-676, 732-749, 72-107)
int32_t plan_compress(const dxb200_image* src, size_t n, uint32_t dstFormat, uint32_t flags, float threshold,
                      const dxb200_image* dst, CompressPlan* plan)
{
    if (!src || !dst || !n) return DXB_E_INVALIDARG;
    const uint32_t srcFormat = src[0].format;
    if (is_compressed(srcFormat) || !is_compressed(dstFormat)) return DXB_E_INVALIDARG;
    if (!is_supported_pixel_format(srcFormat)) return DXB_E_NOT_SUPPORTED;        // no CPU fallback for other formats
    for (size_t i = 0; i < n; ++i)
    {
        if (!src[i].pixels || !dst[i].pixels) return DXB_E_POINTER;
        if (src[i].format != srcFormat || dst[i].format != dstFormat) return DXB_E_INVALIDARG;
        if (src[i].width != dst[i].width || src[i].height != dst[i].height) return DXB_E_FAIL;
        if (!src[i].width || !src[i].height || src[i].width > 0xFFFFFFFFull || src[i].height > 0xFFFFFFFFull) return DXB_E_INVALIDARG;
    }
    dxb_compress_params& P = plan->P;
    P.srcFormat = srcFormat; P.dstFormat = dstFormat;
    P.inF = dxb_convert_flags(srcFormat); P.outF = dxb_convert_flags(dstFormat);
    uint32_t cflags = 0;                                                       // DetermineEncoderSettings :46-68
    if (dstFormat == DXB_FMT_BC4_UNORM || dstFormat == DXB_FMT_BC4_SNORM) cflags = DXB_FILTER_RGB_COPY_RED;
    if (dstFormat == DXB_FMT_BC5_UNORM || dstFormat == DXB_FMT_BC5_SNORM) cflags = DXB_FILTER_RGB_COPY_RED | DXB_FILTER_RGB_COPY_GREEN;
    cflags |= (flags & DXB_FILTER_SRGB_MASK);                                  // GetSRGBFlags :37-44
    P.cflags = dxb_resolve_srgb_convert(cflags, srcFormat, dstFormat);
    P.bcflags = flags & (DXB_BC_FLAGS_DITHER_RGB | DXB_BC_FLAGS_DITHER_A | DXB_BC_FLAGS_UNIFORM |
                         DXB_BC_FLAGS_USE_3SUBSETS | DXB_BC_FLAGS_FORCE_BC7_MODE6);                 // GetBCFlags :26-35
    P.threshold = threshold;
    plan->bc7 = (dxb_make_linear(dstFormat) == DXB_FMT_BC7_UNORM);
    plan->bc6h = (dstFormat == DXB_FMT_BC6H_UF16 || dstFormat == DXB_FMT_BC6H_SF16);
    return DXB_S_OK;
}

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
        dxb_launch_bc6h(grid_for(jt.total, 2 * DXB_BC6H_WARPS, (uint32_t)d.gridBC6H * 4u), stream, jt.dev.d, jt.host.data(), P);
        return check_launch("k_compress_bc6h");
    }
    if (plan.bc7)
    {
        // RGBA32F sources of full blocks: persistent kernel fed by TMA tile loads; everything else: the direct kernel with one CTA
        // per 2 * DXB_BC7_WARPS blocks (no grid-stride cap): block costs differ (alpha blocks run the separate-alpha tasks), so the
        // hardware CTA scheduler balances better than a static stride
        if (dxb_launch_bc7_tma((unsigned)d.gridBC7, stream, jt.host.data(), P)) g_tma_launches.fetch_add(1, std::memory_order_relaxed);
        else dxb_launch_bc7(grid_for(jt.total, 2 * DXB_BC7_WARPS, UINT32_MAX), stream, jt.dev.d, jt.host.data(), P);
        return check_launch("k_compress_bc7");
    }
    dxb_launch_bc15(grid_for(jt.total, 128, (uint32_t)d.gridBC15 * 4u), stream, jt.dev.d, jt.host.data(), P);
    return check_launch("k_compress_bc15");
}

// ---- host staging -------------------------------------------------------------------------------------
// How one image of a staged item travels: its host pixels go up before the launch, its device result comes back after the
// launch, or its bytes are only reserved in device memory (the levels of a chain that is compressed where it is built).
enum class Copy : uint8_t { Up, Down, None };

// One array of images of a staged call: item i owns images [i * per, (i + 1) * per) of `host`; image 0 of an item travels as
// `first`, the others as `rest` (a mip chain uploads level 0 and makes the others).
struct Plane { const dxb200_image* host; size_t per; Copy first, rest; };

// Stages items [0, n) of the planes through the calling thread's lane.  Whole items are grouped into chunks of at most `budget`
// bytes of device memory (an item larger than that is a chunk by itself), and chunk c goes through slot c % NSLOT, so the H2D
// copies, kernels and D2H copies of consecutive chunks overlap (fully when the caller's memory is pinned, see
// dxb200_host_alloc).  In the slot's buffer the chunk's images lie plane after plane, each on a 256-byte boundary, so equal
// images of one plane sit at a constant stride (the vector kernels' alignment checks and dxb_launch_bc7_tma rely on both).
// fn(dev, count, stream) enqueues the kernels: dev[p] is plane p's images of the chunk's `count` items, with device pointers.
// prog (optional) is told before each chunk's upload the units[] of the items the chunk completes, and stops the call between
// chunks (E_ABORT).  Every slot is synchronised before returning; the first error wins.
template <typename Fn>
int32_t run_staged(const Plane* planes, size_t nplanes, size_t n, size_t budget, Fn fn, Progress* prog = nullptr, const size_t* units = nullptr)
{
    auto padded = [](const dxb200_image& im) { return (im.slicePitch + 255) & ~size_t(255); };
    Lane& L = *t_v.lane;
    std::vector<std::vector<dxb200_image>> dev(nplanes);
    size_t i = 0; int slot = 0;
    int32_t hr = DXB_S_OK;
    while (i < n && hr == DXB_S_OK)
    {
        size_t bytes = 0, k = i;
        while (k < n)
        {
            size_t b = 0;
            for (size_t p = 0; p < nplanes; ++p)
                for (size_t m = k * planes[p].per; m < (k + 1) * planes[p].per; ++m) b += padded(planes[p].host[m]);
            if (k > i && bytes + b > budget) break;
            bytes += b; ++k;
        }
        cudaStream_t st = L.streams[slot];
        hr = cuda_hr(cudaStreamSynchronize(st), "slot sync"); if (hr) break;
        if (prog)
        {
            size_t add = 0;
            for (size_t m = i; m < k; ++m) add += units[m];
            if (!prog->report(add)) { hr = DXB_E_ABORT; break; }
        }
        hr = ensure_buffer(&L.buf[slot], &L.cap[slot], bytes); if (hr) break;
        size_t off = 0;
        for (size_t p = 0; p < nplanes && hr == DXB_S_OK; ++p)
        {
            const Plane& pl = planes[p];
            const dxb200_image* host = pl.host + i * pl.per;
            dev[p].assign(host, pl.host + k * pl.per);
            for (size_t m = 0; m < dev[p].size() && hr == DXB_S_OK; ++m)
            {
                dev[p][m].pixels = static_cast<uint8_t*>(L.buf[slot]) + off;
                off += padded(dev[p][m]);
                if ((m % pl.per ? pl.rest : pl.first) == Copy::Up)
                    hr = cuda_hr(cudaMemcpyAsync(dev[p][m].pixels, host[m].pixels, host[m].slicePitch, cudaMemcpyHostToDevice, st), "H2D");
            }
        }
        if (hr) break;
        hr = fn(dev.data(), k - i, st); if (hr) break;
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
    for (int s = 0; s < NSLOT; ++s)
    {
        const int32_t h2 = cuda_hr(cudaStreamSynchronize(L.streams[s]), "final sync");
        if (hr == DXB_S_OK) hr = h2;
    }
    return hr;
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
int32_t plan_convert(const dxb200_image* src, size_t n, uint32_t dstFormat, uint32_t filter, const dxb200_image* dst, dxb_convert_params* P)
{
    if (!src || !dst || !n) return DXB_E_INVALIDARG;
    const uint32_t srcFormat = src[0].format;
    // Convert/ConvertEx argument checks (DirectXTexConvert.cpp:5113-5125): same format, BC formats -> E_INVALIDARG
    if (srcFormat == dstFormat) return DXB_E_INVALIDARG;
    if (is_compressed(srcFormat) || is_compressed(dstFormat)) return DXB_E_INVALIDARG;
    if (!is_supported_pixel_format(srcFormat) || !is_supported_pixel_format(dstFormat)) return DXB_E_NOT_SUPPORTED;
    // TEX_FILTER_DITHER = ordered 4x4 dithering; TEX_FILTER_DITHER_DIFFUSION = Floyd-Steinberg (serial per image, :4815-4858)
    if (filter & (DXB_FILTER_DITHER_MASK & ~(DXB_FILTER_DITHER | DXB_FILTER_DITHER_DIFFUSION))) return DXB_E_NOT_SUPPORTED;
    // the 16-bit packed destinations have dithered stores in the reference (:4302-4500) that this backend does not restate yet
    if ((filter & DXB_FILTER_DITHER_MASK) && (dstFormat == DXB_FMT_B5G6R5_UNORM || dstFormat == DXB_FMT_B5G5R5A1_UNORM || dstFormat == DXB_FMT_B4G4R4A4_UNORM))
        return DXB_E_NOT_SUPPORTED;
    for (size_t i = 0; i < n; ++i)
    {
        if (!src[i].pixels || !dst[i].pixels) return DXB_E_POINTER;
        if (src[i].format != srcFormat || dst[i].format != dstFormat) return DXB_E_INVALIDARG;
        if (src[i].width != dst[i].width || src[i].height != dst[i].height) return DXB_E_FAIL;
        if ((uint64_t)src[i].width * src[i].height > 0x7FFFFFFFull) return DXB_E_INVALIDARG;
    }
    P->srcFormat = srcFormat; P->dstFormat = dstFormat;
    P->inF = dxb_convert_flags(srcFormat); P->outF = dxb_convert_flags(dstFormat);
    P->flags = dxb_resolve_srgb_convert(filter, srcFormat, dstFormat);
    P->threshold = 0.5f;
    return DXB_S_OK;
}

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
        dxb_launch_convert_diffuse(stream, (n > 1) ? jt.dev.d : nullptr, jt.host.data(), P, dErr, errStride);
        hr = check_launch("k_convert_diffuse");
        cudaFreeAsync(dErr, stream);
        return hr;
    }
    dxb_launch_convert(grid_for(jt.total, 256, (uint32_t)t_v.dev->gridRow * 8u), stream, jt.dev.d, jt.host.data(), P);
    return check_launch("k_convert");
}

// ---- PremultiplyAlpha ---------------------------------------------------------------------------
int32_t plan_pmalpha(const dxb200_image* src, size_t n, uint32_t flags, const dxb200_image* dst, dxb_convert_params* P)
{
    if (!src || !dst || !n) return DXB_E_INVALIDARG;
    const uint32_t fmt = src[0].format;
    if (is_compressed(fmt)) return DXB_E_NOT_SUPPORTED;                                 // :224-229
    if (!is_supported_pixel_format(fmt)) return DXB_E_NOT_SUPPORTED;
    if (!(dxb_convert_flags(fmt) & DXB_CONVF_A)) return DXB_E_NOT_SUPPORTED;            // !HasAlpha
    for (size_t i = 0; i < n; ++i)
    {
        if (!src[i].pixels || !dst[i].pixels) return DXB_E_POINTER;
        if (src[i].format != fmt || dst[i].format != fmt) return DXB_E_INVALIDARG;
        if (src[i].width != dst[i].width || src[i].height != dst[i].height || !src[i].width || !src[i].height) return DXB_E_INVALIDARG;
    }
    memset(P, 0, sizeof(*P));
    P->srcFormat = fmt; P->dstFormat = fmt; P->inF = P->outF = dxb_convert_flags(fmt);
    // TEX_PMALPHA_IGNORE_SRGB = 0x1, TEX_PMALPHA_REVERSE = 0x2; the SRGB bits equal TEX_FILTER_SRGB_IN/OUT (:21-26)
    const uint32_t lflags = (flags & 0x1u) ? 0u : dxb_resolve_srgb_linear(flags & DXB_FILTER_SRGB_MASK, fmt);
    P->flags = (lflags & (DXB_FILTER_SRGB_IN | DXB_FILTER_SRGB_OUT)) | ((flags & 0x2u) ? 1u : 0u);
    return DXB_S_OK;
}

int32_t launch_pmalpha(dxb_convert_params P, const dxb200_image* src, const dxb200_image* dst, size_t n, cudaStream_t stream)
{
    JobTable jt;
    const int32_t hr = jt.build(src, dst, n, false, stream);
    if (hr != DXB_S_OK) return hr;
    P.totalUnits = jt.total; P.njobs = (uint32_t)n;
    dxb_launch_pmalpha(grid_for(jt.total, 256, (uint32_t)t_v.dev->gridRow * 8u), stream, jt.dev.d, jt.host.data(), P);
    return check_launch("k_pmalpha");
}

// ---- GenerateMipMaps ----------------------------------------------------------------------------
bool ispow2(size_t x) { return ((x != 0) && !(x & (x - 1))); }

int32_t plan_mips(const dxb200_image* chain, size_t items, size_t levels, uint32_t filter, uint32_t* mode)
{
    if (!chain || !items || levels < 2) return DXB_E_INVALIDARG;
    const uint32_t fmt = chain[0].format;
    if (is_compressed(fmt)) return DXB_E_NOT_SUPPORTED;                         // GenerateMipMaps :2852-2856
    if (!is_supported_pixel_format(fmt)) return DXB_E_NOT_SUPPORTED;
    const size_t w = chain[0].width, h = chain[0].height;
    if (levels > count_mips(w, h)) return DXB_E_INVALIDARG;
    for (size_t it = 0; it < items; ++it)
    {
        size_t lw = w, lh = h;
        for (size_t l = 0; l < levels; ++l)
        {
            const dxb200_image& im = chain[it * levels + l];
            if (!im.pixels) return DXB_E_POINTER;
            if (im.format != fmt || im.width != lw || im.height != lh) return DXB_E_INVALIDARG;
            if (lh > 1) lh >>= 1;
            if (lw > 1) lw >>= 1;
        }
    }
    uint32_t m = filter & DXB_FILTER_MODE_MASK;
    if (!m) m = (ispow2(w) && ispow2(h)) ? DXB_FILTER_BOX : DXB_FILTER_LINEAR;   // :3169-3174
    switch (m)
    {
    case DXB_FILTER_BOX: if (!ispow2(w) || !ispow2(h)) return DXB_E_FAIL; break;     // :1005-1006
    case DXB_FILTER_POINT: case DXB_FILTER_LINEAR: case DXB_FILTER_CUBIC: case DXB_FILTER_TRIANGLE: break;
    default: return DXB_E_NOT_SUPPORTED;
    }
    if ((uint64_t)w * h * items > 0x7FFFFFFFull) return DXB_E_INVALIDARG;
    *mode = m;
    return DXB_S_OK;
}

// Resize = one filter pass from src[i] to dst[i] (PerformResizeUsingCustomFilters, DirectXTexResize.cpp:805-837)
int32_t plan_resize(const dxb200_image* src, size_t n, uint32_t filter, const dxb200_image* dst, uint32_t* mode)
{
    if (!src || !dst || !n) return DXB_E_INVALIDARG;
    const uint32_t fmt = src[0].format;
    if (is_compressed(fmt)) return DXB_E_NOT_SUPPORTED;                         // Resize :875-879
    if (!is_supported_pixel_format(fmt)) return DXB_E_NOT_SUPPORTED;
    const size_t sw = src[0].width, sh = src[0].height, dw = dst[0].width, dh = dst[0].height;
    if (!sw || !sh || !dw || !dh) return DXB_E_INVALIDARG;
    if (sw > 0xFFFFFFFFull || sh > 0xFFFFFFFFull || dw > 0xFFFFFFFFull || dh > 0xFFFFFFFFull) return DXB_E_INVALIDARG;
    for (size_t i = 0; i < n; ++i)
    {
        if (!src[i].pixels || !dst[i].pixels) return DXB_E_POINTER;
        if (src[i].format != fmt || dst[i].format != fmt) return DXB_E_INVALIDARG;
        if (src[i].width != sw || src[i].height != sh || dst[i].width != dw || dst[i].height != dh) return DXB_E_INVALIDARG;
    }
    uint32_t m = filter & DXB_FILTER_MODE_MASK;
    if (!m) m = ((dw << 1) == sw && (dh << 1) == sh) ? DXB_FILTER_BOX : DXB_FILTER_LINEAR;      // :812-817
    switch (m)
    {
    case DXB_FILTER_BOX: if ((dw << 1) != sw || (dh << 1) != sh) return DXB_E_FAIL; break;      // :318-319
    case DXB_FILTER_POINT: case DXB_FILTER_LINEAR: case DXB_FILTER_CUBIC: case DXB_FILTER_TRIANGLE: break;
    default: return DXB_E_NOT_SUPPORTED;
    }
    if ((uint64_t)dw * dh * n > 0x7FFFFFFFull) return DXB_E_INVALIDARG;
    *mode = m;
    return DXB_S_OK;
}

// chain[] holds DEVICE pointers; level 0 of each item is populated
int32_t launch_mips(const dxb200_image* chain, size_t items, size_t levels, uint32_t filter, uint32_t mode, cudaStream_t stream)
{
    const uint32_t fmt = chain[0].format;
    dxb_mip_params P; memset(&P, 0, sizeof(P));
    P.format = fmt; P.mode = mode; P.filter = filter;
    P.lflags = dxb_resolve_srgb_linear(filter & DXB_FILTER_SRGB_MASK, fmt);
    // job records of every level, built once and uploaded with ONE copy (a per-level upload left the GPU idle
    // between the small launches of the tail of the chain)
    std::vector<const dxb200_image*> stale(items, nullptr);
    std::vector<dxb_mip_job> all(items * (levels - 1));
    for (size_t l = 1; l < levels; ++l)
    {
        uint64_t total = 0;
        for (size_t it = 0; it < items; ++it)
        {
            const dxb200_image& s = chain[it * levels + l - 1]; const dxb200_image& d = chain[it * levels + l];
            dxb_mip_job& j = all[(l - 1) * items + it];
            j.src = s.pixels; j.dst = d.pixels; j.srcPitch = s.rowPitch; j.dstPitch = d.rowPitch;
            j.sw = (uint32_t)s.width; j.sh = (uint32_t)s.height; j.dw = (uint32_t)d.width; j.dh = (uint32_t)d.height;
            j.firstUnit = (uint32_t)total; total += (uint64_t)j.dw * j.dh;
            if (s.height == 2) stale[it] = &s;          // box filter quirk, see dxb_mip_box
            j.stale = nullptr; j.stalePitch = 0;
            if (mode == DXB_FILTER_BOX && s.height <= 1 && s.width > 1 && stale[it])
            {
                j.stale = stale[it]->pixels + stale[it]->rowPitch;      // row 1 of that level
                j.stalePitch = stale[it]->rowPitch;
            }
        }
    }
    // TRIANGLE's gather lists, X and Y of every level (shared by all items), travel in the same copy after the records
    std::vector<TriLists> tri(mode == DXB_FILTER_TRIANGLE ? 2 * (levels - 1) : 0);
    size_t bytes = all.size() * sizeof(dxb_mip_job);
    for (size_t l = 1; l <= tri.size() / 2; ++l)
    {
        build_triangle_axis(chain[l - 1].width, chain[l].width, (filter & DXB_FILTER_WRAP_U) != 0, tri[2 * (l - 1)]);
        build_triangle_axis(chain[l - 1].height, chain[l].height, (filter & DXB_FILTER_WRAP_V) != 0, tri[2 * (l - 1) + 1]);
    }
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
    const int32_t hr = dxb_launch_mip_chain(stream, reinterpret_cast<const dxb_mip_job*>(dev), all.data(), (uint32_t)items, (uint32_t)levels, P,
                                            tri.empty() ? nullptr : axes.data(), (unsigned)t_v.dev->gridRow * 8u, g_mip_kernels.load() == 1,
                                            check_launch);
    if (dev) cudaFreeAsync(dev, stream);
    return hr;
}

} // namespace

// =================================================================================================
extern "C" {

const char* dxb200_version(void) { return "dxtex_b200 0.1 (sm_90a)"; }
const char* dxb200_last_error(void) { return t_lastError.c_str(); }
uint64_t dxb200_launch_count(void) { return g_launches.load(); }
uint64_t dxb200_tma_launch_count(void) { return g_tma_launches.load(); }
uint64_t dxb200_kernel_launch_count(const char* kernel)
{
    if (!kernel) return 0;
    std::lock_guard<std::mutex> lk(g_count_mu);
    const auto it = g_kernel_launches.find(kernel);
    return it == g_kernel_launches.end() ? 0 : it->second;
}
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
static int32_t plan_decompress(const dxb200_image* src, size_t n, uint32_t dstFormat, const dxb200_image* dst, dxb_compress_params* P)
{
    if (!src || !dst || !n) return DXB_E_INVALIDARG;
    const uint32_t srcFormat = src[0].format;
    if (!is_compressed(srcFormat) || is_compressed(dstFormat)) return DXB_E_INVALIDARG;
    if (!is_supported_pixel_format(dstFormat)) return DXB_E_NOT_SUPPORTED;
    for (size_t i = 0; i < n; ++i)
    {
        if (!src[i].pixels || !dst[i].pixels) return DXB_E_POINTER;
        if (src[i].format != srcFormat || dst[i].format != dstFormat) return DXB_E_INVALIDARG;
        if (src[i].width != dst[i].width || src[i].height != dst[i].height) return DXB_E_FAIL;
        if (!src[i].width || !src[i].height || src[i].width > 0xFFFFFFFFull || src[i].height > 0xFFFFFFFFull) return DXB_E_INVALIDARG;
    }
    memset(P, 0, sizeof(*P));
    P->srcFormat = srcFormat; P->dstFormat = dstFormat;
    P->inF = dxb_convert_flags(srcFormat); P->outF = dxb_convert_flags(dstFormat);
    P->cflags = dxb_resolve_srgb_convert(0, srcFormat, dstFormat);          // ConvertScanline(..., TEX_FILTER_DEFAULT) (:500)
    return DXB_S_OK;
}

static int32_t launch_decompress(dxb_compress_params P, const dxb200_image* src, const dxb200_image* dst, size_t n, cudaStream_t stream)
{
    JobTable jt;
    const int32_t hr = jt.build(src, dst, n, true, stream);
    if (hr != DXB_S_OK) return hr;
    P.totalUnits = jt.total; P.njobs = (uint32_t)n;
    dxb_launch_decompress(grid_for(jt.total, 128, (uint32_t)t_v.dev->gridBC15 * 8u), stream, jt.dev.d, jt.host.data(), P);
    return check_launch("k_decompress");
}

int32_t dxb200_decompress_device(const dxb200_image* src, size_t nimages, uint32_t dstFormat, const dxb200_image* dst, void* stream)
{
    dxb_compress_params P;
    int32_t hr = plan_decompress(src, nimages, dstFormat, dst, &P);
    if (hr != DXB_S_OK) return hr;
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

// ---- GenerateMipMaps + Compress in one call: the mip chain never leaves HBM --------------------------------------------
// texconv runs GenerateMipMaps and then Compress on the result (Texconv/texconv.cpp; SURVEY 3.5); with the two host-pointer calls
// the chain travels device -> host -> device in between.  Here level 0 of every item goes up once, the chain is built and
// compressed in device memory, and only the packed blocks come back: 4 B/texel up + 1.33 B/texel down (BC3 from RGBA8)
// instead of 4 + 5.33 + 5.33 + 1.33.  Per item: base[i] = level 0 (host), dst[i * levels + l] = the BC image of level l (host).
// Chunks of whole items are pipelined over the lane's NSLOT (stream, buffer) slots: H2D, mip kernels, compress kernel, D2H.
int32_t dxb200_mipmaps_compress(const dxb200_image* base, size_t items, size_t levels, uint32_t filter, uint32_t dstFormat,
                                uint32_t flags, float threshold, float alphaWeight, const dxb200_image* dst)
{
    (void)alphaWeight;
    if (!base || !dst || !items || !levels) return DXB_E_INVALIDARG;
    // the chain every item will have on the device (ScratchImage layout of the source format)
    std::vector<dxb200_image> chain(items * levels);
    for (size_t i = 0; i < items; ++i)
    {
        size_t w = base[i].width, h = base[i].height;
        if (!base[i].pixels) return DXB_E_POINTER;
        if (levels > count_mips(w, h)) return DXB_E_INVALIDARG;
        for (size_t l = 0; l < levels; ++l)
        {
            dxb200_image& c = chain[i * levels + l];
            c.width = w; c.height = h; c.format = base[i].format;
            const int32_t hp = compute_pitch(c.format, w, h, &c.rowPitch, &c.slicePitch);
            if (hp != DXB_S_OK) return hp;
            c.pixels = const_cast<uint8_t*>(base[i].pixels);          // level 0's upload source; the other levels only need it for validation
            if (h > 1) h >>= 1;
            if (w > 1) w >>= 1;
        }
        chain[i * levels].rowPitch = base[i].rowPitch; chain[i * levels].slicePitch = base[i].slicePitch;
    }
    uint32_t mode = 0;
    int32_t hr = plan_mips(chain.data(), items, levels, filter, &mode);
    if (hr != DXB_S_OK) return hr;
    CompressPlan plan;
    hr = plan_compress(chain.data(), items * levels, dstFormat, flags, threshold, dst, &plan);
    if (hr != DXB_S_OK) return hr;
    return run_sharded(items, [&](size_t i) { return base[i].slicePitch; },
        [&](size_t lo, size_t hi)
        {
            const Plane planes[2] = { { chain.data() + lo * levels, levels, Copy::Up, Copy::None }, { dst + lo * levels, levels, Copy::Down, Copy::Down } };
            return run_staged(planes, 2, hi - lo, ITEM_CHUNK,
                [&](const std::vector<dxb200_image>* dev, size_t cnt, cudaStream_t st)
                {
                    const int32_t h2 = launch_mips(dev[0].data(), cnt, levels, filter, mode, st);
                    return h2 != DXB_S_OK ? h2 : launch_compress(plan, dev[0].data(), dev[1].data(), cnt * levels, st);
                });
        });
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

// ---- ScaleMipMapsAlphaForCoverage ----------------------------------------------------------------
static int32_t plan_alpha_coverage(const dxb200_image* src, size_t n, const dxb200_image* dst)
{
    if (!src || !dst || !n) return DXB_E_INVALIDARG;
    const uint32_t fmt = src[0].format;
    if (is_compressed(fmt)) return DXB_E_NOT_SUPPORTED;                         // :3495-3497
    if (!is_supported_pixel_format(fmt)) return DXB_E_NOT_SUPPORTED;
    for (size_t i = 0; i < n; ++i)
    {
        if (!src[i].pixels || !dst[i].pixels) return DXB_E_POINTER;
        if (src[i].format != fmt || dst[i].format != fmt) return DXB_E_INVALIDARG;
        if (src[i].width != dst[i].width || src[i].height != dst[i].height || !src[i].width || !src[i].height) return DXB_E_INVALIDARG;
        if ((uint64_t)src[i].width * src[i].height > 0x7FFFFFFFull) return DXB_E_INVALIDARG;
    }
    return DXB_S_OK;
}

// device pointers; count = device scratch (8 bytes).  Mirrors CalculateAlphaCoverage / EstimateAlphaScaleForCoverage.
static int32_t alpha_coverage_device(const dxb200_image& img, float ref, float scale, unsigned long long* dCount, cudaStream_t st, float* coverage)
{
    *coverage = 0.0f;
    if (img.width < 2 || img.height < 2) return DXB_S_OK;                      // no 2x2 cell: the reference's loops do not run
    dxb_job j; memset(&j, 0, sizeof(j));
    j.src = img.pixels; j.srcPitch = img.rowPitch; j.width = (uint32_t)img.width; j.height = (uint32_t)img.height;
    DXB_CUDA(cudaMemsetAsync(dCount, 0, sizeof(unsigned long long), st));
    const uint64_t cells = (uint64_t)(img.width - 1) * (img.height - 1);
    const uint32_t grid = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((cells + 255) / 256, (uint64_t)t_v.dev->gridRow * 8u));
    dxb_launch_alpha_coverage(grid, st, j, img.format, scale, ref, dCount);
    int32_t hr = check_launch("k_alpha_coverage");
    if (hr != DXB_S_OK) return hr;
    unsigned long long hCount = 0;
    DXB_CUDA(cudaMemcpyAsync(&hCount, dCount, sizeof(hCount), cudaMemcpyDeviceToHost, st));
    DXB_CUDA(cudaStreamSynchronize(st));
    const float cscale = static_cast<float>((img.width - 1) * (img.height - 1) * 8 * 8);          // :300-304
    if (cscale > 0.0f) *coverage = static_cast<float>(hCount) / cscale;
    return DXB_S_OK;
}

static int32_t scale_alpha_for_coverage_device(const dxb200_image* src, size_t n, float ref, const dxb200_image* dst, cudaStream_t st)
{
    unsigned long long* dCount = nullptr;
    DXB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&dCount), sizeof(unsigned long long), st));
    float target = 0.0f;
    int32_t hr = alpha_coverage_device(src[0], ref, 1.0f, dCount, st, &target);
    // base level: plain copy (:3511-3530)
    if (hr == DXB_S_OK)
        hr = cuda_hr(cudaMemcpy2DAsync(dst[0].pixels, dst[0].rowPitch, src[0].pixels, src[0].rowPitch, std::min(src[0].rowPitch, dst[0].rowPitch),
                                       src[0].slicePitch / std::max<size_t>(src[0].rowPitch, 1), cudaMemcpyDeviceToDevice, st), "copy base level");
    for (size_t l = 1; l < n && hr == DXB_S_OK; ++l)
    {
        // EstimateAlphaScaleForCoverage (:310-355): bisection on [0, 4], at most 10 coverage evaluations
        float lo = 0.0f, hi = 4.0f, scale = 1.0f;
        for (int it = 0; it < 10 && hr == DXB_S_OK; ++it)
        {
            float cov = 0.0f;
            hr = alpha_coverage_device(src[l], ref, scale, dCount, st, &cov);
            if (hr != DXB_S_OK) break;
            if (cov < target) lo = scale;
            else if (cov > target) hi = scale;
            else break;
            scale = (lo + hi) * 0.5f;
        }
        if (hr != DXB_S_OK) break;
        dxb_job j; memset(&j, 0, sizeof(j));
        j.src = src[l].pixels; j.dst = dst[l].pixels; j.srcPitch = src[l].rowPitch; j.dstPitch = dst[l].rowPitch;
        j.width = (uint32_t)src[l].width; j.height = (uint32_t)src[l].height;
        const uint64_t px = (uint64_t)j.width * j.height;
        const uint32_t grid = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((px + 255) / 256, (uint64_t)t_v.dev->gridRow * 8u));
        dxb_launch_scale_alpha(grid, st, j, src[l].format, scale);
        hr = check_launch("k_scale_alpha");
    }
    cudaFreeAsync(dCount, st);
    return hr;
}

int32_t dxb200_scale_mipmaps_alpha_for_coverage_device(const dxb200_image* src, size_t nlevels, float alphaReference, const dxb200_image* dst, void* stream)
{
    int32_t hr = plan_alpha_coverage(src, nlevels, dst);
    if (hr != DXB_S_OK) return hr;
    DevScope scope;
    hr = scope.enter(src[0].pixels);
    if (hr != DXB_S_OK) return hr;
    return scale_alpha_for_coverage_device(src, nlevels, alphaReference, dst, static_cast<cudaStream_t>(stream));
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

// a resize is a two-"level" chain per item whose second level has an arbitrary size
static int32_t launch_resize(const dxb200_image* src, const dxb200_image* dst, size_t n, uint32_t filter, uint32_t mode, cudaStream_t stream)
{
    std::vector<dxb200_image> pairs(2 * n);
    for (size_t i = 0; i < n; ++i) { pairs[2 * i] = src[i]; pairs[2 * i + 1] = dst[i]; }
    return launch_mips(pairs.data(), n, 2, filter, mode, stream);
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
