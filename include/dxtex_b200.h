/* dxtex_b200.h — C ABI of libdxtex_b200.so, the H100 (sm_90a) backend for the DirectXTex hot path:
 * DirectX::Compress / Decompress-side block codecs, DirectX::Convert, DirectX::GenerateMipMaps.
 *
 * Every entry point names the reference interface it replaces (paths relative to the reference
 * repository microsoft/DirectXTex @ 0bb96f0).  The design precedent inside the reference for an
 * accelerator boundary at per-image granularity is GPUCompressBC::{Initialize,Prepare,Compress}
 * (DirectXTex/BCDirectCompute.cpp:109, 203, 373), used by DirectX::Compress(ID3D11Device*, ...)
 * (DirectXTex/DirectXTexCompressGPU.cpp:249-319).
 *
 * Conventions
 *   - plain C: pointers + sizes, no C++/torch types; all functions return an HRESULT bit pattern
 *     (S_OK = 0; E_INVALIDARG, E_POINTER, E_OUTOFMEMORY, E_FAIL, HRESULT_E_NOT_SUPPORTED as in
 *     DirectXTexP.h:210-234 / SURVEY.md 8(b)).  CUDA failures map to E_FAIL / E_OUTOFMEMORY.
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails with E_FAIL,
 *     and format pairs the kernels do not implement fail with HRESULT_E_NOT_SUPPORTED.
 *   - `dxb200_image` mirrors DirectX::Image (DirectXTex/DirectXTex.h:437-445) field for field.
 *   - the host-pointer entry points never allocate caller-visible memory: the caller sizes the
 *     destination exactly as ScratchImage::Initialize2D would (DirectXTexImage.cpp:405-455; pitches
 *     from dxb200_compute_pitch == ComputePitch, DirectXTexUtil.cpp:961-1183) and the call fills it.
 *   - `_device` variants take device pointers in the same struct and a CUstream/cudaStream_t
 *     (as void*, may be NULL for the default stream); they only enqueue work.
 *   - thread safety: entry points may be called concurrently from several host threads; each host-pointer call takes one of a
 *     device's two staging lanes (own streams and buffers), so two calls per device really overlap; more wait.
 */
#ifndef DXTEX_B200_H
#define DXTEX_B200_H

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define DXB200_API __attribute__((visibility("default")))
#else
#define DXB200_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dxb200_image
{
    size_t   width;
    size_t   height;
    uint32_t format;      /* DXGI_FORMAT value */
    size_t   rowPitch;
    size_t   slicePitch;
    uint8_t* pixels;
} dxb200_image;

/* library / device management (GPUCompressBC::Initialize, BCDirectCompute.cpp:109) */
DXB200_API const char* dxb200_version(void);
DXB200_API int32_t  dxb200_init(int device);                 /* = dxb200_init_devices(1, &device); idempotent */
/* Multi-GPU inside the library (SURVEY.md 8(b), 8(e); the reference parallelises inside the call too: CompressBC_Parallel,
 * DirectXTexCompress.cpp:210-372).  After dxb200_init_devices(n, devs) every host-pointer entry point shards its work over
 * the n devices: contiguous ranges of images (array calls, mip chains: a chain never spans devices) or of block-row bands
 * (one large image), one host thread and one stream set per device, no collective.  `_device` variants always run on the
 * device that owns the caller's pointers.  Devices can be added by further calls; idempotent per device. */
DXB200_API int32_t  dxb200_init_devices(int ndev, const int* devices);
DXB200_API int32_t  dxb200_initialized_devices(int* devices, int maxDevices);   /* returns how many are initialised */
DXB200_API void     dxb200_shutdown(void);                   /* release cached device / pinned buffers */
DXB200_API int32_t  dxb200_device_count(void);
DXB200_API uint64_t dxb200_launch_count(void);               /* number of kernels this library has launched so far */
DXB200_API uint64_t dxb200_tma_launch_count(void);           /* ... of which fed by TMA tensor-map tile loads (k_compress_bc7_tma) */
/* ... of which launched the __global__ function `kernel`, named without template arguments (e.g. "k_compress_bc15_t" and
 * "k_compress_bc15", "k_compress_bc7_tma" and the direct "k_compress_bc7", "k_convert_vec", "k_mip_box3", "k_mip_level");
 * 0 for a name that never ran.  Lets a caller or a test see which route a call took. */
DXB200_API uint64_t dxb200_kernel_launch_count(const char* kernel);
/* process-wide tuning options (no reference counterpart; results never depend on them).
 *   DXB200_OPT_BC7_FEED  how k_compress_bc7 gets RGBA32F sources made of full blocks: 0 = direct vector loads, one CTA per 16 blocks,
 *                        1 = persistent CTAs fed by TMA tensor-map tile loads with an atomic tile counter, 2 = the same with statically
 *                        strided tiles, 3 = TMA with one CTA per tile, 4 = automatic (default): 1 for batches of images, 0 for a single
 *                        image -- whichever measured faster.  Initial value: environment variable DXB200_BC7_TMA.
 *   DXB200_OPT_MIP_KERNELS  which kernels GenerateMipMaps / Resize levels run on: 0 (default) = the specialised kernels where they apply
 *                        (k_mip_box3, k_mip_tail, k_mip_sep, k_mip_tile), 1 = every level on the generic k_mip_level, so that the
 *                        specialised routes can be checked against it; any other value means 0. */
#define DXB200_OPT_BC7_FEED 1u
#define DXB200_OPT_MIP_KERNELS 2u
DXB200_API int32_t  dxb200_set_option(uint32_t option, int32_t value);      /* E_INVALIDARG for an unknown option */
DXB200_API int32_t  dxb200_get_option(uint32_t option);                     /* -1 for an unknown option */
DXB200_API const char* dxb200_last_error(void);              /* text of the last CUDA error seen by the calling thread's call */

/* pinned host allocations for callers that want full-rate H2D/D2H (optional; any host pointer works) */
DXB200_API void*    dxb200_host_alloc(size_t bytes);
DXB200_API void     dxb200_host_free(void* p);

/* ComputePitch (DirectXTexUtil.cpp:961-1183), CP_FLAGS_NONE, for the implemented formats */
DXB200_API int32_t  dxb200_compute_pitch(uint32_t format, size_t width, size_t height, size_t* rowPitch, size_t* slicePitch);
/* CalculateMipLevels (DirectXTexMipmaps.cpp:359-380): *levels==0 -> full chain */
DXB200_API int32_t  dxb200_calculate_mip_levels(size_t width, size_t height, size_t* levels);

/* DirectX::Compress / CompressEx, single image and array overloads
 * (DirectXTexCompress.cpp:632-845; block walk CompressBC :72-205).
 *   flags     = TEX_COMPRESS_FLAGS (DirectXTex.h:887-917); TEX_COMPRESS_PARALLEL is accepted and ignored
 *   threshold = BC1 alpha threshold (TEX_THRESHOLD_DEFAULT 0.5)
 * src[i] and dst[i] must have equal width/height; dst[i].format == dstFormat, pitches per dxb200_compute_pitch.
 * The row pitch of a BC image (the destination here, the source of a decompress) must be a multiple of its block size (8 bytes
 * for BC1 / BC4, 16 for the others), and so must its pixel pointer in the _device variants: the kernels move whole blocks.
 * Other layouts are refused with E_INVALIDARG. */
DXB200_API int32_t  dxb200_compress(const dxb200_image* src, size_t nimages, uint32_t dstFormat,
                         uint32_t flags, float threshold, float alphaWeight, const dxb200_image* dst);
DXB200_API int32_t  dxb200_compress_device(const dxb200_image* src, size_t nimages, uint32_t dstFormat,
                                uint32_t flags, float threshold, float alphaWeight, const dxb200_image* dst, void* stream);
/* CompressEx / ConvertEx status callback (DirectXTex.h:929-944; DirectXTexCompress.cpp:115-121, 356-360, 785-837): called with
 * (done, total) before every chunk of bands goes to the device -- pixel rows of a single image, images of an array, done
 * before that chunk (a chunk holds whole bands of work rows, about 48 MiB of source and destination) -- and with (total, total)
 * at the end; returning 0 stops the call between chunks with E_ABORT (0x80004004).  With several devices each device reports
 * its own chunks, so the values need not rise; the callback is serialised but may come from worker threads. */
typedef int (*dxb200_status_fn)(size_t done, size_t total, void* user);
DXB200_API int32_t  dxb200_compress_ex(const dxb200_image* src, size_t nimages, uint32_t dstFormat, uint32_t flags, float threshold,
                            float alphaWeight, const dxb200_image* dst, dxb200_status_fn status, void* user);

/* DirectX::Decompress (DirectXTexCompress.cpp:852-979; DecompressBC :425-535) */
DXB200_API int32_t  dxb200_decompress(const dxb200_image* src, size_t nimages, uint32_t dstFormat, const dxb200_image* dst);
DXB200_API int32_t  dxb200_decompress_device(const dxb200_image* src, size_t nimages, uint32_t dstFormat, const dxb200_image* dst, void* stream);

/* DirectX::Convert / ConvertEx (DirectXTexConvert.cpp:5091-5404; ConvertCustom no-dither path :4888-4908).
 *   filter = TEX_FILTER_FLAGS; TEX_FILTER_DITHER = ordered dithering (StoreScanlineDither :4049-4567 without diffusion errors);
 *   TEX_FILTER_DITHER_DIFFUSION = Floyd-Steinberg error diffusion (serial per image; ConvertCustom :4815-4858) */
DXB200_API int32_t  dxb200_convert(const dxb200_image* src, size_t nimages, uint32_t dstFormat,
                        uint32_t filter, float threshold, const dxb200_image* dst);
DXB200_API int32_t  dxb200_convert_device(const dxb200_image* src, size_t nimages, uint32_t dstFormat,
                               uint32_t filter, float threshold, const dxb200_image* dst, void* stream);
DXB200_API int32_t  dxb200_convert_ex(const dxb200_image* src, size_t nimages, uint32_t dstFormat, uint32_t filter, float threshold,
                           const dxb200_image* dst, dxb200_status_fn status, void* user);

/* DirectX::GenerateMipMaps (DirectXTexMipmaps.cpp:2828-3247; Generate2DMips{Point,Box,Linear,Cubic,Triangle}Filter :907-1602).
 *   chain = items*levels images laid out item-major, mip-minor (TexMetadata::ComputeIndex, DirectXTexUtil.cpp:1695-1741);
 *   level 0 of every item is filled by the caller, levels 1.. are written.
 *   filter = TEX_FILTER_FLAGS; mode 0 selects BOX for power-of-two sizes else LINEAR (:3169-3174). */
DXB200_API int32_t  dxb200_generate_mipmaps(const dxb200_image* chain, size_t items, size_t levels, uint32_t filter);
DXB200_API int32_t  dxb200_generate_mipmaps_device(const dxb200_image* chain, size_t items, size_t levels, uint32_t filter, void* stream);

/* GenerateMipMaps followed by Compress (what texconv does, Texconv/texconv.cpp -m / -f) as ONE call whose mip chain never leaves
 * HBM: base[i] = level 0 of item i (host), dst[i * levels + l] = the compressed image of level l of item i (host, sized by the
 * caller as ScratchImage::Initialize2D(dstFormat, w, h, items, levels) would).  Results are identical to
 * dxb200_generate_mipmaps + dxb200_compress (same kernels); host<->device traffic drops from (1 + 2 x 1.33) x source bytes up/down
 * to the source up and the blocks down.  filter as dxb200_generate_mipmaps, flags / threshold as dxb200_compress. */
DXB200_API int32_t  dxb200_mipmaps_compress(const dxb200_image* base, size_t items, size_t levels, uint32_t filter, uint32_t dstFormat,
                                 uint32_t flags, float threshold, float alphaWeight, const dxb200_image* dst);
/* The steps texconv runs between GenerateMipMaps and Compress, done in device memory by dxb200_mipmaps_compress_ex on every chain
 * after its mips and before its compression, in this order (Texconv/texconv.cpp:3480, 3526). */
typedef struct dxb200_chain_steps
{
    float    alphaReference;  /* > 0: ScaleMipMapsAlphaForCoverage of every item at this reference (texconv :3304, :3480); <= 0: skipped */
    uint32_t premultiply;     /* nonzero: PremultiplyAlpha of every image of every chain with pmalphaFlags (texconv :3526) */
    uint32_t pmalphaFlags;    /* TEX_PMALPHA_FLAGS, as dxb200_premultiply_alpha */
} dxb200_chain_steps;
/* dxb200_mipmaps_compress with `steps` (NULL: none, exactly dxb200_mipmaps_compress).  Results are identical to
 * dxb200_generate_mipmaps, then dxb200_scale_mipmaps_alpha_for_coverage per item, then dxb200_premultiply_alpha, then
 * dxb200_compress; every argument is checked before anything is uploaded, and the call returns the HRESULT of the first of those
 * four calls that would fail.  Each chunk of items runs the coverage search of all its chains as 10 + 1 kernel launches. */
DXB200_API int32_t  dxb200_mipmaps_compress_ex(const dxb200_image* base, size_t items, size_t levels, uint32_t filter,
                                               const dxb200_chain_steps* steps, uint32_t dstFormat, uint32_t flags,
                                               float threshold, float alphaWeight, const dxb200_image* dst);
/* texconv's steps in front of GenerateMipMaps, run in device memory by dxb200_mipmaps_compress_from on every item before its
 * mips, in this order: Decompress (Texconv/texconv.cpp:2316-2480), Resize (:2576-2643). */
typedef struct dxb200_chain_source
{
    uint32_t decompressFormat;  /* base in a BC format: Decompress it to this DXGI format first; 0 (UNKNOWN) = DefaultDecompress
                                   (DirectXTexCompress.cpp:377-421).  Ignored for an uncompressed base. */
    size_t   width, height;     /* level 0 of every chain; both 0 = the base's size.  A base of another size is Resized to it. */
    uint32_t resizeFilter;      /* TEX_FILTER_FLAGS of that Resize (texconv passes its mip filter flags) */
} dxb200_chain_source;
/* dxb200_mipmaps_compress_ex of items as they were loaded: base[i] = item i (host), BC or uncompressed, all items of one format
 * and one size; dst[i * levels + l] laid out as ScratchImage::Initialize2D(dstFormat, W, H, items, levels) would, W x H = the
 * chain's level 0.  Results are identical to dxb200_decompress (base -> decompressFormat, if the base is BC), then dxb200_resize
 * (-> W x H with resizeFilter, if the size differs), then dxb200_mipmaps_compress_ex; the decompressed and resized images
 * never leave device memory, so the base goes up and only the blocks come down.  Every argument of every step is checked before
 * anything is uploaded, and the call returns the HRESULT of the first of those calls that would fail.  source == NULL, or a
 * source that changes nothing, is exactly dxb200_mipmaps_compress_ex; only one of width / height 0 -> E_INVALIDARG. */
DXB200_API int32_t  dxb200_mipmaps_compress_from(const dxb200_image* base, size_t items, const dxb200_chain_source* source,
                                                 size_t levels, uint32_t filter, const dxb200_chain_steps* steps, uint32_t dstFormat,
                                                 uint32_t flags, float threshold, float alphaWeight, const dxb200_image* dst);
/* dxb200_mipmaps_compress_from that also answers texconv's next step, "set alpha mode" (Texconv/texconv.cpp:3738-3766):
 * alphaAllOpaque == NULL is exactly dxb200_mipmaps_compress_from; otherwise *alphaAllOpaque = 1 or 0, what
 * ScratchImage::IsAlphaAllOpaque() returns for the output (Initialize2D(dstFormat, W, H, items, levels) holding dst).  The blocks
 * are scanned where they were made, one launch per chunk after its compression, and the answer comes back with the blocks;
 * the blocks are identical to dxb200_mipmaps_compress_from's.  BC4, BC5 and BC6H outputs have no alpha: no scan, 1. */
DXB200_API int32_t  dxb200_mipmaps_compress_from_ex(const dxb200_image* base, size_t items, const dxb200_chain_source* source,
                                                    size_t levels, uint32_t filter, const dxb200_chain_steps* steps, uint32_t dstFormat,
                                                    uint32_t flags, float threshold, float alphaWeight, const dxb200_image* dst,
                                                    int32_t* alphaAllOpaque);

/* texconv's four channel steps between Resize and GenerateMipMaps, each a DirectX::TransformImage (DirectXTexMisc.cpp:606-760) of
 * the image in its own format, run in this order when enabled:
 *   swizzle        (-swizzle, Texconv/texconv.cpp:2645-2694): out[c] = in[swizzle[c]], then the channels of zeroMask (bit c =
 *                  channel c) become 0 and those of oneMask 1.  Enabled unless swizzle == {0, 1, 2, 3} and both masks are 0.
 *   colour key     (-c, :3134-3191): a pixel whose x, y and z each lie within 0.2 of the key colorKeyValue & 0xFFFFFF (0xRRGGBB,
 *                  loaded as an XMCOLOR) becomes (0, 0, 0, 0), every other pixel gets alpha 1.  texconv enables it only for a
 *                  format with alpha.
 *   invert Y       (-inverty, :3193-3240): y = 1 - y.
 *   reconstruct Z  (-reconstructz, :3242-3300): z = sqrt(1 - (x*x + y*y)), on x*2 - 1 and y*2 - 1 and mapped back by z*0.5 + 0.5
 *                  for a UNORM (or sRGB) format; x*x + y*y > 1 gives a NaN z, stored as the format stores a NaN.
 * Each step loads the pixel without an sRGB step and stores it at alpha threshold 0, so a step sees the previous one's stored
 * result (an 8-bit format is quantised between steps). */
typedef struct dxb200_channel_steps
{
    uint8_t  swizzle[4];        /* source channel (0..3) of each output channel */
    uint8_t  zeroMask, oneMask; /* bits 0..3: channels forced to 0, then channels forced to 1 */
    uint8_t  colorKey;          /* nonzero: the colour key step */
    uint8_t  invertY;           /* nonzero: the invert Y step */
    uint8_t  reconstructZ;      /* nonzero: the reconstruct Z step */
    uint32_t colorKeyValue;     /* the key, 0xRRGGBB (higher bits are ignored) */
} dxb200_channel_steps;
/* The enabled steps of `steps` on src[i] -> dst[i], i < n: every source has src[0]'s format, every destination its source's
 * format and size; dst may be src (same pixels and pitch).  HRESULTs, in TransformImage's order: src / dst / steps NULL or n == 0
 * -> E_INVALIDARG; a compressed, typeless, planar or palettized format, or one this library does not implement ->
 * E_NOT_SUPPORTED (0x80070032); src[0] wider or higher than 2^32 - 1 -> E_INVALIDARG; then per image a source of another format or
 * over 32 bits, or a destination of another format or size -> E_FAIL; no step enabled (image 0), a swizzle element above 3 or a
 * mask bit above bit 3 -> E_INVALIDARG; a NULL pixel pointer -> E_POINTER.  The host call stages the images in bands, sharded over
 * the initialised devices, as dxb200_convert does; the _device call enqueues on `stream` and returns. */
DXB200_API int32_t  dxb200_apply_channel_steps(const dxb200_image* src, size_t n, const dxb200_channel_steps* steps, const dxb200_image* dst);
DXB200_API int32_t  dxb200_apply_channel_steps_device(const dxb200_image* src, size_t n, const dxb200_channel_steps* steps,
                                                      const dxb200_image* dst, void* stream);
/* dxb200_mipmaps_compress_from_ex with texconv's channel steps between Resize and GenerateMipMaps (Texconv/texconv.cpp:2645-3300):
 * results identical to dxb200_decompress, dxb200_resize, dxb200_apply_channel_steps on level 0 and
 * dxb200_mipmaps_compress_from_ex.  The steps run in device memory, in place on every chain's level 0: one more k_convert launch
 * per chunk, no more memory.  With steps enabled and decompressFormat == 0, a BC4 / BC5 base decompresses to the format texconv
 * picks (:2393-2447): R8G8B8A8_UNORM (BC4_UNORM, BC5_UNORM) or R8G8B8A8_SNORM (the SNORM twins) when a step needs more channels
 * than R8 / R8G8 hold (BC4: invert Y, reconstruct Z, a swizzle or mask of channels 1-3; BC5: reconstruct Z, a swizzle or mask of
 * channels 2-3), else DefaultDecompress.  A failing call returns the HRESULT of the first of those calls that would fail, the
 * channel steps checked on level 0's format and size.  channels == NULL, or no step enabled, is exactly
 * dxb200_mipmaps_compress_from_ex. */
DXB200_API int32_t  dxb200_mipmaps_compress_from_channels(const dxb200_image* base, size_t items, const dxb200_chain_source* source,
                                                          const dxb200_channel_steps* channels, size_t levels, uint32_t filter,
                                                          const dxb200_chain_steps* steps, uint32_t dstFormat, uint32_t flags,
                                                          float threshold, float alphaWeight, const dxb200_image* dst,
                                                          int32_t* alphaAllOpaque);
/* texconv's path to an uncompressed target (-f R16G16B16A16_FLOAT, B8G8R8A8_UNORM, R8G8_SNORM, ...; Texconv/texconv.cpp:2316-3560)
 * in one call: base, source, channels, levels, filter, steps and alphaAllOpaque mean what they mean for
 * dxb200_mipmaps_compress_from_channels; dst[i * levels + l] = level l of item i in dstFormat, laid out as
 * ScratchImage::Initialize2D(dstFormat, W, H, items, levels) would; convertFilter and threshold are dxb200_convert's filter and
 * threshold.  Results are identical to this sequence of calls, each run only when it does something:
 *   1. dxb200_decompress of a BC base (when source != NULL), to the format dxb200_mipmaps_compress_from_channels picks;
 *   2. dxb200_resize, when the size changes;
 *   3. dxb200_apply_channel_steps with the swizzle and masks of channels, when they are enabled;
 *   4. dxb200_convert to dstFormat with convertFilter and threshold, when level 0's format differs from dstFormat (texconv tests
 *      info.format != tformat, :3100-3132);
 *   5. dxb200_apply_channel_steps with the colour key, invert Y and reconstruct Z of channels, now in dstFormat, when enabled;
 *   6. dxb200_generate_mipmaps of dst;
 *   7. dxb200_scale_mipmaps_alpha_for_coverage per item, when steps->alphaReference > 0;
 *   8. dxb200_premultiply_alpha of every level, when steps->premultiply;
 *   9. dxb200_is_alpha_all_opaque of dst, when alphaAllOpaque != NULL.
 * Every argument is checked before anything is uploaded, and a failing call returns the HRESULT of the first of those calls that
 * would fail, each checked on the format and size the image has at that point.  dst is met first by the Convert (its level 0:
 * another format -> E_INVALIDARG, another size -> E_FAIL), then by GenerateMipMaps (every level).  Without a Convert, dst's level 0
 * must have level 0's format and size (E_INVALIDARG) and non-NULL pixels (E_POINTER), the later channel steps are checked from
 * level 0 (the base itself when no front step runs) into dst's level 0, and GenerateMipMaps is checked on a chain whose level 0 is
 * that image, so a base of another format is E_INVALIDARG and NULL base pixels are E_POINTER there.  A BC dstFormat -> E_INVALIDARG
 * (Convert's answer); a dithered store to B5G6R5, B5G5R5A1 or B4G4R4A4 -> HRESULT_E_NOT_SUPPORTED, as dxb200_convert; levels < 2
 * -> E_INVALIDARG, GenerateMipMaps' answer, after the Convert's checks (levels == 0: the Convert is checked on dst[0]).  The intermediate images
 * never leave device memory: the base goes up and only the finished chain (every level) comes down.  Without a Convert, steps 3
 * and 5 run as one launch, with the same result. */
DXB200_API int32_t  dxb200_mipmaps_convert_from(const dxb200_image* base, size_t items, const dxb200_chain_source* source,
                                                const dxb200_channel_steps* channels, uint32_t dstFormat, uint32_t convertFilter,
                                                float threshold, size_t levels, uint32_t filter, const dxb200_chain_steps* steps,
                                                const dxb200_image* dst, int32_t* alphaAllOpaque);
/* texconv on textures that keep their own mip levels (no -m on an input with mips, Texconv/texconv.cpp:2270, or -m 1) in one call:
 * base[i * levels + l] = level l of item i as loaded (host), BC or uncompressed, every image of base[0]'s format; level sizes need
 * not halve.  dst[i * levels + l] = the same level of the result, laid out as ScratchImage::Initialize2D(dstFormat, W, H, items,
 * levels) would, each of its base's size (or the resized size when levels == 1).  source and channels mean what they mean for
 * dxb200_mipmaps_convert_from, convertFilter is dxb200_convert's filter, compressFlags dxb200_compress's flags and threshold both
 * calls' threshold.  Results are identical to this sequence of calls, each over all items * levels images as one array and each
 * run only when it does something:
 *   1. dxb200_decompress of a BC base, to source->decompressFormat (source == NULL or 0: the format
 *      dxb200_mipmaps_compress_from_channels picks);
 *   2. dxb200_resize to source->width x height with source->resizeFilter, only when levels == 1;
 *   3. dxb200_apply_channel_steps with the swizzle and masks of channels;
 *   4. dxb200_convert to dstFormat with convertFilter and threshold, for an uncompressed dstFormat other than the working format
 *      (texconv :3098);
 *   5. dxb200_apply_channel_steps with the colour key, invert Y and reconstruct Z of channels;
 *   6. dxb200_premultiply_alpha, when steps->premultiply;
 *   7. dxb200_compress into dst with compressFlags and threshold, for a BC dstFormat;
 *   8. dxb200_is_alpha_all_opaque of dst, when alphaAllOpaque != NULL.
 * A BC base whose dstFormat is exactly its own format (BC1_UNORM -> BC1_UNORM_SRGB re-encodes), with no channel step, no
 * premultiply and no resize, passes through as texconv passes it (:3621): dst takes the base's blocks and no decompress or
 * compress kernel runs (the Decompress is still checked, as texconv makes it first); an uncompressed base already in dstFormat
 * with nothing enabled is copied the same way.  Every argument is checked before anything is uploaded.  levels == 0, a size in
 * source that differs from the base's with levels > 1 (texconv's Resize drops the chain and regenerates it, which
 * dxb200_mipmaps_convert_from and dxb200_mipmaps_compress_from_channels do) and steps->alphaReference > 0 (-keepcoverage also
 * regenerates it) -> E_INVALIDARG, in that order; then a failing call returns the HRESULT of the first of the calls above that
 * would fail, each checked on the format and size every image has at that point.  Without a Convert, an uncompressed dst (or a
 * passed-through one) must have the working format and size, and a row pitch of whole blocks (E_INVALIDARG), and pixels
 * (E_POINTER).  A base that is only copied into dst (no decompress, resize, Convert or Compress) is checked last: a format this
 * library does not implement (R8G8B8A8_UINT, R16_UINT, ...) -> HRESULT_E_NOT_SUPPORTED, as every other call answers it; images of
 * other formats, a zero or over-32-bit width or height, or a BC row pitch of part blocks -> E_INVALIDARG; NULL pixels -> E_POINTER.
 * Steps 3 and 5 run as one launch when no Convert sits between them.  The base goes up once, every level of it;
 * only dst comes down. */
DXB200_API int32_t  dxb200_levels_from(const dxb200_image* base, size_t items, size_t levels, const dxb200_chain_source* source,
                                       const dxb200_channel_steps* channels, uint32_t dstFormat, uint32_t convertFilter,
                                       uint32_t compressFlags, float threshold, const dxb200_chain_steps* steps, const dxb200_image* dst,
                                       int32_t* alphaAllOpaque);

/* texconv steps that dxb200_chain_source / dxb200_channel_steps / dxb200_chain_steps do not hold */
typedef struct dxb200_texconv_steps
{
    uint32_t demultiply;       /* nonzero: -alpha: PremultiplyAlpha(TEX_PMALPHA_REVERSE | demultiplyFlags) after Decompress, before Resize */
    uint32_t demultiplyFlags;  /* TEX_PMALPHA_FLAGS (texconv passes its -srgb / -srgbi / -srgbo bits); REVERSE is implied */
    uint32_t bc3Layout;        /* 0 none; 1 DXT5nm / BC3n: (1, y, 0, x); 2 RXGB: (a, g, b, r); after premultiply, before Compress */
} dxb200_texconv_steps;
/* dxb200_mipmaps_compress_from_channels, dxb200_mipmaps_convert_from and dxb200_levels_from with texconv's -alpha
 * (Texconv/texconv.cpp:2483-2531) and -f BC3n / DXT5nm / RXGB (:452-456, 1510-1518, 3553-3617) steps.  ts == NULL, or all zeros, is
 * exactly the call without _ex (those calls are these with NULL).  The steps run in this order, each only when it does something:
 *   Decompress -> demultiply -> Resize -> swizzle / masks -> [Convert] -> colour key / invert Y / reconstruct Z -> GenerateMipMaps
 *   -> coverage -> premultiply -> BC3 layout -> Compress -> IsAlphaAllOpaque,
 * with results identical to the separate calls in that order:
 *   demultiply = dxb200_premultiply_alpha(0x2 REVERSE | ts->demultiplyFlags) of the working images: level 0 of every item for a
 *     generated chain, every level as loaded for dxb200_levels_from_ex;
 *   BC3 layout = dxb200_apply_channel_steps of every image of the chain, in the chain's format, with swizzle { 0, 1, 2, 0 },
 *     zeroMask 0x4 and oneMask 0x1 (DXT5nm) or swizzle { 3, 1, 2, 0 } (RXGB).  Save the RXGB result with DDS_FLAGS_FORCE_DXT5_RXGB.
 * With a layout and no decompress format, a BC4 or BC5 base decompresses to R8G8B8A8_UNORM (R8G8B8A8_SNORM for the SNORM twins), as
 * texconv picks it (:2404-2447).  texconv runs -alpha only on an image whose format has alpha and is not A8_UNORM and whose alpha
 * mode is premultiplied; the caller mirrors that guard.  Here a demultiply on a working format without alpha is PremultiplyAlpha's
 * HRESULT_E_NOT_SUPPORTED.  Every argument is checked before anything is uploaded: first ts's own rules, each E_INVALIDARG
 * (bc3Layout > 2; a layout with a dstFormat other than BC3_UNORM, as texconv asserts at :3556; any layout on
 * dxb200_mipmaps_convert_from_ex, which has no BC target), then the rules of the call without _ex, then the HRESULT of the first
 * separate call above that would fail, each checked on the format and size the image has at that point.  dxb200_levels_from_ex
 * passes no BC chain through when a demultiply or a layout runs (texconv drops the original image after both, :2529, :3616).
 * Neither step adds a staged image: one premultiply launch per chunk for the demultiply and one channel-steps launch per chunk for
 * the layout, both in place. */
DXB200_API int32_t  dxb200_mipmaps_compress_from_channels_ex(const dxb200_image* base, size_t items, const dxb200_chain_source* source,
                                                             const dxb200_channel_steps* channels, size_t levels, uint32_t filter,
                                                             const dxb200_chain_steps* steps, uint32_t dstFormat, uint32_t flags,
                                                             float threshold, float alphaWeight, const dxb200_image* dst,
                                                             int32_t* alphaAllOpaque, const dxb200_texconv_steps* ts);
DXB200_API int32_t  dxb200_mipmaps_convert_from_ex(const dxb200_image* base, size_t items, const dxb200_chain_source* source,
                                                   const dxb200_channel_steps* channels, uint32_t dstFormat, uint32_t convertFilter,
                                                   float threshold, size_t levels, uint32_t filter, const dxb200_chain_steps* steps,
                                                   const dxb200_image* dst, int32_t* alphaAllOpaque, const dxb200_texconv_steps* ts);
DXB200_API int32_t  dxb200_levels_from_ex(const dxb200_image* base, size_t items, size_t levels, const dxb200_chain_source* source,
                                          const dxb200_channel_steps* channels, uint32_t dstFormat, uint32_t convertFilter,
                                          uint32_t compressFlags, float threshold, const dxb200_chain_steps* steps, const dxb200_image* dst,
                                          int32_t* alphaAllOpaque, const dxb200_texconv_steps* ts);

/* One texture of dxb200_texconv_batch: the arguments of the one-call pipeline named by kind.
 *   kind 0 = dxb200_mipmaps_compress_from_channels_ex (compressFlags is its flags; convertFilter is not used),
 *   kind 1 = dxb200_mipmaps_convert_from_ex (compressFlags is not used),
 *   kind 2 = dxb200_levels_from_ex (filter is not used).
 * alphaWeight is not in the record: every one of those calls ignores it. */
typedef struct dxb200_texconv_job
{
    uint32_t kind;
    const dxb200_image* base; size_t items; size_t levels;
    const dxb200_chain_source* source; const dxb200_channel_steps* channels;
    uint32_t filter;            /* GenerateMipMaps' filter (kinds 0, 1) */
    const dxb200_chain_steps* steps; const dxb200_texconv_steps* ts;
    uint32_t dstFormat; uint32_t convertFilter; uint32_t compressFlags; float threshold;
    const dxb200_image* dst; int32_t* alphaAllOpaque;
} dxb200_texconv_job;
/* texconv over a list of textures of any sizes and formats in one call (texconv -r over a folder).  Job i's dst bytes and
 * *alphaAllOpaque are identical to what the call named by its kind writes with the same arguments.  Every job is planned, with that
 * call's own checks, before anything is uploaded; results[i] (when results != NULL) receives job i's HRESULT.  A job that fails its
 * checks does not run and its dst is not written; the other jobs still run.  The return value is S_OK or the HRESULT of the
 * lowest-index job that failed.  A device-side failure is returned and written into results[] of every job that was to run; their
 * dst is then undefined.  jobs == NULL or njobs == 0 -> E_INVALIDARG.  No job's dst may overlap another job's base or dst.
 * Jobs whose plans are equal apart from image pointers and row pitches (same kind, steps, formats, sizes and level counts) run as one
 * multi-item call would, their items in job order; the (job, item) units are split over the initialised devices in contiguous
 * ranges of about equal bytes, as every host call shards its items, and each device stages its share of every group through one
 * pipeline of chunks, so that one texture's upload overlaps the previous one's kernels. */
DXB200_API int32_t  dxb200_texconv_batch(const dxb200_texconv_job* jobs, size_t njobs, int32_t* results);
/* dxb200_texconv_batch on textures already in device memory: every base and dst pixel pointer of every job is device (or managed)
 * memory of one device.  Job i's dst bytes, *alphaAllOpaque, results[i] and the return value are what dxb200_texconv_batch gives
 * for the same jobs on host copies of the same images.  The call runs on the device that owns job 0's base pixels, on `stream`
 * (NULL = the legacy default stream); it neither shards over devices nor uses the host calls' staging buffers, so calls on
 * different streams do not wait for each other.  Base images are never written.  Once a job has passed its planner's checks,
 * an image that is not device or managed memory of that device (pageable or pinned host memory, another device's memory), or a
 * BC image whose pixel pointer is not a multiple of its block size, makes it E_INVALIDARG: it does not run and its dst is not
 * written.  Scratch memory comes from the device's stream-ordered pool (cudaMallocAsync on `stream`).
 * With no job asking for the alpha answer (alphaAllOpaque == NULL), the call only enqueues its work on `stream` and returns without
 * synchronising: dst is complete when the stream's work up to the call is.  When a job asks, the answer is a host value, so the
 * call synchronises `stream` before it returns, as dxb200_is_alpha_all_opaque_device does. */
DXB200_API int32_t  dxb200_texconv_batch_device(const dxb200_texconv_job* jobs, size_t njobs, int32_t* results, void* stream);

/* ScratchImage::IsAlphaAllOpaque (DirectXTexImage.cpp:800-852; IsAlphaAllOpaqueBC, DirectXTexCompress.cpp:539-621) of
 * `nimages` images of one format: *opaque = 1 when every texel inside every image has alpha >= 0.997 (uncompressed, as
 * LoadScanline reads it) or >= 0.99 (decoded BC1 / BC2 / BC3 / BC7 blocks; the padding texels of partial blocks do not count),
 * else 0.  A NaN alpha counts as opaque.  A format without alpha (HasAlpha: BC4, BC5, BC6H, B8G8R8X8, R32_FLOAT, ...) answers 1
 * without a pixel being read and without a device.  HRESULTs: images / opaque NULL or nimages == 0, images of different formats,
 * a zero or over-32-bit size, a BC row pitch that is not a multiple of the block size -> E_INVALIDARG; a NULL pixel pointer ->
 * E_POINTER; a format with alpha this library does not implement -> E_NOT_SUPPORTED (0x80070032).
 * The host call stages the images in bands of whole (block) rows, sharded over the initialised devices; only one result word per
 * band comes back.  The _device call runs on the device that owns the pointers and synchronises `stream` before it returns. */
DXB200_API int32_t  dxb200_is_alpha_all_opaque(const dxb200_image* images, size_t nimages, int32_t* opaque);
DXB200_API int32_t  dxb200_is_alpha_all_opaque_device(const dxb200_image* images, size_t nimages, int32_t* opaque, void* stream);

/* DirectX::Resize (DirectXTexResize.cpp:854-935 single image, :942-1120 arrays; custom filters ResizePointFilter /
 * ResizeBoxFilter / ResizeLinearFilter / ResizeCubicFilter / ResizeTriangleFilter :255-798, selection :805-837).
 *   src[i] -> dst[i], i < nimages; all sources share one size and format, all destinations share one size and the
 *   source format.  filter = TEX_FILTER_FLAGS; mode 0 selects BOX when the target is exactly half the source in both
 *   directions, else LINEAR (:812-817); BOX on any other ratio -> E_FAIL (:318-319); compressed formats ->
 *   HRESULT_E_NOT_SUPPORTED (:875-879).  (SURVEY 8(f) rank 2: the texconv step in front of Convert.) */
DXB200_API int32_t  dxb200_resize(const dxb200_image* src, size_t nimages, uint32_t filter, const dxb200_image* dst);
DXB200_API int32_t  dxb200_resize_device(const dxb200_image* src, size_t nimages, uint32_t filter, const dxb200_image* dst, void* stream);

/* DirectX::PremultiplyAlpha (DirectXTexPMAlpha.cpp:214-344; PremultiplyAlpha_ / PremultiplyAlphaLinear / DemultiplyAlpha /
 * DemultiplyAlphaLinear :30-208).  src[i] -> dst[i], same size and format; flags = TEX_PMALPHA_FLAGS (DirectXTex.h:860-879):
 * 0x1 IGNORE_SRGB, 0x2 REVERSE (premultiplied -> straight), 0x1000000 / 0x2000000 SRGB_IN / SRGB_OUT.
 * Formats without alpha or compressed -> HRESULT_E_NOT_SUPPORTED (:224-229).  (SURVEY 8(f) rank 4, first part.) */
DXB200_API int32_t  dxb200_premultiply_alpha(const dxb200_image* src, size_t nimages, uint32_t flags, const dxb200_image* dst);
DXB200_API int32_t  dxb200_premultiply_alpha_device(const dxb200_image* src, size_t nimages, uint32_t flags, const dxb200_image* dst, void* stream);

/* DirectX::ScaleMipMapsAlphaForCoverage (DirectXTexMipmaps.cpp:3483-3552; CalculateAlphaCoverage :213-308,
 * EstimateAlphaScaleForCoverage :310-355, ScaleAlpha :143-193) for ONE array item: src[0..nlevels) = its mip levels as
 * GenerateMipMaps produced them, dst[0..nlevels) = the same levels of the result.  Level 0 is copied; every other level's
 * alpha is scaled so that its alpha-test coverage at `alphaReference` matches level 0's (10-step bisection).
 * (SURVEY 8(f) rank 4.)  The bisection runs on the device: 10 coverage launches and one scaling launch per call, with no
 * host round trip in between.  The _device variant synchronises `stream` before it returns. */
DXB200_API int32_t  dxb200_scale_mipmaps_alpha_for_coverage(const dxb200_image* src, size_t nlevels, float alphaReference, const dxb200_image* dst);
DXB200_API int32_t  dxb200_scale_mipmaps_alpha_for_coverage_device(const dxb200_image* src, size_t nlevels, float alphaReference,
                                                                   const dxb200_image* dst, void* stream);

/* ---- DDS container (host-side only, no GPU work; SURVEY 8(f) rank 3) ------------------------------------------------
 * dxb200_metadata is a field-for-field mirror of DirectX::TexMetadata (DirectXTex.h:187-216).
 * EncodeDDSHeader (DirectXTexDDS.cpp:711-1043), SaveToDDSMemory (:2403-2620), GetMetadataFromDDSMemory / DecodeDDSHeader
 * (:319-683, 1960-2003), LoadFromDDSMemory (:2008-2100).  TEXTURE2D resources (arrays, cubemaps, mip chains) in the
 * formats this library implements; flags = DDS_FLAGS (DirectXTex.h:232-279): FORCE_DX10_EXT, FORCE_DX10_EXT_MISC2,
 * FORCE_DX9_LEGACY, FORCE_DXT5_RXGB, IGNORE_MIPS, ALLOW_LARGE_FILES are honoured (HRESULT_E_CANNOT_MAKE as in the
 * reference when a format has no legacy encoding); load-side conversion / legacy-expansion flags -> HRESULT_E_NOT_SUPPORTED.
 * save/encode: dst == NULL only computes *required.  load: `images` describes the destination (item-major, mip-minor)
 * as ScratchImage::Initialize(metadata) lays it out. */
typedef struct dxb200_metadata
{
    size_t   width, height, depth, arraySize, mipLevels;
    uint32_t miscFlags, miscFlags2;
    uint32_t format;        /* DXGI_FORMAT */
    uint32_t dimension;     /* TEX_DIMENSION: 3 = TEXTURE2D */
} dxb200_metadata;
DXB200_API int32_t  dxb200_dds_encode_header(const dxb200_metadata* metadata, uint32_t flags, void* dst, size_t maxsize, size_t* required);
DXB200_API int32_t  dxb200_dds_save_memory(const dxb200_image* images, size_t nimages, const dxb200_metadata* metadata, uint32_t flags,
                                           void* dst, size_t maxsize, size_t* required);
DXB200_API int32_t  dxb200_dds_get_metadata(const void* src, size_t size, uint32_t flags, dxb200_metadata* metadata, size_t* dataOffset);
DXB200_API int32_t  dxb200_dds_load_memory(const void* src, size_t size, uint32_t flags, const dxb200_image* images, size_t nimages);

#ifdef __cplusplus
}
#endif
#endif /* DXTEX_B200_H */
