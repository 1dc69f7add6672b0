"""The batches the host staging of libdxtex_b200 builds, restated in Python, and the table of staging cases the suite runs.

Every host-pointer band call (compress, decompress, convert, premultiply) goes through split_bands and run_staged in
dxb_api.cu: images are cut into bands of about BAND_BYTES on work-row boundaries, and the bands are packed into chunks of at
most BAND_CHUNK bytes, each image on a 256-byte boundary of the slot buffer (sources first, then destinations).  Chain calls
(mipmaps_compress) pack whole mip chains into chunks of ITEM_CHUNK bytes.  Which kernel a chunk runs depends on that packing:
the BC7 TMA feed needs equal jobs at a constant stride, the vector kernels aligned pointers and pitches.

The functions below restate that arithmetic for one device (run_sharded hands each device a contiguous range and runs the same
code on it), so that a case can be asked for its band cuts, its chunks and each chunk's jobs.  CASES names, for every case of
tests/test_gpu_staging.py, the edges it exists for; tests/test_cpu_staging.py asserts that each case hits them and that the
constants equal dxb_api.cu's."""
import collections

from directxtex_b200 import formats as F

NSLOT = 3                       # (stream, buffer) slots of one lane
NLANE = 2                       # host-staged calls in flight on one device
BAND_BYTES = 32 << 20           # source + destination bytes of one band
BAND_CHUNK = 48 << 20           # slot buffer bytes of one chunk of a band call
ITEM_CHUNK = 80 << 20           # slot buffer bytes of one chunk of a chain or pair call

COMPRESS, DECOMPRESS, CONVERT, PMALPHA = "compress", "decompress", "convert", "premultiply"


def pad256(n):
    return (n + 255) & ~255


def pitch(fmt, w, extra=0):
    return F.compute_pitch(fmt, w, 1)[0] + extra


def work_rows(op, flags, sizes):
    """(source rows, destination rows, source is BC, destination is BC) of one work row, as each band entry point passes them"""
    if op == COMPRESS:
        return 4, 1, False, True
    if op == DECOMPRESS:
        return 1, 4, True, False
    if op == CONVERT:
        r = 4 if flags & F.TEX_FILTER_DITHER else 1
        if flags & F.TEX_FILTER_DITHER_DIFFUSION:
            r = max([r] + [h for (_, h) in sizes])
        return r, r, False, False
    return 1, 1, False, False


Band = collections.namedtuple("Band", "image row0 rows src_bytes dst_bytes units")     # row0 / rows: pixel rows of the image


def split_bands(op, flags, sizes, spitches, dpitches):
    """split_bands of dxb_api.cu: the bands of images `sizes` ((w, h) each) with the given row pitches"""
    src_rows, dst_rows, src_bc, dst_bc = work_rows(op, flags, sizes)
    out = []
    for m, (w, h) in enumerate(sizes):
        s_total = (h + 3) // 4 if src_bc else h
        d_total = (h + 3) // 4 if dst_bc else h
        units = max(1, -(-s_total // src_rows))
        per = max(1, BAND_BYTES // max(spitches[m] * src_rows + dpitches[m] * dst_rows, 1))
        for u0 in range(0, units, per):
            u1 = min(units, u0 + per)
            sr0, sr1 = u0 * src_rows, min(s_total, u1 * src_rows)
            dr0, dr1 = u0 * dst_rows, min(d_total, u1 * dst_rows)
            rows = min(h, sr1 * 4) - sr0 * 4 if src_bc else sr1 - sr0
            out.append(Band(m, sr0 * 4 if src_bc else sr0, rows, (sr1 - sr0) * spitches[m], (dr1 - dr0) * dpitches[m],
                            rows if len(sizes) == 1 else int(u1 == units)))
    return out


def group_chunks(item_bytes, budget):
    """run_staged's grouping: whole items, at most `budget` bytes per chunk, an item larger than that is a chunk by itself"""
    chunks, i = [], 0
    while i < len(item_bytes):
        k, total = i, 0
        while k < len(item_bytes) and not (k > i and total + item_bytes[k] > budget):
            total += item_bytes[k]
            k += 1
        chunks.append(list(range(i, k)))
        i = k
    return chunks


Job = collections.namedtuple("Job", "band w h src_off dst_off spitch dpitch")


def plan(case, layout="tight"):
    """(bands, chunks as lists of band indices, jobs of each chunk with their offsets in the slot buffer) of a band case"""
    sp, dp = case_pitches(case, layout)
    bands = split_bands(case.op, case.flags, case.sizes, sp, dp)
    chunks = group_chunks([pad256(b.src_bytes) + pad256(b.dst_bytes) for b in bands], BAND_CHUNK)
    jobs = []
    for c in chunks:
        so, do = 0, sum(pad256(bands[i].src_bytes) for i in c)
        js = []
        for i in c:
            b = bands[i]
            js.append(Job(i, case.sizes[b.image][0], b.rows, so, do, sp[b.image], dp[b.image]))
            so, do = so + pad256(b.src_bytes), do + pad256(b.dst_bytes)
        jobs.append(js)
    return bands, chunks, jobs


def tma_eligible(jobs):
    """launch_bc7_tma's batch test on a chunk's jobs (RGBA32F source, the slot buffer 256-byte aligned): full blocks, rows on
    16 bytes, every job of the first one's size and pitches at a constant stride"""
    j0 = jobs[0]
    if j0.w % 4 or j0.h % 4 or j0.spitch % 16:
        return False
    if len(jobs) == 1:
        return True
    ss, ds = jobs[1].src_off - j0.src_off, jobs[1].dst_off - j0.dst_off
    if ss < j0.spitch * (j0.h - 1) + j0.w * 16 or ss % 16 or ds <= 0:
        return False
    return all((j.w, j.h, j.spitch, j.dpitch, j.src_off, j.dst_off) == (j0.w, j0.h, j0.spitch, j0.dpitch, j0.src_off + i * ss, j0.dst_off + i * ds)
               for i, j in enumerate(jobs))


def bc7_kernel(jobs, feed):
    """the kernel dxb_launch_bc7 runs for one chunk of an RGBA32F -> BC7 call under DXB200_OPT_BC7_FEED `feed`"""
    mode = (1 if len(jobs) > 1 else 0) if feed == 4 else feed
    return "k_compress_bc7_tma" if mode and tma_eligible(jobs) else "k_compress_bc7"


# ---- chain calls: dxb200_mipmaps_compress ------------------------------------------------------------------------------------
def chain_chunks(sf, df, w, h, items, levels, extra=0):
    """run_staged's chunks of a mipmaps_compress call: per item, every level of the source chain (level 0 at the caller's row
    pitch, `extra` bytes beyond the tight one) and every BC level take a 256-byte aligned place in the slot buffer"""
    b, lw, lh = 0, w, h
    for lv in range(levels):
        row, sl = F.compute_pitch(sf, lw, lh)
        b += pad256((row + extra) * lh if lv == 0 else sl) + pad256(F.compute_pitch(df, lw, lh)[1])
        lw, lh = max(1, lw >> 1), max(1, lh >> 1)
    return group_chunks([b] * items, ITEM_CHUNK), b


# ---- the case table ------------------------------------------------------------------------------------------------------------
Case = collections.namedtuple("Case", "name op sf df sizes flags edges")

# per image: bytes beyond the tight row pitch, source and destination, of the "wide" layout (+4, +64 and different per image)
WIDE = ((4, 64), (64, 4), (68, 132), (132, 8))


def case_pitches(case, layout):
    """(source, destination) row pitches of every image; a BC side widens by whole 16-byte steps, because its block rows must
    start on a multiple of the block size (the library refuses other pitches)"""
    sizes = case.sizes
    extra = [(0, 0)] * len(sizes) if layout == "tight" else [WIDE[i % len(WIDE)] for i in range(len(sizes))]
    side = lambda fmt, e: -(-e // 16) * 16 if fmt in F.BLOCK_BYTES else e
    return ([pitch(case.sf, w, side(case.sf, e[0])) for (w, _), e in zip(sizes, extra)],
            [pitch(case.df, w, side(case.df, e[1])) for (w, _), e in zip(sizes, extra)])


def units_per_band(op, sf, df, w, flags=0):
    """work rows per band of a tight image of width w"""
    src_rows, dst_rows, _, _ = work_rows(op, flags, [(w, 1)])
    return max(1, BAND_BYTES // (pitch(sf, w) * src_rows + pitch(df, w) * dst_rows))


def height_for(op, sf, df, w, bands, last_rows, flags=0):
    """a height whose tight image is cut into `bands` bands, the last one `last_rows` pixel rows"""
    r = 4 if op in (COMPRESS, DECOMPRESS) else work_rows(op, flags, [(w, 1)])[0]
    return (bands - 1) * units_per_band(op, sf, df, w, flags) * r + last_rows


EDGE_PARTIAL_LAST = "3+ bands, the last one a single block row of 1-3 pixel rows"
EDGE_PARTIAL_END = "2+ bands, the last one ending in a partial block row"
EDGE_MULTI_BAND = "2+ bands of one image"
EDGE_SHARED_CHUNK = "a band of image k and image k+1 in one chunk"
EDGE_OVERSIZED = "an item larger than the chunk budget"
EDGE_TMA_CHUNK = "a chunk whose jobs are equal and at a constant stride"
EDGE_DIRECT_CHUNK = "a chunk whose jobs are not"
EDGE_MULTI_CHUNK = "2+ chunks"
EDGE_UNALIGNED_PITCH = "a tight row pitch that is not a multiple of 16"
EDGE_DITHER_PHASE = "2+ bands, every band starting on a multiple of 4 rows where bands of single rows would not"
EDGE_WHOLE_IMAGES = "one band per image, where DITHER's 4-row bands would cut one"


def _bands_of(bands, m):
    return [b for b in bands if b.image == m]


def has_edge(case, edge, layout="tight"):
    bands, chunks, jobs = plan(case, layout)
    per_image = [_bands_of(bands, m) for m in range(len(case.sizes))]
    if edge == EDGE_PARTIAL_LAST:
        return any(len(bs) >= 3 and bs[-1].rows in (1, 2, 3) for bs in per_image)
    if edge == EDGE_PARTIAL_END:
        return any(len(bs) >= 2 and case.sizes[bs[0].image][1] % 4 and bs[-1].rows % 4 for bs in per_image)
    if edge == EDGE_MULTI_BAND:
        return any(len(bs) >= 2 for bs in per_image)
    if edge == EDGE_SHARED_CHUNK:
        return any(bands[a].image + 1 == bands[b].image for c in chunks for a, b in zip(c, c[1:]))
    if edge == EDGE_OVERSIZED:
        return any(len(c) == 1 and pad256(bands[c[0]].src_bytes) + pad256(bands[c[0]].dst_bytes) > BAND_CHUNK for c in chunks)
    if edge == EDGE_TMA_CHUNK:
        return any(len(js) > 1 and tma_eligible(js) for js in jobs)
    if edge == EDGE_DIRECT_CHUNK:
        return any(len(js) > 1 and not tma_eligible(js) for js in jobs)
    if edge == EDGE_MULTI_CHUNK:
        return len(chunks) >= 2
    if edge == EDGE_UNALIGNED_PITCH:
        return any(pitch(case.sf, w) % 16 or pitch(case.df, w) % 16 for (w, _) in case.sizes)
    if edge == EDGE_DITHER_PHASE:
        # and bands of single rows would cut a multi-band image off the phase
        one_row = [BAND_BYTES // (sp + dp) for sp, dp in zip(*case_pitches(case, layout))]
        return all(b.row0 % 4 == 0 for b in bands) and any(len(bs) >= 2 and one_row[m] % 4 for m, bs in enumerate(per_image))
    if edge == EDGE_WHOLE_IMAGES:
        four_rows = [4 * (BAND_BYTES // (4 * (sp + dp))) for sp, dp in zip(*case_pitches(case, layout))]
        return len(bands) == len(case.sizes) and any(h > r for (_, h), r in zip(case.sizes, four_rows))
    raise KeyError(edge)


def _cases():
    cs = []
    # compress: the last band one partial block row, for every remainder of h % 4
    for sf, df in ((28, 71), (28, 77), (28, 83), (61, 80)):
        for rem in (1, 2, 3):
            w = 1024
            cs.append(Case("bc%d-h%%4=%d" % (df, rem), COMPRESS, sf, df, ((w, height_for(COMPRESS, sf, df, w, 3, rem)),), 0,
                           (EDGE_PARTIAL_LAST, EDGE_MULTI_CHUNK)))
    # BC7 / BC6H from RGBA32F on one image of two bands: full blocks (the TMA feed may take it) and a partial last block row
    w = 256
    cs.append(Case("bc7-2bands", COMPRESS, 2, 98, ((w, height_for(COMPRESS, 2, 98, w, 3, 0)),), 0, (EDGE_MULTI_BAND, EDGE_MULTI_CHUNK)))
    cs.append(Case("bc6h-2bands", COMPRESS, 2, 96, ((w, height_for(COMPRESS, 2, 96, w, 2, 3)),), 0, (EDGE_PARTIAL_END, EDGE_MULTI_BAND)))
    # BC7 array of full-block images over several chunks, every chunk TMA-eligible with more than one job
    cs.append(Case("bc7-array", COMPRESS, 2, 98, ((256, 256),) * 47, 0, (EDGE_TMA_CHUNK, EDGE_MULTI_CHUNK)))
    # mixed sizes: bands of different images share a chunk
    big = (1000, height_for(COMPRESS, 28, 77, 1000, 2, 2))
    cs.append(Case("bc3-mixed", COMPRESS, 28, 77, ((16, 16), big, (7, 5), (13, 9)), 0, (EDGE_SHARED_CHUNK, EDGE_MULTI_BAND, EDGE_DIRECT_CHUNK)))
    big7 = (256, height_for(COMPRESS, 2, 98, 256, 2, 8))
    cs.append(Case("bc7-mixed", COMPRESS, 2, 98, ((16, 16), big7, (7, 5), (13, 9)), 0, (EDGE_SHARED_CHUNK, EDGE_MULTI_BAND, EDGE_DIRECT_CHUNK)))
    # decompress: every BC format, height 4k + 3, two or more bands
    for bc in sorted(F.BLOCK_BYTES):
        for df in decompress_destinations(bc):
            w = 1000
            cs.append(Case("dec%d-%d" % (bc, df), DECOMPRESS, bc, df, ((w, height_for(DECOMPRESS, bc, df, w, 2, 3)),), 0,
                           (EDGE_PARTIAL_END,)))
    # convert: a vector pair and a generic pair, widths whose tight pitch is not a multiple of 16
    for sf, df in ((28, 2), (2, 87)):
        w = 1001
        cs.append(Case("cvt%d-%d" % (sf, df), CONVERT, sf, df, ((w, height_for(CONVERT, sf, df, w, 3, 7)),), 0,
                       (EDGE_MULTI_BAND, EDGE_UNALIGNED_PITCH, EDGE_MULTI_CHUNK)))
        cs.append(Case("cvt%d-%d-mixed" % (sf, df), CONVERT, sf, df, ((16, 16), (w, height_for(CONVERT, sf, df, w, 2, 5)), (7, 5), (13, 9)), 0,
                       (EDGE_SHARED_CHUNK, EDGE_MULTI_BAND, EDGE_UNALIGNED_PITCH)))
    D = F.TEX_FILTER_DITHER
    for sf, df, w in ((2, 28, 999), (10, 61, 998)):
        cs.append(Case("dither%d-%d" % (sf, df), CONVERT, sf, df, ((w, height_for(CONVERT, sf, df, w, 3, 3, D)),), D,
                       (EDGE_DITHER_PHASE, EDGE_UNALIGNED_PITCH)))
    cs.append(Case("dither2-28-mixed", CONVERT, 2, 28, ((16, 16), (999, height_for(CONVERT, 2, 28, 999, 2, 6, D)), (7, 5), (13, 9)), D,
                   (EDGE_DITHER_PHASE, EDGE_SHARED_CHUNK)))
    # error diffusion: one band per image however large the image, so one image is larger than a chunk
    DD = F.TEX_FILTER_DITHER_DIFFUSION
    cs.append(Case("diffusion2-28", CONVERT, 2, 28, ((1003, 3000), (5, 3)), DD, (EDGE_WHOLE_IMAGES, EDGE_OVERSIZED)))
    # premultiply: both directions, formats 28 and 10, several bands
    for fmt in (28, 10):
        for fl in (0, 2):
            w = 1001
            cs.append(Case("pm%d-%s" % (fmt, "rev" if fl else "fwd"), PMALPHA, fmt, fmt, ((w, height_for(PMALPHA, fmt, fmt, w, 3, 5)),), fl,
                           (EDGE_MULTI_BAND, EDGE_UNALIGNED_PITCH, EDGE_MULTI_CHUNK)))
    return cs


GENERIC_DECOMPRESS_DST = 10            # RGBA16F: a destination no BC format has a specialised kernel for


def decompress_destinations(bc):
    """the destination DEC_PAIRS (tests/test_gpu_bc_formats.py, the specialised k_decompress_t routes) lists for `bc`; an sRGB BC
    format takes its UNORM twin's kernel into the twin destination's sRGB form, where the two sRGB sides cancel; and the generic
    destination"""
    from tests.test_gpu_bc_formats import DEC_PAIRS, SRGB_TWIN, UNORM_TWIN
    pairs = dict(DEC_PAIRS)
    df = pairs[UNORM_TWIN[bc]] if bc in UNORM_TWIN else pairs[bc]
    return (SRGB_TWIN[df] if bc in UNORM_TWIN else df, GENERIC_DECOMPRESS_DST)


CASES = _cases()
