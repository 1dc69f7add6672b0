"""The staging case table (tests/staging_cases.py) against the library's band and chunk sizes, without a GPU.

The GPU staging suite only tests what its cases make the staging do.  Each case names the edges it exists for (a partial last
band, bands of two images in one chunk, a TMA-eligible chunk, ...); here every case must hit them under the Python copy of
split_bands / run_staged, and that copy must use the constants dxb_api.cu compiles with, so that a change of the band or chunk
sizes cannot quietly turn the edge cases into single-band calls."""
import os
import re

import numpy as np
import pytest

from directxtex_b200 import capi, formats as F
from tests import staging_cases as SC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("NSLOT", "NLANE", "BAND_BYTES", "BAND_CHUNK", "ITEM_CHUNK")


def test_constants_equal_the_library():
    src = open(os.path.join(ROOT, "directxtex_b200", "csrc", "dxb_api.cu")).read()
    found = {}
    for name, value, shift in re.findall(r"constexpr (?:int|size_t) (\w+) = (?:size_t\()?(\d+)\)?(?: << (\d+))?;", src):
        found[name] = int(value) << int(shift or 0)
    assert {n: found.get(n) for n in NAMES} == {n: getattr(SC, n) for n in NAMES}


@pytest.mark.parametrize("case", SC.CASES, ids=lambda c: c.name)
def test_case_hits_its_edges(case):
    assert case.edges
    for edge in case.edges:
        assert SC.has_edge(case, edge), "%s does not hit: %s" % (case.name, edge)
    # with the wide caller pitches the image is still cut where the case needs it
    if SC.EDGE_MULTI_BAND in case.edges or SC.EDGE_PARTIAL_LAST in case.edges:
        assert SC.has_edge(case, SC.EDGE_MULTI_BAND, "wide"), case.name


def test_every_edge_and_band_call_is_covered():
    edges = {e for c in SC.CASES for e in c.edges}
    assert edges == {v for k, v in vars(SC).items() if k.startswith("EDGE_")}
    assert {c.op for c in SC.CASES} == {SC.COMPRESS, SC.DECOMPRESS, SC.CONVERT, SC.PMALPHA}


def test_split_bands_and_chunks_by_hand():
    """the Python copy on numbers worked out by hand: 1024-wide RGBA8 -> BC1 moves 16384 + 2048 bytes per block row, so a
    band holds 32 MiB // 18432 = 1820 block rows; two such bands do not share a 48 MiB chunk, the last 3 rows join the second"""
    case = SC.Case("", SC.COMPRESS, 28, 71, ((1024, 2 * 7280 + 3),), 0, ())
    bands, chunks, _ = SC.plan(case)
    assert [(b.row0, b.rows, b.units) for b in bands] == [(0, 7280, 7280), (7280, 7280, 7280), (14560, 3, 3)]
    assert [b.src_bytes for b in bands] == [7280 * 4096, 7280 * 4096, 3 * 4096]
    assert chunks == [[0], [1, 2]]
    # an array counts images: only the band that finishes an image reports one
    case = SC.Case("", SC.COMPRESS, 28, 71, ((1024, 7284),) * 2, 0, ())
    assert [b.units for b in SC.plan(case)[0]] == [0, 1, 0, 1]
    # the budget: nine items of 5 MiB + 256 bytes fit 48 MiB, the tenth does not
    assert SC.group_chunks([(5 << 20) + 256] * 10, SC.BAND_CHUNK) == [list(range(9)), [9]]
    assert SC.group_chunks([SC.BAND_CHUNK + 1, 1, 1], SC.BAND_CHUNK) == [[0], [1, 2]]
    assert SC.group_chunks([1, SC.BAND_CHUNK], SC.BAND_CHUNK) == [[0], [1]]


def test_mip_chain_chunks():
    """mipmaps_compress items: eleven 1024^2 RGBA8 -> BC3 chains per 80 MiB chunk (DESIGN.md section 4); a 2048^2 RGBA32F chain
    is larger than a chunk"""
    chunks, b = SC.chain_chunks(28, 77, 1024, 1024, 12, 11)
    assert [len(c) for c in chunks] == [11, 1]
    chunks, b = SC.chain_chunks(2, 98, 2048, 2048, 2, 12)
    assert b > SC.ITEM_CHUNK and chunks == [[0], [1]]


@pytest.mark.parametrize("bc", [71, 77, 98])
def test_bc_rows_off_the_block_size_are_refused(bc):
    """The kernels load and store whole 8- or 16-byte blocks, so a BC row pitch that is not a multiple of the block size would
    fault them: every compress and decompress entry point refuses it with E_INVALIDARG, and the _device ones also refuse such a
    pixel pointer (checked before any device work).  A host-pointer call only passes its row pitch to the device (its images are
    staged into aligned buffers), so an unaligned host pointer passes planning (tests/test_gpu_staging.py runs it)."""
    w, h = 8, 8
    row, sl = F.compute_pitch(bc, w, h)
    pix = np.zeros(w * h * 4 + 64, np.uint8)
    blocks = np.zeros(sl * 2 + 64, np.uint8)
    base = blocks.ctypes.data + (-blocks.ctypes.data) % 16
    L = capi.lib
    for brow, bptr in ((row + 4, base), (row, base + 4)):
        s = capi.images([capi.Image(w, h, 28, w * 4, w * h * 4, pix.ctypes.data)])
        b = capi.images([capi.Image(w, h, bc, brow, brow * 2, bptr)])
        calls = {"compress": lambda: L.dxb200_compress(s, 1, bc, 0, 0.5, 1.0, b), "decompress": lambda: L.dxb200_decompress(b, 1, 28, s),
                 "compress_device": lambda: L.dxb200_compress_device(s, 1, bc, 0, 0.5, 1.0, b, None),
                 "decompress_device": lambda: L.dxb200_decompress_device(b, 1, 28, s, None)}
        for name, call in calls.items():
            refused = brow != row or name.endswith("_device")
            assert (F.hr_u32(call()) == F.E_INVALIDARG) == refused, (bc, name, brow, bptr - base)
