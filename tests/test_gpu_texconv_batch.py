"""GPU suite: dxb200_texconv_batch, texconv over a list of textures of any sizes and formats in one call.

Every dst byte and every alpha answer of every job equals the single call named by the job's kind, made with the same arguments,
over a table that mixes the three kinds, bases, sizes, chain lengths, targets and steps, with tight base pitches, +16, and +4 with
the base 4 bytes off.  One-item jobs of one shape launch what one call over their items launches; failing jobs answer their single
call's HRESULT and leave their dst unwritten; groups larger than a chunk and many small groups give the single calls' bytes; and so
does a batch sharded over every visible device."""
import ctypes as C

import numpy as np
import pytest

from directxtex_b200 import capi, formats as F
from tests import oracle_lib
from tests.test_gpu_chain_steps import launches

pytestmark = pytest.mark.gpu
L = capi.lib
GUARD = 64
FILL = 0xCD
PM = capi.chain_steps(0.0, True)
COV = capi.chain_steps(0.5)
DM = capi.texconv_steps(demultiply=True)
NM = capi.texconv_steps(bc3_layout=1)
SW = capi.channel_steps(swizzle=(2, 1, 0, 3))
CK = capi.channel_steps(color_key=0x102030)
IY = capi.channel_steps(invert_y=True)
SRC = capi.chain_source()


@pytest.fixture(autouse=True)
def one_device():
    L.dxb200_shutdown()
    assert L.dxb200_init(0) == 0


def _sizes(w, h, levels):
    out = []
    for _ in range(levels):
        out.append((w, h))
        w, h = max(1, w // 2), max(1, h // 2)
    return out


def _pointer(x):
    return C.pointer(x) if x is not None else None


class Spec:
    """one job: kind, base format, base size (w, h), items, levels (0 = the full chain), dst format and the optional steps"""

    def __init__(self, kind, bf, w, h, items, levels, df, source=None, channels=None, steps=None, ts=None, scan=True, filter=0, flags=0,
                 bad=None):
        self.kind, self.bf, self.w, self.h, self.items, self.df = kind, bf, w, h, items, df
        ow, oh = (source.width, source.height) if source is not None and source.width else (w, h)
        self.levels = levels or F.count_mips(ow, oh)
        self.source, self.channels, self.steps, self.ts, self.scan, self.filter, self.flags, self.bad = \
            source, channels, steps, ts, scan, filter, flags, bad
        self.bsizes = _sizes(w, h, self.levels) if kind == 2 else [(w, h)]
        self.osizes = [(ow, oh)] if kind == 2 and self.levels == 1 else _sizes(ow, oh, self.levels) if kind != 2 else self.bsizes


def _base_image(fmt, w, h, rng):
    if fmt in F.BLOCK_BYTES:
        return rng.integers(0, 256, F.compute_pitch(fmt, w, h)[1], dtype=np.uint8)
    return oracle_lib.random_image(fmt, w, h, rng).view(np.uint8).reshape(-1)


class Inputs:
    """the host bases of a Spec at a row pitch of tight + extra (rounded up to whole blocks for a BC base), `offset` bytes into their
    buffers"""

    def __init__(self, spec, rng, extra=0, offset=0):
        self.keep, ims = [], []
        for _ in range(spec.items):
            for (w, h) in spec.bsizes:
                img = _base_image(spec.bf, w, h, rng)
                row, _ = F.compute_pitch(spec.bf, w, h)
                rows = max(1, (h + 3) // 4) if spec.bf in F.BLOCK_BYTES else h
                bs = F.BLOCK_BYTES.get(spec.bf, 1)
                pitch = row + ((extra + bs - 1) // bs * bs if spec.bf in F.BLOCK_BYTES else extra)
                buf = np.zeros(offset + pitch * rows, np.uint8)
                for r in range(rows):
                    buf[offset + r * pitch: offset + r * pitch + row] = img[r * row: (r + 1) * row]
                self.keep.append(buf)
                ims.append(capi.Image(w, h, spec.bf, pitch, pitch * rows, buf.ctypes.data + offset))
        if spec.bad is not None:
            i, field, value = spec.bad
            setattr(ims[i], field, value)
        self.base = capi.images(ims)


class Outputs:
    """the dst images of a Spec, each in its own buffer followed by GUARD bytes, every byte FILL at first"""

    def __init__(self, spec):
        self.bufs, ims = [], []
        for _ in range(spec.items):
            for (w, h) in spec.osizes:
                row, sl = F.compute_pitch(spec.df, w, h)
                buf = np.full(sl + GUARD, FILL, np.uint8)
                self.bufs.append(buf)
                ims.append(capi.Image(w, h, spec.df, row, sl, buf.ctypes.data))
        self.dst = capi.images(ims)
        self.opaque = C.c_int32(-1)


def job(spec, inputs, outputs):
    return capi.TexconvJob(spec.kind, inputs.base, spec.items, spec.levels, _pointer(spec.source), _pointer(spec.channels), spec.filter,
                           _pointer(spec.steps), _pointer(spec.ts), spec.df, 0, spec.flags, 0.5, outputs.dst,
                           C.pointer(outputs.opaque) if spec.scan else None)


def single(j):
    """the call named by j.kind with j's arguments"""
    if j.kind == 0:
        return L.dxb200_mipmaps_compress_from_channels_ex(j.base, j.items, j.source, j.channels, j.levels, j.filter, j.steps, j.dstFormat,
                                                          j.compressFlags, j.threshold, 1.0, j.dst, j.alphaAllOpaque, j.ts)
    if j.kind == 1:
        return L.dxb200_mipmaps_convert_from_ex(j.base, j.items, j.source, j.channels, j.dstFormat, j.convertFilter, j.threshold, j.levels,
                                                j.filter, j.steps, j.dst, j.alphaAllOpaque, j.ts)
    return L.dxb200_levels_from_ex(j.base, j.items, j.levels, j.source, j.channels, j.dstFormat, j.convertFilter, j.compressFlags, j.threshold,
                                   j.steps, j.dst, j.alphaAllOpaque, j.ts)


def run_batch(jobs):
    table = (capi.TexconvJob * len(jobs))(*jobs)
    results = (C.c_int32 * len(jobs))()
    hr = F.hr_u32(L.dxb200_texconv_batch(table, len(jobs), results))
    return hr, [F.hr_u32(r) for r in results]


def compare(specs, rng, extra=0, offset=0):
    """runs every spec as a single call and all of them as one batch, on the same inputs; asserts equal HRESULTs, bytes, guards and
    alpha answers, and returns the batch's HRESULT"""
    inputs = [Inputs(s, rng, extra, offset) for s in specs]
    ones, many = [Outputs(s) for s in specs], [Outputs(s) for s in specs]
    want = [F.hr_u32(single(job(s, i, o))) for s, i, o in zip(specs, inputs, ones)]
    jobs = [job(s, i, o) for s, i, o in zip(specs, inputs, many)]
    hr, got = run_batch(jobs)
    assert got == want, [(k, hex(a), hex(b)) for k, (a, b) in enumerate(zip(got, want)) if a != b]
    assert hr == next((w for w in want if w), 0)
    for k, (s, a, b) in enumerate(zip(specs, ones, many)):
        for m, (x, y) in enumerate(zip(a.bufs, b.bufs)):
            assert (y[-GUARD:] == FILL).all(), (k, m)
            if want[k]:
                assert (y == FILL).all(), (k, m)             # a failing job's dst is not written
            else:
                assert np.array_equal(x, y), (k, m, s.kind, s.bf, s.df, s.w, s.h)
        assert a.opaque.value == b.opaque.value, k
        if s.scan and not want[k]:
            assert b.opaque.value in (0, 1), k
    return hr


def table():
    """about 40 jobs: every kind; RGBA8, RGBA8_SRGB, RGBA16F, RGBA32F, BC1, BC3, BC5 and BC7 bases; 1 x 1, 3 x 5, 64^2, 100 x 60,
    256^2 and 1024 x 512; full, partial and single-level chains and kept levels; BC1, BC3, BC3n, BC6H, BC7, RGBA8, BGRA8 and RGBA16F
    targets; with and without source, channels, coverage, premultiply, -alpha and the scan; several jobs of one shape"""
    return [
        Spec(0, 28, 64, 64, 1, 0, 77),
        Spec(0, 28, 64, 64, 2, 0, 77),
        Spec(0, 28, 64, 64, 1, 0, 77, scan=False),
        Spec(0, 29, 100, 60, 1, 0, 72, steps=COV),
        Spec(0, 28, 256, 256, 1, 4, 98, steps=PM),
        Spec(0, 10, 256, 256, 1, 0, 95),
        Spec(0, 2, 1024, 512, 1, 0, 98, channels=SW),
        Spec(0, 2, 64, 64, 1, 3, 95),
        Spec(0, 77, 64, 64, 1, 0, 98, source=SRC, ts=DM),
        Spec(0, 71, 100, 60, 2, 0, 71, source=SRC, channels=CK),
        Spec(0, 83, 64, 64, 1, 0, 77, source=SRC, ts=NM),
        Spec(0, 98, 256, 256, 1, 0, 77, source=capi.chain_source(width=128, height=128, resize_filter=F.TEX_FILTER_LINEAR)),
        Spec(0, 28, 3, 5, 1, 0, 71),
        Spec(0, 28, 3, 5, 2, 0, 71),
        Spec(0, 29, 1024, 512, 1, 0, 77, steps=PM),
        Spec(0, 28, 64, 64, 1, 0, 77, ts=NM),
        Spec(1, 28, 64, 64, 1, 0, 87),
        Spec(1, 28, 64, 64, 1, 0, 87),
        Spec(1, 28, 100, 60, 1, 0, 10, steps=COV),
        Spec(1, 10, 256, 256, 1, 5, 28, channels=SW, steps=PM),
        Spec(1, 2, 64, 64, 2, 0, 10, channels=IY),
        Spec(1, 98, 64, 64, 1, 0, 87, source=SRC, channels=CK, steps=PM, ts=DM),
        Spec(1, 71, 3, 5, 1, 0, 28, source=SRC),
        Spec(1, 77, 1024, 512, 1, 0, 28, source=SRC),
        Spec(1, 28, 100, 60, 1, 0, 28, channels=CK),
        Spec(1, 83, 64, 64, 1, 0, 28, source=SRC, scan=False),
        Spec(2, 77, 64, 64, 1, 0, 98),
        Spec(2, 77, 64, 64, 2, 0, 98),
        Spec(2, 77, 256, 256, 1, 0, 77),
        Spec(2, 71, 100, 60, 1, 0, 28),
        Spec(2, 28, 1, 1, 1, 1, 71),
        Spec(2, 28, 1, 1, 2, 1, 28, scan=False),
        Spec(2, 28, 100, 60, 1, 1, 98, source=capi.chain_source(width=50, height=30)),
        Spec(2, 10, 64, 64, 1, 0, 95),
        Spec(2, 2, 256, 256, 1, 3, 10, steps=PM),
        Spec(2, 29, 3, 5, 1, 0, 87, channels=SW),
        Spec(2, 98, 1024, 512, 1, 0, 87),
        Spec(2, 83, 64, 64, 1, 0, 77, ts=NM),
        Spec(2, 28, 64, 64, 1, 0, 77, ts=DM),
        Spec(2, 77, 64, 64, 1, 0, 98),
    ]


@pytest.mark.parametrize("extra,offset", [(0, 0), (16, 0), (4, 4)], ids=["tight", "pitch16", "pitch4_offset4"])
def test_bytes_equal_the_single_calls(extra, offset):
    rng = np.random.default_rng(7 + extra)
    assert compare(table(), rng, extra, offset) == 0


def test_one_item_jobs_launch_what_one_call_launches():
    """one-item jobs of two shapes, interleaved: per kernel, the launches of one call per shape over all its items"""
    rng = np.random.default_rng(3)
    a = Spec(0, 28, 64, 64, 1, 0, 77, steps=COV)
    b = Spec(1, 71, 64, 64, 1, 0, 87, source=SRC, channels=CK)
    specs = [a, b, a, a, b, a, a, a, b]
    inputs = [Inputs(s, rng) for s in specs]
    outs = [Outputs(s) for s in specs]
    jobs = [job(s, i, o) for s, i, o in zip(specs, inputs, outs)]
    (hr, _), got = launches(run_batch, jobs)
    assert hr == 0

    def grouped(spec, members):
        merged = Spec(spec.kind, spec.bf, spec.w, spec.h, len(members), spec.levels, spec.df, spec.source, spec.channels, spec.steps, spec.ts,
                      spec.scan)
        mi, mo = Inputs(merged, rng), Outputs(merged)
        mi.base = capi.images([inputs[k].base[0] for k in members])
        return job(merged, mi, mo), (mi, mo)                # the buffers stay alive as long as the job

    ja, keep_a = grouped(a, [k for k, s in enumerate(specs) if s is a])
    jb, keep_b = grouped(b, [k for k, s in enumerate(specs) if s is b])
    ra, want_a = launches(single, ja)
    rb, want_b = launches(single, jb)
    assert ra == 0 and rb == 0
    want = {k: want_a.get(k, 0) + want_b.get(k, 0) for k in set(want_a) | set(want_b)}
    assert got == want


def test_failing_jobs_answer_their_single_calls():
    rng = np.random.default_rng(11)
    specs = [
        Spec(0, 28, 64, 64, 1, 0, 77),
        Spec(0, 28, 64, 64, 1, 9, 77),                                   # more levels than 64 x 64 has
        Spec(1, 28, 64, 64, 1, 0, 87),
        Spec(0, 77, 64, 64, 1, 0, 98),                                   # a BC base without a source
        Spec(2, 28, 64, 64, 1, 0, 77, bad=(2, "pixels", None)),
        Spec(2, 77, 64, 64, 1, 0, 98),
        Spec(0, 28, 64, 64, 1, 0, 98, ts=NM),                            # a layout into BC7
        Spec(1, 28, 100, 60, 1, 0, 10, steps=COV),
        Spec(0, 28, 64, 64, 1, 0, 77, steps=COV),
    ]
    hr = compare(specs, rng)
    assert hr == F.E_INVALIDARG


def test_a_group_larger_than_a_chunk():
    """24 one-item jobs of 1024^2 RGBA8 -> BC3 chains: more than one chunk of one group"""
    rng = np.random.default_rng(5)
    assert compare([Spec(0, 28, 1024, 1024, 1, 0, 77)] * 24, rng) == 0


def test_two_hundred_jobs_of_forty_shapes():
    rng = np.random.default_rng(9)
    shapes = []
    for (w, h) in [(8, 8), (16, 16), (32, 32), (64, 64), (24, 40), (40, 24), (100, 60), (128, 64)]:
        shapes += [Spec(0, 28, w, h, 1, 0, 77), Spec(0, 28, w, h, 1, 0, 71, scan=False), Spec(1, 28, w, h, 1, 0, 87),
                   Spec(1, 28, w, h, 1, 0, 10, scan=False), Spec(2, 28, w, h, 1, 0, 98)]
    order = rng.permutation(200) % 40
    assert compare([shapes[k] for k in order], rng) == 0


def test_every_visible_device():
    n = L.dxb200_device_count()
    if n < 2:
        pytest.skip("one device")
    specs = table()
    one = compare(specs, np.random.default_rng(21))
    capi.init_devices(list(range(n)))
    assert compare(specs, np.random.default_rng(21)) == one == 0
