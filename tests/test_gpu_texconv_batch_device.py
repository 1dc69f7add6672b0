"""GPU suite: dxb200_texconv_batch_device, texconv over a list of textures already in device memory, on the caller's stream.

Bases and dsts are torch CUDA buffers followed by guard bytes.  Every dst byte, guard and alpha answer equals dxb200_texconv_batch
run on host copies of the same images, over test_gpu_texconv_batch's 40-job table at three base layouts (BC bases move by a whole
block where the others move by 4 bytes), and the bases are byte-identical after every call, also where the host staging runs a step
in place on the uploaded base.  With caller images laid out as the staging buffer lays them out, the launches per kernel equal the
host batch's.  Failing jobs answer the host batch's HRESULTs; a base or dst in pageable or pinned host memory, on another device or
at a BC pointer that is not a whole number of blocks is E_INVALIDARG for its job alone, which launches nothing and leaves its dst
unwritten.  Work queued on the stream before the call is seen by it, and what is queued after it sees its results; two threads on
two streams, groups larger than a chunk and many small groups give the host batch's bytes, and so does a batch on device 1."""
import ctypes as C
import threading
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from directxtex_b200 import capi, formats as F
from tests.test_gpu_chain_steps import launches
from tests.test_gpu_texconv_batch import CK, COV, DM, FILL, GUARD, NM, SRC, Inputs, Outputs, Spec, job, run_batch, table

pytestmark = pytest.mark.gpu
L = capi.lib


@pytest.fixture(autouse=True)
def one_device():
    L.dxb200_shutdown()
    assert L.dxb200_init(0) == 0


def _tensor(buf, device, fill=FILL):
    """a CUDA copy of the host bytes `buf` followed by GUARD bytes of `fill`"""
    t = torch.full((len(buf) + GUARD,), fill, dtype=torch.uint8, device=device)
    t[:len(buf)].copy_(torch.from_numpy(buf))
    return t


class Device:
    """device copies of a Spec's Inputs and Outputs: each base buffer and each dst buffer (FILL, then GUARD bytes of FILL) in a CUDA
    tensor of its own, the images at the host images' offsets and pitches; job() takes it in place of both"""

    def __init__(self, inputs, outputs, device="cuda"):
        self.tbase, ims = [], []
        for k, buf in enumerate(inputs.keep):
            t = _tensor(buf, device)
            self.tbase.append(t)
            im = capi.Image.from_buffer_copy(inputs.base[k])
            if im.pixels:
                im.pixels = t.data_ptr() + (inputs.base[k].pixels - buf.ctypes.data)
            ims.append(im)
        self.base = capi.images(ims)
        self.tdst, ims = [], []
        for k, buf in enumerate(outputs.bufs):
            t = torch.from_numpy(buf).to(device)            # FILL with its GUARD bytes
            self.tdst.append(t)
            im = capi.Image.from_buffer_copy(outputs.dst[k])
            im.pixels = t.data_ptr()
            ims.append(im)
        self.dst = capi.images(ims)
        self.opaque = C.c_int32(-1)
        self.before = [t.clone() for t in self.tbase]


def _inputs(spec, rng, extra, offset):
    """Inputs at tight + extra pitch, `offset` bytes in; a BC base moves by a whole block instead"""
    bs = F.BLOCK_BYTES.get(spec.bf)
    return Inputs(spec, rng, extra, (bs if offset else 0) if bs else offset)


def prepare(specs, rng, extra=0, offset=0, device="cuda"):
    inputs = [_inputs(s, rng, extra, offset) for s in specs]
    host = [Outputs(s) for s in specs]
    dev = [Device(i, Outputs(s), device) for s, i in zip(specs, inputs)]
    return inputs, host, dev


def host_batch(specs, inputs, host):
    return run_batch([job(s, i, o) for s, i, o in zip(specs, inputs, host)])


def device_batch(specs, dev, stream=None):
    return capi.texconv_batch_device([job(s, d, d) for s, d in zip(specs, dev)], stream)


def check(specs, host, dev, want, got, rejected=()):
    """got = the device batch's (hr, results), want the host batch's; jobs in `rejected` are E_INVALIDARG with their dst unwritten"""
    exp = [F.E_INVALIDARG if k in rejected else w for k, w in enumerate(want[1])]
    assert got[1] == exp, [(k, hex(a), hex(b)) for k, (a, b) in enumerate(zip(got[1], exp)) if a != b]
    assert got[0] == next((w for w in exp if w), 0)
    torch.cuda.synchronize()
    for k, (s, h, d) in enumerate(zip(specs, host, dev)):
        for m, (x, t) in enumerate(zip(h.bufs, d.tdst)):
            y = t.cpu().numpy()
            if exp[k]:
                assert (y == FILL).all(), (k, m)
            else:
                assert np.array_equal(x, y), (k, m, s.kind, s.bf, s.df, s.w, s.h)
        if not exp[k]:
            assert h.opaque.value == d.opaque.value, k
        else:
            assert d.opaque.value == -1, k
        for a, b in zip(d.before, d.tbase):
            assert torch.equal(a, b), k                     # inputs are never written


def compare(specs, rng, extra=0, offset=0, stream="new"):
    inputs, host, dev = prepare(specs, rng, extra, offset)
    want = host_batch(specs, inputs, host)
    st = torch.cuda.Stream() if stream == "new" else stream
    got = device_batch(specs, dev, st)
    check(specs, host, dev, want, got)
    return got[0]


# the plans that write the base in place on the host: the swizzle in front of a Convert (kind 1 RGBA16F -> RGBA8 and kind 2
# RGBA8_SRGB -> BGRA8 are in table()) and the demultiply of an uncompressed base into an uncompressed target
IN_PLACE = [Spec(1, 28, 64, 64, 1, 0, 87, ts=DM), Spec(2, 28, 64, 64, 1, 0, 28, ts=DM, scan=False)]


@pytest.mark.parametrize("extra,offset", [(0, 0), (16, 0), (4, 4)], ids=["tight", "pitch16", "pitch4_offset4"])
def test_bytes_equal_the_host_batch(extra, offset):
    rng = np.random.default_rng(7 + extra)
    assert compare(table() + IN_PLACE, rng, extra, offset) == 0


def test_legacy_default_stream():
    assert compare(table()[:12], np.random.default_rng(13), stream=None) == 0


def _arena(images, bufs, device="cuda"):
    """one CUDA tensor holding every image of `images` (host bytes in bufs) on the next 256-byte boundary, as the staging buffer
    holds a plane: returns (tensor, device images)"""
    offs, at = [], 0
    for b in bufs:
        offs.append(at)
        at += (len(b) + 255) // 256 * 256
    t = torch.zeros(at + GUARD, dtype=torch.uint8, device=device)
    ims = []
    for im, b, o in zip(images, bufs, offs):
        t[o:o + len(b)].copy_(torch.from_numpy(b))
        c = capi.Image.from_buffer_copy(im)
        c.pixels = t.data_ptr() + o
        ims.append(c)
    return t, ims


def test_launches_equal_the_host_batch():
    """one-item jobs of two shapes, interleaved, with every caller image on a 256-byte boundary: per kernel, the host batch's
    launches"""
    rng = np.random.default_rng(3)
    a = Spec(0, 28, 64, 64, 1, 0, 77, steps=COV)
    b = Spec(1, 71, 64, 64, 1, 0, 87, source=SRC, channels=CK)
    specs = [a, b, a, a, b, a, a, a, b]
    inputs = [Inputs(s, rng) for s in specs]
    host = [Outputs(s) for s in specs]
    (want, wl) = launches(host_batch, specs, inputs, host)
    assert want[0] == 0
    tb, bims = _arena([i.base[0] for i in inputs], [i.keep[0] for i in inputs])
    outs = [Outputs(s) for s in specs]
    td, dims = _arena([im for o in outs for im in o.dst[:len(o.bufs)]], [x[:-GUARD] for o in outs for x in o.bufs])
    jobs, keep, at = [], [], 0
    for k, (s, o) in enumerate(zip(specs, outs)):
        keep.append((SimpleNamespace(base=capi.images([bims[k]])), SimpleNamespace(dst=capi.images(dims[at:at + len(o.bufs)]), opaque=o.opaque)))
        jobs.append(job(s, *keep[-1]))
        at += len(o.bufs)
    st = torch.cuda.Stream()
    (got, gl) = launches(capi.texconv_batch_device, jobs, st)
    assert got[0] == 0
    assert gl == wl
    torch.cuda.synchronize()
    got_bytes = td.cpu().numpy()
    at = 0
    for h in host:
        for x in h.bufs:
            n = len(x) - GUARD
            assert np.array_equal(got_bytes[at:at + n], x[:n])
            at += (n + 255) // 256 * 256


def _failing_specs():
    return [
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


def test_failing_jobs_answer_the_host_batch():
    specs = _failing_specs()
    hr = compare(specs, np.random.default_rng(11))
    assert hr == F.E_INVALIDARG


def _pointer_cases():
    """(spec, how its device images are broken): a base in pageable host memory, in pinned host memory, a BC base and a BC dst one
    word off a block"""
    pinned = []

    def pageable(inp, d):
        d.base[0].pixels = inp.base[0].pixels

    def pin(inp, d):
        t = torch.from_numpy(inp.keep[0]).pin_memory()
        pinned.append(t)
        d.base[0].pixels = t.data_ptr()

    def bc_base(inp, d):
        d.base[0].pixels += 4

    def bc_dst(inp, d):
        d.dst[1].pixels += 4

    return [(Spec(0, 28, 64, 64, 1, 0, 77), pageable), (Spec(1, 28, 64, 64, 1, 0, 87), pin),
            (Spec(2, 77, 64, 64, 1, 0, 98), bc_base), (Spec(0, 28, 64, 64, 1, 0, 71), bc_dst)], pinned


def test_pointers_the_device_cannot_use_are_refused_per_job():
    rng = np.random.default_rng(17)
    cases, _pinned = _pointer_cases()
    good = [Spec(0, 28, 64, 64, 1, 0, 77), Spec(2, 77, 64, 64, 1, 0, 98), Spec(1, 28, 64, 64, 1, 0, 87)]
    specs, breaks = [], {}
    for k, (spec, brk) in enumerate(cases):
        specs += [good[k % len(good)], spec]
        breaks[len(specs) - 1] = brk
    inputs, host, dev = prepare(specs, rng)
    for k, brk in breaks.items():
        brk(inputs[k], dev[k])
    want = host_batch(specs, inputs, host)
    assert want[0] == 0
    got = device_batch(specs, dev, torch.cuda.Stream())
    check(specs, host, dev, want, got, rejected=set(breaks))
    # a rejected job launches nothing
    for k in breaks:
        before = L.dxb200_launch_count()
        got = device_batch([specs[k]], [dev[k]], torch.cuda.Stream())
        assert got == (F.E_INVALIDARG, [F.E_INVALIDARG]) and L.dxb200_launch_count() == before, k


def test_a_job_on_another_device_is_refused():
    if torch.cuda.device_count() < 2:
        pytest.skip("one device")
    rng = np.random.default_rng(19)
    specs = [Spec(0, 28, 64, 64, 1, 0, 77), Spec(1, 28, 64, 64, 1, 0, 87), Spec(2, 77, 64, 64, 1, 0, 98)]
    inputs, host, dev = prepare(specs, rng)
    other = [Device(inputs[k], Outputs(specs[k]), "cuda:1") for k in (1, 2)]
    dev[1] = other[0]                                               # base and dst on device 1
    dev[2].dst, dev[2].tdst = other[1].dst, other[1].tdst            # dst on device 1
    want = host_batch(specs, inputs, host)
    got = device_batch(specs, dev, torch.cuda.Stream())
    torch.cuda.synchronize(1)
    check(specs, host, dev, want, got, rejected={1, 2})
    before = L.dxb200_launch_count()
    assert device_batch([specs[2]], [dev[2]], torch.cuda.Stream()) == (F.E_INVALIDARG, [F.E_INVALIDARG])
    assert L.dxb200_launch_count() == before


def test_stream_order():
    """the bases are written by work queued on the stream just before the call, and the dsts read by work queued just after it;
    no job asks for the alpha answer, so nothing in between synchronises"""
    rng = np.random.default_rng(23)
    specs = [Spec(s.kind, s.bf, s.w, s.h, s.items, s.levels, s.df, s.source, s.channels, s.steps, s.ts, False) for s in table()]
    inputs, host, dev = prepare(specs, rng)
    want = host_batch(specs, inputs, host)
    real = [[t.clone() for t in d.tbase] for d in dev]
    for d in dev:
        for t in d.tbase:
            t.zero_()
    torch.cuda.synchronize()
    st = torch.cuda.Stream()
    big = torch.empty(1 << 28, dtype=torch.float32, device="cuda")
    with torch.cuda.stream(st):
        for v in range(8):
            big.fill_(float(v))                             # a large fill ahead of the bases' own bytes
        for d, r in zip(dev, real):
            for t, x in zip(d.tbase, r):
                t.copy_(x)
    got = device_batch(specs, dev, st)
    with torch.cuda.stream(st):
        read = [[t.clone() for t in d.tdst] for d in dev]
    st.synchronize()
    assert got == want
    for h, r in zip(host, read):
        for x, y in zip(h.bufs, r):
            assert np.array_equal(x, y.cpu().numpy())


def test_two_threads_on_two_streams():
    specs = table()
    runs = [prepare(specs, np.random.default_rng(29 + t)) for t in range(2)]
    wants = [host_batch(specs, i, h) for i, h, _ in runs]
    gots = [None, None]

    def work(t):
        st = torch.cuda.Stream()
        gots[t] = device_batch(specs, runs[t][2], st)
        st.synchronize()

    threads = [threading.Thread(target=work, args=(t,)) for t in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for (i, h, d), w, g in zip(runs, wants, gots):
        check(specs, h, d, w, g)


def test_a_group_larger_than_a_chunk():
    """24 one-item jobs of 1024^2 RGBA8 -> BC3 chains: several chunks through one scratch allocation"""
    assert compare([Spec(0, 28, 1024, 1024, 1, 0, 77)] * 24, np.random.default_rng(5)) == 0


def test_two_hundred_jobs_of_forty_shapes():
    rng = np.random.default_rng(9)
    shapes = []
    for (w, h) in [(8, 8), (16, 16), (32, 32), (64, 64), (24, 40), (40, 24), (100, 60), (128, 64)]:
        shapes += [Spec(0, 28, w, h, 1, 0, 77), Spec(0, 28, w, h, 1, 0, 71, scan=False), Spec(1, 28, w, h, 1, 0, 87),
                   Spec(1, 28, w, h, 1, 0, 10, scan=False), Spec(2, 28, w, h, 1, 0, 98)]
    order = rng.permutation(200) % 40
    assert compare([shapes[k] for k in order], rng) == 0


def test_a_batch_on_device_1():
    if torch.cuda.device_count() < 2:
        pytest.skip("one device")
    specs = table()
    inputs, host, _ = prepare(specs, np.random.default_rng(31))
    want = host_batch(specs, inputs, host)
    dev = [Device(i, Outputs(s), "cuda:1") for s, i in zip(specs, inputs)]
    with torch.cuda.device(1):
        st = torch.cuda.Stream()
    got = device_batch(specs, dev, st)
    torch.cuda.synchronize(1)
    check(specs, host, dev, want, got)
