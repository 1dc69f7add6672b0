"""CPU suite: how dxb200_texconv_batch plans a list of textures, without a device, through its planner on the host
(tests/emul/texconv_batch.cpp, emul_texconv_batch).  Every job answers its single call's HRESULT and the batch the lowest-index
failure; jobs whose plans differ only in pointers and row pitches share a group and any planned difference splits them; groups
come in the order of their first job and their items in job order; each group stages what its single call stages; and the units
are split over 1, 2, 3 and 8 devices by the contiguous by-bytes rule every host call shards its items with."""
import ctypes as C
import os

import pytest

from directxtex_b200 import capi, formats as F
from tests.bc7_ranking_build import host_lib
from tests.test_cpu_chain_routing import _chunk_plan
from tests.test_cpu_texconv_steps import CASES, DM, ENTRIES, PM, call_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = capi.lib
NONE = 2 ** 64 - 1
UNIFORM = 0x40000


@pytest.fixture(scope="module")
def em(tmp_path_factory):
    E = host_lib("texconv_batch.cpp", tmp_path_factory.mktemp("texconv_batch_emul"), os.path.join(ROOT, "tests", "emul"))
    for _, name, args in ENTRIES.values():
        getattr(E, name).argtypes = args + [C.POINTER(C.c_uint64)]
        getattr(E, name).restype = C.c_int32
    E.emul_chunk_plan.argtypes = [C.POINTER(C.c_uint64), C.c_size_t]
    E.emul_chunk_plan.restype = C.c_size_t
    E.emul_texconv_batch.argtypes = [C.POINTER(capi.TexconvJob), C.c_size_t, C.POINTER(C.c_int32), C.POINTER(C.c_uint64)]
    E.emul_texconv_batch.restype = C.c_int32
    E.emul_batch_chunk_plan.argtypes = [C.c_size_t]
    E.emul_batch_units.argtypes = [C.c_size_t, C.POINTER(C.c_uint64), C.c_size_t]
    E.emul_batch_units.restype = C.c_size_t
    return E


class Job:
    """one job of a batch and the arguments of its single call: `entry` ("gen", "conv", "lev") with call_args' arguments, the
    TexconvSteps of ts_kw and a scan (alphaAllOpaque) or not"""

    def __init__(self, entry, bf, w, h, items, levels, df, src_kw=None, ch_kw=None, steps=None, ts_kw=None, base_bad=None, dst_bad=None,
                 scan=True, flags=0, threshold=0.5, row_pitch=0, offset=0):
        self.entry = entry
        self.args, self.keep = call_args(entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps, None, base_bad, dst_bad)
        base = self.args[0]
        for im in base:
            if im.pixels:
                im.pixels += offset
            if row_pitch and im.pixels:
                im.rowPitch += row_pitch
                im.slicePitch = im.rowPitch * (max(1, (im.height + 3) // 4) if bf in F.BLOCK_BYTES else im.height)
        self.ts = capi.texconv_steps(**(ts_kw or {}))
        self.opaque = C.c_int32(-1) if scan else None
        source, channels, steps_ = self.keep
        ptr = lambda x: C.pointer(x) if x is not None else None
        a = self.args
        if entry == "gen":
            a = list(a); a[8] = flags; a[9] = threshold; self.args = tuple(a)
            dst = a[11]
            self.job = capi.TexconvJob(0, base, a[1], a[4], ptr(source), ptr(channels), a[5], ptr(steps_), C.pointer(self.ts), df, 0, flags,
                                       threshold, dst, ptr(self.opaque))
        elif entry == "conv":
            a = list(a); a[6] = threshold; self.args = tuple(a)
            self.job = capi.TexconvJob(1, base, a[1], a[7], ptr(source), ptr(channels), a[8], ptr(steps_), C.pointer(self.ts), df, a[5], 0,
                                       threshold, a[10], ptr(self.opaque))
        else:
            a = list(a); a[7] = flags; a[8] = threshold; self.args = tuple(a)
            self.job = capi.TexconvJob(2, base, a[1], a[2], ptr(source), ptr(channels), 0, ptr(steps_), C.pointer(self.ts), df, a[5], flags,
                                       threshold, a[10], ptr(self.opaque))

    def single_hr(self, em):
        """the HRESULT of the job's single call, through its planner on the host"""
        op = C.byref(self.opaque) if self.opaque is not None else None
        return F.hr_u32(getattr(em, ENTRIES[self.entry][1])(*self.args, op, C.byref(self.ts), None))


def batch(em, jobs):
    table = (capi.TexconvJob * len(jobs))(*[j.job for j in jobs])
    results = (C.c_int32 * len(jobs))()
    groups = (C.c_uint64 * len(jobs))()
    hr = F.hr_u32(em.emul_texconv_batch(table, len(jobs), results, groups))
    return hr, [F.hr_u32(r) for r in results], list(groups)


def split(em, devices, nunits):
    """(the unit weights of the last batch, its cut over `devices`)"""
    out = (C.c_uint64 * 4096)()
    words = list(out[:em.emul_batch_units(devices, out, len(out))])
    nd = min(devices, max(nunits, 1))
    assert len(words) == nunits + nd + 1
    return words[:nunits], words[nunits:]


def contiguous_by_bytes(weights, devices):
    """the rule restated: nd = min(devices, max(n, 1)) ranges; range d ends at the first unit where the running weight reaches d / nd
    of the total"""
    n = len(weights)
    nd = min(devices, max(n, 1))
    total = float(sum(weights))
    cut = [0] + [n] * nd
    acc, d = 0.0, 1
    for i, w in enumerate(weights):
        if d >= nd:
            break
        acc += float(w)
        while d < nd and acc >= total * d / nd:
            cut[d] = i + 1
            d += 1
    return cut


# valid jobs of every kind (entry, base fmt, w, h, items, levels, dst fmt, source kwargs, channels kwargs, steps, texconv kwargs)
VALID = [
    ("gen", 28, 32, 32, 2, 6, 77, None, None, None, {}),
    ("gen", 77, 32, 32, 1, 6, 98, {}, None, PM, DM),
    ("gen", 83, 40, 40, 1, 6, 77, dict(width=32, height=32), dict(invert_y=True), None, dict(bc3_layout=1)),
    ("conv", 98, 32, 32, 1, 6, 87, {}, dict(color_key=0x102030), PM, DM),
    ("conv", 10, 32, 32, 2, 5, 28, None, dict(swizzle=(2, 1, 0, 3)), None, {}),
    ("lev", 77, 32, 32, 1, 6, 77, None, None, None, {}),
    ("lev", 28, 32, 32, 2, 6, 98, None, None, PM, {}),
    ("lev", 28, 40, 40, 1, 1, 71, dict(width=20, height=20), None, None, {}),
]


def _mixed():
    jobs = []
    for k, case in enumerate(CASES):
        name, entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps, ts_kw, base_bad, dst_bad, want = case
        jobs.append((Job(entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps, ts_kw, base_bad, dst_bad), want))
        v = VALID[k % len(VALID)]
        jobs.append((Job(*v), 0))
    return jobs


def test_every_job_answers_its_single_call(em):
    mixed = _mixed()
    jobs = [j for j, _ in mixed]
    want = [j.single_hr(em) for j in jobs]
    assert want == [w for _, w in mixed]             # the table holds every class of error the planners return, and valid jobs
    hr, got, groups = batch(em, jobs)
    assert got == want
    assert hr == next(w for w in want if w)
    assert all((g == NONE) == (w != 0) for g, w in zip(groups, want))
    # valid jobs only: S_OK; the lowest-index failure wins wherever it sits
    assert batch(em, [j for j, w in mixed if w == 0])[0] == 0
    assert mixed[26][1] == F.E_POINTER and mixed[0][1] == F.E_INVALIDARG
    assert batch(em, [mixed[1][0], mixed[26][0], mixed[0][0]])[0] == F.E_POINTER


def test_library_answers_every_failing_job_without_a_device():
    """a batch of failing jobs plans as the emulator does and never reaches a device"""
    mixed = [(j, w) for j, w in _mixed() if w]
    table = (capi.TexconvJob * len(mixed))(*[j.job for j, _ in mixed])
    results = (C.c_int32 * len(mixed))()
    hr = F.hr_u32(L.dxb200_texconv_batch(table, len(mixed), results))
    assert [F.hr_u32(r) for r in results] == [w for _, w in mixed]
    assert hr == mixed[0][1]
    assert all(j.opaque.value == -1 for j, _ in mixed)
    # no results array: the same answer
    assert F.hr_u32(L.dxb200_texconv_batch(table, len(mixed), None)) == mixed[0][1]


def test_no_jobs_and_unknown_kind_are_invalid():
    assert F.hr_u32(L.dxb200_texconv_batch(None, 1, None)) == F.E_INVALIDARG
    j = Job("gen", 28, 16, 16, 1, 5, 77)
    table = (capi.TexconvJob * 1)(j.job)
    results = (C.c_int32 * 1)(7)
    assert F.hr_u32(L.dxb200_texconv_batch(table, 0, results)) == F.E_INVALIDARG
    assert results[0] == 7                           # nothing is written
    table[0].kind = 3
    assert F.hr_u32(L.dxb200_texconv_batch(table, 1, results)) == F.E_INVALIDARG
    assert F.hr_u32(results[0]) == F.E_INVALIDARG


BASE = ("gen", 28, 32, 32, 1, 6, 77)
# one planned field changed each: the job does not share the base job's group
CHANGES = {
    "kind": dict(entry="lev"),
    "base_format": dict(bf=29),
    "base_width": dict(w=16),
    "base_height": dict(h=64, levels=6),
    "levels": dict(levels=5),
    "source": dict(src_kw=dict(width=64, height=64)),
    "swizzle": dict(ch_kw=dict(swizzle=(2, 1, 0, 3))),
    "colour_key": dict(ch_kw=dict(color_key=0x102030)),
    "steps": dict(steps=PM),
    "ts": dict(ts_kw=DM),
    "dst_format": dict(df=98),
    "flags": dict(flags=UNIFORM),
    "threshold": dict(threshold=0.25),
    "scan": dict(scan=False),
}


def _job(**kw):
    entry, bf, w, h, items, levels, df = BASE
    a = dict(entry=entry, bf=bf, w=w, h=h, items=items, levels=levels, df=df)
    a.update(kw)
    return Job(**a)


def test_pointers_and_pitches_share_a_group(em):
    jobs = [_job(), _job(items=3), _job(row_pitch=16), _job(row_pitch=4, offset=4), _job(offset=1 << 20)]
    hr, got, groups = batch(em, jobs)
    assert hr == 0 and got == [0] * len(jobs)
    assert groups == [0] * len(jobs)


@pytest.mark.parametrize("field", sorted(CHANGES))
def test_a_planned_field_splits_the_group(field, em):
    changed = _job(**CHANGES[field])
    assert changed.single_hr(em) == 0, field
    hr, got, groups = batch(em, [_job(), changed, _job()])
    assert hr == 0 and got == [0, 0, 0]
    assert groups == [0, 1, 0], field


def test_colour_keys_and_swizzles_that_differ_split(em):
    for a, b in ((dict(color_key=0x102030), dict(color_key=0x102031)), (dict(swizzle=(2, 1, 0, 3)), dict(swizzle=(1, 0, 2, 3)))):
        assert batch(em, [_job(ch_kw=a), _job(ch_kw=b), _job(ch_kw=a)])[2] == [0, 1, 0]


def test_group_order_item_order_and_chunk_plans(em):
    """groups in the order of their first job; units group by group, each group's items in job order; each group's chunk plan is
    its single call's"""
    shapes = [_job(), _job(entry="conv", bf=10, df=28, levels=5, ch_kw=dict(swizzle=(2, 1, 0, 3))), _job(w=64, h=64, levels=7),
              _job(entry="lev", bf=77, df=98)]
    jobs = [shapes[0], shapes[1], _job(items=2), shapes[2], Job(*CASES[0][1:12]), _job(entry="conv", bf=10, df=28, levels=5,
            ch_kw=dict(swizzle=(2, 1, 0, 3)), items=3), shapes[3], _job(w=64, h=64, levels=7)]
    hr, got, groups = batch(em, jobs)
    assert hr == F.E_INVALIDARG and got == [0, 0, 0, 0, F.E_INVALIDARG, 0, 0, 0]
    assert groups == [0, 1, 0, 2, NONE, 1, 3, 2]
    weights, _ = split(em, 1, 3 + 4 + 2 + 1)
    # the bytes of each item's level 0 in the chain: 32 x 32 RGBA8 (the Convert's chain is dst), 64 x 64 RGBA8, 32 x 32 RGBA8 that
    # the kept BC3 levels decompress to
    assert weights == [4096] * 7 + [16384] * 2 + [4096]
    for g, shape in enumerate(shapes):
        em.emul_batch_chunk_plan(g)
        grouped = _chunk_plan(em)
        assert shape.single_hr(em) == 0
        single = _chunk_plan(em)
        assert grouped[:4] == single[:4], g


@pytest.mark.parametrize("devices", [1, 2, 3, 8])
def test_units_split_contiguously_by_bytes(devices, em):
    jobs = [_job(items=9), _job(w=64, h=64, levels=7), _job(entry="lev", bf=77, df=98, items=2), _job(w=16, h=16, levels=5, items=3)]
    assert batch(em, jobs)[0] == 0
    n = 9 + 1 + 2 + 3
    weights, cut = split(em, devices, n)
    assert weights == [4096] * 9 + [16384] + [4096] * 2 + [1024] * 3
    assert cut == contiguous_by_bytes(weights, devices)
    assert cut[0] == 0 and cut[-1] == n and cut == sorted(cut)
    if devices == 2:
        assert 0 < cut[1] < 9                         # the first group is split across the two devices


def test_one_unit_runs_on_one_device(em):
    assert batch(em, [_job()])[0] == 0
    assert split(em, 8, 1)[1] == [0, 1]
