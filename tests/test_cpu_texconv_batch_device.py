"""CPU suite: where dxb200_texconv_batch_device keeps each plane of a chunk, without a device, through the planners on the host
(tests/emul/texconv_batch_device.cpp, emul_device_plan, which plans a job record as the batch does).  For every routing case of test_cpu_chain_routing and every valid plan of
test_cpu_texconv_steps: a plane aliased to the caller's base is never written by a step, so inputs stay as they are; Dst is always
the caller's; a plane with an uploaded image that a step writes lies in scratch and is copied in; chunks are cut exactly as the
host staging cuts them, and a chunk's scratch bytes are its staged bytes less those of its aliased planes, laid out where the staging
buffer would hold them.  Failing jobs answer as dxb200_texconv_batch answers them, without a device."""
import ctypes as C
import os

import pytest

from directxtex_b200 import capi, formats as F
from tests.bc7_ranking_build import host_lib
from tests.test_cpu_chain_routing import CASES as ROUTES, FILTER
from tests.test_cpu_texconv_batch import Job, _mixed
from tests.test_cpu_texconv_steps import CASES, PLANS, SAME

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = capi.lib
BASE, DST = 0, 4                    # plane roles (PlaneRole)
UP = 0                              # Copy::Up
ALL = 1 << 40                       # a budget that keeps every item in one chunk


@pytest.fixture(scope="module")
def em(tmp_path_factory):
    E = host_lib("texconv_batch_device.cpp", tmp_path_factory.mktemp("texconv_batch_device_emul"), os.path.join(ROOT, "tests", "emul"))
    E.emul_device_plan.argtypes = [C.POINTER(capi.TexconvJob), C.c_size_t, C.POINTER(C.c_uint64), C.c_size_t, C.POINTER(C.c_size_t)]
    E.emul_device_plan.restype = C.c_int32
    return E


def _device_plan(em, j, budget):
    """(HRESULT of j's planner, [(role, aliased, first copy, rest copy)] per plane, [(kind, source role, destination role, cover)] per
    step, [(first item, end item, staged, scratch, laid out, keeps caller pixels, [bytes per plane])] per chunk)"""
    out = (C.c_uint64 * 4096)()
    n = C.c_size_t(0)
    hr = F.hr_u32(em.emul_device_plan(C.byref(j.job), budget, out, len(out), C.byref(n)))
    if hr:
        return hr, None, None, None
    w = list(out[:n.value])
    np_ = w[0]
    planes = [tuple(w[1 + 4 * p: 5 + 4 * p]) for p in range(np_)]
    at = 1 + 4 * np_
    steps = [tuple(w[at + 1 + 4 * s: at + 5 + 4 * s]) for s in range(w[at])]
    at += 1 + 4 * w[at]
    chunks = []
    for _ in range(w[at]):
        head = w[at + 1: at + 7]
        chunks.append(tuple(head) + (w[at + 7: at + 7 + np_],))
        at += 6 + np_
    assert at + 1 == len(w)
    return hr, planes, steps, chunks


def _job(entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps, ts_kw, scan, filter=0):
    j = Job(entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps, ts_kw, scan=scan)
    if entry != "lev":
        j.job.filter = filter
    return j


def check_placement(em, name, j, items):
    _, planes, steps, _ = _device_plan(em, j, ALL)
    written = {d for _, _, d, _ in steps}
    roles = [r for r, _, _, _ in planes]
    assert DST in roles, name
    for role, aliased, first, rest in planes:
        if role == DST:
            assert aliased, name
        if aliased:
            assert role in (BASE, DST), name
            if role == BASE:
                assert role not in written, name                 # the caller's inputs are never written
        if UP in (first, rest) and role in written:
            assert not aliased, name                             # copied into scratch
        if role == BASE and role not in written:
            assert aliased, name                                 # no copy where none is needed
    for budget in (0, ALL):
        _, _, _, chunks = _device_plan(em, j, budget)
        assert [(c[0], c[1]) for c in chunks] == ([(i, i + 1) for i in range(items)] if budget == 0 else [(0, items)]), name
        for i, k, staged, scratch, laid, keeps, per_plane in chunks:
            assert staged == sum(per_plane), name
            assert scratch == staged - sum(b for b, p in zip(per_plane, planes) if p[1]), name
            assert laid == scratch and keeps == 1, name


@pytest.mark.parametrize("case", ROUTES, ids=[c[0] for c in ROUTES])
def test_routing_cases(case, em):
    name, entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps, ts_kw, scan = case[:13]
    j = _job(entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps, ts_kw, scan, FILTER)
    assert _device_plan(em, j, ALL)[0] == 0, name
    check_placement(em, name, j, items)


def _texconv_steps_entries():
    """every entry of test_cpu_texconv_steps that plans: its valid plans, its NULL-steps cases, and its failing cases with their
    change undone"""
    out = []
    for p in PLANS:
        name, entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps, ts_kw = p[:12]
        out.append((name, entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps, ts_kw))
    for entry, bf, items, levels, df, src_kw, ch_kw, steps in SAME:
        out.append(("same_%s_%d_%d" % (entry, bf, df), entry, bf, 16, 16, items, levels, df, src_kw, ch_kw, steps, {}))
    for c in CASES:
        name, entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps, ts_kw = c[:12]
        out.append(("fixed_" + name, entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps, ts_kw))
    return out


@pytest.mark.parametrize("scan", [False, True], ids=["no_scan", "scan"])
def test_texconv_steps_entries(scan, em):
    planned = 0
    for name, entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps, ts_kw in _texconv_steps_entries():
        j = _job(entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps, ts_kw, scan)
        if _device_plan(em, j, ALL)[0] != 0:
            continue                        # a case whose check is not the change it makes
        planned += 1
        check_placement(em, name, j, items)
    assert planned >= len(PLANS) + len(SAME)


# routing case -> whether its base plane is the caller's (None: no base plane, level 0 goes straight into the chain)
BASE_ALIASED = {
    "rgba16f_swizzle_convert": False,                       # the swizzle in front of a Convert runs on the base
    "rgba8_demultiply_copy_color_key_premultiply": False,   # the demultiply runs on the base
    "rgba8_demultiply_convert": False,
    "bc3_pass_through": True,
    "bc3_to_bc7": True,
    "bc1_resize_convert_scan": True,
    "rgba16f_resize_swizzle_to_bc7": True,
    "rgba8_to_bc3_scan": None,
    "rgba8_demultiply_to_bc7": None,
}


@pytest.mark.parametrize("name", sorted(BASE_ALIASED))
def test_base_written_in_place_is_copied(name, em):
    """the steps the host staging runs in place on the uploaded base make the base a scratch copy; otherwise it is the caller's"""
    case = next(c for c in ROUTES if c[0] == name)
    _, entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps, ts_kw, scan = case[:13]
    hr, planes, _, _ = _device_plan(em, _job(entry, bf, w, h, items, levels, df, src_kw, ch_kw, steps, ts_kw, False, FILTER), ALL)
    assert hr == 0
    base = [bool(a) for r, a, _, _ in planes if r == BASE]
    assert base == ([] if BASE_ALIASED[name] is None else [BASE_ALIASED[name]])
    assert [bool(a) for r, a, _, _ in planes if r not in (BASE, DST)] == [False] * (len(planes) - len(base) - 1)


def test_failing_jobs_answer_as_the_host_batch_without_a_device():
    mixed = [(j, w) for j, w in _mixed() if w]
    table = (capi.TexconvJob * len(mixed))(*[j.job for j, _ in mixed])
    results = (C.c_int32 * len(mixed))()
    hr = F.hr_u32(L.dxb200_texconv_batch_device(table, len(mixed), results, None))
    assert [F.hr_u32(r) for r in results] == [w for _, w in mixed]
    assert hr == mixed[0][1]
    assert all(j.opaque.value == -1 for j, _ in mixed)
    assert F.hr_u32(L.dxb200_texconv_batch_device(table, len(mixed), None, None)) == mixed[0][1]
    assert F.hr_u32(L.dxb200_texconv_batch_device(None, 1, None, None)) == F.E_INVALIDARG
    assert F.hr_u32(L.dxb200_texconv_batch_device(table, 0, results, None)) == F.E_INVALIDARG
