"""GPU suite for the dense sweep of Resize and GenerateMipMaps extents (tests/resize_sweep.py): every case through the host API.

Each case runs with DXB200_OPT_MIP_KERNELS = 0 and 1 by test_gpu_mip_routes.check_route_and_result: option 0 moves the launch
counters of exactly the kernel families resize_sweep.route() expects, option 1 only k_mip_level's, the two agree bit for bit, and
both equal the oracle bit for bit (with TEX_FILTER_SRGB: the generic kernel level by level within one code, DESIGN.md section
3).  BOX on extents that do not halve exactly fails with E_FAIL, as on the oracle, and launches nothing.  A seeded tenth of the
cases also runs through the device API with rows 16 bytes wider than tight and with rows 4 bytes wider and the base 4 bytes off
(where 8- and 16-byte pixels leave k_mip_sep for k_mip_tile); its bytes equal the host API's.

A host test runs one group of cases (operation, filter, format, sRGB), a device test one operation and filter; each reports
every case that fails, not only the first."""
import contextlib
import io

import numpy as np
import pytest

from directxtex_b200 import capi, formats as F
from tests import resize_sweep as S, test_gpu_mip_routes as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _init():
    assert capi.lib.dxb200_init(0) == 0


def check_fails(oracle, c, src):
    """BOX on sizes that do not halve exactly: E_FAIL from the library and the oracle, and no launch"""
    before = {f: capi.kernel_launch_count(f) for f in R.FAMILIES}
    with pytest.raises(capi.DxTexError) as e:
        R.run_host(c, [src])
    assert e.value.hr == F.E_FAIL, (R.case_id(c), hex(e.value.hr))
    hr = oracle.resize(src, c.w, c.h, c.fmt, c.resize[0], c.resize[1], c.fl)[0] if c.resize else \
        oracle.generate_mipmaps(src, c.w, c.h, c.fmt, c.fl)[0]
    assert hr == F.E_FAIL, (R.case_id(c), hex(hr))
    assert {f: capi.kernel_launch_count(f) for f in R.FAMILIES} == before, R.case_id(c)


def check_all(oracle, cases, one):
    """one(oracle, c) on every case; fails listing every case that failed"""
    bad = []
    with contextlib.redirect_stdout(io.StringIO()):
        for c in cases:
            try:
                one(oracle, c)
            except (AssertionError, capi.DxTexError) as e:
                bad.append("%s: %s" % (R.case_id(c), str(e)[:300]))
    assert not bad, "%d of %d cases failed:\n%s" % (len(bad), len(cases), "\n".join(bad[:40]))


def check_host(oracle, c):
    srcs = R.sources(c)
    if not c.fams:
        check_fails(oracle, c, srcs[0])
    else:
        R.check_route_and_result(oracle, c, srcs)


def check_device(oracle, c):
    srcs = R.sources(c)
    dev = R.check_route_and_result(oracle, c, srcs)
    host = R.run(c._replace(layout="host"), srcs, 0)[0]
    for l in range(len(dev)):
        assert np.array_equal(dev[l], host[l]), (R.case_id(c), "device != host", l)


@pytest.mark.parametrize("key", S.GROUP_KEYS, ids=S.group_id)
def test_sweep_host(oracle, key):
    check_all(oracle, S.host_groups()[key], check_host)


@pytest.mark.parametrize("key", S.DEVICE_KEYS, ids=S.group_id)
def test_sweep_device(oracle, key):
    check_all(oracle, S.device_groups()[key], check_device)
