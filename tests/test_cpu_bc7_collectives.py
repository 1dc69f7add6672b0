"""Host branches of the primitives of the pruned BC7 shape ranking (dxb_warp.cuh: half-warp ballot to a 64-bit mask, n-th set bit,
warp-wide max; dxb_bc7.cuh: s8 x s8 dp4a) against exact references (tests/bc7_ranking/collectives.cu).  The device branches are
checked against the same references on the same inputs by tests/test_gpu_bc7_collectives.py, so device == emulator there."""
import pytest

from tests import bc7_ranking_build as B


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    L = B.host_lib("collectives.cu", tmp_path_factory.mktemp("bc7_collectives_host"))
    assert L.coll_on_device() == 0
    return L


@pytest.mark.parametrize("arg,count", B.COLLECTIVE_DOMAINS, ids=lambda v: B.COLLECTIVE_NAMES.get(v, str(v)))
def test_host_collective_equals_reference(lib, arg, count):
    n, rec = B.run_collective(lib, arg, count)
    assert n == 0, "%s: %d mismatches, first (input, got, want) = %#x, %#x, %#x" % ((B.COLLECTIVE_NAMES[arg], n) + rec)
