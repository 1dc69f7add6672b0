"""Device branches (sm_90a, the library's flags) of the primitives of the pruned BC7 shape ranking against the exact references of
tests/bc7_ranking/collectives.cu; tests/test_cpu_bc7_collectives.py checks the host branches on the same inputs."""
import pytest

from tests import bc7_ranking_build as B


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    L = B.device_lib("collectives.cu", tmp_path_factory.mktemp("bc7_collectives_device"))
    assert L.coll_on_device() == 1
    return L


@pytest.mark.gpu
@pytest.mark.parametrize("arg,count", B.COLLECTIVE_DOMAINS, ids=lambda v: B.COLLECTIVE_NAMES.get(v, str(v)))
def test_device_collective_equals_reference(lib, arg, count):
    n, rec = B.run_collective(lib, arg, count)
    assert n == 0, "%s: %d mismatches, first (input, got, want) = %#x, %#x, %#x" % ((B.COLLECTIVE_NAMES[arg], n) + rec)
