"""GPU tier: the pairing families of tests/pairing_cases.py through the sm_90a build of the harness (one thread per
record, 64-thread blocks as k_verify_miller's): Fp12 products against Python integers, and every output — the Miller
loop on twist points outside the r-torsion included — equal limb for limb to both host builds."""
import pytest

import pairing_cases as PC

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    return PC.DevPairing()


@pytest.fixture(scope="module")
def hosts():
    return [PC.HostPairing(True), PC.HostPairing(False)]


@pytest.mark.parametrize("family", list(PC.FAMILIES))
def test_pairing_edges_gpu(dev, hosts, family):
    fails, got = PC.run_family(dev, family)
    assert fails == {}
    for h in hosts:
        want = PC.run_family(h, family)[1]
        for op in got:
            assert (got[op] == want[op]).all(), op
