"""The picture call with slice tables other than the packed one a decoder stages: every slice's blocks a few blocks apart in the
coefficient buffer, the blocks between them covered by no slice.  Each block's slice then comes from the search over the table rather
than from the picture geometry; the pictures must equal the reference decoder's all the same, and the uncovered blocks write nothing."""
import pytest

import hostsim_build
import prores_util as U


@pytest.fixture(scope="session")
def pref(built):
    lib = U.ref()
    if lib is None:
        pytest.skip("oracle/_ref not built (no reference tree in this environment)")
    return lib


def run(lib, mem, pref, gap):
    decs = [U.Decoded(pref, spec, seed=60 + k) for k, spec in enumerate(U.SMALL_STREAMS)]
    rc, got = U.run_pictures(lib, mem, decs, gap=gap)
    assert rc == 0
    for d, g in zip(decs, got):
        U.check_frame(d, g)


@pytest.mark.parametrize("gap", [1, 3, 40])
def test_spread_slices_cpu(built, pref, gap):
    run(hostsim_build.load(), U.HostMem(), pref, gap)


@pytest.mark.gpu
@pytest.mark.parametrize("gap", [1, 3, 40])
def test_spread_slices_gpu(gpu, pref, gap):
    run(gpu.lib, U.DevMem(), pref, gap)
