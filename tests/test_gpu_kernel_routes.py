"""Every beam-kernel instantiation and the arena-overflow retry pass on the H100 (`pytest -m gpu`), case by case against
the oracle, with the instantiations each call launched asserted from b2c_timings_t.kernels.  The route table is in
tests/kernel_routes.py; tests/test_hostsim_kernel_routes.py asserts the same routes on the CPU simulation build.

Only the device runs the warp-count-dependent code of the one- and two-warp class kernels (classes 128 and 256), of
the 512-thread general kernel and of the 256-thread kernels (hostsim simulates 8 warps for every CTA)."""
import pytest

from tests import kernel_routes as kr

pytestmark = pytest.mark.gpu

ROUTES = kr.route_cases()
RETRIES = kr.retry_cases()


@pytest.fixture(scope="module")
def pkg():
    import __graft_entry__ as g
    g.build()
    import pyctcdecode_b200
    from pyctcdecode_b200 import _lib
    _lib._lib = None  # the real CUDA library, not a test build
    L = _lib.lib()
    assert _lib.library_path() == _lib.DEFAULT_LIBRARY
    if L.b2c_device_count() < 1:
        pytest.skip("no CUDA device on this machine (the GPU tests need one)")
    kr.reset_families()
    yield pyctcdecode_b200
    kr.reset_families()


@pytest.fixture(scope="module")
def orc():
    from oracle import oracle
    oracle.build()
    return oracle


@pytest.fixture(scope="module")
def n_sm(pkg):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_gpu_kernel_routes_case_table_covers_every_instantiation():
    names = [c[0] for c in ROUTES] + [c[0] for c in RETRIES]
    assert len(names) == len(set(names))
    assert {c[6] for c in ROUTES} == set(kr.BITS.values()) == set(range(13))


@pytest.mark.parametrize("case", ROUTES, ids=[c[0] for c in ROUTES])
def test_gpu_kernel_route(pkg, orc, n_sm, case, monkeypatch):
    kr.run_route_case(pkg, orc, case, n_sm, monkeypatch)


@pytest.mark.parametrize("case", RETRIES, ids=[c[0] for c in RETRIES])
def test_gpu_retry_pass(pkg, orc, case, monkeypatch):
    kr.run_retry_case(pkg, orc, case, monkeypatch)


def test_gpu_natural_overflow(pkg, orc, monkeypatch):
    kr.set_env(monkeypatch, {})
    kr.run_natural_overflow(pkg, orc)
