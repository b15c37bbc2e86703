"""decode_batch transcripts written by b2c_finalize's walk and joined on the H100 (`pytest -m gpu`), against
decode_beams_batch's host-built top beam and the oracle, on every route, the retry pass, chunked, gated, pipelined and
hinted calls (tests/device_text.py; tests/test_hostsim_device_text.py runs the same cases on the CPU build)."""
import pytest

from tests import device_text as dt
from tests import kernel_routes as kr

pytestmark = pytest.mark.gpu


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


@pytest.mark.parametrize("case", dt.CASES, ids=[c[0] for c in dt.CASES])
def test_gpu_device_text(pkg, orc, case, monkeypatch):
    dt.run_case(pkg, orc, case, monkeypatch)
