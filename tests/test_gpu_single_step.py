"""The one-token step after a multi-token frame (b2c_fast_single_step) on the device: every case of
tests/single_step.py in every capacity variant of the latency-first kernel, against the oracle and bit for bit
against the same frames taken by the general step (B200CTC_NO_SINGLE_STEP=1)."""
import pytest

from tests import single_step

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pkg():
    import __graft_entry__ as g
    g.build()
    import pyctcdecode_b200
    from pyctcdecode_b200 import _lib
    _lib._lib = None  # make sure the real CUDA library is bound, not a test build
    L = _lib.lib()
    assert _lib.library_path() == _lib.DEFAULT_LIBRARY
    if L.b2c_device_count() < 1:
        pytest.skip("no CUDA device on this machine (the GPU tests need one)")
    return pyctcdecode_b200


@pytest.mark.parametrize("variant", ["0", "1", "2"])
def test_gpu_single_token_step(pkg, variant, monkeypatch):
    from oracle import oracle
    oracle.build()
    monkeypatch.setenv("B200CTC_V5_VARIANT", variant)
    monkeypatch.setenv("B200CTC_FORCE_V5", "1")
    wl = single_step.workload()
    dec = pkg.build_ctcdecoder(wl.labels)
    n = single_step.check_decoder(dec, oracle.OracleDecoder(wl.labels), wl, monkeypatch)
    assert n > 1000 if variant == "0" else n == 0      # compiled into the CAP 1024 variant only
    assert dec.last_timings()["kernel_variant"] == 2
