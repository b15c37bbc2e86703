"""Hostsim twin of tests/test_gpu_single_step.py: the one-token step after a multi-token frame
(b2c_fast_single_step) in the CPU simulation build, in every capacity variant and with the work items of every phase
replayed in other orders (B200CTC_HOSTSIM_ORDER, read once per process: a child process per order)."""
import os
import subprocess
import sys

import pytest

from oracle import oracle as orc
from tests import single_step

HOSTSIM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def sim():
    subprocess.check_call(["make", "-s", "-C", HOSTSIM])
    import pyctcdecode_b200
    from pyctcdecode_b200 import _lib
    _lib.use_library(os.path.join(HOSTSIM, "libb200ctc_hostsim.so"))
    yield pyctcdecode_b200
    _lib._lib = None


@pytest.mark.parametrize("variant", ["0", "1", "2"])
def test_hostsim_single_token_step(sim, variant, monkeypatch):
    monkeypatch.setenv("B200CTC_V5_VARIANT", variant)
    monkeypatch.setenv("B200CTC_FORCE_V5", "1")
    wl = single_step.workload()
    dec = sim.build_ctcdecoder(wl.labels)
    n = single_step.check_decoder(dec, orc.OracleDecoder(wl.labels), wl, monkeypatch)
    assert n > 1000 if variant == "0" else n == 0      # compiled into the CAP 1024 variant only
    assert dec.last_timings()["kernel_variant"] == 2


@pytest.mark.parametrize("order", ["1", "2", "3"])
def test_hostsim_single_token_step_work_item_order(order):
    code = ("import pytest, sys; from tests import single_step; from oracle import oracle as orc; "
            "from pyctcdecode_b200 import _lib; import pyctcdecode_b200 as p; "
            "_lib.use_library(%r); wl = single_step.workload(); mp = pytest.MonkeyPatch(); "
            "n = single_step.check_decoder(p.build_ctcdecoder(wl.labels), orc.OracleDecoder(wl.labels), wl, mp); "
            "sys.exit(0 if n > 1000 else 3)") % os.path.join(HOSTSIM, "libb200ctc_hostsim.so")
    subprocess.check_call(["make", "-s", "-C", HOSTSIM])
    env = dict(os.environ, B200CTC_HOSTSIM_ORDER=order, B200CTC_V5_VARIANT="0", B200CTC_FORCE_V5="1", PYTHONPATH=ROOT)
    subprocess.check_call([sys.executable, "-c", code], cwd=ROOT, env=env)
