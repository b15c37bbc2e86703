"""Hostsim twin of tests/test_gpu_device_text.py: decode_batch transcripts written and joined by the kernel code on the
CPU simulation build, against decode_beams_batch's host-built top beam and the oracle (tests/device_text.py)."""
import os
import subprocess

import pytest

from oracle import oracle as orc
from tests import device_text as dt
from tests import kernel_routes as kr

HOSTSIM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")


@pytest.fixture(scope="module")
def sim():
    subprocess.check_call(["make", "-s", "-C", HOSTSIM])
    import pyctcdecode_b200
    from pyctcdecode_b200 import _lib
    _lib.use_library(os.path.join(HOSTSIM, "libb200ctc_hostsim.so"))
    orc.build()
    kr.reset_families()
    yield pyctcdecode_b200
    _lib._lib = None
    kr.reset_families()


@pytest.mark.parametrize("case", dt.CASES, ids=[c[0] for c in dt.CASES])
def test_hostsim_device_text(sim, case, monkeypatch):
    dt.run_case(sim, orc, case, monkeypatch)
