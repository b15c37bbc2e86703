"""The streaming stage's token lists on the hostsim build (kernel logic on the CPU), case by case against the reference
of tests/streaming_stage.py.  hostsim compiles the `#else` twins of the device-only K1 routines, so this does not
replace tests/test_gpu_streaming_stage.py; it keeps the definition, the host routes and the read-back testable here.
Device-tensor routes need a GPU and are left to the GPU file."""
import os
import subprocess

import pytest

from oracle import oracle as orc
from tests import streaming_stage, synth

HOSTSIM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
CASES = synth.streaming_stage_cases(device_routes=False)


@pytest.fixture(scope="module")
def sim():
    subprocess.check_call(["make", "-s", "-C", HOSTSIM])
    import pyctcdecode_b200
    from pyctcdecode_b200 import _lib
    _lib.use_library(os.path.join(HOSTSIM, "libb200ctc_hostsim.so"))
    orc.build()
    yield pyctcdecode_b200
    _lib._lib = None


@pytest.fixture(scope="module")
def decoders(sim):
    cache = {}

    def get(V):
        if V not in cache:
            cache[V] = sim.build_ctcdecoder(synth.stream_labels(V))
        return cache[V]
    return get


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_hostsim_streaming_stage_token_lists(sim, decoders, case, monkeypatch):
    monkeypatch.setenv("B200CTC_PIPELINE", "1")
    monkeypatch.setenv("B200CTC_PIPELINE_ALL", "1")
    V = case[1]
    streaming_stage.run_case(orc, decoders(V), case, fresh_decoder=lambda: sim.build_ctcdecoder(synth.stream_labels(V)))
