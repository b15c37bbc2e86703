"""Hostsim twin of tests/test_gpu_kernel_routes.py: the route of every case (b2c_timings_t.kernels, cta_threads,
cap_candidates) and the retry pass on the CPU simulation build of the kernels, against the oracle.  The launch plan and
the kernel bit are host code shared with the CUDA build, and hostsim reports 4 SMs; so every route assertion holds here
before it runs on a GPU.  hostsim runs each CTA with 8 simulated warps, so the warp-count-dependent code of the one-
and two-warp kernels is left to the GPU file."""
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle as orc
from tests import kernel_routes as kr

HOSTSIM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
HOSTSIM_SMS = 4            # cudaDevAttrMultiProcessorCount of tests/hostsim/cuda_shim.h
ROUTES = kr.route_cases()
RETRIES = kr.retry_cases()


@pytest.fixture(scope="module")
def sim():
    subprocess.check_call(["make", "-s", "-C", HOSTSIM])
    import pyctcdecode_b200
    from pyctcdecode_b200 import _lib
    _lib.use_library(os.path.join(HOSTSIM, "libb200ctc_hostsim.so"))
    orc.build()
    yield pyctcdecode_b200
    _lib._lib = None
    kr.reset_families()


def test_hostsim_kernel_routes_case_table_covers_every_instantiation():
    names = [c[0] for c in ROUTES] + [c[0] for c in RETRIES]
    assert len(names) == len(set(names))
    assert {c[6] for c in ROUTES} == set(kr.BITS.values()) == set(range(13))
    for b in kr.GENERAL_BITS:
        assert any(c[6] == b for c in ROUTES)


@pytest.mark.parametrize("case", ROUTES, ids=[c[0] for c in ROUTES])
def test_hostsim_kernel_route(sim, case, monkeypatch):
    kr.run_route_case(sim, orc, case, HOSTSIM_SMS, monkeypatch)


@pytest.mark.parametrize("case", RETRIES, ids=[c[0] for c in RETRIES])
def test_hostsim_retry_pass(sim, case, monkeypatch):
    kr.run_retry_case(sim, orc, case, monkeypatch)


def test_hostsim_kernel_route_switch_errors(sim, monkeypatch):
    fam = kr.family(sim, orc, "b32")
    dec = fam.decoder()
    xs = fam.batch(4, 30, seed=5)
    for bad in ("5", "6", "x", "-1"):
        kr.set_env(monkeypatch, {"B200CTC_FORCE_CLASS": bad})
        with pytest.raises(ValueError, match="B200CTC_FORCE_CLASS"):
            dec.decode_batch(None, xs, beam_width=16)
    kr.set_env(monkeypatch, {"B200CTC_FORCE_CLASS": "4"})
    with pytest.raises(ValueError, match="does not fit"):
        dec.decode_batch(None, xs, beam_width=128)
    # below 1 the arena is clamped to the root node: still exact
    kr.set_env(monkeypatch, {"B200CTC_TEXT_ARENA": "0"})
    got = dec.decode_batch(None, xs, beam_width=16, language_model_list=[fam.lm] * 4)
    kr.set_env(monkeypatch, {})
    assert got == dec.decode_batch(None, xs, beam_width=16, language_model_list=[fam.lm] * 4)


def test_hostsim_natural_overflow(sim, monkeypatch):
    kr.set_env(monkeypatch, {})
    kr.run_natural_overflow(sim, orc)
