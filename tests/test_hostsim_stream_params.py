"""Hostsim twin of tests/test_gpu_stream_params.py: per-stream beam width, pruning thresholds and history pruning in
batched streaming, in the CPU simulation build of the kernels; the utt_* search-parameter fields through the C ABI."""
import os
import subprocess

import pytest

from oracle import oracle as orc
from tests import stream_ends as se
from tests import stream_params as sp
from tests import synth
from tests import utt_lms as ul

HOSTSIM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
LIB = os.path.join(HOSTSIM, "libb200ctc_hostsim.so")
CALLS = se.plan(se.POOL_T, 6)


@pytest.fixture(scope="module")
def sim():
    subprocess.check_call(["make", "-s", "-C", HOSTSIM])
    import pyctcdecode_b200
    from pyctcdecode_b200 import _lib
    _lib.use_library(LIB)
    orc.build()
    yield pyctcdecode_b200
    _lib._lib = None


@pytest.fixture(scope="module")
def char_sets(sim):
    return ul.Sets(sim, "char")


def _xs(sets, Ts=se.POOL_T):
    return [sets.wl.utterance(900 + s, T, "diffuse" if s % 2 else "peaky") for s, T in enumerate(Ts)]


def _decoder(sim, sets, own="A"):
    return sim.BeamSearchDecoderCTC(sim.Alphabet.build_alphabet(sets.labels), sets.lm[own] if own else None)


def _streams(sim, sets, variant):
    xs = _xs(sets)
    if variant == "none":
        return se.Streams(_decoder(sim, sets, own=None), xs)
    if variant == "lms":
        # the decoder's own model is never used: every stream has its entry, AB a MultiLanguageModel
        return se.Streams(_decoder(sim, sets), xs, sets, sets.models(sets.names(len(xs))))
    if variant == "hot":
        wl = sets.wl
        scorers = [sim.HotwordScorer.build_scorer([wl.words[3 + s], wl.words[20 + s]], weight=6.0 + s) if s % 3 else None
                   for s in range(len(xs))]
        return se.Streams(_decoder(sim, sets), xs, scorers=scorers)
    return se.Streams(_decoder(sim, sets), xs)


@pytest.mark.parametrize("variant", ["none", "own", "lms", "hot"])
def test_hostsim_stream_params_contract(sim, char_sets, variant):
    outs, differ = sp.run(_streams(sim, char_sets, variant), CALLS, count_differs=True)
    assert differ > 0
    sp.check_not_empty(outs)


def test_hostsim_stream_params_contract_scalars(sim, char_sets):
    # other scalars for the None entries, and no None entries at all
    sp.run(_streams(sim, char_sets, "own"), CALLS, beam_width=7, beam_prune_logp=-3.0, token_min_logp=-2.0, prune_history=True)
    sp.run(_streams(sim, char_sets, "own"), CALLS, nones=False)


def test_hostsim_stream_params_contract_bpe(sim):
    sets = ul.Sets(sim, "bpe")
    Ts = (60, 0, 45, 13, 1, 30, 52, 8)
    calls = se.plan(Ts, 4, chunks=(1, 7, 20))
    xs = [sets.wl.utterance(600 + s, T, "diffuse" if s % 2 else "peaky") for s, T in enumerate(Ts)]
    _, differ = sp.run(se.Streams(_decoder(sim, sets), xs), calls, count_differs=True)
    assert differ > 0
    sp.run(se.Streams(_decoder(sim, sets, own=None), xs, sets, sets.models(sets.names(len(xs), ["A", "B", "none"]))), calls)


def test_hostsim_stream_params_uniform(sim, char_sets):
    xs = [char_sets.wl.utterance(700 + i, 90, "diffuse" if i % 2 else "peaky") for i in range(6)]
    sp.check_uniform(_decoder(sim, char_sets), xs, beam_width=16)
    sp.check_uniform(_decoder(sim, char_sets, own=None), xs, beam_width=16, prune_history=True, token_min_logp=-3.0)


@pytest.mark.parametrize("case", sp.K1_CASES, ids=lambda c: "%s-V%d-%s" % c)
def test_hostsim_stream_params_token_lists(sim, case):
    content, V, dtype = case
    sp.check_token_lists(orc, sim.build_ctcdecoder(synth.stream_labels(V)), content, V, dtype)


def test_hostsim_stream_params_retry(sim, char_sets, monkeypatch):
    """B200CTC_TEXT_ARENA=1: the retry pass decodes the overflowing streams again with their own parameters; `retried`
    is the number of such streams and the results equal the calls without the switch."""
    st = _streams(sim, char_sets, "lms")
    want, _ = sp.run(st, CALLS)
    monkeypatch.setenv("B200CTC_TEXT_ARENA", "1")
    timings = []
    got, _ = sp.run(st, CALLS, timings=timings)
    assert got == want
    assert sum(r for _, r in timings) > 0
    for tm, retried in timings:
        assert tm["retried"] == retried, (tm["retried"], retried)
    assert any(0 < r < len(call) for (_, r), call in zip(timings, CALLS))


def test_hostsim_stream_params_errors(sim, char_sets):
    xs = [char_sets.wl.utterance(40 + i, 30) for i in range(4)]
    sp.check_errors(_decoder(sim, char_sets), xs)


def test_hostsim_stream_params_abi(sim, char_sets):
    xs = [char_sets.wl.utterance(50 + i, 45, "diffuse" if i % 2 else "peaky") for i in range(6)]
    sp.check_abi(_decoder(sim, char_sets), xs)
