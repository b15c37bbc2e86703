"""Hostsim twin of tests/test_gpu_stream_ends.py: per-stream is_end and force_next_word in batched streaming, in the
CPU simulation build of the kernels; the utt_finalize_mode field through the C ABI."""
import os
import subprocess

import pytest

from tests import stream_ends as se
from tests import stream_lms as sl
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


def test_hostsim_stream_ends_plan():
    se.check_plan(CALLS, len(se.POOL_T))


@pytest.mark.parametrize("variant", ["none", "own", "lms", "hot", "prune", "beam1", "beam100", "beam300"])
def test_hostsim_stream_ends_contract(sim, char_sets, variant):
    kw = dict(beam_width=16)
    if variant == "prune":
        kw["prune_history"] = True
    elif variant.startswith("beam"):
        kw["beam_width"] = int(variant[4:])
    se.run(_streams(sim, char_sets, variant), CALLS, **kw)


def test_hostsim_stream_ends_contract_bpe(sim):
    # BPE: force_next_break resets at every call, whatever the stream's mode
    sets = ul.Sets(sim, "bpe")
    Ts = (60, 0, 45, 13, 1, 30, 52, 8)
    calls = se.plan(Ts, 4, chunks=(1, 7, 20))
    se.check_plan(calls, len(Ts))
    xs = [sets.wl.utterance(600 + s, T, "diffuse" if s % 2 else "peaky") for s, T in enumerate(Ts)]
    se.run(se.Streams(_decoder(sim, sets), xs), calls, beam_width=16)
    se.run(se.Streams(_decoder(sim, sets, own=None), xs, sets, sets.models(sets.names(len(xs), ["A", "B", "none"]))), calls,
           beam_width=16)


def test_hostsim_stream_ends_uniform(sim, char_sets):
    xs = [char_sets.wl.utterance(700 + i, 90, "diffuse" if i % 2 else "peaky") for i in range(6)]
    se.check_uniform(_decoder(sim, char_sets), xs, beam_width=16)
    se.check_uniform(_decoder(sim, char_sets, own=None), xs, beam_width=16)


def test_hostsim_stream_ends_not_vacuous(sim, char_sets):
    _, differ = se.run(_streams(sim, char_sets, "own"), CALLS, count_differs=True, beam_width=16)
    assert differ >= 6, differ


@pytest.mark.parametrize("names", sl.golden_groups(), ids=lambda names: names[0])
def test_hostsim_stream_ends_golden(sim, names):
    assert se.run_golden_group(sim, names) == se.golden_steps(names)


def test_hostsim_stream_ends_retry_and_chunks(sim, char_sets, monkeypatch):
    """B200CTC_TEXT_ARENA=1: the first pass overflows the text arena of every stream that commits a word, the retry pass
    decodes them again with their own modes; `retried` is the number of such streams (the sum over the single-stream
    references) and the results equal the calls without the switch.  B200CTC_FORCE_CHUNKS=3 changes nothing."""
    st = _streams(sim, char_sets, "lms")
    want, _ = se.run(st, CALLS, beam_width=16)
    monkeypatch.setenv("B200CTC_TEXT_ARENA", "1")
    timings = []
    got, _ = se.run(st, CALLS, timings=timings, beam_width=16)
    assert got == want
    assert sum(r for _, r in timings) > 0
    for tm, retried in timings:
        assert tm["retried"] == retried, (tm["retried"], retried)
    assert any(0 < r < len(call) for (_, r), call in zip(timings, CALLS))
    monkeypatch.delenv("B200CTC_TEXT_ARENA")
    monkeypatch.setenv("B200CTC_FORCE_CHUNKS", "3")
    assert se.run(st, CALLS, beam_width=16)[0] == want


def test_hostsim_stream_ends_errors(sim, char_sets):
    xs = [char_sets.wl.utterance(40 + i, 30) for i in range(4)]
    se.check_errors(_decoder(sim, char_sets), xs)


def test_hostsim_stream_ends_abi(sim, char_sets):
    xs = [char_sets.wl.utterance(50 + i, 45, "diffuse" if i % 2 else "peaky") for i in range(6)]
    se.check_abi(_decoder(sim, char_sets), xs)
