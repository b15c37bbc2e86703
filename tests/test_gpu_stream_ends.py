"""Per-stream is_end and force_next_word in batched streaming on the device (tests/stream_ends.py): in
continuous-batching schedules every call of every stream equals, bit for bit, partial_decode_beams with that stream's
own flags; lists that give every stream the same flags equal the scalar flags; the streaming goldens of one group pass
with one batched call per step; the retry pass and forced chunks keep the results; the errors; and 64 streams at the
C3 shape with staggered lengths meet the contract on every call."""
import pytest

from tests import stream_ends as se
from tests import stream_lms as sl
from tests import utt_lms as ul

pytestmark = pytest.mark.gpu
CALLS = se.plan(se.POOL_T, 6)


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


@pytest.fixture(scope="module")
def char_sets(pkg):
    return ul.Sets(pkg, "char")


def _xs(sets, Ts=se.POOL_T):
    return [sets.wl.utterance(900 + s, T, "diffuse" if s % 2 else "peaky") for s, T in enumerate(Ts)]


def _decoder(pkg, sets, own="A"):
    return pkg.BeamSearchDecoderCTC(pkg.Alphabet.build_alphabet(sets.labels), sets.lm[own] if own else None)


def _streams(pkg, sets, variant):
    xs = _xs(sets)
    if variant == "none":
        return se.Streams(_decoder(pkg, sets, own=None), xs)
    if variant == "lms":
        return se.Streams(_decoder(pkg, sets), xs, sets, sets.models(sets.names(len(xs))))
    if variant == "hot":
        wl = sets.wl
        scorers = [pkg.HotwordScorer.build_scorer([wl.words[3 + s], wl.words[20 + s]], weight=6.0 + s) if s % 3 else None
                   for s in range(len(xs))]
        return se.Streams(_decoder(pkg, sets), xs, scorers=scorers)
    return se.Streams(_decoder(pkg, sets), xs)


@pytest.mark.parametrize("variant", ["none", "own", "lms", "hot", "prune", "beam1", "beam100", "beam300"])
def test_gpu_stream_ends_contract(pkg, char_sets, variant):
    kw = dict(beam_width=16)
    if variant == "prune":
        kw["prune_history"] = True
    elif variant.startswith("beam"):
        kw["beam_width"] = int(variant[4:])
    se.run(_streams(pkg, char_sets, variant), CALLS, **kw)


def test_gpu_stream_ends_contract_bpe(pkg):
    sets = ul.Sets(pkg, "bpe")
    Ts = (60, 0, 45, 13, 1, 30, 52, 8)
    calls = se.plan(Ts, 4, chunks=(1, 7, 20))
    se.check_plan(calls, len(Ts))
    xs = [sets.wl.utterance(600 + s, T, "diffuse" if s % 2 else "peaky") for s, T in enumerate(Ts)]
    se.run(se.Streams(_decoder(pkg, sets), xs), calls, beam_width=16)
    se.run(se.Streams(_decoder(pkg, sets, own=None), xs, sets, sets.models(sets.names(len(xs), ["A", "B", "none"]))), calls,
           beam_width=16)


def test_gpu_stream_ends_uniform(pkg, char_sets):
    xs = [char_sets.wl.utterance(700 + i, 90, "diffuse" if i % 2 else "peaky") for i in range(6)]
    se.check_uniform(_decoder(pkg, char_sets), xs, beam_width=16)
    se.check_uniform(_decoder(pkg, char_sets, own=None), xs, beam_width=16)


def test_gpu_stream_ends_not_vacuous(pkg, char_sets):
    _, differ = se.run(_streams(pkg, char_sets, "own"), CALLS, count_differs=True, beam_width=16)
    assert differ >= 6, differ


@pytest.mark.parametrize("names", sl.golden_groups(), ids=lambda names: names[0])
def test_gpu_stream_ends_golden(pkg, names):
    assert se.run_golden_group(pkg, names) == se.golden_steps(names)


def test_gpu_stream_ends_retry_and_chunks(pkg, char_sets, monkeypatch):
    st = _streams(pkg, char_sets, "lms")
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


def test_gpu_stream_ends_errors(pkg, char_sets):
    xs = [char_sets.wl.utterance(40 + i, 30) for i in range(4)]
    se.check_errors(_decoder(pkg, char_sets), xs)
    xs = [char_sets.wl.utterance(50 + i, 45, "diffuse" if i % 2 else "peaky") for i in range(6)]
    se.check_abi(_decoder(pkg, char_sets), xs)


def test_gpu_stream_ends_c3_shape(pkg):
    """64 slots at the C3 shape (V = 32, a 3-gram model over 20k words, beam 100, 50-frame chunks), 96 streams of 400 to
    1000 frames: streams end at many different calls and new ones take their slots; every call of every stream against
    partial_decode_beams with its own flags."""
    dec, base = se.c3_streams(pkg)
    Ts = se.staggered(96)
    calls = se.plan(Ts, 64, chunks=(50,))
    se.check_plan(calls, len(Ts))
    xs = [base[j % len(base)][:T] for j, T in enumerate(Ts)]
    se.run(se.Streams(dec, xs), calls, beam_width=100)
