"""Per-stream search parameters in batched streaming on the device (tests/stream_params.py): in continuous-batching
schedules that mix widths 1 to 2000, prune thresholds, token thresholds and both history settings, every call of every
stream equals, bit for bit, partial_decode_beams with that stream's own parameters; lists that repeat the scalars equal
the scalars; the streaming stage's token lists follow each stream's threshold; the retry pass keeps the results; the
errors; and 64 streams at the C3 shape in three parameter tiers meet the contract on every call."""
import pytest

from oracle import oracle as orc
from tests import stream_ends as se
from tests import stream_params as sp
from tests import synth
from tests import utt_lms as ul

pytestmark = pytest.mark.gpu
CALLS = se.plan(se.POOL_T, 6)
WIDTHS = sp.WIDTHS + (2000,)


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


def _wide(s):
    return sp.params_of(s, WIDTHS)


@pytest.mark.parametrize("variant", ["none", "own", "lms", "hot"])
def test_gpu_stream_params_contract(pkg, char_sets, variant):
    outs, differ = sp.run(_streams(pkg, char_sets, variant), CALLS, params=_wide, count_differs=True)
    assert differ > 0
    sp.check_not_empty(outs)


def test_gpu_stream_params_contract_scalars(pkg, char_sets):
    sp.run(_streams(pkg, char_sets, "own"), CALLS, params=_wide, beam_width=7, beam_prune_logp=-3.0, token_min_logp=-2.0,
           prune_history=True)
    sp.run(_streams(pkg, char_sets, "own"), CALLS, params=_wide, nones=False)


def test_gpu_stream_params_contract_bpe(pkg):
    sets = ul.Sets(pkg, "bpe")
    Ts = (60, 0, 45, 13, 1, 30, 52, 8)
    calls = se.plan(Ts, 4, chunks=(1, 7, 20))
    xs = [sets.wl.utterance(600 + s, T, "diffuse" if s % 2 else "peaky") for s, T in enumerate(Ts)]
    _, differ = sp.run(se.Streams(_decoder(pkg, sets), xs), calls, params=_wide, count_differs=True)
    assert differ > 0
    sp.run(se.Streams(_decoder(pkg, sets, own=None), xs, sets, sets.models(sets.names(len(xs), ["A", "B", "none"]))), calls,
           params=_wide)


def test_gpu_stream_params_uniform(pkg, char_sets):
    xs = [char_sets.wl.utterance(700 + i, 90, "diffuse" if i % 2 else "peaky") for i in range(6)]
    sp.check_uniform(_decoder(pkg, char_sets), xs, beam_width=16)
    sp.check_uniform(_decoder(pkg, char_sets, own=None), xs, beam_width=16, prune_history=True, token_min_logp=-3.0)


@pytest.mark.parametrize("case", sp.K1_CASES, ids=lambda c: "%s-V%d-%s" % c)
def test_gpu_stream_params_token_lists(pkg, case):
    orc.build()
    content, V, dtype = case
    sp.check_token_lists(orc, pkg.build_ctcdecoder(synth.stream_labels(V)), content, V, dtype)


def test_gpu_stream_params_retry(pkg, char_sets, monkeypatch):
    st = _streams(pkg, char_sets, "lms")
    want, _ = sp.run(st, CALLS, params=_wide)
    monkeypatch.setenv("B200CTC_TEXT_ARENA", "1")
    timings = []
    got, _ = sp.run(st, CALLS, params=_wide, timings=timings)
    assert got == want
    assert sum(r for _, r in timings) > 0
    for tm, retried in timings:
        assert tm["retried"] == retried, (tm["retried"], retried)
    assert any(0 < r < len(call) for (_, r), call in zip(timings, CALLS))


def test_gpu_stream_params_errors(pkg, char_sets):
    xs = [char_sets.wl.utterance(40 + i, 30) for i in range(4)]
    sp.check_errors(_decoder(pkg, char_sets), xs)
    xs = [char_sets.wl.utterance(50 + i, 45, "diffuse" if i % 2 else "peaky") for i in range(6)]
    sp.check_abi(_decoder(pkg, char_sets), xs)


def test_gpu_stream_params_c3_shape(pkg):
    """64 slots at the C3 shape (V = 32, a 3-gram model over 20k words, 50-frame chunks), 96 streams of 400 to 1000
    frames in three parameter tiers (beam 100 / 128 / 16): every call of every stream against partial_decode_beams with
    its own parameters and flags."""
    dec, base = se.c3_streams(pkg)
    Ts = se.staggered(96)
    calls = se.plan(Ts, 64, chunks=(50,))
    xs = [base[j % len(base)][:T] for j, T in enumerate(Ts)]
    outs, differ = sp.run(se.Streams(dec, xs), calls, params=sp.tiers((100, 128, 16)), nones=False, count_differs=True)
    assert differ > 0
