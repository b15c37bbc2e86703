"""Per-stream language models in batched streaming on the device (tests/stream_lms.py): every call of every stream
equals, bit for bit, partial_decode_beams on a decoder built with that stream's model of the call; the streaming
goldens that share an alphabet and call settings pass as the streams of one batched call; start states are laid out
and checked per stream; and 64 streams at the C3 shape meet the contract on every call."""
import pytest

from tests import stream_lms as sl
from tests import synth
from tests import utt_lms as ul

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


@pytest.fixture(scope="module")
def char_sets(pkg):
    return ul.Sets(pkg, "char")


def _decoder(pkg, sets, own="A"):
    return pkg.BeamSearchDecoderCTC(pkg.Alphabet.build_alphabet(sets.labels), sets.lm[own] if own else None)


@pytest.mark.parametrize("variant", ["plain", "force", "prune", "beam1", "beam100", "hot", "switch"])
def test_gpu_stream_lms_contract(pkg, char_sets, variant):
    sets = char_sets
    xs = sl.streams(sets.wl)
    calls = [sets.models(sets.names(len(xs)))] * (len(sl.BOUNDS) - 1)
    kw = dict(beam_width=16)
    if variant == "force":
        kw["force_next_word"] = True
    elif variant == "prune":
        kw["prune_history"] = True
    elif variant == "beam1":
        kw["beam_width"] = 1
    elif variant == "beam100":
        kw["beam_width"] = 100
    elif variant == "hot":
        wl = sets.wl
        base = [pkg.HotwordScorer.build_scorer([wl.words[3 + i], wl.words[20 + i]], weight=6.0 + i) if i % 3 else None
                for i in range(len(xs))]
        kw["scorers_per_call"] = [base] * len(calls)
    elif variant == "switch":
        calls = [list(c) for c in calls]
        for c, name in enumerate(["A", "B", "none", "AB", "A"]):
            calls[c][0] = sets.lm[name]
    sl.stream_chunks(sets, _decoder(pkg, sets, own="A" if variant != "plain" else None), xs, calls, **kw)


def test_gpu_stream_lms_contract_bpe(pkg):
    sets = ul.Sets(pkg, "bpe")
    xs = sl.streams(sets.wl, n=6, T=(60, 0, 45, 13))
    calls = [sets.models(sets.names(len(xs), ["A", "B", "none"]))] * 4
    sl.stream_chunks(sets, _decoder(pkg, sets), xs, calls, bounds=[0, 1, 8, 40, 60], beam_width=16)


@pytest.mark.parametrize("names", sl.golden_groups(), ids=lambda names: names[0])
def test_gpu_stream_lms_golden(pkg, names):
    assert sl.run_golden_group(pkg, names) >= 1


def test_gpu_stream_lms_not_vacuous(pkg, char_sets):
    xs = [char_sets.wl.utterance(700 + i, 120, "diffuse") for i in range(12)]
    assert sl.differs(char_sets, _decoder(pkg, char_sets, own=None), xs, char_sets.names(12), bounds=[0, 50, 100, 120],
                      beam_width=24) >= 4


def test_gpu_stream_lms_start_states(pkg, char_sets):
    sl.check_start_states(pkg, char_sets, _decoder(pkg, char_sets))
    sl.check_own_model_states(char_sets, _decoder(pkg, char_sets, own="B"))
    sl.check_errors(pkg, char_sets, _decoder(pkg, char_sets))


def test_gpu_stream_lms_c3_shape(pkg):
    """64 streams at the C3 shape (V = 32, 3-gram models over 20k words, beam 100, 50-frame chunks, T = 1000): four
    models, every fifth stream without one; every call of every stream against a decoder built with its model."""
    wls = [synth.CharWorkload("B", n_words=20000, lm_order=3, seed=s) for s in (1, 2, 3)]
    models = [pkg.LanguageModel(pkg.NgramModel(w.arpa), w.words, alpha=0.5, beta=1.0) for w in wls]
    models.append(pkg.LanguageModel(pkg.NgramModel(wls[0].arpa), wls[0].words, alpha=0.9, beta=2.0))
    alphabet = pkg.Alphabet.build_alphabet(wls[0].labels)
    refs = {id(m): pkg.BeamSearchDecoderCTC(alphabet, m) for m in models + [None]}
    lms = [None if i % 5 == 4 else models[i % 4] for i in range(64)]
    xs = wls[0].batch(1, 64, 1000, "peaky")
    dec = pkg.BeamSearchDecoderCTC(alphabet, None)
    caches = [sl.start(dec, lm) for lm in lms]
    b_beams = [list(dec.get_starting_state()[0]) for _ in lms]
    for t0 in range(0, 1000, 50):
        last = t0 + 50 >= 1000
        out = dec.partial_decode_beams_batch([x[t0:t0 + 50] for x in xs], caches, b_beams, [t0] * 64, beam_width=100,
                                             language_model_list=lms, is_end=last)
        for i, lm in enumerate(lms):
            ref_dec = refs[id(lm)]
            ref = ref_dec.partial_decode_beams(xs[i][t0:t0 + 50], ref_dec.get_starting_state()[1], {}, b_beams[i], t0,
                                               beam_width=100, is_end=last)
            assert out[i] == ref, "stream %d frames %d.." % (i, t0)
        b_beams = out
    assert dec.last_timings()["kernel_variant"] == 0
