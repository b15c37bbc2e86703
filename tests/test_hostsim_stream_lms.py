"""Hostsim twin of tests/test_gpu_stream_lms.py: per-stream language models in batched streaming, in the CPU simulation
build of the kernels; the start-state layout and its checks through the C ABI."""
import ctypes as C
import os
import subprocess

import pytest

from tests import stream_lms as sl
from tests import utt_lms as ul

HOSTSIM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
LIB = os.path.join(HOSTSIM, "libb200ctc_hostsim.so")


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


def _decoder(sim, sets, own="A"):
    return sim.BeamSearchDecoderCTC(sim.Alphabet.build_alphabet(sets.labels), sets.lm[own] if own else None)


def _calls(sets, names, n_calls=len(sl.BOUNDS) - 1):
    return [sets.models(names)] * n_calls


@pytest.mark.parametrize("variant", ["plain", "force", "prune", "beam1", "beam100", "hot", "switch"])
def test_hostsim_stream_lms_contract(sim, char_sets, variant):
    sets = char_sets
    xs = sl.streams(sets.wl)
    names = sets.names(len(xs))
    calls = _calls(sets, names)
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
        base = [sim.HotwordScorer.build_scorer([wl.words[3 + i], wl.words[20 + i]], weight=6.0 + i) if i % 3 else None
                for i in range(len(xs))]
        kw["scorers_per_call"] = [base] * len(calls)
    elif variant == "switch":
        # stream 0 goes A -> B -> none -> AB -> A: its carried words are replayed through the model of each call
        calls = [list(c) for c in calls]
        for c, name in enumerate(["A", "B", "none", "AB", "A"]):
            calls[c][0] = sets.lm[name]
    # the decoder's own model is never used: a decoder with model A and one without give the same
    sl.stream_chunks(sets, _decoder(sim, sets, own="A" if variant != "plain" else None), xs, calls, **kw)


def test_hostsim_stream_lms_contract_bpe(sim):
    sets = ul.Sets(sim, "bpe")
    xs = sl.streams(sets.wl, n=6, T=(60, 0, 45, 13))
    names = sets.names(len(xs), ["A", "B", "none"])
    sl.stream_chunks(sets, _decoder(sim, sets), xs, _calls(sets, names, 4), bounds=[0, 1, 8, 40, 60], beam_width=16)


@pytest.mark.parametrize("names", sl.golden_groups(), ids=lambda names: names[0])
def test_hostsim_stream_lms_golden(sim, names):
    assert sl.run_golden_group(sim, names) >= 1


def test_hostsim_stream_lms_not_vacuous(sim, char_sets):
    xs = [char_sets.wl.utterance(700 + i, 120, "diffuse") for i in range(12)]
    assert sl.differs(char_sets, _decoder(sim, char_sets, own=None), xs, char_sets.names(12), bounds=[0, 50, 100, 120],
                      beam_width=24) >= 4


def test_hostsim_stream_lms_start_states(sim, char_sets):
    sl.check_start_states(sim, char_sets, _decoder(sim, char_sets))


def test_hostsim_stream_lms_own_model_states(sim, char_sets):
    sl.check_own_model_states(char_sets, _decoder(sim, char_sets, own="B"))


def test_hostsim_stream_lms_errors(sim, char_sets):
    sl.check_errors(sim, char_sets, _decoder(sim, char_sets))


def test_hostsim_stream_lms_abi(sim, char_sets):
    """The C ABI with utt_lm_set: the start-state layout of a call with sets of different widths, the row width the
    caller states, the checks of every state that is read, streaming calls, and per-beam LM states equal to single
    calls (float32 logits, B2C_DTYPE_F32)."""
    sets = char_sets
    from pyctcdecode_b200 import _lib
    L = _lib.lib()
    handle = _decoder(sim, sets)._handle(None)
    wl = sets.wl
    xs = [wl.utterance(11, 60), wl.utterance(12, 60), wl.utterance(13, 60)]
    ptrs = (C.c_void_p * 3)(*[x.ctypes.data for x in xs])
    Ts = (C.c_int32 * 3)(60, 60, 60)
    a, b = sets.lm["A"], sets.lm["B"]
    lm_sets = (_lib.LmSet * 3)()
    for k, ms in enumerate([[a], [a, b], []]):
        lm_sets[k].n_models = len(ms)
        for j, m in enumerate(ms):
            lm_sets[k].models[j] = m.ngram_model._h()
            lm_sets[k].alpha[j], lm_sets[k].beta[j], lm_sets[k].unk_score_offset[j] = m.alpha, m.beta, m.unk_score_offset
            lm_sets[k].lm_score_boundary[j] = int(m.score_boundary)

    def call(idx=(0, 1, 2), **extra):
        opts = _lib.DecodeOpts()
        L.b2c_decode_opts_default(C.byref(opts))
        opts.beam_width = 8
        opts.max_out_beams = 8
        opts.lm_sets = C.cast(lm_sets, C.POINTER(_lib.LmSet))
        opts.n_lm_sets = 3
        arr = (C.c_int32 * 3)(*idx)
        opts.utt_lm_set = C.cast(arr, C.POINTER(C.c_int32))
        for k, v in extra.items():
            setattr(opts, k, v)
        res = C.c_void_p()
        rc = L.b2c_decode_batch(handle, ptrs, Ts, 3, 0, 0, C.byref(opts), C.byref(res))     # float32 logits
        return rc, res

    # start states, rows of two (the largest set): utterance 0 (set A) reads slot 0, utterance 1 (set AB) both,
    # utterance 2 (no model) nothing.  The slots that are not read hold states the check would refuse.
    own = {0: a, 1: sim.MultiLanguageModel([a, b]), 2: None}
    carried = {u: sets.ref(own[u]).decode_beams(xs[(u + 1) % 3], beam_width=8)[0].last_lm_state for u in (0, 1)}
    start = (_lib.LMState * 6)()
    start[0] = carried[0]._to_c()
    start[2], start[3] = carried[1].states[0]._to_c(), carried[1].states[1]._to_c()
    for k in (1, 4, 5):
        start[k].length = 99
    states = C.cast(start, C.POINTER(_lib.LMState))
    # the caller states the row width: missing or wrong is B2C_E_ARG
    for width in (0, 1, 3):
        assert call(lm_start_states=states, lm_start_width=width)[0] == -1, width
        assert "lm_start_width" in L.b2c_last_error().decode("utf-8")
    rc, res = call(lm_start_states=states, lm_start_width=2)
    assert rc == 0, L.b2c_last_error()
    try:
        for u in range(3):
            want = sets.ref(own[u]).decode_beams(xs[u], beam_width=8, lm_start_state=carried.get(u))
            assert L.b2c_result_n_beams(res, u) == len(want) > 0
            for k, w in enumerate(want):
                assert L.b2c_result_text(res, u, k).decode("utf-8") == w.text
                assert L.b2c_result_lm_score(res, u, k) == w.lm_score
    finally:
        L.b2c_result_free(res)
    # every state that is read is checked: a length above 5, a word id outside its model's vocabulary
    for slot, field, value in ((0, "length", 6), (3, "length", 6), (2, "words", 10 ** 6), (3, "words", 10 ** 6)):
        bad = (_lib.LMState * 6)()
        C.memmove(bad, start, C.sizeof(start))
        if field == "length":
            bad[slot].length = value
        else:
            bad[slot].length = max(1, bad[slot].length)
            bad[slot].words[0] = value
        assert call(lm_start_states=C.cast(bad, C.POINTER(_lib.LMState)), lm_start_width=2)[0] == -1, (slot, field)
        assert "lm_start_states" in L.b2c_last_error().decode("utf-8")
    # streaming with utt_lm_set: three empty streams (EMPTY_START_BEAM) need their rows of start states
    streams = C.cast((_lib.StreamState * 3)(), C.POINTER(_lib.StreamState))
    assert call(stream_states=streams)[0] == -1
    assert "lm_start_states" in L.b2c_last_error().decode("utf-8")
    rc, res = call(stream_states=streams, lm_start_states=states, lm_start_width=2)
    assert rc == 0, L.b2c_last_error()
    L.b2c_result_free(res)
    # per-beam LM states of an offline call (the kernels' default start states) equal single calls
    rc, res = call()
    assert rc == 0
    try:
        for u, own_lm in own.items():
            ref = sets.ref(own_lm)
            rh = ref._handle(None)
            opts = _lib.DecodeOpts()
            L.b2c_decode_opts_default(C.byref(opts))
            opts.beam_width = 8
            opts.max_out_beams = 8
            for idx, m in enumerate(ref._lm_list()):
                L.b2c_decoder_set_params_lm(rh, idx, m.alpha, m.beta, m.unk_score_offset, int(m.score_boundary))
            one = C.c_void_p()
            assert L.b2c_decode_batch(rh, C.cast(C.byref(ptrs, u * C.sizeof(C.c_void_p)), C.POINTER(C.c_void_p)),
                                      C.cast(C.byref(Ts, 4 * u), C.POINTER(C.c_int32)), 1, 0, 0, C.byref(opts), C.byref(one)) == 0
            try:
                nb = L.b2c_result_n_beams(res, u)
                assert nb == L.b2c_result_n_beams(one, 0) > 0
                for beam in range(nb):
                    for j in range(3):
                        s1, s2 = _lib.LMState(), _lib.LMState()
                        r1 = L.b2c_result_lm_state_at(res, u, beam, j, C.byref(s1))
                        r2 = L.b2c_result_lm_state_at(one, 0, beam, j, C.byref(s2))
                        assert r1 == r2, (u, beam, j)
                        assert bytes(s1) == bytes(s2) or r1 == 0, (u, beam, j)
            finally:
                L.b2c_result_free(one)
    finally:
        L.b2c_result_free(res)
