"""Hostsim twin of tests/test_gpu_utt_lms.py: per-utterance language models in the CPU simulation build of the kernels,
in the latency-first variants and the general kernel, and with the work items of every phase replayed in other orders
(B200CTC_HOSTSIM_ORDER, read once per process: a child process per order)."""
import ctypes as C
import os
import subprocess
import sys
import threading

import pytest

from oracle import oracle as orc
from tests import utt_lms as ul

HOSTSIM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
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


@pytest.mark.parametrize("kind", ["char", "bpe"])
@pytest.mark.parametrize("prune_history", [False, True])
def test_hostsim_utt_lms_contract(sim, char_sets, kind, prune_history):
    sets = char_sets if kind == "char" else ul.Sets(sim, "bpe")
    n = 12 if kind == "char" else 6
    names = sets.names(n) if kind == "char" else sets.names(n, ["A", "B", "none"])
    dec = _decoder(sim, sets)
    xs = ul.batch(sets.wl, n=n)
    got = ul.check_contract(sets, dec, xs, sets.models(names), beam_width=24, prune_history=prune_history)
    ul.check_oracle(sets, orc, xs, names, got, beam_width=24, prune_history=prune_history)


@pytest.mark.parametrize("variant", ["0", "1", "2", "general"])
def test_hostsim_utt_lms_kernels(sim, char_sets, variant, monkeypatch):
    if variant == "general":
        bw = 160                  # above the latency-first kernel's 128 beams
    else:
        monkeypatch.setenv("B200CTC_FORCE_V5", "1")
        monkeypatch.setenv("B200CTC_V5_VARIANT", variant)
        bw = 32
    # a MultiLanguageModel set sends the whole call to the general kernel
    names = char_sets.names(12, ul.NAMES if variant == "general" else ["A", "B", "A_params", "A_no_unigrams", "none"])
    dec = _decoder(sim, char_sets)
    xs = ul.batch(char_sets.wl)
    ul.check_contract(char_sets, dec, xs, char_sets.models(names), beam_width=bw)
    ul.check_route(dec, variant)


def test_hostsim_utt_lms_inputs(sim, char_sets, monkeypatch):
    """A padded block with lengths, a host block called three times (pipelined), a ragged host list called twice
    (hinted), chunked launches, hotwords."""
    sets = char_sets
    dec = _decoder(sim, sets, own=None)
    xs = ul.batch(sets.wl)
    lms = sets.models(sets.names(len(xs)))
    block, lengths = ul.padded(xs)
    ul.check_contract(sets, dec, xs, lms, batch_input=block, lengths=lengths, beam_width=16)
    same = [sets.wl.utterance(500 + i, 320, "diffuse") for i in range(6)]
    lms6 = sets.models(sets.names(6, ["A", "none", "B"]))
    block6, _ = ul.padded(same)
    ul.check_pipelined(sets, _decoder(sim, sets, own=None), same, lms6, block6, monkeypatch, beam_width=16)
    # hinted plans exist for single-model sets only (a MultiLanguageModel set takes the general kernel)
    ragged = [sets.wl.utterance(500 + i, 300 + 7 * i, "peaky") for i in range(8)]
    ul.check_hinted(sets, _decoder(sim, sets, own=None), ragged, sets.models(sets.names(8, ["A", "none", "B", "A_params"])),
                    beam_width=16)
    hot = [[sets.wl.words[3]], None, [sets.wl.words[5], sets.wl.words[9]], None, [sets.wl.words[1]], None]
    ul.check_contract(sets, dec, same, lms6, beam_width=16, hotwords_list=hot)
    monkeypatch.setenv("B200CTC_FORCE_CHUNKS", "3")
    monkeypatch.setenv("B200CTC_FORCE_V5", "1")
    ul.check_contract(sets, dec, same, lms6, beam_width=16)


def test_hostsim_utt_lms_not_vacuous(sim, char_sets):
    seeds = [700 + i for i in range(12)]
    xs = [char_sets.wl.utterance(s, 120, "diffuse") for s in seeds]
    assert ul.differs(char_sets, _decoder(sim, char_sets), xs, char_sets.names(12), beam_width=24) >= 4


def test_hostsim_utt_lms_mixed_special_steps(sim, char_sets, monkeypatch):
    monkeypatch.setenv("B200CTC_FORCE_V5", "1")
    monkeypatch.setenv("B200CTC_V5_VARIANT", "0")
    dec = _decoder(sim, char_sets, own=None)
    total = ul.mixed_special_steps(char_sets, dec, ul.batch(char_sets.wl), beam_width=32)
    assert total["inplace_frames"] > 0 and total["single_frames"] > 0


def test_hostsim_utt_lms_reset_params(sim, char_sets):
    """Parameters are read at call time: reset_params on a model applies to the next batched call."""
    sets = ul.Sets(sim, "char")
    dec = _decoder(sim, sets, own=None)
    xs = ul.batch(sets.wl, n=4)
    lms = [sets.lm["A"]] * 4
    ul.check_contract(sets, dec, xs, lms, beam_width=16)
    sets.lm["A"].reset_params(alpha=1.4, beta=-0.5)
    ul.check_contract(sets, dec, xs, lms, beam_width=16)


def test_hostsim_utt_lms_threads(sim, char_sets):
    """Two decoders share the same model objects; 8 threads call them with language_model_list at once."""
    sets = char_sets
    decs = [_decoder(sim, sets), _decoder(sim, sets, own=None)]
    xs = ul.batch(sets.wl, n=6)
    jobs = [(decs[j % 2], sets.models(sets.names(6, ul.NAMES[j % 3:] + ul.NAMES[:j % 3]))) for j in range(8)]
    want = [d.decode_batch(None, xs, beam_width=16, language_model_list=lms) for d, lms in jobs]
    got = [None] * len(jobs)

    def run(j):
        d, lms = jobs[j]
        got[j] = d.decode_batch(None, xs, beam_width=16, language_model_list=lms)

    threads = [threading.Thread(target=run, args=(j,)) for j in range(len(jobs))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert got == want


def test_hostsim_utt_lms_errors(sim, char_sets):
    sets = char_sets
    dec = _decoder(sim, sets)
    xs = [sets.wl.utterance(1, 30), sets.wl.utterance(2, 30)]
    with pytest.raises(ValueError):
        dec.decode_batch(None, xs, language_model_list=[sets.lm["A"]])
    with pytest.raises(ValueError):
        dec.decode_beams_batch(None, xs, language_model_list=sets.lm["A"])

    from pyctcdecode_b200.language_model import AbstractLanguageModel

    class Other(AbstractLanguageModel):
        pass

    with pytest.raises(TypeError):
        dec.decode_batch(None, xs, language_model_list=[Other.__new__(Other), None])
    five = sim.MultiLanguageModel([sets.lm["A"], sets.lm["B"], sets.lm["A_params"], sets.lm["A_no_unigrams"], sets.lm["A"]])
    with pytest.raises(ValueError):
        dec.decode_batch(None, xs, language_model_list=[five, None])
    _abi(sim, sets, dec)


def _abi(sim, sets, dec):
    """B2C_E_ARG from the C ABI, and per-beam LM states from the C accessors equal to single calls."""
    from pyctcdecode_b200 import _lib
    L = _lib.lib()
    handle = dec._handle(None)
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

    def call(idx, **extra):
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
        rc = L.b2c_decode_batch(handle, ptrs, Ts, 3, 1, 0, C.byref(opts), C.byref(res))
        return rc, res

    assert call((0, 3, 1))[0] == -1
    assert call((0, -1, 1))[0] == -1
    start = (_lib.LMState * 3)()
    assert call((0, 1, 2), lm_start_states=C.cast(start, C.POINTER(_lib.LMState)))[0] == -1
    streams = (_lib.StreamState * 3)()          # three empty streams (EMPTY_START_BEAM): valid on their own
    assert call((0, 1, 2), stream_states=C.cast(streams, C.POINTER(_lib.StreamState)))[0] == -1
    rc, res = call((0, 1, 2), stream_states=C.cast(streams, C.POINTER(_lib.StreamState)), utt_lm_set=None)
    assert rc == 0
    L.b2c_result_free(res)
    lm_sets[2].n_models = 5
    assert call((0, 1, 1))[0] == -1
    lm_sets[2].n_models = 1
    assert call((0, 1, 1))[0] == -1             # set 2 now holds a NULL model
    lm_sets[2].n_models = 0
    rc, res = call((0, 1, 2))
    assert rc == 0
    try:
        for u, own in enumerate([a, sim.MultiLanguageModel([a, b]), None]):
            ref = sets.ref(own)
            rh = ref._handle(None)
            opts = _lib.DecodeOpts()
            L.b2c_decode_opts_default(C.byref(opts))
            opts.beam_width = 8
            opts.max_out_beams = 8
            for idx, m in enumerate(ref._lm_list()):
                L.b2c_decoder_set_params_lm(rh, idx, m.alpha, m.beta, m.unk_score_offset, int(m.score_boundary))
            one = C.c_void_p()
            assert L.b2c_decode_batch(rh, C.cast(C.byref(ptrs, u * C.sizeof(C.c_void_p)), C.POINTER(C.c_void_p)),
                                      C.cast(C.byref(Ts, 4 * u), C.POINTER(C.c_int32)), 1, 1, 0, C.byref(opts), C.byref(one)) == 0
            try:
                nb = L.b2c_result_n_beams(res, u)
                assert nb == L.b2c_result_n_beams(one, 0)
                for beam in range(nb):
                    for j in range(3):
                        s1, s2 = _lib.LMState(), _lib.LMState()
                        r1 = L.b2c_result_lm_state_at(res, u, beam, j, C.byref(s1))
                        r2 = L.b2c_result_lm_state_at(one, 0, beam, j, C.byref(s2))
                        assert r1 == r2, (u, beam, j)
                        assert bytes(s1) == bytes(s2) or r1 == 0, (u, beam, j)
            finally:
                L.b2c_result_free(one)
        pk = _lib.Packed()
        assert L.b2c_result_packed(res, C.byref(pk)) == 0
        assert pk.n_models == 2
    finally:
        L.b2c_result_free(res)


@pytest.mark.parametrize("order", ["1", "2", "3"])
def test_hostsim_utt_lms_work_item_order(order):
    code = ("import sys; from tests import utt_lms as ul; from pyctcdecode_b200 import _lib; "
            "import pyctcdecode_b200 as p; _lib.use_library(%r); sets = ul.Sets(p, 'char'); "
            "dec = p.BeamSearchDecoderCTC(p.Alphabet.build_alphabet(sets.labels), sets.lm['A']); "
            "xs = [sets.wl.utterance(300 + i, 90, 'diffuse') for i in range(6)]; "
            "ul.check_contract(sets, dec, xs, sets.models(sets.names(6)), beam_width=24)") % LIB
    subprocess.check_call(["make", "-s", "-C", HOSTSIM])
    env = dict(os.environ, B200CTC_HOSTSIM_ORDER=order, B200CTC_FORCE_V5="1", B200CTC_V5_VARIANT="0", PYTHONPATH=ROOT)
    subprocess.check_call([sys.executable, "-c", code], cwd=ROOT, env=env)
