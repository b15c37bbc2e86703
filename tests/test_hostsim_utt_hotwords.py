"""Hostsim twin of tests/test_gpu_utt_hotwords.py: per-utterance hotwords in the CPU simulation build of the kernels,
in the latency-first variants and the general kernel, and with the work items of every phase replayed in other
orders (B200CTC_HOSTSIM_ORDER, read once per process: a child process per order)."""
import ctypes as C
import os
import subprocess
import sys

import pytest

from oracle import oracle as orc
from tests import utt_hotwords as uh

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


def _batch(wl, n=8, seed0=300, T=(90, 0, 120, 61, 150, 33, 120, 7)):
    xs = [wl.utterance(seed0 + i, T[i % len(T)], "diffuse" if i % 2 else "peaky") for i in range(n)]
    lists, weights = uh.hot_lists(wl, [seed0 + i for i in range(n)], 120)
    return xs, lists, weights


@pytest.mark.parametrize("name", ["char", "char3", "bpe4"])
@pytest.mark.parametrize("prune_history", [False, True])
def test_hostsim_utt_hotwords_contract(sim, name, prune_history):
    wl = uh.workload(name)
    kw = uh.decoder_kwargs(wl)
    dec = sim.build_ctcdecoder(wl.labels, **kw)
    xs, lists, weights = _batch(wl)
    got = uh.check_contract(dec, xs, lists, weights, beam_width=24, prune_history=prune_history)
    uh.check_oracle(orc.OracleDecoder(wl.labels, **kw), xs, lists, weights, got, beam_width=24, prune_history=prune_history)


@pytest.mark.parametrize("variant", ["0", "1", "2", "general"])
def test_hostsim_utt_hotwords_kernels(sim, variant, monkeypatch):
    if variant == "general":
        bw = 160                  # above the latency-first kernel's 128 beams
    else:
        monkeypatch.setenv("B200CTC_FORCE_V5", "1")
        monkeypatch.setenv("B200CTC_V5_VARIANT", variant)
        bw = 32
    wl = uh.workload("char")
    dec = sim.build_ctcdecoder(wl.labels)
    xs, lists, weights = _batch(wl)
    uh.check_contract(dec, xs, lists, weights, beam_width=bw)
    assert dec.last_timings()["kernel_variant"] == (0 if variant == "general" else 2)


def test_hostsim_utt_hotwords_inputs(sim, monkeypatch):
    """A padded block with lengths, a host block called twice (pipelined), chunked launches."""
    wl = uh.workload("char")
    dec = sim.build_ctcdecoder(wl.labels)
    xs, lists, weights = _batch(wl)
    block, lengths = uh.padded(xs)
    uh.check_contract(dec, xs, lists, weights, batch_input=block, lengths=lengths, beam_width=16)
    same = [wl.utterance(500 + i, 320, "diffuse") for i in range(6)]
    lists6, weights6 = uh.hot_lists(wl, [500 + i for i in range(6)], 320)
    block6, _ = uh.padded(same)
    for _ in range(2):
        uh.check_contract(dec, same, lists6, weights6, batch_input=block6, beams=False, beam_width=16)
    monkeypatch.setenv("B200CTC_FORCE_CHUNKS", "3")
    monkeypatch.setenv("B200CTC_FORCE_V5", "1")
    uh.check_contract(dec, same, lists6, weights6, beam_width=16)


def test_hostsim_utt_hotwords_multi_lm(sim):
    a = uh.workload("char3")
    models = [sim.LanguageModel(sim.NgramModel(a.arpa), a.words, alpha=0.5, beta=1.0),
              sim.LanguageModel(sim.NgramModel(a.arpa), a.words[:150], alpha=0.3, beta=0.5, unk_score_offset=-5.0)]
    dec = sim.BeamSearchDecoderCTC(sim.Alphabet.build_alphabet(a.labels), sim.MultiLanguageModel(models))
    xs, lists, weights = _batch(a, n=5)
    uh.check_contract(dec, xs, lists, weights, beam_width=16)


def test_hostsim_utt_hotwords_not_vacuous(sim):
    wl = uh.workload("char")
    dec = sim.build_ctcdecoder(wl.labels)
    seeds = [700 + i for i in range(12)]
    xs = [wl.utterance(s, 120, "diffuse") for s in seeds]
    lists, weights = uh.hot_lists(wl, seeds, 120)
    assert uh.differs(dec, xs, lists, weights, beam_width=24) >= 3


def test_hostsim_utt_hotwords_mixed_special_steps(sim, monkeypatch):
    monkeypatch.setenv("B200CTC_FORCE_V5", "1")
    monkeypatch.setenv("B200CTC_V5_VARIANT", "0")
    wl = uh.workload("char")
    dec = sim.build_ctcdecoder(wl.labels)
    xs, lists, weights = _batch(wl)
    total = uh.mixed_special_steps(dec, xs, lists, weights, beam_width=32)
    assert total["inplace_frames"] > 0 and total["single_frames"] > 0


@pytest.mark.parametrize("name", ["char", "char3"])
def test_hostsim_utt_hotwords_streaming(sim, name):
    wl = uh.workload(name)
    dec = sim.build_ctcdecoder(wl.labels, **uh.decoder_kwargs(wl))
    seeds = [900 + i for i in range(4)]
    xs = [wl.utterance(s, 120, "diffuse") for s in seeds]
    sc = uh.scorers(sim, wl, seeds, 120, 3)
    uh.stream_chunks(dec, sim, xs, sc, [0, 40, 81, 120], beam_width=16)


def test_hostsim_utt_hotwords_errors(sim):
    wl = uh.workload("char")
    dec = sim.build_ctcdecoder(wl.labels)
    xs = [wl.utterance(1, 30), wl.utterance(2, 30)]
    with pytest.raises(ValueError):
        dec.decode_batch(None, xs, hotwords_list=[["a"]])
    with pytest.raises(ValueError):
        dec.decode_batch(None, xs, hotwords_list=[["a"], None], hotword_weight_list=[1.0])
    with pytest.raises(ValueError):
        dec.decode_beams_batch(None, xs, hotwords=["b"], hotwords_list=[["a"], None])
    with pytest.raises(ValueError):
        dec.decode_batch(None, xs, hotword_weight_list=[1.0, 2.0])
    with pytest.raises(ValueError):
        dec.decode_batch(None, xs, hotwords_list=["abc", None])
    scorer = sim.HotwordScorer.build_scorer(["a"])
    st = dec.get_starting_state()
    with pytest.raises(ValueError):
        dec.partial_decode_beams_batch(xs, [st[1]] * 2, [st[0]] * 2, [0, 0], hotword_scorer=scorer,
                                       hotword_scorer_list=[scorer, None])
    with pytest.raises(ValueError):
        dec.partial_decode_beams_batch(xs, [st[1]] * 2, [st[0]] * 2, [0, 0], hotword_scorer_list=[scorer])
    # an empty call-wide list with per-utterance lists is fine
    assert dec.decode_batch(None, xs, hotwords=[], hotwords_list=[["a"], None]) == \
        [dec.decode(xs[0], hotwords=["a"]), dec.decode(xs[1])]
    _abi_errors(sim, dec)


def _abi_errors(sim, dec):
    """B2C_E_ARG from the C ABI: an index outside the sets, and opts->hotwords together with utt_hot_set."""
    from pyctcdecode_b200 import _lib
    L = _lib.lib()
    handle = dec._handle(None)
    x = (C.c_float * 32)()
    ptrs = (C.c_void_p * 2)(C.addressof(x), C.addressof(x))
    Ts = (C.c_int32 * 2)(1, 1)
    words = _lib.cstr_array(["a"])
    sets = (_lib.HotwordSet * 1)()
    sets[0].hotwords = C.cast(words, C.POINTER(C.c_char_p))
    sets[0].n_hotwords = 1
    sets[0].hotword_weight = 10.0
    for idx, n_call_wide in (((0, 1), 0), ((0, -1), 0), ((0, 0), 1)):
        opts = _lib.DecodeOpts()
        L.b2c_decode_opts_default(C.byref(opts))
        opts.hot_sets = C.cast(sets, C.POINTER(_lib.HotwordSet))
        opts.n_hot_sets = 1
        arr = (C.c_int32 * 2)(*idx)
        opts.utt_hot_set = C.cast(arr, C.POINTER(C.c_int32))
        opts.hotwords = C.cast(words, C.POINTER(C.c_char_p))
        opts.n_hotwords = n_call_wide
        res = C.c_void_p()
        assert L.b2c_decode_batch(handle, ptrs, Ts, 2, 0, 0, C.byref(opts), C.byref(res)) == -1
    opts.n_hotwords = 0
    arr = (C.c_int32 * 2)(0, 0)
    opts.utt_hot_set = C.cast(arr, C.POINTER(C.c_int32))
    assert L.b2c_decode_batch(handle, ptrs, Ts, 2, 0, 0, C.byref(opts), C.byref(res)) == 0
    L.b2c_result_free(res)


@pytest.mark.parametrize("order", ["1", "2", "3"])
def test_hostsim_utt_hotwords_work_item_order(order):
    code = ("import sys; from tests import utt_hotwords as uh; from pyctcdecode_b200 import _lib; "
            "import pyctcdecode_b200 as p; _lib.use_library(%r); wl = uh.workload('char3'); "
            "dec = p.build_ctcdecoder(wl.labels, **uh.decoder_kwargs(wl)); "
            "xs = [wl.utterance(300 + i, 90, 'diffuse') for i in range(6)]; "
            "lists, weights = uh.hot_lists(wl, [300 + i for i in range(6)], 90); "
            "uh.check_contract(dec, xs, lists, weights, beam_width=24)") % LIB
    subprocess.check_call(["make", "-s", "-C", HOSTSIM])
    env = dict(os.environ, B200CTC_HOSTSIM_ORDER=order, B200CTC_FORCE_V5="1", B200CTC_V5_VARIANT="0", PYTHONPATH=ROOT)
    subprocess.check_call([sys.executable, "-c", code], cwd=ROOT, env=env)
