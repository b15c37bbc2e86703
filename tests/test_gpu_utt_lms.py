"""Per-utterance language models on the device (tests/utt_lms.py): every batched result equals, bit for bit, the
single-utterance call on a decoder built with that utterance's model, and the oracle per group of utterances sharing a
single-model set; in each latency-first variant, the lean variant and the general kernel, with padded, pipelined,
chunked and device-resident input, together with per-utterance hotwords, and in mixed batches that keep the special
steps."""
import threading

import pytest

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


@pytest.mark.parametrize("kind", ["char", "bpe"])
@pytest.mark.parametrize("prune_history", [False, True])
def test_gpu_utt_lms_contract(pkg, char_sets, kind, prune_history):
    from oracle import oracle
    oracle.build()
    sets = char_sets if kind == "char" else ul.Sets(pkg, "bpe")
    n = 18 if kind == "char" else 9
    names = sets.names(n) if kind == "char" else sets.names(n, ["A", "B", "none"])
    dec = _decoder(pkg, sets)
    xs = ul.batch(sets.wl, n=n)
    got = ul.check_contract(sets, dec, xs, sets.models(names), beam_width=24, prune_history=prune_history)
    ul.check_oracle(sets, oracle, xs, names, got, beam_width=24, prune_history=prune_history)


@pytest.mark.parametrize("variant", ["0", "1", "2", "lean", "general"])
def test_gpu_utt_lms_kernels(pkg, char_sets, variant, monkeypatch):
    if variant == "general":
        bw = 160                  # above the latency-first kernel's 128 beams
    elif variant == "lean":
        monkeypatch.setenv("B200CTC_FORCE_LEAN", "1")
        bw = 16
    else:
        monkeypatch.setenv("B200CTC_FORCE_V5", "1")
        monkeypatch.setenv("B200CTC_V5_VARIANT", variant)
        bw = 32
    # a MultiLanguageModel set sends the whole call to the general kernel
    names = char_sets.names(16, ul.NAMES if variant == "general" else ["A", "B", "A_params", "A_no_unigrams", "none"])
    dec = _decoder(pkg, char_sets, own=None if variant == "lean" else "A")
    xs = ul.batch(char_sets.wl, n=16)
    ul.check_contract(char_sets, dec, xs, char_sets.models(names), beam_width=bw)
    ul.check_route(dec, variant)


def test_gpu_utt_lms_inputs(pkg, char_sets, monkeypatch):
    """A padded block with lengths, a device tensor, a host block called three times (pipelined), a ragged host list
    called twice (hinted), chunked launches, per-utterance hotwords."""
    import torch
    sets = char_sets
    dec = _decoder(pkg, sets, own=None)
    xs = ul.batch(sets.wl, n=16)
    lms = sets.models(sets.names(len(xs)))
    block, lengths = ul.padded(xs)
    ul.check_contract(sets, dec, xs, lms, batch_input=block, lengths=lengths, beam_width=16)
    ul.check_contract(sets, dec, xs, lms, batch_input=torch.from_numpy(block).cuda(), lengths=lengths, beam_width=16)
    ul.check_contract(sets, dec, xs, lms, batch_input=[torch.from_numpy(x).cuda() for x in xs], beam_width=16)
    same = [sets.wl.utterance(500 + i, 320, "diffuse") for i in range(24)]
    lms24 = sets.models(sets.names(24, ["A", "none", "B", "A_params"]))
    block24, _ = ul.padded(same)
    ul.check_pipelined(sets, _decoder(pkg, sets, own=None), same, lms24, block24, monkeypatch, beam_width=16)
    ragged = [sets.wl.utterance(600 + i, 300 + 7 * i, "peaky") for i in range(12)]
    ul.check_hinted(sets, _decoder(pkg, sets, own=None), ragged, sets.models(sets.names(12, ["A", "none", "B", "A_params"])),
                    beam_width=16)
    words = sets.wl.words
    hot = [[words[(3 * i) % 50]] if i % 3 else None for i in range(24)]
    ul.check_contract(sets, dec, same, lms24, beam_width=16, hotwords_list=hot)
    monkeypatch.setenv("B200CTC_FORCE_CHUNKS", "3")
    monkeypatch.setenv("B200CTC_FORCE_V5", "1")
    ul.check_contract(sets, dec, same, lms24, beam_width=16)


def test_gpu_utt_lms_not_vacuous(pkg, char_sets):
    seeds = [700 + i for i in range(12)]
    xs = [char_sets.wl.utterance(s, 120, "diffuse") for s in seeds]
    assert ul.differs(char_sets, _decoder(pkg, char_sets), xs, char_sets.names(12), beam_width=24) >= 4


def test_gpu_utt_lms_mixed_special_steps(pkg, char_sets, monkeypatch):
    monkeypatch.setenv("B200CTC_FORCE_V5", "1")
    monkeypatch.setenv("B200CTC_V5_VARIANT", "0")
    dec = _decoder(pkg, char_sets, own=None)
    total = ul.mixed_special_steps(char_sets, dec, ul.batch(char_sets.wl, n=16), beam_width=32)
    assert total["inplace_frames"] > 0 and total["single_frames"] > 0


def test_gpu_utt_lms_threads(pkg, char_sets):
    """Two decoders share the same model objects; 8 threads call them with language_model_list at once."""
    sets = char_sets
    decs = [_decoder(pkg, sets), _decoder(pkg, sets, own=None)]
    xs = ul.batch(sets.wl, n=8)
    jobs = [(decs[j % 2], sets.models(sets.names(8, ul.NAMES[j % 3:] + ul.NAMES[:j % 3]))) for j in range(8)]
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
