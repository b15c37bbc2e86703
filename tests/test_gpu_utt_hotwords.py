"""Per-utterance hotwords on the device (tests/utt_hotwords.py): every batched result equals the single-utterance call
of the existing API bit for bit, and the oracle per group of utterances sharing a set; in each latency-first variant
and the general kernel, with padded, pipelined, chunked and device-resident input, a MultiLanguageModel, mixed
batches that keep the special steps, and streams with per-stream scorers."""
import pytest

from tests import utt_hotwords as uh

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


def _batch(wl, n=16, seed0=300, T=(90, 0, 120, 61, 150, 33, 120, 7)):
    xs = [wl.utterance(seed0 + i, T[i % len(T)], "diffuse" if i % 2 else "peaky") for i in range(n)]
    lists, weights = uh.hot_lists(wl, [seed0 + i for i in range(n)], 120)
    return xs, lists, weights


@pytest.mark.parametrize("name", ["char", "char3", "bpe4"])
@pytest.mark.parametrize("prune_history", [False, True])
def test_gpu_utt_hotwords_contract(pkg, name, prune_history):
    from oracle import oracle
    oracle.build()
    wl = uh.workload(name)
    kw = uh.decoder_kwargs(wl)
    dec = pkg.build_ctcdecoder(wl.labels, **kw)
    xs, lists, weights = _batch(wl)
    got = uh.check_contract(dec, xs, lists, weights, beam_width=24, prune_history=prune_history)
    uh.check_oracle(oracle.OracleDecoder(wl.labels, **kw), xs, lists, weights, got, beam_width=24,
                    prune_history=prune_history)


@pytest.mark.parametrize("variant", ["0", "1", "2", "general"])
@pytest.mark.parametrize("name", ["char", "char3"])
def test_gpu_utt_hotwords_kernels(pkg, variant, name, monkeypatch):
    if variant == "general":
        bw = 160                  # above the latency-first kernel's 128 beams
    else:
        monkeypatch.setenv("B200CTC_FORCE_V5", "1")
        monkeypatch.setenv("B200CTC_V5_VARIANT", variant)
        bw = 32
    wl = uh.workload(name)
    dec = pkg.build_ctcdecoder(wl.labels, **uh.decoder_kwargs(wl))
    xs, lists, weights = _batch(wl)
    uh.check_contract(dec, xs, lists, weights, beam_width=bw)
    assert dec.last_timings()["kernel_variant"] == (0 if variant == "general" else 2)


def test_gpu_utt_hotwords_inputs(pkg, monkeypatch):
    """A padded block with lengths, a device tensor, a host block called twice (pipelined), chunked launches."""
    import torch
    wl = uh.workload("char")
    dec = pkg.build_ctcdecoder(wl.labels)
    xs, lists, weights = _batch(wl)
    block, lengths = uh.padded(xs)
    uh.check_contract(dec, xs, lists, weights, batch_input=block, lengths=lengths, beam_width=16)
    uh.check_contract(dec, xs, lists, weights, batch_input=torch.from_numpy(block).cuda(), lengths=lengths, beam_width=16)
    uh.check_contract(dec, xs, lists, weights, batch_input=[torch.from_numpy(x).cuda() for x in xs], beam_width=16)
    same = [wl.utterance(500 + i, 320, "diffuse") for i in range(24)]
    lists24, weights24 = uh.hot_lists(wl, [500 + i for i in range(24)], 320)
    block24, _ = uh.padded(same)
    for _ in range(3):
        uh.check_contract(dec, same, lists24, weights24, batch_input=block24, beams=False, beam_width=16)
    monkeypatch.setenv("B200CTC_FORCE_CHUNKS", "3")
    monkeypatch.setenv("B200CTC_FORCE_V5", "1")
    uh.check_contract(dec, same, lists24, weights24, beam_width=16)


def test_gpu_utt_hotwords_multi_lm(pkg):
    a = uh.workload("char3")
    models = [pkg.LanguageModel(pkg.NgramModel(a.arpa), a.words, alpha=0.5, beta=1.0),
              pkg.LanguageModel(pkg.NgramModel(a.arpa), a.words[:150], alpha=0.3, beta=0.5, unk_score_offset=-5.0)]
    dec = pkg.BeamSearchDecoderCTC(pkg.Alphabet.build_alphabet(a.labels), pkg.MultiLanguageModel(models))
    xs, lists, weights = _batch(a, n=8)
    uh.check_contract(dec, xs, lists, weights, beam_width=16)


def test_gpu_utt_hotwords_not_vacuous(pkg):
    wl = uh.workload("char")
    dec = pkg.build_ctcdecoder(wl.labels)
    seeds = [700 + i for i in range(12)]
    xs = [wl.utterance(s, 120, "diffuse") for s in seeds]
    lists, weights = uh.hot_lists(wl, seeds, 120)
    assert uh.differs(dec, xs, lists, weights, beam_width=24) >= 3


def test_gpu_utt_hotwords_mixed_special_steps(pkg, monkeypatch):
    monkeypatch.setenv("B200CTC_FORCE_V5", "1")
    monkeypatch.setenv("B200CTC_V5_VARIANT", "0")
    wl = uh.workload("char")
    dec = pkg.build_ctcdecoder(wl.labels)
    xs, lists, weights = _batch(wl)
    total = uh.mixed_special_steps(dec, xs, lists, weights, beam_width=32)
    assert total["inplace_frames"] > 0 and total["single_frames"] > 0


@pytest.mark.parametrize("name", ["char", "char3"])
def test_gpu_utt_hotwords_streaming(pkg, name):
    wl = uh.workload(name)
    dec = pkg.build_ctcdecoder(wl.labels, **uh.decoder_kwargs(wl))
    seeds = [900 + i for i in range(4)]
    xs = [wl.utterance(s, 120, "diffuse") for s in seeds]
    sc = uh.scorers(pkg, wl, seeds, 120, 3)
    uh.stream_chunks(dec, pkg, xs, sc, [0, 40, 81, 120], beam_width=16)
