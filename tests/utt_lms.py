"""Per-utterance language models (decode_batch / decode_beams_batch with language_model_list), shared by
tests/test_gpu_utt_lms.py and its hostsim twin.

The contract: utterance i of a batched call returns, bit for bit, what BeamSearchDecoderCTC(alphabet,
language_model_list[i]) returns for that utterance decoded alone with the same other arguments.  `check_contract`
asserts it for both batch calls; `check_oracle` compares every utterance with a single-model (or no-model) set with the
oracle, called once per group of utterances that share a set; `differs` counts the utterances whose own model changes
the top text, so that a kernel that ignored the routing could not pass."""
import numpy as np

from tests import goldens, synth

# the sets every mixed batch cycles through
NAMES = ["A", "B", "A_params", "A_no_unigrams", "AB", "none"]


class Sets:
    """Language models over one alphabet, by name, and what the oracle needs to build each single-model set."""

    def __init__(self, pkg, kind="char"):
        if kind == "char":
            a = synth.CharWorkload("B", n_words=300, lm_order=3)           # A: a 3-gram
            b = synth.CharWorkload("B", n_words=250, lm_order=4, seed=2)   # B: a 4-gram over other words
            b_arpa, b_words = b.arpa, b.words
        else:
            a = synth.BpeWorkload(n_words=3000, lm_order=4, V=1024)
            # B: another 4-gram over another word list of the same letters (the pieces are A's)
            b_arpa, b_words, _, _ = synth.cached_arpa(2000, [chr(ord("a") + i) for i in range(26)], 4, seed=2, tag="C")
        self.wl, self.labels = a, a.labels
        self.spec = {
            "A": dict(kenlm_model_path=a.arpa, unigrams=a.words, alpha=0.5, beta=1.0),
            "B": dict(kenlm_model_path=b_arpa, unigrams=b_words, alpha=0.7, beta=2.0),
            "A_params": dict(kenlm_model_path=a.arpa, unigrams=a.words, alpha=0.9, beta=0.25, unk_score_offset=-4.0,
                             lm_score_boundary=False),
            "A_no_unigrams": dict(kenlm_model_path=a.arpa, unigrams=None, alpha=0.5, beta=1.0),
            "none": None,
        }
        self.lm = {}
        for name, kw in self.spec.items():
            self.lm[name] = None if kw is None else self._model(pkg, kw)
        self.lm["AB"] = pkg.MultiLanguageModel([self.lm["A"], self.lm["B"]])
        self.pkg = pkg
        self._refs = {}

    @staticmethod
    def _model(pkg, kw):
        return pkg.LanguageModel(pkg.NgramModel(kw["kenlm_model_path"]), kw["unigrams"], alpha=kw["alpha"], beta=kw["beta"],
                                 unk_score_offset=kw.get("unk_score_offset", -10.0),
                                 score_boundary=kw.get("lm_score_boundary", True))

    def names(self, n, names=NAMES):
        return [names[i % len(names)] for i in range(n)]

    def models(self, names):
        return [self.lm[k] for k in names]

    def ref(self, lm):
        """A decoder built with `lm` as its own model (one per model object)."""
        key = id(lm)
        if key not in self._refs:
            self._refs[key] = (lm, self.pkg.BeamSearchDecoderCTC(self.pkg.Alphabet.build_alphabet(self.labels), lm))
        return self._refs[key][1]


def _beams(out):
    return [(b.text, [(w, tuple(f)) for w, f in b.text_frames], b.logit_score, b.lm_score) for b in out]


def check_contract(sets, dec, xs, lms, beams=True, texts=True, batch_input=None, **kw):
    """Batched call with per-utterance models == one call per utterance on a decoder built with that model, bit for
    bit.  `batch_input` replaces `xs` as what the batched calls get (a padded block, a device tensor), with
    kw["lengths"] if needed.  Returns the batched decode_beams_batch results."""
    inp = xs if batch_input is None else batch_input
    got = None
    single_kw = {k: v for k, v in kw.items() if k not in ("lengths", "hotwords_list")}
    hot = kw.get("hotwords_list")
    if beams:
        got = dec.decode_beams_batch(None, inp, language_model_list=lms, **kw)
        assert len(got) == len(xs)
        for i, x in enumerate(xs):
            extra = {} if hot is None else {"hotwords": hot[i]}
            ref = sets.ref(lms[i]).decode_beams(x, **single_kw, **extra)
            assert _beams(got[i]) == _beams(ref), "utterance %d %r" % (i, kw)
    if texts:
        tkw = {k: v for k, v in kw.items() if k != "prune_history"}
        t = dec.decode_batch(None, inp, language_model_list=lms, **tkw)
        for i, x in enumerate(xs):
            extra = {} if hot is None else {"hotwords": hot[i]}
            ref = sets.ref(lms[i]).decode(x, **{k: v for k, v in single_kw.items() if k != "prune_history"}, **extra)
            assert t[i] == ref, "utterance %d %r" % (i, kw)
    return got


def check_oracle(sets, oracle_mod, xs, names, got, **kw):
    """The batched beams of every utterance with a single-model or no-model set against the oracle, one oracle call per
    group of utterances sharing a set.  The model without unigrams is left out: the oracle, like the reference's
    build_ctcdecoder, reads the unigrams of an ARPA file when none are given."""
    groups = {}
    for i, name in enumerate(names):
        if name in sets.spec and name != "A_no_unigrams":
            groups.setdefault(name, []).append(i)
    for name, idx in groups.items():
        ora = oracle_mod.OracleDecoder(sets.labels, **(sets.spec[name] or {}))
        want = ora.decode_beams_batch([xs[i] for i in idx], **kw)
        for i, beams in zip(idx, want):
            exp = [dict(text=b[0], frames=[(wd, s, e) for wd, (s, e) in b[1]], logit_score=b[2], lm_score=b[3]) for b in beams]
            why = goldens.beams_match_tie_aware(exp, _beams(got[i]))
            assert not why, "utterance %d (%s): %s" % (i, name, why)


def differs(sets, dec, xs, names, **kw):
    """Utterances whose top text with their own set differs from the one set A gives them."""
    own = dec.decode_batch(None, xs, language_model_list=sets.models(names), **kw)
    base = dec.decode_batch(None, xs, language_model_list=[sets.lm["A"]] * len(xs), **kw)
    return sum(1 for a, b in zip(own, base) if a != b)


def mixed_special_steps(sets, dec, xs, **kw):
    """Every other utterance without a model: the counts of the special steps must be the sums of the two halves
    decoded separately (an LM-free utterance keeps its in-place / sorted / one-token steps)."""
    names = ("inplace_frames", "sorted_frames", "single_frames")
    lms = [None if i % 2 else sets.lm["A"] for i in range(len(xs))]
    dec.decode_beams_batch(None, xs, language_model_list=lms, **kw)
    mixed = dec.last_timings()
    total = dict.fromkeys(names, 0)
    for half in (0, 1):
        idx = [i for i in range(len(xs)) if i % 2 == half]
        dec.decode_beams_batch(None, [xs[i] for i in idx], language_model_list=[lms[i] for i in idx], **kw)
        tm = dec.last_timings()
        for k in names:
            total[k] += tm[k]
    assert {k: mixed[k] for k in names} == total
    return total


def check_route(dec, variant):
    """The last call ran the kernel the test forced: the general kernel or a latency-first variant."""
    tm = dec.last_timings()
    if variant == "general":
        assert tm["kernel_variant"] == 0
    else:
        assert tm["kernel_variant"] == 2
        assert tm["cta_threads"] == 128


def check_pipelined(sets, dec, xs, lms, block, monkeypatch, **kw):
    """A [B, T, V] host block called three times on a fresh decoder: the first call is planned from its own statistics,
    the later ones are pipelined (one streaming and one beam launch per chunk, so more launches); every call meets the
    contract."""
    monkeypatch.setenv("B200CTC_PIPELINE", "1")
    monkeypatch.setenv("B200CTC_PIPELINE_ALL", "1")        # also compute-bound calls (by default only copy-bound ones)
    launches = []
    for _ in range(3):
        check_contract(sets, dec, xs, lms, batch_input=block, beams=False, **kw)
        launches.append(dec.last_timings()["launches"])
    assert launches[1] > launches[0] and launches[2] > launches[0], launches
    monkeypatch.delenv("B200CTC_PIPELINE")
    monkeypatch.delenv("B200CTC_PIPELINE_ALL")


def check_hinted(sets, dec, xs, lms, **kw):
    """A ragged list called twice on a fresh decoder: the second call is planned from the first one's statistics
    (b2c_timings_t.hinted) and meets the contract."""
    flags = []
    for _ in range(2):
        check_contract(sets, dec, xs, lms, beams=False, **kw)
        flags.append(dec.last_timings()["hinted"])
    assert flags == [0, 1], flags


def batch(wl, n=12, seed0=300, T=(90, 0, 120, 61, 150, 33, 120, 7)):
    return [wl.utterance(seed0 + i, T[i % len(T)], "diffuse" if i % 2 else "peaky") for i in range(n)]


def padded(xs):
    """[B, T_max, V] float32 block and lengths of a ragged list."""
    T = max(x.shape[0] for x in xs)
    block = np.zeros((len(xs), T, xs[0].shape[1]), dtype=np.float32)
    for i, x in enumerate(xs):
        block[i, :x.shape[0]] = x
    return block, [x.shape[0] for x in xs]
