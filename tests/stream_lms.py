"""Per-stream language models in batched streaming (partial_decode_beams_batch with language_model_list), shared by
tests/test_gpu_stream_lms.py and its hostsim twin.

The contract: stream i of a batched call returns, bit for bit, what BeamSearchDecoderCTC(alphabet,
language_model_list[i]).partial_decode_beams returns for it with the same chunk, cache, beams, processed_frames and
other arguments.  `stream_chunks` asserts it call by call; `run_golden_group` holds the streams of one batched call to
what the unmodified reference returned for each; `differs` counts the streams whose own model changes the final text,
so that a library that ignored the per-stream index could not pass."""
import json

from pyctcdecode_b200.language_model import AbstractLanguageModel
from tests import goldens
from tests.utt_lms import NAMES

# chunk bounds: 1, 7 and 50 frames, then the rest
BOUNDS = [0, 1, 8, 58, 108, 160]


def streams(wl, n=12, seed0=900, T=(150, 0, 120, 61, 160, 33, 8, 1)):
    """Ragged streams, T = 0 and T = 1 included: later chunks of a short stream are empty."""
    return [wl.utterance(seed0 + i, T[i % len(T)], "diffuse" if i % 2 else "peaky") for i in range(n)]


def start(dec, lm):
    """The cache a stream with model `lm` starts from: the decoder's own model's cache without one."""
    return dec.get_starting_state(language_model=lm)[1] if lm is not None else {}


def stream_chunks(sets, dec, xs, lms_per_call, bounds=BOUNDS, scorers_per_call=None, force_next_word=False, **kw):
    """Streams advanced chunk by chunk through partial_decode_beams_batch(language_model_list=lms_per_call[c]) and,
    one stream at a time, through a decoder built with that stream's model of the call: every call's LMBeam lists must
    be identical.  The last call has is_end=True.  Returns the final beams."""
    n = len(xs)
    b_beams = [[b for b in dec.get_starting_state()[0]] for _ in range(n)]
    s_beams = list(b_beams)
    for c in range(len(bounds) - 1):
        t0, t1 = bounds[c], bounds[c + 1]
        last = c == len(bounds) - 2
        lms = lms_per_call[c]
        scorers = scorers_per_call[c] if scorers_per_call is not None else None
        caches = [start(dec, lm) for lm in lms]
        out = dec.partial_decode_beams_batch([x[t0:t1] for x in xs], caches, b_beams, [t0] * n, language_model_list=lms,
                                             hotword_scorer_list=scorers, force_next_word=force_next_word, is_end=last, **kw)
        assert len(out) == n
        for i in range(n):
            ref_dec = sets.ref(lms[i])
            cache = ref_dec.get_starting_state()[1]
            ref = ref_dec.partial_decode_beams(xs[i][t0:t1], cache, {}, s_beams[i], t0,
                                               hotword_scorer=None if scorers is None else scorers[i],
                                               force_next_word=force_next_word, is_end=last, **kw)
            assert out[i] == ref, "stream %d call %d (%s)" % (i, c, lms[i] is not None and type(lms[i]).__name__)
            s_beams[i] = ref
        b_beams = out
    return b_beams


def final_texts(dec, xs, lms, bounds=BOUNDS, **kw):
    """Top text of every stream after the last (is_end) call, every call with the same models."""
    n = len(xs)
    beams = [list(dec.get_starting_state()[0]) for _ in range(n)]
    for c in range(len(bounds) - 1):
        t0, t1 = bounds[c], bounds[c + 1]
        caches = [start(dec, lm) for lm in lms]
        beams = dec.partial_decode_beams_batch([x[t0:t1] for x in xs], caches, beams, [t0] * n, language_model_list=lms,
                                               is_end=c == len(bounds) - 2, **kw)
    return [b[0].text if b else "" for b in beams]


def differs(sets, dec, xs, names, **kw):
    """Streams whose final text with their own set differs from the one set A gives them."""
    own = final_texts(dec, xs, sets.models(names), **kw)
    base = final_texts(dec, xs, [sets.lm["A"]] * len(xs), **kw)
    return sum(1 for a, b in zip(own, base) if a != b)


# ---- against the reference: goldens that share an alphabet and call settings, one batched call --------------------
def golden_groups():
    """Names of the streaming goldens grouped by (labels, call-wide settings); groups of one are left out."""
    groups = {}
    for case in goldens.load_stream()["meta"]["cases"]:
        key = (tuple(case["labels"]), json.dumps(case["common"], sort_keys=True))
        groups.setdefault(key, []).append(case["name"])
    return [names for names in groups.values() if len(names) > 1]


def _match(out, exp, tol):
    """goldens.run_stream_case's comparison of one call: identical strings, frames and last_char, scores within tol,
    the order free only between beams the reference separates by at most 1e-9."""
    if len(out) != len(exp):
        return "%d beams != %d" % (len(out), len(exp))

    def ident(text, nw, pw, lc, tf, pf):
        return (text, nw, pw, lc, tuple(tuple(f) for f in tf), tuple(pf))

    got = {ident(o.text, o.next_word, o.partial_word, o.last_char, o.text_frames, o.partial_frames): (j, o) for j, o in enumerate(out)}
    pos = []
    for j, e in enumerate(exp):
        k = ident(e["text"], e["next_word"], e["partial_word"], e["last_char"], e["text_frames"], e["partial_frames"])
        if k not in got:
            return "reference beam %d %r missing" % (j, k[:4])
        gj, o = got[k]
        if abs(o.logit_score - e["logit_score"]) > tol + 1e-6 * abs(e["logit_score"]):
            return "beam %d logit %r != %r" % (j, o.logit_score, e["logit_score"])
        if abs(o.lm_score - e["lm_score"]) > tol + 1e-6 * abs(e["lm_score"]):
            return "beam %d lm %r != %r" % (j, o.lm_score, e["lm_score"])
        pos.append(gj)
    for a in range(len(exp)):
        for b in range(a + 1, len(exp)):
            if exp[a]["lm_score"] - exp[b]["lm_score"] > 1e-9 and pos[a] > pos[b]:
                return "beams %d and %d swapped" % (a, b)
    return ""


def run_golden_group(pkg, names, tol=2e-4):
    """The cases `names` as the streams of one decoder without a model of its own: every call of the group is one
    partial_decode_beams_batch with each stream's model in language_model_list (and its hotwords in
    hotword_scorer_list); streams whose steps are done drop out.  Streams whose current steps differ in
    force_next_word / is_end go to separate calls.  Returns the number of batched calls."""
    g, s = goldens.load(), goldens.load_stream()
    cases = [next(c for c in s["meta"]["cases"] if c["name"] == name) for name in names]
    labels = cases[0]["labels"]
    dec = pkg.BeamSearchDecoderCTC(pkg.Alphabet.build_alphabet(labels), None)
    lms, xs = [], []
    for case in cases:
        lms.append(goldens.build_product_decoder(pkg, labels, **goldens.lm_kwargs(g, case))._language_model)
        xs.append(s["arrays"][case["array"]] if case["array"] in s["arrays"] else g["arrays"][case["array"]])
    beams = [list(dec.get_starting_state()[0]) for _ in cases]
    caches = [start(dec, lm) for lm in lms]
    common = cases[0]["common"]
    calls = 0
    for step_i in range(max(len(c["steps"]) for c in cases)):
        parts = {}
        for i, case in enumerate(cases):
            if step_i < len(case["steps"]):
                st = case["steps"][step_i]
                parts.setdefault((bool(st["call"].get("force_next_word", False)), bool(st["is_end"])), []).append(i)
        for (force, is_end), idx in parts.items():
            steps = [cases[i]["steps"][step_i] for i in idx]
            scorers = []
            for st in steps:
                hw = st["call"].get("hotwords")
                scorers.append(None if hw is None else pkg.HotwordScorer.build_scorer(hw, weight=st["call"].get("hotword_weight", 10.0)))
            out = dec.partial_decode_beams_batch([xs[i][st["start"]:st["end"]] for i, st in zip(idx, steps)], [caches[i] for i in idx],
                                                 [beams[i] for i in idx], [st["start"] for st in steps],
                                                 hotword_scorer_list=scorers, language_model_list=[lms[i] for i in idx],
                                                 force_next_word=force, is_end=is_end, **common)
            calls += 1
            for i, st, o in zip(idx, steps, out):
                why = _match(o, st["beams"], tol)
                assert not why, "%s call %d: %s" % (names[i], step_i, why)
                beams[i] = o
    return calls


# ---- start states and errors --------------------------------------------------------------------------------------
def _state_key(st):
    return [_state_key(s) for s in st.states] if hasattr(st, "states") else (st.words, st.backoffs)


def _cache_key(cache):
    return {k: (v[0], v[1], _state_key(v[2])) for k, v in cache.items()}


def largest_id_state(lm, words):
    """The state after the word with the largest vocabulary id of `lm` (the largest id of a model over 300 words is
    above the size of a vocabulary over 250)."""
    from pyctcdecode_b200.language_model import B200LMState
    best = None
    for w in words:
        out = B200LMState()
        lm.ngram_model.BaseScore(lm.get_start_state(), w, out)
        if out.words and (best is None or max(out.words) > max(best.words)):
            best = out
    assert best is not None and max(best.words) > 260
    return best


def check_start_states(pkg, sets, dec):
    """get_starting_state(language_model=...), default and carried start states in a call with sets of one and two
    models, and the states the library refuses.  `dec` has model A of its own."""
    from pytest import raises
    for name in NAMES:
        lm = sets.lm[name]
        got, ref = dec.get_starting_state(language_model=lm), sets.ref(lm).get_starting_state()
        assert got[0] == ref[0] and got[2] == ref[2]
        assert _cache_key(got[1]) == _cache_key(ref[1] if lm is not None else dec.get_starting_state()[1])
    xs = streams(sets.wl, n=6, T=(90, 60))
    lms = sets.models(["A", "AB", "B", "none", "A_params", "AB"])
    beams = [list(dec.get_starting_state()[0]) for _ in xs]
    chunk = [x[:40] for x in xs]
    # a missing cache, a cache without the entry and the explicit default state give the same
    explicit = dec.partial_decode_beams_batch(chunk, [start(dec, lm) for lm in lms], beams, [0] * 6, language_model_list=lms)
    assert dec.partial_decode_beams_batch(chunk, [None] * 6, beams, [0] * 6, language_model_list=lms) == explicit
    assert dec.partial_decode_beams_batch(chunk, [{}] * 6, beams, [0] * 6, language_model_list=lms) == explicit
    # carried states: a MultiLanguageModelState for the AB streams next to B200LMStates in one call (rows of two)
    caches = []
    for lm, x in zip(lms, xs):
        st = sets.ref(lm).decode_beams(x[40:90], beam_width=8)[0].last_lm_state if lm is not None else None
        caches.append({("", False): (0.0, 0.0, st)} if st is not None else {})
    assert isinstance(caches[1][("", False)][2], pkg.MultiLanguageModelState)
    out = dec.partial_decode_beams_batch(chunk, caches, beams, [0] * 6, language_model_list=lms, is_end=True)
    for i in range(6):
        assert out[i] == sets.ref(lms[i]).partial_decode_beams(chunk[i], caches[i], {}, beams[i], 0, is_end=True), i
    assert out != dec.partial_decode_beams_batch(chunk, [None] * 6, beams, [0] * 6, language_model_list=lms, is_end=True)
    # the wrong state type for the stream's set
    a_state = sets.lm["A"].get_start_state()
    ab_state = sets.lm["AB"].get_start_state()
    for lm, st in ((sets.lm["AB"], a_state), (sets.lm["A"], ab_state),
                   (sets.lm["AB"], pkg.MultiLanguageModelState([a_state, a_state, a_state]))):
        with raises(AssertionError, match="Wrong input state type"):
            dec.partial_decode_beams_batch(chunk[:2], [None, {("", False): (0.0, 0.0, st)}], beams[:2], [0, 0],
                                           language_model_list=[sets.lm["A"], lm])
    # a stream without a model ignores its entry, whatever it holds
    junk = {("", False): (0.0, 0.0, "not a state")}
    assert dec.partial_decode_beams_batch(chunk[3:4], [junk], beams[:1], [0], language_model_list=[None]) == \
        dec.partial_decode_beams_batch(chunk[3:4], [None], beams[:1], [0], language_model_list=[None])
    # a state of model A whose word id lies beyond model B's vocabulary: refused on a B stream (alone or as model 1 of
    # a MultiLanguageModel), taken on an A stream
    big = largest_id_state(sets.lm["A"], sets.wl.words)
    for lm, st in ((sets.lm["B"], big), (pkg.MultiLanguageModel([sets.lm["A"], sets.lm["B"]]), pkg.MultiLanguageModelState([a_state, big]))):
        with raises(ValueError, match="vocabulary"):
            dec.partial_decode_beams_batch(chunk[:2], [None, {("", False): (0.0, 0.0, st)}], beams[:2], [0, 0],
                                           language_model_list=[sets.lm["A"], lm])
    dec.partial_decode_beams_batch(chunk[:1], [{("", False): (0.0, 0.0, big)}], beams[:1], [0], language_model_list=[sets.lm["A"]])


def check_own_model_states(sets, dec):
    """The check covers a decoder's own model too (`dec` has model B): a state with an id outside its vocabulary is
    refused by decode_beams and partial_decode_beams, the decoder's own start state is taken."""
    from pytest import raises
    big = largest_id_state(sets.lm["A"], sets.wl.words)
    x = sets.wl.utterance(5, 40)
    with raises(ValueError, match="vocabulary"):
        dec.decode_beams(x, beam_width=8, lm_start_state=big)
    beams, cache, pcache = dec.get_starting_state()
    with raises(ValueError, match="vocabulary"):
        dec.partial_decode_beams(x, {("", False): (0.0, 0.0, big)}, pcache, beams, 0)
    assert dec.decode_beams(x, beam_width=8, lm_start_state=cache[("", False)][2])


class OtherLM(AbstractLanguageModel):
    """A language model of another library: the calls take pyctcdecode_b200's own models only (TypeError)."""
    order = 3

    def get_start_state(self):
        return None

    def score_partial_token(self, partial_token):
        return 0.0

    def score(self, prev_state, word, is_last_word=False):
        return 0.0, None


def check_errors(pkg, sets, dec):
    """ValueError / TypeError of partial_decode_beams_batch(language_model_list=...) and
    get_starting_state(language_model=...)."""
    from pytest import raises
    other = OtherLM()
    xs = [sets.wl.utterance(1, 30), sets.wl.utterance(2, 30)]
    caches = [None, None]
    beams = [list(dec.get_starting_state()[0]) for _ in xs]
    five = pkg.MultiLanguageModel([sets.lm["A"], sets.lm["B"], sets.lm["A_params"], sets.lm["A_no_unigrams"], sets.lm["A"]])
    for bad, exc in (([sets.lm["A"]], ValueError), (sets.lm["A"], ValueError), ([five, None], ValueError),
                     ([other, None], TypeError)):
        with raises(exc):
            dec.partial_decode_beams_batch(xs, caches, beams, [0, 0], language_model_list=bad)
    with raises(ValueError):
        dec.get_starting_state(language_model=five)
    with raises(TypeError):
        dec.get_starting_state(language_model=other)
