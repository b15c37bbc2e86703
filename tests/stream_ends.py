"""Per-stream is_end and force_next_word in batched streaming (partial_decode_beams_batch with is_end_list /
force_next_word_list), shared by tests/test_gpu_stream_ends.py and its hostsim twin.

The contract: stream i of a batched call returns, bit for bit, what partial_decode_beams returns for it with the same
chunk, cache, beams and processed_frames and its own force_next_word / is_end.  `plan` lays out continuous-batching
traffic (streams end at different calls and new streams take their slots), `run` holds every call of every stream to
its single-stream reference and can count the streams whose beams under the first stream's flags would differ, so that
a library that gave every stream one mode could not pass; `run_golden_group` runs the streaming goldens of one alphabet
and call settings with one batched call per step."""
import ctypes as C

from tests import goldens
from tests import stream_lms as sl

# chunk sizes a slot cycles through (its stream's processed_frames then differ from the other slots')
CHUNKS = (1, 7, 20, 50)
# stream lengths in the order the streams join: T = 0 and T = 1 included
POOL_T = (150, 0, 120, 61, 1, 95, 33, 8, 70, 1, 0, 44)


def plan(Ts, n_slots, chunks=CHUNKS, max_calls=None):
    """Continuous batching: n_slots slots, each advancing its stream by the next of `chunks` per call; a stream's call
    that reaches its last frame has is_end, every third other call of it force_next_word; a slot whose stream ended
    takes the next stream of Ts at the next call.  Runs until every stream ended, or for max_calls calls.  -> calls,
    each a list of (stream, t0, t1, force_next_word, is_end) in slot order."""
    queue = list(range(len(Ts)))
    slots = [queue.pop(0) if queue else None for _ in range(n_slots)]
    pos = [0] * len(Ts)
    calls = []
    while any(s is not None for s in slots) and (max_calls is None or len(calls) < max_calls):
        c = len(calls)
        call = []
        for k, s in enumerate(slots):
            if s is None:
                continue
            t0 = pos[s]
            t1 = min(Ts[s], t0 + chunks[(k + c) % len(chunks)])
            end = t1 >= Ts[s]
            call.append((s, t0, t1, not end and (k + c + s) % 3 == 0, end))
            pos[s] = t1
            if end:
                slots[k] = queue.pop(0) if queue else None
        calls.append(call)
    return calls


def staggered(n):
    """Lengths of n streams at the C3 shape: between 400 and 1000 frames, staggered so that streams end at many
    different calls of 50-frame chunks."""
    return [400 + (j * 211) % 601 for j in range(n)]


def c3_streams(pkg, n_base=64):
    """The C3 shape (V = 32, a 3-gram model over 20k words, alpha 0.5, beta 1.0): (decoder, model, n_base logits of
    1000 frames).  Stream j of a plan reads the first T_j frames of logits j % n_base."""
    from tests import synth
    wl = synth.CharWorkload("B", n_words=20000, lm_order=3, seed=1)
    lm = pkg.LanguageModel(pkg.NgramModel(wl.arpa), wl.words, alpha=0.5, beta=1.0)
    dec = pkg.BeamSearchDecoderCTC(pkg.Alphabet.build_alphabet(wl.labels), lm)
    return dec, wl.batch(1, n_base, 1000, "peaky")


def mode(force, end):
    return 0 if end else (1 if force else 2)


def check_plan(calls, n_streams):
    """What the schedules must contain: every stream ends once, streams end at different calls, a call with all three
    modes, a call whose streams' processed_frames differ, and streams that join after the first call."""
    ends = [c for c, call in enumerate(calls) for s, _, _, _, e in call if e]
    assert len(ends) == n_streams and len(set(ends)) > 2
    assert any(len({mode(f, e) for _, _, _, f, e in call}) == 3 for call in calls)
    assert any(len({t0 for _, t0, _, _, _ in call}) > 2 for call in calls)
    assert any(t0 == 0 for call in calls[1:] for _, t0, _, _, _ in call)


class Streams:
    """How the streams of a run are decoded: `dec` takes the batched calls; stream s has model lms[s] (with
    language_model_list) and hotword scorer scorers[s] (with hotword_scorer_list).  The reference of a stream is
    partial_decode_beams on `dec`, or on a decoder built with the stream's model with language_model_list."""

    def __init__(self, dec, xs, sets=None, lms=None, scorers=None):
        self.dec, self.xs, self.sets, self.lms, self.scorers = dec, xs, sets, lms, scorers

    def ref_dec(self, s):
        return self.sets.ref(self.lms[s]) if self.lms is not None else self.dec

    def cache(self, s):
        return sl.start(self.dec, self.lms[s]) if self.lms is not None else self.dec.get_starting_state()[1]


def run(st, calls, count_differs=False, timings=None, **kw):
    """The calls of `plan` through partial_decode_beams_batch with is_end_list / force_next_word_list; every stream of
    every call against its reference with its own flags.  -> (outputs per call, number of (call, stream) whose
    reference under the flags of the call's first stream differs from its own; 0 without count_differs).
    `timings`: a list that gets last_timings() of every batched call and the `retried` sum of its references."""
    dec = st.dec
    beams = {}
    outs = []
    differ = 0
    for call in calls:
        ids = [s for s, _, _, _, _ in call]
        for s, t0, _, _, _ in call:
            if t0 == 0 and s not in beams:
                beams[s] = list(dec.get_starting_state()[0])
        extra = dict(kw)
        if st.lms is not None:
            extra["language_model_list"] = [st.lms[s] for s in ids]
        if st.scorers is not None:
            extra["hotword_scorer_list"] = [st.scorers[s] for s in ids]
        out = dec.partial_decode_beams_batch([st.xs[s][t0:t1] for s, t0, t1, _, _ in call], [st.cache(s) for s in ids],
                                             [beams[s] for s in ids], [t0 for _, t0, _, _, _ in call],
                                             force_next_word_list=[f for _, _, _, f, _ in call],
                                             is_end_list=[e for _, _, _, _, e in call], **extra)
        tm = dec.last_timings() if timings is not None else None
        assert len(out) == len(call)
        _, _, _, f0, e0 = call[0]
        retried = 0
        for i, (s, t0, t1, f, e) in enumerate(call):
            rd = st.ref_dec(s)
            cache = rd.get_starting_state()[1] if st.lms is not None else st.cache(s)
            hot = st.scorers[s] if st.scorers is not None else None
            ref = rd.partial_decode_beams(st.xs[s][t0:t1], cache, {}, beams[s], t0, hotword_scorer=hot,
                                          force_next_word=f, is_end=e, **kw)
            if timings is not None:
                retried += rd.last_timings()["retried"]
            assert out[i] == ref, "stream %d frames %d..%d force_next_word=%s is_end=%s" % (s, t0, t1, f, e)
            if count_differs and mode(f, e) != mode(f0, e0):
                alt = rd.partial_decode_beams(st.xs[s][t0:t1], cache, {}, beams[s], t0, hotword_scorer=hot,
                                              force_next_word=f0, is_end=e0, **kw)
                differ += alt != ref
            beams[s] = out[i]
        if timings is not None:
            timings.append((tm, retried))
        outs.append(out)
    return outs, differ


def check_uniform(dec, xs, **kw):
    """Lists that give every stream the same flags return what the scalar flags return: for streams that carry words
    and partial words from a first chunk, each of the three modes, given by one list or by both."""
    n = len(xs)
    beams = dec.partial_decode_beams_batch([x[:40] for x in xs], [dec.get_starting_state()[1]] * n,
                                           [list(dec.get_starting_state()[0]) for _ in xs], [0] * n, **kw)
    assert any(b and b[0].partial_word for b in beams) and any(b and b[0].text for b in beams)
    args = ([x[40:90] for x in xs], [dec.get_starting_state()[1]] * n, beams, [40] * n)
    for scalar, lists in (
            (dict(is_end=True), [dict(is_end_list=[True] * n), dict(is_end_list=[True] * n, force_next_word_list=[False] * n),
                                 dict(is_end_list=[True] * n, force_next_word_list=[True] * n)]),
            (dict(force_next_word=True), [dict(force_next_word_list=[True] * n), dict(is_end_list=[False] * n, force_next_word_list=[True] * n)]),
            (dict(), [dict(is_end_list=[False] * n), dict(force_next_word_list=[False] * n),
                      dict(is_end_list=[False] * n, force_next_word_list=[False] * n)])):
        want = dec.partial_decode_beams_batch(*args, **scalar, **kw)
        for extra in lists:
            assert dec.partial_decode_beams_batch(*args, **extra, **kw) == want, (scalar, extra)
        # one list and the other scalar flag
        if "force_next_word" in scalar:
            assert dec.partial_decode_beams_batch(*args, force_next_word=True, is_end_list=[False] * n, **kw) == want
        if "is_end" in scalar:
            assert dec.partial_decode_beams_batch(*args, is_end=True, force_next_word_list=[False] * n, **kw) == want


# ---- against the reference: the streaming goldens of one group, one batched call per step ------------------------
def run_golden_group(pkg, names, tol=2e-4):
    """The cases `names` (a group of stream_lms.golden_groups) as the streams of one decoder without a model of its
    own, each with its model in language_model_list and its hotwords in hotword_scorer_list: ONE batched call per
    step, each stream with its golden step's own force_next_word and is_end; a case with fewer steps drops out after
    its is_end step.  Returns the number of batched calls."""
    g, s = goldens.load(), goldens.load_stream()
    cases = [next(c for c in s["meta"]["cases"] if c["name"] == name) for name in names]
    labels = cases[0]["labels"]
    dec = pkg.BeamSearchDecoderCTC(pkg.Alphabet.build_alphabet(labels), None)
    lms, xs = [], []
    for case in cases:
        lms.append(goldens.build_product_decoder(pkg, labels, **goldens.lm_kwargs(g, case))._language_model)
        xs.append(s["arrays"][case["array"]] if case["array"] in s["arrays"] else g["arrays"][case["array"]])
    beams = [list(dec.get_starting_state()[0]) for _ in cases]
    caches = [sl.start(dec, lm) for lm in lms]
    common = cases[0]["common"]
    calls = 0
    for step_i in range(max(len(c["steps"]) for c in cases)):
        idx = [i for i, case in enumerate(cases) if step_i < len(case["steps"])]
        steps = [cases[i]["steps"][step_i] for i in idx]
        scorers = []
        for st in steps:
            hw = st["call"].get("hotwords")
            scorers.append(None if hw is None else pkg.HotwordScorer.build_scorer(hw, weight=st["call"].get("hotword_weight", 10.0)))
        out = dec.partial_decode_beams_batch([xs[i][st["start"]:st["end"]] for i, st in zip(idx, steps)], [caches[i] for i in idx],
                                             [beams[i] for i in idx], [st["start"] for st in steps],
                                             hotword_scorer_list=scorers, language_model_list=[lms[i] for i in idx],
                                             force_next_word_list=[bool(st["call"].get("force_next_word", False)) for st in steps],
                                             is_end_list=[bool(st["is_end"]) for st in steps], **common)
        calls += 1
        for i, st, o in zip(idx, steps, out):
            why = sl._match(o, st["beams"], tol)
            assert not why, "%s call %d: %s" % (names[i], step_i, why)
            beams[i] = o
        for i, st in zip(idx, steps):
            assert st["is_end"] == (step_i == len(cases[i]["steps"]) - 1), "%s: is_end before its last step" % names[i]
    return calls


def golden_steps(names):
    """The largest number of steps among the cases `names`."""
    s = goldens.load_stream()
    return max(len(c["steps"]) for c in s["meta"]["cases"] if c["name"] in names)


# ---- errors ---------------------------------------------------------------------------------------------------------
def check_errors(dec, xs):
    """ValueError of partial_decode_beams_batch(is_end_list / force_next_word_list); after each refused call the
    decoder decodes the next call as before."""
    from pytest import raises
    n = len(xs)
    start = dec.get_starting_state()
    args = ([x[:30] for x in xs], [start[1]] * n, [list(start[0]) for _ in xs], [0] * n)
    flags = [i % 2 == 0 for i in range(n)]
    want = dec.partial_decode_beams_batch(*args, is_end_list=flags, beam_width=8)
    for bad in (dict(is_end_list=flags[:-1]), dict(force_next_word_list=flags + [True]), dict(is_end_list=[]),
                dict(is_end=True, is_end_list=flags), dict(force_next_word=True, force_next_word_list=flags)):
        with raises(ValueError):
            dec.partial_decode_beams_batch(*args, beam_width=8, **bad)
        assert dec.partial_decode_beams_batch(*args, is_end_list=flags, beam_width=8) == want, bad
    # is_end=False / force_next_word=False next to a list is what the defaults give
    assert dec.partial_decode_beams_batch(*args, is_end=False, force_next_word=False, is_end_list=flags, beam_width=8) == want


def check_abi(dec, xs):
    """The C ABI: utt_finalize_mode on a streaming call without stream_states (every utterance from EMPTY_START_BEAM at
    frame 0) equals one call per utterance with its finalize_mode and an empty stream state; B2C_E_ARG for a mode outside [0, 2] and for
    finalize_mode != B2C_FIN_EOS together with the array, and the decoder's next call is unchanged after each."""
    from pyctcdecode_b200 import _lib
    L = _lib.lib()
    handle = dec._handle(None)
    n = len(xs)
    ptrs = (C.c_void_p * n)(*[x.ctypes.data for x in xs])
    Ts = (C.c_int32 * n)(*[len(x) for x in xs])

    def call(idx, modes=None, finalize_mode=_lib.FIN_EOS, empty_states=False):
        opts = _lib.DecodeOpts()
        L.b2c_decode_opts_default(C.byref(opts))
        opts.beam_width = 8
        opts.max_out_beams = 8
        opts.finalize_mode = finalize_mode
        states = (_lib.StreamState * len(idx))()
        if empty_states:
            opts.stream_states = C.cast(states, C.POINTER(_lib.StreamState))
        arr = None
        if modes is not None:
            arr = (C.c_int32 * len(modes))(*modes)
            opts.utt_finalize_mode = C.cast(arr, C.POINTER(C.c_int32))
        p = (C.c_void_p * len(idx))(*[ptrs[i] for i in idx])
        t = (C.c_int32 * len(idx))(*[Ts[i] for i in idx])
        res = C.c_void_p()
        rc = L.b2c_decode_batch(handle, p, t, len(idx), 0, 0, C.byref(opts), C.byref(res))    # float32 logits
        if rc != 0:
            return rc, None
        try:
            got = []
            for u in range(len(idx)):
                beams = []
                for b in range(L.b2c_result_n_beams(res, u)):
                    aux = (C.c_int32 * 4)()
                    toks, nt = C.POINTER(C.c_uint32)(), C.c_int32()
                    assert L.b2c_result_stream_beam(res, u, b, C.byref(aux), C.byref(toks), C.byref(nt)) == 0
                    beams.append((L.b2c_result_logit_score(res, u, b), L.b2c_result_lm_score(res, u, b), tuple(aux),
                                  tuple(toks[k] for k in range(nt.value))))
                got.append(beams)
            return rc, got
        finally:
            L.b2c_result_free(res)

    modes = [i % 3 for i in range(n)]
    assert len(set(modes)) == 3
    rc, got = call(list(range(n)), modes)
    assert rc == 0, L.b2c_last_error()
    for u in range(n):
        rc1, one = call([u], finalize_mode=modes[u], empty_states=True)
        assert rc1 == 0 and got[u] == one[0], u
    assert any(len({repr(call([u], finalize_mode=m, empty_states=True)[1]) for m in range(3)}) == 3 for u in range(n))
    for bad, fin in (([3] + modes[1:], _lib.FIN_EOS), ([-1] + modes[1:], _lib.FIN_EOS), (modes, _lib.FIN_FLUSH),
                     (modes, _lib.FIN_KEEP)):
        rc, _ = call(list(range(n)), bad, fin)
        assert rc == -1, (bad, fin)
        assert "finalize_mode" in L.b2c_last_error().decode("utf-8")
        assert call(list(range(n)), modes) == (0, got)
