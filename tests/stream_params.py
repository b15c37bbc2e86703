"""Per-stream search parameters in batched streaming (partial_decode_beams_batch with beam_width_list /
beam_prune_logp_list / token_min_logp_list / prune_history_list), shared by tests/test_gpu_stream_params.py and its
hostsim twin.

The contract: stream i of a batched call returns, bit for bit, what partial_decode_beams returns for it with the same
chunk, cache, beams, processed_frames and flags and its own beam_width, beam_prune_logp, token_min_logp and
prune_history.  The schedules are those of tests/stream_ends.py (continuous batching, ragged chunks, per-stream end
flags); `run` holds every call of every stream to its single-stream reference and can count the streams whose beams
under the first stream's parameters would differ, so that a library that gave every stream one parameter set could not
pass.  `check_token_lists` holds the streaming stage's token lists to numpy's selection with each stream's own
threshold."""
import ctypes as C
import math

from tests import stream_ends as se
from tests import streaming_stage as ss
from tests import synth

DEFAULTS = dict(beam_width=100, beam_prune_logp=-10.0, token_min_logp=-5.0, prune_history=False)
WIDTHS = (1, 2, 16, 100, 128, 129, 300)
PRUNES = (-0.5, -10.0, -40.0)
TOKENS = (-1.0, -5.0, -8.0)
NAMES = ("beam_width", "beam_prune_logp", "token_min_logp", "prune_history")


def params_of(s, widths=WIDTHS):
    """The parameters of stream s: the four values cycle with different periods, so that a call mixes widths,
    thresholds and both history settings."""
    return dict(beam_width=widths[s % len(widths)], beam_prune_logp=PRUNES[s % 3], token_min_logp=TOKENS[(s // 2) % 3],
                prune_history=(s // 3) % 2 == 1)


def tiers(widths):
    """Three parameter tiers (accuracy / latency classes of a server): stream s takes tier s % 3."""
    t = [dict(beam_width=widths[0], beam_prune_logp=-10.0, token_min_logp=-5.0, prune_history=False),
         dict(beam_width=widths[1], beam_prune_logp=-40.0, token_min_logp=-8.0, prune_history=True),
         dict(beam_width=widths[2], beam_prune_logp=-0.5, token_min_logp=-1.0, prune_history=False)]
    return lambda s: t[s % 3]


def run(st, calls, params=params_of, count_differs=False, timings=None, nones=True, **kw):
    """The calls of stream_ends.plan through partial_decode_beams_batch with the four lists and is_end_list /
    force_next_word_list; every stream of every call against partial_decode_beams with its own parameters and flags.
    `kw` are the call's scalars; with `nones`, every fifth stream's entries are None (the scalars).  -> (outputs per
    call, number of (call, stream) whose reference under the parameters of the call's first stream differs from its
    own; 0 without count_differs).  `timings`: gets (last_timings() of every batched call, `retried` sum of its
    references)."""
    dec = st.dec
    scalars = dict(DEFAULTS, **kw)
    beams = {}
    outs = []
    differ = 0

    def own(s):
        return dict(scalars) if nones and s % 5 == 4 else dict(scalars, **params(s))

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
        for name in NAMES:
            extra[name + "_list"] = [None if nones and s % 5 == 4 else params(s)[name] for s in ids]
        out = dec.partial_decode_beams_batch([st.xs[s][t0:t1] for s, t0, t1, _, _ in call], [st.cache(s) for s in ids],
                                             [beams[s] for s in ids], [t0 for _, t0, _, _, _ in call],
                                             force_next_word_list=[f for _, _, _, f, _ in call],
                                             is_end_list=[e for _, _, _, _, e in call], **extra)
        tm = dec.last_timings() if timings is not None else None
        assert len(out) == len(call)
        first = own(call[0][0])
        retried = 0
        for i, (s, t0, t1, f, e) in enumerate(call):
            rd = st.ref_dec(s)
            cache = rd.get_starting_state()[1] if st.lms is not None else st.cache(s)
            hot = st.scorers[s] if st.scorers is not None else None
            mine = own(s)
            ref = rd.partial_decode_beams(st.xs[s][t0:t1], cache, {}, beams[s], t0, hotword_scorer=hot,
                                          force_next_word=f, is_end=e, **mine)
            if timings is not None:
                retried += rd.last_timings()["retried"]
            assert out[i] == ref, "stream %d frames %d..%d %r force_next_word=%s is_end=%s" % (s, t0, t1, mine, f, e)
            assert len(out[i]) <= mine["beam_width"]
            if count_differs and mine != first:
                alt = rd.partial_decode_beams(st.xs[s][t0:t1], cache, {}, beams[s], t0, hotword_scorer=hot,
                                              force_next_word=f, is_end=e, **first)
                differ += alt != ref
            beams[s] = out[i]
        if timings is not None:
            timings.append((tm, retried))
        outs.append(out)
    return outs, differ


def check_uniform(dec, xs, **kw):
    """Lists that repeat the scalars, or hold only None, return what the scalars return; for streams that carry words
    and partial words from a first chunk, with and without per-stream end flags."""
    n = len(xs)
    start = dec.get_starting_state()
    beams = dec.partial_decode_beams_batch([x[:40] for x in xs], [start[1]] * n, [list(start[0]) for _ in xs], [0] * n, **kw)
    assert any(b and b[0].partial_word for b in beams) and any(b and b[0].text for b in beams)
    args = ([x[40:90] for x in xs], [start[1]] * n, beams, [40] * n)
    scalars = dict(DEFAULTS, **kw)
    for flags in (dict(), dict(is_end_list=[i % 2 == 0 for i in range(n)])):
        want = dec.partial_decode_beams_batch(*args, **flags, **kw)
        for lists in ({name + "_list": [scalars[name]] * n for name in NAMES},
                      {name + "_list": [None] * n for name in NAMES},
                      dict(beam_width_list=[scalars["beam_width"]] * n), dict(token_min_logp_list=[None] * n),
                      dict(prune_history_list=[scalars["prune_history"]] * n, beam_prune_logp_list=[None] * n)):
            assert dec.partial_decode_beams_batch(*args, **flags, **lists, **kw) == want, (flags, lists)


# ---- the streaming stage: token lists with per-stream thresholds ----------------------------------------------------
K1_CASES = [("mixed", V, dt) for V in (29, 32, 65, 1024) for dt in ("f32", "f64", "f16")] + [("mixed_prob", 32, "f32"),
                                                                                           ("softmax", 1024, "f64")]


def check_token_lists(orc, dec, content, V, dtype):
    """One streaming call (beam 1) over a case's utterances with one token threshold per stream, among them a
    threshold on a float32 log-prob of one utterance and the next double above it; b2c_decoder_last_tokens then holds,
    utterance by utterance, numpy's selection at that utterance's own threshold in the oracle's set order."""
    name = "%s-V%d-%s-host_list-m5" % (content, V, dtype)
    xs = synth.stream_case_arrays((name, V, content, dtype, "host_list", "m5"))
    assert len(xs) >= 3
    on_lp = dtype == "f32" and content == "mixed"      # a threshold on a float32 log-prob of the longest utterance
    thr_at, pick = ss.resolve_threshold(orc, (name, V, content, dtype, "host_list", ("lp", "at")), xs) if on_lp else (None, None)
    n = len(xs)
    start = dec.get_starting_state()
    for side in ("at", "above"):
        thrs = [(-1.0, -5.0, -8.0, -40.0, ss.LOG_CLIP)[u % 5] for u in range(n)]
        if on_lp:
            thrs[pick[0]] = thr_at if side == "at" else math.nextafter(thr_at, math.inf)
        elif side == "above":
            continue
        dec.partial_decode_beams_batch(xs, [start[1]] * n, [list(start[0]) for _ in xs], [0] * n, beam_width=1,
                                       token_min_logp_list=thrs)
        tok = ss.last_tokens(dec, n)
        total = 0
        f = k = 0
        for u, x in enumerate(xs):
            T = x.shape[0]
            n_u = int(tok["counts"][f:f + T].sum())
            sub = dict(counts=tok["counts"][f:f + T], ids=tok["ids"][k:k + n_u], lps=tok["lps"][k:k + n_u],
                       rec_id0=tok["rec_id0"][f:f + T], rec_lp0=tok["rec_lp0"][f:f + T], is_prob=tok["is_prob"][u:u + 1])
            p = None
            if on_lp and pick[0] == u:
                p = (0, pick[1], pick[2], side == "at")
            ss.check(orc, [x], thrs[u], sub, {"tokens": n_u}, p)
            total += n_u
            f += T
            k += n_u
        assert total == dec.last_timings()["tokens"] == len(tok["ids"])
    return xs


# ---- errors ---------------------------------------------------------------------------------------------------------
def check_errors(dec, xs):
    """ValueError for a list whose length is not the number of streams and for a width outside [1, 65535]; after each
    refused call the decoder decodes the next call as before."""
    from pytest import raises
    n = len(xs)
    start = dec.get_starting_state()
    args = ([x[:30] for x in xs], [start[1]] * n, [list(start[0]) for _ in xs], [0] * n)
    good = dict(beam_width_list=[1 + 3 * i for i in range(n)], token_min_logp_list=[-1.0 - i for i in range(n)])
    want = dec.partial_decode_beams_batch(*args, beam_width=8, **good)
    bads = [dict(beam_width_list=[0] + [4] * (n - 1)), dict(beam_width_list=[65536] + [4] * (n - 1)),
            dict(beam_width_list=[-3] * n), dict(beam_width=0, beam_width_list=[None] * n)]
    for name in NAMES:
        bads += [{name + "_list": [None] * (n - 1)}, {name + "_list": [None] * (n + 1)}, {name + "_list": []}]
    for bad in bads:
        with raises(ValueError):
            dec.partial_decode_beams_batch(*args, **dict(dict(beam_width=8), **bad))
        assert dec.partial_decode_beams_batch(*args, beam_width=8, **good) == want, bad


def check_abi(dec, xs):
    """The C ABI: the four arrays on a call without stream_states, and a width outside [1, 65535], are B2C_E_ARG; the
    decoder's next call is unchanged after each.  With stream_states, utterance i returns at most
    min(max_out_beams, utt_beam_width[i]) beams."""
    from pyctcdecode_b200 import _lib
    L = _lib.lib()
    handle = dec._handle(None)
    n = len(xs)
    ptrs = (C.c_void_p * n)(*[x.ctypes.data for x in xs])
    Ts = (C.c_int32 * n)(*[len(x) for x in xs])
    widths = [1 + 5 * i for i in range(n)]

    def call(stream=True, width=None, prune=None, token=None, history=None, max_out=None):
        opts = _lib.DecodeOpts()
        L.b2c_decode_opts_default(C.byref(opts))
        opts.beam_width = 8
        opts.max_out_beams = max_out if max_out is not None else max(widths)
        keep = []
        if stream:
            states = (_lib.StreamState * n)()
            keep.append(states)
            opts.stream_states = C.cast(states, C.POINTER(_lib.StreamState))
        for field, ctype, vals in (("utt_beam_width", C.c_int32, width), ("utt_beam_prune_logp", C.c_double, prune),
                                   ("utt_token_min_logp", C.c_double, token), ("utt_prune_history", C.c_int32, history)):
            if vals is not None:
                arr = (ctype * n)(*vals)
                keep.append(arr)
                setattr(opts, field, C.cast(arr, C.POINTER(ctype)))
        res = C.c_void_p()
        rc = L.b2c_decode_batch(handle, ptrs, Ts, n, 0, 0, C.byref(opts), C.byref(res))    # float32 logits
        if rc != 0:
            return rc, None
        try:
            return rc, [[(L.b2c_result_logit_score(res, u, b), L.b2c_result_lm_score(res, u, b))
                         for b in range(L.b2c_result_n_beams(res, u))] for u in range(n)]
        finally:
            L.b2c_result_free(res)

    rc, want = call(width=widths)
    assert rc == 0, L.b2c_last_error()
    assert all(len(b) <= w for b, w in zip(want, widths)) and any(len(b) > 1 for b in want)
    rc, capped = call(width=widths, max_out=3)
    assert rc == 0 and [b[:3] for b in want] == capped
    for bad in (dict(stream=False, width=widths), dict(stream=False, prune=[-10.0] * n), dict(stream=False, token=[-5.0] * n),
                dict(stream=False, history=[1] * n), dict(width=[0] + widths[1:]), dict(width=[65536] + widths[1:])):
        rc, _ = call(**bad)
        assert rc == -1, bad
        assert call(width=widths) == (0, want)


def check_not_empty(outs):
    """The schedules decode something: some streams end calls with several beams and text."""
    assert any(len(b) > 1 for out in outs for b in out)
    assert any(b and b[0].text for out in outs for b in out)

