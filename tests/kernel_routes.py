"""Every beam-kernel instantiation and the arena-overflow retry pass, case by case against the oracle, with the kernels
each call launched read back from b2c_timings_t.kernels.  Shared by tests/test_hostsim_kernel_routes.py and
tests/test_gpu_kernel_routes.py.

Route table (csrc/b2c_api.cu: make_plan / plan_launch pick the launch, launch_beam the instantiation; bit = the bit of
b2c_timings_t.kernels, include/b200ctc.h).  Every route is forced by a switch, never inferred from the SM count or a
timing, so the hostsim twin asserts the same bits before anything runs on a GPU:

  bit  instantiation                     forced by                                 cases
  0    b2c_beam_fast_kernel<1024,2,64>   B200CTC_V5_VARIANT=0, V <= 64             v5a_*
  1    b2c_beam_fast_kernel<1024,2,0>    B200CTC_V5_VARIANT=0, V > 64              v5a_g65_*, v5a_bpe_*
  2    b2c_beam_fast_kernel<512,3,64>    B200CTC_V5_VARIANT=1, V <= 64             v5b_*
  3    b2c_beam_fast_kernel<512,3,0>     B200CTC_V5_VARIANT=1, V > 64              v5b_g65_*, v5b_bpe_*
  4    b2c_beam_fast_kernel<256,4,64>    B200CTC_V5_VARIANT=2, V <= 64             v5c_*
  5    b2c_beam_fast_kernel<256,4,0>     B200CTC_V5_VARIANT=2, V > 64              v5c_g65_*, v5c_bpe_*
  6    b2c_beam_kernel<true,256,1>       B200CTC_FORCE_CLASS=4 (class 2048; class 4096 never fits the 200 KB of shared
                                         memory a layout may take, B200CTC_FORCE_CLASS=5 is refused)   cls2048_*
  7    b2c_beam_kernel<true,128,2>       B200CTC_FORCE_CLASS=2 / 3 (classes 512 / 1024)                cls512_*, cls1024_*
  8    b2c_beam_kernel<true,64,4>        B200CTC_FORCE_CLASS=1 (class 256)                             cls256_*
  9    b2c_beam_kernel<true,32,8>        B200CTC_FORCE_CLASS=0 (class 128)                             cls128_*
  10   b2c_beam_kernel<false,256,1>      B200CTC_FORCE_CLASS=general, a launch of at most n_sm utterances whose
                                         widest shared-memory tier leaves one CTA per SM               gen256_*
  11   b2c_beam_kernel<false,512,1>      B200CTC_FORCE_CLASS=general, beam tables in HBM (beam 1200 and up)  gen512_*
  12   b2c_beam_kernel<false,128,2>      B200CTC_FORCE_CLASS=general, more utterances than SMs (the 512-candidate
                                         tier keeps two CTAs per SM)                                   gen128_*

The one- and two-warp class kernels and the 512-thread general kernel run their warp-count-dependent code (per-warp
bucket copies, b2c_bucket_scan_block, B2C_FOR_WARP) only on the device: hostsim runs every CTA with 8 simulated warps.
The classes 128 and 256 get diffuse frames wider than their tier, so that their HBM-tier step runs too
(oversize_frames > 0).

Retry pass (retry_failed): B200CTC_TEXT_ARENA=1 leaves a first pass only the root text node, so the first word an
utterance commits overflows its arena (B2C_ERR_TEXT_FULL) and the host decodes it again on the general kernel with
worst-case arenas.  The class and general kernels commit a text node at every word boundary; the latency-first kernel
only for utterances with a language model or hotwords, except in the frames wider than its shared-memory tier, which
take the general step (b2c_frame_step_slow) and commit every word; the utterances without either are peaky here.  So `retried` is exact: the utterances with a committed word
(T >= 2 and a top beam of two words or more; the batches hold no other kind) in the kernels that commit.  The results
must be bit-identical to the same call without the switch (texts, word frames, both scores, LM end states), and the
call after it, planned from the retried call's statistics, too.
"""
import numpy as np

BITS = {"fast_1024_lt": 0, "fast_1024": 1, "fast_512_lt": 2, "fast_512": 3, "fast_256_lt": 4, "fast_256": 5,
        "class_256t": 6, "class_128t": 7, "class_64t": 8, "class_32t": 9, "general_256t": 10, "general_512t": 11,
        "general_128t": 12}
GENERAL_BITS = (BITS["general_256t"], BITS["general_512t"], BITS["general_128t"])
SWITCHES = ("B200CTC_FORCE_CLASS", "B200CTC_TEXT_ARENA", "B200CTC_FORCE_V5", "B200CTC_V5_VARIANT", "B200CTC_NO_V5",
            "B200CTC_FORCE_CHUNKS", "B200CTC_PIPELINE", "B200CTC_PIPELINE_ALL", "B200CTC_NO_GATE", "B200CTC_NO_HINTED")


def v5_env(variant):
    return {"B200CTC_FORCE_V5": "1", "B200CTC_V5_VARIANT": str(variant)}


def class_env(c):
    return {"B200CTC_FORCE_CLASS": str(c)}


# ---- families -----------------------------------------------------------------------------------------------------
class Family:
    """An alphabet, a language model over it (the decoders' own model is none: the LM is given per utterance), the
    oracles of the model and of no model, and hotwords."""

    def __init__(self, pkg, oracle_mod, key):
        from tests import synth
        if key == "b32":
            wl = synth.CharWorkload("B", n_words=300, lm_order=3)                 # V = 32: the label table is resident
        elif key == "g65":
            wl = synth.CharWorkload(65, n_words=300, lm_order=3)                  # V = 65: staged labels
        else:
            wl = synth.BpeWorkload(n_words=3000, lm_order=4, V=1024)              # BPE, V = 1024
        self.key, self.wl, self.V = key, wl, wl.V
        self.lm_kw = dict(kenlm_model_path=wl.arpa, unigrams=wl.words, alpha=0.5, beta=1.0)
        self.lm = pkg.LanguageModel(pkg.NgramModel(wl.arpa), wl.words, alpha=0.5, beta=1.0)
        self.pkg = pkg
        self.ora = {True: oracle_mod.OracleDecoder(wl.labels, **self.lm_kw), False: oracle_mod.OracleDecoder(wl.labels)}
        self.hot = [wl.words[3], wl.words[8] + " " + wl.words[11]]

    def decoder(self, lm=None):
        return self.pkg.BeamSearchDecoderCTC(self.pkg.Alphabet.build_alphabet(self.wl.labels), lm)

    def batch(self, n, T, seed, kinds=("peaky", "diffuse", "int", "short")):
        """n utterances cycling through `kinds`: peaky, diffuse, integer-valued logits (exact score ties) of T frames,
        and "short": T = 0 and T = 1 in turn."""
        xs = []
        for i in range(n):
            kind = kinds[i % len(kinds)]
            t = (0 if (i // len(kinds)) % 2 == 0 else 1) if kind == "short" else T
            if t == 0:
                xs.append(np.zeros((0, self.V), np.float32))
                continue
            x = self.wl.utterance(seed + i, t, "diffuse" if kind == "diffuse" else "peaky")
            xs.append(np.round(x).astype(np.float32) if kind == "int" else x)
        return xs

    def lms(self, n, every=3):
        """The model for every utterance except each `every`-th (from the second on)."""
        return [None if i % every == 1 else self.lm for i in range(n)]

    def hots(self, n):
        return [self.hot if i % 4 == 0 else None for i in range(n)]


_FAMILIES = {}


def family(pkg, oracle_mod, key):
    if key not in _FAMILIES:
        _FAMILIES[key] = Family(pkg, oracle_mod, key)
    return _FAMILIES[key]


# ---- comparisons --------------------------------------------------------------------------------------------------
def beams_of(out):
    return [(b.text, [(w, tuple(int(v) for v in f)) for w, f in b.text_frames], b.logit_score, b.lm_score) for b in out]


def _state(s):
    """An LM end state as plain data: words, backoffs (and so its length); a MultiLanguageModel state model by model."""
    if s is None:
        return None
    if hasattr(s, "states"):
        return tuple(_state(x) for x in s.states)
    return (s.words, s.backoffs)


def states_of(out):
    return [_state(b.last_lm_state) for b in out]


def compare_oracle(want, got, where, tol=1e-9):
    """Same beams, texts and word frames; scores within `tol` relative."""
    assert len(want) == len(got), "%s: %d beams, oracle %d" % (where, len(got), len(want))
    for k, (r, g) in enumerate(zip(want, got)):
        assert r[0] == g[0], "%s beam %d: text %r, oracle %r" % (where, k, g[0], r[0])
        assert [(w, tuple(f)) for w, f in r[1]] == g[1], "%s beam %d: word frames" % (where, k)
        assert abs(r[2] - g[2]) <= tol * max(1.0, abs(r[2])), "%s beam %d: logit score %r, oracle %r" % (where, k, g[2], r[2])
        assert abs(r[3] - g[3]) <= tol * max(1.0, abs(r[3])), "%s beam %d: lm score %r, oracle %r" % (where, k, g[3], r[3])


def oracle_beams(fam, xs, lms, hots, **kw):
    return [fam.ora[lm is not None].decode_beams(x, hotwords=h, **kw) for x, lm, h in zip(xs, lms, hots)]


def check_oracle_beams(fam, xs, lms, hots, got, **kw):
    for i, (want, g) in enumerate(zip(oracle_beams(fam, xs, lms, hots, **kw), got)):
        compare_oracle(want, beams_of(g), "utterance %d (T=%d)" % (i, xs[i].shape[0]))


def check_oracle_texts(fam, xs, lms, hots, texts, **kw):
    kw = {k: v for k, v in kw.items() if k != "prune_history"}
    for i, (x, lm, h) in enumerate(zip(xs, lms, hots)):
        want = fam.ora[lm is not None].decode(x, hotwords=h, **kw)
        assert texts[i] == want, "utterance %d (T=%d): %r, oracle %r" % (i, x.shape[0], texts[i], want)


# ---- route cases --------------------------------------------------------------------------------------------------
# (name, family, beam_width, switches, n_utts (0: n_sm + 1), T, expected bit, cta_threads, cap_candidates, checks)
# checks: "oversize" -- oversize_frames > 0; "inplace" -- inplace_frames > 0; "no_diffuse" -- no diffuse utterance (a
# diffuse frame of a wide beam fits no class that has room in shared memory: the plan gives it to the general kernel)
def route_cases():
    C = []

    def add(name, fam, bw, env, n, T, bit, threads, cap, checks=()):
        C.append((name, fam, bw, env, n, T, BITS[bit], threads, cap, tuple(checks)))

    for v, (cap, lt, nolt) in enumerate([(1024, "fast_1024_lt", "fast_1024"), (512, "fast_512_lt", "fast_512"),
                                         (256, "fast_256_lt", "fast_256")]):
        tag = "abc"[v]
        for bw in (1, 17, 100, 128):
            add("v5%s_b32_w%d" % (tag, bw), "b32", bw, v5_env(v), 8, 90, lt, 128, cap,
                (("inplace",) if bw > 1 else ()) + (("no_diffuse",) if bw >= 100 else ()))
        for bw in (17, 128):
            add("v5%s_g65_w%d" % (tag, bw), "g65", bw, v5_env(v), 8, 70, nolt, 128, cap, ("no_diffuse",) if bw >= 100 else ())
        add("v5%s_bpe_w100" % tag, "bpe", 100, v5_env(v), 4, 40, nolt, 128, cap, ("no_diffuse",))
    for bw in (1, 17, 100, 129, 256):
        add("cls128_w%d" % bw, "b32", bw, class_env(0), 8, 60, "class_32t", 32, 128, ("oversize",) if bw >= 17 else ())
        add("cls256_w%d" % bw, "b32", bw, class_env(1), 8, 60, "class_64t", 64, 256, ("oversize",) if bw >= 100 else ())
    add("cls128_g65_w200", "g65", 200, class_env(0), 4, 50, "class_32t", 32, 128, ("oversize",))
    add("cls256_bpe_w150", "bpe", 150, class_env(1), 4, 30, "class_64t", 64, 256, ("oversize",))
    for bw in (17, 128, 300):
        add("cls512_w%d" % bw, "b32", bw, class_env(2), 8, 60, "class_128t", 128, 512)
        add("cls1024_w%d" % bw, "b32", bw, class_env(3), 8, 60, "class_128t", 128, 1024)
    add("cls1024_g65_w500", "g65", 500, class_env(3), 4, 40, "class_128t", 128, 1024)
    for bw in (1, 17, 64):
        add("cls2048_w%d" % bw, "b32", bw, class_env(4), 8, 60, "class_256t", 256, 2048)
    add("cls2048_g65_w40", "g65", 40, class_env(4), 4, 50, "class_256t", 256, 2048)
    for bw, fam in ((100, "b32"), (300, "b32"), (500, "b32"), (128, "g65"), (100, "bpe")):
        add("gen256_%s_w%d" % (fam, bw), fam, bw, class_env("general"), 4, 50, "general_256t", 256, 1024)
    for bw in (1200, 2000):
        add("gen512_w%d" % bw, "b32", bw, class_env("general"), 4, 30, "general_512t", 512, 1024)
    for bw, fam in ((17, "b32"), (100, "b32"), (128, "g65")):
        add("gen128_%s_w%d" % (fam, bw), fam, bw, class_env("general"), 0, 12, "general_128t", 128, 512)
    return C


def set_env(monkeypatch, env):
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def run_route_case(pkg, oracle_mod, case, n_sm, monkeypatch):
    name, fkey, bw, env, n, T, bit, threads, cap, checks = case
    fam = family(pkg, oracle_mod, fkey)
    n = n or n_sm + 1
    kinds = ("peaky", "int", "short") if "no_diffuse" in checks else ("peaky", "diffuse", "int", "short")
    xs = fam.batch(n, T, seed=1000 + 37 * len(name), kinds=kinds)
    lms, hots = fam.lms(n), fam.hots(n)
    dec = fam.decoder()
    set_env(monkeypatch, env)
    for prune in (False, True):
        kw = dict(beam_width=bw, prune_history=prune)
        got = dec.decode_beams_batch(None, xs, language_model_list=lms, hotwords_list=hots, **kw)
        tm = dec.last_timings()
        assert tm["kernels"] == 1 << bit, "%s: kernels %#x, expected bit %d" % (name, tm["kernels"], bit)
        assert (tm["cta_threads"], tm["cap_candidates"], tm["retried"]) == (threads, cap, 0), (name, tm)
        if "oversize" in checks:
            assert tm["oversize_frames"] > 0, "%s: no frame took the HBM-tier step" % name
        if "inplace" in checks:
            assert tm["inplace_frames"] > 0, "%s: no in-place frame" % name
        check_oracle_beams(fam, xs, lms, hots, got, **kw)
    texts = dec.decode_batch(None, xs, beam_width=bw, language_model_list=lms, hotwords_list=hots)
    assert dec.last_timings()["kernels"] == 1 << bit, name
    check_oracle_texts(fam, xs, lms, hots, texts, beam_width=bw)


# ---- retry cases --------------------------------------------------------------------------------------------------
# (name, family, beam_width, route switches, first-pass bit (None: a general-kernel bit), commits only with an LM or
#  hotwords (the latency-first kernel), call)
# call: "beams" (decode_beams_batch, with LM end states), "texts" (decode_batch: narrow chain nodes), "partial"
# (partial_decode_beams_batch with carried words), "pipelined" (a [B, T, V] host block, chunked or gated), "hinted",
# "multi" (language_model_list with None and a two-model MultiLanguageModel), "hot" (hotwords_list, no model)
def retry_cases():
    C = []
    for v, (lt, nolt) in enumerate([("fast_1024_lt", "fast_1024"), ("fast_512_lt", "fast_512"), ("fast_256_lt", "fast_256")]):
        C.append(("v5%s_beams" % "abc"[v], "b32", 32, v5_env(v), BITS[lt], True, "beams"))
        C.append(("v5%s_g65_texts" % "abc"[v], "g65", 24, v5_env(v), BITS[nolt], True, "texts"))
    C += [
        ("cls256_beams", "b32", 150, class_env(1), BITS["class_64t"], False, "beams"),
        ("cls128_texts", "b32", 48, class_env(0), BITS["class_32t"], False, "texts"),
        ("general_beams", "b32", 40, class_env("general"), None, False, "beams"),
        ("general_bpe_texts", "bpe", 24, class_env("general"), None, False, "texts"),
        ("v5a_chunks3", "b32", 32, dict(v5_env(0), B200CTC_FORCE_CHUNKS="3"), BITS["fast_1024_lt"], True, "beams"),
        ("v5a_pipelined_chunked", "b32", 16, dict(B200CTC_PIPELINE="1", B200CTC_PIPELINE_ALL="1", B200CTC_NO_GATE="1"),
         BITS["fast_1024_lt"], True, "pipelined"),
        ("v5a_pipelined_gated", "b32", 16, dict(B200CTC_PIPELINE="1", B200CTC_PIPELINE_ALL="1"), BITS["fast_1024_lt"], True,
         "pipelined"),
        ("v5a_hinted", "b32", 32, {}, BITS["fast_1024_lt"], True, "hinted"),
        ("partial_carried_words", "b32", 24, {}, None, False, "partial"),
        ("multi_lm_sets", "b32", 24, {}, None, False, "multi"),
        ("v5a_hotwords_list", "b32", 32, v5_env(0), BITS["fast_1024_lt"], True, "hot"),
    ]
    return C


def _wordy(xs, texts):
    """Every utterance has T <= 1 (no word can be committed) or a top beam of two words or more (one was)."""
    out = []
    for i, (x, t) in enumerate(zip(xs, texts)):
        T = x.shape[0]
        many = len(t.split()) >= 2
        assert T <= 1 or many, "utterance %d (T=%d) has a one-word transcript %r: the expected retry count is not exact" % (i, T, t)
        out.append(T > 1)
    return out


def _expect_retried(wordy, lms, hots, scored_only):
    return sum(1 for w, lm, h in zip(wordy, lms, hots) if w and (not scored_only or lm is not None or h is not None))


def _check_kernels(tm, first, name):
    k = tm["kernels"]
    gen = [b for b in GENERAL_BITS if k & (1 << b)]
    assert gen, "%s: no general-kernel launch in %#x" % (name, k)
    if first is not None:
        assert k & (1 << first), "%s: first-pass bit %d missing from %#x" % (name, first, k)
        assert k & ~(1 << first) & ~sum(1 << b for b in GENERAL_BITS) == 0, "%s: kernels %#x" % (name, k)


def run_retry_case(pkg, oracle_mod, case, monkeypatch):
    name, fkey, bw, env, first, scored_only, call = case
    fam = family(pkg, oracle_mod, fkey)
    T = 40 if fkey == "bpe" else 80
    if call == "partial":
        return _retry_partial(fam, name, bw, env, monkeypatch)
    if call == "pipelined":
        n = 6
        xs = [fam.wl.utterance(2000 + i, 320, "peaky" if i % 2 else "diffuse") for i in range(n)]
        block = np.stack(xs)
    else:
        n = 8
        xs = fam.batch(n, T, seed=3000 + 11 * len(name), kinds=("peaky", "diffuse", "int", "short"))
    if call == "hot":
        lms, hots = [None] * n, [fam.hot if i % 2 == 0 else None for i in range(n)]
    elif call == "multi":
        lms, hots = _multi_lms(pkg, fam, n), [None] * n
    else:
        # the utterances without a model or hotwords are the integer-logit and the short ones: peaky frames, which the
        # latency-first kernel's own steps take (its out-of-line step for wider frames commits every word)
        lms, hots = [None if i % 4 in (2, 3) else fam.lm for i in range(n)], fam.hots(n)
    dec = fam.decoder()
    texts_only = call in ("texts", "pipelined")

    def decode(inp=None):
        inp = xs if inp is None else inp
        if texts_only:
            return dec.decode_batch(None, inp, beam_width=bw, language_model_list=lms, hotwords_list=hots)
        return dec._run(inp, bw, -10.0, -5.0, False, None, 10.0, max_out_beams=bw, with_state=True,
                        hotwords_list=hots, language_model_list=lms)

    def key(out):
        return out if texts_only else [(beams_of(b), states_of(b)) for b in out]

    set_env(monkeypatch, env)
    if call == "pipelined":
        want = decode(block)
        plain = dec.last_timings()["launches"]
    else:
        want = decode()
    tm0 = dec.last_timings()
    assert tm0["retried"] == 0, (name, tm0)
    top = want if texts_only else [b[0].text if b else "" for b in want]
    wordy = _wordy(xs, top)
    expect = _expect_retried(wordy, lms, hots, scored_only)
    assert expect > 0, name
    monkeypatch.setenv("B200CTC_TEXT_ARENA", "1")
    for rep in range(2):       # the second call is planned from the statistics of the retried one
        got = decode(block if call == "pipelined" else None)
        tm = dec.last_timings()
        assert key(got) == key(want), "%s call %d: results differ from the call without B200CTC_TEXT_ARENA" % (name, rep)
        assert tm["retried"] == expect, "%s call %d: retried %d, expected %d" % (name, rep, tm["retried"], expect)
        _check_kernels(tm, first, name)
        if call == "pipelined":
            assert tm["launches"] > plain, "%s: call %d was not pipelined" % (name, rep)
        if call == "hinted":
            assert tm["hinted"] == 1, "%s call %d was not hinted" % (name, rep)
    if texts_only:
        check_oracle_texts(fam, xs, lms, hots, got, beam_width=bw)
    else:
        single = [i for i, lm in enumerate(lms) if lm is None or lm is fam.lm]
        for i in single:
            want_o = fam.ora[lms[i] is not None].decode_beams(xs[i], beam_width=bw, hotwords=hots[i])
            compare_oracle(want_o, beams_of(got[i]), "%s utterance %d" % (name, i))


def _multi_lms(pkg, fam, n):
    other = pkg.LanguageModel(pkg.NgramModel(fam.wl.arpa), fam.wl.words, alpha=0.9, beta=0.25)
    ab = pkg.MultiLanguageModel([fam.lm, other])
    return [[fam.lm, None, ab][i % 3] for i in range(n)]


def _retry_partial(fam, name, bw, env, monkeypatch):
    """partial_decode_beams_batch: the first chunk without the switch, the rest with and without it from the same
    beams (whose words are replayed into the text arena, and overflow it).  Every stream's final beams match the
    oracle's decode of the whole utterance (chunked streaming decodes as the whole utterance does)."""
    dec = fam.decoder(fam.lm)
    T, a = 120, 50
    xs = [fam.wl.utterance(4000 + i, T, "peaky" if i % 2 else "diffuse") for i in range(4)]
    set_env(monkeypatch, env)
    states = [dec.get_starting_state() for _ in xs]
    caches = [s[1] for s in states]
    beams = dec.partial_decode_beams_batch([x[:a] for x in xs], caches, [s[0] for s in states], [0] * len(xs), beam_width=bw)
    assert all(b[0].text for b in beams), "the first chunk must carry words into the second"
    rest = [x[a:] for x in xs]
    want = dec.partial_decode_beams_batch(rest, caches, beams, [a] * len(xs), beam_width=bw, is_end=True)
    assert dec.last_timings()["retried"] == 0
    monkeypatch.setenv("B200CTC_TEXT_ARENA", "1")
    for rep in range(2):
        got = dec.partial_decode_beams_batch(rest, caches, beams, [a] * len(xs), beam_width=bw, is_end=True)
        tm = dec.last_timings()
        assert repr(got) == repr(want), "%s call %d: results differ from the call without B200CTC_TEXT_ARENA" % (name, rep)
        assert tm["retried"] == len(xs), (name, tm["retried"])
        _check_kernels(tm, None, name)
    for i, x in enumerate(xs):
        ref = fam.ora[True].decode_beams(x, beam_width=bw)
        assert [r[0] for r in ref] == [g.text for g in got[i]], "%s stream %d" % (name, i)
        for r, g in zip(ref, got[i]):
            assert [f for _, f in r[1]] == [tuple(f) for f in g.text_frames], "%s stream %d: frames" % (name, i)
            assert abs(r[2] - g.logit_score) <= 1e-9 * max(1.0, abs(r[2]))
            assert abs(r[3] - g.lm_score) <= 1e-9 * max(1.0, abs(r[3]))


def reset_families():
    """Forget the cached families (their models belong to the library that was bound when they were built)."""
    _FAMILIES.clear()


def run_natural_overflow(pkg, oracle_mod):
    """No switch: a diffuse input whose word commits exceed the default text arena (beam_width * T / 4 + 4096 nodes).
    Every other frame makes the space the best token by far, so that nearly every beam finishes a word there; a
    model without weight or unknown-word penalty and a wide pruning margin keep the beams apart."""
    fam = family(pkg, oracle_mod, "b32")
    wl = fam.wl
    rng = np.random.default_rng(1)
    T = 300
    x = rng.normal(0, 1.0, (T, wl.V)).astype(np.float32)
    x[:, wl.blank_id] -= 2
    x[0::2, wl.space_id] += 6
    x[1::2, wl.space_id] -= 3
    xs = [x, wl.utterance(77, 120, "peaky")]
    kw = dict(kenlm_model_path=wl.arpa, unigrams=wl.words, alpha=0.0, beta=0.0, unk_score_offset=0.0)
    lm = pkg.LanguageModel(pkg.NgramModel(wl.arpa), wl.words, alpha=0.0, beta=0.0, unk_score_offset=0.0)
    dec = fam.decoder(lm)
    dkw = dict(beam_width=64, beam_prune_logp=-50.0)
    got = dec.decode_beams_batch(None, xs, **dkw)
    tm = dec.last_timings()
    assert tm["retried"] == 1, tm
    assert tm["kernels"] == (1 << BITS["class_256t"]) | (1 << BITS["general_256t"]), "kernels %#x" % tm["kernels"]
    ora = oracle_mod.OracleDecoder(wl.labels, **kw)
    for i, (want, g) in enumerate(zip(ora.decode_beams_batch(xs, **dkw), got)):
        compare_oracle(want, beams_of(g), "utterance %d" % i)
