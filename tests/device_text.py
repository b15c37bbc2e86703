"""decode_batch transcripts written on the device (b2c_walk_text in b2c_finalize, joined by b2c_join_block) against the
token-chain path of decode_beams_batch, which builds the same top beam's text on the host, and against the oracle.
Shared by tests/test_hostsim_device_text.py and tests/test_gpu_device_text.py.

The alphabets cover what the walk branches on: one-byte and multi-byte UTF-8 labels, empty pieces (a lone U+2581 in a
BPE alphabet, blanks from <pad> / [PAD]), duplicate labels, BPE pieces with and without U+2581, and pieces long
enough that the joined transcripts outgrow the token-chain bytes the call copies back at once (the rest is copied
after the synchronise).  Every case also reads the text-only result through b2c_result_text and b2c_result_packed,
which build its beams from the joined buffer on first use."""
import ctypes as C
import string

import numpy as np

BPE = "▁"

# name -> (labels, is a BPE alphabet)
ALPHABETS = {
    "char29": ([""] + [" "] + list(string.ascii_lowercase) + ["'"], False),
    "utf8": (["", " ", "é", "ü", "中", "文", "a", "b", "<pad>", "x", "[PAD]"], False),
    "bpe_long": (["", BPE, BPE + "internationalization", "ization", BPE + "中文字", "s", BPE + "a",
                  "été", BPE + "b", "xyzxyzxyz", "<pad>"], True),
}


def labels_of(name):
    return ALPHABETS[name][0]


def utterances(V, n, T, seed, long_runs=False):
    """n utterances of T frames (one of T = 0 and one of T = 1 among them when n >= 4).  long_runs: a new non-blank token
    in nearly every frame (one emitted piece per frame: the transcripts outgrow 4 bytes per frame)."""
    rng = np.random.default_rng(seed)
    xs = []
    for i in range(n):
        t = 0 if (n >= 4 and i == 1) else (1 if (n >= 4 and i == 2) else T)
        x = rng.normal(0.0, 1.0, (t, V)).astype(np.float32)
        for f in range(t):
            tok = (f % (V - 1)) + 1 if long_runs else (0 if rng.random() < 0.35 else int(rng.integers(1, V)))
            x[f, tok] += 6.0 if rng.random() < 0.8 else 1.0
        xs.append(x)
    return xs


def read_result(L, _lib, res, n):
    """texts through b2c_result_text (every beam), and through b2c_result_packed"""
    per_beam = []
    for u in range(n):
        per_beam.append([L.b2c_result_text(res, u, b).decode("utf-8") for b in range(L.b2c_result_n_beams(res, u))])
    pk = _lib.Packed()
    assert L.b2c_result_packed(res, C.byref(pk)) == 0
    packed = C.string_at(pk.texts, pk.texts_size).decode("utf-8").split("\x00")[:-1] if pk.texts_size else []
    scores = [L.b2c_result_logit_score(res, u, 0) for u in range(n) if L.b2c_result_n_beams(res, u) > 0]
    return per_beam, packed, scores


def spy_results(monkeypatch, _lib):
    """Wraps b2c_result_top_texts so that every text-only result is also read through the lazy accessors; returns the
    list the reads are appended to."""
    L = _lib.lib()
    orig = L.b2c_result_top_texts
    seen = []

    def spy(res, data, size):
        rc = orig(res, data, size)
        n = L.b2c_result_n_utts(res)
        seen.append(read_result(L, _lib, res, n))
        return rc

    monkeypatch.setattr(L, "b2c_result_top_texts", spy)
    return seen


def check_call(dec, xs, seen, oracle=None, **kw):
    """decode_batch against the top beam of decode_beams_batch (host-built text), the lazy accessors and the oracle;
    returns the texts and the decode_batch call's timings"""
    del seen[:]
    got = dec.decode_batch(None, xs, **kw)
    tm = dec.last_timings()
    beams = dec.decode_beams_batch(None, xs, prune_history=True, **kw)
    want = [b[0].text for b in beams]
    assert got == want
    assert len(seen) == 1
    per_beam, packed, scores = seen[0]
    assert [p[0] for p in per_beam] == got == packed
    assert all(len(p) == 1 for p in per_beam)
    assert np.allclose(scores, [b[0].logit_score for b in beams], rtol=1e-12, atol=0)
    if oracle is not None:
        okw = {k: v for k, v in kw.items() if k in ("beam_width", "beam_prune_logp", "token_min_logp", "hotwords",
                                                    "hotword_weight")}
        assert got == oracle.decode_batch(xs, **okw)
    return got, tm


# (name, alphabet or kernel_routes family, switches, what the call carries)
CASES = [
    ("char29", "char29", {}, "plain"),
    ("utf8_dups_pads", "utf8", {}, "plain"),
    ("bpe_long_pieces", "bpe_long", {}, "plain"),
    ("bpe_long_rest_copy", "bpe_long", {}, "long_runs"),
    ("b32", "b32", {}, "plain"),
    ("b32_lm", "b32", {}, "lm"),
    ("b32_hotwords", "b32", {}, "hot"),
    ("b32_sets", "b32", {}, "sets"),
    ("bpe1024_lm", "bpe", {}, "lm"),
    ("bpe1024_sets", "bpe", {}, "sets"),
    ("v5a", "b32", {"B200CTC_FORCE_V5": "1", "B200CTC_V5_VARIANT": "0"}, "sets"),
    ("v5b", "b32", {"B200CTC_FORCE_V5": "1", "B200CTC_V5_VARIANT": "1"}, "sets"),
    ("v5c", "b32", {"B200CTC_FORCE_V5": "1", "B200CTC_V5_VARIANT": "2"}, "sets"),
    ("v5a_g65", "g65", {"B200CTC_FORCE_V5": "1", "B200CTC_V5_VARIANT": "0"}, "sets"),
    ("cls128", "b32", {"B200CTC_FORCE_CLASS": "0"}, "sets"),
    ("cls256", "b32", {"B200CTC_FORCE_CLASS": "1"}, "sets"),
    ("cls512", "b32", {"B200CTC_FORCE_CLASS": "2"}, "sets"),
    ("cls1024", "b32", {"B200CTC_FORCE_CLASS": "3"}, "sets"),
    ("cls2048", "b32", {"B200CTC_FORCE_CLASS": "4"}, "sets"),
    ("general", "b32", {"B200CTC_FORCE_CLASS": "general"}, "sets"),
    ("general_bpe_lm", "bpe", {"B200CTC_FORCE_CLASS": "general"}, "lm"),
    ("retry_v5", "b32", {"B200CTC_FORCE_V5": "1", "B200CTC_TEXT_ARENA": "1"}, "retry"),
    ("retry_general", "b32", {"B200CTC_FORCE_CLASS": "general", "B200CTC_TEXT_ARENA": "1"}, "retry"),
    ("chunks3", "b32", {"B200CTC_FORCE_V5": "1", "B200CTC_FORCE_CHUNKS": "3"}, "sets"),
    ("pipelined_chunked", "b32", {"B200CTC_PIPELINE": "1", "B200CTC_PIPELINE_ALL": "1", "B200CTC_NO_GATE": "1"}, "block"),
    ("pipelined_gated", "b32", {"B200CTC_PIPELINE": "1", "B200CTC_PIPELINE_ALL": "1"}, "block"),
    ("hinted", "b32", {}, "hinted"),
    ("packed_tensor", "b32", {}, "tensor"),
]


def run_case(pkg, oracle_mod, case, monkeypatch):
    from pyctcdecode_b200 import _lib
    from tests import kernel_routes as kr

    name, key, env, kind = case
    kr.set_env(monkeypatch, env)
    seen = spy_results(monkeypatch, _lib)
    if key in ALPHABETS:
        labels = labels_of(key)
        dec = pkg.build_ctcdecoder(labels)
        xs = utterances(len(labels), 6, 60, seed=len(name), long_runs=kind == "long_runs")
        got, tm = check_call(dec, xs, seen, oracle_mod.OracleDecoder(labels), beam_width=16)
        if kind == "long_runs":        # the joined transcripts outgrow what the token chains would have copied
            joined = 8 + sum(len(t.encode("utf-8")) + 1 for t in got)
            assert joined > 4 * (sum(x.shape[0] for x in xs) + len(xs)), joined
        assert any(" " in t for t in got), got          # the space rule is exercised
        return
    fam = kr.family(pkg, oracle_mod, key)
    n, T, bw = (4, 30, 16) if key == "bpe" else (8, 50, 16)
    xs = fam.batch(n, T, seed=11)
    if kind == "plain":
        check_call(fam.decoder(), xs, seen, fam.ora[False], beam_width=bw)
    elif kind == "lm":
        check_call(fam.decoder(fam.lm), xs, seen, fam.ora[True], beam_width=bw)
    elif kind == "hot":
        check_call(fam.decoder(), xs, seen, fam.ora[False], beam_width=bw, hotwords=fam.hot)
    elif kind == "sets":
        got, _ = check_call(fam.decoder(), xs, seen, beam_width=bw, language_model_list=fam.lms(n), hotwords_list=fam.hots(n))
        kr.check_oracle_texts(fam, xs, fam.lms(n), fam.hots(n), got, beam_width=bw)
    elif kind == "retry":
        _, tm = check_call(fam.decoder(fam.lm), xs, seen, fam.ora[True], beam_width=bw)
        assert tm["retried"] > 0, tm
    elif kind == "block":
        xs = [fam.wl.utterance(20 + i, T, "diffuse" if i % 2 else "peaky") for i in range(n)]
        block = np.stack(xs)
        plain = fam.decoder(fam.lm)
        want = check_call(plain, xs, seen, fam.ora[True], beam_width=bw)[0]
        launches = plain.last_timings()["launches"]
        got, tm = check_call(plain, block, seen, beam_width=bw)
        assert got == want
        assert tm["launches"] > launches, tm          # the block was decoded as a pipelined call
    elif kind == "hinted":
        dec = fam.decoder(fam.lm)
        flags = []
        for _ in range(3):
            _, tm = check_call(dec, xs, seen, fam.ora[True], beam_width=bw)
            flags.append(tm["hinted"])
        assert flags[-1] == 1, flags
    else:                  # one padded [B, T, V] tensor with lengths
        import torch
        lengths = [x.shape[0] for x in xs]
        pad = np.zeros((n, max(lengths), fam.V), np.float32)
        for i, x in enumerate(xs):
            pad[i, :x.shape[0]] = x
        dec = fam.decoder()
        want = check_call(dec, xs, seen, fam.ora[False], beam_width=bw)[0]
        del seen[:]
        assert dec.decode_batch(None, torch.from_numpy(pad), beam_width=bw, lengths=lengths) == want
        assert [p[0] for p in seen[0][0]] == want

