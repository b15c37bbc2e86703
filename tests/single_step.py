"""Inputs and checks for the one-token step after a multi-token frame (b2c_fast_single_step), shared by
tests/test_gpu_single_step.py and its hostsim twin.

`merge_cases` builds logits whose frames alternate between two or three selected tokens and one selected token, so
that the one-token frames meet beams that merge in pairs (X.c from token c meets X + c from the blank) and in threes
(X.c, X.b + c, X.b + blank + c), with integer-valued logits (exact score ties), history-pruned holes
(prune_history=True), tight thresholds and beams from 1 to 128.  `check_decoder` compares a decoder with the oracle
and with itself under B200CTC_NO_SINGLE_STEP=1 (the same frames through the general step): transcripts, word frames
and scores must be identical to the general step's, bit for bit."""
import numpy as np

from tests import synth


def merge_cases(wl, n_cases=40, seed=21):
    """Seeded (logits, decode kwargs) pairs of alternating multi-token / one-token frames."""
    rng = np.random.default_rng(seed)
    letters = [i for i in range(wl.V) if i not in (wl.blank_id, wl.space_id)]
    for i in range(n_cases):
        T = int(rng.integers(30, 220))
        integer = i % 3 == 0
        x = np.full((T, wl.V), -12.0)
        prev = int(rng.choice(letters))
        for t in range(T):
            if t % 2 == 0:                  # two or three tokens: the blank, the previous letter, maybe a new one
                toks = {wl.blank_id, prev}
                if rng.random() < 0.6:
                    toks.add(int(rng.choice(letters)))
                if rng.random() < 0.05:
                    toks.add(wl.space_id)
                for k in toks:
                    x[t, k] = 0.0 if integer else rng.normal(0.0, 0.4)
            else:                           # one token: the previous letter (merges), the blank, a new letter or the space
                r = rng.random()
                k = prev if r < 0.45 else (wl.blank_id if r < 0.75 else (wl.space_id if r < 0.8 else int(rng.choice(letters))))
                x[t, k] = 0.0 if integer else rng.normal(0.0, 0.2)
                if k not in (wl.blank_id, wl.space_id):
                    prev = k
            if not integer:
                x[t] += rng.normal(0.0, 0.05, wl.V)
        kw = dict(beam_width=int(rng.choice([1, 2, 5, 17, 50, 100, 128])), prune_history=bool(i % 2),
                  beam_prune_logp=float(rng.choice([-0.7, -2.0, -3.0, -10.0])), token_min_logp=-5.0)
        yield x.astype(np.float32), kw


def all_cases(wl):
    yield from synth.special_step_cases(wl)
    yield from merge_cases(wl)


def _beams(out):
    return [(b.text, [(w, tuple(f)) for w, f in b.text_frames], b.logit_score, b.lm_score) for b in out]


def _close(ref, got, tol=1e-9):
    assert len(ref) == len(got)
    for r, g in zip(ref, got):
        assert r[0] == g[0]
        assert [(w, tuple(f)) for w, f in r[1]] == g[1]
        assert abs(r[2] - g[2]) <= tol * max(1.0, abs(r[2]))
        assert abs(r[3] - g[3]) <= tol * max(1.0, abs(r[3]))


def check_decoder(dec, ora, wl, monkeypatch):
    """Every case through decode_beams and decode_batch, against the oracle and against the general step; returns the
    frames the one-token step took."""
    single = 0
    for n, (x, kw) in enumerate(all_cases(wl)):
        monkeypatch.delenv("B200CTC_NO_SINGLE_STEP", raising=False)
        got = _beams(dec.decode_beams(x, **kw))
        single += dec.last_timings()["single_frames"]
        kb = {k: v for k, v in kw.items() if k != "prune_history"}
        text = dec.decode_batch(None, [x], **kb)
        monkeypatch.setenv("B200CTC_NO_SINGLE_STEP", "1")
        general = _beams(dec.decode_beams(x, **kw))
        assert dec.last_timings()["single_frames"] == 0
        assert got == general, "case %d %r: the one-token step differs from the general step" % (n, kw)
        assert text == dec.decode_batch(None, [x], **kb), "case %d %r" % (n, kw)
        _close(ora.decode_beams(x, **kw), got)
        assert text == ora.decode_batch([x], **kb)
    monkeypatch.delenv("B200CTC_NO_SINGLE_STEP", raising=False)
    return single


def workload():
    return synth.make_workload(dict(kind="char", vocab="B", n_words=400, lm_order=0))
