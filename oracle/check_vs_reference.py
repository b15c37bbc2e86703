"""TEST INFRASTRUCTURE ONLY (needs a checkout of the reference: $PYCTCDECODE_REFERENCE or ../reference).

Differential check of the C++ oracle (oracle/ctc_oracle.cpp) against the UNMODIFIED reference
imported from that checkout with the stand-ins in oracle/refshim.  Run:
    python oracle/check_vs_reference.py [n_random]
Prints one line per case family and exits non-zero on any mismatch that is neither
  (a) a permutation inside a group of beams the reference itself separates by <= `tie` in lm_score
      (tests/goldens.py beams_match_tie_aware: the same beams -- text and word frames -- with scores within
      tolerance, same order between beams that are not tied; tie = 1e-9 for float64 input, 4e-6 for float32 input,
      where numpy's float32 log-softmax adds ~1e-7 of noise per frame to mathematically equal scores), nor
  (b) a case the UNMODIFIED REFERENCE ITSELF decides by rounding noise: re-run on the input perturbed by
      1e-13 * N(0,1) it returns different outcomes, and the oracle's output lies inside that family (same beam
      set, every beam's scores among those the family gives it, list sorted) -- oracle/gen_golden_unstable.py.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ.get("PYCTCDECODE_REFERENCE") or os.path.join(ROOT, os.pardir, "reference")   # the reference checkout
sys.path.insert(0, os.path.join(HERE, "refshim"))
sys.path.insert(0, REF)
sys.path.insert(0, ROOT)

import logging  # noqa: E402

logging.disable(logging.CRITICAL)

from pyctcdecode import build_ctcdecoder  # noqa: E402  (the reference)

from oracle import oracle as orc  # noqa: E402
from tests import goldens, synth  # noqa: E402

SCORE_TOL = 2e-4  # numpy evaluates log-softmax in float32 with its own SIMD exp/log; see DESIGN.md


def reference_unstable(ref_dec, x, dkw, orc_beams, n=16, eps=1e-13):
    """(b) of the module docstring -> (number of distinct outcomes of the reference, '' or why the oracle is outside)"""
    from oracle import gen_golden_unstable as gu
    if x.dtype == np.float32:
        # float32 input is computed in float32 (decoder.py:180-197): the smallest perturbation is a step to a neighbouring
        # float32 -- the size of the run-to-run differences of numpy's own float32 exp / log (SIMD body vs scalar head /
        # tail of a row, depending on the alignment of the buffer), which were seen to flip this case between two runs of
        # this very script
        beams, n_out, same_set = gu.reference_family(ref_dec, x, dkw, n=4 * n, perturb=gu.one_ulp_float32)   # every tied cut doubles the family
    else:
        x = x.astype(np.float64)        # integer / float64 input: the reference computes in float64
        beams, n_out, same_set = gu.reference_family(ref_dec, x, dkw, n=n, eps=eps)
    if n_out < 2:
        return n_out, "the reference is stable under the perturbation"
    if not same_set:
        return n_out, "reference outcomes differ in their beam sets"
    exp = {(b["text"], tuple((w, s, t) for w, s, t in b["frames"])): b["scores"] for b in beams}
    if len(orc_beams) != len(exp):
        return n_out, "beam count"
    for i, b in enumerate(orc_beams):
        key = (b[0], tuple((w, int(f[0]), int(f[1])) for w, f in b[1]))
        if key not in exp:
            return n_out, "beam %d not in the reference's set" % i
        if not any(abs(p[0] - b[2]) <= SCORE_TOL and abs(p[1] - b[3]) <= SCORE_TOL for p in exp[key]):
            return n_out, "beam %d score outside the family" % i
        if i and orc_beams[i - 1][3] < b[3] - 1e-9:
            return n_out, "not sorted"
    return n_out, ""


def compare(ref_beams, orc_beams, tag, stats, ref_dec=None, x=None, dkw=None):
    ok = True
    if len(ref_beams) != len(orc_beams):
        ok = False
    else:
        for rb, ob in zip(ref_beams, orc_beams):
            if rb.text != ob[0] or [tuple(f) for f in rb.text_frames] != [(w, tuple(fr)) for w, fr in ob[1]]:
                ok = False
                break
            if abs(rb.logit_score - ob[2]) > SCORE_TOL + 1e-6 * abs(rb.logit_score) or \
               abs(rb.lm_score - ob[3]) > SCORE_TOL + 1e-6 * abs(rb.lm_score):
                ok = False
                break
    stats["n"] += 1
    if not ok:
        # a permutation inside tie groups?  (same beams, same scores, order free only where the reference's own
        # scores agree to 1e-9)
        exp = [{"text": b.text, "frames": [(w, f[0], f[1]) for w, f in b.text_frames], "logit_score": b.logit_score,
                "lm_score": b.lm_score} for b in ref_beams]
        tie = 4e-6 if (x is not None and x.dtype == np.float32) else 1e-9
        why = goldens.beams_match_tie_aware(exp, orc_beams, tol=SCORE_TOL, tie=tie)
        verdict = "tie permutation (reference scores within %g)" % tie
        if why and ref_dec is not None:
            n_out, outside = reference_unstable(ref_dec, x, dkw, orc_beams)
            noise = "one-ulp float32 input noise" if (x is not None and x.dtype == np.float32) else "1e-13 input noise"
            verdict = ("reference-unstable: %d distinct reference outcomes under %s, oracle inside the family" % (n_out, noise)
                       if not outside else "HARD: %s; %s" % (why, outside))
        elif why:
            verdict = "HARD: " + why
        top_same = bool(ref_beams) and bool(orc_beams) and ref_beams[0].text == orc_beams[0][0]
        stats["mismatch"].append((tag, len(ref_beams), len(orc_beams), top_same, verdict))
    return ok


def main():
    n_random = int(sys.argv[1]) if len(sys.argv) > 1 else 40
    stats = {"n": 0, "mismatch": []}
    ref_tests = os.path.join(REF, "pyctcdecode", "tests")
    arpa = os.path.join(ref_tests, "sample_data", "bugs_bunny_kenlm.arpa")

    # ---- the reference's own fixtures -------------------------------------------------
    sys.path.insert(0, os.path.dirname(ref_tests))
    SAMPLE_LABELS = [" ", "b", "g", "n", "s", "u", "y", ""]
    vocab = {c: n for n, c in enumerate(SAMPLE_LABELS)}

    def onehot(chars):
        m = np.zeros((len(chars), len(SAMPLE_LABELS)))
        for i, c in enumerate(chars):
            m[i][vocab[c]] = 1
        return m

    bugs, bunny = onehot("bugs"), onehot(["b", "u", "n", "", "n", "y"])
    blank, space = onehot([""]), onehot([" "])
    test_probs = np.vstack([np.vstack([bugs, blank, blank]) * 0.49 + bunny * 0.51, space, bunny])
    test_logits = np.log(np.clip(test_probs, 1e-15, 1))
    with open(os.path.join(ref_tests, "sample_data", "libri_logits.json")) as fh:
        libri = np.array(json.load(fh))

    fixtures = [("test_logits", SAMPLE_LABELS, test_logits), ("test_probs", SAMPLE_LABELS, test_probs),
                ("libri", synth.LIBRI_LABELS, libri),
                ("libri_f32", synth.LIBRI_LABELS, libri.astype(np.float32))]
    lm_variants = [dict(), dict(kenlm_model_path=arpa), dict(kenlm_model_path=arpa, unigrams=["bugs", "bunny"]),
                   dict(kenlm_model_path=arpa, unigrams=["bunny"], alpha=1.0),
                   dict(kenlm_model_path=arpa, alpha=1.0, unk_score_offset=0.0, lm_score_boundary=False)]
    dec_variants = [dict(), dict(prune_history=True), dict(hotwords=["bugs"], hotword_weight=20.0),
                    dict(beam_prune_logp=-20.0, token_min_logp=-8.0), dict(beam_width=3),
                    dict(hotwords=["bunny bugs", "i have"], hotword_weight=5.0, prune_history=True)]
    for name, labels, logits in fixtures:
        for li, lmkw in enumerate(lm_variants):
            if "libri" in name and lmkw:
                continue
            ref = build_ctcdecoder(labels, **lmkw)
            mine = orc.OracleDecoder(labels, **lmkw)
            for di, dkw in enumerate(dec_variants):
                compare(ref.decode_beams(logits, **dkw), mine.decode_beams(logits, **dkw), "%s/lm%d/d%d" % (name, li, di), stats,
                        ref, np.asarray(logits), dkw)
    print("fixtures: %d cases, %d mismatches" % (stats["n"], len(stats["mismatch"])))

    # ---- random synthetic -----------------------------------------------------------
    wl_nolm = synth.CharWorkload("B", n_words=2000, lm_order=0)
    wl_lm = synth.CharWorkload("B", n_words=2000, lm_order=3)
    wl_a = synth.CharWorkload("A", n_words=2000, lm_order=2)
    bpe = synth.BpeWorkload(n_words=2000, lm_order=3)
    rng = np.random.default_rng(123)
    fams = [("B/nolm", wl_nolm, {}), ("B/3gram", wl_lm, dict(kenlm_model_path=wl_lm.arpa, unigrams=wl_lm.words, alpha=0.5, beta=1.0)),
            ("A/2gram", wl_a, dict(kenlm_model_path=wl_a.arpa, unigrams=wl_a.words)),
            ("C/bpe-nolm", bpe, {}), ("C/bpe-3gram", bpe, dict(kenlm_model_path=bpe.arpa, unigrams=bpe.words))]
    for fam, wl, lmkw in fams:
        ref = build_ctcdecoder(wl.labels, **lmkw)
        mine = orc.OracleDecoder(wl.labels, **lmkw)
        n0 = stats["n"]
        m0 = len(stats["mismatch"])
        for i in range(n_random):
            T = int(rng.integers(0, 160))
            regime = ["peaky", "diffuse", "flat"][i % 3] if wl.V <= 64 else ["peaky", "diffuse"][i % 2]
            x = wl.utterance(1000 + i, T, regime) if T > 0 else np.zeros((0, wl.V), np.float32)
            if i % 5 == 4:
                x = x.astype(np.float64)
            if i % 7 == 6 and T > 0:
                e = np.exp(x - x.max(1, keepdims=True))
                x = (e / e.sum(1, keepdims=True)).astype(x.dtype)
            dkw = dict(beam_width=[100, 8, 25][i % 3], prune_history=bool(i % 2))
            if i % 4 == 3:
                dkw.update(hotwords=[wl.words[3], wl.words[10] + " " + wl.words[11]], hotword_weight=6.0)
            compare(ref.decode_beams(x, **dkw), mine.decode_beams(x, **dkw), "%s/%d" % (fam, i), stats, ref, x, dkw)
        print("%s: %d cases, %d mismatches" % (fam, stats["n"] - n0, len(stats["mismatch"]) - m0))

    hard = [m for m in stats["mismatch"] if not m[3] or m[4].startswith("HARD")]
    for m in stats["mismatch"]:
        print("NOT-IDENTICAL", m)
    print("total %d cases, %d identical, %d explained (tie order / reference-unstable), %d hard" %
          (stats["n"], stats["n"] - len(stats["mismatch"]), len(stats["mismatch"]) - len(hard), len(hard)))
    return 1 if hard else 0


if __name__ == "__main__":
    sys.exit(main())
