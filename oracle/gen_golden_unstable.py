"""TEST INFRASTRUCTURE ONLY (needs a checkout of the reference: $PYCTCDECODE_REFERENCE or ../reference).

Golden vectors for cases whose reference output is decided by rounding noise.  LibriSpeech logits of the
reference's test data are INTEGER valued, so with wide settings (beam_prune_logp=-20, token_min_logp=-8) many beams
have mathematically equal scores; which of two tied beams survives the beam_width cut -- and therefore which of two
texts later receives its probability mass -- depends on the last bit of numpy's exp/log.  The UNMODIFIED reference
itself returns different results when the input is perturbed by 1e-13 (oracle/check_vs_reference.py prints the
demonstration).  The outcomes form a combinatorial family (every tied cut doubles it: 22 distinct outcomes in 33
runs), so the golden records what is COMMON to the family and what varies:
  * the set of beams (text + word frames) is the same in every outcome -> must be reproduced exactly;
  * per beam the set of (logit_score, lm_score) pairs the reference attaches to it across the family -> a decoder's
    score for that beam must be one of them (beams the noise does not reach have exactly one pair);
  * a decoder's list must be sorted by lm_score (ties in any order).
tests/goldens.py run_unstable_case checks exactly that.

    python oracle/gen_golden_unstable.py      -> tests/golden/unstable_cases.json
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

from tests import synth  # noqa: E402

REF_TESTS = os.path.join(REF, "pyctcdecode", "tests")
OUT = os.path.join(ROOT, "tests", "golden", "unstable_cases.json")
N_PERTURB = 32
EPS = 1e-13


def beams_to_json(beams):
    return [{"text": b.text, "frames": [[w, int(f[0]), int(f[1])] for w, f in b.text_frames],
             "logit_score": float(b.logit_score), "lm_score": float(b.lm_score)} for b in beams]


def signature(beams):
    """what distinguishes two outcomes beyond tie order: which (text, frames) carries which score"""
    return tuple(sorted((b.text, tuple(tuple(f) for _, f in b.text_frames), round(b.lm_score, 6)) for b in beams))


def one_ulp_float32(x, seed):
    """float32 input: the smallest perturbation there is -- about half of the elements move to a neighbouring float32"""
    rng = np.random.default_rng(seed)
    step = rng.integers(-1, 2, size=x.shape)
    out = x.copy()
    out[step > 0] = np.nextafter(x[step > 0], np.float32(np.inf))
    out[step < 0] = np.nextafter(x[step < 0], np.float32(-np.inf))
    return out.astype(np.float32)


def reference_family(dec, x, dkw, n=N_PERTURB, eps=EPS, perturb=None):
    """the unmodified reference on x and on n copies of x perturbed by eps * N(0, 1) (or by `perturb(x, seed)`): ->
    (beams of the unperturbed run with, per beam, every distinct score pair the family gives it; number of distinct
    outcomes; whether every outcome has the same beam set)"""
    seen = set()
    allowed = {}
    base = None
    same_set = True
    for seed in range(n + 1):
        if seed == 0:
            xp = x
        elif perturb is not None:
            xp = perturb(x, seed)
        else:
            xp = x + np.random.default_rng(seed).standard_normal(x.shape) * eps
        beams = dec.decode_beams(xp, **dkw)
        seen.add(signature(beams))
        ids = set()
        for b in beams:
            key = (b.text, tuple(tuple(f) for _, f in b.text_frames))
            ids.add(key)
            pairs = allowed.setdefault(key, [])
            if not any(abs(p[1] - b.lm_score) < 1e-7 and abs(p[0] - b.logit_score) < 1e-7 for p in pairs):
                pairs.append([float(b.logit_score), float(b.lm_score)])
        if base is None:
            base = (beams, ids)
        elif ids != base[1]:
            same_set = False
    out = []
    for b in base[0]:
        key = (b.text, tuple(tuple(f) for _, f in b.text_frames))
        out.append({"text": b.text, "frames": [[w, int(f[0]), int(f[1])] for w, f in b.text_frames], "scores": allowed[key]})
    return out, len(seen), same_set


def main():
    with open(os.path.join(REF_TESTS, "sample_data", "libri_logits.json")) as fh:
        libri = np.array(json.load(fh))
    dec = build_ctcdecoder(synth.LIBRI_LABELS)
    cases = []
    for name, dkw in (("libri_prune20_tok8", dict(beam_prune_logp=-20.0, token_min_logp=-8.0)),
                      ("libri_prune20_tok8_history", dict(beam_prune_logp=-20.0, token_min_logp=-8.0, prune_history=True))):
        beams, n_out, same_set = reference_family(dec, libri, dkw)
        assert same_set, "the family does not share one beam set: record alternatives instead"
        cases.append({"name": name, "labels": synth.LIBRI_LABELS, "array": "libri", "decode": dkw,
                      "reference_outcomes": n_out, "beams": beams})
        print(name, "distinct reference outcomes under %g perturbation: %d; beams with more than one score: %d" %
              (EPS, n_out, sum(len(b["scores"]) > 1 for b in beams)))
    # the same logits as float32: the reference computes the log-softmax in float32 then, and the smallest perturbation is a
    # step to a neighbouring float32 (numpy's own float32 exp / log differ by that much between two runs on identical input:
    # SIMD body vs scalar head / tail of a row, depending on the alignment of the buffer).  Every tied cut doubles the
    # family, so many more perturbations are drawn.  "cpu_only": pinned on the oracle and on the kernel logic (hostsim).
    libri32 = libri.astype(np.float32)
    for name, dkw in (("libri_f32_prune20_tok8", dict(beam_prune_logp=-20.0, token_min_logp=-8.0)),):
        beams, n_out, same_set = reference_family(dec, libri32, dkw, n=6 * N_PERTURB, perturb=one_ulp_float32)
        assert same_set, "the family does not share one beam set: record alternatives instead"
        cases.append({"name": name, "labels": synth.LIBRI_LABELS, "array": "libri_f32", "decode": dkw, "cpu_only": True,
                      "reference_outcomes": n_out, "beams": beams})
        print(name, "distinct reference outcomes under one-ulp float32 perturbations: %d; beams with more than one score: %d" %
              (n_out, sum(len(b["scores"]) > 1 for b in beams)))
    with open(OUT, "w", encoding="utf-8") as fh:
        json.dump({"cases": cases, "generator": "oracle/gen_golden_unstable.py",
                   "reference": "pyctcdecode 0.6.0 @ afecb676, numpy %s" % np.__version__,
                   "perturbation": "x + %g * N(0,1), seeds 1..%d, plus x itself; float32 cases: about half of the elements moved "
                                   "to a neighbouring float32, seeds 1..%d" % (EPS, N_PERTURB, 6 * N_PERTURB)}, fh, ensure_ascii=False, indent=0)


if __name__ == "__main__":
    main()
