"""Differential fuzzing against the oracle: random vocabulary family, LM / hotwords / prune settings, beam widths
from 1 to 300, logits of random sharpness (incl. integer-valued rows for exact ties), whole-utterance decode and
chunked streaming.  TEST TOOL.
    python tools/fuzz_hostsim.py [n_cases] [seed]          kernel LOGIC on the CPU (tests/hostsim build)
    python tools/fuzz_hostsim.py [n_cases] [seed] --cuda   the CUDA library on a GPU box (also: tests/test_gpu_parity.py)
(B200CTC_HOSTSIM_ORDER / B200CTC_NO_V5 / B200CTC_FORCE_V5 apply)
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

import pyctcdecode_b200 as pkg  # noqa: E402
from oracle import oracle as orc  # noqa: E402
from tests import synth  # noqa: E402

FAMS = {
    "B_nolm": (dict(kind="char", vocab="B", n_words=400, lm_order=0), {}),
    "B_3gram": (dict(kind="char", vocab="B", n_words=400, lm_order=3), dict(alpha=0.5, beta=1.0)),
    "A_2gram": (dict(kind="char", vocab="A", n_words=400, lm_order=2), dict()),
    "B_5gram": (dict(kind="char", vocab="B", n_words=150, lm_order=5), dict(alpha=0.9, beta=0.3, unk_score_offset=-4.0)),
    "C_bpe": (dict(kind="bpe", n_words=400, lm_order=0), {}),
    "C_bpe_4gram": (dict(kind="bpe", n_words=400, lm_order=4), dict(alpha=0.7, beta=2.0)),
    "G5": (dict(kind="char", vocab=5, n_words=300, lm_order=0), {}),
    "G36_3gram": (dict(kind="char", vocab=36, n_words=400, lm_order=3), dict(alpha=0.5, beta=1.0)),
    "G64": (dict(kind="char", vocab=64, n_words=400, lm_order=0), {}),
    "G65_2gram": (dict(kind="char", vocab=65, n_words=400, lm_order=2), dict()),
    "G1025": (dict(kind="char", vocab=1025, n_words=400, lm_order=0), {}),
    "C_bpe64": (dict(kind="bpe", n_words=400, lm_order=0, V=64), {}),
    "C_bpe2000_3gram": (dict(kind="bpe", n_words=3000, lm_order=3, V=2000), dict(alpha=0.5, beta=1.0)),
}


def same(ref, got, tol=1e-9):
    if len(ref) != len(got):
        return False
    for r, g in zip(ref, got):
        if r[0] != g.text or [(w, tuple(f)) for w, f in r[1]] != [(w, tuple(f)) for w, f in g.text_frames]:
            return False
        if abs(r[2] - g.logit_score) > tol * max(1.0, abs(r[2])) or abs(r[3] - g.lm_score) > tol * max(1.0, abs(r[3])):
            return False
    return True


def main():
    argv = [a for a in sys.argv[1:] if not a.startswith("--")]
    if "--cuda" not in sys.argv:
        from pyctcdecode_b200 import _lib
        subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tests", "hostsim")])
        _lib.use_library(os.path.join(ROOT, "tests", "hostsim", "libb200ctc_hostsim.so"))
    return fuzz(int(argv[0]) if len(argv) > 0 else 300, int(argv[1]) if len(argv) > 1 else 1)


def fuzz(n_cases, seed):
    """runs on whichever library pyctcdecode_b200._lib is bound to; returns the number of mismatches"""
    rng = np.random.default_rng(seed)
    decs = {}
    bad = 0
    stats = {"inplace": 0, "sorted": 0, "frames": 0}
    for case in range(n_cases):
        fam = list(FAMS)[int(rng.integers(len(FAMS)))]
        if fam not in decs:
            wkw, lmkw = FAMS[fam]
            wl = synth.make_workload(wkw)
            kw = dict(lmkw)
            if wl.arpa:
                kw.update(kenlm_model_path=wl.arpa, unigrams=wl.words)
            decs[fam] = (wl, pkg.build_ctcdecoder(wl.labels, **kw), orc.OracleDecoder(wl.labels, **kw))
        wl, dec, ora = decs[fam]
        T = int(rng.integers(1, 160 if wl.V <= 64 else 50))
        regime = ["peaky", "peaky", "diffuse", "flat"][int(rng.integers(4))] if wl.V <= 64 else ["peaky", "diffuse"][int(rng.integers(2))]
        x = wl.utterance(int(rng.integers(1 << 30)), T, regime)
        x = (x * float(rng.choice([0.6, 0.8, 1.0, 1.0, 1.3]))).astype(np.float32)
        rounded = rng.random() < 0.15
        if rounded:
            x = np.round(x).astype(np.float32)
        if rng.random() < 0.1:
            x = x.astype(np.float64)
        kw = dict(beam_width=int(rng.choice([1, 2, 3, 8, 17, 50, 100, 128, 129, 300])), prune_history=bool(rng.integers(2)),
                  beam_prune_logp=float(rng.choice([-10.0, -3.0, -20.0, -40.0])), token_min_logp=float(rng.choice([-5.0, -3.0, -7.0])))
        if rng.random() < 0.3:
            kw.update(hotwords=[wl.words[int(rng.integers(50))], wl.words[int(rng.integers(50))] + " " + wl.words[int(rng.integers(50))]],
                      hotword_weight=float(rng.choice([10.0, 6.0, 25.0])))
        ref = ora.decode_beams(x, **kw)
        got = dec.decode_beams(x, **kw)
        tm = dec.last_timings()
        stats["inplace"] += tm["inplace_frames"]
        stats["sorted"] += tm["sorted_frames"]
        stats["frames"] += tm["frames"]
        ok = same(ref, got)
        # the text-only call (decode: 8-byte backtrack nodes, no word frames) must give the top beam's text
        if ok and rng.random() < 0.5:
            dkw = {k: v for k, v in kw.items() if k != "prune_history"}
            ok = dec.decode(x, **dkw) == (got[0].text if got and kw["prune_history"] else ora.decode(x, **dkw))
            if not ok:
                print("TEXT-ONLY", end=" ")
        # chunked streaming must end in the same beams -- for regular alphabets; with BPE the reference itself resets its
        # force_next_break flag at every call, so its chunked and whole results differ (checked against the reference:
        # the product reproduces the reference's CHUNKED result, tests/golden/stream_cases.json)
        # ... and not for integer-valued logits: the reference decides "probabilities or logits" per CALL from the mean of
        # the row sums (decoder.py:702), which can be exactly 1 for a chunk of integer rows and not for the whole matrix
        if ok and T > 4 and wl.V <= 64 and not rounded and rng.random() < 0.4:
            cuts = sorted(set(int(c) for c in rng.integers(1, T, size=int(rng.integers(1, 4)))))
            beams, cache, pcache = dec.get_starting_state()
            start = 0
            skw = {k: v for k, v in kw.items() if k in ("beam_width", "beam_prune_logp", "token_min_logp", "prune_history")}
            scorer = pkg.HotwordScorer.build_scorer(kw["hotwords"], weight=kw["hotword_weight"]) if "hotwords" in kw else None
            for end in cuts + [T]:
                beams = dec.partial_decode_beams(x[start:end], cache, pcache, beams, start, hotword_scorer=scorer, is_end=(end == T), **skw)
                start = end
            ok = len(beams) == len(ref) and all(b.text == r[0] and [tuple(f) for f in b.text_frames] == [tuple(f) for _, f in r[1]]
                                                and abs(b.lm_score - r[3]) <= 1e-9 * max(1.0, abs(r[3])) for b, r in zip(beams, ref))
            if not ok:
                print("STREAM cuts %r" % (cuts,), end=" ")
                if os.environ.get("FUZZ_DUMP"):
                    import json
                    np.save(os.path.join(os.environ["FUZZ_DUMP"], "case%d_seed%d.npy" % (case, seed)), x)
                    with open(os.path.join(os.environ["FUZZ_DUMP"], "case%d_seed%d.json" % (case, seed)), "w") as fh:
                        json.dump({"fam": fam, "kw": kw, "cuts": cuts}, fh)
        if not ok:
            bad += 1
            print("MISMATCH case %d fam %s T=%d regime %s %r variant %d" % (case, fam, T, regime, kw, tm["kernel_variant"]), flush=True)
    print("cases %d mismatches %d  (frames %d, in place %d, sorted %d)" % (n_cases, bad, stats["frames"], stats["inplace"], stats["sorted"]))
    return bad


if __name__ == "__main__":
    sys.exit(1 if main() else 0)
