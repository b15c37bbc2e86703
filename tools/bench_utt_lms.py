"""What per-utterance language models cost and save, on one GPU.

    python tools/bench_utt_lms.py [--steps K] [--warmup W] [--out FILE]

C3 shape (V=32, T=1000, batch 1024, beam 100).  Utterances alternate between two synthetic 3-grams over different word
lists (A: bench.py's C3 model, B: another 20k-word list), and every fourth utterance has no language model:
  (a) one decode_batch call with language_model_list;
  (b) one decode_batch call per group on one decoder per model (A, B, none): what a caller without
      language_model_list must do; wall time and beam-kernel ms are the sums over the three calls;
  (c) the whole batch with model A, bench.py's C3 configuration.
For each: wall time per call (host clock around the synchronous call) and beam-kernel ms (CUDA events inside the
library), and the host time the library spends building the language-model sets of (a) (B200CTC_HOST_PROFILE=1).
Prints one JSON line per measurement, with the card's name and power limit.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.bench_utt_hotwords import card, host_profile_ms, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import numpy as np
    import torch
    import __graft_entry__ as g
    g.build()
    import pyctcdecode_b200 as pkg
    from tests import synth

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    info = card()
    lines = []

    def emit(obj):
        obj.update(info)
        lines.append(json.dumps(obj))
        print(lines[-1], flush=True)

    B, T, beam = 1024, 1000, 100
    wa = synth.CharWorkload("B", n_words=20000, lm_order=3)
    wb = synth.CharWorkload("B", n_words=20000, lm_order=3, seed=2)
    lm_a = pkg.LanguageModel(pkg.NgramModel(wa.arpa), wa.words, alpha=0.5, beta=1.0)
    lm_b = pkg.LanguageModel(pkg.NgramModel(wb.arpa), wb.words, alpha=0.5, beta=1.0)
    alphabet = pkg.Alphabet.build_alphabet(wa.labels)
    xs = torch.from_numpy(np.stack(wa.batch(1, B, T, "peaky"))).cuda()
    lms = [None if i % 4 == 3 else (lm_a if i % 2 == 0 else lm_b) for i in range(B)]
    dec = pkg.BeamSearchDecoderCTC(alphabet, lm_a, device=0)
    own = {id(m): pkg.BeamSearchDecoderCTC(alphabet, m, device=0) for m in (lm_a, lm_b, None)}
    groups = {}
    for i, m in enumerate(lms):
        groups.setdefault(id(m), []).append(i)
    index = {k: torch.tensor(v, device="cuda") for k, v in groups.items()}

    def call_a():
        out = dec.decode_batch(None, xs, beam_width=beam, language_model_list=lms)
        return out, dec.last_timings()["ms_beam"]

    def call_b():
        out, ms = [None] * B, 0.0
        for k, idx in groups.items():
            d = own[k]
            texts = d.decode_batch(None, xs.index_select(0, index[k]), beam_width=beam)
            ms += d.last_timings()["ms_beam"]
            for i, t in zip(idx, texts):
                out[i] = t
        return out, ms

    def call_c():
        out = dec.decode_batch(None, xs, beam_width=beam)
        return out, dec.last_timings()["ms_beam"]

    shape = {"B": B, "T": T, "V": wa.V, "beam": beam, "lms": "3-gram A / 3-gram B alternating, every 4th utterance none"}
    ra, out_a = timed(torch, call_a, args.steps, args.warmup)
    emit(dict(name="c3_language_model_list", shape=shape, **ra))
    rb, out_b = timed(torch, call_b, args.steps, args.warmup)
    emit(dict(name="c3_call_per_model", shape=shape, calls_per_step=len(groups), **rb))
    rc, _ = timed(torch, call_c, args.steps, args.warmup)
    emit(dict(name="c3_one_model", shape=dict(shape, lms="3-gram A for every utterance"), **rc))
    emit(dict(name="c3_summary", a_vs_b_wall_speedup=rb["wall_ms"] / ra["wall_ms"],
              a_vs_b_beam_kernel_speedup=rb["beam_kernel_ms"] / ra["beam_kernel_ms"],
              a_vs_c_beam_kernel_ratio=ra["beam_kernel_ms"] / rc["beam_kernel_ms"], a_equals_b=out_a == out_b))
    emit(dict(name="c3_language_model_list_host_ms", sections=host_profile_ms(call_a)))
    emit(dict(name="c3_one_model_host_ms", sections=host_profile_ms(call_c)))
    if args.out:
        with open(args.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
