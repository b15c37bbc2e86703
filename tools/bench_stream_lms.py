"""What per-stream language models cost and save in batched streaming, on one GPU.

    python tools/bench_stream_lms.py [--passes K] [--warmup W] [--out FILE]

C3 shape (V=32, beam 100, synthetic 3-grams over 20k words), 64 streams of T=1000 host logits advancing by 50 frames
per call, beams carried as LMBeam lists (bench.py's stream64_lm entry).  Streams cycle through four models (three
3-grams over different word lists, and the first one with other alpha / beta); every fifth stream has none:
  (a) one partial_decode_beams_batch per chunk with language_model_list;
  (b) one partial_decode_beams_batch per chunk and model group, on one decoder per model: what a caller without
      language_model_list must do; wall time and beam-kernel ms per chunk are the sums over the group calls;
  (c) every stream with the first model, one call per chunk (bench.py's stream64_lm configuration).
For each: wall time per chunk (host clock around the synchronous calls; median over the chunks of the timed passes) and
beam-kernel ms per chunk (CUDA events inside the library), and the host time the library spends building the
language-model sets of one call of (a) and (c) (`lm_sets=` of B200CTC_HOST_PROFILE=1).  Prints one JSON line per
measurement, with the card's name and power limit.
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.bench_utt_hotwords import card, host_profile_ms  # noqa: E402

N, T, CHUNK, BEAM = 64, 1000, 50, 100


def run_pass(groups, xs):
    """One pass over the streams, chunk by chunk.  groups: [(decoder, stream indices, language_model_list or None)]
    whose calls together advance every stream by one chunk.  -> (wall ms per chunk, beam-kernel ms per chunk, final
    top-1 texts)"""
    beams = [None] * N
    caches = [None] * N
    for dec, idx, lms in groups:
        for k, i in enumerate(idx):
            lm = lms[k] if lms is not None else None
            st = dec.get_starting_state(language_model=lm) if lm is not None else dec.get_starting_state()
            beams[i], caches[i] = list(st[0]), st[1]
    walls, kernels = [], []
    for t0 in range(0, T, CHUNK):
        last = t0 + CHUNK >= T
        ms = 0.0
        t = time.perf_counter()
        for dec, idx, lms in groups:
            out = dec.partial_decode_beams_batch([xs[i][t0:t0 + CHUNK] for i in idx], [caches[i] for i in idx],
                                                 [beams[i] for i in idx], [t0] * len(idx), beam_width=BEAM, is_end=last,
                                                 language_model_list=lms)
            ms += dec.last_timings()["ms_beam"]
            for i, b in zip(idx, out):
                beams[i] = b
        walls.append(1e3 * (time.perf_counter() - t))
        kernels.append(ms)
    return walls, kernels, [b[0].text if b else "" for b in beams]


def first_chunk(dec, lms, xs):
    """The first chunk of every stream in one call: with language_model_list=lms, or on dec's own model (lms None)."""
    def fn():
        if lms is None:
            caches = [dec.get_starting_state()[1]] * N
        else:
            caches = [dec.get_starting_state(language_model=m)[1] if m is not None else {} for m in lms]
        dec.partial_decode_beams_batch([x[:CHUNK] for x in xs], caches, [list(dec.get_starting_state()[0]) for _ in xs],
                                       [0] * N, beam_width=BEAM, language_model_list=lms)
    return fn


def measure(groups, xs, passes, warmup):
    for _ in range(warmup):
        run_pass(groups, xs)
    walls, kernels = [], []
    for _ in range(passes):
        w, k, texts = run_pass(groups, xs)
        walls += w
        kernels += k
    return {"wall_ms_per_chunk": statistics.median(walls), "beam_kernel_ms_per_chunk": statistics.median(kernels),
            "wall_ms_per_chunk_max": max(walls), "chunks": len(walls)}, texts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=3, help="timed passes over the 20 chunks")
    ap.add_argument("--warmup", type=int, default=1, help="untimed passes first")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
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

    wls = [synth.CharWorkload("B", n_words=20000, lm_order=3, seed=s) for s in (1, 2, 3)]
    models = [pkg.LanguageModel(pkg.NgramModel(w.arpa), w.words, alpha=0.5, beta=1.0) for w in wls]
    models.append(pkg.LanguageModel(pkg.NgramModel(wls[0].arpa), wls[0].words, alpha=0.9, beta=2.0))
    alphabet = pkg.Alphabet.build_alphabet(wls[0].labels)
    lms = [None if i % 5 == 4 else models[i % 4] for i in range(N)]
    xs = wls[0].batch(1, N, T, "peaky")
    everyone = list(range(N))

    dec = pkg.BeamSearchDecoderCTC(alphabet, None, device=0)
    by_model = {}
    for i, m in enumerate(lms):
        by_model.setdefault(id(m), (m, []))[1].append(i)
    own = [(pkg.BeamSearchDecoderCTC(alphabet, m, device=0), idx, None) for m, idx in by_model.values()]
    one = pkg.BeamSearchDecoderCTC(alphabet, models[0], device=0)

    shape = {"streams": N, "T": T, "chunk_frames": CHUNK, "V": wls[0].V, "beam": BEAM,
             "lms": "four 3-gram models over 20k words cycling, every 5th stream none"}
    ra, out_a = measure([(dec, everyone, lms)], xs, args.passes, args.warmup)
    emit(dict(name="stream64_language_model_list", shape=shape, calls_per_chunk=1, **ra))
    rb, out_b = measure(own, xs, args.passes, args.warmup)
    emit(dict(name="stream64_call_per_model", shape=shape, calls_per_chunk=len(own), **rb))
    rc, _ = measure([(one, everyone, None)], xs, args.passes, args.warmup)
    emit(dict(name="stream64_one_model", shape=dict(shape, lms="the first model for every stream"), calls_per_chunk=1, **rc))
    emit(dict(name="stream64_summary", a_vs_b_wall_speedup=rb["wall_ms_per_chunk"] / ra["wall_ms_per_chunk"],
              a_vs_b_beam_kernel_speedup=rb["beam_kernel_ms_per_chunk"] / ra["beam_kernel_ms_per_chunk"],
              a_vs_c_wall_ratio=ra["wall_ms_per_chunk"] / rc["wall_ms_per_chunk"],
              a_vs_c_beam_kernel_ratio=ra["beam_kernel_ms_per_chunk"] / rc["beam_kernel_ms_per_chunk"], a_equals_b=out_a == out_b))
    emit(dict(name="stream64_language_model_list_host_ms", sections=host_profile_ms(first_chunk(dec, lms, xs))))
    emit(dict(name="stream64_one_model_host_ms", sections=host_profile_ms(first_chunk(one, None, xs))))
    if args.out:
        with open(args.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
