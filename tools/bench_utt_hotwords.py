"""What per-utterance hotwords cost and save, on one GPU.

    python tools/bench_utt_hotwords.py [--steps K] [--warmup W] [--out FILE]

C4 shape (BPE V=1024, T=500, batch 512, beam 100, synthetic 4-gram), every utterance with its own 16 hotwords drawn
from a fixed seed:
  (a) one decode_batch call with hotwords_list;
  (b) the same batch with one shared 16-word list (hotwords=, the C4 configuration of bench.py);
  (c) one decode_batch call per utterance, each with its own list: what a caller without hotwords_list must do.
For each: wall time per call (host clock around the synchronous call) and beam-kernel ms (CUDA events inside the
library, summed over the calls of (c)).  Also the host time the library spends building the hotword tables of (a)
(B200CTC_HOST_PROFILE=1) and the C2 shape (V=32, T=1000, batch 256, no LM) with lists on every other utterance
against the same batch without hotwords.  Prints one JSON line per measurement, with the card's name and power limit.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                           stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": limit}
    except Exception as exc:          # the figures are still tied to the device torch reports
        import torch
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": "unknown (%r)" % (exc,)}


def per_utt_lists(words, B, n=16, seed=11):
    import numpy as np
    rng = np.random.default_rng(seed)
    return [[words[int(k)] for k in rng.choice(2000, size=n, replace=False)] for _ in range(B)]


def timed(torch, fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    walls, beams = [], []
    for _ in range(steps):
        t0 = time.perf_counter()
        out, ms_beam = fn()
        walls.append(1e3 * (time.perf_counter() - t0))
        beams.append(ms_beam)
    walls.sort()
    beams.sort()
    return {"wall_ms": walls[len(walls) // 2], "beam_kernel_ms": beams[len(beams) // 2], "steps": steps}, out


def host_profile_ms(fn):
    """Run fn once with B200CTC_HOST_PROFILE=1 and return the library's host sections (ms) from its stderr line."""
    os.environ["B200CTC_HOST_PROFILE"] = "1"
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+") as tmp:
        os.dup2(tmp.fileno(), 2)
        try:
            fn()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            del os.environ["B200CTC_HOST_PROFILE"]
        tmp.seek(0)
        text = tmp.read()
    lines = [ln for ln in text.splitlines() if ln.startswith("[b2c host ms]")]
    return {k: float(v) for k, v in re.findall(r"(\w+)=([0-9.]+)", lines[-1])} if lines else {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--single-steps", type=int, default=1, help="timed repetitions of (c), one call per utterance")
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

    # ---- C4 shape ----------------------------------------------------------------------------------------------
    B, T, beam = 512, 500, 100
    wl = synth.BpeWorkload(n_words=50000, lm_order=4)
    dec = pkg.build_ctcdecoder(wl.labels, kenlm_model_path=wl.arpa, unigrams=wl.words, alpha=0.5, beta=1.0, device=0)
    xs = torch.from_numpy(__import__("numpy").stack(wl.batch(1, B, T, "peaky"))).cuda()
    lists = per_utt_lists(wl.words, B)
    shared = wl.hotwords(16)

    def call_a():
        out = dec.decode_batch(None, xs, beam_width=beam, hotwords_list=lists)
        return out, dec.last_timings()["ms_beam"]

    def call_b():
        out = dec.decode_batch(None, xs, beam_width=beam, hotwords=shared)
        return out, dec.last_timings()["ms_beam"]

    def call_c():
        out, ms = [], 0.0
        for i in range(B):
            out += dec.decode_batch(None, xs[i:i + 1], beam_width=beam, hotwords=lists[i])
            ms += dec.last_timings()["ms_beam"]
        return out, ms

    shape = {"B": B, "T": T, "V": wl.V, "beam": beam, "lm": "synthetic 4-gram", "hotwords_per_utt": 16}
    ra, out_a = timed(torch, call_a, args.steps, args.warmup)
    emit(dict(name="c4_hotwords_list", shape=shape, **ra))
    rb, _ = timed(torch, call_b, args.steps, args.warmup)
    emit(dict(name="c4_shared_list", shape=shape, **rb))
    rc, out_c = timed(torch, call_c, args.single_steps, 1)
    emit(dict(name="c4_call_per_utterance", shape=shape, calls_per_step=B, **rc))
    emit(dict(name="c4_summary", a_vs_c_wall_speedup=rc["wall_ms"] / ra["wall_ms"],
              a_vs_c_beam_kernel_speedup=rc["beam_kernel_ms"] / ra["beam_kernel_ms"],
              a_vs_b_beam_kernel_ratio=ra["beam_kernel_ms"] / rb["beam_kernel_ms"], a_equals_c=out_a == out_c))
    emit(dict(name="c4_hotwords_list_host_ms", sections=host_profile_ms(call_a)))
    del dec, xs
    torch.cuda.empty_cache()

    # ---- C2 shape, lists on every other utterance --------------------------------------------------------------
    B, T = 256, 1000
    wl = synth.CharWorkload("B", n_words=20000, lm_order=0)
    dec = pkg.build_ctcdecoder(wl.labels, device=0)
    xs = torch.from_numpy(__import__("numpy").stack(wl.batch(1, B, T, "peaky"))).cuda()
    half = [ws if i % 2 == 0 else None for i, ws in enumerate(per_utt_lists(wl.words, B))]

    def c2_half():
        out = dec.decode_batch(None, xs, beam_width=beam, hotwords_list=half)
        return out, dec.last_timings()["ms_beam"]

    def c2_none():
        out = dec.decode_batch(None, xs, beam_width=beam)
        return out, dec.last_timings()["ms_beam"]

    shape = {"B": B, "T": T, "V": wl.V, "beam": beam, "lm": None, "hotwords_per_utt": "16 on every other utterance"}
    emit(dict(name="c2_half_hotwords_list", shape=shape, **timed(torch, c2_half, args.steps, args.warmup)[0]))
    emit(dict(name="c2_no_hotwords", shape=shape, **timed(torch, c2_none, args.steps, args.warmup)[0]))
    if args.out:
        with open(args.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
