"""What per-stream search parameters save in batched streaming, on one GPU.

    python tools/bench_stream_params.py [--steps K] [--warmup W] [--out FILE]

Continuous-batching traffic at the C3 shape (V=32, a synthetic 3-gram over 20k words): 64 slots, each advancing its
stream by a 50-frame chunk of host logits per step; stream lengths are staggered between 400 and 1000 frames, and a new
stream from get_starting_state() takes each freed slot (tests/stream_ends.plan, with its per-stream end flags).  Stream s
runs in parameter tier s % 3 (tests/stream_params.tiers): beam 100 / prune -10 / token -5; beam 128 / prune -40 /
token -8 / prune_history; beam 16 / prune -0.5 / token -1.
  (A) one partial_decode_beams_batch per step with beam_width_list / beam_prune_logp_list / token_min_logp_list /
      prune_history_list;
  (B) one partial_decode_beams_batch per distinct parameter tuple of the step: what a caller without the lists must do.
Both arms pass is_end_list / force_next_word_list.  The arms run step by step in alternating order, each from its own
beams; every step asserts that they return identical beams.  Per arm: wall time per step (host clock around the
synchronous calls; median and max over the timed steps) and device time per step (ms_prepare + ms_beam of
last_timings(), summed over the step's calls).  Prints one JSON line per measurement, with the card's name and power
limit.
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

from tools.bench_utt_hotwords import card  # noqa: E402

SLOTS, CHUNK, WIDTHS = 64, 50, (100, 128, 16)
NAMES = ("beam_width", "beam_prune_logp", "token_min_logp", "prune_history")


def step_calls(call, tier_of, per_stream):
    """The calls one step takes: [(indices into `call`, scalar parameters or None for the lists)]."""
    if per_stream:
        return [(list(range(len(call))), None)]
    groups = {}
    for i, row in enumerate(call):
        groups.setdefault(tuple(sorted(tier_of(row[0]).items())), []).append(i)
    return [(idx, dict(key)) for key, idx in groups.items()]


def run_step(dec, xs, beams, cache, call, tier_of, per_stream):
    """One step of one arm; updates `beams`.  -> (wall ms, device ms, calls, beams of the step in slot order)"""
    out = [None] * len(call)
    device = 0.0
    parts = step_calls(call, tier_of, per_stream)
    t = time.perf_counter()
    for idx, scalars in parts:
        rows = [call[i] for i in idx]
        if scalars is None:
            params = {name + "_list": [tier_of(r[0])[name] for r in rows] for name in NAMES}
        else:
            params = scalars
        got = dec.partial_decode_beams_batch([xs[s][t0:t1] for s, t0, t1, _, _ in rows], [cache] * len(rows),
                                             [beams[s] for s, _, _, _, _ in rows], [t0 for _, t0, _, _, _ in rows],
                                             force_next_word_list=[r[3] for r in rows], is_end_list=[r[4] for r in rows],
                                             **params)
        tm = dec.last_timings()
        device += tm["ms_prepare"] + tm["ms_beam"]
        for i, b in zip(idx, got):
            out[i] = b
    wall = 1e3 * (time.perf_counter() - t)
    for (s, _, _, _, _), b in zip(call, out):
        beams[s] = b
    return wall, device, len(parts), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40, help="timed steps")
    ap.add_argument("--warmup", type=int, default=5, help="untimed steps first")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build()
    import pyctcdecode_b200 as pkg
    from tests import stream_ends as se
    from tests import stream_params as sp

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    info = card()
    lines = []

    def emit(obj):
        obj.update(info)
        lines.append(json.dumps(obj))
        print(lines[-1], flush=True)

    dec, base = se.c3_streams(pkg)
    tier_of = sp.tiers(WIDTHS)
    n_steps = args.warmup + args.steps
    Ts = se.staggered(SLOTS * (1 + n_steps * CHUNK // 400))
    calls = se.plan(Ts, SLOTS, chunks=(CHUNK,), max_calls=n_steps)
    assert len(calls) == n_steps and all(len(c) == SLOTS for c in calls)
    xs = [base[j % len(base)][:T] for j, T in enumerate(Ts)]
    start, cache = list(dec.get_starting_state()[0]), dec.get_starting_state()[1]
    beams = {True: {}, False: {}}
    rec = {True: ([], [], []), False: ([], [], [])}
    for c, call in enumerate(calls):
        for arm in beams.values():
            for s, t0, _, _, _ in call:
                if t0 == 0:
                    arm[s] = start
        res = {}
        for per_stream in ((True, False) if c % 2 == 0 else (False, True)):
            res[per_stream] = run_step(dec, xs, beams[per_stream], cache, call, tier_of, per_stream)
        assert res[True][3] == res[False][3], "step %d: the arms return different beams" % c
        if c >= args.warmup:
            for per_stream, (wall, device, n_calls, _) in res.items():
                rec[per_stream][0].append(wall)
                rec[per_stream][1].append(device)
                rec[per_stream][2].append(n_calls)
    shape = {"slots": SLOTS, "chunk_frames": CHUNK, "V": 32, "lm": "3-gram over 20k words",
             "tiers": [tier_of(k) for k in range(3)], "stream_frames": "400..1000 staggered", "timed_steps": args.steps}
    out = {}
    for per_stream, name in ((True, "stream_params_per_stream_lists"), (False, "stream_params_call_per_tuple")):
        walls, devs, n_calls = rec[per_stream]
        out[per_stream] = dict(wall_ms_per_step=statistics.median(walls), wall_ms_per_step_max=max(walls),
                               device_ms_per_step=statistics.median(devs), calls_per_step=statistics.mean(n_calls))
        emit(dict(name=name, shape=shape, **out[per_stream]))
    a, b = out[True], out[False]
    emit(dict(name="stream_params_summary", b_over_a_wall=b["wall_ms_per_step"] / a["wall_ms_per_step"],
              b_over_a_device=b["device_ms_per_step"] / a["device_ms_per_step"], identical_beams=True))
    if args.out:
        with open(args.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
