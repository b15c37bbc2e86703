"""Where the cycles of the latency-first beam kernel go, per kind of frame step, on the headline workload.

    python tools/phase_clocks.py                  # build the phase-clock library if needed, run C2 on cuda:0, print the table
    python tools/phase_clocks.py --host-profile   # also a short run with B200CTC_HOST_PROFILE=1: host time per call by section
    python tools/phase_clocks.py --src OTHER_TREE --lib build/phase_clocks/other.so   # the same for another checkout

The library is a `-DB2C_PHASE_CLOCKS` build of `libb200ctc.so` with the flags of `__graft_entry__.NVCC_FLAGS`, written to
`build/phase_clocks/` (ignored by git).  In that build thread 0 of every CTA adds the cycles between consecutive marks of
`b2c_beam_fast.h` into per-key counters, summed over CTAs and printed on stderr after each call; `bench.py` loads it
through `B200CTC_PROFILING_LIB`.  The counters of the timed device-resident steps are combined by the median per key.
Cycles are SM cycles of thread 0 of each CTA, so the shares are shares of the kernel's critical path summed over CTAs,
not of issue slots.
"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT_LIB = os.path.join(ROOT, "build", "phase_clocks", "libb200ctc.so")

# mark keys (B2C_FMARK in b2c_beam_fast.h) that partition thread 0's time; 9-15 split the general step (p0-p4),
# 12-14, 23 and 25-27 count frames
MARK_KEYS = [0, 1, 2, 3, 4, 5, 6, 7, 8, 16, 17, 18, 19, 20, 21, 22, 24]
STEP_KINDS = [   # (name, cycle keys, frame-count keys or the bench.py timing field)
    ("general step, K = 1, after a multi-token frame", [9], 12),
    ("general step, K = 1, after a one-token frame", [15], 23),
    ("general step, K = 2", [10], 13),
    ("general step, K >= 3", [11], 14),
    ("single-token step, three phases", [], 25),
    ("single-token step, no-merge exit (in place)", [], 26),
    ("single-token step, all frames", [24], [25, 26]),
    ("sorted step", [7, 20, 21, 22], "sorted_frames"),
    ("in-place runs", [5, 17, 18], "inplace_frames"),
]


def build(src, lib, force=False):
    """compile the phase-clock variant of the library from the tree `src` into `lib` (skipped when it is up to date)"""
    sys.path.insert(0, ROOT)
    import __graft_entry__ as graft
    csrc = os.path.join(src, "pyctcdecode_b200", "csrc")
    sources = [os.path.join(csrc, f) for f in sorted(os.listdir(csrc))] + [os.path.join(src, "include", "b200ctc.h")]
    if not force and os.path.exists(lib) and all(os.path.getmtime(s) <= os.path.getmtime(lib) for s in sources):
        return
    os.makedirs(os.path.dirname(lib), exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    tmp = "%s.build.%d" % (lib, os.getpid())
    cmd = [nvcc] + graft.NVCC_FLAGS + ["-DB2C_PHASE_CLOCKS", "-o", tmp, os.path.join(csrc, "b2c_api.cu")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    with open(lib + ".log", "w") as fh:
        fh.write(" ".join(cmd) + "\n" + r.stdout)
    if r.returncode != 0:
        if os.path.exists(tmp):
            os.remove(tmp)
        raise RuntimeError("nvcc failed:\n" + r.stdout[-4000:])
    os.replace(tmp, lib)


def run_bench(env_extra, steps, warmup, extra):
    env = dict(os.environ, **env_extra)
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup),
           "--no-secondary", "--no-cpu-baseline"] + extra
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, cwd=ROOT, env=env)
    if r.returncode != 0:
        raise RuntimeError("bench.py failed (%d):\n%s" % (r.returncode, r.stderr[-4000:]))
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1]
    return json.loads(line), r.stderr.splitlines()


def parse_clocks(lines):
    out = []
    for ln in lines:
        if ln.startswith("[b2c phase clocks"):
            out.append({int(k): float(v) for k, v in re.findall(r" p(\d+)=([0-9]+)", ln)})
    return out


def table(res, calls, n_utts):
    med = {k: statistics.median(c.get(k, 0.0) for c in calls) for k in range(32)}
    total = sum(med[k] for k in MARK_KEYS)
    bkc = res["beam_kernel_config"]
    rows = []
    for name, keys, fk in STEP_KINDS:
        cyc = sum(med[k] for k in keys)
        if isinstance(fk, str):
            frames = bkc[{"sorted_frames": "sorted_no_merge_frames_per_step", "inplace_frames": "inplace_single_token_frames_per_step"}[fk]]
        else:
            frames = sum(med[k] for k in (fk if isinstance(fk, list) else [fk]))
        if not frames and not cyc:
            continue
        rows.append((name, frames, cyc))
    fin = med[8]
    lines = ["kernel cycles summed over CTAs (thread 0, median of %d calls): %.1f M; frames per call: %d" %
             (len(calls), total / 1e6, res["config"]["batch_per_gpu"] * res["config"]["T"])]
    lines.append("| step kind | frames per call | share of kernel cycles | cycles per frame |")
    lines.append("|---|---|---|---|")
    for name, frames, cyc in rows:
        lines.append("| %s | %d | %s | %s |" % (name, frames, "%.1f %%" % (100.0 * cyc / total) if cyc else "-",
                                                 "%.0f" % (cyc / frames) if frames and cyc else "-"))
    lines.append("| finalize + backtrack walk (p8) | %d utterances | %.1f %% | %.0f per utterance |" %
                 (n_utts, 100.0 * fin / total, fin / n_utts))
    if med[27]:
        lines.append("single-token step: %d frames handed to the general step (counted there as well)" % med[27])
    other = {k: med[k] for k in (0, 1, 2, 3, 4, 6, 16, 19) if med[k]}
    lines.append("other marks (share): " + ", ".join("p%d %.1f %%" % (k, 100.0 * v / total) for k, v in other.items()))
    return "\n".join(lines), med, total


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--src", default=ROOT, help="tree whose kernel sources are built (default: this one)")
    ap.add_argument("--lib", default=DEFAULT_LIB, help="where the phase-clock library goes / is read from")
    ap.add_argument("--no-build", action="store_true", help="use --lib as it is")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-profile", action="store_true", help="also a run of the default library with B200CTC_HOST_PROFILE=1")
    ap.add_argument("--json", default="", help="also write the medians of every key to this file")
    ap.add_argument("bench_args", nargs="*", help="more bench.py arguments (after --), e.g. -- --beam 50")
    args = ap.parse_args()
    lib = os.path.abspath(args.lib)
    if not args.no_build:
        build(os.path.abspath(args.src), lib)
    warmup = max(args.warmup, 3)          # bench.py runs at least three warm-up calls
    res, err = run_bench({"B200CTC_PROFILING_LIB": lib}, args.steps, warmup, args.bench_args)
    calls = parse_clocks(err)
    if len(calls) < warmup + args.steps:
        raise SystemExit("expected %d phase-clock lines, got %d (is %s a -DB2C_PHASE_CLOCKS build?)" % (warmup + args.steps, len(calls), lib))
    timed = calls[warmup:warmup + args.steps]           # the device-resident arm's timed calls come first
    text, med, total = table(res, timed, res["config"]["batch_per_gpu"])
    print(text)
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"lib": lib, "median_cycles": med, "total": total, "bench": res}, fh, indent=1)
    if args.host_profile:
        res_h, err_h = run_bench({"B200CTC_HOST_PROFILE": "1"}, args.steps, warmup, args.bench_args)
        host = [dict((k, float(v)) for k, v in re.findall(r"(\w+)=([0-9.]+)", ln)) for ln in err_h if ln.startswith("[b2c host ms]")]
        host = host[warmup:warmup + args.steps]
        keys = list(host[0]) if host else []
        print("host time per device-resident call, ms (median of %d): " % len(host) +
              ", ".join("%s %.3f" % (k, statistics.median(h[k] for h in host)) for k in keys))
        print("wall ms per step %.3f, device ms per step (first event to D2H done) %.3f, beam kernel %.3f, streaming stage %.3f" %
              (res_h["ms_per_step"], res_h["device_ms_per_step"], res_h["roofline"]["kernel_ms"], res_h["roofline_prepare"]["kernel_ms"]))


if __name__ == "__main__":
    main()
