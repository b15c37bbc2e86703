import time, sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import synth
from oracle import oracle as orc
print("cpu_count", os.cpu_count(), "affinity", len(os.sched_getaffinity(0)))
try: print("cpu.max", open("/sys/fs/cgroup/cpu.max").read().strip())
except Exception as e: print("cpu.max n/a", e)
wl = synth.CharWorkload("B", n_words=20000, lm_order=0)
xs = wl.batch(1, 256, 1000, "peaky")
ora = orc.OracleDecoder(wl.labels)
for nt in [1, 8, 16, 32, 64, 128]:
    n = min(256, 2*nt)
    t0=time.perf_counter(); ora.decode_batch(xs[:n], n_threads=nt, beam_width=100); dt=time.perf_counter()-t0
    print(nt, n, "%.2fs"%dt, "%.0f frames/s total, %.0f /thread"%(n*1000/dt, n*1000/dt/nt), flush=True)
