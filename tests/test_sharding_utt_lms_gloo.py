"""world_size-2 `gloo` test of decode_batch_sharded with per-utterance language models: language_model_list is
sharded together with the utterances, so the sharded decode equals the single-process call and the decode of each
utterance on a decoder built with its own model.  The kernels are the tests/hostsim simulation build here; the plumbing under test is the product's."""
import json
import os
import socket
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

WORKER = r'''
import json, os, sys
sys.path.insert(0, %(root)r)
import numpy as np
import torch.distributed as dist
from pyctcdecode_b200 import _lib, sharding
import pyctcdecode_b200 as pkg
from tests import utt_lms as ul
_lib.use_library(os.path.join(%(root)r, "tests", "hostsim", "libb200ctc_hostsim.so"))
os.environ["B200CTC_DEVICE"] = "0"   # the simulation build exposes a single fake device
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
sets = ul.Sets(pkg, "char")
wl = sets.wl
dec = pkg.BeamSearchDecoderCTC(pkg.Alphabet.build_alphabet(sets.labels), sets.lm["A"])
Ts = [50, 0, 120, 7, 33, 90, 64, 1, 15]
xs = [wl.utterance(300 + i, T, "diffuse") if T else np.zeros((0, wl.V), np.float32) for i, T in enumerate(Ts)]
lms = sets.models(sets.names(len(Ts)))
texts = sharding.decode_batch_sharded(dec, xs, beam_width=20, language_model_list=lms)
out = [None] * world
dist.all_gather_object(out, texts)
if rank == 0:
    single = dec.decode_batch(None, xs, beam_width=20, language_model_list=lms)
    alone = [sets.ref(m).decode(x, beam_width=20) for x, m in zip(xs, lms)]
    print(json.dumps({"texts": out, "single": single, "alone": alone}))
dist.destroy_process_group()
'''


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def test_two_rank_gloo_sharded_decode_with_language_model_list(tmp_path):
    subprocess.check_call(["make", "-s", "-C", os.path.join(HERE, "hostsim")])
    script = tmp_path / "worker.py"
    script.write_text(WORKER % {"root": ROOT})
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", OMP_NUM_THREADS="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), str(script)]
    res = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-3000:]
    out = json.loads([line for line in res.stdout.splitlines() if line.startswith("{")][-1])
    assert out["texts"][0] == out["texts"][1] == out["single"] == out["alone"]
