"""Multi-GPU plumbing for decode_batch: one process per GPU, utterances sharded, no data-path
collective.

The reference's only parallelism is ``multiprocessing.Pool.map`` over utterances with the LM
shared by fork copy-on-write (reference decoder.py:895-945, :262-269).  The GPU equivalent:
every rank owns one GPU and a shard of the utterances; the flattened LM is built once (rank
``src`` parses the ARPA file) and shipped to the other ranks with ONE ``torch.distributed``
broadcast (NCCL over NVLink on a GPU box, gloo in the CPU tests); after that ranks never talk
during decoding.  Results are gathered only if the caller asks for it.
"""
import ctypes as C
from typing import Any, Collection, List, Optional, Sequence

import numpy as np

from . import _lib
from .alphabet import Alphabet, verify_alphabet_coverage
from .constants import DEFAULT_ALPHA, DEFAULT_BETA, DEFAULT_SCORE_LM_BOUNDARY, DEFAULT_UNK_LOGP_OFFSET
from .decoder import BeamSearchDecoderCTC
from .language_model import LanguageModel, NgramModel, load_unigram_set_from_arpa


# what the last broadcast_ngram_model call moved: {"bytes", "ms", "gb_per_s", "backend"} (bench.py reports it)
last_broadcast: dict = {}


def shard_utterances(lengths: Sequence[int], world_size: int) -> List[List[int]]:
    """Longest-processing-time-first partition of utterance indices over ``world_size`` ranks.
    Deterministic (ties broken by index) so that every rank computes the same partition."""
    order = sorted(range(len(lengths)), key=lambda i: (-int(lengths[i]), i))
    loads = [0] * world_size
    shards: List[List[int]] = [[] for _ in range(world_size)]
    for i in order:
        r = min(range(world_size), key=lambda k: (loads[k], k))
        shards[r].append(i)
        loads[r] += int(lengths[i]) + 1
    for s in shards:
        s.sort()
    return shards


def broadcast_ngram_model(path: Optional[str], unigrams: Optional[Collection[str]], device: Optional[int], src: int = 0,
                          group: Any = None) -> Optional[NgramModel]:
    """Rank ``src`` builds the flattened model from ``path``; all ranks return an NgramModel over
    bit-identical tables.  With a CUDA device the broadcast buffer itself becomes the resident
    device copy (no second upload)."""
    import torch
    import torch.distributed as dist

    rank = dist.get_rank(group)
    use_cuda = device is not None and torch.cuda.is_available() and dist.get_backend(group) == "nccl"
    meta = [None]
    model = None
    if rank == src:
        if path is None:
            meta = [(None, 0)]
        else:
            model = NgramModel(path, unigrams)
            _, size = model.blob()
            meta = [(path, size)]
    dist.broadcast_object_list(meta, src=src, group=group)
    path_b, size = meta[0]
    if path_b is None:
        return None
    dev = torch.device("cuda", device) if use_cuda else torch.device("cpu")
    buf = torch.empty(size, dtype=torch.uint8, device=dev)
    if rank == src:
        addr, _ = model.blob()
        host = np.ctypeslib.as_array((C.c_uint8 * size).from_address(addr))
        buf.copy_(torch.from_numpy(host))
    import time

    if use_cuda:
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        dist.broadcast(buf, src=src, group=group)
        ev1.record()
        ev1.synchronize()
        ms = float(ev0.elapsed_time(ev1))
    else:
        t0 = time.perf_counter()
        dist.broadcast(buf, src=src, group=group)
        ms = 1e3 * (time.perf_counter() - t0)
    last_broadcast.clear()
    last_broadcast.update(bytes=int(size), ms=ms, gb_per_s=(size / 1e9) / max(ms * 1e-3, 1e-9), backend=str(dist.get_backend(group)),
                          world_size=int(dist.get_world_size(group)))
    if rank != src:
        host_copy = buf.cpu().numpy()
        model = NgramModel.from_blob(path_b, host_copy.ctypes.data, size)
    if use_cuda:
        _lib.check(_lib.lib().b2c_lm_adopt_device_blob(model._h(), device, C.c_void_p(buf.data_ptr()), size))
        model._device_blob = buf  # keep the broadcast buffer alive: it IS the device-resident LM
    return model


def build_ctcdecoder_broadcast(labels: List[str], kenlm_model_path: Optional[str] = None,
                               unigrams: Optional[Collection[str]] = None, alpha: float = DEFAULT_ALPHA,
                               beta: float = DEFAULT_BETA, unk_score_offset: float = DEFAULT_UNK_LOGP_OFFSET,
                               lm_score_boundary: bool = DEFAULT_SCORE_LM_BOUNDARY, device: Optional[int] = None,
                               src: int = 0, group: Any = None) -> BeamSearchDecoderCTC:
    """build_ctcdecoder() for one-process-per-GPU jobs: only rank ``src`` reads the ARPA file."""
    import torch.distributed as dist

    rank = dist.get_rank(group)
    if unigrams is None and kenlm_model_path is not None and kenlm_model_path.endswith(".arpa"):
        holder = [sorted(load_unigram_set_from_arpa(kenlm_model_path)) if rank == src else None]
        dist.broadcast_object_list(holder, src=src, group=group)
        unigrams = holder[0]
    alphabet = Alphabet.build_alphabet(labels)
    if unigrams is not None:
        verify_alphabet_coverage(alphabet, unigrams)
    ulist = None if unigrams is None else sorted(set(unigrams))
    ngram = broadcast_ngram_model(kenlm_model_path, ulist, device, src=src, group=group)
    lm = None
    if ngram is not None:
        lm = LanguageModel.__new__(LanguageModel)
        lm._unigram_list = ulist
        lm._blob_unigrams = False
        lm._kenlm_model = ngram
        lm.alpha, lm.beta, lm.unk_score_offset, lm.score_boundary = alpha, beta, unk_score_offset, lm_score_boundary
    return BeamSearchDecoderCTC(alphabet, lm, device=device)


def decode_batch_sharded(decoder: BeamSearchDecoderCTC, logits_list: Sequence[Any], group: Any = None, **kwargs: Any) -> List[str]:
    """Every rank passes the SAME list; each decodes its shard on its own GPU; all ranks return the
    full list of transcripts (one all_gather_object of strings -- not on the data path)."""
    import torch.distributed as dist

    world, rank = dist.get_world_size(group), dist.get_rank(group)
    shards = shard_utterances([x.shape[0] for x in logits_list], world)
    mine = decoder.decode_batch(None, [logits_list[i] for i in shards[rank]], **kwargs)
    gathered: List[Any] = [None] * world
    dist.all_gather_object(gathered, mine, group=group)
    out: List[Optional[str]] = [None] * len(logits_list)
    for idx, texts in zip(shards, gathered):
        for i, t in zip(idx, texts):
            out[i] = t
    return out  # type: ignore[return-value]
