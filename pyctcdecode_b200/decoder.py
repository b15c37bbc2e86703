"""BeamSearchDecoderCTC / build_ctcdecoder with the reference's call surface, dispatching the
whole beam search to the sm_90a kernels through the C ABI (include/b200ctc.h).

What stays on the host: argument checking (reference decoder.py:330-344), packaging the list
of [T_i, V] matrices into one ``b2c_decode_batch`` call, turning results into ``OutputBeam``.
What moved to the GPU: input normalisation (:756-765), the per-frame loop of
``_partial_decode_logits`` (:443-554), LM / hotword fusion (:346-424), ``_finalize_beams``
(:558-602).  ``pool`` arguments are accepted and ignored: utterance parallelism is one CTA per
utterance on the device (and one rank per GPU above that), not ``multiprocessing``.
"""
import ctypes as C
import dataclasses
import logging
import os
import threading
from typing import Any, Collection, Dict, Iterable, List, NamedTuple, Optional, Sequence, Tuple, Union

import numpy as np

from . import _lib
from .alphabet import Alphabet, verify_alphabet_coverage
from .constants import (
    DEFAULT_ALPHA,
    DEFAULT_BEAM_WIDTH,
    DEFAULT_BETA,
    DEFAULT_HOTWORD_WEIGHT,
    DEFAULT_MIN_TOKEN_LOGP,
    DEFAULT_PRUNE_BEAMS,
    DEFAULT_PRUNE_LOGP,
    DEFAULT_SCORE_LM_BOUNDARY,
    DEFAULT_UNK_LOGP_OFFSET,
)
from .language_model import (
    AbstractLanguageModel,
    AbstractLMState,
    B200LMState,
    HotwordScorer,
    LanguageModel,
    MultiLanguageModel,
    MultiLanguageModelState,
    NgramModel,
    load_unigram_set_from_arpa,
)

logger = logging.getLogger(__name__)

Frames = Tuple[int, int]
WordFrames = Tuple[str, Frames]


@dataclasses.dataclass(frozen=True)
class Beam:
    """reference decoder.py:69-94 (what partial_decode_beams takes and, as LMBeam, returns)"""

    text: str
    next_word: str
    partial_word: str
    last_char: Optional[str]
    text_frames: List[Frames]
    partial_frames: Frames
    logit_score: float

    @classmethod
    def from_lm_beam(cls, lm_beam: "LMBeam") -> "Beam":
        return Beam(lm_beam.text, lm_beam.next_word, lm_beam.partial_word, lm_beam.last_char, lm_beam.text_frames,
                    lm_beam.partial_frames, lm_beam.logit_score)


@dataclasses.dataclass(frozen=True)
class LMBeam(Beam):
    """reference decoder.py:97-100"""

    lm_score: float


NULL_FRAMES: Frames = (-1, -1)
EMPTY_START_BEAM = Beam("", "", "", None, [], NULL_FRAMES, 0.0)
LMScoreCache = Dict[Tuple[str, bool], Tuple[float, float, AbstractLMState]]


def _merge_tokens(token_1: str, token_2: str) -> str:
    """reference decoder.py:200-208"""
    if len(token_2) == 0:
        return token_1
    if len(token_1) == 0:
        return token_2
    return token_1 + " " + token_2


class OutputBeam(NamedTuple):
    """reference decoder.py:102-118; a NamedTuple so that both ``beam.text`` and the
    positional access HF's Wav2Vec2ProcessorWithLM uses (``beam[0]`` ... ``beam[4]``) work."""

    text: str
    last_lm_state: Optional[AbstractLMState]
    text_frames: List[WordFrames]
    logit_score: float
    lm_score: float

    def get_mp_safe_beam(self) -> "OutputBeam":
        state = None if self.last_lm_state is None else self.last_lm_state.get_mp_safe_state()
        return self._replace(last_lm_state=state)


def _default_device() -> int:
    env = os.environ.get("B200CTC_DEVICE")
    if env is not None:
        return int(env)
    return int(os.environ.get("LOCAL_RANK", "0"))


def _cuda_index(t: Any) -> Optional[int]:
    """CUDA device index of a torch tensor, None for host tensors / arrays."""
    if getattr(t, "is_cuda", False):
        return int(t.device.index if t.device.index is not None else 0)
    return None


def _as_matrix(logits: Any) -> Tuple[Any, int, int, int, bool]:
    """-> (owner, address, T, dtype_code, is_device).  float32/float64 are passed through, integer inputs are
    computed in float64 like numpy would, float16 / bfloat16 travel as they are (dtype codes 2 / 3) and are widened
    to float32 on the device."""
    if hasattr(logits, "is_cuda") and hasattr(logits, "data_ptr"):  # torch tensor
        t = logits
        if t.dim() != 2:
            raise ValueError("Input logits have %s dimensions, but need 2: (time, vocabulary)" % t.dim())
        import torch

        codes = {torch.float32: 0, torch.float64: 1, torch.float16: 2, torch.bfloat16: 3}
        if t.dtype not in codes:
            t = t.to(torch.float64 if not t.dtype.is_floating_point else torch.float32)
        t = t.contiguous()
        return t, t.data_ptr(), t.shape[0], codes[t.dtype], bool(t.is_cuda)
    arr = np.asarray(logits)
    if arr.ndim != 2:
        raise ValueError("Input logits have %s dimensions, but need 2: (time, vocabulary)" % arr.ndim)
    if arr.dtype == np.float32:
        arr = np.ascontiguousarray(arr)
        code = 0
    elif arr.dtype == np.float16:
        arr = np.ascontiguousarray(arr)
        code = 2
    else:
        arr = np.ascontiguousarray(arr, dtype=np.float64)
        code = 1
    return arr, arr.ctypes.data, arr.shape[0], code, False


class BeamSearchDecoderCTC:
    # the language model lives in a class variable keyed by a random token, like the reference
    # (decoder.py:262-269), so that code poking at model_container keeps working
    model_container: Dict[bytes, Optional[AbstractLanguageModel]] = {}

    _ALPHABET_SERIALIZED_FILENAME = "alphabet.json"
    _LANGUAGE_MODEL_SERIALIZED_DIRECTORY = "language_model"

    def __init__(self, alphabet: Alphabet, language_model: Optional[AbstractLanguageModel] = None,
                 device: Optional[int] = None) -> None:
        self._alphabet = alphabet
        self._idx2vocab = {n: c for n, c in enumerate(self._alphabet.labels)}
        self._is_bpe = alphabet.is_bpe
        self._model_key = os.urandom(16)
        BeamSearchDecoderCTC.model_container[self._model_key] = language_model
        self._device = device
        self._handles: Dict[int, int] = {}   # device -> b2c_decoder_t*
        self._lock = threading.Lock()
        # decode calls on one decoder object are serialised: parameters (alpha, beta, ...) are set on the handle right
        # before the call, and the handle's scratch buffers are per handle.  Any number of threads may call
        # decode()/decode_batch()/... concurrently, like with the reference; they run one after another on the GPU.
        self._run_lock = threading.RLock()
        self._label_ids: Dict[str, int] = {}                              # last_char -> canonical token id
        self._word_hash: Dict[str, Tuple[bytes, bytes, int, int]] = {}    # streaming host path, see _stream_states
        self._text_cache: List[Dict[str, Tuple[bytes, bytes, int]]] = [{}, {}]
        self._labels_with_space = any(len(lbl) > 1 and len(lbl.split()) != 1 for lbl in alphabet.labels)

    # ---- life cycle ---------------------------------------------------------------------
    def reset_params(self, alpha: Optional[float] = None, beta: Optional[float] = None,
                     unk_score_offset: Optional[float] = None, lm_score_boundary: Optional[bool] = None) -> None:
        language_model = self._language_model
        if language_model is None:
            return
        params: Dict[str, Any] = {}
        if alpha is not None:
            params["alpha"] = alpha
        if beta is not None:
            params["beta"] = beta
        if unk_score_offset is not None:
            params["unk_score_offset"] = unk_score_offset
        if lm_score_boundary is not None:
            params["score_boundary"] = lm_score_boundary
        language_model.reset_params(**params)

    @classmethod
    def clear_class_models(cls) -> None:
        cls.model_container = {}

    def cleanup(self) -> None:
        if self._model_key in BeamSearchDecoderCTC.model_container:
            del BeamSearchDecoderCTC.model_container[self._model_key]

    @property
    def _language_model(self) -> Optional[AbstractLanguageModel]:
        return BeamSearchDecoderCTC.model_container[self._model_key]

    def __del__(self) -> None:
        if _lib._lib is None:
            return
        for h in getattr(self, "_handles", {}).values():
            try:
                _lib._lib.b2c_decoder_destroy(h)
            except Exception:  # pragma: no cover
                pass
        self._handles = {}

    # ---- device objects -------------------------------------------------------------------
    def _handle(self, device: Optional[int] = None) -> int:
        dev = device if device is not None else (self._device if self._device is not None else _default_device())
        with self._lock:
            h = self._handles.get(dev)
            if h is None:
                lm = self._language_model
                models = self._lm_list()
                labels = self._alphabet.labels
                out = C.c_void_p()
                lm_handle = models[0].ngram_model._h() if models else None
                _lib.check(_lib.lib().b2c_decoder_create(_lib.cstr_array(labels), len(labels), int(self._is_bpe),
                                                         lm_handle, dev, C.byref(out)))
                for extra in models[1:]:          # MultiLanguageModel: models 1..
                    _lib.check(_lib.lib().b2c_decoder_add_lm(out, extra.ngram_model._h()))
                h = self._handles[dev] = out.value
        return h

    def _lm_list(self) -> List[LanguageModel]:
        """[] without a language model, [lm] for a LanguageModel, the member models of a MultiLanguageModel."""
        lm = self._language_model
        if lm is None:
            return []
        models = list(lm.language_models) if isinstance(lm, MultiLanguageModel) else [lm]
        if len(models) > 4:
            raise ValueError("pyctcdecode_b200 supports at most 4 models in a MultiLanguageModel")
        for m in models:
            if not isinstance(m, LanguageModel):
                raise TypeError("language_model must be a pyctcdecode_b200 LanguageModel (or a MultiLanguageModel of them)")
        return models

    def _check_logits_dimension(self, logits: Any) -> None:
        """reference decoder.py:330-344"""
        shape = tuple(logits.shape)
        if len(shape) != 2:
            raise ValueError("Input logits have %s dimensions, but need 2: (time, vocabulary)" % len(shape))
        if shape[-1] != len(self._idx2vocab):
            raise ValueError("Input logits shape is %s, but vocabulary is size %s. Need logits of shape: "
                             "(time, vocabulary)" % (shape, len(self._idx2vocab)))

    def _as_packed_batch(self, logits_list: Any) -> Optional[Tuple[Any, int, int, int, int, bool]]:
        """A single 3-D [B, T, V] float32/float64 numpy array or torch tensor -> (owner, address,
        B, T, dtype_code, is_device); anything else -> None (generic per-utterance path)."""
        V = len(self._idx2vocab)
        if hasattr(logits_list, "data_ptr") and hasattr(logits_list, "is_cuda"):
            import torch

            t = logits_list
            if t.dim() != 3:
                return None
            codes = {torch.float32: 0, torch.float64: 1, torch.float16: 2, torch.bfloat16: 3}
            if t.dtype not in codes:
                return None
            if t.shape[2] != V:
                raise ValueError("Input logits shape is %s, but vocabulary is size %s. Need logits of shape: "
                                 "(time, vocabulary)" % (tuple(t.shape[1:]), V))
            t = t.contiguous()
            return t, t.data_ptr(), t.shape[0], t.shape[1], codes[t.dtype], bool(t.is_cuda)
        if isinstance(logits_list, np.ndarray) and logits_list.ndim == 3 and logits_list.dtype in (np.float32, np.float64, np.float16):
            if logits_list.shape[2] != V:
                raise ValueError("Input logits shape is %s, but vocabulary is size %s. Need logits of shape: "
                                 "(time, vocabulary)" % (logits_list.shape[1:], V))
            a = np.ascontiguousarray(logits_list)
            return a, a.ctypes.data, a.shape[0], a.shape[1], {np.dtype(np.float32): 0, np.dtype(np.float64): 1, np.dtype(np.float16): 2}[a.dtype], False
        return None

    # ---- the one place that talks to the kernels ------------------------------------------
    def _run(self, logits_list: Sequence[Any], beam_width: int, beam_prune_logp: float, token_min_logp: float,
             prune_history: bool, hotwords: Optional[Iterable[str]], hotword_weight: float, max_out_beams: int,
             lm_start_states: Optional[Sequence[Optional[AbstractLMState]]] = None, with_state: bool = True,
             device: Optional[int] = None, texts_only: bool = False, lengths: Optional[Sequence[int]] = None,
             stream: Optional[Sequence[Tuple[Sequence[Beam], int]]] = None, finalize_mode: int = _lib.FIN_EOS) -> Any:
        packed = self._as_packed_batch(logits_list)
        if lengths is not None and packed is None:
            raise ValueError("lengths= needs one padded [B, T, V] array or tensor")
        if packed is not None:
            # one [B, T, V] array / tensor: no per-utterance conversion, pointers by arithmetic
            owner, base, n, t_each, dtype_code, is_device = packed
            if n == 0:
                return []
            step = t_each * len(self._idx2vocab) * {0: 4, 1: 8, 2: 2, 3: 2}[dtype_code]
            if lengths is None:
                mats = [(owner, base + i * step, t_each, dtype_code, is_device) for i in range(n)]
            else:
                lens = [int(x) for x in lengths]
                if len(lens) != n or any(x < 0 or x > t_each for x in lens):
                    raise ValueError("lengths must hold one value in [0, T] per utterance of the padded batch")
                mats = [(owner, base + i * step, lens[i], dtype_code, is_device) for i in range(n)]
        else:
            for logits in logits_list:
                self._check_logits_dimension(logits)
            n = len(logits_list)
            if n == 0:
                return []
            mats = [_as_matrix(x) for x in logits_list]
            codes = {m[3] for m in mats}
            devs = {m[4] for m in mats}
            if len(codes) > 1 or len(devs) > 1:  # mixed batch: bring everything to host float64
                mats = [_as_matrix(x.detach().cpu().double().numpy() if hasattr(x, "cpu") else np.asarray(x, dtype=np.float64))
                        for x in logits_list]
        dtype_code, is_device = mats[0][3], mats[0][4]
        # device-resident input: the decoder that runs must live on the tensors' device (raw pointers cross the ABI)
        torch_stream = None
        if is_device:
            owners = {id(m[0]): m[0] for m in mats}.values()
            where = {_cuda_index(o) for o in owners}
            if len(where) != 1:
                raise ValueError("logits of one call live on different CUDA devices: %s" % sorted(where))
            (tensor_dev,) = where
            pinned = device if device is not None else self._device
            if pinned is not None and pinned != tensor_dev:
                raise ValueError("logits are on cuda:%d but this decoder is bound to cuda:%d" % (tensor_dev, pinned))
            device = tensor_dev
            import torch

            torch_stream = torch.cuda.current_stream(tensor_dev).cuda_stream
        with self._run_lock:
            return self._run_locked(mats, n, dtype_code, is_device, device, torch_stream, beam_width, beam_prune_logp,
                                    token_min_logp, prune_history, hotwords, hotword_weight, max_out_beams, lm_start_states,
                                    with_state, texts_only, stream, finalize_mode)

    def _run_locked(self, mats: List[Tuple[Any, int, int, int, bool]], n: int, dtype_code: int, is_device: bool,
                    device: Optional[int], torch_stream: Optional[int], beam_width: int, beam_prune_logp: float,
                    token_min_logp: float, prune_history: bool, hotwords: Optional[Iterable[str]], hotword_weight: float,
                    max_out_beams: int, lm_start_states: Optional[Sequence[Optional[AbstractLMState]]], with_state: bool,
                    texts_only: bool, stream: Optional[Sequence[Tuple[Sequence[Beam], int]]], finalize_mode: int) -> Any:
        handle = self._handle(device)
        lm = self._language_model
        L = _lib.lib()
        if torch_stream is not None:
            # the logits may still be in flight on torch's current stream: the decoder's stream waits for it
            _lib.check(L.b2c_decoder_wait_stream(handle, C.c_void_p(torch_stream)))
        models = self._lm_list()
        for idx, m in enumerate(models):
            _lib.check(L.b2c_decoder_set_params_lm(handle, idx, float(m.alpha), float(m.beta), float(m.unk_score_offset),
                                                   int(bool(m.score_boundary))))
        opts = _lib.DecodeOpts()
        L.b2c_decode_opts_default(C.byref(opts))
        opts.beam_width = int(beam_width)
        opts.beam_prune_logp = float(beam_prune_logp)
        opts.token_min_logp = float(token_min_logp)
        opts.prune_history = int(bool(prune_history))
        hot = [s.strip() for s in (hotwords or []) if len(s.strip()) > 0]
        hot_arr = _lib.cstr_array(hot)
        opts.hotwords = C.cast(hot_arr, C.POINTER(C.c_char_p))
        opts.n_hotwords = len(hot)
        opts.hotword_weight = float(hotword_weight)
        opts.max_out_beams = int(max_out_beams)
        states_arr = None
        n_lm = len(models)
        if lm is not None and lm_start_states is not None and any(s is not None for s in lm_start_states):
            states_arr = (_lib.LMState * (n * n_lm))()      # n_lm consecutive states per utterance
            for i, s in enumerate(lm_start_states):
                st = s if s is not None else lm.get_start_state()
                if n_lm > 1:
                    if not isinstance(st, MultiLanguageModelState) or len(st.states) != n_lm:
                        raise AssertionError("Wrong input state type found. Expected MultiLanguageModelState with %d states, "
                                             "got %s" % (n_lm, type(st)))
                    parts = list(st.states)
                else:
                    parts = [st]
                for j, part in enumerate(parts):
                    if not isinstance(part, B200LMState):
                        raise AssertionError("Wrong input state type found. Expected B200LMState, got %s" % type(part))
                    states_arr[i * n_lm + j] = part._to_c()
            opts.lm_start_states = C.cast(states_arr, C.POINTER(_lib.LMState))
        keep_alive: List[Any] = []
        if stream is not None:
            opts.stream_states = C.cast(self._stream_states(handle, stream, keep_alive), C.POINTER(_lib.StreamState))
        opts.finalize_mode = int(finalize_mode)
        opts.text_only = int(bool(texts_only))
        ptrs = (C.c_void_p * n)(*[m[1] for m in mats])
        Ts = (C.c_int32 * n)(*[m[2] for m in mats])
        res = C.c_void_p()
        _lib.check(L.b2c_decode_batch(handle, ptrs, Ts, n, dtype_code, int(is_device), C.byref(opts), C.byref(res)))
        try:
            if texts_only:
                data, size = C.c_void_p(), C.c_size_t()
                _lib.check(L.b2c_result_top_texts(res, C.byref(data), C.byref(size)))
                return C.string_at(data, size.value).decode("utf-8").split("\x00")[:n]
            if stream is not None:
                return self._stream_results(res, stream, finalize_mode)
            out = self._output_beams(L, res, with_state, n_lm)
        finally:
            L.b2c_result_free(res)
        return out

    _STATE_DTYPE = np.dtype([("w", "<u4", (5,)), ("b", "<f4", (5,)), ("n", "<u4")])

    @classmethod
    def _output_beams(cls, L: Any, res: Any, with_state: bool, n_lm: int) -> List[List[OutputBeam]]:
        """OutputBeam lists (reference decoder.py:653-667) from the flat arrays of b2c_result_packed: one library call
        per decode call, list slicing and C-level zip per beam."""
        pk = _lib.Packed()
        _lib.check(L.b2c_result_packed(res, C.byref(pk)))
        nb_total, nw_total = int(pk.n_beams_total), int(pk.n_words_total)
        counts = np.ctypeslib.as_array(pk.n_beams, shape=(pk.n_utts,)).tolist() if pk.n_utts else []
        if nb_total == 0:
            return [[] for _ in counts]
        scores = np.ctypeslib.as_array(pk.scores, shape=(2 * nb_total,)).tolist()
        n_words = np.ctypeslib.as_array(pk.n_words, shape=(nb_total,)).tolist()
        if nw_total:
            fr = np.ctypeslib.as_array(pk.frames, shape=(2 * nw_total,)).tolist()
            pairs = list(zip(fr[0::2], fr[1::2]))
        else:
            pairs = []
        texts = C.string_at(pk.texts, pk.texts_size).decode("utf-8").split("\x00")
        states: List[Any] = []
        if with_state and pk.n_models > 0 and bool(pk.states):
            nm = int(pk.n_models)
            raw = np.frombuffer(C.string_at(pk.states, C.sizeof(_lib.LMState) * nb_total * nm), dtype=cls._STATE_DTYPE)
            lens, ws, bs = raw["n"].tolist(), raw["w"].tolist(), raw["b"].tolist()
            flat = [B200LMState._from_tuples(tuple(w[:k]), tuple(b[:k])) for k, w, b in zip(lens, ws, bs)]
            states = flat if nm == 1 else [MultiLanguageModelState(flat[i:i + nm]) for i in range(0, len(flat), nm)]
        out: List[List[OutputBeam]] = []
        k = wi = 0
        for nb in counts:
            beams = []
            for _ in range(nb):
                nw = n_words[k]
                text = texts[k]
                if nw:
                    # words = the text's words (labels never contain a space inside a word)
                    frames = list(zip(text.split(" "), pairs[wi:wi + nw]))
                    wi += nw
                else:
                    frames = []
                beams.append(OutputBeam(text, states[k] if states else None, frames, scores[2 * k], scores[2 * k + 1]))
                k += 1
            out.append(beams)
        return out

    def last_timings(self, device: Optional[int] = None) -> Dict[str, float]:
        """Device-side timings of the last decode call (CUDA events on the decoder's stream)."""
        tm = _lib.Timings()
        _lib.check(_lib.lib().b2c_decoder_last_timings(self._handle(device), C.byref(tm)))
        out = {name: getattr(tm, name) for name, _ in _lib.Timings._fields_}
        out["cand_hist"] = list(out["cand_hist"])
        return out

    # ---- public decoding API (signatures of reference decoder.py:730-945) ------------------
    def decode_beams(self, logits: Any, beam_width: int = DEFAULT_BEAM_WIDTH, beam_prune_logp: float = DEFAULT_PRUNE_LOGP,
                     token_min_logp: float = DEFAULT_MIN_TOKEN_LOGP, prune_history: bool = DEFAULT_PRUNE_BEAMS,
                     hotwords: Optional[Iterable[str]] = None, hotword_weight: float = DEFAULT_HOTWORD_WEIGHT,
                     lm_start_state: Optional[AbstractLMState] = None) -> List[OutputBeam]:
        return self._run([logits], beam_width, beam_prune_logp, token_min_logp, prune_history, hotwords, hotword_weight,
                         max_out_beams=beam_width, lm_start_states=[lm_start_state])[0]

    def decode_beams_batch(self, pool: Any, logits_list: Sequence[Any], beam_width: int = DEFAULT_BEAM_WIDTH,
                           beam_prune_logp: float = DEFAULT_PRUNE_LOGP, token_min_logp: float = DEFAULT_MIN_TOKEN_LOGP,
                           prune_history: bool = DEFAULT_PRUNE_BEAMS, hotwords: Optional[Iterable[str]] = None,
                           hotword_weight: float = DEFAULT_HOTWORD_WEIGHT,
                           lengths: Optional[Sequence[int]] = None) -> List[List[OutputBeam]]:
        """`lengths` (extension, SURVEY 8f-4): valid frames per utterance when `logits_list` is ONE padded
        [B, T, V] array or (CUDA) tensor -- the padding rows are never read."""
        # the reference strips the LM state for multiprocessing (decoder.py:797-799); keep that
        return self._run(logits_list, beam_width, beam_prune_logp, token_min_logp, prune_history, hotwords,
                         hotword_weight, max_out_beams=beam_width, with_state=False, lengths=lengths)

    def decode(self, logits: Any, beam_width: int = DEFAULT_BEAM_WIDTH, beam_prune_logp: float = DEFAULT_PRUNE_LOGP,
               token_min_logp: float = DEFAULT_MIN_TOKEN_LOGP, hotwords: Optional[Iterable[str]] = None,
               hotword_weight: float = DEFAULT_HOTWORD_WEIGHT, lm_start_state: Optional[AbstractLMState] = None) -> str:
        beams = self._run([logits], beam_width, beam_prune_logp, token_min_logp, True, hotwords, hotword_weight,
                          max_out_beams=1, lm_start_states=[lm_start_state], with_state=False)[0]
        return beams[0].text

    def decode_batch(self, pool: Any, logits_list: Sequence[Any], beam_width: int = DEFAULT_BEAM_WIDTH,
                     beam_prune_logp: float = DEFAULT_PRUNE_LOGP, token_min_logp: float = DEFAULT_MIN_TOKEN_LOGP,
                     hotwords: Optional[Iterable[str]] = None, hotword_weight: float = DEFAULT_HOTWORD_WEIGHT,
                     lengths: Optional[Sequence[int]] = None) -> List[str]:
        return self._run(logits_list, beam_width, beam_prune_logp, token_min_logp, True, hotwords, hotword_weight,
                         max_out_beams=1, with_state=False, texts_only=True, lengths=lengths)

    # ---- streaming (reference decoder.py:669-728) ------------------------------------------------
    def get_starting_state(self) -> Tuple[List[Beam], LMScoreCache, Dict[str, float]]:
        """Starting beams and caches, same shape as the reference returns (decoder.py:669-680).  The caches are
        accepted back by partial_decode_beams for signature compatibility; only the start state stored under
        ("", False) is read -- the kernels recompute LM / hotword scores of the carried beams from their words."""
        language_model = self._language_model
        cached_lm_scores: LMScoreCache = {}
        if language_model is not None:
            cached_lm_scores[("", False)] = (0.0, 0.0, language_model.get_start_state())
        return [EMPTY_START_BEAM], cached_lm_scores, {}

    def _token_id(self, handle: int, label: Optional[str]) -> int:
        if label is None:
            return 0xFFFF
        ids = self._label_ids
        tid = ids.get(label)
        if tid is None:
            tid = int(_lib.lib().b2c_decoder_token_id(handle, label.encode("utf-8")))
            if tid < 0:
                raise ValueError("beam.last_char %r is not a label of this decoder's alphabet" % (label,))
            ids[label] = tid
        return tid

    # ---- streaming host path ---------------------------------------------------------------------------------
    # The beam state travels as Python strings (the reference's API).  The kernels identify words by hashes, so every
    # call has to hand over the word hashes of every carried beam's text.  Two caches keep that linear in what is NEW:
    #   _word_hash    word -> (hash as 8 bytes, code points as 4 bytes, hash, code points), filled by ONE library call
    #                 per decode call for all the words not seen before
    #   _text_cache   text -> (hashes of its words as bytes, their lengths as bytes, word count) for the beams the last
    #                 two calls returned (a call's output texts are the next call's input texts); misses re-split the text
    _SB_DTYPE = np.dtype([("part_hash", "<u8"), ("logit", "<f8"), ("word_off", "<u4"), ("n_words", "<u4"), ("part_len", "<u4"),
                          ("last_tok", "<u4"), ("pf_s", "<i4"), ("pf_e", "<i4")])

    def _hash_words(self, words: Sequence[str]) -> None:
        if not words:
            return
        n = len(words)
        data = b"".join([w.encode("utf-8") + b"\x00" for w in words])
        hs, ls = np.empty(n, dtype=np.uint64), np.empty(n, dtype=np.uint32)
        _lib.check(_lib.lib().b2c_hash_utf8_batch(data, len(data), n, hs.ctypes.data_as(C.POINTER(C.c_uint64)),
                                                  ls.ctypes.data_as(C.POINTER(C.c_uint32))))
        table = self._word_hash
        if len(table) > 1000000:
            table.clear()
        hb, lb, hl, ll = hs.tobytes(), ls.tobytes(), hs.tolist(), ls.tolist()
        for i, w in enumerate(words):
            table[w] = (hb[8 * i:8 * i + 8], lb[4 * i:4 * i + 4], hl[i], ll[i])

    def _text_entry(self, text: str) -> Optional[Tuple[bytes, bytes, int]]:
        ent = self._text_cache[0].get(text)
        if ent is None:
            ent = self._text_cache[1].get(text)
        return ent

    def _stream_states(self, handle: int, stream: Sequence[Tuple[Sequence[Beam], int]], keep_alive: List[Any]) -> Any:
        """List of (beams, processed_frames) per utterance -> b2c_stream_state_t array (words and partial words
        as hashes, last_char as a token id)."""
        table = self._word_hash
        c0, c1 = self._text_cache
        # pass 1: the cached entry of every beam's text; which strings need hashing
        missing: Dict[str, None] = {}
        found: List[Any] = []            # per beam: cache entry, or the text itself on a miss
        for beams, _ in stream:
            for beam in beams:
                text = beam.text if not beam.next_word else _merge_tokens(beam.text, beam.next_word)
                ent = c0.get(text)
                if ent is None:
                    ent = c1.get(text)
                if ent is None:
                    ent = text
                    for w in text.split():
                        if w not in table:
                            missing[w] = None
                found.append(ent)
                pw = beam.partial_word
                if pw and pw not in table:
                    missing[pw] = None
        self._hash_words(list(missing))
        # pass 2: columns of the beam rows and the word arrays (one allocation each for the whole call)
        n_rows = len(found)
        col_ph, col_lg, col_off, col_nw, col_pl, col_lt, col_s, col_e = [], [], [], [], [], [], [], []
        hparts: List[bytes] = []
        lparts: List[bytes] = []
        starts: List[Tuple[int, int, int, int]] = []        # per utterance: first row, rows, first word, words
        n_words_total = r = 0
        ids = self._label_ids
        for beams, _ in stream:
            row0, off = r, 0
            for beam in beams:
                ent = found[r]
                r += 1
                if ent.__class__ is str:
                    words = ent.split()
                    ent = c0[ent] = (b"".join([table[w][0] for w in words]), b"".join([table[w][1] for w in words]), len(words))
                hparts.append(ent[0])
                lparts.append(ent[1])
                pw = beam.partial_word
                if pw:
                    e = table[pw]
                    col_ph.append(e[2])
                    col_pl.append(e[3])
                else:
                    col_ph.append(0)
                    col_pl.append(0)
                col_lg.append(beam.logit_score)
                col_off.append(off)
                col_nw.append(ent[2])
                lc = beam.last_char
                col_lt.append(0xFFFF if lc is None else (ids[lc] if lc in ids else self._token_id(handle, lc)))
                pf = beam.partial_frames
                col_s.append(pf[0])
                col_e.append(pf[1])
                off += ent[2]
            starts.append((row0, r - row0, n_words_total, off))
            n_words_total += off
        a_rows = np.zeros(max(1, n_rows), dtype=self._SB_DTYPE)
        if n_rows:
            for name, col in (("part_hash", col_ph), ("logit", col_lg), ("word_off", col_off), ("n_words", col_nw), ("part_len", col_pl),
                              ("last_tok", col_lt), ("pf_s", col_s), ("pf_e", col_e)):
                a_rows[name] = col
        a_wh = np.frombuffer(b"".join(hparts) or b"\x00" * 8, dtype=np.uint64)
        a_wl = np.frombuffer(b"".join(lparts) or b"\x00" * 4, dtype=np.uint32)
        assert a_rows.itemsize == C.sizeof(_lib.StreamBeam)
        states = (_lib.StreamState * len(stream))()
        p_rows, p_wh, p_wl = a_rows.ctypes.data, a_wh.ctypes.data, a_wl.ctypes.data
        for u, ((_, processed_frames), (row0, n_beams, word0, n_words)) in enumerate(zip(stream, starts)):
            st = states[u]
            st.beams = C.cast(p_rows + row0 * a_rows.itemsize, C.POINTER(_lib.StreamBeam))
            st.n_beams = n_beams
            st.processed_frames = int(processed_frames)
            st.word_hashes = C.cast(p_wh + 8 * word0, C.POINTER(C.c_uint64))
            st.word_lens = C.cast(p_wl + 4 * word0, C.POINTER(C.c_uint32))
            st.n_words = n_words
        keep_alive.extend([a_rows, a_wh, a_wl, states])
        return states

    @staticmethod
    def _new_lm_beam(text: str, partial: str, last_char: Optional[str], frames: List[Frames], pframes: Frames, logit: float,
                     lm: float) -> LMBeam:
        # LMBeam(text, "", partial, last_char, frames, pframes, logit, lm) without the eight object.__setattr__ calls of
        # a frozen dataclass's __init__ (a streaming call returns thousands of beams)
        beam = LMBeam.__new__(LMBeam)
        beam.__dict__.update(text=text, next_word="", partial_word=partial, last_char=last_char, text_frames=frames,
                             partial_frames=pframes, logit_score=logit, lm_score=lm)
        return beam

    def _stream_results(self, res: Any, stream: Sequence[Tuple[Sequence[Beam], int]], finalize_mode: int) -> List[List[LMBeam]]:
        """What the call appended (the token chain since the input beam, replayed into strings by the library; frames of
        the words finished during the call) on top of the input beams' strings -> LMBeam lists (reference
        _finalize_beams output)."""
        L = _lib.lib()
        pk = _lib.Packed()
        _lib.check(L.b2c_result_packed(res, C.byref(pk)))
        nb_total, nw_total = int(pk.n_beams_total), int(pk.n_words_total)
        counts = np.ctypeslib.as_array(pk.n_beams, shape=(pk.n_utts,)).tolist() if pk.n_utts else []
        if nb_total == 0:
            return [[] for _ in counts]
        scores = np.ctypeslib.as_array(pk.scores, shape=(2 * nb_total,)).tolist()
        n_frames = np.ctypeslib.as_array(pk.n_words, shape=(nb_total,)).tolist()
        aux = np.ctypeslib.as_array(pk.stream_aux, shape=(4 * nb_total,)).tolist()
        boundary = np.ctypeslib.as_array(pk.stream_boundary, shape=(nb_total,)).tolist()
        pieces = C.string_at(pk.stream_pieces, pk.stream_pieces_size).decode("utf-8").split("\x00")
        if nw_total:
            fr = np.ctypeslib.as_array(pk.frames, shape=(2 * nw_total,)).tolist()
            pairs = list(zip(fr[0::2], fr[1::2]))
        else:
            pairs = []
        labels = self._alphabet.labels
        keep = finalize_mode == _lib.FIN_KEEP
        table = self._word_hash
        c0, c1 = self._text_cache
        spaced = self._labels_with_space
        new_beam = self._new_lm_beam
        pending: Dict[str, Tuple[Tuple[bytes, bytes, int], List[str]]] = {}     # new text -> (entry of the root text, appended words)
        missing: Dict[str, None] = {}
        out: List[List[LMBeam]] = []
        k = wi = 0
        for u, nb in enumerate(counts):
            roots = stream[u][0]
            beams = []
            for _ in range(nb):
                a0 = aux[4 * k]
                root = roots[a0] if a0 >= 0 else EMPTY_START_BEAM
                root_text = root.text if not root.next_word else _merge_tokens(root.text, root.next_word)
                first, mid, last = pieces[3 * k], pieces[3 * k + 1], pieces[3 * k + 2]
                if boundary[k]:
                    word0 = root.partial_word + first
                    text = root_text
                    if word0:                           # branches (ii) / (iii): a word boundary finishes the partial word
                        text = text + " " + word0 if text else word0
                    if mid:
                        text = text + " " + mid if text else mid
                    partial = last
                else:                                   # branch (iv) only: the partial word grew
                    text, partial = root_text, root.partial_word + first
                nf = n_frames[k]
                frames = list(root.text_frames) + pairs[wi:wi + nf] if nf else list(root.text_frames)
                wi += nf
                if keep:
                    a1 = aux[4 * k + 1]
                    beams.append(new_beam(text, partial, None if a1 < 0 else labels[a1], frames, (aux[4 * k + 2], aux[4 * k + 3]),
                                          scores[2 * k], scores[2 * k + 1]))
                    if text not in pending:
                        ent = c0.get(root_text)
                        if ent is None:
                            ent = c1.get(root_text)
                        if ent is None and not root_text:
                            ent = (b"", b"", 0)
                        if ent is not None:
                            added: List[str] = []
                            if boundary[k]:
                                if word0:
                                    added.append(word0)
                                if mid:
                                    added.extend(mid.split(" "))
                            # labels with white space inside would make text.split() disagree with the word list
                            if not spaced or all(len(w.split()) == 1 for w in added):
                                pending[text] = (ent, added)
                                for w in added:
                                    if w not in table:
                                        missing[w] = None
                else:
                    beams.append(new_beam(_merge_tokens(text, partial), "", None, frames, NULL_FRAMES, scores[2 * k], scores[2 * k + 1]))
                k += 1
            out.append(beams)
        # the texts this call returned are the texts the next call brings back: their word hashes, incrementally
        self._hash_words(list(missing))
        fresh: Dict[str, Tuple[bytes, bytes, int]] = {}
        for text, (ent, added) in pending.items():
            if added:
                fresh[text] = (ent[0] + b"".join([table[w][0] for w in added]), ent[1] + b"".join([table[w][1] for w in added]),
                               ent[2] + len(added))
            else:
                fresh[text] = ent
        self._text_cache = [fresh, c0]
        return out

    def partial_decode_beams(self, logits: Any, cached_lm_scores: LMScoreCache, cached_p_lm_scores: Dict[str, float],
                             beams: List[Beam], processed_frames: int, beam_width: int = DEFAULT_BEAM_WIDTH,
                             beam_prune_logp: float = DEFAULT_PRUNE_LOGP, token_min_logp: float = DEFAULT_MIN_TOKEN_LOGP,
                             prune_history: bool = DEFAULT_PRUNE_BEAMS, hotword_scorer: Optional[HotwordScorer] = None,
                             force_next_word: bool = False, is_end: bool = False) -> List[LMBeam]:
        """Decode one chunk of logits starting from `beams` (reference decoder.py:682-728).  The beam state
        travels as the returned LMBeam list, exactly like in the reference; the chunk itself (input
        normalisation, frame loop, _finalize_beams with force_next_word / is_end) runs on the device."""
        return self.partial_decode_beams_batch([logits], [cached_lm_scores], [beams], [processed_frames], beam_width,
                                               beam_prune_logp, token_min_logp, prune_history, hotword_scorer,
                                               force_next_word, is_end)[0]

    def partial_decode_beams_batch(self, logits_list: Sequence[Any], cached_lm_scores_list: Sequence[Optional[LMScoreCache]],
                                   beams_list: Sequence[List[Beam]], processed_frames_list: Sequence[int],
                                   beam_width: int = DEFAULT_BEAM_WIDTH, beam_prune_logp: float = DEFAULT_PRUNE_LOGP,
                                   token_min_logp: float = DEFAULT_MIN_TOKEN_LOGP, prune_history: bool = DEFAULT_PRUNE_BEAMS,
                                   hotword_scorer: Optional[HotwordScorer] = None, force_next_word: bool = False,
                                   is_end: bool = False) -> List[List[LMBeam]]:
        """Extension: many independent streams advance by one chunk each in ONE kernel launch."""
        n = len(logits_list)
        if not (len(beams_list) == len(processed_frames_list) == len(cached_lm_scores_list) == n):
            raise ValueError("one beam list, cache and processed_frames value per stream")
        lm = self._language_model
        starts: Optional[List[Optional[AbstractLMState]]] = None
        if lm is not None:
            starts = []
            for cache in cached_lm_scores_list:
                entry = (cache or {}).get(("", False))
                starts.append(entry[2] if entry is not None else None)
        hot = hotword_scorer.unigrams if hotword_scorer is not None else None
        weight = hotword_scorer.weight if hotword_scorer is not None else DEFAULT_HOTWORD_WEIGHT
        mode = _lib.FIN_EOS if is_end else (_lib.FIN_FLUSH if force_next_word else _lib.FIN_KEEP)
        return self._run(logits_list, beam_width, beam_prune_logp, token_min_logp, prune_history, hot, weight,
                         max_out_beams=beam_width, lm_start_states=starts, with_state=False,
                         stream=[(list(b), int(p)) for b, p in zip(beams_list, processed_frames_list)], finalize_mode=mode)

    # ---- serialisation (reference decoder.py:947-1005): file plumbing only ------------------
    def save_to_dir(self, filepath: str) -> None:
        with open(os.path.join(filepath, self._ALPHABET_SERIALIZED_FILENAME), "w") as fh:
            fh.write(self._alphabet.dumps())
        lm = self._language_model
        if lm is not None:
            lm_path = os.path.join(filepath, self._LANGUAGE_MODEL_SERIALIZED_DIRECTORY)
            os.makedirs(lm_path)
            lm.save_to_dir(lm_path)

    @staticmethod
    def parse_directory_contents(filepath: str) -> Dict[str, Union[str, None]]:
        contents = [c for c in os.listdir(filepath) if not c.startswith(".") and not c.startswith("__")]
        if BeamSearchDecoderCTC._ALPHABET_SERIALIZED_FILENAME not in contents:
            raise ValueError("Could not find alphabet file %s. Found %s" % (BeamSearchDecoderCTC._ALPHABET_SERIALIZED_FILENAME, contents))
        contents.remove(BeamSearchDecoderCTC._ALPHABET_SERIALIZED_FILENAME)
        lm_directory: Optional[str] = None
        if contents:
            if BeamSearchDecoderCTC._LANGUAGE_MODEL_SERIALIZED_DIRECTORY not in contents:
                raise ValueError("Count not find language model directory. Looking for %s, found %s"
                                 % (BeamSearchDecoderCTC._LANGUAGE_MODEL_SERIALIZED_DIRECTORY, contents))
            lm_directory = os.path.join(filepath, BeamSearchDecoderCTC._LANGUAGE_MODEL_SERIALIZED_DIRECTORY)
        return {"alphabet": os.path.join(filepath, BeamSearchDecoderCTC._ALPHABET_SERIALIZED_FILENAME),
                "language_model": lm_directory}

    @classmethod
    def load_from_dir(cls, filepath: str, unigram_encoding: Optional[str] = None) -> "BeamSearchDecoderCTC":
        names = cls.parse_directory_contents(filepath)
        with open(names["alphabet"]) as fh:  # type: ignore[arg-type]
            alphabet = Alphabet.loads(fh.read())
        lm = None
        if names["language_model"] is not None:
            lm = LanguageModel.load_from_dir(names["language_model"], unigram_encoding=unigram_encoding)
        return cls(alphabet, language_model=lm)


def build_ctcdecoder(labels: List[str], kenlm_model_path: Optional[str] = None, unigrams: Optional[Collection[str]] = None,
                     alpha: float = DEFAULT_ALPHA, beta: float = DEFAULT_BETA,
                     unk_score_offset: float = DEFAULT_UNK_LOGP_OFFSET,
                     lm_score_boundary: bool = DEFAULT_SCORE_LM_BOUNDARY, device: Optional[int] = None) -> BeamSearchDecoderCTC:
    """Same arguments and semantics as reference decoder.py:1051-1099; ``kenlm_model_path`` is an ARPA file, a KenLM
    binary of the probing model type, or a ``*.b2clm`` blob written by ``NgramModel.save_blob``."""
    from_blob = kenlm_model_path is not None and kenlm_model_path.endswith(NgramModel.BLOB_SUFFIX)
    if from_blob:
        # a flattened model written by NgramModel.save_blob: no ARPA parse; it carries its unigram / prefix sets
        ngram = NgramModel.load_blob(kenlm_model_path)
    else:
        ngram = None if kenlm_model_path is None else NgramModel(kenlm_model_path)
    if unigrams is None and kenlm_model_path is not None and not from_blob:
        if kenlm_model_path.endswith(".arpa"):
            unigrams = load_unigram_set_from_arpa(kenlm_model_path)
        else:
            logger.warning("Unigrams not provided and cannot be automatically determined from LM file (only "
                           "arpa format). Decoding accuracy might be reduced.")
    alphabet = Alphabet.build_alphabet(labels)
    if unigrams is not None:
        verify_alphabet_coverage(alphabet, unigrams)
    language_model: Optional[AbstractLanguageModel] = None
    if ngram is not None:
        language_model = LanguageModel(ngram, unigrams, alpha=alpha, beta=beta, unk_score_offset=unk_score_offset,
                                       score_boundary=lm_score_boundary)
    return BeamSearchDecoderCTC(alphabet, language_model, device=device)
