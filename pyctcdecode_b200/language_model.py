"""Host-side language-model objects of the CUDA decoder.

Same surface as reference pyctcdecode/language_model.py (LanguageModel, HotwordScorer, the
state wrappers), but the n-gram engine is the library's own flattened model
(csrc/b2c_lm_host.h, resident in HBM for the kernels) instead of the kenlm package, and the
unigram prefix trie is a hash set inside the same blob instead of pygtrie.  The methods here
evaluate on the HOST copy of the tables; they exist for API compatibility and for tests --
during decoding the same arithmetic runs inside the beam kernel (csrc/b2c_lm.h).
"""
import abc
import ctypes as C
import json
import logging
import os
import shutil
from typing import Any, Collection, Dict, Iterable, List, Optional, Sequence, Set, Tuple

from . import _lib
from .constants import (
    AVG_TOKEN_LEN,
    DEFAULT_ALPHA,
    DEFAULT_BETA,
    DEFAULT_HOTWORD_WEIGHT,
    DEFAULT_SCORE_LM_BOUNDARY,
    DEFAULT_UNK_LOGP_OFFSET,
    LOG_BASE_CHANGE_FACTOR,
)

logger = logging.getLogger(__name__)


class AbstractLMState(abc.ABC):
    def get_mp_safe_state(self) -> Optional["AbstractLMState"]:
        return None


class B200LMState(AbstractLMState):
    """n-gram context (word ids most recent first + their backoffs); plain data, picklable.

    Plays the role of reference ``KenlmState`` (language_model.py:45-53)."""

    def __init__(self, words: Sequence[int] = (), backoffs: Sequence[float] = ()) -> None:
        self.words = tuple(int(w) for w in words)
        self.backoffs = tuple(float(b) for b in backoffs)

    @classmethod
    def _from_c(cls, st: _lib.LMState) -> "B200LMState":
        n = st.length
        return cls(st.words[:n], st.backoff[:n])

    @classmethod
    def _from_tuples(cls, words: Tuple[int, ...], backoffs: Tuple[float, ...]) -> "B200LMState":
        st = cls.__new__(cls)
        st.words = words
        st.backoffs = backoffs
        return st

    def _to_c(self) -> _lib.LMState:
        st = _lib.LMState()
        st.length = len(self.words)
        for i, (w, b) in enumerate(zip(self.words, self.backoffs)):
            st.words[i] = w
            st.backoff[i] = b
        return st

    @property
    def state(self) -> "B200LMState":
        return self

    def get_mp_safe_state(self) -> "B200LMState":
        return self

    def __eq__(self, other: object) -> bool:
        return isinstance(other, B200LMState) and self.words == other.words and self.backoffs == other.backoffs

    def __repr__(self) -> str:
        return "B200LMState(words=%r)" % (self.words,)


KenlmState = B200LMState  # name used by code written against the reference


def load_unigram_set_from_arpa(arpa_path: str) -> Set[str]:
    """Unigrams of an ARPA file -- only lines with three tab separated fields count, exactly
    like reference language_model.py:67-84."""
    found: Set[str] = set()
    in_unigrams = False
    with open(arpa_path, encoding="utf-8") as fh:
        for raw in fh:
            line = raw.strip()
            if line == "\\1-grams:":
                in_unigrams = True
            elif line == "\\2-grams:":
                break
            if in_unigrams and line:
                fields = line.split("\t")
                if len(fields) == 3:
                    found.add(fields[1])
    if not found:
        raise ValueError("No unigrams found in arpa file. Something is wrong with the file.")
    return found


class NgramModel:
    """``kenlm.Model`` look-alike over the library's flattened n-gram tables: ARPA files and KenLM binaries of the
    probing model type (what ``build_binary`` writes by default; trie / quantised binaries raise).

    Covers the calls the reference makes on a kenlm model: ``word in model``, ``.order``,
    ``.path``, ``BeginSentenceWrite``, ``NullContextWrite``, ``BaseScore``."""

    def __init__(self, path: str, unigrams: Optional[Collection[str]] = None, _handle: Optional[int] = None) -> None:
        self.path = os.path.abspath(path).encode("utf-8")
        if not os.path.exists(path):
            raise OSError("Cannot read model '%s'" % path)
        self._unigrams = None if unigrams is None else list(unigrams)
        self._handle = _handle

    def _h(self) -> int:
        if self._handle is None:
            out = C.c_void_p()
            if self._unigrams is None:
                rc = _lib.lib().b2c_lm_build_from_file(self.path, None, -1, C.byref(out))
            else:
                arr = _lib.cstr_array(self._unigrams)
                rc = _lib.lib().b2c_lm_build_from_file(self.path, arr, len(self._unigrams), C.byref(out))
            _lib.check(rc)
            self._handle = out.value
        return self._handle

    def with_unigrams(self, unigrams: Optional[Collection[str]]) -> "NgramModel":
        """A model over the same ARPA file whose blob carries the unigram set / prefix set."""
        if getattr(self, "_from_blob_file", False):
            return self            # a saved blob already carries the unigram / prefix sets it was built with
        if unigrams is None and self._unigrams is None:
            return self
        return NgramModel(self.path.decode("utf-8"), unigrams)

    @property
    def order(self) -> int:
        return int(_lib.lib().b2c_lm_order(self._h()))

    def __contains__(self, word: str) -> bool:
        return bool(_lib.lib().b2c_lm_contains(self._h(), word.encode("utf-8")))

    def in_unigrams(self, word: str) -> bool:
        return bool(_lib.lib().b2c_lm_in_unigrams(self._h(), word.encode("utf-8")))

    def has_prefix(self, prefix: str) -> bool:
        return bool(_lib.lib().b2c_lm_has_prefix(self._h(), prefix.encode("utf-8")))

    @property
    def have_unigrams(self) -> bool:
        """The tables carry a unigram set / prefix set (the model was built with a unigram list)."""
        return bool(_lib.lib().b2c_lm_have_unigrams(self._h()))

    def BeginSentenceWrite(self, state: B200LMState) -> None:  # noqa: N802 (kenlm naming)
        st = _lib.LMState()
        _lib.lib().b2c_lm_begin_sentence(self._h(), C.byref(st))
        state.words, state.backoffs = tuple(st.words[: st.length]), tuple(st.backoff[: st.length])

    def NullContextWrite(self, state: B200LMState) -> None:  # noqa: N802
        state.words, state.backoffs = (), ()

    def BaseScore(self, in_state: B200LMState, word: str, out_state: B200LMState) -> float:  # noqa: N802
        a, b = in_state._to_c(), _lib.LMState()
        score = _lib.lib().b2c_lm_base_score(self._h(), C.byref(a), word.encode("utf-8"), C.byref(b))
        out_state.words, out_state.backoffs = tuple(b.words[: b.length]), tuple(b.backoff[: b.length])
        return float(score)

    def blob(self) -> Tuple[int, int]:
        """(address, size) of the relocatable table blob (what an NCCL broadcast ships)."""
        data, size = C.c_void_p(), C.c_size_t()
        _lib.check(_lib.lib().b2c_lm_blob(self._h(), C.byref(data), C.byref(size)))
        return data.value, size.value

    @classmethod
    def from_blob(cls, path: str, address: int, size: int) -> "NgramModel":
        out = C.c_void_p()
        _lib.check(_lib.lib().b2c_lm_from_blob(C.c_void_p(address), size, C.byref(out)))
        obj = cls.__new__(cls)
        obj.path = os.path.abspath(path).encode("utf-8")
        obj._unigrams = None
        obj._handle = out.value
        return obj

    BLOB_SUFFIX = ".b2clm"

    def save_blob(self, path: str) -> None:
        """Write the flattened model (n-gram / vocabulary / unigram-prefix hash tables, SURVEY 8f-3) to `path`.
        Loading it back with :meth:`load_blob` skips the ARPA parse, which dominates start-up for large models."""
        address, size = self.blob()
        with open(path, "wb") as fh:
            fh.write(C.string_at(address, size))

    @classmethod
    def load_blob(cls, path: str) -> "NgramModel":
        """A model from a file written by :meth:`save_blob` (the blob is validated by magic and size)."""
        with open(path, "rb") as fh:
            data = fh.read()
        buf = C.create_string_buffer(data, len(data))
        obj = cls.from_blob(path, C.addressof(buf), len(data))
        obj._from_blob_file = True
        return obj

    def __del__(self) -> None:
        h = getattr(self, "_handle", None)
        if h and _lib._lib is not None:
            try:
                _lib._lib.b2c_lm_destroy(h)
            except Exception:  # pragma: no cover - interpreter shutdown
                pass
            self._handle = None


class HotwordScorer:
    """Host mirror of reference HotwordScorer (language_model.py:115-189).

    ``score(text)`` is weight x number of whitespace separated words of ``text`` that are hotword
    unigrams (what the reference's look-around regex counts); the partial score is
    ``weight * len(prefix) / len(shortest hotword starting with prefix)``.  The kernels use a
    hash table with the same content (csrc/b2c_api.cu build_hot)."""

    def __init__(self, unigrams: Iterable[str] = (), weight: float = DEFAULT_HOTWORD_WEIGHT) -> None:
        self._weight = weight
        self._words = set(unigrams)
        self._prefix_min_len: Dict[str, int] = {}
        for w in self._words:
            for i in range(len(w) + 1):
                p = w[:i]
                if p not in self._prefix_min_len or len(w) < self._prefix_min_len[p]:
                    self._prefix_min_len[p] = len(w)

    @property
    def unigrams(self) -> List[str]:
        return sorted(self._words)

    @property
    def weight(self) -> float:
        return self._weight

    def __contains__(self, item: str) -> bool:
        return item in self._prefix_min_len

    def score(self, text: str) -> float:
        return self._weight * sum(1 for w in text.split() if w in self._words)

    def score_partial_token(self, token: str) -> float:
        if token in self._prefix_min_len:
            return self._weight * len(token) / self._prefix_min_len[token]
        return 0.0

    @classmethod
    def build_scorer(cls, hotwords: Optional[Iterable[str]] = None, weight: float = DEFAULT_HOTWORD_WEIGHT) -> "HotwordScorer":
        unigrams: List[str] = []
        for phrase in hotwords or []:
            unigrams.extend(phrase.split())
        return cls(unigrams, weight)


class AbstractLanguageModel(abc.ABC):
    @property
    @abc.abstractmethod
    def order(self) -> int:
        raise NotImplementedError()

    @abc.abstractmethod
    def get_start_state(self) -> AbstractLMState:
        raise NotImplementedError()

    @abc.abstractmethod
    def score_partial_token(self, partial_token: str) -> float:
        raise NotImplementedError()

    @abc.abstractmethod
    def score(self, prev_state: AbstractLMState, word: str, is_last_word: bool = False) -> Tuple[float, AbstractLMState]:
        raise NotImplementedError()

    def save_to_dir(self, filepath: str) -> None:
        raise NotImplementedError()

    @classmethod
    def load_from_dir(cls, filepath: str) -> "AbstractLanguageModel":
        raise NotImplementedError()

    def reset_params(self, **params: Any) -> None:
        """Reset some of the parameters in place."""


class LanguageModel(AbstractLanguageModel):
    JSON_ATTRS = ("alpha", "beta", "unk_score_offset", "score_boundary")
    _ATTRS_SERIALIZED_FILENAME = "attrs.json"
    _UNIGRAMS_SERIALIZED_FILENAME = "unigrams.txt"

    def __init__(
        self,
        kenlm_model: Any,
        unigrams: Optional[Collection[str]] = None,
        alpha: float = DEFAULT_ALPHA,
        beta: float = DEFAULT_BETA,
        unk_score_offset: float = DEFAULT_UNK_LOGP_OFFSET,
        score_boundary: bool = DEFAULT_SCORE_LM_BOUNDARY,
    ) -> None:
        """``kenlm_model``: an :class:`NgramModel` or the path of an ARPA file (reference
        language_model.py:237-269 takes a ``kenlm.Model``)."""
        if isinstance(kenlm_model, (str, bytes, os.PathLike)):
            kenlm_model = NgramModel(os.fsdecode(kenlm_model))
        if not isinstance(kenlm_model, NgramModel):
            raise TypeError("kenlm_model must be a pyctcdecode_b200 NgramModel or an ARPA path")
        self._blob_unigrams = bool(getattr(kenlm_model, "_from_blob_file", False)) and unigrams is None and kenlm_model.have_unigrams
        if self._blob_unigrams:
            # a saved *.b2clm blob carries the unigram / prefix sets it was built with; the word list itself is not stored
            self._unigram_list: Optional[List[str]] = None
        elif unigrams is None:
            logger.warning("No known unigrams provided, decoding results might be a lot worse.")
            self._unigram_list = None
        else:
            if len(unigrams) < 1000:
                logger.warning("Only %s unigrams passed as vocabulary. Is this small or artificial data?", len(unigrams))
            self._unigram_list = sorted(set(unigrams))
        # the device blob carries the (filtered) unigram set and its prefix set
        self._kenlm_model = kenlm_model.with_unigrams(self._unigram_list)
        self.alpha = alpha
        self.beta = beta
        self.unk_score_offset = unk_score_offset
        self.score_boundary = score_boundary

    # ---- pieces of the reference object the tests / HF integration look at ----------------
    @property
    def _unigram_set(self) -> Set[str]:
        if self._unigram_list is None:
            return set()
        return {w for w in self._unigram_list if w in self._kenlm_model}

    @property
    def ngram_model(self) -> NgramModel:
        return self._kenlm_model

    def reset_params(self, **params: Any) -> None:
        """reference language_model.py:271-301 (same type checks, same messages)."""
        for name, typ in (("alpha", float), ("beta", float), ("unk_score_offset", float), ("score_boundary", bool)):
            value = params.get(name)
            if value is None:
                continue
            if not isinstance(value, typ):
                raise ValueError("%s must be a %s. Got %s." % (name, typ.__name__, type(value)))
            setattr(self, name, value)

    @property
    def order(self) -> int:
        return self._kenlm_model.order

    def get_start_state(self) -> B200LMState:
        state = B200LMState()
        if self.score_boundary:
            self._kenlm_model.BeginSentenceWrite(state)
        else:
            self._kenlm_model.NullContextWrite(state)
        return state

    def _get_raw_end_score(self, start_state: B200LMState) -> float:
        if not self.score_boundary:
            return 0.0
        return self._kenlm_model.BaseScore(start_state, "</s>", B200LMState())

    def score_partial_token(self, partial_token: str) -> float:
        if self._blob_unigrams:
            is_oov = int(not self._kenlm_model.has_prefix(partial_token))
        elif self._unigram_list is None:
            is_oov = 1.0
        else:
            is_oov = int(not self._kenlm_model.has_prefix(partial_token)) if partial_token else int(len(self._unigram_set) == 0)
        unk_score = self.unk_score_offset * is_oov
        if len(partial_token) > AVG_TOKEN_LEN:
            unk_score = unk_score * len(partial_token) / AVG_TOKEN_LEN
        return unk_score

    def score(self, prev_state: AbstractLMState, word: str, is_last_word: bool = False) -> Tuple[float, B200LMState]:
        if not isinstance(prev_state, B200LMState):
            raise AssertionError("Wrong input state type found. Expected B200LMState, got %s" % type(prev_state))
        end_state = B200LMState()
        lm_score = self._kenlm_model.BaseScore(prev_state, word, end_state)
        have_unigrams = (self._unigram_list is not None and len(self._unigram_set) > 0) or \
            (self._blob_unigrams and self._kenlm_model.has_prefix(""))
        if (have_unigrams and not self._kenlm_model.in_unigrams(word)) or word not in self._kenlm_model:
            lm_score += self.unk_score_offset
        if is_last_word:
            lm_score = lm_score + self._get_raw_end_score(end_state)
        return self.alpha * lm_score * LOG_BASE_CHANGE_FACTOR + self.beta, end_state

    # ---- serialisation (reference language_model.py:371-452): file plumbing, pure python --------
    @property
    def serializable_attrs(self) -> Dict[str, Any]:
        return {attr: getattr(self, attr) for attr in LanguageModel.JSON_ATTRS}

    def save_to_dir(self, filepath: str, unigram_encoding: Optional[str] = None) -> None:
        src = self._kenlm_model.path.decode("utf-8")
        with open(os.path.join(filepath, self._ATTRS_SERIALIZED_FILENAME), "w") as fh:
            json.dump(self.serializable_attrs, fh)
        with open(os.path.join(filepath, self._UNIGRAMS_SERIALIZED_FILENAME), "w", encoding=unigram_encoding) as fh:
            for unigram in sorted(self._unigram_set):
                fh.write(unigram + "\n")
        shutil.copy2(src, os.path.join(filepath, os.path.split(src)[1]))

    @staticmethod
    def parse_directory_contents(filepath: str) -> Dict[str, str]:
        contents = [c for c in os.listdir(filepath) if not c.startswith(".") and not c.startswith("__")]
        if len(contents) != 3:
            raise ValueError("Found wrong number of files in directory. Expected 3 files, found %s" % contents)
        for needed in (LanguageModel._ATTRS_SERIALIZED_FILENAME, LanguageModel._UNIGRAMS_SERIALIZED_FILENAME):
            if needed not in contents:
                raise ValueError("did not find %s in files: %s" % (needed, contents))
            contents.remove(needed)
        if os.path.splitext(contents[0])[1] not in {".arpa", ".bin", ".binary", NgramModel.BLOB_SUFFIX}:
            raise ValueError("Explected kenlm file to end in `.arpa` or `.bin(ary)`. Found %s" % contents[0])
        return {
            "json_attrs": os.path.join(filepath, LanguageModel._ATTRS_SERIALIZED_FILENAME),
            "unigrams": os.path.join(filepath, LanguageModel._UNIGRAMS_SERIALIZED_FILENAME),
            "kenlm": os.path.join(filepath, contents[0]),
        }

    @classmethod
    def load_from_dir(cls, filepath: str, unigram_encoding: Optional[str] = None) -> "LanguageModel":
        names = cls.parse_directory_contents(filepath)
        with open(names["json_attrs"]) as fh:
            attrs = json.load(fh)
        if set(attrs.keys()) != set(cls.JSON_ATTRS):
            raise ValueError("Expected json serialized attributes to be %s but found %s" % (cls.JSON_ATTRS, attrs.keys()))
        with open(names["unigrams"], encoding=unigram_encoding) as fh:
            unigrams = fh.read().splitlines()
        if names["kenlm"].endswith(NgramModel.BLOB_SUFFIX):
            # a flattened model: its unigram / prefix sets are inside the blob (unigrams.txt is empty for it)
            return cls(NgramModel.load_blob(names["kenlm"]), unigrams or None, **attrs)
        return cls(NgramModel(names["kenlm"]), unigrams, **attrs)


class MultiLanguageModelState(AbstractLMState):
    """reference language_model.py:56-64"""

    def __init__(self, states: Sequence[AbstractLMState]) -> None:
        self._states = states

    @property
    def states(self) -> Sequence[AbstractLMState]:
        return self._states

    def get_mp_safe_state(self) -> "MultiLanguageModelState":
        return self


class MultiLanguageModel(AbstractLanguageModel):
    """Mean of several language models (reference language_model.py:455-502).  On the device every model keeps
    its own tables, vocabulary, unigram set and alpha / beta / unk offset / boundary flag; a word's score is the
    sum of the models' scores divided by their number, the state is the list of the models' states
    (csrc/b2c_beam.h b2c_text_extend).  At most 4 models."""

    def __init__(self, language_models: Sequence[AbstractLanguageModel]) -> None:
        if len(language_models) < 2:
            raise ValueError("This class is meant to contain at least 2 language models.")
        self._language_models = language_models

    @property
    def language_models(self) -> Sequence[AbstractLanguageModel]:
        return self._language_models

    @property
    def order(self) -> int:
        return max(lm.order for lm in self._language_models)

    def get_start_state(self) -> MultiLanguageModelState:
        return MultiLanguageModelState([lm.get_start_state() for lm in self._language_models])

    def score_partial_token(self, partial_token: str) -> float:
        return float(sum(lm.score_partial_token(partial_token) for lm in self._language_models) / len(self._language_models))

    def score(self, prev_state: AbstractLMState, word: str, is_last_word: bool = False) -> Tuple[float, MultiLanguageModelState]:
        if not isinstance(prev_state, MultiLanguageModelState):
            raise AssertionError("Wrong input state type found. Expected MultiLanguageModelState, got %s" % type(prev_state))
        if len(prev_state.states) != len(self._language_models):
            raise AssertionError("Number of states (%d) does not match number of language models (%d)."
                                 % (len(prev_state.states), len(self._language_models)))
        score = 0.0
        end_state = []
        for lm_prev_state, lm in zip(prev_state.states, self._language_models):
            lm_score, lm_end_state = lm.score(lm_prev_state, word, is_last_word=is_last_word)
            score += lm_score
            end_state.append(lm_end_state)
        return score / len(self._language_models), MultiLanguageModelState(end_state)
