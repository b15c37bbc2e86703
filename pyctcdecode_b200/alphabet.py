"""Label normalisation for the CUDA decoder.

Host-side, O(V), build time only -- but it decides which token is the CTC blank, which one
separates words and whether the alphabet is BPE, i.e. what the kernels are specialised on, so
the behaviour follows reference pyctcdecode/alphabet.py:22-170 case by case (checked against
the reference's outputs in tests/test_alphabet.py).
"""
import json
import logging
import re
from typing import Collection, List

BPE_TOKEN = "▁"
UNK_TOKEN = "⁇"
UNK_BPE_TOKEN = BPE_TOKEN + UNK_TOKEN + BPE_TOKEN

_SPECIAL = re.compile(r"^[<\[].+[>\]]$")
_BLANK = re.compile(r"^[<\[]pad[>\]]$", flags=re.IGNORECASE)
_UNK = re.compile(r"^[<\[]unk[>\]]$", flags=re.IGNORECASE)

logger = logging.getLogger(__name__)


def _looks_like_bpe(labels: List[str]) -> bool:
    """reference alphabet.py:22-31"""
    return any(s.startswith("##") for s in labels) or any(s.startswith(BPE_TOKEN) for s in labels)


def _to_sentencepiece_style(token: str) -> str:
    """'##x' word-piece style -> U+2581 style (reference alphabet.py:76-85)."""
    if token.startswith("##"):
        return token[2:]
    if _SPECIAL.match(token) or token in ("", BPE_TOKEN, UNK_BPE_TOKEN, "<unk>"):
        return token
    return BPE_TOKEN + token


def _substitute(labels: List[str], pattern, replacement: str) -> List[str]:
    return [replacement if pattern.match(tok) else tok for tok in labels]


def _normalize_char_labels(labels: List[str]) -> List[str]:
    """reference alphabet.py:34-73"""
    out = list(labels)
    if "|" in out and " " not in out:
        out[out.index("|")] = " "
    out = _substitute(out, _BLANK, "")
    if "_" in out and "" not in out:
        out[out.index("_")] = ""
    if "" not in out:
        out.append("")
    out = _substitute(out, _UNK, UNK_TOKEN)
    if any(len(c) > 1 for c in out):
        logger.warning("Labels longer than one character in a non-BPE alphabet -- is this intended?")
    if " " not in out:
        logger.warning("Space token ' ' missing from vocabulary.")
    return out


def _normalize_bpe_labels(labels: List[str]) -> List[str]:
    """reference alphabet.py:88-110"""
    out = list(labels)
    if any(s.startswith("##") for s in labels):
        out = [_to_sentencepiece_style(tok) for tok in out]
    out = _substitute(out, _BLANK, "")
    if "" not in out:
        out.append("")
    out = _substitute(out, _UNK, UNK_BPE_TOKEN)
    if UNK_BPE_TOKEN not in out:
        logger.warning("UNK token %s not found, is this a mistake?", UNK_BPE_TOKEN)
    return out


class Alphabet:
    def __init__(self, labels: List[str], is_bpe: bool) -> None:
        self._labels = labels
        self._is_bpe = is_bpe

    @property
    def is_bpe(self) -> bool:
        return self._is_bpe

    @property
    def labels(self) -> List[str]:
        return self._labels[:]

    @classmethod
    def build_alphabet(cls, labels: List[str]) -> "Alphabet":
        """reference alphabet.py:139-148 (incl. the checks of _verify_alphabet :113-120)."""
        is_bpe = _looks_like_bpe(labels)
        if len(labels) != len(set(labels)):
            raise ValueError("Alphabet contains duplicate entries, this is not allowed.")
        if is_bpe and any(" " in s for s in labels):
            raise ValueError("Space token ' ' found in vocabulary even though it looks like BPE.")
        normalized = _normalize_bpe_labels(labels) if is_bpe else _normalize_char_labels(labels)
        return cls(normalized, is_bpe)

    def dumps(self) -> str:
        return json.dumps({"labels": self.labels, "is_bpe": self.is_bpe})

    @classmethod
    def loads(cls, s: str) -> "Alphabet":
        d = json.loads(s)
        if set(d.keys()) != {"is_bpe", "labels"}:
            raise ValueError("unexpected keys found. Expected {'is_bpe', 'labels'}, found %s" % set(d.keys()))
        return cls(d["labels"], d["is_bpe"])


def verify_alphabet_coverage(alphabet: Alphabet, unigrams: Collection[str]) -> None:
    """reference alphabet.py:165-170"""
    label_chars = set(alphabet.labels)
    unigram_chars = set("".join(unigrams))
    if len(unigram_chars - label_chars) / len(unigram_chars) > 0.2:
        logger.warning("Unigrams and labels don't seem to agree.")
