"""pyctcdecode_b200 -- CUDA-native (H100) CTC prefix beam-search decoder with the pyctcdecode API.

    from pyctcdecode_b200 import build_ctcdecoder
    decoder = build_ctcdecoder(labels, kenlm_model_path="lm.arpa", alpha=0.5, beta=1.0)
    texts = decoder.decode_batch(None, logits_list, beam_width=100)

The per-frame beam update runs in hand-written sm_90a CUDA kernels behind a C ABI
(include/b200ctc.h, pyctcdecode_b200/libb200ctc.so).  There is no CPU fallback.
"""
from .alphabet import Alphabet  # noqa: F401
from .decoder import Beam, BeamSearchDecoderCTC, LMBeam, OutputBeam, build_ctcdecoder  # noqa: F401
from .language_model import HotwordScorer, LanguageModel, MultiLanguageModel, MultiLanguageModelState, NgramModel  # noqa: F401

__version__ = "0.2.0"


def install_alias(name: str = "pyctcdecode") -> None:
    """Make ``import pyctcdecode`` (and ``pyctcdecode.decoder`` / ``.language_model`` / ``.alphabet`` / ``.constants``)
    resolve to this package, so that code written against the reference -- ``from pyctcdecode import
    build_ctcdecoder, BeamSearchDecoderCTC, Alphabet, LanguageModel`` (reference __init__.py:2-4), or
    transformers' Wav2Vec2ProcessorWithLM -- runs on the CUDA decoder without an edit.  Opt-in and explicit: nothing
    is aliased at import time (the real reference must stay importable where it is installed, e.g. for the golden
    vector generators under oracle/).  Raises if a different ``pyctcdecode`` is already imported."""
    import sys

    from . import alphabet, constants, decoder, language_model

    this = sys.modules[__name__]
    have = sys.modules.get(name)
    if have is not None and have is not this:
        raise ImportError("%r is already imported from %s; call install_alias() before anything imports it"
                          % (name, getattr(have, "__file__", "?")))
    sys.modules[name] = this
    for sub, mod in (("alphabet", alphabet), ("constants", constants), ("decoder", decoder), ("language_model", language_model)):
        sys.modules["%s.%s" % (name, sub)] = mod
