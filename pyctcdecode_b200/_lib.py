"""ctypes binding of libb200ctc.so (C ABI declared in include/b200ctc.h).

The shared library is built in-tree by ``__graft_entry__.build()`` (nvcc, sm_90a).  There is
no CPU implementation: if the library is missing, or the machine has no CUDA device, every
decode call raises -- loudly, by design.
"""
import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_LIBRARY = os.path.join(_HERE, "libb200ctc.so")

_lock = threading.Lock()
_lib = None
_lib_path = None


class LMState(C.Structure):
    _fields_ = [("words", C.c_uint32 * 5), ("backoff", C.c_float * 5), ("length", C.c_uint32)]


class StreamBeam(C.Structure):
    _fields_ = [("part_hash", C.c_uint64), ("logit_score", C.c_double), ("word_off", C.c_uint32), ("n_words", C.c_uint32),
                ("part_len", C.c_uint32), ("last_tok", C.c_uint32), ("pf_s", C.c_int32), ("pf_e", C.c_int32)]


class StreamState(C.Structure):
    _fields_ = [("beams", C.POINTER(StreamBeam)), ("n_beams", C.c_int), ("processed_frames", C.c_int),
                ("word_hashes", C.POINTER(C.c_uint64)), ("word_lens", C.POINTER(C.c_uint32)), ("n_words", C.c_int)]


FIN_EOS, FIN_FLUSH, FIN_KEEP = 0, 1, 2


class HotwordSet(C.Structure):
    _fields_ = [("hotwords", C.POINTER(C.c_char_p)), ("n_hotwords", C.c_int), ("hotword_weight", C.c_double)]


class LmSet(C.Structure):
    _fields_ = [("n_models", C.c_int), ("models", C.c_void_p * 4), ("alpha", C.c_double * 4), ("beta", C.c_double * 4),
                ("unk_score_offset", C.c_double * 4), ("lm_score_boundary", C.c_int * 4)]


class DecodeOpts(C.Structure):
    _fields_ = [
        ("beam_width", C.c_int),
        ("beam_prune_logp", C.c_double),
        ("token_min_logp", C.c_double),
        ("prune_history", C.c_int),
        ("hotwords", C.POINTER(C.c_char_p)),
        ("n_hotwords", C.c_int),
        ("hotword_weight", C.c_double),
        ("max_out_beams", C.c_int),
        ("lm_start_states", C.POINTER(LMState)),
        ("stream_states", C.POINTER(StreamState)),
        ("finalize_mode", C.c_int),
        ("text_only", C.c_int),
        ("hot_sets", C.POINTER(HotwordSet)),
        ("n_hot_sets", C.c_int),
        ("utt_hot_set", C.POINTER(C.c_int32)),
        ("lm_sets", C.POINTER(LmSet)),
        ("n_lm_sets", C.c_int),
        ("utt_lm_set", C.POINTER(C.c_int32)),
        ("lm_start_width", C.c_int),
        ("utt_finalize_mode", C.POINTER(C.c_int32)),
        ("utt_beam_width", C.POINTER(C.c_int32)),
        ("utt_beam_prune_logp", C.POINTER(C.c_double)),
        ("utt_token_min_logp", C.POINTER(C.c_double)),
        ("utt_prune_history", C.POINTER(C.c_int32)),
    ]


class Packed(C.Structure):
    _fields_ = [("n_utts", C.c_int32), ("n_models", C.c_int32), ("n_beams_total", C.c_int64), ("n_words_total", C.c_int64),
                ("n_beams", C.POINTER(C.c_int32)), ("scores", C.POINTER(C.c_double)), ("n_words", C.POINTER(C.c_int32)),
                ("frames", C.POINTER(C.c_int32)), ("texts", C.c_void_p), ("texts_size", C.c_size_t),
                ("states", C.POINTER(LMState)), ("stream_aux", C.POINTER(C.c_int32)), ("n_stream_toks", C.POINTER(C.c_int32)),
                ("stream_toks", C.POINTER(C.c_uint32)), ("n_stream_toks_total", C.c_int64),
                ("stream_pieces", C.c_void_p), ("stream_pieces_size", C.c_size_t), ("stream_boundary", C.POINTER(C.c_int32))]


class Timings(C.Structure):
    _fields_ = [
        ("ms_prepare", C.c_float),
        ("ms_beam", C.c_float),
        ("ms_total", C.c_float),
        ("launches", C.c_int),
        ("h2d_bytes", C.c_longlong),
        ("d2h_bytes", C.c_longlong),
        ("frames", C.c_longlong),
        ("tokens", C.c_longlong),
        ("cap_candidates", C.c_int),
        ("cta_threads", C.c_int),
        ("cta_slots", C.c_int),
        ("oversize_frames", C.c_longlong),
        ("kernel_variant", C.c_int),
        ("cand_hist", C.c_longlong * 7),
        ("inplace_frames", C.c_longlong),
        ("sorted_frames", C.c_longlong),
        ("single_frames", C.c_longlong),
        ("hinted", C.c_int),
        ("kernels", C.c_int),
        ("retried", C.c_int),
    ]


def _declare(L):
    vp, cp, i32, f64 = C.c_void_p, C.c_char_p, C.c_int, C.c_double
    pp = C.POINTER(vp)
    L.b2c_last_error.restype = cp
    L.b2c_version.restype = i32
    L.b2c_device_count.restype = i32
    L.b2c_lm_build_from_arpa.argtypes = [cp, C.POINTER(cp), C.c_long, pp]
    L.b2c_lm_build_from_file.argtypes = [cp, C.POINTER(cp), C.c_long, pp]
    L.b2c_lm_blob.argtypes = [vp, pp, C.POINTER(C.c_size_t)]
    L.b2c_lm_from_blob.argtypes = [vp, C.c_size_t, pp]
    L.b2c_lm_upload.argtypes = [vp, i32]
    L.b2c_lm_adopt_device_blob.argtypes = [vp, i32, vp, C.c_size_t]
    L.b2c_lm_destroy.argtypes = [vp]
    L.b2c_lm_destroy.restype = None
    L.b2c_lm_order.argtypes = [vp]
    L.b2c_lm_contains.argtypes = [vp, cp]
    L.b2c_lm_in_unigrams.argtypes = [vp, cp]
    L.b2c_lm_has_prefix.argtypes = [vp, cp]
    L.b2c_lm_have_unigrams.argtypes = [vp]
    L.b2c_lm_begin_sentence.argtypes = [vp, C.POINTER(LMState)]
    L.b2c_lm_begin_sentence.restype = None
    L.b2c_lm_null_context.argtypes = [vp, C.POINTER(LMState)]
    L.b2c_lm_null_context.restype = None
    L.b2c_lm_base_score.argtypes = [vp, C.POINTER(LMState), cp, C.POINTER(LMState)]
    L.b2c_lm_base_score.restype = C.c_float
    L.b2c_decoder_create.argtypes = [C.POINTER(cp), i32, i32, vp, i32, pp]
    L.b2c_decoder_destroy.argtypes = [vp]
    L.b2c_decoder_destroy.restype = None
    L.b2c_decoder_set_params.argtypes = [vp, f64, f64, f64, i32]
    L.b2c_decoder_device.argtypes = [vp]
    L.b2c_decoder_wait_stream.argtypes = [vp, vp]
    L.b2c_decode_opts_default.argtypes = [C.POINTER(DecodeOpts)]
    L.b2c_decode_opts_default.restype = None
    L.b2c_decode_batch.argtypes = [vp, C.POINTER(vp), C.POINTER(C.c_int32), i32, i32, i32, C.POINTER(DecodeOpts), pp]
    L.b2c_result_free.argtypes = [vp]
    L.b2c_result_free.restype = None
    L.b2c_result_n_utts.argtypes = [vp]
    L.b2c_result_n_beams.argtypes = [vp, i32]
    L.b2c_result_text.argtypes = [vp, i32, i32]
    L.b2c_result_text.restype = cp
    L.b2c_result_top_texts.argtypes = [vp, C.POINTER(vp), C.POINTER(C.c_size_t)]
    L.b2c_result_logit_score.argtypes = [vp, i32, i32]
    L.b2c_result_logit_score.restype = f64
    L.b2c_result_lm_score.argtypes = [vp, i32, i32]
    L.b2c_result_lm_score.restype = f64
    L.b2c_result_n_words.argtypes = [vp, i32, i32]
    L.b2c_result_word.argtypes = [vp, i32, i32, i32]
    L.b2c_result_word.restype = cp
    L.b2c_result_packed.argtypes = [vp, C.POINTER(Packed)]
    L.b2c_hash_utf8_batch.argtypes = [C.c_char_p, C.c_size_t, C.c_int64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
    L.b2c_result_frames.argtypes = [vp, i32, i32]
    L.b2c_result_frames.restype = C.POINTER(C.c_int32)
    L.b2c_result_lm_state.argtypes = [vp, i32, i32, C.POINTER(LMState)]
    L.b2c_decoder_last_timings.argtypes = [vp, C.POINTER(Timings)]
    L.b2c_decoder_last_tokens.argtypes = [vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64), vp, vp, vp, vp, vp, vp]
    L.b2c_decoder_add_lm.argtypes = [vp, vp]
    L.b2c_decoder_set_params_lm.argtypes = [vp, i32, f64, f64, f64, i32]
    L.b2c_result_lm_state_at.argtypes = [vp, i32, i32, i32, C.POINTER(LMState)]
    L.b2c_result_stream_beam.argtypes = [vp, i32, i32, C.POINTER(C.c_int32 * 4), C.POINTER(C.POINTER(C.c_uint32)), C.POINTER(i32)]
    L.b2c_result_n_frames.argtypes = [vp, i32, i32]
    L.b2c_hash_utf8.argtypes = [cp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
    L.b2c_decoder_token_id.argtypes = [vp, cp]
    return L


def use_library(path):
    """Bind a specific build of the C ABI.  Used by the CPU-only logic tests to point the host
    code at tests/hostsim's simulation build; product code never calls this."""
    global _lib, _lib_path
    with _lock:
        _lib = _declare(C.CDLL(path))
        _lib_path = path
    return _lib


def lib():
    global _lib, _lib_path
    if _lib is None:
        with _lock:
            if _lib is None:
                if not os.path.exists(DEFAULT_LIBRARY):
                    raise RuntimeError(
                        "libb200ctc.so is not built (%s). Run `python -c 'import __graft_entry__ as g; g.build()'`; "
                        "pyctcdecode_b200 has no CPU fallback." % DEFAULT_LIBRARY)
                _lib = _declare(C.CDLL(DEFAULT_LIBRARY))
                _lib_path = DEFAULT_LIBRARY
    return _lib


def library_path():
    return _lib_path


class B200Error(RuntimeError):
    pass


def check(rc):
    """Map C return codes to the exceptions the reference raises (ValueError for bad input)."""
    if rc == 0:
        return
    msg = lib().b2c_last_error().decode("utf-8", "replace")
    if rc == -1:
        raise ValueError(msg)
    if rc == -3:
        raise OSError(msg)
    if rc == -4:
        raise MemoryError(msg)
    raise B200Error("libb200ctc error %d: %s" % (rc, msg))


def cstr_array(strings):
    arr = (C.c_char_p * max(1, len(strings)))()
    for i, s in enumerate(strings):
        arr[i] = s.encode("utf-8")
    return arr
