/* b200ctc.h -- C ABI of libb200ctc.so, the CUDA-native (H100, sm_90a) CTC prefix beam-search decoder.
 *
 * The reference (kensho-technologies/pyctcdecode 0.6.0) has no FFI: its "plugin API" for
 * this path is the Python class BeamSearchDecoderCTC.  This header is the boundary a
 * maintainer of the reference would bind with ctypes/cffi to replace the body of
 * decode()/decode_batch()/decode_beams()/decode_beams_batch() -- see INTEGRATION.md.
 * Each entry point cites the reference interface it replaces (paths relative to
 * /root/reference/pyctcdecode/).
 *
 * Conventions: plain pointers and sizes only; every function returns 0 on success or a
 * negative B2C_E_* code (b2c_last_error() gives the message for the calling thread); the
 * library owns every object it returns until the matching *_free/_destroy; inputs stay
 * caller-owned and are never modified (reference decoder.py:762-765 allocates instead of
 * mutating); calls are synchronous and use the decoder's own CUDA stream; any number of threads
 * may call b2c_decode_batch on one handle -- the calls are serialised by a mutex inside the handle
 * (results are independent objects).  Parameter setters (b2c_decoder_set_params*) are plain stores:
 * a caller that changes parameters between calls from several threads serialises setter + decode
 * itself (the Python layer does).  Device-resident logits written on another stream than the
 * legacy default stream: call b2c_decoder_wait_stream first.  There is no CPU fallback: without a
 * CUDA device b2c_decoder_create fails with B2C_E_CUDA.
 */
#ifndef B200CTC_H
#define B200CTC_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2C_E_OK 0
#define B2C_E_ARG (-1)      /* bad argument (python side raises ValueError, like decoder.py:335-344) */
#define B2C_E_CUDA (-2)     /* CUDA runtime failure / no device */
#define B2C_E_IO (-3)       /* cannot read the ARPA file */
#define B2C_E_NOMEM (-4)
#define B2C_E_INTERNAL (-5)

#define B2C_DTYPE_F32 0
#define B2C_DTYPE_F64 1
#define B2C_DTYPE_F16 2     /* IEEE half: copied as 2-byte elements, widened to float32 on the device (exact) */
#define B2C_DTYPE_BF16 3    /* bfloat16: likewise */

typedef struct b2c_lm b2c_lm_t;            /* flattened n-gram model (host blob + device copies) */
typedef struct b2c_decoder b2c_decoder_t;  /* one decoder bound to one CUDA device */
typedef struct b2c_result b2c_result_t;    /* results of one decode_batch call */

const char* b2c_last_error(void);
int b2c_version(void);
/* number of visible CUDA devices (0 when there is none) */
int b2c_device_count(void);

/* ---- n-gram model ------------------------------------------------------------------------
 * Replaces kenlm.Model(kenlm_model_path) + _prepare_unigram_set + CharTrie.fromkeys
 * (decoder.py:1074-1096, language_model.py:87-103, :237-269).  `unigrams` NULL or
 * n_unigrams < 0 means "no unigram list" (LanguageModel(unigrams=None)). */
int b2c_lm_build_from_arpa(const char* arpa_path, const char* const* unigrams, long n_unigrams, b2c_lm_t** out);
/* the same from whatever kenlm.Model(path) accepts (decoder.py:1074, language_model.py:422-426): ARPA text, or a KenLM
 * BINARY file of the probing model type (what kenlm's build_binary writes by default) -- told apart by the first
 * bytes.  Trie / quantised binaries are rejected with a message (B2C_E_IO). */
int b2c_lm_build_from_file(const char* path, const char* const* unigrams, long n_unigrams, b2c_lm_t** out);
/* the relocatable blob (for a NCCL broadcast) and its reconstruction on another rank; from_blob validates every
 * offset, mask and id of the header against `size` before use */
int b2c_lm_blob(const b2c_lm_t* lm, const void** data, size_t* size);
int b2c_lm_from_blob(const void* data, size_t size, b2c_lm_t** out);
/* make the model resident on `device` by cudaMemcpy, or adopt a device copy that already
 * exists (e.g. the torch tensor an NCCL broadcast wrote); adopted memory stays caller-owned */
int b2c_lm_upload(b2c_lm_t* lm, int device);
int b2c_lm_adopt_device_blob(b2c_lm_t* lm, int device, const void* device_ptr, size_t size);
void b2c_lm_destroy(b2c_lm_t* lm);
/* kenlm.Model look-alike queries, evaluated on the host copy of the tables
 * (language_model.py:95,306,312-314,347,352) */
int b2c_lm_order(const b2c_lm_t* lm);
int b2c_lm_contains(const b2c_lm_t* lm, const char* word);
int b2c_lm_in_unigrams(const b2c_lm_t* lm, const char* word);
int b2c_lm_has_prefix(const b2c_lm_t* lm, const char* prefix);
/* 1 when the model was built with a unigram list (LanguageModel(unigrams=...) not None) */
int b2c_lm_have_unigrams(const b2c_lm_t* lm);
/* state: `words` most recent first; BaseScore writes the out state and returns log10 p */
typedef struct { uint32_t words[5]; float backoff[5]; uint32_t length; } b2c_lm_state_t;
void b2c_lm_begin_sentence(const b2c_lm_t* lm, b2c_lm_state_t* st);
void b2c_lm_null_context(const b2c_lm_t* lm, b2c_lm_state_t* st);
float b2c_lm_base_score(const b2c_lm_t* lm, const b2c_lm_state_t* in, const char* word, b2c_lm_state_t* out);

/* ---- decoder -----------------------------------------------------------------------------
 * Replaces BeamSearchDecoderCTC.__init__ (decoder.py:275-290).  `labels` are the NORMALISED
 * labels (Alphabet.labels, alphabet.py:139-148): "" is the CTC blank, " " the word separator
 * of a regular alphabet, U+2581-prefixed pieces start a word in a BPE alphabet.
 * `lm` may be NULL.  The decoder keeps a reference to `lm` (destroy the decoder first). */
int b2c_decoder_create(const char* const* labels, int n_labels, int is_bpe, b2c_lm_t* lm, int device,
                       b2c_decoder_t** out);
void b2c_decoder_destroy(b2c_decoder_t* dec);
/* the CUDA device the decoder was created on */
int b2c_decoder_device(const b2c_decoder_t* dec);
/* order the next decode call after everything `cuda_stream` (a cudaStream_t, e.g. torch's current stream) holds now:
 * needed when device-resident logits were produced on a stream other than the legacy default stream */
int b2c_decoder_wait_stream(b2c_decoder_t* dec, void* cuda_stream);
/* LanguageModel.reset_params (language_model.py:271-301): plain scalars handed to the kernels */
int b2c_decoder_set_params(b2c_decoder_t* dec, double alpha, double beta, double unk_score_offset,
                           int lm_score_boundary);

#define B2C_FIN_EOS 0
#define B2C_FIN_FLUSH 1
#define B2C_FIN_KEEP 2
/* One input beam of a streaming call, string-free (reference Beam, decoder.py:69-94): the finished words of
 * `text` as (hash, code points) pairs from b2c_hash_utf8, the partial word likewise, last_char as a token id. */
typedef struct {
    uint64_t part_hash;        /* b2c_hash_utf8(partial_word) */
    double logit_score;
    uint32_t word_off, n_words;/* words of `text`: word_hashes / word_lens [word_off, word_off + n_words) of the state */
    uint32_t part_len;         /* code points of partial_word */
    uint32_t last_tok;         /* b2c_decoder_token_id(last_char); 0xFFFF for None */
    int32_t pf_s, pf_e;        /* partial_frames */
} b2c_stream_beam_t;
typedef struct b2c_stream_state {
    const b2c_stream_beam_t* beams;   /* in the order the previous call returned them */
    int n_beams;
    int processed_frames;             /* frame index of the first row of this call's logits */
    const uint64_t* word_hashes;
    const uint32_t* word_lens;
    int n_words;
} b2c_stream_state_t;

/* MultiLanguageModel (language_model.py:455-502, the mean of >= 2 models): the decoder is created with model 0,
 * further models (at most 4 in total) are added here; every model keeps its own alpha / beta / unk offset /
 * boundary flag (index 0 = the model given to b2c_decoder_create).  With more than one model
 * opts->lm_start_states holds n_models consecutive states per utterance and b2c_result_lm_state_at returns the
 * state of each model (MultiLanguageModelState.states). */
int b2c_decoder_add_lm(b2c_decoder_t* dec, b2c_lm_t* lm);
int b2c_decoder_set_params_lm(b2c_decoder_t* dec, int lm_index, double alpha, double beta, double unk_score_offset,
                              int lm_score_boundary);

/* One hotword set (HotwordScorer, language_model.py:152-189): what opts->hotwords / hotword_weight give a whole call. */
typedef struct {
    const char* const* hotwords; /* raw hotword strings, split on whitespace */
    int n_hotwords;
    double hotword_weight;
} b2c_hotword_set_t;

/* One language-model set: no model (n_models == 0), a LanguageModel (1) or a MultiLanguageModel of 2..4 models, each
 * with its own alpha / beta / unk offset / boundary flag, as b2c_decoder_set_params_lm gives a decoder's own models. */
typedef struct b2c_lm_set {
    int n_models;
    b2c_lm_t* models[4];
    double alpha[4], beta[4], unk_score_offset[4];
    int lm_score_boundary[4];
} b2c_lm_set_t;

typedef struct {
    int beam_width;            /* DEFAULT_BEAM_WIDTH 100          (constants.py:8)  */
    double beam_prune_logp;    /* DEFAULT_PRUNE_LOGP -10          (constants.py:10) */
    double token_min_logp;     /* DEFAULT_MIN_TOKEN_LOGP -5       (constants.py:12) */
    int prune_history;         /* decode(): 1 (decoder.py:888); decode_beams(): 0  */
    const char* const* hotwords; /* raw hotword strings, split on whitespace like language_model.py:160-166 */
    int n_hotwords;
    double hotword_weight;     /* DEFAULT_HOTWORD_WEIGHT 10       (constants.py:9)  */
    int max_out_beams;         /* 1 for decode()/decode_batch(); beam_width for decode_beams*() */
    /* NULL, or the start states (lm_start_state, decoder.py:612-625): n_utts rows of W states, W = the number of models
     * of the call's largest set (the decoder's own models without utt_lm_set; at least 1).  Utterance i uses the first
     * n_models entries of its row, one per model of its own set in set order; the rest of the row, and the whole row of
     * an utterance without a model, is not read.  Every state that is read is checked on the host before anything is
     * enqueued: B2C_E_ARG for a length above 5 or for a word id among the first `length` that is not below its model's
     * vocabulary size.  A state of another model whose ids all lie inside the vocabulary cannot be told apart. */
    const b2c_lm_state_t* lm_start_states;
    /* streaming (partial_decode_beams, decoder.py:669-728): NULL, or one state per utterance = the beams the call
     * starts from (NULL beams / n_beams == 0: EMPTY_START_BEAM) and processed_frames */
    const struct b2c_stream_state* stream_states;
    int finalize_mode;         /* B2C_FIN_EOS (default): decode_beams / is_end=True; B2C_FIN_FLUSH: force_next_word=True,
                                  is_end=False; B2C_FIN_KEEP: neither -- beams keep their partial words (decoder.py:571-593) */
    int text_only;             /* decode() / decode_batch() (decoder.py:859-945 return beam.text only): word frames are
                                  neither copied back nor assembled; b2c_result_n_words is 0 */
    /* per-utterance hotwords: utterance i is decoded exactly as a call of its own with hotwords / hotword_weight of
     * hot_sets[utt_hot_set[i]].  utt_hot_set NULL: every utterance uses hotwords / hotword_weight above and hot_sets is
     * not read.  B2C_E_ARG: an index outside [0, n_hot_sets), or n_hotwords > 0 together with utt_hot_set.  Utterances
     * that share an index share one table on the device. */
    const b2c_hotword_set_t* hot_sets;
    int n_hot_sets;
    const int32_t* utt_hot_set; /* NULL, or [n_utts] indices into hot_sets */
    /* per-utterance language models: utterance i is decoded exactly as a call of its own on a decoder created with the
     * models of lm_sets[utt_lm_set[i]] (and their parameters).  utt_lm_set NULL: every utterance uses the decoder's
     * own model(s) and lm_sets is not read.  Models are uploaded to the decoder's device on first use.  B2C_E_ARG: an
     * index outside [0, n_lm_sets), or a set with a NULL model or with n_models outside [0, 4].  Composes with
     * lm_start_states (layout above; lm_start_width must state W) and with stream_states: a streaming utterance starts
     * from its row of lm_start_states, which a streaming call with utt_lm_set must give (B2C_E_ARG without it), and
     * replays the words of its input beams through its own set.  Streaming calls and calls with a set of more
     * than one model run on the general kernel.  Results: b2c_result_lm_state(_at) return the states of the utterance's
     * own set (0 for an utterance without a model); in b2c_packed_t n_models is the largest set of the call, and a
     * beam of a smaller set has its models' states first, then zeroed states (length 0). */
    const struct b2c_lm_set* lm_sets;
    int n_lm_sets;
    const int32_t* utt_lm_set; /* NULL, or [n_utts] indices into lm_sets */
    /* W of the lm_start_states layout, stated by the caller when utt_lm_set is given together with lm_start_states: it
     * must equal the number of models of the call's largest set (at least 1), else B2C_E_ARG (the library cannot see
     * the extent of the array).  Not read without utt_lm_set. */
    int lm_start_width;
    /* per-utterance finalize modes: NULL, or [n_utts] B2C_FIN_* values; utterance i then ends its call as a call of its
     * own with finalize_mode = utt_finalize_mode[i] (batched streaming where some streams end, some flush their partial
     * words and the rest keep them), and finalize_mode is not read.  B2C_E_ARG: a value outside [B2C_FIN_EOS,
     * B2C_FIN_KEEP], or finalize_mode != B2C_FIN_EOS together with utt_finalize_mode.  The call is a streaming call
     * when stream_states is given or some utterance's mode is not B2C_FIN_EOS. */
    const int32_t* utt_finalize_mode;
    /* per-utterance search parameters: each NULL, or [n_utts] values; a given array replaces its scalar field
     * (beam_width, beam_prune_logp, token_min_logp, prune_history) for every utterance, which is then decoded exactly
     * as a call of its own with those values (batched streaming where streams run at different widths or thresholds),
     * and returns at most min(max_out_beams, utt_beam_width[i]) beams.  Accepted only together with stream_states (they
     * run on the general kernel), else B2C_E_ARG; B2C_E_ARG also for a width outside [1, 65535].  Both checks run
     * before anything is enqueued.  The beam tables, candidate tiers, history-prune tables and arenas are sized by the
     * call's largest width, and the shared-memory limit is checked against it. */
    const int32_t* utt_beam_width;
    const double* utt_beam_prune_logp;
    const double* utt_token_min_logp;
    const int32_t* utt_prune_history;
} b2c_decode_opts_t;
void b2c_decode_opts_default(b2c_decode_opts_t* opts);

/* Replaces decode_batch / decode_beams_batch (decoder.py:801-857, :895-945) and, with
 * n_utts == 1, decode / decode_beams (:730-775, :859-893).
 *   logits[i]  -> C-contiguous [T[i], V] matrix of dtype (B2C_DTYPE_*; half types are computed as float32), host pointers when
 *                 is_device == 0 (copied host->device inside the call), device pointers on the
 *                 decoder's device when is_device != 0 (used in place when contiguous);
 *   ragged T and T == 0 are allowed.                                                      */
int b2c_decode_batch(b2c_decoder_t* dec, const void* const* logits, const int32_t* T, int n_utts, int dtype,
                     int is_device, const b2c_decode_opts_t* opts, b2c_result_t** out);

/* ---- results (OutputBeam, decoder.py:102-118, built at :653-667) ------------------------- */
void b2c_result_free(b2c_result_t* res);
int b2c_result_n_utts(const b2c_result_t* res);
int b2c_result_n_beams(const b2c_result_t* res, int utt);
const char* b2c_result_text(const b2c_result_t* res, int utt, int beam);          /* utf-8 */
/* top-1 text of every utterance in one buffer, each text followed by a NUL byte (one call instead of
 * n_utts; what decode_batch needs); the buffer lives as long as the result */
int b2c_result_top_texts(b2c_result_t* res, const char** data, size_t* size);
double b2c_result_logit_score(const b2c_result_t* res, int utt, int beam);
double b2c_result_lm_score(const b2c_result_t* res, int utt, int beam);
int b2c_result_n_words(const b2c_result_t* res, int utt, int beam);
const char* b2c_result_word(const b2c_result_t* res, int utt, int beam, int word);
/* 2 * n_words ints: (start_frame, end_frame) per word */
const int32_t* b2c_result_frames(const b2c_result_t* res, int utt, int beam);
/* LM state after the last word (OutputBeam.last_lm_state); returns 0 when there is no LM */
int b2c_result_lm_state(const b2c_result_t* res, int utt, int beam, b2c_lm_state_t* out);
int b2c_result_lm_state_at(const b2c_result_t* res, int utt, int beam, int lm_index, b2c_lm_state_t* out);
/* Every beam of every utterance in flat arrays (one call instead of ~6 per beam; what decode_beams_batch needs to
 * build its OutputBeam lists, decoder.py:653-667).  Beams are numbered utterance by utterance in rank order.  All
 * pointers live as long as the result. */
typedef struct {
    int32_t n_utts;
    int32_t n_models;             /* LM states per beam (0: no language model, states == NULL) */
    int64_t n_beams_total;
    int64_t n_words_total;
    const int32_t* n_beams;       /* [n_utts] */
    const double* scores;         /* [n_beams_total][2]: logit_score, lm_score */
    const int32_t* n_words;       /* [n_beams_total] */
    const int32_t* frames;        /* [n_words_total][2]: (start_frame, end_frame) per word, beam after beam */
    const char* texts;            /* utf-8, every beam's text followed by a NUL byte */
    size_t texts_size;
    const b2c_lm_state_t* states; /* [n_beams_total][n_models] */
    /* streaming calls only (NULL otherwise): what b2c_result_stream_beam returns, for every beam at once; `frames` /
     * `n_words` then describe the words finished during the call */
    const int32_t* stream_aux;    /* [n_beams_total][4] */
    const int32_t* n_stream_toks; /* [n_beams_total] */
    const uint32_t* stream_toks;  /* emitted tokens (token | kind << 16), oldest first, beam after beam */
    int64_t n_stream_toks_total;
    /* the same token chains replayed into strings, three per beam, each followed by a NUL byte: what the chain appends
     * to the input beam's partial word before the first word boundary; the words finished after that boundary, joined
     * by single spaces; the partial word after the last boundary.  stream_boundary[beam] says whether the chain
     * contains a word boundary at all (0: everything went to the first string). */
    const char* stream_pieces;
    size_t stream_pieces_size;
    const int32_t* stream_boundary; /* [n_beams_total] */
} b2c_packed_t;
int b2c_result_packed(b2c_result_t* res, b2c_packed_t* out);
/* streaming calls (opts->stream_states != NULL): what the call appended to an input beam instead of assembled
 * strings.  aux = {input beam index (-1: none), token id of last_char (-1: None), partial_frames start, end};
 * toks = the emitted tokens since the input beam, oldest first, token | kind << 16 with kind B2C_KIND_CONT = appended
 * to the partial word, B2C_KIND_SPACE = the word separator, B2C_KIND_BPE = BPE piece that starts a word; b2c_result_frames / b2c_result_n_frames give the frames
 * of the words finished during the call (LMBeam, decoder.py:97-100; the host replays them onto the input beam). */
#define B2C_KIND_CONT 0
#define B2C_KIND_SPACE 1
#define B2C_KIND_BPE 2
int b2c_result_stream_beam(const b2c_result_t* res, int utt, int beam, int32_t aux[4], const uint32_t** toks, int* n_toks);
int b2c_result_n_frames(const b2c_result_t* res, int utt, int beam);
/* string -> (hash, code points) as the kernels identify words and partial words; label -> canonical token id
 * (-1 when the alphabet has no such label) */
int b2c_hash_utf8(const char* s, uint64_t* hash, uint32_t* n_chars);
/* the same for `count` strings stored back to back, each followed by a NUL byte */
int b2c_hash_utf8_batch(const char* data, size_t size, int64_t count, uint64_t* hashes, uint32_t* n_chars);
int b2c_decoder_token_id(const b2c_decoder_t* dec, const char* label);

/* ---- measurement hooks (bench.py) ---------------------------------------------------------
 * Device time of the kernels of the LAST decode call, measured with CUDA events on the
 * decoder's stream, and launch / traffic counters. */
typedef struct {
    float ms_prepare;          /* prepare kernel (normalise + token select)               */
    float ms_beam;             /* beam-search kernel                                       */
    float ms_total;            /* first H2D copy .. last D2H copy                          */
    int launches;              /* kernels launched                                         */
    long long h2d_bytes, d2h_bytes;
    long long frames;          /* sum of T                                                 */
    long long tokens;          /* (frame, token) pairs the streaming stage emitted          */
    int cap_candidates;        /* shared-memory candidate capacity class chosen for the call */
    int cta_threads;           /* threads per CTA of the beam kernel                        */
    int cta_slots;             /* resident CTAs (utterances in flight)                      */
    long long oversize_frames; /* frames that took the out-of-line HBM-tier step           */
    int kernel_variant;        /* 0 general, 1 capacity-class fast kernel, 2 latency-first kernel (beam_width <= 128) */
    long long cand_hist[7];    /* frames with more than 128,256,...,4096 candidates; [6] = frames counted */
    long long inplace_frames;  /* single-token frames that updated the beam table in place (b2c_fast_cheap_step) */
    long long sorted_frames;   /* multi-token frames ranked by binary search, no grouping (b2c_fast_sorted_step) */
    long long single_frames;   /* one-token frames after a multi-token frame, one candidate per thread (b2c_fast_single_step) */
    int hinted;                /* 1: the beam kernel was planned from the previous call's statistics and launched without
                                  waiting for this call's (no mid-call synchronisation); same results either way */
    int kernels;               /* one bit per beam-kernel instantiation launched by the call, the retry launch included:
                                    bit 0  b2c_beam_fast_kernel<1024,2,64>   latency-first variant 0, V <= 64
                                    bit 1  b2c_beam_fast_kernel<1024,2,0>    latency-first variant 0, V > 64
                                    bit 2  b2c_beam_fast_kernel<512,3,64>    latency-first variant 1, V <= 64
                                    bit 3  b2c_beam_fast_kernel<512,3,0>     latency-first variant 1, V > 64
                                    bit 4  b2c_beam_fast_kernel<256,4,64>    latency-first variant 2, V <= 64
                                    bit 5  b2c_beam_fast_kernel<256,4,0>     latency-first variant 2, V > 64
                                    bit 6  b2c_beam_kernel<true,256,1>       capacity class 2048 / 4096
                                    bit 7  b2c_beam_kernel<true,128,2>       capacity class 512 / 1024
                                    bit 8  b2c_beam_kernel<true,64,4>        capacity class 256
                                    bit 9  b2c_beam_kernel<true,32,8>        capacity class 128
                                    bit 10 b2c_beam_kernel<false,256,1>      general kernel, one CTA per SM
                                    bit 11 b2c_beam_kernel<false,512,1>      general kernel, beam tables in HBM
                                    bit 12 b2c_beam_kernel<false,128,2>      general kernel, two CTAs per SM */
    int retried;               /* utterances whose first-pass arenas overflowed and that the general kernel decoded again
                                  with worst-case arenas (their results are those of the second decode) */
} b2c_timings_t;
int b2c_decoder_last_timings(const b2c_decoder_t* dec, b2c_timings_t* out);
/* Diagnostics: the (token id, log-prob) lists the streaming stage wrote in the LAST call, as the beam kernel consumed
 * them -- every frame's list in emission order, frame after frame, utterance after utterance.  With NULL arrays only
 * the sizes are returned.  counts / rec_id0 / rec_lp0: [n_frames] (list length, and the first token and log-prob of
 * the frame's record); ids / lps: [n_entries]; is_prob: one flag per utterance of the last call (1: the utterance was
 * taken as probabilities). */
int b2c_decoder_last_tokens(const b2c_decoder_t* dec, int64_t* n_frames, int64_t* n_entries, int32_t* counts, uint32_t* ids,
                            double* lps, uint16_t* rec_id0, double* rec_lp0, int32_t* is_prob);

#ifdef __cplusplus
}
#endif
#endif /* B200CTC_H */
