// b200ctc -- n-gram shallow fusion and hotword scoring on the flattened tables.
//
// Replaces, on the device, what the reference does through kenlm + pygtrie:
//   kenlm.Model.BaseScore ............ b2c_lm_base_score   (reference language_model.py:321,347)
//   LanguageModel.score .............. b2c_lm_score_word   (language_model.py:338-360)
//   LanguageModel.score_partial_token  b2c_partial_score   (language_model.py:326-336)
//   HotwordScorer.score / partial .... b2c_hot_*           (language_model.py:133-150)
// All tables are open-addressing hash tables in HBM probed linearly; a lookup touches one
// 32-byte sector in the common case.
#pragma once
#include "b2c_common.h"

B2C_HD u32 b2c_f32_bits(float f) {
    union { float f; u32 u; } c;
    c.f = f;
    return c.u;
}
B2C_HD bool b2c_has_extension(float backoff) { return b2c_f32_bits(backoff) != 0x80000000u; }

// string-hash keyed tables store hash+1 so that 0 can mean "empty"
B2C_HD const B2cVocab* b2c_vocab_find(const B2cLmView& lm, u64 word_hash) {
    u64 key = word_hash + 1;
    u64 slot = b2c_mix64(key) & lm.vocab_mask;
    while (true) {
        const B2cVocab* e = lm.vocab + slot;
        u64 k = e->key;
        if (k == key) return e;
        if (k == 0) return nullptr;
        slot = (slot + 1) & lm.vocab_mask;
    }
}
B2C_HD bool b2c_prefix_contains(const B2cLmView& lm, u64 prefix_hash) {
    u64 key = prefix_hash + 1;
    u64 slot = b2c_mix64(key) & lm.prefix_mask;
    while (true) {
        u64 k = lm.prefixes[slot];
        if (k == key) return true;
        if (k == 0) return false;
        slot = (slot + 1) & lm.prefix_mask;
    }
}
B2C_HD const B2cNgram* b2c_ngram_find(const B2cLmView& lm, u64 key) {
    u64 slot = b2c_mix64(key) & lm.ngram_mask;
    while (true) {
        const B2cNgram* e = lm.ngrams + slot;
        u64 k = e->key;
        if (k == key) return e;
        if (k == 0) return nullptr;
        slot = (slot + 1) & lm.ngram_mask;
    }
}
B2C_HD const B2cHot* b2c_hot_find(const B2cHotSet& H, u64 prefix_hash) {
    u64 key = prefix_hash + 1;
    u64 slot = b2c_mix64(key) & H.mask;
    while (true) {
        const B2cHot* e = H.tab + slot;
        u64 k = e->key;
        if (k == key) return e;
        if (k == 0) return nullptr;
        slot = (slot + 1) & H.mask;
    }
}

// KenLM FullScore for one word: longest matching n-gram + backoffs of the skipped contexts,
// float32 arithmetic, state minimised to the longest match that has an extension.
B2C_HD float b2c_lm_base_score(const B2cLmView& lm, const B2cLmState& in, u32 w, B2cLmState& out) {
    B2cUni u = lm.uni[w];
    float prob = u.prob;
    out.backoff[0] = u.backoff;
    out.words[0] = w;
    u32 out_len = b2c_has_extension(u.backoff) ? 1u : 0u;
    u32 matched = 1;
    const bool kenlm_keys = lm.key_scheme == B2C_KEYS_KENLM;
    u64 h = kenlm_keys ? b2c_kenlm_start(w) : b2c_ngram_start(w);
    for (u32 k = 0; k < in.length; ++k) {
        if (static_cast<int>(k) + 2 > lm.order) break;
        h = kenlm_keys ? b2c_kenlm_extend(h, in.words[k]) : b2c_ngram_extend(h, in.words[k]);
        if (h == 0) break;      // 0 marks an empty slot (KenLM's tables reserve it as well)
        const B2cNgram* e = b2c_ngram_find(lm, h);
        if (!e) break;
        prob = e->prob;
        matched = k + 2;
        if (static_cast<int>(matched) < lm.order) {
            out.backoff[k + 1] = e->backoff;
            if (b2c_has_extension(e->backoff)) out_len = matched;
        }
    }
    for (u32 i = matched - 1; i < in.length; ++i) prob = prob + in.backoff[i];
    for (u32 i = 1; i < out_len; ++i) out.words[i] = in.words[i - 1];
    out.length = out_len;
    return prob;
}

// LanguageModel.score(prev_state, word, is_last_word) -> alpha * ln10 * log10 score + beta
B2C_HD double b2c_lm_score_word_v(const B2cLmView& lm, double alpha, double beta, double unk_offset, int score_boundary,
                                  double log_base_change, const B2cLmState& prev, u64 word_hash, u32 word_len, bool is_last,
                                  B2cLmState& end_state) {
    u32 wid = 0, flags = 0;
    if (word_len) {
        const B2cVocab* v = b2c_vocab_find(lm, word_hash);
        if (v) { wid = v->id; flags = v->flags; }
    }
    double s = static_cast<double>(b2c_lm_base_score(lm, prev, wid, end_state));
    if ((lm.n_unigrams > 0 && !(flags & 1u)) || wid == 0) s += unk_offset;
    if (is_last) {
        double e = 0.0;
        if (score_boundary) {
            B2cLmState tmp;
            e = static_cast<double>(b2c_lm_base_score(lm, end_state, lm.eos_id, tmp));
        }
        s = s + e;
    }
    return alpha * s * log_base_change + beta;
}
// model 0 of a set
B2C_HD double b2c_lm_score_word(const B2cLmSet& M, const B2cLmState& prev, u64 word_hash, u32 word_len,
                                bool is_last, B2cLmState& end_state) {
    return b2c_lm_score_word_v(M.lm, M.alpha, M.beta, M.unk_offset, M.score_boundary, M.log_base_change, prev, word_hash,
                               word_len, is_last, end_state);
}
// LanguageModel.score_partial_token of one model (language_model.py:326-336)
B2C_HD double b2c_lm_partial_v(const B2cLmView& lm, double unk_offset, u64 part_hash, u32 part_len) {
    double is_oov = 1.0;
    if (lm.have_unigrams) is_oov = b2c_prefix_contains(lm, part_hash) ? 0.0 : 1.0;
    double unk = unk_offset * is_oov;
    if (part_len > B2C_AVG_TOKEN_LEN) unk = unk * static_cast<double>(part_len) / B2C_AVG_TOKEN_LEN;
    return unk;
}

// score of an unfinished word.  LM mode (reference decoder.py:397-409): hotword prefix score
// if the partial is a prefix of a hotword, else the LM's OOV-prefix penalty.  No-LM mode
// (decoder.py:363-367): hotword prefix score or 0.  M, H: the utterance's language-model set (model 0) and hotword set.
B2C_HD double b2c_partial_score(const B2cLmSet& M, const B2cHotSet& H, u64 part_hash, u32 part_len) {
    if (H.min_len > 0) {
        if (part_len == 0) return H.weight * 0 / H.min_len;
        const B2cHot* h = b2c_hot_find(H, part_hash);
        if (h) return H.weight * static_cast<double>(part_len) / static_cast<double>(h->min_len);
    }
    if (M.lm.order == 0) return 0.0;
    double is_oov = 1.0;
    if (M.lm.have_unigrams) is_oov = b2c_prefix_contains(M.lm, part_hash) ? 0.0 : 1.0;
    double unk = M.unk_offset * is_oov;
    if (part_len > B2C_AVG_TOKEN_LEN) unk = unk * static_cast<double>(part_len) / B2C_AVG_TOKEN_LEN;
    return unk;
}

B2C_HD u32 b2c_hot_is_word(const B2cHotSet& H, u64 word_hash, u32 word_len) {
    if (H.min_len == 0 || word_len == 0) return 0;
    const B2cHot* h = b2c_hot_find(H, word_hash);
    return (h && h->is_word) ? 1u : 0u;
}
