// b200ctc -- the per-utterance prefix beam search (one CTA per utterance, all T frames).
//
// Restates, string-free, the body of BeamSearchDecoderCTC._partial_decode_logits
// (reference decoder.py:443-554) and _finalize_beams/_decode_logits (:558-667):
//   expand (4 branches, :452-534) -> merge by (text, partial_word, last_char) with
//   log-sum-exp in iteration order (:211-224) -> LM / hotword fusion (:346-424) ->
//   score threshold (:545-546) -> stable top-N (:165-167) -> history prune (:227-258).
//
// Order dependence of the reference that is reproduced exactly:
//   * candidates are enumerated token-major in the CPython set order of the frame's tokens
//     (computed by the prepare kernels), beams in rank order inside a token;
//   * a merged group sits at the position of its FIRST member, takes the metadata (frames,
//     text/next_word split) of its LAST member, and folds scores left to right;
//   * ties in lm_score keep enumeration order (heapq.nlargest is stable);
//   * the single force_next_break flag of BPE alphabets (:442,474-482).
//
// Per-frame structure (4 block barriers):
//   A  expand every (token, beam) pair ONCE, cache the result, group equal keys      | barrier
//   B  group leaders: fold scores, LM / hotword fusion, score bucket, running max     | barrier
//   C  every warp scans the buckets (redundantly); leaders above the threshold get their
//      exact rank = bucket prefix + order inside the bucket; history keys are grouped  | barrier
//   D  every warp compacts the kept ranks (redundantly) and commits its share of the new
//      beams; tables are cleared for the next frame                                    | barrier
// The latency of a frame, not its instruction count, bounds a single utterance, so rare paths
// (n-gram word scoring, prefix / hotword probes, BPE force logic, finalisation) are kept out of
// line to keep the hot loop small in the instruction cache.
#pragma once
#include "b2c_cta.h"
#include "b2c_lm.h"

#if defined(__CUDACC__)
#define B2C_HDN __host__ __device__ __noinline__
#else
#define B2C_HDN __attribute__((noinline))
#endif

struct B2cBeamTab {
    double* logit;      // logit_score
    double* lm_hw;      // LM + hotword score of the beam's text (reference cached lm_hw_score)
    double* pscore;     // score of the unfinished word (0 when empty)
    u64* text_hash;
    u64* part_hash;
    u64* hist_hash;     // hash of the last hist_n finished words (history-prune key)
    u32* text_node;     // -> B2cText arena
    u32* chain;         // -> B2cChain arena (backtrack)
    int* pf_s;          // partial_frames
    int* pf_e;
    u16* last_tok;      // canonical token id or B2C_NO_TOK
    u16* part_len;      // python len(partial_word)
};

struct B2cScalars {
    u64 max_key;
    double prev_max;     // best lm_score of the previous frame: reference point of the score buckets
    B2cHotSet hot;       // this utterance's hotword set (b2c_utt_begin; parked with the rest by chunked launches)
    u32 n_beams, n_sel, n_new, chain_used, text_used, status, force_break;
    u32 flags;           // B2C_FL_*: mode bits re-read from shared memory every frame so that the compiler
                         // cannot unswitch (= replicate) the frame loop on them
    u32 m_over[6];       // frames whose candidate count exceeded 128,256,512,1024,2048,4096 (adaptive sizing)
    u32 m_frames;
    u32 inplace_bad;     // a thread's exactness check of b2c_inplace_step failed (rare)
    u32 m_inplace;       // frames handled by b2c_inplace_step
    u32 clean_s, clean_g; // leading slots of the shared-memory / HBM tier's grouping table that are known to be clear
    u32 lm_set;          // this utterance's language-model set, an index into B2cParams::lm_sets (b2c_utt_begin)
};
// the language-model set of the CTA's current utterance
B2C_HD const B2cLmSet& b2c_lm_of(const B2cParams& P, const B2cScalars* sc) { return P.lm_sets[sc->lm_set]; }
enum { B2C_FL_BPE = 1, B2C_FL_PRUNE = 2, B2C_FL_LM = 4, B2C_FL_PSCORE = 8, B2C_FL_NO_SINGLE = 16 };

#define B2C_NBUCKET 256      // score buckets of the O(m) ranking (monotone in the score)
#define B2C_NBUCKET_WIDE 2048 // the same for launches that rank hundreds to thousands of candidates per frame (general kernel,
                              // the 2048 / 4096-candidate classes): a bucket then holds ~1 candidate instead of ~10
#define B2C_MAXWARPS 8       // warps per CTA of the beam kernel (64-, 128- and 256-thread variants)
#define B2C_STAGE_K 64       // most tokens of a frame whose label records are staged in shared memory (general kernels)

struct B2cCandTier {     // per-frame candidate working set (shared memory tier or HBM tier)
    u32 cap;             // candidates
    u32 ht_cap;          // hash slots (power of two >= 2*cap)
    u64* ckey;           // merge key; after phase B: order-preserving lm_score key of group leaders, 0 otherwise
    double* cfold;       // merged logit_score of group leaders
    u64* cth;            // cached expansion: text hash of the candidate
    u64* cph;            //                   partial-word hash | branch type << 61
    u32* cmeta;          //                   partial length | canonical token << 16
    u32* cslot;          // candidate -> group slot
    u32* cnext;          // bucket list link
    u32* clast;          // leader -> last member of its group (metadata donor)
    u32* ht_idx;         // slot -> representative candidate
    u32* ht_min;         // slot -> first member (dict position)
    u32* ht_max;         // slot -> last member
    u32* ht_cnt;
};

struct B2cWork {
    B2cScalars* sc;
    B2cBeamTab cur, nxt;
    B2cCandTier tier_s, tier_g;
    // selection (capacity beam_width)
    u32* ord;            // rank -> candidate index
    u64* phk;            // rank -> history-prune key
    u32* pslot;          // rank -> slot in the prune table
    u32* pt_idx;         // history-prune table: slot -> representative rank
    u32* pt_min;         //                      slot -> best rank with that key
    u32 pt_cap;          // power of two >= 2 * beam_width
    u32 n_bucket;        // B2C_NBUCKET or B2C_NBUCKET_WIDE
    u32* bcnt;           // [n_bucket] leaders per score bucket
    u32* bhead;          // [n_bucket] list heads
    u32* bpre;           // exclusive prefix: [n_warps][B2C_NBUCKET], one private copy per warp, or ONE [B2C_NBUCKET_WIDE + 32]
    // label records / log-probs / ids of the current frame's tokens, staged once per frame (frames of up to
    // B2C_STAGE_K tokens; nullptr: no staging area, e.g. the out-of-line step of the latency-first kernel)
    B2cTok* stok;
    double* slp;
    u32* sid;
    // per-frame token side arrays for BPE force_next_break (capacity V, HBM)
    u32* tk_ffirst;
    u8* tk_fall;
    // arenas (HBM)
    B2cChain* chain;
    u32 chain_cap;
    B2cText* text;
    u32 text_cap;
#if defined(B2C_PHASE_CLOCKS)
    u64 clk[16];
    long long clk_last;
#endif
};

#define B2C_PH_MASK B2C_P61

// ---------------------------------------------------------------------------------------
// workspace layout (shared memory + per-slot HBM workspace): computed on the host
// (b2c_api.cu make_layout), interpreted here
// ---------------------------------------------------------------------------------------
struct B2cLayout {
    int W;                      // beam_width (capacity of the beam tables)
    u32 cap_s, ht_s;            // shared-memory candidate tier
    u32 cap_g, ht_g;            // HBM candidate tier (0: absent)
    int beams_in_smem;
    int n_warps;                // warps per CTA of the launch (sizes the per-warp scratch)
    int n_bucket;               // score buckets (B2C_NBUCKET / B2C_NBUCKET_WIDE)
    u32 chain_cap, text_cap;
    int V;
    u32 smem_bytes;
    u64 gws_bytes;              // per slot
    // offsets
    u32 s_sc, s_tab[2], s_sel, s_tier;
    u64 g_tab[2], g_sel, g_tier, g_tk, g_chain, g_text;
};

B2C_HD u32 pt_cap_for(int W) { u32 p = 16; while (p < 2u * static_cast<u32>(W)) p <<= 1; return p; }

B2C_HD u8* b2c_carve(u8*& p, u64 bytes) {
    u8* r = p;
    p += (bytes + 15) & ~15ull;
    return r;
}
B2C_HD void b2c_carve_tab(u8* base, int W, B2cBeamTab& t) {
    u8* p = base;
    t.logit = reinterpret_cast<double*>(b2c_carve(p, 8ull * W));
    t.lm_hw = reinterpret_cast<double*>(b2c_carve(p, 8ull * W));
    t.pscore = reinterpret_cast<double*>(b2c_carve(p, 8ull * W));
    t.text_hash = reinterpret_cast<u64*>(b2c_carve(p, 8ull * W));
    t.part_hash = reinterpret_cast<u64*>(b2c_carve(p, 8ull * W));
    t.hist_hash = reinterpret_cast<u64*>(b2c_carve(p, 8ull * W));
    t.text_node = reinterpret_cast<u32*>(b2c_carve(p, 4ull * W));
    t.chain = reinterpret_cast<u32*>(b2c_carve(p, 4ull * W));
    t.pf_s = reinterpret_cast<int*>(b2c_carve(p, 4ull * W));
    t.pf_e = reinterpret_cast<int*>(b2c_carve(p, 4ull * W));
    t.last_tok = reinterpret_cast<u16*>(b2c_carve(p, 2ull * W));
    t.part_len = reinterpret_cast<u16*>(b2c_carve(p, 2ull * W));
}
B2C_HD void b2c_carve_tier(u8* base, u32 cap, u32 ht, B2cCandTier& c) {
    u8* p = base;
    c.cap = cap;
    c.ht_cap = ht;
    c.ckey = reinterpret_cast<u64*>(b2c_carve(p, 8ull * cap));
    c.cfold = reinterpret_cast<double*>(b2c_carve(p, 8ull * cap));
    c.cth = reinterpret_cast<u64*>(b2c_carve(p, 8ull * cap));
    c.cph = reinterpret_cast<u64*>(b2c_carve(p, 8ull * cap));
    c.cmeta = reinterpret_cast<u32*>(b2c_carve(p, 4ull * cap));
    c.cslot = reinterpret_cast<u32*>(b2c_carve(p, 4ull * cap));
    c.cnext = reinterpret_cast<u32*>(b2c_carve(p, 4ull * cap));
    c.clast = reinterpret_cast<u32*>(b2c_carve(p, 4ull * cap));
    c.ht_idx = reinterpret_cast<u32*>(b2c_carve(p, 4ull * ht));
    c.ht_min = reinterpret_cast<u32*>(b2c_carve(p, 4ull * ht));
    c.ht_max = reinterpret_cast<u32*>(b2c_carve(p, 4ull * ht));
    c.ht_cnt = reinterpret_cast<u32*>(b2c_carve(p, 4ull * ht));
}


// build the work descriptor of one CTA; `parity` says which of the two beam tables is current
B2C_HD void b2c_make_work(const B2cLayout& L, u8* smem, u8* g, int parity, bool beams_s, B2cWork& W) {
    W.sc = reinterpret_cast<B2cScalars*>(smem + L.s_sc);
    if (beams_s) {
        b2c_carve_tab(smem + L.s_tab[parity], L.W, W.cur);
        b2c_carve_tab(smem + L.s_tab[parity ^ 1], L.W, W.nxt);
    } else {
        b2c_carve_tab(g + L.g_tab[parity], L.W, W.cur);
        b2c_carve_tab(g + L.g_tab[parity ^ 1], L.W, W.nxt);
    }
    {
        u8* p = smem + L.s_sel;
        W.phk = reinterpret_cast<u64*>(b2c_carve(p, 8ull * L.W));
        W.ord = reinterpret_cast<u32*>(b2c_carve(p, 4ull * L.W));
        W.pslot = reinterpret_cast<u32*>(b2c_carve(p, 4ull * L.W));
        W.pt_cap = pt_cap_for(L.W);
        W.pt_idx = reinterpret_cast<u32*>(b2c_carve(p, 4ull * W.pt_cap));
        W.pt_min = reinterpret_cast<u32*>(b2c_carve(p, 4ull * W.pt_cap));
        W.n_bucket = static_cast<u32>(L.n_bucket);
        W.bcnt = reinterpret_cast<u32*>(b2c_carve(p, 4ull * L.n_bucket));
        W.bhead = reinterpret_cast<u32*>(b2c_carve(p, 4ull * L.n_bucket));
        W.bpre = reinterpret_cast<u32*>(b2c_carve(p, L.n_bucket == B2C_NBUCKET ? 4ull * B2C_NBUCKET * L.n_warps : 4ull * (L.n_bucket + 32)));
        W.stok = reinterpret_cast<B2cTok*>(b2c_carve(p, sizeof(B2cTok) * B2C_STAGE_K));
        W.slp = reinterpret_cast<double*>(b2c_carve(p, 8ull * B2C_STAGE_K));
        W.sid = reinterpret_cast<u32*>(b2c_carve(p, 4ull * B2C_STAGE_K));
    }
    b2c_carve_tier(smem + L.s_tier, L.cap_s, L.ht_s, W.tier_s);
    if (L.cap_g) b2c_carve_tier(g + L.g_tier, L.cap_g, L.ht_g, W.tier_g);
    else W.tier_g = W.tier_s;
    {
        u8* p = g + L.g_tk;
        W.tk_ffirst = reinterpret_cast<u32*>(b2c_carve(p, 4ull * L.V));
        W.tk_fall = reinterpret_cast<u8*>(b2c_carve(p, static_cast<u64>(L.V)));
    }
    W.chain = reinterpret_cast<B2cChain*>(g + L.g_chain);
    W.chain_cap = L.chain_cap;
    W.text = reinterpret_cast<B2cText*>(g + L.g_text);
    W.text_cap = L.text_cap;
}

B2C_HD void b2c_swap_tabs(B2cBeamTab& a, B2cBeamTab& b) {
    B2cBeamTab t = a;
    a = b;
    b = t;
}

B2C_HD int b2c_warp_id() {
#if defined(__CUDA_ARCH__)
    return static_cast<int>(threadIdx.x >> 5);
#else
    return 0;
#endif
}

// ---------------------------------------------------------------------------------------
// out-of-line rare paths
// ---------------------------------------------------------------------------------------
// text-level quantities of "text + word" (reference _get_lm_beams cache miss, decoder.py:388-395)
struct B2cTextNew {
    double raw_lm, lm_hw;
    u32 hw_count;
    B2cLmState st;
};
// LM states of models 1.. of a text node live behind the node arena: [text_cap][n_lm - 1]
B2C_HD B2cLmState* b2c_text_states_x(const B2cText* arena, u32 text_cap, int n_lm, u32 node) {
    return reinterpret_cast<B2cLmState*>(const_cast<B2cText*>(arena) + text_cap) + static_cast<u64>(node) * static_cast<u64>(n_lm - 1);
}
// out_x: where the end states of models 1.. go (MultiLanguageModel; nullptr: not wanted)
B2C_HDN void b2c_text_extend(const B2cLmSet& M, const B2cHotSet& H, const B2cText* arena, u32 text_cap, u32 parent_id, u64 word_hash,
                             u32 word_len, int is_eos, B2cTextNew* out, B2cLmState* out_x) {
    const B2cText* parent = arena + parent_id;
    out->hw_count = parent->hw_count + b2c_hot_is_word(H, word_hash, word_len);
    if (M.n_lm > 1) {
        // MultiLanguageModel.score (language_model.py:485-502): sum of the models' scores, left to right, / N
        const B2cLmState* px = b2c_text_states_x(arena, text_cap, M.n_lm, parent_id);
        B2cLmState in = parent->st;
        double sc = b2c_lm_score_word(M, in, word_hash, word_len, is_eos != 0, out->st);
        for (int j = 1; j < M.n_lm; ++j) {
            const B2cLmExtra X = M.lmx[j - 1];
            in = px[j - 1];
            B2cLmState end;
            sc = sc + b2c_lm_score_word_v(X.lm, X.alpha, X.beta, X.unk_offset, X.score_boundary, M.log_base_change, in, word_hash,
                                          word_len, is_eos != 0, end);
            if (out_x) out_x[j - 1] = end;
        }
        sc = sc / static_cast<double>(M.n_lm);
        out->raw_lm = parent->raw_lm + sc;
        out->lm_hw = out->raw_lm + H.weight * static_cast<double>(out->hw_count);
    } else if (M.lm.order > 0) {
        B2cLmState in = parent->st;
        double sc = b2c_lm_score_word(M, in, word_hash, word_len, is_eos != 0, out->st);
        out->raw_lm = parent->raw_lm + sc;
        out->lm_hw = out->raw_lm + H.weight * static_cast<double>(out->hw_count);
    } else {
        out->raw_lm = 0.0;
        out->st.length = 0;
        out->lm_hw = H.weight * static_cast<double>(out->hw_count);
    }
}

// score of an unfinished word, scalar arguments only (no parameter block copy on this path)
B2C_HDN double b2c_partial_score_ool(const B2cHotSet& H, int lm_order, int have_unigrams, const u64* prefixes, u64 prefix_mask,
                                     double unk_offset, u64 part_hash, u32 part_len) {
    if (H.min_len > 0) {
        if (part_len == 0) return H.weight * 0 / H.min_len;
        const B2cHot* e = b2c_hot_find(H, part_hash);
        if (e) return H.weight * static_cast<double>(part_len) / static_cast<double>(e->min_len);
    }
    if (lm_order == 0) return 0.0;
    double is_oov = 1.0;
    if (have_unigrams) {
        const u64 key = part_hash + 1;
        u64 slot = b2c_mix64(key) & prefix_mask;
        while (true) {
            const u64 k = prefixes[slot];
            if (k == key) { is_oov = 0.0; break; }
            if (k == 0) break;
            slot = (slot + 1) & prefix_mask;
        }
    }
    double unk = unk_offset * is_oov;
    if (part_len > B2C_AVG_TOKEN_LEN) unk = unk * static_cast<double>(part_len) / B2C_AVG_TOKEN_LEN;
    return unk;
}
// MultiLanguageModel.score_partial_token (language_model.py:478-483): mean over the models; the hotword prefix
// score takes precedence exactly as with one model (decoder.py:397-409)
B2C_HDN double b2c_partial_score_multi(const B2cLmSet& M, const B2cHotSet& H, u64 part_hash, u32 part_len) {
    if (H.min_len > 0) {
        if (part_len == 0) return H.weight * 0 / H.min_len;
        const B2cHot* h = b2c_hot_find(H, part_hash);
        if (h) return H.weight * static_cast<double>(part_len) / static_cast<double>(h->min_len);
    }
    double s = b2c_lm_partial_v(M.lm, M.unk_offset, part_hash, part_len);
    for (int j = 1; j < M.n_lm; ++j) {
        const B2cLmExtra X = M.lmx[j - 1];
        s = s + b2c_lm_partial_v(X.lm, X.unk_offset, part_hash, part_len);
    }
    return s / static_cast<double>(M.n_lm);
}
B2C_HD double b2c_partial_score_of(const B2cLmSet& M, const B2cHotSet& H, bool need, u64 part_hash, u32 part_len) {
    if (!need) return 0.0;
    if (M.n_lm > 1) return b2c_partial_score_multi(M, H, part_hash, part_len);
    return b2c_partial_score_ool(H, M.lm.order, M.lm.have_unigrams, M.lm.prefixes, M.lm.prefix_mask, M.unk_offset, part_hash, part_len);
}

// history-prune hash of "text + word" (last hist_n words)
B2C_HDN u64 b2c_hist_extend(const B2cText* par, int hist_n, u64 word_hash) {
    const u32 keep = (par->n_win + 1 < static_cast<u32>(hist_n)) ? par->n_win : static_cast<u32>(hist_n) - 1;
    u64 hh = B2C_HIST_SEED;
    for (int w = static_cast<int>(keep) - 1; w >= 0; --w) hh = b2c_hist_fold(hh, par->win[w]);
    return b2c_hist_fold(hh, word_hash);
}

// a surviving beam finished a word: create the text node (LM state, raw score, hotword count, history)
struct B2cTextCommit { u32 node; double lm_hw; u64 hist_hash; };
B2C_HDN void b2c_commit_text(const B2cLmSet& M, const B2cHotSet& H, B2cText* arena, u32 text_cap, u32* text_used, u32* status, u32 parent_id,
                             u64 word_hash, u32 word_len, B2cTextCommit* out) {
    const B2cText* par = arena + parent_id;
    // the node is allocated first so that a MultiLanguageModel's other end states are written in place
    const u32 id = b2c_atomic_add_u32(text_used, 1u);
    B2cTextNew tn;
    b2c_text_extend(M, H, arena, text_cap, parent_id, word_hash, word_len, 0, &tn,
                    (M.n_lm > 1 && id < text_cap) ? b2c_text_states_x(arena, text_cap, M.n_lm, id) : nullptr);
    out->lm_hw = tn.lm_hw;
    out->node = parent_id;
    const u32 keep = (par->n_win + 1 < static_cast<u32>(M.hist_n)) ? par->n_win : static_cast<u32>(M.hist_n) - 1;
    B2cText nt;
    nt.win[0] = word_hash;
    for (u32 w = 0; w < keep; ++w) nt.win[w + 1] = par->win[w];
    for (u32 w = keep + 1; w < B2C_MAX_HIST; ++w) nt.win[w] = 0;
    nt.n_win = keep + 1;
    u64 hh = B2C_HIST_SEED;
    for (int w = static_cast<int>(nt.n_win) - 1; w >= 0; --w) hh = b2c_hist_fold(hh, nt.win[w]);
    nt.hist_hash = hh;
    out->hist_hash = hh;
    nt.raw_lm = tn.raw_lm;
    nt.st = tn.st;
    nt.hw_count = tn.hw_count;
    if (id < text_cap) {
        arena[id] = nt;
        out->node = id;
    } else {
        b2c_atomic_or_u32(status, B2C_ERR_TEXT_FULL);
    }
}

// log-sum-exp merge, out of line: float64 exp + log are ~150 instructions that only merged groups need
B2C_HDN double b2c_sum_log_scores_ool(double s1, double s2) { return b2c_sum_log_scores(s1, s2); }

// BPE only: who consumes force_next_break (decoder.py:442,474-482); contains two block barriers
B2C_HDN void b2c_bpe_force(const B2cTok* toks, const u32* tk_id, int K, const u16* last_tok, u32 n, u32* ffirst, u8* fall,
                           u32* force_break) {
    // tk_id == nullptr: `toks` is already the frame's token list (staged records of the fast kernel)
    B2C_FOR(k, K) {
        const B2cTok ti = toks[tk_id ? tk_id[k] : k];
        u32 first = B2C_NONE_U32;
        if (!(ti.flags & B2C_TF_BLANK)) {
            for (u32 b = 0; b < n; ++b) {
                if (last_tok[b] == 0xFFFEu) continue;      // dead slot of the latency-first kernel (B2C_INVALID_TOK)
                if (last_tok[b] != ti.canon) { first = b; break; }
            }
        }
        ffirst[k] = first;
    }
    B2C_SYNC();
    B2C_LEADER {
        u32 F = *force_break;
        for (int k = 0; k < K; ++k) {
            const u16 fl = toks[tk_id ? tk_id[k] : k].flags;
            const u32 first = ffirst[k];
            u8 all = 0;
            u32 one = B2C_NONE_U32;
            if (first != B2C_NONE_U32) {
                const u32 trail = (fl & B2C_TF_BPE_TRAIL) ? 1u : 0u;
                if (fl & B2C_TF_BPE_LEAD) { all = 1; F = trail; }
                else if (F) { one = first; all = static_cast<u8>(trail); F = trail; }
            }
            ffirst[k] = one;
            fall[k] = all;
        }
        *force_break = F;
    }
    B2C_SYNC();
}

// ---------------------------------------------------------------------------------------
// small inline helpers of the hot path
// ---------------------------------------------------------------------------------------
B2C_HD double b2c_combine_score(bool has_lm, double logit, double lm_hw, double pscore, u32 part_len) {
    double s;
    if (has_lm) {
        double l = lm_hw;                                  // decoder.py:396-420
        if (part_len > 0) l += pscore;
        s = logit + l;
    } else {
        s = logit + lm_hw + pscore;                        // decoder.py:363-367
    }
    return s + 0.0;                                        // -0.0 -> +0.0 so that key order == float order
}

B2C_HD B2cCandTier b2c_pick_tier(const B2cWork& W, u32 M) {
    B2cCandTier c = W.tier_s;
    if (M > W.tier_s.cap) c = W.tier_g;
    return c;
}

B2C_HD u32 b2c_ht_size(u32 M) {   // power of two >= max(16, 2*M)
    if (M <= 8) return 16;
#if defined(__CUDA_ARCH__)
    return 1u << (32 - __clz(static_cast<int>(2 * M - 1)));
#else
    u32 h = 16;
    while (h < 2 * M) h <<= 1;
    return h;
#endif
}

B2C_HD void b2c_fence_block() {
#if defined(__CUDA_ARCH__)
    asm volatile("fence.acq_rel.cta;" ::: "memory");   // release before / acquire after the slot CAS
#endif
}

// group candidates with equal keys.  The caller has stored C.ckey[i] and issued a block fence;
// a thread that loses the slot race reads the winner's key, which the winner published
// (store, fence) before its CAS.
B2C_HD void b2c_group_insert(const B2cCandTier& C, u32 hmask, u32 i, u64 key) {
    u32 slot = static_cast<u32>(b2c_mix64(key)) & hmask;
    bool claimed = false;
    while (true) {
        const u32 rep = b2c_atomic_cas_u32(&C.ht_idx[slot], B2C_NONE_U32, i);
        if (rep == B2C_NONE_U32) { claimed = true; break; }
        b2c_fence_block();
        if (C.ckey[rep] == key) break;
        slot = (slot + 1) & hmask;
    }
    C.cslot[i] = slot;
    // the member that claimed the slot is known from ht_idx; only JOINERS (merges: a few percent of the candidates) pay
    // for the three atomics that track the group's extent
    if (!claimed) {
        b2c_atomic_min_u32(&C.ht_min[slot], i);
        b2c_atomic_max_u32(&C.ht_max[slot], i);
        b2c_atomic_add_u32(&C.ht_cnt[slot], 1u);
    }
}
// first / last member and size of the group in `slot` (after the barrier that ends the insert phase)
B2C_HD void b2c_group_extent(const B2cCandTier& C, u32 slot, u32& first, u32& last, u32& cnt) {
    const u32 rep = C.ht_idx[slot], joined = C.ht_cnt[slot];
    first = rep;
    last = rep;
    cnt = joined + 1;
    if (joined) {
        const u32 lo = C.ht_min[slot], hi = C.ht_max[slot];
        if (lo < first) first = lo;
        if (hi > last) last = hi;
    }
}

// clear the grouping table (first H slots) and the score buckets for the next frame; called in
// phase D, where neither is read any more.  (The history-prune table IS read in phase D by every
// warp's compaction loop, so it is cleared in phase A of the next frame instead.)
B2C_HD void b2c_clear_tables(const B2cWork& W, const B2cCandTier& C, u32 H) {
    B2C_FOR(s, H) {
        C.ht_idx[s] = B2C_NONE_U32;
        C.ht_min[s] = B2C_NONE_U32;
        C.ht_max[s] = 0;
        C.ht_cnt[s] = 0;
    }
    B2C_FOR(s, W.n_bucket) { W.bcnt[s] = 0; W.bhead[s] = B2C_NONE_U32; }
}
// The same with bookkeeping: sc->clean_s / clean_g say how many leading slots of each tier's table are known to be
// clear, so that frames which never touch the table (in-place steps) do not sweep it again.  `used_g` / `H_used`: the
// tier and extent the calling step has dirtied (H_used == 0: none).  Every thread computes the same values from the
// scalars it read BEFORE the closing barrier of the step; the leader stores them (block-uniform control flow).
B2C_HD void b2c_prepare_tables(const B2cWork& W, u32 M_next, bool used_g, u32 H_used, bool buckets) {
    B2cScalars* sc = W.sc;
    const bool next_g = M_next > W.tier_s.cap && W.tier_g.cap > W.tier_s.cap;
    const B2cCandTier Cn = next_g ? W.tier_g : W.tier_s;
    u32 Hn = b2c_ht_size(M_next);
    if (Hn > Cn.ht_cap) Hn = Cn.ht_cap;
    u32 cs = sc->clean_s, cg = sc->clean_g;
    if (H_used) { if (used_g) cg = 0; else cs = 0; }
    const u32 have = next_g ? cg : cs;
    if (have < Hn) {
        B2C_FOR(q, Hn - have) {
            const u32 s = have + static_cast<u32>(q);
            Cn.ht_idx[s] = B2C_NONE_U32;
            Cn.ht_min[s] = B2C_NONE_U32;
            Cn.ht_max[s] = 0;
            Cn.ht_cnt[s] = 0;
        }
        if (next_g) cg = Hn; else cs = Hn;
    }
    if (buckets) { B2C_FOR(s, W.n_bucket) { W.bcnt[s] = 0; W.bhead[s] = B2C_NONE_U32; } }
    B2C_SYNC();         // everybody has read the old extents
    B2C_LEADER { sc->clean_s = cs; sc->clean_g = cg; }
}

// i -> (i / n, i % n) without an integer division (float reciprocal + exact correction)
B2C_HD void b2c_divmod(u32 i, u32 n, float rcp, u32& q, u32& r) {
    if (i >= (1u << 22)) { q = i / n; r = i - q * n; return; }
    q = static_cast<u32>(static_cast<float>(i) * rcp);
    r = i - q * n;
    if (static_cast<int>(r) < 0) { --q; r += n; }
    else if (r >= n) { ++q; r -= n; }
}

// score bucket relative to a reference score, monotone non-increasing in the score: a larger score
// never gets a larger bucket (scores above the reference share bucket 0, far-away ones the last)
B2C_HD u32 b2c_bucket_n(double ref, double score, double scale, u32 nb) {
    const double d = (ref - score) * scale;
    if (!(d > 0.0)) return 0;
    return d >= static_cast<double>(nb - 1) ? nb - 1 : static_cast<u32>(d);
}
B2C_HD u32 b2c_bucket(double ref, double score, double scale) { return b2c_bucket_n(ref, score, scale, B2C_NBUCKET); }
B2C_HD double b2c_bucket_scale(double prune_logp) {
    double range = -prune_logp + 2.0;      // the reference point is the previous frame's best score
    if (!(range >= 1.0)) range = 1.0;      // also catches NaN
    if (range > 34.0) range = 34.0;
    return static_cast<double>(B2C_NBUCKET) / range;
}

// exclusive prefix over the bucket counts, computed by the calling warp into ITS copy `pre`
B2C_HD void b2c_bucket_scan_warp(const u32* bcnt, u32* pre) {
#if defined(__CUDA_ARCH__)
    const u32 lane = threadIdx.x & 31;
    const u32 per = B2C_NBUCKET / 32;
    u32 v[B2C_NBUCKET / 32];
    u32 sum = 0;
#pragma unroll
    for (u32 q = 0; q < per; ++q) { v[q] = bcnt[lane * per + q]; sum += v[q]; }
    u32 incl = sum;
    for (int off = 1; off < 32; off <<= 1) {
        const u32 o = __shfl_up_sync(0xFFFFFFFFu, incl, off);
        if (lane >= static_cast<u32>(off)) incl += o;
    }
    u32 run = incl - sum;
#pragma unroll
    for (u32 q = 0; q < per; ++q) { pre[lane * per + q] = run; run += v[q]; }
    __syncwarp();
#else
    u32 run = 0;
    for (u32 b = 0; b < B2C_NBUCKET; ++b) { pre[b] = run; run += bcnt[b]; }
#endif
}

// the same for B2C_NBUCKET_WIDE buckets: ONE copy computed by the whole CTA (two block barriers inside; nb is a multiple
// of 4 * blockDim.x); pre[nb .. nb + 32) is scratch for the warp totals
B2C_HD void b2c_bucket_scan_block(const u32* bcnt, u32* pre, u32 nb) {
#if defined(__CUDA_ARCH__)
    const u32 tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const u32 per4 = nb / (4 * blockDim.x);
    const uint4* src = reinterpret_cast<const uint4*>(bcnt) + tid * per4;
    u32 sum = 0;
    for (u32 q = 0; q < per4; ++q) { const uint4 a = src[q]; sum += a.x + a.y + a.z + a.w; }
    u32 incl = sum;
    for (int off = 1; off < 32; off <<= 1) {
        const u32 o = __shfl_up_sync(0xFFFFFFFFu, incl, off);
        if (lane >= static_cast<u32>(off)) incl += o;
    }
    if (lane == 31) pre[nb + w] = incl;
    __syncthreads();
    u32 run = incl - sum;
    for (u32 q = 0; q < w; ++q) run += pre[nb + q];
    uint4* dst = reinterpret_cast<uint4*>(pre) + tid * per4;
    for (u32 q = 0; q < per4; ++q) {
        const uint4 a = src[q];
        uint4 o;
        o.x = run; o.y = o.x + a.x; o.z = o.y + a.y; o.w = o.z + a.z;
        run = o.w + a.w;
        dst[q] = o;
    }
    __syncthreads();
#else
    u32 run = 0;
    for (u32 b = 0; b < nb; ++b) { pre[b] = run; run += bcnt[b]; }
#endif
}

B2C_HD void b2c_block_max_u64(u64 v, u64* target) {
#if defined(__CUDA_ARCH__)
    for (int off = 16; off >= 1; off >>= 1) {
        const u64 o = __shfl_xor_sync(0xFFFFFFFFu, v, off);
        if (o > v) v = o;
    }
    if ((threadIdx.x & 31) == 0 && v) atomicMax(target, v);
#else
    if (v > *target) *target = v;
#endif
}
B2C_HD void b2c_block_add_u32(u32 v, u32* target) {
#if defined(__CUDA_ARCH__)
    for (int off = 16; off >= 1; off >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, off);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(target, v);
#else
    *target += v;
#endif
}

// opt-in phase timing (-DB2C_PHASE_CLOCKS, profiling builds only): thread 0 accumulates the cycles
// between consecutive marks into W.clk[]
#if defined(B2C_PHASE_CLOCKS) && defined(__CUDA_ARCH__)
#define B2C_MARK(idx) do { if (threadIdx.x == 0) { const long long _c = clock64(); W.clk[idx] += static_cast<u64>(_c - W.clk_last); W.clk_last = _c; } } while (0)
#else
#define B2C_MARK(idx) ((void)0)
#endif

// one new beam: rank r of this frame becomes beam j of the next frame
template <class Tier>
B2C_HD void b2c_commit_one(const B2cParams& P, const B2cWork& W, const Tier& C, const B2cBeamTab& cur, const B2cBeamTab& nx,
                           const u32* tk_id, const B2cTok* toks_s, u32 n, float rcp_n, int t, u32 j, u32 r, u32 flags) {
    B2cScalars* sc = W.sc;
    const u32 i = W.ord[r];
    const u32 last = C.clast[i];
    u32 k, bl;
    b2c_divmod(last, n, rcp_n, k, bl);
    const u64 cph = C.cph[last];
    const u32 type = static_cast<u32>(cph >> 61);
    const u64 part_hash = cph & B2C_PH_MASK;
    const u32 meta = C.cmeta[last];
    const u32 part_len = meta & 0xFFFFu;
    nx.logit[j] = C.cfold[i];
    nx.text_hash[j] = C.cth[last];
    nx.part_hash[j] = part_hash;
    nx.part_len[j] = static_cast<u16>(part_len);
    nx.last_tok[j] = static_cast<u16>(meta >> 16);
    // partial_frames (decoder.py:454-461,495,513,519-523)
    const int ps0 = cur.pf_s[bl], pe0 = cur.pf_e[bl];
    int pfs, pfe;
    if (type == 0) { pfs = ps0; pfe = ((toks_s ? toks_s[k].flags : P.toks[tk_id[k]].flags) & B2C_TF_BLANK) ? pe0 : t + 1; }
    else if (type == 1) { pfs = t; pfe = t + 1; }
    else if (type == 2) { pfs = -1; pfe = -1; }
    else { pfs = ps0 < 0 ? t : ps0; pfe = t + 1; }
    nx.pf_s[j] = pfs;
    nx.pf_e[j] = pfe;
    const u32 word_len = (type == 1 || type == 2) ? static_cast<u32>(cur.part_len[bl]) : 0u;
    // backtrack chain
    u32 chain = cur.chain[bl];
    if (type != 0) {
        const u32 id = b2c_alloc_one(&sc->chain_used);
        if (id < W.chain_cap) {
            B2cChain c;
            c.parent = chain;
            c.tok = static_cast<u16>(tk_id[k]);
            c.kind = type == 3 ? B2C_CK_CONT : (type == 2 ? B2C_CK_SPACE : B2C_CK_BPE);
            c.has_word = word_len > 0 ? 1 : 0;
            c.ws = ps0;
            c.we = pe0;
            b2c_chain_store(W.chain, id, c, P.narrow_chain != 0);
            chain = id;
        } else {
            b2c_atomic_or_u32(&sc->status, B2C_ERR_CHAIN_FULL);
        }
    }
    nx.chain[j] = chain;
    // text level
    u32 tnode = cur.text_node[bl];
    double lm_hw = cur.lm_hw[bl];
    u64 hh = cur.hist_hash[bl];
    if (word_len > 0) {
        B2cTextCommit tc;
        b2c_commit_text(b2c_lm_of(P, sc), sc->hot, W.text, W.text_cap, &sc->text_used, &sc->status, tnode, cur.part_hash[bl], word_len, &tc);
        tnode = tc.node;
        lm_hw = tc.lm_hw;
        hh = tc.hist_hash;
    }
    nx.text_node[j] = tnode;
    nx.lm_hw[j] = lm_hw;
    nx.hist_hash[j] = hh;
    double ps = 0.0;
    if (type == 0) ps = cur.pscore[bl];
    else if (part_len > 0) ps = b2c_partial_score_of(b2c_lm_of(P, sc), sc->hot, (flags & B2C_FL_PSCORE) != 0, part_hash, part_len);
    nx.pscore[j] = ps;
}

// -----------------------------------------------------------------------------------------
// one frame.  kFast: the candidate tier is the shared-memory one; all table views are value copies
// so that the compiler keeps them in registers and can prove the shared-memory address space of
// every access.  On entry the grouping table (first ht_size(n*K) slots), the buckets and the
// prune table are clear (previous frame's phase D / b2c_utt_begin).
// -----------------------------------------------------------------------------------------
template <bool kFast>
B2C_HD void b2c_frame_step(const B2cParams& P, B2cWork& W, int t, const u32* tk_id_g, const double* tk_lp_g, int K, int K_next) {
    B2cScalars* sc = W.sc;
    const u32 n = sc->n_beams;
    const u32 M = n * static_cast<u32>(K);
    const float rcp_n = 1.0f / static_cast<float>(n);
    const B2cCandTier C = kFast ? W.tier_s : b2c_pick_tier(W, M);
    if (M > C.cap) {  // cannot happen: the host sizes the tiers from beam_width and the token counts
        B2C_LEADER { sc->status = B2C_ERR_CAND_FULL; }
        B2C_SYNC();
        return;
    }
    B2C_MARK(0);
    B2C_LEADER {
        ++sc->m_frames;
        for (int q = 0; q < 6; ++q)
            if (M > (128u << q)) ++sc->m_over[q];
    }
    const u32 hmask = b2c_ht_size(M) - 1;
    const B2cBeamTab cur = W.cur;
    const B2cBeamTab nx = W.nxt;
    u32* const ord = W.ord;
    u64* const phk = W.phk;
    u32* const pslot = W.pslot;
    u32* const bcnt = W.bcnt;
    u32* const bhead = W.bhead;
    const u32 nb = W.n_bucket;
    u32* const bpre = nb == B2C_NBUCKET ? W.bpre + static_cast<u32>(b2c_warp_id()) * B2C_NBUCKET : W.bpre;
    u32* const pt_idx = W.pt_idx;
    u32* const pt_min = W.pt_min;
    const u32 ptmask = W.pt_cap - 1;
    const double ref = sc->prev_max;
    const double bscale = P.bucket_scale * static_cast<double>(nb / B2C_NBUCKET);
    const u32 flags = sc->flags;
    const bool is_bpe = (flags & B2C_FL_BPE) != 0, prune = (flags & B2C_FL_PRUNE) != 0;

    // label records / log-probs of this frame's tokens: once into shared memory instead of two dependent global
    // loads per candidate (frames of up to B2C_STAGE_K tokens)
    const bool staged = W.stok != nullptr && K <= B2C_STAGE_K;
    const B2cTok* const toks_s = staged ? W.stok : nullptr;
    if (staged) {
        B2C_FOR(k, K) {
            const u32 id = tk_id_g[k];
            W.sid[k] = id;
            W.stok[k] = P.toks[id];
            W.slp[k] = tk_lp_g[k];
        }
    }
    const u32* const tk_id = staged ? W.sid : tk_id_g;
    const double* const tk_lp = staged ? W.slp : tk_lp_g;
    if (prune) { B2C_FOR(s, W.pt_cap) { pt_idx[s] = B2C_NONE_U32; pt_min[s] = B2C_NONE_U32; } }
    if (staged) B2C_SYNC();

    if (is_bpe) b2c_bpe_force(toks_s ? toks_s : P.toks, toks_s ? nullptr : tk_id, K, cur.last_tok, n, W.tk_ffirst, W.tk_fall, &sc->force_break);

    // ---- phase A: expand once, cache, merge key, grouping (publish key, fence, claim slot) -----
    B2C_FOR(i, M) {
        u32 k, b;
        b2c_divmod(static_cast<u32>(i), n, rcp_n, k, b);
        const B2cTok ti = toks_s ? toks_s[k] : P.toks[tk_id[k]];
        const u32 plen = cur.part_len[b];
        const u64 ph = cur.part_hash[b];
        u64 th = cur.text_hash[b];
        u64 nph;
        u32 nplen, type;
        if ((ti.flags & B2C_TF_BLANK) || cur.last_tok[b] == ti.canon) {                        // (i)
            type = 0; nph = ph; nplen = plen;
        } else if (is_bpe && ((ti.flags & B2C_TF_BPE_LEAD) || W.tk_fall[k] || W.tk_ffirst[k] == b)) {       // (ii)
            type = 1; nph = ti.clean_hash; nplen = ti.clean_nchars;
            if (plen) th = b2c_text_append(th, ph);
        } else if (!is_bpe && (ti.flags & B2C_TF_SPACE)) {                                     // (iii)
            type = 2; nph = 0; nplen = 0;
            if (plen) th = b2c_text_append(th, ph);
        } else {                                                                               // (iv)
            type = 3; nph = b2c_hash_append(ph, ti.raw_hash, ti.raw_pow); nplen = plen + ti.raw_nchars;
        }
        C.cth[i] = th;
        C.cph[i] = nph | (static_cast<u64>(type) << 61);
        C.cmeta[i] = (nplen & 0xFFFFu) | (static_cast<u32>(ti.canon) << 16);
        const u64 key = b2c_beam_key(th, nph, nplen, ti.canon);
        C.ckey[i] = key;
        b2c_fence_block();
        b2c_group_insert(C, hmask, static_cast<u32>(i), key);
    }
    B2C_LEADER { sc->max_key = 0; sc->n_sel = 0; }
    B2C_SYNC();
    B2C_MARK(1);

    // ---- phase B: fold scores of each group, LM / hotword fusion, bucket, running max ----------
    {
        u64 tmax = 0;
        B2C_FOR(i, M) {
            const u32 slot = C.cslot[i];
            u32 first, last, cnt;
            b2c_group_extent(C, slot, first, last, cnt);
            if (first != static_cast<u32>(i)) { C.ckey[i] = 0; continue; }
            // members of a group normally share the token; tokens with identical label strings
            // (string compare in the reference) may merge across tokens, so decode every index
            u32 k0, b0, kl, bl;
            b2c_divmod(static_cast<u32>(i), n, rcp_n, k0, b0);
            b2c_divmod(last, n, rcp_n, kl, bl);
            double s = cur.logit[b0] + tk_lp[k0];
            for (u32 j = (cnt == 2) ? last : static_cast<u32>(i) + 1; cnt > 1 && j <= last; ++j) {
                if (C.cslot[j] != slot) continue;
                u32 kj, bj;
                b2c_divmod(j, n, rcp_n, kj, bj);
                s = b2c_sum_log_scores_ool(s, cur.logit[bj] + tk_lp[kj]);
            }
            C.cfold[i] = s;
            C.clast[i] = last;
            const u64 cph = C.cph[last];
            const u32 type = static_cast<u32>(cph >> 61);
            const u32 part_len = C.cmeta[last] & 0xFFFFu;
            double lm_hw = cur.lm_hw[bl];
            if ((type == 1 || type == 2) && cur.part_len[bl] > 0) {
                B2cTextNew tn;
                b2c_text_extend(b2c_lm_of(P, sc), sc->hot, W.text, W.text_cap, cur.text_node[bl], cur.part_hash[bl], cur.part_len[bl], 0, &tn, nullptr);
                lm_hw = tn.lm_hw;
            }
            double ps = 0.0;
            if (type == 0) ps = cur.pscore[bl];
            else if (part_len > 0) ps = b2c_partial_score_of(b2c_lm_of(P, sc), sc->hot, (flags & B2C_FL_PSCORE) != 0, cph & B2C_PH_MASK, part_len);
            const double sco = b2c_combine_score((flags & B2C_FL_LM) != 0, s, lm_hw, ps, part_len);
            const u64 key = b2c_f64_key(sco);
            C.ckey[i] = key;
            const u32 bkt = b2c_bucket_n(ref, sco, bscale, nb);
            b2c_atomic_add_u32(&bcnt[bkt], 1u);
#if defined(__CUDA_ARCH__)
            C.cnext[i] = atomicExch(&bhead[bkt], static_cast<u32>(i));
#else
            C.cnext[i] = bhead[bkt];
            bhead[bkt] = static_cast<u32>(i);
#endif
            if (key > tmax) tmax = key;
        }
        b2c_block_max_u64(tmax, &sc->max_key);
    }
    B2C_SYNC();
    B2C_MARK(2);

    // ---- phase C: threshold (decoder.py:545-546), stable top-N (decoder.py:548): rank = bucket
    //      prefix + exact order inside the bucket; history keys of the selected go to the prune table
    if (nb == B2C_NBUCKET) b2c_bucket_scan_warp(bcnt, bpre);
    else b2c_bucket_scan_block(bcnt, bpre, nb);
    const double max_score = b2c_key_f64(sc->max_key);
    const double thr = max_score + P.prune_logp;
    const u32 width = static_cast<u32>(P.beam_width);
    {
        u32 my_sel = 0;
        B2C_FOR(i, M) {
            const u64 key = C.ckey[i];
            if (key == 0) continue;
            const double sco = b2c_key_f64(key);
            if (!(sco >= thr)) continue;
            const u32 bkt = b2c_bucket_n(ref, sco, bscale, nb);
            u32 rank = bpre[bkt];
            if (rank >= width) continue;          // every candidate of a better bucket outranks it: no need to walk its own
            for (u32 j = bhead[bkt]; j != B2C_NONE_U32;) {      // the candidate itself adds 0; the two loads of a step are
                const u64 kj = C.ckey[j];                        // independent (on the HBM tier: one L2 round trip, not two)
                const u32 jn = C.cnext[j];
                const u32 gt = kj > key ? 1u : 0u, eq_before = (kj == key ? 1u : 0u) & (j < static_cast<u32>(i) ? 1u : 0u);
                rank += gt | eq_before;
                j = jn;
            }
            if (rank >= width) continue;
            ord[rank] = static_cast<u32>(i);
            ++my_sel;
            if (prune) {
                const u32 last = C.clast[i];
                u32 kl, bl;
                b2c_divmod(last, n, rcp_n, kl, bl);
                const u64 cph = C.cph[last];
                const u32 type = static_cast<u32>(cph >> 61);
                const u32 meta = C.cmeta[last];
                u64 hh = cur.hist_hash[bl];
                if ((type == 1 || type == 2) && cur.part_len[bl] > 0)
                    hh = b2c_hist_extend(W.text + cur.text_node[bl], b2c_lm_of(P, sc).hist_n, cur.part_hash[bl]);
                const u64 hk = b2c_beam_key(hh, cph & B2C_PH_MASK, meta & 0xFFFFu, meta >> 16);
                phk[rank] = hk;
                b2c_fence_block();
                u32 slot = static_cast<u32>(b2c_mix64(hk)) & ptmask;
                while (true) {
                    const u32 rep = b2c_atomic_cas_u32(&pt_idx[slot], B2C_NONE_U32, rank);
                    if (rep == B2C_NONE_U32) break;
                    b2c_fence_block();
                    if (phk[rep] == hk) break;
                    slot = (slot + 1) & ptmask;
                }
                pslot[rank] = slot;
                b2c_atomic_min_u32(&pt_min[slot], rank);
            }
        }
        b2c_block_add_u32(my_sel, &sc->n_sel);
    }
    B2C_SYNC();
    B2C_MARK(3);

    // ---- phase D: history prune (decoder.py:550-552) = keep the best rank of every key; every warp
    //      compacts the kept ranks redundantly and commits the blocks of 32 ranks it owns ----------
    const u32 nsel = sc->n_sel;
    u32 n_new = 0;
#if defined(__CUDA_ARCH__)
    {
        const u32 lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
        const u32 lt = (1u << lane) - 1u;
        for (u32 blk = 0; blk * 32 < nsel; ++blk) {
            const u32 r = blk * 32 + lane;
            const bool kept = r < nsel && (!prune || pt_min[pslot[r]] == r);
            const u32 mask = __ballot_sync(0xFFFFFFFFu, kept);
            if (kept && (blk % nw) == w) b2c_commit_one(P, W, C, cur, nx, tk_id, toks_s, n, rcp_n, t, n_new + __popc(mask & lt), r, flags);
            n_new += __popc(mask);
        }
    }
#else
    for (u32 r = 0; r < nsel; ++r) {
        const bool kept = !prune || pt_min[pslot[r]] == r;
        if (kept) b2c_commit_one(P, W, C, cur, nx, tk_id, toks_s, n, rcp_n, t, n_new++, r, flags);
    }
#endif
    // the next frame may take the other tier; this frame dirtied the first hmask + 1 slots of its own
    b2c_prepare_tables(W, n_new * static_cast<u32>(K_next), !kFast && M > W.tier_s.cap && W.tier_g.cap > W.tier_s.cap, hmask + 1, true);
    B2C_LEADER { sc->n_beams = n_new; sc->prev_max = max_score; }
    B2C_SYNC();
    B2C_MARK(4);
    b2c_swap_tabs(W.cur, W.nxt);
}

// -----------------------------------------------------------------------------------------
// single-token frame right after a single-token frame, updated IN PLACE (general kernel; the latency-first kernel
// has its own copy working on its table with holes, b2c_fast_cheap_step in b2c_beam_fast.h, where the argument is
// spelled out): every beam ends in the previous token c', so a frame that selects only c', only the blank, or (no
// LM, no hotwords, regular alphabet) one ordinary character maps every beam to exactly one new beam in the same
// order with the same log-prob added -- no merge, no reordering, no new history-prune victim.  What float64
// rounding could change (order, threshold) is re-checked; on failure the state is untouched and the caller runs the
// general step.  No table swap; leaves the tables clear for the next frame like phase D does.
// -----------------------------------------------------------------------------------------
enum { B2C_INPLACE_NO = 0, B2C_INPLACE_T0 = 1, B2C_INPLACE_T3 = 2, B2C_INPLACE_T3P = 3 };
B2C_HD int b2c_inplace_kind(u32 flags, u32 prev_single, u16 tok_flags, u16 tok_canon) {
    if (prev_single == B2C_NONE_U32) return B2C_INPLACE_NO;
    if ((tok_flags & B2C_TF_BLANK) || prev_single == tok_canon) return B2C_INPLACE_T0;
    if ((flags & B2C_FL_BPE) || (tok_flags & B2C_TF_SPACE)) return B2C_INPLACE_NO;
    // an ordinary character; with LM / hotwords (T3P) the new per-beam scores are computed first and the frame is
    // in place only if they stay in order and above the threshold (same as b2c_fast_scored_step)
    return (flags & B2C_FL_PSCORE) ? B2C_INPLACE_T3P : B2C_INPLACE_T3;
}
// Inline, by reference: an out-of-line copy would take the parameter block and the work descriptor by value (~1 KB of
// local-memory traffic per frame) or force the descriptor into local memory for the whole kernel.
B2C_HD bool b2c_inplace_step(const B2cParams& P, const B2cWork& W, int t, int kind, u16 tok_id, const B2cTok& ti, double p, int K_next) {
    B2cScalars* sc = W.sc;
    const u32 n = sc->n_beams;
    const u32 flags = sc->flags;
    const bool has_lm = (flags & B2C_FL_LM) != 0, plain = (flags & B2C_FL_PSCORE) == 0;
    const B2cBeamTab cur = W.cur;
    const bool scored = kind == B2C_INPLACE_T3P;
    const B2cCandTier Cs = b2c_pick_tier(W, n);        // scratch of the scored form: new lm_score, new partial score
    if (scored) {
        B2C_FOR(b, n) {
            const u64 nph = b2c_hash_append(cur.part_hash[b], ti.raw_hash, ti.raw_pow);
            const u32 nplen = (static_cast<u32>(cur.part_len[b]) + ti.raw_nchars) & 0xFFFFu;
            const double ps = b2c_partial_score_of(b2c_lm_of(P, sc), sc->hot, true, nph, nplen);
            union { double d; u64 u; } c;
            c.d = ps;
            Cs.ckey[b] = c.u;
            Cs.cfold[b] = b2c_combine_score(has_lm, cur.logit[b] + p, cur.lm_hw[b], ps, nplen);
        }
        B2C_SYNC();
    }
    const double top = scored ? Cs.cfold[0]
                              : (plain ? (cur.logit[0] + p) + 0.0
                                       : b2c_combine_score(has_lm, cur.logit[0] + p, cur.lm_hw[0], cur.pscore[0], cur.part_len[0]));
    const double thr = top + P.prune_logp;
    B2C_FOR(b, n) {
        if (scored) {
            const double mine = Cs.cfold[b];
            bool ok = mine >= thr;
            if (static_cast<u32>(b) + 1 < n) ok = ok && mine >= Cs.cfold[b + 1];
            if (!ok) sc->inplace_bad = 1;
            continue;
        }
        if (plain) {      // order is preserved by monotone rounding; only the threshold needs the check
            if (!((cur.logit[b] + p) + 0.0 >= thr)) sc->inplace_bad = 1;
            continue;
        }
        const double mine = b2c_combine_score(has_lm, cur.logit[b] + p, cur.lm_hw[b], cur.pscore[b], cur.part_len[b]);
        bool ok = mine >= thr;
        if (static_cast<u32>(b) + 1 < n) {
            const double next = b2c_combine_score(has_lm, cur.logit[b + 1] + p, cur.lm_hw[b + 1], cur.pscore[b + 1], cur.part_len[b + 1]);
            ok = ok && mine >= next;
        }
        if (!ok) sc->inplace_bad = 1;
    }
    B2C_SYNC();
    if (sc->inplace_bad) {      // block-uniform
        B2C_SYNC();
        B2C_LEADER { sc->inplace_bad = 0; }
        B2C_SYNC();
        return false;
    }
    const bool blank = (ti.flags & B2C_TF_BLANK) != 0;
    const u32 chain_base = sc->chain_used;        // branch (iv): beam b takes node chain_base + b (no per-beam atomic)
    B2C_FOR(b, n) {
        cur.logit[b] = cur.logit[b] + p;
        cur.last_tok[b] = ti.canon;
        if (kind == B2C_INPLACE_T0) {
            if (!blank) cur.pf_e[b] = t + 1;
        } else {
            const int ps0 = cur.pf_s[b], pe0 = cur.pf_e[b];
            cur.part_hash[b] = b2c_hash_append(cur.part_hash[b], ti.raw_hash, ti.raw_pow);
            cur.part_len[b] = static_cast<u16>(cur.part_len[b] + ti.raw_nchars);
            if (scored) {
                union { double d; u64 u; } c;
                c.u = Cs.ckey[b];
                cur.pscore[b] = c.d;
            }
            if (ps0 < 0) cur.pf_s[b] = t;
            cur.pf_e[b] = t + 1;
            const u32 id = chain_base + static_cast<u32>(b);
            if (id < W.chain_cap) {
                B2cChain c;
                c.parent = cur.chain[b];
                c.tok = tok_id;
                c.kind = B2C_CK_CONT;
                c.has_word = 0;
                c.ws = ps0;
                c.we = pe0;
                b2c_chain_store(W.chain, id, c, P.narrow_chain != 0);
                cur.chain[b] = id;
            } else {
                b2c_atomic_or_u32(&sc->status, B2C_ERR_CHAIN_FULL);
            }
        }
    }
    // what phase D of the general step leaves behind: tables clear for the next frame (this step touched neither
    // the grouping table nor the buckets: only what a wider next frame needs beyond the clear extent is swept)
    b2c_prepare_tables(W, n * static_cast<u32>(K_next), false, 0, false);
    B2C_LEADER {
        if (kind != B2C_INPLACE_T0) sc->chain_used = chain_base + n;
        sc->prev_max = top;
        ++sc->m_frames;
        ++sc->m_inplace;
        for (int q = 0; q < 6; ++q)
            if (n > (128u << q)) ++sc->m_over[q];
    }
    B2C_SYNC();
    return true;
}

// frames whose candidate count exceeds the shared-memory tier (a few very wide frames per
// utterance, flat logits) take this out-of-line copy that works on the HBM tier through generic
// pointers.  It operates on a COPY of the work descriptor so that the hot path's descriptor never
// has its address taken (which would push it to local memory).
B2C_HDN void b2c_frame_step_slow(B2cParams P, B2cLayout L, u8* smem, u8* g, int parity, int t, const u32* tk_id,
                                 const double* tk_lp, int K, int K_next) {
    B2cWork Wc;
    b2c_make_work(L, smem, g, parity, true, Wc);
    b2c_frame_step<false>(P, Wc, t, tk_id, tk_lp, K, K_next);   // the caller swaps its own tables
}

// -----------------------------------------------------------------------------------------
// start of an utterance: EMPTY_START_BEAM (decoder.py:130,628) and the root text node
// -----------------------------------------------------------------------------------------
struct B2cStreamIn {           // streaming input of one utterance (n_beams == 0: start from EMPTY_START_BEAM)
    const B2cStreamBeam* beams;
    u32 n_beams;
    const u64* word_hash;
    const u32* word_len;
};
B2C_HDN void b2c_utt_begin(B2cParams P, B2cWork W, int u, const B2cLmState* start_state, int K_first, B2cStreamIn in) {
    const u32 M0 = static_cast<u32>(K_first > 0 ? K_first : 1) * (in.n_beams > 0 ? in.n_beams : 1u);
    {
        const B2cCandTier C0 = b2c_pick_tier(W, M0);
        b2c_clear_tables(W, C0, b2c_ht_size(M0));
    }
    B2C_LEADER {
        B2cScalars* sc = W.sc;
        {   // clear extents of the two grouping tables (b2c_prepare_tables)
            const bool g0 = M0 > W.tier_s.cap && W.tier_g.cap > W.tier_s.cap;
            sc->clean_s = g0 ? 0u : b2c_ht_size(M0);
            sc->clean_g = g0 ? b2c_ht_size(M0) : 0u;
        }
        sc->n_beams = 1;
        sc->chain_used = 0;
        sc->text_used = 1;
        sc->status = B2C_OK;
        sc->force_break = 0;
        sc->inplace_bad = 0;
        sc->prev_max = 0.0;
        sc->hot = P.hot_utt[u];
        sc->lm_set = P.utt_lm[u];
        const B2cLmSet& M = P.lm_sets[sc->lm_set];
        u32 fl = 0;
        if (P.is_bpe) fl |= B2C_FL_BPE;
        if (P.prune_history) fl |= B2C_FL_PRUNE;
        if (M.lm.order > 0) fl |= B2C_FL_LM;
        if (sc->hot.min_len > 0 || M.lm.order > 0) fl |= B2C_FL_PSCORE;
        fl |= static_cast<u32>(P.kflags) & B2C_FL_NO_SINGLE;
        sc->flags = fl;
        B2cText root;
        for (int w = 0; w < B2C_MAX_HIST; ++w) { root.win[w] = 0; root.st.words[w] = 0; root.st.backoff[w] = 0.0f; }
        root.n_win = 0;
        root.hist_hash = B2C_HIST_SEED;
        root.raw_lm = 0.0;
        root.hw_count = 0;
        root.st.length = 0;
        if (M.lm.order > 0) {
            if (start_state) {
                root.st = *start_state;
            } else if (M.score_boundary) {   // BeginSentenceWrite (language_model.py:311-312)
                root.st.length = 1;
                root.st.words[0] = M.lm.bos_id;
                root.st.backoff[0] = M.lm.uni[M.lm.bos_id].backoff;
            }
        }
        W.text[0] = root;
        if (M.n_lm > 1) {       // start states of models 1.. (start_state, if given, holds n_lm consecutive states)
            B2cLmState* x = b2c_text_states_x(W.text, W.text_cap, M.n_lm, 0);
            for (int j = 1; j < M.n_lm; ++j) {
                B2cLmState st;
                st.length = 0;
                for (int w = 0; w < B2C_MAX_HIST; ++w) { st.words[w] = 0; st.backoff[w] = 0.0f; }
                if (start_state) {
                    st = start_state[j];
                } else if (M.lmx[j - 1].score_boundary) {
                    st.length = 1;
                    st.words[0] = M.lmx[j - 1].lm.bos_id;
                    st.backoff[0] = M.lmx[j - 1].lm.uni[M.lmx[j - 1].lm.bos_id].backoff;
                }
                x[j - 1] = st;
            }
        }
        const B2cBeamTab& c = W.cur;
        c.logit[0] = 0.0;
        c.lm_hw[0] = M.lm.order > 0 ? 0.0 : sc->hot.weight * 0;
        c.pscore[0] = 0.0;
        c.text_hash[0] = B2C_TEXT_SEED;
        c.part_hash[0] = 0;
        c.hist_hash[0] = B2C_HIST_SEED;
        c.text_node[0] = 0;
        c.chain[0] = B2C_NONE_U32;
        c.pf_s[0] = -1;
        c.pf_e[0] = -1;
        c.last_tok[0] = B2C_NO_TOK;
        c.part_len[0] = 0;
        if (in.n_beams > 0) {
            sc->n_beams = in.n_beams;
            sc->chain_used = in.n_beams;     // chain nodes [0, n_beams) are the ROOT markers of the input beams
        }
    }
    B2C_SYNC();
    // streaming: the beams of the previous call, in their given (rank) order.  The words of each beam's text are
    // replayed from the start state: text identity, LM state, raw LM score, hotword count and history window come
    // out exactly as if the beam had been decoded in this call (reference: cached_lm_scores carried between calls)
    B2C_FOR(b, in.n_beams) {
        B2cScalars* sc = W.sc;
        const B2cStreamBeam sb = in.beams[b];
        u64 th = B2C_TEXT_SEED, hh = B2C_HIST_SEED;
        u32 node = 0;
        const B2cLmSet& M = b2c_lm_of(P, sc);
        double lm_hw = M.lm.order > 0 ? 0.0 : sc->hot.weight * 0;
        for (u32 w = 0; w < sb.n_words; ++w) {
            const u64 wh = in.word_hash[sb.word_off + w];
            B2cTextCommit tc;
            b2c_commit_text(M, sc->hot, W.text, W.text_cap, &sc->text_used, &sc->status, node, wh, in.word_len[sb.word_off + w], &tc);
            node = tc.node;
            lm_hw = tc.lm_hw;
            hh = tc.hist_hash;
            th = b2c_text_append(th, wh);
        }
        const B2cBeamTab& c = W.cur;
        c.logit[b] = sb.logit;
        c.lm_hw[b] = lm_hw;
        c.pscore[b] = sb.part_len > 0 ? b2c_partial_score_of(M, sc->hot, (sc->flags & B2C_FL_PSCORE) != 0, sb.part_hash, sb.part_len) : 0.0;
        c.text_hash[b] = th;
        c.part_hash[b] = sb.part_hash;
        c.hist_hash[b] = hh;
        c.text_node[b] = node;
        c.chain[b] = static_cast<u32>(b);
        c.pf_s[b] = sb.pf_s;
        c.pf_e[b] = sb.pf_e;
        c.last_tok[b] = static_cast<u16>(sb.last_tok);
        c.part_len[b] = static_cast<u16>(sb.part_len);
        B2cChain root;
        root.parent = B2C_NONE_U32;
        root.tok = static_cast<u16>(b);
        root.kind = B2C_CK_ROOT;
        root.has_word = 0;
        root.ws = -1;
        root.we = -1;
        b2c_chain_store(W.chain, static_cast<u32>(b), root, P.narrow_chain != 0);
    }
    if (in.n_beams > 0) B2C_SYNC();
}

// -----------------------------------------------------------------------------------------
// _finalize_beams(force_next_word=True, is_end=True) + output (decoder.py:558-667); once per
// utterance, out of line
// -----------------------------------------------------------------------------------------
struct B2cOut {              // per-utterance output views (HBM)
    int* n_beams;            // [1]
    int* status;             // [1]
    double* scores;          // [out_beams][2]  logit_score, lm_score
    int* n_tok;              // [out_beams]
    int* n_words;            // [out_beams]
    u32* toks;               // [out_beams][stride]  token | kind << 16, last emission first
    int* frames;             // [out_beams][stride][2] word frames, last word first
    B2cLmState* states;      // [out_beams] LM state after the last word (last_lm_state)
    B2cLmState* states_x;    // [out_beams][P.lm_x] MultiLanguageModel: the other models' states, the first n_lm - 1 of
                             // each beam's row (nullptr when no set of the call has more than one model)
    int* aux;                // [out_beams][4] streaming: input beam the output descends from (-1: none), canonical
                             // token of last_char (-1: None), partial_frames; nullptr outside streaming calls
    u32 stride;              // T + 1
    // text-only calls (P.narrow_chain): no toks / frames / n_words; the transcript of beam r ends at the end of its
    // region [r, r + 1) * stride * P.text_node_bytes of `text`, its length in bytes goes to n_tok[r]
    u8* text;
};

// The transcript of one beam, walked from its newest node and written backwards so that it ends at `end`; the same bytes
// as joining the beam's non-empty words with one space (a word: the clean piece of its BPE node, if any, then its CONT
// labels; SPACE and BPE nodes end the word before them).  Returns its length.  Out of line: finalize only.
B2C_HDN u32 b2c_walk_text(const B2cChain* chain, u32 node, u32 max_nodes, const B2cPiece* pieces, u8* end) {
    const u8* bytes = reinterpret_cast<const u8*>(pieces);
    const u64* nodes = reinterpret_cast<const u64*>(chain);      // the 8-byte nodes of b2c_chain_store
    u8* p = end;
    bool open = false;           // the word being written (its last bytes first) has a byte
    u64 v = node != B2C_NONE_U32 ? nodes[node] : 0;
    for (u32 nt = 0; node != B2C_NONE_U32 && nt < max_nodes; ++nt) {
        const u32 parent = static_cast<u32>(v), tok = static_cast<u16>(v >> 32), kind = static_cast<u8>(v >> 48);
        if (kind == B2C_CK_ROOT) break;
        // the parent's load goes out before this node's piece is copied: the chase of parent pointers (HBM latency
        // per node) stays the only serial chain of the walk
        const u64 pv = parent != B2C_NONE_U32 ? nodes[parent] : 0;
        if (kind != B2C_CK_SPACE) {
            const B2cPiece pc = pieces[2u * tok + (kind == B2C_CK_BPE ? 1u : 0u)];
            if (pc.len) {
                if (!open && p != end) *--p = ' ';      // a later word is written already
                p -= pc.len;
                for (u32 i = 0; i < pc.len; ++i) p[i] = bytes[pc.off + i];
                open = true;
            }
        }
        if (kind != B2C_CK_CONT) open = false;
        node = parent;
        v = pv;
    }
    return static_cast<u32>(end - p);
}

B2C_HDN void b2c_finalize(B2cParams P, B2cWork W, B2cOut O, int fin_mode) {
    const bool keep = fin_mode == B2C_FIN_KEEP;
    const int is_eos = fin_mode == B2C_FIN_EOS ? 1 : 0;
    // on entry the grouping table is clear for ht_size(n_beams) slots (last phase D / utt_begin)
    B2cScalars* sc = W.sc;
    const B2cLmSet& M = b2c_lm_of(P, sc);
    const u32 n = sc->n_beams;
    const B2cCandTier C = b2c_pick_tier(W, n);
    const u32 hmask = b2c_ht_size(n) - 1;
    const B2cBeamTab cur = W.cur;
    B2C_FOR(b, n) {
        // B2C_FIN_KEEP: new_beams = list(beams), nothing merges (decoder.py:592-593): one group per beam
        const u64 th = cur.part_len[b] ? b2c_text_append(cur.text_hash[b], cur.part_hash[b]) : cur.text_hash[b];
        const u64 key = keep ? b2c_beam_key(b2c_mix64(static_cast<u64>(b) + 1), 1, 0, B2C_NO_TOK) : b2c_beam_key(th, 0, 0, B2C_NO_TOK);
        C.ckey[b] = key;
        b2c_fence_block();
        b2c_group_insert(C, hmask, static_cast<u32>(b), key);
    }
    B2C_LEADER { sc->max_key = 0; sc->n_sel = 0; }
    B2C_SYNC();
    B2C_FOR(b, n) {
        const u32 slot = C.cslot[b];
        u32 first, last, cnt;
        b2c_group_extent(C, slot, first, last, cnt);
        if (first != static_cast<u32>(b)) { C.ckey[b] = 0; continue; }
        double s = cur.logit[b];
        for (u32 j = static_cast<u32>(b) + 1; j <= last; ++j)
            if (C.cslot[j] == slot) s = b2c_sum_log_scores(s, cur.logit[j]);
        C.cfold[b] = s;
        C.clast[b] = last;
        // the LAST duplicate decides the (text, next_word) split that gets scored with is_eos
        // (decoder.py:387-395: an empty next_word is scored as a word -> <unk>)
        double lm_hw;
        if (keep) {
            lm_hw = cur.lm_hw[last];        // next_word == "": cache hit on (text, False) (decoder.py:387-396)
        } else if ((M.lm.order > 0 && (is_eos || cur.part_len[last] > 0)) || cur.part_len[last] > 0) {
            // is_eos=False with an empty next_word is a cache hit on (text, False) as well
            B2cTextNew tn;
            b2c_text_extend(M, sc->hot, W.text, W.text_cap, cur.text_node[last], cur.part_hash[last], cur.part_len[last], is_eos, &tn, nullptr);
            lm_hw = tn.lm_hw;
        } else {
            lm_hw = cur.lm_hw[last];
        }
        const u64 key = keep ? b2c_f64_key(b2c_combine_score(M.lm.order > 0, s, lm_hw, cur.pscore[last], cur.part_len[last]))
                             : b2c_f64_key(b2c_combine_score(M.lm.order > 0, s, lm_hw, 0.0, 0));
        C.ckey[b] = key;
        b2c_atomic_max_u64(&sc->max_key, key);
    }
    B2C_SYNC();
    const double thr = b2c_key_f64(sc->max_key) + P.prune_logp;
    B2C_FOR(b, n) {
        const u64 key = C.ckey[b];
        if (key == 0) continue;
        if (b2c_key_f64(key) >= thr) b2c_atomic_add_u32(&sc->n_sel, 1u);
        else C.ckey[b] = 0;
    }
    B2C_SYNC();
    // once per utterance: plain counting rank over the survivors
    const u32 m = sc->n_sel;
    const u32 nsel = m < static_cast<u32>(P.beam_width) ? m : static_cast<u32>(P.beam_width);
    B2C_FOR(b, n) {
        const u64 key = C.ckey[b];
        if (key == 0) continue;
        u32 rank = 0;
        for (u32 j = 0; j < n; ++j) {
            const u64 kj = C.ckey[j];
            rank += (kj > key || (kj == key && j < static_cast<u32>(b))) ? 1u : 0u;
        }
        if (rank < nsel) W.ord[rank] = static_cast<u32>(b);
    }
    B2C_SYNC();
    const u32 n_out = nsel < static_cast<u32>(P.out_beams) ? nsel : static_cast<u32>(P.out_beams);
    B2C_LEADER { *O.n_beams = static_cast<int>(n_out); *O.status = static_cast<int>(sc->status); }
    // ---- backtrack: one thread per output beam walks its chain ---------------------------
    B2C_FOR(r, n_out) {
        const u32 b = W.ord[r];
        const u32 last = C.clast[b];
        O.scores[2 * r] = C.cfold[b];
        O.scores[2 * r + 1] = b2c_key_f64(C.ckey[b]);
        B2cLmState st;
        st.length = 0;
        for (int w = 0; w < B2C_MAX_HIST; ++w) { st.words[w] = 0; st.backoff[w] = 0.0f; }
        if (M.lm.order > 0) {
            if (keep || (!is_eos && cur.part_len[last] == 0)) {
                st = W.text[cur.text_node[last]].st;
                if (M.n_lm > 1 && O.states_x) {
                    const B2cLmState* x = b2c_text_states_x(W.text, W.text_cap, M.n_lm, cur.text_node[last]);
                    for (int j = 1; j < M.n_lm; ++j) O.states_x[static_cast<u64>(r) * P.lm_x + (j - 1)] = x[j - 1];
                }
            } else {
                B2cTextNew tn;
                b2c_text_extend(M, sc->hot, W.text, W.text_cap, cur.text_node[last], cur.part_hash[last], cur.part_len[last], is_eos, &tn,
                                (M.n_lm > 1 && O.states_x) ? O.states_x + static_cast<u64>(r) * P.lm_x : nullptr);
                st = tn.st;
            }
        }
        O.states[r] = st;
        if (P.narrow_chain) {
            u8* end = O.text + (static_cast<u64>(r) + 1) * O.stride * P.text_node_bytes;
            const B2cPiece* pieces = reinterpret_cast<const B2cPiece*>(P.toks + P.V);
            O.n_tok[r] = static_cast<int>(b2c_walk_text(W.chain, cur.chain[last], O.stride, pieces, end));
            continue;
        }
        u32* toks = O.toks + static_cast<u64>(r) * O.stride;
        int* frames = O.frames + static_cast<u64>(r) * O.stride * 2;
        u32 nt = 0, nw = 0;
        if (!keep && cur.part_len[last] > 0) {
            frames[0] = cur.pf_s[last];
            frames[1] = cur.pf_e[last];
            nw = 1;
        }
        int root = -1;
        u32 node = cur.chain[last];
        while (node != B2C_NONE_U32 && nt < O.stride) {
            const B2cChain c = b2c_chain_load(W.chain, node, P.narrow_chain != 0);
            if (c.kind == B2C_CK_ROOT) { root = static_cast<int>(c.tok); break; }
            toks[nt++] = static_cast<u32>(c.tok) | (static_cast<u32>(c.kind) << 16);
            if (c.kind != B2C_CK_CONT && c.has_word && nw < O.stride) {
                frames[2 * nw] = c.ws;
                frames[2 * nw + 1] = c.we;
                ++nw;
            }
            node = c.parent;
        }
        O.n_tok[r] = static_cast<int>(nt);
        O.n_words[r] = static_cast<int>(nw);
        if (O.aux) {
            int* a = O.aux + 4 * static_cast<u64>(r);
            a[0] = root;
            a[1] = (keep && cur.last_tok[last] != B2C_NO_TOK) ? static_cast<int>(cur.last_tok[last]) : -1;
            a[2] = keep ? cur.pf_s[last] : -1;
            a[3] = keep ? cur.pf_e[last] : -1;
        }
    }
    // leave the tables clear for the next utterance handled by this CTA (utt_begin clears again)
    B2C_SYNC();
}
