// b200ctc -- host side of the n-gram model: ARPA text -> flat, relocatable tables.
//
// GPU-native replacement for what the reference gets from the third-party kenlm package
// (kenlm.Model(path): reference decoder.py:1074, language_model.py:451) and from
// pygtrie.CharTrie over the unigram list (language_model.py:263).  The result is ONE
// contiguous blob (header + unigram array + n-gram hash table + vocabulary hash table +
// unigram-prefix hash set) that is uploaded to HBM as is and can be broadcast between
// GPUs with a single NCCL call.  Sources: ARPA text (b2c_lm_build) and KenLM binary files of the
// probing model type (b2c_lm_build_kenlm_binary; the format kenlm's build_binary writes by default).
#pragma once
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "b2c_common.h"
#include "b2c_lm.h"

inline u64 b2c_hash_bytes(const char* s, size_t n) {
    u64 h = 0;
    for (size_t i = 0; i < n; ++i)
        h = b2c_addmod61(b2c_mulmod61(h, B2C_HASH_BASE), static_cast<u64>(static_cast<unsigned char>(s[i])) + 1);
    return h;
}
inline u64 b2c_pow_bytes(size_t n) {
    u64 p = 1;
    for (size_t i = 0; i < n; ++i) p = b2c_mulmod61(p, B2C_HASH_BASE);
    return p;
}
inline u32 b2c_utf8_len(const char* s, size_t n) {
    u32 c = 0;
    for (size_t i = 0; i < n; ++i) c += ((static_cast<unsigned char>(s[i]) & 0xC0) != 0x80) ? 1u : 0u;
    return c;
}

struct B2cLmHeader {          // first bytes of the blob
    u64 magic;                // "B2CLM002"
    u64 total_bytes;
    int order;
    u32 bos_id, eos_id, n_vocab;
    int have_unigrams, n_unigrams;
    int key_scheme;           // B2C_KEYS_B2C: keys chained by b2c_ngram_start / _extend (ARPA source);
                              // B2C_KEYS_KENLM: KenLM's own chain (tables taken from a KenLM binary)
    int reserved;
    u64 off_uni, off_ngrams, ngram_mask, off_vocab, vocab_mask, off_prefix, prefix_mask;
    u64 n_ngrams_total;
    u64 counts[B2C_MAX_ORDER + 1];
};
#define B2C_LM_MAGIC 0x3230304D4C433242ull

struct B2cLmHost {
    std::vector<unsigned char> blob;
    std::string path;
    std::string error;
    // host-side dictionaries kept for the python-facing helper API (word in model, etc.)
    std::unordered_map<std::string, u32> vocab;
    std::unordered_set<std::string> unigram_set;

    const B2cLmHeader* header() const { return reinterpret_cast<const B2cLmHeader*>(blob.data()); }

    B2cLmView view(const void* base) const {   // view over a copy of the blob at `base` (host or device)
        const B2cLmHeader* h = header();
        const unsigned char* b = static_cast<const unsigned char*>(base);
        B2cLmView v;
        v.order = h->order;
        v.bos_id = h->bos_id; v.eos_id = h->eos_id; v.n_vocab = h->n_vocab;
        v.have_unigrams = h->have_unigrams; v.n_unigrams = h->n_unigrams;
        v.key_scheme = h->key_scheme; v.pad_view = 0;
        v.uni = reinterpret_cast<const B2cUni*>(b + h->off_uni);
        v.ngrams = reinterpret_cast<const B2cNgram*>(b + h->off_ngrams); v.ngram_mask = h->ngram_mask;
        v.vocab = reinterpret_cast<const B2cVocab*>(b + h->off_vocab); v.vocab_mask = h->vocab_mask;
        v.prefixes = reinterpret_cast<const u64*>(b + h->off_prefix); v.prefix_mask = h->prefix_mask;
        return v;
    }
};

static inline u64 b2c_pow2_at_least(u64 n) {
    u64 p = 16;
    while (p < n) p <<= 1;
    return p;
}

// Splits an ARPA line in place: returns number of whitespace separated fields (pointers into buf)
static inline int b2c_split_fields(char* buf, char** fields, int max_fields) {
    int n = 0;
    char* p = buf;
    while (*p && n < max_fields) {
        while (*p == ' ' || *p == '\t' || *p == '\r' || *p == '\n') ++p;
        if (!*p) break;
        fields[n++] = p;
        while (*p && *p != ' ' && *p != '\t' && *p != '\r' && *p != '\n') ++p;
        if (*p) *p++ = 0;
    }
    return n;
}

// last stage of every source: vocabulary table keyed by the string hash the kernels compute token by token, unigram
// set / prefix set (reference language_model.py:87-103, :263), one contiguous blob.  `table`: the finished
// open-addressing n-gram table (size a power of two), keys in `key_scheme`.
static inline bool b2c_lm_assemble(B2cLmHost& lm, int order, const std::vector<std::string>& id2word, const std::vector<B2cUni>& uni,
                                   const std::vector<B2cNgram>& table, const char* const* unigrams, long n_unigrams, int key_scheme,
                                   const std::vector<u64>& counts) {
    const u32 n_vocab = static_cast<u32>(id2word.size());
    const u64 ng_size = table.size();
    // ---- vocabulary hash + unigram set ------------------------------------------------------
    lm.unigram_set.clear();
    const bool have_uni = (unigrams != nullptr && n_unigrams >= 0);
    if (have_uni) {
        for (long i = 0; i < n_unigrams; ++i) {
            auto it = lm.vocab.find(unigrams[i]);
            if (it != lm.vocab.end() && it->second != 0) lm.unigram_set.insert(unigrams[i]);  // language_model.py:94-95
        }
    }
    const u64 vsize = b2c_pow2_at_least(static_cast<u64>(n_vocab) * 2 + 16);
    std::vector<B2cVocab> vtab(vsize, B2cVocab{0, 0, 0});
    for (u32 w = 1; w < n_vocab; ++w) {   // id 0 (<unk>) is "not in the model" (kenlm __contains__)
        const std::string& s = id2word[w];
        const u64 key = b2c_hash_bytes(s.data(), s.size()) + 1;
        u64 slot = b2c_mix64(key) & (vsize - 1);
        while (vtab[slot].key != 0 && vtab[slot].key != key) slot = (slot + 1) & (vsize - 1);
        if (vtab[slot].key == key) { lm.error = "word hash collision in vocabulary: " + s; return false; }
        vtab[slot].key = key;
        vtab[slot].id = w;
        vtab[slot].flags = lm.unigram_set.count(s) ? 1u : 0u;
    }
    // ---- prefix set over the (filtered) unigrams --------------------------------------------
    std::unordered_set<u64> pref;
    for (const std::string& s : lm.unigram_set) {
        u64 h = 0;
        for (size_t i = 0; i < s.size(); ++i) {
            h = b2c_addmod61(b2c_mulmod61(h, B2C_HASH_BASE), static_cast<u64>(static_cast<unsigned char>(s[i])) + 1);
            const bool boundary = (i + 1 == s.size()) || ((static_cast<unsigned char>(s[i + 1]) & 0xC0) != 0x80);
            if (boundary) pref.insert(h + 1);
        }
    }
    const u64 psize = b2c_pow2_at_least(pref.size() * 2 + 16);
    std::vector<u64> ptab(psize, 0);
    for (u64 key : pref) {
        u64 slot = b2c_mix64(key) & (psize - 1);
        while (ptab[slot] != 0) slot = (slot + 1) & (psize - 1);
        ptab[slot] = key;
    }
    // ---- assemble the blob ------------------------------------------------------------------
    auto align = [](u64 x) { return (x + 255) & ~255ull; };
    B2cLmHeader h;
    std::memset(&h, 0, sizeof(h));
    h.magic = B2C_LM_MAGIC;
    h.order = order;
    auto bos = lm.vocab.find("<s>");
    auto eos = lm.vocab.find("</s>");
    h.bos_id = bos == lm.vocab.end() ? 0 : bos->second;
    h.eos_id = eos == lm.vocab.end() ? 0 : eos->second;
    h.n_vocab = n_vocab;
    h.have_unigrams = have_uni ? 1 : 0;
    h.n_unigrams = static_cast<int>(lm.unigram_set.size());
    h.off_uni = align(sizeof(B2cLmHeader));
    h.off_ngrams = align(h.off_uni + sizeof(B2cUni) * n_vocab);
    h.ngram_mask = ng_size - 1;
    h.off_vocab = align(h.off_ngrams + sizeof(B2cNgram) * ng_size);
    h.vocab_mask = vsize - 1;
    h.off_prefix = align(h.off_vocab + sizeof(B2cVocab) * vsize);
    h.prefix_mask = psize - 1;
    h.total_bytes = align(h.off_prefix + sizeof(u64) * psize);
    h.key_scheme = key_scheme;
    h.n_ngrams_total = 0;
    for (int o = 1; o <= order; ++o) { h.counts[o] = counts[o]; h.n_ngrams_total += counts[o]; }
    lm.blob.assign(h.total_bytes, 0);
    std::memcpy(lm.blob.data(), &h, sizeof(h));
    std::memcpy(lm.blob.data() + h.off_uni, uni.data(), sizeof(B2cUni) * n_vocab);
    std::memcpy(lm.blob.data() + h.off_ngrams, table.data(), sizeof(B2cNgram) * ng_size);
    std::memcpy(lm.blob.data() + h.off_vocab, vtab.data(), sizeof(B2cVocab) * vsize);
    std::memcpy(lm.blob.data() + h.off_prefix, ptab.data(), sizeof(u64) * psize);
    return true;
}

// unigrams == nullptr / n_unigrams < 0: "no unigrams given" (reference LanguageModel(unigrams=None))
static inline bool b2c_lm_build(B2cLmHost& lm, const char* arpa_path, const char* const* unigrams, long n_unigrams) {
    lm.path = arpa_path;
    FILE* fp = std::fopen(arpa_path, "rb");
    if (!fp) { lm.error = std::string("cannot open ") + arpa_path; return false; }
    struct Gram { std::vector<u32> ids; float prob, backoff; bool has_bo; };
    std::vector<std::vector<Gram>> grams(B2C_MAX_ORDER + 2);
    lm.vocab.clear();
    lm.vocab.emplace("<unk>", 0u);
    std::vector<std::string> id2word{"<unk>"};
    int order = 0, cur = 0;
    std::vector<char> line(1 << 16);
    char* fields[B2C_MAX_ORDER + 4];
    bool ok = true;
    while (std::fgets(line.data(), static_cast<int>(line.size()), fp)) {
        char* s = line.data();
        while (*s == ' ' || *s == '\t') ++s;
        if (*s == 0 || *s == '\n' || *s == '\r') continue;
        if (*s == '\\') {
            if (std::strstr(s, "-grams:")) {
                cur = std::atoi(s + 1);
                if (cur > B2C_MAX_ORDER) { lm.error = "n-gram order above the supported maximum"; ok = false; break; }
                if (cur > order) order = cur;
            } else if (std::strncmp(s, "\\end\\", 5) == 0) {
                break;
            }
            continue;
        }
        if (cur == 0) continue;  // "ngram N=count" header lines
        int nf = b2c_split_fields(s, fields, cur + 2);
        if (nf < cur + 1) continue;
        Gram g;
        g.prob = static_cast<float>(std::strtod(fields[0], nullptr));
        g.has_bo = nf > cur + 1;
        g.backoff = g.has_bo ? static_cast<float>(std::strtod(fields[cur + 1], nullptr)) : 0.0f;
        g.ids.resize(cur);
        for (int i = 0; i < cur; ++i) {
            auto it = lm.vocab.find(fields[1 + i]);
            if (it == lm.vocab.end()) {
                it = lm.vocab.emplace(fields[1 + i], static_cast<u32>(id2word.size())).first;
                id2word.emplace_back(fields[1 + i]);
            }
            g.ids[i] = it->second;
        }
        grams[cur].push_back(std::move(g));
    }
    std::fclose(fp);
    if (!ok) return false;
    if (order == 0) { lm.error = "no n-gram sections found in ARPA file"; return false; }

    const u32 n_vocab = static_cast<u32>(id2word.size());
    // ---- unigram array ------------------------------------------------------------------
    std::vector<B2cUni> uni(n_vocab, B2cUni{0.0f, 0.0f});
    std::vector<char> uni_present(n_vocab, 0);
    for (const Gram& g : grams[1]) {
        uni[g.ids[0]] = B2cUni{g.prob, g.backoff};
        uni_present[g.ids[0]] = 1;
    }
    if (!uni_present[0]) uni[0] = B2cUni{-100.0f, 0.0f};  // KenLM default for a missing <unk>
    // ---- n-gram table (orders >= 2), keys chained from the LAST word backwards -------------
    u64 n_hi = 0;
    for (int o = 2; o <= order; ++o) n_hi += grams[o].size();
    const u64 ng_size = b2c_pow2_at_least(n_hi * 2 + 16);
    std::vector<B2cNgram> table(ng_size, B2cNgram{0, 0.0f, 0.0f});
    auto key_of = [](const std::vector<u32>& ids, size_t n) {
        u64 h = b2c_ngram_start(ids[n - 1]);
        for (size_t k = 1; k < n; ++k) h = b2c_ngram_extend(h, ids[n - 1 - k]);
        return h;
    };
    auto find_slot = [&](u64 key) -> B2cNgram* {
        u64 slot = b2c_mix64(key) & (ng_size - 1);
        while (table[slot].key != 0 && table[slot].key != key) slot = (slot + 1) & (ng_size - 1);
        return &table[slot];
    };
    for (int o = 2; o <= order; ++o) {
        for (const Gram& g : grams[o]) {
            B2cNgram* e = find_slot(key_of(g.ids, g.ids.size()));
            e->key = key_of(g.ids, g.ids.size());
            e->prob = g.prob;
            e->backoff = g.backoff;
        }
    }
    // ---- extension marks: backoff == -0.0f  <=>  "no extension" (KenLM kNoExtensionBackoff) ----
    // an n-gram has an extension when its backoff is non-zero or it is the context (first n
    // words) of a longer n-gram.
    auto is_zero = [](float f) { return f == 0.0f; };
    const float neg_zero = -0.0f;
    for (u32 w = 0; w < n_vocab; ++w) if (is_zero(uni[w].backoff)) uni[w].backoff = neg_zero;
    for (u64 s = 0; s < ng_size; ++s) if (table[s].key && is_zero(table[s].backoff)) table[s].backoff = neg_zero;
    for (int o = 2; o <= order; ++o) {
        for (const Gram& g : grams[o]) {
            if (o == 2) {
                if (b2c_f32_bits(uni[g.ids[0]].backoff) == 0x80000000u) uni[g.ids[0]].backoff = 0.0f;
            } else {
                B2cNgram* e = find_slot(key_of(g.ids, g.ids.size() - 1));
                if (e->key && b2c_f32_bits(e->backoff) == 0x80000000u) e->backoff = 0.0f;
            }
        }
    }
    std::vector<u64> counts(B2C_MAX_ORDER + 1, 0);
    for (int o = 1; o <= order; ++o) counts[o] = grams[o].size();
    return b2c_lm_assemble(lm, order, id2word, uni, table, unigrams, n_unigrams, B2C_KEYS_B2C, counts);
}

// =========================================================================================
// KenLM binary files (reference decoder.py:1074 kenlm.Model(path) accepts them; language_model.py:422-426 lists the
// extensions .bin / .binary).  Restated from the published layout of kenlm's lm/binary_format.cc, lm/vocab.cc,
// lm/search_hashed.{hh,cc}, util/probing_hash_table.hh (the kenlm package is a third-party dependency that is absent
// from this environment: PARITY UNPINNED against a kenlm-built file -- the reader is pinned by an independent writer
// of the same layout (tests/kenlm_binary.py) and by the self-checks below, which fail loudly on any layout drift):
//   [Sanity 88 B: "mmap lm http://kheafield.com/code format version 5\n\0" padded to 56, 0.0f 1.0f -0.5f, u32 1,
//    u32 max, u64 1]
//   [FixedWidthParameters 20 B: u8 order, f32 probing_multiplier, i32 model_type, u8 has_vocabulary, u32 search_version]
//   [u64 counts[order]]                                   header padded to a multiple of 8
//   [vocabulary: {u32 version, u32 bound} + probing table of {u64 MurmurHash64A(word), u32 index}, 16-byte entries,
//    max(n + 1, multiplier * n) buckets]
//   [unigrams: (counts[0] + 1) x {f32 prob, f32 backoff}, indexed by word]
//   [orders 2 .. N-1: probing tables of {u64 key, f32 prob, f32 backoff};  order N: {u64 key, f32 prob} packed to 12 B]
//   [vocabulary strings: "<unk>\0" then every word in index order, NUL separated]   (has_vocabulary)
// key of an n-gram = CombineWordHash chained from the LAST word backwards (b2c_kenlm_start / _extend); the stored sign
// bit of prob is a flag ("independent left"), the value is -|prob|; backoff -0.0f means "no extension".
// Supported: model_type 0 (probing).  Trie / quantised / rest-cost models are rejected with a message.
// =========================================================================================
static inline u64 b2c_murmur64a(const void* key, size_t len, u64 seed) {
    const u64 m = 0xc6a4a7935bd1e995ull;
    const int r = 47;
    u64 h = seed ^ (len * m);
    const unsigned char* data = static_cast<const unsigned char*>(key);
    const unsigned char* end = data + (len / 8) * 8;
    while (data != end) {
        u64 k;
        std::memcpy(&k, data, 8);
        data += 8;
        k *= m; k ^= k >> r; k *= m;
        h ^= k; h *= m;
    }
    switch (len & 7) {
        case 7: h ^= static_cast<u64>(data[6]) << 48;  // fall through
        case 6: h ^= static_cast<u64>(data[5]) << 40;  // fall through
        case 5: h ^= static_cast<u64>(data[4]) << 32;  // fall through
        case 4: h ^= static_cast<u64>(data[3]) << 24;  // fall through
        case 3: h ^= static_cast<u64>(data[2]) << 16;  // fall through
        case 2: h ^= static_cast<u64>(data[1]) << 8;   // fall through
        case 1: h ^= static_cast<u64>(data[0]); h *= m;
    }
    h ^= h >> r; h *= m; h ^= h >> r;
    return h;
}

#define B2C_KENLM_MAGIC "mmap lm http://kheafield.com/code format version 5\n"

static inline bool b2c_is_kenlm_binary(const char* path) {
    FILE* fp = std::fopen(path, "rb");
    if (!fp) return false;
    char buf[32] = {0};
    const size_t n = std::fread(buf, 1, 28, fp);
    std::fclose(fp);
    return n == 28 && std::memcmp(buf, "mmap lm http://kheafield.com", 28) == 0;
}

static inline u64 b2c_kenlm_buckets(u64 entries, float multiplier) {
    const u64 a = entries + 1, b = static_cast<u64>(multiplier * static_cast<float>(entries));
    return a > b ? a : b;
}

static inline bool b2c_lm_build_kenlm_binary(B2cLmHost& lm, const char* path, const char* const* unigrams, long n_unigrams) {
    lm.path = path;
    FILE* fp = std::fopen(path, "rb");
    if (!fp) { lm.error = std::string("cannot open ") + path; return false; }
    std::fseek(fp, 0, SEEK_END);
    const long fsize_l = std::ftell(fp);
    std::fseek(fp, 0, SEEK_SET);
    if (fsize_l < 128) { std::fclose(fp); lm.error = "KenLM binary: file too short"; return false; }
    const u64 fsize = static_cast<u64>(fsize_l);
    std::vector<unsigned char> file(fsize);
    const size_t got = std::fread(file.data(), 1, fsize, fp);
    std::fclose(fp);
    if (got != fsize) { lm.error = "KenLM binary: short read"; return false; }
    const unsigned char* f = file.data();
    auto fail = [&](const std::string& why) { lm.error = "KenLM binary " + std::string(path) + ": " + why; return false; };
    // ---- Sanity ------------------------------------------------------------------------------------------------
    const size_t magic_len = sizeof(B2C_KENLM_MAGIC);          // including the terminating NUL, as in kenlm
    if (std::memcmp(f, "mmap lm http://kheafield.com/code format version", 48) != 0) return fail("not a KenLM binary");
    if (std::memcmp(f, B2C_KENLM_MAGIC, magic_len) != 0) return fail("unsupported format version (only version 5 is read)");
    const size_t sanity_magic = (magic_len + 7) & ~size_t(7);   // ALIGN8: 56
    float zf, of, mhf;
    u32 one_w, max_w;
    u64 one_u;
    std::memcpy(&zf, f + sanity_magic, 4);
    std::memcpy(&of, f + sanity_magic + 4, 4);
    std::memcpy(&mhf, f + sanity_magic + 8, 4);
    std::memcpy(&one_w, f + sanity_magic + 12, 4);
    std::memcpy(&max_w, f + sanity_magic + 16, 4);
    std::memcpy(&one_u, f + sanity_magic + 24, 8);              // u64 aligned to 8 inside the struct
    if (zf != 0.0f || of != 1.0f || mhf != -0.5f || one_w != 1u || max_w != 0xFFFFFFFFu || one_u != 1ull)
        return fail("sanity block mismatch (file from a machine with another byte order or type sizes)");
    const size_t sanity_size = sanity_magic + 32;               // 88
    // ---- FixedWidthParameters + counts -----------------------------------------------------------------------------
    const unsigned order = f[sanity_size];
    float mult;
    int model_type;
    unsigned search_version;
    std::memcpy(&mult, f + sanity_size + 4, 4);
    std::memcpy(&model_type, f + sanity_size + 8, 4);
    const bool has_vocab = f[sanity_size + 12] != 0;
    std::memcpy(&search_version, f + sanity_size + 16, 4);
    if (order < 2 || order > B2C_MAX_ORDER) return fail("n-gram order " + std::to_string(order) + " outside the supported range 2.." + std::to_string(B2C_MAX_ORDER));
    if (model_type != 0) {
        static const char* names[] = {"probing", "rest-cost probing", "trie", "quantised trie", "array trie", "quantised array trie"};
        return fail(std::string("model type '") + (model_type > 0 && model_type < 6 ? names[model_type] : "unknown") +
                    "' is not supported: rebuild with `build_binary probing` or pass the ARPA file");
    }
    if (!(mult > 1.0f) || mult > 100.0f) return fail("implausible probing multiplier");
    if (!has_vocab) return fail("the file was written without its vocabulary strings; the decoder needs the words");
    const size_t fixed_size = 20;
    std::vector<u64> kcounts(order);
    if (sanity_size + fixed_size + 8ull * order > fsize) return fail("truncated header");
    std::memcpy(kcounts.data(), f + sanity_size + fixed_size, 8ull * order);
    const u64 header_size = (sanity_size + fixed_size + 8ull * order + 7) & ~7ull;
    // ---- section sizes ---------------------------------------------------------------------------------------------
    for (unsigned o = 0; o < order; ++o)
        if (kcounts[o] == 0 || kcounts[o] > (1ull << 40)) return fail("implausible n-gram count");
    const u64 vocab_buckets = b2c_kenlm_buckets(kcounts[0], mult);
    const u64 vocab_size = 8 + vocab_buckets * 16;
    const u64 off_vocab = header_size;
    const u64 off_uni = off_vocab + vocab_size;
    const u64 uni_size = (kcounts[0] + 1) * 8;
    std::vector<u64> off_mid(order), buckets(order, 0);
    u64 cur = off_uni + uni_size;
    for (unsigned n = 2; n < order; ++n) {
        off_mid[n - 1] = cur;
        buckets[n - 1] = b2c_kenlm_buckets(kcounts[n - 1], mult);
        cur += buckets[n - 1] * 16;
    }
    const u64 off_longest = cur;
    buckets[order - 1] = b2c_kenlm_buckets(kcounts[order - 1], mult);
    cur += buckets[order - 1] * 12;
    const u64 off_strings = cur;
    if (off_strings + 6 > fsize) return fail("sections run past the end of the file (layout mismatch)");
    if (std::memcmp(f + off_strings, "<unk>\0", 6) != 0) return fail("vocabulary strings not found where the layout puts them (layout mismatch)");
    // ---- vocabulary strings, index order -----------------------------------------------------------------------------
    std::vector<std::string> id2word;
    {
        u64 p = off_strings;
        while (p < fsize) {
            const void* z = std::memchr(f + p, 0, fsize - p);
            if (!z) break;
            const u64 q = static_cast<u64>(static_cast<const unsigned char*>(z) - f);
            id2word.emplace_back(reinterpret_cast<const char*>(f + p), q - p);
            p = q + 1;
        }
    }
    if (id2word.size() < 2 || id2word.size() > kcounts[0] + 1) return fail("vocabulary string count does not match the unigram count");
    // every word must be in the probing vocabulary under its MurmurHash64A with its index (the buckets are scanned, so
    // the check does not depend on how the table maps a hash to its first bucket)
    {
        u32 bound;
        std::memcpy(&bound, f + off_vocab + 4, 4);
        if (bound != id2word.size()) return fail("vocabulary bound does not match the number of strings");
        const unsigned char* vt = f + off_vocab + 8;
        std::unordered_map<u64, u32> seen;
        seen.reserve(id2word.size() * 2);
        for (u64 b = 0; b < vocab_buckets; ++b) {
            u64 k;
            u32 v;
            std::memcpy(&k, vt + b * 16, 8);
            std::memcpy(&v, vt + b * 16 + 8, 4);
            if (k != 0) seen.emplace(k, v);
        }
        if (seen.size() + 1 != id2word.size()) return fail("vocabulary table entries do not match the number of strings (layout mismatch)");
        for (size_t w = 1; w < id2word.size(); ++w) {
            auto it = seen.find(b2c_murmur64a(id2word[w].data(), id2word[w].size(), 0));
            if (it == seen.end() || it->second != w)
                return fail("word '" + id2word[w] + "' is not in the probing vocabulary under its hash (layout mismatch)");
        }
    }
    lm.vocab.clear();
    for (size_t w = 0; w < id2word.size(); ++w) lm.vocab.emplace(id2word[w], static_cast<u32>(w));
    if (id2word[0] != "<unk>") return fail("index 0 is not <unk>");
    // ---- unigrams ------------------------------------------------------------------------------------------------------
    const u32 n_vocab = static_cast<u32>(id2word.size());
    std::vector<B2cUni> uni(n_vocab);
    for (u32 w = 0; w < n_vocab; ++w) {
        float p, b;
        std::memcpy(&p, f + off_uni + 8ull * w, 4);
        std::memcpy(&b, f + off_uni + 8ull * w + 4, 4);
        uni[w] = B2cUni{-std::fabs(p), b};
    }
    // ---- higher orders: every occupied bucket keeps KenLM's key --------------------------------------------------------
    u64 n_hi = 0;
    for (unsigned n = 2; n <= order; ++n) n_hi += kcounts[n - 1];
    const u64 ng_size = b2c_pow2_at_least(n_hi * 2 + 16);
    std::vector<B2cNgram> table(ng_size, B2cNgram{0, 0.0f, 0.0f});
    u64 inserted = 0;
    auto insert = [&](u64 key, float prob, float backoff) {
        u64 slot = b2c_mix64(key) & (ng_size - 1);
        while (table[slot].key != 0 && table[slot].key != key) slot = (slot + 1) & (ng_size - 1);
        if (table[slot].key == 0) ++inserted;
        table[slot] = B2cNgram{key, prob, backoff};
    };
    const float neg_zero = -0.0f;
    for (unsigned n = 2; n < order; ++n) {
        const unsigned char* t = f + off_mid[n - 1];
        u64 seen = 0;
        for (u64 b = 0; b < buckets[n - 1]; ++b) {
            u64 k;
            float p, bo;
            std::memcpy(&k, t + b * 16, 8);
            if (k == 0) continue;
            std::memcpy(&p, t + b * 16 + 8, 4);
            std::memcpy(&bo, t + b * 16 + 12, 4);
            insert(k, -std::fabs(p), bo);
            ++seen;
        }
        if (seen != kcounts[n - 1]) return fail("order " + std::to_string(n) + ": " + std::to_string(seen) + " occupied buckets for " + std::to_string(kcounts[n - 1]) + " n-grams (layout mismatch)");
    }
    {
        const unsigned char* t = f + off_longest;
        u64 seen = 0;
        for (u64 b = 0; b < buckets[order - 1]; ++b) {
            u64 k;
            float p;
            std::memcpy(&k, t + b * 12, 8);
            if (k == 0) continue;
            std::memcpy(&p, t + b * 12 + 8, 4);
            insert(k, -std::fabs(p), neg_zero);
            ++seen;
        }
        if (seen != kcounts[order - 1]) return fail("order " + std::to_string(order) + ": occupied buckets do not match the n-gram count (layout mismatch)");
    }
    if (inserted != n_hi) return fail("n-gram keys of different orders collide");
    std::vector<u64> counts(B2C_MAX_ORDER + 1, 0);
    counts[1] = n_vocab;
    for (unsigned n = 2; n <= order; ++n) counts[n] = kcounts[n - 1];
    return b2c_lm_assemble(lm, static_cast<int>(order), id2word, uni, table, unigrams, n_unigrams, B2C_KEYS_KENLM, counts);
}
