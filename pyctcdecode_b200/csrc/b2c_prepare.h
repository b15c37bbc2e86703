// b200ctc -- prepare kernel body: input normalisation + per-frame token selection.
//
// One CTA per utterance.  Restates reference decoder.py:756-765 (probabilities vs logits,
// log-softmax, clipping) and decoder.py:444-445 (tokens >= token_min_logp united with the
// argmax, in CPython set iteration order) and writes one compact (token id, log-prob) list
// per frame, so that the beam kernel never touches the [T,V] matrix again.
//
// Streaming and HBM bound: every logit is read from HBM once (the second and third pass of
// a row hit L1/L2), algorithmic bytes per frame = V * sizeof(dtype).
//
// Numerical definition shared with the oracle (oracle/ctc_oracle.cpp normalise_rows):
//   logits branch, float32 (computed IN float32 like the reference, decoder.py:180-197):
//                  d = x - max;  e = b2c_sm_expf(d) (fixed sequence of IEEE operations, b2c_softmath.h);
//                  S = fl32(sum rint(e * 2^32)) * 2^-32 -- an INTEGER sum: exact, independent of the order of
//                  summation, so one lane per row, one warp per row or any other decomposition gives the same bits;
//                  lp = d - b2c_sm_logf(S), clipped in float64 to [log(1e-15), 0];
//   logits branch, float64: d = x - max, S = sum exp(d) in "warp order" (32 lane-strided partial sums, then xor
//                  butterfly 16,8,4,2,1), lp = d - log S (libm / CUDA double exp and log);
//   probs branch   lp = fl_T(log((double)clip(x, fl_T(1e-15), 1)));
//   the branch decision is math.isclose(x.sum(axis=1).mean(), 1) evaluated bit-exactly like numpy does (pairwise
//   summation in the input dtype) -- but only for utterances whose approximate mean row sum is anywhere near 1: the
//   streaming pass accumulates sum(x) and sum(|x|) per utterance, and an utterance with |mean - 1| > 0.01 + 1e-4 *
//   mean|x| cannot be "probabilities" whatever the order of summation (numpy's float32 pairwise error is below
//   2e-6 * mean|x|), so the exact evaluation -- a second read of the utterance -- happens for probability inputs only.
#pragma once
#include "b2c_cta.h"
#include "b2c_softmath.h"

// ---------------------------------------------------------------------------------------
// numpy pairwise summation (numpy/_core/src/umath/loops_utils.h.src, PW_BLOCKSIZE = 128)
// ---------------------------------------------------------------------------------------
template <class T>
B2C_HD T b2c_np_leaf_sum(const T* a, long n) {
    if (n < 8) {
        T res = static_cast<T>(-0.0);
        for (long i = 0; i < n; ++i) res = res + a[i];
        return res;
    }
    T r0 = a[0], r1 = a[1], r2 = a[2], r3 = a[3], r4 = a[4], r5 = a[5], r6 = a[6], r7 = a[7];
    long i;
    for (i = 8; i < n - (n % 8); i += 8) {
        r0 = r0 + a[i + 0]; r1 = r1 + a[i + 1]; r2 = r2 + a[i + 2]; r3 = r3 + a[i + 3];
        r4 = r4 + a[i + 4]; r5 = r5 + a[i + 5]; r6 = r6 + a[i + 6]; r7 = r7 + a[i + 7];
    }
    T res = ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7));
    for (; i < n; ++i) res = res + a[i];
    return res;
}

// full pairwise sum; `leaf` returns the sum of the leaf block [off, off+n) (n <= 128)
struct B2cPwFrame { long off, n; int st; };
template <class T, class LeafFn>
B2C_HD T b2c_np_pairwise_generic(long n, LeafFn leaf) {
    B2cPwFrame stk[48];
    T left[48];
    int sp = 0;
    T ret = static_cast<T>(0);
    stk[0].off = 0; stk[0].n = n; stk[0].st = 0;
    sp = 1;
    while (sp > 0) {
        B2cPwFrame& f = stk[sp - 1];
        if (f.n <= 128) { ret = leaf(f.off, f.n); --sp; continue; }
        long n2 = f.n / 2;
        n2 -= n2 % 8;
        if (f.st == 0) {
            f.st = 1;
            stk[sp].off = f.off; stk[sp].n = n2; stk[sp].st = 0;
            ++sp;
        } else if (f.st == 1) {
            left[sp - 1] = ret;
            f.st = 2;
            stk[sp].off = f.off + n2; stk[sp].n = f.n - n2; stk[sp].st = 0;
            ++sp;
        } else {
            ret = left[sp - 1] + ret;
            --sp;
        }
    }
    return ret;
}
template <class T>
struct B2cLeafDirect {
    const T* a;
    B2C_HD T operator()(long off, long n) const { return b2c_np_leaf_sum(a + off, n); }
};
template <class T>
B2C_HD T b2c_np_pairwise(const T* a, long n) {
    B2cLeafDirect<T> lf;
    lf.a = a;
    return b2c_np_pairwise_generic<T>(n, lf);
}

// math.isclose(x, 1.0) with the default rel_tol=1e-9, abs_tol=0
B2C_HD bool b2c_isclose_one(double x) {
    if (x == 1.0) return true;
    if (!(x - x == 0.0)) return false;  // inf or nan
    double diff = fabs(1.0 - x);
    return (diff <= fabs(1e-9 * 1.0)) || (diff <= fabs(1e-9 * x));
}

// ---------------------------------------------------------------------------------------
// per-element log-probability
// ---------------------------------------------------------------------------------------
template <class T>
B2C_HD double b2c_lp_logit(T x, T m, double ls) {
    const T d = x - m;
    // float32 rows: `ls` holds a float32 value and the subtraction is the float32 one (one rounding); float64: as is
    double lp = sizeof(T) == 4 ? static_cast<double>(B2C_SM_ADD(static_cast<float>(d), -static_cast<float>(ls)))
                               : static_cast<double>(d) - ls;
    if (lp < B2C_LOG_MIN_CLIP) lp = B2C_LOG_MIN_CLIP;
    if (lp > 0.0) lp = 0.0;
    return lp;
}
// the integer addend of one element in the softmax denominator of a float32 row, and the flags of the special values
B2C_HD u64 b2c_sm_quantum(float e, bool& any_nan, bool& any_inf) {
    if (!(e == e)) { any_nan = true; return 0; }
    if (e > 1.0f) { any_inf = true; return 0; }          // only exp(+inf): d <= 0 for finite rows
#if defined(__CUDA_ARCH__)
    return __float2ull_rn(B2C_SM_MUL(e, 4294967296.0f));
#else
    return static_cast<u64>(llrintf(e * 4294967296.0f));
#endif
}
B2C_HD float b2c_sm_finish(u64 q, bool any_nan, bool any_inf) {
    if (any_nan) return b2c_sm_from_bits(0x7FC00000u);
    if (any_inf) return b2c_sm_from_bits(0x7F800000u);
#if defined(__CUDA_ARCH__)
    const float S = B2C_SM_MUL(__ull2float_rn(q), 2.3283064365386963e-10f);
#else
    const float S = static_cast<float>(q) * 2.3283064365386963e-10f;
#endif
    return b2c_sm_logf(S);
}
template <class T>
B2C_HD double b2c_lp_prob(T x) {
    const T lo = static_cast<T>(1e-15);
    T c = x;
    if (c < lo) c = lo;
    if (c > static_cast<T>(1)) c = static_cast<T>(1);
    return static_cast<double>(static_cast<T>(log(static_cast<double>(c))));
}
template <class T>
B2C_HD double b2c_lp(T x, bool is_prob, T m, double ls) { return is_prob ? b2c_lp_prob<T>(x) : b2c_lp_logit<T>(x, m, ls); }

// ---------------------------------------------------------------------------------------
// CPython 3.12 set of small non-negative ints (Objects/setobject.c), tables of u16.
// Two ping-pong buffers of `cap` entries each; 0xFFFF marks an empty slot.
// ---------------------------------------------------------------------------------------
struct B2cPySet {
    u16* buf[2];
    int cur;
    u32 mask, fill;
};
B2C_HD void b2c_pyset_clear(u16* t, u32 size) { for (u32 i = 0; i < size; ++i) t[i] = 0xFFFFu; }
B2C_HD void b2c_pyset_init(B2cPySet& s, u16* b0, u16* b1) {
    s.buf[0] = b0; s.buf[1] = b1; s.cur = 0; s.mask = 7; s.fill = 0;
    b2c_pyset_clear(b0, 8);
}
B2C_HD void b2c_pyset_insert_clean(u16* t, u32 mask, u32 key) {
    u32 perturb = key;
    u32 i = key & mask;
    while (true) {
        if (t[i] == 0xFFFFu) { t[i] = static_cast<u16>(key); return; }
        if (i + 9 <= mask) {
            for (u32 j = 1; j <= 9; ++j)
                if (t[i + j] == 0xFFFFu) { t[i + j] = static_cast<u16>(key); return; }
        }
        perturb >>= 5;
        i = (i * 5 + 1 + perturb) & mask;
    }
}
B2C_HD void b2c_pyset_resize(B2cPySet& s, u32 minused) {
    u32 newsize = 8;
    while (newsize <= minused) newsize <<= 1;
    u16* old = s.buf[s.cur];
    u16* nt = s.buf[s.cur ^ 1];
    b2c_pyset_clear(nt, newsize);
    for (u32 i = 0; i <= s.mask; ++i)
        if (old[i] != 0xFFFFu) b2c_pyset_insert_clean(nt, newsize - 1, old[i]);
    s.cur ^= 1;
    s.mask = newsize - 1;
}
B2C_HD void b2c_pyset_add(B2cPySet& s, u32 key) {
    u16* t = s.buf[s.cur];
    u32 perturb = key;
    u32 i = key & s.mask;
    while (true) {
        const u32 probes = (i + 9 <= s.mask) ? 9u : 0u;
        for (u32 j = 0; j <= probes; ++j) {
            const u16 e = t[i + j];
            if (e == 0xFFFFu) {
                t[i + j] = static_cast<u16>(key);
                ++s.fill;
                if (s.fill * 5 >= s.mask * 3) b2c_pyset_resize(s, s.fill > 50000 ? s.fill * 2 : s.fill * 4);
                return;
            }
            if (e == key) return;
        }
        perturb >>= 5;
        i = (i * 5 + 1 + perturb) & s.mask;
    }
}
// result = copy(s) | {extra}: set_copy (set_merge into an empty set) then set_merge of a 1-element set.
// On return s holds the result; iterate slots 0..mask ascending for the iteration order.
B2C_HD void b2c_pyset_copy_or(B2cPySet& s, u32 extra) {
    // --- copy: new empty table with mask 7 receives all of s
    const u32 used = s.fill;
    u32 nmask = 7;
    if (used > 0) {
        if ((0 + used) * 5 >= nmask * 3) {
            u32 newsize = 8;
            while (newsize <= used * 2) newsize <<= 1;
            nmask = newsize - 1;
        }
        if (nmask != s.mask) {
            // different size: set_insert_clean in slot order of the source
            u16* old = s.buf[s.cur];
            u16* nt = s.buf[s.cur ^ 1];
            b2c_pyset_clear(nt, nmask + 1);
            for (u32 i = 0; i <= s.mask; ++i)
                if (old[i] != 0xFFFFu) b2c_pyset_insert_clean(nt, nmask, old[i]);
            s.cur ^= 1;
            s.mask = nmask;
        }
        // same size: slots are copied verbatim -> nothing to do
    } else {
        b2c_pyset_clear(s.buf[s.cur], 8);
        s.mask = 7;
    }
    // --- merge {extra}
    if ((s.fill + 1) * 5 >= s.mask * 3) b2c_pyset_resize(s, (s.fill + 1) * 2);
    if (s.fill == 0) {
        // empty target, same mask (7) as the one-element source: slot copy
        s.buf[s.cur][extra & 7] = static_cast<u16>(extra);
        s.fill = 1;
        return;
    }
    b2c_pyset_add(s, extra);
}

// ---------------------------------------------------------------------------------------
// kernel bodies.  Three launches:
//   rowsum  -- numpy-order sum of every logit row (coalesced: 8 lanes per row, 4 rows per warp)
//   decide  -- per utterance: numpy-order mean of the row sums, math.isclose(mean, 1)
//   tokens  -- one warp per RUN of 8 consecutive frames of one utterance, persistent grid, no
//              block barrier: log-softmax, clip, token selection, CPython set order, compact lists
// Token lists are compact inside a run; the run starting at frame t0 of utterance u owns the
// entry range beginning at (frame_off[u] + t0) * V.
// ---------------------------------------------------------------------------------------
#define B2C_RUN 8                   // frames per run
#define B2C_PREP_WARPS 8
#define B2C_PREP_SMEM_SET 128       // entries per smem set buffer (enough for 32 selected tokens)
#define B2C_PREP_LEAF_CAP 1024
#define B2C_ROWSUM_MAX_LEAF 64      // rows up to 8192 elements take the coalesced warp-per-row sum

// token list of one frame: offset inside its run, length, and the FIRST token of the list inline (a single-token
// frame -- most frames of ASR posteriors -- is fully described by its 16-byte record: the beam kernel's in-place
// runs never touch the token arrays)
struct B2cFrameRec { u32 off; u16 cnt; u16 id0; double lp0; };

struct B2cPrepArgs {
    const void* logits;      // packed [total_frames, V]
    const u64* frame_off;    // [B]
    const int* T;            // [B]
    const u64* run_off;      // [B+1] exclusive prefix of ceil(T/8)
    int n_utts;
    u64 total_frames;
    int V;
    double token_min_logp;
    const double* utt_token_min_logp;  // [B] per-utterance thresholds (streaming calls that give them), or NULL: token_min_logp
    B2cFrameRec* tok_rec;    // [total_frames]
    u32* tok_ids;            // [total_frames * V]  (32-bit: the beam kernel stages them with 4-byte cp.async)
    double* tok_lp;
    void* rowsum;            // [total_frames] scratch, input dtype (exact numpy row sums, probability-like utterances only)
    u16* set_scratch;        // [total warps][2][set_cap] spill space for large token sets
    u32 set_cap;             // power of two >= 8 * (V + 1)
    int mode;                // 0: streaming pass (every utterance as logits, approximate row sums accumulated);
                             // 1: second pass over the utterances the decide kernel found to be probabilities
    double* approx;          // [B][2] sum of all elements, sum of their absolute values (zeroed before the launch)
    int run_lo, run_hi;      // run-based kernels: runs [run_lo, run_hi) of 8 frames of EVERY utterance are the work items
                             // (utterance = item / (run_hi - run_lo); runs past an utterance's end are skipped)
    int tile_lo, tile_hi;    // lane-per-row kernel (V <= 32): tiles [tile_lo, tile_hi) of 32 frames of EVERY utterance are the
                             // work items (utterance = item / (tile_hi - tile_lo); tiles past an utterance's end are skipped)
    int* is_prob;            // [B]
    u32* max_k;              // [B] largest per-frame token count (zeroed before the launch)
    u32* sum_k;              // [B] total number of selected tokens (zeroed before the launch)
};

// the token threshold of utterance u
B2C_HD double b2c_token_min_of(const B2cPrepArgs& A, int u) { return A.utt_token_min_logp ? A.utt_token_min_logp[u] : A.token_min_logp; }

// ---- rowsum ---------------------------------------------------------------------------------
template <class T>
struct B2cLeafShared {
    const double* sums;
    mutable int next;
    B2C_HD T operator()(long, long) const { return static_cast<T>(sums[next++]); }
};

B2C_HD void b2c_atomic_add_f64(double* p, double v) {
#if defined(__CUDA_ARCH__)
    atomicAdd(p, v);
#else
    *p += v;
#endif
}

// streaming pass: sum(x) and sum(|x|) of `n` consecutive elements (the rows of one run / tile are adjacent) added to
// the utterance's accumulators; one warp, coalesced
template <class T>
B2C_HD void b2c_accum_approx(double* acc, const T* x, long n, int lane) {
#if defined(__CUDA_ARCH__)
    double sx = 0.0, sa = 0.0;
    for (long i = lane; i < n; i += 32) {
        const double v = static_cast<double>(x[i]);
        sx += v;
        sa += fabs(v);
    }
    for (int off = 16; off >= 1; off >>= 1) {
        sx += __shfl_xor_sync(0xFFFFFFFFu, sx, off);
        sa += __shfl_xor_sync(0xFFFFFFFFu, sa, off);
    }
    if (lane == 0) { atomicAdd(acc, sx); atomicAdd(acc + 1, sa); }
#else
    (void)lane;
    double sx = 0.0, sa = 0.0;
    for (long i = 0; i < n; ++i) { sx += static_cast<double>(x[i]); sa += fabs(static_cast<double>(x[i])); }
    acc[0] += sx;
    acc[1] += sa;
#endif
}

// ---- decide ---------------------------------------------------------------------------------
struct B2cDecideShared { double leaf_sum[B2C_PREP_LEAF_CAP]; int far; };

B2C_HD int b2c_count_leaves(long n) {
    long st[48];
    int sp = 0, nl = 0;
    st[sp++] = n;
    while (sp > 0) {
        long q = st[--sp];
        if (q <= 128) { ++nl; continue; }
        long q2 = q / 2;
        q2 -= q2 % 8;
        st[sp++] = q - q2;
        st[sp++] = q2;
    }
    return nl;
}

template <class T>
B2C_HD void b2c_decide_block(const B2cPrepArgs& A, int u, B2cDecideShared* sh) {
    const int Tn = A.T[u];
    // far from 1 by a margin no order of summation can bridge -> logits, nothing else to do (see the file header)
    B2C_LEADER {
        const double mean = Tn > 0 ? A.approx[2 * u] / Tn : 0.0, mabs = Tn > 0 ? A.approx[2 * u + 1] / Tn : 0.0;
        sh->far = (Tn == 0 || fabs(mean - 1.0) > 0.01 + 1e-4 * mabs) ? 1 : 0;
        if (sh->far) A.is_prob[u] = 0;
    }
    B2C_SYNC();
    if (sh->far) return;
    // exact: numpy-order row sums of this utterance (one row per thread; probability-like input only)
    {
        const T* x = static_cast<const T*>(A.logits) + A.frame_off[u] * static_cast<u64>(A.V);
        T* out = static_cast<T*>(A.rowsum) + A.frame_off[u];
        B2C_FOR(r, Tn) { out[r] = b2c_np_pairwise<T>(x + static_cast<u64>(r) * A.V, A.V); }
    }
    B2C_SYNC();
    const T* rs = static_cast<const T*>(A.rowsum) + A.frame_off[u];
    const int n_leaf = b2c_count_leaves(Tn);
    const bool par_leaves = n_leaf <= B2C_PREP_LEAF_CAP && Tn > 128;
    if (par_leaves) {
        B2C_FOR(lf, n_leaf) {
            long off = 0, n = Tn;
            int idx = lf;
            while (n > 128) {
                long n2 = n / 2;
                n2 -= n2 % 8;
                const int nl = b2c_count_leaves(n2);
                if (idx < nl) { n = n2; } else { idx -= nl; off += n2; n = n - n2; }
            }
            sh->leaf_sum[lf] = static_cast<double>(b2c_np_leaf_sum<T>(rs + off, n));
        }
        B2C_SYNC();
    }
    B2C_LEADER {
        int isp = 0;
        if (Tn > 0) {
            T tot;
            if (par_leaves) {
                B2cLeafShared<T> lf;
                lf.sums = sh->leaf_sum;
                lf.next = 0;
                tot = b2c_np_pairwise_generic<T>(Tn, lf);
            } else {
                tot = b2c_np_pairwise<T>(rs, Tn);
            }
            const T mean = tot / static_cast<T>(Tn);
            isp = b2c_isclose_one(static_cast<double>(mean)) ? 1 : 0;
        }
        A.is_prob[u] = isp;
        if (isp) {                                          // the second pass recounts this utterance's tokens
            A.max_k[u] = 0;
            A.sum_k[u] = 0;
            b2c_atomic_or_u32(reinterpret_cast<u32*>(A.approx + 2 * A.n_utts), 1u);     // "some utterance is probabilities"
        }
    }
}

// ---- tokens ---------------------------------------------------------------------------------
struct B2cPrepShared { u16 sets[B2C_PREP_WARPS][2][B2C_PREP_SMEM_SET]; };

// row statistics: max, log-sum-exp, argmax of the clipped log-probs, and the selected set
// fed in ascending order into `set`.  Warp-cooperative on the device, a plain loop in hostsim.
// kMaskOnly (V <= 32): the selected set is returned as a bit mask in nsel_out instead of being inserted
template <class T, bool kMaskOnly>
B2C_HD void b2c_prep_row(const T* row, int V, bool is_prob, double thr, int lane, B2cPySet& set, T& m_out,
                         double& ls_out, int& amax_out, u32& nsel_out) {
#if defined(__CUDA_ARCH__)
    const unsigned full = 0xFFFFFFFFu;
    T m = static_cast<T>(0);
    double ls = 0.0;
    if (!is_prob) {
        bool have = false;
        for (int v = lane; v < V; v += 32) {
            const T x = row[v];
            if (!have || x > m) { m = x; have = true; }
        }
        for (int off = 16; off >= 1; off >>= 1) {
            const T o = __shfl_xor_sync(full, m, off);
            const int oh = __shfl_xor_sync(full, have ? 1 : 0, off);
            if (oh && (!have || o > m)) { m = o; have = true; }
        }
        if (!(static_cast<double>(m) - static_cast<double>(m) == 0.0)) m = static_cast<T>(0);
        if (sizeof(T) == 4) {
            u64 q = 0;
            bool nn = false, ni = false;
            for (int v = lane; v < V; v += 32) q += b2c_sm_quantum(b2c_sm_expf(static_cast<float>(row[v] - m)), nn, ni);
            for (int off = 16; off >= 1; off >>= 1) q += __shfl_xor_sync(full, q, off);
            ls = static_cast<double>(b2c_sm_finish(q, __any_sync(full, nn), __any_sync(full, ni)));
        } else {
            double part = 0.0;
            for (int v = lane; v < V; v += 32) part += exp(static_cast<double>(static_cast<T>(row[v] - m)));
            for (int off = 16; off >= 1; off >>= 1) part = part + __shfl_xor_sync(full, part, off);
            ls = log(part);
        }
    }
    double best = 0.0;
    int besti = -1;
    u32 nsel = 0;
    if (!kMaskOnly && lane == 0) b2c_pyset_init(set, set.buf[0], set.buf[1]);
    for (int base = 0; base < V; base += 32) {
        const int v = base + lane;
        bool sel = false;
        if (v < V) {
            const double lp = b2c_lp<T>(row[v], is_prob, m, ls);
            if (besti < 0 || lp > best) { best = lp; besti = v; }
            sel = lp >= thr;
        }
        unsigned mask = __ballot_sync(full, sel);
        if (kMaskOnly) { nsel = mask; continue; }
        nsel += __popc(mask);
        if (lane == 0) {
            while (mask) {
                const int bit = __ffs(mask) - 1;
                mask &= mask - 1;
                b2c_pyset_add(set, static_cast<u32>(base + bit));
            }
        }
        __syncwarp();
    }
    for (int off = 16; off >= 1; off >>= 1) {
        const double ob = __shfl_xor_sync(full, best, off);
        const int oi = __shfl_xor_sync(full, besti, off);
        if (oi >= 0 && (besti < 0 || ob > best || (ob == best && oi < besti))) { best = ob; besti = oi; }
    }
    m_out = m; ls_out = ls; amax_out = besti; nsel_out = nsel;
#else
    (void)lane;
    T m = static_cast<T>(0);
    double ls = 0.0;
    if (!is_prob) {
        m = row[0];
        for (int v = 1; v < V; ++v) if (row[v] > m) m = row[v];
        if (!(static_cast<double>(m) - static_cast<double>(m) == 0.0)) m = static_cast<T>(0);
        if (sizeof(T) == 4) {
            u64 q = 0;
            bool nn = false, ni = false;
            for (int v = 0; v < V; ++v) q += b2c_sm_quantum(b2c_sm_expf(static_cast<float>(row[v] - m)), nn, ni);
            ls = static_cast<double>(b2c_sm_finish(q, nn, ni));
        } else {
            double part[32];
            for (int l = 0; l < 32; ++l) {
                double s = 0.0;
                for (int v = l; v < V; v += 32) s += exp(static_cast<double>(static_cast<T>(row[v] - m)));
                part[l] = s;
            }
            for (int off = 16; off >= 1; off >>= 1) {
                double nxt[32];
                for (int l = 0; l < 32; ++l) nxt[l] = part[l] + part[l ^ off];
                for (int l = 0; l < 32; ++l) part[l] = nxt[l];
            }
            ls = log(part[0]);
        }
    }
    double best = 0.0;
    int besti = -1;
    u32 nsel = 0;
    if (!kMaskOnly) b2c_pyset_init(set, set.buf[0], set.buf[1]);
    for (int v = 0; v < V; ++v) {
        const double lp = b2c_lp<T>(row[v], is_prob, m, ls);
        if (besti < 0 || lp > best) { best = lp; besti = v; }
        if (lp >= thr) {
            if (kMaskOnly) nsel |= 1u << v;
            else { ++nsel; b2c_pyset_add(set, static_cast<u32>(v)); }
        }
    }
    m_out = m; ls_out = ls; amax_out = besti; nsel_out = nsel;
#endif
}

#if defined(__CUDA_ARCH__)
// float32 logits, rows WITHOUT NaN / infinity (the common case), one warp per row: the same definition as
// b2c_prep_row -- same maximum, same integer softmax denominator, same float32 log-probabilities, same selected set in
// the same insertion order, same arg-max -- evaluated without the special-value branches and without float64 per element:
//   pass 1  maximum, and sum(x) / sum(|x|) for the probabilities-or-logits decision (a separate read of the run before);
//           a NaN or an infinity makes sum(|x|) non-finite -> return false, the general routine redoes the row
//   pass 2  denominator through b2c_sm_quantum_fast (bit-identical to the definition on this domain)
//   pass 3  float32 comparison against the threshold rounded UP to float32 ((double)lp >= thr <=> lp >= thr_up; the clip
//           at log 1e-15 cannot move the arg-max and matters for the set only when thr is below it: thr_all)
// ~40 warp instructions per 32 elements instead of ~64 (the streaming stage is instruction-bound at V = 1024).
__device__ __forceinline__ bool b2c_prep_row_f32_fast(const float* row, int V, double thr, int lane, B2cPySet& set, float& m_out,
                                                      double& ls_out, int& amax_out, u32& nsel_out, float& sx_out, float& sa_out) {
    const unsigned full = 0xFFFFFFFFu;
    float mx = -3.402823466e38f, sx = 0.0f, sa = 0.0f;
    for (int v = lane; v < V; v += 32) {
        const float x = row[v];
        sx += x;
        sa += fabsf(x);
        mx = fmaxf(mx, x);
    }
    sx_out = sx;
    sa_out = sa;
    if (__any_sync(full, !(sa < 3.0e38f))) return false;
    for (int off = 16; off >= 1; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(full, mx, off));
    const float m = mx;
    u64 q = 0;
    for (int v = lane; v < V; v += 32) q += b2c_sm_quantum_fast(row[v] - m);
    for (int off = 16; off >= 1; off >>= 1) q += __shfl_xor_sync(full, q, off);
    const float lsf = b2c_sm_finish(q, false, false);
    const float thr_up = __double2float_ru(thr);
    const bool thr_all = thr <= B2C_LOG_MIN_CLIP;
    float best = -3.402823466e38f;
    int besti = -1;
    u32 nsel = 0;
    if (lane == 0) b2c_pyset_init(set, set.buf[0], set.buf[1]);
    for (int base = 0; base < V; base += 32) {
        const int v = base + lane;
        bool sel = false;
        if (v < V) {
            const float lp = B2C_SM_ADD(row[v] - m, -lsf);
            if (lp > best || besti < 0) { best = lp; besti = v; }
            sel = thr_all || lp >= thr_up;
        }
        unsigned mask = __ballot_sync(full, sel);
        nsel += __popc(mask);
        if (lane == 0) {
            while (mask) {
                const int bit = __ffs(mask) - 1;
                mask &= mask - 1;
                b2c_pyset_add(set, static_cast<u32>(base + bit));
            }
        }
        __syncwarp();
    }
    for (int off = 16; off >= 1; off >>= 1) {
        const float ob = __shfl_xor_sync(full, best, off);
        const int oi = __shfl_xor_sync(full, besti, off);
        if (oi >= 0 && (besti < 0 || ob > best || (ob == best && oi < besti))) { best = ob; besti = oi; }
    }
    m_out = m;
    ls_out = static_cast<double>(lsf);
    amax_out = besti;
    nsel_out = nsel;
    return true;
}

// The same for rows that are 16-byte aligned with V a multiple of 4: a lane reads FOUR consecutive logits per load
// (v = base + 4 lane + j) -- a quarter of the load instructions, and four independent exp chains per lane hide the
// latency of the dependent fused multiply-adds.  Maximum, sums and the integer denominator do not depend on the order of
// the walk; the selected set is fed in ascending token order from four ballots per 128 tokens (bit L of ballot j is
// token base + 4 L + j), the arg-max keeps the lowest index among equal values.
__device__ __forceinline__ bool b2c_prep_row_f32_fast4(const float* row, int V, double thr, int lane, B2cPySet& set, float& m_out,
                                                       double& ls_out, int& amax_out, u32& nsel_out, float& sx_out, float& sa_out) {
    const unsigned full = 0xFFFFFFFFu;
    const float4* const row4 = reinterpret_cast<const float4*>(row);
    const int V4 = V >> 2;
    float mx = -3.402823466e38f, sx = 0.0f, sa = 0.0f;
    for (int q = lane; q < V4; q += 32) {
        const float4 x = row4[q];
        sx += (x.x + x.y) + (x.z + x.w);
        sa += (fabsf(x.x) + fabsf(x.y)) + (fabsf(x.z) + fabsf(x.w));
        mx = fmaxf(fmaxf(mx, x.x), fmaxf(x.y, fmaxf(x.z, x.w)));
    }
    sx_out = sx;
    sa_out = sa;
    if (__any_sync(full, !(sa < 3.0e38f))) return false;
    for (int off = 16; off >= 1; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(full, mx, off));
    const float m = mx;
    u64 q0 = 0, q1 = 0;
    for (int q = lane; q < V4; q += 32) {
        const float4 x = row4[q];
        q0 += b2c_sm_quantum_fast(x.x - m);
        q1 += b2c_sm_quantum_fast(x.y - m);
        q0 += b2c_sm_quantum_fast(x.z - m);
        q1 += b2c_sm_quantum_fast(x.w - m);
    }
    u64 qs = q0 + q1;
    for (int off = 16; off >= 1; off >>= 1) qs += __shfl_xor_sync(full, qs, off);
    const float lsf = b2c_sm_finish(qs, false, false);
    const float thr_up = __double2float_ru(thr);
    const bool thr_all = thr <= B2C_LOG_MIN_CLIP;
    float best = -3.402823466e38f;
    int besti = -1;
    u32 nsel = 0;
    if (lane == 0) b2c_pyset_init(set, set.buf[0], set.buf[1]);
    for (int base4 = 0; base4 < V4; base4 += 32) {
        const int q = base4 + lane;
        bool s0 = false, s1 = false, s2 = false, s3 = false;
        if (q < V4) {
            const float4 x = row4[q];
            const float l0 = B2C_SM_ADD(x.x - m, -lsf), l1 = B2C_SM_ADD(x.y - m, -lsf), l2 = B2C_SM_ADD(x.z - m, -lsf),
                        l3 = B2C_SM_ADD(x.w - m, -lsf);
            const int v = 4 * q;
            if (l0 > best || besti < 0) { best = l0; besti = v; }
            if (l1 > best) { best = l1; besti = v + 1; }
            if (l2 > best) { best = l2; besti = v + 2; }
            if (l3 > best) { best = l3; besti = v + 3; }
            s0 = thr_all || l0 >= thr_up;
            s1 = thr_all || l1 >= thr_up;
            s2 = thr_all || l2 >= thr_up;
            s3 = thr_all || l3 >= thr_up;
        }
        const unsigned b0 = __ballot_sync(full, s0), b1 = __ballot_sync(full, s1), b2 = __ballot_sync(full, s2), b3 = __ballot_sync(full, s3);
        unsigned any = b0 | b1 | b2 | b3;
        nsel += __popc(b0) + __popc(b1) + __popc(b2) + __popc(b3);
        if (lane == 0) {
            while (any) {
                const int L = __ffs(any) - 1;
                any &= any - 1;
                const u32 v = 4u * static_cast<u32>(base4 + L);
                if ((b0 >> L) & 1u) b2c_pyset_add(set, v);
                if ((b1 >> L) & 1u) b2c_pyset_add(set, v + 1);
                if ((b2 >> L) & 1u) b2c_pyset_add(set, v + 2);
                if ((b3 >> L) & 1u) b2c_pyset_add(set, v + 3);
            }
        }
        __syncwarp();
    }
    for (int off = 16; off >= 1; off >>= 1) {
        const float ob = __shfl_xor_sync(full, best, off);
        const int oi = __shfl_xor_sync(full, besti, off);
        if (oi >= 0 && (besti < 0 || ob > best || (ob == best && oi < besti))) { best = ob; besti = oi; }
    }
    m_out = m;
    ls_out = static_cast<double>(lsf);
    amax_out = besti;
    nsel_out = nsel;
    return true;
}
#endif

// CPython iteration order of set(ascending ints of `mask`) | {amax} for at most 3 selected tokens < 32 with
// amax among them (or none selected): the table keeps its initial 8 slots (no resize below 5 entries, the
// linear-probe window i+9 <= mask is never open at mask 7), one byte per slot in a 64-bit register.
// Returns the number of tokens written to out[0..2].
B2C_HD u32 b2c_pyset_small_order(u32 mask, u32 amax, u32* out) {
    if (mask == 0) { out[0] = amax; return 1; }
    u64 tab = ~0ull;
    u32 mm = mask;
    while (mm) {
#if defined(__CUDA_ARCH__)
        const u32 key = static_cast<u32>(__ffs(static_cast<int>(mm)) - 1);
#else
        u32 key = 0;
        while (!((mm >> key) & 1u)) ++key;
#endif
        mm &= mm - 1;
        u32 perturb = key, i = key & 7u;
        while (((tab >> (8 * i)) & 0xFFull) != 0xFFull) {
            perturb >>= 5;
            i = (i * 5 + 1 + perturb) & 7u;
        }
        tab = (tab & ~(0xFFull << (8 * i))) | (static_cast<u64>(key) << (8 * i));
    }
    u32 n = 0;
    for (u32 i = 0; i < 8; ++i) {
        const u32 e = static_cast<u32>((tab >> (8 * i)) & 0xFFull);
        if (e != 0xFFu) out[n++] = e;
    }
    return n;
}

// V <= 32: one run (<= 8 frames) per warp.  Row statistics are warp-wide per frame and leave the frame's
// selected set as a bit mask in lane f; the ordering of the (typically 1-3) tokens, the offsets inside the
// run and the compact writes are then done by 8 lanes in parallel, one frame each.  Frames with more than
// 3 selected tokens go through the general set emulation afterwards, at offsets that are already known.
template <class T>
B2C_HD void b2c_tokens_run_v32(const B2cPrepArgs& A, u64 run, int lane, u16* set0, u16* set1) {
    const u32 per = static_cast<u32>(A.run_hi - A.run_lo);
    const int u = static_cast<int>(run / per);
    const int Tn = A.T[u];
    const int t0 = (A.run_lo + static_cast<int>(run % per)) * B2C_RUN;
    if (t0 >= Tn) return;                                   // a run past the end of a short utterance of a ragged batch
    const int t1 = t0 + B2C_RUN < Tn ? t0 + B2C_RUN : Tn;
    const int nf = t1 - t0;
    const int V = A.V;
    const u64 f0 = A.frame_off[u];
    if (A.mode == 1 && A.is_prob[u] == 0) return;          // second pass: probability utterances only
    const bool is_prob = A.mode == 1;
    const double thr = b2c_token_min_of(A, u);
    const T* x = static_cast<const T*>(A.logits) + f0 * static_cast<u64>(V);
    const u64 base = (f0 + static_cast<u64>(t0)) * static_cast<u64>(V);
    if (A.mode == 0) b2c_accum_approx<T>(A.approx + 2 * u, x + static_cast<u64>(t0) * V, static_cast<long>(nf) * V, lane);
    u32* ids = A.tok_ids + base;
    double* lps = A.tok_lp + base;
    B2cPySet set;
    set.buf[0] = set0;
    set.buf[1] = set1;
#if defined(__CUDA_ARCH__)
    const unsigned full = 0xFFFFFFFFu;
    u32 my_mask = 0, my_amax = 0;
    T my_m = static_cast<T>(0);
    double my_ls = 0.0;
    {
        for (int f = 0; f < nf; ++f) {
            T m;
            double ls;
            int amax;
            u32 mask;
            b2c_prep_row<T, true>(x + static_cast<u64>(t0 + f) * V, V, is_prob, thr, lane, set, m, ls, amax, mask);
            amax = __shfl_sync(full, amax, 0);          // lane 0's view, like the general path
            if (lane == f) { my_mask = mask; my_amax = static_cast<u32>(amax); my_m = m; my_ls = ls; }
        }
    }
    const bool mine = lane < nf;
    const u32 nsel = __popc(my_mask);
    const bool small = nsel == 0 || (nsel <= 3 && ((my_mask >> my_amax) & 1u));
    const u32 cnt = mine ? static_cast<u32>(__popc(my_mask | (1u << my_amax))) : 0u;
    u32 incl = cnt;
    for (int off = 1; off < B2C_RUN; off <<= 1) {
        const u32 o = __shfl_up_sync(full, incl, off);
        if (lane >= off) incl += o;
    }
    const u32 my_off = incl - cnt;
    if (mine) {
        B2cFrameRec rec;
        rec.off = my_off;
        rec.cnt = static_cast<u16>(cnt);
        rec.id0 = 0;
        rec.lp0 = 0.0;
        if (small) {
            const T* row = x + static_cast<u64>(t0 + lane) * V;
            u32 toks[3];
            const u32 n = b2c_pyset_small_order(my_mask, my_amax, toks);
            for (u32 q = 0; q < n; ++q) {
                const double lp = b2c_lp<T>(row[toks[q]], is_prob, my_m, my_ls);
                ids[my_off + q] = toks[q];
                lps[my_off + q] = lp;
                if (q == 0) { rec.id0 = static_cast<u16>(toks[0]); rec.lp0 = lp; }
            }
        }
        A.tok_rec[f0 + static_cast<u64>(t0 + lane)] = rec;     // frames of the general set emulation: first token patched below
    }
    u32 big = __ballot_sync(full, mine && !small);
    while (big) {
        const int f = __ffs(static_cast<int>(big)) - 1;
        big &= big - 1;
        const T* row = x + static_cast<u64>(t0 + f) * V;
        T m;
        double ls;
        int amax;
        u32 ns;
        b2c_prep_row<T, false>(row, V, is_prob, thr, lane, set, m, ls, amax, ns);
        u32 off = __shfl_sync(full, my_off, f);
        if (lane == 0) {
            b2c_pyset_copy_or(set, static_cast<u32>(amax));
            const u16* tab = set.buf[set.cur];
            bool first = true;
            for (u32 s = 0; s <= set.mask; ++s) {
                const u16 tok = tab[s];
                if (tok == 0xFFFFu) continue;
                const double lp = b2c_lp<T>(row[tok], is_prob, m, ls);
                ids[off] = tok;
                lps[off] = lp;
                if (first) {
                    B2cFrameRec* r = A.tok_rec + f0 + static_cast<u64>(t0 + f);
                    r->id0 = tok;
                    r->lp0 = lp;
                    first = false;
                }
                ++off;
            }
        }
        __syncwarp();
    }
    u32 mx = cnt;
    for (int off = 1; off < B2C_RUN; off <<= 1) {
        const u32 o = __shfl_xor_sync(full, mx, off);
        mx = o > mx ? o : mx;
    }
    const u32 total = __shfl_sync(full, incl, B2C_RUN - 1);
    if (lane == 0 && mx > 0) {
        b2c_atomic_max_u32(&A.max_k[u], mx);
        b2c_atomic_add_u32(&A.sum_k[u], total);
    }
#else
    (void)lane;
    u32 off = 0, mx = 0;
    for (int f = 0; f < nf; ++f) {
        const T* row = x + static_cast<u64>(t0 + f) * V;
        T m;
        double ls;
        int amax;
        u32 mask;
        b2c_prep_row<T, true>(row, V, is_prob, thr, 0, set, m, ls, amax, mask);
        u32 nsel = 0;
        for (u32 b = 0; b < 32; ++b) nsel += (mask >> b) & 1u;
        const bool small = nsel == 0 || (nsel <= 3 && ((mask >> amax) & 1u));
        B2cFrameRec rec;
        rec.off = off;
        rec.id0 = 0;
        rec.lp0 = 0.0;
        if (small) {
            u32 toks[3];
            const u32 n = b2c_pyset_small_order(mask, static_cast<u32>(amax), toks);
            for (u32 q = 0; q < n; ++q) {
                ids[off] = toks[q];
                lps[off] = b2c_lp<T>(row[toks[q]], is_prob, m, ls);
                if (q == 0) { rec.id0 = static_cast<u16>(toks[0]); rec.lp0 = lps[off]; }
                ++off;
            }
            rec.cnt = static_cast<u16>(n);
        } else {
            u32 ns;
            b2c_prep_row<T, false>(row, V, is_prob, thr, 0, set, m, ls, amax, ns);
            b2c_pyset_copy_or(set, static_cast<u32>(amax));
            rec.cnt = static_cast<u16>(set.fill);
            const u16* tab = set.buf[set.cur];
            bool first = true;
            for (u32 s2 = 0; s2 <= set.mask; ++s2) {
                const u16 tok = tab[s2];
                if (tok == 0xFFFFu) continue;
                ids[off] = tok;
                lps[off] = b2c_lp<T>(row[tok], is_prob, m, ls);
                if (first) { rec.id0 = tok; rec.lp0 = lps[off]; first = false; }
                ++off;
            }
        }
        A.tok_rec[f0 + static_cast<u64>(t0 + f)] = rec;
        if (rec.cnt > mx) mx = rec.cnt;
    }
    if (mx > 0) {
        b2c_atomic_max_u32(&A.max_k[u], mx);
        b2c_atomic_add_u32(&A.sum_k[u], off);
    }
#endif
}

// one run (<= 8 frames) handled by one warp
template <class T>
B2C_HD void b2c_tokens_run(const B2cPrepArgs& A, u64 run, int lane, u16* set0, u16* set1) {
    // locate the utterance of this run (binary search over the prefix of runs per utterance)
    const u32 per = static_cast<u32>(A.run_hi - A.run_lo);
    const int u = static_cast<int>(run / per);
    const int Tn = A.T[u];
    const int t0 = (A.run_lo + static_cast<int>(run % per)) * B2C_RUN;
    if (t0 >= Tn) return;                                   // a run past the end of a short utterance of a ragged batch
    const int t1 = t0 + B2C_RUN < Tn ? t0 + B2C_RUN : Tn;
    const int V = A.V;
    const u64 f0 = A.frame_off[u];
    if (A.mode == 1 && A.is_prob[u] == 0) return;          // second pass: probability utterances only
    const bool is_prob = A.mode == 1;
    const double thr = b2c_token_min_of(A, u);
    const T* x = static_cast<const T*>(A.logits) + f0 * static_cast<u64>(V);
    const u64 base = (f0 + static_cast<u64>(t0)) * static_cast<u64>(V);
#if defined(__CUDA_ARCH__)
    // float32 streaming pass: the row sums of the probabilities-or-logits decision come out of pass 1 of the fast row
    // routine (float32 per row and lane, float64 across rows) instead of a separate read of the run
    constexpr bool kFastRows = sizeof(T) == 4;
    const bool fast_rows = kFastRows && A.mode == 0;
    double run_sx = 0.0, run_sa = 0.0;
#else
    const bool fast_rows = false;
#endif
    if (A.mode == 0 && !fast_rows) b2c_accum_approx<T>(A.approx + 2 * u, x + static_cast<u64>(t0) * V, static_cast<long>(t1 - t0) * V, lane);
    u32* ids = A.tok_ids + base;
    double* lps = A.tok_lp + base;
    u32 off = 0, mx = 0;
    for (int t = t0; t < t1; ++t) {
        const T* row = x + static_cast<u64>(t) * V;
        B2cPySet set;
        set.buf[0] = set0;
        set.buf[1] = set1;
        T m;
        double ls;
        int amax;
        u32 nsel;
        bool row_done = false;
#if defined(__CUDA_ARCH__)
        if constexpr (kFastRows) {
            if (fast_rows) {
                float fm, fsx, fsa;
                const float* const frow = reinterpret_cast<const float*>(row);
                const bool vec4 = (V & 3) == 0 && (reinterpret_cast<unsigned long long>(frow) & 15ull) == 0;
                row_done = vec4 ? b2c_prep_row_f32_fast4(frow, V, thr, lane, set, fm, ls, amax, nsel, fsx, fsa)
                                : b2c_prep_row_f32_fast(frow, V, thr, lane, set, fm, ls, amax, nsel, fsx, fsa);
                m = fm;
                run_sx += static_cast<double>(fsx);
                run_sa += static_cast<double>(fsa);
            }
        }
#endif
        if (!row_done) b2c_prep_row<T, false>(row, V, is_prob, thr, lane, set, m, ls, amax, nsel);
        if (lane == 0) {
            b2c_pyset_copy_or(set, static_cast<u32>(amax));
            const u32 cnt = set.fill;
            B2cFrameRec rec;
            rec.off = off;
            rec.cnt = static_cast<u16>(cnt);
            rec.id0 = 0;
            rec.lp0 = 0.0;
            const u16* tab = set.buf[set.cur];
            bool first = true;
            for (u32 s = 0; s <= set.mask; ++s) {
                const u16 tok = tab[s];
                if (tok == 0xFFFFu) continue;
                ids[off] = tok;
                lps[off] = b2c_lp<T>(row[tok], is_prob, m, ls);
                if (first) { rec.id0 = tok; rec.lp0 = lps[off]; first = false; }
                ++off;
            }
            A.tok_rec[f0 + static_cast<u64>(t)] = rec;
            if (cnt > mx) mx = cnt;
        }
#if defined(__CUDA_ARCH__)
        __syncwarp();
#endif
    }
    if (lane == 0 && mx > 0) {
        b2c_atomic_max_u32(&A.max_k[u], mx);
        b2c_atomic_add_u32(&A.sum_k[u], off);
    }
#if defined(__CUDA_ARCH__)
    if (fast_rows) {
        for (int o = 16; o >= 1; o >>= 1) {
            run_sx += __shfl_xor_sync(0xFFFFFFFFu, run_sx, o);
            run_sa += __shfl_xor_sync(0xFFFFFFFFu, run_sa, o);
        }
        if (lane == 0) { atomicAdd(A.approx + 2 * u, run_sx); atomicAdd(A.approx + 2 * u + 1, run_sa); }
    }
#endif
}

template <class T>
B2C_HD void b2c_tokens_block(const B2cPrepArgs& A, int block_idx, int n_blocks, B2cPrepShared* sh) {
    const u64 total_runs = static_cast<u64>(A.n_utts) * static_cast<u64>(A.run_hi - A.run_lo);
    const bool small = A.V <= 32;
    if (A.mode == 1 && *reinterpret_cast<const u32*>(A.approx + 2 * A.n_utts) == 0) return;   // no probability input
#if defined(__CUDA_ARCH__)
    const int w = static_cast<int>(threadIdx.x >> 5), lane = static_cast<int>(threadIdx.x & 31);
    const u64 gw = static_cast<u64>(block_idx) * B2C_PREP_WARPS + w;
    const u64 n_warps = static_cast<u64>(n_blocks) * B2C_PREP_WARPS;
    u16* b0 = small ? sh->sets[w][0] : A.set_scratch + (gw * 2 + 0) * A.set_cap;
    u16* b1 = small ? sh->sets[w][1] : A.set_scratch + (gw * 2 + 1) * A.set_cap;
    if (small) { for (u64 run = gw; run < total_runs; run += n_warps) b2c_tokens_run_v32<T>(A, run, lane, b0, b1); }
    else { for (u64 run = gw; run < total_runs; run += n_warps) b2c_tokens_run<T>(A, run, lane, b0, b1); }
#else
    for (int w = 0; w < B2C_PREP_WARPS; ++w) {
        const u64 gw = static_cast<u64>(block_idx) * B2C_PREP_WARPS + w;
        const u64 n_warps = static_cast<u64>(n_blocks) * B2C_PREP_WARPS;
        u16* b0 = small ? sh->sets[w][0] : A.set_scratch + (gw * 2 + 0) * A.set_cap;
        u16* b1 = small ? sh->sets[w][1] : A.set_scratch + (gw * 2 + 1) * A.set_cap;
        for (u64 run = gw; run < total_runs; run += n_warps) {
            if (small) b2c_tokens_run_v32<T>(A, run, 0, b0, b1);
            else b2c_tokens_run<T>(A, run, 0, b0, b1);
        }
    }
#endif
}

// ---------------------------------------------------------------------------------------
// float32 logits, V <= 32: ONE LANE PER ROW.  A warp takes a tile of 32 consecutive frames of one utterance (4 runs);
// the tile (<= 4 KB) is brought into shared memory by ONE bulk asynchronous copy (cp.async.bulk + mbarrier, the next
// tile in flight while the current one is processed; rows that are not 16-byte aligned take a coalesced load
// instead) and every lane walks its own row three times out of shared memory, in an order rotated by its lane index
// so that the 32 lanes hit 32 different banks: maximum, sum of exponentials (an integer sum: the order of the walk
// does not matter, see the file header), log-probabilities / selection mask / arg-max.  No shuffle, no ballot and
// no float64 transcendental per element: ~35 warp instructions per row instead of ~350.  The (typically 1-3)
// selected tokens are ordered like CPython's set iteration and written by the row's lane; frames with more than
// three selected tokens fall back to the warp-cooperative set emulation at offsets that are already known.
// Streaming pass only (mode 0); hostsim and the second pass use b2c_tokens_run_v32.
// ---------------------------------------------------------------------------------------
#define B2C_TILE_WARPS 4
#define B2C_TILE_ROWS 32
#if defined(__CUDACC__)
struct B2cTileShared {
    alignas(128) float tile[B2C_TILE_WARPS][2][B2C_TILE_ROWS * 32];
    alignas(8) u64 mbar[B2C_TILE_WARPS][2];
    u16 sets[B2C_TILE_WARPS][2][B2C_PREP_SMEM_SET];
};

struct B2cTileInfo { int u, t0, nrows; const float* src; u32 bytes; bool bulk; };

__device__ __forceinline__ B2cTileInfo b2c_tile_locate(const B2cPrepArgs& A, u64 item) {
    const u32 per = static_cast<u32>(A.tile_hi - A.tile_lo);
    B2cTileInfo ti;
    ti.u = static_cast<int>(item / per);
    const int Tn = A.T[ti.u];
    ti.t0 = (A.tile_lo + static_cast<int>(item % per)) * B2C_TILE_ROWS;
    ti.nrows = Tn - ti.t0 < B2C_TILE_ROWS ? Tn - ti.t0 : B2C_TILE_ROWS;          // <= 0: past the end of this utterance
    if (ti.nrows < 0) ti.nrows = 0;
    ti.src = static_cast<const float*>(A.logits) + (A.frame_off[ti.u] + static_cast<u64>(ti.t0)) * static_cast<u64>(A.V);
    ti.bytes = static_cast<u32>(ti.nrows) * static_cast<u32>(A.V) * 4u;
    ti.bulk = ti.nrows > 0 && (reinterpret_cast<u64>(ti.src) & 15ull) == 0 && (ti.bytes & 15u) == 0;
    return ti;
}

__device__ __forceinline__ void b2c_tile_issue(const B2cTileInfo& ti, float* dst, u64* mbar, int lane) {
    if (ti.bulk && lane == 0) {
        const u32 bar = static_cast<u32>(__cvta_generic_to_shared(mbar));
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(ti.bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                         static_cast<u32>(__cvta_generic_to_shared(dst))),
                     "l"(ti.src), "r"(ti.bytes), "r"(bar)
                     : "memory");
    }
}
__device__ __forceinline__ void b2c_tile_wait(u64* mbar, u32 parity) {
    const u32 bar = static_cast<u32>(__cvta_generic_to_shared(mbar));
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "B2C_TILE_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra B2C_TILE_DONE;\n"
        "bra B2C_TILE_WAIT;\n"
        "B2C_TILE_DONE:\n"
        "}\n" ::"r"(bar),
        "r"(parity)
        : "memory");
}

__device__ inline void b2c_tokens_tiles_v32(const B2cPrepArgs& A, int block_idx, int n_blocks, B2cTileShared* sh) {
    const unsigned full = 0xFFFFFFFFu;
    const int w = static_cast<int>(threadIdx.x >> 5), lane = static_cast<int>(threadIdx.x & 31);
    const u64 total = static_cast<u64>(A.n_utts) * static_cast<u64>(A.tile_hi - A.tile_lo);
    const u64 gw = static_cast<u64>(block_idx) * B2C_TILE_WARPS + w, n_warps = static_cast<u64>(n_blocks) * B2C_TILE_WARPS;
    const int V = A.V;
    if (lane == 0) {
        for (int b = 0; b < 2; ++b) {
            const u32 bar = static_cast<u32>(__cvta_generic_to_shared(&sh->mbar[w][b]));
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar) : "memory");
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    u32 parity[2] = {0u, 0u};
    int buf = 0;
    if (gw >= total) return;
    B2cTileInfo cur = b2c_tile_locate(A, gw);
    b2c_tile_issue(cur, sh->tile[w][0], &sh->mbar[w][0], lane);
    const int lr = lane % V;                 // rotation of this lane's walk over its row
    for (u64 tile = gw; tile < total; tile += n_warps) {
        B2cTileInfo nxt;
        nxt.nrows = 0;
        const bool has_next = tile + n_warps < total;
        if (has_next) {
            nxt = b2c_tile_locate(A, tile + n_warps);
            b2c_tile_issue(nxt, sh->tile[w][buf ^ 1], &sh->mbar[w][buf ^ 1], lane);
        }
        float* T0 = sh->tile[w][buf];
        if (cur.nrows <= 0) {                 // a tile past the end of a short utterance of a ragged batch
            cur = nxt;
            buf ^= 1;
            continue;
        }
        if (cur.bulk) {
            b2c_tile_wait(&sh->mbar[w][buf], parity[buf]);
            parity[buf] ^= 1u;
        } else {
            const int n = cur.nrows * V;
            for (int i = lane; i < n; i += 32) T0[i] = cur.src[i];
            __syncwarp();
        }
        const double thr = b2c_token_min_of(A, cur.u);      // every row of a tile belongs to one utterance
        // ---- one row per lane ----------------------------------------------------------------------------------
        const bool mine = lane < cur.nrows;
        const float* row = T0 + lane * V;
        u32 mask = 0, amax = 0;
        float m = 0.0f, lsf = 0.0f, sx = 0.0f, sa = 0.0f;
        bool odd_row = false;       // a NaN / infinity in the row: the warp-cooperative general path decides everything
        if (mine) {
            if (V == 32) {
                // rows of exactly 32 float32: four elements per shared-memory access (LDS.128), quads rotated by the
                // lane index (8 lanes of a quarter warp -> 8 different quads -> no bank conflict)
                // pass 1: maximum, sums
                float mx = -3.402823466e38f;
#pragma unroll 2
                for (int qq = 0; qq < 8; ++qq) {
                    const float4 v = *reinterpret_cast<const float4*>(row + 4 * ((qq + lane) & 7));
                    sx += (v.x + v.y) + (v.z + v.w);
                    sa += (fabsf(v.x) + fabsf(v.y)) + (fabsf(v.z) + fabsf(v.w));
                    mx = fmaxf(fmaxf(mx, v.x), fmaxf(v.y, fmaxf(v.z, v.w)));
                }
                odd_row = !(sa < 3.0e38f);                          // NaN or infinity somewhere (or a sum that overflows)
                m = mx;
                // pass 2: softmax denominator, integer sum (order free)
                u64 qs = 0;
#pragma unroll 2
                for (int qq = 0; qq < 8; ++qq) {
                    const float4 v = *reinterpret_cast<const float4*>(row + 4 * ((qq + lane) & 7));
                    // rows with NaN / infinity (odd_row) are redone by the general routine below: the branch-free form
                    // of the definition (bit-identical for finite rows) is enough here
                    qs += b2c_sm_quantum_fast(v.x - m);
                    qs += b2c_sm_quantum_fast(v.y - m);
                    qs += b2c_sm_quantum_fast(v.z - m);
                    qs += b2c_sm_quantum_fast(v.w - m);
                }
                lsf = b2c_sm_finish(qs, false, false);
                // pass 3 in float32: (double)lp >= thr  <=>  lp >= thr rounded up to float32; the clip at log(1e-15)
                // cannot move the arg-max and matters for the mask only when thr is below it (thr_all)
                const float thr_up = __double2float_ru(thr);
                const bool thr_all = thr <= B2C_LOG_MIN_CLIP;
                float best = -3.402823466e38f;
                u32 bi = 32;
#pragma unroll 2
                for (int qq = 0; qq < 8; ++qq) {
                    const u32 j0 = 4u * ((qq + lane) & 7);
                    const float4 v = *reinterpret_cast<const float4*>(row + j0);
                    const float l0 = B2C_SM_ADD(v.x - m, -lsf), l1 = B2C_SM_ADD(v.y - m, -lsf), l2 = B2C_SM_ADD(v.z - m, -lsf),
                                l3 = B2C_SM_ADD(v.w - m, -lsf);
                    const u32 bits = (l0 >= thr_up ? 1u : 0u) | (l1 >= thr_up ? 2u : 0u) | (l2 >= thr_up ? 4u : 0u) | (l3 >= thr_up ? 8u : 0u);
                    mask |= (thr_all ? 15u : bits) << j0;
                    // largest value, lowest index among equals (the quads are visited in a rotated order)
                    if (l0 > best || (l0 == best && j0 < bi)) { best = l0; bi = j0; }
                    if (l1 > best || (l1 == best && j0 + 1 < bi)) { best = l1; bi = j0 + 1; }
                    if (l2 > best || (l2 == best && j0 + 2 < bi)) { best = l2; bi = j0 + 2; }
                    if (l3 > best || (l3 == best && j0 + 3 < bi)) { best = l3; bi = j0 + 3; }
                }
                amax = bi & 31u;
            } else {
            // pass 1: maximum (a NaN in column 0 makes the reference's running maximum NaN -> "not finite" -> 0)
            float mx = -3.402823466e38f;
            bool seen = false;
            for (int q = 0; q < V; ++q) {
                int j = q + lr;
                if (j >= V) j -= V;
                const float x = row[j];
                sx += x;
                sa += fabsf(x);
                if (x == x) { mx = seen ? fmaxf(mx, x) : x; seen = true; }
            }
            const float x0 = row[0];
            m = (x0 == x0 && seen) ? mx : x0;                   // NaN first element: NaN (falls to 0 below)
            if (!(m - m == 0.0f)) m = 0.0f;                     // inf / NaN
            // pass 2: softmax denominator, integer sum (order free)
            u64 qs = 0;
            bool nn = false, ni = false;
            for (int q = 0; q < V; ++q) {
                int j = q + lr;
                if (j >= V) j -= V;
                qs += b2c_sm_quantum(b2c_sm_expf(row[j] - m), nn, ni);
            }
            lsf = b2c_sm_finish(qs, nn, ni);
            // pass 3: log-probabilities, selection mask, arg-max (largest value, lowest index; NaN never wins, a NaN
            // in column 0 keeps index 0 like the reference's sequential scan)
            double best = 0.0;
            int bi = -1;
            bool nan0 = false;
            for (int q = 0; q < V; ++q) {
                int j = q + lr;
                if (j >= V) j -= V;
                double lp = static_cast<double>(B2C_SM_ADD(row[j] - m, -lsf));
                if (lp < B2C_LOG_MIN_CLIP) lp = B2C_LOG_MIN_CLIP;
                if (lp > 0.0) lp = 0.0;
                if (lp >= thr) mask |= 1u << j;
                if (j == 0 && !(lp == lp)) nan0 = true;
                if (lp == lp && (bi < 0 || lp > best || (lp == best && j < bi))) { best = lp; bi = j; }
            }
            amax = (nan0 || bi < 0) ? 0u : static_cast<u32>(bi);
            }
        }
        // ---- approximate row sums of the tile (decide kernel) -------------------------------------------------------
        {
            double dx = static_cast<double>(sx), da = static_cast<double>(sa);
            for (int off = 16; off >= 1; off >>= 1) {
                dx += __shfl_xor_sync(full, dx, off);
                da += __shfl_xor_sync(full, da, off);
            }
            if (lane == 0) { atomicAdd(A.approx + 2 * cur.u, dx); atomicAdd(A.approx + 2 * cur.u + 1, da); }
        }
        // ---- offsets inside each run of 8 frames, records, small token lists ---------------------------------------
        // a row with special values: its statistics come from the warp-cooperative general routine (same definition)
        {
            u32 odd = __ballot_sync(full, mine && odd_row);
            while (odd) {
                const int f = __ffs(static_cast<int>(odd)) - 1;
                odd &= odd - 1;
                B2cPySet tmp;
                tmp.buf[0] = sh->sets[w][0];
                tmp.buf[1] = sh->sets[w][1];
                float gm;
                double gls;
                int gamax;
                u32 gmask;
                b2c_prep_row<float, true>(cur.src + static_cast<u64>(f) * V, V, false, thr, lane, tmp, gm, gls, gamax, gmask);
                gamax = __shfl_sync(full, gamax, 0);
                if (lane == f) { mask = gmask; amax = static_cast<u32>(gamax); m = gm; lsf = static_cast<float>(gls); }
            }
        }
        const u32 nsel = __popc(mask);
        const bool small = nsel == 0 || (nsel <= 3 && ((mask >> amax) & 1u));
        const u32 cnt = mine ? static_cast<u32>(__popc(mask | (1u << amax))) : 0u;
        u32 incl = cnt;
        for (int off = 1; off < B2C_RUN; off <<= 1) {
            const u32 o = __shfl_up_sync(full, incl, off, B2C_RUN);
            if ((lane & (B2C_RUN - 1)) >= off) incl += o;
        }
        const u32 my_off = incl - cnt;
        const u64 f0 = A.frame_off[cur.u];
        const u64 run_base = (f0 + static_cast<u64>(cur.t0 + (lane & ~(B2C_RUN - 1)))) * static_cast<u64>(V);
        if (mine) {
            B2cFrameRec rec;
            rec.off = my_off;
            rec.cnt = static_cast<u16>(cnt);
            rec.id0 = 0;
            rec.lp0 = 0.0;
            if (small) {
                u32 toks[3];
                const u32 n = b2c_pyset_small_order(mask, amax, toks);
                for (u32 q = 0; q < n; ++q) {
                    const double lp = b2c_lp_logit<float>(row[toks[q]], m, static_cast<double>(lsf));
                    A.tok_ids[run_base + my_off + q] = toks[q];
                    A.tok_lp[run_base + my_off + q] = lp;
                    if (q == 0) { rec.id0 = static_cast<u16>(toks[0]); rec.lp0 = lp; }
                }
            }
            A.tok_rec[f0 + static_cast<u64>(cur.t0 + lane)] = rec;       // big frames: first token patched below
        }
        // ---- frames with more than three selected tokens: the general set emulation ---------------------------------
        u32 big = __ballot_sync(full, mine && !small);
        while (big) {
            const int f = __ffs(static_cast<int>(big)) - 1;
            big &= big - 1;
            const float* grow = cur.src + static_cast<u64>(f) * V;
            B2cPySet set;
            set.buf[0] = sh->sets[w][0];
            set.buf[1] = sh->sets[w][1];
            float gm;
            double gls;
            int gamax;
            u32 ns;
            b2c_prep_row<float, false>(grow, V, false, thr, lane, set, gm, gls, gamax, ns);
            u32 off = __shfl_sync(full, my_off, f);
            const u64 rb = (f0 + static_cast<u64>(cur.t0 + (f & ~(B2C_RUN - 1)))) * static_cast<u64>(V);
            if (lane == 0) {
                b2c_pyset_copy_or(set, static_cast<u32>(gamax));
                const u16* tab = set.buf[set.cur];
                bool first = true;
                for (u32 s = 0; s <= set.mask; ++s) {
                    const u16 tok = tab[s];
                    if (tok == 0xFFFFu) continue;
                    const double lp = b2c_lp_logit<float>(grow[tok], gm, gls);
                    A.tok_ids[rb + off] = tok;
                    A.tok_lp[rb + off] = lp;
                    if (first) {
                        B2cFrameRec* r = A.tok_rec + f0 + static_cast<u64>(cur.t0 + f);
                        r->id0 = tok;
                        r->lp0 = lp;
                        first = false;
                    }
                    ++off;
                }
            }
            __syncwarp();
        }
        // ---- token statistics of the utterance (launch planning) -----------------------------------------------------
        {
            u32 mx = cnt, tot = cnt;
            for (int off = 16; off >= 1; off >>= 1) {
                const u32 o = __shfl_xor_sync(full, mx, off);
                mx = o > mx ? o : mx;
                tot += __shfl_xor_sync(full, tot, off);
            }
            if (lane == 0 && mx > 0) {
                atomicMax(&A.max_k[cur.u], mx);
                atomicAdd(&A.sum_k[cur.u], tot);
            }
        }
        __syncwarp();          // every lane is done with this buffer before the copy after next overwrites it
        cur = nxt;
        buf ^= 1;
    }
}
#endif
