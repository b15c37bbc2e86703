"""Per-utterance hotwords (decode_batch / decode_beams_batch with hotwords_list, partial_decode_beams_batch with
hotword_scorer_list), shared by tests/test_gpu_utt_hotwords.py and its hostsim twin.

The contract: utterance i of a batched call returns, bit for bit, what the same decoder returns for that utterance
decoded alone with hotwords=hotwords_list[i] and hotword_weight=hotword_weight_list[i].  `check_contract` asserts it
for both batch calls; `check_oracle` compares the batch with the oracle, called once per group of utterances that
share a set; `differs` counts the utterances whose own lists change the outcome, so that a kernel that ignored the
routing could not pass."""
import numpy as np

from tests import goldens, synth

WEIGHTS = [10.0, 0.0, 4.0, 25.0, 10.0, 7.5]


def workload(name):
    if name == "char":            # V = 32, no language model
        return synth.CharWorkload("B", n_words=400, lm_order=0)
    if name == "char3":           # V = 32, 3-gram model
        return synth.CharWorkload("B", n_words=300, lm_order=3)
    if name == "bpe4":            # BPE V = 1024, 4-gram model (a small C4 shape)
        return synth.BpeWorkload(n_words=3000, lm_order=4, V=1024)
    raise KeyError(name)


def decoder_kwargs(wl):
    return {} if wl.arpa is None else dict(kenlm_model_path=wl.arpa, unigrams=wl.words, alpha=0.5, beta=1.0)


def hot_lists(wl, seeds, T, seed=5):
    """One list per utterance from words of its own truth() plus distractors.  Covers phrases, duplicates, empty,
    whitespace-only and None entries, and one list shared by several utterances; weights differ, 0 included."""
    rng = np.random.default_rng(seed)
    shared = [wl.words[3], wl.words[11] + " " + wl.words[12]]
    lists, weights = [], []
    for i, s in enumerate(seeds):
        truth = wl.truth(s, T).split()
        if i % 5 == 4:
            lists.append(None)
        elif i % 7 == 3:
            lists.append(shared)
        else:
            own = [truth[j] for j in rng.choice(len(truth), size=min(2, len(truth)), replace=False)] if truth else []
            other = [wl.words[int(k)] for k in rng.integers(0, min(len(wl.words), 2000), size=2)]
            entry = own + other
            if i % 3 == 0 and len(entry) >= 2:
                entry = entry + [entry[0] + " " + entry[-1], entry[0], "", "   "]
            lists.append(entry)
        weights.append(WEIGHTS[i % len(WEIGHTS)])
    return lists, weights


def _strip(words):
    return [w.strip() for w in (words or []) if w.strip()]


def _beams(out):
    return [(b.text, [(w, tuple(f)) for w, f in b.text_frames], b.logit_score, b.lm_score) for b in out]


def check_contract(dec, xs, lists, weights, beams=True, texts=True, batch_input=None, **kw):
    """Batched call with per-utterance lists == one call per utterance, bit for bit.  `batch_input` replaces `xs`
    as what the batched calls get (a padded block, a device tensor), with kw["lengths"] if needed.  Returns the
    batched decode_beams_batch results."""
    inp = xs if batch_input is None else batch_input
    got = None
    single_kw = {k: v for k, v in kw.items() if k != "lengths"}
    if beams:
        got = dec.decode_beams_batch(None, inp, hotwords_list=lists, hotword_weight_list=weights, **kw)
        assert len(got) == len(xs)
        for i, x in enumerate(xs):
            ref = dec.decode_beams(x, hotwords=lists[i], hotword_weight=weights[i], **single_kw)
            assert _beams(got[i]) == _beams(ref), "utterance %d (%r, %r) %r" % (i, lists[i], weights[i], kw)
    if texts:
        tkw = {k: v for k, v in kw.items() if k != "prune_history"}
        t = dec.decode_batch(None, inp, hotwords_list=lists, hotword_weight_list=weights, **tkw)
        for i, x in enumerate(xs):
            ref = dec.decode(x, hotwords=lists[i], hotword_weight=weights[i], **{k: v for k, v in single_kw.items() if k != "prune_history"})
            assert t[i] == ref, "utterance %d (%r, %r) %r" % (i, lists[i], weights[i], kw)
    return got


def check_oracle(ora, xs, lists, weights, got, **kw):
    """The batched beams against the oracle, one oracle call per group of utterances sharing (list, weight)."""
    groups = {}
    for i in range(len(xs)):
        groups.setdefault((tuple(_strip(lists[i])), weights[i]), []).append(i)
    for (words, w), idx in groups.items():
        want = ora.decode_beams_batch([xs[i] for i in idx], hotwords=list(words), hotword_weight=w, **kw)
        for i, beams in zip(idx, want):
            exp = [dict(text=b[0], frames=[(wd, s, e) for wd, (s, e) in b[1]], logit_score=b[2], lm_score=b[3]) for b in beams]
            why = goldens.beams_match_tie_aware(exp, _beams(got[i]))
            assert not why, "utterance %d (%r, %r): %s" % (i, words, w, why)


def differs(dec, xs, lists, weights, **kw):
    """Utterances whose per-utterance top text differs both from the decode without hotwords and from the decode
    with the union of every list (at each utterance's own weight)."""
    union = sorted({w for ws in lists for w in _strip(ws)})
    own = dec.decode_batch(None, xs, hotwords_list=lists, hotword_weight_list=weights, **kw)
    plain = dec.decode_batch(None, xs, **kw)
    uni = dec.decode_batch(None, xs, hotwords_list=[union] * len(xs), hotword_weight_list=weights, **kw)
    return sum(1 for a, b, c in zip(own, plain, uni) if a != b and a != c)


def mixed_special_steps(dec, xs, lists, weights, **kw):
    """A no-LM batch in which every other utterance has no list: the counts of the special steps must be the sums of
    the two halves decoded separately (a hotword-free utterance keeps its in-place / sorted / one-token steps)."""
    names = ("inplace_frames", "sorted_frames", "single_frames")
    lists = [None if i % 2 else ws for i, ws in enumerate(lists)]
    dec.decode_beams_batch(None, xs, hotwords_list=lists, hotword_weight_list=weights, **kw)
    mixed = dec.last_timings()
    total = dict.fromkeys(names, 0)
    for half in (0, 1):
        idx = [i for i in range(len(xs)) if i % 2 == half]
        dec.decode_beams_batch(None, [xs[i] for i in idx], hotwords_list=[lists[i] for i in idx],
                               hotword_weight_list=[weights[i] for i in idx], **kw)
        tm = dec.last_timings()
        for k in names:
            total[k] += tm[k]
    assert {k: mixed[k] for k in names} == total
    return total


def stream_chunks(dec, pkg, xs, scorers_per_chunk, bounds, **kw):
    """Streams advanced chunk by chunk through partial_decode_beams_batch(hotword_scorer_list=...) and, one stream
    at a time, through partial_decode_beams: every call's LMBeam lists must be identical."""
    n = len(xs)
    starts = [dec.get_starting_state() for _ in range(n)]
    b_beams = [s[0] for s in starts]
    s_beams = [s[0] for s in starts]
    for c in range(len(bounds) - 1):
        t0, t1 = bounds[c], bounds[c + 1]
        last = c == len(bounds) - 2
        scorers = scorers_per_chunk[c]
        out = dec.partial_decode_beams_batch([x[t0:t1] for x in xs], [s[1] for s in starts], b_beams, [t0] * n,
                                             hotword_scorer_list=scorers, is_end=last, **kw)
        for i in range(n):
            ref = dec.partial_decode_beams(xs[i][t0:t1], starts[i][1], starts[i][2], s_beams[i], t0,
                                           hotword_scorer=scorers[i], is_end=last, **kw)
            assert out[i] == ref, "stream %d chunk %d" % (i, c)
            s_beams[i] = ref
        b_beams = out
    return b_beams


def scorers(pkg, wl, seeds, T, n_chunks):
    """Per-stream HotwordScorers for each chunk: stream 1's scorer changes after the first chunk, stream 2 has none."""
    lists, weights = hot_lists(wl, seeds, T, seed=9)
    base = [pkg.HotwordScorer.build_scorer(ws, weight=w) if ws else None for ws, w in zip(lists, weights)]
    base[2 % len(base)] = None
    out = []
    for c in range(n_chunks):
        cur = list(base)
        if c > 0 and len(cur) > 1:
            cur[1] = pkg.HotwordScorer.build_scorer([wl.words[7], wl.words[8]], weight=15.0)
        out.append(cur)
    return out


def padded(xs):
    """[B, T_max, V] float32 block and lengths of a ragged list."""
    T = max(x.shape[0] for x in xs)
    block = np.zeros((len(xs), T, xs[0].shape[1]), dtype=np.float32)
    for i, x in enumerate(xs):
        block[i, :x.shape[0]] = x
    return block, [x.shape[0] for x in xs]
