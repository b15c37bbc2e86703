"""Token lists of the streaming stage (K1, csrc/b2c_prepare.h) read back from the decoder and checked against a
reference of the same operation.  Shared by tests/test_hostsim_streaming_stage.py and tests/test_gpu_streaming_stage.py.

K1 turns every logit row into the (token id, float64 log-prob) list the beam kernel consumes.  After a normal
decode_beams_batch call, b2c_decoder_last_tokens returns exactly those lists, so every input route (host lists, pipelined
host blocks, device tensors in place, gathered device lists, half-precision widening, the second pass over probability
utterances) is checked on what the beam kernel really read.
"""
import ctypes as C
import math

import numpy as np

from tests import synth

LOG_CLIP = math.log(1e-15)


def last_tokens(dec, n_utts, device=None):
    """What K1 wrote in the decoder's last call: dict of counts [frames], ids / lps [entries], rec_id0 / rec_lp0
    [frames] (the frame records), is_prob [n_utts]."""
    from pyctcdecode_b200 import _lib
    L = _lib.lib()
    h = dec._handle(device)
    nf, ne = C.c_int64(), C.c_int64()
    _lib.check(L.b2c_decoder_last_tokens(h, C.byref(nf), C.byref(ne), None, None, None, None, None, None))
    out = dict(counts=np.zeros(nf.value, np.int32), ids=np.zeros(ne.value, np.uint32), lps=np.zeros(ne.value, np.float64),
               rec_id0=np.zeros(nf.value, np.uint16), rec_lp0=np.zeros(nf.value, np.float64), is_prob=np.zeros(n_utts, np.int32))
    _lib.check(L.b2c_decoder_last_tokens(h, C.byref(nf), C.byref(ne), *[out[k].ctypes.data for k in
                                                                          ("counts", "ids", "lps", "rec_id0", "rec_lp0", "is_prob")]))
    assert ne.value == len(out["ids"])
    return out


def scan_argmax(row):
    """The reference's sequential arg-max (`row[v] > row[best]` from best = 0): the first maximum; a NaN never wins,
    except in column 0 where it stays (np.argmax would return the first NaN instead)."""
    if np.isnan(row[0]) or np.isnan(row).all():
        return 0
    return int(np.nanargmax(row))


def reference(orc, x, thr):
    """Expected K1 output for one utterance `x` ([T, V] float32 / float64, as the device computes on it)."""
    T = x.shape[0]
    with np.errstate(all="ignore"):
        is_prob = T > 0 and math.isclose(x.sum(axis=1).mean(), 1)      # the reference's own rule (decoder.py:702)
    assert orc.looks_like_probs(x) == is_prob, "the oracle's emulation of the probabilities test disagrees with numpy"
    lp = orc.normalise(x)
    counts, ids = [], []
    for t in range(T):
        row = lp[t]
        sel = np.nonzero(row >= thr)[0].tolist()
        order = orc.token_order(sel, scan_argmax(row))
        counts.append(len(order))
        ids.extend(order)
    ids = np.asarray(ids, dtype=np.int64)
    frame_of = np.repeat(np.arange(T), counts) if T else np.zeros(0, np.int64)
    lps = lp[frame_of, ids] if len(ids) else np.zeros(0)
    return is_prob, np.asarray(counts, np.int64), ids, lps, lp


def same_bits(a, b):
    """Element-wise bit equality of float64 arrays, any NaN equal to any NaN."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return (a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))


def close_f64(a, b):
    """float64 log-probs that may differ by CUDA's vs glibc's exp / log in the last bit: within 2^-49 (2 + |b|), a few
    ulp of log S (S <= V) and of the log-prob; NaN equal to NaN."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    with np.errstate(invalid="ignore"):
        return same_bits(a, b) | (np.abs(a - b) <= 2.0 ** -49 * (2.0 + np.abs(b)))


def float64_bound(x, lp32):
    """Check float32 logit rows against plain float64 math that shares nothing with b2c_softmath.h / the oracle.

    lp64 = log-softmax of the float32 input evaluated in float64, clipped to [log 1e-15, 0].  The float32 definition
    (DESIGN section 2) differs from it by at most, per token v of a row with maximum m and exact d_v = x_v - m:
      - d rounded to float32:                                   2^-24 |d_v|
      - log S, with S = sum of the quantised exponentials:
          each term e_w = expf(fl32(d_w)) is within 0.99 ulp (<= 0.99 * 2^-23 relative) of exp(fl32(d_w)), which is
          within 2^-24 |d_w| (relative) of exp(d_w); rounding e_w to a multiple of 2^-32 adds 2^-32 (absolute, at most
          a full quantum); S >= 1 (the maximum contributes 1), so relative to S:
            delta = (sum_w e_w (0.99 * 2^-23 + 2^-24 |d_w|) + V * 2^-32) / S  +  2^-24 (the integer sum rounded to
            float32); log S then moves by at most delta / (1 - delta), and logf adds 0.74 ulp of log S
      - lp = fl32(d - log S):                                   0.5 ulp of lp
    plus 2^-50 (|d_v| + log S + 1) for the float64 evaluation itself.  Clipping both sides to [log 1e-15, 0] cannot
    increase the difference.  Returns (lp64, bound), [T, V] each."""
    x64 = x.astype(np.float64)
    m = x64.max(axis=1, keepdims=True)
    d = x64 - m
    e = np.exp(d)
    S = e.sum(axis=1, keepdims=True)
    ls = np.log(S)
    lp64 = np.clip(d - ls, LOG_CLIP, 0.0)
    V = x.shape[1]
    delta = (np.sum(e * (0.99 * 2.0 ** -23 + 2.0 ** -24 * np.abs(d)), axis=1, keepdims=True) + V * 2.0 ** -32) / S + 2.0 ** -24
    ulp_ls = np.spacing(np.abs(ls).astype(np.float32)).astype(np.float64)
    ulp_lp = np.spacing(np.abs(lp32).astype(np.float32)).astype(np.float64)
    bound = (2.0 ** -24 * np.abs(d) + delta / (1.0 - delta) + 0.74 * ulp_ls + 0.5 * ulp_lp
             + 2.0 ** -50 * (np.abs(d) + ls + 1.0))
    return lp64, bound


def float64_bound_f64(x):
    """The same for float64 rows (libm exp / log, warp-order sum): a few ulp of float64.  d = x - m is one rounding
    (2^-53 |d|), every exp and the log within 1 ulp, the sum of V positive terms within (V - 1) 2^-53 relative."""
    m = x.max(axis=1, keepdims=True)
    d = x - m
    S = np.exp(d).sum(axis=1, keepdims=True)
    ls = np.log(S)
    lp64 = np.clip(d - ls, LOG_CLIP, 0.0)
    V = x.shape[1]
    bound = 4 * 2.0 ** -53 * (np.abs(d) + np.abs(ls) + 1.0) + (V + 2) * 2.0 ** -52
    return lp64, bound


def resolve_threshold(orc, case, xs):
    """A case's token_min_logp and, for the thresholds placed on a float32 log-prob, the (utterance, frame, token) that
    must be selected at the value ("at") and not at the next double above it ("above")."""
    thr = case[5]
    if isinstance(thr, str):
        return synth.STREAM_THR[thr], None
    u = max(range(len(xs)), key=lambda i: xs[i].shape[0])
    lp = orc.normalise(xs[u])
    t = next(t for t in range(3, lp.shape[0]) if ((lp[t] > -6.0) & (lp[t] < -1.0)).any())
    cand = np.nonzero((lp[t] > -6.0) & (lp[t] < -1.0))[0]
    v = int(cand[len(cand) // 2])
    value = float(lp[t, v])
    assert value == float(np.float32(value))
    return (value if thr[1] == "at" else math.nextafter(value, math.inf)), (u, t, v, thr[1] == "at")


def check(orc, xs, thr, tok, timings, pick=None):
    """Assert that the read-back lists `tok` are K1's definition for the utterances `xs` at threshold `thr`: token ids,
    counts, records and the probabilities flag exactly; log-probs bit for bit where K1 computes in float32 (float32,
    float16, bfloat16 input).  float64 input is computed with libm exp / log in the oracle and CUDA's on the device,
    which may differ in the last bit (DESIGN section 2): there the log-probs must agree to a few ulp."""
    exact = xs[0].dtype != np.float64
    n_frames = sum(x.shape[0] for x in xs)
    assert len(tok["counts"]) == n_frames
    k = f = 0
    total = 0
    for u, x in enumerate(xs):
        x = x.astype(np.float32) if x.dtype == np.float16 else x
        T = x.shape[0]
        is_prob, counts, ids, lps, lp = reference(orc, x, thr)
        n = int(counts.sum())
        got_c = tok["counts"][f:f + T]
        got_ids = tok["ids"][k:k + n] if np.array_equal(got_c, counts) else None
        where = "utterance %d (T=%d)" % (u, T)
        assert bool(tok["is_prob"][u]) == is_prob, "%s: is_prob %d, numpy says %s" % (where, tok["is_prob"][u], is_prob)
        if got_ids is None:
            bad = int(np.nonzero(got_c != counts)[0][0])
            raise AssertionError("%s frame %d: %d tokens, expected %d" % (where, bad, got_c[bad], counts[bad]))
        if not np.array_equal(got_ids, ids):
            bad = int(np.nonzero(got_ids != ids)[0][0])
            raise AssertionError("%s: token ids differ at entry %d of the utterance: %r vs %r" % (where, bad, got_ids[max(0, bad - 3):bad + 4],
                                                                                                ids[max(0, bad - 3):bad + 4]))
        got_lps = tok["lps"][k:k + n]
        ok = same_bits(got_lps, lps) if exact else close_f64(got_lps, lps)
        if not ok.all():
            bad = int(np.nonzero(~ok)[0][0])
            raise AssertionError("%s: log-prob of token %d differs: %r vs %r" % (where, ids[bad], got_lps[bad], lps[bad]))
        first = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64) if T else np.zeros(0, np.int64)
        assert np.array_equal(tok["rec_id0"][f:f + T], ids[first]), "%s: frame record's first token" % where
        got0 = tok["rec_lp0"][f:f + T]
        assert (same_bits(got0, lps[first]) if exact else close_f64(got0, lps[first])).all(), "%s: frame record's first log-prob" % where
        if T and not is_prob:
            _check_float64(x, lp, thr, where)
        if pick is not None and pick[0] == u:
            _, t, v, at = pick
            sel = ids[first[t]:first[t] + counts[t]]
            assert (v in sel) == at, "%s frame %d: token %d (log-prob %r) selected=%s at threshold %r" % (where, t, v, lp[t, v], v in sel, thr)
        total += n
        k += n
        f += T
    assert k == len(tok["ids"])
    assert timings["tokens"] == total, (timings["tokens"], total)


def _check_float64(x, lp, thr, where):
    finite = np.isfinite(x).all(axis=1)
    if x.dtype == np.float32:
        with np.errstate(over="ignore", invalid="ignore"):
            finite &= np.isfinite(x.max(axis=1) - x.min(axis=1))
        lp64, bound = float64_bound(x[finite], lp[finite]) if finite.any() else (None, None)
    else:
        with np.errstate(over="ignore", invalid="ignore"):
            finite &= np.isfinite(x.max(axis=1) - x.min(axis=1))
        lp64, bound = float64_bound_f64(x[finite]) if finite.any() else (None, None)
    if lp64 is None:
        return
    err = np.abs(lp[finite] - lp64)
    assert (err <= bound).all(), "%s: |lp - lp64| = %r above the bound %r" % (where, err.max(), bound[err > bound][0])
    # away from the threshold the selection is the float64 one
    clear = np.abs(lp64 - thr) > bound
    sel = lp[finite] >= thr
    assert np.array_equal(sel[clear], (lp64 >= thr)[clear]), "%s: selection differs from float64 math away from the threshold" % where


def _device_inputs(xs, dtype, route):
    """Device tensors for a case: adjacent slices of one tensor (in place; dev_offset1: storage offset one element, so
    no row is 16-byte aligned) or separately placed tensors with gaps between them (the gather kernel)."""
    import torch
    tdt = {"f32": torch.float32, "f64": torch.float64, "f16": torch.float16, "bf16": torch.bfloat16}[dtype]
    host = [torch.from_numpy(np.ascontiguousarray(x)).to(tdt) for x in xs]
    V = xs[0].shape[1]
    Ts = [x.shape[0] for x in xs]
    if route in ("dev_inplace", "dev_offset1"):
        off = 1 if route == "dev_offset1" else 0
        buf = torch.zeros(off + sum(Ts) * V, dtype=tdt, device="cuda")
        flat = buf[off:].view(sum(Ts), V)
        flat.copy_(torch.cat(host).cuda())
        out, o = [], 0
        for T in Ts:
            out.append(flat[o:o + T])
            o += T
        if route == "dev_offset1":
            assert flat.data_ptr() % 16 != 0 and flat.storage_offset() == 1
        else:
            assert flat.data_ptr() % 16 == 0
        return out
    gap = V + 1                                   # one row and one element between utterances: never adjacent
    buf = torch.zeros(sum(Ts) * V + gap * len(Ts), dtype=tdt, device="cuda")
    out, o = [], 0
    for h, T in zip(host, Ts):
        out.append(buf[o:o + T * V].view(T, V))
        out[-1].copy_(h.cuda())
        o += T * V + gap
    assert len(out) > 4
    esz = buf.element_size()
    assert all(b.data_ptr() != a.data_ptr() + a.shape[0] * V * esz for a, b in zip(out[:-1], out[1:]))
    return out


def run_case(orc, dec, case, fresh_decoder=None):
    """Decode the case's batch with beam_width=1 through its input route and check what K1 wrote."""
    name, V, content, dtype, route, _ = case
    xs = synth.stream_case_arrays(case)
    thr, pick = resolve_threshold(orc, case, xs)
    kw = dict(beam_width=1, token_min_logp=thr)
    if route == "host_list":
        if dtype == "bf16":
            import torch
            inp = [torch.from_numpy(x).to(torch.bfloat16) for x in xs]
            assert all(np.array_equal(t.float().numpy(), x, equal_nan=True) for t, x in zip(inp, xs))
        else:
            inp = xs
        dec.decode_beams_batch(None, inp, **kw)
    elif route == "host_block":
        # a fresh decoder: the first call is plain (no hint yet), the second one pipelined, K1 chunk by chunk
        dec = fresh_decoder()
        block = np.stack(xs)
        assert block.dtype == np.float32 and block.shape[1] >= 256
        dec.decode_beams_batch(None, block, **kw)
        plain = dec.last_timings()["launches"]
        dec.decode_beams_batch(None, block, **kw)
        assert dec.last_timings()["launches"] > plain, "the second call of the block was not pipelined"
    else:
        dec.decode_beams_batch(None, _device_inputs(xs, dtype, route), **kw)
    tok = last_tokens(dec, len(xs))
    check(orc, xs, thr, tok, dec.last_timings(), pick)
