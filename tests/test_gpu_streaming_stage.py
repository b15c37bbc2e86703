"""The streaming stage's token lists on the H100 (`pytest -m gpu`) against the reference of tests/streaming_stage.py
(bit for bit; float64 input to a few ulp), at every alphabet size and row layout K1 branches on.

Route table (csrc/b2c_prepare.h; which device code a case drives):
  float32, V <= 32, streaming pass    b2c_tokens_tiles_v32 (one lane per row):
      V == 32                         LDS.128 walk over rotated quads, its own tie rule (mixed-V32 "tie" rows, thr p05)
      V != 32                         scalar rotated walk (V = 1 .. 31)
      16-byte aligned tile            bulk copy + mbarrier; otherwise the coalesced load (odd V, dev_offset1)
      NaN / inf rows (V == 32)        fallback to the warp routine (special-V32)
      more than three tokens          fallback to the warp set emulation (mixed "nsel" rows, thr m40 / ninf / clip)
      pipelined host block            the same per chunk over tile_lo / tile_hi (host_block, V = 29, 32)
  float32, V > 32, streaming pass     b2c_tokens_run, one warp per run of 8 frames:
      V % 4 == 0 and aligned rows     b2c_prep_row_f32_fast4 (V = 8 .. 32 take the tile kernel; 36, 64, 128, 1024)
      otherwise                       b2c_prep_row_f32_fast (V = 33, 63, 65, 127, 129, 1023, 1025, 4097; dev_offset1)
      NaN / inf / overflowing rows    b2c_prep_row, warp-cooperative (special)
      thr <= log(1e-15)               thr_all branch (clip, clip_lo, m40, ninf); thr on a float32 log-prob (lp_at/above)
      33 <= V <= 64                   the latency-first beam kernel with its resident label table (B2C_FAST_LT)
      V > 1024                        set_cap growth of the set emulation (V = 1025, 4097 with thr ninf / nsel rows)
  float64 (any V), probability pass   b2c_prep_row: b2c_tokens_run_v32 (V <= 32) / b2c_tokens_run
  probabilities or logits             approximate sums (float32 lanes, double atomics), margin, exact numpy-order pass
                                      (softmax, onehot, isclose_in / isclose_out, cancel; mixed_prob: second pass for
                                      some utterances only)
  device input                        in place (dev_inplace), misaligned (dev_offset1), gather kernel (dev_gather,
                                      float32 and float64), widen kernel (f16 / bf16 device tensors)
"""
import pytest

from tests import streaming_stage, synth

pytestmark = pytest.mark.gpu

CASES = synth.streaming_stage_cases(device_routes=True)


@pytest.fixture(scope="module")
def pkg():
    import __graft_entry__ as g
    g.build()
    import pyctcdecode_b200
    from pyctcdecode_b200 import _lib
    _lib._lib = None  # the real CUDA library, not a test build
    L = _lib.lib()
    assert _lib.library_path() == _lib.DEFAULT_LIBRARY
    if L.b2c_device_count() < 1:
        pytest.skip("no CUDA device on this machine (the GPU tests need one)")
    return pyctcdecode_b200


@pytest.fixture(scope="module")
def orc():
    from oracle import oracle
    oracle.build()
    return oracle


@pytest.fixture(scope="module")
def decoders(pkg):
    cache = {}

    def get(V):
        if V not in cache:
            cache[V] = pkg.build_ctcdecoder(synth.stream_labels(V))
        return cache[V]
    return get


def test_gpu_streaming_stage_case_matrix_covers_every_route():
    names = [c[0] for c in CASES]
    assert len(names) == len(set(names))
    Vs = {c[1] for c in CASES}
    assert set(synth.STREAM_V) <= Vs
    for route in ("host_list", "host_block", "dev_inplace", "dev_offset1", "dev_gather"):
        assert any(c[4] == route for c in CASES), route
    for thr in synth.STREAM_THR:
        assert any(c[5] == thr for c in CASES), thr
    for V in (31, 32, 33, 36, 1024, 1025):           # tile / LDS.128 / _fast / _fast4 / growth: misaligned and aligned
        assert any(c[1] == V and c[4] == "dev_offset1" for c in CASES)
        assert any(c[1] == V and c[4] == "dev_inplace" for c in CASES)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_gpu_streaming_stage_token_lists(pkg, orc, decoders, case, monkeypatch):
    monkeypatch.setenv("B200CTC_PIPELINE", "1")
    monkeypatch.setenv("B200CTC_PIPELINE_ALL", "1")
    V = case[1]
    streaming_stage.run_case(orc, decoders(V), case, fresh_decoder=lambda: pkg.build_ctcdecoder(synth.stream_labels(V)))
