"""The state_len 3 decode runs one chunk per warp and packs ceil(N * R / 132) chunks (at most 16) into a CTA, R being the
engine's num_runners (decode.cu, crf_decode_warp_kernel).  Whatever the packing, every chunk must decode exactly as the C
oracle decodes the engine's own scores: moves, sequence, qstring and n_bases.

Fast-topology models have no variable-chunk-size mode (the reference has none for lstm_size 96), so the ragged case here is
a call on fewer chunks than the runner's batch, which leaves the last CTA partly empty."""
import math

import numpy as np
import pytest

from conftest import model_dir, synthetic_scores

pytestmark = pytest.mark.gpu

MAX_CHUNKS_PER_CTA = 16
NUM_SMS = 132


def _chunks_per_cta(N, R):
    return min(MAX_CHUNKS_PER_CTA, max(1, math.ceil(N * R / NUM_SMS)))


def _check(crf_oracle, cfg, scores, got, idx):
    moves, seq, qstr, nb = got
    ref = crf_oracle.decode(scores[idx], clamp_val=5.0 if cfg.clamp else 0.0, q_shift=cfg.qbias, q_scale=cfg.qscale)
    np.testing.assert_array_equal(nb[idx], ref.n_bases)
    np.testing.assert_array_equal(moves[idx], ref.moves)
    np.testing.assert_array_equal(seq[idx], ref.seq_buf)
    np.testing.assert_array_equal(qstr[idx], ref.qstr_buf)


@pytest.mark.parametrize("R", [1, 2, 4, 8])
def test_runner_decode_matches_oracle_at_every_packing(crf_oracle, R):
    from dorado_b200.config import load_model_config
    from dorado_b200.runner import B200Caller, B200ModelRunner
    from dorado_b200.weights import synthetic_weights
    cfg = load_model_config(model_dir("fast"))
    caller = B200Caller(cfg, synthetic_weights(cfg, 42), num_runners=R)
    rng = np.random.default_rng(100 + R)
    # (batch, chunk size, chunks called): 16 and 48 in full, 37 of a batch of 64, and the flagship batch of 512
    for N, T, n in [(16, 1200, 16), (48, 1200, 48), (64, 1200, 37), (512, 3000, 512)]:
        runner = B200ModelRunner(caller, N, T)
        sig = rng.standard_normal((N, runner.chunk_size())).astype(np.float16)
        for i in range(N):
            runner.accept_chunk(i, sig[i])
        scores = runner.forward_scores(n)
        got = [np.array(a)[:n] for a in runner.call_chunks_raw(n)]
        if n <= 64:
            idx = np.arange(n)
        else:   # the scalar oracle is too slow for all 512: the first and last chunk of every CTA, and a seeded sample
            cpc = _chunks_per_cta(n, R)
            edges = {c for b in range(0, n, cpc) for c in (b, min(b + cpc, n) - 1)}
            idx = np.array(sorted(edges | set(rng.choice(n, size=16, replace=False).tolist())))
        _check(crf_oracle, cfg, scores, got, idx)
        runner.close()
    caller.close()


@pytest.mark.parametrize("N", [1, 15, 16, 17, 33, 301])
def test_standalone_decode_bit_exact(crf_oracle, N):
    """decode_scores packs for one batch in flight: one chunk per CTA up to 132 chunks, then 3 per CTA at N = 301 (the
    last CTA holding a single chunk)."""
    from dorado_b200 import lib as L
    T = 120
    scores = synthetic_scores(N, T, 3, seed=N, scale=1.5)
    moves, seq, qstr, nb = L.decode_scores(scores, clamp_val=5.0)
    idx = np.arange(N) if N <= 64 else np.array(sorted({0, 1, 2, 150, 297, 298, 299, 300}))
    ref = crf_oracle.decode(scores[idx], clamp_val=5.0)
    np.testing.assert_array_equal(nb[idx], ref.n_bases)
    np.testing.assert_array_equal(moves[idx], ref.moves)
    np.testing.assert_array_equal(seq[idx], ref.seq_buf)
    np.testing.assert_array_equal(qstr[idx], ref.qstr_buf)
