"""GPU parity at the sizes bench.py times (BASELINE configs: fast/hac batch 512 x 9996 samples, sup batch 128 x 9984),
pinned to the reference itself through tests/golden/full_*.npz and decode_full.npz (tools/make_golden_full.py: the
unmodified reference CPU sources, fp32 forward + CPUDecoder, run on full-length chunks).

Three contracts, each printed as measured numbers (run with -s to see them; tools/verify_round.sh keeps the log):
  1. decode: on identical fp16 scores the engine is BIT-IDENTICAL (sequence, qstring, moves) to the C oracle for EVERY
     chunk of the full batch, and -- on well-conditioned (planted-path) scores -- identical in sequence and moves to the
     reference's own CPUDecoder, with the qstring differing only where libtorch's vectorised scans differ from the
     contract's in the last ulp (the quality is 1 - sum(p^0.4)/sum(...), which cancels for confident bases).
  2. scores: distribution of |engine - reference fp32| / max(1, |reference|) over the committed score rows
     (north_star: 1e-3 relative for fp16).
  3. end to end: engine(signal) strings against reference(signal) strings over >= 1e5 bases (fast, hac), reported as
     edit-distance rate / moves mismatch rate next to the reference's own sensitivity to rounding its scores to fp16
     (the synthetic random-weight models are ill-conditioned: that rounding alone moves ~2 % of the bases).
"""
import concurrent.futures as cf
import os
import pathlib

import numpy as np
import pytest

from conftest import edit_distance, model_dir, planted_scores, synthetic_scores, unpack_rows

pytestmark = pytest.mark.gpu
GOLD = pathlib.Path(__file__).resolve().parent / "golden"
BATCH = {"fast": 512, "hac": 512, "sup": 128}


def _oracle_decode_parallel(crf_oracle, scores, **kw):
    """C oracle over all chunks, one slice per host thread (ctypes releases the GIL)."""
    N = scores.shape[0]
    workers = max(1, min(os.cpu_count() or 1, 64, N))
    bounds = np.linspace(0, N, workers + 1).astype(int)
    with cf.ThreadPoolExecutor(workers) as ex:
        parts = list(ex.map(lambda i: crf_oracle.decode(scores[bounds[i]:bounds[i + 1]], **kw), range(workers)))
    cat = lambda name: np.concatenate([getattr(p, name) for p in parts])
    return cat("seq_buf"), cat("qstr_buf"), cat("moves"), cat("n_bases")


def _rate(a, b):
    return a / max(1, b)


@pytest.mark.parametrize("kind", ["fast", "hac", "sup"])
def test_full_batch_against_reference(crf_oracle, kind):
    from dorado_b200.config import load_model_config
    from dorado_b200.runner import B200Caller, B200ModelRunner
    from dorado_b200.weights import synthetic_weights
    g = np.load(GOLD / f"full_{kind}.npz")
    cfg = load_model_config(model_dir(kind))
    M, T, T_out = int(g["M"]), int(g["T"]), int(g["T_out"])
    N = BATCH[kind]
    sig = np.random.default_rng(int(g["signal_seed"])).standard_normal((M, T)).astype(np.float16)
    import hashlib
    assert hashlib.sha256(sig.tobytes()).hexdigest() == str(g["sha_signal"]), "fixture signal not reproduced from its seed"
    caller = B200Caller(cfg, synthetic_weights(cfg, int(g["weights_seed"])))
    runner = B200ModelRunner(caller, N, T)
    assert runner.chunk_size() == T and runner.out_len() == T_out
    for i in range(N):
        runner.accept_chunk(i, sig[i % M])                   # the batch = the fixture's chunks, tiled
    scores = runner.forward_scores(N)                        # [N, T_out, C] fp16 (un-clamped)
    moves, seq, qstr, nb = (np.array(a) for a in runner.call_chunks_raw(N))

    # -- 1. decode of the engine's own scores: bit-identical to the C oracle, every chunk of the full batch
    o_seq, o_qstr, o_moves, o_nb = _oracle_decode_parallel(crf_oracle, scores, clamp_val=5.0 if cfg.clamp else 0.0,
                                                           q_shift=cfg.qbias, q_scale=cfg.qscale)
    np.testing.assert_array_equal(nb, o_nb)
    np.testing.assert_array_equal(moves, o_moves)
    np.testing.assert_array_equal(seq, o_seq)
    np.testing.assert_array_equal(qstr, o_qstr)
    # chunks are independent: every copy of a fixture chunk decodes identically wherever it sits in the batch
    for i in range(M, N):
        assert nb[i] == nb[i % M] and (moves[i] == moves[i % M]).all() and (seq[i] == seq[i % M]).all()
        assert (qstr[i] == qstr[i % M]).all()
    del o_seq, o_qstr, o_moves

    # -- 2. scores against the reference's fp32 forward (committed rows)
    rows = g["rows"]                                          # [row_chunks, n_rows, C] fp32, Clamp already applied
    rc, step = int(g["row_chunks"]), int(g["row_step"])
    got = scores[:rc, ::step].astype(np.float32)
    if cfg.clamp:
        got = np.clip(got, -5.0, 5.0)
    rel = np.abs(got - rows) / np.maximum(1.0, np.abs(rows))
    scale = max(1.0, float(np.abs(rows).max()))
    pct = {p: float(np.percentile(rel, p)) for p in (50, 90, 99, 99.9)}
    rel_l2 = float(np.linalg.norm(got - rows) / np.linalg.norm(rows))
    print(f"\n[{kind} N={N} T={T}] scores vs reference fp32 over {rel.size} values: |d|/max(1,|ref|) "
          f"p50 {pct[50]:.2e} p90 {pct[90]:.2e} p99 {pct[99]:.2e} p99.9 {pct[99.9]:.2e} max {rel.max():.2e}; "
          f"within 1e-3: {(rel <= 1e-3).mean():.4f}; rel-L2 {rel_l2:.2e}; max|ref| {scale:.2f}")
    # fp16 storage of weights, activations and the recurrent state against an fp32 reference: the error comes from the
    # fp16 rounding points (DESIGN.md), not from the kernels' accumulation order; the test prints the measured figures
    assert rel_l2 <= 5e-3, rel_l2
    assert pct[50] <= 3e-3 and pct[99] <= 2.5e-2 and rel.max() <= 0.1, (pct, float(rel.max()))

    # -- 3. end to end strings against the reference's own forward + decode of the same signal
    r_nb = g["ref_n_bases"]
    r_seq, r_q = unpack_rows(g["ref_seq"], r_nb), unpack_rows(g["ref_qstr"], r_nb)
    r_mv = np.unpackbits(g["ref_moves"], axis=1)[:, :T_out]
    h_nb = g["ref16_n_bases"]
    h_seq = unpack_rows(g["ref16_seq"], h_nb)
    h_mv = np.unpackbits(g["ref16_moves"], axis=1)[:, :T_out]
    e_seq = [bytes(seq[i, :nb[i]]) for i in range(M)]
    with cf.ThreadPoolExecutor(min(32, os.cpu_count() or 1)) as ex:
        d_eng = list(ex.map(lambda i: edit_distance(e_seq[i], r_seq[i]), range(M)))
        d_h = list(ex.map(lambda i: edit_distance(h_seq[i], r_seq[i]), range(M)))
    bases = int(r_nb.sum())
    eng_rate, h_rate = _rate(sum(d_eng), bases), _rate(sum(d_h), bases)
    mv_eng, mv_h = float((moves[:M] != r_mv).mean()), float((h_mv != r_mv).mean())
    q_same = q_tot = 0
    for i in range(M):
        if e_seq[i] == r_seq[i]:
            q_tot += len(r_q[i])
            q_same += sum(x == y for x, y in zip(bytes(qstr[i, :nb[i]]), r_q[i]))
    print(f"[{kind}] engine(signal) vs reference(signal) over {bases} bases / {M} chunks: base edit rate {eng_rate:.4f}, "
          f"moves mismatch {mv_eng:.4f}, identical chunks {sum(d == 0 for d in d_eng)}/{M}; "
          f"yardstick = reference on its own scores rounded to fp16: edit rate {h_rate:.4f}, moves mismatch {mv_h:.4f}; "
          f"qstring equal on identical sequences {q_same}/{q_tot}")
    # the engine's whole fp16 pipeline must stay within a small multiple of what rounding the final scores alone does
    assert eng_rate <= 6.0 * h_rate + 0.01, (eng_rate, h_rate)
    assert mv_eng <= 6.0 * mv_h + 0.02, (mv_eng, mv_h)


@pytest.mark.parametrize("state_len", [3, 4, 5])
def test_full_length_decode_against_reference(crf_oracle, state_len):
    """Full-length chunks (T = 1666 / 1664) of every state length, i.i.d. and planted-path scores regenerated from their
    seeds: engine == C oracle bit for bit; engine vs the reference CPUDecoder's committed output."""
    from dorado_b200 import lib as L
    g = np.load(GOLD / "decode_full.npz")
    N, T = (int(v) for v in g[f"sl{state_len}_shape"])
    o = L.default_decoder_options()
    o.q_shift, o.q_scale = float(g["q_shift"]), float(g["q_scale"])
    for tag, s16 in (("sl", synthetic_scores(N, T, state_len, seed=int(g["seed_base"]) + state_len, scale=float(g["scale"]))),
                     ("pl", planted_scores(N, T, state_len, seed=int(g["planted_seed_base"]) + state_len))):
        moves, seq, qstr, nb = L.decode_scores(s16, clamp_val=float(g["clamp"]), opts=o)
        ref = crf_oracle.decode(s16, clamp_val=float(g["clamp"]), q_shift=o.q_shift, q_scale=o.q_scale)
        np.testing.assert_array_equal(nb, ref.n_bases)
        np.testing.assert_array_equal(moves, ref.moves)
        np.testing.assert_array_equal(seq, ref.seq_buf)
        np.testing.assert_array_equal(qstr, ref.qstr_buf)
        r_nb = g[f"{tag}{state_len}_n_bases"]
        r_seq, r_q = unpack_rows(g[f"{tag}{state_len}_seq"], r_nb), unpack_rows(g[f"{tag}{state_len}_qstr"], r_nb)
        r_mv = np.unpackbits(g[f"{tag}{state_len}_moves"], axis=1)[:, :T]
        same = [bytes(seq[i, :nb[i]]) == r_seq[i] for i in range(N)]
        q_bad = sum(sum(x != y for x, y in zip(bytes(qstr[i, :nb[i]]), r_q[i])) for i in range(N) if same[i])
        q_tot = sum(len(r_q[i]) for i in range(N) if same[i])
        print(f"\n[decode state_len {state_len} {'iid' if tag == 'sl' else 'planted'} {N}x{T}] vs reference CPUDecoder: identical "
              f"sequences {sum(same)}/{N}, identical move tables {int((moves == r_mv).all(axis=1).sum())}/{N}, "
              f"qstring characters differing {q_bad}/{q_tot}")
        if tag == "pl":
            assert all(same) and (moves == r_mv).all()
            assert q_bad <= 0.015 * q_tot   # measured 0.5 %: last-ulp noise of libtorch's scans under the quality's cancellation
        else:
            assert sum(same) >= N // 2      # i.i.d. scores are full of near-ties (see the module docstring)
            assert q_bad <= 0.002 * q_tot + 1
