"""GPU parity of the network forward + the whole call_chunks path through the C ABI.

Scores (north_star: "CRF score tensors within 1e-3 relative (fp16)").  The engine, like the reference's own
CUDA path, keeps weights and inter-layer activations in fp16 with fp32 accumulation, so the oracle it is held
to 1e-3 against is oracle/nn_oracle.py with emulate_fp16=True (same rounding points, fp32 arithmetic):
  * >= 99.9 % of scores within 1e-3 * max|ref| (scores span [-5, 5]: 5e-3 absolute), none beyond 4e-3 * max|ref|.
The 18-layer transformer (sup) re-rounds its fp16 residual stream 36 times, so there the fraction within
1e-3 * max|ref| is ~98.7 % (bound: 97 %), still none beyond 4e-3 * max|ref|.
Against the pure-fp32 oracle (== the reference's CPU path, see tests/test_oracle_vs_reference.py) the fp16
storage itself costs ~2e-3 relative L2 on these synthetic weights, so that comparison is bounded looser:
  * relative L2 error <= 5e-3 and max error <= 2e-2 * max|ref|.
Decode: the engine's sequence / qstring / moves must be bit-identical to the CPU oracle decoding the engine's
own fp16 scores.
"""
import numpy as np
import pytest

from conftest import model_dir

pytestmark = pytest.mark.gpu


def _setup(kind, N, T, seed=1234):
    from dorado_b200.config import load_model_config
    from dorado_b200.runner import B200Caller, B200ModelRunner
    from dorado_b200.weights import synthetic_weights
    cfg = load_model_config(model_dir(kind))
    w = synthetic_weights(cfg, 42)
    caller = B200Caller(cfg, w)
    runner = B200ModelRunner(caller, N, T)
    rng = np.random.default_rng(seed)
    sig = rng.standard_normal((N, runner.chunk_size())).astype(np.float16)
    for i in range(N):
        runner.accept_chunk(i, sig[i])
    return cfg, w, caller, runner, sig


def _check_scores(got, ref16, ref32, clamp, max_frac_bad=1e-3):
    got = got.astype(np.float32)
    if clamp:
        got = np.clip(got, -5.0, 5.0)  # the engine defers the clamp to the decoder's score read, like the reference
    scale = max(1.0, float(np.abs(ref16).max()))
    err = np.abs(got - ref16)
    frac_bad = float((err > 1e-3 * scale).mean())
    assert frac_bad <= max_frac_bad, f"{frac_bad:.2e} of scores off by more than 1e-3 relative (max err {err.max():.4f})"
    assert err.max() <= 4e-3 * scale, f"max score error vs fp16-storage oracle {err.max():.4f}"
    rel_l2 = float(np.linalg.norm(got - ref32) / np.linalg.norm(ref32))
    assert rel_l2 <= 5e-3, f"relative L2 error vs fp32 oracle {rel_l2:.2e}"
    assert np.abs(got - ref32).max() <= 2e-2 * scale


@pytest.mark.parametrize("kind,N,T", [("fast", 16, 1200), ("fast", 48, 3000), ("fast", 800, 600), ("fast", 1664, 300), ("hac", 32, 1200), ("hac", 64, 1998), ("hac", 512, 300)])
def test_lstm_model_scores(kind, N, T):
    from oracle import nn_oracle
    cfg, w, caller, runner, sig = _setup(kind, N, T)
    got = runner.forward_scores(N)
    ref32 = nn_oracle.forward(cfg, w, sig.astype(np.float32))
    ref16 = nn_oracle.forward(cfg, w, sig.astype(np.float32), emulate_fp16=True)
    assert got.shape == ref32.shape
    _check_scores(got, ref16, ref32, cfg.clamp)


def test_flstm_model_reuses_the_lstm_kernels():
    """FLSTM (nn/FLSTMStack.cpp:108-124; SURVEY section 8f row 4): the factorised gate matrices are folded at load time, so an
    FLSTM model and the LSTM model with the products up @ dn as its weights give bit-identical scores and calls; the
    scores also sit on the numpy oracle's (the reference has no CPU forward for FLSTM to pin against)."""
    from oracle import nn_oracle
    from dorado_b200.config import load_model_config
    from dorado_b200.runner import B200Caller, B200ModelRunner
    from dorado_b200.weights import fold_flstm_weights, synthetic_weights
    N, T = 32, 3000
    cfg_f = load_model_config(model_dir("flstm"))
    cfg_l = load_model_config(model_dir("fast"))
    assert cfg_f.is_flstm_model and cfg_f.lstm_inner_dim == 32 and cfg_f.lstm_layers == cfg_l.lstm_layers
    w_f = synthetic_weights(cfg_f, 11)
    w_l = fold_flstm_weights(cfg_f, w_f)
    assert list(w_l) == list(synthetic_weights(cfg_l, 11))          # same tensor names as a plain LSTM model
    sig = np.random.default_rng(5).standard_normal((N, cfg_f.normalise_chunk_size(T))).astype(np.float16)
    out = []
    for cfg, w in ((cfg_f, w_f), (cfg_l, w_l)):
        caller = B200Caller(cfg, w)
        runner = B200ModelRunner(caller, N, T)
        assert not runner.variable_chunk_sizes()                    # api/runner_creation.cpp:28
        for i in range(N):
            runner.accept_chunk(i, sig[i])
        out.append((runner.forward_scores(N).copy(), [np.array(a) for a in runner.call_chunks_raw(N)]))
    np.testing.assert_array_equal(out[0][0], out[1][0])
    for a, b in zip(out[0][1], out[1][1]):
        np.testing.assert_array_equal(a, b)
    assert int(out[0][1][3].sum()) > N * 20                        # real calls, not empty strings
    ref32 = nn_oracle.forward(cfg_f, w_f, sig.astype(np.float32))
    ref16 = nn_oracle.forward(cfg_f, w_f, sig.astype(np.float32), emulate_fp16=True)
    _check_scores(out[0][0], ref16, ref32, cfg_f.clamp)


@pytest.mark.parametrize("N,T", [(2, 1920), (3, 3264)])
def test_tx_model_scores(N, T):
    """sup topology: conv x5 -> 18 transformer layers -> upsample -> scaled CRF linear.  The oracle uses the true
    attention window [-127, +128] (cpu_split_quirk=False); the reference's CPU fallback drops one key for the last
    query of each of its 12 splits, which tests/test_oracle_vs_reference.py pins separately."""
    from oracle import nn_oracle
    cfg, w, caller, runner, sig = _setup("sup", N, T)
    got = runner.forward_scores(N)
    ref32 = nn_oracle.forward(cfg, w, sig.astype(np.float32))
    ref16 = nn_oracle.forward(cfg, w, sig.astype(np.float32), emulate_fp16=True)
    assert got.shape == ref32.shape == (N, runner.chunk_size() // cfg.stride, 4096)
    # 18 layers re-round the fp16 residual stream 36 times: the rounding noise of two fp16 pipelines decorrelates,
    # so ~1.3 % of scores sit beyond 1e-3 * scale (measured; relative L2 1.6e-3, max 2.2e-3 * scale)
    _check_scores(got, ref16, ref32, cfg.clamp, max_frac_bad=3e-2)


@pytest.mark.parametrize("kind,N,T", [("fast", 32, 3000), ("hac", 32, 1998), ("sup", 2, 1920)])
def test_call_chunks_end_to_end(crf_oracle, kind, N, T):
    cfg, w, caller, runner, sig = _setup(kind, N, T)
    scores = runner.forward_scores(N)
    chunks = runner.call_chunks(N)
    assert len(chunks) == N
    ref = crf_oracle.decode(scores, clamp_val=5.0 if cfg.clamp else 0.0, q_shift=cfg.qbias, q_scale=cfg.qscale)
    for i, c in enumerate(chunks):
        assert c.sequence == ref.sequences[i]
        assert c.qstring == ref.qstrings[i]
        np.testing.assert_array_equal(c.moves, ref.moves[i])
        assert len(c.moves) == runner.chunk_size() // cfg.stride
        assert len(c.sequence) == len(c.qstring) == int(c.moves.sum())
    # partial batch: the first k results do not depend on what the other slots hold
    k = min(5, N - 1)
    part = runner.call_chunks(k)
    assert [p.sequence for p in part] == [c.sequence for c in chunks[:k]]
    stats = runner.sample_stats()
    assert stats["batches_called"] == 2 and stats["model_decode_ms"] > 0
    assert caller.stats()["gpu_launches"] > 0


def test_runner_rejects_bad_shapes():
    from dorado_b200 import lib as L
    from dorado_b200.config import load_model_config
    from dorado_b200.runner import B200Caller, B200ModelRunner
    from dorado_b200.weights import synthetic_weights
    cfg = load_model_config(model_dir("fast"))
    caller = B200Caller(cfg, synthetic_weights(cfg, 1))
    with pytest.raises(L.B200Error):
        B200ModelRunner(caller, 7, 1200)  # LSTM batch must be a multiple of 16 (32 for hac)
    r = B200ModelRunner(caller, 16, 1203)  # normalised down to a multiple of the stride (BatchParams::normalise)
    assert r.chunk_size() == 1200
    with pytest.raises(L.B200Error):
        r.accept_chunk(16, np.zeros(1200, np.float16))
    with pytest.raises(L.B200Error):
        r.accept_chunk(0, np.zeros(1199, np.float16))
    with pytest.raises(L.B200Error):
        r.call_chunks(17)


@pytest.mark.parametrize("kind,N,T", [("fast", 64, 3000), ("hac", 64, 1200), ("sup", 4, 1920)])
def test_concurrent_runners_match_serial(kind, N, T):
    """Two runners of one caller (dorado's num_runners = 2 per device, api/runner_creation.cpp:91-123), each on its own
    stream and driven from its own thread, must return exactly what they return one at a time."""
    import threading
    from dorado_b200.runner import B200ModelRunner
    cfg, w, caller, r0, sig0 = _setup(kind, N, T, seed=5)
    r1 = B200ModelRunner(caller, N, T)
    sig1 = np.random.default_rng(6).standard_normal((N, r1.chunk_size())).astype(np.float16)
    for i in range(N):
        r1.accept_chunk(i, sig1[i])
    runners = [r0, r1]
    serial = [[(c.sequence, c.qstring, bytes(c.moves)) for c in r.call_chunks(N)] for r in runners]
    assert serial[0] != serial[1]
    got = [[], []]

    def drive(i):
        for _ in range(4):
            got[i].append([(c.sequence, c.qstring, bytes(c.moves)) for c in runners[i].call_chunks(N)])

    ths = [threading.Thread(target=drive, args=(i,)) for i in range(2)]
    for th in ths:
        th.start()
    for th in ths:
        th.join()
    for i in range(2):
        assert len(got[i]) == 4
        for g in got[i]:
            assert g == serial[i]
    # the device-resident pipelined loop (bench.py's `value`) leaves each runner's result intact as well
    ms = B200ModelRunner.step_device_runners(runners, N, 6)
    assert ms > 0
    for i, r in enumerate(runners):
        assert [(c.sequence, c.qstring, bytes(c.moves)) for c in r.call_chunks(N)] == serial[i]


def test_caller_lifecycle_and_low_latency():
    """CudaCaller::terminate / restart (CudaCaller.cpp:273-287) and the low-latency variant (:126-138, 216-222)."""
    from dorado_b200 import lib as L
    from dorado_b200.config import load_model_config
    from dorado_b200.runner import B200Caller, B200ModelRunner
    from dorado_b200.weights import synthetic_weights
    cfg = load_model_config(model_dir("fast"))
    w = synthetic_weights(cfg, 42)
    caller = B200Caller(cfg, w)
    runner = B200ModelRunner(caller, 16, 1200)
    assert runner.batch_timeouts_ms() == (300000, 30000) and not runner.is_low_latency()
    sig = np.random.default_rng(0).standard_normal((16, runner.chunk_size())).astype(np.float16)
    for i in range(16):
        runner.accept_chunk(i, sig[i])
    first = runner.call_chunks(16)
    runner.terminate()
    runner.terminate()                      # once per runner sharing the caller
    with pytest.raises(L.B200Error) as e:
        runner.call_chunks(16)
    assert "terminated" in str(e.value)
    runner.restart()
    runner.restart()                        # idempotent
    again = runner.call_chunks(16)
    assert [c.sequence for c in again] == [c.sequence for c in first]
    assert [c.qstring for c in again] == [c.qstring for c in first]
    # low-latency caller: 350 ms timeouts, highest-priority streams, same results
    ll = B200Caller(cfg, w, low_latency=True)
    r2 = B200ModelRunner(ll, 16, 1200)
    assert r2.batch_timeouts_ms() == (350, 350) and r2.is_low_latency()
    for i in range(16):
        r2.accept_chunk(i, sig[i])
    assert [c.sequence for c in r2.call_chunks(16)] == [c.sequence for c in first]


def test_decoder_options_struct_mirrors_the_reference():
    from dorado_b200 import lib as L
    o = L.default_decoder_options()
    assert (o.beam_width, o.beam_cut, o.blank_score, o.q_shift, o.q_scale, o.temperature, o.move_pad) == (32, 100.0, 2.0, 0.0, 1.0, 1.0, 0)
    scores = np.zeros((1, 8, 256), np.float16)
    for field, val in (("move_pad", 1), ("temperature", 0.5)):
        o = L.default_decoder_options()
        setattr(o, field, val)
        with pytest.raises(L.B200Error) as e:
            L.decode_scores(scores, opts=o)
        assert e.value.status == L.B200_ERR_UNSUPPORTED


def test_pool_feeds_every_runner_and_matches_a_single_runner():
    """b200_pool (one process, an engine per listed device, runners fed from one shared cursor) returns, chunk for chunk,
    what a single runner returns; every runner takes part.  Listing device 0 twice exercises the multi-engine code on the
    one-GPU test box (tools/bench_pool.py runs it across real devices)."""
    from dorado_b200.config import load_model_config
    from dorado_b200.runner import B200Caller, B200ModelRunner, B200Pool
    from dorado_b200.weights import synthetic_weights
    cfg = load_model_config(model_dir("fast"))
    w = synthetic_weights(cfg, 42)
    n, B, T = 150, 16, 1200
    pool = B200Pool(cfg, w, [0, 0], 2, B, T)
    assert pool.num_runners() == 4
    sig = np.random.default_rng(5).standard_normal((n, pool.chunk_size)).astype(np.float16)
    secs, moves, seq, qs, nb = pool.call_chunks(sig)
    assert secs > 0
    secs2, *_ = pool.call_chunks(sig, want_output=False)      # a second job on the same pool
    taken = [pool.runner_info(i)["batches"] for i in range(4)]
    assert sum(taken) == 2 * ((n + B - 1) // B) and min(taken) >= 1, taken
    caller = B200Caller(cfg, w)
    runner = B200ModelRunner(caller, B, T)
    for start in range(0, n, B):
        cnt = min(B, n - start)
        for i in range(cnt):
            runner.accept_chunk(i, sig[start + i])
        ref = runner.call_chunks(cnt)
        for i, c in enumerate(ref):
            k = start + i
            assert nb[k] == len(c.sequence)
            assert bytes(seq[k, :nb[k]]).decode() == c.sequence and bytes(qs[k, :nb[k]]).decode() == c.qstring
            assert (moves[k] == c.moves).all()
    pool.close()


def test_cluster_shapes_agree():
    """The hac recurrence runs 16, 32 or 64 chunks per cluster of 8 CTAs (chosen from the batch size and the engine's
    num_runners): the result must not depend on that choice -- bit for bit, fixed and variable chunk sizes --
    and the 16-chunk shape is the one the other tests pin against the oracle."""
    import os
    from dorado_b200.config import load_model_config
    from dorado_b200.runner import B200Caller, B200ModelRunner
    from dorado_b200.weights import synthetic_weights
    cfg = load_model_config(model_dir("hac"))
    caller = B200Caller(cfg, synthetic_weights(cfg, 42))
    N, T = 128, 1200
    rng = np.random.default_rng(3)
    sig = rng.standard_normal((N, cfg.normalise_chunk_size(T))).astype(np.float16)
    lens = rng.integers(10, sig.shape[1] // cfg.stride + 1, size=N) * cfg.stride
    got = {}
    try:
        for un in (16, 32, 64):
            os.environ["B200_CLUSTER_CHUNKS"] = str(un)
            runner = B200ModelRunner(caller, N, T)
            assert runner.plan_info()["lstm_rec.chunks_per_cluster"] == un and runner.plan_info()["lstm_rec.ctas"] == N // un * 8
            for i in range(N):
                runner.accept_chunk(i, sig[i])
            fixed = runner.forward_scores(N).copy()
            for i in range(N):
                runner.accept_chunk_var(i, sig[i, :lens[i]])
            got[un] = (fixed, runner.forward_scores(N).copy(), [np.array(a) for a in runner.call_chunks_raw(N)])
            runner.close()
    finally:
        os.environ.pop("B200_CLUSTER_CHUNKS", None)
    for un in (32, 64):
        np.testing.assert_array_equal(got[un][0], got[16][0])
        for i in range(N):   # beyond a chunk's own length the score rows are unspecified
            tn = int(lens[i]) // cfg.stride
            np.testing.assert_array_equal(got[un][1][i, :tn], got[16][1][i, :tn])
        (mv, sq, qs, nb), (mv0, sq0, qs0, nb0) = got[un][2], got[16][2]
        np.testing.assert_array_equal(nb, nb0)
        for i in range(N):
            tn = int(lens[i]) // cfg.stride
            assert (mv[i, :tn] == mv0[i, :tn]).all() and (sq[i, :nb[i]] == sq0[i, :nb[i]]).all() and (qs[i, :nb[i]] == qs0[i, :nb[i]]).all()


def test_variable_chunk_sizes_match_each_chunk_alone(crf_oracle):
    """Variable chunk sizes (SURVEY 8f row 1; nn/AuxiliaryData.cpp, CudaModelRunner.cpp:21-31, CUDADecoder.cpp:35-62): a batch
    of hac chunks of different lengths.  Every chunk must come out as if it were basecalled alone at its own length: scores
    against the numpy oracle run per chunk, strings bit-identical to the C oracle decoding the engine's scores, moves of
    len / stride blocks -- and equal to what a fixed-shape runner of exactly that chunk size returns."""
    from oracle import nn_oracle
    from dorado_b200.config import load_model_config
    from dorado_b200.runner import B200Caller, B200ModelRunner
    from dorado_b200.weights import synthetic_weights
    cfg = load_model_config(model_dir("hac"))
    w = synthetic_weights(cfg, 42)
    caller = B200Caller(cfg, w)
    N, T = 64, 1998
    runner = B200ModelRunner(caller, N, T)
    assert runner.variable_chunk_sizes()
    fast_runner = B200ModelRunner(B200Caller(load_model_config(model_dir("fast")), synthetic_weights(load_model_config(model_dir("fast")), 42)), 16, 1200)
    assert not fast_runner.variable_chunk_sizes()   # lstm_size 96: the reference has no such mode either (runner_creation.cpp:27-31)
    rng = np.random.default_rng(77)
    lens = rng.integers(40, T // cfg.stride + 1, size=N) * cfg.stride
    lens[0], lens[1], lens[2], lens[33] = T, cfg.stride * 40, cfg.stride, T          # full, short, one block, full
    lens[32:40] = np.sort(lens[32:40])
    sig = [rng.standard_normal(int(l)).astype(np.float16) for l in lens]
    for i in range(N):
        runner.accept_chunk_var(i, sig[i])
    scores = runner.forward_scores(N)
    called = runner.call_chunks(N)
    clamp = 5.0 if cfg.clamp else 0.0
    worst = 0.0
    for i in range(N):
        tn = int(lens[i]) // cfg.stride
        assert len(called[i].moves) == tn and int(called[i].moves.sum()) == len(called[i].sequence) == len(called[i].qstring)
        ref = crf_oracle.decode(scores[i:i + 1, :tn], clamp_val=clamp, q_shift=cfg.qbias, q_scale=cfg.qscale)
        assert called[i].sequence == ref.sequences[0] and called[i].qstring == ref.qstrings[0]
        assert (called[i].moves == ref.moves[0]).all()
        if i in (0, 1, 2, 5, 33, 39, 63):   # numpy forward of the chunk alone, at its own length
            want = nn_oracle.forward(cfg, w, sig[i][None].astype(np.float32), emulate_fp16=True)[0]
            got = np.clip(scores[i, :tn].astype(np.float32), -5, 5) if cfg.clamp else scores[i, :tn].astype(np.float32)
            err = np.abs(got - want)
            scale = max(1.0, float(np.abs(want).max()))
            assert (err > 1e-3 * scale).mean() <= 2e-3 and err.max() <= 6e-3 * scale, (i, tn, float(err.max()))
            worst = max(worst, float(err.max()) / scale)
    # a fixed-shape runner of exactly that chunk size gives the same call
    for i in (1, 5):
        alone = B200ModelRunner(caller, 32, int(lens[i]))
        alone.accept_chunk(0, sig[i])
        a = alone.call_chunks(1)[0]
        assert a.sequence == called[i].sequence and a.qstring == called[i].qstring and (a.moves == called[i].moves).all()
    print(f"\n[variable chunk sizes] {N} hac chunks of {int(lens.min())}..{int(lens.max())} samples: worst score error {worst:.2e} of max|ref|")
    # fixed-size chunks through the same runner afterwards: the slots revert to full length
    full = rng.standard_normal((N, runner.chunk_size())).astype(np.float16)
    for i in range(N):
        runner.accept_chunk(i, full[i])
    again = runner.call_chunks(N)
    assert all(len(c.moves) == runner.out_len() for c in again)


def test_conv12_tensor_core_kernel_matches_the_fma_kernel_and_the_oracle(monkeypatch):
    """conv1 + conv2 of the v5 LSTM models: the tensor-core kernel (conv2 as a 128 x 16 x 80 mma.sync contraction per tile of 128 samples,
    conv1's output as its fp16 operand) against the fp32 FMA-pipe kernel (B200_CONV12_FMA=1) and against nn_oracle's conv2
    output with the same rounding points.  The conv2 output buffer x2 [N][T + 2 * pad + 8][16] is the first workspace block;
    its padding rows must stay zero.  Ragged T (not a multiple of the 128-sample tile) and several tiles per chunk."""
    from oracle import nn_oracle
    from dorado_b200.runner import B200ModelRunner
    N, T = 32, 1998
    cfg, w, caller, runner, sig = _setup("fast", N, T)
    T = runner.chunk_size()
    pad = cfg.convs[2].winlen // 2
    Tp = T + 2 * pad + 8

    def x2_of(r):
        r.forward_scores(N)
        return r.debug_read_workspace(0, N * Tp * 16 * 2).view(np.float16).reshape(N, Tp, 16).astype(np.float32)

    tc_out = x2_of(runner)
    monkeypatch.setenv("B200_CONV12_FMA", "1")
    fma_runner = B200ModelRunner(caller, N, T)
    monkeypatch.delenv("B200_CONV12_FMA")
    for i in range(N):
        fma_runner.accept_chunk(i, sig[i])
    fma_out = x2_of(fma_runner)
    _, inter = nn_oracle.forward(cfg, w, sig.astype(np.float32), return_intermediates=True, emulate_fp16=True)
    ref = inter["conv1"].transpose(0, 2, 1)  # conv index 1 = conv2's output, [N][T][16]
    scale = max(1.0, float(np.abs(ref).max()))
    assert np.abs(tc_out[:, :pad]).max() == 0 and np.abs(tc_out[:, pad + T:]).max() == 0, "padding rows must stay zero"
    err_ref = np.abs(tc_out[:, pad:pad + T] - ref)
    err_fma = np.abs(tc_out - fma_out)
    print(f"\n[conv12 tensor-core kernel] vs oracle: max {err_ref.max():.2e} mean {err_ref.mean():.2e}; "
          f"vs fp32 FMA kernel: max {err_fma.max():.2e} mean {err_fma.mean():.2e} (scale {scale:.2f})")
    assert err_ref.max() <= 2e-3 * scale    # one fp16 rounding of the output + accumulation order
    assert err_fma.max() <= 6e-3 * scale    # the FMA kernel keeps conv1's output and conv2's weights in fp32
