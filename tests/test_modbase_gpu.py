"""conv_lstm_v3 modified-base models on the GPU (dorado_b200/csrc/modbase_model.cu): probabilities against the
fp16-emulating numpy oracle, each LSTM layer against the teacher-forced float64 reference of tests/lstm_layer_ref.py,
bit-exact invariances of the batch, and the error codes of the C ABI."""
import threading

import numpy as np
import pytest

from lstm_layer_ref import check_layer, make_layer_weights
from test_modbase_cpu import MODBASE, modbase_dir, modbase_inputs

pytestmark = pytest.mark.gpu

# engine vs fp16-emulating oracle, probabilities in [0, 1]: the engine's activations (tanh.approx in the LSTM gates, ex2/rcp
# in the convolutions) and its fp32 summation order move a probability by an fp16 ulp or two.  Measured on an H100 over
# both fixtures at batch 64 and 1024 and the 768-wide variant: max 2.4e-3, p99.9 9.8e-4, mean 1.5e-4.
PROB_MAX = 5e-3
PROB_P999 = 2e-3
PROB_MEAN = 3e-4
_cache = {}


def _cfg_w(kind, tmp_factory=None):
    from dorado_b200.config import load_modbase_config
    from dorado_b200.weights import synthetic_modbase_weights
    if kind not in _cache:
        cfg = load_modbase_config(_wide_dir(tmp_factory) if kind == "mb768" else modbase_dir(kind))
        _cache[kind] = (cfg, synthetic_modbase_weights(cfg, 5))
    return _cache[kind]


def _resize(src, tmp_dir, old, new):
    """The 384 fixture with its LSTM width replaced (merge conv size, both LSTMs, the linear's input, model size)."""
    text = (modbase_dir("mb384") / "config.toml").read_text()
    assert text.count(f"size = {old}") == 4 and text.count(f"in_features = {old}") == 1
    text = text.replace(f"size = {old}", f"size = {new}").replace(f"in_features = {old}", f"in_features = {new}")
    tmp_dir.mkdir(parents=True, exist_ok=True)
    (tmp_dir / "config.toml").write_text(text)
    return tmp_dir


def _wide_dir(tmp_factory):
    return _resize(modbase_dir("mb384"), tmp_factory.mktemp("mb768"), 384, 768)


def _runner(caller, N, sig, seq, n_accept=None):
    from dorado_b200.modbase import B200ModBaseRunner
    r = B200ModBaseRunner(caller, N)
    assert (r.sig_len, r.seq_len) == (sig.shape[1], seq.shape[1])
    for i in range(N if n_accept is None else n_accept):
        r.accept_chunk(i, sig[i], seq[i])
    return r


@pytest.mark.parametrize("kind,N", [("mb384", 64), ("mb384", 1024), ("mb192", 64), ("mb192", 1024), ("mb768", 64)])
def test_probabilities(tmp_path_factory, kind, N):
    from dorado_b200.modbase import B200ModBaseCaller
    from oracle.modbase_oracle import modbase_forward
    cfg, w = _cfg_w(kind, tmp_path_factory)
    sig, seq = modbase_inputs(cfg, N, 21)
    caller = B200ModBaseCaller(cfg, w)
    r = _runner(caller, N, sig, seq)
    assert r.out_len == cfg.out_steps()
    got = r.call_chunks(N).astype(np.float32)
    ref = modbase_forward(cfg, w, sig, seq, emulate_fp16=True)
    assert got.shape == ref.shape == (N, cfg.out_steps() * cfg.num_out)
    assert np.isfinite(got).all()
    assert np.allclose(got.reshape(N, -1, cfg.num_out).sum(-1), 1.0, atol=1e-2)
    err = np.abs(got - ref)
    p50, p99, p999 = np.percentile(err, [50, 99, 99.9])
    print(f"{kind} N={N}: |p - oracle| p50 {p50:.2e} p99 {p99:.2e} p99.9 {p999:.2e} max {err.max():.2e} "
          f"mean {err.mean():.2e}")
    assert err.max() <= PROB_MAX and p999 <= PROB_P999 and err.mean() <= PROB_MEAN


def _read_after(monkeypatch, caller, N, sig, seq, layers):
    """The sequence buffer after `layers` LSTM layers (B200_DEBUG_LSTM_LAYERS is read when the runner is created)."""
    monkeypatch.setenv("B200_DEBUG_LSTM_LAYERS", str(layers))
    r = _runner(caller, N, sig, seq)
    monkeypatch.delenv("B200_DEBUG_LSTM_LAYERS")
    r.call_chunks(N)
    return r.read_sequence_buffer()


@pytest.mark.parametrize("kind", ["mb384", "mb192", "mb768"])
def test_lstm_layers_teacher_forced(tmp_path_factory, monkeypatch, kind):
    from dorado_b200.modbase import B200ModBaseCaller
    from oracle.modbase_oracle import modbase_forward
    cfg, w = _cfg_w(kind, tmp_path_factory)
    N = 64
    sig, seq = modbase_inputs(cfg, N, 33)
    caller = B200ModBaseCaller(cfg, w)
    X = _read_after(monkeypatch, caller, N, sig, seq, 0)
    H1 = _read_after(monkeypatch, caller, N, sig, seq, 1)
    H2 = _read_after(monkeypatch, caller, N, sig, seq, 2)
    # the merge conv output itself, against the oracle's
    _, inter = modbase_forward(cfg, w, sig, seq, emulate_fp16=True, return_intermediates=True)
    merge_err = np.abs(X.astype(np.float32) - inter["merge"])
    print(f"{kind}: merge conv output vs oracle max |diff| {merge_err.max():.3g}")
    assert merge_err.max() <= 1e-2
    ratios = []
    for l, (Xl, Hl) in enumerate([(X, H1), (H1, H2)]):
        p = f"lstm{l + 1}."
        lw = make_layer_weights(w[p + "weight_ih_l0.tensor"], w[p + "weight_hh_l0.tensor"], w[p + "bias_ih_l0.tensor"],
                                w[p + "bias_hh_l0.tensor"])
        reverse = l == 1   # lstm1 forward in time, lstm2 reversed
        chk = check_layer(Xl.astype(np.float64), Hl.astype(np.float64), lw, reverse, label=f"{kind} {p[:-1]}")
        print(chk.describe())
        assert chk.ok, chk.describe()
        wrong = check_layer(Xl.astype(np.float64), Hl.astype(np.float64), lw, not reverse)
        assert wrong.max_ratio >= 10.0, f"{p[:-1]} in the wrong direction only reaches {wrong.max_ratio:.3g} x the budget"
        ratios.append(chk.max_ratio)
    print(f"{kind}: worst error / budget per layer {ratios}")


def test_batch_invariances():
    from dorado_b200.modbase import B200ModBaseCaller
    cfg, w = _cfg_w("mb384")
    N = 96
    sig, seq = modbase_inputs(cfg, N, 44)
    caller = B200ModBaseCaller(cfg, w)
    full = _runner(caller, N, sig, seq).call_chunks(N)
    # a partial batch: 40 chunks in a fresh runner whose other slots were never written
    part = _runner(caller, N, sig, seq, n_accept=40).call_chunks(40)
    assert np.array_equal(part.view(np.uint16), full[:40].view(np.uint16))
    # the same runner called again for fewer chunks
    r = _runner(caller, N, sig, seq)
    r.call_chunks(N)
    assert np.array_equal(r.call_chunks(17).view(np.uint16), full[:17].view(np.uint16))
    # permuted chunks give permuted outputs
    perm = np.random.default_rng(3).permutation(N)
    permuted = _runner(caller, N, sig[perm], seq[perm]).call_chunks(N)
    assert np.array_equal(permuted.view(np.uint16), full[perm].view(np.uint16))


def _concurrently(*fns):
    out = [None] * len(fns)
    errs = []

    def run(i):
        try:
            out[i] = fns[i]()
        except Exception as e:  # surfaced below
            errs.append(e)
    ts = [threading.Thread(target=run, args=(i,)) for i in range(len(fns))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs
    return out


def test_concurrent_runners_match_alone():
    from dorado_b200.config import load_model_config
    from dorado_b200.modbase import B200ModBaseCaller
    from dorado_b200.runner import B200Caller, B200ModelRunner
    from dorado_b200.weights import synthetic_weights
    from conftest import model_dir
    cfg, w = _cfg_w("mb384")
    N = 128
    sig_a, seq_a = modbase_inputs(cfg, N, 1)
    sig_b, seq_b = modbase_inputs(cfg, N, 2)
    caller = B200ModBaseCaller(cfg, w)
    ra, rb = _runner(caller, N, sig_a, seq_a), _runner(caller, N, sig_b, seq_b)
    alone_a, alone_b = ra.call_chunks(N), rb.call_chunks(N)
    # two runners of one engine in flight at once, several batches each
    for _ in range(3):
        got_a, got_b = _concurrently(lambda: ra.call_chunks(N), lambda: rb.call_chunks(N))
        assert np.array_equal(got_a.view(np.uint16), alone_a.view(np.uint16))
        assert np.array_equal(got_b.view(np.uint16), alone_b.view(np.uint16))
    # a modbase runner next to a basecall runner on the same device
    bcfg = load_model_config(model_dir("hac"))
    bcaller = B200Caller(bcfg, synthetic_weights(bcfg, 42))
    br = B200ModelRunner(bcaller, 64, 1200)
    bsig = np.random.default_rng(9).standard_normal((64, 1200)).astype(np.float16)
    for i in range(64):
        br.accept_chunk(i, bsig[i])
    scores_alone = br.forward_scores(64)
    for _ in range(3):
        got_a, scores = _concurrently(lambda: ra.call_chunks(N), lambda: br.forward_scores(64))
        assert np.array_equal(got_a.view(np.uint16), alone_a.view(np.uint16))
        assert np.array_equal(scores.view(np.uint16), scores_alone.view(np.uint16))


def test_error_codes(tmp_path):
    from dorado_b200 import lib as L
    from dorado_b200.config import load_modbase_config
    from dorado_b200.modbase import B200ModBaseCaller, B200ModBaseRunner
    from dorado_b200.weights import synthetic_modbase_weights
    # widths without a recurrence instantiation
    for width in (512, 96):
        cfg = load_modbase_config(_resize(modbase_dir("mb384"), tmp_path / f"w{width}", 384, width))
        assert cfg.lstm_size == width
        with pytest.raises(L.B200Error) as e:
            B200ModBaseCaller(cfg, synthetic_modbase_weights(cfg, 1))
        assert e.value.status == L.B200_ERR_UNSUPPORTED, str(e.value)
    cfg, w = _cfg_w("mb192")
    caller = B200ModBaseCaller(cfg, w)
    for bad in (48, 16, 0):
        with pytest.raises(L.B200Error) as e:
            B200ModBaseRunner(caller, bad)
        assert e.value.status == L.B200_ERR_INVALID
    r = B200ModBaseRunner(caller, 32)
    sig, seq = modbase_inputs(cfg, 1, 0)
    r.accept_chunk(0, sig[0], seq[0])
    for s, q in ((sig[0][:-6], seq[0]), (sig[0], seq[0][:-1]), (np.concatenate([sig[0], sig[0][:6]]), seq[0])):
        with pytest.raises(L.B200Error) as e:
            r.accept_chunk(0, s, q)
        assert e.value.status == L.B200_ERR_INVALID
    with pytest.raises(L.B200Error) as e:
        r.accept_chunk(32, sig[0], seq[0])
    assert e.value.status == L.B200_ERR_INVALID
    with pytest.raises(L.B200Error) as e:
        r.call_chunks(33)
    assert e.value.status == L.B200_ERR_INVALID
    # a missing or misshapen weight tensor
    w2 = dict(w)
    w2["fc.weight.tensor"] = w2["fc.weight.tensor"][:, :-1]
    with pytest.raises(L.B200Error) as e:
        B200ModBaseCaller(cfg, w2)
    assert e.value.status == L.B200_ERR_INVALID


@pytest.mark.parametrize("kind,batch,n", [("mb384", 64, 50), ("mb192", 32, 32)])
def test_dorado_binding_matches_python(tmp_path, kind, batch, n):
    """include/B200ModBaseModel.h compiled against the reference's headers (oracle/_ref/modbase_host) and run once: its
    forward gives the probabilities of the ctypes path, bit for bit."""
    import pathlib
    import subprocess
    from dorado_b200.modbase import B200ModBaseCaller
    from oracle.modbase_oracle import ModBaseReference
    host = pathlib.Path(__file__).resolve().parents[1] / "oracle" / "_ref" / "modbase_host"
    if not host.exists() or not ModBaseReference.available():
        pytest.skip("oracle/_ref/modbase_host not built (needs the reference tree where it is built)")
    cfg, w = _cfg_w(kind)
    sig, seq = modbase_inputs(cfg, n, 77)
    model_dir = ModBaseReference().write_model_dir(modbase_dir(kind), w, tmp_path / "model")
    sig.tofile(tmp_path / "sig.f16")
    seq.tofile(tmp_path / "seq.i8")
    run = subprocess.run([str(host), str(model_dir), str(batch), str(n), str(tmp_path / "sig.f16"), str(tmp_path / "seq.i8"),
                          str(tmp_path / "out.f16")], capture_output=True, text=True, timeout=300)
    assert run.returncode == 0, run.stderr
    got = np.fromfile(tmp_path / "out.f16", np.float16).reshape(n, -1)
    want = _runner(B200ModBaseCaller(cfg, w), batch, sig, seq, n_accept=n).call_chunks(n)
    assert np.array_equal(got.view(np.uint16), want.view(np.uint16))
