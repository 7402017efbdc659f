"""Per-layer errors of an LSTM model's forward against nn_oracle (fp16 storage points): conv2, conv3 and the output of
every LSTM layer, then the CRF linear.  usage: python tools/debug_forward.py fast|hac|sup N T

B200_DEBUG_LSTM_LAYERS=k stops the forward after k LSTM layers; it is read when a runner is built, so each k gets a runner
of its own.  The workspace offsets come from tests/lstm_layer_ref.workspace_layout, which the layer tests use too."""
import os, sys, numpy as np
sys.path.insert(0, '.'); sys.path.insert(0, 'tests')
from conftest import model_dir
from lstm_layer_ref import read_seq, read_x2, workspace_layout
from dorado_b200.config import load_model_config
from dorado_b200.runner import B200Caller, B200ModelRunner
from dorado_b200.weights import synthetic_weights
from oracle import nn_oracle
kind, N, T = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
np.set_printoptions(linewidth=220, precision=4, suppress=True)
cfg = load_model_config(model_dir(kind)); w = synthetic_weights(cfg, 42)
caller = B200Caller(cfg, w)
T = cfg.normalise_chunk_size(T)
pad = workspace_layout(cfg, N, T)["pad"]
sig = np.random.default_rng(1234).standard_normal((N, T)).astype(np.float16)
ref, inter = nn_oracle.forward(cfg, w, sig.astype(np.float32), return_intermediates=True, emulate_fp16=True)


def make_runner(k):
    if k is None:
        os.environ.pop("B200_DEBUG_LSTM_LAYERS", None)
    else:
        os.environ["B200_DEBUG_LSTM_LAYERS"] = str(k)
    r = B200ModelRunner(caller, N, T)
    for i in range(N): r.accept_chunk(i, sig[i])
    return r


for k in range(0, cfg.lstm_layers + 1):
    runner = make_runner(k)
    runner.forward_scores(N)
    if k == 0:
        x2 = read_x2(runner, cfg, N, T)
        r2 = inter["conv1"].transpose(0, 2, 1)
        e = np.abs(x2[:, pad:pad + T] - r2)
        print("conv2 out: max err", e.max(), "mean", e.mean(), "pad rows max", np.abs(x2[:, :pad]).max(), np.abs(x2[:, pad + T:]).max())
    seq = read_seq(runner, cfg, N, T).astype(np.float32).transpose(1, 0, 2)
    runner.close()
    r = inter["conv2"].transpose(0, 2, 1) if k == 0 else inter[f"lstm{k-1}"]
    e = np.abs(seq - r)
    print(f"after {k} lstm layers: max {e.max():.4f} mean {e.mean():.5f}  per-t max first/last 6 {e.max(axis=(0,2))[:6]} {e.max(axis=(0,2))[-6:]}")
    if k >= 1:
        eu = e.max(axis=(0, 1)); print("   per-unit max", eu.reshape(-1, 32).max(axis=1), " worst units", np.argsort(eu)[-8:], "per-n max", e.max(axis=(1,2))[:8])
runner = make_runner(None)
got = runner.forward_scores(N).astype(np.float32)
seq = read_seq(runner, cfg, N, T).astype(np.float32)
W = w[f"{3 + cfg.lstm_layers + 1}.linear.weight.tensor"].astype(np.float16).astype(np.float32)
exp = np.clip(seq @ W.T, -5, 5) if cfg.clamp else seq @ W.T   # [T][N][out]
exp_raw = seq @ W.T
g = got.transpose(1, 0, 2)
e = np.abs(np.clip(g, -5, 5) - exp)
print("linear check: max", e.max(), "mean", e.mean())
er = e.max(axis=2)  # [T][N]
print("rows (t,n) with err>0.05:", np.argwhere(er > 0.05)[:40].tolist())
print("per-t max", er.max(axis=1)[:24], "...", er.max(axis=1)[-10:])
bad = np.argwhere(e > 0.05)
print("bad count", len(bad), "cols of bad (first 30)", sorted(set(bad[:, 2].tolist()))[:30])
t, n = (bad[0][0], bad[0][1]) if len(bad) else (0, 0)
print("example row", t, n, "got", g[t, n, :8], "exp", exp_raw[t, n, :8])
