"""A runner's device memory: b200_engine_runner_bytes is exactly what building the runner adds to the engine's arena bytes,
for every fixture model at two shapes, and it refuses exactly the shapes runner creation refuses.  Both come from one
layout function per buffer owner (dorado_b200/csrc/engine.h, Bump)."""
import ctypes as C

import numpy as np
import pytest

from conftest import CONFIG_DIR, model_dir
from test_modbase_cpu import modbase_dir, modbase_inputs
from test_tx1536_cpu import config_variant

pytestmark = pytest.mark.gpu

# (fixture, precision, [(batch, chunk), (batch, chunk)]); hac is a variable-chunk-size model (a per-chunk length buffer)
CASES = [
    ("fast", "fp16", [(64, 1200), (128, 6000)]),
    ("flstm", "fp16", [(64, 1200), (256, 3000)]),
    ("hac", "fp16", [(64, 1200), (192, 6000)]),
    ("synthetic_lstm128@v0", "fp16", [(64, 1200), (128, 6000)]),
    ("synthetic_lstm256@v0", "fp16", [(64, 1200), (128, 6000)]),
    ("synthetic_lstm768_prev4@v0", "fp16", [(64, 1000), (128, 5000)]),
    ("synthetic_lstm1024@v0", "fp16", [(64, 1200), (128, 6000)]),
    ("sup", "fp16", [(32, 1920), (128, 9984)]),
    ("sup", "fp8_ffn", [(32, 1920), (128, 9984)]),
    ("tx1536", "fp16", [(1, 1920), (64, 12288)]),
]


def _caller(kind, precision, tmp_path):
    from dorado_b200.config import load_model_config
    from dorado_b200.runner import B200Caller
    from dorado_b200.weights import synthetic_weights
    if kind == "tx1536":
        path = config_variant(tmp_path, depth=1)  # the workspace does not depend on the depth
    elif kind.startswith("synthetic_"):
        path = CONFIG_DIR / kind
    else:
        path = model_dir(kind)
    cfg = load_model_config(path)
    return B200Caller(cfg, synthetic_weights(cfg, 3), precision=precision)


@pytest.mark.parametrize("kind,precision,shapes", CASES, ids=[f"{k}-{p}" for k, p, _ in CASES])
def test_runner_bytes_is_the_arena_growth(tmp_path, kind, precision, shapes):
    from dorado_b200.runner import B200ModelRunner
    caller = _caller(kind, precision, tmp_path)
    for N, T in shapes:
        want = caller.runner_bytes(N, T)
        before = caller.stats()["arena_bytes"]
        runner = B200ModelRunner(caller, N, T)
        assert caller.stats()["arena_bytes"] - before == want, (N, T)
        print(f"\n[{kind} {precision}] runner_bytes({N}, {T}) = {want}")
        runner.close()
        assert caller.stats()["arena_bytes"] == before
    caller.close()


# shapes runner creation refuses: a transformer chunk that is a multiple of the stride but not of the chunk granularity
# (stride x upsample x 16 = 192), a chunk beyond the RoPE table, an LSTM batch that is not a multiple of 16 or 32
@pytest.mark.parametrize("kind,N,T", [("sup", 32, 1926), ("sup", 1, 24576 + 192), ("fast", 7, 1200), ("hac", 48, 1200)])
def test_runner_bytes_refuses_what_runner_creation_refuses(tmp_path, kind, N, T):
    from dorado_b200 import lib as L
    caller = _caller(kind, "fp16", tmp_path)
    with pytest.raises(L.B200Error) as e:
        caller.runner_bytes(N, T)
    assert e.value.status == L.B200_ERR_INVALID
    handle = C.c_void_p()
    assert L.load_library().b200_runner_create(caller.handle, N, T, C.byref(handle)) == L.B200_ERR_INVALID
    assert not handle.value
    caller.close()


@pytest.mark.parametrize("kind", ["mb384", "mb192"])
def test_modbase_runner_workspace(kind):
    """The modbase runner's workspace starts with the sequence buffer and bounds debug reads, at two batch sizes."""
    from dorado_b200 import lib as L
    from dorado_b200.config import load_modbase_config
    from dorado_b200.modbase import B200ModBaseCaller, B200ModBaseRunner
    from dorado_b200.weights import synthetic_modbase_weights
    cfg = load_modbase_config(modbase_dir(kind))
    caller = B200ModBaseCaller(cfg, synthetic_modbase_weights(cfg, 5))
    for N in (32, 96):
        sig, seq = modbase_inputs(cfg, N, 7)
        r = B200ModBaseRunner(caller, N)
        for i in range(N):
            r.accept_chunk(i, sig[i], seq[i])
        assert np.isfinite(r.call_chunks(N).astype(np.float32)).all()
        assert r.read_sequence_buffer().shape == (cfg.lstm_steps(), N, cfg.lstm_size)
        with pytest.raises(L.B200Error):
            r.debug_read_workspace(0, 1 << 40)
        r.close()
    caller.close()
