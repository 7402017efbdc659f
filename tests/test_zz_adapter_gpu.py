"""The reference-side binding EXECUTED: oracle/_ref/adapter_host is include/B200ModelRunner.h compiled against the reference's
own headers (ModelRunnerBase, BasecallModelConfig, crf_utils) and libtorch (oracle/Makefile `ref`, built by build() where
the reference sources are available; the binary travels with the tree to the GPU machine).  It drives the engine only through dorado::basecall::ModelRunnerBase --
accept_chunk(at::Tensor), call_chunks(), sample_stats(), terminate()/restart() -- and must return exactly what the ctypes
path returns for the same chunks."""
import pathlib
import subprocess

import numpy as np
import pytest

from conftest import model_dir

pytestmark = pytest.mark.gpu
ROOT = pathlib.Path(__file__).resolve().parents[1]
HOST = ROOT / "oracle" / "_ref" / "adapter_host"


@pytest.mark.parametrize("kind,batch,chunk,n", [("fast", 16, 1200, 40), ("sup", 4, 1536, 6)])
def test_cpp_adapter_matches_ctypes_path(tmp_path, kind, batch, chunk, n):
    from dorado_b200.config import load_model_config
    from dorado_b200.runner import B200Caller, B200ModelRunner
    from dorado_b200.weights import save_b2w, synthetic_weights
    if not HOST.exists():
        pytest.fail(f"{HOST} is missing: run `make -C oracle ref` where the reference sources exist (it travels with the tree)")
    cfg = load_model_config(model_dir(kind))
    w = synthetic_weights(cfg, 42)
    T = cfg.normalise_chunk_size(chunk)
    sig = np.random.default_rng(11).standard_normal((n, T)).astype(np.float16)
    save_b2w(tmp_path / "w.b2w", w)
    sig.tofile(tmp_path / "sig.f16")
    out = tmp_path / "out.txt"
    r = subprocess.run([str(HOST), str(model_dir(kind)), str(tmp_path / "w.b2w"), str(tmp_path / "work"), str(batch), str(chunk),
                        str(tmp_path / "sig.f16"), str(n), str(out)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = out.read_text().splitlines()
    head = {l.split()[0]: l.split()[1:] for l in lines if not l.startswith("chunk")}
    assert head["name"][0].startswith("B200ModelRunner_0_")
    assert [int(x) for x in head["dims"]] == [batch, T, cfg.stride]
    assert head["timeouts"][:2] == ["300000", "30000"] and head["timeouts"][3] == "0"
    assert head["stats"][0] == "batches_called" and float(head["stats"][1]) == (n + batch - 1) // batch
    assert float(head["stats"][3]) > 0                      # model_decode_ms
    assert head["terminate_refuses"] == ["1", "restart_ok", "1"]
    got = [l.split()[1:] for l in lines if l.startswith("chunk")]
    assert len(got) == n
    runner = B200ModelRunner(B200Caller(cfg, w), batch, chunk)
    k = 0
    for start in range(0, n, batch):
        cnt = min(batch, n - start)
        for i in range(cnt):
            runner.accept_chunk(i, sig[start + i])
        for c in runner.call_chunks(cnt):
            seq, qstr, mv = got[k]
            assert seq == c.sequence and qstr == c.qstring
            assert mv == "".join("1" if m else "0" for m in c.moves)
            k += 1
