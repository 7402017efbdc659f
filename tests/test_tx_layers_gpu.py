"""Every kernel launch of the transformer plan, one at a time, against the float64 reference of tests/tx_layer_ref.py.

B200_DEBUG_TX_LAUNCHES=k (read when a runner is built) makes the forward return after its first k launches.  Each case
builds one runner per k = 0 .. launches from one B200Caller and snapshots the whole workspace after the forward, so
launch k is checked on its own, teacher-forced: its output buffer in snapshot k against the reference computed from
the input buffers of snapshot k - 1, every element within its bound.  Besides:
  - no stray writes, determinism: every buffer launch k does not write is bit-identical in snapshots k - 1 and k (two
    runners), so the buffers written before k are the same in every stopped runner;
  - the conv buffers' padding rows stay exactly zero (the next conv reads them as its padding);
  - the partial sums of squares (ss_a after fc2, ss_b after out_proj) against the float64 sums of the stored rows;
  - in fp8_ffn, norm1's E4M3 copy is the satfinite cast of its fp16 output, bit for bit;
  - the profile lists exactly the plan's launches, 5, 7 or 6 per layer, and the layout's size is the workspace's;
  - sensitivity: each mistake of tx_layer_ref.MUTATIONS, applied to the reference of one launch, puts the engine's real
    output at least 3 bounds away at the worst element.
The last launch (the CRF GEMM) writes the scores, read with the stop unset.

Chunk sizes are whole multiples of 16 tokens (the runner's granularity), so the token rows N T are a multiple of 16 in
every plan: the row counts below are ragged against the GEMMs' 128-row tiles and the attention's 128-query tiles, but
rmsnorm_kernel's 8-row grid tail cannot be reached through a model.

Measured worst error / bound of each launch kind and mode: DESIGN.md section 2.
"""
import time
import zlib

import numpy as np
import pytest

import tx_layer_ref as X
from conftest import CONFIG_DIR
from test_tx1536_cpu import config_variant

pytestmark = pytest.mark.gpu

SUP = CONFIG_DIR / "dna_r10.4.1_e8.2_400bps_sup@v5.0.0"
MARGIN = 3.0   # a simulated mistake must reach this many bounds at its worst element

# name: (model, depth, mode, N, samples per chunk, Wqkv gain)
CASES = {
    # 992 tokens: a ragged last query tile; chunk boundaries inside GEMM row tiles (RoPE at g % T); layer 0 without a norm
    "sup_fold": ("sup", 3, "fold", 3, 11904, 1.0),
    "sup_rmsnorm_pass": ("sup", 3, "rmsnorm_pass", 3, 11904, 1.0),
    "sup_fp8_ffn": ("sup", 3, "fp8_ffn", 3, 11904, 1.0),
    # peaked softmax: the running-max rescaling across key blocks
    "sup_wqkv_x3": ("sup", 3, "fold", 3, 11904, 3.0),
    # 640 tokens: five key blocks per query tile, K 6144
    "tx1536_fold": ("tx1536", 2, "fold", 1, 7680, 1.0),
    "tx1536_fp8_ffn": ("tx1536", 2, "fp8_ffn", 1, 7680, 1.0),
    # 336 tokens, 672 rows: no tile split when out_ss is set
    "dm128_fold": ("dm128", 2, "fold", 2, 4032, 1.0),
    "dm128_rmsnorm_pass": ("dm128", 2, "rmsnorm_pass", 2, 4032, 1.0),
}

_stats = {}        # (kind, mode) -> worst ratio
_sensitivity = {}  # mutation -> least worst ratio over the cases


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    print("\n[transformer launches vs float64 reference] worst error / bound per launch kind and mode:")
    for (kind, mode), r in sorted(_stats.items()):
        print(f"  {kind:18s} {mode:13s} {r:.3f}")
    print("[transformer launches] simulated mistakes, least worst ratio over the cases (must be >= 3):")
    for m, r in sorted(_sensitivity.items()):
        print(f"  {m:24s} {r:.1f}")


def _config(tmp_path, model, depth):
    from dorado_b200.config import load_model_config
    if model == "sup":
        text = (SUP / "config.toml").read_text()
        assert text.count("depth = 18\n") == 1
        d = tmp_path / f"sup_d{depth}"
        d.mkdir()
        (d / "config.toml").write_text(text.replace("depth = 18\n", f"depth = {depth}\n"))
    elif model == "tx1536":
        d = config_variant(tmp_path, depth=depth, name=f"tx1536_d{depth}")
    else:
        d = config_variant(tmp_path, depth=depth, d_model=128, nhead=2, ff=512, name=f"dm128_d{depth}")
    return load_model_config(d)


def _stat(kind, mode, r):
    _stats[(kind, mode)] = max(_stats.get((kind, mode), 0.0), r)


def _applies(mutation, mode, l, N):
    if mutation in ("qkv_gain_of_layer_l", "out_proj_raw_residual"):
        return mode != "rmsnorm_pass" and l == 1
    if mutation == "fc2_n2_gain":
        return mode == "fold" and l == 1
    if mutation == "rope_global_position":
        return N >= 2 and l == 1
    return mutation == "upsample_step_major" or l == 1


def _split(cfg, lay, ws):
    return {name: ws[off:off + nb] for name, (off, nb) in lay["buffers"].items()}


@pytest.mark.parametrize("case", list(CASES))
def test_every_launch(tmp_path, monkeypatch, case):
    from dorado_b200 import lib as L
    from dorado_b200.runner import B200Caller, B200ModelRunner
    from dorado_b200.weights import synthetic_weights
    t0 = time.time()
    model, depth, mode, N, T_in, wqkv_gain = CASES[case]
    cfg = _config(tmp_path, model, depth)
    assert cfg.normalise_chunk_size(T_in) == T_in
    w = synthetic_weights(cfg, 42)
    if wqkv_gain != 1.0:
        w = dict(w)
        for l in range(depth):
            k = f"transformer_encoder.{l}.self_attn.Wqkv.weight.tensor"
            w[k] = w[k] * np.float32(wqkv_gain)
    if mode == "rmsnorm_pass":
        monkeypatch.setenv("B200_TX_RMSNORM_PASS", "1")
    caller = B200Caller(cfg, w, **({"precision": "fp8_ffn"} if mode == "fp8_ffn" else {}))
    monkeypatch.delenv("B200_TX_RMSNORM_PASS", raising=False)
    ref = X.TxLayerRef(cfg, w, mode, N, T_in)
    lay = ref.lay
    plan = X.launches(cfg, mode)
    n = len(plan)
    assert n == X.launch_count(cfg, mode)
    sig = np.random.default_rng(zlib.crc32(case.encode())).standard_normal((N, T_in)).astype(np.float16)

    def snapshot(k):
        if k < n:
            monkeypatch.setenv("B200_DEBUG_TX_LAUNCHES", str(k))
        else:
            monkeypatch.delenv("B200_DEBUG_TX_LAUNCHES", raising=False)
        runner = B200ModelRunner(caller, N, T_in)
        try:
            for i in range(N):
                runner.accept_chunk(i, sig[i])
            scores = runner.forward_scores(N).astype(np.float64)
            ws = runner.debug_read_workspace(0, lay["bytes"])
            extra = {}
            if k == 0:
                with pytest.raises(L.B200Error):   # the layout's size is the workspace's
                    runner.debug_read_workspace(0, lay["bytes"] + 1)
            if k in (3, n):   # a stopped plan and the whole plan
                extra["profile"] = [name for name, _ in runner.profile(N)]
        finally:
            runner.close()
            monkeypatch.delenv("B200_DEBUG_TX_LAUNCHES", raising=False)
        return _split(cfg, lay, ws), scores, extra

    prev, _, _ = snapshot(0)
    assert all((b == 0).all() for b in prev.values()), "the workspace is not all zero before the first launch"
    worst = {}
    short = []   # simulated mistakes below the margin, asserted after every launch has been checked
    for k in range(1, n + 1):
        name, kind, idx = plan[k - 1]
        cur, scores, extra = snapshot(k)
        if "profile" in extra:
            names = extra["profile"]
            assert names[:k] == [p[0] for p in plan[:k]], names[:k + 1]
            if k < n:   # the plan stopped: what follows is the decode
                assert len(names) == k or names[k] not in {p[0] for p in plan}, names[:k + 1]
        # no stray writes, determinism
        written = X.writes(cfg, lay, kind, idx, mode)
        for buf, b in cur.items():
            if buf in written:
                rng_ = written[buf]
                if rng_ is not None:
                    lo, hi = rng_
                    assert np.array_equal(b[hi:], prev[buf][hi:]), f"launch {k} ({name}) wrote {buf} beyond its range"
                continue
            assert np.array_equal(b, prev[buf]), \
                f"launch {k} ({name}): {buf} changed, which it does not write (a stray write, or an earlier launch is not deterministic)"
        for i in range(len(cfg.convs) - 1):
            assert X.cbuf_padding_nonzero(cfg, lay, cur, i) == 0, f"launch {k} ({name}): padding rows of cbuf{i} not zero"
        inp = X.logical_inputs(cfg, lay, prev, mode)
        inp["signal"] = sig.astype(np.float64)
        got_all = X.logical_inputs(cfg, lay, cur, mode)
        got_all["scores"] = scores
        refs = ref.reference(kind, idx, inp)
        for out, (r, bnd) in refs.items():
            if out == "hid8":
                ff = cfg.tx.dim_feedforward
                outside, ratio = X.e4m3_cast_check(cur["hid"][:lay["rows"] * ff].reshape(-1, ff), r, bnd)
                assert outside == 0, f"launch {k} ({name}): {outside} E4M3 outputs outside the casts of their interval"
                wr = float(ratio.max())
            else:
                got = got_all[out]
                assert np.isfinite(got).all(), f"launch {k} ({name}): non-finite {out}"
                wr = X.worst_ratio(got, r, bnd)
                assert wr <= 1.0, f"launch {k} ({name}) {out}: worst error {wr:.3f} of the bound"
            _stat(kind, mode, wr)
            worst[f"{k}:{name}"] = wr
        if kind == "norm1" and mode == "fp8_ffn":
            rows, dm = lay["rows"], cfg.tx.d_model
            want = X.e4m3_sat_bytes(cur["att"].view(np.float16).astype(np.float32))
            assert np.array_equal(cur["qkv"][:rows * dm], want), f"launch {k}: the E4M3 copy is not the cast of the fp16 output"
        if "ss_b" in written:
            r = X.ss_ratio(got_all["y"], cur["ss_b"].view(np.float32))
            assert r <= 1.0
            _stat("ss_b", mode, r)
        if "ss_a" in written:
            r = X.ss_ratio(got_all["x"], cur["ss_a"].view(np.float32))
            assert r <= 1.0
            _stat("ss_a", mode, r)
        for m, mk in X.MUTATIONS.items():
            if mk != kind or not _applies(m, mode, idx, N):
                continue
            (out, (r, bnd)), = ref.reference(kind, idx, inp, mutation=m).items()
            if out == "hid8":
                ff = cfg.tx.dim_feedforward
                _, ratio = X.e4m3_cast_check(cur["hid"][:lay["rows"] * ff].reshape(-1, ff), r, bnd)
                mr = float(ratio.max())
            else:
                mr = X.worst_ratio(got_all[out], r, bnd)
            print(f"\n  [{case}] {m} at launch {k} ({name}): worst ratio {mr:.1f}")
            _sensitivity[m] = min(_sensitivity.get(m, np.inf), mr)
            if mr < MARGIN:
                short.append(f"{m}: the mistake reaches only {mr:.2f} bounds")
        prev = cur
    print(f"\n[{case}] {n} launches, worst ratio {max(worst.values()):.3f} ({max(worst, key=worst.get)}), "
          f"{time.time() - t0:.0f} s")
    caller.close()
    assert not short, short

