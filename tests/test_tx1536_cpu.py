"""The 1536-wide transformer without a GPU: the fixture, the numpy oracle against the reference's own CPU TxModel forward,
a restatement of how tx_attention_tc_kernel (dorado_b200/csrc/tx_model.cu) picks the key blocks of a query tile, and the
build's ptxas report of that kernel.  The GPU side is tests/test_tx1536_gpu.py.

The fixture synthetic_tx1536@v0 is synthetic: its encoder layer (d_model 1536, 24 heads, window (255, 256), feed-forward
6144) is the second shape the reference's tiled transformer path names; the rest of it copies the sup@v5 fixture."""
import pathlib
import re

import numpy as np
import pytest

from conftest import CONFIG_DIR

MODEL = "synthetic_tx1536@v0"
PTXAS_LOG = pathlib.Path(__file__).resolve().parents[1] / "dorado_b200" / "csrc" / "build" / "tx_model.ptxas.log"

# tx_model.cu constants
AT_BQ = AT_BK = 128
AT_MAX_WIN = 256
AT_MAXBLK = 5
AT_SLOTS = 3
AT_SMEM = 1024 + (1 + 2 * AT_SLOTS) * 128 * 64 * 2 + 64


def model_dir():
    return CONFIG_DIR / MODEL


def config_variant(tmp_path, depth=None, d_model=None, nhead=None, ff=None, window=None, name="variant"):
    """A copy of the fixture's config.toml with the encoder shape changed; returns its directory."""
    text = (model_dir() / "config.toml").read_text()

    def sub(pattern, value, count):
        nonlocal text
        text, n = re.subn(pattern, value, text)
        assert n == count, (pattern, n)

    if depth is not None:
        sub(r"depth = 18\n", f"depth = {depth}\n", 1)
    if d_model is not None:
        sub(r"(?m)^size = 1536\n", f"size = {d_model}\n", 1)            # the last conv
        sub(r"insize = 1536\n", f"insize = {d_model}\n", 1)              # the CRF linear
        sub(r"d_model = 1536\n", f"d_model = {d_model}\n", 2)            # upsample and encoder layer
    if nhead is not None:
        sub(r"nhead = 24\n", f"nhead = {nhead}\n", 1)
    if ff is not None:
        sub(r"dim_feedforward = 6144\n", f"dim_feedforward = {ff}\n", 1)
    if window is not None:
        sub(r"attn_window = \[ 255, 256,\]", f"attn_window = [ {window[0]}, {window[1]},]", 1)
    d = tmp_path / name
    d.mkdir()
    (d / "config.toml").write_text(text)
    return d


def test_fixture_parses():
    from dorado_b200.config import load_model_config
    from dorado_b200.weights import tensor_specs
    cfg = load_model_config(model_dir())
    tx = cfg.tx
    assert (tx.d_model, tx.nhead, tx.attn_window, tx.dim_feedforward) == (1536, 24, (255, 256), 6144)
    assert (tx.depth, tx.upsample_scale, tx.crf_scale, tx.max_seq_len) == (18, 2, 5.0, 2048)
    assert abs(tx.deepnorm_alpha - 2.4494897) < 1e-6
    assert (cfg.stride, cfg.state_len, cfg.outsize, cfg.blank_score) == (6, 5, 4096, 2.0)
    assert cfg.chunk_size_granularity() == 192
    assert cfg.convs[-1].size == 1536 and cfg.convs[-1].winlen == 5 and cfg.convs[-1].insize == 128
    specs = tensor_specs(cfg)
    assert specs["transformer_encoder.0.self_attn.Wqkv.weight.tensor"] == (4608, 1536)
    assert specs["transformer_encoder.17.ff.fc1.weight.tensor"] == (12288, 1536)
    assert specs["upsample.linear.weight.tensor"] == (3072, 1536)
    assert specs["crf.linear.weight.tensor"] == (4096, 1536)
    # the C descriptor carries the shape unchanged
    from dorado_b200 import lib as L
    d = L.model_desc_from_config(cfg)
    assert (d.d_model, d.nhead, d.dim_feedforward, d.depth, d.attn_window_upper, d.attn_window_lower) == (
        1536, 24, 6144, 18, 255, 256)


def test_fixture_says_it_is_synthetic():
    assert "SYNTHETIC" in (model_dir() / "config.toml").read_text().splitlines()[0]


# The reference's CPU forward drops one key per query split (cpu_split_quirk, oracle/nn_oracle.py); against the true window the
# fp32 oracle differs by that.  Measured at depth 2, N = 1, 7680 samples (640 tokens), weights seed 42, signal seed 7:
# max |true window - reference| = 2.2e-4, no score beyond 1e-3.
TRUE_WINDOW_MAX = 1e-3
TRUE_WINDOW_FRAC = 0.0


def test_forward_matches_reference(reference, tmp_path):
    from oracle import nn_oracle
    from dorado_b200.config import load_model_config
    from dorado_b200.weights import save_b2w, synthetic_weights
    d = config_variant(tmp_path, depth=2, name="tx1536_depth2")
    cfg = load_model_config(d)
    w = synthetic_weights(cfg, 42)
    save_b2w(tmp_path / "w.b2w", w)
    h = reference.load_model(d, tmp_path / "w.b2w")
    info = reference.model_info(h)
    assert info["stride"] == cfg.stride and info["outsize"] == cfg.outsize and info["state_len"] == cfg.state_len
    T = 7680   # 640 tokens: the middle query tiles see all five key blocks
    assert cfg.normalise_chunk_size(T) == T and T // (cfg.stride * cfg.tx.upsample_scale) == 640
    sig = np.random.default_rng(7).standard_normal((1, T)).astype(np.float32)
    ref = reference.forward(h, sig)
    mine = nn_oracle.forward(cfg, w, sig, cpu_split_quirk=True)
    assert ref.shape == mine.shape == (1, T // cfg.stride, 4096)
    np.testing.assert_allclose(mine, ref, rtol=0, atol=5e-5)
    true_win = nn_oracle.forward(cfg, w, sig, cpu_split_quirk=False)
    diff = np.abs(true_win - ref)
    print(f"\n[tx1536 depth 2] true window vs reference CPU forward: max {diff.max():.2e}, "
          f"{(diff > 1e-3).mean():.2e} of scores beyond 1e-3")
    assert diff.max() > 0                      # the quirk does change something at this length
    assert diff.max() <= TRUE_WINDOW_MAX and (diff > 1e-3).mean() <= TRUE_WINDOW_FRAC
    reference.free_model(h)


# ---- key blocks of a query tile (tx_attention_tc_kernel) ---------------------------------------------------------------
def kernel_blocks(q0, T, win_upper, win_lower):
    """The kernel's kb_first .. kb_last for the query tile starting at q0."""
    kb_first = 0 if q0 - win_upper < 0 else (q0 - win_upper) // AT_BK
    kb_last = min((q0 + AT_BQ - 1 + win_lower) // AT_BK, (T - 1) // AT_BK)
    return kb_first, kb_last


WINDOWS = sorted({(u, l) for u in list(range(0, AT_MAX_WIN + 1, 17)) + [127, 128, 129, 255, 256]
                  for l in list(range(0, AT_MAX_WIN + 1, 17)) + [127, 128, 129, 255, 256]})
TS = [1, 100, 127, 128, 129, 640, 1000, 1024, 2048]


@pytest.mark.parametrize("T", TS)
def test_block_range_covers_the_window(T):
    worst = 0
    i = np.arange(T)
    for wu, wl in WINDOWS:
        for q0 in range(0, T, AT_BQ):
            kb_first, kb_last = kernel_blocks(q0, T, wu, wl)
            nblk = kb_last - kb_first + 1
            worst = max(worst, nblk)
            assert 1 <= nblk <= AT_MAXBLK, (T, wu, wl, q0, nblk)
            assert kb_last * AT_BK < T                                   # no block starts past the chunk
            rows = i[q0:q0 + AT_BQ]
            first_key = np.maximum(rows - wu, 0)
            last_key = np.minimum(rows + wl, T - 1)
            assert (first_key >= kb_first * AT_BK).all()                 # every visible key is in a loaded block
            assert (last_key < (kb_last + 1) * AT_BK).all()
            assert (nblk - 1) // AT_SLOTS <= 1                           # block b uses slot b % 3: refilled at most once
    if T >= 640:
        assert worst == AT_MAXBLK                                        # some tiles of long chunks see all five
    if T >= 384:
        assert max(kernel_blocks(q0, T, 127, 128)[1] - kernel_blocks(q0, T, 127, 128)[0] + 1
                   for q0 in range(0, T, AT_BQ)) == 3                     # sup keeps its three blocks


def test_block_bound_is_tight():
    """AT_MAXBLK = 1 + ceil(256 / 128) + floor((127 + 256) / 128) = 5 is reached by (255, 256) and (256, 256) and not
    exceeded by any window in range."""
    assert 1 + -(-AT_MAX_WIN // AT_BK) + (AT_BQ - 1 + AT_MAX_WIN) // AT_BK == AT_MAXBLK
    for w in ((255, 256), (256, 256)):
        assert max(kernel_blocks(q0, 2048, *w)[1] - kernel_blocks(q0, 2048, *w)[0] + 1 for q0 in range(0, 2048, 128)) == 5


def _attention_ptxas():
    text = PTXAS_LOG.read_text()
    for block in re.split(r"ptxas info\s*: Compiling entry function ", text)[1:]:
        if "tx_attention_tc_kernel" not in block.split("'")[1]:
            continue
        frame = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
        regs = re.search(r"Used (\d+) registers", block)
        return int(regs.group(1)), *(int(x) for x in frame.groups())
    return None


# tx_attention_tc_kernel at the 128-register cap of __launch_bounds__(256, 2): its 64 fp32 scores, 32 output accumulators and
# the P / V fragments leave no room for a few per-row and address values, which ptxas keeps on the stack.  The
# three-block kernel this one replaced already spilled (144-byte frame, 164 / 160 bytes of spill stores / loads); the ring
# bookkeeping adds some (144-byte frame, 264 / 212 bytes).  The bounds hold it there.
MAX_STACK_BYTES = 144
MAX_SPILL_BYTES = 264


def test_ptxas_attention_kernel():
    """One attention instantiation for every window: at most 128 registers (two CTAs of 256 threads per SM by registers)
    and the 113 KB shared-memory footprint sup had before, with spills no larger than measured."""
    if not PTXAS_LOG.is_file():
        pytest.skip("dorado_b200/csrc/build/tx_model.ptxas.log not built")
    entry = _attention_ptxas()
    assert entry is not None, "no tx_attention_tc_kernel in the ptxas log"
    regs, stack, spill_st, spill_ld = entry
    print(f"\n[tx_attention_tc_kernel] {regs} registers, {stack} B stack, {spill_st} B spill stores, {spill_ld} B spill loads, "
          f"{AT_SMEM} B dynamic shared memory")
    assert regs <= 128
    assert 2 * regs * 256 <= 65536
    assert stack <= MAX_STACK_BYTES and spill_st <= MAX_SPILL_BYTES and spill_ld <= MAX_SPILL_BYTES
    assert AT_SMEM == 115776 and AT_SMEM <= 227 * 1024
    assert len(re.findall(r"Compiling entry function '\w*tx_attention_tc_kernel", PTXAS_LOG.read_text())) == 1
