"""lstm_size 128 and 256 without a GPU: the two fixtures, the numpy oracle against the reference's own forward, and a CPU
model of how lstm_rec_kernel (dorado_b200/csrc/lstm_model.cu) partitions the recurrence over a thread-block cluster at
these widths.  The GPU side is tests/test_lstm128_256_gpu.py, which also pins the launch-shape model below to the plan
the library builds.

Both widths run the x-projection GEMM followed by the fp16 form lstm_rec_kernel<false, C, CL, NB>, with
CL = rec_cluster(C): 4 CTAs for 128, 8 for 256, so every CTA owns U = 32 hidden units (128 gate rows, 8 warps)."""
import pathlib
import re

import numpy as np
import pytest

from conftest import CONFIG_DIR

MODELS = {
    "lstm128": "synthetic_lstm128@v0",   # the fast@v5.0.0 shape at lstm_size 128 (state_len 3)
    "lstm256": "synthetic_lstm256@v0",   # the hac@v5.0.0 shape at lstm_size 256 (state_len 4)
}
WIDTHS = {"lstm128": 128, "lstm256": 256}
NBS = (16, 32, 64)                       # chunks per cluster: lstm_rec_chunks and B200_CLUSTER_CHUNKS
MAX_SMEM = 227 * 1024                    # dynamic shared memory of one sm_90a CTA
PTXAS_LOG = pathlib.Path(__file__).resolve().parents[1] / "dorado_b200" / "csrc" / "build" / "lstm_model.ptxas.log"


def model_dir(kind):
    return CONFIG_DIR / MODELS[kind]


def rec_cluster(C):
    """lstm_model.cu rec_cluster: CTAs per cluster."""
    return 4 if C <= 192 else 8


class RecCfg:
    """lstm_model.cu RecCfg<I8, C, CL, NB>, with its static_asserts; the fp16 form unless i8."""

    def __init__(self, C, CL, NB, i8=False):
        self.C, self.CL, self.NB = C, CL, NB
        self.EB = 1 if i8 else 2          # bytes per element of W_hh and h
        self.U = C // CL
        self.MT = 4 * self.U // 16
        self.THREADS = 32 * self.MT
        self.KE = 32 // self.EB
        self.KS = C // self.KE
        self.NT = NB // 8
        self.HS = C + 16 // self.EB
        self.GS = NB + 4
        self.PAIRS = self.U // 2 * NB // self.THREADS
        self.GX_AHEAD = self.PAIRS <= 2
        self.SMEM = 2 * NB * self.HS * self.EB + 4 * self.U * self.GS * 4

    def static_asserts_hold(self):
        shape = (self.C % self.KE == 0 and self.C % self.CL == 0 and self.U % 4 == 0 and self.NT % 2 == 0
                 and self.PAIRS >= 1 and (self.U // 2 * self.NB) % self.THREADS == 0)
        return shape and self.HS * self.EB % 128 == 16 and self.THREADS <= 1024 and 1 < self.CL <= 8


def lstm_rec_chunks(Np, override=None):
    """lstm_model.cu lstm_rec_chunks: chunks per cluster for a padded batch."""
    un = 32 if Np > 256 else 16
    if override is not None:
        assert override in NBS and Np % override == 0
        un = override
    while Np % un:
        un //= 2
    return un


# ---- fixtures and config ----------------------------------------------------------------------------------------------
def test_fixtures_parse():
    from dorado_b200.config import ACT_SWISH, ACT_TANH, load_model_config
    from dorado_b200.weights import tensor_specs
    c128 = load_model_config(model_dir("lstm128"))
    assert (c128.lstm_size, c128.lstm_layers, c128.stride, c128.state_len, c128.outsize) == (128, 5, 6, 3, 256)
    assert [(c.insize, c.size, c.winlen, c.stride, c.activation) for c in c128.convs] == [
        (1, 16, 5, 1, ACT_SWISH), (16, 16, 5, 1, ACT_SWISH), (16, 128, 19, 6, ACT_SWISH)]
    assert c128.clamp and c128.out_features is None and c128.lstm_inner_dim is None and c128.scale == 1.0
    c256 = load_model_config(model_dir("lstm256"))
    assert (c256.lstm_size, c256.lstm_layers, c256.stride, c256.state_len, c256.outsize) == (256, 5, 6, 4, 1024)
    assert [c.activation for c in c256.convs] == [ACT_SWISH, ACT_SWISH, ACT_TANH] and c256.convs[2].size == 256
    # neither CRF linear has a bias: no "9.linear.bias.tensor" among the weights
    for cfg in (c128, c256):
        assert cfg.bias is False
        specs = tensor_specs(cfg)
        assert specs["9.linear.weight.tensor"] == (cfg.outsize, cfg.lstm_size)
        assert "9.linear.bias.tensor" not in specs
        for l in range(5):
            assert specs[f"{4 + l}.rnn.weight_hh_l0.tensor"] == (4 * cfg.lstm_size, cfg.lstm_size)


def test_the_128_fixture_leaves_the_crf_bias_unset():
    text = (model_dir("lstm128") / "config.toml").read_text()
    crf = text[text.index('type = "linearcrfencoder"'):]
    assert "bias" not in crf.split("[[")[0]


@pytest.mark.parametrize("C,bias", [(128, False), (256, True)])
def test_decomposed_linear_bias_defaults_by_width(tmp_path, C, bias):
    """BasecallModelConfig.cpp:251: a decomposition `linear` sublayer without a `bias` key has a bias only above
    lstm_size 128 (config.py applies the same rule)."""
    from dorado_b200.config import load_model_config
    from dorado_b200.weights import tensor_specs
    text = (model_dir("lstm128" if C == 128 else "lstm256") / "config.toml").read_text()
    linear = f'[[encoder.sublayers]]\ntype = "linear"\nin_features = {C}\nout_features = 128\n\n'
    text = text.replace('[[encoder.sublayers]]\ntype = "linearcrfencoder"', linear +
                        '[[encoder.sublayers]]\ntype = "linearcrfencoder"')
    (tmp_path / "config.toml").write_text(text.replace(f"insize = {C}\nn_base", "insize = 128\nn_base"))
    cfg = load_model_config(tmp_path)
    assert cfg.lstm_size == C and cfg.out_features == 128 and cfg.bias is bias
    assert ("9.linear.bias.tensor" in tensor_specs(cfg)) is bias


@pytest.mark.parametrize("kind,N,T", [("lstm128", 2, 600), ("lstm256", 1, 720)])
def test_forward_matches_reference(reference, tmp_path, kind, N, T):
    from oracle import nn_oracle
    from dorado_b200.config import load_model_config
    from dorado_b200.weights import save_b2w, synthetic_weights
    cfg = load_model_config(model_dir(kind))
    w = synthetic_weights(cfg, 42)
    save_b2w(tmp_path / "w.b2w", w)
    h = reference.load_model(model_dir(kind), tmp_path / "w.b2w")
    info = reference.model_info(h)
    assert info["stride"] == cfg.stride and info["outsize"] == cfg.outsize and info["state_len"] == cfg.state_len
    assert info["clamp"] == cfg.clamp
    sig = np.random.default_rng(7).standard_normal((N, cfg.normalise_chunk_size(T))).astype(np.float32)
    ref = reference.forward(h, sig)
    mine = nn_oracle.forward(cfg, w, sig)
    assert ref.shape == mine.shape == (N, sig.shape[1] // cfg.stride, cfg.outsize)
    np.testing.assert_allclose(mine, ref, rtol=0, atol=5e-5)
    reference.free_model(h)


# ---- partition of lstm_rec_kernel at 128 and 256 ----------------------------------------------------------------------
SHAPES = [(C, NB) for C in (128, 256) for NB in NBS]


@pytest.mark.parametrize("C,NB", SHAPES)
def test_rec_cfg(C, NB):
    cfg = RecCfg(C, rec_cluster(C), NB)
    assert cfg.static_asserts_hold()
    assert (cfg.CL, cfg.U, cfg.THREADS, cfg.KS) == ((4, 32, 256, 8) if C == 128 else (8, 32, 256, 16))
    assert cfg.PAIRS == NB // 16 and cfg.GX_AHEAD == (NB <= 32)
    assert cfg.SMEM <= MAX_SMEM
    # 4 KS A-fragment registers per thread hold W_hh: 32 for 128, 64 for 256
    assert 4 * cfg.KS == C // 4
    if C == 256:   # the int8 form: the same partition and gx schedule, half the K steps, h rows of C + 16 bytes
        i8 = RecCfg(C, rec_cluster(C), NB, i8=True)
        assert i8.static_asserts_hold()
        assert (i8.THREADS, i8.PAIRS, i8.GX_AHEAD, i8.KS, i8.HS) == (cfg.THREADS, cfg.PAIRS, cfg.GX_AHEAD, C // 32, C + 16)
        assert i8.SMEM < cfg.SMEM


@pytest.mark.parametrize("C", [128, 256])
def test_every_weight_is_held_once(C):
    """Warp w of CTA `rank` holds local gate rows 16 w + lane / 4 (+ 8) <-> W_hh rows (r / U) C + rank U + r % U, all
    K = C columns 16 ks + 2 (lane % 4) (+ 1, + 8, + 9): every W_hh element sits in exactly one register of the cluster."""
    cfg = RecCfg(C, rec_cluster(C), 16)
    U = cfg.U
    held = np.zeros((4 * C, C), np.int32)
    cols = np.array([ks * 16 + d for ks in range(cfg.KS) for d in (0, 1, 8, 9)])
    for rank in range(cfg.CL):
        for warp in range(cfg.MT):
            for lane in range(32):
                for r in (warp * 16 + lane // 4, warp * 16 + lane // 4 + 8):
                    np.add.at(held[(r // U) * C + rank * U + r % U], cols + 2 * (lane % 4), 1)
    assert (held == 1).all()


@pytest.mark.parametrize("C,NB", SHAPES)
def test_every_cell_has_one_owner_and_reads_its_own_gate_rows(C, NB):
    """Cells: pair q = tid + j THREADS -> units rank U + u, + 1 (u = 2 (q % (U / 2))), chunk q / (U / 2).  Each (unit,
    chunk) of the NB chunks has one owner thread in one CTA, and the four gate pre-activations it reads from the gate
    buffer, rows g U + u + e, were written by exactly one (warp, lane, n tile, element) of its own CTA, whose accumulator
    is W_hh row g C + rank U + u + e times h of that chunk."""
    cfg = RecCfg(C, rec_cluster(C), NB)
    U = cfg.U
    written = {}   # (rank, local gate row, chunk) -> writer
    for rank in range(cfg.CL):
        for warp in range(cfg.MT):
            for lane in range(32):
                for nt in range(cfg.NT):
                    for e in range(4):
                        r = warp * 16 + lane // 4 + 8 * (e // 2)
                        n = nt * 8 + 2 * (lane % 4) + e % 2
                        key = (rank, r, n)
                        assert key not in written
                        written[key] = (warp, lane, nt, e)
    assert len(written) == cfg.CL * 4 * U * NB
    cells = {}
    for rank in range(cfg.CL):
        for tid in range(cfg.THREADS):
            for j in range(cfg.PAIRS):
                q = tid + j * cfg.THREADS
                u, n = 2 * (q % (U // 2)), q // (U // 2)
                assert n < NB
                for e in range(2):
                    cell = (rank * U + u + e, n)
                    assert cell not in cells
                    cells[cell] = (rank, tid)
                    for g in range(4):
                        r = g * U + u + e
                        assert (rank, r, n) in written
                        assert (r // U) * C + rank * U + r % U == g * C + cell[0]
    assert len(cells) == C * NB
    # h_t of a cell goes to columns rank U + u, + 1 of its chunk's row in every CTA's copy: each copy gets all C x NB
    assert sorted(cells) == [(c, n) for c in range(C) for n in range(NB)]


@pytest.mark.parametrize("C", [128, 256])
def test_launch_shape(C):
    """lstm_rec.ctas = Np / NB x CL for every padded batch, default and overridden chunks per cluster."""
    CL = rec_cluster(C)
    for Np in range(32, 4097, 32):
        nb = lstm_rec_chunks(Np)
        assert nb == (32 if Np > 256 else 16) and Np % nb == 0
        assert Np // nb * CL == (Np // 32 * CL if Np > 256 else Np // 16 * CL)
        for override in NBS:
            if Np % override == 0:
                assert lstm_rec_chunks(Np, override) == override
    assert lstm_rec_chunks(512) == 32 and 512 // 32 * CL == (64 if C == 128 else 128)


def _ptxas_entries():
    """(C, CL, NB) -> (registers, stack bytes, spill store bytes, spill load bytes) of the fp16 form of lstm_rec_kernel from
    the build's ptxas log."""
    text = PTXAS_LOG.read_text()
    out = {}
    for block in re.split(r"ptxas info\s*: Compiling entry function ", text)[1:]:
        m = re.match(r"'_ZN4b200\w*?15lstm_rec_kernelILb0ELi(\d+)ELi(\d+)ELi(\d+)E", block)
        if not m:
            continue
        frame = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
        regs = re.search(r"Used (\d+) registers", block)
        out[tuple(int(x) for x in m.groups())] = (int(regs.group(1)), *(int(x) for x in frame.groups()))
    return out


def test_ptxas_reports_no_spills_in_the_fp16_rec_form():
    """Every lstm_rec_kernel<false, 128 | 256, CL, NB> of the built library: no stack frame, no spills, one CTA of 256 threads
    within the 255-register cap."""
    if not PTXAS_LOG.is_file():
        pytest.skip("dorado_b200/csrc/build/lstm_model.ptxas.log not built")
    entries = _ptxas_entries()
    for C, NB in SHAPES:
        key = (C, rec_cluster(C), NB)
        assert key in entries, f"no lstm_rec_kernel<false, {C}, {key[1]}, {NB}> in the ptxas log"
        regs, stack, st, ld = entries[key]
        assert (stack, st, ld) == (0, 0, 0), (key, entries[key])
        assert regs <= 255
