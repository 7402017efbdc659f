"""lstm_size 768 and 1024 without a GPU: the config parser (pre-v4 and v4 layouts), the numpy oracle against the
reference's own forward, and a CPU model of how lstm_grid_rec_kernel (dorado_b200/csrc/lstm_model.cu) partitions the
recurrence and sizes its launches.  The GPU side is tests/test_wide_lstm_gpu.py, which also pins the launch-shape model
below to the plan the library builds."""
import pathlib

import numpy as np
import pytest

from conftest import CONFIG_DIR

WIDE_MODELS = {
    "lstm768": "synthetic_lstm768_prev4@v0",   # pre-v4 layout, lstm_size 768 (the RNA sup shape)
    "lstm1024": "synthetic_lstm1024@v0",       # v4 layout, lstm_size 1024
}


def model_dir(kind):
    return CONFIG_DIR / WIDE_MODELS[kind]


REF_RNA004 = pathlib.Path("/root/reference/tests/data/model_configs/rna004_130bps_sup@v3.0.1")

UNITS = 16       # GR_UNITS: hidden units per CTA
THREADS = 256    # GR_THREADS: 8 warps, gate = warp % 4, K half = warp // 4
SMS = 132        # H100 SXM
CTAS_PER_SM = 1  # ptxas: 179-243 registers x 256 threads per CTA (DESIGN.md section 3)


def test_pre_v4_config():
    from dorado_b200.config import ACT_SWISH, load_model_config
    cfg = load_model_config(model_dir("lstm768"))
    assert (cfg.lstm_size, cfg.lstm_layers, cfg.stride, cfg.state_len, cfg.outsize) == (768, 5, 5, 5, 4096)
    assert cfg.bias and not cfg.clamp and cfg.out_features is None and cfg.lstm_inner_dim is None
    assert cfg.scale == 5.0 and cfg.blank_score == 2.0 and cfg.num_features == 1
    assert [(c.insize, c.size, c.winlen, c.stride, c.activation) for c in cfg.convs] == [
        (1, 4, 5, 1, ACT_SWISH), (4, 16, 5, 1, ACT_SWISH), (16, 768, 19, 5, ACT_SWISH)]
    assert (cfg.qscale, cfg.qbias) == (pytest.approx(0.9), pytest.approx(-0.1))


def test_pre_v4_config_matches_the_reference_fields():
    """The fields BasecallModelConfigTest.cpp pins for rna004_130bps_sup@v3.0.1, parsed from the reference's own file."""
    from dorado_b200.config import ACT_SWISH, load_model_config
    try:
        present = (REF_RNA004 / "config.toml").is_file()
    except OSError:
        present = False
    if not present:
        pytest.skip("reference model configs not available")
    cfg = load_model_config(REF_RNA004)
    assert cfg.bias is True and cfg.num_features == 1 and cfg.stride == 5 and cfg.lstm_size == 768
    assert cfg.blank_score == 2.0 and cfg.scale == 5.0 and cfg.state_len == 5 and cfg.outsize == 4096
    assert cfg.clamp is False and cfg.out_features is None
    assert cfg.qbias == pytest.approx(-0.1) and cfg.qscale == pytest.approx(0.9)
    assert [(c.insize, c.size, c.winlen, c.stride, c.activation) for c in cfg.convs] == [
        (1, 4, 5, 1, ACT_SWISH), (4, 16, 5, 1, ACT_SWISH), (16, 768, 19, 5, ACT_SWISH)]


def test_v4_config_of_width_1024():
    from dorado_b200.config import ACT_SWISH, ACT_TANH, load_model_config
    cfg = load_model_config(model_dir("lstm1024"))
    assert (cfg.lstm_size, cfg.lstm_layers, cfg.stride, cfg.state_len, cfg.outsize) == (1024, 5, 6, 5, 4096)
    assert cfg.clamp and not cfg.bias and cfg.scale == 1.0 and cfg.out_features is None
    assert [c.activation for c in cfg.convs] == [ACT_SWISH, ACT_SWISH, ACT_TANH]


def test_pre_v4_weights_carry_the_crf_bias():
    """crf_utils.cpp: the linear bias follows the linear weight whenever the config has a bias, decomposed or not."""
    from dorado_b200.config import load_model_config
    from dorado_b200.weights import tensor_specs
    specs = tensor_specs(load_model_config(model_dir("lstm768")))
    assert specs["9.linear.weight.tensor"] == (4096, 768) and specs["9.linear.bias.tensor"] == (4096,)
    assert list(specs)[-2:] == ["9.linear.weight.tensor", "9.linear.bias.tensor"]
    assert "9.linear.bias.tensor" not in tensor_specs(load_model_config(model_dir("lstm1024")))


@pytest.mark.parametrize("kind,N,T", [("lstm768", 1, 400), ("lstm1024", 1, 360)])
def test_wide_forward_matches_reference(reference, tmp_path, kind, N, T):
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
    assert ref.shape == mine.shape
    # 5 tanh(z) (the 768 model) multiplies fp32 rounding differences in z by up to 5
    np.testing.assert_allclose(mine, ref, rtol=0, atol=5e-5 * (5.0 if cfg.scale == 5.0 else 1.0))
    reference.free_model(h)


# ---- partition of lstm_grid_rec_kernel -------------------------------------------------------------------------------
def a_fragment_rows(C, rank, warp, lane):
    """W_hh rows and columns a thread holds: tile gate = warp % 4, rows gate * C + 16 rank + lane / 4 (+ 8), K half
    warp / 4 of C / 32 k steps, columns 16 ks + 2 (lane % 4) (+ 1, + 8, + 9)."""
    gate, kh = warp % 4, warp // 4
    rows = [gate * C + UNITS * rank + lane // 4 + 8 * hi for hi in range(2)]
    cols = [kh * (C // 2) + ks * 16 + 2 * (lane % 4) + d for ks in range(C // 32) for d in (0, 1, 8, 9)]
    return rows, cols


@pytest.mark.parametrize("C", [768, 1024])
def test_every_weight_is_held_once(C):
    """Each W_hh element sits in exactly one register of one thread of the group, and the two K halves of a row
    cover K exactly once."""
    G = C // UNITS
    held = np.zeros((4 * C, C), np.int32)
    for rank in range(G):
        for warp in range(THREADS // 32):
            for lane in range(32):
                rows, cols = a_fragment_rows(C, rank, warp, lane)
                for r in rows:
                    np.add.at(held[r], cols, 1)
    assert (held == 1).all()


@pytest.mark.parametrize("C,NB", [(768, 32), (768, 64), (1024, 32), (1024, 64)])
def test_every_gate_unit_chunk_has_one_owner(C, NB):
    """Accumulators: warp (gate, K half) lane holds rows lane / 4 (+ 8) of its gate tile for chunks 8 nt + 2 (lane % 4)
    (+ 1); both K halves of a (gate, unit, chunk) are summed by exactly one gate-math thread, which owns whole cells."""
    G = C // UNITS
    partial = {}
    for rank in range(G):
        for warp in range(THREADS // 32):
            gate, kh = warp % 4, warp // 4
            for lane in range(32):
                for nt in range(NB // 8):
                    for e in range(4):
                        unit = UNITS * rank + lane // 4 + 8 * (e // 2)
                        chunk = 8 * nt + 2 * (lane % 4) + e % 2
                        key = (gate, unit, chunk, kh)
                        assert key not in partial
                        partial[key] = (rank, warp, lane, nt, e)
    assert len(partial) == 4 * C * NB * 2
    cells = {}
    pairs = UNITS // 2 * NB // THREADS
    for rank in range(G):
        for tid in range(THREADS):
            for j in range(pairs):
                q = tid + j * THREADS
                u, n = 2 * (q % (UNITS // 2)), q // (UNITS // 2)
                for e in range(2):
                    cell = (UNITS * rank + u + e, n)
                    assert cell not in cells
                    cells[cell] = (rank, tid)
                    for g in range(4):
                        assert (g, cell[0], n, 0) in partial and (g, cell[0], n, 1) in partial
    assert len(cells) == C * NB


@pytest.mark.parametrize("C", [768, 1024])
def test_barrier_targets(C):
    """CTAs arrive once per step on their group's counter (zeroed before the launch) and step s waits for G s arrivals,
    so the count after step s is G (s + 1).  Under any interleaving a CTA that starts step s finds every row h_{s-1}
    stored, and no CTA is ever more than one step ahead of another (so the row it writes is not one still being read)."""
    G = C // UNITS
    steps = 12
    rng = np.random.default_rng(C)
    done = [0] * G        # steps completed (h stored, arrival counted) per CTA
    counter = 0
    while min(done) < steps:
        r = int(rng.integers(G))
        s = done[r]
        if s == steps or counter < G * s:
            continue      # finished, or still waiting for step s - 1 of the group
        assert all(d >= s for d in done)          # every h_{s-1} row of the group is stored
        assert max(done) - min(done) <= 1
        done[r] += 1
        counter += 1
        if min(done) == max(done):
            assert counter == G * done[0]         # the target after step s is G (s + 1)
    assert counter == G * steps


def grid_shape(Np, max_groups32, max_groups64, runners):
    """lstm_model.cu grid_shape: (chunks per group, groups per launch, launches per layer)."""
    nb = 64 if (max_groups64 >= 1 and Np % 64 == 0 and Np // 64 >= max_groups64) else 32
    max_groups = max_groups64 if nb == 64 else max_groups32
    tiles = Np // nb
    groups = min(tiles, max(1, max_groups // max(1, runners)))
    return nb, groups, -(-tiles // groups)


@pytest.mark.parametrize("C", [768, 1024])
def test_launch_shapes_fit_the_gpu_and_cover_the_batch(C):
    G = C // UNITS
    mg = CTAS_PER_SM * SMS // G
    for Np in range(32, 2049, 32):
        for runners in range(1, 5):
            nb, groups, launches = grid_shape(Np, mg, mg, runners)
            assert Np % nb == 0
            assert groups * G <= CTAS_PER_SM * SMS
            covered = [i * groups + g for i in range(launches) for g in range(min(groups, Np // nb - i * groups))]
            assert covered == list(range(Np // nb))     # every chunk tile exactly once
            assert min(groups, Np // nb - (launches - 1) * groups) >= 1
