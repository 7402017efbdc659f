"""conv_lstm_v3 modified-base models without a GPU: config parsing against the reference's rules, and the numpy oracle
(oracle/modbase_oracle.py) against the reference's own CPU model (oracle/_ref/libmodbase_ref.so, built from the
reference tree where it is available).

Output length: every ModsConv pads by winlen // 2, so 600-sample chunks of the 6mA shape give 101 steps
((600 + 16 - 16) / 6 + 1 for sig_conv3, (100 + 16 - 16) + 1 for seq_conv2), not chunked_output_TC's 600 / 6 = 100.
test_oracle_matches_reference pins that to the reference's forward."""
import os
import pathlib

import numpy as np
import pytest

from conftest import CONFIG_DIR

MODBASE = {
    "mb384": "synthetic_modbase_v3_384@v0",      # the 6mA@v4 shape: lstm 384, 2 classes, no upsample
    "mb192": "synthetic_modbase_v3_192_up@v0",   # lstm 192, 3 classes, LinearUpsample x 2
}
REF_ROOT = pathlib.Path(os.environ.get("DORADO_REFERENCE", "/root/reference"))
REF_6MA = REF_ROOT / "tests" / "data" / "model_configs" / "dna_r10.4.1_e8.2_400bps_sup@v5.0.0_6mA@v4"
# fp16-emulating oracle vs the fp32 oracle, probabilities (measured 2.0e-3 / 1.5e-3 at most on 4 chunks)
FP16_VS_FP32_MAX = 8e-3


def modbase_dir(kind):
    return CONFIG_DIR / MODBASE[kind]


def modbase_inputs(cfg, N, seed):
    """fp16 signal [N, chunk_size] and a random k-mer one-hot encoding [N, T_seq, 4 kmer_len] int8."""
    rng = np.random.default_rng(seed)
    sig = rng.standard_normal((N, cfg.chunk_size)).astype(np.float16)
    T, Cc = cfg.chunked_sequence_input_TC()
    seq = np.zeros((N, T, Cc), np.int8)
    base = rng.integers(0, 4, (N, T, cfg.kmer_len))
    for k in range(cfg.kmer_len):
        seq[np.arange(N)[:, None], np.arange(T)[None, :], 4 * k + base[:, :, k]] = 1
    return sig, seq


def _load(kind):
    from dorado_b200.config import load_modbase_config
    return load_modbase_config(modbase_dir(kind))


def test_fixtures_parse():
    c = _load("mb384")
    m = c.modules
    assert (c.model_type, c.size, c.kmer_len, c.num_out, c.stride, c.sequence_stride) == ("conv_lstm_v3", 384, 9, 2, 6, 1)
    assert [(s.insize, s.size, s.winlen, s.stride) for s in m.signal_convs] == [(1, 4, 5, 1), (4, 16, 5, 1), (16, 128, 16, 6)]
    assert [(s.insize, s.size, s.winlen, s.stride) for s in m.sequence_convs] == [(36, 16, 5, 1), (16, 128, 16, 1)]
    assert (m.merge_conv.insize, m.merge_conv.size, m.merge_conv.winlen) == (256, 384, 5)
    assert m.lstms == [(384, False), (384, True)] and m.linear == (384, 2) and m.upsample is None
    assert c.chunked_sequence_input_TC() == (100, 36) and c.chunked_output_TC() == (100, 2)
    assert (c.encoder_steps(), c.lstm_steps(), c.out_steps()) == (101, 101, 101)
    assert c.refine_do_rough_rescale and c.refine_center_idx == 6 and c.mod_codes == ["a"]
    c = _load("mb192")
    assert (c.lstm_size, c.num_out, c.upsample_scale, c.kmer_len) == (192, 3, 2, 5)
    assert c.mod_codes == ["h", "m"] and c.mod_long_names == ["5hmC", "5mC"]
    assert c.chunked_sequence_input_TC() == (80, 20)
    assert (c.encoder_steps(), c.lstm_steps(), c.out_steps()) == (81, 81, 162)


def _flatten(c):
    """Our config in the order of ref_modbase_config (oracle/modbase_ref_driver.cpp)."""
    m = c.modules
    v = [2, c.size, c.kmer_len, c.num_out, c.stride, c.sequence_stride]   # ModelType::CONV_LSTM_V3 == 2
    for cv in m.signal_convs + m.sequence_convs + [m.merge_conv]:
        v += [cv.insize, cv.size, cv.winlen, cv.stride, cv.activation]
    v.append(len(m.lstms))
    for size, rev in m.lstms:
        v += [size, int(rev)]
    v += list(m.linear) + (list(m.upsample) if m.upsample else [-1, -1])
    v += [c.samples_before, c.samples_after, c.chunk_size, c.bases_before, c.bases_after, c.kmer_len, int(c.reverse_signal),
          int(c.base_start_justify), int(c.refine_do_rough_rescale), c.refine_center_idx, len(c.mod_codes), c.motif_offset,
          ord(c.motif[c.motif_offset])]
    v += list(c.chunked_sequence_input_TC()) + list(c.chunked_signal_input_TC()) + list(c.chunked_output_TC())
    return v


@pytest.fixture(scope="module")
def mbref():
    from oracle.modbase_oracle import ModBaseReference
    if not ModBaseReference.available():
        pytest.skip("oracle/_ref/libmodbase_ref.so not built (needs the reference tree)")
    return ModBaseReference()


def test_reference_6ma_config_field_for_field(mbref):
    from dorado_b200.config import load_modbase_config
    if not (REF_6MA / "config.toml").exists():
        pytest.skip("the reference tree's 6mA@v4 config is not present")
    assert _flatten(load_modbase_config(REF_6MA)) == mbref.config(REF_6MA)


@pytest.mark.parametrize("kind", sorted(MODBASE))
def test_fixture_config_field_for_field(mbref, kind):
    from dorado_b200.config import load_modbase_config
    assert _flatten(load_modbase_config(modbase_dir(kind))) == mbref.config(modbase_dir(kind))


def _edited(tmp_path, name, old, new):
    src = (modbase_dir("mb384") / "config.toml").read_text()
    assert old in src
    d = tmp_path / name
    d.mkdir()
    (d / "config.toml").write_text(src.replace(old, new, 1))
    return d


@pytest.mark.parametrize("model", ["conv_lstm", "conv_lstm_v2", "conv_only", "conv_v1", "lstm_v9"])
def test_other_model_types_rejected(tmp_path, model):
    from dorado_b200.config import load_modbase_config
    d = _edited(tmp_path, model, 'model = "conv_lstm_v3"', f'model = "{model}"')
    with pytest.raises(ValueError, match="not supported|Unknown modbase model type"):
        load_modbase_config(d)


@pytest.mark.parametrize("old,new,match", [
    ("type = \"lstm\"\nsize = 384\nreverse = 0", "type = \"lstm\"\nsize = 384\nreverse = 1", "first lstm layer must be forward"),
    ("kmer_len = 9", "kmer_len = 7", "inconsistent kmer_len"),
    ("num_out = 2", "num_out = 3", "linear and num_out mismatch"),
    ("stride = 6\nsequence_stride", "stride = 3\nsequence_stride", "signal convolution stride mismatch"),
    ("size = 384\nkmer_len", "size = 192\nkmer_len", "lstm size mismatch"),
    ("chunk_size = 600", "chunk_size = 200", "not in range"),
    ("activation = \"tanh\"", "activation = \"relu\"", "Unknown activation"),
])
def test_reference_consistency_checks(tmp_path, old, new, match):
    """ModelGeneralParams / ContextParams / parse_lstms checks (ModBaseModelConfig.cpp:123-147, 220-245, 337-360, 470-480)."""
    from dorado_b200.config import load_modbase_config
    with pytest.raises(ValueError, match=match):
        load_modbase_config(_edited(tmp_path, "bad", old, new))


@pytest.mark.parametrize("kind", sorted(MODBASE))
def test_oracle_matches_reference(mbref, tmp_path, kind):
    from dorado_b200.weights import synthetic_modbase_weights
    from oracle.modbase_oracle import modbase_forward
    cfg = _load(kind)
    w = synthetic_modbase_weights(cfg, 7)
    sig, seq = modbase_inputs(cfg, 3, 11)
    got = modbase_forward(cfg, w, sig.astype(np.float32), seq)
    ref = mbref.forward(modbase_dir(kind), w, tmp_path / "model", sig.astype(np.float32), seq)
    assert ref.shape == got.shape == (3, cfg.out_steps() * cfg.num_out)
    assert np.abs(got - ref).max() <= 2e-5, f"oracle vs reference max |diff| {np.abs(got - ref).max():.3g}"
    if kind == "mb384":
        assert ref.shape[1] == 101 * 2


@pytest.mark.parametrize("kind", sorted(MODBASE))
def test_fp16_oracle_within_bound_of_fp32(kind):
    from dorado_b200.weights import synthetic_modbase_weights
    from oracle.modbase_oracle import modbase_forward
    cfg = _load(kind)
    w = synthetic_modbase_weights(cfg, 7)
    sig, seq = modbase_inputs(cfg, 8, 3)
    p32 = modbase_forward(cfg, w, sig, seq)
    p16 = modbase_forward(cfg, w, sig, seq, emulate_fp16=True)
    err = np.abs(p16 - p32)
    print(f"{kind}: fp16 vs fp32 oracle |dp| p50 {np.percentile(err, 50):.2e} p99 {np.percentile(err, 99):.2e} "
          f"max {err.max():.2e}")
    assert err.max() <= FP16_VS_FP32_MAX
    # the synthetic weights give confident, not flat, class probabilities
    assert np.median(p32.reshape(8, -1, cfg.num_out).max(-1)) > 1.5 / cfg.num_out


def test_modbase_weight_specs():
    from dorado_b200.weights import modbase_tensor_specs
    specs = list(modbase_tensor_specs(_load("mb192")).items())
    assert specs[0] == ("sig_conv1.weight.tensor", (8, 1, 7))
    assert [n for n, _ in specs[-4:]] == ["fc.weight.tensor", "fc.bias.tensor", "linear_up.linear.weight.tensor",
                                         "linear_up.linear.bias.tensor"]
    assert dict(specs)["linear_up.linear.weight.tensor"] == (6, 3)
    assert "linear_up.linear.weight.tensor" not in dict(modbase_tensor_specs(_load("mb384")))
