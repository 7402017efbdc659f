import pathlib
import sys

import numpy as np
import pytest

ROOT = pathlib.Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

CONFIG_DIR = ROOT / "tests" / "data" / "model_configs"
MODELS = {
    "fast": "dna_r10.4.1_e8.2_400bps_fast@v5.0.0",
    "hac": "dna_r10.4.1_e8.2_400bps_hac@v5.0.0",
    "sup": "dna_r10.4.1_e8.2_400bps_sup@v5.0.0",
    "flstm": "synthetic_fast_flstm@v0",   # fast topology with factorised LSTM layers (nn/FLSTMStack.cpp)
}


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a) GPU")


def model_dir(kind: str) -> pathlib.Path:
    return CONFIG_DIR / MODELS[kind]


def synthetic_scores(N, T, state_len, seed, scale=2.0, dtype=np.float16):
    """Random CRF transition scores with some temporal structure so the beam has real choices."""
    rng = np.random.default_rng(seed)
    C = 4 ** (state_len + 1)
    base = rng.standard_normal((N, T, C)).astype(np.float32) * scale
    # favour a random "true" path so stays and steps alternate
    return np.clip(base, -6, 6).astype(dtype)


def planted_scores(N, T, state_len, seed, margin=4.0, noise=1.0, dtype=np.float16):
    """CRF transition scores with a planted best path: per block the path either stays (probability 0.45, every step
    transition then sits below the fixed stay score 2.0) or steps to a random base (that transition gets +margin).
    Decoding is well conditioned here -- unlike i.i.d. scores, where fp16 rounding alone moves 2 % of the bases -- so
    implementations that differ only in the last ulp of their scans must agree on every base."""
    rng = np.random.default_rng(seed)
    S = 4 ** state_len
    C = 4 * S
    out = (rng.standard_normal((N, T, C)).astype(np.float32) * noise - 1.5)
    for n in range(N):
        state = int(rng.integers(S))
        stay = rng.random(T) < 0.45
        bases = rng.integers(4, size=T)
        for t in range(T):
            if t > 0 and stay[t]:
                continue
            new_state = ((state << 2) & (S - 1)) | int(bases[t])
            dropped = (state << 2) >> (2 * state_len)
            out[n, t, new_state * 4 + dropped] = margin + 0.25 * rng.standard_normal()
            state = new_state
    return np.clip(out, -6, 6).astype(dtype)


def unpack_rows(flat, n_bases):
    """Inverse of tools/make_golden_full.pack_rows: list of per-chunk byte strings."""
    o = np.concatenate([[0], np.cumsum(n_bases)])
    return [bytes(flat[o[i]:o[i + 1]]) for i in range(len(n_bases))]


def edit_distance(a: bytes, b: bytes) -> int:
    """Levenshtein distance, one numpy row per character of a."""
    x = np.frombuffer(a, np.uint8)
    y = np.frombuffer(b, np.uint8)
    if len(x) == 0 or len(y) == 0:
        return max(len(x), len(y))
    idx = np.arange(len(y) + 1)
    prev = idx.copy()
    for i, c in enumerate(x):
        m = np.minimum(prev[:-1] + (y != c), prev[1:] + 1)
        m2 = np.concatenate([[i + 1], m])
        prev = np.minimum.accumulate(m2 - idx) + idx   # insertions: cur[j] = min_k<=j (m2[k] + j - k)
    return int(prev[-1])


@pytest.fixture(scope="session")
def crf_oracle():
    from oracle.oracle import CrfOracle, build
    build(ref=False)
    return CrfOracle()


@pytest.fixture(scope="session")
def reference():
    from oracle.oracle import Reference, reference_available
    if not reference_available():
        pytest.skip("oracle/_ref/libdorado_ref.so not built (needs /root/reference)")
    return Reference()
