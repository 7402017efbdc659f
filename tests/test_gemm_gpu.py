"""wgmma GEMM (dorado_b200/csrc/gemm.cu) vs an fp32 matmul of the same fp16 operands.

Tolerance: the kernel accumulates in fp32 and rounds once to fp16, so |err| <= fp16 half-ulp of the result
plus accumulation-order noise: rtol 2e-3 (two fp16 ulps), atol 2e-3.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ACT_NONE, ACT_SWISH, ACT_SWISH_CLAMP, ACT_TANH, ACT_TANH_X5, ACT_SWIGLU = -1, 0, 1, 2, 3, 4


def _ref(a, b, bias, act):
    y = a.astype(np.float32) @ b.astype(np.float32).T
    if bias is not None:
        y = y + bias
    sig = lambda v: 1.0 / (1.0 + np.exp(-v))
    if act == ACT_SWISH:
        y = y * sig(y)
    elif act == ACT_SWISH_CLAMP:
        y = np.minimum(y * sig(y), 3.5)
    elif act == ACT_TANH:
        y = np.tanh(y)
    elif act == ACT_TANH_X5:
        y = 5 * np.tanh(y)
    elif act == ACT_SWIGLU:
        yy, g = y[:, 0::2], y[:, 1::2]
        y = yy * (g * sig(g))
    return y


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (128, 32, 128), (300, 96, 320), (1000, 1024, 384), (77, 256, 512),
                                   (4096, 512, 2048), (130, 1536, 512)])
@pytest.mark.parametrize("act,use_bias", [(ACT_NONE, False), (ACT_SWISH, True), (ACT_TANH, True)])
def test_gemm_matches_fp32(M, N, K, act, use_bias):
    from dorado_b200 import lib as L
    rng = np.random.default_rng(M * 7 + N * 3 + K)
    a = (rng.standard_normal((M, K)) * 0.5).astype(np.float16)
    b = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float16)
    bias = (rng.standard_normal(N) * 0.1).astype(np.float32) if use_bias else None
    c = L.test_gemm(a, b, bias, act)
    np.testing.assert_allclose(c.astype(np.float32), _ref(a, b, bias, act), rtol=2e-3, atol=2e-3)


def test_gemm_k_not_multiple_of_64_and_other_acts():
    from dorado_b200 import lib as L
    rng = np.random.default_rng(5)
    a = (rng.standard_normal((200, 304)) * 0.5).astype(np.float16)  # K = 19 * 16 (last conv of the LSTM models)
    b = (rng.standard_normal((384, 304)) / 17).astype(np.float16)
    bias = (rng.standard_normal(384) * 0.1).astype(np.float32)
    for act in (ACT_SWISH_CLAMP, ACT_TANH_X5):
        c = L.test_gemm(a, b, bias, act)
        np.testing.assert_allclose(c.astype(np.float32), _ref(a, b, bias, act), rtol=2e-3, atol=4e-3)


def test_gemm_swiglu():
    from dorado_b200 import lib as L
    rng = np.random.default_rng(6)
    a = (rng.standard_normal((256, 512)) * 0.5).astype(np.float16)
    b = (rng.standard_normal((4096, 512)) / 22).astype(np.float16)
    c = L.test_gemm(a, b, None, ACT_SWIGLU)
    assert c.shape == (256, 2048)
    np.testing.assert_allclose(c.astype(np.float32), _ref(a, b, None, ACT_SWIGLU), rtol=2e-3, atol=2e-3)
